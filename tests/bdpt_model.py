"""numpy restatement of the bidirectional path tracer's sample set-up (examples/bidir_path_tracer/main.cc): the
xorshift128 generator Random (main.cc:132-157), the sample seed of main()'s loop (main.cc:1382) and the camera ray of
eyeSubpath (main.cc:1022-1027) under nrt_bdpt_params' camera block."""
import numpy as np

F = np.float32
REFERENCE_CAMERA = np.array([0, 5, 20, 1, 0, 0, 0, 1, 0, 0, 0, -1], np.float32)


def seed(x, y, width, spp_total, i):
    """(uint32)((y * W + x) * spp_total + i), as the reference's int arithmetic wraps"""
    return ((int(y) * int(width) + int(x)) * int(spp_total) + int(i)) & 0xFFFFFFFF


def _init(s):
    st = []
    for i in range(1, 5):
        s = (1812433253 * (s ^ (s >> 30)) + i) & 0xFFFFFFFF
        st.append(s)
    return st


def random_ints(s, n):
    st = _init(int(s) & 0xFFFFFFFF)
    out = np.zeros(n, np.uint64)
    for k in range(n):
        t = (st[0] ^ (st[0] << 11)) & 0xFFFFFFFF
        st[0], st[1], st[2] = st[1], st[2], st[3]
        st[3] = ((st[3] ^ (st[3] >> 19)) ^ (t ^ (t >> 8))) & 0xFFFFFFFF
        out[k] = st[3]
    return out


def random_reals(s, n):
    """Random(s).nextReal() x n: (float)nextInt() / (float)UINT_MAX, in float32 (can be 1.0)"""
    return (random_ints(s, n).astype(np.float32) / F(4294967296.0)).astype(np.float32)


def _normalize(v):
    """float3::normalize: the threshold and 1.0 / len in double, the scaling in float"""
    ln = np.sqrt(F(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]), dtype=np.float32)
    if abs(float(ln)) > 1.0e-6:
        inv = F(1.0 / float(ln))
        v = np.array([v[0] * inv, v[1] * inv, v[2] * inv], np.float32)
    return v


def camera_ray(cam, x, y, width, height, s):
    """(org, unit dir) of loop pixel (x, y) for sample seed s: px = x + (u0 - 0.5), py = y + (u1 - 0.5),
    dir = normalize(sx * right + sy * up + forward) with sx = px / W - 0.5, sy = py / H - 0.5"""
    cam = np.asarray(cam, np.float32)
    u = random_reals(s, 2)
    px = F(F(x) + F(u[0] - F(0.5)))
    py = F(F(y) + F(u[1] - F(0.5)))
    sx = F(F(px / F(width)) - F(0.5))
    sy = F(F(py / F(height)) - F(0.5))
    d = np.array([F(F(sx * cam[3 + k]) + F(sy * cam[6 + k])) + cam[9 + k] for k in range(3)], np.float32)
    return cam[0:3].copy(), _normalize(d)


def flat_normals(verts, faces):
    """face-varying normals [n, 9]: the example loader's calcNormal, normalize(cross(v2 - v0, v1 - v0)) (main.cc:299-305)
    at all three corners, in float32"""
    v = np.asarray(verts, np.float32)[np.asarray(faces, np.int64)]
    a, b = v[:, 2] - v[:, 0], v[:, 1] - v[:, 0]
    n = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                  a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1).astype(np.float32)
    out = np.zeros_like(n)
    for i in range(len(n)):
        out[i] = _normalize(n[i])
    return np.repeat(out, 3, axis=0).reshape(-1, 9)
