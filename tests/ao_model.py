"""Host model of the primary + 1-bounce AO pass (csrc/wavefront.cuh: camera_ray, CameraRays::load, make_ao_ray;
csrc/scene.cu: scene_gen_ao_kernel), restated from those kernels -- which in turn restate the reference path tracer's
examples/path_tracer/main.cc:809-817 (camera), 860 (hit point), 306-312 + 878-881 (normal flipped to the viewer) and
216-250 (orthonormal basis + cosine direction).

The library is built with --fmad=false and without fast-math, so every operation of those functions except sincosf is an
IEEE-rounded float32 operation, and numpy float32 reproduces it when it runs the same operations in the same order.
Two levels:
  * the f32 model: the device's operation order; sincosf(ph) is replaced by the float64 sin / cos of the same float32 ph,
    rounded to float32 (`sincos`).  Everything else is bit-exact to the device.
  * the f64 ideal: the same construction in float64 from the float32 inputs (hit point, normal, basis, direction).
"""
import numpy as np

F32 = np.float32
TWO_PI_F = F32(6.28318530718)  # the literal 6.28318530718f of make_ao_ray


def slots(W, H, tile_w, tile_h, spp, sample0=0, shard=0, n_shards=1):
    """(pixel, sample) of every ray slot of a shard in queue order (-1 outside the image); sample includes sample0."""
    from nanort_b200 import dist as nd

    pix, smp = nd.slot_pixels(W, H, tile_w, tile_h, shard, n_shards, spp)
    return pix, smp + sample0


def camera_dirs(cam, W, H, seed, pix, smp):
    """camera_ray(): float32 [n,3] unit directions of (pixel, sample)."""
    from nanort_b200 import scenes as S

    cam = np.asarray(cam, F32)
    jx = S.rand_ps(pix, smp, 0, seed)
    jy = S.rand_ps(pix, smp, 1, seed)
    px = (pix % W).astype(F32)
    py = (pix // W).astype(F32)
    sx = (px + jx) / F32(W) - F32(0.5)
    sy = F32(0.5) - (py + jy) / F32(H)
    d = [cam[3 + k] * sx + cam[6 + k] * sy + cam[9 + k] for k in range(3)]
    inv = F32(1.0) / np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2])
    return np.stack([d[0] * inv, d[1] * inv, d[2] * inv], axis=1)


def sincos(ph):
    """sincosf replaced by float64 sin / cos of the float32 argument, rounded once."""
    ph64 = ph.astype(np.float64)
    return np.sin(ph64).astype(F32), np.cos(ph64).astype(F32)


def unit_normals(a, b, c):
    """make_ao_ray's normal: normalize(cross(b - a, c - a)) in float32, device order; a, b, c: [n,3] float32."""
    e1x, e1y, e1z = b[:, 0] - a[:, 0], b[:, 1] - a[:, 1], b[:, 2] - a[:, 2]
    e2x, e2y, e2z = c[:, 0] - a[:, 0], c[:, 1] - a[:, 1], c[:, 2] - a[:, 2]
    nx = e1y * e2z - e1z * e2y
    ny = e1z * e2x - e1x * e2z
    nz = e1x * e2y - e1y * e2x
    ln = np.sqrt(nx * nx + ny * ny + nz * nz)
    with np.errstate(divide="ignore"):
        ln = np.where(ln > 0, F32(1.0) / ln, F32(0.0)).astype(F32)
    return nx * ln, ny * ln, nz * ln


def cosine_dirs(nx, ny, nz, d, u1, u2, sn=None, cs=None):
    """The rest of make_ao_ray from the unit normal (float32): viewer flip against d [n,3], branch-free basis, cosine
    direction, normalisation.  Returns (dir [n,3], flipped normal (nx, ny, nz), sg).  sn / cs override sincos()."""
    flip = (nx * d[:, 0] + ny * d[:, 1] + nz * d[:, 2]) > 0
    nx, ny, nz = np.where(flip, -nx, nx), np.where(flip, -ny, ny), np.where(flip, -nz, nz)
    sg = np.where(nz >= 0, F32(1.0), F32(-1.0))
    a = F32(-1.0) / (sg + nz)
    b = nx * ny * a
    t1x, t1y, t1z = F32(1.0) + sg * nx * nx * a, sg * b, -sg * nx
    t2x, t2y, t2z = b, sg + ny * ny * a, -ny
    r = np.sqrt(u1)
    ph = TWO_PI_F * u2
    if sn is None:
        sn, cs = sincos(ph)
    lx, ly, lz = r * cs, r * sn, np.sqrt(np.maximum(F32(0.0), F32(1.0) - u1))
    wx = t1x * lx + t2x * ly + nx * lz
    wy = t1y * lx + t2y * ly + ny * lz
    wz = t1z * lx + t2z * ly + nz * lz
    il = F32(1.0) / np.sqrt(wx * wx + wy * wy + wz * wz)
    return np.stack([wx * il, wy * il, wz * il], axis=1), (nx, ny, nz), sg


def ao_samples(pix, smp, seed):
    from nanort_b200 import scenes as S

    return S.rand_ps(pix, smp, 2, seed), S.rand_ps(pix, smp, 3, seed)


def ao_rays_f32(verts, faces, org, d, t, prim, pix, smp, seed):
    """make_ao_ray for hits (org [3] or [n,3], d [n,3], t [n], prim [n]): (P [n,3], dir [n,3], n_viewer, sg)."""
    org = np.broadcast_to(np.asarray(org, F32), d.shape)
    P = org + d * t[:, None]  # o.x + d.x * t, per component
    f = faces[prim]
    nx, ny, nz = unit_normals(verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]])
    u1, u2 = ao_samples(pix, smp, seed)
    w, n, sg = cosine_dirs(nx, ny, nz, d, u1, u2)
    return P, w, n, sg


def dirs_within_sincos_ulps(verts, faces, d, prim, pix, smp, seed, got, k=3):
    """True where `got` equals, bit for bit, the f32 model evaluated with sin / cos moved by at most k ulp from the
    correctly rounded values: the device differs from the model only through sincosf (<= 2 ulp)."""
    f = faces[prim]
    nx, ny, nz = unit_normals(verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]])
    u1, u2 = ao_samples(pix, smp, seed)
    sn0, cs0 = sincos(TWO_PI_F * u2)
    ok = np.zeros(len(prim), bool)
    gb = np.ascontiguousarray(got, F32).view(np.uint32)
    for i in range(-k, k + 1):
        sn = _nudge(sn0, i)
        for j in range(-k, k + 1):
            w, _, _ = cosine_dirs(nx, ny, nz, d, u1, u2, sn=sn, cs=_nudge(cs0, j))
            ok |= np.all(w.view(np.uint32) == gb, axis=1)
    return ok


def _nudge(x, k):
    """x moved by k float32 ulps (towards +inf for k > 0)."""
    out = x.copy()
    for _ in range(abs(k)):
        out = np.nextafter(out, F32(np.inf) if k > 0 else F32(-np.inf)).astype(F32)
    return out


def ideal_f64(verts, faces, org, d, t, prim, pix, smp, seed, n32, sg):
    """The f64 ideal of make_ao_ray from the same float32 inputs.  The normal is oriented like the f32 model's flipped
    normal n32 and the basis takes the f32 sign sg (a normal with |nz| ~ 0 may pick the other, equally valid, basis).
    Returns (P64, dir64, n64, cond) with cond = |e1| |e2| / |e1 x e2| (1 / sine of the corner angle)."""
    org = np.broadcast_to(np.asarray(org, np.float64), d.shape)
    P = org + d.astype(np.float64) * t.astype(np.float64)[:, None]
    f = faces[prim]
    p0, p1, p2 = (verts[f[:, k]].astype(np.float64) for k in range(3))
    e1, e2 = p1 - p0, p2 - p0
    n = np.cross(e1, e2)
    ln = np.linalg.norm(n, axis=1)
    cond = np.linalg.norm(e1, axis=1) * np.linalg.norm(e2, axis=1) / np.maximum(ln, 1e-300)
    n = n / np.maximum(ln, 1e-300)[:, None]
    n32 = np.stack(n32, axis=1).astype(np.float64)
    n = np.where(((n * n32).sum(axis=1) < 0)[:, None], -n, n)
    s = sg.astype(np.float64)
    a = -1.0 / (s + n[:, 2])
    b = n[:, 0] * n[:, 1] * a
    t1 = np.stack([1.0 + s * n[:, 0] * n[:, 0] * a, s * b, -s * n[:, 0]], axis=1)
    t2 = np.stack([b, s + n[:, 1] * n[:, 1] * a, -n[:, 1]], axis=1)
    u1, u2 = (u.astype(np.float64) for u in ao_samples(pix, smp, seed))
    r, ph = np.sqrt(u1), 2.0 * np.pi * u2
    w = t1 * (r * np.cos(ph))[:, None] + t2 * (r * np.sin(ph))[:, None] + n * np.sqrt(1.0 - u1)[:, None]
    return P, w / np.linalg.norm(w, axis=1)[:, None], n, cond


def mat_apply(X, p):
    """scene.cu:multv -- row-vector transform with the reference's sum order, float32: X [4,4], p [n,3]."""
    X = np.asarray(X, F32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([((X[0, k] * x + X[1, k] * y) + X[2, k] * z) + X[3, k] for k in range(3)], axis=1)


def scene_ao_rays_f32(insts, xforms, hits, d, pix, smp, seed, ao_min_t, ao_max_t):
    """scene_gen_ao_kernel for scene hits (SCENE_HIT_DTYPE) of camera directions d: AO rays (RAY_DTYPE).
    insts = [(verts, faces, _)], xforms = the instances' local -> world matrices (Scene.InstanceStates()["xform"])."""
    from nanort_b200 import scenes as S

    n = len(hits)
    A, B, C = (np.zeros((n, 3), F32) for _ in range(3))
    for i in np.unique(hits["node_id"]):
        sel = hits["node_id"] == i
        v, f, _ = insts[i]
        tri = f[hits["prim_id"][sel]]
        A[sel], B[sel], C[sel] = (mat_apply(xforms[i], v[tri[:, k]]) for k in range(3))
    nx, ny, nz = unit_normals(A, B, C)
    u1, u2 = ao_samples(pix, smp, seed)
    w, (nx, ny, nz), _ = cosine_dirs(nx, ny, nz, d, u1, u2)
    m = F32(ao_min_t)
    out = np.zeros(n, S.RAY_DTYPE)
    out["org"] = np.stack([hits["P"][:, 0] + nx * m, hits["P"][:, 1] + ny * m, hits["P"][:, 2] + nz * m], axis=1)
    out["dir"] = w
    out["min_t"] = 0.0
    out["max_t"] = ao_max_t
    return out
