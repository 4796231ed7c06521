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


K_EPS = np.float32(0.001)
K_INF = np.float32(1.0e30)
K_PI = float(np.float32(4.0) * np.arctan(np.float32(1.0)))  # 4.0f * std::atan(1.0f)
NONE = 0xFFFFFFFF
LIGHT = 0  # NRT_BDPT_LIGHT


def light_total_area(verts, faces, mats16, ids):
    """LightSampler's totalArea_ (main.cc:698-715) in float32: 0.5f * |cross(v2 - v0, v1 - v0)| of every face with
    max(Le) > kEps, summed in face order.  Also returns the (area, face) pairs in that order."""
    v = np.asarray(verts, np.float32)[np.asarray(faces, np.int64)]
    le = np.asarray(mats16, np.float32)[np.asarray(ids, np.int64), 9:12]
    lit = np.nonzero(np.maximum(le[:, 0], np.maximum(le[:, 1], le[:, 2])) > K_EPS)[0]
    a, b = v[lit, 2] - v[lit, 0], v[lit, 1] - v[lit, 0]
    c = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                  a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)
    area = F(0.5) * np.sqrt(c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1] + c[:, 2] * c[:, 2])
    total = F(0.0)
    for x in area:
        total = F(total + x)
    return total, area.astype(np.float32), lit


# ---- connectPath (main.cc:1081-1289) in float64 over nrt_bdpt_vertex records.  Vectors are tuples of Python floats
# (IEEE double); a vertex is a dict of its fields and its material's 16 floats (None: the lens and light-origin
# vertices, which have no material).
def _sub(a, b):
    return (a[0] - b[0], a[1] - b[1], a[2] - b[2])


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _length(a):
    return _dot(a, a) ** 0.5


def _unit(a):
    n = _length(a)
    return (a[0] / n, a[1] / n, a[2] / n) if n > 1e-6 else a


def _vertex(rec, mats):
    m = int(rec["material"])
    vec = lambda k: tuple(float(x) for x in rec[k])
    return dict(p=vec("position"), on=vec("original_norm"), n=vec("norm"), beta=vec("beta"), wo=vec("wo"),
                fwd=float(rec["pdf_fwd"]), rev=float(rec["pdf_rev"]), type=int(rec["type"]),
                mat=None if m == NONE else [float(x) for x in mats[m]])


def _delta(v):
    """Vertex::isDelta: any specular or transmittance; no material: not delta"""
    m = v["mat"]
    return m is not None and any(x != 0.0 for x in m[3:9])


def _lobes(m, wo, on, n):
    """the Fresnel factor and the normalised (rhoS, rhoD, rhoR) of Vertex::f / pdfBRDF, or None when totalrho < 1e-4"""
    inside = -1.0 if _dot((-wo[0], -wo[1], -wo[2]), on) < 0 else 1.0
    n1 = 1.0 / m[12] if inside < 0 else m[12]
    n2 = 1.0 / n1
    r0 = ((n1 - n2) / (n1 + n2)) ** 2
    fresnel = r0 + (1.0 - r0) * (1.0 - _dot(wo, n)) ** 5
    third = lambda c: (c[0] + c[1] + c[2]) / 3.0
    rs = third(m[3:6]) * fresnel
    rd = third(m[0:3]) * (1.0 - fresnel) * (1.0 - m[13])
    rr = third(m[6:9]) * (1.0 - fresnel) * m[13]
    total = rs + rd + rr
    if total < 0.0001:
        return None
    return rs / total, rd / total, rr / total


def vertex_f(v, q):
    """Vertex::f (main.cc:634-689) of v towards position q: only the diffuse lobe has a value"""
    if v["mat"] is None:
        return (0.0, 0.0, 0.0)
    m, n = v["mat"], v["n"]
    refl = _dot(_sub(q, v["p"]), n) * _dot(v["wo"], n) > 0.0
    rho = _lobes(m, v["wo"], v["on"], n)
    if rho is None:
        return (0.0, 0.0, 0.0)
    rs, rd, rr = rho
    weight = (rs if rs > 0.0 and refl else 0.0) + (rd if rd > 0.0 and refl else 0.0) + \
             (rr if rr > 0.0 and not refl else 0.0)
    if not (rd > 0.0 and refl):
        return (0.0, 0.0, 0.0)
    return tuple(rd * m[k] / K_PI / weight for k in range(3))


def pdf_brdf(m, wi, wo, on, n):
    """pdfBRDF (main.cc:839-886); no material: 0"""
    if m is None:
        return 0.0
    refl = _dot(wi, n) * _dot(wo, n) > 0.0
    rho = _lobes(m, wo, on, n)
    if rho is None or not (rho[1] > 0.0 and refl):
        return 0.0
    return rho[1] * abs(_dot(wi, n)) / K_PI


def _pdf_area(v_from, v_to, wi_pos):
    """pdfBRDF at v_from from wi_pos towards v_to, per unit area at v_to: pdfOmega * |n . wo| / dist^2"""
    wo = _sub(v_to["p"], v_from["p"])
    dist = _length(wo)
    wi, wo = _unit(_sub(wi_pos, v_from["p"])), _unit(wo)
    return pdf_brdf(v_from["mat"], wi, wo, v_from["on"], v_from["n"]) * abs(_dot(v_from["n"], wo)) / (dist * dist)


def _pdf_light(v_from, v_to):
    """weightMIS's cosine pdf from an emitting vertex: max(0, n . to) * (n . to) / dist^2"""
    to = _sub(v_to["p"], v_from["p"])
    dist = _length(to)
    to = (to[0] / dist, to[1] / dist, to[2] / dist)
    c = _dot(v_from["n"], to)
    return max(0.0, c) * c / (dist * dist)


def weight_mis(E, Lv, ne, nl, inv_area):
    """weightMIS (main.cc:1081-1211) of eye vertices E[:ne] and light vertices Lv[:nl]"""
    if ne <= 2 and nl == 0:
        return 1.0
    length = ne + nl
    path = [[E[i]["fwd"], E[i]["rev"]] for i in range(ne)] + \
           [[Lv[i]["fwd"], Lv[i]["rev"]] for i in range(nl - 1, -1, -1)]
    ve, vl = E[ne - 1], (Lv[nl - 1] if nl >= 1 else None)
    vem, vlm = (E[ne - 2] if ne >= 2 else None), (Lv[nl - 2] if nl >= 2 else None)
    if nl == 0:
        path[ne - 1][1] = inv_area
    elif nl == 1:
        path[ne - 1][1] = _pdf_light(vl, ve)
    else:
        path[ne - 1][1] = _pdf_area(vl, ve, vlm["p"])
    if vl is not None:
        path[ne][1] = _pdf_area(ve, vl, vem["p"])
    if vem is not None:
        path[ne - 2][1] = _pdf_light(ve, vem) if nl == 0 else _pdf_area(ve, vem, vl["p"])
    if vlm is not None:
        path[ne + 1][1] = _pdf_area(vl, vlm, ve["p"])
    mis, prob = 0.0, 1.0
    for i in range(ne - 1, 1, -1):
        fwd, rev = (x if x != 0.0 else 1.0 for x in path[i])  # 0 counts as 1
        prob *= rev / fwd
        if _delta(E[i]) or _delta(E[i - 1]):
            continue
        mis += prob * prob
    prob = 1.0
    for i in range(ne, length):
        fwd, rev = (x if x != 0.0 else 1.0 for x in path[i])
        prob *= rev / fwd
        if _delta(Lv[length - i - 1]) or (i + 1 < length and _delta(Lv[length - i - 2])):
            continue
        mis += prob * prob
    return 1.0 / (1.0 + mis)


def conn_rays(pe, pl):
    """calcG's rays as the device's conn_ray builds them, in float32: (org, unit dir, dist) of pe -> pl"""
    pe, pl = np.asarray(pe, np.float32).reshape(-1, 3), np.asarray(pl, np.float32).reshape(-1, 3)
    to = pl - pe
    dist = np.sqrt(to[:, 0] * to[:, 0] + to[:, 1] * to[:, 1] + to[:, 2] * to[:, 2])
    return pe, to / dist[:, None], dist


def connection_terms(eye, light, mats, total_area, max_bounces, trace):
    """connectPath's terms (main.cc:1246-1289) of one sample over exported records eye[:ne], light[:nl] and the 16-float
    material table, with max_bounces in place of uMaxBounces: [(e, l, float64 rgb)], the emission term as (ne, 0).
    The skips: delta vertices, e + l - 2 > max_bounces and L == 0.  calcG's ray is built in float32 as the device
    builds it; `trace(org, dir) -> (hit, t)` gives its nearest hit and |dist - t| > kEps is decided in float32.  Its
    cosines and 1 / dist^2 are float64."""
    mats = np.asarray(mats, np.float32).reshape(-1, 16)
    E = [_vertex(r, mats) for r in eye]
    Lv = [_vertex(r, mats) for r in light]
    ne, nl = len(E), len(Lv)
    inv_area = 1.0 / float(total_area)
    terms = []
    if E[-1]["type"] == LIGHT:
        w = weight_mis(E, Lv, ne, 0, inv_area)
        terms.append((ne, 0, np.array([w * b for b in E[-1]["beta"]])))
    pending = []  # (e, l, L * mis) waiting for calcG
    for e in range(2, ne + 1):
        ev = E[e - 1]
        if _delta(ev) or ev["type"] == LIGHT:
            continue
        for l in range(1, nl + 1):
            if e + l - 2 > max_bounces:
                continue
            lv = Lv[l - 1]
            if l != 1 and _delta(lv):
                continue
            fe = vertex_f(ev, lv["p"])
            if l == 1:
                c = abs(_dot(lv["n"], _unit(_sub(ev["p"], lv["p"]))))
                L = [ev["beta"][k] * fe[k] * lv["beta"][k] * c for k in range(3)]
            else:
                fl = vertex_f(lv, ev["p"])
                L = [ev["beta"][k] * fe[k] * fl[k] * lv["beta"][k] for k in range(3)]
            if L[0] == 0.0 and L[1] == 0.0 and L[2] == 0.0:
                continue
            pending.append((e, l, np.array(L) * weight_mis(E, Lv, e, l, inv_area)))
    if pending:
        org, d, dist = conn_rays([eye[e - 1]["position"] for e, _, _ in pending],
                                 [light[l - 1]["position"] for _, l, _ in pending])
        hit, t = trace(org, d)
        t = np.asarray(t, np.float32)
        seen = hit & ~(np.abs(dist - t) > K_EPS)
        for k, (e, l, Lm) in enumerate(pending):
            G = 0.0
            if seen[k]:
                ev, lv = E[e - 1], Lv[l - 1]
                to = _unit(_sub(lv["p"], ev["p"]))
                dd = _length(_sub(lv["p"], ev["p"]))
                G = max(0.0, _dot(to, ev["n"])) * max(0.0, -_dot(to, lv["n"])) / (dd * dd)
            terms.append((e, l, Lm * G))
    return terms


def connect_path(eye, light, mats, total_area, max_bounces, trace):
    """connectPath's colour and its sum of |term| per channel (float64)"""
    terms = connection_terms(eye, light, mats, total_area, max_bounces, trace)
    rgb, mag = np.zeros(3), np.zeros(3)
    for _, _, t in terms:
        rgb += t
        mag += np.abs(t)
    return rgb, mag


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
