"""The scene pass's rules of nrt_scene_render_bdpt_device (include/nanort_b200_scene_bdpt.h) restated in numpy over a
flattened scene: the lift of a spawned ray (SceneSpawn::lifted), the connection's visibility (SceneSpawn::plane_max_t
with the walk's nearest hit from orc.PortScene) and connectPath's terms with bdpt_model's weight_mis / vertex_f.

float32 where the device decides (ray origins, max_t, the comparison with the hit distance), in the device's operation
order (the library is compiled with --fmad=false); the terms themselves in float64, as bdpt_model's."""
import numpy as np

import bdpt_model as M

F = np.float32
K_EPS = F(0.001)
K_INF = F(1.0e30)


def dot3(a, b):
    """a.x * b.x + a.y * b.y + a.z * b.z per row, float32, left to right"""
    a, b = np.asarray(a, F), np.asarray(b, F)
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def unit_cross(tri):
    """world_normal(): unit cross(e1, e2) of float32 triangles [n, 3, 3]"""
    tri = np.asarray(tri, F)
    e1, e2 = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], axis=1).astype(F)
    ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    il = np.where(ln > 0, F(1.0) / np.where(ln > 0, ln, F(1.0)), F(0.0)).astype(F)
    return n * il[:, None]


def lifted(g, p, d):
    """SceneSpawn::lifted(kEps, p, d): p + kEps g, g turned to the side d leaves"""
    g, p = np.asarray(g, F), np.asarray(p, F)
    g = np.where((dot3(g, d) < 0)[:, None], -g, g)
    return p + g * K_EPS


def plane_max_t(p, o, d, dist, ln):
    """SceneSpawn::plane_max_t: where the ray from o (p lifted) along d meets the plane of unit normal ln through the
    point at dist from p, less 1e-5"""
    ndl = dot3(ln, d)
    ndo = dot3(ln, np.asarray(o, F) - np.asarray(p, F))
    safe = np.where(ndl != 0, ndl, F(1.0))
    return np.where(ndl != 0, np.asarray(dist, F) - ndo / safe, np.asarray(dist, F)) - F(0.00001)


def walk(port, org, d, max_t=K_INF):
    """the reference's Scene::Traverse of float32 rays {org, d, kEps, max_t}: (hits, mask)"""
    from oracle import orc

    rays = np.zeros(len(org), orc.RAY_DTYPE)
    rays["org"], rays["dir"] = org, d
    rays["min_t"], rays["max_t"] = K_EPS, max_t
    return port.traverse(rays)


def connection_terms(ex, i, flat, mats, total_area, max_bounces, port):
    """connectPath's terms of exported slot i under the scene rules: [(e, l, float64 rgb)].  `flat` maps (instance,
    face) to the flattened face and holds the world triangles (flat.tri, flat.offsets)."""
    ne, nl = int(ex["ne"][i]), int(ex["nl"][i])
    eye, light = ex["eye"][i, :ne], ex["light"][i, :nl]
    mats = np.asarray(mats, np.float32).reshape(-1, 16)
    E = [M._vertex(r, mats) for r in eye]
    Lv = [M._vertex(r, mats) for r in light]
    inv_area = 1.0 / float(total_area)
    terms = []
    if E[-1]["type"] == M.LIGHT:
        terms.append((ne, 0, np.array([M.weight_mis(E, Lv, ne, 0, inv_area) * b for b in E[-1]["beta"]])))
    pending = []
    for e in range(2, ne + 1):
        ev = E[e - 1]
        if M._delta(ev) or ev["type"] == M.LIGHT:
            continue
        for l in range(1, nl + 1):
            if e + l - 2 > max_bounces:
                continue
            lv = Lv[l - 1]
            if l != 1 and M._delta(lv):
                continue
            fe = M.vertex_f(ev, lv["p"])
            if l == 1:
                c = abs(M._dot(lv["n"], M._unit(M._sub(ev["p"], lv["p"]))))
                L = [ev["beta"][k] * fe[k] * lv["beta"][k] * c for k in range(3)]
            else:
                fl = M.vertex_f(lv, ev["p"])
                L = [ev["beta"][k] * fe[k] * fl[k] * lv["beta"][k] for k in range(3)]
            if L[0] == 0.0 and L[1] == 0.0 and L[2] == 0.0:
                continue
            pending.append((e, l, np.array(L) * M.weight_mis(E, Lv, e, l, inv_area)))
    if not pending:
        return terms
    es = np.array([e for e, _, _ in pending]) - 1
    ls = np.array([l for _, l, _ in pending]) - 1
    pe, d, dist = M.conn_rays(eye["position"][es], light["position"][ls])
    fe = flat.offsets[ex["eye_inst"][i, es].astype(np.int64)] + eye["prim_id"][es].astype(np.int64)
    pair = ex["pair"][i].astype(np.int64)
    origin = ls == 0  # the light-origin vertex: the sampled pair's plane
    li = np.where(origin, 0, ex["light_inst"][i, ls]).astype(np.int64)
    lp = np.where(origin, 0, light["prim_id"][ls]).astype(np.int64)
    fl = np.where(origin, flat.offsets[pair[0]] + pair[1], flat.offsets[li] + lp)
    o = lifted(unit_cross(flat.tri[fe]), pe, d)
    max_t = plane_max_t(pe, o, d, dist, unit_cross(flat.tri[fl]))
    hits, mask = walk(port, o, d, max_t)
    blocked = (mask != 0) & (hits["t"] < max_t)
    for k, (e, l, Lm) in enumerate(pending):
        G = 0.0
        if not blocked[k]:
            ev, lv = E[e - 1], Lv[l - 1]
            to = M._unit(M._sub(lv["p"], ev["p"]))
            dd = M._length(M._sub(lv["p"], ev["p"]))
            G = max(0.0, M._dot(to, ev["n"])) * max(0.0, -M._dot(to, lv["n"])) / (dd * dd)
        terms.append((e, l, Lm * G))
    return terms


def hit_normal(fn9, u, v):
    """subpath_hit's interpolation of face-varying normals fn9 [n, 9] at (u, v): (1.0 - u - v) in double, the
    reference's normalize (threshold and 1.0 / len in double)"""
    fn = np.asarray(fn9, F).reshape(-1, 3, 3)
    u, v = np.asarray(u, F), np.asarray(v, F)
    w = (1.0 - u.astype(np.float64) - v.astype(np.float64)).astype(F)
    n = (fn[:, 0] * w[:, None] + fn[:, 1] * u[:, None]) + fn[:, 2] * v[:, None]
    ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    inv = np.where(np.abs(ln.astype(np.float64)) > 1e-6, (1.0 / np.maximum(ln.astype(np.float64), 1e-30)).astype(F),
                   F(1.0))
    return n * inv[:, None]
