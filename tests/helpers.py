"""Shared parity checker: GPU results vs the oracle, with exact-t tie classification (SURVEY.md F3)."""
import numpy as np


def compare_hits(port, verts, faces, rays, got_hits, got_mask, want_hits, want_mask, topts=None, cpp11=True,
                 exact=True, rel_tol=1e-5):
    """Returns a dict of mismatch counts.  `exact`: t/u/v must match bit-for-bit; otherwise within rel_tol
    (the north star's 1e-5 relative).  A prim_id difference is a tie when the oracle, re-testing the GPU's
    primitive alone with the reference arithmetic, reports exactly the same t."""
    got_mask = got_mask.astype(bool)
    want_mask = want_mask.astype(bool)
    out = {"n": len(rays), "hits": int(want_mask.sum()), "mask_diff": int((got_mask != want_mask).sum()),
           "prim_diff": 0, "ties": 0, "near_ties": 0, "tuv_diff": 0}
    both = got_mask & want_mask
    g, w = got_hits[both], want_hits[both]
    pd = g["prim_id"] != w["prim_id"]
    idx_both = np.nonzero(both)[0]
    for j in np.nonzero(pd)[0]:
        ok, h = port.test_prim(verts, faces, rays[idx_both[j]], int(g["prim_id"][j]), topts=topts, cpp11=cpp11)
        # the GPU's record must be exactly what the reference arithmetic gives for that primitive
        valid = ok and all(h[k] == g[k][j] for k in ("t", "u", "v"))
        if valid and g["t"][j] == w["t"][j]:
            out["ties"] += 1
        elif valid and abs(float(g["t"][j]) - float(w["t"][j])) <= rel_tol * abs(float(w["t"][j])):
            # two different primitives (coplanar, overlapping) whose hits differ by an ulp or so: which one the
            # REFERENCE reports depends on its own visiting order, because its box test culls with the current
            # best t at that precision (SURVEY.md F3); t is within the north star's 1e-5
            out["near_ties"] += 1
        else:
            out["prim_diff"] += 1
    same = ~pd
    if exact:
        bad = np.zeros(same.sum(), bool)
        for k in ("t", "u", "v"):
            bad |= g[k][same].view(np.uint32) != w[k][same].view(np.uint32)
    else:
        bad = np.zeros(same.sum(), bool)
        for k in ("t", "u", "v"):
            a, b = g[k][same].astype(np.float64), w[k][same].astype(np.float64)
            bad |= np.abs(a - b) > rel_tol * np.maximum(np.abs(b), 1e-30) + 1e-12
    out["tuv_diff"] = int(bad.sum())
    return out


def assert_parity(res, allow_ties=True, max_near_ties=None):
    assert res["mask_diff"] == 0, res
    assert res["prim_diff"] == 0, res
    assert res["tuv_diff"] == 0, res
    if not allow_ties:
        assert res["ties"] == 0 and res["near_ties"] == 0, res
    if max_near_ties is not None:
        assert res["near_ties"] <= max_near_ties, res


def scene_len2(rays):
    """|d|^2 in float32 in the scene kernel's order, (dx dx + dy dy) + dz dz"""
    d = rays["dir"].astype(np.float32)
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def scene_handed_over_len(rays):
    """rays the production scene walk hands to the list kernel for their direction's length: |d|^2 not within
    1e-5 of 1 (NaN included)"""
    with np.errstate(invalid="ignore"):
        return ~(np.abs(scene_len2(rays) - np.float32(1.0)) <= np.float32(1e-5))


NEAR_ULPS = 8  # world-distance ulps of a near tie: a few ulps of local t, moved through the transform


def _ulp(x):
    return np.spacing(np.abs(np.float32(x)))


def classify_scene_hits(port_scene, rays, got_hits, got_mask, top, top_idx, exact_rays=None):
    """Production two-level walk vs the oracle's Scene::Traverse over the GPU's own top-level tree (`top`,
    `top_idx` = Scene.GetTopLevel()), ray by ray.  Asserts:
      * the same hit mask;
      * every GPU record is exactly what the reference arithmetic gives for the GPU's (instance, triangle)
        (PortScene.prim_hit), and its t is the nearest distance inside that instance (PortScene.instance_hit);
      * where the pick is the oracle's, the whole record is the oracle's;
      * a different pick is one of three classes:
        (a) an exact tie, the same bits of t;
        (b) a distance-versus-entry cull: the reference skips an instance box when the running nearest world
            DISTANCE is below the box's entry ray PARAMETER tmin, and a hit inside the box can lie below tmin by
            |1 - |d|| tmin (direction length) plus the rounding of the transform, so the answer depends on the
            visiting order.  (b) needs the winner's box listed with tmin above the loser's distance (the loser's
            running nearest can have skipped it) and t_lose - t_win <= |1 - |d|| tmin + NEAR_ULPS ulp;
        (c) a near tie inside one instance: two triangles of the same instance (coplanar, or meeting at an edge)
            whose hits lie within NEAR_ULPS ulp; which one the reference reports depends on its visiting order,
            because its box test culls with the running best t at that precision -- the near tie of compare_hits.
            The GPU's pick is likewise within NEAR_ULPS ulp of PortScene.instance_hit.
    `exact_rays` (bool mask): rays that must equal the oracle bit for bit (handed to the list kernel, which runs
    the reference's own order); a tie is still allowed there when the instance trees are not the oracle's.
    Returns ({"hits", "same", "ties", "order", "near", "exact_rays"} counts, the oracle's records)."""
    ph, pm = port_scene.traverse(rays, threads=8, top=top, top_idx=top_idx)
    got_mask = np.asarray(got_mask).astype(bool)
    want_mask = pm.astype(bool)
    bad = np.flatnonzero(got_mask != want_mask)
    assert len(bad) == 0, f"hit mask differs on {len(bad)} rays, first {bad[:8]}"
    hit = np.flatnonzero(want_mask)
    g, w = got_hits[hit], ph[hit]
    # the GPU's record is the reference arithmetic for its own pick
    rt, ok = port_scene.prim_hit(rays[hit], g["node_id"], g["prim_id"])
    assert ok.all() and rt.tobytes() == g.tobytes(), "a GPU record is not prim_hit(node_id, prim_id)"
    it, ok = port_scene.instance_hit(rays[hit], g["node_id"])
    assert ok.all()
    near = np.abs(it["t"].astype(np.float64) - g["t"]) <= NEAR_ULPS * _ulp(it["t"])
    assert near.all(), f"{int((~near).sum())} GPU picks are not the nearest hit of their instance, first " \
        f"{hit[~near][:4]}"
    same = (g["node_id"] == w["node_id"]) & (g["prim_id"] == w["prim_id"])
    assert g[same].tobytes() == w[same].tobytes()
    out = {"hits": len(hit), "same": int(same.sum()), "ties": 0, "order": 0, "near": 0, "exact_rays": 0}
    if exact_rays is not None:
        ex = np.asarray(exact_rays, bool)[hit]
        out["exact_rays"] = int(ex.sum())
    else:
        ex = np.zeros(len(hit), bool)
    len2 = scene_len2(rays[hit])
    unexplained = []
    for j in np.flatnonzero(~same):
        tg, tr = np.float32(g["t"][j]), np.float32(w["t"][j])
        if tg.view(np.uint32) == tr.view(np.uint32):
            out["ties"] += 1
            continue
        if not ex[j]:
            t_win, t_lose = min(tg, tr), max(tg, tr)
            win_node = g["node_id"][j] if tg < tr else w["node_id"][j]
            tmin, _, ids = port_scene.list_node_intersections(rays[hit[j]], top=top, top_idx=top_idx)
            k = np.flatnonzero(ids == win_node)
            if len(k):
                tb = np.float32(tmin[k[0]])
                slack = abs(1.0 - np.sqrt(np.float64(len2[j]))) * float(tb) + NEAR_ULPS * float(_ulp(t_lose))
                if t_lose < tb and float(t_lose) - float(t_win) <= slack:
                    out["order"] += 1
                    continue
        if g["node_id"][j] == w["node_id"][j] and abs(float(tg) - float(tr)) <= NEAR_ULPS * float(_ulp(max(tg, tr))):
            out["near"] += 1
            continue
        unexplained.append((int(hit[j]), g[j], w[j]))
    assert not unexplained, f"{len(unexplained)} picks differ outside the three classes, first: {unexplained[:3]}"
    return out, ph


def check_tree_structure(nodes, indices, verts, faces, min_leaf=4, max_depth=256, preorder=True):
    """Structural invariants every nanort-layout tree must satisfy (SURVEY.md section 4.3, 8b)."""
    n_prims = len(faces)
    n = len(nodes)
    assert n >= 1
    assert np.array_equal(np.sort(indices), np.arange(n_prims, dtype=np.uint32)), "each primitive exactly once"
    flag = nodes["flag"]
    assert np.all((flag == 0) | (flag == 1))
    leaf = flag == 1
    n_leaf, n_branch = int(leaf.sum()), int((~leaf).sum())
    assert n_leaf == n_branch + 1
    # exact triangle boxes
    tri = verts[faces]  # [nf,3,3]
    tmin, tmax = tri.min(axis=1), tri.max(axis=1)
    depth = np.zeros(n, np.int64)
    bmin = np.zeros((n, 3), np.float32)
    bmax = np.zeros((n, 3), np.float32)
    covered = np.zeros(n_prims, np.int64)
    # children always follow their parent in the array -> reverse sweep propagates boxes bottom-up
    d0, d1 = nodes["data"][:, 0].astype(np.int64), nodes["data"][:, 1].astype(np.int64)
    br = np.nonzero(~leaf)[0]
    assert np.all(d0[br] > br) and np.all(d1[br] > br) and np.all(d0[br] < n) and np.all(d1[br] < n)
    assert np.all((nodes["axis"][br] >= 0) & (nodes["axis"][br] <= 2))
    if preorder:
        assert np.all(d0[br] == br + 1), "left child directly follows its parent (DFS pre-order)"
    for i in range(n):
        if not leaf[i]:
            depth[d0[i]] = depth[i] + 1
            depth[d1[i]] = depth[i] + 1
    first = np.zeros(n, np.int64)
    count = np.zeros(n, np.int64)
    for i in range(n - 1, -1, -1):
        if leaf[i]:
            c, f0 = int(d0[i]), int(d1[i])
            assert c >= 1 and f0 + c <= n_prims
            p = indices[f0:f0 + c]
            covered[f0:f0 + c] += 1
            bmin[i], bmax[i] = tmin[p].min(axis=0), tmax[p].max(axis=0)
            first[i], count[i] = f0, c
            assert c <= min_leaf or depth[i] >= max_depth, (i, c, depth[i])
        else:
            a, b = d0[i], d1[i]
            bmin[i] = np.minimum(bmin[a], bmin[b])
            bmax[i] = np.maximum(bmax[a], bmax[b])
            assert first[a] + count[a] == first[b], "children cover adjacent index ranges"
            first[i], count[i] = first[a], count[a] + count[b]
    assert np.all(covered == 1), "leaves partition indices_"
    assert first[0] == 0 and count[0] == n_prims
    assert np.all(depth <= max_depth)
    # boxes are the exact float min/max of the member triangles (numerically: -0.0 == 0.0)
    assert np.array_equal(nodes["bmin"], bmin) and np.array_equal(nodes["bmax"], bmax), "exact node boxes"
    return {"max_tree_depth": int(depth.max()), "num_leaf_nodes": n_leaf, "num_branch_nodes": n_branch}


def random_soup(rng, n):
    """Clustered triangle soup: cluster centres on very different scales, many coincident centroids, some slivers."""
    k = int(rng.integers(1, 6))
    centres = rng.normal(0, 10.0 ** rng.uniform(-2, 2), (k, 3))
    which = rng.integers(0, k, n)
    spread = 10.0 ** rng.uniform(-3, 0.5, k)
    c = centres[which] + rng.normal(0, 1, (n, 3)) * spread[which][:, None]
    dup = rng.random(n) < 0.15  # exact duplicates of another triangle's centroid position
    c[dup] = c[rng.integers(0, n, int(dup.sum()))]
    size = 10.0 ** rng.uniform(-3, 0, (n, 1, 1))
    tri = c[:, None, :] + rng.normal(0, 1, (n, 3, 3)) * size
    flat = rng.random(n) < 0.1  # axis-aligned flat triangles: zero-thickness boxes
    tri[flat, :, int(rng.integers(0, 3))] = c[flat, int(rng.integers(0, 3))][:, None]
    v = tri.reshape(-1, 3).astype(np.float32)
    return v, np.arange(3 * n, dtype=np.uint32).reshape(n, 3)


def degenerate_mesh(kind):
    """Small or degenerate triangle sets: one triangle, five, 3000 copies of one, 700 centroids on a line."""
    if kind == "one":
        v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
        return v, np.array([[0, 1, 2]], np.uint32)
    if kind == "five":
        v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 1], [3, 1, 1], [2, 2, 2], [5, 5, 5]], np.float32)
        return v, np.array([[0, 1, 2], [1, 2, 3], [2, 3, 4], [3, 4, 5], [4, 5, 6]], np.uint32)
    if kind == "identical":  # 3000 copies of one triangle: no plane separates the centroids -> median cuts
        v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
        return v, np.tile(np.array([[0, 1, 2]], np.uint32), (3000, 1))
    if kind == "line":  # centroids on a line along x only
        k = 700
        x = np.arange(k, dtype=np.float32)
        v = np.stack([np.stack([x, 0 * x, 0 * x], 1), np.stack([x + 0.5, 0 * x, 0 * x + 1], 1),
                      np.stack([x, 0 * x + 1, 0 * x], 1)], 1).reshape(-1, 3)
        return v.astype(np.float32), np.arange(3 * k, dtype=np.uint32).reshape(k, 3)
    raise KeyError(kind)
