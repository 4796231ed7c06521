"""Non-triangle primitives (csrc/prims.cu): the device kinds of nanort's Prim / Pred / Intersector concept against the
reference's own models running on the unmodified nanort.h.

  * spheres: examples/particle_primitive/main.cc's SphereGeometry / SpherePred / SphereIntersector
             (oracle/_ref/libprim_ref.so).  The trees differ (the reference builds its own), hits do not depend on the
             topology: hit flag and prim_id identical, t bit-identical, u / v within 1e-6 (atan2 / acos of two libms).
  * boxes:   BVHAccel::ListNodeIntersections with nanosg's NodeBBoxIntersector (oracle/_ref/libnanosg_ref.so): the same
             nearest-first list of pierced boxes, bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _spheres(n, seed, rmax=0.35):
    rng = np.random.default_rng(seed)
    centers = rng.uniform(-6, 6, size=(n, 3)).astype(np.float32)
    radii = rng.uniform(0.02, rmax, size=n).astype(np.float32)
    return centers, radii


def _rays(n, seed, lo=-8.0, hi=8.0):
    from nanort_b200 import scenes as S

    r = S.incoherent_rays(np.float32([lo] * 3), np.float32([hi] * 3), n, seed=seed, axis_parallel_fraction=1.0 / 64)
    r["min_t"] = 0.0
    return r


@pytest.mark.parametrize("n_spheres", [1, 7, 5000, 200000])
def test_spheres_match_the_reference_particle_primitive_model(n_spheres):
    from oracle import orc
    from nanort_b200 import api

    if not orc.ReferenceSpheres.available():
        pytest.skip("oracle/_ref/libprim_ref.so not built")
    centers, radii = _spheres(n_spheres, seed=n_spheres)
    ref = orc.ReferenceSpheres(centers, radii)
    acc = api.BVHAccel()
    assert acc.BuildSpheres(centers, radii)
    gb, rb = acc.BoundingBox(), ref.bounding_box()
    assert np.array_equal(gb[0], rb[0]) and np.array_equal(gb[1], rb[1])
    st = acc.GetStatistics()
    assert st["num_leaf_nodes"] == st["num_branch_nodes"] + 1
    rays = _rays(60000, seed=3)
    # rays starting inside spheres and rays with a short range exercise the t0 < 0 and the `t > t_inout` branches
    rays["org"][:2000] = centers[np.arange(2000) % n_spheres] + np.float32(0.01)
    rays["max_t"][2000:6000] = np.float32(3.0)
    want_h, want_m = ref.traverse(rays)
    got_h, got_m = acc.Traverse(rays)
    assert np.array_equal(got_m, want_m), int((got_m != want_m).sum())
    hit = want_m.astype(bool)
    assert hit.sum() > (100 if n_spheres > 100 else 0)
    same_prim = got_h["prim_id"][hit] == want_h["prim_id"][hit]
    # overlapping spheres can be hit at exactly the same distance: the reference keeps whichever it tested last
    ties = ~same_prim & (got_h["t"][hit] == want_h["t"][hit])
    assert int((~same_prim).sum()) == int(ties.sum())
    assert np.array_equal(got_h["t"][hit].view(np.uint32), want_h["t"][hit].view(np.uint32)), "t must be bit-identical"
    ok = same_prim
    assert np.max(np.abs(got_h["u"][hit][ok] - want_h["u"][hit][ok]), initial=0.0) <= 1e-6
    assert np.max(np.abs(got_h["v"][hit][ok] - want_h["v"][hit][ok]), initial=0.0) <= 1e-6


def test_sphere_prim_id_range_filter():
    from oracle import orc
    from nanort_b200 import api

    if not orc.ReferenceSpheres.available():
        pytest.skip("oracle/_ref/libprim_ref.so not built")
    centers, radii = _spheres(3000, seed=5)
    ref = orc.ReferenceSpheres(centers, radii)
    acc = api.BVHAccel()
    acc.BuildSpheres(centers, radii)
    rays = _rays(20000, seed=9)
    opt = api.BVHTraceOptions(prim_ids_range=(500, 1500))
    want_h, want_m = ref.traverse(rays, prim_range=(500, 1500))
    got_h, got_m = acc.Traverse(rays, options=opt)
    assert np.array_equal(got_m, want_m)
    hit = want_m.astype(bool)
    assert hit.any() and got_h["prim_id"][hit].min() >= 500 and got_h["prim_id"][hit].max() < 1500
    assert np.array_equal(got_h["t"][hit].view(np.uint32), want_h["t"][hit].view(np.uint32))


def test_sphere_build_of_nothing_fails_like_the_reference():
    from nanort_b200 import api

    acc = api.BVHAccel()
    assert acc.BuildSpheres(np.zeros((0, 3), np.float32), np.zeros(0, np.float32)) is False


@pytest.mark.parametrize("max_hits", [64, 5, 1])
def test_list_node_intersections_matches_the_reference(max_hits):
    """The boxes are the world boxes of a reference nanosg scene's nodes.  BVHAccel::ListNodeIntersections is a property
    of the TREE, not only of the boxes: the leaf-level NodeBBoxIntersector has no [min_t, max_t] clamp (nanosg.h:597-634),
    so a box behind the origin is listed iff it shares a leaf with a box the range-clamped node test lets through.  The
    device list is therefore compared, bit for bit, with the reference algorithm walking the DEVICE's tree (the oracle's
    restatement, itself pinned to the unmodified nanosg.h on the reference's tree -- re-checked below), and with the
    reference's own list on every ray whose answer cannot depend on the leaves (all listed boxes start in front of
    min_t)."""
    from edge_cases import hostile_rays
    from oracle import orc
    from nanort_b200 import api, scenes as S

    if not orc.ReferenceScene.available(True):
        pytest.skip("oracle/_ref/libnanosg_ref.so not built")
    insts = S.instances_row(80)  # a row of overlapping instances: rays along the row pierce > 64 boxes
    ref = orc.ReferenceScene(insts, cpp11=True)
    port = orc.Port()
    st = ref.node_states()
    ref_nodes, ref_idx = ref.top()
    boxes = np.concatenate([st["xbmin"], st["xbmax"]], axis=1).astype(np.float32)
    acc = api.BVHAccel()
    assert acc.BuildBoxes(boxes)
    dev_nodes, dev_idx = acc.GetNodes(), acc.GetIndices()
    bmin, bmax = boxes[:, :3].min(axis=0), boxes[:, 3:].max(axis=0)
    rays = S.incoherent_rays(bmin - 1, bmax + 1, 3000, seed=4, axis_parallel_fraction=0.25)
    # rays down the row (both ways, slightly tilted, some starting inside it): these pierce tens of boxes, more than 64
    # for the long ones, and meet the coincident instances at exactly equal distances
    k = np.arange(240)
    down = np.zeros(len(k), S.RAY_DTYPE)
    fwd = (k % 2) == 0
    down["org"][:, 0] = np.where(fwd, -2.0 + 0.37 * (k % 60), 82.0 - 0.41 * (k % 50))
    down["org"][:, 1] = 0.3 * np.sin(k * 0.7)
    down["org"][:, 2] = 0.3 * np.cos(k * 1.3)
    d = np.stack([np.where(fwd, 1.0, -1.0), 0.004 * np.sin(k * 2.1), 0.004 * np.cos(k * 0.9)], axis=1)
    down["dir"] = (d / np.linalg.norm(d, axis=1)[:, None]).astype(np.float32)
    down["max_t"] = np.where(k % 3 == 0, 30.0, 1e30)
    rays = np.concatenate([rays, down])
    rays["min_t"] = 0.0
    hits, counts = acc.ListNodeIntersections(rays, max_intersections=max_hits)
    many = tree_independent = 0
    for i in range(len(rays)):
        r_tmin, r_tmax, r_ids = ref.list_node_intersections(rays[i], max_hits)
        if i < 300:  # the restatement on the reference's tree is the reference (pinned on CPU too)
            o_tmin, o_tmax, o_ids = orc.list_node_intersections_on_tree(port, ref_nodes, ref_idx, st, rays[i], max_hits)
            assert np.array_equal(o_ids, r_ids) and np.array_equal(o_tmin.view(np.uint32), r_tmin.view(np.uint32)), i
        tmin, tmax, ids = orc.list_node_intersections_on_tree(port, dev_nodes, dev_idx, st, rays[i], max_hits)
        assert counts[i] == len(ids), (i, counts[i], len(ids))
        g = hits[i, : counts[i]]
        assert np.array_equal(g["t_min"].view(np.uint32), tmin.view(np.uint32)), i
        assert np.array_equal(g["node_id"], ids), i  # same tree, same heap: same order, ties included
        assert np.array_equal(g["t_max"].view(np.uint32), tmax.view(np.uint32)), i
        if len(r_ids) == len(ids) and len(ids) < max_hits and (len(ids) == 0 or (tmin.min() > 0.0 and r_tmin.min() > 0.0)):
            # nothing was dropped and nothing lies behind the origin: the set of boxes is the same in any tree
            assert sorted(ids) == sorted(r_ids), i
            tree_independent += 1
        many += int(counts[i] >= min(max_hits, 10))
    assert many > 20 and tree_independent > 100
    # the C++03 inverse (-0.0 -> +inf) and the hostile rays of tests/edge_cases.py (NaN / inf / zero components,
    # inverted and NaN ranges), against the restatement on the device's tree in each convention; the restatement's
    # C++03 convention is pinned to the unmodified nanosg.h built without NANORT_USE_CPP11_FEATURE on its own tree
    hostile = hostile_rays(bmin - 1, bmax + 1, 1200, seed=6)
    both = np.concatenate([rays, hostile])
    for cpp11 in (True, False):
        flags = 0 if cpp11 else api.TRAVERSE_CPP03_INVERSE
        hits, counts = acc.ListNodeIntersections(both, max_intersections=max_hits, flags=flags)
        for i in range(len(rays) if cpp11 else 0, len(both)):
            tmin, tmax, ids = orc.list_node_intersections_on_tree(port, dev_nodes, dev_idx, st, both[i], max_hits,
                                                                  cpp11=cpp11)
            assert counts[i] == len(ids), (cpp11, i, counts[i], len(ids))
            g = hits[i, : counts[i]]
            assert np.array_equal(g["node_id"], ids), (cpp11, i)
            assert _same_f32(g["t_min"], tmin) and _same_f32(g["t_max"], tmax), (cpp11, i)
    if orc.ReferenceScene.available(False):
        ref03 = orc.ReferenceScene(insts, cpp11=False)
        n03, i03 = ref03.top()
        st03 = ref03.node_states()
        for i in range(len(rays), len(both), 3):
            r_tmin, r_tmax, r_ids = ref03.list_node_intersections(both[i], max_hits)
            o_tmin, o_tmax, o_ids = orc.list_node_intersections_on_tree(port, n03, i03, st03, both[i], max_hits, cpp11=False)
            assert np.array_equal(o_ids, r_ids) and _same_f32(o_tmin, r_tmin), i


def _same_f32(a, b):
    """bit for bit, except that any NaN equals any NaN (the device and the host spell NaN differently)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    if a.shape != b.shape:
        return False
    both_nan = np.isnan(a) & np.isnan(b)
    return bool(np.all(both_nan | (a.view(np.uint32) == b.view(np.uint32))))
