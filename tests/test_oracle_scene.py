"""The two-level scene restatement (oracle/nanort_oracle.c, "two-level scene" section) against the unmodified
reference scene graph (examples/nanosg/nanosg.h via oracle/ref_sg_shim.cc): per-instance matrices and boxes,
the top-level tree, the sorted node-hit list and Scene::Traverse's records, all bit for bit."""
import numpy as np
import pytest

from nanort_b200 import scenes as S
from oracle import orc

pytestmark = pytest.mark.skipif(not orc.ReferenceScene.available(), reason="oracle/_ref not built")


def _scene_rays(insts, n, seed):
    lo = np.min([np.min(v @ x[:3, :3] + x[3, :3], axis=0) for v, f, x in insts], axis=0)
    hi = np.max([np.max(v @ x[:3, :3] + x[3, :3], axis=0) for v, f, x in insts], axis=0)
    pad = 0.25 * (hi - lo) + 0.5
    rays = S.incoherent_rays(lo - pad, hi + pad, n, seed=seed)
    rays["min_t"] = 0.0
    return rays


def _same_bits(a, b):
    return a.tobytes() == b.tobytes()


def _same_tree(a, b):
    """bit-equal node arrays; a leaf's `axis` is never written by the reference (nanort.h:1795-1813)"""
    br = a["flag"] == 0
    return (len(a) == len(b) and all(_same_bits(a[k], b[k]) for k in ("bmin", "bmax", "flag", "data"))
            and np.array_equal(a["axis"][br], b["axis"][br]))


@pytest.mark.parametrize("cpp11", [True, False])
@pytest.mark.parametrize("kind", ["mixed", "row"])
def test_port_scene_matches_reference(kind, cpp11):
    if not orc.ReferenceScene.available(cpp11):
        pytest.skip("mode not built")
    insts = S.instances_mixed() if kind == "mixed" else S.instances_row()
    ref = orc.ReferenceScene(insts, cpp11)
    port = orc.PortScene(insts, cpp11)
    # Node::Update: matrices, local and world boxes
    st = ref.node_states()
    for name in st.dtype.names:
        assert _same_bits(st[name], port.sg[name]), name
    # top-level tree + every bottom-level tree
    tn, ti = ref.top()
    assert _same_tree(tn, port.top) and _same_bits(ti, port.top_idx)
    for i in (0, 1, 2, len(insts) - 1):
        bn, bi = ref.node_tree(i)
        assert _same_tree(bn, port.blas[i][0]) and _same_bits(bi, port.blas[i][1])
    rays = _scene_rays(insts, 20000, seed=5)
    if kind == "row":  # rays down the row: > 64 boxes pierced, exact entry ties at the duplicates
        k = np.arange(2000)
        rays["org"][:2000] = np.stack([-3.0 - 0.01 * (k % 7), 0.3 * S.rand01(k, 0, 9) - 0.15,
                                       0.3 * S.rand01(k, 1, 9) - 0.15], axis=1)
        d = np.stack([np.ones(2000), 0.002 * (S.rand01(k, 2, 9) - 0.5), 0.002 * (S.rand01(k, 3, 9) - 0.5)], axis=1)
        rays["dir"][:2000] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
        rays["dir"][:50, 1:] = 0.0
        rays["dir"][:50, 0] = 1.0
        rays["max_t"][:2000] = 1e30
    # first stage: the node-hit list in its exact order
    saw_full = False
    for r in list(range(0, 300)) + list(range(5000, 5100)):
        a = ref.list_node_intersections(rays[r])
        b = port.list_node_intersections(rays[r])
        assert len(a[0]) == len(b[0])
        saw_full |= len(a[0]) == 64
        for x, y in zip(a, b):
            assert _same_bits(x, y), r
    if kind == "row":
        assert saw_full
    # Scene::Traverse
    rh, rm = ref.traverse(rays, threads=4)
    ph, pm = port.traverse(rays, threads=4)
    assert rm.sum() > 500
    assert np.array_equal(rm, pm)
    hit = rm == 1
    assert _same_bits(rh[hit], ph[hit])


@pytest.mark.parametrize("cpp11", [True, False])
@pytest.mark.parametrize("kind", ["mixed", "row", "hostile"])
def test_instance_and_prim_hit_reproduce_every_reference_record(kind, cpp11):
    """PortScene.instance_hit / prim_hit (the per-instance body of Scene::Traverse, on the whole local tree or on one
    triangle) give back every record of the unmodified nanosg.h bit for bit: the GPU scene tests re-test picks with
    them."""
    from edge_cases import hostile_rays

    if not orc.ReferenceScene.available(cpp11):
        pytest.skip("mode not built")
    insts = S.instances_row() if kind == "row" else S.instances_mixed(12 if kind == "hostile" else 24)
    ref = orc.ReferenceScene(insts, cpp11)
    port = orc.PortScene(insts, cpp11)
    if kind == "hostile":
        rays = hostile_rays(np.float32([-8, -4, -8]), np.float32([8, 4, 8]), n=8000, seed=6)
    else:
        rays = _scene_rays(insts, 8000, seed=9)
    rh, rm = ref.traverse(rays, threads=4)
    hit = np.flatnonzero(rm)
    assert len(hit) > 300
    want = rh[hit]
    for got, ok in (port.prim_hit(rays[hit], want["node_id"], want["prim_id"]),
                    port.instance_hit(rays[hit], want["node_id"])):
        assert ok.all() and _same_bits(got, want)
    # the list cut: max_hits=64 is the reference; a larger cut can only add boxes behind the 64 nearest
    ph, pm = port.traverse(rays, threads=4, max_hits=64)
    assert np.array_equal(pm, rm) and _same_bits(ph[hit], want)
    if kind == "row":
        k = np.arange(200)
        rows = rays[:200].copy()
        rows["org"] = np.stack([-3.0 + 0 * k, 0.3 * S.rand01(k, 0, 4) - 0.15, 0.3 * S.rand01(k, 1, 4) - 0.15], axis=1)
        rows["dir"] = (1.0, 0.0, 0.0)
        rows["min_t"], rows["max_t"] = 0.0, 1e30
        assert all(len(port.list_node_intersections(r, max_hits=128)[0]) > 64 for r in rows)
        h64, m64 = port.traverse(rows, max_hits=64)
        h128, m128 = port.traverse(rows, max_hits=128)
        assert np.array_equal(m64, m128) and _same_bits(h64[m64 == 1], h128[m128 == 1])  # the first sphere wins


def test_cull_back_face_flag_is_inert_and_local_ray_is_unbounded():
    """S2 / S4 of the restatement header: the world ray's min_t/max_t gate only the top-level walk."""
    insts = S.instances_mixed(6)
    ref = orc.ReferenceScene(insts)
    port = orc.PortScene(insts)
    rays = _scene_rays(insts, 4000, seed=8)
    rays["max_t"] = 0.75  # far smaller than most hit distances
    rh, rm = ref.traverse(rays)
    ph, pm = port.traverse(rays)
    assert np.array_equal(rm, pm) and _same_bits(rh[rm == 1], ph[pm == 1])
    assert (rh["t"][rm == 1] > 0.75).any()  # hits beyond the world max_t are still reported


def test_port_scene_matches_reference_on_hostile_rays():
    """Non-finite, zero-length and far-from-unit directions through Scene::Traverse: raw bits must match."""
    from edge_cases import hostile_rays

    insts = S.instances_mixed(12)
    ref = orc.ReferenceScene(insts)
    port = orc.PortScene(insts)
    rays = hostile_rays(np.float32([-8, -4, -8]), np.float32([8, 4, 8]), n=8000, seed=5)
    rays["min_t"] = np.where(np.isnan(rays["min_t"]), rays["min_t"], 0.0)
    rh, rm = ref.traverse(rays, threads=4)
    ph, pm = port.traverse(rays, threads=4)
    assert np.array_equal(rm, pm) and _same_bits(rh[rm == 1], ph[pm == 1])
    assert rm.sum() > 300
