"""The sphere oracle's entry points (oracle/prim_ref_shim.cc over the unmodified examples/particle_primitive/main.cc)
pinned to the reference's own behaviour, without a GPU: `adopt` of the reference's own tree reproduces its own
Traverse bit for bit, and `test_prim` on the prim Traverse reported reproduces every hit record.  These are what
tests/test_gpu_prims_exact.py builds its ray-by-ray check of the device's sphere kernel on."""
import numpy as np
import pytest

from edge_cases import hostile_rays
from nanort_b200 import scenes as S
from oracle import orc


def _need(cpp11):
    if not orc.ReferenceSpheres.exact_available(cpp11):
        pytest.skip("oracle/_ref/libprim_ref{,03}.so not built from the current oracle/prim_ref_shim.cc "
                    "(no reference tree at build time)")


def _spheres(n, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(-6, 6, size=(n, 3)).astype(np.float32), rng.uniform(0.05, 0.6, size=n).astype(np.float32)


def _rays(centers, n, seed):
    rays = S.incoherent_rays(np.float32([-8] * 3), np.float32([8] * 3), n, seed=seed, axis_parallel_fraction=1.0 / 16)
    rays["min_t"] = 0.0
    k = n // 4
    rays["org"][:k] = centers[np.arange(k) % len(centers)]  # from the centres: the far root, and hits below min_t
    rays["min_t"][: k // 2] = np.float32(0.3)
    rays["max_t"][k : 2 * k] = np.float32(2.5)
    return rays


@pytest.mark.parametrize("cpp11", [True, False])
@pytest.mark.parametrize("n,leaf", [(1, 4), (7, 1), (5000, 4), (5000, 200), (20000, 8)])
def test_adopting_the_reference_tree_reproduces_its_traverse(cpp11, n, leaf):
    _need(cpp11)
    centers, radii = _spheres(n, seed=n + leaf)
    opts = orc.build_options(min_leaf_primitives=leaf)
    ref = orc.ReferenceSpheres(centers, radii, cpp11=cpp11, options=opts)
    nodes, idx = ref.nodes(), ref.indices()
    assert len(idx) == n and sorted(idx) == list(range(n))
    adopted = orc.ReferenceSpheres.adopt(nodes, idx, centers, radii, cpp11=cpp11)
    assert adopted.nodes().tobytes() == nodes.tobytes() and np.array_equal(adopted.indices(), idx)
    rays = np.concatenate([_rays(centers, 20000, seed=n), hostile_rays(np.float32([-7] * 3), np.float32([7] * 3), 4000)])
    topts = orc.trace_options(prim_ids_range=(0, max(1, n // 2)))
    for t in (None, topts):
        wh, wm = ref.traverse(rays, topts=t)
        gh, gm = adopted.traverse(rays, topts=t)
        assert np.array_equal(gm, wm) and gh.tobytes() == wh.tobytes()
    assert wm.sum() > 100


@pytest.mark.parametrize("cpp11", [True, False])
def test_test_prim_of_the_reported_prim_reproduces_every_hit_record(cpp11):
    _need(cpp11)
    centers, radii = _spheres(3000, seed=11)
    ref = orc.ReferenceSpheres(centers, radii, cpp11=cpp11)
    rays = _rays(centers, 40000, seed=5)
    rays["dir"][::7] *= np.float32(1e3)  # non-unit directions
    rays["dir"][1::7] *= np.float32(1e-3)
    for t in (None, orc.trace_options(prim_ids_range=(100, 2000))):
        h, m = ref.traverse(rays, topts=t)
        hit = m.astype(bool)
        assert hit.sum() > 5000
        rec, ok = ref.test_prim(rays[hit], h["prim_id"][hit], topts=t)
        assert ok.all() and rec.tobytes() == h[hit].tobytes()
        # from t_inout = the reported t, the reported prim is still accepted (ties replace: `t > *t_inout` rejects)
        rec, ok = ref.test_prim(rays[hit], h["prim_id"][hit], t_inout=h["t"][hit], topts=t)
        assert ok.all() and rec.tobytes() == h[hit].tobytes()
    # outside the id range Intersect refuses
    _, ok = ref.test_prim(rays[:10], 5, prim_range=(6, 7))
    assert not ok.any()


def test_nan_rays_and_leaf_boxes():
    _need(True)
    centers, radii = _spheres(40, seed=2)
    ref = orc.ReferenceSpheres(centers, radii, options=orc.build_options(min_leaf_primitives=1))
    rays = _rays(centers, 200, seed=3)
    assert not ref.nan_rays(rays).any()
    bad = rays.copy()
    bad["org"][:, 1] = np.nan  # every sphere: NaN discriminant -> NaN t, accepted
    assert ref.nan_rays(bad).all()
    assert not ref.nan_rays(bad, prim_range=(5, 5)).any()  # an empty id range tests nothing
    # the leaf of a sphere the ray hits passes the slab test over [min_t, max_t]
    leaf = ref.leaf_of()
    assert (leaf >= 0).all() and (ref.nodes()["flag"][leaf] == 1).all()
    h, m = ref.traverse(rays)
    for i in np.flatnonzero(m)[:50]:
        assert ref.box_hit(rays[i], leaf[h["prim_id"][i]])
    far = rays[:1].copy()
    far["org"] = (100.0, 100.0, 100.0)
    far["dir"] = (1.0, 0.0, 0.0)
    assert not ref.box_hit(far[0], 0) and not ref.box_hit(far[0], leaf[0])
