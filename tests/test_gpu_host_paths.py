"""The host-side call paths of the float accel, the double accel and the two-level scene under concurrent host threads
and after a failed call: the zero-copy pool of small calls, the chunked staging pipeline of the host-pointer entries,
the lazy host mirrors of the trees, and the ring of per-launch scratch behind them.  Every record is checked against
the same rays traced in one call (or through the device-pointer entry); every mirror against a later single-threaded
call and, for reference builds, against the oracle's arrays."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CHUNK = 1 << 20  # rays per chunk of the staging pipeline


def _run_threads(fns):
    """runs the callables on threads that start together; re-raises the first failure"""
    barrier = threading.Barrier(len(fns))
    errors = []

    def wrap(fn):
        try:
            barrier.wait()
            fn()
        except BaseException as e:  # noqa: BLE001 -- handed to the main thread
            errors.append(e)

    th = [threading.Thread(target=wrap, args=(fn,)) for fn in fns]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errors:
        raise errors[0]


def _scene64(seed):
    """sphere grid with coordinates that do not survive a round trip through float"""
    from nanort_b200 import scenes as S

    v, f = S.sphere_grid(nx=3, nz=3)
    rng = np.random.default_rng(seed)
    return v.astype(np.float64) * (1.0 + 1e-9 * rng.standard_normal(v.shape)), f


def _rays64(v64, n, seed):
    from nanort_b200 import api, scenes as S

    r32 = S.incoherent_rays(v64.min(axis=0).astype(np.float32), v64.max(axis=0).astype(np.float32), n, seed=seed)
    r = np.zeros(n, api.RAY64_DTYPE)
    r["org"], r["dir"] = r32["org"], r32["dir"]
    r["min_t"], r["max_t"] = r32["min_t"], r32["max_t"]
    return r


def _bounds(insts):
    lo = np.min([np.min(v @ x[:3, :3] + x[3, :3], axis=0) for v, f, x in insts], axis=0)
    hi = np.max([np.max(v @ x[:3, :3] + x[3, :3], axis=0) for v, f, x in insts], axis=0)
    return lo, hi


def _scene_rays(insts, n, seed):
    from nanort_b200 import scenes as S

    lo, hi = _bounds(insts)
    rays = S.incoherent_rays(lo - 1.0, hi + 1.0, n, seed=seed)
    rays["min_t"] = 0.0
    rays["dir"][::5] *= np.float32(0.5)  # some rays through the list kernel
    return rays


def _scene(insts, flags=0):
    from nanort_b200 import api

    accels, sc = [], api.Scene()
    for v, f, x in insts:
        a = api.BVHAccel()
        assert a.Build(len(f), v, f, flags=flags)
        accels.append(a)
        sc.AddNode(a, x)
    assert sc.Commit(flags)
    return sc, accels


def _scene_device_records(sc, rays):
    """the same rays through nrt_scene_traverse_device"""
    import torch

    n = len(rays)
    d_rays = torch.from_numpy(rays.view(np.uint8).reshape(-1, 36).copy()).cuda()
    d_hits = torch.full((n, 32), 0xFF, dtype=torch.uint8, device="cuda")
    d_mask = torch.full((n,), 0xFF, dtype=torch.uint8, device="cuda")
    sc.TraverseDevice(d_rays.data_ptr(), n, d_hits.data_ptr(), d_mask.data_ptr(),
                      stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return d_hits.cpu().numpy().tobytes(), d_mask.cpu().numpy()


def test_f64_small_calls_from_threads_equal_one_batched_call():
    """Eight threads make reference-order calls of 1..65 rays (every other one without hit flags) on one
    BVHAccelF64 while a ninth makes fast calls of more than 64 rays: every record is the bits of one batched call."""
    from nanort_b200 import api

    v64, f = _scene64(seed=41)
    acc = api.BVHAccelF64()
    assert acc.Build(len(f), v64, f)
    sizes = [1 + k % 65 for k in range(4 * 65)]
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    rays = _rays64(v64, int(sum(sizes)), seed=43)
    want_h, want_m = acc.Traverse(rays, flags=api.TRAVERSE_CONFORMANCE)
    fast_rays = _rays64(v64, 40 * 300, seed=47)
    want_fh, want_fm = acc.Traverse(fast_rays)
    assert want_m.sum() > len(rays) // 20 and want_fm.sum() > len(fast_rays) // 20

    got_h, got_m = np.zeros(len(rays), api.HIT64_DTYPE), np.full(len(rays), 0xFF, np.uint8)
    got_fh, got_fm = np.zeros(len(fast_rays), api.HIT64_DTYPE), np.full(len(fast_rays), 0xFF, np.uint8)
    L = api.lib()

    def small_calls(t):
        for k in range(t, len(sizes), 8):
            a, m = int(starts[k]), sizes[k]
            mask = api._p(got_m[a:a + m]) if k % 2 == 0 else None
            api._check(L.nrt_traverse_f64(acc._h, api._p(rays[a:a + m]), m, api._p(got_h[a:a + m]), mask, None,
                                          api.TRAVERSE_CONFORMANCE))

    def fast_calls():
        for a in range(0, len(fast_rays), 300):
            acc.Traverse(fast_rays[a:a + 300], hits=got_fh[a:a + 300], mask=got_fm[a:a + 300])

    _run_threads([lambda t=t: small_calls(t) for t in range(8)] + [fast_calls])
    assert got_h.tobytes() == want_h.tobytes()
    flagged = np.concatenate([np.arange(starts[k], starts[k] + sizes[k]) for k in range(0, len(sizes), 2)])
    assert np.array_equal(got_m[flagged], want_m[flagged])
    unflagged = np.setdiff1d(np.arange(len(rays)), flagged)
    assert np.all(got_m[unflagged] == 0xFF)  # no flags were asked for: none were written
    assert got_fh.tobytes() == want_fh.tobytes() and np.array_equal(got_fm, want_fm)


def test_two_scenes_traversed_from_host_threads_at_once():
    """Four threads over two scenes, one of them with a call of 2^20 + 777 rays (two chunks), the others with calls
    of 40 K rays: every record equals the device entry's on the same rays."""
    from nanort_b200 import scenes as S

    scenes = [_scene(S.instances_mixed()), _scene(S.instances_row())]
    insts = [S.instances_mixed(), S.instances_row()]
    jobs = [(0, _scene_rays(insts[0], CHUNK + 777, seed=51), 1)]  # (scene, rays, calls)
    jobs += [(k % 2, _scene_rays(insts[k % 2], 3 * 40_000, seed=52 + k), 3) for k in range(1, 4)]
    got = [None] * len(jobs)

    def work(j):
        s, rays, calls = jobs[j]
        parts = [scenes[s][0].Traverse(r) for r in np.array_split(rays, calls)]
        got[j] = (np.concatenate([h for h, _ in parts]), np.concatenate([m for _, m in parts]))

    _run_threads([lambda j=j: work(j) for j in range(len(jobs))])
    for j, (s, rays, _) in enumerate(jobs):
        want_h, want_m = _scene_device_records(scenes[s][0], rays)
        assert want_m.sum() > 0.01 * len(rays), j
        assert np.array_equal(got[j][1], want_m), j
        assert got[j][0].tobytes() == want_h, j


@pytest.mark.parametrize("build", ["fast", "reference"])
def test_mirrors_from_threads(port, build):
    """GetNodes / GetIndices of a freshly built float accel, double accel and scene (GetTopLevel) from eight threads
    at once: all equal a later single-threaded call and, for reference builds, the oracle's arrays."""
    from nanort_b200 import api, scenes as S
    from oracle import orc

    flags = api.BUILD_REFERENCE_TREE if build == "reference" else api.BUILD_FAST
    v, f = S.make_scene("sphere_grid", nx=4, nz=4)
    v64, f64 = _scene64(seed=61)
    insts = S.instances_mixed()
    acc = api.BVHAccel()
    assert acc.Build(len(f), v, f, flags=flags)
    acc64 = api.BVHAccelF64()
    assert acc64.Build(len(f64), v64, f64, flags=flags)
    sc, _keep = _scene(insts, flags)
    getters = {"float": lambda: (acc.GetNodes(), acc.GetIndices()),
               "f64": lambda: (acc64.GetNodes(), acc64.GetIndices()),
               "scene": sc.GetTopLevel}
    got = {name: [None] * 8 for name in getters}

    def work(t):
        for name, get in getters.items():
            got[name][t] = get()

    _run_threads([lambda t=t: work(t) for t in range(8)])
    oracle = {}
    if build == "reference":
        oracle["float"] = port.build(v, f, mode=orc.MODE_CPP11)[:2]
        oracle["f64"] = orc.Port64().build(v64, f64, mode=orc.MODE_CPP11)[:2]
        ps = orc.PortScene(insts, cpp11=True, port=port)
        oracle["scene"] = (ps.top, ps.top_idx)
    for name, get in getters.items():
        nodes, idx = get()
        assert len(nodes) > 1 and len(idx) > 0, name
        for t, (n_t, i_t) in enumerate(got[name]):
            assert n_t.tobytes() == nodes.tobytes() and np.array_equal(i_t, idx), (name, t)
        if name in oracle:
            want_nodes, want_idx = oracle[name]
            assert np.array_equal(idx, want_idx), name
            for k in ("bmin", "bmax", "flag", "data"):
                assert nodes[k].tobytes() == want_nodes[k].tobytes(), (name, k)


def test_a_failed_host_call_leaves_the_accel_and_the_scene_usable():
    """nrt_traverse and nrt_scene_traverse of more than one chunk with reserved flag bits return the error; the next
    call on the same object gives the device entry's records."""
    import torch
    from nanort_b200 import api, scenes as S

    v, f = S.make_scene("sphere_grid", nx=4, nz=4)
    acc = api.BVHAccel()
    assert acc.Build(len(f), v, f)
    rays = S.incoherent_rays(v.min(axis=0), v.max(axis=0), CHUNK + 777, seed=71)
    with pytest.raises(api.NanortB200Error, match="reserved"):
        acc.Traverse(rays, flags=(3 << 8))
    h, m = acc.Traverse(rays)
    d_rays = torch.from_numpy(rays.view(np.uint8).reshape(-1, 36).copy()).cuda()
    d_hits = torch.full((len(rays), 16), 0xFF, dtype=torch.uint8, device="cuda")
    d_mask = torch.full((len(rays),), 0xFF, dtype=torch.uint8, device="cuda")
    acc.TraverseDevice(d_rays.data_ptr(), len(rays), d_hits.data_ptr(), d_mask.data_ptr(),
                       stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert m.sum() > 0.05 * len(rays)
    assert np.array_equal(m, d_mask.cpu().numpy()) and h.tobytes() == d_hits.cpu().numpy().tobytes()

    insts = S.instances_mixed()
    sc, _keep = _scene(insts)
    rays = _scene_rays(insts, CHUNK + 777, seed=73)
    with pytest.raises(api.NanortB200Error, match="reserved"):
        sc.Traverse(rays, flags=(2 << 8))
    h, m = sc.Traverse(rays)
    want_h, want_m = _scene_device_records(sc, rays)
    assert m.sum() > 0.05 * len(rays)
    assert np.array_equal(m, want_m) and h.tobytes() == want_h
