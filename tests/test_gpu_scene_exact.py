"""The production two-level walk (scene_unified_kernel, what nrt_scene_traverse[_device] and the scene AO pass run by
default) ray by ray against the oracle's Scene::Traverse over the GPU's own top-level tree.

Per ray (helpers.classify_scene_hits): the same hit mask; every GPU record is the reference arithmetic for its own
(instance, triangle) and the nearest hit of that instance; the whole record is the oracle's where the pick is the
same; a different pick is an exact tie (same bits of t), a distance-versus-entry cull or a near tie between two
triangles of one instance (helpers.classify_scene_hits states the three classes).  Rays the kernel hands to the list kernel (|d|^2 off 1 by more than 1e-5, more than 64 instance
boxes) equal the oracle bit for bit.  Every family first asserts, with the oracle, that it reaches what it is there
to test.  Then: the 2^20-ray host chunking, and launches on eight streams at once against serial ones."""
import threading

import numpy as np
import pytest

from helpers import classify_scene_hits, scene_handed_over_len, scene_len2

pytestmark = pytest.mark.gpu


def _bounds(insts):
    lo = np.min([np.min(v @ x[:3, :3] + x[3, :3], axis=0) for v, f, x in insts], axis=0)
    hi = np.max([np.max(v @ x[:3, :3] + x[3, :3], axis=0) for v, f, x in insts], axis=0)
    return lo, hi


def _hollow_instances(n=80, seed=3):
    """n overlapping, rotated and scaled copies of a hollow box: two triangles at opposite corners of [-0.5, 0.5]^3.
    A ray through the middle pierces most of the n boxes and misses most of the geometry, so the 64 boxes with the
    nearest entries often hold no hit or not the nearest one."""
    from nanort_b200 import scenes as S

    v = np.array([[0, 0, 0], [0.6, 0, 0], [0, 0.6, 0.1], [1, 1, 1], [0.4, 1, 0.9], [1, 0.4, 1]], np.float32) - 0.5
    f = np.array([[0, 1, 2], [3, 4, 5]], np.uint32)
    i = np.arange(n, dtype=np.int64)
    r = [S.rand01(i, k, seed) for k in range(8)]
    return [(v, f, S.xform(translate=((r[0][k] - 0.5), (r[1][k] - 0.5), (r[2][k] - 0.5)),
                           scale=(2.0 + 2.0 * r[3][k], 2.0 + 2.0 * r[4][k], 2.0 + 2.0 * r[5][k]),
                           yaw=float(r[6][k]) * 6.2831853, pitch=(float(r[7][k]) - 0.5) * 1.5)) for k in range(n)]


def _mirror_instances():
    """27 axis-aligned, scaled and mirrored Cornell boxes on a grid: a world direction with +0.0 components becomes a
    local one with -0.0 components, where the C++03 and C++11 inverses (+inf / -inf) disagree"""
    from nanort_b200 import scenes as S

    v, f = S.cornell()
    v = v * np.float32(0.2)
    return [(v, f, S.xform(translate=(3.0 * (k % 3), 3.0 * ((k // 3) % 3), 3.0 * (k // 9)),
                           scale=(0.5 + 0.5 * (k % 3), -1.0 if k % 2 else 1.0, 1.0 if (k // 2) % 2 else -1.0)))
            for k in range(27)]


def _instances(kind):
    from nanort_b200 import scenes as S

    return {"mixed": S.instances_mixed, "row": S.instances_row, "hollow": _hollow_instances,
            "mirror": _mirror_instances}[kind]()


def _incoherent(insts, n, seed):
    from nanort_b200 import scenes as S

    lo, hi = _bounds(insts)
    pad = 0.25 * (hi - lo) + 0.5
    rays = S.incoherent_rays(lo - pad, hi + pad, n, seed=seed)
    rays["min_t"] = 0.0
    return rays


def _toward(insts, n, seed, spread=0.35):
    """rays from a sphere around the scene towards random points of its middle: unit directions (rounded in float64
    first), [0, 1e30]; returns (rays, distance from the origin to the aim point)"""
    from nanort_b200 import scenes as S

    lo, hi = _bounds(insts)
    c, ext = 0.5 * (lo + hi), 0.5 * (hi - lo)
    i = np.arange(n, dtype=np.int64)
    u = np.stack([S.rand01(i, k, seed) for k in range(6)], axis=1).astype(np.float64)
    z, ph = 2.0 * u[:, 0] - 1.0, 2.0 * np.pi * u[:, 1]
    s = np.sqrt(1.0 - z * z)
    org = c + 1.5 * np.linalg.norm(ext) * np.stack([s * np.cos(ph), z, s * np.sin(ph)], axis=1)
    aim = c + spread * ext * (2.0 * u[:, 2:5] - 1.0)
    d = aim - org
    dist = np.linalg.norm(d, axis=1)
    rays = np.zeros(n, S.RAY_DTYPE)
    rays["org"] = org.astype(np.float32)
    rays["dir"] = (d / dist[:, None]).astype(np.float32)
    rays["min_t"], rays["max_t"] = 0.0, 1e30
    return rays, dist


def _with_len2(rays, target, seed):
    """directions scaled to |d|^2 = target, kept where float32 (kernel order) rounds it to the same side of the
    1e-5 handoff threshold as `target`"""
    d = rays["dir"].astype(np.float64)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    out = rays.copy()
    out["dir"] = (d * np.sqrt(target)).astype(np.float32)
    want = abs(target - 1.0) > 1e-5
    keep = scene_handed_over_len(out) == want
    assert keep.mean() > 0.9
    return out[keep]


def _axis_rays(insts, n, seed):
    """axis-parallel directions with +0.0 / -0.0 in the other components, aimed along the axis at a random point
    near the middle of a random instance's world box from outside the scene"""
    from nanort_b200 import scenes as S

    rays = _incoherent(insts, n, seed)
    i = np.arange(n, dtype=np.int64)
    axis, sgn = (i % 3), np.where(S.rand01(i, 11, seed) < 0.5, -1.0, 1.0).astype(np.float32)
    z0 = np.where(S.rand01(i, 12, seed) < 0.5, np.float32(-0.0), np.float32(0.0))
    z1 = np.where(S.rand01(i, 13, seed) < 0.5, np.float32(-0.0), np.float32(0.0))
    z2 = np.where(S.rand01(i, 14, seed) < 0.5, np.float32(-0.0), np.float32(0.0))
    d = np.stack([z0, z1, z2], axis=1).astype(np.float32)
    d[i, axis] = sgn
    lo, hi = _bounds(insts)
    boxes = [(np.min(v @ x[:3, :3] + x[3, :3], axis=0), np.max(v @ x[:3, :3] + x[3, :3], axis=0)) for v, f, x in insts]
    k = (S.rand01(i, 15, seed) * len(insts)).astype(np.int64)
    b0, b1 = np.array([boxes[j][0] for j in k]), np.array([boxes[j][1] for j in k])
    jit = np.stack([S.rand01(i, 16 + a, seed) for a in range(3)], axis=1) - 0.5
    org = 0.5 * (b0 + b1) + 0.6 * (b1 - b0) * jit
    org[i, axis] = np.where(sgn > 0, lo[axis] - 1.0, hi[axis] + 1.0)
    rays["org"] = org.astype(np.float32)
    rays["dir"] = d
    rays["max_t"] = 1e30
    return rays


def _row_rays(n):
    from nanort_b200 import scenes as S

    k = np.arange(n)
    rays = np.zeros(n, S.RAY_DTYPE)
    rays["org"] = np.stack([-3.0 - 0.01 * (k % 7), 0.3 * S.rand01(k, 0, 9) - 0.15, 0.3 * S.rand01(k, 1, 9) - 0.15], 1)
    d = np.stack([np.ones(n), 0.002 * (S.rand01(k, 2, 9) - 0.5), 0.002 * (S.rand01(k, 3, 9) - 0.5)], axis=1)
    rays["dir"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    rays["dir"][:50, 1:] = 0.0
    rays["dir"][:50, 0] = 1.0
    rays["max_t"] = 1e30
    return rays


def _families(insts, kind, port, seed):
    """name -> rays"""
    fam = {"incoherent": _incoherent(insts, 60000, seed)}
    t, dist = _toward(insts, 30000, seed + 1)
    h, m = port.traverse(t, threads=8)
    # [min_t, max_t] ends near the first hit of [0, inf): the range cuts through instance boxes, and the boxes that
    # lie wholly outside it drop out of the top-level walk
    u = np.random.default_rng(seed).uniform(0.5, 1.5, len(t))
    cut = (np.where(m == 1, h["t"], 0.5 * dist) * u).astype(np.float32)
    fam["min_t"] = t.copy()
    fam["min_t"]["min_t"] = cut
    fam["max_t"] = t.copy()
    fam["max_t"]["max_t"] = cut
    t, _ = _toward(insts, 40000, seed + 2)
    fam["len2_in"] = np.concatenate([_with_len2(t[:20000], 1.0 + 0.9e-5, seed), _with_len2(t[20000:], 1.0 - 0.9e-5, seed)])
    fam["len2_out"] = np.concatenate([_with_len2(t[:20000], 1.0 + 1.1e-5, seed),
                                      _with_len2(t[20000:], 1.0 - 1.1e-5, seed)])
    t, _ = _toward(insts, 20000, seed + 3)
    fam["len_half"], fam["len_three"] = t.copy(), t.copy()
    fam["len_half"]["dir"] *= np.float32(0.5)
    fam["len_three"]["dir"] *= np.float32(3.0)
    fam["axis"] = _axis_rays(insts, 12000, seed + 4)
    if kind == "row":
        fam["row"] = _row_rays(4000)
    return fam


def _gpu_scene(insts, blas_flags, top_flags):
    from nanort_b200 import api

    accels = {}
    sc = api.Scene()
    for v, f, x in insts:
        key = (v.ctypes.data, f.ctypes.data)
        if key not in accels:
            a = api.BVHAccel()
            a.Build(len(f), v, f, flags=blas_flags)
            accels[key] = a
        sc.AddNode(accels[key], x)
    assert sc.Commit(top_flags)
    return sc


def _assert_preconditions(kind, fam, port, top, ti, cpp11, cpp03_ports):
    """each family reaches what it is there to test (the oracle over the GPU's top-level tree)"""
    def trav(rays, **kw):
        return port.traverse(rays, threads=8, top=top, top_idx=ti, **kw)

    def differ(a, b):
        (ha, ma), (hb, mb) = a, b
        return (ma != mb) | ((ma == 1) & (ha["t"] != hb["t"]))

    for name in ("min_t", "max_t"):
        rays = fam[name]
        full = rays.copy()
        full["min_t"], full["max_t"] = 0.0, 1e30
        h, m = trav(rays)
        assert differ((h, m), trav(full)).sum() >= 30, name  # the [min_t, max_t] gate of the top level matters
        if name == "min_t":  # hits nearer than min_t are still reported: the instance walk runs {0, FLT_MAX}
            assert ((m == 1) & (h["t"] < rays["min_t"])).sum() >= 30
    if kind == "hollow":  # the 64-box cut changes the reference's answer
        rays = np.concatenate([fam["incoherent"], fam["len2_in"]])
        assert differ(trav(rays), trav(rays, max_hits=128)).sum() >= 100
    if kind == "mixed":  # |d| = 0.5: the visiting order decides; the nearest hit over all instances is not the answer
        rays = fam["len_half"]
        h, m = trav(rays)
        best = np.full(len(rays), np.inf, np.float32)
        for i in range(len(port.sg)):
            hi, ok = port.instance_hit(rays, i)
            best = np.where(ok & (hi["t"] < best), hi["t"], best)
        assert ((m == 1) & (h["t"] != best)).sum() >= 10
    if kind == "mirror" and not cpp11:  # local -0.0 components: the C++03 inverse (+inf) and the C++11 one (-inf)
        p11, p03 = cpp03_ports
        rays = fam["axis"]
        a = p11.traverse(rays, threads=8, top=top, top_idx=ti)
        b = p03.traverse(rays, threads=8, top=top, top_idx=ti)
        assert differ(a, b).sum() >= 100


COUNTS = {}


@pytest.mark.parametrize("mode", ["cpp11", "cpp03"])
@pytest.mark.parametrize("top_build", ["fast", "ref"])
@pytest.mark.parametrize("blas_build", ["ref", "fast"])
@pytest.mark.parametrize("kind", ["mixed", "row", "hollow", "mirror"])
def test_production_scene_walk_ray_by_ray(kind, blas_build, top_build, mode):
    from nanort_b200 import api
    from oracle import orc

    cpp11 = mode == "cpp11"
    ref_flags = api.BUILD_REFERENCE_TREE | (0 if cpp11 else api.BUILD_REFERENCE_CPP03_ORDER)
    insts = _instances(kind)
    port = orc.PortScene(insts, cpp11=cpp11)
    sc = _gpu_scene(insts, ref_flags if blas_build == "ref" else api.BUILD_FAST,
                    ref_flags if top_build == "ref" else api.BUILD_FAST)
    top, ti = sc.GetTopLevel()
    if top_build == "ref":
        assert top.tobytes() == port.top.tobytes() and ti.tobytes() == port.top_idx.tobytes()
    fam = _families(insts, kind, port, seed=17)
    _assert_preconditions(kind, fam, port, top, ti, cpp11,
                          (orc.PortScene(insts, cpp11=True), port) if not cpp11 else None)
    flags = api.TRAVERSE_FAST if cpp11 else api.TRAVERSE_CPP03_INVERSE
    counts = {}
    for name, rays in fam.items():
        gh, gm = sc.Traverse(rays, flags=flags)
        handed = scene_handed_over_len(rays)
        if name in ("len2_out", "len_half", "len_three"):
            assert handed.all()
        if name == "len2_in":
            assert not handed.any() and (scene_len2(rays) != 1.0).all()
        res, ph = classify_scene_hits(port, rays, gh, gm, top, ti, exact_rays=handed)
        if blas_build == "ref":  # the list kernel walks the oracle's own trees in the reference's order
            ex = handed & (gm == 1)
            assert gh[ex].tobytes() == ph[ex].tobytes(), name
        counts[name] = res
    COUNTS[(kind, blas_build, top_build, mode)] = counts
    print(kind, blas_build, top_build, mode, {k: (v["hits"], v["ties"], v["order"], v["near"]) for k, v in counts.items()})


def test_production_scene_walk_on_hostile_rays():
    """non-finite, zero-length, denormal and far-from-unit directions, inverted and NaN ranges, over production-built
    instance and top-level trees"""
    from edge_cases import hostile_rays
    from nanort_b200 import api
    from oracle import orc

    for kind, n_inst in (("mixed", 12), ("hollow", 80)):
        from nanort_b200 import scenes as S

        insts = S.instances_mixed(n_inst) if kind == "mixed" else _hollow_instances(n_inst)
        port = orc.PortScene(insts, cpp11=True)
        sc = _gpu_scene(insts, api.BUILD_FAST, api.BUILD_FAST)
        top, ti = sc.GetTopLevel()
        lo, hi = _bounds(insts)
        rays = hostile_rays(lo - 1.0, hi + 1.0, n=40000, seed=23)
        gh, gm = sc.Traverse(rays)
        res, _ = classify_scene_hits(port, rays, gh, gm, top, ti, exact_rays=scene_handed_over_len(rays))
        assert res["hits"] > 1000, res
        print(kind, "hostile", res)


def test_host_chunking_equals_one_device_call():
    """nrt_scene_traverse moves rays through 2^20-ray chunks; 2^20 + 777 rays give the device entry's records"""
    import torch
    from nanort_b200 import api, scenes as S

    insts = S.instances_mixed()
    sc = _gpu_scene(insts, api.BUILD_FAST, api.BUILD_FAST)
    n = (1 << 20) + 777
    rays = _incoherent(insts, n, seed=29)
    rays["dir"][::5] *= np.float32(0.5)  # some rays through the list kernel in both chunks
    hh, hm = sc.Traverse(rays)
    d_rays = torch.from_numpy(rays.view(np.uint8).reshape(-1, 36)).cuda()
    d_hits = torch.full((n, 32), 0xFF, dtype=torch.uint8, device="cuda")
    d_mask = torch.full((n,), 0xFF, dtype=torch.uint8, device="cuda")
    sc.TraverseDevice(d_rays.data_ptr(), n, d_hits.data_ptr(), d_mask.data_ptr(),
                      stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert hm.sum() > 0.1 * n and hm[(1 << 20):].sum() > 50
    assert np.array_equal(d_mask.cpu().numpy(), hm)
    assert d_hits.cpu().numpy().tobytes() == hh.tobytes()


def _gated_launches(sc, d_rays, n, outs, streams, gate_cycles=50_000_000):
    """one TraverseDevice per stream, all held back by one event that a gate stream records after a spin, so the
    launches start together"""
    import torch

    gate = torch.cuda.Stream()
    with torch.cuda.stream(gate):
        torch.cuda._sleep(gate_cycles)
    ev = torch.cuda.Event()
    ev.record(gate)
    for s, (h, m) in zip(streams, outs):
        s.wait_event(ev)
        sc.TraverseDevice(d_rays.data_ptr(), n, h.data_ptr(), m.data_ptr(), stream=s.cuda_stream)


@pytest.mark.parametrize("handed_over", [False, True])
def test_concurrent_launches_on_eight_streams_equal_serial_ones(handed_over):
    """Eight nrt_scene_traverse_device calls in flight at once on eight streams (more than the scene's four scratch
    slots), 8 K rays / 64 CTAs each so that all of them are resident together: every output equals the single-stream
    records.  handed_over: |d| = 3, every ray goes through the overflow list to the list kernel."""
    import torch
    from nanort_b200 import api, scenes as S

    insts = S.instances_mixed()
    sc = _gpu_scene(insts, api.BUILD_FAST, api.BUILD_FAST)
    n = 8192
    lo, hi = _bounds(insts)
    rays = S.incoherent_rays(lo - 1.0, hi + 1.0, n, seed=31, axis_parallel_fraction=0.0)
    rays["min_t"] = 0.0
    if handed_over:
        rays["dir"] *= np.float32(3.0)
    assert scene_handed_over_len(rays).all() if handed_over else not scene_handed_over_len(rays).any()
    d_rays = torch.from_numpy(rays.view(np.uint8).reshape(-1, 36)).cuda()

    def fresh():
        return (torch.full((n, 32), 0xFF, dtype=torch.uint8, device="cuda"),
                torch.full((n,), 0xFF, dtype=torch.uint8, device="cuda"))

    want_h, want_m = fresh()
    sc.TraverseDevice(d_rays.data_ptr(), n, want_h.data_ptr(), want_m.data_ptr(),
                      stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert int(want_m.sum().item()) > 0.2 * n
    streams = [torch.cuda.Stream() for _ in range(8)]
    for rep in range(3):
        outs = [fresh() for _ in streams]
        torch.cuda.synchronize()
        _gated_launches(sc, d_rays, n, outs, streams)
        torch.cuda.synchronize()
        for k, (h, m) in enumerate(outs):
            assert torch.equal(m, want_m), (rep, k, int((m != want_m).sum().item()))
            assert torch.equal(h, want_h), (rep, k)


def test_scene_ao_passes_next_to_traversals_equal_serial_runs():
    """two scene AO passes on two streams from two host threads while traversals run on six more: both frames equal
    the frames of serial runs pixel for pixel"""
    import torch
    from nanort_b200 import api, scenes as S
    from test_gpu_scene import _ao_params

    insts = S.instances_mixed()
    sc = _gpu_scene(insts, api.BUILD_FAST, api.BUILD_FAST)
    W, H, spp = 256, 128, 2
    cams = [S.look_at((0.0, 12.0, 20.0), (0.0, 0.0, 0.0), aspect=W / H),
            S.look_at((14.0, 6.0, -12.0), (0.0, 0.0, 0.0), aspect=W / H)]
    params = [_ao_params(api, cam, W, H, spp, 3.0) for cam in cams]
    for p in params:
        p.ray_min_t = 0.0

    def render(p, stream=None):
        a = torch.zeros(W * H, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        r = sc.RenderAO(p, a.data_ptr(), stream=stream.cuda_stream if stream is not None else None)
        return a, r

    serial = [render(p) for p in params]
    torch.cuda.synchronize()
    n = 8192
    lo, hi = _bounds(insts)
    rays = S.incoherent_rays(lo - 1.0, hi + 1.0, n, seed=37, axis_parallel_fraction=0.0)
    rays["min_t"] = 0.0
    rays["dir"][::3] *= np.float32(0.5)
    d_rays = torch.from_numpy(rays.view(np.uint8).reshape(-1, 36)).cuda()
    want_h, want_m = sc.Traverse(rays)
    frames = [None, None]
    ao_streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    accs = [torch.zeros(W * H, dtype=torch.float32, device="cuda") for _ in params]
    torch.cuda.synchronize()

    def worker(k):
        frames[k] = sc.RenderAO(params[k], accs[k].data_ptr(), stream=ao_streams[k].cuda_stream)

    th = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    streams = [torch.cuda.Stream() for _ in range(6)]
    outs = [(torch.full((n, 32), 0xFF, dtype=torch.uint8, device="cuda"),
             torch.full((n,), 0xFF, dtype=torch.uint8, device="cuda")) for _ in streams]
    torch.cuda.synchronize()
    for t in th:
        t.start()
    for _ in range(4):
        _gated_launches(sc, d_rays, n, outs, streams, gate_cycles=5_000_000)
    for t in th:
        t.join()
    torch.cuda.synchronize()
    for k in range(2):
        assert torch.equal(accs[k], serial[k][0]), k
        assert (frames[k].primary_rays, frames[k].ao_rays, frames[k].ao_hits) == \
            (serial[k][1].primary_rays, serial[k][1].ao_rays, serial[k][1].ao_hits)
    for h, m in outs:
        assert np.array_equal(m.cpu().numpy(), want_m) and h.cpu().numpy().tobytes() == want_h.tobytes()
