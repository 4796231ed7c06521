"""Every instantiation of the float traversal kernels that a launcher can pick, compared with the oracle:

  * the 512-entry stack (tree depth + 2 > 64): synthetic "caterpillar" trees of depth 62 ... 500, reference-built
    trees of terrain(128) (depth 99) and of the 100 K-triangle sphere grid (depth 66), the primary + AO pass and the
    path tracer's launches on such trees, and the two-level scene walk with its 1024-entry stack;
  * the WideNode policies of the coherent launches (a PairNode array above 38 MiB): terrain(900), production- and
    reference-built;
  * the counting instantiation (CountDevice, LaneStatsDevice): its box and primitive counts are the reference's
    nodes popped and primitives tested.

Every test first asserts that its tree really selects the instantiation it is about, so that a builder change that
makes a tree shallower or smaller fails here instead of quietly testing the already-covered kernel."""
import numpy as np
import pytest

from helpers import assert_parity, compare_hits

pytestmark = pytest.mark.gpu

STACK_SMALL = 64             # traverse.cu: needs_deep_stack() picks 512 entries above this
PAIR128_MAX = 38 << 20       # traverse.cu: kPair128MaxBytes, coherent launches read WideNodes above it
PAIR_NODE_BYTES = 128
TRACE_OPTION_SETS = [None, dict(cull_back_face=1), dict(skip_prim_id=17), dict(prim_ids_range=(1000, 3000)),
                     dict(cull_back_face=1, prim_ids_range=(0, 2500), skip_prim_id=2001)]


def _deep(acc):
    return acc.GetStatistics()["max_tree_depth"] + 2 > STACK_SMALL


def _wide(acc):
    return acc.GetStatistics()["num_branch_nodes"] * PAIR_NODE_BYTES > PAIR128_MAX


def _topts(tkw):
    from oracle import orc

    return None if tkw is None else orc.trace_options(**tkw)


def _opts(tkw):
    from nanort_b200 import api

    return None if tkw is None else api.BVHTraceOptions(**tkw)


def _bits(h):
    return np.ascontiguousarray(h).view(np.uint32).reshape(len(h), -1)


def _d_rays(torch, rays):
    return torch.from_numpy(np.ascontiguousarray(rays).view(np.uint8).reshape(-1, 36).copy()).cuda()


def _device_hits(acc, rays, flags=0, options=None):
    import torch
    from nanort_b200 import scenes as S

    d_r = _d_rays(torch, rays)
    d_h = torch.empty(len(rays) * 16, dtype=torch.uint8, device="cuda")
    acc.TraverseDevice(d_r.data_ptr(), len(rays), d_h.data_ptr(), options=options, flags=flags)
    torch.cuda.synchronize()
    return d_h.cpu().numpy().view(S.HIT_DTYPE)


def _ray32(rays):
    r32 = np.ascontiguousarray(np.ascontiguousarray(rays).view(np.uint8).reshape(-1, 36)[:, :32])
    return r32.view(np.dtype((np.void, 32))).reshape(-1)


def _check_ray32(acc, rays, want_h, base=0):
    """NRT_TRAVERSE_RAY32, host and device forms: the records of the 36-byte call, bit for bit."""
    import torch
    from nanort_b200 import api, scenes as S

    from_host, m = acc.Traverse(_ray32(rays), flags=base | api.TRAVERSE_RAY32, mask=False)
    assert m is None and np.array_equal(_bits(from_host), _bits(want_h))
    d_r = torch.from_numpy(np.ascontiguousarray(_ray32(rays)).view(np.uint8).copy()).cuda()
    d_h = torch.empty(len(rays) * 16, dtype=torch.uint8, device="cuda")
    acc.TraverseDevice(d_r.data_ptr(), len(rays), d_h.data_ptr(), flags=base | api.TRAVERSE_RAY32)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(d_h.cpu().numpy().view(S.HIT_DTYPE)), _bits(want_h))


def _check_any_hit(acc, rays, ch, cm, base=0, max_retrace=200):
    """NRT_TRAVERSE_ANY_HIT: the same hit flags as the closest-hit call; a record that differs from the closest one is
    a genuine hit of its own triangle (re-traced alone with prim_ids_range, it gives the same record)."""
    from nanort_b200 import api

    ah, am = acc.Traverse(rays, flags=base | api.TRAVERSE_ANY_HIT)
    assert np.array_equal(am, cm)
    hit = cm.astype(bool)
    assert np.all(ah["prim_id"][~hit] == 0xFFFFFFFF)
    assert np.all(ah["t"][hit] >= ch["t"][hit]) and np.all(ah["t"][hit] < rays["max_t"][hit])
    other = np.flatnonzero(hit & (ah["prim_id"] != ch["prim_id"]))
    for i in other[:: max(1, len(other) // max_retrace)]:
        o = api.BVHTraceOptions(prim_ids_range=(int(ah["prim_id"][i]), int(ah["prim_id"][i]) + 1))
        h1, m1 = acc.Traverse(rays[i:i + 1], options=o, flags=base)
        assert m1[0] == 1 and _bits(h1).tolist() == _bits(ah[i:i + 1]).tolist(), i
    return len(other)


# ------------------------------------------------------------------ A. synthetic deep trees
def caterpillar(D):
    """A tree of depth D over D + 1 triangles: triangle i lies in the plane x = D - i + 1 (they overlap in y / z,
    odd ones wound the other way); branch 2i (axis 0) has the children (2i + 2, 2i + 1), leaf 2i + 1 holds triangle i
    and the last branch's deeper child, leaf 2D, holds triangle D.  Boxes are exact unions.  A ray going +x from x = 0
    descends into the nearer child at every level and pushes the leaf; a ray going -x meets triangle 0 first."""
    from oracle import orc

    n = D + 1
    x = (D - np.arange(n) + 1).astype(np.float32)
    tri = np.zeros((n, 3, 3), np.float32)
    tri[:, :, 0] = x[:, None]
    tri[:, 0, 1:], tri[:, 1, 1:], tri[:, 2, 1:] = (-4.0, -4.0), (8.0, -4.0), (-4.0, 8.0)
    tri[1::2, 1:3] = tri[1::2, 2:0:-1].copy()  # alternating winding
    v = tri.reshape(-1, 3)
    f = np.arange(3 * n, dtype=np.uint32).reshape(n, 3)
    lo, hi = tri.min(axis=1), tri.max(axis=1)
    nodes = np.zeros(2 * D + 1, orc.NODE_DTYPE)
    br = 2 * np.arange(D)
    nodes["flag"][br], nodes["axis"][br] = 0, 0
    nodes["data"][br, 0], nodes["data"][br, 1] = br + 2, br + 1
    # a branch holds triangles i..D: suffix min / max
    nodes["bmin"][br] = np.minimum.accumulate(lo[::-1], axis=0)[::-1][:D]
    nodes["bmax"][br] = np.maximum.accumulate(hi[::-1], axis=0)[::-1][:D]
    lf = np.concatenate([br + 1, [2 * D]])
    nodes["flag"][lf] = 1
    # children cover adjacent index ranges, the deeper one first (as the reference's builder lays them out)
    nodes["data"][lf, 0], nodes["data"][lf, 1] = 1, D - np.arange(n)
    nodes["bmin"][lf], nodes["bmax"][lf] = lo, hi
    return v, f, nodes, np.ascontiguousarray(np.arange(n, dtype=np.uint32)[::-1])


def caterpillar_rays(D, n=1024, seed=3):
    """+x rays from x = 0 (jittered, some exactly axis-parallel with a -0.0 component: the two inverse conventions
    differ there), the same rays ending at max_t = 0.5 (before every triangle), and -x rays from x = D + 3."""
    from nanort_b200 import scenes as S

    k = np.arange(n)
    yz = np.stack([1.8 * S.rand01(k, 0, seed) - 0.9, 1.8 * S.rand01(k, 1, seed) - 0.9], axis=1)
    jit = 2e-3 * (np.stack([S.rand01(k, 2, seed), S.rand01(k, 3, seed)], axis=1) - 0.5)
    d = np.concatenate([np.ones((n, 1)), jit], axis=1)
    d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    d[: n // 8] = (1.0, 0.0, 0.0)
    d[: n // 16, 1] = -0.0
    fwd = np.zeros(n, S.RAY_DTYPE)
    fwd["org"][:, 1:] = yz
    fwd["dir"], fwd["min_t"], fwd["max_t"] = d, 0.0, 1e30
    short = fwd.copy()
    short["max_t"] = 0.5
    back = fwd.copy()
    back["org"][:, 0] = D + 3
    back["dir"][:, 0] = -back["dir"][:, 0]
    return np.concatenate([fwd, short, back])


def _caterpillar_options(D):
    # reject the nearest triangles: the walk unwinds through that many stack entries before it finds a hit
    return [None, dict(prim_ids_range=(0, D - 9)), dict(skip_prim_id=D), dict(cull_back_face=1),
            dict(prim_ids_range=(0, D // 2), cull_back_face=1)]


@pytest.mark.parametrize("D", [62, 63, 200, 500])
def test_caterpillar_fast_conformance_and_oracle_are_bit_identical(port, D):
    from nanort_b200 import api

    v, f, nodes, idx = caterpillar(D)
    acc = api.BVHAccel()
    acc.Adopt(nodes, idx, v, f)
    assert acc.GetStatistics()["max_tree_depth"] == D
    assert _deep(acc) == (D >= 63)
    rays = caterpillar_rays(D)
    n = len(rays) // 3
    for cpp11 in (True, False):
        base = 0 if cpp11 else api.TRAVERSE_CPP03_INVERSE
        for tkw in _caterpillar_options(D):
            want_h, want_m, ctr = port.traverse(nodes, idx, v, f, rays, topts=_topts(tkw), cpp11=cpp11, counters=True)
            # the construction does what it promises; the first n / 16 rays have a -0.0 direction component, whose
            # inverse is -inf in the C++11 convention: those rays miss every box there (the reference's behaviour)
            z = n // 16
            if tkw is None:
                assert ctr["max_stack"] == D
                assert np.all(want_m[z:n] == 1) and np.all(want_h["prim_id"][z:n] == D) and np.all(want_m[n:2 * n] == 0)
                assert np.all(want_m[:z] == (0 if cpp11 else 1)) and np.all(want_h["prim_id"][2 * n:] == 0)
            if tkw == dict(prim_ids_range=(0, D - 9)):
                assert np.all(want_h["prim_id"][z:n] == D - 10)
            hit = want_m.astype(bool)
            fast_h, fast_m = acc.Traverse(rays, options=_opts(tkw), flags=base)
            conf_h, conf_m = acc.Traverse(rays, options=_opts(tkw), flags=base | api.TRAVERSE_CONFORMANCE)
            # the triangles lie at distinct x: no ties, so every record is bit-identical, misses included
            assert np.array_equal(fast_m, want_m) and np.array_equal(conf_m, want_m), (cpp11, tkw)
            assert np.array_equal(_bits(fast_h[hit]), _bits(want_h[hit])), (cpp11, tkw)
            assert np.array_equal(_bits(fast_h), _bits(conf_h)), (cpp11, tkw)
        # the other calls of the same kernel
        want_h, want_m = acc.Traverse(rays, flags=base)
        assert np.array_equal(_bits(_device_hits(acc, rays, flags=base)), _bits(want_h))
        _check_ray32(acc, rays, want_h, base)
        _check_any_hit(acc, rays, want_h, want_m, base)
        for lo, cnt in ((0, 1), (5, 33), (n - 20, 64), (2 * n + 7, 64)):  # <= 64 rays: the zero-copy path
            h, m = acc.Traverse(rays[lo:lo + cnt], flags=base)
            assert np.array_equal(m, want_m[lo:lo + cnt]) and np.array_equal(_bits(h), _bits(want_h[lo:lo + cnt]))


def test_caterpillar_deeper_than_500_is_refused():
    from nanort_b200 import api

    v, f, nodes, idx = caterpillar(501)
    with pytest.raises(api.NanortB200Error, match="deeper than 500"):
        api.BVHAccel().Adopt(nodes, idx, v, f)


# ------------------------------------------------------------------ B. reference-shaped deep trees
def _reference_shaped(port, name):
    """(acc, nodes, indices, verts, faces, scene name) of a deep tree the reference's builder shapes."""
    from nanort_b200 import api, scenes as S

    if name == "bench_ref":
        v, f = S.make_scene("sphere_grid")
        scene = "sphere_grid"
    else:
        v, f = S.make_scene("terrain", n=128)
        scene = "terrain"
    acc = api.BVHAccel()
    if name == "terrain128_adopted":
        nodes, idx, _ = port.build(v, f)
        acc.Adopt(nodes, idx, v, f)
    else:
        flags = api.BUILD_REFERENCE_TREE | (api.BUILD_REFERENCE_CPP03_ORDER if name == "terrain128_ref03" else 0)
        acc.Build(len(f), v, f, flags=flags)
        nodes, idx = acc.GetNodes(), acc.GetIndices()
    return acc, nodes, idx, v, f, scene


def _scene_rays(S, scene, v, W=160, H=96, n_inc=20000):
    from edge_cases import hostile_rays

    bmin, bmax = v.min(axis=0), v.max(axis=0)
    return np.concatenate([S.primary_rays(S.scene_camera(scene, W, H), W, H, spp=1, seed=9),
                           S.incoherent_rays(bmin, bmax, n_inc, seed=10), hostile_rays(bmin, bmax)])


@pytest.mark.parametrize("name", ["terrain128_ref", "terrain128_ref03", "terrain128_adopted", "bench_ref"])
def test_reference_shaped_deep_tree_fast_kernel_matches_oracle(port, name):
    from nanort_b200 import api, scenes as S

    acc, nodes, idx, v, f, scene = _reference_shaped(port, name)
    depth = acc.GetStatistics()["max_tree_depth"]
    assert _deep(acc), depth
    assert depth >= (66 if name == "bench_ref" else 90), depth
    rays = _scene_rays(S, scene, v)
    option_sets = TRACE_OPTION_SETS if name != "bench_ref" else TRACE_OPTION_SETS[:2]
    for cpp11 in (True, False):
        base = 0 if cpp11 else api.TRAVERSE_CPP03_INVERSE
        for tkw in option_sets:
            t = _topts(tkw)
            want_h, want_m = port.traverse(nodes, idx, v, f, rays, topts=t, cpp11=cpp11, threads=8)
            got_h, got_m = acc.Traverse(rays, options=_opts(tkw), flags=base)
            assert_parity(compare_hits(port, v, f, rays, got_h, got_m, want_h, want_m, topts=t, cpp11=cpp11))
        got_h, got_m = acc.Traverse(rays, flags=base)
        _check_ray32(acc, rays, got_h, base)
        _check_any_hit(acc, rays, got_h, got_m, base)


# ------------------------------------------------------------------ C. passes and scenes on deep trees
def _ao_params(api, S, scene, W, H, spp, bbox, flags=0):
    cam = S.scene_camera(scene, W, H)
    p = api.AoParams()
    for i in range(12):
        p.cam[i] = float(cam[i])
    p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, 0, 1
    p.tile_w, p.tile_h, p.shard, p.n_shards = 64, 8, 0, 1
    p.ray_min_t, p.ray_max_t, p.ao_min_t, p.ao_max_t = 1e-3, 1e30, 1e-3, 0.25 * float(np.linalg.norm(bbox[1] - bbox[0]))
    p.flags = flags
    return p, cam


def _render(torch, acc, p, W, H):
    accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r = acc.RenderAO(p, accum.data_ptr())
    return accum.cpu().numpy(), (r.primary_rays, r.ao_rays, r.ao_hits)


def _ao_pass_matches_oracle(port, acc, v, f, scene, W, H, spp, oracle_stride=1):
    """The primary + AO pass on `acc`: fused == AO_UNFUSED == ANY_HIT frames bit for bit with equal counts; both
    exported ray queues hit what the oracle finds walking the same arrays; frame.sum() == primary - occluded."""
    import torch
    from nanort_b200 import api, dist as nd, scenes as S

    bbox = acc.BoundingBox()
    frames, results = [], []
    for flags in (0, api.AO_UNFUSED, api.TRAVERSE_ANY_HIT):
        p, _ = _ao_params(api, S, scene, W, H, spp, bbox, flags=flags)
        fr, res = _render(torch, acc, p, W, H)
        frames.append(fr)
        results.append(res)
    assert results[0] == results[1] == results[2] and results[0][0] == W * H * spp and results[0][2] > 0
    assert np.array_equal(frames[0], frames[1]) and np.array_equal(frames[0], frames[2])

    p, _ = _ao_params(api, S, scene, W, H, spp, bbox)
    pix, _ = nd.slot_pixels(W, H, 64, 8, 0, 1, spp)
    n_slots = len(pix)
    d_p = torch.empty(n_slots * 36, dtype=torch.uint8, device="cuda")
    d_a = torch.empty(n_slots * 36, dtype=torch.uint8, device="cuda")
    accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    n_p, n_a = acc.ExportAOWorkload(p, accum.data_ptr(), d_p.data_ptr(), d_a.data_ptr())
    assert n_p == W * H * spp == int((pix >= 0).sum()) and n_a == results[0][1]
    assert np.array_equal(accum.cpu().numpy(), frames[0])
    nodes, idx = acc.GetNodes(), acc.GetIndices()
    prim = d_p.cpu().numpy().view(S.RAY_DTYPE)[pix >= 0]  # the queue is in tile order; padding slots hold no ray
    ao = d_a[: n_a * 36].cpu().numpy().view(S.RAY_DTYPE)
    occluded = 0
    for rays in (prim, ao):
        got_h, got_m = acc.Traverse(rays)
        sel = np.arange(0, len(rays), oracle_stride)
        want_h, want_m = port.traverse(nodes, idx, v, f, rays[sel], threads=8)
        assert_parity(compare_hits(port, v, f, rays[sel], got_h[sel], got_m[sel], want_h, want_m), max_near_ties=8)
        occluded = int(got_m.sum())
    assert int((acc.Traverse(prim)[1]).sum()) == n_a, "one AO ray per primary hit"
    assert occluded == results[0][2]
    assert float(frames[0].astype(np.float64).sum()) == float(n_p - occluded)


def test_ao_pass_on_the_reference_built_bench_scene(port):
    """The fused camera and AO launches at 512 entries (CameraPolicy, IncoherentPolicy, their ANY_HIT forms)."""
    from nanort_b200 import api, scenes as S

    v, f = S.make_scene("sphere_grid")
    acc = api.BVHAccel()
    acc.Build(len(f), v, f, flags=api.BUILD_REFERENCE_TREE)
    assert _deep(acc) and not _wide(acc)
    _ao_pass_matches_oracle(port, acc, v, f, "sphere_grid", 200, 104, 3)


def test_fused_ao_frame_of_several_waves_equals_the_unfused_frame():
    """1920x1080x9 camera rays are more than one 16 Mi-ray wave: the fused pass carries its queues across waves."""
    import torch
    from nanort_b200 import api, scenes as S

    W, H, spp = 1920, 1080, 9
    assert W * H * spp > 1 << 24
    v, f = S.make_scene("sphere_grid")
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    bbox = acc.BoundingBox()
    out = []
    for flags in (0, api.AO_UNFUSED):
        p, _ = _ao_params(api, S, "sphere_grid", W, H, spp, bbox, flags=flags)
        out.append(_render(torch, acc, p, W, H))
    assert out[0][1] == out[1][1] and out[0][1][0] == W * H * spp
    assert np.array_equal(out[0][0], out[1][0])
    assert float(out[0][0].astype(np.float64).sum()) == float(out[0][1][0] - out[0][1][2])


def _deep_scene_instances():
    from nanort_b200 import scenes as S

    v, f = S.make_scene("terrain", n=128)
    return [(v, f, S.xform()),
            (v, f, S.xform(translate=(12.0, 0.5, 0.0), yaw=0.7)),
            (v, f, S.xform(translate=(0.0, -1.0, 12.0), scale=(1.5, 0.6, 0.8), pitch=0.3)),
            (v, f, S.xform(translate=(-12.0, 0.0, 3.0), scale=(-1.0, 1.0, 1.0))),       # mirrored
            (v, f, S.xform(translate=(4.0, 3.0, -10.0), scale=(0.7, -1.3, 1.1), yaw=-1.1, pitch=0.5))]


def _tree_depth(nodes):
    depth = np.zeros(len(nodes), np.int64)
    for i in np.flatnonzero(nodes["flag"] == 0):
        depth[nodes["data"][i]] = depth[i] + 1
    return int(depth.max())


def test_scene_with_deep_instances_matches_the_oracle_scene():
    """BLAS built by the reference-exact builder (depth 99) under rotated, non-uniformly scaled and mirrored
    transforms: the two-level walk needs more than 64 entries and runs scene_unified_kernel<1024, 2>."""
    import torch
    from nanort_b200 import api, scenes as S
    from oracle import orc
    from test_gpu_scene import _gpu_scene, _rays_for, _same_bits

    insts = _deep_scene_instances()
    port = orc.PortScene(insts, cpp11=True)
    for top in (api.BUILD_FAST, api.BUILD_REFERENCE_TREE):
        sc = _gpu_scene(insts, api.BUILD_REFERENCE_TREE, top)
        blas = api.BVHAccel()
        blas.Build(len(insts[0][1]), insts[0][0], insts[0][1], flags=api.BUILD_REFERENCE_TREE)
        need = _tree_depth(sc.GetTopLevel()[0]) + blas.GetStatistics()["max_tree_depth"] + 6
        assert STACK_SMALL < need <= 1024, need
        rays = _rays_for(insts, 100000, seed=21)
        ph, pm = port.traverse(rays, threads=8)
        gh, gm = sc.Traverse(rays)
        assert pm.sum() > 2000
        assert np.array_equal(pm, gm)
        hit = pm == 1
        same_pick = hit & (ph["node_id"] == gh["node_id"]) & (ph["prim_id"] == gh["prim_id"])
        assert _same_bits(ph[same_pick], gh[same_pick])
        other = hit & ~same_pick
        assert other.sum() <= 0.005 * hit.sum()  # shared edges of the heightfield: equal distances only
        if other.any():
            rel = np.abs(ph["t"][other] - gh["t"][other]) / np.maximum(ph["t"][other], 1e-6)
            assert rel.max() <= 1e-5
        if top == api.BUILD_REFERENCE_TREE:
            ch, cm = sc.Traverse(rays, flags=api.TRAVERSE_CONFORMANCE)
            assert np.array_equal(pm, cm) and _same_bits(ph[hit], ch[cm == 1])

    # the pass over the scene: production walk against the conformance (list) walk
    from test_gpu_scene import _ao_params as scene_ao_params

    W, H, spp, radius = 256, 144, 2, 3.0
    cam = S.look_at((0.0, 14.0, 26.0), (0.0, 0.0, 0.0), aspect=W / H)
    frames = []
    for flags in (0, api.TRAVERSE_CONFORMANCE):
        p = scene_ao_params(api, cam, W, H, spp, radius)
        p.flags = flags
        a = torch.zeros(W * H, dtype=torch.float32, device="cuda")
        r = sc.RenderAO(p, a.data_ptr())
        assert r.primary_rays == W * H * spp and 0 < r.ao_hits < r.ao_rays
        assert float(a.double().sum().item()) == float(r.primary_rays - r.ao_hits)
        frames.append((a, r))
    (a0, r0), (a1, r1) = frames
    assert abs(int(r0.ao_rays) - int(r1.ao_rays)) <= 4
    assert float((a0 != a1).double().mean().item()) < 1e-3


# ------------------------------------------------------------------ D. WideNode launches past the 38 MiB cut-off
def _large_tree_checks(port, acc, v, f, W=1920, H=1080, n_inc=1_000_000):
    """Fast == conformance on every ray (differences only as classified ties), a strided oracle sample over the same
    arrays, RAY32, ANY_HIT, the fused AO frame == AO_UNFUSED, and the visit counters on a sample."""
    import torch
    from nanort_b200 import api, scenes as S

    rays = np.concatenate([S.primary_rays(S.scene_camera("terrain", W, H), W, H, spp=1, seed=5),
                           S.incoherent_rays(v.min(axis=0), v.max(axis=0), n_inc, seed=6)])
    n = len(rays)
    fast = _device_hits(acc, rays)
    conf = _device_hits(acc, rays, flags=api.TRAVERSE_CONFORMANCE)
    diff = np.flatnonzero((_bits(fast) != _bits(conf)).any(axis=1))
    assert len(diff) <= 2e-5 * n, len(diff)
    mask = (fast["prim_id"] != 0xFFFFFFFF).astype(np.uint8)
    assert mask.mean() > 0.3
    nodes, idx = acc.GetNodes(), acc.GetIndices()
    sel = np.unique(np.concatenate([np.arange(0, n, 97), diff]))
    want_h, want_m = port.traverse(nodes, idx, v, f, rays[sel], threads=32)
    assert_parity(compare_hits(port, v, f, rays[sel], fast[sel], mask[sel], want_h, want_m), max_near_ties=8)

    head = rays[: 1 << 18]
    ch, cm = acc.Traverse(head)
    assert np.array_equal(_bits(ch), _bits(fast[: len(head)]))
    _check_ray32(acc, head, ch)
    _check_any_hit(acc, head, ch, cm)

    bbox = acc.BoundingBox()
    out = []
    for flags in (0, api.AO_UNFUSED):
        p, _ = _ao_params(api, S, "terrain", 640, 360, 2, bbox, flags=flags)
        out.append(_render(torch, acc, p, 640, 360))
    assert out[0][1] == out[1][1] and out[0][1][2] > 0
    assert np.array_equal(out[0][0], out[1][0])

    _fast_counts_match_oracle(port, acc, nodes, idx, v, f, rays[:: max(1, n // 30000)])


@pytest.fixture(scope="module")
def terrain900():
    from nanort_b200 import scenes as S

    v, f = S.make_scene("terrain", n=900)
    assert len(f) == 1_620_000
    return v, f


def test_widenode_coherent_launches_on_the_production_tree(port, terrain900):
    """1.62 M triangles: the PairNode array is past the cut-off, so caller rays run IncoherentPolicy and the camera
    launch IncoherentCameraPolicy, both at 64 entries."""
    from nanort_b200 import api

    v, f = terrain900
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    st = acc.GetStatistics()
    assert st["num_branch_nodes"] * PAIR_NODE_BYTES > 55e6, st  # about 0.297 branches per triangle
    assert _wide(acc) and not _deep(acc)
    _large_tree_checks(port, acc, v, f)


def test_widenode_coherent_launches_on_the_reference_built_tree(port, terrain900):
    """The same mesh from the reference-exact builder: deep AND past the cut-off, i.e. <AosRays, 512,
    IncoherentPolicy> and <CameraRays, 512, IncoherentCameraPolicy>."""
    from nanort_b200 import api

    v, f = terrain900
    acc = api.BVHAccel()
    acc.Build(len(f), v, f, flags=api.BUILD_REFERENCE_TREE)
    assert _wide(acc) and _deep(acc), acc.GetStatistics()
    _large_tree_checks(port, acc, v, f, n_inc=400_000)


# ------------------------------------------------------------------ E. visit counters
def _count(acc, rays, tkw=None, flags=0):
    import torch

    d_r = _d_rays(torch, rays)
    return acc.CountDevice(d_r.data_ptr(), len(rays), options=_opts(tkw), flags=flags)


def _oracle_count(port, nodes, idx, v, f, rays, tkw=None, cpp11=True):
    h, m, c = port.traverse(nodes, idx, v, f, rays, topts=_topts(tkw), cpp11=cpp11, threads=8, counters=True)
    return h, m, (c["nodes_popped"], c["prims_tested"])


def _fast_counts_match_oracle(port, acc, nodes, idx, v, f, rays, tkw=None, cpp11=True):
    """The fast kernel visits in distance order, so its counts equal the reference's only where the visit set does not
    depend on the order: on rays that miss, and on hit rays re-cast with max_t = the closest hit's t.  Rays with a
    non-finite origin or direction, a zero direction, or an origin so far out (1e30) that the edge functions overflow
    are left out: they can accept a triangle at t = NaN, which ends the reference's walk wherever its order first meets
    such a triangle (the conformance counts include them)."""
    from nanort_b200 import api

    base = 0 if cpp11 else api.TRAVERSE_CPP03_INVERSE
    d = rays["dir"]
    rays = rays[(np.abs(rays["org"]) < 1e20).all(axis=1) & np.isfinite(d).all(axis=1) & (np.abs(d).max(axis=1) > 0)]
    h, m, _ = _oracle_count(port, nodes, idx, v, f, rays, tkw, cpp11)
    miss = rays[m == 0]
    assert _count(acc, miss, tkw, base) == _oracle_count(port, nodes, idx, v, f, miss, tkw, cpp11)[2]
    hit = rays[m == 1].copy()
    hit["max_t"] = h["t"][m == 1]
    assert _count(acc, hit, tkw, base) == _oracle_count(port, nodes, idx, v, f, hit, tkw, cpp11)[2]
    return len(miss), len(hit)


def _count_case(port, name):
    from nanort_b200 import api, scenes as S

    acc = api.BVHAccel()
    if name == "single_leaf":
        v = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 1]])
        f = np.uint32([[0, 1, 2], [0, 3, 1], [2, 3, 4]])
        acc.Build(len(f), v, f)
        assert acc.GetStatistics()["num_branch_nodes"] == 0
        nodes, idx = acc.GetNodes(), acc.GetIndices()
    elif name.startswith("caterpillar"):
        v, f, nodes, idx = caterpillar(int(name[len("caterpillar"):]))
        acc.Adopt(nodes, idx, v, f)
    elif name == "cornell_built":
        v, f = S.make_scene("cornell")
        acc.Build(len(f), v, f)
        nodes, idx = acc.GetNodes(), acc.GetIndices()
    elif name == "sphere_grid_adopted":
        v, f = S.make_scene("sphere_grid", nx=3, nz=3)
        nodes, idx, _ = port.build(v, f)
        acc.Adopt(nodes, idx, v, f)
    else:
        acc, nodes, idx, v, f, _ = _reference_shaped(port, "terrain128_ref")
    from edge_cases import hostile_rays

    bmin, bmax = v.min(axis=0), v.max(axis=0)
    pad = 0.5 * (bmax - bmin) + 0.5
    rays = np.concatenate([S.incoherent_rays(bmin - pad, bmax + pad, 12000, seed=31),  # many miss the root box
                           hostile_rays(bmin, bmax, 4000, seed=32)])
    if name.startswith("caterpillar"):
        rays = np.concatenate([rays, caterpillar_rays(len(f) - 1, n=512)])
    return acc, nodes, idx, v, f, rays


COUNT_CASES = ["single_leaf", "cornell_built", "sphere_grid_adopted", "caterpillar62", "caterpillar200",
               "terrain128_ref"]


@pytest.mark.parametrize("name", COUNT_CASES)
def test_conformance_counts_equal_the_oracle(port, name):
    """CountDevice over the conformance walk == the reference's (nodes popped, primitives tested), every ray counted,
    NaN ranges and rays that miss the root box included."""
    from nanort_b200 import api

    acc, nodes, idx, v, f, rays = _count_case(port, name)
    assert np.isnan(rays["min_t"]).any() and np.isnan(rays["max_t"]).any()
    for cpp11 in (True, False):
        flags = api.TRAVERSE_CONFORMANCE | (0 if cpp11 else api.TRAVERSE_CPP03_INVERSE)
        for tkw in (None, dict(cull_back_face=1, prim_ids_range=(0, max(1, len(f) // 2)), skip_prim_id=1)):
            want = _oracle_count(port, nodes, idx, v, f, rays, tkw, cpp11)[2]
            assert _count(acc, rays, tkw, flags) == want, (cpp11, tkw)


@pytest.mark.parametrize("name", COUNT_CASES)
def test_fast_counts_equal_the_oracle_where_the_visit_set_is_fixed(port, name):
    acc, nodes, idx, v, f, rays = _count_case(port, name)
    assert _deep(acc) == (name in ("caterpillar200", "terrain128_ref"))
    for cpp11 in (True, False):
        n_miss, n_hit = _fast_counts_match_oracle(port, acc, nodes, idx, v, f, rays, cpp11=cpp11)
        assert n_miss > 1000 and n_hit > 20, (n_miss, n_hit)
    _fast_counts_match_oracle(port, acc, nodes, idx, v, f, rays, tkw=dict(cull_back_face=1, skip_prim_id=0))


@pytest.mark.parametrize("name", ["cornell_built", "caterpillar200", "terrain128_ref"])
def test_lane_stats_invariants(port, name):
    """Within one call: every ray retires once, every box counted is the root's or one of a tested pair's two, and
    every ray was handed to a lane."""
    import torch

    acc, nodes, idx, v, f, rays = _count_case(port, name)
    d_r = _d_rays(torch, rays)
    n = len(rays)
    s = acc.LaneStatsDevice(d_r.data_ptr(), n)
    assert s["lanes_retired"] == n, s
    assert s["boxes"] == n + 2 * s["lanes_testing"], s
    assert s["lanes_refilled"] >= n, s
    assert (s["boxes"], s["prims"]) == acc.CountDevice(d_r.data_ptr(), n)
