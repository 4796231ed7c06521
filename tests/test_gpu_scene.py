"""Two-level scene (instancing) on the GPU against the oracle's restatement of examples/nanosg (which
tests/test_oracle_scene.py pins bit-for-bit to the unmodified reference):
  * instance state (matrices, inverse, world boxes) bit-equal,
  * conformance commit: top-level tree bit-equal,
  * conformance traversal: every record bit-equal,
  * fast traversal: same hit mask; records bit-equal where the same (instance, triangle) is picked, and a different
    pick only at an exact tie or by a parameter-versus-distance cull (tests/test_gpu_scene_exact.py goes further),
  * the 64-box limit and the flattened-scene cross-check."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _rays_for(insts, n, seed):
    from nanort_b200 import scenes as S

    lo = np.min([np.min(v @ x[:3, :3] + x[3, :3], axis=0) for v, f, x in insts], axis=0)
    hi = np.max([np.max(v @ x[:3, :3] + x[3, :3], axis=0) for v, f, x in insts], axis=0)
    pad = 0.25 * (hi - lo) + 0.5
    rays = S.incoherent_rays(lo - pad, hi + pad, n, seed=seed)
    rays["min_t"] = 0.0
    return rays


def _row_rays(rays):
    from nanort_b200 import scenes as S

    k = np.arange(2000)
    rays["org"][:2000] = np.stack([-3.0 - 0.01 * (k % 7), 0.3 * S.rand01(k, 0, 9) - 0.15,
                                   0.3 * S.rand01(k, 1, 9) - 0.15], axis=1)
    d = np.stack([np.ones(2000), 0.002 * (S.rand01(k, 2, 9) - 0.5), 0.002 * (S.rand01(k, 3, 9) - 0.5)], axis=1)
    rays["dir"][:2000] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    rays["dir"][:50, 1:] = 0.0
    rays["dir"][:50, 0] = 1.0
    rays["max_t"][:2000] = 1e30
    return rays


def _gpu_scene(insts, build_flags, commit_flags):
    from nanort_b200 import api

    accels = {}
    sc = api.Scene()
    for v, f, x in insts:
        key = (v.ctypes.data, f.ctypes.data)
        if key not in accels:
            a = api.BVHAccel()
            a.Build(len(f), v, f, flags=build_flags)
            accels[key] = a
        sc.AddNode(accels[key], x)
    assert sc.Commit(commit_flags)
    return sc


def _same_bits(a, b):
    return a.tobytes() == b.tobytes()


def _same_tree(a, b):
    br = a["flag"] == 0
    return (len(a) == len(b) and all(_same_bits(a[k], b[k]) for k in ("bmin", "bmax", "flag", "data"))
            and np.array_equal(a["axis"][br], b["axis"][br]))


@pytest.mark.parametrize("kind", ["mixed", "row"])
def test_conformance_scene_is_bit_exact(kind):
    from nanort_b200 import api, scenes as S
    from oracle import orc

    insts = S.instances_mixed() if kind == "mixed" else S.instances_row()
    port = orc.PortScene(insts, cpp11=True)
    sc = _gpu_scene(insts, api.BUILD_REFERENCE_TREE, api.BUILD_REFERENCE_TREE)
    st = sc.InstanceStates()
    for name in st.dtype.names:
        assert _same_bits(st[name], port.sg[name]), name
    tn, ti = sc.GetTopLevel()
    assert _same_tree(port.top, tn) and _same_bits(port.top_idx, ti)
    assert _same_bits(np.concatenate(sc.GetBoundingBox()), np.concatenate([port.top["bmin"][0], port.top["bmax"][0]]))
    rays = _rays_for(insts, 60000, seed=5)
    if kind == "row":
        rays = _row_rays(rays)
    ph, pm = port.traverse(rays, threads=8)
    gh, gm = sc.Traverse(rays, flags=api.TRAVERSE_CONFORMANCE)
    assert pm.sum() > 1000
    assert np.array_equal(pm, gm)
    assert _same_bits(ph[pm == 1], gh[gm == 1])
    miss = gm == 0
    assert np.all(gh["prim_id"][miss] == 0xFFFFFFFF) and np.all(gh["node_id"][miss] == 0xFFFFFFFF)


@pytest.mark.parametrize("kind,top_flags", [("mixed", "fast"), ("row", "fast"), ("mixed", "ref")])
def test_fast_scene_matches_reference_up_to_equal_distance_ties(kind, top_flags):
    from helpers import classify_scene_hits, scene_handed_over_len
    from nanort_b200 import api, scenes as S
    from oracle import orc

    insts = S.instances_mixed() if kind == "mixed" else S.instances_row()
    port = orc.PortScene(insts, cpp11=True)
    sc = _gpu_scene(insts, api.BUILD_FAST, api.BUILD_FAST if top_flags == "fast" else api.BUILD_REFERENCE_TREE)
    rays = _rays_for(insts, 200000, seed=6)
    if kind == "row":
        rays = _row_rays(rays)
    gh, gm = sc.Traverse(rays)
    top, ti = sc.GetTopLevel()
    # a different pick only at an exact tie of t or by a parameter-versus-distance cull (helpers.classify_scene_hits)
    res, _ = classify_scene_hits(port, rays, gh, gm, top, ti, exact_rays=scene_handed_over_len(rays))
    assert res["hits"] > 1000, res


def test_two_level_equals_flattened_scene():
    """Pure translations: the instanced grid and the same triangles flattened into one soup must see the same
    surfaces (t up to the rounding of the transform, same triangle)."""
    from nanort_b200 import api, scenes as S

    base = S.sphere_grid(nx=3, nz=3)
    insts = S.instances_grid(4, 3, base=base)
    sc = _gpu_scene(insts, api.BUILD_FAST, api.BUILD_FAST)
    vs = np.concatenate([v + x[3, :3] for v, f, x in insts]).astype(np.float32)
    fs = np.concatenate([f + np.uint32(i * len(base[0])) for i, (v, f, x) in enumerate(insts)]).astype(np.uint32)
    flat = api.BVHAccel()
    flat.Build(len(fs), vs, fs)
    cam = S.look_at((0.0, 14.0, 30.0), (0.0, 0.0, 0.0), aspect=16 / 9)
    rays = S.primary_rays(cam, 640, 360, spp=1, seed=3, min_t=0.0)
    fh, fm = flat.Traverse(rays)
    gh, gm = sc.Traverse(rays)
    assert fm.sum() > 0.05 * len(rays)
    agree = fm == gm
    assert agree.mean() > 0.9999
    both = (fm == 1) & (gm == 1)
    nf = len(base[1])
    same = (gh["node_id"][both] * nf + gh["prim_id"][both]) == fh["prim_id"][both]
    assert same.mean() > 0.999
    dt = np.abs(gh["t"][both][same] - fh["t"][both][same]) / fh["t"][both][same]
    assert dt.max() < 1e-4


def test_device_pointer_scene_traverse_and_empty_commit():
    import torch
    from nanort_b200 import api, scenes as S

    assert api.Scene().Commit() is False  # nanosg.h:708-711
    insts = S.instances_mixed(9)
    sc = _gpu_scene(insts, api.BUILD_FAST, api.BUILD_FAST)
    rays = _rays_for(insts, 50000, seed=12)
    hh, hm = sc.Traverse(rays)
    d_rays = torch.from_numpy(rays.view(np.uint8).reshape(-1, 36)).cuda()
    d_hits = torch.zeros(len(rays), 32, dtype=torch.uint8, device="cuda")
    d_mask = torch.zeros(len(rays), dtype=torch.uint8, device="cuda")
    sc.TraverseDevice(d_rays.data_ptr(), len(rays), d_hits.data_ptr(), d_mask.data_ptr(),
                      stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(d_mask.cpu().numpy(), hm)
    assert d_hits.cpu().numpy().tobytes() == hh.tobytes()


def _ao_params(api, cam, W, H, spp, radius, shard=0, n_shards=1):
    p = api.AoParams()
    for i in range(12):
        p.cam[i] = float(cam[i])
    p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, 0, 1
    p.tile_w, p.tile_h, p.shard, p.n_shards = 64, 8, shard, n_shards
    p.ray_min_t, p.ray_max_t, p.ao_min_t, p.ao_max_t = 1e-3, 1e30, 1e-3, radius
    p.flags = 0
    return p


def test_scene_ao_pass_against_the_flattened_scene():
    """nrt_scene_render_ao_device: the wavefront primary + AO pass with Scene::Traverse as its traversal step.  Against the
    same triangles flattened into one soup and rendered by nrt_render_ao_device: the same camera rays hit the same
    surfaces (primary hit counts equal up to grazing rays), frame.sum() == primary - occluded exactly, and the
    visibility images agree (the scene pass lifts the AO origin by ao_min_t along the normal and works in world space,
    so pixels may differ by a sample here and there, not systematically); tile shards add up to the whole frame."""
    import torch
    from nanort_b200 import api, scenes as S

    base = S.sphere_grid(nx=3, nz=3)
    insts = [(base[0], base[1], S.xform(translate=(-6.0, 0.0, 0.0))),
             (base[0], base[1], S.xform(translate=(6.0, 0.5, 1.0), yaw=0.6)),
             (base[0], base[1], S.xform(translate=(0.0, 0.0, -9.0), scale=(1.5, 1.0, 0.75), pitch=0.2))]
    sc = _gpu_scene(insts, api.BUILD_FAST, api.BUILD_FAST)
    vs, fs = [], []
    for i, (v, f, x) in enumerate(insts):
        x64 = x.astype(np.float64)
        vs.append((v.astype(np.float64) @ x64[:3, :3] + x64[3, :3]).astype(np.float32))
        fs.append(f + np.uint32(i * len(v)))
    vs, fs = np.concatenate(vs), np.concatenate(fs).astype(np.uint32)
    flat = api.BVHAccel()
    flat.Build(len(fs), vs, fs)
    W, H, spp = 320, 176, 4
    cam = S.look_at((0.0, 12.0, 26.0), (0.0, 0.0, -2.0), aspect=W / H)
    radius = 4.0
    p = _ao_params(api, cam, W, H, spp, radius)
    a_flat = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r_flat = flat.RenderAO(p, a_flat.data_ptr())
    a_sc = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r_sc = sc.RenderAO(p, a_sc.data_ptr())
    assert r_sc.primary_rays == r_flat.primary_rays == W * H * spp
    assert abs(int(r_sc.ao_rays) - int(r_flat.ao_rays)) <= 1e-4 * r_flat.ao_rays + 4, (r_sc.ao_rays, r_flat.ao_rays)
    assert r_sc.ao_hits > 0.05 * r_sc.ao_rays  # something is occluded
    fsum = float(a_sc.double().sum().item())
    assert fsum == float(r_sc.primary_rays - r_sc.ao_hits)
    f_flat, f_sc = a_flat.cpu().numpy() / spp, a_sc.cpu().numpy() / spp
    assert abs(f_sc.mean() - f_flat.mean()) < 2e-3, (f_sc.mean(), f_flat.mean())
    differ = np.abs(f_sc - f_flat) > 1e-6
    assert differ.mean() < 0.01, differ.mean()
    assert np.abs(f_sc - f_flat).max() <= 2.0 / spp + 1e-6
    # conformance walk of the scene (the reference's list algorithm): the same frame up to exact-distance ties
    pc = _ao_params(api, cam, W, H, spp, radius)
    pc.flags = api.TRAVERSE_CONFORMANCE
    a_c = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r_c = sc.RenderAO(pc, a_c.data_ptr())
    assert r_c.primary_rays == r_sc.primary_rays and abs(int(r_c.ao_rays) - int(r_sc.ao_rays)) <= 4
    assert float((a_c != a_sc).double().mean().item()) < 1e-3
    # shards
    total = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    rays = 0
    for shard in range(3):
        ps = _ao_params(api, cam, W, H, spp, radius, shard=shard, n_shards=3)
        part = torch.zeros(W * H, dtype=torch.float32, device="cuda")
        r = sc.RenderAO(ps, part.data_ptr())
        total += part
        rays += r.primary_rays
    assert rays == W * H * spp and torch.equal(total, a_sc)


def test_scene_ao_pass_without_a_result():
    """nrt_scene_render_ao_device with res == NULL, which the C ABI allows: the call succeeds and renders the frame it
    renders with a result struct, bit for bit (nothing is timed)."""
    import ctypes as C

    import torch
    from nanort_b200 import api, scenes as S

    base = S.sphere_grid(nx=2, nz=2)
    insts = [(base[0], base[1], S.xform(translate=(-4.0, 0.0, 0.0))),
             (base[0], base[1], S.xform(translate=(4.0, 0.5, 1.0), yaw=0.6))]
    sc = _gpu_scene(insts, api.BUILD_FAST, api.BUILD_FAST)
    W, H, spp = 160, 96, 2
    p = _ao_params(api, S.look_at((0.0, 8.0, 18.0), (0.0, 0.0, 0.0), aspect=W / H), W, H, spp, 3.0)
    with_res = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r = sc.RenderAO(p, with_res.data_ptr())
    assert r.primary_rays == W * H * spp and r.ao_hits > 0
    without = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    rc = api.lib().nrt_scene_render_ao_device(sc._h, C.byref(p), C.c_void_p(without.data_ptr()), None, None)
    assert rc == 0, api.lib().nrt_last_error()
    assert torch.equal(without, with_res)
