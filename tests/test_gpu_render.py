"""The wavefront primary+AO pass: fused == stand-alone stages, rays == numpy generators, hits == oracle,
tile sharding == single shard."""
import numpy as np
import pytest

from helpers import assert_parity, compare_hits

pytestmark = pytest.mark.gpu


def _params(api, S, name, W, H, spp, bbox, shard=0, n_shards=1, flags=0, tile=(64, 8)):
    cam = S.scene_camera(name, W, H)
    p = api.AoParams()
    for i in range(12):
        p.cam[i] = float(cam[i])
    p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, 0, 1
    p.tile_w, p.tile_h, p.shard, p.n_shards = tile[0], tile[1], shard, n_shards
    p.ray_min_t, p.ray_max_t, p.ao_min_t, p.ao_max_t = 1e-3, 1e30, 1e-3, 0.25 * float(np.linalg.norm(bbox[1] - bbox[0]))
    p.flags = flags
    return p, cam


@pytest.mark.parametrize("name,kw,W,H,spp", [("sphere_grid", dict(nx=4, nz=4), 200, 104, 3), ("cornell", {}, 96, 64, 2)])
def test_pass_fused_equals_unfused_and_matches_oracle(port, name, kw, W, H, spp):
    import torch
    from oracle import orc
    from nanort_b200 import api, dist as nd, scenes as S

    v, f = S.make_scene(name, **kw)
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    bbox = acc.BoundingBox()
    frames, results = [], []
    for flags in (0, 0x10000):  # fused, NRT_AO_UNFUSED
        p, cam = _params(api, S, name, W, H, spp, bbox, flags=flags)
        accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
        r = acc.RenderAO(p, accum.data_ptr())
        frames.append(accum.cpu().numpy())
        results.append((r.primary_rays, r.ao_rays, r.ao_hits))
    assert results[0] == results[1]
    assert np.array_equal(frames[0], frames[1])
    assert results[0][0] == W * H * spp

    # exported queues: primary rays equal the numpy generator (same hash), all hits equal the oracle's
    p, cam = _params(api, S, name, W, H, spp, bbox)
    slots = nd.shard_ray_count(W, H, 64, 8, 0, 1, spp)
    pix, smp = nd.slot_pixels(W, H, 64, 8, 0, 1, spp)
    n_slots = len(pix)
    d_p = torch.empty(n_slots * 36, dtype=torch.uint8, device="cuda")
    d_a = torch.empty(n_slots * 36, dtype=torch.uint8, device="cuda")
    accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    n_p, n_a = acc.ExportAOWorkload(p, accum.data_ptr(), d_p.data_ptr(), d_a.data_ptr())
    assert n_p == slots == int((pix >= 0).sum()) and n_a == results[0][1]
    assert np.array_equal(accum.cpu().numpy(), frames[0])
    prim = d_p.cpu().numpy().view(S.RAY_DTYPE)
    valid = pix >= 0
    want = np.zeros(n_slots, S.RAY_DTYPE)
    for s in range(spp):
        sel = valid & (smp == s)
        want[sel] = S.primary_rays(cam, W, H, spp=1, seed=1, pixels=pix[sel], sample0=s)
    assert np.array_equal(prim["dir"][valid].view(np.uint32), want["dir"][valid].view(np.uint32))  # bit for bit
    assert np.array_equal(prim["org"][valid], want["org"][valid])
    assert np.all(prim["max_t"][~valid] < 0)

    rn, ri, _ = port.build(v, f, mode=orc.MODE_CPP11)
    ao = d_a[: n_a * 36].cpu().numpy().view(S.RAY_DTYPE)
    occluded = None
    for rays in (prim[valid], ao):
        want_h, want_m = port.traverse(rn, ri, v, f, rays, threads=8)
        got_h, got_m = acc.Traverse(rays)
        assert_parity(compare_hits(port, v, f, rays, got_h, got_m, want_h, want_m))
        occluded = int(want_m.sum())
    assert int(want_m.sum()) == results[0][2]
    assert float(frames[0].sum()) == float(n_p - occluded)
    # pixels whose primaries all miss are fully visible; no pixel exceeds spp
    ph, pm = port.traverse(rn, ri, v, f, prim[valid], threads=8)
    miss_per_pix = np.bincount(pix[valid][pm == 0], minlength=W * H)
    assert np.all(frames[0] >= miss_per_pix) and np.all(frames[0] <= spp)
    assert np.all(frames[0][miss_per_pix == spp] == spp)


def test_tile_shards_add_up_to_the_single_shard_frame():
    """rays shard by tile across GPUs: the union of the shards' frames is the 1-shard frame, bit for bit."""
    import torch
    from nanort_b200 import api, dist as nd, scenes as S

    name, W, H, spp = "sphere_grid", 200, 104, 2
    v, f = S.make_scene(name, nx=4, nz=4)
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    bbox = acc.BoundingBox()
    p, _ = _params(api, S, name, W, H, spp, bbox)
    full = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r_full = acc.RenderAO(p, full.data_ptr())
    total = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    rays = 0
    for shard in range(3):
        ps, _ = _params(api, S, name, W, H, spp, bbox, shard=shard, n_shards=3)
        part = torch.zeros(W * H, dtype=torch.float32, device="cuda")
        r = acc.RenderAO(ps, part.data_ptr())
        mine = torch.as_tensor(nd.shard_pixels(W, H, 64, 8, shard, 3), device="cuda")
        other = torch.ones(W * H, dtype=torch.bool, device="cuda")
        other[mine] = False
        assert float(part[other].abs().sum().item()) == 0.0, "a shard only touches its own pixels"
        assert r.primary_rays == len(mine) * spp
        total += part
        rays += r.primary_rays + r.ao_rays
    assert torch.equal(total, full)
    assert rays == r_full.primary_rays + r_full.ao_rays


@pytest.mark.parametrize("name,kw,W,H,spp", [("sphere_grid", dict(nx=4, nz=4), 200, 104, 4), ("terrain", dict(n=96), 160, 96, 3)])
def test_any_hit_occlusion_rays_give_the_same_frame(name, kw, W, H, spp):
    """NRT_TRAVERSE_ANY_HIT on the AO launch (nanort has only closest-hit, examples/path_tracer/main.cc:675-701 looks at
    the bool): framebuffer and occluded count identical bit for bit; through nrt_traverse the hit flags are identical
    and every record is a real hit at or behind the closest one."""
    import torch
    from nanort_b200 import api, scenes as S

    v, f = S.make_scene(name, **kw)
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    bbox = acc.BoundingBox()
    out = []
    for flags in (0, api.TRAVERSE_ANY_HIT):
        p, _ = _params(api, S, name, W, H, spp, bbox, flags=flags)
        accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
        r = acc.RenderAO(p, accum.data_ptr())
        out.append((accum.cpu().numpy(), (r.primary_rays, r.ao_rays, r.ao_hits)))
    assert out[0][1] == out[1][1] and out[0][1][2] > 0
    assert np.array_equal(out[0][0], out[1][0])

    p, _ = _params(api, S, name, W, H, spp, bbox)
    n_slots = W * H * spp * 2
    d_p = torch.empty(n_slots * 36, dtype=torch.uint8, device="cuda")
    d_a = torch.empty(n_slots * 36, dtype=torch.uint8, device="cuda")
    accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    n_p, n_a = acc.ExportAOWorkload(p, accum.data_ptr(), d_p.data_ptr(), d_a.data_ptr())
    ao = d_a[: n_a * 36].cpu().numpy().view(S.RAY_DTYPE)
    ch, cm = acc.Traverse(ao)
    ah, am = acc.Traverse(ao, flags=api.TRAVERSE_ANY_HIT)
    assert np.array_equal(am, cm)
    hit = cm.astype(bool)
    assert np.all(ah["prim_id"][~hit] == 0xFFFFFFFF) and np.all(ah["prim_id"][hit] < len(f))
    assert np.all(ah["t"][hit] >= ch["t"][hit]) and np.all(ah["t"][hit] < ao["max_t"][hit]) and np.all(ah["t"][hit] >= ao["min_t"][hit])
    # a record that differs from the closest one is a genuine hit of ITS triangle: re-trace with only that triangle allowed
    other = np.flatnonzero(hit & (ah["prim_id"] != ch["prim_id"]))[:200]
    for i in other:
        o = api.BVHTraceOptions(prim_ids_range=(int(ah["prim_id"][i]), int(ah["prim_id"][i]) + 1))
        h1, m1 = acc.Traverse(ao[i:i + 1], options=o)
        assert m1[0] == 1 and h1.view(np.uint32).tolist() == ah[i:i + 1].view(np.uint32).tolist()


@pytest.mark.parametrize("unfused", [False, True])
def test_pass_times_split_into_primary_and_ao_launches(unfused):
    """The AO pass's traversal time is the sum of its camera-ray and AO-ray launch times, both inside the pass's time;
    with no result struct the pass renders the same frame."""
    import torch
    from nanort_b200 import api, scenes as S

    name, W, H, spp = "sphere_grid", 200, 104, 2
    v, f = S.make_scene(name, nx=4, nz=4)
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    p, _ = _params(api, S, name, W, H, spp, acc.BoundingBox(), flags=api.AO_UNFUSED if unfused else 0)
    accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r = acc.RenderAO(p, accum.data_ptr())
    assert r.primary_traverse_ms > 0.0 and r.ao_traverse_ms > 0.0
    assert abs(r.traverse_ms - (r.primary_traverse_ms + r.ao_traverse_ms)) <= 1e-4 * r.traverse_ms
    assert r.traverse_ms <= r.total_ms
    quiet = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    acc.RenderAO(p, quiet.data_ptr(), want_result=False)
    torch.cuda.synchronize()
    assert torch.equal(quiet, accum)
