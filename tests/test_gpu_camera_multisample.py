"""The packet walk of the AO pass's camera launch takes two samples of each 8x4-pixel block per warp, two rays per lane
(traverse3.cuh: traverse_packet_kernel, wavefront.cuh: CameraUnits, traverse.cu: CameraPacketPolicy).

Every case compares the fused frame bit for bit with the AO_UNFUSED frame, whose primary launch is the per-lane
while-while kernel over a ray queue, and compares the primary, AO and occluded ray counts.  The cases cover how work
units map to slots (odd and even spp, where the last unit of a block holds a sample past spp; sample0 != 0; tiles that
reach past the image; packed tiles of two shards), the 512-entry stack, units whose samples diverge (camera inside the
scene, a 170 degree field of view: the two rays of a lane may then differ in direction signs, and the warp loads planes
and triangles per ray) and rays that end early (a short ray_max_t)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

AO_UNFUSED = 0x10000
AO_PACKED_TILES = 0x20000


def _params(api, cam, W, H, spp, sample0=0, tile=(64, 8), max_t=1e30, shard=0, n_shards=1, flags=0):
    p = api.AoParams()
    for i in range(12):
        p.cam[i] = float(cam[i])
    p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, sample0, 5
    p.tile_w, p.tile_h, p.shard, p.n_shards = tile[0], tile[1], shard, n_shards
    p.ray_min_t, p.ray_max_t, p.ao_min_t, p.ao_max_t = 1e-3, max_t, 1e-3, 1.0
    p.flags = flags
    return p


def _render(acc, p, n_floats):
    import torch

    accum = torch.zeros(n_floats, dtype=torch.float32, device="cuda")
    r = acc.RenderAO(p, accum.data_ptr())
    return accum.cpu().numpy(), (r.primary_rays, r.ao_rays, r.ao_hits)


def _check(acc, cam, W, H, spp, **kw):
    """Fused and unfused frames and counts agree bit for bit; returns the counts."""
    from nanort_b200 import api

    fused, c0 = _render(acc, _params(api, cam, W, H, spp, **kw), W * H)
    unfused, c1 = _render(acc, _params(api, cam, W, H, spp, flags=AO_UNFUSED, **kw), W * H)
    assert c0 == c1, (c0, c1)
    assert np.array_equal(fused.view(np.uint32), unfused.view(np.uint32)), int((fused != unfused).sum())
    assert c0[0] == W * H * spp
    return c0


def _build(v, f, flags=0):
    from nanort_b200 import api

    acc = api.BVHAccel()
    acc.Build(len(f), v, f, flags=flags)
    return acc


@pytest.fixture(scope="module")
def grid():
    from nanort_b200 import scenes as S

    v, f = S.make_scene("sphere_grid", nx=3, nz=3)
    return _build(v, f)


def _cam(W, H, fov=20.0):
    from nanort_b200 import scenes as S

    return S.look_at((0.37, 6.53, 11.1), (0.0, 0.3, 0.0), fov_y_deg=fov, aspect=W / H)


@pytest.mark.parametrize("spp", [1, 2, 3, 4])
def test_odd_and_even_spp(grid, spp):
    W, H = 64, 32
    rays = _check(grid, _cam(W, H), W, H, spp)
    assert 0 < rays[2] < rays[1]


@pytest.mark.parametrize("spp,sample0", [(3, 5), (2, 7)])
def test_sample0(grid, spp, sample0):
    W, H = 64, 32
    rays = _check(grid, _cam(W, H), W, H, spp, sample0=sample0)
    assert rays[1] > 0


@pytest.mark.parametrize("spp", [1, 3])
def test_partial_tiles(grid, spp):
    """61 x 29 pixels in 64 x 8 tiles: the last tile column and row hold slots outside the image."""
    W, H = 61, 29
    rays = _check(grid, _cam(W, H), W, H, spp)
    assert rays[1] > 0


@pytest.mark.parametrize("spp", [1, 3])
def test_packed_tiles_two_shards(grid, spp):
    """Two shards of one rank each, accumulating tile-major: each shard's packed frame is the packing of its part of
    the unfused single-shard frame, and the two parts add up to it."""
    from nanort_b200 import api, dist as nd

    W, H, tile = 75, 37, (16, 8)
    cam = _cam(W, H)
    full, c_full = _render(grid, _params(api, cam, W, H, spp, tile=tile, flags=AO_UNFUSED), W * H)
    n_packed = nd.packed_slot_floats(W, H, tile[0], tile[1], 2)
    total, counts = np.zeros(W * H, np.float32), np.zeros(3, np.int64)
    for shard in range(2):
        part, c_part = _render(grid, _params(api, cam, W, H, spp, tile=tile, shard=shard, n_shards=2,
                                             flags=AO_UNFUSED), W * H)
        packed, c_packed = _render(grid, _params(api, cam, W, H, spp, tile=tile, shard=shard, n_shards=2,
                                                 flags=AO_PACKED_TILES), n_packed)
        assert c_packed == c_part
        want = nd.pack_own_tiles(part, W, H, tile[0], tile[1], shard, 2)
        assert np.array_equal(packed.view(np.uint32), want.view(np.uint32))
        total += part
        counts += np.array(c_part)
    assert np.array_equal(total, full) and tuple(counts) == c_full


def test_reference_built_deep_tree():
    """terrain(128) with the reference's builder: deeper than 62 levels, so the 512-entry stack."""
    from nanort_b200 import api, scenes as S

    v, f = S.make_scene("terrain", n=128)
    acc = _build(v, f, flags=api.BUILD_REFERENCE_TREE)
    assert acc.GetStatistics()["max_tree_depth"] + 2 > 64
    W, H = 96, 56
    rays = _check(acc, S.scene_camera("terrain", W, H), W, H, 3)
    assert rays[1] > 0 and rays[2] > 0


@pytest.mark.parametrize("case", ["inside", "wide_fov"])
def test_diverging_samples(grid, case):
    """Samples of one pixel that leave in different directions and reach different spheres."""
    from nanort_b200 import scenes as S

    W, H = 64, 32
    if case == "inside":
        cam = S.look_at((-0.5, 0.3, -0.5), (1.0, 0.3, 1.0), fov_y_deg=70.0, aspect=W / H)
    else:
        cam = S.look_at((0.2, 1.9, 4.1), (0.0, 0.2, 0.0), fov_y_deg=170.0, aspect=W / H)
    rays = _check(grid, cam, W, H, 3)
    assert rays[1] > 0


def test_short_max_t(grid):
    """ray_max_t shorter than the distance to most spheres: rays drop out at inner nodes."""
    W, H = 64, 32
    org = np.array([0.37, 6.53, 11.1])
    max_t = float(np.linalg.norm(org - np.array([0.0, 0.3, 0.0])))
    short = _check(grid, _cam(W, H), W, H, 3, max_t=max_t)
    full = _check(grid, _cam(W, H), W, H, 3)
    assert 0 < short[1] < full[1]
