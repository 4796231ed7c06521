"""The AO pass's camera launch over the camera-relative copies walks each 8x4-pixel packet as one warp (traverse3.cuh:
traverse_packet_kernel, selected by traverse.cu: launch_traverse_camera_fused).

Every case compares the fused frame bit for bit with the AO_UNFUSED frame, whose primary launch is the per-lane
while-while kernel over a ray queue, and compares the primary, AO and occluded ray counts.  A packet walk visits each
lane's nodes in the warp's order instead of the lane's own; the closest hit is the same, so the AO rays it spawns and
the frame are too (an exact-t tie between primitives with different normals would show here as a frame difference).
The cases cover both packet instantiations (the 64- and the 512-entry stack), packets whose lanes diverge (camera
inside the scene, a very wide field of view, an image of one packet), and lanes that start inactive or stop early
(slots outside the image, empty or NaN ranges, a short ray_max_t)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# Which camera launch a pass takes is not observable from outside, so the tests recompute the selection of
# traverse.cu's launch_traverse_camera_fused and needs_deep_stack from copies of their constants and assert which side
# each scene lies on; they must change together with kCameraRelMaxBytes / kPair128MaxBytes, sizeof(PairNode) /
# sizeof(TriCM) and the 64-entry stack.
CAMERA_REL_MAX = 24 << 20  # traverse.cu: kCameraRelMaxBytes
PAIR128_MAX = 38 << 20     # traverse.cu: kPair128MaxBytes
PAIR_NODE_BYTES, TRI_CM_BYTES = 128, 48  # common.cuh: PairNode, TriCM
STACK_SMALL = 64           # traverse.cu: needs_deep_stack() picks 512 entries above this
AO_UNFUSED = 0x10000


def _path(acc, n_prims):
    """(packet walk?, 512-entry stack?) of the fused camera launch on this accel: the packet walk reads the
    camera-relative copies, which exist only for PairNode trees whose arrays and copies fit the copy budget."""
    st = acc.GetStatistics()
    pair_bytes = st["num_branch_nodes"] * PAIR_NODE_BYTES
    packet = pair_bytes <= PAIR128_MAX and 2 * (pair_bytes + n_prims * TRI_CM_BYTES) <= CAMERA_REL_MAX
    return packet, st["max_tree_depth"] + 2 > STACK_SMALL


def _params(api, cam, W, H, spp, ao_max_t, min_t=1e-3, max_t=1e30, tile=(64, 8), flags=0):
    p = api.AoParams()
    for i in range(12):
        p.cam[i] = float(cam[i])
    p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, 0, 3
    p.tile_w, p.tile_h, p.shard, p.n_shards = tile[0], tile[1], 0, 1
    p.ray_min_t, p.ray_max_t, p.ao_min_t, p.ao_max_t = min_t, max_t, 1e-3, ao_max_t
    p.flags = flags
    return p


def _check_fused_equals_unfused(acc, cam, W, H, spp=2, ao_max_t=1.0, **kw):
    """Renders the pass fused and unfused; returns (primary, AO, occluded) rays after asserting both agree."""
    import torch
    from nanort_b200 import api

    frames, counts = [], []
    for flags in (0, AO_UNFUSED):
        accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
        r = acc.RenderAO(_params(api, cam, W, H, spp, ao_max_t, flags=flags, **kw), accum.data_ptr())
        frames.append(accum.cpu().numpy())
        counts.append((r.primary_rays, r.ao_rays, r.ao_hits))
    assert counts[0] == counts[1], counts
    assert np.array_equal(frames[0].view(np.uint32), frames[1].view(np.uint32)), int((frames[0] != frames[1]).sum())
    assert counts[0][0] == W * H * spp
    return counts[0]


def _build(v, f, flags=0):
    from nanort_b200 import api

    acc = api.BVHAccel()
    acc.Build(len(f), v, f, flags=flags)
    return acc


@pytest.fixture(scope="module")
def grid():
    from nanort_b200 import scenes as S

    v, f = S.make_scene("sphere_grid", nx=3, nz=3)
    return _build(v, f), len(f)


# ------------------------------------------------------------------ the three instantiations
def test_headline_scene_production_tree():
    """The bench scene (100 K-triangle sphere grid) on the production tree at a reduced resolution: 64-entry
    stack."""
    from nanort_b200 import scenes as S

    v, f = S.make_scene("sphere_grid")
    acc = _build(v, f)
    assert _path(acc, len(f)) == (True, False)
    W, H = 320, 184
    rays = _check_fused_equals_unfused(acc, S.scene_camera("sphere_grid", W, H), W, H, spp=2, ao_max_t=2.0)
    assert 0 < rays[2] < rays[1] < rays[0]


def test_reference_built_deep_tree():
    """terrain(128) with the reference's builder: deeper than 62 levels, so the 512-entry stack."""
    from nanort_b200 import api, scenes as S

    v, f = S.make_scene("terrain", n=128)
    acc = _build(v, f, flags=api.BUILD_REFERENCE_TREE)
    assert _path(acc, len(f)) == (True, True), acc.GetStatistics()["max_tree_depth"]
    W, H = 192, 104
    rays = _check_fused_equals_unfused(acc, S.scene_camera("terrain", W, H), W, H, spp=2, ao_max_t=1.0)
    assert rays[1] > 0 and rays[2] > 0


# ------------------------------------------------------------------ packets whose lanes diverge
@pytest.mark.parametrize("case", ["inside", "wide_fov", "one_packet"])
def test_diverging_packets(grid, case):
    from nanort_b200 import scenes as S

    acc, n = grid
    assert _path(acc, n) == (True, False)
    if case == "inside":  # within the scene box, spheres on every side
        W, H = 64, 32
        cam = S.look_at((-0.5, 0.3, -0.5), (1.0, 0.3, 1.0), fov_y_deg=70.0, aspect=W / H)
    elif case == "wide_fov":  # a packet spans a wide cone of directions
        W, H = 64, 32
        cam = S.look_at((0.2, 1.9, 4.1), (0.0, 0.2, 0.0), fov_y_deg=170.0, aspect=W / H)
    else:  # the whole image is one 8 x 4 packet
        W, H = 8, 4
        cam = S.look_at((0.37, 6.53, 11.1), (0.0, 0.3, 0.0), fov_y_deg=60.0, aspect=W / H)
    rays = _check_fused_equals_unfused(acc, cam, W, H, spp=4, tile=(8, 4) if case == "one_packet" else (64, 8))
    assert rays[1] > 0


# ------------------------------------------------------------------ lanes that start inactive or stop early
def test_partial_tiles(grid):
    """61 x 29 pixels in 64 x 8 tiles: the last tile column and row hold slots outside the image, which take part in
    their packets' walks without a ray."""
    from nanort_b200 import scenes as S

    acc, n = grid
    W, H = 61, 29
    cam = S.look_at((0.37, 6.53, 11.1), (0.0, 0.3, 0.0), fov_y_deg=20.0, aspect=W / H)
    rays = _check_fused_equals_unfused(acc, cam, W, H, spp=3)
    assert rays[1] > 0


@pytest.mark.parametrize("rng", [(5.0, 1.0), (1e-3, float("nan")), (float("nan"), 1e30)])
def test_every_lane_starts_inactive(grid, rng):
    """An empty or NaN range: no lane of any packet enters the root; every ray misses."""
    from nanort_b200 import scenes as S

    acc, n = grid
    W, H = 64, 32
    cam = S.look_at((0.37, 6.53, 11.1), (0.0, 0.3, 0.0), fov_y_deg=20.0, aspect=W / H)
    rays = _check_fused_equals_unfused(acc, cam, W, H, min_t=rng[0], max_t=rng[1])
    assert rays[1] == 0


def test_short_max_t_ends_packets_mid_tree(grid):
    """ray_max_t shorter than the distance to most spheres: lanes drop out at inner nodes, and packets end while
    their stacks still hold entries that every lane culls."""
    from nanort_b200 import scenes as S

    acc, n = grid
    W, H = 64, 32
    org = np.array([0.37, 6.53, 11.1])
    cam = S.look_at(tuple(org), (0.0, 0.3, 0.0), fov_y_deg=20.0, aspect=W / H)
    max_t = float(np.linalg.norm(org - np.array([0.0, 0.3, 0.0])))  # the grid's centre sphere and nearer ones only
    rays = _check_fused_equals_unfused(acc, cam, W, H, spp=2, max_t=max_t)
    full = _check_fused_equals_unfused(acc, cam, W, H, spp=2)
    assert 0 < rays[1] < full[1]
