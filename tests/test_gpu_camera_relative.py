"""The AO pass's camera launch over camera-relative nodes and triangles (traverse.cu: launch_traverse_camera_fused,
layout.cu: camera_relative_layout) and its AO spawn from per-primitive normals (render.cu: face_normals_kernel).

The fused pass is compared bit for bit with the AO_UNFUSED pass, whose primary launch reads the accel's own arrays
and subtracts the origin per ray: cameras whose origin subtraction rounds, the copies' cache across origins, accel
rebuilds and adoptions, two streams sharing one accel, and a scene too large for the copies."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# Which camera launch a pass takes is not observable from outside, so the tests recompute the selection of
# traverse.cu's launch_traverse_camera_fused from these copies of its constants and assert which side each scene lies
# on; they must change together with kCameraRelMaxBytes / kPair128MaxBytes and sizeof(PairNode) / sizeof(TriCM).
CAMERA_REL_MAX = 24 << 20  # traverse.cu: kCameraRelMaxBytes
PAIR128_MAX = 38 << 20     # traverse.cu: kPair128MaxBytes
PAIR_NODE_BYTES, TRI_CM_BYTES = 128, 48  # common.cuh: PairNode, TriCM
AO_UNFUSED = 0x10000


def _copy_bytes(acc, n_prims):
    return 2 * (acc.GetStatistics()["num_branch_nodes"] * PAIR_NODE_BYTES + n_prims * TRI_CM_BYTES)


def _params(api, cam, W, H, spp, ao_max_t, flags=0):
    p = api.AoParams()
    for i in range(12):
        p.cam[i] = float(cam[i])
    p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, 0, 1
    p.tile_w, p.tile_h, p.shard, p.n_shards = 64, 8, 0, 1
    p.ray_min_t, p.ray_max_t, p.ao_min_t, p.ao_max_t = 1e-3, 1e30, 1e-3, ao_max_t
    p.flags = flags
    return p


def _render(torch, acc, cam, W, H, spp=2, ao_max_t=1.0, flags=0):
    from nanort_b200 import api

    accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r = acc.RenderAO(_params(api, cam, W, H, spp, ao_max_t, flags), accum.data_ptr())
    return accum.cpu().numpy(), (r.primary_rays, r.ao_rays, r.ao_hits)


def _cam(S, org, target, fov=20.0, W=64, H=32, zero=()):
    cam = S.look_at(org, target, fov_y_deg=fov, aspect=W / H)
    for k in zero:  # an origin component of -0.0 (look_at would give +0.0)
        cam[k] = np.float32(-0.0)
    return cam


def _cameras(S):
    """(name, camera) of the 3 x 3 sphere grid (spheres at -1, 0, 1 on the floor y = 0), origins whose subtraction
    from the planes and vertices rounds: odd offsets, far away (1e6 + odd), negative, -0.0 components, inside the
    scene box."""
    far = np.array([1e6 + 0.371, 2.0e5 - 0.113, -3.0e5 + 0.777])
    dist = float(np.linalg.norm(far))
    return [
        ("odd", _cam(S, (0.37, 6.53, 11.1), (0.0, 0.3, 0.0))),
        ("far", _cam(S, tuple(far), (0.0, 0.3, 0.0), fov=np.degrees(4.0 / dist))),
        ("negative", _cam(S, (-3.3, -0.9, -4.7), (0.0, 0.1, 0.0))),
        ("minus_zero", _cam(S, (0.0, 6.5, 11.0), (0.0, 0.3, 0.0), zero=(0,))),
        ("minus_zero_y", _cam(S, (2.0, 0.0, 9.0), (0.0, 0.3, 0.0), zero=(1,))),
        ("inside", _cam(S, (-0.5, 0.3, -0.5), (1.0, 0.3, 1.0), fov=70.0)),
    ]


@pytest.fixture(scope="module")
def grid():
    from nanort_b200 import scenes as S

    return S.make_scene("sphere_grid", nx=3, nz=3)


def _fresh(torch, v, f, cam, **kw):
    from nanort_b200 import api

    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    return _render(torch, acc, cam, 64, 32, **kw)


def test_fused_equals_unfused_for_rounding_origins(grid):
    import torch
    from nanort_b200 import api, scenes as S

    v, f = grid
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    assert _copy_bytes(acc, len(f)) <= CAMERA_REL_MAX  # the fused pass reads the copies
    for name, cam in _cameras(S):
        fused, rf = _render(torch, acc, cam, 64, 32)
        unfused, ru = _render(torch, acc, cam, 64, 32, flags=AO_UNFUSED)
        assert rf == ru and rf[1] > 0, (name, rf, ru)
        assert np.array_equal(fused.view(np.uint32), unfused.view(np.uint32)), name


def test_origin_changes_on_one_accel_equal_fresh_accels(grid):
    """The copies follow the origin: every pass on one accel equals the same pass on a fresh accel."""
    import torch
    from nanort_b200 import api, scenes as S

    v, f = grid
    cams = _cameras(S)
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    for name, cam in cams + cams[:2]:  # back to origins it held before
        got, rg = _render(torch, acc, cam, 64, 32)
        want, rw = _fresh(torch, v, f, cam)
        assert rg == rw and np.array_equal(got.view(np.uint32), want.view(np.uint32)), name


def test_passes_after_rebuild_and_adopt_equal_fresh_accels(grid):
    """Re-Build and Adopt on one BVHAccel object after a pass.  Both create a new native accel (nrt_build_ex /
    nrt_adopt), so this checks what a caller sees -- no copies or normals of the old geometry survive -- not the
    invalidation inside derive_private_layout, which no entry point reaches on an accel that already rendered."""
    import torch
    from nanort_b200 import api, scenes as S

    v, f = grid
    cam = _cameras(S)[0][1]
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    _render(torch, acc, cam, 64, 32)
    # other geometry under the same origin: stale copies would keep the old spheres
    v2 = (v + np.float32([0.5, 0.0, -0.25])).astype(np.float32)
    acc.Build(len(f), v2, f)
    got, rg = _render(torch, acc, cam, 64, 32)
    want, rw = _fresh(torch, v2, f, cam)
    assert rg == rw and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    unfused, ru = _render(torch, acc, cam, 64, 32, flags=AO_UNFUSED)
    assert rg == ru and np.array_equal(got.view(np.uint32), unfused.view(np.uint32))
    # the Load path (a dumped tree adopted as it is)
    ref = api.BVHAccel()
    ref.Build(len(f), v, f)
    nodes, idx = ref.GetNodes(), ref.GetIndices()
    acc.Adopt(nodes, idx, v, f)
    got, rg = _render(torch, acc, cam, 64, 32)
    want, rw = _render(torch, ref, cam, 64, 32)
    assert rg == rw and np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_two_streams_on_one_accel(grid):
    """Passes with different origins enqueued on two streams with no synchronisation between them: each pass waits
    for the one enqueued before it, so neither reads copies (or wave scratch) that the other rewrites."""
    import torch
    from nanort_b200 import api, scenes as S

    v, f = grid
    cams = _cameras(S)
    a_cam, b_cam = cams[0][1], cams[2][1]
    W, H, spp = 256, 128, 4
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    want_a, _ = _render(torch, acc, a_cam, W, H, spp)
    want_b, _ = _render(torch, acc, b_cam, W, H, spp)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    frames = [torch.zeros(W * H, dtype=torch.float32, device="cuda") for _ in range(4)]
    torch.cuda.synchronize()  # the zeroing is done before either stream starts; nothing waits from here on
    for k, accum in enumerate(frames):
        cam, s = (a_cam, s1) if k % 2 == 0 else (b_cam, s2)
        acc.RenderAO(_params(api, cam, W, H, spp, 1.0), accum.data_ptr(), stream=s.cuda_stream, want_result=False)
    torch.cuda.synchronize()
    for k, accum in enumerate(frames):
        want = want_a if k % 2 == 0 else want_b
        assert np.array_equal(accum.cpu().numpy().view(np.uint32), want.view(np.uint32)), k


def test_scene_above_the_copy_budget():
    """A PairNode scene whose arrays and copies would exceed kCameraRelMaxBytes: the camera launch reads the accel's
    own arrays and subtracts the origin per ray."""
    import torch
    from nanort_b200 import api, scenes as S

    v, f = S.make_scene("sphere_grid", nx=16, nz=16)
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    assert _copy_bytes(acc, len(f)) > CAMERA_REL_MAX
    assert acc.GetStatistics()["num_branch_nodes"] * PAIR_NODE_BYTES <= PAIR128_MAX
    cam = _cam(S, (0.37, 9.53, 16.1), (0.0, 0.2, 0.0), W=128, H=64)
    fused, rf = _render(torch, acc, cam, 128, 64, spp=1)
    unfused, ru = _render(torch, acc, cam, 128, 64, spp=1, flags=AO_UNFUSED)
    assert rf == ru and rf[2] > 0
    assert np.array_equal(fused.view(np.uint32), unfused.view(np.uint32))


@pytest.mark.parametrize("kind", ["spheres", "boxes"])
def test_pass_on_a_non_triangle_accel_is_refused(kind):
    """Sphere and box accels have no triangle layout to derive the copies or the normals from: RenderAO refuses them
    before it derives or launches anything, fused or not."""
    import torch
    from nanort_b200 import api, scenes as S

    acc = api.BVHAccel()
    centers = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    if kind == "spheres":
        assert acc.BuildSpheres(centers, np.full(4, 0.25, np.float32))
    else:
        assert acc.BuildBoxes(np.concatenate([centers - 0.25, centers + 0.25], axis=1))
    cam = _cam(S, (0.37, 2.53, 5.1), (0.0, 0.3, 0.0))
    accum = torch.zeros(64 * 32, dtype=torch.float32, device="cuda")
    for flags in (0, AO_UNFUSED):
        with pytest.raises(api.NanortB200Error, match="triangle accel"):
            acc.RenderAO(_params(api, cam, 64, 32, 1, 1.0, flags), accum.data_ptr())
    torch.cuda.synchronize()  # the context is still usable
    assert float(accum.sum().item()) == 0.0
