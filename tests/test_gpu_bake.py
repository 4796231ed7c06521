"""Texture-space baking (include/nanort_b200_bake.h) against the reference's arithmetic:
  * the texel cast (nrt_uv_raster_device) over a reference-exact UV tree with the conformance walk writes, texel by
    texel, the record CPU nanort's Traverse returns for the reference uv_raster's ray (flips, UV regions, texel offsets,
    sizes that are not multiples of 8 or 32); the production tree and walk agree on coverage and distance; the
    position and normal AOVs equal the float32 Lerp of main.cc bit for bit;
  * the bake's exported AO rays are the host model's (tests/bake_model.py: bake_rays), lie in the normal's hemisphere
    and are cosine distributed;
  * the bake's accumulator equals, texel by texel, the number of exported rays the reference finds unoccluded, for the
    fast walk, ANY_HIT and the 512-entry stack;
  * sample ranges, launches split at the 32-bit slot cap and two streams compose exactly; refusals launch nothing."""
import os

import numpy as np
import pytest

import bake_model as B

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
MISS = 0xFFFFFFFF
# direction bound against the f32 model (tests/test_gpu_ao_exact.py derives it: sincosf's ulps through the
# 1-Lipschitz direction plus the f32 evaluation's own rounding)
DIR_BOUND_F32 = 1.7e-6
KS_MIN_P = 1e-3


def load_obj_uv(path):
    """(verts, faces, uv mesh (verts, faces), facevarying normals [n, 9]) of an OBJ with v / vt / vn, quads split as
    the reference uv_raster splits them, (p0, p1, p2), (p2, p3, p0) (examples/uv_raster/main.cc:373-404)."""
    v, vt, vn, corners = [], [], [], []
    for line in open(path):
        t = line.split()
        if not t:
            continue
        if t[0] == "v":
            v.append([float(x) for x in t[1:4]])
        elif t[0] == "vt":
            vt.append([float(x) for x in t[1:3]])
        elif t[0] == "vn":
            vn.append([float(x) for x in t[1:4]])
        elif t[0] == "f":
            idx = [[int(x) - 1 for x in c.split("/")] for c in t[1:]]
            tris = [idx] if len(idx) == 3 else [[idx[0], idx[1], idx[2]], [idx[2], idx[3], idx[0]]]
            corners.extend(tris)
    c = np.asarray(corners)  # [n, 3, (v, vt, vn)]
    verts = np.asarray(v, np.float32)
    faces = c[:, :, 0].astype(np.uint32)
    uv = np.asarray(vt, np.float32)[c[:, :, 1]]
    uv_verts = np.zeros((len(c) * 3, 3), np.float32)
    uv_verts[:, :2] = uv.reshape(-1, 2)
    uv_faces = np.arange(len(c) * 3, dtype=np.uint32).reshape(-1, 3)
    fvn = np.asarray(vn, np.float32)[c[:, :, 2]].reshape(-1, 9)
    return verts, faces, (uv_verts, uv_faces), fvn


_MESHES = {}


def mesh(name):
    """(world verts, world faces, uv verts, uv faces, facevarying normals [n, 9] float32)."""
    from nanort_b200 import scenes as S

    if name not in _MESHES:
        if name == "suzanne":
            v, f, (uv, uf), fvn = load_obj_uv(os.path.join(HERE, "golden", "suzanne_uv.obj"))
        else:
            base = "terrain" if name.startswith("terrain") else name
            v, f = S.make_scene(base, **({"n": 96} if base == "terrain" else {}))
            if name == "terrain_reversed":
                f = np.ascontiguousarray(f[:, [0, 2, 1]])
            uv, uf = S.planar_uv(v, f) if name.startswith("terrain") else S.per_face_atlas(len(f))
            # face-varying normals that are not the geometric ones: a deterministic tilt of each corner
            rng = np.random.default_rng(len(f))
            fvn = rng.normal(size=(len(f), 9)).astype(np.float32)
        _MESHES[name] = (v, f, uv, uf, fvn)
    return _MESHES[name]


def _accel(v, f, flags=0):
    from nanort_b200 import api

    acc = api.BVHAccel()
    assert acc.Build(len(f), v, f, flags=flags)
    return acc


def _raster_params(W, H, flip=(0, 0), region=(0.0, 1.0, 0.0, 1.0), offset=(0.5, 0.5), flags=0):
    from nanort_b200 import api

    p = api.UvRasterParams()
    p.width, p.height = W, H
    p.uv_region[:] = list(region)
    p.texel_offset[:] = list(offset)
    p.flip_x, p.flip_y = flip
    p.flags = flags
    return p


def _raster(uv_acc, p, world=None, fvn=None):
    """(records HIT_DTYPE [W*H], position [W*H, 3] or None, normal or None, covered count)."""
    import torch

    from nanort_b200 import scenes as S

    n = p.width * p.height
    rec = torch.full((n, 4), -3.0, dtype=torch.float32, device="cuda")  # every texel must be written
    pos = nrm = d_fvn = None
    if world is not None:
        pos = torch.full((n, 3), -5.0, dtype=torch.float32, device="cuda")
        nrm = torch.full((n, 3), -5.0, dtype=torch.float32, device="cuda")
        d_fvn = torch.from_numpy(fvn).cuda()
    covered = uv_acc.UVRaster(p, rec.data_ptr(), world=world, d_position_ptr=pos.data_ptr() if pos is not None else None,
                              d_normal_ptr=nrm.data_ptr() if nrm is not None else None,
                              d_facevarying_normals_ptr=d_fvn.data_ptr() if d_fvn is not None else None)
    records = rec.cpu().numpy().view(S.HIT_DTYPE).reshape(-1)
    return (records, pos.cpu().numpy() if pos is not None else None, nrm.cpu().numpy() if nrm is not None else None,
            covered)


RASTER_CASES = [  # W, H, flip, region, offset
    (257, 131, (0, 0), (0.0, 1.0, 0.0, 1.0), (0.5, 0.5)),
    (100, 60, (1, 0), (0.0, 1.0, 0.0, 1.0), (0.5, 0.5)),
    (96, 77, (0, 1), (0.1, 0.9, 0.2, 0.8), (0.25, 0.75)),
    (64, 64, (1, 1), (-0.1, 1.1, 1.0, 0.0), (0.0, 0.0)),
]


def _want_records(ref_hits, ref_mask, dest):
    from nanort_b200 import scenes as S

    want = np.zeros(len(dest), S.HIT_DTYPE)
    want["t"] = np.float32(1e30)
    want["prim_id"] = MISS
    hit = ref_mask.astype(bool)
    want[dest[hit]] = ref_hits[hit]
    return want


@pytest.mark.parametrize("name", ["suzanne", "terrain", "cornell"])
@pytest.mark.parametrize("case", range(len(RASTER_CASES)))
def test_raster_conformance_equals_the_reference(name, case):
    from nanort_b200 import api
    from oracle import orc

    W, H, flip, region, offset = RASTER_CASES[case]
    v, f, uv, uf, fvn = mesh(name)
    world = _accel(v, f)
    uv_acc = _accel(uv, uf, flags=api.BUILD_REFERENCE_TREE)
    ref = orc.Reference().build(uv, uf)
    rays = B.texel_rays(W, H, region, offset)
    rh, rm = ref.traverse(rays, threads=8)
    want = _want_records(rh, rm, B.texel_dest(W, H, *flip))
    got, pos, nrm, covered = _raster(uv_acc, _raster_params(W, H, flip, region, offset, api.TRAVERSE_CONFORMANCE),
                                     world, fvn)
    assert got.tobytes() == want.tobytes()
    assert covered == int(rm.sum()) > 0
    _check_aovs(v, f, fvn, got, pos, nrm)


def _check_aovs(v, f, fvn, rec, pos, nrm):
    hit = rec["prim_id"] != MISS
    r = rec[hit]
    tri = f[r["prim_id"]]
    want_p = B.lerp3(v[tri[:, 0]], v[tri[:, 1]], v[tri[:, 2]], r["u"], r["v"])
    n = fvn.reshape(-1, 3, 3)[r["prim_id"]]
    want_n = B.lerp3(n[:, 0], n[:, 1], n[:, 2], r["u"], r["v"])
    assert np.array_equal(pos[hit].view(np.uint32), want_p.view(np.uint32))
    assert np.array_equal(nrm[hit].view(np.uint32), want_n.view(np.uint32))
    assert np.all(pos[~hit] == 0) and np.all(nrm[~hit] == 0)


@pytest.mark.parametrize("name", ["suzanne", "terrain", "cornell"])
def test_raster_production_walk_agrees_with_the_reference(name):
    from oracle import orc

    port = orc.Port()
    v, f, uv, uf, fvn = mesh(name)
    uv_acc, world = _accel(uv, uf), _accel(v, f)
    ref = orc.Reference().build(uv, uf)
    for W, H, flip, region, offset in RASTER_CASES:
        rays = B.texel_rays(W, H, region, offset)
        dest = B.texel_dest(W, H, *flip)
        want = _want_records(*ref.traverse(rays, threads=8), dest)
        for cpp03 in (0, 2):
            got, pos, nrm, covered = _raster(uv_acc, _raster_params(W, H, flip, region, offset, cpp03), world, fvn)
            hit = want["prim_id"] != MISS
            assert np.array_equal(got["prim_id"] != MISS, hit), "covered texels differ"
            assert covered == int(hit.sum())
            assert np.array_equal(got["t"].view(np.uint32), want["t"].view(np.uint32))
            other = np.flatnonzero(hit & (got["prim_id"] != want["prim_id"]))
            same = hit & (got["prim_id"] == want["prim_id"])
            assert got[same].tobytes() == want[same].tobytes()
            # a texel on a shared UV edge or in overlapping charts: the other primitive is hit at the same t
            inv = np.empty_like(dest)
            inv[dest] = np.arange(len(dest))
            for k in other:
                ok, h = port.test_prim(uv, uf, rays[inv[k]], int(got["prim_id"][k]))
                assert ok and h["t"] == got["t"][k] and h["u"] == got["u"][k] and h["v"] == got["v"][k], k
            _check_aovs(v, f, fvn, got, pos, nrm)


# ------------------------------------------------------------------ bake
def _bake_params(W, H, spp, sample0=0, seed=3, ao=(1e-3, 1.0), flags=0, fvn_ptr=None):
    from nanort_b200 import api

    p = api.BakeParams()
    p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, sample0, seed
    p.ao_min_t, p.ao_max_t = ao
    p.flags = flags
    p.d_facevarying_normals = fvn_ptr
    return p


def _export(world, d_rec, p, n_cov):
    import torch

    from nanort_b200 import scenes as S

    buf = torch.zeros(max(n_cov * p.spp, 1) * 9, dtype=torch.float32, device="cuda")
    n = world.ExportBakeRays(d_rec.data_ptr(), p, buf.data_ptr(), n_cov * p.spp)
    assert n == n_cov * p.spp
    return buf.cpu().numpy().view(S.RAY_DTYPE)[:n]


def _bake(world, d_rec, p, accum=None, stream=None):
    import torch

    if accum is None:
        accum = torch.zeros(p.width * p.height, dtype=torch.float32, device="cuda")
    r = world.BakeAO(d_rec.data_ptr(), p, accum.data_ptr(), stream=stream.cuda_stream if stream is not None else None)
    return accum, r


def _records(name, W=160, H=128):
    """Production raster of `name` as (records numpy, records on the device, world accel, v, f, fvn)."""
    import torch

    v, f, uv, uf, fvn = mesh(name)
    world = _accel(v, f)
    rec, _, _, covered = _raster(_accel(uv, uf), _raster_params(W, H))
    assert covered > 0
    return rec, torch.from_numpy(rec.view(np.float32).reshape(-1, 4).copy()).cuda(), world, v, f, fvn


@pytest.mark.parametrize("name,use_fvn", [("suzanne", True), ("suzanne", False), ("terrain", False),
                                          ("terrain_reversed", False), ("terrain_reversed", True), ("cornell", False)])
def test_bake_rays_equal_the_model(name, use_fvn):
    import torch
    from scipy import stats

    rec, d_rec, world, v, f, fvn = _records(name)
    d_fvn = torch.from_numpy(fvn).cuda() if use_fvn else None
    n_cov = int((rec["prim_id"] != MISS).sum())
    p = _bake_params(160, 128, spp=3, sample0=5, seed=11, ao=(2e-3, 0.75),
                     fvn_ptr=d_fvn.data_ptr() if use_fvn else None)
    got = _export(world, d_rec, p, n_cov)
    want, texel, smp = B.bake_rays(v, f, rec, 3, 11, 2e-3, 0.75, sample0=5, fv_normals=fvn if use_fvn else None)
    assert np.array_equal(got["org"].view(np.uint32), want["org"].view(np.uint32))
    assert np.all(got["min_t"] == np.float32(2e-3)) and np.all(got["max_t"] == np.float32(0.75))
    assert np.abs(got["dir"] - want["dir"]).max() <= DIR_BOUND_F32
    assert B.bake_dirs_within_sincos_ulps(v, f, rec, texel, smp, 11, got["dir"],
                                          fv_normals=fvn if use_fvn else None).all()
    # hemisphere, from float64 geometry: the wound normal, or the side of the interpolated face-varying normal
    r = rec[texel]
    tri = f[r["prim_id"]].astype(np.int64)
    p0, p1, p2 = (v[tri[:, k]].astype(np.float64) for k in range(3))
    n64 = np.cross(p1 - p0, p2 - p0)
    n64 /= np.linalg.norm(n64, axis=1)[:, None]
    if use_fvn:
        fn = fvn.reshape(-1, 3, 3)[r["prim_id"]].astype(np.float64)
        u, w = r["u"].astype(np.float64)[:, None], r["v"].astype(np.float64)[:, None]
        s = (1 - u - w) * fn[:, 0] + u * fn[:, 1] + w * fn[:, 2]
        side = np.sign((n64 * s).sum(axis=1))
        clear = np.abs((n64 * s).sum(axis=1)) > 1e-4 * np.linalg.norm(s, axis=1)
        n64, got_dir = n64[clear] * side[clear, None], got["dir"][clear]
    else:
        got_dir = got["dir"]
    cos = (got_dir.astype(np.float64) * n64).sum(axis=1)
    assert cos.min() > -1e-4, cos.min()  # the f32 normal against the f64 one, on grazing directions
    assert stats.kstest(np.clip(cos, 0, 1) ** 2, "uniform").pvalue >= KS_MIN_P
    if name == "terrain_reversed" and not use_fvn:  # reversed winding: the rays leave through the underside
        assert (got["dir"][:, 1] < 0).mean() > 0.9


def _unoccluded_counts(ref, rays, texel, n):
    _, mask = ref.traverse(rays, threads=8)
    return np.bincount(texel[mask == 0], minlength=n).astype(np.float32)


@pytest.mark.parametrize("name,flags", [("suzanne", 0), ("suzanne", 8), ("terrain", 0), ("terrain", 8),
                                        ("cornell", 0), ("cornell", 2)])
def test_bake_equals_the_reference_per_texel(name, flags):
    from oracle import orc

    rec, d_rec, world, v, f, fvn = _records(name)
    n_cov = int((rec["prim_id"] != MISS).sum())
    radius = 0.25 * float(np.linalg.norm(v.max(axis=0) - v.min(axis=0)))
    p = _bake_params(160, 128, spp=4, seed=7, ao=(1e-3, radius), flags=flags)
    rays = _export(world, d_rec, p, n_cov)
    texel, _ = B.bake_slots(rec, 4)
    want = _unoccluded_counts(orc.Reference().build(v, f), rays, texel, 160 * 128)
    accum, r = _bake(world, d_rec, p)
    got = accum.cpu().numpy()
    assert np.array_equal(got, want)
    assert (r.texels, r.ao_rays) == (n_cov, 4 * n_cov)
    assert r.ao_hits == 4 * n_cov - int(want.sum()) and 0 < r.ao_hits < r.ao_rays
    assert r.traverse_launches == 1 and r.launches >= 4


def test_bake_on_a_deep_adopted_tree_equals_the_reference():
    import torch

    from nanort_b200 import api, scenes as S
    from oracle import orc

    port = orc.Port()
    v, f = S.make_scene("terrain", n=128)
    nodes, idx, _ = port.build(v, f)
    world = api.BVHAccel()
    world.Adopt(nodes, idx, v, f)
    assert world.GetStatistics()["max_tree_depth"] + 2 > 64  # the 512-entry stack
    uv, uf = S.planar_uv(v, f)
    rec, _, _, _ = _raster(_accel(uv, uf), _raster_params(128, 128))
    d_rec = torch.from_numpy(rec.view(np.float32).reshape(-1, 4).copy()).cuda()
    n_cov = int((rec["prim_id"] != MISS).sum())
    for flags in (0, api.TRAVERSE_ANY_HIT):
        p = _bake_params(128, 128, spp=4, seed=9, ao=(1e-3, 2.0), flags=flags)
        rays = _export(world, d_rec, p, n_cov)
        texel, _ = B.bake_slots(rec, 4)
        want = _unoccluded_counts(orc.Reference().adopt(nodes, idx, v, f), rays, texel, 128 * 128)
        accum, r = _bake(world, d_rec, p)
        assert np.array_equal(accum.cpu().numpy(), want)
        assert r.ao_hits == 4 * n_cov - int(want.sum()) > 0


# ------------------------------------------------------------------ composition
def test_sample_ranges_compose_and_empty_texels_keep_their_value():
    import torch

    rec, d_rec, world, v, f, fvn = _records("cornell")
    empty = rec["prim_id"] == MISS
    assert empty.any()
    whole, _ = _bake(world, d_rec, _bake_params(160, 128, spp=8))
    parts = torch.full((160 * 128,), -7.0, dtype=torch.float32, device="cuda")
    _bake(world, d_rec, _bake_params(160, 128, spp=4, sample0=0), parts)
    _bake(world, d_rec, _bake_params(160, 128, spp=4, sample0=4), parts)
    w, pt = whole.cpu().numpy(), parts.cpu().numpy()
    assert np.all(pt[empty] == -7.0) and np.all(w[empty] == 0.0)
    assert np.array_equal(pt[~empty] + 7.0, w[~empty])


def test_launches_split_at_the_slot_cap_compose_exactly():
    import torch

    from nanort_b200 import api, scenes as S

    v, f = S.make_scene("terrain", n=32)
    uv, uf = S.planar_uv(v, f)
    W = H = 1024
    rec, _, _, n_cov = _raster(_accel(uv, uf), _raster_params(W, H))
    assert n_cov > 1000000
    d_rec = torch.from_numpy(rec.view(np.float32).reshape(-1, 4).copy()).cuda()
    world = _accel(v, f)
    per_launch = 0xFFFFFFFF // n_cov  # whole samples whose slots fit 32 bits
    spp = per_launch + 3
    flags = api.TRAVERSE_ANY_HIT
    whole, r = _bake(world, d_rec, _bake_params(W, H, spp, ao=(1e-3, 0.3), flags=flags))
    assert r.traverse_launches == 2 and r.ao_rays == spp * n_cov > 2**32
    parts = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r1 = _bake(world, d_rec, _bake_params(W, H, per_launch, ao=(1e-3, 0.3), flags=flags), parts)[1]
    r2 = _bake(world, d_rec, _bake_params(W, H, 3, sample0=per_launch, ao=(1e-3, 0.3), flags=flags), parts)[1]
    assert r1.traverse_launches == 1 and r2.traverse_launches == 1
    assert np.array_equal(whole.cpu().numpy(), parts.cpu().numpy())
    assert r.ao_hits == r1.ao_hits + r2.ao_hits > 0


def test_two_streams_on_one_accel_equal_serial_runs():
    import torch

    rec, d_rec, world, v, f, fvn = _records("suzanne")
    ps = [_bake_params(160, 128, spp=6, seed=s, ao=(1e-3, 1.0)) for s in (1, 2)]
    serial = [_bake(world, d_rec, p)[0].cpu().numpy() for p in ps]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    outs = [torch.zeros(160 * 128, dtype=torch.float32, device="cuda") for _ in ps]
    torch.cuda.synchronize()
    for _ in range(3):
        for o in outs:
            o.zero_()
        torch.cuda.synchronize()
        for p, o, s in zip(ps, outs, streams):
            world.BakeAO(d_rec.data_ptr(), p, o.data_ptr(), stream=s.cuda_stream, want_result=False)
        torch.cuda.synchronize()
        for o, want in zip(outs, serial):
            assert np.array_equal(o.cpu().numpy(), want)


def test_refusals_launch_nothing():
    import torch

    from nanort_b200 import api

    rec, d_rec, world, v, f, fvn = _records("cornell")
    accum = torch.full((160 * 128,), 2.5, dtype=torch.float32, device="cuda")
    spheres = api.BVHAccel()
    spheres.BuildSpheres(np.zeros((4, 3), np.float32) + np.arange(4, dtype=np.float32)[:, None], np.ones(4, np.float32))
    boxes = api.BVHAccel()
    boxes.BuildBoxes(np.float32([[0, 0, 0, 1, 1, 1], [2, 2, 2, 3, 3, 3]]))
    bad = rec.copy()
    bad["prim_id"][np.flatnonzero(bad["prim_id"] != MISS)[7]] = len(f) + 5
    d_bad = torch.from_numpy(bad.view(np.float32).reshape(-1, 4).copy()).cuda()
    ok = _bake_params(160, 128, spp=2)
    cases = [
        (world, 0, ok), (spheres, d_rec.data_ptr(), ok), (boxes, d_rec.data_ptr(), ok),
        (world, d_rec.data_ptr(), _bake_params(160, 128, spp=0)),
        (world, d_rec.data_ptr(), _bake_params(0, 128, spp=2)),
        (world, d_rec.data_ptr(), _bake_params(160, 128, spp=2, flags=api.TRAVERSE_CONFORMANCE)),
        (world, d_bad.data_ptr(), ok),
    ]
    rays = torch.zeros(160 * 128 * 2 * 9, dtype=torch.float32, device="cuda")
    for acc, ptr, p in cases:
        with pytest.raises(api.NanortB200Error, match="error -1"):
            api._check(api.lib().nrt_bake_ao_device(acc._h, ptr or None, p, accum.data_ptr(), None, None))
        with pytest.raises(api.NanortB200Error, match="error -1"):
            acc.ExportBakeRays(ptr or None, p, rays.data_ptr(), len(rays) // 9)
    with pytest.raises(api.NanortB200Error, match="error -1"):
        api._check(api.lib().nrt_bake_ao_device(world._h, d_rec.data_ptr(), None, accum.data_ptr(), None, None))
    with pytest.raises(api.NanortB200Error, match="error -1"):
        world.BakeAO(d_rec.data_ptr(), ok, 0)
    with pytest.raises(api.NanortB200Error, match="error -1"):  # the rays do not fit
        world.ExportBakeRays(d_rec.data_ptr(), ok, rays.data_ptr(), 10)
    torch.cuda.synchronize()
    assert torch.all(accum == 2.5) and torch.all(rays == 0)
    # the texel cast: a world accel of another face count, AOVs without a world accel, no normals for the normal AOV
    v2, f2, uv2, uf2, fvn2 = mesh("cornell")
    uv_acc = _accel(uv2, uf2)
    out = torch.zeros((160 * 128, 4), dtype=torch.float32, device="cuda")
    small = _accel(v2, f2[:-1])
    for kw in (dict(world=small), dict(d_position_ptr=out.data_ptr()),
               dict(world=world, d_normal_ptr=out.data_ptr())):
        with pytest.raises(api.NanortB200Error, match="error -1"):
            uv_acc.UVRaster(_raster_params(160, 128), out.data_ptr(), **kw)
    with pytest.raises(api.NanortB200Error, match="error -1"):
        spheres.UVRaster(_raster_params(160, 128), out.data_ptr())
    torch.cuda.synchronize()
    assert torch.all(out == 0)
