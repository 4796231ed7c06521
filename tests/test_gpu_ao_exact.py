"""The primary + 1-bounce AO pass, ray by ray and pixel by pixel, against the host model of tests/ao_model.py:
  * exported camera rays are bit-exact to the f32 model;
  * exported AO rays are exactly one per primary hit, matched to their slot by the bits of their origin; the origin
    and the [min_t, max_t] range are bit-exact, the direction equals the f32 model up to sincosf's ulps and the f64
    ideal within 1e-5 away from sliver triangles; directions are unit, face the viewer-side hemisphere, start on
    the hit triangle and are cosine distributed;
  * the frame is exact per pixel: primary misses + AO rays the conformance walk finds unoccluded, for the exported,
    fused, AO_UNFUSED and ANY_HIT passes;
  * progressive samples, tile shards, packed tiles, nrt_render_ao_sharded at world 1 and the wave bookkeeping compose
    exactly;
  * the two-level scene pass equals the model per pixel up to borderline samples."""
import numpy as np
import pytest

import ao_model as M
from helpers import assert_parity, compare_hits

pytestmark = pytest.mark.gpu

# Direction bound against the f32 model.  The device differs from the model only in sincosf, <= 2 ulp (CUDA C
# Programming Guide, single-precision functions) against the model's <= 0.5 ulp, so |d cs|, |d sn| <= 2.5 * 2^-24
# (|cs|, |sn| <= 1).  The exact direction is 1-Lipschitz in (cs, sn) (the r <= 1 scaling, unit t1 / t2, and the
# normalisation of a unit vector do not amplify), which bounds the change of the exact result by sqrt(2) * 2.5 * 2^-24
# = 2.1e-7.  Each float32 evaluation then adds its own forward error: about 12 roundings on values of magnitude <= ~1
# (lx, ly, three products and two sums per component, squares, sums, sqrt, reciprocal, final product), at most
# 12 * 2^-24 = 7.2e-7 each, twice.  Total <= 2.1e-7 + 1.43e-6 < 1.7e-6.  The stronger check is bit equality with the
# model evaluated at sin / cos moved by at most 3 ulp (`M.dirs_within_sincos_ulps`).
DIR_BOUND_F32 = 1.7e-6
# Against the f64 ideal: the f32 normal's error is about 3 * 2^-24 * cond per component (cancellation in the cross
# product, cond = 1 / sine of the corner angle); with the f32 tail's 1.7e-6 that stays below 1e-5 for cond <= 16.
# Triangles with cond > 16 are slivers whose f32 normal is ill-conditioned: excluded and counted.
DIR_TOL_F64 = 1e-5
SLIVER_COND = 16.0
# KS tests of cos^2(theta) and the azimuth: the rays are deterministic, so is the p-value.  Observed on an H100:
# p >= 0.03 over the configurations below.
KS_MIN_P = 1e-3
# Two-level scene pass: total |frame - model| over all pixels, every unit explained by a borderline sample (none
# observed on the two scenes below, H100 80GB HBM3 at 400 W).
SCENE_BORDERLINE_BUDGET = 4

_ACCELS = {}


def _scene(name, flags, reversed_winding=False):
    """(verts, faces, accel) per scene and build flavour, built once per session.  reversed_winding: every triangle's
    cross(e1, e2) points away from the camera, so every AO normal is flipped towards the viewer."""
    from nanort_b200 import api, scenes as S

    key = (name, flags, reversed_winding)
    if key not in _ACCELS:
        kw = {"sphere_grid": dict(nx=4, nz=4), "terrain": dict(n=96), "cornell": {}}[name]
        v, f = S.make_scene(name, **kw)
        if reversed_winding:
            f = np.ascontiguousarray(f[:, [0, 2, 1]])
        acc = api.BVHAccel()
        acc.Build(len(f), v, f, flags=flags)
        _ACCELS[key] = (v, f, acc)
    return _ACCELS[key]


def _radius(acc):
    bmin, bmax = acc.BoundingBox()
    return 0.25 * float(np.linalg.norm(bmax - bmin))


def _params(api, cam, W, H, spp, tile, sample0=0, seed=1, ao=(1e-3, 1.0), flags=0, shard=0, n_shards=1):
    p = api.AoParams()
    for i in range(12):
        p.cam[i] = float(cam[i])
    p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, sample0, seed
    p.tile_w, p.tile_h, p.shard, p.n_shards = tile[0], tile[1], shard, n_shards
    p.ray_min_t, p.ray_max_t, p.ao_min_t, p.ao_max_t = 1e-3, 1e30, ao[0], ao[1]
    p.flags = flags
    return p


def _render(acc, p, W, H):
    import torch

    accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r = acc.RenderAO(p, accum.data_ptr())
    return accum.cpu().numpy(), r


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _match_by_origin(dev_org, dev_dir, mod_org, mod_dir):
    """Indices m with dev ray j <-> model ray m[j]: sort both sides by origin bits, then direction bits.  Asserts that
    the origins are the same multiset bit for bit: one AO ray per primary hit, no extras, none missing."""
    assert len(dev_org) == len(mod_org), (len(dev_org), len(mod_org))
    do, dd, mo, md = _bits(dev_org), _bits(dev_dir), _bits(mod_org), _bits(mod_dir)
    od = np.lexsort((dd[:, 2], dd[:, 1], dd[:, 0], do[:, 2], do[:, 1], do[:, 0]))
    om = np.lexsort((md[:, 2], md[:, 1], md[:, 0], mo[:, 2], mo[:, 1], mo[:, 0]))
    assert np.array_equal(do[od], mo[om]), "AO origins are not bit-exact, one per primary hit"
    m = np.empty(len(od), np.int64)
    m[od] = om
    return m


def _tie_alternatives(port, v, f, ray, prim, t):
    """Triangles other than `prim` that the reference arithmetic hits at exactly the same t (exact-t ties: the device
    may have picked any of them).  Candidates: triangles sharing a vertex with `prim`, or lying in its plane."""
    fv = f[prim]
    cand = np.flatnonzero(np.isin(f, fv).any(axis=1))
    if len(f) <= 4096:
        cand = np.arange(len(f))
    out = []
    for c in cand:
        if c == prim:
            continue
        ok, h = port.test_prim(v, f, ray, int(c))
        if ok and _bits(h["t"]) == _bits(t):
            out.append(int(c))
    return out


def _property_checks(v, f, cam, d, t, prim, dirs, stats):
    """Checks that do not come from restating the formula: unit length, viewer-side hemisphere, origin on the hit
    triangle (float64), cosine distribution by KS tests."""
    from scipy import stats as sst

    dirs64 = dirs.astype(np.float64)
    nrm = np.linalg.norm(dirs64, axis=1)
    assert np.all(np.abs(nrm - 1.0) <= 1e-6), np.abs(nrm - 1.0).max()
    tri = v[f[prim]].astype(np.float64)
    e1, e2 = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    n = np.cross(e1, e2)
    n /= np.linalg.norm(n, axis=1)[:, None]
    d64 = d.astype(np.float64)
    cosv = (n * d64).sum(axis=1)
    n_viewer = np.where((cosv > 0)[:, None], -n, n)
    graze = np.abs(cosv) < 1e-6  # the f32 flip may legitimately choose the other side
    c = (dirs64 * n_viewer).sum(axis=1)
    assert np.all(c[~graze] >= -1e-6), c[~graze].min()
    stats["grazing"] = int(graze.sum())
    # the origin lies on the hit triangle: plane distance and barycentrics, scale-relative
    o = np.asarray(cam[:3], np.float64)
    P = o + d64 * t.astype(np.float64)[:, None]
    scale = np.abs(o).max() + t + np.abs(tri).max(axis=(1, 2))
    q = P - tri[:, 0]
    assert np.all(np.abs((q * n).sum(axis=1)) <= 1e-5 * scale)
    g11, g12, g22 = (e1 * e1).sum(1), (e1 * e2).sum(1), (e2 * e2).sum(1)
    r1, r2 = (q * e1).sum(1), (q * e2).sum(1)
    det = g11 * g22 - g12 * g12
    beta, gamma = (g22 * r1 - g12 * r2) / det, (g11 * r2 - g12 * r1) / det
    longest = np.sqrt(np.maximum(np.maximum(g11, g22), ((e2 - e1) ** 2).sum(1)))
    tol_b = 1e-5 * scale * longest / np.sqrt(det)  # distance tolerance over the smallest altitude
    assert np.all(beta >= -tol_b) and np.all(gamma >= -tol_b) and np.all(beta + gamma <= 1 + tol_b)
    # cosine-weighted: cos^2(theta) ~ U(0, 1); azimuth ~ U(0, 2 pi) about any per-ray basis
    keep = ~graze
    p_cos = sst.kstest(c[keep] ** 2, "uniform").pvalue
    nv = n_viewer[keep]
    ax = np.where((np.abs(nv[:, 0]) < 0.9)[:, None], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0])
    b1 = np.cross(nv, ax)
    b1 /= np.linalg.norm(b1, axis=1)[:, None]
    b2 = np.cross(nv, b1)
    dk = dirs64[keep]
    phi = np.arctan2((dk * b2).sum(1), (dk * b1).sum(1)) / (2 * np.pi) + 0.5
    p_phi = sst.kstest(phi, "uniform").pvalue
    stats["ks_p_cos2"], stats["ks_p_azimuth"] = float(p_cos), float(p_phi)
    assert p_cos >= KS_MIN_P and p_phi >= KS_MIN_P, (p_cos, p_phi)


def _check_exported_pass(port, v, f, acc, cam, p, light=False, oracle_stride=7):
    """Runs the exported (unfused) pass of `p` and checks it ray by ray against the model.  Returns (the exported
    frame, the expected frame, stats).  light: only camera rays, origin matching, ranges and the frame (huge passes)."""
    import torch
    from nanort_b200 import api, scenes as S

    W, H, spp, seed = p.width, p.height, p.spp, p.seed
    pix, smp = M.slots(W, H, p.tile_w, p.tile_h, spp, p.sample0, p.shard, p.n_shards)
    n_slots = len(pix)
    d_p = torch.empty(n_slots * 36, dtype=torch.uint8, device="cuda")
    d_a = torch.empty(n_slots * 36, dtype=torch.uint8, device="cuda")
    accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    n_p, n_a = acc.ExportAOWorkload(p, accum.data_ptr(), d_p.data_ptr(), d_a.data_ptr())
    frame = accum.cpu().numpy()
    valid = pix >= 0
    assert n_p == int(valid.sum())
    stats = {"primary": int(n_p), "ao": int(n_a)}

    # camera rays: bit-exact; padding slots retire at the root
    prim = d_p.cpu().numpy().view(S.RAY_DTYPE)
    del d_p
    assert np.all(prim["max_t"][~valid] < 0)
    pr = prim[valid]
    pv, sv = pix[valid], smp[valid]
    d = M.camera_dirs(cam, W, H, seed, pv, sv)
    assert np.array_equal(_bits(pr["dir"]), _bits(d)), "camera directions are not bit-exact"
    assert np.array_equal(_bits(pr["org"]), np.broadcast_to(_bits(np.asarray(cam[:3], np.float32)), pr["org"].shape))
    assert np.all(_bits(pr["min_t"]) == _bits(np.float32(p.ray_min_t)))
    assert np.all(_bits(pr["max_t"]) == _bits(np.float32(p.ray_max_t)))

    # primary hits: fast == conformance walk (t bit for bit), oracle on a sample
    hc, mc = acc.Traverse(pr, flags=api.TRAVERSE_CONFORMANCE)
    hf, mf = (hc, mc) if light else acc.Traverse(pr)
    assert np.array_equal(mf, mc)
    hit = mf.astype(bool)
    assert np.array_equal(_bits(hf["t"][hit]), _bits(hc["t"][hit]))
    nodes, idx = acc.GetNodes(), acc.GetIndices()
    sel = np.arange(0, len(pr), oracle_stride * (50 if light else 1))
    wh, wm = port.traverse(nodes, idx, v, f, pr[sel], threads=8)
    assert_parity(compare_hits(port, v, f, pr[sel], hc[sel], mc[sel], wh, wm), allow_ties=False)

    # AO rays: one per primary hit, matched by origin
    ao = d_a[: n_a * 36].cpu().numpy().view(S.RAY_DTYPE)
    del d_a
    src = np.flatnonzero(hit)
    tsrc, psrc = hf["t"][src], hf["prim_id"][src]
    P, w, n32, sg = M.ao_rays_f32(v, f, cam[:3], d[src], tsrc, psrc, pv[src], sv[src], seed)
    m = _match_by_origin(ao["org"], ao["dir"], P, w)
    s = src[m]  # primary slot (into pr) of every device AO ray
    assert np.all(_bits(ao["min_t"]) == _bits(np.float32(p.ao_min_t)))
    assert np.all(_bits(ao["max_t"]) == _bits(np.float32(p.ao_max_t)))
    stats["ties"] = 0
    if not light:
        prim_used = psrc[m].copy()
        ok = M.dirs_within_sincos_ulps(v, f, d[s], prim_used, pv[s], sv[s], seed, ao["dir"])
        for j in np.flatnonzero(~ok):  # exact-t ties: the device may have used another triangle at the same t
            for c in _tie_alternatives(port, v, f, pr[s[j]], int(prim_used[j]), hf["t"][s[j]]):
                cj = np.array([c])
                if M.dirs_within_sincos_ulps(v, f, d[s[j]:s[j] + 1], cj, pv[s[j]:s[j] + 1], sv[s[j]:s[j] + 1], seed,
                                             ao["dir"][j:j + 1])[0]:
                    prim_used[j], ok[j] = c, True
                    stats["ties"] += 1
                    break
        assert ok.all(), f"{int((~ok).sum())} AO directions differ from the model by more than sincosf's ulps"
        _, w_used, n_used, sg_used = M.ao_rays_f32(v, f, cam[:3], d[s], hf["t"][s], prim_used, pv[s], sv[s], seed)
        err32 = np.abs(ao["dir"].astype(np.float64) - w_used.astype(np.float64)).max(axis=1)
        assert err32.max() <= DIR_BOUND_F32, err32.max()
        _, w64, _, cond = M.ideal_f64(v, f, cam[:3], d[s], hf["t"][s], prim_used, pv[s], sv[s], seed, n_used, sg_used)
        err64 = np.abs(ao["dir"].astype(np.float64) - w64).max(axis=1)
        sliver = cond > SLIVER_COND
        assert err64[~sliver].max() <= DIR_TOL_F64, err64[~sliver].max()
        assert sliver.mean() <= 0.01
        stats.update(err_f32=float(err32.max()), err_f64=float(err64[~sliver].max()), slivers=int(sliver.sum()))
        _property_checks(v, f, cam, d[s], hf["t"][s], prim_used, ao["dir"], stats)

    # occlusion: conformance walk on the GPU; the fast kernel agrees; the oracle on a sample + every disagreement
    ch, cm = acc.Traverse(ao, flags=api.TRAVERSE_CONFORMANCE)
    fm = cm if light else acc.Traverse(ao)[1]  # huge passes: the fused frame below is the fast kernel's answer
    disagree = np.flatnonzero(cm != fm)
    assert len(disagree) == 0, disagree[:10]
    sel = np.union1d(np.arange(0, len(ao), oracle_stride * (50 if light else 1)), disagree)
    wh, wm = port.traverse(nodes, idx, v, f, ao[sel], threads=8)
    assert_parity(compare_hits(port, v, f, ao[sel], ch[sel], cm[sel], wh, wm), max_near_ties=8)
    stats["occluded"] = int(cm.sum())

    expected = (np.bincount(pv[~hit], minlength=W * H) + np.bincount(pv[s[cm == 0]], minlength=W * H)).astype(np.float32)
    assert np.array_equal(frame, expected), f"{int((frame != expected).sum())} pixels differ from the expected frame"
    return frame, expected, stats


# (scene, build, W, H, tile, spp, sample0, seed, ao_min_t, ao_max_t); ao_max_t None = a quarter of the diagonal
CONFIGS = [
    ("cornell", "prod", 203, 101, (8, 4), 1, 0, 1, 1e-3, None),
    ("cornell", "ref", 37, 9, (40, 20), 3, 7, 0xFFFFFFFF, 0.0, 1e30),  # one tile larger than the image
    ("sphere_grid", "prod", 203, 101, (16, 12), 3, 7, 0xFFFFFFFF, 0.0, None),  # self-hits
    ("terrain", "prod", 203, 101, (40, 20), 5, 0, 1, 1e-3, 1e30),
    ("sphere_grid", "ref", 203, 101, (64, 8), 3, 0, 1, 1e-3, 1e-6),  # nothing occluded
    ("terrain", "ref", 37, 9, (64, 8), 1, 7, 0xFFFFFFFF, 0.0, None),
    # the scenes' triangles face the camera where it sees them; reversed, the viewer flip of the normal is exercised
    ("cornell", "prod-reversed", 203, 101, (16, 12), 3, 7, 1, 1e-3, None),
    ("terrain", "ref-reversed", 96, 40, (8, 4), 2, 0, 0xFFFFFFFF, 0.0, None),
]


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: f"{c[0]}-{c[1]}-{c[2]}x{c[3]}-t{c[4][0]}x{c[4][1]}-spp{c[5]}"
                                                       f"-s{c[6]}-seed{c[7]:x}-ao{c[8]:g}-{c[9] or 'r'}")
def test_exported_pass_matches_the_model_ray_by_ray(port, cfg):
    from nanort_b200 import api, scenes as S

    name, build, W, H, tile, spp, sample0, seed, ao_min, ao_max = cfg
    v, f, acc = _scene(name, api.BUILD_FAST if build.startswith("prod") else api.BUILD_REFERENCE_TREE,
                       reversed_winding=build.endswith("reversed"))
    cam = S.scene_camera(name, W, H)
    ao = (ao_min, _radius(acc) if ao_max is None else ao_max)
    p = _params(api, cam, W, H, spp, tile, sample0, seed, ao)
    frame, expected, stats = _check_exported_pass(port, v, f, acc, cam, p)
    print("\nAO_EXACT", cfg, stats)
    assert stats["primary"] == W * H * spp
    if ao[1] < ao[0]:
        assert stats["occluded"] == 0 and np.all(frame == spp)
    else:
        assert stats["occluded"] > 0
    # the fused, AO_UNFUSED and ANY_HIT passes of the same parameters give the same frame, per pixel
    for flags in (0, api.AO_UNFUSED, api.TRAVERSE_ANY_HIT):
        fr, r = _render(acc, _params(api, cam, W, H, spp, tile, sample0, seed, ao, flags=flags), W, H)
        assert np.array_equal(fr, expected), (flags, int((fr != expected).sum()))
        assert (r.primary_rays, r.ao_rays, r.ao_hits) == (stats["primary"], stats["ao"], stats["occluded"])


def test_progressive_samples_add_up():
    """sample0 shifts the RNG sample index of the camera and AO rays: frame(spp = a + b) = frame(a, sample0 = 0) +
    frame(b, sample0 = a), exactly, fused and unfused."""
    from nanort_b200 import api, scenes as S

    v, f, acc = _scene("sphere_grid", api.BUILD_FAST)
    W, H, tile, a, b = 203, 101, (16, 12), 2, 3
    cam = S.scene_camera("sphere_grid", W, H)
    ao = (1e-3, _radius(acc))
    for flags in (0, api.AO_UNFUSED):
        whole, _ = _render(acc, _params(api, cam, W, H, a + b, tile, 0, 5, ao, flags=flags), W, H)
        first, _ = _render(acc, _params(api, cam, W, H, a, tile, 0, 5, ao, flags=flags), W, H)
        rest, _ = _render(acc, _params(api, cam, W, H, b, tile, a, 5, ao, flags=flags), W, H)
        assert np.array_equal(whole, first + rest), flags


@pytest.mark.parametrize("n_shards,tile", [(3, (40, 20)), (4, (8, 4)), (4, (64, 8))])
def test_shards_and_packed_tiles(n_shards, tile):
    """Each shard touches only its own pixels and the shard frames add up to the single-shard frame; the packed
    (tile-major) accumulation of a shard equals dist.pack_own_tiles of its row-major frame bit for bit, padding of
    partial tiles included; AO_UNFUSED | AO_PACKED_TILES is refused."""
    import ctypes as C

    import torch
    from nanort_b200 import api, dist as nd, scenes as S

    v, f, acc = _scene("sphere_grid", api.BUILD_FAST)
    W, H, spp = 203, 101, 2
    cam = S.scene_camera("sphere_grid", W, H)
    ao = (1e-3, _radius(acc))
    full, r_full = _render(acc, _params(api, cam, W, H, spp, tile, 3, 1, ao), W, H)
    total = np.zeros_like(full)
    rays = 0
    n_packed = nd.packed_slot_floats(W, H, tile[0], tile[1], n_shards)
    for shard in range(n_shards):
        ps = _params(api, cam, W, H, spp, tile, 3, 1, ao, shard=shard, n_shards=n_shards)
        part, r = _render(acc, ps, W, H)
        mine = nd.shard_pixels(W, H, tile[0], tile[1], shard, n_shards)
        other = np.ones(W * H, bool)
        other[mine] = False
        assert np.all(part[other] == 0), "a shard only touches its own pixels"
        assert r.primary_rays == len(mine) * spp
        ps.flags = api.AO_UNFUSED
        assert np.array_equal(_render(acc, ps, W, H)[0], part)
        total += part
        rays += r.primary_rays + r.ao_rays
        # packed tiles
        ps.flags = api.AO_PACKED_TILES
        buf = torch.zeros(n_packed, dtype=torch.float32, device="cuda")
        rp = acc.RenderAO(ps, buf.data_ptr())
        want = nd.pack_own_tiles(part, W, H, tile[0], tile[1], shard, n_shards)
        got = buf.cpu().numpy()
        assert np.array_equal(got, want)
        pad = np.ones(n_packed, bool)
        pad[nd.pack_own_tiles(np.arange(W * H, dtype=np.int64) + 1, W, H, tile[0], tile[1], shard, n_shards) > 0] = False
        assert np.all(got[pad] == 0) and (rp.primary_rays, rp.ao_rays) == (r.primary_rays, r.ao_rays)
        ps.flags = api.AO_PACKED_TILES | api.AO_UNFUSED
        rc = api.lib().nrt_render_ao_device(acc._h, C.byref(ps), C.c_void_p(buf.data_ptr()), None, None)
        assert rc == -1  # NRT_ERR_INVALID
    assert np.array_equal(total, full)
    assert rays == r_full.primary_rays + r_full.ao_rays


def test_sharded_pass_at_world_one_unpacks_partial_tiles():
    """nrt_render_ao_sharded with a communicator of one rank: packed accumulation + unpack_tiles_kernel, no
    all-gather; the frame equals RenderAO's, and every pixel is written (the frame starts as NaN)."""
    import torch
    from nanort_b200 import api, scenes as S

    v, f, acc = _scene("terrain", api.BUILD_FAST)
    W, H, spp, tile = 203, 101, 2, (40, 20)
    cam = S.scene_camera("terrain", W, H)
    p = _params(api, cam, W, H, spp, tile, 0, 1, (1e-3, _radius(acc)))
    want, r_want = _render(acc, p, W, H)
    try:
        comm = api.Comm(api.Comm.unique_id(), 0, 1)
    except api.NanortB200Error as e:
        pytest.skip(str(e))
    try:
        frame = torch.full((W * H,), float("nan"), dtype=torch.float32, device="cuda")
        r = comm.RenderAO(acc, p, frame.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(frame.cpu().numpy(), want)
        assert r.launches == r_want.launches + 1
        assert (r.primary_rays, r.ao_rays, r.ao_hits) == (r_want.primary_rays, r_want.ao_rays, r_want.ao_hits)
    finally:
        comm.free()


@pytest.mark.parametrize("W,H,tile,spp,waves", [(300, 200, (256, 64), 257, 3), (128, 64, (64, 64), 4097, 2)])
def test_wave_bookkeeping(port, W, H, tile, spp, waves):
    """300x200 in 256x64 tiles at 257 spp: 3 tiles of 4.2 M slots per 16 Mi-slot wave, waves of 3 + 3 + 2 tiles ending
    after partial tiles (the host-side valid-slot count).  128x64 in 64x64 tiles at 4097 spp: one tile alone exceeds a
    wave, one tile per wave.  Wave count, primary count and the per-pixel frame are exact."""
    from nanort_b200 import api, scenes as S

    v, f, acc = _scene("cornell", api.BUILD_FAST)
    cam = S.scene_camera("cornell", W, H)
    p = _params(api, cam, W, H, spp, tile, 0, 1, (1e-3, _radius(acc)))
    fused, r = _render(acc, p, W, H)
    assert r.traverse_launches == 2 * waves
    assert r.primary_rays == W * H * spp
    frame, expected, stats = _check_exported_pass(port, v, f, acc, cam, p, light=True)
    print("\nAO_WAVES", (W, H, tile, spp), stats)
    assert np.array_equal(fused, expected)
    assert (r.ao_rays, r.ao_hits) == (stats["ao"], stats["occluded"])


# ------------------------------------------------------------------ two-level scene pass
def _scene_instances(kind):
    from nanort_b200 import scenes as S

    if kind == "mixed":
        return S.instances_mixed()
    grid = S.instances_grid(2, 2, base=S.sphere_grid(nx=2, nz=2))
    return [(v, f, S.xform(translate=tuple(x[3, :3] * 0.5), scale=(1.3, 0.8, 1.1), yaw=0.4 + 0.3 * k, pitch=0.2))
            for k, (v, f, x) in enumerate(grid)]


@pytest.mark.parametrize("kind", ["mixed", "grid"])
def test_scene_pass_matches_the_model_up_to_borderline_samples(kind):
    """Scene.RenderAO with the conformance walk against the model driven by the oracle scene: camera rays of the model,
    primary hits of orc.PortScene (bit-exact to the conformance kernel), world normal from the instance matrix, origin
    lifted by ao_min_t along the viewer-facing normal, occluded iff the oracle's t < ao_max_t.  A differing pixel must
    be explained by borderline samples: ones whose occlusion flips when the model direction moves by 4 ulp."""
    import torch
    from nanort_b200 import api, scenes as S
    from oracle import orc
    from test_gpu_scene import _gpu_scene

    insts = _scene_instances(kind)
    port = orc.PortScene(insts, cpp11=True)
    sc = _gpu_scene(insts, api.BUILD_REFERENCE_TREE, api.BUILD_REFERENCE_TREE)
    xf = sc.InstanceStates()["xform"]
    assert xf.tobytes() == port.sg["xform"].tobytes()
    lo, hi = sc.GetBoundingBox()
    W, H, spp, tile, sample0, seed = 160, 96, 2, (16, 12), 7, 0xFFFFFFFF
    ctr = 0.5 * (lo + hi)
    cam = S.look_at(ctr + np.array([0.0, 0.25, 0.5]) * float(np.linalg.norm(hi - lo)), ctr, aspect=W / H)
    radius = 0.2 * float(np.linalg.norm(hi - lo))
    p = _params(api, cam, W, H, spp, tile, sample0, seed, (1e-3, radius), flags=api.TRAVERSE_CONFORMANCE)
    accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r = sc.RenderAO(p, accum.data_ptr())
    frame = accum.cpu().numpy()

    pix, smp = M.slots(W, H, tile[0], tile[1], spp, sample0)
    valid = pix >= 0
    pv, sv = pix[valid], smp[valid]
    rays = np.zeros(len(pv), S.RAY_DTYPE)
    rays["org"] = cam[:3]
    rays["dir"] = M.camera_dirs(cam, W, H, seed, pv, sv)
    rays["min_t"], rays["max_t"] = p.ray_min_t, p.ray_max_t
    ph, pm = port.traverse(rays, threads=8)
    gh, gm = sc.Traverse(rays, flags=api.TRAVERSE_CONFORMANCE)
    assert np.array_equal(pm, gm) and ph[pm == 1].tobytes() == gh[gm == 1].tobytes()
    hit = pm == 1
    src = np.flatnonzero(hit)
    ao = M.scene_ao_rays_f32(insts, xf, ph[src], rays["dir"][src], pv[src], sv[src], seed, p.ao_min_t, p.ao_max_t)
    ah, am = port.traverse(ao, threads=8)
    occ = (am == 1) & (ah["t"] < np.float32(p.ao_max_t))
    model = (np.bincount(pv[~hit], minlength=W * H) + np.bincount(pv[src[~occ]], minlength=W * H)).astype(np.float32)
    assert r.primary_rays == W * H * spp and r.ao_rays == len(src) and 0 < r.ao_hits < r.ao_rays

    diff = frame - model
    bad = np.flatnonzero(diff != 0)
    borderline_total = 0
    if len(bad):
        j = np.flatnonzero(np.isin(pv[src], bad))  # AO rays of the differing pixels
        border = np.zeros(len(j), bool)
        base_dir = ao["dir"][j]
        for sx in (-4, 4):
            for sy in (-4, 4):
                for sz in (-4, 4):
                    nudged = ao[j].copy()
                    nudged["dir"] = np.stack([M._nudge(base_dir[:, k], s) for k, s in enumerate((sx, sy, sz))], axis=1)
                    nh, nm = port.traverse(nudged, threads=8)
                    border |= ((nm == 1) & (nh["t"] < np.float32(p.ao_max_t))) != occ[j]
        per_pix = np.bincount(pv[src[j]][border], minlength=W * H)
        assert np.all(np.abs(diff[bad]) <= per_pix[bad]), "a pixel differs without a borderline sample"
        borderline_total = int(np.abs(diff[bad]).sum())
    print("\nAO_SCENE", kind, {"pixels_differing": len(bad), "borderline_mismatches": borderline_total,
                               "ao_rays": len(src)})
    assert borderline_total <= SCENE_BORDERLINE_BUDGET

    # the production walk against the conformance walk: the same frame up to exact-distance ties
    p.flags = 0
    a0 = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    r0 = sc.RenderAO(p, a0.data_ptr())
    assert r0.primary_rays == r.primary_rays and abs(int(r0.ao_rays) - int(r.ao_rays)) <= 4
    assert float((a0 != accum).double().mean().item()) < 1e-3
