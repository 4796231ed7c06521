"""Slot bookkeeping of the two passes that run in waves of ray slots: the path-tracing pass (csrc/path.cu,
nrt_render_path_device) and the two-level scene AO pass (csrc/scene.cu, nrt_scene_render_ao_device).  A frame must not
depend on how its (pixel, sample) set is split into waves, tile shards, tile sizes and sample ranges.

Path pass, on a tie-free Cornell box (`untied`): no two triangles share an edge or a plane, so every radiance hit -- and
with it every decision and contribution of a path -- depends on (pixel, sample, seed) only, not on how the slots were
split and queued; the shadow pass's "any hit below max_t" does not depend on order either.  Ray counts are therefore
exact across splits.  The frame is a sum of float atomicAdds whose order does change: every term is non-negative and a
path adds at most one term per bounce, so a pixel holds at most m = spp * max_bounces terms and two orders agree within
    |a - b| <= 2 * m * 2^-24 * max(a, b) * 1.01.
Scene AO pass, conformance walk: deterministic per ray and a frame of 1.0f terms, so every comparison is bit-exact.

The wave counts below follow from path.cu (kMaxWave = 8 Mi slots; waves are whole tiles, at least one) and scene.cu
(whole tiles of at most 1 << 22 slots, at least one); each test asserts them through traverse_launches."""
import numpy as np
import pytest

import ao_model as M

pytestmark = pytest.mark.gpu

PATH_MAX_WAVE = 8 << 20  # path.cu: kMaxWave
SCENE_MAX_WAVE = 1 << 22  # scene.cu: ray slots per wave
U = 2.0 ** -24
SEED = 7
# config (a): 16 x 88 tiles of 64 x 8 (partial on the right and at the bottom), 6144 slots per tile at 12 spp,
# 8 Mi // 6144 = 1365 tiles per wave -> waves of 1365 + 43 tiles
A = dict(W=1000, H=700, spp=12, bounces=10, tile=(64, 8))
A_WAVE1 = 1365 * 64 * 8 * 12  # first slot of the second wave: 8 386 560


def narrow_camera():
    """The Cornell camera with a field of view narrowed to the box's opening: every pixel, the image's edges included,
    sees the inside of the box."""
    from nanort_b200 import scenes as S

    cam = S.scene_camera("cornell", 1, 1).copy()
    cam[3:9] *= np.float32(0.6)
    return cam


def _n_tiles(W, H, tile, shard=0, n_shards=1):
    n = (-(-W // tile[0])) * (-(-H // tile[1]))
    return (n - shard + n_shards - 1) // n_shards if n > shard else 0


def path_waves(W, H, tile, spp, shard=0, n_shards=1):
    per_tile = tile[0] * tile[1] * spp
    slots = _n_tiles(W, H, tile, shard, n_shards) * per_tile
    cap = min(slots, max(1, PATH_MAX_WAVE // per_tile) * per_tile)
    return -(-slots // cap) if slots else 0


def scene_waves(W, H, tile, spp, shard=0, n_shards=1):
    per_tile = tile[0] * tile[1] * spp
    slots = _n_tiles(W, H, tile, shard, n_shards) * per_tile
    wave = max(per_tile, (SCENE_MAX_WAVE // per_tile) * per_tile)
    return -(-slots // wave) if slots else 0


def _print(name, stats):
    print("\nPASS_SLOTS", name, stats)


# ------------------------------------------------------------------ the tie-free path scene
def untied_cornell():
    """S.cornell_with_materials() with every triangle on its own three vertices, shrunk towards its centroid by a
    relative 1e-3 (no shared edges) and moved along its own normal by (1 + k mod 7) * 1e-4 of the scene's extent (the box
    bottoms leave the floor plane).  Face order, material ids and the emissive faces are unchanged.

    The second light triangle is wound the other way.  Emission takes the loader's flat normal and next-event
    estimation the opposite one (main.cc:306-312 and 337-392), so a one-sided light either shines into the room when hit
    or when sampled, never both; with one triangle of each winding, both kinds of term reach the frame."""
    from nanort_b200 import scenes as S

    v, f, mats, ids, emissive = S.cornell_with_materials()
    f = f.copy()
    f[emissive[-1]] = f[emissive[-1]][[0, 2, 1]]
    tri = v[f].astype(np.float64)
    c = tri.mean(axis=1, keepdims=True)
    tri = c + (tri - c) * (1.0 - 1e-3)
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    n /= np.linalg.norm(n, axis=1)[:, None]
    ext = float(np.linalg.norm(v.max(axis=0) - v.min(axis=0)))
    k = np.arange(len(f))
    tri += (n * ((1 + k % 7) * 1e-4 * ext)[:, None])[:, None, :]
    v2 = np.ascontiguousarray(tri.reshape(-1, 3), np.float32)
    f2 = np.arange(3 * len(f), dtype=np.uint32).reshape(-1, 3)
    # no two triangles left in one plane: parallel ones sit at least 1e-5 * extent apart
    t32 = v2[f2].astype(np.float64)
    n32 = np.cross(t32[:, 1] - t32[:, 0], t32[:, 2] - t32[:, 0])
    n32 /= np.linalg.norm(n32, axis=1)[:, None]
    for i in range(len(f)):
        par = np.abs(n32 @ n32[i]) > 1.0 - 1e-9
        par[i] = False
        gap = np.abs((t32[par, 0] - t32[i, 0]) @ n32[i])
        assert np.all(gap > 1e-5 * ext), (i, np.flatnonzero(par), gap)
    return v2, f2, mats, ids, emissive


@pytest.fixture(scope="module")
def untied():
    return untied_cornell()


class _PathPass:
    """RenderPath on the tie-free scene with one accel; frames come back as float64 [W * H, 3]."""

    def __init__(self, scene):
        import torch
        from nanort_b200 import api, scenes as S
        from test_gpu_path import _setup

        v, f, mats, ids, emissive = scene
        self.torch, self.api = torch, api
        self.acc, self.p, _, self.keep = _setup(torch, api, S, v, f, mats, ids, emissive, None, 64, 48, 1, 1, SEED)
        self.cam = narrow_camera()
        for i in range(12):
            self.p.cam[i] = float(self.cam[i])

    def params(self, W, H, spp, bounces, tile, sample0=0, shard=0, n_shards=1, flags=0):
        p = self.api.PathParams.from_buffer_copy(self.p)
        p.width, p.height, p.spp, p.sample0, p.max_bounces = W, H, spp, sample0, bounces
        p.tile_w, p.tile_h, p.shard, p.n_shards, p.flags = tile[0], tile[1], shard, n_shards, flags
        return p

    def render(self, W, H, spp, bounces, tile, **kw):
        torch = self.torch
        accum = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
        r = self.acc.RenderPath(self.params(W, H, spp, bounces, tile, **kw), accum.data_ptr())
        return accum.cpu().numpy().astype(np.float64).reshape(-1, 3), r


@pytest.fixture(scope="module")
def path_pass(untied):
    return _PathPass(untied)


def _assert_waves(r, bounces, waves):
    assert r.traverse_launches == 2 * bounces * waves, (r.traverse_launches, bounces, waves)
    assert r.launches == waves * (1 + 4 * bounces), (r.launches, bounces, waves)


def _within_bound(a, b, m):
    """max |a - b| / bound over the pixels; asserts every pixel is within the reassociation bound."""
    bound = 2.0 * m * U * np.maximum(a, b) * 1.01
    d = np.abs(a - b)
    over = d > bound
    assert not over.any(), (int(over.any(axis=1).sum()), float(d[over].max()), float(bound[over].min()))
    return float(np.max(np.where(bound > 0, d / np.where(bound > 0, bound, 1.0), 0.0)))


def _nonzero_pixels(frame):
    return float(np.mean(frame.sum(axis=1) > 0))


def _compare_splits(pp, name, cfg, waves, splits):
    """The whole frame of cfg against each split: a list of part configurations whose frames are summed in float64."""
    W, H, spp, bounces, tile = cfg["W"], cfg["H"], cfg["spp"], cfg["bounces"], cfg["tile"]
    assert path_waves(W, H, tile, spp) == waves
    whole, rw = pp.render(W, H, spp, bounces, tile)
    _assert_waves(rw, bounces, waves)
    assert rw.camera_rays == W * H * spp and rw.shadow_rays > 0
    assert _nonzero_pixels(whole) > 0.8, "the frame must have something to compare"
    m = spp * bounces
    stats = {"waves": waves, "pixels": W * H, "max_diff_of_bound": 0.0, "splits": {}}
    for label, parts in splits:
        total = np.zeros_like(whole)
        counts = np.zeros(3, np.int64)
        part_waves = []
        for kw in parts:
            c = dict(cfg, **kw)
            extra = {k: c[k] for k in ("sample0", "shard", "n_shards", "flags") if k in c}
            fr, r = pp.render(W, H, c["spp"], bounces, c["tile"], **extra)
            w = path_waves(W, H, c["tile"], c["spp"], c.get("shard", 0), c.get("n_shards", 1))
            _assert_waves(r, bounces, w)
            part_waves.append(w)
            total += fr
            counts += (r.camera_rays, r.radiance_rays, r.shadow_rays)
        assert counts[0] == W * H * spp, (label, counts[0])
        assert (counts[1], counts[2]) == (rw.radiance_rays, rw.shadow_rays), (label, counts, rw.radiance_rays, rw.shadow_rays)
        frac = _within_bound(whole, total, m)
        stats["splits"][label] = {"waves": part_waves, "max_diff_of_bound": round(frac, 4)}
        stats["max_diff_of_bound"] = max(stats["max_diff_of_bound"], round(frac, 4))
    _print(name, stats)
    return whole, rw


# ------------------------------------------------------------------ path pass: splits of one frame
def test_path_pass_two_waves_with_partial_tiles(path_pass):
    """(a) 1000 x 700, 12 spp, 10 bounces, 64 x 8 tiles: 2 waves.  Three shards (one wave each), spp 5 + 7 at sample0 5,
    8 x 4 tiles (21845 + 30 tiles of 384 slots) and 40 x 20 tiles (873 + 2 tiles of 9600 slots), and ANY_HIT shadow
    launches give the same frame and the same ray counts."""
    from nanort_b200 import api

    assert path_waves(A["W"], A["H"], (8, 4), A["spp"]) == 2 and path_waves(A["W"], A["H"], (40, 20), A["spp"]) == 2
    _compare_splits(path_pass, "a", A, 2, [
        ("3 shards", [dict(shard=s, n_shards=3) for s in range(3)]),
        ("spp 5 + 7", [dict(spp=5), dict(spp=7, sample0=5)]),
        ("tiles 8x4", [dict(tile=(8, 4))]),
        ("tiles 40x20", [dict(tile=(40, 20))]),
        ("any hit", [dict(flags=api.TRAVERSE_ANY_HIT)]),
    ])


def test_path_pass_one_tile_larger_than_a_wave(path_pass):
    """(b) 128 x 64 in 64 x 64 tiles at 2049 spp: a tile holds 8 392 704 > 8 Mi slots, one tile per wave, 2 waves;
    the two tiles rendered as shards 0 and 1 of 2."""
    cfg = dict(W=128, H=64, spp=2049, bounces=6, tile=(64, 64))
    _compare_splits(path_pass, "b", cfg, 2, [("2 shards", [dict(shard=0, n_shards=2), dict(shard=1, n_shards=2)])])


def test_path_pass_in_the_benchmarked_wave_layout(path_pass):
    """(c) bench.py configs[2]'s pass shape: 1920 x 1080, 64 spp, 10 bounces, 64 x 8 tiles -> 4050 tiles of 32768 slots,
    256 per wave, 16 waves with a partial last one; against 4 shards and against 32 + 32 samples."""
    cfg = dict(W=1920, H=1080, spp=64, bounces=10, tile=(64, 8))
    _compare_splits(path_pass, "c", cfg, 16, [
        ("4 shards", [dict(shard=s, n_shards=4) for s in range(4)]),
        ("spp 32 + 32", [dict(spp=32), dict(spp=32, sample0=32)]),
    ])


def test_path_pass_equals_its_paths_driven_bounce_by_bounce(path_pass):
    """(d) The whole pass of (a) against the same paths driven from the host: every valid slot in one queue (path id =
    global slot), camera rays of ao_model.camera_dirs, nrt_path_bounce_device per bounce with its shadow pass skipped;
    the shadow rays are traced with ANY_HIT and their visible contributions summed in float64.  Ray counts are exact,
    the frame is within the reassociation bound."""
    import torch
    from nanort_b200 import api

    pp = path_pass
    W, H, spp, bounces, tile = A["W"], A["H"], A["spp"], A["bounces"], A["tile"]
    whole, rw = pp.render(W, H, spp, bounces, tile)
    _assert_waves(rw, bounces, 2)
    p = pp.params(W, H, spp, bounces, tile)
    pix_of_slot, smp_of_slot = M.slots(W, H, tile[0], tile[1], spp)
    valid = np.flatnonzero(pix_of_slot >= 0)
    n = len(valid)
    assert n == W * H * spp
    dev = "cuda"
    dirs = M.camera_dirs(pp.cam, W, H, SEED, pix_of_slot[valid], smp_of_slot[valid])
    q = [[torch.empty((n, 4), dtype=torch.float32, device=dev) for _ in range(2)] + [torch.empty(n, dtype=torch.int32, device=dev)]
         for _ in range(2)]
    q[0][0][:, :3] = torch.as_tensor(np.asarray(pp.cam[:3], np.float32), device=dev)
    q[0][0][:, 3] = 1e-3
    q[0][1][:, :3] = torch.as_tensor(dirs, device=dev)
    q[0][1][:, 3] = 1e30
    q[0][2].copy_(torch.as_tensor(valid.astype(np.int32), device=dev))
    del dirs
    sh = [torch.empty((n, 4), dtype=torch.float32, device=dev) for _ in range(3)]
    weight = torch.ones((len(pix_of_slot), 4), dtype=torch.float32, device=dev)
    emission = torch.zeros(W * H * 3, dtype=torch.float32, device=dev)
    shadow64 = torch.zeros((W * H, 3), dtype=torch.float64, device=dev)
    terms = torch.zeros(W * H, dtype=torch.int64, device=dev)  # non-zero terms per pixel (emission: one per bounce at most)
    rays32 = torch.empty((n, 8), dtype=torch.float32, device=dev)
    hits = torch.empty((n, 4), dtype=torch.float32, device=dev)
    mask = torch.empty(n, dtype=torch.uint8, device=dev)
    per_bounce, radiance, shadow, visible, cur, k = [], 0, 0, 0, 0, n
    for b in range(bounces):
        if k == 0:
            break
        per_bounce.append(k)
        radiance += k
        before = emission.clone()
        nc, ns = pp.acc.PathBounce(p, b, k, q[cur][0].data_ptr(), q[cur][1].data_ptr(), q[cur][2].data_ptr(),
                                   weight.data_ptr(), q[cur ^ 1][0].data_ptr(), q[cur ^ 1][1].data_ptr(),
                                   q[cur ^ 1][2].data_ptr(), sh[0].data_ptr(), sh[1].data_ptr(), sh[2].data_ptr(),
                                   emission.data_ptr(), skip_shadow_pass=True)
        terms += (emission != before).view(-1, 3).any(dim=1)
        shadow += ns
        if ns:
            rays32[:ns, 0:3], rays32[:ns, 3:6] = sh[0][:ns, :3], sh[1][:ns, :3]
            rays32[:ns, 6], rays32[:ns, 7] = sh[0][:ns, 3], sh[1][:ns, 3]
            pp.acc.TraverseDevice(rays32.data_ptr(), ns, hits.data_ptr(), mask.data_ptr(),
                                  flags=api.TRAVERSE_RAY32 | api.TRAVERSE_ANY_HIT)
            vis = mask[:ns] == 0
            contrib = sh[2][:ns][vis][:, :3]
            pix = sh[2][:ns].view(torch.int32)[:, 3][vis].long()
            shadow64.index_add_(0, pix, contrib.double())
            nz = (contrib > 0).any(dim=1)
            terms.index_add_(0, pix[nz], torch.ones_like(pix[nz]))
            visible += int(nz.sum())
        k, cur = nc, cur ^ 1
    assert (radiance, shadow) == (rw.radiance_rays, rw.shadow_rays), (radiance, shadow, rw.radiance_rays, rw.shadow_rays)
    host = emission.double().view(-1, 3).cpu().numpy() + shadow64.cpu().numpy()
    frac = _within_bound(whole, host, spp * bounces)
    # the comparison checks something: emission and light samples reach the frame, paths live past bounce 4 (Russian
    # roulette decides every continuation from bounce 3 on), and most pixels are sums of several terms
    t = terms.cpu().numpy()
    assert float(emission.sum()) > 0 and visible > 0 and len(per_bounce) == bounces and per_bounce[-1] > 0
    assert np.mean(t >= 2) > 0.5, np.mean(t >= 2)
    _print("d", {"waves": 2, "pixels": W * H, "max_diff_of_bound": round(frac, 4), "paths_per_bounce": per_bounce,
                 "pixels_with_2_terms": round(float(np.mean(t >= 2)), 4)})


def test_path_pass_of_an_empty_shard(path_pass):
    """A shard number past the last tile: zero frame, zero counts, NRT_OK, no launches."""
    W, H, tile = A["W"], A["H"], A["tile"]
    n = _n_tiles(W, H, tile)
    assert n == 16 * 88 and path_waves(W, H, tile, A["spp"], n, n + 1) == 0
    fr, r = path_pass.render(W, H, A["spp"], A["bounces"], tile, shard=n, n_shards=n + 1)
    assert not fr.any()
    assert (r.camera_rays, r.radiance_rays, r.shadow_rays, r.launches, r.traverse_launches) == (0, 0, 0, 0, 0)


# ------------------------------------------------------------------ path pass: the reference's shading at other tile maps
def test_every_bounce_matches_the_reference_on_shard_1_of_3(untied):
    """_bounce_by_bounce at 203 x 101 in 40 x 20 tiles, shard 1 of 3, sample0 5, 3 spp (partial tiles)."""
    from test_gpu_path import _bounce_by_bounce

    n = _bounce_by_bounce(with_normals=True, scene=untied,
                          frame=dict(W=203, H=101, spp=3, tile=(40, 20), sample0=5, shard=1, n_shards=3,
                                     cam=narrow_camera()))
    _print("bounces shard 1/3", {"slots_checked": n})


def test_every_bounce_matches_the_reference_in_the_second_wave(untied):
    """_bounce_by_bounce on 30 000 slots of config (a)'s second wave (slot ids >= 8 386 560), partial edge tiles
    included, through all 10 bounces."""
    from test_gpu_path import _bounce_by_bounce

    W, H, tile, spp = A["W"], A["H"], A["tile"], A["spp"]
    pix, _ = M.slots(W, H, tile[0], tile[1], spp)
    cand = np.flatnonzero(pix >= 0)
    cand = cand[cand >= A_WAVE1]
    pick = np.sort(np.random.default_rng(11).choice(cand, 30000, replace=False))
    edge = (pix[pick] % W >= 960) | (pix[pick] // W >= 696)  # pixels of the partial tiles
    assert edge.sum() > 1000 and np.any(pix[pick] % W >= 960) and np.any(pix[pick] // W >= 696)
    n = _bounce_by_bounce(with_normals=False, scene=untied, frame=dict(A, seed=SEED, cam=narrow_camera()), slots=pick)
    _print("bounces wave 2", {"slots": len(pick), "edge_slots": int(edge.sum()), "slots_checked": n})


# ------------------------------------------------------------------ scene AO pass
E = dict(W=500, H=290, spp=31, tile=(40, 20))  # 13 x 15 tiles of 24 800 slots, 169 per wave: 2 waves (169 + 26)


class _ScenePass:
    def __init__(self):
        import torch
        from nanort_b200 import api
        from test_gpu_ao_exact import _scene_instances
        from test_gpu_scene import _gpu_scene

        self.torch, self.api = torch, api
        self.insts = _scene_instances("grid")
        self.sc = _gpu_scene(self.insts, api.BUILD_REFERENCE_TREE, api.BUILD_REFERENCE_TREE)
        self.lo, self.hi = self.sc.GetBoundingBox()
        self.radius = 0.2 * float(np.linalg.norm(self.hi - self.lo))

    def camera(self, W, H):
        from nanort_b200 import scenes as S

        ctr = 0.5 * (self.lo + self.hi)
        return S.look_at(ctr + np.array([0.0, 0.25, 0.5]) * float(np.linalg.norm(self.hi - self.lo)), ctr, aspect=W / H)

    def params(self, W, H, spp, tile, sample0=0, shard=0, n_shards=1):
        from test_gpu_ao_exact import _params

        return _params(self.api, self.camera(W, H), W, H, spp, tile, sample0, SEED, (1e-3, self.radius),
                       flags=self.api.TRAVERSE_CONFORMANCE, shard=shard, n_shards=n_shards)

    def render(self, W, H, spp, tile, **kw):
        torch = self.torch
        accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
        r = self.sc.RenderAO(self.params(W, H, spp, tile, **kw), accum.data_ptr())
        return accum.cpu().numpy(), r


@pytest.fixture(scope="module")
def scene_pass():
    return _ScenePass()


def _compare_scene_splits(sp, name, cfg, waves, splits):
    W, H, spp, tile = cfg["W"], cfg["H"], cfg["spp"], cfg["tile"]
    assert scene_waves(W, H, tile, spp) == waves
    whole, rw = sp.render(W, H, spp, tile)
    assert rw.traverse_launches == 2 * waves and rw.launches == 5 * waves
    assert rw.primary_rays == W * H * spp and 0 < rw.ao_hits < rw.ao_rays
    assert 0 < float(np.mean(whole)) < spp - 1, "the frame mixes hits, misses and occlusion"
    stats = {"waves": waves, "pixels": W * H, "splits": {}}
    for label, parts in splits:
        total = np.zeros_like(whole)
        counts = np.zeros(3, np.int64)
        part_waves = []
        for kw in parts:
            c = dict(cfg, **kw)
            extra = {k: c[k] for k in ("sample0", "shard", "n_shards") if k in c}
            fr, r = sp.render(W, H, c["spp"], c["tile"], **extra)
            w = scene_waves(W, H, c["tile"], c["spp"], c.get("shard", 0), c.get("n_shards", 1))
            assert r.traverse_launches == 2 * w, (label, r.traverse_launches, w)
            part_waves.append(w)
            total += fr
            counts += (r.primary_rays, r.ao_rays, r.ao_hits)
        assert np.array_equal(total, whole), (label, int((total != whole).sum()))
        assert tuple(counts) == (rw.primary_rays, rw.ao_rays, rw.ao_hits), (label, counts)
        stats["splits"][label] = part_waves
    _print(name, stats)
    return whole, rw


def test_scene_pass_two_waves_with_partial_tiles(scene_pass):
    """(e) 500 x 290, 40 x 20 tiles, 31 spp: 2 waves; equal bit for bit to 3 shards, 16 + 15 samples and 8 x 4 tiles;
    every 97th pixel with all its samples equals the model driven by the oracle scene up to borderline samples."""
    from oracle import orc

    sp = scene_pass
    assert scene_waves(E["W"], E["H"], (8, 4), E["spp"]) == 2  # 63 x 73 tiles of 992 slots, 4228 per wave
    whole, rw = _compare_scene_splits(sp, "e", E, 2, [
        ("3 shards", [dict(shard=s, n_shards=3) for s in range(3)]),
        ("spp 16 + 15", [dict(spp=16), dict(spp=15, sample0=16)]),
        ("tiles 8x4", [dict(tile=(8, 4))]),
    ])

    # anchor against the model: every 97th pixel, all of its samples
    from test_gpu_ao_exact import SCENE_BORDERLINE_BUDGET
    from nanort_b200 import api, scenes as S

    W, H, spp = E["W"], E["H"], E["spp"]
    p = sp.params(W, H, spp, E["tile"])
    cam = sp.camera(W, H)
    port = orc.PortScene(sp.insts, cpp11=True)
    xf = sp.sc.InstanceStates()["xform"]
    assert xf.tobytes() == port.sg["xform"].tobytes()
    pixels = np.arange(0, W * H, 97)
    pv = np.repeat(pixels, spp)
    sv = np.tile(np.arange(spp), len(pixels))
    rays = np.zeros(len(pv), S.RAY_DTYPE)
    rays["org"] = cam[:3]
    rays["dir"] = M.camera_dirs(cam, W, H, SEED, pv, sv)
    rays["min_t"], rays["max_t"] = p.ray_min_t, p.ray_max_t
    ph, pm = port.traverse(rays, threads=8)
    gh, gm = sp.sc.Traverse(rays, flags=api.TRAVERSE_CONFORMANCE)
    assert np.array_equal(pm, gm) and ph[pm == 1].tobytes() == gh[gm == 1].tobytes()
    hit = pm == 1
    src = np.flatnonzero(hit)
    ao = M.scene_ao_rays_f32(sp.insts, xf, ph[src], rays["dir"][src], pv[src], sv[src], SEED, p.ao_min_t, p.ao_max_t)
    ah, am = port.traverse(ao, threads=8)
    occ = (am == 1) & (ah["t"] < np.float32(p.ao_max_t))
    model = (np.bincount(pv[~hit], minlength=W * H) + np.bincount(pv[src[~occ]], minlength=W * H)).astype(np.float32)
    assert hit.any() and (~hit).any() and occ.any() and (~occ).any()
    diff = whole[pixels] - model[pixels]
    bad = pixels[diff != 0]
    borderline = 0
    if len(bad):
        j = np.flatnonzero(np.isin(pv[src], bad))
        border = np.zeros(len(j), bool)
        for sx in (-4, 4):
            for sy in (-4, 4):
                for sz in (-4, 4):
                    nudged = ao[j].copy()
                    nudged["dir"] = np.stack([M._nudge(ao["dir"][j][:, c], s) for c, s in enumerate((sx, sy, sz))], axis=1)
                    nh, nm = port.traverse(nudged, threads=8)
                    border |= ((nm == 1) & (nh["t"] < np.float32(p.ao_max_t))) != occ[j]
        per_pix = np.bincount(pv[src[j]][border], minlength=W * H)
        d = whole[bad] - model[bad]
        assert np.all(np.abs(d) <= per_pix[bad]), "a pixel differs from the model without a borderline sample"
        borderline = int(np.abs(d).sum())
    assert borderline <= SCENE_BORDERLINE_BUDGET
    _print("e anchor", {"pixels": len(pixels), "samples": len(pv), "ao_rays": len(src), "pixels_differing": len(bad),
                        "borderline_mismatches": borderline})


def test_scene_pass_one_tile_larger_than_a_wave(scene_pass):
    """(f) 100 x 64 in 64 x 64 tiles at 1025 spp: a tile holds 4 198 400 > 4 Mi slots, one tile per wave, 2 waves
    (the second partial); equal bit for bit to its two tiles rendered as shards."""
    cfg = dict(W=100, H=64, spp=1025, tile=(64, 64))
    _compare_scene_splits(scene_pass, "f", cfg, 2, [("2 shards", [dict(shard=0, n_shards=2), dict(shard=1, n_shards=2)])])


def test_scene_pass_of_an_empty_shard(scene_pass):
    """A shard number past the last tile: zero frame, zero counts, NRT_OK, no launches."""
    W, H, tile, spp = E["W"], E["H"], E["tile"], E["spp"]
    n = _n_tiles(W, H, tile)
    assert n == 13 * 15 and scene_waves(W, H, tile, spp, n, n + 1) == 0
    fr, r = scene_pass.render(W, H, spp, tile, shard=n, n_shards=n + 1)
    assert not fr.any()
    assert (r.primary_rays, r.ao_rays, r.ao_hits, r.launches, r.traverse_launches) == (0, 0, 0, 0, 0)
