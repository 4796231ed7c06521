"""Path-traced lightmaps (include/nanort_b200_lightmap.h) against the reference path tracer's own functions and a float64
restatement of the texel vertex (tests/lightmap_model.py):
  * bounce 0, the texel vertex: origins are the position AOV, the slots with a shadow ray and with a continuation are
    the model's, rays / contributions / weights agree to 1e-5, no shadow ray leaves below the texel's hemisphere and the
    continuations are cosine distributed about the texel's normal;
  * bounces 1 and up: test_gpu_path.py's bounce-by-bounce harness with (texel, sample) in place of (pixel, sample),
    checked against oracle/_ref/libpt_ref.so (the unmodified examples/path_tracer/main.cc) on the device's continuation
    queue;
  * the whole pass equals the sum of its bounces; waves, sample ranges, ANY_HIT, repeated calls and two streams compose;
  * a furnace: every texel of a quad inside a closed box of unit emitters bakes to 1;
  * refusals launch nothing."""
import numpy as np
import pytest

import bake_model as B
import lightmap_model as LM

pytestmark = pytest.mark.gpu

MISS = 0xFFFFFFFF


def _rel(a, b, floor=1e-3):
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), floor))) if a.size else 0.0


# ------------------------------------------------------------------ scenes
def cornell():
    """Cornell box with the reference's material set, one chart per face: (v, f, mats, ids, emissive, uv, uf)."""
    from nanort_b200 import scenes as S

    v, f, mats, ids, emissive = S.cornell_with_materials()
    uv, uf = S.per_face_atlas(len(f))
    return v, f, mats, ids, emissive, uv, uf


def cornell_diffuse():
    """The Cornell box, every wall and box diffuse 0.7, under an area light: no lobe depends on which of two faces at
    the same distance a ray reports, so ray counts do not depend on the queue order."""
    from nanort_b200 import scenes as S

    v, f = S.make_scene("cornell")
    v, f, l0, ln = S.with_area_light(v, f, (0.0, 9.99, 0.0), 2.0, 2.0)
    mats = np.concatenate([S.material(diffuse=(0.7, 0.7, 0.7)), S.material(emission=(10, 10, 10))])
    ids = np.zeros(len(f), np.uint32)
    ids[l0:] = 1
    uv, uf = S.per_face_atlas(len(f))
    return v, f, mats, ids, np.arange(l0, l0 + ln, dtype=np.uint32), uv, uf


def _terrain_uv(v, f, l0):
    """planar UVs of the terrain's faces; the light's faces charted at u, v in [2.2, 2.8], outside the atlas region"""
    from nanort_b200 import scenes as S

    uv, uf = S.planar_uv(v[:int(f[:l0].max()) + 1], f[:l0])
    n_l = len(f) - l0
    lv = np.zeros((3 * n_l, 3), np.float32)
    lv[:, :2] = np.tile(np.float32([[2.2, 2.2], [2.8, 2.2], [2.2, 2.8]]), (n_l, 1))
    return np.concatenate([uv, lv]), np.arange(3 * len(f), dtype=np.uint32).reshape(-1, 3)


def terrain():
    """The 1,002,528-triangle terrain under an area light (BASELINE.json configs[2]), planar UVs."""
    from nanort_b200 import scenes as S

    v, f = S.make_scene("terrain")
    v, f, l0, ln = S.with_area_light(v, f, (0.0, 6.0, 0.0), 2.0, 2.0)
    mats = np.concatenate([S.material(diffuse=(0.7, 0.7, 0.7)), S.material(emission=(20, 20, 20))])
    ids = np.zeros(len(f), np.uint32)
    ids[l0:] = 1
    uv, uf = _terrain_uv(v, f, l0)
    return v, f, mats, ids, np.arange(l0, l0 + ln, dtype=np.uint32), uv, uf


class Bake:
    """World accel, records (host and device), position AOV and device shading arrays of a scene."""

    def __init__(self, scene, W, H, fvn=None):
        import torch

        from nanort_b200 import api

        self.v, self.f, self.mats, self.ids, self.emissive, uv, uf = scene
        self.W, self.H = W, H
        self.world = api.BVHAccel()
        assert self.world.Build(len(self.f), self.v, self.f)
        uv_acc = api.BVHAccel()
        assert uv_acc.Build(len(uf), uv, uf)
        rp = api.UvRasterParams()
        rp.width, rp.height = W, H
        rp.uv_region[:] = [0.0, 1.0, 0.0, 1.0]
        rp.texel_offset[:] = [0.5, 0.5]
        rec = torch.zeros((W * H, 4), dtype=torch.float32, device="cuda")
        pos = torch.zeros((W * H, 3), dtype=torch.float32, device="cuda")
        self.n_cov = uv_acc.UVRaster(rp, rec.data_ptr(), world=self.world, d_position_ptr=pos.data_ptr())
        assert self.n_cov > 0
        from nanort_b200 import scenes as S

        self.d_rec = rec
        self.rec = rec.cpu().numpy().view(S.HIT_DTYPE).reshape(-1)
        self.pos = pos.cpu().numpy()
        self.fvn = fvn
        self.keep = {"m": torch.as_tensor(np.ascontiguousarray(self.mats).view(np.float32).reshape(-1), device="cuda"),
                     "i": torch.as_tensor(self.ids.astype(np.int32), device="cuda"),
                     "e": torch.as_tensor(self.emissive.astype(np.int32), device="cuda"),
                     "n": torch.as_tensor(np.ascontiguousarray(fvn, np.float32).reshape(-1), device="cuda")
                     if fvn is not None else None}

    def params(self, spp, bounces, seed=5, sample0=0, flags=0):
        from nanort_b200 import api

        p = api.LightmapParams()
        p.width, p.height, p.spp, p.sample0, p.seed, p.max_bounces = self.W, self.H, spp, sample0, seed, bounces
        p.ray_min_t, p.ray_max_t = 1e-3, 1e30
        p.n_materials, p.n_emissive = len(self.mats), len(self.emissive)
        p.d_materials, p.d_material_ids = self.keep["m"].data_ptr(), self.keep["i"].data_ptr()
        p.d_emissive_faces = self.keep["e"].data_ptr()
        p.d_facevarying_normals = self.keep["n"].data_ptr() if self.fvn is not None else None
        p.flags = flags
        return p

    def bake(self, p, accum=None, stream=None):
        import torch

        if accum is None:
            accum = torch.zeros(self.W * self.H * 3, dtype=torch.float32, device="cuda")
        r = self.world.BakeLightmap(self.d_rec.data_ptr(), p, accum.data_ptr(),
                                    stream=stream.cuda_stream if stream is not None else None)
        return accum, r


class Queues:
    """Caller-owned queues of LightmapBounce for n rays and `paths` path ids."""

    def __init__(self, n, paths):
        import torch

        z = lambda *s, dt=torch.float32: torch.zeros(s, dtype=dt, device="cuda")
        self.out_o, self.out_d, self.out_pid = z(n, 4), z(n, 4), z(n, dt=torch.int32)
        self.sh_o, self.sh_d, self.sh_c = z(n, 4), z(n, 4), z(n, 4)
        self.weight = z(paths, 4)

    def run(self, bk, p, b, n, accum, d_in=(None, None, None), skip_shadow=False):
        return bk.world.LightmapBounce(bk.d_rec.data_ptr(), p, b, n, *[x.data_ptr() if x is not None else None for x in d_in],
                                       self.weight.data_ptr(), self.out_o.data_ptr(), self.out_d.data_ptr(),
                                       self.out_pid.data_ptr(), self.sh_o.data_ptr(), self.sh_d.data_ptr(),
                                       self.sh_c.data_ptr(), accum.data_ptr(), skip_shadow_pass=skip_shadow)


def _waves(r, bounces):
    assert r.traverse_launches % (2 * bounces - 1) == 0
    return r.traverse_launches // (2 * bounces - 1)


# ------------------------------------------------------------------ bounce 0: the texel vertex
@pytest.mark.parametrize("name,with_normals", [("cornell", False), ("cornell", True), ("terrain", False)])
def test_texel_vertex_equals_the_model(name, with_normals):
    import torch
    from scipy import stats

    from oracle import orc

    scene = cornell() if name == "cornell" else terrain()
    fvn = None
    if with_normals:  # the example loader's flat normals: the opposite side of the wound normal
        fvn = orc.ReferencePathTracer(scene[0], scene[1], scene[3], scene[2]).fvn if orc.ReferencePathTracer.available() \
            else None
        if fvn is None:
            pytest.skip("oracle/_ref/libpt_ref.so not built")
    W, H, spp, bounces, seed = (160, 128, 4, 6, 7) if name == "cornell" else (256, 256, 2, 6, 3)
    bk = Bake(scene, W, H, fvn)
    if name == "terrain":
        light_faces = np.arange(len(bk.f) - 2, len(bk.f))
        assert not np.isin(bk.rec["prim_id"], light_faces).any(), "the light's faces cover no texel"
    n = bk.n_cov * spp
    p = bk.params(spp, bounces, seed, sample0=3)
    q = Queues(n, n)
    accum = torch.full((W * H * 3,), 0.25, dtype=torch.float32, device="cuda")
    n_cont, n_sh = q.run(bk, p, 0, n, accum, skip_shadow=True)
    torch.cuda.synchronize()
    assert torch.all(accum == 0.25), "bounce 0 adds nothing to the lightmap before its shadow pass"
    want = LM.texel_vertex(bk.v, bk.f, bk.rec, spp, seed, bk.emissive, bk.mats, bk.ids, bounces, sample0=3, fv_normals=fvn)
    # ---- continuations: one per path (every texel vertex scatters diffusely), origin = the position AOV bit for bit
    assert n_cont == n
    pid = q.out_pid.cpu().numpy()[:n_cont].astype(np.int64)
    assert np.array_equal(np.sort(pid), np.arange(n))
    co, cd = q.out_o.cpu().numpy()[:n_cont], q.out_d.cpu().numpy()[:n_cont]
    order = np.argsort(pid)
    co, cd = co[order], cd[order]
    assert np.array_equal(co[:, :3].view(np.uint32), bk.pos[want["texel"]].view(np.uint32))
    assert np.all(co[:, 3] == np.float32(1e-3)) and np.all(cd[:, 3] == np.float32(1e30))
    assert float(np.abs(cd[:, :3] - want["cont_dir"]).max()) <= 1e-5
    w = q.weight.cpu().numpy()[:n]
    assert np.all(w == np.float32([1, 1, 1, 0])), "weight 1, do_emission 0"
    cos = (cd[:, :3].astype(np.float64) * want["n"]).sum(axis=1)
    assert cos.min() > -1e-5
    assert stats.kstest(np.clip(cos / np.linalg.norm(cd[:, :3], axis=1), 0, 1) ** 2, "uniform").pvalue >= 1e-3
    # ---- shadow rays: the set of slots is exact away from grazing light samples (|dot(l, n)| below 1e-5: a light
    # sampled in the texel's own plane, e.g. a texel on the light itself, whose float32 sign is rounding)
    assert n_sh > 0
    so, sd, sc = q.sh_o.cpu().numpy()[:n_sh], q.sh_d.cpu().numpy()[:n_sh], q.sh_c.cpu().numpy()[:n_sh]
    got_texel = sc[:, 3].copy().view(np.uint32).astype(np.int64)
    grazing = np.abs(want["cos_s"]) < 1e-5
    assert grazing.mean() < 0.08  # Cornell: the texels of the light's 2 of 36 faces
    # match by (texel, direction): a texel's samples have distinct light samples
    kg = np.lexsort((sd[:, 1], sd[:, 0], got_texel))
    ws = np.flatnonzero(want["shadow"])
    kr = ws[np.lexsort((want["shadow_dir"][ws, 1], want["shadow_dir"][ws, 0], want["texel"][ws]))]
    got_clear = np.ones(n_sh, bool)
    if grazing.any():  # drop grazing samples on both sides before pairing (a texel keeps its clear ones)
        gm = np.zeros(n_sh, bool)
        for t in np.unique(want["texel"][grazing]):
            gm |= got_texel == t
        keep_t = ~np.isin(want["texel"], np.unique(want["texel"][grazing]))
        got_clear = ~gm
        kg = kg[got_clear[kg]]
        kr = kr[keep_t[kr]]
        assert int(want["shadow"][keep_t].sum()) == int(got_clear.sum())
    else:
        assert n_sh == int(want["shadow"].sum())
    assert np.array_equal(got_texel[kg], want["texel"][kr])
    assert np.array_equal(so[kg][:, :3].view(np.uint32), bk.pos[want["texel"][kr]].view(np.uint32))
    assert np.all(so[:, 3] == np.float32(1e-5))
    assert float(np.abs(sd[kg][:, :3] - want["shadow_dir"][kr]).max()) <= 1e-5
    assert _rel(sd[kg][:, 3], want["shadow_max_t"][kr]) <= 1e-5
    err = np.abs(sc[kg][:, :3] - want["contrib"][kr]).max(axis=1) / np.maximum(want["contrib_scale"][kr], 1e-30)
    assert float(err.max()) <= 1e-5, float(err.max())
    # no shadow ray below the texel's hemisphere (float64 normal; the device decided on its float32 one)
    first = {int(t): i for i, t in enumerate(want["texel"][:bk.n_cov])}
    nrm = want["n"][[first[int(t)] for t in got_texel]]
    assert float((sd[:, :3].astype(np.float64) * nrm).sum(axis=1).min()) > -1e-5


# ------------------------------------------------------------------ bounces 1 and up: the reference's own functions
def _bounce_by_bounce(scene_fn, with_normals, W, H, spp, bounces, seed, min_checked):
    import torch

    from nanort_b200 import scenes as S
    from oracle import orc

    if not orc.ReferencePathTracer.available():
        pytest.skip("oracle/_ref/libpt_ref.so not built (no reference tree at build time)")
    scene = scene_fn()
    v, f, mats, ids, emissive = scene[:5]
    ref = orc.ReferencePathTracer(v, f, ids, mats)
    assert np.array_equal(ref.emissive_faces(), emissive)
    fvn = ref.fvn if with_normals else None
    bk = Bake(scene, W, H, fvn)
    n_paths = bk.n_cov * spp
    p = bk.params(spp, bounces, seed)
    texel_of, smp_of = B.bake_slots(bk.rec, spp)
    q = Queues(n_paths, n_paths)
    accum = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
    n_cont, _ = q.run(bk, p, 0, n_paths, accum)
    expect = accum.cpu().numpy().reshape(-1, 3).astype(np.float64)  # bounce 0's visible light samples
    pid = q.out_pid.cpu().numpy()[:n_cont].astype(np.int64)
    org, dirs = q.out_o.cpu().numpy()[:n_cont, :3].copy(), q.out_d.cpu().numpy()[:n_cont, :3].copy()
    checked, lobes = 0, set()
    dev = "cuda"
    f4 = lambda xyz, w: torch.as_tensor(np.concatenate([xyz, np.full((len(xyz), 1), w, np.float32)], axis=1), device=dev)
    for b in range(1, bounces):
        n = len(pid)
        if n == 0:
            break
        d_in = (f4(org, 1e-3), f4(dirs, 1e30), torch.as_tensor(pid.astype(np.int32), device=dev))
        w_in = q.weight[torch.as_tensor(pid, device=dev)].cpu().numpy()
        out = Queues(n, 0)
        out.weight = q.weight
        n_cont, n_sh = out.run(bk, p, b, n, accum, d_in)
        r = np.zeros(n, S.RAY_DTYPE)
        r["org"], r["dir"], r["min_t"], r["max_t"] = org, dirs, np.float32(1e-3), np.float32(1e30)
        hits, mask = bk.world.Traverse(r)
        h = np.flatnonzero(mask.astype(bool))
        tex, smp = texel_of[pid], smp_of[pid]
        dim = 8 + 8 * b
        draws = np.stack([S.rand_ps(tex, smp, dim + k, seed) for k in range(6)], axis=1).astype(np.float32)
        want = ref.shade(b, bounces, org[h], dirs[h], np.stack([hits["u"][h], hits["v"][h], hits["t"][h]], axis=1),
                         hits["prim_id"][h], w_in[h], draws[h])
        checked += len(h)
        cont, shad, emit = ((want["flags"] & k) != 0 for k in (1, 2, 4))
        assert n_cont == int(cont.sum()) and n_sh == int(shad.sum()), (b, n_cont, int(cont.sum()), n_sh, int(shad.sum()))
        got_pid = out.out_pid.cpu().numpy()[:n_cont].astype(np.int64)
        ref_pid = pid[h][cont]
        assert np.array_equal(np.sort(got_pid), np.sort(ref_pid)), f"bounce {b}: different set of continuing paths"
        go, gd = out.out_o.cpu().numpy()[:n_cont], out.out_d.cpu().numpy()[:n_cont]
        gs, rs = np.argsort(got_pid), np.argsort(ref_pid)
        assert _rel(go[gs][:, :3], want["next_org"][cont][rs]) <= 1e-5
        assert (float(np.abs(gd[gs][:, :3] - want["next_dir"][cont][rs]).max()) <= 2e-5) if n_cont else True
        w_out = q.weight[torch.as_tensor(ref_pid, device=dev)].cpu().numpy()
        assert _rel(w_out[:, :3], want["weight"][cont][:, :3], floor=1e-6) <= 1e-5
        assert np.array_equal(w_out[:, 3] != 0, want["weight"][cont][:, 3] != 0), "do_emission flag"
        so, sd, sc = (x.cpu().numpy()[:n_sh] for x in (out.sh_o, out.sh_d, out.sh_c))
        got_tex = sc[:, 3].copy().view(np.uint32)
        ref_tex = tex[h][shad].astype(np.uint32)
        kg = np.lexsort((so[:, 2], so[:, 1], so[:, 0], got_tex))
        ro = want["shadow_org"][shad]
        kr = np.lexsort((ro[:, 2], ro[:, 1], ro[:, 0], ref_tex))
        assert np.array_equal(got_tex[kg], ref_tex[kr])
        assert _rel(so[kg][:, :3], ro[kr]) <= 1e-5
        assert (float(np.abs(sd[kg][:, :3] - want["shadow_dir"][shad][kr]).max()) <= 2e-5) if n_sh else True
        assert _rel(sd[kg][:, 3], want["shadow_max_t"][shad][kr]) <= 1e-5
        # as in test_gpu_path.py: both cosines of a light sample agree to 2e-5 absolute, grazing ones a little less
        cdf = np.abs(sc[kg][:, :3] - want["shadow_contrib"][shad][kr]) / np.maximum(np.abs(want["shadow_contrib"][shad][kr]), 1e-6)
        assert (float(cdf.max()) <= 1e-3 and float(np.quantile(cdf, 0.999)) <= 2e-5) if n_sh else True
        sr = np.zeros(n_sh, S.RAY_DTYPE)
        sr["org"], sr["dir"], sr["min_t"], sr["max_t"] = so[:, :3], sd[:, :3], so[:, 3], sd[:, 3]
        _, smask = bk.world.Traverse(sr) if n_sh else (None, np.zeros(0, np.uint8))
        np.add.at(expect, tex[h][emit].astype(np.int64), want["emission"][emit].astype(np.float64))
        vis = smask == 0
        np.add.at(expect, got_tex[vis].astype(np.int64), sc[vis][:, :3].astype(np.float64))
        got = accum.cpu().numpy().reshape(-1, 3).astype(np.float64)
        assert np.max(np.abs(got - expect) / np.maximum(np.abs(expect), 1.0)) <= 1e-4, b
        lobes |= {("cont", bool(cont.any())), ("shadow", bool(shad.any())), ("emit", bool(emit.any()))}
        pid, org, dirs = got_pid, go[:, :3].copy(), gd[:, :3].copy()
    assert checked >= min_checked and ("shadow", True) in lobes, (checked, lobes)
    return lobes


def test_bounces_match_the_reference_functions_on_cornell():
    lobes = _bounce_by_bounce(cornell, False, 96, 96, 4, 8, 5, 15000)
    assert ("emit", True) in lobes


def test_bounces_match_the_reference_functions_on_cornell_with_facevarying_normals():
    _bounce_by_bounce(cornell, True, 96, 96, 4, 8, 5, 15000)


def test_bounces_match_the_reference_functions_on_the_1m_triangle_terrain():
    _bounce_by_bounce(terrain, False, 512, 512, 1, 5, 3, 25000)


# ------------------------------------------------------------------ the whole pass
def test_whole_pass_equals_the_sum_of_its_bounces():
    import torch

    bk = Bake(cornell(), 128, 128)
    spp, bounces = 4, 7
    p = bk.params(spp, bounces, seed=9)
    whole, r = bk.bake(p)
    n_paths = bk.n_cov * spp
    assert (r.texels, r.paths) == (bk.n_cov, n_paths) and _waves(r, bounces) == 1
    q = Queues(n_paths, n_paths)
    accum = torch.zeros(128 * 128 * 3, dtype=torch.float32, device="cuda")
    n, shadow = q.run(bk, p, 0, n_paths, accum)
    radiance = 0
    cur = (q.out_o.clone(), q.out_d.clone(), q.out_pid.clone())
    for b in range(1, bounces):
        if n == 0:
            break
        radiance += n
        nc, ns = q.run(bk, p, b, n, accum, cur)
        shadow += ns
        n, cur = nc, (q.out_o.clone(), q.out_d.clone(), q.out_pid.clone())
    # equal up to exact-distance ties (test_gpu_path.py: a ray hitting two faces at the same t, e.g. the glass box's
    # bottom lying in the floor, may report either, depending on the queue order)
    assert abs(radiance - r.radiance_rays) <= 4 and abs(shadow - r.shadow_rays) <= 4, (radiance, shadow, r.radiance_rays,
                                                                                     r.shadow_rays)
    a, b = accum.cpu().numpy().reshape(-1, 3).astype(np.float64), whole.cpu().numpy().reshape(-1, 3).astype(np.float64)
    rel = np.max(np.abs(a - b) / np.maximum(np.abs(b), 1.0), axis=1)
    assert np.count_nonzero(rel > 1e-5) <= 4, np.count_nonzero(rel > 1e-5)
    empty = bk.rec["prim_id"] == MISS
    assert empty.any() and np.all(b[empty] == 0) and np.count_nonzero(b[~empty].sum(axis=1) > 0) > 0.5 * bk.n_cov


def _sphere_furnace(n_lat=48, n_lon=96, half=0.05):
    """A 2 half x 2 half quad (normal +y) at the centre of a closed unit sphere of n_lat x n_lon facets, all unit emitters
    wound inward; only the quad is charted in the atlas.  Returns the scene and cos_min, the smallest cos_l between a
    facet's normal and the direction from a facet vertex to a quad corner or centre."""
    from nanort_b200 import scenes as S

    th = np.pi * np.arange(1, n_lat) / n_lat
    ph = 2 * np.pi * np.arange(n_lon) / n_lon
    ring = np.stack([np.sin(th)[:, None] * np.cos(ph)[None], np.cos(th)[:, None] + 0 * ph[None],
                     np.sin(th)[:, None] * np.sin(ph)[None]], axis=2).reshape(-1, 3)
    v = np.concatenate([[[0, 1, 0]], ring, [[0, -1, 0]]]).astype(np.float32)
    south = len(v) - 1
    at = lambda i, j: 1 + i * n_lon + (j % n_lon)
    faces = []
    for j in range(n_lon):
        faces.append((0, at(0, j), at(0, j + 1)))
        faces.append((south, at(n_lat - 2, j + 1), at(n_lat - 2, j)))
        for i in range(n_lat - 2):
            faces += [(at(i, j), at(i + 1, j), at(i + 1, j + 1)), (at(i, j), at(i + 1, j + 1), at(i, j + 1))]
    f = np.asarray(faces, np.uint32)
    e1, e2 = v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]
    inward = (np.cross(e1, e2) * -v[f].mean(axis=1)).sum(axis=1) > 0
    f[~inward] = f[~inward][:, [0, 2, 1]]
    n_e = len(f)
    qv = np.float32([[-half, 0, -half], [half, 0, -half], [half, 0, half], [-half, 0, half]])
    base = len(v)
    qf = np.uint32([[base, base + 2, base + 1], [base, base + 3, base + 2]])  # cross(e1, e2) = +y
    v, f = np.concatenate([v, qv]), np.concatenate([f, qf])
    assert np.cross(v[qf[0, 1]] - v[qf[0, 0]], v[qf[0, 2]] - v[qf[0, 0]])[1] > 0
    nrm = np.cross(v[f[:n_e, 1]] - v[f[:n_e, 0]], v[f[:n_e, 2]] - v[f[:n_e, 0]]).astype(np.float64)
    nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    pts = np.concatenate([qv, [[0, 0, 0]]]).astype(np.float64)
    cos_min = 1.0
    for k in range(3):
        d = pts[None] - v[f[:n_e, k]].astype(np.float64)[:, None]
        cos_min = min(cos_min, float(((d / np.linalg.norm(d, axis=2)[..., None]) * nrm[:, None]).sum(axis=2).min()))
    mats = np.concatenate([S.material(emission=(1, 1, 1)), S.material(diffuse=(0.5, 0.5, 0.5))])
    ids = np.zeros(len(f), np.uint32)
    ids[n_e:] = 1
    uvs = np.zeros((len(f), 3, 2), np.float32) + 2.5  # the emitters: outside the atlas
    uvs[n_e] = [[0, 0], [1, 1], [1, 0]]
    uvs[n_e + 1] = [[0, 0], [0, 1], [1, 1]]
    uv = np.zeros((3 * len(f), 3), np.float32)
    uv[:, :2] = uvs.reshape(-1, 2)
    scene = (v, f, mats, ids, np.arange(n_e, dtype=np.uint32), uv, np.arange(3 * len(f), dtype=np.uint32).reshape(-1, 3))
    return scene, cos_min


@pytest.mark.parametrize("bounces", [1, 8])
def test_furnace_every_texel_bakes_to_one(bounces):
    """Inside a closed sphere of unit emitters every texel sees emitters over its whole hemisphere, and light from
    below the quad must not count: with the path tracer's |cos| at the texel the bake would give 2.  The reference's
    emitters have a cosine EDF (radiance Le * cos_l, main.cc:943-950), so E / pi = (1 / pi) * integral of cos_l cos dw
    lies in [cos_min, 1], cos_min the facets' smallest cos_l towards the quad (0.99 and more: small quad, fine facets)."""
    scene, cos_min = _sphere_furnace()
    assert cos_min > 0.98
    bk = Bake(scene, 32, 32)
    spp = 1024
    accum, r = bk.bake(bk.params(spp, bounces, seed=4))
    m = accum.cpu().numpy().reshape(-1, 3).astype(np.float64)[bk.rec["prim_id"] != MISS] / spp
    assert len(m) == bk.n_cov > 800 and np.allclose(m[:, 0], m[:, 1], rtol=1e-5) and np.allclose(m[:, 0], m[:, 2], rtol=1e-5)
    m = m[:, 0]
    # the texels' means scatter with the per-sample spread / sqrt(spp): the bounds are 5 standard errors for their mean
    # and 6 of their standard deviations for every texel, around [cos_min, 1]
    sd = float(m.std())
    assert sd < 0.1, sd
    se = 5 * sd / np.sqrt(len(m))
    assert cos_min - se <= float(m.mean()) <= 1.0 + se, (float(m.mean()), sd, cos_min)
    assert float(m.min()) >= cos_min - 6 * sd and float(m.max()) <= 1.0 + 6 * sd, (float(m.min()), float(m.max()), sd)
    assert r.radiance_rays == (bk.n_cov * spp if bounces > 1 else 0)  # every continuation is traced, then stops


# ------------------------------------------------------------------ splits, waves, streams
def _same(a, b, n_out=16):
    """equal within the reassociation of float atomics (per-texel sums of the same positive terms in another order:
    1e-5 relative), but for a few texels whose path hit two faces at exactly the same distance (the boxes' edges), where
    the traversal reports either face depending on the queue order and the continuation leaves along the other normal"""
    a, b = a.cpu().numpy().astype(np.float64), b.cpu().numpy().astype(np.float64)
    rel = np.abs(a - b) / np.maximum(np.abs(b), 1e-3)
    return np.count_nonzero(rel > 1e-5) <= n_out, (np.count_nonzero(rel > 1e-5), float(rel.max()))


def test_waves_sample_ranges_any_hit_and_repeated_calls_compose():
    import torch

    from nanort_b200 import api

    bk = Bake(cornell_diffuse(), 2048, 2048)
    bounces = 4
    spp = 16
    whole, r = bk.bake(bk.params(spp, bounces))
    assert r.paths == bk.n_cov * spp and _waves(r, bounces) == -(-r.paths // (8 << 20)) >= 2
    parts = torch.zeros_like(whole)
    r1 = bk.bake(bk.params(8, bounces), parts)[1]
    r2 = bk.bake(bk.params(8, bounces, sample0=8), parts)[1]
    assert _waves(r1, bounces) == _waves(r2, bounces) == -(-bk.n_cov * 8 // (8 << 20))
    assert (r1.radiance_rays + r2.radiance_rays, r1.shadow_rays + r2.shadow_rays) == (r.radiance_rays, r.shadow_rays)
    ok, worst = _same(parts, whole)
    assert ok, worst
    anyhit, ra = bk.bake(bk.params(spp, bounces, flags=api.TRAVERSE_ANY_HIT))
    assert (ra.radiance_rays, ra.shadow_rays, ra.traverse_launches) == (r.radiance_rays, r.shadow_rays, r.traverse_launches)
    ok, worst = _same(anyhit, whole)
    assert ok, worst
    again, rr = bk.bake(bk.params(spp, bounces))
    assert (rr.radiance_rays, rr.shadow_rays) == (r.radiance_rays, r.shadow_rays)
    ok, worst = _same(again, whole)
    assert ok, worst
    assert r.traverse_ms > 0 and r.total_ms >= r.traverse_ms


def test_lightmap_and_path_pass_on_two_streams_equal_their_solo_runs():
    import torch

    from nanort_b200 import api, scenes as S

    bk = Bake(cornell_diffuse(), 256, 256)
    p = bk.params(8, 5, seed=2)
    pp = api.PathParams()
    cam = S.scene_camera("cornell", 128, 96)
    for i in range(12):
        pp.cam[i] = float(cam[i])
    pp.width, pp.height, pp.spp, pp.sample0, pp.seed = 128, 96, 8, 0, 3
    pp.tile_w, pp.tile_h, pp.shard, pp.n_shards = 64, 8, 0, 1
    pp.max_bounces, pp.ray_min_t, pp.ray_max_t = 5, 1e-3, 1e30
    pp.n_materials, pp.n_emissive = len(bk.mats), len(bk.emissive)
    pp.d_materials, pp.d_material_ids, pp.d_emissive_faces = bk.keep["m"].data_ptr(), bk.keep["i"].data_ptr(), bk.keep["e"].data_ptr()
    solo_l, rl = bk.bake(p)
    solo_p = torch.zeros(128 * 96 * 3, dtype=torch.float32, device="cuda")
    rp = bk.world.RenderPath(pp, solo_p.data_ptr())
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for _ in range(2):
        lm = torch.zeros_like(solo_l)
        img = torch.zeros_like(solo_p)
        torch.cuda.synchronize()
        bk.world.BakeLightmap(bk.d_rec.data_ptr(), p, lm.data_ptr(), stream=streams[0].cuda_stream, want_result=False)
        bk.world.RenderPath(pp, img.data_ptr(), stream=streams[1].cuda_stream, want_result=False)
        torch.cuda.synchronize()
        for got, want in ((lm, solo_l), (img, solo_p)):
            ok, worst = _same(got, want)
            assert ok, worst
    assert rl.traverse_launches == 9 and rp.traverse_launches == 10


def test_refusals_launch_nothing():
    import torch

    from nanort_b200 import api

    bk = Bake(cornell(), 160, 128)
    accum = torch.full((160 * 128 * 3,), 2.5, dtype=torch.float32, device="cuda")
    spheres = api.BVHAccel()
    spheres.BuildSpheres(np.zeros((4, 3), np.float32) + np.arange(4, dtype=np.float32)[:, None], np.ones(4, np.float32))
    bad = bk.rec.copy()
    bad["prim_id"][np.flatnonzero(bad["prim_id"] != MISS)[7]] = len(bk.f) + 5
    d_bad = torch.from_numpy(bad.view(np.float32).reshape(-1, 4).copy()).cuda()
    unaligned = bk.d_rec.data_ptr() + 4

    def with_(**kw):
        p = bk.params(2, 3)
        for k, v in kw.items():
            setattr(p, k, v)
        return p

    cases = [(bk.world, 0, with_()), (spheres, bk.d_rec.data_ptr(), with_()), (bk.world, unaligned, with_()),
             (bk.world, d_bad.data_ptr(), with_()), (bk.world, bk.d_rec.data_ptr(), with_(spp=0)),
             (bk.world, bk.d_rec.data_ptr(), with_(width=0)), (bk.world, bk.d_rec.data_ptr(), with_(width=1 << 16, height=1 << 16)),
             (bk.world, bk.d_rec.data_ptr(), with_(max_bounces=0)), (bk.world, bk.d_rec.data_ptr(), with_(n_materials=0)),
             (bk.world, bk.d_rec.data_ptr(), with_(d_materials=None)),
             (bk.world, bk.d_rec.data_ptr(), with_(d_emissive_faces=None)),
             (bk.world, bk.d_rec.data_ptr(), with_(flags=api.TRAVERSE_CONFORMANCE)),
             (bk.world, bk.d_rec.data_ptr(), with_(flags=1 << 20))]
    n = bk.n_cov * 2
    q = Queues(n, n)
    for acc, ptr, p in cases:
        with pytest.raises(api.NanortB200Error, match="error -1"):
            api._check(api.lib().nrt_bake_lightmap_device(acc._h, ptr or None, p, accum.data_ptr(), None, None))
        with pytest.raises(api.NanortB200Error, match="error -1"):
            acc.LightmapBounce(ptr or None, p, 0, n, None, None, None, q.weight.data_ptr(), q.out_o.data_ptr(),
                               q.out_d.data_ptr(), q.out_pid.data_ptr(), q.sh_o.data_ptr(), q.sh_d.data_ptr(),
                               q.sh_c.data_ptr(), accum.data_ptr())
    with pytest.raises(api.NanortB200Error, match="error -1"):
        api._check(api.lib().nrt_bake_lightmap_device(bk.world._h, bk.d_rec.data_ptr(), None, accum.data_ptr(), None, None))
    with pytest.raises(api.NanortB200Error, match="error -1"):
        bk.world.BakeLightmap(bk.d_rec.data_ptr(), with_(), 0)
    for b, nn in ((0, n + 1), (1, 1 << 32)):  # more texel vertices than slots; a path id beyond 32 bits
        with pytest.raises(api.NanortB200Error, match="error -1"):
            bk.world.LightmapBounce(bk.d_rec.data_ptr(), with_(), b, nn, q.out_o.data_ptr(), q.out_d.data_ptr(),
                                    q.out_pid.data_ptr(), q.weight.data_ptr(), q.out_o.data_ptr(), q.out_d.data_ptr(),
                                    q.out_pid.data_ptr(), q.sh_o.data_ptr(), q.sh_d.data_ptr(), q.sh_c.data_ptr(),
                                    accum.data_ptr())
    with pytest.raises(api.NanortB200Error, match="error -1"):  # bounce >= 1 needs its input queue
        bk.world.LightmapBounce(bk.d_rec.data_ptr(), with_(), 1, 8, None, None, None, q.weight.data_ptr(),
                                q.out_o.data_ptr(), q.out_d.data_ptr(), q.out_pid.data_ptr(), q.sh_o.data_ptr(),
                                q.sh_d.data_ptr(), q.sh_c.data_ptr(), accum.data_ptr())
    torch.cuda.synchronize()
    assert torch.all(accum == 2.5)
    for t in (q.weight, q.out_o, q.out_d, q.sh_o, q.sh_d, q.sh_c):
        assert torch.all(t == 0)
    assert torch.all(q.out_pid == 0)
