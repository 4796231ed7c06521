"""Texel cast, AO bake and lightmap bake over two-level scenes (csrc/scene_bake.cu, include/nanort_b200_scene_bake.h).

The scene is test_gpu_scene_path.py's instanced Cornell box with reference-built trees: the walls, the light (no chart),
and one box mesh shared by a rotated, non-uniformly scaled instance and a mirrored one.  The two boxes also share one
UV accel.  Charts: the walls at (0, 0) 64 x 64; the rotated box at (64, 0) 48 x 40 with both flips and a non-default
region; the mirrored box at (64, 40) 48 x 40, in a 128 x 128 atlas (so that the charts with x0 and y0 swapped stay
inside it).  Flattened on the host (world vertices by the float32 MultV order, world
face-varying normals by inverse_transpose33, face id = instance offset + prim) the scene is an ordinary mesh that the
flat calls (nrt_uv_raster_device, nrt_bake_lightmap_device) take."""
import ctypes as C
import threading

import numpy as np
import pytest

from test_gpu_scene_path import SceneSetup, _multv, _unit_cross

pytestmark = pytest.mark.gpu

AW, AH = 128, 128
CHARTS = {0: (0, 0, 64, 64, (0.0, 1.0, 0.0, 1.0), (0.5, 0.5), 0, 0),
          2: (64, 0, 48, 40, (0.05, 0.95, 0.1, 0.9), (0.25, 0.75), 1, 1),
          3: (64, 40, 48, 40, (0.0, 1.0, 0.0, 1.0), (0.5, 0.5), 0, 0)}
MIN_T = np.float32(1e-3)


def _grid_uvs(nf):
    """a UV mesh in SetupVerticesForUVRaster's layout: triangle i in cell i of a square grid over [0, 1]^2"""
    g = int(np.ceil(np.sqrt(nf)))
    v = np.zeros((nf, 3, 3), np.float32)
    for i in range(nf):
        x, y = (i % g) / g, (i // g) / g
        e = 0.9 / g
        v[i] = [[x + 0.05 / g, y + 0.05 / g, 0], [x + e, y + 0.05 / g, 0], [x + 0.05 / g, y + e, 0]]
    return v.reshape(-1, 3), np.arange(3 * nf, dtype=np.uint32).reshape(-1, 3)


class Bake:
    """The scene, its UV accels and charts, and the atlas buffers."""

    def __init__(self, with_normals, charts=CHARTS, aw=AW, ah=AH):
        import torch
        from nanort_b200 import api

        self.torch, self.api = torch, api
        self.ss = ss = SceneSetup(with_normals)
        if with_normals:  # the tilted normals face the walls' outside and the boxes' inside: bake the lit sides
            for d_n in ss.keep[1::2]:
                d_n.neg_()
            ss.fvn = -ss.fvn
        self.states = ss.sc.InstanceStates()
        self.aw, self.ah = aw, ah
        self.uv = {}
        for i in charts:
            v, f = ss.insts[i][0], ss.insts[i][1]
            key = (v.ctypes.data, f.ctypes.data)
            if key not in self.uv:
                uvv, uvf = _grid_uvs(len(f))
                a = api.BVHAccel()
                a.Build(len(uvf), uvv, uvf)
                self.uv[key] = a
        self.charts = []
        for i in range(len(ss.insts)):
            c = api.SceneChart()
            if i in charts:
                x0, y0, w, h, region, off, fx, fy = charts[i]
                c.uv = self.uv[(ss.insts[i][0].ctypes.data, ss.insts[i][1].ctypes.data)]._h
                c.x0, c.y0, c.width, c.height = x0, y0, w, h
                c.uv_region[:], c.texel_offset[:] = region, off
                c.flip_x, c.flip_y = fx, fy
            self.charts.append(c)
        self.with_normals = with_normals

    def uv_accel(self, i):
        return self.uv[(self.ss.insts[i][0].ctypes.data, self.ss.insts[i][1].ctypes.data)]

    def raster(self, flags=0, aovs=True):
        torch = self.torch
        AW, AH = self.aw, self.ah
        rec = torch.zeros(AW * AH * 4, dtype=torch.int32, device="cuda")
        inst = torch.zeros(AW * AH, dtype=torch.int32, device="cuda")
        pos = torch.full((AW * AH * 3,), 7.0, device="cuda") if aovs else None
        nrm = torch.full((AW * AH * 3,), 7.0, device="cuda") if aovs and self.with_normals else None
        n = self.ss.sc.UVRaster(self.charts, AW, AH, rec.data_ptr(), inst.data_ptr(),
                                shading=self.ss.shading if nrm is not None else None,
                                d_position_ptr=pos.data_ptr() if pos is not None else None,
                                d_normal_ptr=nrm.data_ptr() if nrm is not None else None, flags=flags)
        self.d_rec, self.d_inst = rec, inst
        out = (rec.cpu().numpy().view(np.float32).reshape(-1, 4), inst.cpu().numpy().view(np.uint32))
        return n, out[0], out[1], (pos.cpu().numpy().reshape(-1, 3) if pos is not None else None), \
            (nrm.cpu().numpy().reshape(-1, 3) if nrm is not None else None)

    def texel_model(self, rec, inst):
        """float32 restatement of the texel point: P, n of every covered texel (host-flattened triangles)"""
        ss = self.ss
        cov = np.flatnonzero(rec[:, 3].view(np.uint32) != 0xFFFFFFFF)
        face = ss.offsets[inst[cov]] + rec[cov, 3].view(np.uint32)
        tri = ss.v[ss.f[face]]
        u, v = rec[cov, 0], rec[cov, 1]
        w = np.float32(1.0) - u - v
        P = (w[:, None] * tri[:, 0] + u[:, None] * tri[:, 1]) + v[:, None] * tri[:, 2]
        n = _unit_cross(tri)
        if ss.fvn is not None:
            fn = ss.fvn[face].reshape(-1, 3, 3)
            s = (w[:, None] * fn[:, 0] + u[:, None] * fn[:, 1]) + v[:, None] * fn[:, 2]
            flip = np.sum(n * s, axis=1) < 0
        else:
            det = np.array([np.linalg.det(self.states["xform"][i][:3, :3].astype(np.float64)) for i in range(len(ss.insts))])
            flip = det[inst[cov]] < 0
        n[flip] *= -1
        return cov, face, P, n


def _flat_world(ss, i):
    """a world accel of instance i's host-flattened triangles, its world normals, and the instance's state"""
    from nanort_b200 import api

    v, f = ss.insts[i][0], ss.insts[i][1]
    st = ss.sc.InstanceStates()[i]
    a = api.BVHAccel()
    a.Build(len(f), _multv(st["xform"], v), f)
    return a


# ------------------------------------------------------------------ 1. texel cast
@pytest.mark.parametrize("with_normals", [False, True])
def test_charts_are_the_flat_cast_bit_for_bit(with_normals):
    import torch
    from nanort_b200 import api

    bk = Bake(with_normals)
    ss = bk.ss
    for flags in (api.TRAVERSE_FAST, api.TRAVERSE_CONFORMANCE):
        n, rec, inst, pos, nrm = bk.raster(flags)
        owner = np.full((AH, AW), 0xFFFFFFFF, np.uint32)
        covered = 0
        for i, (x0, y0, w, h, region, off, fx, fy) in CHARTS.items():
            p = api.UvRasterParams()
            p.width, p.height, p.flip_x, p.flip_y, p.flags = w, h, fx, fy, flags
            p.uv_region[:], p.texel_offset[:] = region, off
            world = _flat_world(ss, i)
            frec = torch.zeros(w * h * 4, dtype=torch.int32, device="cuda")
            fpos = torch.zeros(w * h * 3, device="cuda")
            fnrm = torch.zeros(w * h * 3, device="cuda") if with_normals else None
            keep = None
            if with_normals:
                ln = ss.keep[2 * i + 1].cpu().numpy().reshape(-1, 3)
                keep = torch.as_tensor(_multv(bk.states["invT33"][i], ln).reshape(-1), device="cuda")
            c = bk.uv_accel(i).UVRaster(p, frec.data_ptr(), world=world, d_position_ptr=fpos.data_ptr(),
                                        d_normal_ptr=fnrm.data_ptr() if fnrm is not None else None,
                                        d_facevarying_normals_ptr=keep.data_ptr() if keep is not None else None)
            covered += c
            sl = (slice(y0, y0 + h), slice(x0, x0 + w))
            got = rec.reshape(AH, AW, 4)[sl]
            assert got.tobytes() == frec.cpu().numpy().view(np.float32).reshape(h, w, 4).tobytes(), (i, flags)
            assert pos.reshape(AH, AW, 3)[sl].tobytes() == fpos.cpu().numpy().reshape(h, w, 3).tobytes(), (i, flags)
            if with_normals:
                assert nrm.reshape(AH, AW, 3)[sl].tobytes() == fnrm.cpu().numpy().reshape(h, w, 3).tobytes(), i
            hit = got[..., 3].view(np.uint32) != 0xFFFFFFFF
            owner[sl][hit] = i
            assert 0 < hit.sum() < w * h
        assert n == covered
        assert np.array_equal(inst.reshape(AH, AW), owner)
        empty = owner.reshape(-1) == 0xFFFFFFFF
        want = np.array([0, 0, 1e30, 0], np.float32)
        want[3] = np.uint32(0xFFFFFFFF).view(np.float32)
        assert np.all(rec[empty].view(np.uint32) == want.view(np.uint32))
        assert not pos[empty].any() and (nrm is None or not nrm[empty].any())


# ------------------------------------------------------------------ 2. texel point, 3. AO bake
def _ao_params(bk, spp, seed=3, flags=0, sample0=0):
    p = bk.api.BakeParams()
    p.width, p.height, p.spp, p.sample0, p.seed = bk.aw, bk.ah, spp, sample0, seed
    p.ao_min_t, p.ao_max_t, p.flags, p.d_facevarying_normals = float(MIN_T), 3.0, flags, None
    return p


def _export(bk, p, shading, cap=None):
    torch = bk.torch
    cap = bk.aw * bk.ah * p.spp if cap is None else cap
    d = torch.zeros(cap * 9, dtype=torch.int32, device="cuda")
    n = bk.ss.sc.ExportBakeRays(bk.d_rec.data_ptr(), bk.d_inst.data_ptr(), p, d.data_ptr(), cap, shading=shading)
    from nanort_b200 import scenes as S

    return d.cpu().numpy().view(S.RAY_DTYPE)[:n].copy()


@pytest.mark.parametrize("with_normals", [False, True])
def test_texel_normals_and_ao_origins(with_normals):
    bk = Bake(with_normals)
    ss = bk.ss
    _, rec, inst, _, _ = bk.raster()
    cov, face, P, n = bk.texel_model(rec, inst)
    p = _ao_params(bk, 2)
    rays = _export(bk, p, ss.shading if with_normals else None)
    assert len(rays) == 2 * len(cov)
    k = np.arange(len(rays)) % len(cov)
    want = P[k] + n[k] * MIN_T
    assert np.max(np.abs(rays["org"] - want) / np.maximum(np.abs(want), 1e-3)) <= 1e-6
    assert np.all(np.sum(rays["dir"] * n[k], axis=1) >= 0)  # cosine directions about n
    assert np.all(rays["min_t"] == 0) and np.all(rays["max_t"] == np.float32(3.0))
    if not with_normals:  # both boxes (one mirrored) bake their outside
        for i in (2, 3):
            m = inst[cov] == i
            c = _multv(bk.states["xform"][i], ss.insts[i][0].mean(axis=0, keepdims=True))[0]
            assert m.sum() > 100 and np.all(np.sum(n[m] * (P[m] - c), axis=1) > 0), i


def test_ao_bake_equals_the_reference_walk_of_its_rays():
    """conformance walk: exact per-texel counts of orc.PortScene over the exported rays; production walk: the same
    except on exact-distance ties"""
    from oracle import orc
    from nanort_b200 import api

    torch = pytest.importorskip("torch")
    bk = Bake(False)
    ss = bk.ss
    bk.raster()
    rec = bk.d_rec.cpu().numpy().view(np.uint32).reshape(-1, 4)
    texels = np.flatnonzero(rec[:, 3] != 0xFFFFFFFF)
    port = orc.PortScene([(v, f, x) for v, f, x, _ in ss.insts])
    for flags in (api.TRAVERSE_CONFORMANCE, api.TRAVERSE_FAST):
        p = _ao_params(bk, 4, flags=flags)
        rays = _export(bk, p, None)
        h, m = port.traverse(rays, threads=4)
        occ = (m == 1) & (h["t"] < np.float32(3.0))
        want = np.zeros(AW * AH)
        np.add.at(want, texels[np.arange(len(rays)) % len(texels)], (~occ).astype(np.float64))
        acc = torch.zeros(AW * AH, device="cuda")
        r = ss.sc.BakeAO(bk.d_rec.data_ptr(), bk.d_inst.data_ptr(), p, acc.data_ptr())
        got = acc.cpu().numpy()
        assert r.texels == len(texels) and r.ao_rays == len(rays) and r.traverse_launches == 1
        if flags == api.TRAVERSE_CONFORMANCE:
            assert np.array_equal(got, want) and r.ao_hits == int(occ.sum())
        else:
            diff = int(np.abs(got - want).sum())
            print(f"production walk: {diff} of {len(rays)} AO rays differ (exact-distance ties)")
            assert diff <= 1e-3 * len(rays) and abs(r.ao_hits - int(occ.sum())) <= diff


# ------------------------------------------------------------------ 4. lightmap bounce 0
def _lm_params(bk, spp, bounces, seed=5, sample0=0, flags=0):
    ss = bk.ss
    p = bk.api.LightmapParams()
    p.width, p.height, p.spp, p.sample0, p.seed, p.max_bounces = bk.aw, bk.ah, spp, sample0, seed, bounces
    p.ray_min_t, p.ray_max_t = float(MIN_T), 1e30
    p.n_materials, p.n_emissive = len(ss.mats), len(ss.pairs)
    p.d_materials, p.d_material_ids, p.d_emissive_faces = ss.d_mats.data_ptr(), None, ss.d_pairs.data_ptr()
    p.d_facevarying_normals, p.flags = None, flags
    return p


class Queues:
    def __init__(self, torch, n):
        z = lambda *s: torch.zeros(s, dtype=torch.float32, device="cuda")
        self.q = [[z(n, 4), z(n, 4), torch.zeros(n, dtype=torch.int32, device="cuda")] for _ in range(2)]
        self.sh = [z(n, 4) for _ in range(3)]
        self.w = z(n, 4)

    def run(self, bk, p, b, n, accum, cur=0):
        a, o = self.q[cur], self.q[cur ^ 1]
        return bk.ss.sc.LightmapBounce(bk.d_rec.data_ptr(), bk.d_inst.data_ptr(), p, bk.ss.shading, b, n,
                                       a[0].data_ptr(), a[1].data_ptr(), a[2].data_ptr(), self.w.data_ptr(),
                                       o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), self.sh[0].data_ptr(),
                                       self.sh[1].data_ptr(), self.sh[2].data_ptr(), accum.data_ptr())


@pytest.mark.parametrize("with_normals", [False, True])
def test_texel_vertex_spawns_lifted_rays_above_the_texel(with_normals):
    import torch

    bk = Bake(with_normals)
    _, rec, inst, _, _ = bk.raster()
    cov, face, P, n = bk.texel_model(rec, inst)
    spp = 2
    N = len(cov) * spp
    p = _lm_params(bk, spp, 3)
    qs = Queues(torch, N)
    accum = torch.zeros(AW * AH * 3, device="cuda")
    nc, ns = qs.run(bk, p, 0, N, accum, cur=1)
    assert nc == N and 0 < ns <= N  # white Lambertian: every path continues
    pid = qs.q[0][2].cpu().numpy()[:nc]
    assert np.array_equal(np.sort(pid), np.arange(N))
    k = pid % len(cov)
    co, cd = qs.q[0][0].cpu().numpy()[:nc], qs.q[0][1].cpu().numpy()[:nc]
    want = P[k] + n[k] * MIN_T  # lifted along n: the continuation leaves on n's side
    assert np.max(np.abs(co[:, :3] - want) / np.maximum(np.abs(want), 1e-3)) <= 1e-6
    assert np.all(np.sum(cd[:, :3] * n[k], axis=1) >= 0) and np.all(qs.w.cpu().numpy()[:N, :3] == 1.0)
    so, sd, sc = (x.cpu().numpy()[:ns] for x in qs.sh)
    tex = sc[:, 3].view(np.uint32)
    km = {t: j for j, t in enumerate(cov)}
    kk = np.array([km[t] for t in tex])
    assert np.all(np.sum(sd[:, :3] * n[kk], axis=1) > 0), "a shadow ray below the texel's hemisphere"
    want = P[kk] + n[kk] * MIN_T
    assert np.max(np.abs(so[:, :3] - want) / np.maximum(np.abs(want), 1e-3)) <= 1e-6
    # the cosine continuation: cos^2 of the angle to n is uniform on [0, 1]
    from scipy import stats

    c2 = np.clip(np.sum(cd[:, :3] * n[k], axis=1), 0.0, 1.0) ** 2
    assert stats.kstest(c2, "uniform").pvalue > 1e-3
    # against the flat bake's texel vertex (checked against the float64 model in test_gpu_lightmap.py) on the flattened
    # mesh with mapped records: the same paths continue in the same directions, the same texels get a shadow ray, with
    # the same direction and contribution; only the origins differ, by the lift
    acc, d_rec, pf, _keep = _flat(bk, rec, inst, spp, 3)
    fq = Queues(torch, N)
    faccum = torch.zeros(AW * AH * 3, device="cuda")
    f_in, f_out = fq.q[1], fq.q[0]
    fnc, fns = acc.LightmapBounce(d_rec.data_ptr(), pf, 0, N, None, None, None, fq.w.data_ptr(), f_out[0].data_ptr(),
                                  f_out[1].data_ptr(), f_out[2].data_ptr(), fq.sh[0].data_ptr(), fq.sh[1].data_ptr(),
                                  fq.sh[2].data_ptr(), faccum.data_ptr(), skip_shadow_pass=True)
    assert (fnc, fns) == (nc, ns)
    fpid = f_out[2].cpu().numpy()[:fnc]
    fcd = f_out[1].cpu().numpy()[:fnc]
    assert np.max(np.abs(fcd[np.argsort(fpid)][:, :3] - cd[np.argsort(pid)][:, :3])) <= 1e-6
    assert np.array_equal(fq.w.cpu().numpy()[:N], qs.w.cpu().numpy()[:N])
    fsd, fsc = fq.sh[1].cpu().numpy()[:fns], fq.sh[2].cpu().numpy()[:fns]
    ftex = fsc[:, 3].view(np.uint32)
    kg = np.lexsort((sd[:, 2], sd[:, 1], sd[:, 0], tex))
    kf = np.lexsort((fsd[:, 2], fsd[:, 1], fsd[:, 0], ftex))
    assert np.array_equal(tex[kg], ftex[kf])
    assert np.max(np.abs(sd[kg][:, :3] - fsd[kf][:, :3])) <= 1e-6
    rel = np.abs(sc[kg][:, :3] - fsc[kf][:, :3]) / np.maximum(np.abs(fsc[kf][:, :3]), 1e-6)
    assert float(rel.max()) <= 1e-5, float(rel.max())


# ------------------------------------------------------------------ 6. composition
@pytest.fixture(scope="module")
def bk():
    b = Bake(True)
    b.raster()
    return b


def _bake(bk, p, stream=None):
    accum = bk.torch.zeros(bk.aw * bk.ah * 3, device="cuda")
    r = bk.ss.sc.BakeLightmap(bk.d_rec.data_ptr(), bk.d_inst.data_ptr(), p, bk.ss.shading, accum.data_ptr(),
                              stream=stream)
    return accum.cpu().numpy().astype(np.float64).reshape(-1, 3), r


def _within(a, b, m):
    bound = 2.0 * m * 2.0 ** -24 * np.maximum(a, b) * 1.01
    assert not (np.abs(a - b) > bound).any(), float(np.abs(a - b).max())


def test_whole_bake_equals_the_sum_of_its_bounces(bk):
    import torch
    from nanort_b200 import api

    spp, bounces = 3, 5
    p = _lm_params(bk, spp, bounces, flags=api.TRAVERSE_CONFORMANCE)
    whole, r = _bake(bk, p)
    n_cov = int((bk.d_rec.cpu().numpy().view(np.uint32).reshape(-1, 4)[:, 3] != 0xFFFFFFFF).sum())
    assert r.texels == n_cov and r.paths == n_cov * spp and r.shadow_rays > 0 and whole.sum() > 0
    N = n_cov * spp
    qs = Queues(torch, N)
    accum = torch.zeros(AW * AH * 3, device="cuda")
    k, cur, radiance, shadow, walks = N, 1, 0, 0, 0
    for b in range(bounces):
        if k == 0:
            break
        nc, ns = qs.run(bk, p, b, k, accum, cur=cur if b else 1)
        radiance += k if b else 0
        shadow += ns
        walks += (1 if b else 0) + (1 if ns else 0)
        k, cur = nc, (cur ^ 1 if b else 0)
    assert (radiance, shadow, walks) == (r.radiance_rays, r.shadow_rays, r.traverse_launches)
    _within(whole, accum.cpu().numpy().astype(np.float64).reshape(-1, 3), spp * bounces)


def test_sample_ranges_repeated_calls_and_two_streams_compose(bk):
    import torch
    from nanort_b200 import api

    f = api.TRAVERSE_CONFORMANCE
    whole, r = _bake(bk, _lm_params(bk, 6, 4, flags=f))
    a, ra = _bake(bk, _lm_params(bk, 2, 4, flags=f))
    b, rb = _bake(bk, _lm_params(bk, 4, 4, sample0=2, flags=f))
    assert (ra.shadow_rays + rb.shadow_rays, ra.radiance_rays + rb.radiance_rays) == (r.shadow_rays, r.radiance_rays)
    _within(whole, a + b, 6 * 4)
    again, _ = _bake(bk, _lm_params(bk, 6, 4, flags=f))
    _within(whole, again, 6 * 4)
    streams = [torch.cuda.Stream() for _ in range(2)]
    accs = [torch.zeros(AW * AH * 3, device="cuda") for _ in range(2)]
    cfg = [_lm_params(bk, 6, 4, flags=f), _lm_params(bk, 3, 2, seed=9, flags=f)]
    torch.cuda.synchronize()

    def run(k):
        bk.ss.sc.BakeLightmap(bk.d_rec.data_ptr(), bk.d_inst.data_ptr(), cfg[k], bk.ss.shading, accs[k].data_ptr(),
                              stream=streams[k].cuda_stream)

    th = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    torch.cuda.synchronize()
    _within(whole, accs[0].cpu().numpy().astype(np.float64).reshape(-1, 3), 6 * 4)
    solo, _ = _bake(bk, cfg[1])
    _within(solo, accs[1].cpu().numpy().astype(np.float64).reshape(-1, 3), 3 * 2)


# ------------------------------------------------------------------ 7. against the flat bake of the flattened mesh
def _flat(bk, rec, inst, spp, bounces):
    """the flattened mesh as a flat accel, the scene records mapped to it (prim = offset[instance] + prim) and the flat
    bake's parameters.  Without normals the flat bake gets constant per-face normals: on charted instances the unit
    cross(e1, e2) times the sign of the determinant (the texel normal's rule), on the light -cross(e1, e2)
    (calcNormal's orientation, which its cosine EDF reads at bounces 1 and up, as the scene pass does)"""
    torch, ss = bk.torch, bk.ss
    flat_rec = rec.copy()
    cov = inst != 0xFFFFFFFF
    flat_rec[cov, 3] = (ss.offsets[inst[cov]] + rec[cov, 3].view(np.uint32)).view(np.float32)
    acc, keep = ss.flat_accel()
    if bk.with_normals:
        fvn = keep[2]
    else:
        det = np.array([np.linalg.det(bk.states["xform"][i][:3, :3].astype(np.float64)) for i in range(len(ss.insts))])
        sign = np.concatenate([np.full(len(x[1]), np.sign(det[i]) if i in CHARTS else -1.0, np.float32)
                               for i, x in enumerate(ss.insts)])
        g = _unit_cross(ss.v[ss.f]) * sign[:, None]
        fvn = torch.as_tensor(np.repeat(g, 3, axis=0).reshape(-1), device="cuda")
    d_rec = torch.as_tensor(flat_rec.view(np.int32).reshape(-1), device="cuda")
    p = _lm_params(bk, spp, bounces)
    p.d_material_ids, p.d_emissive_faces, p.d_facevarying_normals = keep[0].data_ptr(), keep[1].data_ptr(), fvn.data_ptr()
    return acc, d_rec, p, (keep, fvn)


@pytest.mark.parametrize("with_normals", [False, True])
@pytest.mark.parametrize("bounces", [1, 5])
def test_the_scene_bakes_like_its_flattened_mesh(with_normals, bounces):
    """records mapped to the flattened mesh (prim = offset[instance] + prim), same atlas and seeds: every 16 x 16 block
    mean within 4 sigma, total energy within 1 % (the flat inputs: _flat)"""
    import torch

    bk = Bake(with_normals)
    _, rec, inst, _, _ = bk.raster()
    spp = 64
    scene, _ = _bake(bk, _lm_params(bk, spp, bounces))
    cov = inst != 0xFFFFFFFF
    acc, d_rec, p, _keep = _flat(bk, rec, inst, spp, bounces)
    accum = torch.zeros(AW * AH * 3, device="cuda")
    acc.BakeLightmap(d_rec.data_ptr(), p, accum.data_ptr())
    flat = accum.cpu().numpy().astype(np.float64).reshape(-1, 3)
    a, b = scene.sum(axis=1).reshape(AH, AW) / spp, flat.sum(axis=1).reshape(AH, AW) / spp
    assert abs(a.sum() - b.sum()) <= 0.01 * b.sum(), (a.sum(), b.sum())
    worst = 0.0
    for y in range(0, AH, 16):
        for x in range(0, AW, 16):
            m = cov.reshape(AH, AW)[y:y + 16, x:x + 16]
            if m.sum() < 8:
                continue
            ba, bb = a[y:y + 16, x:x + 16][m], b[y:y + 16, x:x + 16][m]
            sigma = np.sqrt((ba.var() + bb.var()) / len(ba)) + 1e-6
            worst = max(worst, abs(ba.mean() - bb.mean()) / sigma)
    assert worst <= 4.0, worst
    # the two boxes share a mesh and a UV accel, yet bake different charts
    c2 = a[0:40, 64:112][cov.reshape(AH, AW)[0:40, 64:112]]
    c3 = a[40:80, 64:112][cov.reshape(AH, AW)[40:80, 64:112]]
    assert abs(c2.mean() - c3.mean()) > 1e-3 * max(c2.mean(), c3.mean())


# ------------------------------------------------------------------ 9. refusals
def test_refusals_write_nothing(bk):
    import torch
    from nanort_b200 import api

    L = api.lib()
    ss = bk.ss
    vp = C.c_void_p
    rec = torch.full((AW * AH * 4,), 7, dtype=torch.int32, device="cuda")
    inst = torch.full((AW * AH,), 7, dtype=torch.int32, device="cuda")

    def chart_case(over):
        arr = bk.ss.sc._charts(bk.charts)
        for (i, k), v in over.items():
            setattr(arr[i], k, v)
        return L.nrt_scene_uv_raster_device(ss.sc._h, C.cast(arr, vp), AW, AH, 0, None, vp(rec.data_ptr()),
                                            vp(inst.data_ptr()), None, None, None, None)

    assert chart_case({(3, "y0"): 30}) == -1  # overlaps chart 2
    assert chart_case({(0, "width"): AW + 1}) == -1  # outside the atlas
    assert chart_case({(1, "uv"): bk.uv_accel(0)._h, (1, "x0"): 112, (1, "width"): 16, (1, "height"): 16}) == -1
    torch.cuda.synchronize()
    assert bool((rec == 7).all()) and bool((inst == 7).all())

    accum = torch.zeros(AW * AH * 3, device="cuda")
    arr = ss.sc._shading(ss.shading)

    def lm(p, sh=arr, d_inst=bk.d_inst):
        return L.nrt_scene_bake_lightmap_device(ss.sc._h, vp(bk.d_rec.data_ptr()), vp(d_inst.data_ptr()), C.byref(p),
                                                C.cast(sh, vp) if sh is not None else None, vp(accum.data_ptr()), None,
                                                None)

    bad_pairs = torch.as_tensor(np.array([3, 12], np.int32), device="cuda")
    bad_inst = bk.d_inst.clone()
    bad_inst[bk.d_rec.view(-1, 4)[:, 3] != -1] = 1  # instance 1 (the light) has 2 faces
    cases = [
        (lambda: lm(_lm_params(bk, 2, 2, flags=api.TRAVERSE_ANY_HIT))),
        (lambda: lm(_lm_params(bk, 2, 2), sh=None)),
        (lambda: lm(_lm_params(bk, 2, 2), d_inst=bad_inst)),
    ]
    p = _lm_params(bk, 2, 2)
    p.d_material_ids = ss.keep[0].data_ptr()
    cases.append(lambda: lm(p))
    p2 = _lm_params(bk, 2, 2)
    p2.n_emissive, p2.d_emissive_faces = 1, bad_pairs.data_ptr()
    cases.append(lambda: lm(p2))
    bp = _ao_params(bk, 2)
    bp.d_facevarying_normals = ss.keep[1].data_ptr()
    acc1 = torch.zeros(AW * AH, device="cuda")
    cases.append(lambda: L.nrt_scene_bake_ao_device(ss.sc._h, vp(bk.d_rec.data_ptr()), vp(bk.d_inst.data_ptr()), None,
                                                    C.byref(bp), vp(acc1.data_ptr()), None, None))
    ba = _ao_params(bk, 2, flags=api.TRAVERSE_ANY_HIT)
    cases.append(lambda: L.nrt_scene_bake_ao_device(ss.sc._h, vp(bk.d_rec.data_ptr()), vp(bk.d_inst.data_ptr()), None,
                                                    C.byref(ba), vp(acc1.data_ptr()), None, None))
    for k, c in enumerate(cases):
        assert c() == -1 and L.nrt_last_error().decode(), k
    torch.cuda.synchronize()
    assert not accum.any() and not acc1.any()


# ------------------------------------------------------------------ waves
# 512^2 walls and two 384 x 320 box charts in a 1024 x 640 atlas: enough covered texels for a lightmap bake of more
# than one 8 Mi-path wave and an AO bake of more than one 4 Mi-ray wave at a few dozen samples per texel
WAVE_CHARTS = {0: (0, 0, 512, 512, (0.0, 1.0, 0.0, 1.0), (0.5, 0.5), 0, 0),
               2: (512, 0, 384, 320, (0.05, 0.95, 0.1, 0.9), (0.25, 0.75), 1, 1),
               3: (512, 320, 384, 320, (0.0, 1.0, 0.0, 1.0), (0.5, 0.5), 0, 0)}


@pytest.fixture(scope="module")
def wave_bk():
    b = Bake(False, WAVE_CHARTS, 1024, 640)
    n, _, _, _, _ = b.raster(aovs=False)
    b.n_cov = n
    return b


def test_lightmap_bake_across_waves_equals_its_sample_ranges(wave_bk):
    """conformance walk: a bake of two 8 Mi-path waves (the second starting inside a texel's samples) against the same
    samples as two single-wave calls; equal ray counts, the atlas within the atomic-order bound"""
    from nanort_b200 import api

    bk, f, bounces = wave_bk, api.TRAVERSE_CONFORMANCE, 3
    spp = (9 << 20) // bk.n_cov + 1
    s1 = spp // 2
    assert bk.n_cov * spp > 8 << 20 and bk.n_cov * (spp - s1) <= 8 << 20 and (8 << 20) % bk.n_cov != 0
    whole, r = _bake(bk, _lm_params(bk, spp, bounces, flags=f))
    assert r.paths == bk.n_cov * spp and r.traverse_launches > 2 * bounces - 1  # one wave walks at most 2 b - 1 times
    a, ra = _bake(bk, _lm_params(bk, s1, bounces, flags=f))
    b, rb = _bake(bk, _lm_params(bk, spp - s1, bounces, sample0=s1, flags=f))
    assert ra.traverse_launches <= 2 * bounces - 1 and rb.traverse_launches <= 2 * bounces - 1
    assert (ra.radiance_rays + rb.radiance_rays, ra.shadow_rays + rb.shadow_rays) == (r.radiance_rays, r.shadow_rays)
    assert whole.sum() > 0
    _within(whole, a + b, spp * bounces)


def test_ao_bake_across_waves_equals_the_reference_walk_of_its_rays(wave_bk):
    """conformance walk: more than 4 Mi AO rays (two waves); the exported rays walked by orc.PortScene give the bake's
    per-texel counts and ao_hits exactly"""
    from oracle import orc
    from nanort_b200 import api

    bk = wave_bk
    torch = bk.torch
    spp = (4 << 20) // bk.n_cov + 2
    total = bk.n_cov * spp
    assert total > 4 << 20
    p = _ao_params(bk, spp, flags=api.TRAVERSE_CONFORMANCE)
    rays = _export(bk, p, None, cap=total)
    assert len(rays) == total
    rec = bk.d_rec.cpu().numpy().view(np.uint32).reshape(-1, 4)
    texels = np.flatnonzero(rec[:, 3] != 0xFFFFFFFF)
    h, m = orc.PortScene([(v, f, x) for v, f, x, _ in bk.ss.insts]).traverse(rays, threads=8)
    occ = (m == 1) & (h["t"] < np.float32(3.0))
    want = np.zeros(bk.aw * bk.ah)
    np.add.at(want, texels[np.arange(total) % len(texels)], (~occ).astype(np.float64))
    acc = torch.zeros(bk.aw * bk.ah, device="cuda")
    r = bk.ss.sc.BakeAO(bk.d_rec.data_ptr(), bk.d_inst.data_ptr(), p, acc.data_ptr())
    assert r.traverse_launches == 2 and r.ao_rays == total
    assert np.array_equal(acc.cpu().numpy(), want) and r.ao_hits == int(occ.sum())


# ------------------------------------------------------------------ 8. furnace over instances
def test_furnace_over_instances_every_texel_bakes_to_one():
    """test_gpu_lightmap.py's furnace as a scene: the faceted sphere of unit emitters as two instances (its two halves of
    faces), the quad as two instances of one triangle (identity, and rotated 180 degrees about y), each quad instance
    with its own chart over one shared UV accel.  Every texel's E / pi lies in [cos_min, 1] within the flat test's
    bounds, and both charts agree."""
    import torch
    from nanort_b200 import api
    from test_gpu_lightmap import _sphere_furnace

    (v, f, mats, ids, emissive, _, _), cos_min = _sphere_furnace()
    n_e = len(emissive)
    half = [np.ascontiguousarray(f[:n_e // 2]), np.ascontiguousarray(f[n_e // 2:n_e])]
    qv = v[f[n_e]].astype(np.float32)  # one triangle of the quad, normal +y
    rot = np.diag([-1.0, 1.0, -1.0, 1.0]).astype(np.float32)
    tri = np.arange(3, dtype=np.uint32).reshape(1, 3)
    sc, keep, shading = api.Scene(), [], []
    sphere = []
    for hf in half:
        a = api.BVHAccel()
        a.Build(len(hf), v, hf)
        sphere.append(a)
        sc.AddNode(a, np.eye(4, dtype=np.float32))
    quad = api.BVHAccel()
    quad.Build(1, qv, tri)
    sc.AddNode(quad, np.eye(4, dtype=np.float32))
    sc.AddNode(quad, rot)
    assert sc.Commit()
    for i, nf in enumerate([len(half[0]), len(half[1]), 1, 1]):
        d = torch.as_tensor(np.full(nf, 0 if i < 2 else 1, np.int32), device="cuda")
        keep.append(d)
        shading.append(api.SceneShading(d.data_ptr(), None))
    uv = api.BVHAccel()
    uv.Build(1, np.float32([[0, 0, 0], [1, 1, 0], [1, 0, 0]]), tri)
    charts = []
    for i in range(4):
        c = api.SceneChart()
        if i >= 2:
            c.uv, c.x0, c.y0, c.width, c.height = uv._h, 32 * (i - 2), 0, 32, 32
            c.uv_region[:], c.texel_offset[:] = (0.0, 1.0, 0.0, 1.0), (0.5, 0.5)
        charts.append(c)
    W, H = 64, 32
    rec = torch.zeros(W * H * 4, dtype=torch.int32, device="cuda")
    inst = torch.zeros(W * H, dtype=torch.int32, device="cuda")
    n_cov = sc.UVRaster(charts, W, H, rec.data_ptr(), inst.data_ptr())
    pairs = np.concatenate([np.stack([np.full(len(hf), i), np.arange(len(hf))], axis=1) for i, hf in enumerate(half)])
    d_pairs = torch.as_tensor(pairs.astype(np.int32).reshape(-1), device="cuda")
    d_mats = torch.as_tensor(np.ascontiguousarray(mats).view(np.float32).reshape(-1), device="cuda")
    spp = 1024
    for bounces in (1, 8):
        p = api.LightmapParams()
        p.width, p.height, p.spp, p.sample0, p.seed, p.max_bounces = W, H, spp, 0, 4, bounces
        p.ray_min_t, p.ray_max_t = 1e-3, 1e30
        p.n_materials, p.n_emissive = len(mats), len(pairs)
        p.d_materials, p.d_emissive_faces = d_mats.data_ptr(), d_pairs.data_ptr()
        accum = torch.zeros(W * H * 3, device="cuda")
        r = sc.BakeLightmap(rec.data_ptr(), inst.data_ptr(), p, shading, accum.data_ptr())
        ins = inst.cpu().numpy().view(np.uint32)
        got = accum.cpu().numpy().reshape(-1, 3).astype(np.float64)
        m = got[ins != 0xFFFFFFFF] / spp
        assert len(m) == n_cov > 800 and np.allclose(m[:, 0], m[:, 1], rtol=1e-5)
        m = m[:, 0]
        sd = float(m.std())
        assert sd < 0.1, sd
        se = 5 * sd / np.sqrt(len(m))
        assert cos_min - se <= float(m.mean()) <= 1.0 + se, (float(m.mean()), sd, cos_min)
        assert float(m.min()) >= cos_min - 6 * sd and float(m.max()) <= 1.0 + 6 * sd
        a, b = got[ins == 2, 0] / spp, got[ins == 3, 0] / spp
        assert len(a) == len(b) and abs(a.mean() - b.mean()) <= 5 * sd * np.sqrt(2.0 / len(a))
        assert r.radiance_rays == (n_cov * spp if bounces > 1 else 0)


# ------------------------------------------------------------------ refusals: a sphere instance
def test_a_sphere_instance_is_refused():
    """a chart on a sphere instance, and a lightmap bake of a scene with one, are refused before any launch"""
    import torch
    from nanort_b200 import api

    bk = Bake(False)
    walls = bk.ss.accels[(bk.ss.insts[0][0].ctypes.data, bk.ss.insts[0][1].ctypes.data)]
    sph = api.BVHAccel()
    sph.BuildSpheres(np.float32([[0.0, 2.0, 0.0]]), np.float32([0.5]))
    sc = api.Scene()
    sc.AddNode(walls, np.eye(4, dtype=np.float32))
    sc.AddNode(sph, np.eye(4, dtype=np.float32))
    assert sc.Commit()
    rec = torch.full((AW * AH * 4,), 7, dtype=torch.int32, device="cuda")
    inst = torch.full((AW * AH,), 7, dtype=torch.int32, device="cuda")
    charts = [bk.charts[0], api.SceneChart()]
    charts[1].uv, charts[1].x0, charts[1].y0, charts[1].width, charts[1].height = bk.uv_accel(0)._h, 64, 64, 32, 32
    with pytest.raises(api.NanortB200Error, match="not a triangle accel"):
        sc.UVRaster(charts, AW, AH, rec.data_ptr(), inst.data_ptr())
    assert bool((rec == 7).all()) and bool((inst == 7).all())
    p = _lm_params(bk, 2, 2)
    p.n_emissive = 0
    ids = torch.zeros(10, dtype=torch.int32, device="cuda")
    accum = torch.zeros(AW * AH * 3, device="cuda")
    with pytest.raises(api.NanortB200Error, match="triangle instances only"):
        sc.BakeLightmap(rec.data_ptr(), inst.data_ptr(), p,
                        [api.SceneShading(ids.data_ptr(), None), api.SceneShading(None, None)], accum.data_ptr())
    torch.cuda.synchronize()
    assert not accum.any()
