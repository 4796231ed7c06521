"""Path tracing over two-level scenes (csrc/scene.cu: nrt_scene_render_path_device, nrt_scene_path_bounce_device).

The test scene is S.cornell_with_materials() split into instances: the walls as one identity instance, the ceiling light
as its own translated and uniformly scaled instance, and the tall box as one mesh shared by two instances -- one rotated
with a non-uniform scale (the specular material), one mirrored (negative determinant, the glass material).  Flattened on
the host -- world vertices by the float32 MultV order, world face-varying normals by inverse_transpose33, face id =
instance offset + prim -- it is an ordinary mesh that the reference path tracer's own shading code
(oracle/_ref/libpt_ref.so, orc.ReferencePathTracer) and the flat pass (nrt_render_path_device) can render.

Scene::Traverse walks an instance with the local range {0, FLT_MAX}, so spawned rays are lifted off the surface by
ray_min_t along the unit geometric normal (continuation: the side the ray leaves; shadow: the light's side), and a shadow
ray is occluded iff it hits nearer than its max_t: where the lifted ray meets the sampled light's plane, less 1e-5 (with
dist - 1e-5 the light would occlude its own samples).  The checks below restate that rule."""
import ctypes as C

import numpy as np
import pytest

import ao_model as M

pytestmark = pytest.mark.gpu

TILE = (64, 8)
MIN_T = np.float32(1e-3)
U = 2.0 ** -24


def _xform(scale, angle_deg, translate):
    """row-vector 4x4 (p' = p . M): scale, then rotation about y, then translation"""
    c, s = np.cos(np.radians(angle_deg)), np.sin(np.radians(angle_deg))
    R = np.array([[c, 0, -s, 0], [0, 1, 0, 0], [s, 0, c, 0], [0, 0, 0, 1]], np.float64)
    S_ = np.diag([scale[0], scale[1], scale[2], 1.0])
    T = np.eye(4)
    T[3, :3] = translate
    return (S_ @ R @ T).astype(np.float32)


def _multv(m, p):
    """Matrix::MultV in float32: t[k] = ((m[0][k] x + m[1][k] y) + m[2][k] z) + m[3][k]"""
    m = np.asarray(m, np.float32).reshape(4, 4)
    p = np.asarray(p, np.float32)
    return np.stack([((m[0, k] * p[:, 0] + m[1, k] * p[:, 1]) + m[2, k] * p[:, 2]) + m[3, k] for k in range(3)], axis=1)


def _unit_cross(tri):
    """unit cross(v1 - v0, v2 - v0) of float32 triangles [n, 3, 3], the device's arithmetic"""
    e1, e2 = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], axis=1).astype(np.float32)
    ln = np.sqrt(n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2])
    il = np.where(ln > 0, np.float32(1.0) / np.where(ln > 0, ln, np.float32(1.0)), np.float32(0.0)).astype(np.float32)
    return n * il[:, None]


def _local_normals(v, f):
    """face-varying normals of a local mesh that are not its flat normal: face normal tilted towards the vertex"""
    tri = v[f].astype(np.float64)
    n = np.cross(tri[:, 2] - tri[:, 0], tri[:, 1] - tri[:, 0])
    n /= np.linalg.norm(n, axis=1)[:, None]
    c = v.astype(np.float64).mean(axis=0)
    r = tri - c
    r /= np.linalg.norm(r, axis=2)[..., None]
    return (n[:, None, :] + 0.3 * r).astype(np.float32).reshape(-1, 9)


def instanced_cornell():
    """[(verts, faces, xform, material ids)] and the material table"""
    from nanort_b200 import scenes as S

    v, f, mats, ids, emissive = S.cornell_with_materials()
    walls = (v, np.ascontiguousarray(f[0:10]), np.eye(4, dtype=np.float32), ids[0:10].copy())
    lv = v[f[emissive]].reshape(-1, 3).astype(np.float32)
    lc = np.float32([0.0, 9.99, 0.0])
    light_v = np.ascontiguousarray((lv - lc) / np.float32(2.0), np.float32)
    light = (light_v, np.arange(6, dtype=np.uint32).reshape(2, 3), _xform((2, 2, 2), 0, (0.0, 9.99, 0.0)),
             np.full(2, 5, np.uint32))
    bv = v[f[10:22]].reshape(-1, 3).astype(np.float64)
    base = np.float64([(bv[:, 0].min() + bv[:, 0].max()) / 2, 0.0, (bv[:, 2].min() + bv[:, 2].max()) / 2])
    box_v = np.ascontiguousarray(bv - base, np.float32)
    box_f = np.arange(36, dtype=np.uint32).reshape(12, 3)
    tall = (box_v, box_f, _xform((0.8, 0.9, 0.7), 25.0, (-2.0, 0.0, -1.8)), np.full(12, 3, np.uint32))
    mirrored = (box_v, box_f, _xform((-0.6, 0.45, 0.6), -15.0, (2.1, 0.0, 1.7)), np.full(12, 4, np.uint32))
    assert np.linalg.det(mirrored[2][:3, :3]) < 0
    return [walls, light, tall, mirrored], mats


class SceneSetup:
    """The device scene (reference-built trees, so that the conformance walk equals orc.PortScene bit for bit), the
    per-instance shading, the emissive pairs and the flattened mesh."""

    def __init__(self, with_normals):
        import torch
        from nanort_b200 import api

        self.torch, self.api = torch, api
        insts, mats = instanced_cornell()
        self.insts, self.mats = insts, mats
        self.sc = api.Scene()
        self.accels = {}
        for v, f, x, _ in insts:
            key = (v.ctypes.data, f.ctypes.data)
            if key not in self.accels:
                a = api.BVHAccel()
                a.Build(len(f), v, f, flags=api.BUILD_REFERENCE_TREE)
                self.accels[key] = a
            self.sc.AddNode(self.accels[key], x)
        assert self.sc.Commit(api.BUILD_REFERENCE_TREE)
        st = self.sc.InstanceStates()
        self.keep = []
        self.shading = []
        fv, ff, fids, fn = [], [], [], []
        pairs = []
        self.offsets = []
        nv = nf = 0
        for i, (v, f, x, ids) in enumerate(insts):
            ln = _local_normals(v, f) if with_normals else None
            d_ids = torch.as_tensor(ids.astype(np.int32), device="cuda")
            d_n = torch.as_tensor(ln.reshape(-1), device="cuda") if with_normals else None
            self.keep += [d_ids, d_n]
            self.shading.append(api.SceneShading(d_ids.data_ptr(), d_n.data_ptr() if d_n is not None else None))
            wv = _multv(st["xform"][i], v)
            fv.append(wv)
            ff.append(f.astype(np.uint32) + nv)
            fids.append(ids)
            if with_normals:
                fn.append(_multv(st["invT33"][i], ln.reshape(-1, 3)).reshape(-1, 9))
            for k in np.flatnonzero(mats["emission"][ids].sum(axis=1) > 0):
                pairs.append((i, k))
            self.offsets.append(nf)
            nv += len(v)
            nf += len(f)
        self.offsets = np.asarray(self.offsets, np.uint32)
        self.v, self.f, self.ids = np.concatenate(fv), np.concatenate(ff), np.concatenate(fids)
        self.fvn = np.concatenate(fn) if with_normals else None
        self.pairs = np.asarray(pairs, np.uint32)
        self.emissive = self.offsets[self.pairs[:, 0]] + self.pairs[:, 1]
        self.d_mats = torch.as_tensor(np.ascontiguousarray(mats).view(np.float32).reshape(-1), device="cuda")
        self.d_pairs = torch.as_tensor(self.pairs.reshape(-1).astype(np.int32), device="cuda")

    def params(self, W, H, spp, bounces, seed, tile=TILE, sample0=0, shard=0, n_shards=1, flags=0, cam=None):
        from nanort_b200 import scenes as S

        p = self.api.PathParams()
        cam = S.scene_camera("cornell", W, H) if cam is None else cam
        for i in range(12):
            p.cam[i] = float(cam[i])
        p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, sample0, seed
        p.tile_w, p.tile_h, p.shard, p.n_shards = tile[0], tile[1], shard, n_shards
        p.max_bounces, p.ray_min_t, p.ray_max_t = bounces, float(MIN_T), 1e30
        p.n_materials, p.n_emissive = len(self.mats), len(self.pairs)
        p.d_materials, p.d_material_ids, p.d_emissive_faces = self.d_mats.data_ptr(), None, self.d_pairs.data_ptr()
        p.d_facevarying_normals, p.flags = None, flags
        return p, cam

    def render(self, W, H, spp, bounces, seed, stream=None, **kw):
        torch = self.torch
        p, _ = self.params(W, H, spp, bounces, seed, **kw)
        accum = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
        r = self.sc.RenderPath(p, self.shading, accum.data_ptr(), stream=stream)
        return accum.cpu().numpy().astype(np.float64).reshape(-1, 3), r

    def flat_accel(self):
        """the flattened mesh as an ordinary accel + its flat-pass parameters"""
        torch, api = self.torch, self.api
        acc = api.BVHAccel()
        acc.Build(len(self.f), self.v, self.f)
        keep = [torch.as_tensor(self.ids.astype(np.int32), device="cuda"),
                torch.as_tensor(self.emissive.astype(np.int32), device="cuda")]
        if self.fvn is not None:
            keep.append(torch.as_tensor(self.fvn.reshape(-1), device="cuda"))
        return acc, keep


def _rel(a, b, floor=1e-3):
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), floor))) if a.size else 0.0


def _lift_ok(got, base, g, d):
    """got == base + ray_min_t * g flipped to the side of d; where d grazes the surface either side is accepted"""
    dot = np.sum(g * d, axis=1)
    s = np.where(dot < 0, np.float32(-1), np.float32(1)).astype(np.float32)
    want = base + (g * s[:, None]) * MIN_T
    alt = base - (g * s[:, None]) * MIN_T
    err = np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-3), axis=1)
    err_alt = np.max(np.abs(got - alt) / np.maximum(np.abs(alt), 1e-3), axis=1)
    graze = np.abs(dot) < 1e-4
    return bool(np.all((err <= 1e-5) | (graze & (err_alt <= 1e-5)))), float(err.max()) if len(err) else 0.0


def _bounce_by_bounce(with_normals, flags):
    import torch
    from nanort_b200 import api, scenes as S
    from oracle import orc

    if not orc.ReferencePathTracer.available():
        pytest.skip("oracle/_ref/libpt_ref.so not built (no reference tree at build time)")
    ss = SceneSetup(with_normals)
    W, H, spp, bounces, seed = 64, 48, 4, 8, 5
    ref = orc.ReferencePathTracer(ss.v, ss.f, ss.ids, ss.mats, facevarying_normals=ss.fvn)
    assert np.array_equal(ref.emissive_faces(), ss.emissive), "MeshLight's list != the {instance, face} pairs"
    port = orc.PortScene([(v, f, x) for v, f, x, _ in ss.insts]) if flags == api.TRAVERSE_CONFORMANCE else None
    p, cam = ss.params(W, H, spp, bounces, seed, flags=flags)
    world_tri = ss.v[ss.f]  # [n, 3, 3] float32, the device's world vertices
    g_of_face = _unit_cross(world_tri)

    pix_of_slot, smp_of_slot = M.slots(W, H, TILE[0], TILE[1], spp)
    valid = np.nonzero(pix_of_slot >= 0)[0]
    order = np.lexsort((smp_of_slot[valid], pix_of_slot[valid]))
    pid = valid[order].astype(np.uint32)
    n = len(pid)
    o4 = np.zeros((n, 4), np.float32)
    o4[:, :3], o4[:, 3] = np.asarray(cam[:3], np.float32), MIN_T
    d4 = np.zeros((n, 4), np.float32)
    d4[:, :3], d4[:, 3] = M.camera_dirs(cam, W, H, seed, pix_of_slot[pid], smp_of_slot[pid]), 1e30
    dev = "cuda"
    d_weight = torch.ones((len(pix_of_slot), 4), dtype=torch.float32, device=dev)
    accum = torch.zeros(W * H * 3, dtype=torch.float32, device=dev)
    expect = np.zeros((W * H, 3), np.float64)
    checked, seen = 0, set()
    for b in range(bounces):
        n = len(pid)
        if n == 0:
            break
        d_o, d_d = torch.as_tensor(o4, device=dev), torch.as_tensor(d4, device=dev)
        d_pid = torch.as_tensor(pid.astype(np.int32), device=dev)
        out = [torch.zeros((n, 4), dtype=torch.float32, device=dev) for _ in range(2)] + [torch.zeros(n, dtype=torch.int32, device=dev)]
        sh = [torch.zeros((n, 4), dtype=torch.float32, device=dev) for _ in range(3)]
        w_in = d_weight[torch.as_tensor(pid.astype(np.int64), device=dev)].cpu().numpy()
        n_cont, n_sh = ss.sc.PathBounce(p, ss.shading, b, n, d_o.data_ptr(), d_d.data_ptr(), d_pid.data_ptr(),
                                        d_weight.data_ptr(), out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(),
                                        sh[0].data_ptr(), sh[1].data_ptr(), sh[2].data_ptr(), accum.data_ptr())
        r = np.zeros(n, S.RAY_DTYPE)
        r["org"], r["dir"], r["min_t"], r["max_t"] = o4[:, :3], d4[:, :3], o4[:, 3], d4[:, 3]
        hits, mask = ss.sc.Traverse(r, flags=flags)
        if port is not None:  # the conformance walk is the reference's Scene::Traverse bit for bit
            ph, pm = port.traverse(r, threads=4)
            assert np.array_equal(pm, mask) and hits[mask == 1].tobytes() == ph[pm == 1].tobytes(), b
        hit = mask.astype(bool)
        h = np.nonzero(hit)[0]
        face = ss.offsets[hits["node_id"][h]] + hits["prim_id"][h]
        pix, smp = pix_of_slot[pid], smp_of_slot[pid]
        dim = 8 + 8 * b
        draws = np.stack([S.rand_ps(pix, smp, dim + k, seed) for k in range(6)], axis=1).astype(np.float32)
        want = ref.shade(b, bounces, o4[h, :3], d4[h, :3], np.stack([hits["u"][h], hits["v"][h], hits["t"][h]], axis=1),
                         face, w_in[h], draws[h])
        checked += len(h)
        cont, shad, emit = ((want["flags"] & k) != 0 for k in (1, 2, 4))
        # ---- decisions
        assert n_cont == int(cont.sum()) and n_sh == int(shad.sum()), (b, n_cont, int(cont.sum()), n_sh, int(shad.sum()))
        got_pid = out[2].cpu().numpy()[:n_cont].astype(np.uint32)
        ref_pid = pid[h][cont]
        assert np.array_equal(np.sort(got_pid), np.sort(ref_pid)), f"bounce {b}: different set of continuing paths"
        # ---- continuation rays: the reference's origin lifted off the hit triangle, its direction, the throughput
        go, gd = out[0].cpu().numpy()[:n_cont], out[1].cpu().numpy()[:n_cont]
        gs, rs = np.argsort(got_pid), np.argsort(ref_pid)
        g_cont = g_of_face[face[cont]][rs]
        ref_dir = want["next_dir"][cont][rs]
        ok, err = _lift_ok(go[gs][:, :3], want["next_org"][cont][rs], g_cont, ref_dir)
        assert ok, (b, err)
        assert float(np.max(np.abs(gd[gs][:, :3] - ref_dir))) <= 2e-5 if n_cont else True
        zero = np.all(ref_dir == 0, axis=1)  # total internal reflection: a radiance ray that misses at the root
        assert np.all(gd[gs][zero, 3] < go[gs][zero, 3]) and np.all(gd[gs][~zero, 3] == np.float32(1e30))
        w_out = d_weight[torch.as_tensor(ref_pid.astype(np.int64), device=dev)].cpu().numpy()
        assert _rel(w_out[:, :3], want["weight"][cont][:, :3], floor=1e-6) <= 1e-5
        assert np.array_equal(w_out[:, 3] != 0, want["weight"][cont][:, 3] != 0)
        # ---- shadow rays: origin lifted towards the light from the reference's, direction, max_t and contribution
        so, sd, sc_ = (x.cpu().numpy()[:n_sh] for x in sh)
        got_pix = sc_[:, 3].copy().view(np.uint32)
        ref_pix = pix[h][shad].astype(np.uint32)
        ref_org = want["shadow_org"][shad]
        ref_sd = want["shadow_dir"][shad]
        g_sh = g_of_face[face[shad]]
        lifted = ref_org + (g_sh * np.where(np.sum(g_sh * ref_sd, axis=1) < 0, np.float32(-1), np.float32(1))[:, None]) * MIN_T
        kg = np.lexsort((so[:, 2], so[:, 1], so[:, 0], got_pix))
        kr = np.lexsort((lifted[:, 2], lifted[:, 1], lifted[:, 0], ref_pix))
        assert np.array_equal(got_pix[kg], ref_pix[kr])
        ok, err = _lift_ok(so[kg][:, :3], ref_org[kr], g_sh[kr], ref_sd[kr])
        assert ok, (b, err)
        assert float(np.max(np.abs(sd[kg][:, :3] - ref_sd[kr]))) <= 2e-5 if n_sh else True
        # max_t: where the lifted ray meets the sampled light's plane, less 1e-5
        nf = len(ss.emissive)
        k_light = np.minimum(np.floor(draws[h][shad][:, 0] * np.float32(nf)).astype(np.int64), nf - 1)
        n_l = g_of_face[ss.emissive[k_light]][kr]
        l_dir = ref_sd[kr]
        g_up = g_sh[kr] * np.where(np.sum(g_sh[kr] * l_dir, axis=1) < 0, -1.0, 1.0)[:, None]
        ndl = np.sum(n_l * l_dir, axis=1)
        steep = np.abs(ndl) > 0.05  # edge-on light samples add nothing; their bound is ill-conditioned
        want_max_t = want["shadow_max_t"][shad][kr] - float(MIN_T) * np.sum(n_l * g_up, axis=1) / np.where(steep, ndl, 1.0)
        # the device takes the lift's length along ln from its rounded lifted origin: a few 1e-5 where ln . l is small
        rel_t = np.abs(sd[kg][steep, 3] - want_max_t[steep]) / np.abs(want_max_t[steep])
        assert (float(rel_t.max()) <= 1e-4 and float(np.quantile(rel_t, 0.999)) <= 1e-5) if steep.any() else True
        cd = np.abs(sc_[kg][:, :3] - want["shadow_contrib"][shad][kr]) / np.maximum(np.abs(want["shadow_contrib"][shad][kr]), 1e-6)
        assert (float(cd.max()) <= 1e-3 and float(np.quantile(cd, 0.999)) <= 2e-5) if n_sh else True
        # ---- the frame: emission + the light samples whose shadow ray hits nothing nearer than max_t
        sr = np.zeros(n_sh, S.RAY_DTYPE)
        sr["org"], sr["dir"], sr["min_t"], sr["max_t"] = so[:, :3], sd[:, :3], so[:, 3], sd[:, 3]
        if n_sh:
            shh, shm = ss.sc.Traverse(sr, flags=flags)
            vis = ~((shm == 1) & (shh["t"] < sd[:, 3]))
            np.add.at(expect, got_pix[vis].astype(np.int64), sc_[vis][:, :3].astype(np.float64))
        np.add.at(expect, pix[h][emit], want["emission"][emit].astype(np.float64))
        got = accum.cpu().numpy().reshape(-1, 3).astype(np.float64)
        assert np.max(np.abs(got - expect) / np.maximum(np.abs(expect), 1.0)) <= 1e-4, b
        seen |= {k for k, m in (("shadow", shad), ("emit", emit), ("cont", cont)) if m.any()}
        pid, o4, d4 = got_pid, go.copy(), gd.copy()
    assert checked > 15000 and seen == {"shadow", "emit", "cont"}, (checked, seen)


def test_every_bounce_matches_the_reference_with_facevarying_normals_conformance_walk():
    from nanort_b200 import api

    _bounce_by_bounce(True, api.TRAVERSE_CONFORMANCE)


def test_every_bounce_matches_the_reference_with_flat_normals_conformance_walk():
    from nanort_b200 import api

    _bounce_by_bounce(False, api.TRAVERSE_CONFORMANCE)


def test_every_bounce_matches_the_reference_with_facevarying_normals_production_walk():
    _bounce_by_bounce(True, 0)


def test_every_bounce_matches_the_reference_with_flat_normals_production_walk():
    _bounce_by_bounce(False, 0)


# ------------------------------------------------------------------ the whole pass
@pytest.fixture(scope="module")
def setup():
    return SceneSetup(with_normals=True)


def _within_bound(a, b, m):
    """a frame of non-negative atomicAdd terms, at most m per pixel, summed in two orders"""
    bound = 2.0 * m * U * np.maximum(a, b) * 1.01
    over = np.abs(a - b) > bound
    assert not over.any(), (int(over.any(axis=1).sum()), float(np.abs(a - b)[over].max()))


def test_whole_pass_equals_its_bounces(setup):
    """RenderPath against the same slots driven bounce by bounce from the host (conformance walk: per-ray
    deterministic): identical ray counts, the frame within the atomic-order bound."""
    import torch
    from nanort_b200 import api

    ss = setup
    W, H, spp, bounces, seed = 96, 64, 6, 7, 11
    whole, rw = ss.render(W, H, spp, bounces, seed, flags=api.TRAVERSE_CONFORMANCE)
    assert rw.camera_rays == W * H * spp and rw.shadow_rays > 0
    p, cam = ss.params(W, H, spp, bounces, seed, flags=api.TRAVERSE_CONFORMANCE)
    pix_of_slot, smp_of_slot = M.slots(W, H, TILE[0], TILE[1], spp)
    valid = np.flatnonzero(pix_of_slot >= 0)
    n = len(valid)
    dev = "cuda"
    q = [[torch.zeros((n, 4), dtype=torch.float32, device=dev) for _ in range(2)] + [torch.zeros(n, dtype=torch.int32, device=dev)]
         for _ in range(2)]
    q[0][0][:, :3] = torch.as_tensor(np.asarray(cam[:3], np.float32), device=dev)
    q[0][0][:, 3] = float(MIN_T)
    q[0][1][:, :3] = torch.as_tensor(M.camera_dirs(cam, W, H, seed, pix_of_slot[valid], smp_of_slot[valid]), device=dev)
    q[0][1][:, 3] = 1e30
    q[0][2].copy_(torch.as_tensor(valid.astype(np.int32), device=dev))
    sh = [torch.zeros((n, 4), dtype=torch.float32, device=dev) for _ in range(3)]
    weight = torch.ones((len(pix_of_slot), 4), dtype=torch.float32, device=dev)
    accum = torch.zeros(W * H * 3, dtype=torch.float32, device=dev)
    radiance, shadow, cur, k = 0, 0, 0, n
    for b in range(bounces):
        if k == 0:
            break
        radiance += k
        nc, ns = ss.sc.PathBounce(p, ss.shading, b, k, q[cur][0].data_ptr(), q[cur][1].data_ptr(), q[cur][2].data_ptr(),
                                  weight.data_ptr(), q[cur ^ 1][0].data_ptr(), q[cur ^ 1][1].data_ptr(),
                                  q[cur ^ 1][2].data_ptr(), sh[0].data_ptr(), sh[1].data_ptr(), sh[2].data_ptr(),
                                  accum.data_ptr())
        shadow += ns
        k, cur = nc, cur ^ 1
    assert (radiance, shadow) == (rw.radiance_rays, rw.shadow_rays)
    _within_bound(whole, accum.cpu().numpy().astype(np.float64).reshape(-1, 3), spp * bounces)


def _compare_splits(ss, cfg, splits):
    from nanort_b200 import api

    base = dict(seed=3, flags=api.TRAVERSE_CONFORMANCE)
    whole, rw = ss.render(**dict(base, **cfg))
    assert rw.camera_rays == cfg["W"] * cfg["H"] * cfg["spp"] and float(whole.sum()) > 0
    for label, parts in splits:
        total = np.zeros_like(whole)
        counts = np.zeros(3, np.int64)
        for kw in parts:
            fr, r = ss.render(**dict(base, **dict(cfg, **kw)))
            total += fr
            counts += (r.camera_rays, r.radiance_rays, r.shadow_rays)
        assert tuple(counts) == (rw.camera_rays, rw.radiance_rays, rw.shadow_rays), (label, counts)
        _within_bound(whole, total, cfg["spp"] * cfg["bounces"])
    return rw


def test_splitting_the_frame_does_not_change_it(setup):
    """500 x 300 in 64 x 8 tiles (partial on the right and at the bottom) at 28 spp: 304 tiles of 14336 slots, 292 per
    wave (1 << 22 slots) -> two waves; against shard k of 3, spp 13 + 15 at sample0 13, and 8 x 4 tiles."""
    cfg = dict(W=500, H=300, spp=28, bounces=4, tile=(64, 8))
    rw = _compare_splits(setup, cfg, [
        ("3 shards", [dict(shard=s, n_shards=3) for s in range(3)]),
        ("spp 13 + 15", [dict(spp=13), dict(spp=15, sample0=13)]),
        ("tiles 8x4", [dict(tile=(8, 4))]),
    ])
    assert rw.traverse_launches > 2 * 4  # more than one wave of 4 bounces


def test_a_tile_larger_than_a_wave(setup):
    """128 x 64 in 64 x 64 tiles at 1025 spp: a tile holds 4 198 400 > 1 << 22 slots, one tile per wave, two waves;
    against the two tiles as shards 0 and 1 of 2."""
    cfg = dict(W=128, H=64, spp=1025, bounces=2, tile=(64, 64))
    _compare_splits(setup, cfg, [("2 shards", [dict(shard=0, n_shards=2), dict(shard=1, n_shards=2)])])


def test_a_shard_past_the_last_tile(setup):
    fr, r = setup.render(100, 60, 4, 5, 3, shard=20, n_shards=21)  # 2 x 8 tiles
    assert not fr.any()
    assert (r.camera_rays, r.radiance_rays, r.shadow_rays, r.launches, r.traverse_launches) == (0, 0, 0, 0, 0)


def test_two_streams_give_the_frames_each_gives_alone(setup):
    import torch
    from nanort_b200 import api

    ss = setup
    cfgs = [dict(W=160, H=120, spp=8, bounces=6, seed=1), dict(W=128, H=96, spp=6, bounces=5, seed=2)]
    alone = [ss.render(flags=api.TRAVERSE_CONFORMANCE, **c) for c in cfgs]
    streams = [torch.cuda.Stream() for _ in cfgs]
    accs = [torch.zeros(c["W"] * c["H"] * 3, dtype=torch.float32, device="cuda") for c in cfgs]
    torch.cuda.synchronize()
    import threading

    res = [None, None]

    def run(k):
        p, _ = ss.params(cfgs[k]["W"], cfgs[k]["H"], cfgs[k]["spp"], cfgs[k]["bounces"], cfgs[k]["seed"],
                         flags=api.TRAVERSE_CONFORMANCE)
        res[k] = ss.sc.RenderPath(p, ss.shading, accs[k].data_ptr(), stream=streams[k].cuda_stream)

    th = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    torch.cuda.synchronize()
    for k, c in enumerate(cfgs):
        fr = accs[k].cpu().numpy().astype(np.float64).reshape(-1, 3)
        assert (res[k].radiance_rays, res[k].shadow_rays) == (alone[k][1].radiance_rays, alone[k][1].shadow_rays)
        _within_bound(alone[k][0], fr, c["spp"] * c["bounces"])


# ------------------------------------------------------------------ against the flat pass over the flattened mesh
@pytest.mark.parametrize("with_normals", [False, True])
def test_the_scene_renders_like_its_flattened_mesh(with_normals):
    """Same spp, same random draws: per 16 x 16 block the mean radiance agrees within 4 sigma of the blocks' pixel
    spread, and the total energy within 1 % -- a wrong light area, a flipped normal under the mirroring matrix, or a
    lift that leaks light would show here."""
    import torch

    ss = SceneSetup(with_normals)
    W, H, spp, bounces, seed = 128, 96, 64, 8, 21
    scene, _ = ss.render(W, H, spp, bounces, seed)
    acc, keep = ss.flat_accel()
    p, _ = ss.params(W, H, spp, bounces, seed)
    p.d_material_ids, p.d_emissive_faces = keep[0].data_ptr(), keep[1].data_ptr()
    p.d_facevarying_normals = keep[2].data_ptr() if with_normals else None
    accum = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
    acc.RenderPath(p, accum.data_ptr())
    flat = accum.cpu().numpy().astype(np.float64).reshape(-1, 3)
    a, b = scene.sum(axis=1).reshape(H, W) / spp, flat.sum(axis=1).reshape(H, W) / spp
    assert abs(a.sum() - b.sum()) <= 0.01 * b.sum(), (a.sum(), b.sum())
    worst = 0.0
    for y in range(0, H, 16):
        for x in range(0, W, 16):
            ba, bb = a[y:y + 16, x:x + 16].ravel(), b[y:y + 16, x:x + 16].ravel()
            sigma = np.sqrt((ba.var() + bb.var()) / len(ba)) + 1e-6
            worst = max(worst, abs(ba.mean() - bb.mean()) / sigma)
    assert worst <= 4.0, worst


# ------------------------------------------------------------------ refusals
def test_refusals_launch_nothing(setup):
    import torch
    from nanort_b200 import api

    ss = setup
    L = api.lib()
    W, H = 64, 48
    accum = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
    arr = ss.sc._shading(ss.shading)
    bad_pairs = torch.as_tensor(np.array([0, 0, 3, 12], np.int32), device="cuda")  # instance 3 has 12 faces
    bad_inst = torch.as_tensor(np.array([4, 0], np.int32), device="cuda")

    def variant(**kw):
        p, _ = ss.params(W, H, 2, 3, 1)
        for k, v in kw.items():
            setattr(p, k, v)
        return p

    cases = {
        "material ids in the params": (variant(d_material_ids=ss.keep[0].data_ptr()), arr),
        "normals in the params": (variant(d_facevarying_normals=ss.keep[1].data_ptr()), arr),
        "NULL shading": (variant(), None),
        "any hit": (variant(flags=api.TRAVERSE_ANY_HIT), arr),
        "packed tiles": (variant(flags=api.AO_PACKED_TILES), arr),
        "tile width": (variant(tile_w=12), arr),
        "no bounces": (variant(max_bounces=0), arr),
        "shard": (variant(shard=2, n_shards=2), arr),
        "face out of range": (variant(n_emissive=2, d_emissive_faces=bad_pairs.data_ptr()), arr),
        "instance out of range": (variant(n_emissive=1, d_emissive_faces=bad_inst.data_ptr()), arr),
    }
    res = api.PathResult()
    n = 32
    q = [torch.full((n, 4), 7.0, device="cuda") for _ in range(7)]
    pid = torch.zeros(n, dtype=torch.int32, device="cuda")
    for name, (p, sh) in cases.items():
        rc = L.nrt_scene_render_path_device(ss.sc._h, C.byref(p), C.cast(sh, C.c_void_p) if sh is not None else None,
                                            C.c_void_p(accum.data_ptr()), C.byref(res), None)
        assert rc == -1 and L.nrt_last_error().decode(), name
        nc, ns = C.c_uint64(5), C.c_uint64(5)
        vp = C.c_void_p
        rc = L.nrt_scene_path_bounce_device(ss.sc._h, C.byref(p), C.cast(sh, vp) if sh is not None else None, 0, n,
                                            vp(q[0].data_ptr()), vp(q[1].data_ptr()), vp(pid.data_ptr()),
                                            vp(q[2].data_ptr()), vp(q[3].data_ptr()), vp(q[4].data_ptr()),
                                            vp(pid.data_ptr()), vp(q[5].data_ptr()), vp(q[6].data_ptr()),
                                            vp(q[5].data_ptr()), vp(accum.data_ptr()), C.byref(nc), C.byref(ns), 0, None)
        assert rc == -1 and L.nrt_last_error().decode() and (nc.value, ns.value) == (0, 0), name
    torch.cuda.synchronize()
    assert not accum.any() and all(bool((x == 7.0).all()) for x in q)
