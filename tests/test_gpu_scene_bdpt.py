"""The bidirectional path tracer over two-level scenes (csrc/bdpt.cu: nrt_scene_render_bdpt_device,
nrt_scene_bdpt_export_device).

The scene is test_gpu_scene_path.instanced_cornell(): the walls, a x2-scaled light, and one box mesh shared by a rotated,
non-uniformly scaled instance and a mirrored one, each with its own material, with per-instance face-varying normals.
A second scene adds a smaller, non-uniformly scaled instance of the light, so that the light table's (area, pair) order
is not its pair order.
The trees are reference-built, so the conformance walk is orc.PortScene's.  Flattened on the host (world vertices by
the float32 MultV order, world normals by inverse_transpose33, face = instance offset + prim) it is an ordinary mesh
that the reference (oracle/_ref/libbdpt_ref.so) and the flat pass (nrt_render_bdpt_device) render."""
import numpy as np
import pytest

import bdpt_model as M
import scene_bdpt_model as SM
from bdpt_helpers import FIELDS, _bits, frame_from_samples, slot_map
from test_gpu_scene_path import _local_normals, _multv, _xform, instanced_cornell

pytestmark = pytest.mark.gpu

MB = 10
CONF = 1  # NRT_TRAVERSE_CONFORMANCE
NONE = 0xFFFFFFFF
BDPT_SURFACE = 2
WAVE_BUDGET = 512 << 20


class SceneBdpt:
    def __init__(self, ref_mod, extra_light=False):
        import torch
        from nanort_b200 import api
        from oracle import orc

        self.api, self.torch = api, torch
        insts, mats = instanced_cornell()
        if extra_light:  # the light's mesh again, smaller and stretched, under the ceiling
            lv, lf, _, lids = insts[1]
            insts = insts + [(lv, lf, _xform((1.2, 1.0, 0.7), 30.0, (1.0, 8.5, -2.0)), lids)]
        self.insts = insts
        self.port = orc.PortScene([(v, f, x) for v, f, x, _ in insts], cpp11=True)
        self.mats = np.ascontiguousarray(np.asarray(mats).view(np.float32).reshape(-1, 16))
        self.sc = api.Scene()
        self.accels = {}
        for v, f, x, _ in insts:
            key = (v.ctypes.data, f.ctypes.data)
            if key not in self.accels:
                a = api.BVHAccel()
                assert a.Build(len(f), v, f, flags=api.BUILD_REFERENCE_TREE)
                self.accels[key] = a
            self.sc.AddNode(self.accels[key], x)
        assert self.sc.Commit(api.BUILD_REFERENCE_TREE)
        st = self.sc.InstanceStates()
        self.keep, self.shading, self.offsets = [], [], []
        fv, ff, fids, fn = [], [], [], []
        nv = nf = 0
        for i, (v, f, x, ids) in enumerate(insts):
            ln = _local_normals(v, f)
            d_ids = torch.as_tensor(ids.astype(np.int32), device="cuda")
            d_n = torch.as_tensor(ln.reshape(-1), device="cuda")
            self.keep += [d_ids, d_n]
            self.shading.append(api.SceneShading(d_ids.data_ptr(), d_n.data_ptr()))
            wv = _multv(st["xform"][i], v)
            fv.append(wv)
            ff.append(f.astype(np.uint32) + nv)
            fids.append(ids)
            fn.append(_multv(st["invT33"][i], ln.reshape(-1, 3)).reshape(-1, 9))
            self.offsets.append(nf)
            nv += len(v)
            nf += len(f)
        self.offsets = np.asarray(self.offsets, np.int64)
        self.v, self.f = np.concatenate(fv), np.concatenate(ff)
        self.ids = np.concatenate(fids).astype(np.uint32)
        self.fvn = np.concatenate(fn).astype(np.float32)
        self.tri = self.v[self.f]  # world triangles of the flattened mesh
        self.ref = ref_mod.BdptReference(self.v, self.f, self.ids, self.mats, self.fvn, api.BDPT_VERTEX_DTYPE)
        self.d_mats = torch.from_numpy(self.mats.copy()).to("cuda")
        self.d_ids = torch.from_numpy(self.ids.view(np.int32).copy()).to("cuda")
        self.d_fvn = torch.from_numpy(self.fvn.reshape(-1).copy()).to("cuda")

    def params(self, W, H, spp, sample0=0, spp_total=None, tile=(16, 8), shard=0, n_shards=1, max_bounces=MB,
               flags=CONF, flat=False):
        p = self.api.BdptParams()
        for k in range(12):
            p.cam[k] = float(M.REFERENCE_CAMERA[k])
        p.width, p.height, p.spp, p.sample0 = W, H, spp, sample0
        p.spp_total = spp_total if spp_total is not None else sample0 + spp
        p.tile_w, p.tile_h, p.shard, p.n_shards = tile[0], tile[1], shard, n_shards
        p.max_bounces, p.n_materials = max_bounces, len(self.mats)
        p.d_materials = self.d_mats.data_ptr()
        p.d_material_ids = self.d_ids.data_ptr() if flat else None
        p.d_facevarying_normals = self.d_fvn.data_ptr() if flat else None
        p.flags = flags
        return p

    def render(self, p, stream=None, shading=None, accum=None):
        if accum is None:
            accum = self.torch.zeros(3 * p.width * p.height, dtype=self.torch.float32, device="cuda")
        r = self.sc.RenderBDPT(p, self.shading if shading is None else shading, accum.data_ptr(), stream)
        self.torch.cuda.synchronize()
        return accum.cpu().numpy().reshape(-1, 3), r, accum

    def export(self, p):
        torch = self.torch
        n = self.api.bdpt_slots(p)
        rec = p.max_bounces + 1
        eye = torch.zeros(n * rec * 80, dtype=torch.uint8, device="cuda")
        light = torch.zeros_like(eye)
        ei = torch.full((n * rec,), -1, dtype=torch.int32, device="cuda")
        li = torch.full_like(ei, -1)
        pair = torch.zeros(2 * n, dtype=torch.int32, device="cuda")
        ne = torch.zeros(n, dtype=torch.int32, device="cuda")
        nl = torch.zeros_like(ne)
        rgb = torch.zeros(3 * n, dtype=torch.float32, device="cuda")
        r = self.sc.ExportBDPT(p, self.shading, eye.data_ptr(), light.data_ptr(), ei.data_ptr(), li.data_ptr(),
                               pair.data_ptr(), ne.data_ptr(), nl.data_ptr(), rgb.data_ptr())
        torch.cuda.synchronize()
        dt = self.api.BDPT_VERTEX_DTYPE
        u32 = lambda t: t.cpu().numpy().view(np.uint32)
        return dict(eye=eye.cpu().numpy().view(dt).reshape(n, rec), light=light.cpu().numpy().view(dt).reshape(n, rec),
                    eye_inst=u32(ei).reshape(n, rec), light_inst=u32(li).reshape(n, rec),
                    pair=u32(pair).reshape(n, 2), ne=ne.cpu().numpy().astype(np.int64),
                    nl=nl.cpu().numpy().astype(np.int64), rgb=rgb.cpu().numpy().reshape(n, 3), res=r)

    def flat_faces(self, prim, inst):
        """flattened face ids of (instance, prim) records; NONE stays NONE"""
        prim, inst = np.asarray(prim, np.int64), np.asarray(inst, np.int64)
        out = np.full(prim.shape, NONE, np.int64)
        m = prim != NONE
        out[m] = self.offsets[inst[m]] + prim[m]
        return out


def api_slots(p):
    from nanort_b200 import api

    return api.bdpt_slots(p)


def scene_waves(p, exported):
    """waves of a call: the wave-scratch formula of bdpt.cu (make_layout + the scene walk's records)"""
    return -(-api_slots(p) // wave_slots(p, exported))


def wave_slots(p, exported):
    """slots of a full wave (whole tiles)"""
    B = p.max_bounces
    stride, mc = B + 1, B * (B + 1) // 2
    per_slot = 64 + (0 if exported else 2 * stride * 80 + 8 + 12) + 8 + 4 + 4 + 12 + mc * 24 + 8
    per_slot += (0 if exported else 2 * stride * 4 + 8) + mc * (36 + 32 + 1)
    per_tile = p.tile_w * p.tile_h * p.spp
    tpw = max(1, WAVE_BUDGET // (per_slot * per_tile))
    return min(api_slots(p), tpw * per_tile)


@pytest.fixture(scope="module")
def ref_mod():
    from oracle import bdpt_ref

    if not bdpt_ref.available():
        pytest.skip("oracle/_ref/libbdpt_ref.so is not built")
    return bdpt_ref


@pytest.fixture(scope="module")
def scene(ref_mod):
    return SceneBdpt(ref_mod)


@pytest.fixture(scope="module")
def two_lights(ref_mod):
    return SceneBdpt(ref_mod, extra_light=True)


@pytest.mark.parametrize("which", ["scene", "two_lights"])
def test_whole_samples_against_the_reference(which, request):
    """Samples whose structure (lengths, types, flattened faces, materials) matches the reference's on the flattened
    mesh; for those, the lens vertex and the light-origin vertex (position, normal, beta, pdfPos) are bit-exact: the
    pair light table, the world-area sum and the (area, pair) CDF order are the reference's.  In the two-light scene
    the second light's triangles are smaller, so the CDF's (area, pair) order differs from pair order, and both
    lights are picked."""
    scene = request.getfixturevalue(which)
    p = scene.params(48, 32, 2)
    ex = scene.export(p)
    pix, smp, valid = slot_map(p)
    same = total = 0
    exact_bad = []
    for i in np.nonzero(valid)[0]:
        x, r = int(pix[i] % p.width), int(pix[i] // p.width)
        y = p.height - 1 - r
        seed = M.seed(x, y, p.width, p.spp_total, p.sample0 + int(smp[i]))
        eye, light, _ = scene.ref.sample(x, y, p.width, p.height, seed)
        ne, nl = ex["ne"][i], ex["nl"][i]
        ge, gl = ex["eye"][i, :ne], ex["light"][i, :nl]
        total += 1
        if len(eye) != ne or len(light) != nl:
            continue
        fe = scene.flat_faces(ge["prim_id"], ex["eye_inst"][i, :ne])
        fl = scene.flat_faces(gl["prim_id"], ex["light_inst"][i, :nl])
        if not (np.array_equal(eye["type"], ge["type"]) and np.array_equal(light["type"], gl["type"])
                and np.array_equal(eye["prim_id"].astype(np.int64), fe)
                and np.array_equal(light["prim_id"].astype(np.int64), fl)
                and np.array_equal(eye["material"], ge["material"]) and np.array_equal(light["material"], gl["material"])):
            continue
        same += 1
        for name, a, b, keys in (("lens", eye[:1], ge[:1], ("position", "original_norm", "norm", "beta", "wo",
                                                             "pdf_fwd")),
                                 ("light", light[:1], gl[:1], ("position", "norm", "beta", "pdf_fwd"))):
            for k in keys:
                if len(a) and not np.array_equal(_bits(a[k]), _bits(b[k])):
                    exact_bad.append((int(i), name, k))
    frac = same / total
    print(f"scene bdpt: {same} of {total} samples structurally identical to the reference ({100 * frac:.2f} %)")
    assert not exact_bad, exact_bad[:10]
    assert frac >= 0.99
    picked = ex["pair"][ex["nl"] > 0, 0]
    if which == "two_lights":
        total, area, lit = M.light_total_area(scene.v, scene.f, scene.mats, scene.ids)
        assert not np.array_equal(np.argsort(area, kind="stable"), np.arange(len(area)))
        assert set(picked.tolist()) == {1, 4}


def _lift_origins(scene, ex, path, inst, slots, k):
    """where the ray that found vertex k of each slot started: the lens (camera rays are not lifted), the light origin
    lifted along the sampled pair's normal, or vertex k - 1 lifted along its face's normal; and its direction -wo"""
    recs = ex[path]
    d = -recs["wo"][slots, k].astype(np.float32)
    prev = recs["position"][slots, k - 1].astype(np.float32)
    if k == 1 and path == "eye":
        return prev, d
    if k == 1:
        pair = ex["pair"][slots].astype(np.int64)
        fid = scene.offsets[pair[:, 0]] + pair[:, 1]
    else:
        fid = scene.flat_faces(recs["prim_id"][slots, k - 1], ex[inst][slots, k - 1])
    return SM.lifted(SM.unit_cross(scene.tri[fid]), prev, d), d


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) / np.maximum(np.maximum(np.abs(a), np.abs(b)), 1e-30)


def test_vertex_consistency(scene):
    """For every exported vertex k >= 1:
    - the instance arrays are NONE exactly where prim_id is, and every sampled pair is emissive;
    - it lies on the plane of its (instance, face);
    - the walk from where its ray started (the lens, or vertex k - 1 lifted kEps along its geometric normal) along -wo
      hits that (instance, face) first (-wo is the ray's direction rounded through normalize, so a ray through an edge
      may take the neighbour: at most 0.2 % of them);
    - its shading normal (original_norm) is the instance's face-varying normals moved by inverse_transpose33 and
      interpolated at that walk's (u, v);
    - beta, pdf_fwd and the previous vertex's pdf_rev follow from vertex_f / pdf_brdf within 1e-5 relative, where the
      previous vertex is diffuse (the lobe that was sampled is then known); cosines below 0.05 are skipped, because the
      device's cosine and the restated one differ by an ulp of the direction."""
    p = scene.params(32, 32, 2)
    ex = scene.export(p)
    mats = scene.mats
    stats = dict(vertices=0, walk_miss=0, beta=0, pdf_fwd=0, pdf_rev=0)
    for path, cnt, inst in (("eye", "ne", "eye_inst"), ("light", "nl", "light_inst")):
        n = ex[cnt]
        recs = ex[path]
        for i in np.nonzero(n > 0)[0]:
            assert np.array_equal(recs["prim_id"][i, :n[i]] == NONE, ex[inst][i, :n[i]] == NONE)
            assert recs["prim_id"][i, 0] == NONE
        for k in range(1, int(n.max())):
            slots = np.nonzero(n > k)[0]
            fid = scene.flat_faces(recs["prim_id"][slots, k], ex[inst][slots, k])
            tri = scene.tri[fid].astype(np.float64)
            g = SM.unit_cross(scene.tri[fid]).astype(np.float64)
            pos = recs["position"][slots, k].astype(np.float64)
            dplane = np.abs(np.einsum("ij,ij->i", pos - tri[:, 0], g))
            assert np.all(dplane <= 2e-5 * (np.abs(tri).max(axis=(1, 2)) + 1.0)), (path, k, dplane.max())
            o, d = _lift_origins(scene, ex, path, inst, slots, k)
            hits, mask = SM.walk(scene.port, o, d)
            got = np.where(mask != 0, scene.offsets[np.minimum(hits["node_id"], len(scene.offsets) - 1)] +
                           hits["prim_id"].astype(np.int64), -1)
            same = got == fid
            stats["walk_miss"] += int((~same).sum())
            stats["vertices"] += len(slots)
            wn = SM.hit_normal(scene.fvn[fid[same]], hits["u"][same], hits["v"][same])
            on = recs["original_norm"][slots[same], k]
            assert np.all(np.abs(wn - on) <= 2e-5), (path, k, float(np.abs(wn - on).max()))
            # the previous vertex's BRDF sample
            if k < 2:
                if path == "eye":  # from the lens: pdf 1, beta 1 (unless the hit is a light)
                    to = pos - recs["position"][slots, 0].astype(np.float64)
                    dist = np.linalg.norm(to, axis=1)
                    want = np.einsum("ij,ij->i", to / dist[:, None], recs["norm"][slots, 0]) / (dist * dist)
                    assert np.all(_rel(recs["pdf_fwd"][slots, k], want) <= 1e-5)
                continue
            for j, i in enumerate(slots):
                pv = M._vertex(recs[i, k - 1], mats)
                v = M._vertex(recs[i, k], mats)
                if pv["mat"] is None or M._delta(pv) or pv["type"] != BDPT_SURFACE or v["type"] != BDPT_SURFACE:
                    continue
                out = M._unit(tuple(-float(x) for x in recs["wo"][i, k]))
                c = abs(M._dot(pv["n"], out))
                if c < 0.05:
                    continue
                pdf = M.pdf_brdf(pv["mat"], out, pv["wo"], pv["on"], pv["n"])
                f = M.vertex_f(pv, tuple(pv["p"][q] + out[q] for q in range(3)))
                beta = np.array([pv["beta"][q] * f[q] * c / pdf for q in range(3)])
                assert np.all(_rel(beta, v["beta"]) <= 1e-5), (path, i, k, beta, v["beta"])
                stats["beta"] += 1
                to = M._sub(v["p"], pv["p"])
                dist = M._length(to)
                want = pdf * (M._dot(M._unit(to), pv["n"]) / (dist * dist))
                assert _rel(v["fwd"], want) <= 1e-5, (path, i, k, v["fwd"], want)
                stats["pdf_fwd"] += 1
                # pdf_rev of vertex k - 1: vertex k's pdfBRDF back along its incoming ray, per unit area at k - 1
                if n[i] > k + 1 and v["mat"] is not None:
                    nxt = M._unit(tuple(-float(x) for x in recs["wo"][i, k + 1]))
                    if abs(M._dot(v["n"], nxt)) < 0.05 or abs(M._dot(v["n"], M._unit(to))) < 0.05:
                        continue
                    back = M.pdf_brdf(v["mat"], nxt, v["wo"], v["on"], v["n"])
                    want = back * abs(M._dot(M._unit(to), v["n"])) / (dist * dist)
                    assert _rel(recs["pdf_rev"][i, k - 1], want) <= 1e-5, (path, i, k, recs["pdf_rev"][i, k - 1], want)
                    stats["pdf_rev"] += 1
    live = ex["nl"] > 0
    pairs = ex["pair"][live].astype(np.int64)
    assert np.all(scene.mats[scene.ids[scene.offsets[pairs[:, 0]] + pairs[:, 1]], 9:12].max(axis=1) > 0.001)
    assert np.all(ex["pair"][~live] == NONE)
    print(f"scene bdpt vertex consistency: {stats}")
    assert stats["walk_miss"] <= 0.002 * stats["vertices"]
    assert stats["vertices"] > 1000 and stats["beta"] > 200 and stats["pdf_rev"] > 200


@pytest.mark.parametrize("flags", [CONF, 0])
def test_connections_against_the_scene_rules(scene, flags):
    """Every exported sample's colour is connectPath's sum over its own subpaths with bdpt_model's weight_mis /
    vertex_f and the scene's visibility rule (the lifted connection ray, max_t at the light vertex's plane less 1e-5,
    the walk's nearest hit from orc.PortScene), within 1e-4 of its sum of |term|.  The production walk returns the
    reference's distance for a face and may differ only in which face it names at a tie, which visibility does not
    read, so it is held to the same bound."""
    p = scene.params(32, 24, 2, flags=flags)
    ex = scene.export(p)
    total, _, _ = M.light_total_area(scene.v, scene.f, scene.mats, scene.ids)
    bad, worst, n_terms, blocked = [], 0.0, 0, 0
    for i in np.nonzero(ex["ne"] > 1)[0]:
        terms = SM.connection_terms(ex, i, scene, scene.mats, total, p.max_bounces, scene.port)
        want = sum((t for _, _, t in terms), np.zeros(3))
        mag = sum((np.abs(t) for _, _, t in terms), np.zeros(3))
        n_terms += len(terms)
        blocked += sum(1 for e, l, t in terms if l > 0 and not np.any(t))
        err = np.abs(ex["rgb"][i].astype(np.float64) - want)
        if np.any(err > 1e-4 * mag + 1e-30):
            bad.append((int(i), ex["rgb"][i], want))
        worst = max(worst, float(np.max(err / np.maximum(mag, 1e-30))))
    print(f"scene bdpt connections (flags {flags}): {n_terms} terms, {blocked} zero, worst {worst:.2e} of sum|term|, "
          f"{len(bad)} samples off")
    assert not bad, (len(bad), bad[:5])
    assert n_terms > 1000 and blocked > 0


def test_splits_are_bit_identical(scene):
    """Under the conformance walk: a call across >= 3 waves equals its single-wave shards, a sample0 split, a second call
    and two calls on two streams; the frame is the ordered sum of the exported sample colours."""
    import torch

    B = 64
    p = scene.params(64, 48, 4, max_bounces=B)
    nw = scene_waves(p, exported=False)
    assert nw >= 3, nw
    frame, r, _ = scene.render(p)
    assert np.all(np.isfinite(frame)) and np.count_nonzero(frame) > 0
    again = scene.render(p)[0]
    assert np.array_equal(_bits(again), _bits(frame))
    # the walks each wave of the formula's partition can run, from the subpaths: eye and light walks reach the longest
    # subpath of the wave (one more when its last ray missed), plus at most one connection walk
    ex = scene.export(p)
    cap = wave_slots(p, exported=False)
    lo = hi = 0
    for s0 in range(0, api_slots(p), cap):
        ne, nl = ex["ne"][s0:s0 + cap], ex["nl"][s0:s0 + cap]
        me, ml = int(ne.max()), int(nl.max())
        lo += max(me - 1, 0) + max(ml - 1, 0)
        hi += min(me, B) + min(ml, B) + 1
    assert lo <= r.traverse_launches <= hi, (lo, r.traverse_launches, hi)
    acc = np.zeros_like(frame)
    for sh in range(nw):
        q = scene.params(64, 48, 4, max_bounces=B, shard=sh, n_shards=nw)
        assert scene_waves(q, exported=False) == 1
        acc += scene.render(q)[0]
    assert np.array_equal(_bits(acc), _bits(frame))
    _, _, split = scene.render(scene.params(64, 48, 2, spp_total=4, max_bounces=B))
    halves = scene.render(scene.params(64, 48, 2, sample0=2, spp_total=4, max_bounces=B), accum=split)[0]
    assert np.array_equal(_bits(halves), _bits(frame))
    assert np.array_equal(_bits(frame_from_samples(p, ex).reshape(-1, 3)), _bits(frame))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    out = []
    for s in (s1, s2):
        acc_t = torch.zeros(3 * 64 * 48, dtype=torch.float32, device="cuda")
        scene.sc.RenderBDPT(p, scene.shading, acc_t.data_ptr(), s.cuda_stream)
        out.append(acc_t)
    torch.cuda.synchronize()
    for o in out:
        assert np.array_equal(_bits(o.cpu().numpy().reshape(-1, 3)), _bits(frame))
    print(f"scene bdpt splits: {nw} waves, {r.traverse_launches} walks, {r.connection_rays} connection rays")


def test_against_the_flat_pass(scene):
    """Same seeds, the scene against the flattened mesh through nrt_render_bdpt_device: every 16x16 block mean within
    4 sigma, total energy within 1 %"""
    W = H = 128
    K, spp = 16, 4
    acc = scene.api.BVHAccel()
    assert acc.Build(len(scene.f), scene.v, scene.f, flags=scene.api.BUILD_REFERENCE_TREE)
    torch = scene.torch
    blocks = {"scene": [], "flat": []}
    for k in range(K):
        ps = scene.params(W, H, spp, sample0=spp * k, spp_total=spp * K)
        fs = scene.render(ps)[0]
        pf = scene.params(W, H, spp, sample0=spp * k, spp_total=spp * K, flat=True)
        af = torch.zeros(3 * W * H, dtype=torch.float32, device="cuda")
        acc.RenderBDPT(pf, af.data_ptr())
        torch.cuda.synchronize()
        ff = af.cpu().numpy().reshape(-1, 3)
        for name, fr in (("scene", fs), ("flat", ff)):
            img = fr.astype(np.float64).sum(axis=1).reshape(H // 16, 16, W // 16, 16)
            blocks[name].append(img.mean(axis=(1, 3)) / spp)
    s, f = np.asarray(blocks["scene"]), np.asarray(blocks["flat"])
    ms, mf = s.mean(axis=0), f.mean(axis=0)
    se = np.sqrt(s.var(axis=0, ddof=1) / K + f.var(axis=0, ddof=1) / K)
    z = np.abs(ms - mf) / np.maximum(se, 1e-12)
    e_s, e_f = ms.sum(), mf.sum()
    print(f"scene vs flat bdpt: worst block {z.max():.2f} sigma, energy {e_s:.4f} vs {e_f:.4f} "
          f"({100 * (e_s / e_f - 1):+.3f} %)")
    assert np.all(np.abs(ms - mf) <= 4 * se + 1e-6 * np.abs(mf)), z.max()
    assert abs(e_s / e_f - 1) <= 0.01


@pytest.mark.parametrize("B", [1, 3, 16])
def test_subpaths_are_prefixes_of_max_bounces_64(scene, B):
    """Eye subpaths at B are prefixes of those at 64; so are light subpaths where the eye subpath ended before B + 1
    vertices.  The last vertex's pdf_rev is written by the next bounce, which a cut subpath does not trace."""
    short = scene.export(scene.params(24, 16, 2, max_bounces=B))
    full = scene.export(scene.params(24, 16, 2, max_bounces=64))
    assert np.all(short["ne"] == np.minimum(full["ne"], B + 1))
    same_start = (short["ne"] > 1) & (short["ne"] < B + 1)
    assert np.all(short["nl"][same_start] == np.minimum(full["nl"][same_start], B + 1))
    fields = FIELDS + ("type", "prim_id", "material")
    for k, cnt, ik, rows in (("eye", "ne", "eye_inst", np.nonzero(short["ne"] > 0)[0]),
                             ("light", "nl", "light_inst", np.nonzero(same_start)[0])):
        for i in rows:
            n = short[cnt][i]
            a, c = short[k][i, :n], full[k][i, :n]
            assert np.array_equal(short[ik][i, :n], full[ik][i, :n])
            for key in fields:
                x, y = a[key], c[key]
                if key == "pdf_rev":
                    x, y = x[:-1], y[:-1]
                assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32)), (k, i, key)


def test_refusals_launch_nothing(scene):
    import torch
    from nanort_b200 import api

    p = scene.params(16, 8, 1)
    accum = torch.full((3 * 16 * 8,), 7.0, dtype=torch.float32, device="cuda")

    def refused(q, shading=None):
        with pytest.raises(Exception):
            scene.sc.RenderBDPT(q, scene.shading if shading is None else shading, accum.data_ptr())
        torch.cuda.synchronize()
        assert torch.all(accum == 7.0)

    refused(scene.params(16, 8, 1, flat=True))  # ids / normals in the params
    q = scene.params(16, 8, 1)
    q.flags = api.TRAVERSE_ANY_HIT
    refused(q)
    q = scene.params(16, 8, 1)
    q.max_bounces = 65
    refused(q)
    q = scene.params(16, 8, 1)
    q.tile_w = 12
    refused(q)
    missing = list(scene.shading)
    missing[2] = api.SceneShading(scene.shading[2].d_material_ids, None)
    refused(p, missing)
    missing = list(scene.shading)
    missing[1] = api.SceneShading(None, scene.shading[1].d_facevarying_normals)
    refused(p, missing)
    bad_ids = torch.full((12,), len(scene.mats), dtype=torch.int32, device="cuda")
    bad = list(scene.shading)
    bad[3] = api.SceneShading(bad_ids.data_ptr(), scene.shading[3].d_facevarying_normals)
    refused(p, bad)
    dark_ids = [torch.zeros(12 if i >= 2 else (10 if i == 0 else 2), dtype=torch.int32, device="cuda")
                for i in range(4)]
    dark = [api.SceneShading(d.data_ptr(), s.d_facevarying_normals) for d, s in zip(dark_ids, scene.shading)]
    refused(p, dark)
    assert api.lib().nrt_scene_render_bdpt_device(scene.sc._h, p, None, accum.data_ptr(), None, None) != 0
    torch.cuda.synchronize()
    assert torch.all(accum == 7.0)
    # an instance that is not a triangle accel
    spheres = api.BVHAccel()
    assert spheres.BuildSpheres(np.float32([[0.0, 2.0, 0.0]]), np.float32([1.0]))
    mixed = api.Scene()
    mixed.AddNode(scene.accels[next(iter(scene.accels))], np.eye(4, dtype=np.float32))
    mixed.AddNode(spheres, np.eye(4, dtype=np.float32))
    assert mixed.Commit()
    with pytest.raises(Exception):
        mixed.RenderBDPT(p, [scene.shading[0], scene.shading[0]], accum.data_ptr())
    torch.cuda.synchronize()
    assert torch.all(accum == 7.0)
