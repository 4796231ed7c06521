"""Shared pieces of the bidirectional path tracer's tests (test_gpu_bdpt.py, test_gpu_bdpt_slots.py, test_bdpt_model.py):
the device/reference set-up of a mesh, the slot map of a call, the frame as the device sums it, the whole-sample
comparison against the reference, the reference's closest hit as the model's visibility, and the many-light panel
scene."""
import numpy as np

import bdpt_model as M

MB = 10  # the reference's uMaxBounces
LIGHT, LENS, SURFACE = 0, 1, 2  # NRT_BDPT_LIGHT / LENS / SURFACE


class Setup:
    """A mesh with materials on the device and in the reference, with a reference-tree accel and a production one."""

    def __init__(self, ref_mod, v, f, mats, ids):
        import torch

        from nanort_b200 import api

        self.api = api
        self.v, self.f = np.ascontiguousarray(v, np.float32), np.ascontiguousarray(f, np.uint32)
        self.mats = np.ascontiguousarray(np.asarray(mats).view(np.float32).reshape(-1, 16))
        self.ids = np.ascontiguousarray(ids, np.uint32)
        self.fvn = M.flat_normals(self.v, self.f)
        self.ref = ref_mod.BdptReference(self.v, self.f, self.ids, self.mats, self.fvn, api.BDPT_VERTEX_DTYPE)
        dev = "cuda:0"
        self.d_mats = torch.from_numpy(self.mats.copy()).to(dev)
        self.d_ids = torch.from_numpy(self.ids.view(np.int32).copy()).to(dev)
        self.d_fvn = torch.from_numpy(self.fvn.copy()).to(dev)
        self.conf = api.BVHAccel(device=0)
        assert self.conf.Build(len(self.f), self.v, self.f, flags=api.BUILD_REFERENCE_TREE)
        self.fast = api.BVHAccel(device=0)
        assert self.fast.Build(len(self.f), self.v, self.f)

    def params(self, W, H, spp, sample0=0, spp_total=None, tile=(16, 8), shard=0, n_shards=1, max_bounces=MB,
               flags=1, cam=M.REFERENCE_CAMERA):
        p = self.api.BdptParams()
        for k in range(12):
            p.cam[k] = float(cam[k])
        p.width, p.height, p.spp, p.sample0 = W, H, spp, sample0
        p.spp_total = spp_total if spp_total is not None else sample0 + spp
        p.tile_w, p.tile_h, p.shard, p.n_shards = tile[0], tile[1], shard, n_shards
        p.max_bounces, p.n_materials = max_bounces, len(self.mats)
        p.d_materials, p.d_material_ids, p.d_facevarying_normals = (self.d_mats.data_ptr(), self.d_ids.data_ptr(),
                                                                    self.d_fvn.data_ptr())
        p.flags = flags
        return p

    def export(self, p, accel=None, stream=None):
        import torch

        accel = accel or (self.conf if p.flags else self.fast)
        n = self.api.bdpt_slots(p)
        rec = p.max_bounces + 1
        eye = torch.zeros(n * rec * 80, dtype=torch.uint8, device="cuda:0")
        light = torch.zeros_like(eye)
        ne = torch.zeros(n, dtype=torch.int32, device="cuda:0")
        nl = torch.zeros_like(ne)
        rgb = torch.zeros(3 * n, dtype=torch.float32, device="cuda:0")
        r = accel.ExportBDPT(p, eye.data_ptr(), light.data_ptr(), ne.data_ptr(), nl.data_ptr(), rgb.data_ptr(), stream)
        torch.cuda.synchronize()
        dt = self.api.BDPT_VERTEX_DTYPE
        return dict(eye=eye.cpu().numpy().view(dt).reshape(n, rec), light=light.cpu().numpy().view(dt).reshape(n, rec),
                    ne=ne.cpu().numpy().astype(np.int64), nl=nl.cpu().numpy().astype(np.int64),
                    rgb=rgb.cpu().numpy().reshape(n, 3), res=r)

    def render(self, p, accum=None, accel=None, stream=None):
        import torch

        accel = accel or (self.conf if p.flags else self.fast)
        if accum is None:
            accum = torch.zeros(3 * p.width * p.height, dtype=torch.float32, device="cuda:0")
        r = accel.RenderBDPT(p, accum.data_ptr(), stream)
        return accum, r


def slot_map(p):
    """(pix, smp, valid) of every slot of a call: the path pass's tile map"""
    from nanort_b200 import api

    n = api.bdpt_slots(p)
    tp = p.tile_w * p.tile_h
    s = np.arange(n, dtype=np.int64)
    k, rem = s // (tp * p.spp), s % (tp * p.spp)
    smp, q = rem // tp, rem % tp
    bw = p.tile_w // 8
    blk, inn = q // 32, q % 32
    lx, ly = (blk % bw) * 8 + (inn & 7), (blk // bw) * 4 + (inn >> 3)
    tiles_x = -(-p.width // p.tile_w)
    tile = k * p.n_shards + p.shard
    x, y = (tile % tiles_x) * p.tile_w + lx, (tile // tiles_x) * p.tile_h + ly
    valid = (x < p.width) & (y < p.height)
    return y * p.width + x, smp, valid


def frame_from_samples(p, ex, frame=None):
    """d_accum as the device adds it: per pixel, the sample colours in ascending sample order"""
    pix, smp, valid = slot_map(p)
    frame = np.zeros((p.width * p.height, 3), np.float32) if frame is None else frame
    for s in range(p.spp):
        m = valid & (smp == s) & (ex["ne"] > 1)
        frame[pix[m]] += ex["rgb"][m]
    return frame


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


FIELDS = ("position", "original_norm", "norm", "beta", "wo", "pdf_fwd", "pdf_rev")
# Fields that depend on no cosf / sinf of the sample (directionCosTheta), so must be the reference's bit for bit:
# the lens vertex, the first eye hit (its ray is the camera ray) and the light-origin vertex (LightSampler::sample).
# pdf_rev is left out of all three: the next bounce writes it from a BRDF sample.
EXACT = (("eye", 0, ("position", "original_norm", "norm", "beta", "wo", "pdf_fwd")),
         ("eye", 1, ("position", "original_norm", "norm", "beta", "wo", "pdf_fwd")),
         ("light", 0, ("position", "norm", "beta", "pdf_fwd")))


def _close(a, b, rel):
    """|a - b| <= rel * the larger magnitude, per scalar or, for rows of vectors (position, normal, colour), per row:
    a coordinate near 0 is held to the precision of its vector"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = np.maximum(np.abs(a), np.abs(b))
    if a.ndim > 1:
        scale = scale.max(axis=-1, keepdims=True)
    return bool(np.all(np.abs(a - b) <= rel * scale))


def _exact_mismatches(ref_paths, dev_paths):
    """[(path, vertex, field)] of the EXACT fields that differ in their bits"""
    bad = []
    for name, k, keys in EXACT:
        a, b = ref_paths[name], dev_paths[name]
        if len(a) <= k:
            continue
        for key in keys:
            if not np.array_equal(_bits(a[k][key]), _bits(b[k][key])):
                bad.append((name, k, key))
    return bad


def _compare_samples(setup, p, ex, slots):
    """(structure matches, value mismatches) of the device's samples against bdpt_ref_sample.  Where the structure
    matches, every vertex agrees to 1e-4 and the colour to 1e-3, and the EXACT fields bit for bit."""
    pix, smp, valid = slot_map(p)
    same, diverged, value_bad = 0, [], []
    for i in slots:
        if not valid[i]:
            continue
        x, r = int(pix[i] % p.width), int(pix[i] // p.width)
        y = p.height - 1 - r
        seed = M.seed(x, y, p.width, p.spp_total, p.sample0 + int(smp[i]))
        eye, light, rgb = setup.ref.sample(x, y, p.width, p.height, seed)
        ge, gl = ex["eye"][i, :ex["ne"][i]], ex["light"][i, :ex["nl"][i]]
        structure = len(eye) == len(ge) and len(light) == len(gl) and all(
            np.array_equal(a[k], b[k]) for a, b in ((eye, ge), (light, gl)) for k in ("type", "prim_id", "material"))
        if not structure:
            diverged.append(int(i))
            continue
        same += 1
        ok = all(_close(a[k], b[k], 1e-4) for a, b in ((eye, ge), (light, gl)) for k in FIELDS)
        ok = ok and _close(rgb[None], ex["rgb"][i][None], 1e-3)
        ok = ok and not _exact_mismatches(dict(eye=eye, light=light), dict(eye=ge, light=gl))
        if not ok:
            value_bad.append(int(i))
    return same, diverged, value_bad


def reference_trace(v, f):
    """The model's visibility: the reference's closest hit (oracle/_ref/libnanort_ref.so) over (v, f), as
    trace(org, dir) -> (hit, t) for float32 [n, 3] rays on [kEps, kInf)"""
    from oracle import orc

    acc = orc.Reference(True).build(v, f)

    def trace(org, d):
        rays = np.zeros(len(org), orc.RAY_DTYPE)
        rays["org"], rays["dir"] = org, d
        rays["min_t"], rays["max_t"] = M.K_EPS, M.K_INF
        hits, mask = acc.traverse(rays)
        return mask.astype(bool), hits["t"].copy()

    trace.accel = acc  # keeps the tree alive with the closure
    return trace


# ---------------------------------------------------------------- the many-light panel scene
# The Cornell box with its ceiling light replaced by a tilted panel of PANEL_N x PANEL_N cells of side 1/16 in the plane
# y = 9.25 - x/4 - z/8 (every vertex a dyadic rational, exact in float32; no cross product has a zero component).  Each
# cell is two triangles with separate vertices, both facing down; cells alternate emissive and not (a checkerboard), so
# the light table's compaction skips every other pair of faces.  Translated triangles have the same area bits, so
# the sorted table holds long tie groups across its 1024-key sort tiles; some emissive triangles have a corner pulled
# in by k/256 (distinct, smaller areas).  Three more emitters: a back-wall triangle whose max(Le) is exactly 0.001f
# (not a light: LightSampler keeps max(Le) > kEps, yet a hit ends an eye subpath, isLight), a panel triangle at the
# next float above 0.001f (a light) and one emitting in the blue channel only.
PANEL_N = 52
PANEL_H = 1.0 / 16.0
PANEL_X0 = -PANEL_N * PANEL_H / 2
THRESHOLD_FACE = 4  # the first back-wall triangle of scenes.cornell()


def _panel_y(x, z):
    return 9.25 - x / 4.0 - z / 8.0


def many_lights_scene():
    """(verts, faces, materials, ids, info): info has the panel's face base, the special faces and the cell of every
    panel face"""
    from nanort_b200 import scenes as S

    v, f = S.cornell()
    nv = len(v)
    mats = np.concatenate([
        S.material(diffuse=(0.8, 0.8, 0.8)),                                    # 0 grey
        S.material(diffuse=(0.8, 0.05, 0.05)),                                  # 1 red
        S.material(diffuse=(0.023, 0.41, 0.048)),                               # 2 green
        S.material(specular=(1.0, 1.0, 1.0)),                                   # 3 mirror
        S.material(specular=(0.9, 0.9, 1.0), transmittance=(0.9, 0.9, 1.0), ior=1.5, dissolve=1.0),  # 4 glass
        S.material(diffuse=(0.5, 0.5, 0.5), emission=(15.0, 14.0, 13.0)),      # 5 panel light
        S.material(diffuse=(1.0, 0.8, 0.8), specular=(0.2, 0.2, 0.2)),          # 6 floor
        S.material(diffuse=(0.6, 0.6, 0.6)),                                    # 7 dark panel cell
        S.material(diffuse=(0.8, 0.8, 0.8), emission=(0.001, 0.0005, 0.001)),   # 8 max(Le) == kEps: no light
        S.material(diffuse=(0.6, 0.6, 0.6),
                   emission=(float(np.nextafter(np.float32(0.001), np.float32(1))), 0.0, 0.0)),  # 9 just a light
        S.material(diffuse=(0.6, 0.6, 0.6), emission=(0.0, 0.0, 20.0)),        # 10 blue only
    ])
    ids = np.zeros(len(f), np.uint32)
    ids[0:2] = 6
    ids[2:6] = 0
    ids[THRESHOLD_FACE] = 8
    ids[6:8] = 1
    ids[8:10] = 2
    ids[10:22] = 3
    ids[22:34] = 4
    base = len(f)
    pv, pf, pids, cells = [], [], [], []
    h = PANEL_H
    jitter_k = 0
    for i in range(PANEL_N):
        for j in range(PANEL_N):
            x0, z0 = PANEL_X0 + i * h, PANEL_X0 + j * h
            lit = (i + j) % 2 == 0
            corner = x0 + h
            if lit and (i * PANEL_N + j) % 37 == 0:  # pull the lower triangle's right-angle corner in
                jitter_k = jitter_k % 8 + 1
                corner = x0 + h - jitter_k / 256.0
            lower = [(x0, z0), (x0 + h, z0 + h), (corner, z0)]
            upper = [(x0, z0), (x0, z0 + h), (x0 + h, z0 + h)]
            for half, tri in ((0, lower), (1, upper)):
                n0 = len(pv)
                pv += [(x, _panel_y(x, z), z) for x, z in tri]
                pf.append((n0, n0 + 1, n0 + 2))
                pids.append(5 if lit else 7)
                cells.append((i, j, half))
    pids = np.asarray(pids, np.uint32)
    cells = np.asarray(cells, np.int64)
    # the two single emitters on dark cells: (1, 2) lower and (2, 1) upper
    just = int(np.nonzero((cells[:, 0] == 1) & (cells[:, 1] == 2) & (cells[:, 2] == 0))[0][0])
    blue = int(np.nonzero((cells[:, 0] == 2) & (cells[:, 1] == 1) & (cells[:, 2] == 1))[0][0])
    pids[just], pids[blue] = 9, 10
    pv = np.asarray(pv, np.float64)
    assert np.array_equal(pv.astype(np.float32).astype(np.float64), pv)  # dyadic: exact in float32
    v = np.concatenate([v, pv.astype(np.float32)]).astype(np.float32)
    f = np.concatenate([f, np.asarray(pf, np.uint32) + nv]).astype(np.uint32)
    ids = np.concatenate([ids, pids])
    info = dict(base=base, just=base + just, blue=base + blue, threshold=THRESHOLD_FACE, cells=cells)
    return v, f, mats, ids, info


def panel_faces_of(points, info):
    """The panel face holding each light-origin position (float [n, 3]), from its cell and the cell's diagonal; -1 for
    a point outside the panel"""
    p = np.asarray(points, np.float64)
    i = np.floor((p[:, 0] - PANEL_X0) / PANEL_H).astype(np.int64)
    j = np.floor((p[:, 2] - PANEL_X0) / PANEL_H).astype(np.int64)
    fx = p[:, 0] - (PANEL_X0 + i * PANEL_H)
    fz = p[:, 2] - (PANEL_X0 + j * PANEL_H)
    half = (fz > fx).astype(np.int64)  # the lower triangle lies under the diagonal z - z0 = x - x0
    inside = (i >= 0) & (i < PANEL_N) & (j >= 0) & (j < PANEL_N)
    inside &= np.abs(p[:, 1] - _panel_y(p[:, 0], p[:, 2])) < 1e-4
    face = info["base"] + (np.clip(i, 0, PANEL_N - 1) * PANEL_N + np.clip(j, 0, PANEL_N - 1)) * 2 + half
    return np.where(inside, face, -1)
