"""Host model of the texel cast and the AO bake (csrc/wavefront.cuh: TexelRays, TexelStore, BakeAoRays), restated from
those loaders -- which restate the reference uv_raster's texel ray (examples/uv_raster/main.cc:752-770), its flips
(:779-782) and Lerp (:58-60), and the AO pass's orthonormal basis + cosine direction (ao_direction).

As in tests/ao_model.py, every operation is an IEEE-rounded float32 operation in the device's order (the library is built
with --fmad=false), except sincosf, which the f32 model replaces by the correctly rounded sin / cos of the float32 angle.
The basis and cosine direction are ao_model's own code: cosine_dirs flips the normal towards a viewer, and a viewer
direction of -n leaves the bake's normal as it is."""
import numpy as np

import ao_model as M

F32 = np.float32


def texel_rays(W, H, uv_region, texel_offset):
    """TexelRays::load, the reference uv_raster's texel ray (examples/uv_raster/main.cc:752-770), ray i = texel
    (i % W, i // W): RAY_DTYPE [W * H]."""
    from nanort_b200 import scenes as S

    r = np.asarray(uv_region, F32)
    off = np.asarray(texel_offset, F32)
    i = np.arange(W * H, dtype=np.int64)
    x, y = (i % W).astype(F32), (i // W).astype(F32)
    out = np.zeros(W * H, S.RAY_DTYPE)
    out["org"][:, 0] = r[0] + (x * (r[1] - r[0]) + off[0]) / F32(W)
    out["org"][:, 1] = r[2] + (y * (r[3] - r[2]) + off[1]) / F32(H)
    out["org"][:, 2] = 1.0
    out["dir"][:, 2] = -1.0
    out["min_t"] = 0.0
    out["max_t"] = F32(1e30)
    return out


def texel_dest(W, H, flip_x, flip_y):
    """Texel that ray i's record goes to (main.cc:779-782)."""
    i = np.arange(W * H, dtype=np.int64)
    x, y = i % W, i // W
    px = W - 1 - x if flip_x else x
    py = H - 1 - y if flip_y else y
    return py * W + px


def lerp3(a, b, c, u, v):
    """uv_raster's Lerp (main.cc:58-60) in float32: (1 - u - v) a + u b + v c, per component, left to right."""
    w = (F32(1.0) - u - v)[:, None]
    return w * a + u[:, None] * b + v[:, None] * c


def bake_slots(records, spp, sample0=0):
    """(texel, sample) of every slot of a bake call: covered texels ascending, slot i = sample sample0 + i // n_cov of
    covered texel i % n_cov."""
    texels = np.flatnonzero(records["prim_id"] != 0xFFFFFFFF)
    i = np.arange(len(texels) * spp, dtype=np.int64)
    return texels[i % len(texels)], (sample0 + i // len(texels)).astype(np.uint64)


def bake_normals(verts, faces, records, texel, fv_normals=None):
    """The bake's normal of each texel: the wound unit geometric normal, flipped to the side of the interpolated
    face-varying normal when those are given.  (nx, ny, nz) float32."""
    rec = records[texel]
    f = faces[rec["prim_id"]]
    nx, ny, nz = M.unit_normals(verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]])
    if fv_normals is not None:
        fn = np.asarray(fv_normals, F32).reshape(-1, 3, 3)[rec["prim_id"]]
        s = lerp3(fn[:, 0], fn[:, 1], fn[:, 2], rec["u"], rec["v"])
        flip = nx * s[:, 0] + ny * s[:, 1] + nz * s[:, 2] < 0
        nx, ny, nz = np.where(flip, -nx, nx), np.where(flip, -ny, ny), np.where(flip, -nz, nz)
    return nx, ny, nz


def _dirs(nx, ny, nz, u1, u2, sn=None, cs=None):
    """ao_direction about the normal as given: ao_model.cosine_dirs seen from the viewer direction -n (never flipped)."""
    return M.cosine_dirs(nx, ny, nz, -np.stack([nx, ny, nz], axis=1), u1, u2, sn=sn, cs=cs)[0]


def bake_rays(verts, faces, records, spp, seed, ao_min_t, ao_max_t, sample0=0, fv_normals=None):
    """BakeAoRays::load for every slot (f32 model): (rays RAY_DTYPE, texel, sample)."""
    from nanort_b200 import scenes as S

    texel, smp = bake_slots(records, spp, sample0)
    rec = records[texel]
    f = faces[rec["prim_id"]]
    P = lerp3(verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]], rec["u"], rec["v"])
    nx, ny, nz = bake_normals(verts, faces, records, texel, fv_normals)
    u1, u2 = M.ao_samples(texel, smp, seed)
    out = np.zeros(len(texel), S.RAY_DTYPE)
    out["org"] = P
    out["dir"] = _dirs(nx, ny, nz, u1, u2)
    out["min_t"] = ao_min_t
    out["max_t"] = ao_max_t
    return out, texel, smp


def bake_dirs_within_sincos_ulps(verts, faces, records, texel, smp, seed, got, fv_normals=None, k=3):
    """ao_model.dirs_within_sincos_ulps for bake rays: True where `got` equals, bit for bit, the f32 model evaluated
    with sin / cos moved by at most k ulp from the correctly rounded values."""
    nx, ny, nz = bake_normals(verts, faces, records, texel, fv_normals)
    u1, u2 = M.ao_samples(texel, smp, seed)
    sn0, cs0 = M.sincos(M.TWO_PI_F * u2)
    ok = np.zeros(len(u2), bool)
    gb = np.ascontiguousarray(got, F32).view(np.uint32)
    for i in range(-k, k + 1):
        sn = M._nudge(sn0, i)
        for j in range(-k, k + 1):
            ok |= np.all(_dirs(nx, ny, nz, u1, u2, sn=sn, cs=M._nudge(cs0, j)).view(np.uint32) == gb, axis=1)
    return ok
