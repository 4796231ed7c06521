"""Float64 restatement of the lightmap bake's texel vertex (csrc/wavefront.cuh: lightmap_texel_vertex, the path tracer's
diffuse branch of main.cc:930-960 at bounce 0 with albedo 1 and the texel's one-sided light rule).

Geometry, light samples, cosines and directions are evaluated in float64 from the float32 inputs.  Two decisions are
taken as the device takes them, in float32, because a float64 value on the other side of the threshold would not be a
different answer but a different question: the light face picked by floor(xi1 * n_emissive) and the sign of the
normal's z, which chooses the branch of the orthonormal basis.  Everything else the tests compare with a tolerance."""
import numpy as np

import bake_model as B

F32 = np.float32
INV_PI = 1.0 / 3.14159265358979


def unit_normals64(verts, faces, prim):
    """normalize(cross(v1 - v0, v2 - v0)) of the faces `prim`, and their areas, in float64."""
    tri = np.asarray(faces, np.int64)[prim]
    p0, p1, p2 = (np.asarray(verts, np.float64)[tri[:, k]] for k in range(3))
    c = np.cross(p1 - p0, p2 - p0)
    l = np.linalg.norm(c, axis=1)
    return c / np.where(l > 0, l, 1.0)[:, None], 0.5 * l


def texel_vertex(verts, faces, records, spp, seed, emissive, mats, ids, max_bounces, sample0=0, n_paths=None,
                 fv_normals=None):
    """The texel vertex of paths 0 .. n_paths - 1 of a call (slot map of bake_model.bake_slots).  Returns a dict of
    per-path arrays: texel, sample, P (float64 position), n (float64 unit normal), n32 (the device's float32 normal),
    shadow (bool), shadow_dir, shadow_max_t, contrib (rgb), contrib_scale (the contribution with both cosines 1: the
    scale on which the cosines' float32 rounding, absolute, shows), cos_s (dot(l, n)), cont (bool), cont_dir."""
    from nanort_b200 import scenes as S

    texel, smp = B.bake_slots(records, spp, sample0)
    if n_paths is not None:
        texel, smp = texel[:n_paths], smp[:n_paths]
    rec = records[texel]
    prim = rec["prim_id"].astype(np.int64)
    tri = np.asarray(faces, np.int64)[prim]
    v64 = np.asarray(verts, np.float64)
    u, w = rec["u"].astype(np.float64)[:, None], rec["v"].astype(np.float64)[:, None]
    P = (1 - u - w) * v64[tri[:, 0]] + u * v64[tri[:, 1]] + w * v64[tri[:, 2]]
    n, _ = unit_normals64(verts, faces, prim)
    n32 = np.stack(B.bake_normals(verts, faces, records, texel, fv_normals), axis=1)
    if fv_normals is not None:
        fn = np.asarray(fv_normals, np.float64).reshape(-1, 3, 3)[prim]
        s = (1 - u - w) * fn[:, 0] + u * fn[:, 1] + w * fn[:, 2]
        n = np.where(((n * s).sum(axis=1) < 0)[:, None], -n, n)
    m = len(texel)
    out = {"texel": texel, "sample": smp, "P": P, "n": n, "n32": n32, "shadow": np.zeros(m, bool),
           "shadow_dir": np.zeros((m, 3)), "shadow_max_t": np.zeros(m), "contrib": np.zeros((m, 3)),
           "contrib_scale": np.zeros(m), "cos_s": np.zeros(m), "cont": np.zeros(m, bool), "cont_dir": np.zeros((m, 3))}
    # ---- next-event estimation: MeshLight::sampleDirect from dimensions 8 and 9 (main.cc:337-392)
    ne = len(emissive)
    if ne > 0:
        xi1 = S.rand_ps(texel, smp, 8, seed)
        xi2 = S.rand_ps(texel, smp, 9, seed).astype(np.float64)
        nf = F32(ne)
        k = np.minimum(np.floor(xi1 * nf).astype(np.int64), ne - 1)  # float32, as the device picks
        xi = (xi1 * nf - k.astype(F32)).astype(np.float64)
        fid = np.asarray(emissive, np.int64)[k]
        ltri = np.asarray(faces, np.int64)[fid]
        s1 = np.sqrt(xi)
        c0, c1, c2 = 1 - s1, s1 * (1 - xi2), s1 * xi2
        Q = c0[:, None] * v64[ltri[:, 0]] + c1[:, None] * v64[ltri[:, 1]] + c2[:, None] * v64[ltri[:, 2]]
        l = Q - P
        dist = np.linalg.norm(l, axis=1)
        ok = dist > 1e-6
        l = l / np.where(ok, dist, 1.0)[:, None]
        ln, area = unit_normals64(verts, faces, fid)
        cos_l = np.maximum(-(l * ln).sum(axis=1), 0.0)
        cos_s = (l * n).sum(axis=1)
        sample = ok & (cos_s > 0)
        le = np.asarray(mats["emission"], np.float64)[np.asarray(ids, np.int64)[fid]]
        with np.errstate(divide="ignore", invalid="ignore"):
            # brdf * cosine EDF * cos_s / pdf (main.cc:943-950): the emitted radiance is Le * cos_l, and the area
            # pdf's change to solid angle brings cos_l again; cos_s is left out here
            g = INV_PI * cos_l * cos_l * (ne * area) / (dist * dist)
        out["shadow"] = sample
        out["shadow_dir"] = l
        out["shadow_max_t"] = dist - 1e-5
        out["cos_s"] = cos_s
        out["contrib"] = np.where(sample[:, None], (g * cos_s)[:, None] * le, 0.0)
        with np.errstate(divide="ignore", invalid="ignore"):
            out["contrib_scale"] = np.where(sample, INV_PI * (ne * area) / (dist * dist) * le.max(axis=1), 0.0)
    # ---- continuation: cosine direction about n from dimensions 10 and 11, path_shade_hit's basis (main.cc:216-250)
    if max_bounces > 1:
        u1 = S.rand_ps(texel, smp, 10, seed).astype(np.float64)
        u2 = S.rand_ps(texel, smp, 11, seed).astype(np.float64)
        nx, ny, nz = n[:, 0], n[:, 1], n[:, 2]
        sg = np.where(n32[:, 2] >= 0, 1.0, -1.0)  # the basis branch, from the device's float32 normal
        a = -1.0 / (sg + nz)
        b = nx * ny * a
        t1 = np.stack([1.0 + sg * nx * nx * a, sg * b, -sg * nx], axis=1)
        t2 = np.stack([b, sg + ny * ny * a, -ny], axis=1)
        r = np.sqrt(u1)
        ph = 2.0 * np.pi * u2
        hx, hy, hz = r * np.cos(ph), r * np.sin(ph), np.sqrt(np.maximum(0.0, 1.0 - u1))
        out["cont"] = np.ones(m, bool)
        out["cont_dir"] = t1 * hx[:, None] + t2 * hy[:, None] + n * hz[:, None]
    return out
