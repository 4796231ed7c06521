"""Times the scene bakes (nrt_scene_bake_lightmap_device, nrt_scene_bake_ao_device) against the flat bakes of the
flattened mesh with mapped records (nrt_bake_lightmap_device, nrt_bake_ao_device).

Scene: the 1,002,528-triangle terrain under its area light, the terrain's faces cut into 16 identity instances plus the
light (tools/scene_bdpt_probe.py's scene).  Each terrain instance gets a 4 x 4 grid cell of the atlas as its chart, with
planar UVs of its own faces; the light has no chart.  The flat bakes take the same texels: the scene records with
prim = offset[instance] + prim.  Atlases 2048^2 and 4096^2, 16 spp, lightmaps at max_bounces 1 and 5, AO with
ao_max_t 2.  The passes alternate; best of `reps` calls after one warm-up call each.  Reported: total_ms,
traverse_ms (the scene lightmap times its walks as part of the call: 0), paths/s (rays/s for AO) over the whole call,
rays/s over the traversal launches, with the card's name and power limit read in the same run.

    python tools/scene_bake_probe.py [reps]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch

from nanort_b200 import api
from scene_bdpt_probe import card, terrain_instances


def uv_mesh(v, f):
    """planar (x, z) UVs of these faces, normalised to [0.01, 0.99]^2, in SetupVerticesForUVRaster's layout"""
    t = v[f.astype(np.int64)][:, :, [0, 2]].astype(np.float64)
    lo, hi = t.reshape(-1, 2).min(axis=0), t.reshape(-1, 2).max(axis=0)
    uv = 0.01 + 0.98 * (t - lo) / np.maximum(hi - lo, 1e-30)
    out = np.zeros((3 * len(f), 3), np.float32)
    out[:, :2] = uv.reshape(-1, 2)
    return out, np.arange(3 * len(f), dtype=np.uint32).reshape(-1, 3)


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    if not torch.cuda.is_available():
        raise SystemExit("scene_bake_probe needs a CUDA device")
    insts, mats = terrain_instances()
    sc, keep, shading, uv_accels, offsets, nf = api.Scene(), [], [], [], [], 0
    accels = {}
    for v, f, x, ids in insts:
        key = (v.ctypes.data, f.ctypes.data)
        if key not in accels:
            accels[key] = api.BVHAccel()
            accels[key].Build(len(f), v, f)
        sc.AddNode(accels[key], x)
        d_ids = torch.from_numpy(ids.astype(np.int32)).cuda()
        keep.append(d_ids)
        shading.append(api.SceneShading(d_ids.data_ptr(), None))
        offsets.append(nf)
        nf += len(f)
    assert sc.Commit()
    v = insts[0][0]
    f = np.concatenate([x[1] for x in insts])
    ids = np.concatenate([x[3] for x in insts])
    flat = api.BVHAccel()
    flat.Build(len(f), v, f)
    light = len(insts) - 1
    pairs = np.array([(light, k) for k in range(len(insts[light][1]))], np.int32)
    d_pairs = torch.from_numpy(pairs.reshape(-1).copy()).cuda()
    d_emit = torch.from_numpy((offsets[light] + pairs[:, 1]).astype(np.int32)).cuda()
    d_fids = torch.from_numpy(ids.astype(np.int32)).cuda()
    d_mats = torch.from_numpy(np.ascontiguousarray(mats).view(np.float32).reshape(-1).copy()).cuda()
    for v_, f_, _, _ in insts[:light]:
        a = api.BVHAccel()
        uvv, uvf = uv_mesh(v_, f_)
        a.Build(len(uvf), uvv, uvf)
        uv_accels.append(a)
    offsets = np.asarray(offsets, np.uint32)
    rows = []
    for size in (2048, 4096):
        cell = size // 4
        charts = []
        for i in range(len(insts)):
            c = api.SceneChart()
            if i < light:
                c.uv = uv_accels[i]._h
                c.x0, c.y0, c.width, c.height = (i % 4) * cell, (i // 4) * cell, cell, cell
                c.uv_region[:], c.texel_offset[:] = (0.0, 1.0, 0.0, 1.0), (0.5, 0.5)
            charts.append(c)
        rec = torch.zeros(size * size * 4, dtype=torch.int32, device="cuda")
        inst = torch.zeros(size * size, dtype=torch.int32, device="cuda")
        n_cov = sc.UVRaster(charts, size, size, rec.data_ptr(), inst.data_ptr())
        hr, hi = rec.view(-1, 4).cpu().numpy().view(np.uint32), inst.cpu().numpy().view(np.uint32)
        cov = hi != 0xFFFFFFFF
        hr[cov, 3] = offsets[hi[cov]] + hr[cov, 3]
        frec = torch.from_numpy(hr.view(np.int32).reshape(-1).copy()).cuda()
        for bounces in (1, 5):
            p = api.LightmapParams()
            p.width = p.height = size
            p.spp, p.sample0, p.seed, p.max_bounces = 16, 0, 7, bounces
            p.ray_min_t, p.ray_max_t = 1e-3, 1e30
            p.n_materials, p.n_emissive = len(mats), len(pairs)
            p.d_materials, p.d_emissive_faces = d_mats.data_ptr(), d_pairs.data_ptr()
            pf = api.LightmapParams.from_buffer_copy(p)
            pf.d_material_ids, pf.d_emissive_faces = d_fids.data_ptr(), d_emit.data_ptr()
            acc = torch.zeros(size * size * 3, dtype=torch.float32, device="cuda")
            runs = {"scene": lambda: sc.BakeLightmap(rec.data_ptr(), inst.data_ptr(), p, shading, acc.data_ptr()),
                    "flat": lambda: flat.BakeLightmap(frec.data_ptr(), pf, acc.data_ptr())}
            res = {k: [r()] for k, r in runs.items()}  # warm-up
            for _ in range(reps):
                for k, r in runs.items():
                    res[k].append(r())
            row = {"bake": "lightmap", "atlas": size, "spp": 16, "max_bounces": bounces, "texels": n_cov}
            for k, rs in res.items():
                r = min(rs[1:], key=lambda x: x.total_ms)
                rays = r.radiance_rays + r.shadow_rays
                row[k] = {"total_ms": round(r.total_ms, 2), "traverse_ms": round(r.traverse_ms, 2),
                          "paths_per_s": round(r.paths / (r.total_ms * 1e-3)),
                          "rays_per_s": round(rays / (r.total_ms * 1e-3)),
                          "rays_per_s_traversal": round(rays / (r.traverse_ms * 1e-3)) if r.traverse_ms else None,
                          "traverse_launches": r.traverse_launches}
            row["scene_over_flat_paths_per_s"] = round(row["flat"]["total_ms"] / row["scene"]["total_ms"], 3)
            rows.append(row)
            print(json.dumps(row), flush=True)
        b = api.BakeParams()
        b.width = b.height = size
        b.spp, b.sample0, b.seed, b.ao_min_t, b.ao_max_t, b.flags = 16, 0, 3, 1e-3, 2.0, 0
        acc = torch.zeros(size * size, dtype=torch.float32, device="cuda")
        runs = {"scene": lambda: sc.BakeAO(rec.data_ptr(), inst.data_ptr(), b, acc.data_ptr()),
                "flat": lambda: flat.BakeAO(frec.data_ptr(), b, acc.data_ptr())}
        res = {k: [r()] for k, r in runs.items()}
        for _ in range(reps):
            for k, r in runs.items():
                res[k].append(r())
        row = {"bake": "ao", "atlas": size, "spp": 16, "texels": n_cov}
        for k, rs in res.items():
            r = min(rs[1:], key=lambda x: x.total_ms)
            row[k] = {"total_ms": round(r.total_ms, 2), "traverse_ms": round(r.traverse_ms, 2),
                      "rays_per_s": round(r.ao_rays / (r.total_ms * 1e-3)),
                      "rays_per_s_traversal": round(r.ao_rays / (r.traverse_ms * 1e-3)),
                      "traverse_launches": r.traverse_launches}
        row["scene_over_flat_rays_per_s"] = round(row["flat"]["total_ms"] / row["scene"]["total_ms"], 3)
        rows.append(row)
        print(json.dumps(row), flush=True)
        del rec, inst, frec
    print(json.dumps({"results": rows, **card()}))


if __name__ == "__main__":
    main()
