"""Times the lightmap bake (nrt_bake_lightmap_device) on the 1 M-triangle terrain under its area light (planar UVs, the
light charted outside the atlas) and on the Cornell box (one chart per face), next to the path pass on the same accel.

For each configuration, best of 3 calls: total_ms, traverse_ms, paths/s over the whole call and rays/s (radiance +
shadow rays) over the traversal launches.  The path pass line is nrt_render_path_device at 1920x1080 with the same
max_bounces, rays/s over its traversal launches (camera, continuation and shadow rays).
usage: python tools/lightmap_probe.py [--quick] [--out file.json]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nanort_b200 import api, scenes as S  # noqa: E402


def terrain_scene():
    v, f = S.make_scene("terrain")
    v, f, l0, ln = S.with_area_light(v, f, (0.0, 6.0, 0.0), 2.0, 2.0)
    mats = np.concatenate([S.material(diffuse=(0.7, 0.7, 0.7)), S.material(emission=(20, 20, 20))])
    ids = np.zeros(len(f), np.uint32)
    ids[l0:] = 1
    uv, _ = S.planar_uv(v[:int(f[:l0].max()) + 1], f[:l0])
    lv = np.zeros((3 * ln, 3), np.float32)
    lv[:, :2] = np.tile(np.float32([[2.2, 2.2], [2.8, 2.2], [2.2, 2.8]]), (ln, 1))
    uv = np.concatenate([uv, lv])
    return v, f, mats, ids, np.arange(l0, l0 + ln, dtype=np.uint32), uv, "terrain"


def cornell_scene():
    v, f, mats, ids, emissive = S.cornell_with_materials()
    uv, _ = S.per_face_atlas(len(f))
    return v, f, mats, ids, emissive, uv, "cornell"


def best_of(fn, k=3):
    rs = [fn() for _ in range(k)]
    return min(rs, key=lambda r: r.total_ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="2048^2 only")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = []
    for make, sizes, spps in ((terrain_scene, (2048,) if a.quick else (2048, 4096), (16,)), (cornell_scene, (2048,), (16,))):
        v, f, mats, ids, emissive, uv, name = make()
        world = api.BVHAccel()
        world.Build(len(f), v, f)
        uv_acc = api.BVHAccel()
        uv_acc.Build(len(f), uv, np.arange(3 * len(f), dtype=np.uint32).reshape(-1, 3))
        d_m = torch.as_tensor(np.ascontiguousarray(mats).view(np.float32).reshape(-1), device="cuda")
        d_i = torch.as_tensor(ids.astype(np.int32), device="cuda")
        d_e = torch.as_tensor(emissive.astype(np.int32), device="cuda")
        for bounces in (1, 5):
            pp = api.PathParams()
            cam = S.scene_camera(name, 1920, 1080)
            for i in range(12):
                pp.cam[i] = float(cam[i])
            pp.width, pp.height, pp.spp, pp.sample0, pp.seed = 1920, 1080, 4, 0, 1
            pp.tile_w, pp.tile_h, pp.shard, pp.n_shards = 64, 8, 0, 1
            pp.max_bounces, pp.ray_min_t, pp.ray_max_t = bounces, 1e-3, 1e30
            pp.n_materials, pp.n_emissive = len(mats), len(emissive)
            pp.d_materials, pp.d_material_ids, pp.d_emissive_faces = d_m.data_ptr(), d_i.data_ptr(), d_e.data_ptr()
            img = torch.zeros(1920 * 1080 * 3, dtype=torch.float32, device="cuda")
            world.RenderPath(pp, img.data_ptr())  # warm-up
            rp = best_of(lambda: world.RenderPath(pp, img.data_ptr()))
            path_rays = rp.radiance_rays + rp.shadow_rays
            for size in sizes:
                rec = torch.zeros((size * size, 4), dtype=torch.float32, device="cuda")
                rparams = api.UvRasterParams()
                rparams.width = rparams.height = size
                rparams.uv_region[:] = [0.0, 1.0, 0.0, 1.0]
                rparams.texel_offset[:] = [0.5, 0.5]
                n_cov = uv_acc.UVRaster(rparams, rec.data_ptr())
                for spp in spps:
                    p = api.LightmapParams()
                    p.width = p.height = size
                    p.spp, p.sample0, p.seed, p.max_bounces = spp, 0, 7, bounces
                    p.ray_min_t, p.ray_max_t = 1e-3, 1e30
                    p.n_materials, p.n_emissive = len(mats), len(emissive)
                    p.d_materials, p.d_material_ids, p.d_emissive_faces = d_m.data_ptr(), d_i.data_ptr(), d_e.data_ptr()
                    accum = torch.zeros(size * size * 3, dtype=torch.float32, device="cuda")
                    world.BakeLightmap(rec.data_ptr(), p, accum.data_ptr())  # warm-up
                    r = best_of(lambda: world.BakeLightmap(rec.data_ptr(), p, accum.data_ptr()))
                    rays = r.radiance_rays + r.shadow_rays
                    row = {"scene": name, "atlas": size, "spp": spp, "max_bounces": bounces, "texels": n_cov,
                           "paths": r.paths, "total_ms": round(r.total_ms, 2), "traverse_ms": round(r.traverse_ms, 2),
                           "paths_per_s": r.paths / (r.total_ms * 1e-3),
                           "rays_per_s_traversal": rays / max(r.traverse_ms * 1e-3, 1e-9),
                           "traverse_launches": r.traverse_launches,
                           "path_pass_rays_per_s_traversal": path_rays / max(rp.traverse_ms * 1e-3, 1e-9),
                           "path_pass_traverse_ms": round(rp.traverse_ms, 2)}
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                del rec
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
