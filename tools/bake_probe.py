"""Texel cast + AO bake of a UV atlas, timed, next to the flat AO pass on the same accel.

The 1,002,528-triangle terrain (bench.py's configs[2] mesh) with planar UVs is rastered at 2048^2 and 4096^2 texels
(nrt_uv_raster_device, production walk), then baked at 64 spp (nrt_bake_ao_device) with and without ANY_HIT; the bake's
AO launch is the flat pass's AO launch with another ray loader, so the same run also prints nrt_render_ao_device's
ao_traverse_ms / ao_rays on the same world accel.  Rates are rays over the traversal launches' device time (CUDA
events), best of `reps`; the card's name and power limit are read in the same run.

    python tools/bake_probe.py [spp reps]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from nanort_b200 import api, scenes as S


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return r, e0.elapsed_time(e1)


def main():
    spp, reps = (int(a) for a in (sys.argv[1:3] + ["64", "3"][len(sys.argv[1:3]):]))
    if not torch.cuda.is_available():
        raise SystemExit("bake_probe needs a CUDA device")
    v, f = S.make_scene("terrain")
    uv, uf = S.planar_uv(v, f)
    world, uv_acc = api.BVHAccel(), api.BVHAccel()
    world.Build(len(f), v, f)
    uv_acc.Build(len(uf), uv, uf)
    radius = 0.25 * float(np.linalg.norm(v.max(axis=0) - v.min(axis=0)))
    out = {"workload": f"terrain ({len(f)} triangles), planar UVs, AO range [1e-3, {radius:.3f}), {spp} spp"}

    # the flat AO pass on the same accel (bench.py's camera and pass parameters at 1920x1080, 4 spp)
    W, H = 1920, 1080
    cam = S.scene_camera("terrain", W, H)
    p = api.AoParams()
    for i in range(12):
        p.cam[i] = float(cam[i])
    p.width, p.height, p.spp, p.sample0, p.seed = W, H, 4, 0, 1
    p.tile_w, p.tile_h, p.shard, p.n_shards = 64, 8, 0, 1
    p.ray_min_t, p.ray_max_t, p.ao_min_t, p.ao_max_t = 1e-3, 1e30, 1e-3, radius
    frame = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    world.RenderAO(p, frame.data_ptr())
    best = min((world.RenderAO(p, frame.data_ptr()) for _ in range(reps)), key=lambda r: r.ao_traverse_ms)
    out["render_ao"] = {"ao_rays": best.ao_rays, "ao_traverse_ms": round(best.ao_traverse_ms, 3),
                        "ao_mrays_per_s": round(best.ao_rays / (best.ao_traverse_ms * 1e3), 1)}

    for T in (2048, 4096):
        rp = api.UvRasterParams()
        rp.width, rp.height = T, T
        rp.uv_region[:] = [0.0, 1.0, 0.0, 1.0]
        rp.texel_offset[:] = [0.5, 0.5]
        rec = torch.empty((T * T, 4), dtype=torch.float32, device="cuda")
        uv_acc.UVRaster(rp, rec.data_ptr())  # warm-up
        raster_ms = min(timed(lambda: uv_acc.UVRaster(rp, rec.data_ptr()))[1] for _ in range(reps))
        row = {"raster_ms": round(raster_ms, 3)}
        accum = torch.zeros(T * T, dtype=torch.float32, device="cuda")
        for label, flags in (("closest", 0), ("any_hit", api.TRAVERSE_ANY_HIT)):
            bp = api.BakeParams()
            bp.width, bp.height, bp.spp, bp.sample0, bp.seed = T, T, spp, 0, 1
            bp.ao_min_t, bp.ao_max_t, bp.flags = 1e-3, radius, flags
            world.BakeAO(rec.data_ptr(), bp, accum.data_ptr())  # warm-up
            runs = [timed(lambda: world.BakeAO(rec.data_ptr(), bp, accum.data_ptr())) for _ in range(reps)]
            r, ms = min(runs, key=lambda x: x[0].traverse_ms)
            row[label] = {"texels": r.texels, "ao_rays": r.ao_rays, "occluded": r.ao_hits, "bake_ms": round(ms, 1),
                          "traverse_ms": round(r.traverse_ms, 1), "traverse_launches": r.traverse_launches,
                          "mrays_per_s": round(r.ao_rays / (r.traverse_ms * 1e3), 1)}
        out[f"{T}x{T}"] = row
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
