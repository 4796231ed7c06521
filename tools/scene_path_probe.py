"""Path-tracing rate of a two-level scene against the same geometry as one flat accel.

The 1,002,528-triangle terrain under its area light (bench.py's configs[2] scene) is rendered twice at the same
parameters: as a scene of 17 instances (the terrain's faces cut into 16 runs of 1/16 each, each its own accel with an
identity matrix, plus the light) through nrt_scene_render_path_device, and flattened, as one accel, through
nrt_render_path_device.  Prints M rays/s (radiance + shadow Traverse calls over the pass's wall time, CUDA events) for
both, with the card's name and power limit read in the same run.

    python tools/scene_path_probe.py [W H spp reps]"""
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


def main():
    W, H, spp, reps = (int(a) for a in (sys.argv[1:5] + ["1920", "1080", "16", "3"][len(sys.argv[1:5]):]))
    if not torch.cuda.is_available():
        raise SystemExit("scene_path_probe needs a CUDA device")
    v, f = S.make_scene("terrain")
    v, f, l0, ln = S.with_area_light(v, f, (0.0, 6.0, 0.0), 2.0, 2.0)
    mats = np.concatenate([S.material(diffuse=(0.7, 0.7, 0.7)), S.material(emission=(20, 20, 20))])
    ids = np.zeros(len(f), np.uint32)
    ids[l0:] = 1
    d_m = torch.as_tensor(mats.view(np.float32).reshape(-1), device="cuda")
    cam = S.scene_camera("terrain", W, H)
    eye = np.eye(4, dtype=np.float32)

    def params():
        p = api.PathParams()
        for i in range(12):
            p.cam[i] = float(cam[i])
        p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, 0, 3
        p.tile_w, p.tile_h, p.shard, p.n_shards = 64, 8, 0, 1
        p.max_bounces, p.ray_min_t, p.ray_max_t = 10, 1e-3, 1e30
        p.n_materials, p.d_materials, p.flags = len(mats), d_m.data_ptr(), 0
        return p

    # flat
    flat = api.BVHAccel()
    flat.Build(len(f), v, f)
    d_i = torch.as_tensor(ids.astype(np.int32), device="cuda")
    d_e = torch.as_tensor(np.arange(l0, l0 + ln, dtype=np.int32), device="cuda")
    pf = params()
    pf.n_emissive, pf.d_material_ids, pf.d_emissive_faces = ln, d_i.data_ptr(), d_e.data_ptr()
    # scene: 16 runs of the terrain's faces + the light, every instance with the identity matrix
    cuts = np.linspace(0, l0, 17).astype(np.int64)
    parts = [(cuts[k], cuts[k + 1]) for k in range(16)] + [(l0, l0 + ln)]
    sc, accels, keep, shading = api.Scene(), [], [], []
    for a, b in parts:
        acc = api.BVHAccel()
        acc.Build(b - a, v, np.ascontiguousarray(f[a:b]))
        accels.append(acc)
        sc.AddNode(acc, eye)
        t = torch.as_tensor(ids[a:b].astype(np.int32), device="cuda")
        keep.append(t)
        shading.append(api.SceneShading(t.data_ptr(), None))
    assert sc.Commit()
    d_pairs = torch.as_tensor(np.stack([np.full(ln, 16), np.arange(ln)], axis=1).reshape(-1).astype(np.int32), device="cuda")
    ps = params()
    ps.n_emissive, ps.d_emissive_faces = ln, d_pairs.data_ptr()

    accum = torch.zeros(W * H * 3, dtype=torch.float32, device="cuda")
    runs = {"flat": lambda: flat.RenderPath(pf, accum.data_ptr()),
            "scene": lambda: sc.RenderPath(ps, shading, accum.data_ptr())}
    out = {"workload": f"terrain + area light ({len(f)} triangles), {W}x{H}x{spp} spp, <= 10 bounces; scene = 16 + 1 instances"}
    for name in runs:  # warm-up
        runs[name]()
    torch.cuda.synchronize()
    rates = {k: [] for k in runs}
    images = {}
    for _ in range(reps):  # alternate the two passes
        for name, run in runs.items():
            accum.zero_()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = run()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
            rates[name].append((r.radiance_rays + r.shadow_rays) / (ms * 1e3))
            images[name] = float(accum.double().sum()) / (W * H * spp)
    out.update({f"{k}_mrays_per_s": [round(x, 1) for x in rates[k]] for k in rates})
    out.update({f"{k}_mean_radiance": round(images[k], 6) for k in images})
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
