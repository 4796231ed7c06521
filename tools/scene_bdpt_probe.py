"""The bidirectional path tracer over a two-level scene (nrt_scene_render_bdpt_device) against the same geometry as one
flat accel (nrt_render_bdpt_device), timed after warm-up, the two passes alternated.

Workloads, both from the reference's camera {0,5,20, 1,0,0, 0,1,0, 0,0,-1}, max_bounces 10, flat face-varying
normals, production walk and trees:
  - the instanced Cornell box at 512x512x4: tests/test_gpu_scene_path.py's instanced_cornell() (the walls, the light
    x2, one box mesh shared by a rotated, non-uniformly scaled instance and a mirrored one);
  - the 1,002,528-triangle terrain under its area light, the terrain's faces cut into 16 identity instances plus the
    light (tools/scene_path_probe.py's scene), at 512x512x1.
Reported per workload and pass: samples/s over the call's device time (CUDA events inside the call) and over the host
wall time of the call (which includes the scene pass's per-call allocation and free), the scene walks' (or traversal
launches') device time and share of the call (best of `reps`), with the card's name and power limit read in the same
run.

    python tools/scene_bdpt_probe.py [reps]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

from nanort_b200 import api, scenes as S
from test_gpu_scene_path import instanced_cornell  # the scene the scene pass's tests render

CAM = [0, 5, 20, 1, 0, 0, 0, 1, 0, 0, 0, -1]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def flat_normals(v, f):
    """normalize(cross(v2 - v0, v1 - v0)) at the three corners of every face"""
    t = v[f.astype(np.int64)]
    n = np.cross(t[:, 2] - t[:, 0], t[:, 1] - t[:, 0]).astype(np.float32)
    n /= np.maximum(np.linalg.norm(n, axis=1, keepdims=True), np.float32(1e-30))
    return np.repeat(n, 3, axis=0).reshape(-1, 9).astype(np.float32)


def terrain_instances():
    v, f = S.make_scene("terrain")
    v, f, l0, ln = S.with_area_light(v, f, (0.0, 6.0, 0.0), 2.0, 2.0)
    mats = np.concatenate([S.material(diffuse=(0.7, 0.7, 0.7)), S.material(emission=(20, 20, 20))])
    ids = np.zeros(len(f), np.uint32)
    ids[l0:] = 1
    cuts = np.linspace(0, l0, 17).astype(np.int64)
    parts = [(cuts[k], cuts[k + 1]) for k in range(16)] + [(l0, l0 + ln)]
    eye = np.eye(4, dtype=np.float32)
    return [(v, np.ascontiguousarray(f[a:b]), eye, ids[a:b].copy()) for a, b in parts], mats


def params(W, H, spp, d_mats, n_mats, d_ids=None, d_fvn=None):
    p = api.BdptParams()
    for k in range(12):
        p.cam[k] = float(CAM[k])
    p.width, p.height, p.spp, p.sample0, p.spp_total = W, H, spp, 0, spp
    p.tile_w, p.tile_h, p.shard, p.n_shards = 64, 8, 0, 1
    p.max_bounces, p.n_materials = 10, n_mats
    p.d_materials = d_mats.data_ptr()
    p.d_material_ids = d_ids.data_ptr() if d_ids is not None else None
    p.d_facevarying_normals = d_fvn.data_ptr() if d_fvn is not None else None
    p.flags = 0
    return p


def run(name, insts, mats, W, H, spp, reps):
    d_mats = torch.from_numpy(np.ascontiguousarray(mats).view(np.float32).reshape(-1, 16).copy()).cuda()
    keep, shading, accels = [], [], {}
    sc = api.Scene()
    fv, ff, fids, nv = [], [], [], 0
    for v, f, x, ids in insts:
        key = (v.ctypes.data, f.ctypes.data)
        if key not in accels:
            accels[key] = api.BVHAccel()
            accels[key].Build(len(f), v, f)
        sc.AddNode(accels[key], x)
        d_ids = torch.from_numpy(ids.astype(np.int32)).cuda()
        d_n = torch.from_numpy(flat_normals(v, f).reshape(-1).copy()).cuda()
        keep += [d_ids, d_n]
        shading.append(api.SceneShading(d_ids.data_ptr(), d_n.data_ptr()))
        wv = (np.c_[v.astype(np.float64), np.ones(len(v))] @ x.astype(np.float64))[:, :3].astype(np.float32)
        fv.append(wv)
        ff.append(f.astype(np.uint32) + nv)
        fids.append(ids)
        nv += len(v)
    assert sc.Commit()
    v, f, ids = np.concatenate(fv), np.concatenate(ff), np.concatenate(fids)
    flat = api.BVHAccel()
    flat.Build(len(f), v, f)
    d_fids = torch.from_numpy(ids.astype(np.int32)).cuda()
    d_ffvn = torch.from_numpy(flat_normals(v, f).reshape(-1).copy()).cuda()
    ps = params(W, H, spp, d_mats, len(d_mats))
    pf = params(W, H, spp, d_mats, len(d_mats), d_fids, d_ffvn)
    frame = torch.zeros(3 * W * H, dtype=torch.float32, device="cuda")
    runs = {"flat": lambda: flat.RenderBDPT(pf, frame.data_ptr()),
            "scene": lambda: sc.RenderBDPT(ps, shading, frame.data_ptr())}
    for r in runs.values():  # warm-up
        r()
    best, host = {}, {}
    for _ in range(reps):
        for k, r in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = r()
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3
            host[k] = min(host.get(k, ms), ms)
            if k not in best or res.total_ms < best[k].total_ms:
                best[k] = res
    out = {"workload": f"{name} ({len(f)} triangles, {len(insts)} instances), {W}x{H}, {spp} spp, max_bounces 10"}
    for k, r in best.items():
        out[k] = {"total_ms": round(r.total_ms, 2), "traverse_ms": round(r.traverse_ms, 2),
                  "traverse_share": round(r.traverse_ms / r.total_ms, 3),
                  "msamples_per_s": round(W * H * spp / (r.total_ms * 1e3), 3), "host_ms": round(host[k], 2),
                  "msamples_per_s_host": round(W * H * spp / (host[k] * 1e3), 3),
                  "rays": int(r.eye_rays + r.light_rays + r.connection_rays), "launches": int(r.launches)}
    out["scene_over_flat_samples_per_s"] = round(best["flat"].total_ms / best["scene"].total_ms, 3)
    out["scene_over_flat_host"] = round(host["flat"] / host["scene"], 3)
    return out


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    if not torch.cuda.is_available():
        raise SystemExit("scene_bdpt_probe needs a CUDA device")
    res = [run("instanced Cornell", *instanced_cornell(), 512, 512, 4, reps),
           run("terrain in 16 instances + area light", *terrain_instances(), 512, 512, 1, reps)]
    print(json.dumps({"results": res, **card()}))


if __name__ == "__main__":
    main()
