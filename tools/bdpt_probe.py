"""The bidirectional path tracer (nrt_render_bdpt_device), timed after warm-up.

Workloads: the Cornell box with the reference's material set (scenes.cornell_with_materials) at 512x512, and the
1,002,528-triangle terrain under an area light (scenes.with_area_light), both from the reference's camera
{0,5,20, 1,0,0, 0,1,0, 0,0,-1}, max_bounces 10, flat face-varying normals, production walk and tree.  Reported per
workload: samples/s over the whole call, rays/s by kind (eye, light, connection) over the traversal launches' device
time (CUDA events, best of `reps`), and the traversal launches' share of the call.  The card's name and power limit
are read in the same run.

    python tools/bdpt_probe.py [spp reps]"""
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


def flat_normals(v, f):
    """normalize(cross(v2 - v0, v1 - v0)) at the three corners of every face (the example loader's calcNormal)"""
    t = v[f.astype(np.int64)]
    n = np.cross(t[:, 2] - t[:, 0], t[:, 1] - t[:, 0]).astype(np.float32)
    n /= np.maximum(np.linalg.norm(n, axis=1, keepdims=True), np.float32(1e-30))
    return np.repeat(n, 3, axis=0).reshape(-1, 9).astype(np.float32)


def run(name, v, f, mats, ids, W, H, spp, reps):
    acc = api.BVHAccel()
    acc.Build(len(f), v, f)
    d_mats = torch.from_numpy(np.ascontiguousarray(mats).view(np.float32).reshape(-1, 16).copy()).cuda()
    d_ids = torch.from_numpy(ids.astype(np.int32)).cuda()
    d_fvn = torch.from_numpy(flat_normals(v, f)).cuda()
    p = api.BdptParams()
    cam = [0, 5, 20, 1, 0, 0, 0, 1, 0, 0, 0, -1]
    for k in range(12):
        p.cam[k] = float(cam[k])
    p.width, p.height, p.spp, p.sample0, p.spp_total = W, H, spp, 0, spp
    p.tile_w, p.tile_h, p.shard, p.n_shards = 64, 8, 0, 1
    p.max_bounces, p.n_materials = 10, len(d_mats)
    p.d_materials, p.d_material_ids, p.d_facevarying_normals = d_mats.data_ptr(), d_ids.data_ptr(), d_fvn.data_ptr()
    p.flags = 0
    frame = torch.zeros(3 * W * H, dtype=torch.float32, device="cuda")
    acc.RenderBDPT(p, frame.data_ptr())  # warm-up
    r = min((acc.RenderBDPT(p, frame.data_ptr()) for _ in range(reps)), key=lambda x: x.total_ms)
    rays = r.eye_rays + r.light_rays + r.connection_rays
    return {"workload": f"{name} ({len(f)} triangles), {W}x{H}, {spp} spp, max_bounces 10",
            "total_ms": round(r.total_ms, 2), "traverse_ms": round(r.traverse_ms, 2),
            "traverse_share": round(r.traverse_ms / r.total_ms, 3),
            "msamples_per_s": round(W * H * spp / (r.total_ms * 1e3), 2),
            "eye_rays": r.eye_rays, "light_rays": r.light_rays, "connection_rays": r.connection_rays,
            "mrays_per_s_traversal": round(rays / (r.traverse_ms * 1e3), 1),
            "mrays_per_s_call": round(rays / (r.total_ms * 1e3), 1),
            "connection_share_of_rays": round(r.connection_rays / rays, 3),
            "launches": r.launches, "traverse_launches": r.traverse_launches}


def main():
    spp, reps = (int(a) for a in (sys.argv[1:3] + ["4", "3"][len(sys.argv[1:3]):]))
    if not torch.cuda.is_available():
        raise SystemExit("bdpt_probe needs a CUDA device")
    out = {}
    v, f, mats, ids, _ = S.cornell_with_materials()
    out["cornell"] = run("cornell", v, f, mats, ids, 512, 512, spp, reps)
    v, f = S.make_scene("terrain")
    v, f, l0, ln = S.with_area_light(v, f, (0.0, 3.0, 0.0), 1.0, 1.0)
    mats = np.concatenate([S.material(diffuse=(0.7, 0.6, 0.5)), S.material(emission=(20.0, 20.0, 20.0))])
    ids = np.zeros(len(f), np.uint32)
    ids[l0:l0 + ln] = 1
    out["terrain"] = run("terrain + area light", v, f, mats, ids, 512, 512, max(1, spp // 4), reps)
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
