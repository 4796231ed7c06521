"""Lane-state histogram of the persistent traversal warps on the exported primary / AO ray sets
(nrt_traverse_lane_stats_device): where the 32 lanes go in the node phase, the leaf phase, refills and retires."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import json
import numpy as np
import torch
from nanort_b200 import api, scenes as S

scenes = sys.argv[1].split(",") if len(sys.argv) > 1 else ["sphere_grid", "terrain"]
W, H, spp = 1920, 1080, 2
for scene in scenes:
    v, f = S.make_scene(scene)
    acc = api.BVHAccel(); acc.Build(len(f), v, f)
    cam = S.scene_camera(scene, W, H)
    bmin, bmax = acc.BoundingBox()
    p = api.AoParams()
    for i in range(12): p.cam[i] = float(cam[i])
    p.width, p.height, p.spp, p.sample0, p.seed = W, H, spp, 0, 1
    p.tile_w, p.tile_h, p.shard, p.n_shards = 64, 8, 0, 1
    p.ray_min_t, p.ray_max_t, p.ao_min_t, p.ao_max_t = 1e-3, 1e30, 1e-3, 0.25 * float(np.linalg.norm(bmax - bmin))
    n = W * H * spp
    accum = torch.zeros(W * H, dtype=torch.float32, device="cuda")
    d_p = torch.empty(n * 36, dtype=torch.uint8, device="cuda")
    d_a = torch.empty(n * 36, dtype=torch.uint8, device="cuda")
    n_p, n_a = acc.ExportAOWorkload(p, accum.data_ptr(), d_p.data_ptr(), d_a.data_ptr())
    for name, d_r, cnt in (("primary", d_p, n_p), ("ao", d_a, n_a)):
        s = acc.LaneStatsDevice(d_r.data_ptr(), cnt)
        ns, lr, ts = max(s["node_steps"], 1), max(s["leaf_rounds"], 1), max(s["tri_steps"], 1)
        print(json.dumps({"scene": scene, "rays": name, "n": cnt,
                          "node_steps_per_ray": s["boxes"] / 2 / cnt, "prims_per_ray": s["prims"] / cnt,
                          "node_phase_lanes": {"testing": s["lanes_testing"] / ns, "no_ray": s["lanes_no_ray"] / ns,
                                               "finished": s["lanes_finished"] / ns,
                                               "parked_on_leaves": s["lanes_parked_on_leaves"] / ns},
                          "leaf_round_lanes": s["lanes_with_leaf"] / lr, "tri_step_lanes": s["prims"] / ts,
                          "tri_steps_per_round": ts / lr, "node_steps_per_outer": ns / max(s["outer_iterations"], 1),
                          "refill_lanes": s["lanes_refilled"] / max(s["refill_events"], 1),
                          "retire_lanes": s["lanes_retired"] / max(s["retire_events"], 1),
                          "outer_per_ray_x32": 32 * s["outer_iterations"] / cnt, "raw": s}), flush=True)
