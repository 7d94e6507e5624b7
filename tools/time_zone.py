#!/usr/bin/env python
"""Zone monitoring on the GPU (ob_zone_render, ob_zone_monitor_update) at 128x2048 (785.json's beams, 2048 columns):
  * render of 1 zone and of 16 zones of 2048 triangles each (height fields around the sensor, tests/test_gpu_zone),
    and of one 2048-triangle box that encloses the sensor, so every ray tests every triangle (the worst case);
  * one monitor update of 16 live zones on a device range image, bitmask included.
Reports CUDA-event ms per call (a render call ends in a synchronise: it checks the hit counts on the host), and the
one-core oracle (oracle/orc_zone.c) for the 1-zone and box renders.  Writes h100_zone.json into --out (default: a
directory under the system temporary directory) with the card's name and power limit read in the same run.

    python tools/time_zone.py [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import __graft_entry__ as graft  # noqa: E402
from oracle import zone as oz  # noqa: E402
from tests.test_gpu_zone import grid_mesh, random_range, random_zones, subsample  # noqa: E402
from tests.test_oracle_zone import s2b_z1, sensor_meta  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ouster_b200_profiles"))
args = ap.parse_args()
ob = graft.load_package()
if ob.device_count() == 0:
    sys.exit("time_zone.py needs a CUDA device")
dev = torch.device("cuda", 0)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()[0]
ST = ob.Stream(0, cuda_stream=torch.cuda.current_stream(dev).cuda_stream)
H, W = 128, 2048
meta = subsample(sensor_meta("785.json"), H, W)
cfg = ob.pyapi.BeamConfig.from_sensor_info(meta, s2b_z1())
out = {"gpu": gpu, "reps": args.reps, "shape": [H, W], "cases": {},
       "input": "785.json's 128 beams at 2048 columns, sensor_to_body z = 1 m; meshes of 2048 triangles"}


def event_ms(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def oriented(k, seed):
    t = grid_mesh(32, 1.0 + 0.25 * (k // 6), seed).reshape(-1, 3, 3)
    t = np.roll(t, k % 3, axis=2)
    if (k // 3) % 2:
        t = -t
    return t.reshape(-1, 9)


def enclosing_box():
    faces = []
    for ax in range(3):
        for s in (-1, 1):
            q = grid_mesh(13, 0, ax)[:341].reshape(-1, 3, 3) * np.float32(2.5)
            q[..., 2] = 4 * s
            faces.append(np.roll(q, ax, axis=2).reshape(-1, 9))
    t = np.concatenate(faces)
    return np.concatenate([t, t[:2048 - len(t)]])


box = enclosing_box()
assert len(box) == 2048
cases = {"render_1_zone": [{"triangles": oriented(0, 0), "coordinate_frame": 1}],
         "render_16_zones": [{"triangles": oriented(k, k), "coordinate_frame": 1 + k % 2} for k in range(16)],
         "render_box_every_ray_hits": [{"triangles": box, "coordinate_frame": 2}]}
sensor_lut = cfg.lut_no_sensor_to_body_transform
for name, zones in cases.items():
    run = lambda: ob.zone_render(zones, H, W, sensor_lut, cfg.lut, stream=ST)
    near, far, px = run()
    ms = event_ms(run, args.reps)
    rec = {"gpu_ms_per_call": ms, "zones": len(zones), "triangles_per_zone": 2048,
           "pixels_with_intersections": [int(v) for v in px]}
    if len(zones) == 1:
        lut = cfg.lut if zones[0]["coordinate_frame"] == 1 else sensor_lut
        t0 = time.perf_counter()
        rn, rf, rpx = oz.render(zones[0]["triangles"], lut.direction, lut.offset, H, W)
        rec["oracle_one_core_ms"] = (time.perf_counter() - t0) * 1e3
        rec["bit_exact_vs_oracle"] = bool(np.array_equal(near[0].cpu().numpy().view(np.uint32), rn) and
                                          np.array_equal(far[0].cpu().numpy().view(np.uint32), rf) and px[0] == rpx)
    out["cases"][name] = rec
    print(name, json.dumps(rec), flush=True)

zones = random_zones(H, W, 16, 7)
live = [{"id": z[0], "mode": z[1], "point_count": z[2], "frame_count": z[3], "near_mm": z[4], "far_mm": z[5]}
        for z in zones]
mon = ob.ZoneMonitor(live, H, W)
rng = torch.from_numpy(random_range(zones, H, W, 1).view(np.int32)).to(dev)
bm = torch.zeros((H, W), dtype=torch.int32, device=dev)
ms = event_ms(lambda: mon.update(rng, bm, stream=ST), max(args.reps, 200))
t0 = time.perf_counter()
for z in zones:
    oz.counts(rng.cpu().numpy().view(np.uint32), z[4], z[5])
orc_ms = (time.perf_counter() - t0) * 1e3
out["cases"]["monitor_update_16_zones"] = {"gpu_ms_per_update": ms, "launches_per_update": 2,
                                           "oracle_one_core_ms": orc_ms,
                                           "bytes_read_per_update": int(H * W * 4 * (1 + 2 * 16) + H * W * 4 * 2)}
print("monitor_update_16_zones", json.dumps(out["cases"]["monitor_update_16_zones"]), flush=True)
os.makedirs(args.out, exist_ok=True)
with open(os.path.join(args.out, "h100_zone.json"), "w") as f:
    json.dump(out, f, indent=1)
print("wrote", os.path.join(args.out, "h100_zone.json"))
