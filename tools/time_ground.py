#!/usr/bin/env python
"""Ground segmentation (ob_ground_mask) on the GPU: whole calls timed with CUDA events after a warm-up, device
buffers, for one 128x2048 dual-return frame of `box_rooftop` and of `room` (NORMALS given, and computed by the call),
and a 16-frame set; the per-kernel times of one profiled call, which give each pass's share (the sequential fallback
sum is header_kernel; whole-call times up to a pass are dominated by the call's fixed costs), the
prune's BFS levels, and the oracle on one core for the same frames.  The card's name and power limit are read in
the same run.

    python tools/time_ground.py [--out profiles/h100_ground.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import __graft_entry__ as graft  # noqa: E402
from oracle import ground as og  # noqa: E402
from tests import ground_scenes as gs  # noqa: E402

ob = graft.load_package()


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def device_frame(f, normals):
    dev = torch.device("cuda", 0)
    return {"lut": ob.core.XYZLutT.from_arrays(f["direction"], f["offset"], f["h"], f["w"]),
            "ranges": [torch.from_numpy(r.view(np.int32)).to(dev) for r in f["ranges"]],
            "status": torch.from_numpy(f["status"].view(np.int32)).to(dev),
            "poses": torch.from_numpy(f["poses"]).to(dev),
            "normals": torch.from_numpy(normals[0]).to(dev), "normals2": torch.from_numpy(normals[1]).to(dev)}


def kernel_times(frames):
    from torch.profiler import ProfilerActivity, profile
    ob.core.ground_mask(frames)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ob.core.ground_mask(frames)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if ev.device_time_total > 0:
            m = re.search(r"(\w+_kernel)", ev.key)
            name = m.group(1) if m else ev.key[:60]
            out[name] = round(out.get(name, 0.0) + ev.device_time_total / 1000.0, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_ground.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_ground.py needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "unavailable",
           "method": "CUDA events around whole ob_ground_mask calls (device buffers), 3 warm-up + 50 timed calls (5 for the 16-frame set)",
           "cases": {}}
    for name in ("box_rooftop", "room"):
        f = gs.make_frame(name, h=128, w=2048, dual=True)
        nrm = [x.astype(np.float32) for x in og.computed_normals(f["ranges"], f["direction"], f["offset"],
                                                                 f["poses"], f["sensor_to_body"])]
        d = device_frame(f, nrm)
        case = {"call_ms": round(timeit(lambda: ob.core.ground_mask([d]), n=50), 4)}
        dn = {k: v for k, v in d.items() if k not in ("normals", "normals2")}
        dn["sensor_to_body"] = f["sensor_to_body"]
        case["call_computed_normals_ms"] = round(timeit(lambda: ob.core.ground_mask([dn]), n=50), 4)
        gn = ob.core.ground_mask([dn])[0]
        own = og.run(f["ranges"], f["status"], f["direction"], f["offset"], f["poses"],
                     og.computed_normals(f["ranges"], f["direction"], f["offset"], f["poses"], f["sensor_to_body"]))[0]
        case["computed_normals_pixels_differing_from_oracle_own_subtent"] = int(
            sum(int((m.cpu().numpy() != w).sum()) for m, w in zip(gn["masks"], own)))
        got = ob.core.ground_mask([d], model=True)[0]
        case["grid"] = [got["model"]["rows"], got["model"]["cols"]]
        case["prune_bfs_levels"] = got["prune_levels"]
        case["kernel_ms"] = kernel_times([d])
        want = og.run(f["ranges"], f["status"], f["direction"], f["offset"], f["poses"],
                      [x.astype(np.float64) for x in nrm])[0]
        case["masks_equal_oracle"] = all(np.array_equal(m.cpu().numpy(), w) for m, w in zip(got["masks"], want))
        t0 = time.perf_counter()
        for _ in range(3):
            og.run(f["ranges"], f["status"], f["direction"], f["offset"], f["poses"],
                   [x.astype(np.float64) for x in nrm])
        # og.run calls orc_ground_run twice (once for the grid shape): half its time is one oracle run
        case["oracle_one_core_ms"] = round((time.perf_counter() - t0) / 3 / 2 * 1000.0, 2)
        res["cases"][name + "_128x2048_dual"] = case
        if name == "box_rooftop":
            frames16 = [d] * 16
    t = timeit(lambda: ob.core.ground_mask(frames16), n=5)
    res["cases"]["box_rooftop_16_frames"] = {"call_ms": round(t, 4), "per_frame_ms": round(t / 16, 4),
                                             "kernel_ms": kernel_times(frames16)}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    json.dump(res, open(args.out, "w"), indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
