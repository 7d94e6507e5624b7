#!/usr/bin/env python
"""Cloud-to-cloud ICP (ob_cloud_align) on the GPU: point_to_point_align and point_to_plane_align on
  * a room-scene frame pair (tests/test_gpu_align.room_pair at 128x2048) after voxel_downsample_with_normals, and
  * the full 128x2048 pair (262 144 rows a side) without downsampling.
Reports CUDA-event ms per call and per iteration (with the row counts and iteration count), the one-core oracle
(oracle/orc_align.c) for the same call beside each figure and the largest |GPU - oracle| pose entry; then a
torch.profiler run of one call per case, summed by kernel group, to say which step dominates (the 27-cell search in
the association kernel, or the per-iteration median sort).  Writes h100_align.json into --out (default: a
directory under the system temporary directory) with the card's name and power limit read in the same run.

    python tools/time_align.py [--reps 20] [--out DIR]
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
from oracle import align as oa  # noqa: E402
from tests.test_gpu_align import room_pair  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ouster_b200_profiles"))
args = ap.parse_args()
ob = graft.load_package()
if ob.device_count() == 0:
    sys.exit("time_align.py needs a CUDA device")
dev = torch.device("cuda", 0)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()[0]
out = {"gpu": gpu, "reps": args.reps, "cases": {},
       "input": "10 m room scene (tests/test_oracle_normals.room_scene, 128x2048) seen from two poses 1.05 deg and "
                "0.14 m apart, 2 mm point noise, analytic wall normals with 0.01 noise; max_corr_dist 0.5"}
ST = ob.Stream(0, cuda_stream=torch.cuda.current_stream(dev).cuda_stream)
GROUPS = [("association (27-cell search)", "al_assoc"), ("compaction", "al_compact"), ("median sort", "RadixSort"),
          ("sums (leaves)", "al_leaf"), ("tree root + solve", "_solve_kernel"), ("centroid root", "al_centroid"),
          ("grid build", "gr_"), ("grid build", "DeviceScan"), ("init / finish", "al_init"),
          ("init / finish", "al_finish")]


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


def kernel_split(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {}
    for ev in prof.key_averages():
        if ev.device_type.name != "CUDA":
            continue
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = ev.cuda_time_total
        group = next((g for g, key in GROUPS if key in ev.key), "other")
        split[group] = split.get(group, 0.0) + us / 1000.0
    return {k: round(v, 4) for k, v in sorted(split.items(), key=lambda kv: -kv[1])}


def case(name, src, tgt, ns, nt):
    s, t = torch.from_numpy(src).to(dev), torch.from_numpy(tgt).to(dev)
    sn, tn = torch.from_numpy(ns).to(dev), torch.from_numpy(nt).to(dev)
    for mode in ("point_to_point", "point_to_plane"):
        plane = mode == "point_to_plane"
        def call():
            return ob.cloud_align(s, t, sn if plane else None, tn if plane else None, max_corr_dist=0.5, stream=ST)
        ms = event_ms(call, args.reps)
        pose, it = call()
        pose, it = pose.cpu().numpy(), int(it.item())
        t0 = time.perf_counter()
        if plane:
            want, wit = oa.point_to_plane_align(src, tgt, ns, nt, None, 0.5)
        else:
            want, wit = oa.point_to_point_align(src, tgt, None, 0.5)
        oracle_ms = (time.perf_counter() - t0) * 1e3
        out["cases"][f"{name}/{mode}"] = {
            "source_rows": len(src), "target_rows": len(tgt), "iterations": it, "oracle_iterations": wit,
            "gpu_ms_per_call": round(ms, 4), "gpu_ms_per_iteration": round(ms / max(it, 1), 4),
            "oracle_one_core_ms_per_call": round(oracle_ms, 2),
            "oracle_one_core_ms_per_iteration": round(oracle_ms / max(wit, 1), 2),
            "speedup_vs_one_core": round(oracle_ms / ms, 1),
            "max_abs_pose_diff_vs_oracle": float(np.abs(pose - want).max()),
            "gpu_ms_by_kernel_group_one_call": kernel_split(call)}
        print(name, mode, out["cases"][f"{name}/{mode}"], flush=True)


src, tgt, ns, nt, _ = room_pair(128, 2048)
case("full_128x2048", src, tgt, ns, nt)
ds = []
for p, n in ((src, ns), (tgt, nt)):
    pts, nrm, _ = ob.voxel_downsample(p, 0.25, "point_normal", normals=n)
    ds += [pts, nrm]
case("voxel_0.25m_with_normals", ds[0], ds[2], ds[1], ds[3])
os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "h100_align.json")
with open(path, "w") as f:
    json.dump(out, f, indent=1)
print("wrote", path)
