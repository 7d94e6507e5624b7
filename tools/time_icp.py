#!/usr/bin/env python
"""Frame-to-map registration (ob_voxel_map / ob_icp_align) on the GPU: a SLAM chain on the 128x2048 room scene with a
known per-frame motion -- 2x voxel_downsample (device counts) -> align_points_to_map (device pose) -> transform +
add_points -> cull, the order of lio_slam.cpp:155-231 -- after a map warmed up with 20 frames.  Reports CUDA-event
ms for add_points per frame, closest-neighbour queries per second for the ICP source and a full 262 k-point frame, align_points_to_map per
call and per iteration (with the source size and iteration count), and the one-core oracle (oracle/orc_icp.c) for the
same work beside each figure, plus whether the GPU result equals the oracle's.  The input cloud is already in the
sensor frame: dewarping is timed by tools/time_voxel.py and not repeated here.  Writes h100_icp.json into --out
(default: a directory under the system temporary directory) with the card's name and power limit read in the same run.

    python tools/time_icp.py [--reps 20] [--out DIR]
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
from scipy.spatial.transform import Rotation  # noqa: E402

import __graft_entry__ as graft  # noqa: E402
from oracle import icp as oi  # noqa: E402
from oracle import voxel as orv  # noqa: E402
from tests.test_gpu_icp import scene  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ouster_b200_profiles"))
args = ap.parse_args()
ob = graft.load_package()
if ob.device_count() == 0:
    sys.exit("time_icp.py needs a CUDA device")
dev = torch.device("cuda", 0)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()[0]
out = {"gpu": gpu, "reps": args.reps, "cases": {},
       "input": "128x2048 room scene moved by a known per-frame motion, generated directly in the sensor frame: the "
                "dewarp step is not part of this workload (tools/time_voxel.py times dewarp + downsampling)"}

VS, MAX_DIST, MAX_PTS = 1.0, 100.0, 20          # lio_slam voxel size 1 m: passes at 0.5 and 1.5 m
ICP_DIST, KERNEL = 3.0, 1.0
ST = ob.Stream(0, cuda_stream=torch.cuda.current_stream(dev).cuda_stream)


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


def cpu_ms(fn):
    t0 = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t0) * 1e3, r


cloud = scene()
step = np.eye(4)
step[:3, :3] = Rotation.from_rotvec(np.radians([0.1, -0.2, 0.9])).as_matrix()
step[:3, 3] = [0.05, 0.02, 0.0]


def frame_at(k):
    world = np.linalg.matrix_power(step, k)
    inv = np.linalg.inv(world)
    return (inv[:3, :3] @ cloud.T).T + inv[:3, 3]


def slam_step(m, frame_dev, n):
    p1, _, c1 = ob.voxel_downsample(frame_dev, 0.5 * VS, n=n, stream=ST)
    p2, _, c2 = ob.voxel_downsample(p1, 1.5 * VS, n=c1, stream=ST)
    pose, it = ob.icp_align(m, p2, ICP_DIST, KERNEL, 50, n=c2, stream=ST)
    m.add_points(ob.transform(p1, pose, stream=ST), n=c1, stream=ST)
    m.remove_far(pose[:3, 3].contiguous(), stream=ST)
    return p1, c1, p2, c2, pose, it


# warm map: 20 frames through the whole chain, GPU map and oracle map side by side
gm, om = ob.VoxelMap(VS, MAX_DIST, MAX_PTS), oi.VoxelHashMap3d(VS, MAX_DIST, MAX_PTS)
n_rows = torch.tensor([cloud.shape[0]], dtype=torch.int64, device=dev)
orc_ms = {"add": [], "align": []}
for k in range(1, 21):
    f = frame_at(k)
    p1, c1, p2, c2, pose, it = slam_step(gm, torch.from_numpy(f).to(dev), n_rows)
    o1, _ = orv.voxel_downsample(f, 0.5 * VS)
    o2, _ = orv.voxel_downsample(o1, 1.5 * VS)
    t_al, (opose, oit) = cpu_ms(lambda: oi.align_points_to_map(o2, om, ICP_DIST, KERNEL, 50))
    moved = (opose[:3, :3] @ o1.T).T + opose[:3, 3]
    t_add, _ = cpu_ms(lambda: om.add_points(moved))
    om.remove_voxels_far_from_location(opose[:3, 3])
    orc_ms["align"].append((t_al, oit))
    orc_ms["add"].append(t_add)
torch.cuda.synchronize()
out["warm_map"] = {"frames": 20, "voxels": gm.size()[0], "points": gm.size()[1],
                   "oracle_voxels": om.size()[0], "oracle_points": om.size()[1]}
out["chain_pose_max_abs_diff_vs_oracle"] = float(np.abs(pose.cpu().numpy() - opose).max())

# the next frame's inputs
f = frame_at(21)
fd = torch.from_numpy(f).to(dev)
p1, _, c1 = ob.voxel_downsample(fd, 0.5 * VS, n=n_rows, stream=ST)
p2, _, c2 = ob.voxel_downsample(p1, 1.5 * VS, n=c1, stream=ST)
torch.cuda.synchronize()
k1, k2 = int(c1.item()), int(c2.item())
src = p2[:k2].contiguous()
fine = p1[:k1].contiguous()

# the oracle's copy of the GPU map: re-inserting the stored points in creation order rebuilds the same buckets, so the
# per-call comparisons below run both sides on one map
oc = oi.VoxelHashMap3d(VS, MAX_DIST, MAX_PTS)
oc.add_points(gm.point_cloud())

# align_points_to_map on the warm map (device pose: no host wait)
res = {}
al_ms = event_ms(lambda: res.update(r=ob.icp_align(gm, src, ICP_DIST, KERNEL, 50, stream=ST)), args.reps)
g_pose, g_it = res["r"]
iters = int(g_it.item())
o_src = src.cpu().numpy()
t_o, (o_pose, o_it) = cpu_ms(lambda: oi.align_points_to_map(o_src, oc, ICP_DIST, KERNEL, 50))
out["cases"]["align_points_to_map"] = {
    "source_points": k2, "iterations": iters, "oracle_iterations": o_it, "gpu_ms": al_ms,
    "gpu_ms_per_iteration": al_ms / max(iters, 1), "oracle_ms": t_o, "oracle_ms_per_iteration": t_o / max(o_it, 1),
    "max_abs_pose_diff_vs_oracle": float(np.abs(g_pose.cpu().numpy() - o_pose).max())}
# 1 iteration; 500 (the reference's SLAM default, slam_engine.h:25) with the default criterion 1e-4, where the
# iterations after convergence are launches that return at once; and 500 with criterion 1e-12
for it_max, crit in ((1, 1e-4), (500, 1e-4), (500, 1e-12)):
    res = {}
    ms = event_ms(lambda: res.update(r=ob.icp_align(gm, src, ICP_DIST, KERNEL, it_max, crit, stream=ST)),
                  max(2, args.reps // 4))
    out["cases"][f"align_max_iterations_{it_max}_criterion_{crit:g}"] = {
        "source_points": k2, "gpu_ms": ms, "iterations_run": int(res["r"][1].item())}

# closest-neighbour queries
# the ICP source, ~30 k rows of the fine cloud, and a full 128x2048 frame
for nq, q in (("source", src), ("30k", fine[:30000].contiguous()), ("frame", fd)):
    qn = int(q.shape[0])
    ms = event_ms(lambda: gm.closest_neighbors(q, stream=ST), args.reps)
    nb, d2 = gm.closest_neighbors(q, stream=ST)
    torch.cuda.synchronize()
    qh = q.cpu().numpy()
    sub = qh[:: max(1, qn // 20000)]
    t_o, (wnb, wd2) = cpu_ms(lambda: oc.get_closest_neighbors(sub))
    gnb, gd2 = gm.closest_neighbors(sub)
    out["cases"][f"closest_{nq}"] = {
        "queries": qn, "gpu_ms": ms, "gpu_queries_per_s": qn / ms * 1e3,
        "oracle_queries_per_s": len(sub) / t_o * 1e3, "oracle_sampled_queries": len(sub),
        "bit_exact_on_sample": bool(np.array_equal(gnb, wnb) and np.array_equal(gd2, wd2))}

# add_points per frame: the fine cloud of the next frame into a copy of the warm state each time
moved = ob.transform(fine, g_pose, stream=ST)


def add_once():
    m = ob.VoxelMap(VS, MAX_DIST, MAX_PTS)
    m.add_points(gm.point_cloud(device=True), stream=ST)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    m.add_points(moved, stream=ST)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


add_ms = sorted(add_once() for _ in range(max(5, args.reps // 2)))
out["cases"]["add_points"] = {"rows": k1, "gpu_ms_median": add_ms[len(add_ms) // 2],
                              "oracle_ms_median_warmup_frames": float(np.median(orc_ms["add"]))}
# the same rows through the device-count path on the warm map itself (row capacity 128x2048): this is the call
# that reads the counters when the host bound says the table might have to grow
dev_moved = torch.zeros((cloud.shape[0], 3), dtype=torch.float64, device=dev)
dev_moved[:k1] = moved
c_fine = torch.tensor([k1], dtype=torch.int64, device=dev)
dev_add_ms = []
for _ in range(5):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    gm.add_points(dev_moved, n=c_fine, stream=ST)
    e1.record()
    torch.cuda.synchronize()
    dev_add_ms.append((e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3))
out["cases"]["add_points_device_count_warm_map"] = {
    "rows": k1, "row_capacity": int(cloud.shape[0]), "gpu_ms": [round(a, 4) for a, _ in dev_add_ms],
    "host_ms": [round(b, 4) for _, b in dev_add_ms],
    "note": "re-adds the same rows, so the voxels exist; host_ms includes any counter read the growth check makes"}
cull_ms = event_ms(lambda: gm.remove_far(g_pose[:3, 3].contiguous(), stream=ST), args.reps)
out["cases"]["remove_voxels_far_from_location"] = {"gpu_ms": cull_ms}
out["cases"]["slam_step"] = {"gpu_ms": event_ms(lambda: slam_step(gm, fd, n_rows), max(2, args.reps // 4)),
                             "steps": "2x voxel_downsample + align + transform + add_points + cull"}
out["oracle_align_ms_warmup_frames"] = [round(t, 3) for t, _ in orc_ms["align"]]
os.makedirs(args.out, exist_ok=True)
path = os.path.join(args.out, "h100_icp.json")
with open(path, "w") as fh:
    json.dump(out, fh, indent=1)
print(json.dumps(out, indent=1))
print("wrote", path)
