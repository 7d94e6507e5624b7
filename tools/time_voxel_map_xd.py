#!/usr/bin/env python
"""The voxel map with per-point attributes (VoxelHashMapXd, DESIGN f-11) on the GPU: the map exporter's loop on a
128x2048 dual-return room scene with 3 attribute columns (REFLECTIVITY uint16, SIGNAL uint32, NEAR_IR float32) --
map_rows (range -> dewarped rows with attributes, both returns in one launch, device count) -> add_points (device
count) -- on a map warmed with 20 frames; an extract after a move; align_points_to_map on the attribute map against
the 3-d map with the same x, y, z.  CUDA-event ms per call, and the one-core CPU time of the same step beside each:
the exporter's numpy step (oracle cartesian + dewarp + indexing + concatenate) and the plain-Python VoxelHashMapXd
statement for map and extract (tests/voxel_map_xd_reference.py, a Python port, marked as such), the registration
oracle (oracle/orc_icp.c) for ICP.  Writes h100_voxel_map_xd.json into --out (default: a directory under the system
temporary directory) with the card's name and power limit read in the same run.

With --parent-tree DIR (a built checkout of the commit to compare with, e.g. `git worktree add DIR HEAD~1` and
`python DIR/ouster-sdk_b200/build.py`), the same run also times the 3-d map: tools/time_icp.py of DIR and of this tree,
alternately, --icp-rounds times each with the same --reps, into the section `icp_3d_map_parent_vs_change_ms`.

    python tools/time_voxel_map_xd.py [--reps 20] [--out DIR] [--parent-tree DIR [--icp-rounds 2]]
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
from tests import voxel_map_xd_reference as xr  # noqa: E402
from tests.test_oracle_normals import room_scene  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ouster_b200_profiles"))
ap.add_argument("--parent-tree", default=None)
ap.add_argument("--icp-rounds", type=int, default=2)
args = ap.parse_args()
ob = graft.load_package()
if ob.device_count() == 0:
    sys.exit("time_voxel_map_xd.py needs a CUDA device")
dev = torch.device("cuda", 0)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()[0]
H, W = 128, 2048
VS, MAX_DIST, MAX_PTS = 0.5, 100.0, 20
out = {"gpu": gpu, "reps": args.reps, "cases": {},
       "input": f"{H}x{W} room scene, dual return (15 % zero range each), per-column poses of a known motion, fields "
                "uint16 + uint32 + float32 (3 attribute columns; on the device the unsigned ones sit in int16 / "
                "int32 tensors as a DeviceLidarScan holds them, with their types stated); map voxel 0.5 m, 20 points "
                "per voxel"}
ST = ob.Stream(0, cuda_stream=torch.cuda.current_stream(dev).cuda_stream)


def event_ms(fn, reps):
    for _ in range(2):
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


_, RNG, D = room_scene(H, W)
LUT_D = np.ascontiguousarray(D.reshape(-1, 3)) * 0.001     # range in mm, XYZ in metres
LUT_O = np.zeros_like(LUT_D)
lut = ob.XYZLutT.from_arrays(LUT_D, LUT_O, H, W)
step = np.eye(4)
step[:3, :3] = Rotation.from_rotvec(np.radians([0.0, 0.0, 0.8])).as_matrix()
step[:3, 3] = [0.3, 0.1, 0.0]


def frame(k):
    rs = np.random.default_rng(k)
    base = np.linalg.matrix_power(step, k)
    poses = np.repeat(base[None], W, 0)
    poses[:, 0, 3] += np.linspace(0, 0.05, W)            # motion within the sweep
    items = []
    for r in range(2):
        rg = (RNG.astype(np.int64) + rs.integers(-30, 31, RNG.shape) + 500 * r).astype(np.uint32)
        rg[rs.random(RNG.shape) < 0.15] = 0
        fields = [rs.integers(0, 65535, (H, W)).astype(np.uint16), rs.integers(0, 1 << 20, (H, W)).astype(np.uint32),
                  rs.normal(0, 100.0, (H, W)).astype(np.float32)]
        items.append({"range": rg, "poses": poses, "fields": fields, "direction": LUT_D, "offset": LUT_O})
    return items


SIGNED = {np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32}


def device_items(items):
    """the frame's images on the device as a DeviceLidarScan holds them: unsigned fields in signed tensors of the
    same width, passed with their types"""
    return [{"lut": lut, "range": torch.from_numpy(it["range"].view(np.int32)).to(dev),
             "poses": torch.from_numpy(it["poses"]).to(dev),
             "fields": [(torch.from_numpy(f.view(SIGNED[f.dtype])).to(dev), f.dtype) if f.dtype in SIGNED
                        else torch.from_numpy(f).to(dev) for f in it["fields"]]}
            for it in items]


# warm map: 20 frames, GPU and the Python statement side by side (the latter only for the first: a Python loop)
gm = ob.VoxelMap(VS, MAX_DIST, MAX_PTS, num_attributes=3)
xm = xr.VoxelHashMapXd(VS, MAX_DIST, MAX_PTS, num_attributes=3)
ref_ms = {"map_rows": [], "add": []}
for k in range(1, 21):
    its = frame(k)
    rows, n = ob.map_rows(device_items(its), stream=ST)
    gm.add_points(rows, n=n, stream=ST)
    if k == 1:
        t_rows, hrows = cpu_ms(lambda: xr.map_rows(its))
        t_add, _ = cpu_ms(lambda: xm.add_points(hrows))
        ref_ms["map_rows"].append(t_rows)
        ref_ms["add"].append(t_add)
        out["warm_map_matches_python_statement_after_1_frame"] = bool(
            np.array_equal(gm.point_cloud(), xm.point_cloud()))
torch.cuda.synchronize()
out["warm_map"] = {"frames": 20, "voxels": gm.size()[0], "points": gm.size()[1]}

its = frame(21)
ditems = device_items(its)
res = {}
mr_ms = event_ms(lambda: res.update(r=ob.map_rows(ditems, stream=ST)), args.reps)
rows, n = res["r"]
n_rows = int(n.item())


def add_once():
    m = ob.VoxelMap(VS, MAX_DIST, MAX_PTS, num_attributes=3)
    m.add_points(gm.point_cloud(device=True), stream=ST)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    r, c = ob.map_rows(ditems, stream=ST)
    m.add_points(r, n=c, stream=ST)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


both = sorted(add_once() for _ in range(max(5, args.reps // 2)))
out["cases"]["map_rows"] = {"rows": n_rows, "cols": int(rows.shape[1]), "gpu_ms": mr_ms,
                            "cpu_ms_exporter_numpy_step": float(np.median(ref_ms["map_rows"]))}
out["cases"]["map_rows_plus_add_points_per_frame"] = {
    "rows": n_rows, "gpu_ms_median": both[len(both) // 2],
    "cpu_ms_python_statement_add_points": float(np.median(ref_ms["add"])),
    "cpu_note": "the CPU add figure is a pure-Python statement (one core), not the reference's C++ map"}

# extract after a move: voxels beyond max_distance of a far origin
far = np.array([150.0, 0.0, 0.0])
ext_ms = []
for _ in range(5):
    m = ob.VoxelMap(VS, MAX_DIST, MAX_PTS, num_attributes=3)
    m.add_points(gm.point_cloud(device=True), stream=ST)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e = m.remove_far(far, extract=True, stream=ST)
    ext_ms.append((time.perf_counter() - t0) * 1e3)
x2 = xr.VoxelHashMapXd(VS, MAX_DIST, MAX_PTS, num_attributes=3)
x2.add_points(gm.point_cloud())
t_x, xe = cpu_ms(lambda: x2.extract_voxels_far_from_location(far))
out["cases"]["extract_after_move"] = {
    "rows_extracted": int(len(e)), "map_points": gm.size()[1], "gpu_call_ms_median_incl_host_copy": sorted(ext_ms)[2],
    "cpu_ms_python_statement": t_x, "matches_python_statement": bool(np.array_equal(e, xe)),
    "cpu_note": "the CPU figure is a pure-Python statement (one core), not the reference's C++ map"}

# ICP on the attribute map against the 3-d map with the same x, y, z
pc = gm.point_cloud()
g3 = ob.VoxelMap(VS, MAX_DIST, MAX_PTS)
g3.add_points(np.ascontiguousarray(pc[:, :3]))
hrows = rows[:n_rows].cpu().numpy()
src0, _ = orv.voxel_downsample(np.ascontiguousarray(hrows[:, :3]), 1.5)
src = torch.from_numpy(src0).to(dev)
res = {}
xd_ms = event_ms(lambda: res.update(r=ob.icp_align(gm, src, 3.0, 1.0, 50, stream=ST)), args.reps)
px, itx = res["r"]
d3_ms = event_ms(lambda: res.update(r=ob.icp_align(g3, src, 3.0, 1.0, 50, stream=ST)), args.reps)
p3, it3 = res["r"]
om = oi.VoxelHashMap3d(VS, MAX_DIST, MAX_PTS)
om.add_points(np.ascontiguousarray(pc[:, :3]))
t_o, (wp, wit) = cpu_ms(lambda: oi.align_points_to_map(src0, om, 3.0, 1.0, 50))
out["cases"]["align_points_to_map"] = {
    "source_points": int(src.shape[0]), "iterations_xd": int(itx.item()), "iterations_3d": int(it3.item()),
    "oracle_iterations": wit, "gpu_ms_xd_map": xd_ms, "gpu_ms_3d_map": d3_ms, "oracle_ms": t_o,
    "xd_pose_equals_3d_pose": bool(torch.equal(px, p3)),
    "max_abs_pose_diff_vs_oracle": float(np.abs(px.cpu().numpy() - wp).max())}
os.makedirs(args.out, exist_ok=True)
if args.parent_tree:
    # the 3-d map before and after: tools/time_icp.py of both trees, alternately, same reps, same card
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cases = ("align_points_to_map", "add_points", "remove_voxels_far_from_location", "slam_step", "closest_frame",
             "closest_source", "closest_30k")
    ab = {c: {"parent": [], "change": []} for c in cases}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.icp_rounds):
            for side, tree in (("parent", os.path.abspath(args.parent_tree)), ("change", here)):
                od = os.path.join(tmp, f"{side}_{r}")
                subprocess.run([sys.executable, os.path.join(tree, "tools", "time_icp.py"), "--reps", str(args.reps),
                                "--out", od], cwd=tree, check=True, capture_output=True)
                got = json.load(open(os.path.join(od, "h100_icp.json")))["cases"]
                for c in cases:
                    ab[c][side].append(round(got[c].get("gpu_ms", got[c].get("gpu_ms_median")), 4))
    out["icp_3d_map_parent_vs_change_ms"] = {
        "tool": f"tools/time_icp.py --reps {args.reps} of the parent tree and of this tree, alternately, "
                f"{args.icp_rounds} rounds, in this run", "cases": ab}
path = os.path.join(args.out, "h100_voxel_map_xd.json")
with open(path, "w") as fh:
    json.dump(out, fh, indent=1)
print(json.dumps(out, indent=1))
print("wrote", path)
