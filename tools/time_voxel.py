#!/usr/bin/env python
"""Voxel-grid downsampling (ob_voxel_downsample) on the GPU: CUDA-event ms per call and Mpoints/s for every mode
on the 128x2048 room scene, the SLAM two-pass chain on a dewarped FrameSet (device-side counts, lio_slam.cpp:140-160),
and the worst case of one voxel holding 90 % of the points; the oracle's one-core CPU time beside each (kind
"port": it restates the reference's sequential hash-map loop in C), and whether the GPU result equals the oracle's.
Writes h100_voxel.json into --out (default: a directory under the system temporary directory) with the card's
name and power limit read in the same run.

    python tools/time_voxel.py [--reps 20] [--out DIR]
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
from oracle import oracle as orc  # noqa: E402
from oracle import voxel as orv  # noqa: E402
from tests.helpers import random_lut, random_range  # noqa: E402
from tests.test_gpu_dewarp import _random_poses  # noqa: E402
from tests.test_gpu_voxel import STRATEGY, dense_cloud, scene_points  # noqa: E402
from tests.test_oracle_normals import room_scene  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ouster_b200_profiles"))
args = ap.parse_args()
ob = graft.load_package()
dev = torch.device("cuda", 0)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()[0]
out = {"gpu": gpu, "reps": args.reps, "cases": {}}


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


def record(name, n_in, fn_gpu, fn_cpu, check):
    ms = event_ms(fn_gpu, args.reps)
    c_ms, want = cpu_ms(fn_cpu)
    rec = {"ms_per_call": ms, "mpoints_s": n_in / ms / 1e3, "points_in": n_in,
           "oracle_cpu_1thread_ms": c_ms, "oracle_kind": "port", "matches_oracle": bool(check(want))}
    out["cases"][name] = rec
    print(name, rec, flush=True)


def same(got, want):
    return all(np.array_equal(g.cpu().numpy().view(np.uint32) if g.dtype == torch.int32 else g.cpu().numpy(), w)
               for g, w in zip(got, want))


st = ob.Stream(0, cuda_stream=torch.cuda.current_stream(dev).cuda_stream)
pts = scene_points()
t_pts = torch.from_numpy(pts).to(dev)
for vs in (0.1, 0.5):
    run = lambda: ob.voxel_downsample(t_pts, vs, stream=st)                                   # noqa: E731
    record(f"shuffle_first_vs{vs}", len(pts), run, lambda: orv.voxel_downsample(pts, vs), lambda w: same(run(), w))
    for mode in ("first_n", "average", "random"):
        run = lambda: ob.voxel_downsample(t_pts, vs, mode, max_points_per_voxel=3, stream=st)  # noqa: E731
        record(f"{mode}_max3_vs{vs}", len(pts), run,
               lambda: orv.voxel_downsample_xd(pts, vs, 3, 1, STRATEGY[mode], with_indices=True),
               lambda w: same(run(), w))
# with normals
h, w = 128, 2048
xyz, rng, _ = room_scene(h, w)
nrm = orc.normals(xyz, rng, sensor_origins_xyz=np.zeros((w, 3))).reshape(-1, 3)
t_xyz, t_nrm = torch.from_numpy(xyz.reshape(-1, 3).copy()).to(dev), torch.from_numpy(nrm).to(dev)
run = lambda: ob.voxel_downsample(t_xyz, 0.5, "point_normal", normals=t_nrm, stream=st)      # noqa: E731
record("point_normal_vs0.5", h * w, run,
       lambda: orv.voxel_downsample_with_normals(xyz.reshape(-1, 3), nrm, 0.5, with_indices=True),
       lambda wnt: same(run(), wnt))
# worst case: one voxel with 90 % of the points, one thread walks it
dc = dense_cloud(h * w)
t_dc = torch.from_numpy(dc).to(dev)
for mode in ("first_n", "average", "random"):
    run = lambda: ob.voxel_downsample(t_dc, 0.5, mode, max_points_per_voxel=8, stream=st)      # noqa: E731
    record(f"dense_voxel_{mode}_max8", len(dc), run,
           lambda: orv.voxel_downsample_xd(dc, 0.5, 8, 1, STRATEGY[mode], with_indices=True), lambda wnt: same(run(), wnt))
run = lambda: ob.voxel_downsample(t_dc, 0.5, stream=st)                                        # noqa: E731
record("dense_voxel_shuffle_first", len(dc), run, lambda: orv.voxel_downsample(dc, 0.5), lambda wnt: same(run(), wnt))

# SLAM chain per FrameSet: dewarp (device count) -> 0.5 vs -> 1.5 vs, vs = 1 m, no host wait inside
capi = ob._capi
import ctypes as C  # noqa: E402
shapes = [(128, 2048)]
frames = (capi.DewarpFramesIO * len(shapes))()
keep, want = [], []
for i, (hh, ww) in enumerate(shapes):
    rg = random_range(hh, ww, 31 + i, p_zero=0.1, max_range=60000)
    d, o = random_lut(hh * ww, 7 + i, np.float64)
    poses = _random_poses(ww, np.float64, 13 + i)
    status = np.ones(ww, np.uint32)
    lut = ob.XYZLutT.from_arrays(d, o, hh, ww)
    t = [torch.from_numpy(a).to(dev) for a in (rg.view(np.int32), poses, status.view(np.int32))]
    keep += t + [lut]
    frames[i].lut, frames[i].range, frames[i].poses, frames[i].status = lut._h, *(x.data_ptr() for x in t)
    want.append(orc.dewarp_frame(rg, d, o, poses, status, np.zeros(ww, np.uint64), 0.5, 45.0)[0])
cap = sum(a * b for a, b in shapes)
dpts = torch.empty((cap, 3), dtype=torch.float64, device=dev)
n_pts = torch.zeros(1, dtype=torch.int64, device=dev)


def chain():
    capi.check(capi.lib.ob_dewarp_frames(frames, len(shapes), 0.5, 45.0, dpts.data_ptr(), cap, None, None, None, None,
                                         C.cast(n_pts.data_ptr(), C.POINTER(C.c_size_t)), st.h))
    p1, i1, c1 = ob.voxel_downsample(dpts, 0.5, n=n_pts, stream=st)
    return p1, i1, c1, ob.voxel_downsample(p1, 1.5, n=c1, stream=st)


def chain_check(ref):
    p1, i1, c1, (p2, i2, c2) = chain()
    torch.cuda.synchronize()
    k1, k2 = int(c1.item()), int(c2.item())
    (w1, wi1), (w2, wi2) = ref
    g1, g2 = i1[:k1].cpu().numpy().view(np.uint32), i2[:k2].cpu().numpy().view(np.uint32)
    return k1 == len(w1) and k2 == len(w2) and np.array_equal(p2[:k2].cpu().numpy(), w2) and \
        np.array_equal(g1[g2], wi1[wi2])


cloud = np.concatenate(want)


def chain_cpu():
    a = orv.voxel_downsample(cloud, 0.5)
    return a, orv.voxel_downsample(a[0], 1.5)


ms_dewarp = event_ms(lambda: capi.check(capi.lib.ob_dewarp_frames(
    frames, len(shapes), 0.5, 45.0, dpts.data_ptr(), cap, None, None, None, None,
    C.cast(n_pts.data_ptr(), C.POINTER(C.c_size_t)), st.h)), args.reps)
record("slam_chain_frameset_128x2048", cap, chain, chain_cpu, chain_check)
out["cases"]["slam_chain_frameset_128x2048"]["dewarp_only_ms"] = ms_dewarp
out["cases"]["slam_chain_frameset_128x2048"]["oracle_cpu_excludes_dewarp"] = True
os.makedirs(args.out, exist_ok=True)
json.dump(out, open(os.path.join(args.out, "h100_voxel.json"), "w"), indent=1)
print("matches_oracle all:", all(c["matches_oracle"] for c in out["cases"].values()))
