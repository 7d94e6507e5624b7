#!/usr/bin/env python
"""Frame operations on the GPU (ob_frame_mask_fields, ob_frame_select_rows) at 128x2048 dual return
(RNG19_RFL8_SIG16_NIR16_DUAL, 4 718 592 B of pixel fields per frame): clip, filter_field, filter_uv "u" and "v",
mask, filter_xyz (XYZLutFloat) and reduce_by_factor(2), on DeviceLidarScans of 1 and 32 frames per call.
Reports two CUDA-event times per operation: `call_ms`, the Python call repeated back to back (it includes building
the field table on the host, which bounds a small call), and `device_ms`, the operation's launch replayed from a CUDA
graph after a graph that restores the input (timed alone and subtracted), so every replay changes what the first call
changed.  Beside them: the one-core oracle (oracle/orc_frame_ops.c) on one frame, and the fraction of the copy peak
measured in the same run: bytes read plus the bytes that actually change (as the oracle counts them) over
device_ms, divided by the rate of a device-to-device copy of 32 frames' fields.  Writes h100_frame_ops.json into --out with
the card's name and power limit read in the same run.

    python tools/time_frame_ops.py [--reps 50] [--out DIR]
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
from oracle import frame_ops as ofo  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=50)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ouster_b200_profiles"))
args = ap.parse_args()
ob = graft.load_package()
if ob.device_count() == 0:
    sys.exit("time_frame_ops.py needs a CUDA device")
from ouster_sdk_b200 import pyapi  # noqa: E402

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()[0]
meta = json.load(open(os.path.join(os.path.dirname(__file__), "..", "tests", "golden",
                                   "OS-1-128_767798045_1024x10_20230712_120049.json")))
meta = dict(meta, profile="RNG19_RFL8_SIG16_NIR16_DUAL", w=2048, columns_per_packet=16, column_window=[0, 2047])
info = ob.SensorInfo.from_meta(meta)
H, W = info.h, info.w
rs = np.random.default_rng(0)
host = ob.LidarScan(info)
masks = {f[0]: f[6] for f in info.fields()}
for n in host.fields:
    a = host.field(n)
    a[...] = (rs.integers(0, 1 << 32, size=a.shape, dtype=np.uint64) & np.uint64(masks[n])).astype(a.dtype)
frame_bytes = sum(host.field(n).nbytes for n in host.fields)
lut = pyapi.XYZLutFloat(info)
mask = torch.as_tensor((rs.random((H, W)) < 0.5).astype(np.uint8)).cuda()


def scans(n):
    out = []
    for _ in range(n):
        s = pyapi.DeviceLidarScan(info)
        for k in host.fields:
            a = host.field(k)
            s._fields[k] = torch.from_numpy(a.view({1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[a.itemsize])
                                            .copy()).cuda()
        out.append(s)
    return out


def event_ms(fn, reps):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


fo = ob.frame_ops
ops = {
    "clip": (lambda f: fo.clip(f, [], 1000, 200000, 0), lambda o: ofo.clip(o, [], 1000, 200000, 0)),
    "filter_field": (lambda f: fo.filter_field(f, "RANGE", 0, 100000), lambda o: ofo.filter_field(o, "RANGE", 0, 100000)),
    "filter_uv_u": (lambda f: fo.filter_uv(f, "u", 0, 32), lambda o: ofo.filter_uv(o, "u", 0, 32)),
    "filter_uv_v": (lambda f: fo.filter_uv(f, "v", 0, 512), lambda o: ofo.filter_uv(o, "v", 0, 512, literal=False)),
    "mask": (lambda f: fo.mask(f, [], mask), lambda o: ofo.mask(o, [], mask.cpu().numpy())),
    "filter_xyz": (lambda f: fo.filter_xyz(f, lut, 2, -0.5, 0.5), None),
}
# copy peak: device-to-device copy of 32 frames' fields
big = torch.empty(32 * frame_bytes, dtype=torch.uint8, device="cuda")
big2 = torch.empty_like(big)
copy_ms = event_ms(lambda: big2.copy_(big), args.reps)
copy_rate = 2 * big.numel() / (copy_ms * 1e-3)
out = {"gpu": gpu, "reps": args.reps, "shape": [H, W], "profile": "RNG19_RFL8_SIG16_NIR16_DUAL",
       "frame_bytes": frame_bytes, "copy_peak_GBps": copy_rate / 1e9, "cases": {}}
for name, (g, r) in ops.items():
    # bytes the oracle reads and changes on one frame
    o = ofo.Frame(H, W, info.pixel_shift_by_row)
    for k in host.fields:
        o.add(k, host.field(k).copy(), host.field_tag(k))
    before = {k: o.field(k).copy() for k in o.fields}
    t0 = time.perf_counter()
    if r is not None:
        r(o)
    cpu_ms = (time.perf_counter() - t0) * 1e3 if r is not None else None
    changed = sum(int(np.count_nonzero(before[k] != o.field(k))) * o.field(k).itemsize for k in o.fields) if r else None
    case = {"oracle_one_core_ms": cpu_ms, "changed_bytes_per_frame": changed}
    for n in (1, 32):
        fs, base = scans(n), scans(n)
        arg = fs if n > 1 else fs[0]
        l0 = ob.kernel_launch_count("frame_ops")
        g(arg)
        launches = ob.kernel_launch_count("frame_ops") - l0
        call_ms = event_ms(lambda: g(arg), args.reps)
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            g(arg)
        torch.cuda.current_stream().wait_stream(st)
        g_restore, g_op = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(g_restore, stream=st):
            for a, b in zip(fs, base):
                for k in host.fields:
                    a.field(k).copy_(b.field(k))
        with torch.cuda.graph(g_op, stream=st):
            g(arg)
        restore_ms = event_ms(g_restore.replay, args.reps)
        both_ms = event_ms(lambda: (g_restore.replay(), g_op.replay()), args.reps)
        ms = max(both_ms - restore_ms, 1e-6)
        # filter_xyz reads the range field again for each return, and the float LUT (24 B per pixel, read once per return: 2 x 12 B)
        read = n * frame_bytes + (n * H * W * 2 * 12 if name == "filter_xyz" else 0)
        moved = read + (n * (changed or 0) if changed is not None else 0)
        case[f"{n}_frames"] = {"call_ms": call_ms, "device_ms": ms, "restore_ms": restore_ms, "launches": launches,
                               "GBps": moved / (ms * 1e-3) / 1e9, "fraction_of_copy_peak": moved / (ms * 1e-3) / copy_rate}
        del fs, base, arg, g_restore, g_op
    out["cases"][name] = case
    print(name, json.dumps(case), flush=True)
for n in (1, 32):
    fs = scans(n)
    arg = fs if n > 1 else fs[0]
    ms = event_ms(lambda: fo.reduce_by_factor(arg, 2), max(args.reps // 5, 5))
    out["cases"].setdefault("reduce_by_factor_2", {})[f"{n}_frames"] = {"ms": ms, "note": "includes allocating the result"}
    del fs, arg
print(json.dumps(out["cases"]["reduce_by_factor_2"]))
os.makedirs(args.out, exist_ok=True)
with open(os.path.join(args.out, "h100_frame_ops.json"), "w") as fh:
    json.dump(out, fh, indent=1)
print("gpu:", gpu, "copy peak GB/s:", round(copy_rate / 1e9, 1), "->", os.path.join(args.out, "h100_frame_ops.json"))
