#!/usr/bin/env python
"""Image post-processing on the GPU (ob_image_proc_update) at 128x2048: AutoExposure on mono, RGB and float16 RGB,
BeamUniformityCorrector on mono and LocalToneMapper on RGB and float16 RGB, float32, on device images updated in
place on the torch stream.  AE and LTM run with update_every = 1 (every update selects its order statistics, the
costly case); BUC keeps its fixed every-8th-frame recompute, and its figure is the mean over whole 8-frame cycles.
Reports CUDA-event ms per update (for the in-place cases including a device copy of the input, timed on its own
beside it) and the launches of one update, beside the one-core oracle (oracle/orc_image.c) on the same input, and writes
h100_image.json into --out (default: a directory under the system temporary directory) with the card's name and
power limit read in the same run.

    python tools/time_image.py [--reps 64] [--out DIR]
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
from oracle import image as oi  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=64)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ouster_b200_profiles"))
args = ap.parse_args()
ob = graft.load_package()
if ob.device_count() == 0:
    sys.exit("time_image.py needs a CUDA device")
dev = torch.device("cuda", 0)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()[0]
H, W = 128, 2048
r = np.random.default_rng(0)
mono = r.uniform(0, 4000, (H, W)).astype(np.float32) + np.linspace(0, 300, H, dtype=np.float32)[:, None]
mono[r.random((H, W)) < 0.1] = 0
rgb = r.uniform(0, 1.5, (H, W, 3)).astype(np.float32)
half = rgb.astype(np.float16)
out = {"gpu": gpu, "reps": args.reps, "shape": [H, W], "dtype": "float32", "cases": {},
       "input": "uniform values with 10 % zeros (mono, plus a row ramp) or uniform RGB in [0, 1.5)"}


def event_ms(fn, reps):
    for _ in range(8):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def oracle_ms(make, img, reps=4):
    o = make()
    t = 0.0
    for _ in range(reps):
        x = img.copy()
        t0 = time.perf_counter()
        o.update(x)
        t += time.perf_counter() - t0
    return t / reps * 1e3


cases = [("auto_exposure_mono", "auto_exposure", mono, lambda: oi.AutoExposure(0.1, 0.1, 1, 0.9)),
         ("auto_exposure_rgb", "auto_exposure", rgb, lambda: oi.AutoExposure(0.1, 0.1, 1, 0.9)),
         ("auto_exposure_rgb_f16", "auto_exposure", half, lambda: oi.AutoExposure(0.1, 0.1, 1, 0.9)),
         ("beam_uniformity_mono", "beam_uniformity", mono, oi.BeamUniformityCorrector),
         ("local_tone_map_rgb", "local_tone_map", rgb, oi.LocalToneMapper),
         ("local_tone_map_rgb_f16", "local_tone_map", half, oi.LocalToneMapper)]
for name, kind, host, make in cases:
    kw = {} if kind == "beam_uniformity" else {"update_every": 1}
    proc = ob.ImageProcessor(kind, **kw)
    src = torch.from_numpy(host.copy()).to(dev)
    x = src.clone()
    if host.dtype == np.float16:
        res = torch.empty(x.shape, dtype=torch.float32, device=dev)
        fn = lambda: proc.update(src, out=res)
        copy = None
    else:
        copy = lambda: x.copy_(src)  # every update sees the same input, not its own previous output

        def fn():
            copy()
            proc.update(x)
    launches0 = ob.kernel_launch_count("image")
    fn()
    torch.cuda.synchronize()
    launches = ob.kernel_launch_count("image") - launches0
    reps = max(8, args.reps // 8 * 8)
    rec = {"gpu_ms_per_update": event_ms(fn, reps), "launches_per_update": launches,
           "oracle_one_core_ms_per_update": oracle_ms(make, host)}
    if copy is not None:
        rec["included_input_copy_ms"] = event_ms(copy, reps)
    out["cases"][name] = rec
    print(name, json.dumps(rec), flush=True)
os.makedirs(args.out, exist_ok=True)
with open(os.path.join(args.out, "h100_image.json"), "w") as f:
    json.dump(out, f, indent=1)
print("wrote", os.path.join(args.out, "h100_image.json"))
