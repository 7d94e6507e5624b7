"""Times pose interpolation (DESIGN f-12) on the GPU and writes a profile (profiles/h100_pose.json).

    python tools/time_interp_pose.py --out profiles/h100_pose.json [--reps 50]

Sizes: one 2048-column frame (ob_frames_interp_pose), a 64-frame set of 2048 columns, the reference perf test's
4096 queries over 2 knots (python/tests/test_performance.py:417-438), and 10^6 and 1.6 * 10^7 queries over 1000
knots (ob_interp_pose).  Device inputs, device outputs and a device error word, so no call waits; kernel time is
CUDA events around `reps` back-to-back calls after a warm-up.  For the large sizes, compulsory bytes (x in, 128 B
per pose out) over time against a device-to-device copy peak measured in the same run.  CPU figure: the oracle
(oracle/orc_pose.c) on one core.  Also the largest |gpu - oracle| / max(1, |oracle|) of each size.  The card's name,
power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as graft  # noqa: E402
from oracle import pose as op  # noqa: E402


def gpu_info():
    try:
        q = "name,power.limit,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception as e:  # the timing itself does not depend on it
        return {"error": str(e)}


def events_ms(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def copy_peak_gbs(torch):
    src = torch.empty(1 << 30, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    ms = events_ms(lambda: dst.copy_(src), 20)
    return 2 * src.numel() / (ms * 1e-3) / 1e9


def knot_case(n, m, seed):
    rs = np.random.default_rng(seed)
    k = np.cumsum(rs.random(m) + 0.01)
    pk = [np.eye(4)]
    for _ in range(m - 1):
        ax = rs.normal(size=3)
        pk.append(pk[-1] @ op.posev_exp(np.concatenate([ax / np.linalg.norm(ax) * 0.2, rs.normal(size=3)])))
    return np.sort(rs.uniform(k[0] - 0.5, k[-1] + 0.5, n)), k, np.stack(pk)


def rel_diff(got, want):
    return float(np.max(np.abs(got - want) / np.maximum(1.0, np.abs(want))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    ob = graft.load_package()
    assert ob.device_count() > 0, "this measurement needs a CUDA device"
    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_info(), "reps": args.reps, "copy_peak_gbs": copy_peak_gbs(torch), "entries": []}
    err = torch.zeros(3, dtype=torch.int64, device=dev)
    st = ob.Stream(0, cuda_stream=torch.cuda.current_stream(dev).cuda_stream)
    for name, n, m in (("perf_test_4096_queries", 4096, 2), ("queries_1e6_knots_1000", 10**6, 1000),
                       ("queries_1.6e7_knots_1000", 16 * 10**6, 1000)):
        x, k, pk = knot_case(n, m, n + m)
        dx, dk, dpk = (torch.from_numpy(a).to(dev) for a in (x, k, pk))
        out = torch.empty((n, 4, 4), dtype=torch.float64, device=dev)
        ms = events_ms(lambda: ob.core.interp_pose(dx, dk, dpk, out=out, error=err, stream=st), args.reps)
        t = time.perf_counter()
        want = op.interp_pose(x, k, pk)
        cpu_ms = (time.perf_counter() - t) * 1e3
        e = {"case": name, "n": n, "m": m, "gpu_ms": ms, "cpu_oracle_one_core_ms": cpu_ms,
             "max_rel_diff_vs_oracle": rel_diff(out.cpu().numpy(), want)}
        if n >= 10**6:
            gbs = n * (8 + 128) / (ms * 1e-3) / 1e9
            e.update(compulsory_bytes=n * (8 + 128), achieved_gbs=gbs, frac_of_copy_peak=gbs / res["copy_peak_gbs"])
        res["entries"].append(e)
    for name, n_frames in (("frame_2048_columns", 1), ("frameset_64x2048", 64)):
        w = 2048
        rs = np.random.default_rng(n_frames)
        frames = []
        for f in range(n_frames):
            tsf = (10**18 + (np.arange(w) + f * w) * 48828).astype(np.uint64)
            stf = (rs.random(w) < 0.9).astype(np.uint32)
            frames.append((tsf, stf, np.zeros((w, 4, 4))))
        x0 = np.eye(4)
        x1 = op.posev_exp(np.array([0.0, 0.0, 0.05, 1.0, 0.1, 0.0]))
        t1 = float(frames[-1][0][-1]) * 1e-9
        t0 = t1 - 0.1
        dfr = [(torch.from_numpy(a.view(np.int64)).to(dev), torch.from_numpy(b.view(np.int32)).to(dev),
                torch.from_numpy(c).to(dev)) for a, b, c in frames]
        dx0, dx1 = torch.from_numpy(x0).to(dev), torch.from_numpy(x1).to(dev)
        ms = events_ms(lambda: ob.core.frames_interp_pose(dfr, t0, dx0, t1, dx1, error=err, stream=st), args.reps)
        t = time.perf_counter()
        op.frames_interp_pose(frames, t0, x0, t1, x1)
        cpu_ms = (time.perf_counter() - t) * 1e3
        d = max(rel_diff(g[2].cpu().numpy(), f[2]) for g, f in zip(dfr, frames))
        res["entries"].append({"case": name, "frames": n_frames, "columns": w, "gpu_ms": ms,
                               "cpu_oracle_one_core_ms": cpu_ms, "max_rel_diff_vs_oracle": d})
    torch.cuda.synchronize()
    assert err.cpu().tolist() == [0, 0, 0]
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
