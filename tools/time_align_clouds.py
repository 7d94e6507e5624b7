#!/usr/bin/env python
"""Global cloud alignment (ob_align_clouds) on the GPU: whole calls timed with CUDA events after a warm-up, device
buffers, for a pair of 128x2048 scans of the `open` scene of tests/align_scenes.py (source yawed 137 degrees and
moved), without and with normals; the CUDA-event split of a traced call into features, pass 1, pass 2, ICP and
confidence; and the oracle on one core for the same pair.  The card's name and power limit are read in the same run.

    python tools/time_align_clouds.py [--out profiles/h100_align_clouds.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import __graft_entry__ as graft  # noqa: E402
from oracle import align_clouds as oac  # noqa: E402
from tests import align_scenes as A  # noqa: E402

ob = graft.load_package()
STAGES = ("features", "pass1", "pass2", "icp", "confidence")


def timeit(fn, n=20):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_align_clouds.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_align_clouds.py needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else "unavailable",
           "method": "CUDA events around whole ob_align_clouds calls (device inputs and outputs), 3 warm-up + 20 "
                     "timed calls; stage split: median of 5 traced calls (CUDA events inside the call); oracle: one "
                     "call on one core",
           "cases": {}}
    truth = A.pose(137.0, (-2.0, 1.5, 0.2))
    sp, sn, tp, tn = A.pair("open", truth, 128, 2048)
    dev = [torch.as_tensor(a, device="cuda") for a in (sp, tp, sn, tn)]
    for normals in (False, True):
        args_dev = dev if normals else dev[:2]
        case = {"source_rows": len(sp), "target_rows": len(tp)}
        case["call_ms"] = round(timeit(lambda: ob.core.align_clouds(*args_dev, compute_confidence=True)), 3)
        traces = [ob.core.align_clouds(*args_dev, compute_confidence=True, trace=True)[2] for _ in range(5)]
        split = np.median(np.array([t["stage_ms"] for t in traces]), axis=0)
        case["stage_ms"] = {k: round(float(v), 3) for k, v in zip(STAGES, split)}
        tr = traces[0]
        case["features"] = [int(tr["source_features"]), int(tr["target_features"])]
        case["grid"] = {"bound_m": tr["bound_m"], "fine": [tr["fine_base_n"], tr["fine_fft_n"]],
                        "coarse": [tr["coarse_base_n"], tr["coarse_fft_n"]]}
        pose, conf = ob.core.align_clouds(sp, tp, sn if normals else None, tn if normals else None,
                                          compute_confidence=True)
        e_t, e_r = A.pose_error(pose, truth)
        case["error_vs_truth"] = {"m": round(e_t, 5), "deg": round(e_r, 5), "confidence": round(conf, 4)}
        t0 = time.perf_counter()
        o, _, _ = oac.align_clouds(sp, tp, None, sn if normals else None, tn if normals else None)
        case["oracle_one_core_ms"] = round((time.perf_counter() - t0) * 1000.0, 1)
        case["max_pose_difference_from_oracle"] = float(np.abs(o - pose).max())
        res["cases"]["open_128x2048" + ("_normals" if normals else "_points")] = case
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    json.dump(res, open(args.out, "w"), indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
