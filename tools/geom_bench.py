"""Geometric-filter throughput, F (7-point) against E (five-point), at bench.py's geom shape: 2000 pairs x 800 putative
matches, 35 % outliers, 1600x1200 views, host arrays in and out.  F and E calls alternate after one warm-up call each;
the card and its power limit are read in the same run.  With oracle/_ref/libref_geom_essential.so present, the
reference E filter is also timed on 200 pairs on one thread.  The oracle's trace on 100 pairs gives the mean number of
AC-RANSAC iterations and of real five-point models per iteration.  --profile adds a torch.profiler pass (device time of
each kernel) in a separate run.

    python tools/geom_bench.py [--calls 5] [--profile]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from openmvg_b200 import geometry, synth  # noqa: E402

PAIRS, MATCHES, WH = 2000, 800, (1600, 1200)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def inputs():
    xs = [synth.calibrated_two_view_matches(MATCHES, 0.35, seed=10_000 + p, wh=WH) for p in range(PAIRS)]
    off = np.arange(PAIRS + 1, dtype=np.uint64) * MATCHES
    xI = np.concatenate([x[0] for x in xs]); xJ = np.concatenate([x[1] for x in xs])
    sz = np.tile(np.array(WH + WH, np.int32), (PAIRS, 1)); intr = np.array([x[3] + x[4] for x in xs])
    return off, xI, xJ, sz, intr


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--calls", type=int, default=5); ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    off, xI, xJ, sz, intr = inputs()
    f_call = lambda: geometry.fundamental_acransac(off, xI, xJ, sz, 4.0, 2048)  # noqa: E731
    e_call = lambda: geometry.essential_acransac(off, xI, xJ, sz, intr, 4.0, 2048)  # noqa: E731
    f_call(); e_res = e_call()
    tf, te = [], []
    for _ in range(a.calls):
        t0 = time.perf_counter(); f_call(); tf.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); e_call(); te.append(time.perf_counter() - t0)
    out = dict(card=card(), pairs=PAIRS, matches_per_pair=MATCHES,
               F_pairs_per_s=[PAIRS / t for t in tf], E_pairs_per_s=[PAIRS / t for t in te],
               E_kept=int(sum(len(r["inliers"]) > 12.5 for r in e_res)))
    import checkers_essential as ce
    tr = [ce.oracle_acransac_essential(xI[MATCHES * p:MATCHES * (p + 1)], xJ[MATCHES * p:MATCHES * (p + 1)], WH + WH, intr[p], 4.0, 2048)["trace"] for p in range(100)]
    it = np.array([t[0] for t in tr], float); mo = np.array([t[1] for t in tr], float)
    out.update(E_mean_iterations=float(it.mean()), E_real_models_per_iteration=float(mo.sum() / it.sum()))
    if os.path.exists(ce.REF_GEOM_E_SO):
        t0 = time.perf_counter()
        for p in range(200):
            ce.ref_acransac_essential.__wrapped__(xI[MATCHES * p:MATCHES * (p + 1)], xJ[MATCHES * p:MATCHES * (p + 1)], WH + WH, intr[p], 4.0, 2048)
        out["E_reference_1thread_pairs_per_s"] = 200 / (time.perf_counter() - t0)
    if a.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            f_call(); e_call()
            torch.cuda.synchronize()
        out["kernel_ms"] = {e.key: e.device_time_total / 1e3 for e in prof.key_averages() if "acransac" in e.key}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
