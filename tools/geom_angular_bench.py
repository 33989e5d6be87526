"""Angular essential-matrix filters (`-g a` eight-point, `-g u` upright three-point) against F (7-point) at bench.py's geom
shape: 2000 pairs x 800 putative matches, 35 % outliers, host arrays in and out.  The angular filters run on general
motion of a 360° pair; the upright one also on upright motion (a rotation about y, t_y = 0), the motion its solver
models.  The calls alternate after one warm-up call each; the card and its power limit are read in the same run.  Also reports: the oracle's mean
AC-RANSAC iterations per pair (100 pairs), torch.profiler device time of each kernel for one call of each model, the
compiled reference on 200 pairs on one thread (when oracle/_ref/libref_geom_angular.so is present), and how often the
device's asin differs from glibc's on 10^6 random arguments in [-1, 1] (measured through torch.asin, which calls
CUDA's asin: a proxy for the kernel's own call).

    python tools/geom_angular_bench.py [--calls 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
from openmvg_b200 import geometry, synth  # noqa: E402
from geom_bench import card  # noqa: E402

PAIRS, MATCHES = 2000, 800


def inputs():
    xs = [synth.spherical_two_view_matches(MATCHES, 0.35, seed=20_000 + p, motion="general") for p in range(PAIRS)]
    us = [synth.spherical_two_view_matches(MATCHES, 0.35, seed=30_000 + p, motion="upright") for p in range(PAIRS)]
    fs = [synth.two_view_matches(MATCHES, 0.35, seed=500 + k, wh=(1600, 1200))[:2] for k in range(PAIRS)]
    off = np.arange(PAIRS + 1, dtype=np.uint64) * MATCHES
    return (off, np.concatenate([x[2] for x in xs]), np.concatenate([x[3] for x in xs]),
            np.concatenate([x[2] for x in us]), np.concatenate([x[3] for x in us]),
            np.concatenate([f[0] for f in fs]), np.concatenate([f[1] for f in fs]))


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--calls", type=int, default=5)
    a = ap.parse_args()
    off, bI, bJ, uI, uJ, xI, xJ = inputs()
    sz = np.tile(np.array([1600, 1200, 1600, 1200], np.int32), (PAIRS, 1))
    calls = {"F": lambda: geometry.fundamental_acransac(off, xI, xJ, sz, 4.0, 2048),
             "angular": lambda: geometry.angular_essential_acransac(off, bI, bJ, False, 4.0, 2048),
             "upright": lambda: geometry.angular_essential_acransac(off, bI, bJ, True, 4.0, 2048),
             "upright_on_upright_motion": lambda: geometry.angular_essential_acransac(off, uI, uJ, True, 4.0, 2048)}
    res = {k: f() for k, f in calls.items()}
    t = {k: [] for k in calls}
    for _ in range(a.calls):
        for k, f in calls.items():
            t0 = time.perf_counter(); f(); t[k].append(time.perf_counter() - t0)
    out = dict(card=card(), pairs=PAIRS, matches_per_pair=MATCHES, calls=a.calls)
    for k in calls:
        out[f"{k}_pairs_per_s"] = [round(PAIRS / s, 1) for s in t[k]]
    out["angular_kept"] = int(sum(len(r["inliers"]) > 20 for r in res["angular"]))
    out["upright_kept"] = int(sum(len(r["inliers"]) > 7.5 for r in res["upright"]))
    out["upright_on_upright_motion_kept"] = int(sum(len(r["inliers"]) > 7.5 for r in res["upright_on_upright_motion"]))
    import checkers_angular as ca
    for name, model, b1, b2 in (("angular", ca.ANGULAR, bI, bJ), ("upright", ca.UPRIGHT, bI, bJ), ("upright_on_upright_motion", ca.UPRIGHT, uI, uJ)):
        it = [ca.oracle_angular_acransac(model, b1[MATCHES * p:MATCHES * (p + 1)], b2[MATCHES * p:MATCHES * (p + 1)])["trace"][0] for p in range(100)]
        out[f"{name}_mean_iterations"] = float(np.mean(it))
    import torch
    from torch.profiler import ProfilerActivity, profile
    for k, f in calls.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            f()
        ev = [e for e in prof.key_averages() if e.device_type.name == "CUDA" and "acransac" in e.key]
        out[f"{k}_kernel_ms"] = {e.key[:60]: round(e.device_time_total / 1e3, 3) for e in ev}
    if os.path.exists(ca.REF_GEOM_A_SO):
        for name, model in (("angular", ca.ANGULAR), ("upright", ca.UPRIGHT)):
            t0 = time.perf_counter()
            for p in range(200):
                ca.ref_angular_acransac.__wrapped__(model, bI[MATCHES * p:MATCHES * (p + 1)], bJ[MATCHES * p:MATCHES * (p + 1)], 4.0, 2048)
            out[f"{name}_reference_1thread_pairs_per_s"] = round(200 / (time.perf_counter() - t0), 1)
    x = np.random.default_rng(0).uniform(-1.0, 1.0, 1_000_000)
    dev = torch.asin(torch.from_numpy(x).cuda()).cpu().numpy()
    host = ca.oracle_asin(x)
    ulp = np.abs(dev.view(np.int64) - host.view(np.int64))
    out["asin_differ_of_1e6"] = int((ulp != 0).sum()); out["asin_max_ulp"] = int(ulp.max())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
