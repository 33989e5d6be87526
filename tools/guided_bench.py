"""Guided-matching throughput (omvg_match_guided_run, DESIGN §3.9) at a realistic shape: 64 views x 5000 features at
1600x1200 from one seeded scene (synth.guided_scene), all 2016 pairs.  The models are the fundamental matrices our
AC-RANSAC finds on each pair's putative matches (the true correspondences plus 35 % wrong ones), thresholds
Square(errorMax), ratio Square(0.6); pairs AC-RANSAC does not keep are left out, as the filter leaves them out.
Timed: --calls calls of guided_run + fetch on the resident context after one warm-up call; reported as pairs/s and
candidate tests/s (sum of N_I * N_J over the pairs / time), with the card and power limit read in the same run.
A separate torch.profiler pass gives the guided kernel's device time.  With oracle/_ref/libref_guided.so present, the
reference GuidedMatching is timed on --ref-pairs pairs on one thread.

    python tools/guided_bench.py [--views 64] [--features 5000] [--calls 5] [--ref-pairs 4] [--no-profile]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
os.environ.setdefault("OMP_NUM_THREADS", "1")                  # the reference timing is single-threaded
from openmvg_b200 import geometry, matching, synth  # noqa: E402

WH = (1600, 1200)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def putatives(s, a, b, rng):
    pa, pb = s["point"][a], s["point"][b]
    ib = {p: k for k, p in enumerate(pb) if p >= 0}
    m = np.array([(i, ib[p]) for i, p in enumerate(pa) if p >= 0 and p in ib], np.int64).reshape(-1, 2)
    n_bad = int(0.35 / 0.65 * len(m))
    bad = np.stack([rng.integers(0, len(pa), n_bad), rng.integers(0, len(pb), n_bad)], 1)
    return np.concatenate([m, bad])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=64); ap.add_argument("--features", type=int, default=5000)
    ap.add_argument("--calls", type=int, default=5); ap.add_argument("--ref-pairs", type=int, default=4)
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    s = synth.guided_scene(a.views, a.features, seed=77, wh=WH)
    rng = np.random.default_rng(78)
    pi_all, pj_all = synth.exhaustive_pairs(a.views)
    puts = [putatives(s, int(i), int(j), rng) for i, j in zip(pi_all, pj_all)]
    off = np.concatenate([[0], np.cumsum([len(m) for m in puts])]).astype(np.uint64)
    xI = np.concatenate([s["xy"][int(i)][m[:, 0]] for (i, m) in zip(pi_all, puts)])
    xJ = np.concatenate([s["xy"][int(j)][m[:, 1]] for (j, m) in zip(pj_all, puts)])
    res = geometry.fundamental_acransac(off, xI, xJ, np.tile(np.array(WH + WH, np.int32), (len(puts), 1)), 4.0, 2048)
    keep = [k for k, r in enumerate(res) if len(r["inliers"]) > 2.5 * 7]
    pi, pj = pi_all[keep], pj_all[keep]
    M = np.stack([res[k]["F"] for k in keep]); thr = np.array([res[k]["error_max"] ** 2 for k in keep])
    ratio = 0.6 * 0.6
    ctx = matching.MatchContext(0)
    ctx.load(s["desc"])
    for k, xy in enumerate(s["xy"]):
        ctx.upload_positions(k, xy)
    counts = np.array([len(x) for x in s["xy"]], np.float64)
    tests = float(np.sum(counts[pi] * counts[pj]))

    def call():
        ctx.guided_run(pi, pj, M, thr, ratio, matching.GUIDED_EPIPOLAR)
        return ctx.fetch()

    off_g, ij = call()
    ctx.kernel_time(reset=True)
    times = []
    for _ in range(a.calls):
        t0 = time.perf_counter(); call(); times.append(time.perf_counter() - t0)
    kms, kl = ctx.kernel_time(reset=True)
    out = dict(card=card(), views=a.views, features=a.features, pairs=len(pi), candidate_tests=tests, matches=int(len(ij)),
               mean_threshold_px2=float(thr.mean()), call_s=times, pairs_per_s=[len(pi) / t for t in times],
               candidate_tests_per_s=[tests / t for t in times], event_kernel_ms_per_call=kms / max(kl, 1))
    if not a.no_profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        out["profiler_kernel_ms"] = {e.key: e.device_time_total / 1e3 for e in prof.key_averages() if "guided" in e.key}
    ctx.close()
    import checkers_guided as cg
    if os.path.exists(cg.REF_G_SO) and a.ref_pairs:
        t0 = time.perf_counter(); ref_tests = 0.0
        for k in range(a.ref_pairs):
            i, j = int(pi[k]), int(pj[k])
            cg.ref_guided.__wrapped__(0, s["xy"][i], s["desc"][i], s["xy"][j], s["desc"][j], M[k], thr[k], ratio)
            ref_tests += counts[i] * counts[j]
        dt = time.perf_counter() - t0
        out.update(reference_1thread_pairs_per_s=a.ref_pairs / dt, reference_1thread_candidate_tests_per_s=ref_tests / dt)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
