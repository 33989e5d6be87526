"""Per-kernel device time of BA Adjust on one GPU (torch.profiler, CUDA activities), by default on bench.py's
headline scene (1000 cameras / 100k points / 1M observations, seed 42).

  python tools/ba_profile.py [--cams 1000 --points 100000 --obs-per-point 10 --runs 2] [--json OUT]

Prints the GPU name and power limit, the device memory the context holds after a solve, and a table of kernels
sorted by device time: total ms over the profiled runs, ms per LM iteration and share of all device time.
The profiled runs are taken after one warm-up solve; tracing slows the host, so take end-to-end rates from bench.py.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                                       # the numbers still stand; the card is then unnamed
        return dict(error=str(e)[:200])


def short(name: str) -> str:
    """'void omvg::ba::schur_stage_kernel<3>(omvg::ba::SchurArgs, ...)' -> 'schur_stage_kernel<3>'"""
    name = re.sub(r"^void ", "", name.split("(")[0])
    return re.sub(r"^(omvg::)?(ba::)?(\(anonymous namespace\)::)?", "", name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cams", type=int, default=1000)
    ap.add_argument("--points", type=int, default=100_000)
    ap.add_argument("--obs-per-point", type=int, default=10)
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--json", default=None, help="also write the table as JSON to this path")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from openmvg_b200 import ba, synth

    torch.cuda.init()
    free0, total = torch.cuda.mem_get_info()
    scene = synth.ba_scene(args.cams, args.points, args.obs_per_point, seed=args.seed)
    ctx = ba.BAContext(scene, device=0)
    ctx.reset(); ctx.run()                                     # warm-up: module load, lazily allocated buffers
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    iters = lm_steps = 0; dev_ms = 0.0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.runs):
            ctx.reset(); r = ctx.run()
            iters += r["iterations"]; lm_steps += r["lm_steps"]; dev_ms += r["device_ms"]
        torch.cuda.synchronize()
    ctx.close()

    per = collections.defaultdict(lambda: [0.0, 0])            # name -> [device us, launches]
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = e.device_time_total
        k = short(e.name); per[k][0] += t; per[k][1] += 1
    total_us = sum(v[0] for v in per.values())
    rows = sorted(((k, v[0] / 1e3, v[1]) for k, v in per.items()), key=lambda x: -x[1])
    info = gpu_info()
    res = dict(gpu=info, scene=dict(cams=args.cams, points=args.points, obs=args.points * args.obs_per_point, seed=args.seed),
               runs=args.runs, iterations=iters, lm_steps=lm_steps, device_ms_events=dev_ms, kernel_ms=total_us / 1e3,
               context_mib=(free0 - free1) / 2**20,
               kernels=[dict(name=k, ms=ms, launches=n, ms_per_lm_iter=ms / max(iters, 1), share=ms * 1e3 / total_us) for k, ms, n in rows])
    print(f"GPU: {info}")
    print(f"{args.runs} solves, {iters} LM iterations ({lm_steps} LM steps), {dev_ms:.2f} ms by CUDA events, "
          f"{total_us / 1e3:.2f} ms of kernels and copies in the trace; device memory held by the context {res['context_mib']:.0f} MiB")
    print(f"{'kernel':<48} {'ms':>9} {'launches':>9} {'ms/iter':>9} {'share':>7}")
    for k, ms, n in rows:
        print(f"{k[:48]:<48} {ms:9.3f} {n:9d} {ms / max(iters, 1):9.4f} {100 * ms * 1e3 / total_us:6.1f}%")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(res, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
