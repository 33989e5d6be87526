"""Compare the SASS of two source trees, function by function.

    python tools/sass_compare.py OLD_ROOT NEW_ROOT [--out DIR]

Each root is a checkout of this repository (for instance `git worktree add /tmp/old <rev>`).  Every translation unit
of openmvg_b200/build.py is compiled in both with the flags build.py uses, then `cuobjdump -sass` is split into
functions and the instruction text (addresses and encodings stripped) is compared.  A host-only change must report
every function identical: identical SASS means identical device time.  Needs nvcc, no GPU.
"""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from openmvg_b200 import build as B  # noqa: E402


def compile_tu(root: str, src: str, out_dir: str) -> str:
    obj = os.path.join(out_dir, src[:-3] + ".o")
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")] + B.EXTRA_FLAGS.get(src, [])
    subprocess.check_call([B._nvcc()] + flags + ["-c", os.path.join(root, "openmvg_b200", "csrc", src), "-o", obj])
    return obj


def sass_functions(obj: str) -> dict[str, list[str]]:
    text = subprocess.run([os.path.join(os.path.dirname(B._nvcc()), "cuobjdump"), "-sass", obj],
                          check=True, capture_output=True, text=True).stdout
    funcs: dict[str, list[str]] = {}
    cur = None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)   # "/*0040*/  IMAD.MOV.U32 R1, ... ;  /* 0x... */"
        if cur is not None and m:
            cur.append(m.group(1))
    return funcs


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("old_root")
    ap.add_argument("new_root")
    ap.add_argument("--out", help="keep the objects here (default: a temporary directory)")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        base = a.out or tmp
        dirs = {r: os.path.join(base, tag) for r, tag in ((a.old_root, "old"), (a.new_root, "new"))}
        for d in dirs.values():
            os.makedirs(d, exist_ok=True)
        jobs = [(r, s, d) for r, d in dirs.items() for s in B.SOURCES]
        with ThreadPoolExecutor(max_workers=len(jobs)) as ex:
            objs = list(ex.map(lambda j: compile_tu(*j), jobs))
        bad = 0
        for k, src in enumerate(B.SOURCES):
            old, new = sass_functions(objs[k]), sass_functions(objs[len(B.SOURCES) + k])
            same = sum(old[f] == new.get(f) for f in old)
            diff = sorted(f for f in old.keys() | new.keys() if old.get(f) != new.get(f))
            n_ins = sum(len(v) for v in new.values())
            print(f"{src}: {len(old)} functions old, {len(new)} new ({n_ins} instructions), {same} identical"
                  + ("" if not diff else f", {len(diff)} differ"))
            for f in diff:
                print(f"  differs: {f}")
            bad += len(diff)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
