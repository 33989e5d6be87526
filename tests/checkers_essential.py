"""ctypes bindings for the checkers of the essential-matrix geometric filter (DESIGN §3.8):
oracle/_build/liboracle_essential.so (our CPU restatement) and oracle/_ref/libref_geom_essential.so (the reference
itself), both built by oracle/essential.mk.

Without oracle/_ref the ref_* calls are answered from tests/golden/reference_calls_essential.pkl.gz, recorded with
OMVG_RECORD_REFERENCE=1 and oracle/_ref built, e.g.
`OMVG_RECORD_REFERENCE=1 pytest tests/test_oracle_geom_essential.py`.

Test infrastructure only."""
from __future__ import annotations

import atexit
import ctypes
import functools
import gzip
import hashlib
import os
import pickle
import subprocess

import numpy as np

from checkers import _digest, _P, ROOT

ORACLE_E_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_essential.so")
REF_GEOM_E_SO = os.path.join(ROOT, "oracle", "_ref", "libref_geom_essential.so")
REF_CALLS_E = os.path.join(ROOT, "tests", "golden", "reference_calls_essential.pkl.gz")

_cache = {}


def oracle_e():
    if "o" not in _cache:
        if not os.path.exists(ORACLE_E_SO):
            subprocess.check_call(["make", "-s", "-f", os.path.join(ROOT, "oracle", "essential.mk"), "essential-oracle"])
        _cache["o"] = ctypes.CDLL(ORACLE_E_SO)
    return _cache["o"]


def have_ref_geom_e(replay=False):
    return os.path.exists(REF_GEOM_E_SO) or (replay and os.path.exists(REF_CALLS_E))


def _recorded():
    if "calls" not in _cache:
        _cache["calls"] = {}
        if os.path.exists(REF_CALLS_E):
            with gzip.open(REF_CALLS_E, "rb") as f:
                _cache["calls"] = pickle.load(f)
    return _cache["calls"]


def _save():
    calls = dict(_recorded()); calls.update(_cache.get("record", {}))
    with gzip.GzipFile(REF_CALLS_E, "wb", compresslevel=9, mtime=0) as f:
        pickle.dump(calls, f, protocol=4)


def _replayable(fn):
    """The reference when oracle/_ref has it, else its recorded answer for the same arguments."""
    @functools.wraps(fn)
    def call(*args, **kw):
        h = hashlib.sha1(fn.__name__.encode()); _digest(h, args); _digest(h, sorted(kw.items()))
        key = h.hexdigest()
        if not os.path.exists(REF_GEOM_E_SO):
            calls = _recorded()
            if key not in calls:
                raise KeyError(f"{fn.__name__}: no recorded reference output for these arguments ({REF_CALLS_E}); "
                               "build oracle/_ref and record with OMVG_RECORD_REFERENCE=1")
            return pickle.loads(pickle.dumps(calls[key]))
        out = fn(*args, **kw)
        if os.environ.get("OMVG_RECORD_REFERENCE"):
            rec = _cache.setdefault("record", {})
            if not rec:
                atexit.register(_save)
            rec[key] = out
        return out
    return call


def _ref():
    if "r" not in _cache:
        _cache["r"] = ctypes.CDLL(REF_GEOM_E_SO)
    return _cache["r"]


def _five_point(fn, b1, b2):
    b1 = np.ascontiguousarray(b1, np.float64).reshape(-1, 5, 3); b2 = np.ascontiguousarray(b2, np.float64).reshape(-1, 5, 3)
    n = len(b1)
    E = np.zeros((max(n, 1), 10, 9)); k = np.zeros(max(n, 1), np.int32)
    fn(n, _P(b1), _P(b2), _P(E), _P(k))
    return dict(E=E[:n].reshape(n, 10, 3, 3).copy(), n_models=k[:n].copy())


@_replayable
def ref_five_point(b1, b2):
    """FivePointsRelativePose (multiview/solver_essential_five_point.cpp:170-212) on n samples [n][5][3]."""
    return _five_point(_ref().ref_five_point, b1, b2)


def oracle_five_point(b1, b2):
    return _five_point(oracle_e().oracle_five_point, b1, b2)


def _acransac_e(fn, xI, xJ, wh, intr, precision, iterations, with_trace):
    xI = np.ascontiguousarray(xI, np.float64); xJ = np.ascontiguousarray(xJ, np.float64)
    k6 = np.ascontiguousarray(intr, np.float64).reshape(6)
    n = len(xI)
    inl = np.zeros(max(n, 1), np.uint32); E = np.zeros(9); stats = np.zeros(2); trace = np.zeros(4, np.int32)
    args = [_P(xI), _P(xJ), n, int(wh[0]), int(wh[1]), int(wh[2]), int(wh[3]), _P(k6), ctypes.c_double(precision),
            ctypes.c_uint(iterations), _P(inl), _P(E), _P(stats)]
    if with_trace:
        args.append(_P(trace))
    k = fn(*args)
    return dict(inliers=inl[:k].copy(), F=E.reshape(3, 3), error_max=float(stats[0]), min_nfa=float(stats[1]), trace=trace)


@_replayable
def ref_acransac_essential(xI, xJ, wh, intr, precision=4.0, iterations=2048):
    """The reference's ACRANSAC + ACKernelAdaptorEssential<FivePointSolver, EpipolarDistanceError> (E_ACRobust.hpp:111-133);
    intr = (f, ppx, ppy) of I then J.  `F` of the result holds E."""
    out = _acransac_e(_ref().ref_acransac_essential, xI, xJ, wh, intr, precision, iterations, False)
    out.pop("trace")
    return out


def oracle_acransac_essential(xI, xJ, wh, intr, precision=4.0, iterations=2048):
    """trace: iterations run, models evaluated, iteration AC-RANSAC mode was entered (-1: never), samples without a model."""
    return _acransac_e(oracle_e().oracle_acransac_essential, xI, xJ, wh, intr, precision, iterations, True)


def same_solution_set(A, B, tol=1e-9):
    """Two lists of 3x3 E (any order, any scale and sign) are the same set: each unit-normalised E of A has one
    partner in B within tol, and the counts agree."""
    if len(A) != len(B):
        return False
    un = lambda E: E / np.linalg.norm(E)  # noqa: E731
    left = [un(e) for e in B]
    for e in A:
        e = un(e)
        d = [min(np.abs(e - f).max(), np.abs(e + f).max()) for f in left]
        if not d or min(d) > tol:
            return False
        left.pop(int(np.argmin(d)))
    return True
