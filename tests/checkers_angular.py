"""ctypes bindings for the checkers of the angular essential-matrix geometric filters (`-g a` / `-g u`, DESIGN §3.10):
oracle/_build/liboracle_angular.so (our CPU restatement) and oracle/_ref/libref_geom_angular.so (the reference itself),
both built by oracle/angular.mk.

Without oracle/_ref the ref_* calls are answered from tests/golden/reference_calls_angular.pkl.gz, recorded with
OMVG_RECORD_REFERENCE=1 and oracle/_ref built, e.g.
`OMVG_RECORD_REFERENCE=1 pytest tests/test_oracle_geom_angular.py`.

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

ORACLE_A_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_angular.so")
REF_GEOM_A_SO = os.path.join(ROOT, "oracle", "_ref", "libref_geom_angular.so")
REF_CALLS_A = os.path.join(ROOT, "tests", "golden", "reference_calls_angular.pkl.gz")

ANGULAR, UPRIGHT = 3, 4
MS = {ANGULAR: 8, UPRIGHT: 3}

_cache = {}


def oracle_a():
    if "o" not in _cache:
        if not os.path.exists(ORACLE_A_SO):
            subprocess.check_call(["make", "-s", "-f", os.path.join(ROOT, "oracle", "angular.mk"), "angular-oracle"])
        _cache["o"] = ctypes.CDLL(ORACLE_A_SO)
    return _cache["o"]


def have_ref_geom_a(replay=False):
    return os.path.exists(REF_GEOM_A_SO) or (replay and os.path.exists(REF_CALLS_A))


def _recorded():
    if "calls" not in _cache:
        _cache["calls"] = {}
        if os.path.exists(REF_CALLS_A):
            with gzip.open(REF_CALLS_A, "rb") as f:
                _cache["calls"] = pickle.load(f)
    return _cache["calls"]


def _save():
    calls = dict(_recorded()); calls.update(_cache.get("record", {}))
    with gzip.GzipFile(REF_CALLS_A, "wb", compresslevel=9, mtime=0) as f:
        pickle.dump(calls, f, protocol=4)


def _replayable(fn):
    """The reference when oracle/_ref has it, else its recorded answer for the same arguments."""
    @functools.wraps(fn)
    def call(*args, **kw):
        h = hashlib.sha1(fn.__name__.encode()); _digest(h, args); _digest(h, sorted(kw.items()))
        key = h.hexdigest()
        if not os.path.exists(REF_GEOM_A_SO):
            calls = _recorded()
            if key not in calls:
                raise KeyError(f"{fn.__name__}: no recorded reference output for these arguments ({REF_CALLS_A}); "
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
        _cache["r"] = ctypes.CDLL(REF_GEOM_A_SO)
    return _cache["r"]


def _f64(a, shape):
    return np.ascontiguousarray(a, np.float64).reshape(shape)


def _solver(fn, model, b1, b2):
    ms = MS[model]
    b1 = _f64(b1, (-1, ms, 3)); b2 = _f64(b2, (-1, ms, 3))
    n = len(b1)
    E = np.zeros((max(n, 1), 9))
    fn(int(model), n, _P(b1), _P(b2), _P(E))
    return E[:n].reshape(n, 3, 3).copy()


@_replayable
def ref_angular_solver(model, b1, b2):
    """EightPointRelativePoseSolver (model 3) / ThreePointUprightRelativePoseSolver (model 4) on samples [n][ms][3]."""
    return _solver(_ref().ref_angular_solver, model, b1, b2)


def oracle_angular_solver(model, b1, b2):
    return _solver(oracle_a().oracle_angular_solver, model, b1, b2)


def _error(fn, E, b1, b2):
    E = _f64(E, (-1, 9)); b1 = _f64(b1, (-1, 3)); b2 = _f64(b2, (-1, 3))
    n = len(E)
    out = np.zeros(max(n, 1))
    fn(n, _P(E), _P(b1), _P(b2), _P(out))
    return out[:n].copy()


@_replayable
def ref_angular_error(E, b1, b2):
    """AngularError::Error(E_k, b1_k, b2_k) of n candidates (radians)."""
    return _error(_ref().ref_angular_error, E, b1, b2)


def oracle_angular_error(E, b1, b2):
    return _error(oracle_a().oracle_angular_error, E, b1, b2)


def oracle_asin(x):
    x = np.ascontiguousarray(x, np.float64)
    y = np.zeros(max(len(x), 1))
    oracle_a().oracle_asin(len(x), _P(x), _P(y))
    return y[:len(x)].copy()


def oracle_motion_from_essential(E):
    R = np.zeros((4, 9)); t = np.zeros((4, 3))
    oracle_a().oracle_motion_from_essential(_P(_f64(E, 9)), _P(R), _P(t))
    return R.reshape(4, 3, 3), t


@_replayable
def ref_relative_pose(E, b1, b2, index):
    """RelativePoseFromEssential(b1, b2, E, index) -> dict(counts [4], selected, ok)."""
    E = _f64(E, 9); b1 = _f64(b1, (-1, 3)); b2 = _f64(b2, (-1, 3)); idx = np.ascontiguousarray(index, np.uint32)
    counts = np.zeros(4, np.int32); sel = np.zeros(max(len(idx), 1), np.uint32); ns = np.zeros(1, np.int32)
    ok = _ref().ref_relative_pose(_P(E), len(b1), _P(b1), _P(b2), len(idx), _P(idx), _P(counts), _P(sel), _P(ns))
    return dict(counts=counts, selected=sel[:int(ns[0])].copy(), ok=bool(ok))


def oracle_relative_pose(E, b1, b2, index):
    E = _f64(E, 9); b1 = _f64(b1, (-1, 3)); b2 = _f64(b2, (-1, 3)); idx = np.ascontiguousarray(index, np.uint32)
    counts = np.zeros(4, np.int32); sel = np.zeros(max(len(idx), 1), np.uint32); ns = np.zeros(1, np.int32)
    ok = oracle_a().oracle_relative_pose(_P(E), _P(b1), _P(b2), len(idx), _P(idx), _P(counts), _P(sel), _P(ns))
    return dict(counts=counts, selected=sel[:int(ns[0])].copy(), ok=bool(ok))


def _acransac(fn, model, b1, b2, precision_deg, iterations, with_counts_trace):
    b1 = _f64(b1, (-1, 3)); b2 = _f64(b2, (-1, 3))
    n = len(b1)
    ri = np.zeros(max(n, 1), np.uint32); fi = np.zeros(max(n, 1), np.uint32); nf = np.zeros(1, np.int32)
    E = np.zeros(9); st = np.zeros(2); counts = np.zeros(4, np.int32); trace = np.zeros(3, np.int32)
    args = [int(model), _P(b1), _P(b2), n, ctypes.c_double(precision_deg), ctypes.c_uint(iterations), _P(ri), _P(fi), _P(nf), _P(E), _P(st), _P(counts)]
    if with_counts_trace:
        args.append(_P(trace))
    k = fn(*args)
    out = dict(ransac_inliers=ri[:k].copy(), inliers=fi[:int(nf[0])].copy(), F=E.reshape(3, 3), error_max=float(st[0]),
               min_nfa=float(st[1]), counts=counts)
    if with_counts_trace:
        out["trace"] = trace
    return out


@_replayable
def ref_angular_acransac(model, b1, b2, precision_deg=4.0, iterations=2048):
    """The reference functor's steps on bearing vectors: ACRANSAC + ACKernelAdaptor_AngularRadianError, then
    RelativePoseFromEssential.  `F` holds E; error_max in radians."""
    return _acransac(_ref().ref_angular_acransac, model, b1, b2, precision_deg, iterations, False)


def oracle_angular_acransac(model, b1, b2, precision_deg=4.0, iterations=2048):
    """trace: iterations run, models evaluated, iteration AC-RANSAC mode was entered (-1: never)."""
    return _acransac(oracle_a().oracle_angular_acransac, model, b1, b2, precision_deg, iterations, True)


def same_up_to_sign(A, B, tol):
    A = np.asarray(A).reshape(-1); B = np.asarray(B).reshape(-1)
    return min(np.abs(A - B).max(), np.abs(A + B).max()) <= tol


def golden_pairs():
    """The fixed pairs both models are checked on: (name, model, bI, bJ).  Chosen to reach every branch of the
    functor: too few matches, AC-RANSAC failing, the cheirality ratio test failing, results on both sides of the
    keep threshold, points behind the camera."""
    from openmvg_b200 import synth
    out = []
    for model in (ANGULAR, UPRIGHT):
        for name, n, frac, seed, motion in (("general", 300, 0.3, 1, "general"), ("short", 250, 0.2, 2, "short"),
                                            ("forward", 250, 0.35, 3, "forward"), ("full", 400, 0.4, 4, "full"),
                                            ("upright", 300, 0.3, 5, "upright"), ("upright_tilt", 300, 0.3, 6, "upright_tilt"),
                                            ("rotation", 300, 0.1, 7, "rotation"), ("outliers70", 300, 0.7, 8, "general"),
                                            ("all_outliers", 200, 1.0, 9, "general"), ("few", 24, 0.1, 10, "general")):
            _, _, bI, bJ, _ = synth.spherical_two_view_matches(n, frac, seed=seed + 100 * model, motion=motion)
            out.append((name, model, bI, bJ))
        # the keep rule is "more than 2.5 * MINIMUM_SAMPLES": final lists of 20 / 21 (eight-point), 7 / 8 (upright)
        for k, n, seed in (((20, 21, 11), (21, 21, 1)) if model == ANGULAR else ((7, 8, 22), (8, 8, 28))):
            _, _, bI, bJ, _ = synth.spherical_two_view_matches(n, 0.1, seed=seed, motion="general")
            out.append((f"keep{k}", model, bI, bJ))
        _, _, bI, bJ, _ = synth.spherical_two_view_matches(MS[model], 0.0, seed=11, motion="general")
        out.append(("n_eq_ms", model, bI, bJ))
    return out
