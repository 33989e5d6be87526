"""ctypes bindings for the checkers of guided matching (DESIGN §3.9): oracle/_build/liboracle_guided.so (our CPU
restatement) and oracle/_ref/libref_guided.so (the reference's own geometry_aware::GuidedMatching), both built by
oracle/guided.mk.

Without oracle/_ref the ref_* calls are answered from tests/golden/reference_calls_guided.pkl.gz, recorded with
OMVG_RECORD_REFERENCE=1 and oracle/_ref built, e.g. `OMVG_RECORD_REFERENCE=1 pytest tests/test_oracle_guided.py`.

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

ORACLE_G_SO = os.path.join(ROOT, "oracle", "_build", "liboracle_guided.so")
REF_G_SO = os.path.join(ROOT, "oracle", "_ref", "libref_guided.so")
REF_CALLS_G = os.path.join(ROOT, "tests", "golden", "reference_calls_guided.pkl.gz")

_cache = {}


def oracle_g():
    if "o" not in _cache:
        if not os.path.exists(ORACLE_G_SO):
            subprocess.check_call(["make", "-s", "-f", os.path.join(ROOT, "oracle", "guided.mk"), "guided-oracle"])
        L = ctypes.CDLL(ORACLE_G_SO)
        L.oracle_guided.restype = ctypes.c_uint32
        _cache["o"] = L
    return _cache["o"]


def have_ref_guided(replay=False):
    return os.path.exists(REF_G_SO) or (replay and os.path.exists(REF_CALLS_G))


def _recorded():
    if "calls" not in _cache:
        _cache["calls"] = {}
        if os.path.exists(REF_CALLS_G):
            with gzip.open(REF_CALLS_G, "rb") as f:
                _cache["calls"] = pickle.load(f)
    return _cache["calls"]


def _save():
    calls = dict(_recorded()); calls.update(_cache.get("record", {}))
    with gzip.GzipFile(REF_CALLS_G, "wb", compresslevel=9, mtime=0) as f:
        pickle.dump(calls, f, protocol=4)


def _replayable(fn):
    """The reference when oracle/_ref has it, else its recorded answer for the same arguments."""
    @functools.wraps(fn)
    def call(*args, **kw):
        h = hashlib.sha1(fn.__name__.encode()); _digest(h, args); _digest(h, sorted(kw.items()))
        key = h.hexdigest()
        if not os.path.exists(REF_G_SO):
            calls = _recorded()
            if key not in calls:
                raise KeyError(f"{fn.__name__}: no recorded reference output for these arguments ({REF_CALLS_G}); "
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
        L = ctypes.CDLL(REF_G_SO)
        L.ref_guided.restype = ctypes.c_uint32
        _cache["r"] = L
    return _cache["r"]


def _arrays(xI, dI, xJ, dJ, M):
    xI = np.ascontiguousarray(xI, np.float64).reshape(-1, 2); xJ = np.ascontiguousarray(xJ, np.float64).reshape(-1, 2)
    dI = np.ascontiguousarray(dI, np.uint8).reshape(-1, 128); dJ = np.ascontiguousarray(dJ, np.uint8).reshape(-1, 128)
    M = np.ascontiguousarray(M, np.float64).reshape(9)
    return xI, dI, xJ, dJ, M


@_replayable
def ref_guided(model, xI, dI, xJ, dJ, M, thr, ratio, camI=None, camJ=None):
    """The reference's GuidedMatching for one pair.  model 0 = EpipolarDistanceError, 1 = AsymmetricError; ratio >= 0:
    the descriptor variant on SIFT_Regions (feature coordinates are floats there), < 0: the descriptor-free variant.
    camI / camJ: {w, h, f, ppx, ppy, k1} of a Pinhole_Intrinsic_Radial_K1 that un-distorts the positions, or None.
    -> [m, 2] uint32 (i, j)."""
    xI, dI, xJ, dJ, M = _arrays(xI, dI, xJ, dJ, M)
    out = np.zeros((max(len(xI), 1), 2), np.uint32)
    cI = None if camI is None else np.ascontiguousarray(camI, np.float64)
    cJ = None if camJ is None else np.ascontiguousarray(camJ, np.float64)
    n = _ref().ref_guided(int(model), _P(xI), len(xI), _P(dI), _P(xJ), len(xJ), _P(dJ), _P(M), ctypes.c_double(thr),
                          ctypes.c_double(ratio), None if cI is None else _P(cI), None if cJ is None else _P(cJ), _P(out))
    return out[:n].copy()


@_replayable
def ref_ud_pixels(cam, xy):
    """Pinhole_Intrinsic_Radial_K1{w, h, f, ppx, ppy, k1}::get_ud_pixel of every row of xy."""
    c = np.ascontiguousarray(cam, np.float64); xy = np.ascontiguousarray(xy, np.float64).reshape(-1, 2)
    out = np.zeros_like(xy)
    _ref().ref_ud_pixels(_P(c), _P(xy), len(xy), _P(out))
    return out


def _errors(fn, model, M, xI, xJ):
    M = np.ascontiguousarray(M, np.float64).reshape(9)
    xI = np.ascontiguousarray(xI, np.float64).reshape(-1, 2); xJ = np.ascontiguousarray(xJ, np.float64).reshape(-1, 2)
    err = np.zeros(len(xI))
    fn(int(model), _P(M), _P(xI), _P(xJ), len(xI), _P(err))
    return err


@_replayable
def ref_guided_errors(model, M, xI, xJ):
    """EpipolarDistanceError::Error / AsymmetricError::Error of the rows (xI[k], xJ[k])."""
    return _errors(_ref().ref_guided_errors, model, M, xI, xJ)


def oracle_guided_errors(model, M, xI, xJ):
    return _errors(oracle_g().oracle_guided_errors, model, M, xI, xJ)


def oracle_guided(model, xI, dI, xJ, dJ, M, thr, ratio):
    """guided_oracle.cpp on positions as given (already un-distorted).  -> [m, 2] uint32 (i, j), ascending i."""
    xI, dI, xJ, dJ, M = _arrays(xI, dI, xJ, dJ, M)
    out = np.zeros((max(len(xI), 1), 2), np.uint32)
    n = oracle_g().oracle_guided(int(model), _P(xI), len(xI), _P(dI), _P(xJ), len(xJ), _P(dJ), _P(M), ctypes.c_double(thr),
                                 ctypes.c_double(ratio), _P(out))
    return out[:n].copy()


def oracle_guided_collection(model, xys, descs, pi, pj, models, thresholds, ratio):
    """The oracle over a pair list, in omvg_match_fetch's CSR layout: (offsets [n+1] uint64, ij [m, 2] uint32)."""
    rows = [oracle_guided(model, xys[a], descs[a], xys[b], descs[b], models[p], thresholds[p], ratio)
            for p, (a, b) in enumerate(zip(pi, pj))]
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.uint64)
    ij = np.concatenate(rows).astype(np.uint32) if rows else np.zeros((0, 2), np.uint32)
    return off, ij.reshape(-1, 2)
