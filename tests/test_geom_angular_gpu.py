"""The GPU angular essential-matrix filters (`-g a` eight-point, `-g u` upright three-point: omvg_geom_angular_acransac)
against the CPU restatement (oracle/angular_oracle.cpp), which tests/test_oracle_geom_angular.py pins to the reference."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest

import checkers_angular as ca
from openmvg_b200 import geometry, synth
from openmvg_b200._lib import lib

pytestmark = pytest.mark.gpu

MODELS = [ca.ANGULAR, ca.UPRIGHT]


def _csr(pairs):
    off = np.concatenate([[0], np.cumsum([len(b) for b, _ in pairs])]).astype(np.uint64)
    return off, np.concatenate([b for b, _ in pairs]).reshape(-1, 3), np.concatenate([b for _, b in pairs]).reshape(-1, 3)


def _check(pairs, model, iters):
    off, bI, bJ = _csr(pairs)
    res = geometry.angular_essential_acransac(off, bI, bJ, upright=model == ca.UPRIGHT, precision_deg=4.0, max_iterations=iters)
    for k, ((b1, b2), r) in enumerate(zip(pairs, res)):
        o = ca.oracle_angular_acransac(model, b1, b2, 4.0, iters)
        assert np.array_equal(r["ransac_inliers"], o["ransac_inliers"]), k
        assert np.array_equal(r["inliers"], o["inliers"]), k
        assert (r["error_max"] == o["error_max"]) and (r["min_nfa"] == o["min_nfa"] or abs(r["min_nfa"] - o["min_nfa"]) <= 1e-12), k
        assert np.abs(r["F"] - o["F"]).max() <= 1e-12, k
    return res


@pytest.mark.parametrize("model", MODELS)
def test_goldens_one_launch(model):
    pairs = [(bI, bJ) for _, m, bI, bJ in ca.golden_pairs() if m == model]
    _check(pairs, model, 2048)


@pytest.mark.parametrize("iters", [64, 2048])
@pytest.mark.parametrize("model", MODELS)
def test_random_pairs(model, iters):
    rng = np.random.default_rng(77 + model)
    pairs = []
    for k in range(60):
        motion = synth.ANGULAR_MOTIONS[k % len(synth.ANGULAR_MOTIONS)]
        _, _, bI, bJ, _ = synth.spherical_two_view_matches(int(rng.integers(10, 600)), float(rng.uniform(0, 0.7)), seed=3000 + k, motion=motion)
        pairs.append((bI, bJ))
    res = _check(pairs, model, iters)
    assert sum(len(r["inliers"]) > 2.5 * ca.MS[model] for r in res) >= 10


@pytest.mark.parametrize("model", MODELS)
def test_solver_debug_entry(model):
    ms = ca.MS[model]
    _, _, bI, bJ, _ = synth.spherical_two_view_matches(10000 * ms, 0.0, seed=91, motion="full")
    b1, b2 = bI.reshape(-1, ms, 3), bJ.reshape(-1, ms, 3)
    g = geometry.debug_angular_solver(b1, b2, upright=model == ca.UPRIGHT)
    o = ca.oracle_angular_solver(model, b1, b2)
    assert np.abs(g - o).max() <= 1e-12


def _pose_cases():
    _, _, bI, bJ, _ = synth.spherical_two_view_matches(40, 0.0, seed=21, motion="general")
    E = ca.oracle_angular_acransac(ca.ANGULAR, bI, bJ)["F"]
    idx = np.arange(40, dtype=np.uint32)
    def flip(k, m):
        return np.concatenate([bI[:k], -bI[k:k + m]]), np.concatenate([bJ[:k], -bJ[k:k + m]]), np.arange(k + m, dtype=np.uint32)
    return {"good": (E, bI, bJ, idx), "empty": (E, bI, bJ, idx[:0]), "ratio_0.7": (E,) + flip(10, 7), "ratio_0.6": (E,) + flip(10, 6),
            "tie": (E,) + flip(10, 10), "all_behind": (E, -bI, -bJ, idx), "parallel": (E, bI, bI.copy(), idx),
            "subset_unordered": (E, bI, bJ, idx[::-3].copy())}


@pytest.mark.parametrize("case", ["good", "empty", "ratio_0.7", "ratio_0.6", "tie", "all_behind", "parallel", "subset_unordered"])
def test_relative_pose_debug_entry(case):
    E, b1, b2, idx = _pose_cases()[case]
    g = geometry.debug_relative_pose(E, b1, b2, idx)
    o = ca.oracle_relative_pose(E, b1, b2, idx)
    assert np.array_equal(g["counts"], o["counts"]) and g["ok"] == o["ok"] and np.array_equal(g["selected"], o["selected"])
    top = sorted(o["counts"])[-2:]
    expect = {"empty": ([0, 0], False), "ratio_0.7": ([7, 10], False), "ratio_0.6": ([6, 10], True), "tie": ([10, 10], False)}
    if case in expect:
        assert (top, g["ok"]) == expect[case]


def test_error_codes():
    L = lib()
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    _, _, bI, bJ, _ = synth.spherical_two_view_matches(50, 0.2, seed=4)
    off = np.array([0, 50], np.uint64)
    inl = np.zeros(50, np.uint32); n = np.zeros(1, np.uint32); E = np.zeros(9); st = np.zeros(2)

    def call(model=3, offsets=off, b1=bI, b2=bJ, prec=4.0):
        return L.omvg_geom_angular_acransac(0, model, ctypes.c_uint64(len(offsets) - 1), p(offsets), p(np.ascontiguousarray(b1)), p(np.ascontiguousarray(b2)),
                                            ctypes.c_double(prec), ctypes.c_uint32(2048), p(inl), p(n), p(E), p(st), None, None)
    assert call() == 0
    for prec in (float("inf"), float("nan"), 0.0, -1.0):
        assert call(prec=prec) == -4
    bad = bI.copy(); bad[7, 1] = np.nan
    assert call(b1=bad) == -1
    assert call(offsets=np.array([0, 30, 20], np.uint64)) == -1
    assert call(model=2) == -1
    assert L.omvg_geom_angular_acransac(0, 3, ctypes.c_uint64(1), p(off), None, None, ctypes.c_double(4.0), ctypes.c_uint32(2048),
                                        p(inl), p(n), p(E), p(st), None, None) == -1
    # omvg_geom_acransac takes pixels: it rejects the bearing-vector models
    xy = np.zeros((50, 2)); sz = np.array([[100, 100, 100, 100]], np.int32)
    for model in (3, 4):
        assert L.omvg_geom_acransac(0, model, ctypes.c_uint64(1), p(off), p(xy), p(xy), p(sz), ctypes.c_double(4.0), ctypes.c_uint32(2048),
                                    p(inl), p(n), p(E), p(st)) == -4
