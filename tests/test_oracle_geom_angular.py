"""The CPU restatement of the angular essential-matrix filters (`-g a` / `-g u`, oracle/angular_oracle.cpp) against the
reference's own solvers, AngularError, ACRANSAC + ACKernelAdaptor_AngularRadianError and RelativePoseFromEssential
(oracle/_ref/libref_geom_angular.so, or its recorded answers in tests/golden/reference_calls_angular.pkl.gz)."""
from __future__ import annotations

import numpy as np
import pytest

import checkers_angular as ca
from openmvg_b200 import synth

pytestmark = pytest.mark.skipif(not ca.have_ref_geom_a(replay=True), reason="no reference answers (oracle/_ref or golden)")

MODELS = [ca.ANGULAR, ca.UPRIGHT]


def _samples(model, motion, n, seed):
    ms = ca.MS[model]
    _, _, bI, bJ, _ = synth.spherical_two_view_matches(n * ms, 0.0, seed=seed, motion=motion)
    return bI.reshape(n, ms, 3), bJ.reshape(n, ms, 3)


def _same_result(r, o):
    assert np.array_equal(r["ransac_inliers"], o["ransac_inliers"])
    assert np.array_equal(r["inliers"], o["inliers"])
    # the order of the four poses depends on the signs the SVD picks; the multiset of counts does not
    assert np.array_equal(np.sort(r["counts"]), np.sort(o["counts"]))
    for k in ("error_max", "min_nfa"):
        a, b = r[k], o[k]
        assert (a == b) or abs(a - b) <= 1e-9, (k, a, b)
    E1, E2 = np.asarray(r["F"]), np.asarray(o["F"])                 # the solver's bound (test_solver_matches_reference)
    assert ca.same_up_to_sign(E1 / np.linalg.norm(E1), E2 / np.linalg.norm(E2), 1e-7)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("motion", ["general", "short", "full", "upright"])
def test_solver_matches_reference(model, motion):
    b1, b2 = _samples(model, motion, 1000, seed=17 + model)
    r = ca.ref_angular_solver(model, b1, b2); o = ca.oracle_angular_solver(model, b1, b2)
    # a minimal sample's null vector is only as well defined as the gap to the next eigenvalue of A'A: Jacobi and
    # Eigen's tridiagonal QR differ by up to 3.1e-8 (eight-point, short baseline) on these samples, 99 % within 5e-9
    d = np.array([min(np.abs(a - b).max(), np.abs(a + b).max()) for a, b in zip(r, o)])
    assert d.max() <= 1e-7 and np.percentile(d, 99) <= 1e-8, (d.max(), np.percentile(d, 99))


def test_angular_error_bit_for_bit():
    """AngularError with the reference's FMAs: identical bits on 40 000 candidates (random models, and solver models
    against their own and other bearings)."""
    rng = np.random.default_rng(5)
    n = 20000
    E = rng.normal(size=(n, 9))
    _, _, b1, b2, _ = synth.spherical_two_view_matches(n, 0.5, seed=6, motion="full")
    b1s, b2s = _samples(ca.ANGULAR, "general", n // 8, seed=8)
    Es = np.repeat(ca.oracle_angular_solver(ca.ANGULAR, b1s, b2s).reshape(-1, 9), 8, axis=0)
    E = np.concatenate([E, Es]); B1 = np.concatenate([b1, b1s.reshape(-1, 3)]); B2 = np.concatenate([b2, b2s.reshape(-1, 3)])
    r = ca.ref_angular_error(E, B1, B2); o = ca.oracle_angular_error(E, B1, B2)
    assert np.array_equal(r.view(np.uint64), o.view(np.uint64))


def _pose_cases():
    """(E, b1, b2, index) covering the edges of RelativePoseFromEssential."""
    _, _, bI, bJ, inl = synth.spherical_two_view_matches(40, 0.0, seed=21, motion="general")
    o = ca.oracle_angular_acransac(ca.ANGULAR, bI, bJ)
    E = o["F"]
    idx = np.arange(40, dtype=np.uint32)
    cases = {"good": (E, bI, bJ, idx), "empty": (E, bI, bJ, idx[:0])}
    flip = np.concatenate([bI[:10], -bI[10:17]]), np.concatenate([bJ[:10], -bJ[10:17]])
    cases["ratio_0.7"] = (E, flip[0], flip[1], np.arange(17, dtype=np.uint32))          # counts {10, 7, 0, 0}
    tie = np.concatenate([bI[:10], -bI[10:20]]), np.concatenate([bJ[:10], -bJ[10:20]])
    cases["tie"] = (E, tie[0], tie[1], np.arange(20, dtype=np.uint32))                  # counts {10, 10, 0, 0}
    cases["all_behind"] = (E, -bI, -bJ, idx)                                             # every point behind both cameras
    cases["parallel"] = (E, bI, bI.copy(), idx)                                          # identical rays
    cases["subset"] = (E, bI, bJ, idx[::3].copy())
    return cases


@pytest.mark.parametrize("case", ["good", "empty", "ratio_0.7", "tie", "all_behind", "parallel", "subset"])
def test_relative_pose_matches_reference(case):
    E, b1, b2, idx = _pose_cases()[case]
    r = ca.ref_relative_pose(E, b1, b2, idx); o = ca.oracle_relative_pose(E, b1, b2, idx)
    assert np.array_equal(np.sort(r["counts"]), np.sort(o["counts"]))
    assert r["ok"] == o["ok"] and np.array_equal(r["selected"], o["selected"])
    if case == "ratio_0.7":
        assert sorted(o["counts"])[-2:] == [7, 10] and not o["ok"]
    if case == "tie":
        assert sorted(o["counts"])[-2:] == [10, 10] and not o["ok"]
    if case == "empty":
        assert max(o["counts"]) == 0 and not o["ok"]


@pytest.mark.parametrize("k", range(len(ca.golden_pairs())))
def test_golden_pairs_match_reference(k):
    name, model, bI, bJ = ca.golden_pairs()[k]
    _same_result(ca.ref_angular_acransac(model, bI, bJ), ca.oracle_angular_acransac(model, bI, bJ))


RANDOM = [(model, iters, seed) for model in MODELS for iters, seed in ((64, 1), (256, 2), (2048, 3), (2048, 4), (256, 5), (64, 6))]


@pytest.mark.parametrize("model,iters,seed", RANDOM)
def test_random_pairs_match_reference(model, iters, seed):
    rng = np.random.default_rng(1000 + 10 * seed + model)
    motion = synth.ANGULAR_MOTIONS[int(rng.integers(len(synth.ANGULAR_MOTIONS)))]
    _, _, bI, bJ, _ = synth.spherical_two_view_matches(int(rng.integers(30, 500)), float(rng.uniform(0, 0.7)), seed=seed + 50 * model, motion=motion)
    _same_result(ca.ref_angular_acransac(model, bI, bJ, 4.0, iters), ca.oracle_angular_acransac(model, bI, bJ, 4.0, iters))


def test_goldens_reach_every_branch():
    """The golden pairs take every branch of the functor: nData <= MINIMUM_SAMPLES, AC-RANSAC failing, the cheirality
    best count 0 (no AC-RANSAC inliers), the ratio test failing with inliers, final lists at and just above the keep
    threshold (20 / 21 for the eight-point, 7 / 8 for upright) and points behind camera I."""
    seen = set()
    for name, model, bI, bJ in ca.golden_pairs():
        o = ca.oracle_angular_acransac(model, bI, bJ)
        nr, nf, ms = len(o["ransac_inliers"]), len(o["inliers"]), ca.MS[model]
        if len(bI) <= ms:
            seen.add("ndata_le_ms")
        elif nr == 0:
            seen.add("acransac_failed")
        if max(o["counts"]) == 0:
            seen.add("best_count_0")
        if nr > 0 and nf == 0:
            seen.add("ratio_ge_0.7")
        thr = 20 if model == ca.ANGULAR else 7
        if nf in (thr, thr + 1):
            seen.add(f"keep_edge_{model}_{nf}")
        if nf and (bI[o["inliers"], 2] < 0).any():
            seen.add("behind")
    assert seen >= {"ndata_le_ms", "acransac_failed", "best_count_0", "ratio_ge_0.7", "behind",
                    "keep_edge_3_20", "keep_edge_3_21", "keep_edge_4_7", "keep_edge_4_8"}, seen
