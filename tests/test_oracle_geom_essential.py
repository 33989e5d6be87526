"""CPU: the essential-matrix filter's oracle (oracle/essential_oracle.cpp, DESIGN §3.8) against the reference's own
FivePointsRelativePose and ACRANSAC + ACKernelAdaptorEssential (oracle/_ref/libref_geom_essential.so, or its recorded
answers in tests/golden/reference_calls_essential.pkl.gz).

The five-point solver is pinned as a SET of solutions per sample: the order of the models depends on which basis of
the 4-D null space an eigen-solver returns, which rounding decides.  The filter is pinned on identical inlier lists."""
import numpy as np
import pytest

import checkers_essential as ce
from openmvg_b200 import synth

pytestmark = pytest.mark.skipif(not ce.have_ref_geom_e(replay=True), reason="no reference essential filter and no recorded answers")

WH = (1600, 1200)
# golden pairs: (name, n, outlier fraction, seed, motion)
GOLD_E = [
    ("p200_no_model", 200, 1.0, 71, "general"),
    ("p5", 5, 0.0, 72, "general"),
    ("p6", 6, 0.0, 73, "general"),
    ("p30_too_few", 30, 0.6, 210, "general"),
    ("p400_clean", 400, 0.0, 75, "general"),
    ("p1500_half_outliers", 1500, 0.5, 76, "general"),
    ("p800_short_baseline", 800, 0.3, 77, "short"),
    ("p800_forward", 800, 0.3, 78, "forward"),
    ("p600_near_planar", 600, 0.2, 79, "planar"),
]


def gold_inputs(n, of, seed, motion):
    xI, xJ, _, kI, kJ = synth.calibrated_two_view_matches(max(n, 1), of, seed=seed, wh=WH, motion=motion)
    return xI[:n], xJ[:n], WH + WH, np.array(kI + kJ)


def bearings(x, k):
    u = (x[:, 0] - k[1]) / k[0]; v = (x[:, 1] - k[2]) / k[0]
    b = np.stack([u, v, np.ones_like(u)], 1)
    return b / np.linalg.norm(b, axis=1, keepdims=True)


def five_point_samples(n, seed, motion):
    """n samples of 5 noisy, outlier-free correspondences as bearing pairs [n, 5, 3]."""
    xI, xJ, _, kI, kJ = synth.calibrated_two_view_matches(5 * n, 0.0, seed=seed, wh=WH, motion=motion)
    return bearings(xI, kI).reshape(n, 5, 3), bearings(xJ, kJ).reshape(n, 5, 3)


# Tolerances per family (set comparison, residuals of each solution).  General views are well conditioned; a short
# baseline, a forward motion or a near-planar scene make the five-point problem itself ill-conditioned, and the
# rounding differences between the reference's Eigen solvers and ours grow with it (DESIGN §3.8).  Worst values
# observed on the pinned samples, set / residual: general 6.1e-9 / 1.4e-9, short 9.3e-8 / 6.0e-9,
# forward 1.9e-8 / 2.7e-8, planar 5.5e-9 / 1.3e-9; the bounds are 1.6 to 8 times those.
FAMILIES = [("general", 1e-8, 1e-8), ("short", 5e-7, 3e-8), ("forward", 1e-7, 1e-7), ("planar", 3e-8, 1e-8)]


@pytest.mark.parametrize("motion,tol,rtol", FAMILIES, ids=[f[0] for f in FAMILIES])
def test_five_point_oracle_against_reference(motion, tol, rtol):
    b1, b2 = five_point_samples(500, 90 + len(motion), motion)
    r = ce.ref_five_point(b1, b2); o = ce.oracle_five_point(b1, b2)
    assert np.array_equal(r["n_models"], o["n_models"])
    for s in range(len(b1)):
        k = o["n_models"][s]
        assert ce.same_solution_set(r["E"][s][:k], o["E"][s][:k], tol), (motion, s)
        for E in o["E"][s][:k]:
            E = E / np.linalg.norm(E)
            assert np.abs(np.einsum("ti,ij,tj->t", b2[s], E, b1[s])).max() < rtol
            assert abs(np.linalg.det(E)) < rtol
            assert np.abs(2 * E @ E.T @ E - np.trace(E @ E.T) * E).max() < rtol


def check_same(r, o, what):
    assert np.array_equal(r["inliers"], o["inliers"]), what
    if len(o["inliers"]):
        assert abs(r["error_max"] - o["error_max"]) <= 1e-9 * abs(r["error_max"]), what
        assert abs(r["min_nfa"] - o["min_nfa"]) <= 1e-9 * abs(r["min_nfa"]), what
        E = r["F"] / np.linalg.norm(r["F"]); G = o["F"] / np.linalg.norm(o["F"])
        assert min(np.abs(E - G).max(), np.abs(E + G).max()) <= 1e-7, what


@pytest.mark.parametrize("c", GOLD_E, ids=[c[0] for c in GOLD_E])
def test_oracle_against_reference_golden(c):
    xI, xJ, wh, k = gold_inputs(*c[1:])
    check_same(ce.ref_acransac_essential(xI, xJ, wh, k, 4.0, 2048), ce.oracle_acransac_essential(xI, xJ, wh, k, 4.0, 2048), c[0])


def test_goldens_exercise_every_branch():
    """Early exit without a model, <= 5 matches, a pair too weak to keep, a model at iteration 0, the focused phase,
    K_I != K_J (every case)."""
    res = {c[0]: ce.oracle_acransac_essential(*gold_inputs(*c[1:]), 4.0, 2048) for c in GOLD_E}
    assert len(res["p200_no_model"]["inliers"]) == 0 and res["p200_no_model"]["trace"][2] == -1
    assert res["p5"]["trace"][0] == 0 and len(res["p5"]["inliers"]) == 0
    assert 0 < len(res["p30_too_few"]["inliers"]) <= 12          # a model, but the filter does not keep the pair
    assert res["p400_clean"]["trace"][2] == 0 and len(res["p400_clean"]["inliers"]) > 300
    assert len(res["p1500_half_outliers"]["inliers"]) > 600
    assert res["p1500_half_outliers"]["trace"][0] < 2048          # the focused phase ended the search early
    kI, kJ = gold_inputs(*GOLD_E[0][1:])[3].reshape(2, 3)
    assert kI[0] != kJ[0] and kI[1] != kJ[1]


@pytest.mark.parametrize("seed", range(120, 132))
def test_oracle_against_compiled_reference(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(7, 900)); of = float(rng.uniform(0.0, 0.7)); it = [64, 256, 2048][seed % 3]
    motion = ["general", "short", "forward", "planar"][seed % 4]
    xI, xJ, wh, k = gold_inputs(n, of, seed, motion)
    check_same(ce.ref_acransac_essential(xI, xJ, wh, k, 4.0, it), ce.oracle_acransac_essential(xI, xJ, wh, k, 4.0, it), (n, of, it, motion))
