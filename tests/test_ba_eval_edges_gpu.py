"""The residual / Jacobian evaluation on the GPU (omvg_ba_debug_eval, omvg_ba_residual_norms, omvg_ba_debug_prior)
entry by entry against the extended-precision reference of tests/ba_eval_reference.py, on scenes built to hit the
edges of the evaluation: rotation angles on both sides of AngleAxisRotatePoint's theta^2 <= eps branch and near or
beyond pi, depths from 1e-3 to 1e4 and behind the camera, landmarks 1e4 from the origin seen from nearby, the fisheye
r = 1e-8 switch and r = 0, distortion at r ~ 1, the spherical poles and lon = +-pi seam, the Huber switch at
|r|^2 = a^2 (1 +- 1e-9) and the far tail, weights 0 .. 1e3, no-loss flags, fixed landmarks, every option mask, four
camera models in one scene (kiu = 8), a grid-stride scene of 60 001 observations on a one-wave grid, and the
pose-centre prior rows.

Bar: |gpu - reference| <= TAU m per entry, m the sum of |terms| that forms it (the reference's magnitude).  The
kernel forms each entry from the same terms in another order (analytic distortion derivatives, R (j_k x X) for the
rotation columns, FMA contraction).  m already carries the first-order propagation of every operand of every
operation on every term (it is typically 30 |J| on the pose and point blocks), so a rounding of eps/2 relative in any
one operation, or an ulp of CUDA's sin / cos / atan / atan2, moves an entry by well under 1 eps of m; a correct
evaluation in any order stays below about 1 eps m (0.74 measured, below).  TAU = 4 eps leaves a factor of 5 over the
measured worst, for contraction and libm differences, and still catches one wrong term.  The cost is a sum over
observations in a fixed tree (<= 2^7 per CTA, then the CTA partials): its bar is 2 TAU of the summed magnitudes.
Masked columns and removed observations must be exactly 0.

Worst measured on one H100 80GB HBM3 (power limit 400 W), in eps of m, per family (r / J_intr / J_pose / J_point):
  rotations 0.25 / 0.50 / 0.61 / 0.61    depth 0.35 / 0.50 / 0.32 / 0.40    fisheye 0.15 / 0.39 / 0.13 / 0.13
  radial    0.37 / 0.43 / 0.35 / 0.30    spherical 0.17 / 0 / 0.21 / 0.18   loss 0.30 / 0.32 / 0.28 / 0.34
  weights   0.24 / 0.62 / 0.45 / 0.50    mixed 0.30 / 0.45 / 0.40 / 0.45    masks 0.20 / 0.42 / 0.38 / 0.50
  grid      0.41 / 0.70 / 0.66 / 0.74    priors r 0.12, J 0.18;  norms <= 0.29, cost <= 0.033 of eps m.
With the pose record before its Taylor-branch fix (dR_k X = R (j_k x X) for R = I + [aa]x) the J_pose columns of
the small-angle poses deviated by 7.7e5 (spherical) to 5.7e8 (rotations) eps of m, and 5.1e12 on the grid scene;
every other block stayed below 0.71 eps."""
import json
import os

import numpy as np
import pytest

import ba_eval_reference as er

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
TAU = 4 * EPS
WORST = {}
BLOCKS = (("r", 1), ("J_intr", 2), ("J_pose", 3), ("J_point", 4))
FAMILIES = {"rotations": er.scene_rotations, "depth": er.scene_depth, "fisheye": er.scene_fisheye, "radial": er.scene_radial,
            "spherical": er.scene_spherical, "mixed": er.scene_mixed}


@pytest.fixture(scope="module")
def ba():
    from openmvg_b200 import ba as m
    return m


@pytest.fixture(scope="module", autouse=True)
def _report():
    """OMVG_BA_EVAL_REPORT=<file>: the worst measured deviation per family and block, in eps of m, as JSON."""
    yield
    path = os.environ.get("OMVG_BA_EVAL_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(WORST, f, indent=1, sort_keys=True)


def _check(family, name, got, ref, mag, tau=TAU):
    got = np.asarray(got, np.float64); ref = np.asarray(ref, er.LD); mag = np.asarray(mag, er.LD)
    assert np.isfinite(got).all(), (family, name, "not finite")
    err = np.abs(got.astype(er.LD) - ref)
    zero = mag == 0                                          # masked columns, removed observations: exactly 0
    assert not got[zero].any(), (family, name, "non-zero where the reference is exactly 0", int((got[zero] != 0).sum()))
    ratio = float((err[~zero] / mag[~zero]).max() / EPS) if (~zero).any() else 0.0
    key = f"{family}:{name}"
    if key not in WORST or ratio > WORST[key]:
        WORST[key] = ratio
    bad = err > tau * mag
    if bad.any():
        rows = np.unique(np.nonzero(bad)[0])[:8]
        raise AssertionError(f"{family} {name}: {int(bad.sum())} entries over {tau / EPS:.0f} eps of m, worst {ratio:.3g} eps; rows {rows.tolist()}")


def check_eval(ba, s, family, **opts):
    """debug_eval (+ residual_norms) of scene s against the reference, every block, the cost."""
    ctx = ba.BAContext(s)
    try:
        got = ctx.debug_eval(**opts)
        norms = ctx.residual_norms()
    finally:
        ctx.close()
    o = {k: opts[k] for k in ("intrinsics_opt", "extrinsics_opt", "structure_opt") if k in opts}
    ref = er.evaluate(s, opts.get("use_loss", 1), opts.get("huber_a", 16.0), **o)
    for name, i in BLOCKS:
        _check(family, name, got[i], ref[name], ref["m_" + name])
    _check(family, "norms", norms, ref["norms"], ref["m_norms"])
    _check(family, "cost", got[0], ref["cost"], ref["m_cost"], 2 * TAU)
    return ref


@pytest.mark.parametrize("family", list(FAMILIES))
def test_eval_edges(ba, family):
    ref = check_eval(ba, FAMILIES[family](), family)
    if family in ("rotations", "mixed"):
        assert ref["taylor"].any() and not ref["taylor"].all()


@pytest.mark.parametrize("use_loss,huber_a", [(1, 16.0), (1, 3.5), (0, 16.0)])
def test_eval_loss(ba, use_loss, huber_a):
    check_eval(ba, er.scene_loss(), "loss", use_loss=use_loss, huber_a=huber_a)


@pytest.mark.parametrize("use_loss", [1, 0])
def test_eval_weights_flags_fixed(ba, use_loss):
    """Weights 0 / 1e-3 / 7 / 1e3, no-loss flags and fixed landmarks (the instantiation with the extensions); the
    removed observation behind the camera gives exact zeros."""
    s = er.scene_weights()
    check_eval(ba, s, "weights", use_loss=use_loss)
    ctx = ba.BAContext(s)
    try:
        _, r, Ji, Jc, Jp = ctx.debug_eval(use_loss=use_loss)
    finally:
        ctx.close()
    dead = np.asarray(s["obs_weight"]) == 0
    for a in (r, Ji, Jc, Jp):
        assert np.isfinite(a[dead]).all() and not a[dead].any()


@pytest.mark.parametrize("intrinsics_opt", [1, 2, 4, 8, 6, 10, 12, 14])
def test_eval_masks(ba, intrinsics_opt):
    """Every option mask on the four-model scene: free columns to the bar, masked columns exactly 0."""
    s = er.scene_mixed(per=3)
    for extrinsics_opt in (1, 2, 4, 6):
        for structure_opt in (0, 1):
            check_eval(ba, s, "masks", intrinsics_opt=intrinsics_opt, extrinsics_opt=extrinsics_opt, structure_opt=structure_opt)


def test_eval_grid_stride(ba, monkeypatch):
    """60 001 observations on a one-wave grid: every thread takes several observations through the prefetch."""
    monkeypatch.setenv("OMVG_BA_EVAL_WAVES", "1")
    s = er.scene_grid()
    assert len(s["obs_view"]) % 128 and len(s["obs_view"]) >= 60000
    check_eval(ba, s, "grid")


@pytest.mark.parametrize("extrinsics_opt", [6, 2, 4, 1])
def test_prior_rows(ba, extrinsics_opt):
    """The pose-centre prior rows (omvg_ba_debug_prior), Taylor-branch poses included."""
    s = er.scene_priors()
    ctx = ba.BAContext(s)
    try:
        cost, r, J = ctx.debug_prior(extrinsics_opt=extrinsics_opt)
    finally:
        ctx.close()
    ref = er.evaluate_priors(s, extrinsics_opt)
    _check("priors", "r", r, ref["r"], ref["m_r"])
    _check("priors", "J", J, ref["J"], ref["m_J"])
    _check("priors", "cost", cost, ref["cost"], ref["m_cost"], 2 * TAU)
    assert er.taylor_branch(s["poses"][:, :3]).any()
