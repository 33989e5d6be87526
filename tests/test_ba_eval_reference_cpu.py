"""CPU: the extended-precision evaluation reference (tests/ba_eval_reference.py) against the oracle, whose double jets
restate Ceres' expressions (oracle_ba_eval, oracle_ba_cost), on the edge scenes of the GPU evaluation check; and a
numpy model of the compact per-pose record of cam_prep_kernel, which shows why its Taylor branch needs e_k x X.

Bar: |oracle - reference| <= TAU m per entry, m the entry's magnitude.  The oracle evaluates the same expressions in
double: each operation rounds once (<= eps/2 of its result, which m carries forward term by term), and libm's
sin / cos / atan / atan2 are within an ulp, so a correct oracle stays below about 1 eps m (0.61 measured over all
scenes and loss settings of this file).  TAU = 4 eps."""
import numpy as np
import pytest

import ba_eval_reference as er
import checkers as ck

EPS = np.finfo(np.float64).eps
TAU = 4 * EPS
SCENES = {"rotations": er.scene_rotations, "depth": er.scene_depth, "fisheye": er.scene_fisheye, "radial": er.scene_radial,
          "spherical": er.scene_spherical, "loss": er.scene_loss, "weights": er.scene_weights, "mixed": er.scene_mixed,
          "priors": er.scene_priors}


def oracle_eval(s, use_loss=1, huber_a=16.0):
    """(rows, r, J_intr, J_pose, J_point) of the oracle with the scene's weights, no-loss flags and fixed landmarks
    applied by hand (oracle_ba_eval takes the plain problem).  Weighting after the evaluation is exact only where no
    loss applies or the weight is 0 or 1: `rows` marks those (the cost, from oracle_ba_cost_ex, covers the others)."""
    plain = {k: v for k, v in s.items() if k not in ("obs_weight", "obs_no_loss", "point_fixed", "prior_pose")}
    if s.get("obs_weight") is None:
        return (np.ones(len(s["obs_view"]), bool),) + ck.oracle_ba_eval(plain, use_loss, huber_a)[1:]
    a = ck.oracle_ba_eval(plain, use_loss, huber_a)
    b = ck.oracle_ba_eval(plain, 0, huber_a)
    nl = np.asarray(s["obs_no_loss"]).astype(bool); w = np.asarray(s["obs_weight"], np.float64)
    out = []
    for x, y in zip(a[1:], b[1:]):
        sh = (-1,) + (1,) * (x.ndim - 1)
        out.append(np.where(nl.reshape(sh), y, x) * w.reshape(sh))
    out[3] = out[3] * (~np.asarray(s["point_fixed"]).astype(bool))[s["obs_point"]][:, None, None]
    return (nl | (use_loss == 0) | (w == 0) | (w == 1),) + tuple(out)


def _within(name, got, ref, mag, tau=TAU):
    got = np.asarray(got, np.float64); ref = np.asarray(ref, er.LD); mag = np.asarray(mag, er.LD)
    assert np.isfinite(got).all(), name
    err = np.abs(got.astype(er.LD) - ref)
    bad = err > tau * mag
    assert not bad.any(), (name, int(bad.sum()), float((err / np.maximum(mag, 1e-300)).max() / EPS), "eps of m")


@pytest.mark.parametrize("name", list(SCENES))
@pytest.mark.parametrize("use_loss,huber_a", [(1, 16.0), (1, 3.5), (0, 16.0)])
def test_reference_matches_oracle(name, use_loss, huber_a):
    s = SCENES[name]()
    ref = er.evaluate(s, use_loss, huber_a)
    rows, r, Ji, Jc, Jp = oracle_eval(s, use_loss, huber_a)
    for k, got in (("r", r), ("J_intr", Ji), ("J_pose", Jc), ("J_point", Jp)):
        _within(f"{name}:{k}", got[rows], ref[k][rows], ref["m_" + k][rows])
    cost = ck.oracle_ba_cost({k: v for k, v in s.items() if k != "prior_pose"}, use_loss=use_loss, huber_a=huber_a)
    assert abs(cost - float(ref["cost"])) <= TAU * float(ref["m_cost"]), (name, cost, float(ref["cost"]))
    if name == "rotations":
        assert ref["taylor"].any() and not ref["taylor"].all()


def test_edge_scene_coverage():
    """The scenes reach the edges they are built for."""
    for th in er.ROT_ANGLES:
        t2 = th * th
        assert abs(t2 - er.DBL_EPSILON) > 4 * np.spacing(er.DBL_EPSILON)      # branch decided the same in every build
    assert set(er.TAYLOR_ANGLES) == {0.0, 1e-12, 1e-10, 1e-9, 1.2e-8}
    s = er.scene_rotations()
    taylor = er.taylor_branch(s["poses"][:, :3])
    th = np.linalg.norm(s["poses"][:, :3], axis=1)
    assert np.array_equal(taylor, th * th <= er.DBL_EPSILON)
    assert ((th > 3.14) & (th < 3.15)).sum() == 2 and (th > 2 * np.pi).sum() == 1
    # fisheye: r = 0 exactly and both sides of r = 1e-8
    s = er.scene_fisheye(); p = s["points"][:7]
    r = np.hypot(p[:, 0] / p[:, 2], p[:, 1] / p[:, 2])
    assert (r == 0).sum() == 2 and (r > 1e-8).sum() == 3 and ((r > 0) & (r < 1e-8)).sum() == 2
    # Huber: |r|^2 within 1e-9 of a^2 on both sides
    ref = er.evaluate(er.scene_loss(), use_loss=0)
    s2 = (ref["r"].astype(np.float64) ** 2).sum(1)
    for a in (16.0, 3.5):
        q = s2 / a ** 2 - 1
        assert ((q > 0) & (q < 2e-9)).sum() >= 4 and ((q < 0) & (q > -2e-9)).sum() >= 4
    # landmarks far from the origin: the projection cancels
    s = er.scene_depth()
    assert np.abs(s["points"]).max() > 9e3
    assert er.scene_grid(n_obs=1000)["obs_view"].size == 1000


def test_prior_reference_matches_oracle_cost():
    """Pose-centre prior rows (Taylor-branch poses included): the cost of the reference equals the oracle's; the
    reference J equals central differences of the reference residual in long double."""
    s = er.scene_priors()
    pr = er.evaluate_priors(s)
    obs = er.evaluate(s)
    want = ck.oracle_ba_cost(s)
    got = float(obs["cost"] + pr["cost"])
    assert abs(got - want) <= TAU * float(obs["m_cost"] + pr["m_cost"]), (got, want)
    assert (np.abs(pr["r"]).max(1) > 0).all()
    # the Huber tail is reached by some rows and not by others
    n2 = (pr["r"].astype(np.float64) ** 2).sum(1)
    assert (n2 < s["prior_huber_a"] ** 2).any()
    # extrinsics masks: masked columns exactly zero
    for ext, cols in ((1, []), (2, [0, 1, 2]), (4, [3, 4, 5])):
        J = er.evaluate_priors(s, extrinsics_opt=ext)["J"]
        off = [c for c in range(6) if c not in cols]
        assert not J[:, :, off].any()


@pytest.mark.parametrize("theta", er.ROT_ANGLES)
def test_pose_record_model(theta):
    """dR_k X from the compact record.  R' dR_k is skew only for a rotation; in the Taylor branch R = I + [aa]x is not
    one, and R (j_k x X) misses Ceres' derivative e_k x X by O(theta).  The fixed record (Jr = I, e_k x X) is exact."""
    rng = np.random.default_rng(int(theta * 1e3) % 1000)
    a = rng.normal(size=3); a /= np.linalg.norm(a)
    aa = theta * a
    X = rng.normal(size=3) * 5
    # Ceres' derivative: the jets of AngleAxisRotatePoint in long double
    E = [er.Jet.var(np.array([aa[k]]), er.KI + k) for k in range(3)]
    P = [er.Jet.const(X[i], 1) for i in range(3)]
    out = er.rotate(E, P, er.taylor_branch(aa[None]))
    want = np.array([[float(out[i].v[0, er.KI + k]) for k in range(3)] for i in range(3)])
    mag = np.array([[float(out[i].mv[0, er.KI + k]) for k in range(3)] for i in range(3)])
    old = er.record_model(aa, fixed=False)(X)
    new = er.record_model(aa, fixed=True)(X)
    scale = np.abs(X).sum()
    err_old = np.abs(old - want).max() / scale
    err_new = np.abs(new - want).max() / scale
    if theta not in er.TAYLOR_ANGLES:
        # outside the Taylor branch R is a rotation and the record's R (j_k x X) is Ceres' derivative to rounding:
        # within 8 eps of the magnitude of Ceres' own double evaluation of it (which grows as 1/theta just above
        # the branch switch, where 1 - cos theta cancels)
        err = np.abs(new - want)
        assert (err <= 8 * EPS * (mag + scale)).all(), (theta, float((err / (mag + scale)).max() / EPS))
        return
    assert err_new <= 8 * EPS, (theta, err_new)
    if theta >= 1e-10:
        assert err_old >= 0.1 * theta, (theta, err_old)                    # the defect: O(theta), not rounding
    if theta == 0.0:
        assert err_old <= 8 * EPS, (theta, err_old)                        # aa = 0: R = I, the old record was exact
