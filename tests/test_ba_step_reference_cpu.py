"""CPU: the extended-precision LM-step reference (tests/ba_step_reference.py) from the oracle's Jacobian.
The reduced solve plus back-substitution equals a dense solve of the unreduced system, and the first step at
initial_radius reproduces the oracle's own first step (its candidate cost and model cost change), which ties the
reference's scaling, clamps, signs and masks to the oracle and through it to Ceres."""
import numpy as np
import pytest

import ba_step_reference as bref
import checkers as ck
from openmvg_b200 import synth

OPTION_MIXES = [
    dict(),
    dict(intrinsics_opt=1, extrinsics_opt=6, structure_opt=1),
    dict(intrinsics_opt=14, extrinsics_opt=4, structure_opt=1),
    dict(intrinsics_opt=2, extrinsics_opt=2, structure_opt=1),
    dict(intrinsics_opt=14, extrinsics_opt=6, structure_opt=0),
    dict(intrinsics_opt=1, extrinsics_opt=1, structure_opt=1),
    dict(use_loss=0),
]


def oracle_jacobian(s, use_loss=1):
    """(r, J_intr, J_pose, J_point) as the GPU's debug_eval returns them: for a scene with control points the
    oracle's plain evaluation, weighted by hand, without the loss on flagged observations, no columns for fixed points."""
    if not ck.has_ext(s):
        return ck.oracle_ba_eval(s, use_loss=use_loss)[1:]
    plain = {k: v for k, v in s.items() if k not in ("obs_weight", "obs_no_loss", "point_fixed")}
    a = ck.oracle_ba_eval(plain, use_loss=use_loss)[1:]
    b = ck.oracle_ba_eval(plain, use_loss=0)[1:]
    nl = np.asarray(s["obs_no_loss"]).astype(bool)
    w = np.asarray(s["obs_weight"], np.float64)
    out = []
    for x, y in zip(a, b):
        x = np.where(nl.reshape((-1,) + (1,) * (x.ndim - 1)), y, x) * w.reshape((-1,) + (1,) * (x.ndim - 1))
        out.append(x)
    out[3] = out[3] * (~np.asarray(s["point_fixed"]).astype(bool))[s["obs_point"]][:, None, None]
    return tuple(out)


def _scenes():
    for model in (1, 4, 3):
        for k, opts in enumerate(OPTION_MIXES):
            if model != 1 and k not in (0, 4):
                continue
            yield f"model{model}-mix{k}", dict(model=model), opts
    yield "gcp", dict(gcp=True), dict()


@pytest.mark.parametrize("name,scene,opts", list(_scenes()), ids=[n for n, _, _ in _scenes()])
def test_reduced_step_equals_unreduced_solve(name, scene, opts):
    s = synth.ba_scene(6, 80, 4, seed=3, model=scene.get("model", 1), outlier_frac=0.05)
    if scene.get("gcp"):
        s = synth.add_gcp(s, 4, weight=9.0)
    r, Ji, Jc, Jp = oracle_jacobian(s, opts.get("use_loss", 1))
    ref = bref.StepReference(s, r, Ji, Jc, Jp, 1e4, **opts)
    dp, dr, z = ref.step()
    up, ur = bref.unreduced_step(ref)
    d = np.concatenate([dp.ravel(), dr]); u = np.concatenate([up.ravel(), ur])
    assert np.abs(u).max() > 0
    err = float(np.abs(d - u).max() / np.abs(u).max())
    assert err <= 1e-10, (name, err)
    if not opts.get("structure_opt", 1):
        assert not dp.any()

    # the first step of the oracle at initial_radius: candidate cost and model cost change
    o = ck.oracle_ba_solve(s, **opts)
    tr = o["trace"]
    assert len(tr) >= 2 and tr[1][3] > 0, tr[:2]                    # a successful first step
    poses, intr, pts = ref.candidate(dp, dr)
    cand = ck.oracle_ba_cost(dict(s, poses=poses, intrinsics=intr, points=pts), use_loss=opts.get("use_loss", 1))
    assert abs(cand - tr[1][0]) <= 1e-12 * tr[1][0], (name, cand, tr[1][0])
    model = float(ref.model_change(dp, dr))
    want = tr[1][1] / tr[1][3]
    assert abs(model - want) <= 1e-8 * abs(want), (name, model, want)


def test_reference_identity_rows_and_masks():
    """Constant coordinates of the reduced system are identity rows with a zero right-hand side; intrinsic slots
    past a model's parameter count are constant."""
    s = synth.ba_scene(6, 80, 4, seed=3, model=2)
    r, Ji, Jc, Jp = oracle_jacobian(s)
    ref = bref.StepReference(s, r, Ji, Jc, Jp, 1e4, intrinsics_opt=2, extrinsics_opt=4)
    const = np.flatnonzero(~ref.free_r)
    assert len(const) == 6 * 3 + 7                                   # rotations of 6 poses (18), 7 of 8 intrinsic slots
    S = ref.S
    assert np.all(S[const][:, const] == np.eye(len(const))) and not ref.b[const].any()
    mask = np.ones(ref.nd, bool); mask[const] = False
    assert not S[const][:, mask].any() and not S[mask][:, const].any()
    assert np.all(np.linalg.eigvalsh(S.astype(np.float64)) > 0)
