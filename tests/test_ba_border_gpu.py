"""The intrinsics border, the camera right-hand side and the intrinsics corner are sums in a fixed order (per pose over
its observations grouped by intrinsic group, per group over its landmarks): poses seen through two intrinsic groups
against the oracle, and bitwise reproducible solves where no order-dependent sum is left."""
import numpy as np
import pytest

import checkers as ck
from openmvg_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ba():
    from openmvg_b200 import ba as m
    return m


def _two_group_scene(n_cams, n_points, obs_per_point, seed):
    """Every pose has a second view with its own pinhole group (focal length 30 px longer); every third landmark is seen
    through the second views only, so each landmark keeps one group and most poses see landmarks of both groups.
    Observations are re-projected through the oracle at the initial parameters, plus 0.5 px noise; then the landmarks
    are perturbed."""
    s = synth.ba_scene(n_cams, n_points, obs_per_point, seed=seed)
    intr = np.repeat(s["intrinsics"][:1], 2, axis=0); intr[1, 0] += 30.0
    second = s["obs_point"] % 3 == 0
    s.update(intrinsics=np.ascontiguousarray(intr), intr_model=np.full(2, 1, np.int32),
             view_pose=np.tile(np.arange(n_cams, dtype=np.int32), 2), view_intr=np.repeat(np.arange(2, dtype=np.int32), n_cams),
             obs_view=np.ascontiguousarray(s["obs_view"] + np.where(second, n_cams, 0)).astype(np.int32), obs_xy=np.zeros_like(s["obs_xy"]))
    proj = ck.oracle_ba_eval(s, use_loss=0)[1]                  # residual = projection - observation (0)
    rng = np.random.default_rng(seed)
    s["obs_xy"] = np.ascontiguousarray(proj + rng.normal(0, 0.5, proj.shape))
    s["points"] = np.ascontiguousarray(s["points"] + rng.normal(0, 0.01, s["points"].shape))
    return s


@pytest.mark.parametrize("cfg", [(24, 1200, 6), (60, 3000, 8), (120, 4000, 8)])   # direct solve, explicit inverse, PCG
def test_poses_seen_through_two_groups(ba, cfg):
    s = _two_group_scene(*cfg, seed=cfg[0])
    pose_groups = np.zeros((cfg[0], 2), bool)
    pose_groups[s["view_pose"][s["obs_view"]], s["view_intr"][s["obs_view"]]] = True
    assert pose_groups.all(axis=1).mean() > 0.9
    g = ba.solve(s)
    o = ck.oracle_ba_solve(s)
    assert g["ok"] and o["usable"]
    assert abs(g["final_cost"] - o["final_cost"]) <= 1e-6 * o["final_cost"], (g["final_cost"], o["final_cost"])
    assert g["iterations"] == o["iterations"]


@pytest.mark.parametrize("cams", [20, 60])                      # dense_solve_kernel; the explicit inverse
def test_direct_path_solve_is_bitwise_reproducible(ba, cams):
    """With tracks of at most 32 views and one intrinsic group every sum of a direct-path solve runs in a fixed order
    (back-substitution adds at most two warp partials per landmark, which commute): two runs agree bit for bit."""
    s = synth.ba_scene(cams, 50 * cams, 8, seed=11 + cams)
    ctx = ba.BAContext(s)
    a = ctx.run(); pa = ctx.download()
    ctx.reset()
    b = ctx.run(); pb = ctx.download()
    ctx.close()
    assert a["ok"] and a["pcg_iterations"] == 0
    assert a["iterations"] == b["iterations"] and a["final_cost"] == b["final_cost"]
    for x, y in zip(pa, pb):
        assert x.tobytes() == y.tobytes()
