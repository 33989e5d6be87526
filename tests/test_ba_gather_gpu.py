"""Camera blocks of the reduced system summed over per-block observation-pair lists (schur_gather_kernel):
cases the lists must get right beyond the one-view-per-pose scenes of test_ba_gpu.py."""
import numpy as np
import pytest

import checkers as ck
from openmvg_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ba():
    from openmvg_b200 import ba as m
    return m


def test_two_views_of_one_pose_see_the_same_landmark(ba):
    """A second view on every pose (a rig whose cameras share one pose) re-observes a third of the landmarks, so one
    landmark has two observations in the same diagonal camera block: both cross terms belong to that block."""
    s = synth.ba_scene(16, 600, 6, seed=7)
    nv = len(s["view_pose"])
    rng = np.random.default_rng(7)
    pick = np.flatnonzero(rng.random(len(s["obs_view"])) < 0.06)                 # observations to repeat through the twin view
    s["view_pose"] = np.ascontiguousarray(np.concatenate([s["view_pose"], s["view_pose"]]).astype(np.int32))
    s["view_intr"] = np.ascontiguousarray(np.concatenate([s["view_intr"], s["view_intr"]]).astype(np.int32))
    s["obs_view"] = np.ascontiguousarray(np.concatenate([s["obs_view"], s["obs_view"][pick] + nv]).astype(np.int32))
    s["obs_point"] = np.ascontiguousarray(np.concatenate([s["obs_point"], s["obs_point"][pick]]).astype(np.int32))
    s["obs_xy"] = np.ascontiguousarray(np.concatenate([s["obs_xy"], s["obs_xy"][pick] + rng.normal(0, 0.5, (len(pick), 2))]))
    g = ba.solve(s)
    o = ck.oracle_ba_solve(s)
    assert g["ok"] and o["usable"]
    assert abs(g["final_cost"] - o["final_cost"]) <= 1e-6 * o["final_cost"], (g["final_cost"], o["final_cost"])
    assert g["iterations"] == o["iterations"]
