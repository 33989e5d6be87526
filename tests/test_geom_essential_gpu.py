"""GPU: the essential-matrix filter (omvg_geom_essential_acransac, DESIGN §3.8) against the oracle: identical inlier
lists, (errorMax, minNFA) to 1e-9, E up to scale to 1e-7; the device five-point solver against the oracle's."""
import numpy as np
import pytest

import checkers_essential as ce
from openmvg_b200 import synth
from test_oracle_geom_essential import GOLD_E, WH, check_same, five_point_samples, gold_inputs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def geometry():
    from openmvg_b200 import geometry as g
    return g


def run(geometry, pairs, iterations):
    off = np.concatenate([[0], np.cumsum([len(p[0]) for p in pairs])]).astype(np.uint64)
    return geometry.essential_acransac(off, np.concatenate([p[0] for p in pairs]).reshape(-1, 2), np.concatenate([p[1] for p in pairs]).reshape(-1, 2),
                                       np.array([p[2] for p in pairs]), np.array([p[3] for p in pairs]), 4.0, iterations)


def test_golden_cases_in_one_launch(geometry):
    """All golden pairs as ONE CSR call, pairs with <= 5 matches included."""
    xs = [gold_inputs(*c[1:]) for c in GOLD_E]
    for x, r, c in zip(xs, run(geometry, xs, 2048), GOLD_E):
        o = ce.oracle_acransac_essential(*x, 4.0, 2048)
        check_same(o, r, c[0])
        if not len(o["inliers"]):
            assert len(r["inliers"]) == 0


@pytest.mark.parametrize("iterations", [64, 2048])
def test_many_pairs_against_oracle(geometry, iterations):
    rng = np.random.default_rng(17)
    pairs = []
    for k in range(60):
        n = int(rng.integers(0, 1200)); of = float(rng.uniform(0.0, 0.7)); motion = ["general", "short", "forward", "planar"][k % 4]
        pairs.append(gold_inputs(n, of, 500 + k, motion))
    kept = 0
    for p, r in zip(pairs, run(geometry, pairs, iterations)):
        o = ce.oracle_acransac_essential(*p, 4.0, iterations)
        check_same(o, r, (len(p[0]), iterations))
        kept += len(o["inliers"]) > 12.5
    assert kept > 20


def test_five_point_solver_against_oracle(geometry):
    for motion, seed in (("general", 1), ("short", 2), ("forward", 3), ("planar", 4)):
        b1, b2 = five_point_samples(2500, 700 + seed, motion)
        d = geometry.debug_five_point(b1, b2); o = ce.oracle_five_point(b1, b2)
        assert np.array_equal(d["n_models"], o["n_models"]), motion
        for s in range(len(b1)):
            k = o["n_models"][s]
            assert ce.same_solution_set(o["E"][s][:k], d["E"][s][:k], 1e-12), (motion, s)


def test_rejections(geometry):
    from openmvg_b200._lib import OmvgError
    xI, xJ, wh, k = gold_inputs(50, 0.2, 1, "general")
    with pytest.raises(OmvgError):
        geometry.essential_acransac([0, 50], xI, xJ, [wh], [k], precision=float("inf"))
    bad = k.copy(); bad[3] = 0.0
    with pytest.raises(OmvgError):
        geometry.essential_acransac([0, 50], xI, xJ, [wh], [bad])
    bad = k.copy(); bad[0] = -5.0
    with pytest.raises(OmvgError):
        geometry.essential_acransac([0, 50], xI, xJ, [wh], [bad])
    from openmvg_b200._lib import lib
    import ctypes
    off = np.array([0, 50], np.uint64); sz = np.array([wh], np.int32)
    out = [np.zeros(50, np.uint32), np.zeros(1, np.uint32), np.zeros(9), np.zeros(2)]
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    rc = lib().omvg_geom_essential_acransac(0, ctypes.c_uint64(1), p(off), p(xI), p(xJ), p(sz), None, ctypes.c_double(4.0),
                                            ctypes.c_uint32(2048), *[p(a) for a in out])
    assert rc != 0
    # the model-as-argument entry has no intrinsics: it keeps rejecting the essential model
    rc = lib().omvg_geom_acransac(0, 2, ctypes.c_uint64(1), p(off), p(xI), p(xJ), p(sz), ctypes.c_double(4.0), ctypes.c_uint32(2048), *[p(a) for a in out])
    assert rc != 0
