"""CPU: guided matching's oracle (oracle/guided_oracle.cpp, DESIGN §3.9) against the reference's own
geometry_aware::GuidedMatching (oracle/_ref/libref_guided.so, or its recorded answers in
tests/golden/reference_calls_guided.pkl.gz), list for list."""
import numpy as np
import pytest

import checkers_guided as cg
from openmvg_b200 import synth

pytestmark = pytest.mark.skipif(not cg.have_ref_guided(replay=True), reason="no reference guided matching and no recorded answers")

EPI, TRANSFER = 0, 1
RATIOS = [0.36, 0.64, 1.0, -1.0]          # Square(0.6), Square(0.8), 1, the descriptor-free variant


def _scene(counts, seed, planar=False, n_dup=0):
    return synth.guided_scene(len(counts), counts, seed=seed, planar=planar, n_dup=n_dup)


def _model(s, model, a, b):
    return synth.scene_fundamental(s, a, b) if model == EPI else synth.scene_homography(s, a, b)


def _same(model, xI, dI, xJ, dJ, M, thr, ratio, camI=None, camJ=None, uI=None, uJ=None):
    ref = cg.ref_guided(model, xI, dI, xJ, dJ, M, thr, ratio, camI, camJ)
    ora = cg.oracle_guided(model, xI if uI is None else uI, dI, xJ if uJ is None else uJ, dJ, M, thr, ratio)
    assert np.array_equal(ref, ora), f"{len(ref)} reference matches vs {len(ora)} oracle matches"
    return ref


# golden pairs: (name, counts, seed, planar, duplicated coordinates)
GOLD = [("v900_v700", [900, 700], 11, False, 0), ("v1500_v1200_dups", [1500, 1200], 12, False, 40),
        ("planar_800_800", [800, 800], 13, True, 0), ("planar_600_900_dups", [600, 900], 14, True, 25)]


@pytest.mark.parametrize("model", [EPI, TRANSFER])
@pytest.mark.parametrize("ratio", RATIOS)
@pytest.mark.parametrize("name,counts,seed,planar,dups", GOLD, ids=[g[0] for g in GOLD])
def test_golden_pairs(name, counts, seed, planar, dups, model, ratio):
    s = _scene(counts, seed, planar, dups)
    thr = 4.0 if model == EPI else 9.0
    m = _same(model, s["xy"][0], s["desc"][0], s["xy"][1], s["desc"][1], _model(s, model, 0, 1), thr, ratio)
    if planar or model == EPI:
        assert len(m) > 0


@pytest.mark.parametrize("seed", range(6))
def test_seeded_random_pairs(seed):
    rng = np.random.default_rng(1000 + seed)
    counts = [int(rng.integers(50, 1200)), int(rng.integers(50, 1200))]
    planar = bool(seed % 2)
    s = _scene(counts, 2000 + seed, planar, int(rng.integers(0, 20)))
    for model in (EPI, TRANSFER):
        thr = float(rng.uniform(1.0, 25.0))
        M = _model(s, model, 0, 1) if (model == EPI or planar) else rng.normal(size=(3, 3))
        for ratio in RATIOS:
            _same(model, s["xy"][0], s["desc"][0], s["xy"][1], s["desc"][1], M, thr, ratio)


@pytest.mark.parametrize("nI,nJ", [(0, 300), (300, 0), (0, 0), (1, 400), (400, 1)])
def test_empty_and_single_feature_images(nI, nJ):
    s = _scene([max(nI, 1), max(nJ, 1)], 21)
    xI, dI, xJ, dJ = s["xy"][0][:nI], s["desc"][0][:nI], s["xy"][1][:nJ], s["desc"][1][:nJ]
    for model in (EPI, TRANSFER):
        for ratio in RATIOS:
            m = _same(model, xI, dI, xJ, dJ, _model(s, EPI, 0, 1) if model == EPI else np.eye(3), 1e4, ratio)
            if min(nI, nJ) == 0 or (nJ == 1 and ratio >= 0):
                assert len(m) == 0                                      # no second distance: never valid


def test_radial_view_undistorted_positions():
    """The reference un-distorts with Pinhole_Intrinsic_Radial_K1::get_ud_pixel; the oracle takes those positions."""
    s = _scene([900, 800], 31)
    camI = np.array([1600, 1200, 1700, 810, 590, 0.03]); camJ = np.array([1600, 1200, 1500, 790, 610, -0.02])
    uI, uJ = cg.ref_ud_pixels(camI, s["xy"][0]), cg.ref_ud_pixels(camJ, s["xy"][1])
    assert np.abs(uI - s["xy"][0]).max() > 1.0
    F = _model(s, EPI, 0, 1)
    for ratio in RATIOS:
        _same(EPI, s["xy"][0], s["desc"][0], s["xy"][1], s["desc"][1], F, 25.0, ratio, camI, camJ, uI, uJ)


@pytest.mark.parametrize("model", [EPI, TRANSFER])
def test_threshold_equal_to_a_candidate_error_excludes_it(model):
    s = _scene([400, 500], 41, planar=True)
    M = _model(s, model, 0, 1)
    xI, xJ = s["xy"][0], s["xy"][1]
    m = cg.oracle_guided(model, xI, s["desc"][0], xJ, s["desc"][1], M, 9.0, -1.0)
    i, j = (int(v) for v in m[len(m) // 2])
    e = float(cg.oracle_guided_errors(model, M, xI[i:i + 1], xJ[j:j + 1])[0])
    assert e == float(cg.ref_guided_errors(model, M, xI[i:i + 1], xJ[j:j + 1])[0]) and e > 0
    at = _same(model, xI, s["desc"][0], xJ, s["desc"][1], M, e, -1.0)
    assert not any(r[0] == i and r[1] == j for r in at)               # err < thr is strict
    above = _same(model, xI, s["desc"][0], xJ, s["desc"][1], M, float(np.nextafter(e, np.inf)), -1.0)
    assert any(r[0] == i and r[1] == j for r in above)


def test_descriptor_ties_and_geometry_ties():
    """Equal descriptor distances give sbd == bd (rejected); an exact position duplicate in J ties the geometric error
    and the lowest j wins in the descriptor-free variant."""
    s = _scene([300, 300], 51, planar=True)
    xJ, dJ = s["xy"][1].copy(), s["desc"][1].copy()
    xJ = np.concatenate([xJ, xJ[:150]]); dJ = np.concatenate([dJ, dJ[:150]])      # rows 300.. repeat rows 0..149
    for model in (EPI, TRANSFER):
        M = _model(s, model, 0, 1)
        with_desc = _same(model, s["xy"][0], s["desc"][0], xJ, dJ, M, 16.0, 1.0)
        assert not any(j < 150 or j >= 300 for _, j in with_desc)
        geo = _same(model, s["xy"][0], s["desc"][0], xJ, dJ, M, 16.0, -1.0)
        assert len(geo) and not any(j >= 300 for _, j in geo)


@pytest.mark.parametrize("model", [EPI, TRANSFER])
@pytest.mark.parametrize("seed", [61, 62])
def test_error_functions_bit_for_bit(model, seed):
    """EpipolarDistanceError / AsymmetricError as the reference's build rounds them (one FMA per row of M [x; 1])."""
    s = _scene([700, 600], seed, planar=True)
    rng = np.random.default_rng(seed)
    xI = s["xy"][0][rng.integers(0, 700, 5000)]; xJ = s["xy"][1][rng.integers(0, 600, 5000)]
    for M in (_model(s, model, 0, 1), rng.normal(size=(3, 3))):
        ref, ora = cg.ref_guided_errors(model, M, xI, xJ), cg.oracle_guided_errors(model, M, xI, xJ)
        assert np.array_equal(ref.view(np.uint64), ora.view(np.uint64))
