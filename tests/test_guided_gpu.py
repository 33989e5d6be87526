"""GPU: guided matching (omvg_match_guided_run, DESIGN §3.9) against the oracle (oracle/guided_oracle.cpp, pinned to the
reference by tests/test_oracle_guided.py): CSR bit-identical, every collection in ONE guided_run call."""
import numpy as np
import pytest

import checkers_guided as cg
from openmvg_b200 import matching, synth
from openmvg_b200._lib import OmvgError

pytestmark = pytest.mark.gpu

EPI, TRANSFER = matching.GUIDED_EPIPOLAR, matching.GUIDED_TRANSFER
COUNTS = [0, 1, 2, 127, 128, 129, 900, 3000, 5000, 5000]
E_ARG, E_STATE = -1, -3


def _pairs(n_img, n, seed):
    rng = np.random.default_rng(seed)
    fixed = [(8, 9), (9, 8), (0, 5), (5, 0), (1, 6), (6, 1), (2, 3), (3, 4), (4, 5), (7, 8)]
    rest = [tuple(int(v) for v in rng.choice(n_img, 2, replace=False)) for _ in range(n - len(fixed))]
    pi, pj = zip(*(fixed + rest))
    return np.array(pi, np.uint32), np.array(pj, np.uint32)


def _load(s):
    ctx = matching.MatchContext(0)
    ctx.load(s["desc"])
    for k, xy in enumerate(s["xy"]):
        ctx.upload_positions(k, xy)
    return ctx


def _models(s, model, pi, pj, seed):
    rng = np.random.default_rng(seed)
    M = np.stack([synth.scene_fundamental(s, a, b) if model == EPI else synth.scene_homography(s, a, b) for a, b in zip(pi, pj)])
    thr = rng.uniform(2.0, 20.0, len(pi))
    return M, thr


def _check(ctx, s, model, pi, pj, M, thr, ratio):
    ctx.guided_run(pi, pj, M, thr, ratio, model)
    off, ij = ctx.fetch()
    ooff, oij = cg.oracle_guided_collection(model, s["xy"], s["desc"], pi, pj, M, thr, ratio)
    assert np.array_equal(off, ooff), "per-pair match counts differ"
    assert np.array_equal(ij, oij), "matches differ"
    return off, ij


@pytest.fixture(scope="module")
def scene():
    return synth.guided_scene(len(COUNTS), COUNTS, seed=101, n_dup=30)


@pytest.fixture(scope="module")
def planar():
    return synth.guided_scene(len(COUNTS), COUNTS, seed=102, planar=True, n_dup=30)


@pytest.mark.parametrize("ratio", [0.36, 0.64, 1.0, -1.0])
def test_epipolar_collection(scene, ratio):
    pi, pj = _pairs(len(COUNTS), 40, 7)
    M, thr = _models(scene, EPI, pi, pj, 8)
    ctx = _load(scene)
    off, ij = _check(ctx, scene, EPI, pi, pj, M, thr, ratio)
    ctx.close()
    assert len(ij) > 1000 and off[1] > off[0]                      # the 5000 x 5000 pair has matches


@pytest.mark.parametrize("ratio", [0.36, 1.0, -1.0])
def test_transfer_planar_collection(planar, ratio):
    pi, pj = _pairs(len(COUNTS), 40, 9)
    M, thr = _models(planar, TRANSFER, pi, pj, 10)
    ctx = _load(planar)
    _, ij = _check(ctx, planar, TRANSFER, pi, pj, M, thr, ratio)
    ctx.close()
    assert len(ij) > 1000


@pytest.mark.parametrize("model", [EPI, TRANSFER])
def test_strict_threshold_boundary(planar, model):
    """A threshold equal to a candidate's error excludes it; the next double up includes it."""
    a, b = 6, 7
    M = synth.scene_fundamental(planar, a, b) if model == EPI else synth.scene_homography(planar, a, b)
    m = cg.oracle_guided(model, planar["xy"][a], planar["desc"][a], planar["xy"][b], planar["desc"][b], M, 9.0, -1.0)
    picks = m[:: max(1, len(m) // 8)][:8]
    errs = [float(cg.oracle_guided_errors(model, M, planar["xy"][a][i:i + 1], planar["xy"][b][j:j + 1])[0]) for i, j in picks]
    thr = np.array([v for e in errs for v in (e, np.nextafter(e, np.inf))])
    pi = np.full(len(thr), a, np.uint32); pj = np.full(len(thr), b, np.uint32)
    ctx = _load(planar)
    off, ij = _check(ctx, planar, model, pi, pj, np.stack([M] * len(thr)), thr, -1.0)
    ctx.close()
    for k, (i, j) in enumerate(picks):
        at, up = ij[off[2 * k]:off[2 * k + 1]], ij[off[2 * k + 1]:off[2 * k + 2]]
        assert not any((r == (i, j)).all() for r in at)
        assert any((r == (i, j)).all() for r in up)


def test_ties_and_single_candidates(planar):
    """Rows of J repeated exactly (position and descriptor): equal distances are rejected by the ratio test, a lone
    candidate is rejected, and the descriptor-free variant keeps the lowest j of the tied errors."""
    s = {k: list(v) if isinstance(v, list) else v for k, v in planar.items()}
    n = len(s["xy"][7])
    s["xy"].append(np.concatenate([s["xy"][7], s["xy"][7][: n // 2]]))            # a copy of view 7, half its rows twice
    s["desc"].append(np.concatenate([s["desc"][7], s["desc"][7][: n // 2]]))
    s["K"].append(s["K"][7]); s["R"].append(s["R"][7]); s["C"].append(s["C"][7])
    last = len(s["xy"]) - 1
    pi = np.array([5, 6, 8, 5], np.uint32); pj = np.array([last, last, last, 1], np.uint32)
    ctx = _load(s)
    for model in (EPI, TRANSFER):
        M, thr = _models(s, model, pi, pj, 11)
        off, ij = _check(ctx, s, model, pi, pj, M, thr, 1.0)
        assert off[4] == off[3]                                     # image 1 has one feature: never a second distance
        assert not np.any(ij[:off[3], 1] < n // 2) and not np.any(ij[:off[3], 1] >= n)   # tied rows never match
        off, ij = _check(ctx, s, model, pi, pj, M, thr, -1.0)
        assert off[3] > 0 and not np.any(ij[:off[3], 1] >= n)       # the lowest j of a geometric tie wins
    ctx.close()


def test_several_batches(scene, monkeypatch):
    pi, pj = _pairs(len(COUNTS), 40, 12)
    M, thr = _models(scene, EPI, pi, pj, 13)
    ctx = _load(scene)
    ctx.guided_run(pi, pj, M, thr, 0.36, EPI); off1, ij1 = ctx.fetch(); ctx.close()
    monkeypatch.setenv("OMVG_MATCH_K12_MB", "0")                   # 0 MB => one pair per batch
    ctx = _load(scene)
    ctx.guided_run(pi, pj, M, thr, 0.36, EPI); off2, ij2 = ctx.fetch(); ctx.close()
    assert np.array_equal(off1, off2) and np.array_equal(ij1, ij2)


def test_match_run_unchanged_by_guided_run(scene):
    pi, pj = _pairs(len(COUNTS), 20, 14)
    ctx = _load(scene)
    ctx.run(pi, pj, 0.8); off1, ij1 = ctx.fetch()
    M, thr = _models(scene, EPI, pi, pj, 15)
    ctx.guided_run(pi, pj, M, thr, 0.36, EPI); ctx.fetch()
    ctx.run(pi, pj, 0.8); off2, ij2 = ctx.fetch()
    ctx.close()
    assert np.array_equal(off1, off2) and np.array_equal(ij1, ij2)


def _code(fn):
    with pytest.raises(OmvgError) as e:
        fn()
    return e.value.code


def test_bad_input_rejected(scene):
    pi, pj = np.array([6], np.uint32), np.array([7], np.uint32)
    M, thr = _models(scene, EPI, pi, pj, 16)
    ctx = matching.MatchContext(0)
    ctx.set_images([len(x) for x in scene["xy"]])
    for k, d in enumerate(scene["desc"]):
        ctx.upload_host(k, d)
    ctx.upload_positions(6, scene["xy"][6])
    assert _code(lambda: ctx.guided_run(pi, pj, M, thr, 0.36)) == E_STATE          # before prepare
    ctx.prepare()
    assert _code(lambda: ctx.guided_run(pi, pj, M, thr, 0.36)) == E_STATE          # image 7 has no positions
    ctx.upload_positions(7, scene["xy"][7])
    assert _code(lambda: ctx.guided_run(pi, np.array([len(COUNTS)], np.uint32), M, thr, 0.36)) == E_ARG
    bad = M.copy(); bad[0, 1, 1] = np.inf
    assert _code(lambda: ctx.guided_run(pi, pj, bad, thr, 0.36)) == E_ARG
    bad[0, 1, 1] = np.nan
    assert _code(lambda: ctx.guided_run(pi, pj, bad, thr, 0.36)) == E_ARG
    assert _code(lambda: ctx.guided_run(pi, pj, M, [np.inf], 0.36)) == E_ARG
    assert _code(lambda: ctx.guided_run(pi, pj, M, [np.nan], 0.36)) == E_ARG
    assert _code(lambda: ctx.guided_run(pi, pj, M, thr, float("nan"))) == E_ARG
    assert _code(lambda: ctx.guided_run(pi, pj, M, thr, 0.36, error_model=2)) == E_ARG
    ctx.guided_run(pi, pj, M, thr, 0.36)                                          # and now it runs
    off, ij = ctx.fetch()
    ctx.close()
    ooff, oij = cg.oracle_guided_collection(EPI, scene["xy"], scene["desc"], pi, pj, M, thr, 0.36)
    assert np.array_equal(off, ooff) and np.array_equal(ij, oij)
