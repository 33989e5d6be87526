"""One LM step of the GPU BA path taken apart (omvg_ba_debug_step) and every stage checked against the extended-precision
reference of tests/ba_step_reference.py, fed the GPU's own r and J (debug_eval) so that a failure names the stage:

  stage              compared with                                   bar
  scale, lm_diag     reference from the same J (free columns)        BAR_VEC relative, elementwise
  S, rhs             reference S, b                                  per 6x6 / 6x8 / 8x8 block: BAR_S x the largest sum of
                                                                     |terms| in its block row; exactly 0 where two poses
                                                                     share no landmark; identity rows bit for bit
  z                  the GPU's own S, rhs                            direct L D L': normwise backward error <= BAR_LDLT;
                                                                     explicit inverse: forward error against z* <= 100 kappa eps;
                                                                     PCG: the residual bound its stopping rule guarantees
  step_point         reference back-substitution of the GPU's z      BAR_STEP relative per landmark block; constant landmarks 0
  model change       reference model change of the GPU's step        BAR_MODEL relative
  whole chain        reference step from the reference S, b          forward error <= 10 kappa(S) (eta_S + eta_b + eta_solve)

Worst measured on one H100 80GB HBM3 (SXM, 700 W) over all cases of this file, against the bar:
  scale 3.4e-16, lm_diag 4.6e-16 (1e-14);  S 2.8e-14, rhs 3.3e-14 (1e-12);  L D L' backward error 2.7e-16 (1e-14);
  explicit inverse 1.6 kappa eps (100 kappa eps);  PCG residuals 0.46 of the guaranteed bound (1);
  step_point 6.3e-12 (1e-10);  model change 2.1e-16 (1e-12);  whole chain 0.25 of kappa eta (10).
S is measured against the sum of |terms| rather than the largest entry of the block row because the one-pose scene
(every view on one pose centre: landmark depths are unobservable but for D^2) cancels: there the error is 2.1e-10 of
the block row's largest entry and 2.8e-14 of its terms.  The same scene sets step_point: the landmark step solves
(A_pp + D_p^2) with kappa ~1/D^2 and a right-hand side g_p - A_pr z that cancels, so its bar is 1e-10, not 1e-12.

The PCG stopping rules (pcg3_kernel / pcg5_kernel, pcg_kernel) and the bound they guarantee:
  pcg3 / pcg5 iterate on Scc X_j = B_j for B_0 = b_c and B_a = the border column of each free intrinsic coordinate,
  and stop when the recursive residual of every right-hand side satisfies |E_j| <= tol |B_j|.  The border is then
  eliminated exactly (z_i = T^-1 (b_i - Sci X_0), z_c = X_0 - X_a z_i), so the camera rows of S z - b equal
  E_0 - sum_a E_a z_i,a:  |r_c| <= tol (|b_c| + sum_a |z_i,a| |B_a|).  The intrinsic rows would be zero to rounding,
  but T = Sii - B'X is symmetrised first, which moves T_ab by (E_a'X_b - E_b'X_a) / 2:
  |r_i,a| <= tol / 2 sum_b (|X_a| |B_b| + |B_a| |X_b|) |z_i,b|.  pcg_kernel stops at |r| <= tol |b| on the whole system.
The bounds hold for the recursive residual; the true residual is checked against twice the bound plus a rounding
term (1e-14 |S| |z| on the camera rows, 1e-12 (|S_i| |z| + |b_i|) on the intrinsic rows)."""
import json
import os

import numpy as np
import pytest

import ba_step_reference as bref
import checkers as ck
from openmvg_b200 import synth

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
BAR_VEC, BAR_S, BAR_LDLT, BAR_STEP, BAR_MODEL = 1e-14, 1e-12, 1e-14, 1e-10, 1e-12
WORST = {}


@pytest.fixture(scope="module")
def ba():
    from openmvg_b200 import ba as m
    return m


@pytest.fixture(scope="module", autouse=True)
def _report():
    """OMVG_BA_STEP_REPORT=<file>: the worst measured deviation per stage, as JSON (to set the bars above)."""
    yield
    path = os.environ.get("OMVG_BA_STEP_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(WORST, f, indent=1, sort_keys=True)


def _note(stage, value, case):
    value = float(value)
    if stage not in WORST or value > WORST[stage][0]:
        WORST[stage] = [value, case]
    return value


def _blocks(nc, ni):
    return [(6 * a, 6) for a in range(nc)] + [(6 * nc + 8 * q, 8) for q in range(ni)]


def check_step(ctx, s, radius=1e4, solver=None, case="", point_constant=None, **opts):
    """debug_step at `radius` against the reference, stage by stage; returns the step record."""
    _, r, Ji, Jc, Jp = ctx.debug_eval(**opts)
    g = ctx.debug_step(radius, **opts)
    if solver is not None:
        assert g["solver"] == solver, (case, g["solver"])
    ref = bref.StepReference(s, r, Ji, Jc, Jp, radius, point_constant=point_constant, **opts)
    nc, ni, nd = ref.nc, ref.ni, ref.nd
    fail = []

    def bar(stage, value, limit):
        if not value <= limit:
            fail.append((stage, value, limit))
        _note(stage, value, case)

    # ---- scale, LM diagonal
    f = ref.free
    for name, want in (("scale", ref.scale), ("lm_diag", ref.lm_diag)):
        got = g[name][f].astype(bref.LD)
        bar(name, np.max(np.abs(got - want[f]) / np.abs(want[f])) if f.any() else 0.0, BAR_VEC)
    # ---- reduced system
    S, b = g["S"], g["rhs"]
    Sr, br = ref.S, ref.b
    const = np.flatnonzero(~ref.free_r)
    if len(const):
        eye = np.zeros((len(const), nd)); eye[np.arange(len(const)), const] = 1.0
        assert np.array_equal(S[const], eye) and np.array_equal(S[:, const], eye.T) and not b[const].any(), (case, "identity rows")
    werr_s = werr_t = werr_b = 0.0
    for r0, nr in _blocks(nc, ni):
        rowmax = float(np.abs(Sr[r0:r0 + nr]).max())
        termmax = float(ref.Smag[r0:r0 + nr].max())
        for c0, ncol in _blocks(nc, ni):
            blk, want = S[r0:r0 + nr, c0:c0 + ncol], Sr[r0:r0 + nr, c0:c0 + ncol]
            if not want.any() and (r0 < 6 * nc and c0 < 6 * nc and r0 != c0):
                assert not blk.any(), (case, "camera block without co-visibility is not 0", r0 // 6, c0 // 6)
            e = float(np.abs(blk - want).max())
            werr_s = max(werr_s, e / rowmax); werr_t = max(werr_t, e / termmax)
        mag = float(ref.bmag[r0:r0 + nr].max())
        e = float(np.abs(b[r0:r0 + nr] - br[r0:r0 + nr]).max())
        werr_b = max(werr_b, e / mag if mag > 0 else (0.0 if e == 0 else np.inf))
    _note("S_over_entries", werr_s, case)
    bar("S", werr_t, BAR_S); bar("rhs", werr_b, BAR_S)
    # ---- the solver on the GPU's own S, rhs
    z = g["z"]
    SL, bL, zL = S.astype(bref.LD), b.astype(bref.LD), z.astype(bref.LD)
    res = bL - SL @ zL
    nS = np.linalg.norm(S, 2)
    kappa = np.linalg.cond(S)
    if g["solver"] == "dense_ldlt":
        eta = float(np.linalg.norm(res) / (nS * np.linalg.norm(z) + np.linalg.norm(b)))
        bar("z_ldlt_backward", eta, BAR_LDLT)
    elif g["solver"] == "dense_inverse":
        zs = bref.solve_refined(SL, bL)
        fe = float(np.linalg.norm(zL - zs) / np.linalg.norm(zs))
        bar("z_inverse_forward_over_kappa_eps", fe / (kappa * EPS), 100.0)
        eta = float(np.linalg.norm(res) / (nS * np.linalg.norm(z) + np.linalg.norm(b)))
    else:
        tol = opts.get("pcg_tolerance", 1e-8)
        assert g["pcg_iterations"] > 0 and g["pcg_relres"] <= tol, (case, g["pcg_iterations"], g["pcg_relres"])
        nc6 = 6 * nc
        drift = 1e-14 * nS * np.linalg.norm(z)
        if g["solver"] == "pcg":
            bound = tol * np.linalg.norm(b)
            bar("z_pcg_residual_over_bound", float(np.linalg.norm(res)) / (2 * bound + drift), 1.0)
        else:
            fi = np.flatnonzero(ref.free_r[nc6:]) + nc6
            B = S[:nc6, fi]                                          # border columns B_a
            bound = tol * (np.linalg.norm(b[:nc6]) + sum(abs(z[q]) * np.linalg.norm(S[:nc6, q]) for q in fi))
            bar("z_block_pcg_camera_residual_over_bound", float(np.linalg.norm(res[:nc6])) / (2 * bound + drift), 1.0)
            # intrinsic rows: T = Sii - B' X is symmetrised, which moves T_ab by (E_a' X_b - E_b' X_a) / 2
            X = np.linalg.solve(S[:nc6, :nc6], B)                    # X_a = Scc^-1 B_a
            nB, nX, zi = np.linalg.norm(B, axis=0), np.linalg.norm(X, axis=0), np.abs(z[fi])
            bi = 0.5 * tol * (nX[:, None] * nB[None, :] + nB[:, None] * nX[None, :]) @ zi
            ri = float(np.linalg.norm(res[nc6:]))
            bar("z_block_pcg_border_residual_over_bound",
                ri / (2 * np.linalg.norm(bi) + 1e-12 * (np.linalg.norm(S[nc6:], 2) * np.linalg.norm(z) + np.linalg.norm(b[nc6:]))), 1.0)
        eta = float(np.linalg.norm(res) / (nS * np.linalg.norm(z) + np.linalg.norm(b)))
    # ---- back-substitution and model change from the GPU's z
    sp = g["step_point"]
    want = ref.back_substitute(z)
    cp = ~ref.fp.any(1)
    assert not sp[cp].any(), (case, "constant landmark with a nonzero step")
    wm = np.abs(want).max(1)
    live = ~cp & (wm > 0)
    assert not sp[~cp & (wm == 0)].any()
    bar("step_point", float((np.abs(sp[live] - want[live]).max(1) / wm[live]).max()) if live.any() else 0.0, BAR_STEP)
    m = ref.model_change(sp, -z)
    bar("model_change", float(abs(g["model_change"] - m) / abs(m)), BAR_MODEL)
    # ---- whole chain: the GPU's z against the reference's exact z*
    zs = bref.solve_refined(Sr, br)
    eta_s = float(np.linalg.norm((S - Sr.astype(np.float64)), 2) / np.linalg.norm(Sr.astype(np.float64), 2))
    eta_b = float(np.linalg.norm(b - br.astype(np.float64)) / np.linalg.norm(br.astype(np.float64)))
    tot = eta_s + eta_b + eta
    if kappa * tot < 0.1:
        fe = float(np.linalg.norm(zL - zs) / np.linalg.norm(zs))
        bar("chain_forward_over_kappa_eta", fe / (kappa * tot), 10.0)
    assert not fail, (case, g["solver"], fail)
    return g


def _reproject(s, seed, noise=0.5):
    """Observations re-projected through the oracle at the initial parameters plus noise; landmarks then perturbed."""
    s["obs_xy"] = np.zeros((len(s["obs_view"]), 2))
    proj = ck.oracle_ba_eval(s, use_loss=0)[1]
    rng = np.random.default_rng(seed)
    s["obs_xy"] = np.ascontiguousarray(proj + rng.normal(0, noise, proj.shape))
    s["points"] = np.ascontiguousarray(s["points"] + rng.normal(0, 0.01, s["points"].shape))
    return s


def _custom_scene(n_cams, tracks, seed, n_intrinsics=1):
    """Poses / intrinsics of synth.ba_scene, one landmark per track (a list of views), observations re-projected."""
    s = synth.ba_scene(n_cams, 1, 1, seed=seed, n_intrinsics=n_intrinsics)
    rng = np.random.default_rng(seed)
    s["points"] = np.ascontiguousarray(rng.uniform(-0.5, 0.5, (len(tracks), 3)))
    s["obs_view"] = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in tracks]))
    s["obs_point"] = np.ascontiguousarray(np.repeat(np.arange(len(tracks), dtype=np.int32), [len(t) for t in tracks]))
    return _reproject(s, seed)


def _pair_counts(s):
    """Observation pairs of every camera block on the co-visibility lists (pair_count_kernel: landmarks of one intrinsic
    group and at most 32 views; pairs (t, u) with pose(u) >= pose(t))."""
    pose = s["view_pose"][s["obs_view"]]; grp = s["view_intr"][s["obs_view"]]
    counts = {}
    for j in range(len(s["points"])):
        o = np.flatnonzero(s["obs_point"] == j)
        if len(o) > 32 or len(set(grp[o])) > 1:
            continue
        for t in o:
            for u in o:
                if pose[u] >= pose[t]:
                    counts[(pose[t], pose[u])] = counts.get((pose[t], pose[u]), 0) + 1
    return counts


def _ctx(ba, s):
    return ba.BAContext(s)


# ----------------------------------------------------------------------------- KIU instantiations, masks, radius
@pytest.mark.parametrize("model", [1, 2, 3, 4, 5, 7, "mix"])
def test_step_every_kiu(ba, model):
    """dispatch_kiu K = 3 (pinhole, spherical, pinhole + spherical), 4, 6, 7, 8: schur_stage / schur_border / corner."""
    if model == "mix":
        s = synth.ba_scene(12, 300, 5, seed=4, n_intrinsics=2)
        sp = synth.ba_scene(12, 300, 5, seed=4, n_intrinsics=2, model=7)
        s["intr_model"] = np.array([1, 7], np.int32); s["intrinsics"][1] = sp["intrinsics"][1]
        sph = s["view_intr"][s["obs_view"]] == 1
        s["obs_xy"][sph] = sp["obs_xy"][sph]
    else:
        s = synth.ba_scene(12, 300, 5, seed=3, model=model, n_intrinsics=2, outlier_frac=0.05)
        s["intrinsics"][:, 3:] += s["gt_dist"][3:] * 0.9
    ctx = _ctx(ba, s)
    check_step(ctx, s, solver="dense_ldlt", case=f"kiu-model{model}")
    ctx.close()


@pytest.mark.parametrize("opts", [dict(intrinsics_opt=1), dict(intrinsics_opt=2), dict(intrinsics_opt=4), dict(intrinsics_opt=8),
                                  dict(intrinsics_opt=14), dict(extrinsics_opt=1), dict(extrinsics_opt=2), dict(extrinsics_opt=4),
                                  dict(extrinsics_opt=6), dict(structure_opt=0), dict(use_loss=0)],
                         ids=lambda k: "_".join(f"{a}{b}" for a, b in k.items()))
def test_step_option_masks(ba, opts):
    s = synth.ba_scene(14, 400, 5, seed=6, model=4, outlier_frac=0.03)
    s["intrinsics"][:, 3:] += s["gt_dist"][3:] * 0.5
    ctx = _ctx(ba, s)
    g = check_step(ctx, s, solver="dense_ldlt", case=f"mask-{opts}", **opts)
    if opts.get("structure_opt") == 0:
        assert not g["step_point"].any()
    ctx.close()


@pytest.mark.parametrize("radius", [1e-3, 1e4, 1e16])
@pytest.mark.parametrize("cams", [20, 60])
def test_step_radius(ba, radius, cams):
    """The clamps of lm_diag3_kernel bind at both ends; at 1e16 the gauge directions make kappa ~1e20 and only the
    backward-error bars speak."""
    s = synth.ba_scene(cams, 30 * cams, 6, seed=cams, outlier_frac=0.02)
    ctx = _ctx(ba, s)
    check_step(ctx, s, radius=radius, solver="dense_ldlt" if cams == 20 else "dense_inverse", case=f"radius{radius:g}-{cams}")
    ctx.close()


# ----------------------------------------------------------------------------- co-visibility lists
def test_step_gather_chunk_boundaries(ba):
    """Camera blocks whose pair lists are 1, 29, 30, 31, 119, 120, 121, 240, 241 and 1000 (9 chunks) long: GATHER_CHUNK =
    120 pairs per warp, 30 per load round, the ticketed sum of the partials of a multi-chunk block."""
    lengths = [1, 29, 30, 31, 119, 120, 121, 240, 241, 1000]
    n_cams = 22
    tracks = []
    for k, n in enumerate(lengths):                     # n two-view landmarks on cameras (2k, 2k+1)
        tracks += [[2 * k, 2 * k + 1]] * n
    for j in range(300):                                # background tracks on cameras of one parity only
        c = (2 * j + j % 2) % n_cams
        tracks.append([(c + 2 * i) % n_cams for i in range(4)])
    s = _custom_scene(n_cams, tracks, seed=31)
    counts = _pair_counts(s)
    for k, n in enumerate(lengths):
        assert counts[(2 * k, 2 * k + 1)] == n
    assert max(counts.values()) >= 8 * 120
    ctx = _ctx(ba, s)
    a = check_step(ctx, s, solver="dense_ldlt", case="gather-chunks")
    b = ctx.debug_step(1e4)
    for k in ("S", "rhs", "z", "step_point", "model_change"):      # the tickets were reset by the first call
        assert np.array_equal(a[k], b[k]), k
    ctx.close()


def test_step_fast_and_slow_landmarks_in_one_block(ba):
    """Tracks of exactly 32 views (co-visibility lists) and 33 views (schur_kernel atomics + mirror_kernel) through
    the same cameras, so that both land on the same gathered blocks."""
    n_cams = 34
    tracks = [list(range(32))] * 15 + [list(range(33))] * 15
    tracks += [[(j + 3 * i) % n_cams for i in range(5)] for j in range(400)]
    s = _custom_scene(n_cams, tracks, seed=5)
    ctx = _ctx(ba, s)
    check_step(ctx, s, solver="dense_ldlt", case="slow-32-33")
    ctx.close()


def test_step_landmarks_through_two_groups(ba):
    """Views alternate between two intrinsic groups: landmarks seen through both (not on the lists) give Sii its
    off-diagonal group block."""
    s = synth.ba_scene(16, 500, 5, seed=8, n_intrinsics=2)
    grp = s["view_intr"][s["obs_view"]]
    both = np.zeros(len(s["points"]), bool)
    both[np.unique(s["obs_point"][grp == 0])] = True
    assert (both & np.isin(np.arange(len(both)), s["obs_point"][grp == 1])).any()
    ctx = _ctx(ba, s)
    g = check_step(ctx, s, solver="dense_ldlt", case="two-groups")
    nc6 = 6 * 16
    assert np.abs(g["S"][nc6:nc6 + 3, nc6 + 8:nc6 + 11]).max() > 0
    ctx.close()


def test_step_two_views_of_one_pose(ba):
    """A rig: a second view on every pose re-observes some landmarks, two observations of one landmark in the same
    diagonal block."""
    s = synth.ba_scene(16, 600, 6, seed=7)
    nv = len(s["view_pose"])
    rng = np.random.default_rng(7)
    pick = np.flatnonzero(rng.random(len(s["obs_view"])) < 0.06)
    s["view_pose"] = np.ascontiguousarray(np.concatenate([s["view_pose"], s["view_pose"]]).astype(np.int32))
    s["view_intr"] = np.ascontiguousarray(np.concatenate([s["view_intr"], s["view_intr"]]).astype(np.int32))
    s["obs_view"] = np.ascontiguousarray(np.concatenate([s["obs_view"], s["obs_view"][pick] + nv]).astype(np.int32))
    s["obs_point"] = np.ascontiguousarray(np.concatenate([s["obs_point"], s["obs_point"][pick]]).astype(np.int32))
    s["obs_xy"] = np.ascontiguousarray(np.concatenate([s["obs_xy"], s["obs_xy"][pick] + rng.normal(0, 0.5, (len(pick), 2))]))
    ctx = _ctx(ba, s)
    check_step(ctx, s, solver="dense_ldlt", case="rig")
    ctx.close()


# ----------------------------------------------------------------------------- empty and removed structure
def test_step_pose_without_observations(ba):
    s = synth.ba_scene(12, 300, 5, seed=2)
    s["poses"] = np.ascontiguousarray(np.concatenate([s["poses"], s["poses"][:1] + 0.01]))
    s["view_pose"] = np.ascontiguousarray(np.append(s["view_pose"], 12).astype(np.int32))
    s["view_intr"] = np.ascontiguousarray(np.append(s["view_intr"], 0).astype(np.int32))
    ctx = _ctx(ba, s)
    g = check_step(ctx, s, solver="dense_ldlt", case="empty-pose")
    lm = g["lm_diag"][3 * len(s["points"]) + 72:3 * len(s["points"]) + 78]
    assert np.array_equal(g["S"][72:78, 72:78], np.diag(lm * lm))
    assert not g["S"][72:78, :72].any() and not g["S"][72:78, 78:].any() and not g["z"][72:78].any()
    ctx.close()


def test_step_pose_with_zero_weights(ba):
    s = synth.ba_scene(12, 300, 5, seed=2)
    w = np.ones(len(s["obs_view"])); w[s["view_pose"][s["obs_view"]] == 5] = 0.0
    ctx = _ctx(ba, s)
    ctx.set_obs_weights(w)
    g = check_step(ctx, s, solver="dense_ldlt", case="zero-weight-pose")
    assert not g["S"][30:36, :30].any() and not g["z"][30:36].any()
    ctx.close()


def test_step_removed_tracks(ba):
    s = synth.ba_scene(12, 600, 5, seed=4)
    ctx = _ctx(ba, s)
    mask = np.zeros(len(s["points"]), np.uint8); mask[::7] = 1
    ctx.remove_points(mask)
    g = check_step(ctx, s, solver="dense_ldlt", case="removed", point_constant=mask)
    assert not g["step_point"][mask == 1].any()
    ctx.close()


def test_step_control_points(ba):
    s = synth.add_gcp(synth.ba_scene(12, 300, 5, seed=3, model=3, outlier_frac=0.05), 5, weight=7.0)
    ctx = _ctx(ba, s)
    g = check_step(ctx, s, solver="dense_ldlt", case="gcp")
    assert not g["step_point"][s["point_fixed"] == 1].any()
    ctx.close()


# ----------------------------------------------------------------------------- every solver at its boundary
def _one_pose_scene(n_views=6, n_points=300, seed=9):
    s = synth.ba_scene(n_views, n_points, 4, seed=seed)
    intr = np.repeat(s["intrinsics"][:1], n_views, axis=0); intr[:, 0] += 20.0 * np.arange(n_views)
    s.update(poses=np.ascontiguousarray(s["poses"][:1]), intrinsics=np.ascontiguousarray(intr), intr_model=np.full(n_views, 1, np.int32),
             view_pose=np.zeros(n_views, np.int32), view_intr=np.arange(n_views, dtype=np.int32))
    return _reproject(s, seed)


SOLVER_CASES = [
    ("34x2", dict(n_cams=34, n_intrinsics=2), {}, {}, "dense_ldlt"),            # nd = 220
    ("33x3", dict(n_cams=33, n_intrinsics=3), {}, {}, "dense_inverse"),         # nd = 222
    ("104x2", dict(n_cams=104, n_intrinsics=2), {}, {}, "dense_inverse"),       # nd = 640
    ("103x3", dict(n_cams=103, n_intrinsics=3), {}, {}, "pcg3"),                # nd = 642, 9 free intrinsic columns
    ("103x3-focal", dict(n_cams=103, n_intrinsics=3), dict(intrinsics_opt=2), {}, "pcg5"),   # 3 free columns
    ("12-one-cta", dict(n_cams=12, n_intrinsics=1), {}, dict(OMVG_BA_DENSE_MAX="0", OMVG_BA_DENSE2_MAX="0"), "pcg3"),
    ("one-pose", None, {}, dict(OMVG_BA_DENSE_MAX="0", OMVG_BA_DENSE2_MAX="0"), "pcg3"),
    ("brown6", dict(n_cams=30, n_intrinsics=6, model=4), {}, dict(OMVG_BA_DENSE_MAX="0", OMVG_BA_DENSE2_MAX="0"), "pcg"),   # 48 free columns
    ("pcg1", dict(n_cams=40, n_intrinsics=1), {}, dict(OMVG_BA_DENSE_MAX="0", OMVG_BA_DENSE2_MAX="0", OMVG_BA_PCG1="1"), "pcg"),
]


@pytest.mark.parametrize("tol", [1e-8, 1e-12])
@pytest.mark.parametrize("name,scene,opts,env,solver", SOLVER_CASES, ids=[c[0] for c in SOLVER_CASES])
def test_step_every_solver(ba, monkeypatch, name, scene, opts, env, solver, tol):
    if solver.startswith("dense") and tol != 1e-8:
        pytest.skip("pcg_tolerance does not reach the direct solves")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    if scene is None:
        s = _one_pose_scene()
    else:
        kw = dict(scene); n = kw.pop("n_cams")
        s = synth.ba_scene(n, 20 * n, 6, seed=n, outlier_frac=0.02, **kw)
    if s["intr_model"][0] == 4:
        s["intrinsics"][:, 3:] += s["gt_dist"][3:] * 0.5
    ctx = _ctx(ba, s)
    check_step(ctx, s, solver=solver, case=f"solver-{name}-tol{tol:g}", pcg_tolerance=tol, **opts)
    ctx.close()


# ----------------------------------------------------------------------------- state between calls on one context
def test_step_state_between_calls(ba):
    """The first call on a fresh context (the H records still hold the create-time sort buffers), a second identical
    call bitwise equal (direct path, no landmark off the lists: the gather tickets reset), calls alternating
    structure_opt 0/1 and intrinsics_opt 1/14, and run() after debug_step equal to run() on a fresh context."""
    s = synth.ba_scene(20, 1000, 6, seed=2)
    ctx = _ctx(ba, s)
    a = check_step(ctx, s, solver="dense_ldlt", case="state-first")
    b = ctx.debug_step(1e4)
    for k in ("S", "rhs", "z", "step_point", "scale", "lm_diag"):
        assert a[k].tobytes() == b[k].tobytes(), k
    assert a["model_change"] == b["model_change"]
    for opts in (dict(structure_opt=0), dict(structure_opt=1), dict(intrinsics_opt=1), dict(intrinsics_opt=14),
                 dict(structure_opt=0, intrinsics_opt=1), dict()):
        check_step(ctx, s, solver="dense_ldlt", case=f"state-{opts}", **opts)
    r1 = ctx.run(); p1 = ctx.download()
    ctx.close()
    fresh = _ctx(ba, s)
    r2 = fresh.run(); p2 = fresh.download()
    fresh.close()
    assert r1["final_cost"] == r2["final_cost"] and r1["iterations"] == r2["iterations"]
    for x, y in zip(p1, p2):
        assert x.tobytes() == y.tobytes()
