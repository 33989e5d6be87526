"""Python binding of the BA C-ABI (tests / bench plumbing; the drop-in host shim is the C++ class
in openmvg_b200/host/Bundle_Adjustment_B200.hpp).

Mirrors openMVG::sfm::Bundle_Adjustment_Ceres::Adjust (reference: sfm/sfm_data_BA_ceres.cpp:165-608)
on the flat scene of include/omvg_b200.h: same options (Optimize_Options, sfm_data_BA.hpp:66-89),
same outcome convention (returns the refined parameters iff the solution is usable).
"""
from __future__ import annotations

import ctypes

import numpy as np

from ._lib import OmvgError, check, lib

_vp = ctypes.c_void_p
_dp = ctypes.POINTER(ctypes.c_double)
_ip = ctypes.POINTER(ctypes.c_int32)
_bp = ctypes.POINTER(ctypes.c_uint8)


class Problem(ctypes.Structure):
    _fields_ = [("n_poses", ctypes.c_int32), ("n_intrinsics", ctypes.c_int32), ("n_points", ctypes.c_int32),
                ("n_views", ctypes.c_int32), ("n_obs", ctypes.c_int64), ("poses", _dp), ("intrinsics", _dp),
                ("intr_model", _ip), ("points", _dp), ("view_pose", _ip), ("view_intr", _ip), ("obs_view", _ip),
                ("obs_point", _ip), ("obs_xy", _dp),
                # optional extensions (NULL / 0 = absent): GCP weights / flags / fixed landmarks, pose-centre priors
                ("obs_weight", _dp), ("obs_no_loss", _bp), ("point_fixed", _bp),
                ("n_priors", ctypes.c_int32), ("reserved_", ctypes.c_int32), ("prior_pose", _ip),
                ("prior_center", _dp), ("prior_weight", _dp), ("prior_huber_a", ctypes.c_double)]


class Options(ctypes.Structure):
    _fields_ = [("intrinsics_opt", ctypes.c_int32), ("extrinsics_opt", ctypes.c_int32), ("structure_opt", ctypes.c_int32),
                ("use_loss", ctypes.c_int32), ("huber_a", ctypes.c_double), ("max_num_iterations", ctypes.c_int32),
                ("max_consecutive_invalid_steps", ctypes.c_int32), ("function_tolerance", ctypes.c_double),
                ("gradient_tolerance", ctypes.c_double), ("parameter_tolerance", ctypes.c_double),
                ("initial_radius", ctypes.c_double), ("max_radius", ctypes.c_double), ("min_radius", ctypes.c_double),
                ("min_relative_decrease", ctypes.c_double), ("min_lm_diagonal", ctypes.c_double),
                ("max_lm_diagonal", ctypes.c_double), ("pcg_tolerance", ctypes.c_double),
                ("pcg_max_iterations", ctypes.c_int32), ("verbose", ctypes.c_int32), ("device", ctypes.c_int32),
                ("reserved_", ctypes.c_int32)]


class Summary(ctypes.Structure):
    _fields_ = [("initial_cost", ctypes.c_double), ("final_cost", ctypes.c_double), ("iterations", ctypes.c_int32),
                ("successful_steps", ctypes.c_int32), ("unsuccessful_steps", ctypes.c_int32), ("lm_steps", ctypes.c_int32),
                ("termination", ctypes.c_int32), ("usable", ctypes.c_int32), ("pcg_iterations", ctypes.c_int64),
                ("kernel_launches", ctypes.c_int64), ("device_ms", ctypes.c_double), ("jacobian_ms", ctypes.c_double),
                ("jacobian_launches", ctypes.c_int64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def default_options(**kw) -> Options:
    o = Options()
    lib().omvg_ba_default_options(ctypes.byref(o))
    for k, v in kw.items():
        if not hasattr(o, k):
            raise TypeError(f"unknown BA option {k}")
        setattr(o, k, v)
    return o


def _problem(s, poses, intr, pts) -> Problem:
    P = Problem()
    P.n_poses, P.n_intrinsics, P.n_points = len(poses), len(intr), len(pts)
    P.n_views, P.n_obs = len(s["view_pose"]), len(s["obs_view"])
    d = lambda a: a.ctypes.data_as(_dp)   # noqa: E731
    i = lambda a: a.ctypes.data_as(_ip)   # noqa: E731
    P.poses, P.intrinsics, P.points = d(poses), d(intr), d(pts)
    P.intr_model, P.view_pose, P.view_intr = i(s["intr_model"]), i(s["view_pose"]), i(s["view_intr"])
    P.obs_view, P.obs_point, P.obs_xy = i(s["obs_view"]), i(s["obs_point"]), d(s["obs_xy"])
    # optional extensions; the converted arrays are kept alive on the struct
    keep = []

    def opt(key, dtype, ptr):
        a = s.get(key)
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype); keep.append(a)
        return a.ctypes.data_as(ptr)
    P.obs_weight = opt("obs_weight", np.float64, _dp)
    P.obs_no_loss = opt("obs_no_loss", np.uint8, _bp)
    P.point_fixed = opt("point_fixed", np.uint8, _bp)
    if s.get("prior_pose") is not None and len(s["prior_pose"]):
        P.n_priors = len(s["prior_pose"])
        P.prior_pose = opt("prior_pose", np.int32, _ip)
        P.prior_center = opt("prior_center", np.float64, _dp)
        P.prior_weight = opt("prior_weight", np.float64, _dp)
        P.prior_huber_a = float(s.get("prior_huber_a", 0.0))
    P._keep = keep
    return P


def solve(s: dict, **opts) -> dict:
    """One-shot Adjust through omvg_ba_solve with HOST buffers (upload, solve, write-back)."""
    poses = np.ascontiguousarray(s["poses"], np.float64).copy()
    intr = np.ascontiguousarray(s["intrinsics"], np.float64).copy()
    pts = np.ascontiguousarray(s["points"], np.float64).copy()
    P = _problem(s, poses, intr, pts)
    o = default_options(**opts)
    sm = Summary()
    rc = lib().omvg_ba_solve(ctypes.byref(P), ctypes.byref(o), ctypes.byref(sm))
    if rc not in (0, -5):
        check(rc)
    out = sm.as_dict()
    out.update(ok=(rc == 0), poses=poses, intrinsics=intr, points=pts)
    return out


class BAContext:
    """Device-resident scene (omvg_ba_ctx): create once, reset/run many times."""

    def __init__(self, s: dict, device: int = 0):
        self._keep = (np.ascontiguousarray(s["poses"], np.float64).copy(),
                      np.ascontiguousarray(s["intrinsics"], np.float64).copy(),
                      np.ascontiguousarray(s["points"], np.float64).copy())
        self._s = s
        P = _problem(s, *self._keep)
        self._h = _vp()
        check(lib().omvg_ba_create(ctypes.byref(self._h), int(device), ctypes.byref(P)))

    def close(self):
        if self._h:
            lib().omvg_ba_destroy(self._h)
            self._h = _vp()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        check(lib().omvg_ba_reset(self._h))

    def run(self, **opts) -> dict:
        o = default_options(**opts)
        sm = Summary()
        rc = lib().omvg_ba_run(self._h, ctypes.byref(o), ctypes.byref(sm))
        if rc not in (0, -5):
            check(rc)
        out = sm.as_dict()
        out["ok"] = rc == 0
        return out

    def download(self):
        poses, intr, pts = (np.zeros_like(a) for a in self._keep)
        check(lib().omvg_ba_download(self._h, poses.ctypes.data_as(_dp), intr.ctypes.data_as(_dp), pts.ctypes.data_as(_dp)))
        return poses, intr, pts

    def residual_norms(self):
        out = np.zeros(len(self._s["obs_view"]))
        check(lib().omvg_ba_residual_norms(self._h, out.ctypes.data_as(_dp)))
        return out

    def set_obs_weights(self, w):
        """Per-observation weights of the resident problem (0 = observation removed)."""
        w = np.ascontiguousarray(w, np.float64)
        assert len(w) == len(self._s["obs_view"])
        check(lib().omvg_ba_set_obs_weights(self._h, w.ctypes.data_as(_dp)))

    def reject_outliers(self, threshold_px: float = 4.0, min_track_length: int = 2):
        """RemoveOutliers_PixelResidualError(threshold, minTrackLength) on the device (sfm_data_filters.cpp:40-73).
        -> (obs_removed[n_obs] bool in the caller's order, point_removed[n_points] bool, n_outliers, n_tracks)"""
        n = len(self._s["obs_view"]); npts = len(self._keep[2])
        bits = np.zeros((n + 31) // 32, np.uint32); pr = np.zeros(npts, np.uint8)
        no = ctypes.c_int64(); nt = ctypes.c_int64()
        check(lib().omvg_ba_reject_outliers(self._h, ctypes.c_double(threshold_px), int(min_track_length), bits.ctypes.data_as(_vp),
                                            pr.ctypes.data_as(_vp), ctypes.byref(no), ctypes.byref(nt)))
        removed = np.unpackbits(bits.view(np.uint8), bitorder="little")[:n].astype(bool)
        return removed, pr.astype(bool), no.value, nt.value

    def remove_points(self, mask):
        """Remove whole tracks (the host-side angle test's verdict).  -> (obs_removed[n_obs] bool, n_tracks)"""
        n = len(self._s["obs_view"])
        m = np.ascontiguousarray(mask, np.uint8); assert len(m) == len(self._keep[2])
        bits = np.zeros((n + 31) // 32, np.uint32); nt = ctypes.c_int64()
        check(lib().omvg_ba_remove_points(self._h, m.ctypes.data_as(_vp), bits.ctypes.data_as(_vp), ctypes.byref(nt)))
        return np.unpackbits(bits.view(np.uint8), bitorder="little")[:n].astype(bool), nt.value

    def commit(self):
        """Make the refined parameters the state reset() restores."""
        check(lib().omvg_ba_commit(self._h))

    def debug_eval(self, **opts):
        o = default_options(**opts)
        n = len(self._s["obs_view"])
        r = np.zeros((n, 2)); Ji = np.zeros((n, 2, 8)); Jc = np.zeros((n, 2, 6)); Jp = np.zeros((n, 2, 3))
        cost = ctypes.c_double()
        d = lambda a: a.ctypes.data_as(_dp)   # noqa: E731
        check(lib().omvg_ba_debug_eval(self._h, ctypes.byref(o), ctypes.byref(cost), d(r), d(Ji), d(Jc), d(Jp)))
        return cost.value, r, Ji, Jc, Jp

    def debug_prior(self, **opts):
        """The pose-centre prior rows at the uploaded parameters (omvg_ba_debug_prior): (cost, r [n_priors][3],
        J [n_priors][3][6]), Huber-corrected, unscaled, masked by the extrinsics option."""
        o = default_options(**opts)
        pp = self._s.get("prior_pose")
        n = 0 if pp is None else len(pp)
        r = np.zeros((n, 3)); J = np.zeros((n, 3, 6)); cost = ctypes.c_double()
        check(lib().omvg_ba_debug_prior(self._h, ctypes.byref(o), ctypes.byref(cost), r.ctypes.data_as(_dp), J.ctypes.data_as(_dp)))
        return cost.value, r, J

    # solver ids of omvg_ba_debug_step
    SOLVERS = ("dense_ldlt", "dense_inverse", "pcg5", "pcg3", "pcg")

    def debug_step(self, radius: float, **opts) -> dict:
        """The first LM step of run() at trust-region radius `radius`, stage by stage (omvg_ba_debug_step): Jacobi
        scaling, LM diagonal, the dense reduced system S and its right-hand side, the solver's z, the landmark step and
        the model cost change.  Vectors over all columns are ordered points (3 n_points), poses (6 n_poses), intrinsic
        slots (8 n_intrinsics); S, rhs and z cover the last two."""
        o = default_options(**opts)
        npt, nc, ni = len(self._keep[2]), len(self._keep[0]), len(self._keep[1])
        nd = 6 * nc + 8 * ni; nx = 3 * npt + nd
        scale = np.zeros(nx); lm = np.zeros(nx); S = np.zeros((nd, nd)); rhs = np.zeros(nd); z = np.zeros(nd)
        step = np.zeros((npt, 3)); model = ctypes.c_double(); solver = ctypes.c_int32(); pcg = np.zeros(3)
        d = lambda a: a.ctypes.data_as(_dp)   # noqa: E731
        check(lib().omvg_ba_debug_step(self._h, ctypes.byref(o), ctypes.c_double(radius), d(scale), d(lm), d(S), d(rhs), d(z), d(step),
                                       ctypes.byref(model), ctypes.byref(solver), d(pcg)))
        return dict(scale=scale, lm_diag=lm, S=S, rhs=rhs, z=z, step_point=step, model_change=model.value,
                    solver=self.SOLVERS[solver.value], pcg_iterations=int(pcg[0]), pcg_relres=pcg[1], pcg_bnorm=pcg[2])


class Bundle_Adjustment_B200:
    """Drop-in for Bundle_Adjustment_Ceres on the flat scene: Adjust(scene, options) -> bool, scene
    updated in place iff the solution is usable (sfm_data_BA.hpp:91-105, sfm_data_BA_ceres.cpp:503-507)."""

    def __init__(self, **ceres_options):
        self.options = ceres_options
        self.summary = None

    def Adjust(self, scene: dict, intrinsics_opt=14, extrinsics_opt=6, structure_opt=1) -> bool:
        r = solve(scene, intrinsics_opt=intrinsics_opt, extrinsics_opt=extrinsics_opt, structure_opt=structure_opt,
                  **self.options)
        self.summary = r
        if r["ok"]:
            scene["poses"][...] = r["poses"]; scene["intrinsics"][...] = r["intrinsics"]; scene["points"][...] = r["points"]
        return bool(r["ok"])
