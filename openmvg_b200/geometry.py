"""Python binding of the geometric-filter C-ABI (tests / bench plumbing).

Mirrors GeometricFilter_FMatrix_AC::Robust_estimation per pair (reference:
matching_image_collection/F_ACRobust.hpp:45-106) over a CSR of putative matches."""
from __future__ import annotations

import ctypes

import numpy as np

from ._lib import check, lib

_vp = ctypes.c_void_p


FUNDAMENTAL, HOMOGRAPHY, ESSENTIAL = 0, 1, 2


def fundamental_acransac(offsets, xI, xJ, image_size, precision: float = 4.0, max_iterations: int = 2048, device: int = 0):
    return acransac(FUNDAMENTAL, offsets, xI, xJ, image_size, precision, max_iterations, device)


def homography_acransac(offsets, xI, xJ, image_size, precision: float = 4.0, max_iterations: int = 2048, device: int = 0):
    """GeometricFilter_HMatrix_AC::Robust_estimation per pair (H_ACRobust.hpp:46-112); `F` of the result holds H."""
    return acransac(HOMOGRAPHY, offsets, xI, xJ, image_size, precision, max_iterations, device)


def acransac(model, offsets, xI, xJ, image_size, precision: float = 4.0, max_iterations: int = 2048, device: int = 0):
    """offsets[n_pairs+1]; xI, xJ [n_matches, 2] float64; image_size [n_pairs, 4] (wI, hI, wJ, hJ).
    -> list of dicts per pair: inliers (uint32 indices into the pair's matches), F [3,3], error_max, min_nfa"""
    off = np.ascontiguousarray(offsets, np.uint64); n_pairs = len(off) - 1
    xI = np.ascontiguousarray(xI, np.float64).reshape(-1, 2); xJ = np.ascontiguousarray(xJ, np.float64).reshape(-1, 2)
    sz = np.ascontiguousarray(image_size, np.int32).reshape(-1, 4)
    nm = int(off[-1]); assert len(xI) == nm == len(xJ) and len(sz) == n_pairs
    inl = np.zeros(max(nm, 1), np.uint32); ninl = np.zeros(max(n_pairs, 1), np.uint32); F = np.zeros((max(n_pairs, 1), 9)); st = np.zeros((max(n_pairs, 1), 2))
    p = lambda a: a.ctypes.data_as(_vp)   # noqa: E731
    check(lib().omvg_geom_acransac(int(device), int(model), ctypes.c_uint64(n_pairs), p(off), p(xI), p(xJ), p(sz), ctypes.c_double(precision),
                                               ctypes.c_uint32(max_iterations), p(inl), p(ninl), p(F), p(st)))
    out = []
    for k in range(n_pairs):
        a = int(off[k])
        out.append(dict(inliers=inl[a:a + int(ninl[k])].copy(), F=F[k].reshape(3, 3).copy(), error_max=float(st[k, 0]), min_nfa=float(st[k, 1])))
    return out


def essential_acransac(offsets, xI, xJ, image_size, intr, precision: float = 4.0, max_iterations: int = 2048, device: int = 0):
    """GeometricFilter_EMatrix_AC::Robust_estimation per pair (E_ACRobust.hpp:55-150) over a CSR of putative matches of
    calibrated pinhole views.  intr [n_pairs, 6] = (f, ppx, ppy) of view I then view J.  Same result dicts as
    acransac; `F` holds E and error_max is in squared pixels, as the reference leaves them.  The reference keeps a
    pair iff it has more than 12.5 inliers."""
    off = np.ascontiguousarray(offsets, np.uint64); n_pairs = len(off) - 1
    xI = np.ascontiguousarray(xI, np.float64).reshape(-1, 2); xJ = np.ascontiguousarray(xJ, np.float64).reshape(-1, 2)
    sz = np.ascontiguousarray(image_size, np.int32).reshape(-1, 4)
    k = np.ascontiguousarray(intr, np.float64).reshape(-1, 6)
    nm = int(off[-1]); assert len(xI) == nm == len(xJ) and len(sz) == n_pairs == len(k)
    inl = np.zeros(max(nm, 1), np.uint32); ninl = np.zeros(max(n_pairs, 1), np.uint32); E = np.zeros((max(n_pairs, 1), 9)); st = np.zeros((max(n_pairs, 1), 2))
    p = lambda a: a.ctypes.data_as(_vp)   # noqa: E731
    check(lib().omvg_geom_essential_acransac(int(device), ctypes.c_uint64(n_pairs), p(off), p(xI), p(xJ), p(sz), p(k), ctypes.c_double(precision),
                                             ctypes.c_uint32(max_iterations), p(inl), p(ninl), p(E), p(st)))
    out = []
    for q in range(n_pairs):
        a = int(off[q])
        out.append(dict(inliers=inl[a:a + int(ninl[q])].copy(), F=E[q].reshape(3, 3).copy(), error_max=float(st[q, 0]), min_nfa=float(st[q, 1])))
    return out


def debug_five_point(b1, b2, device: int = 0):
    """The device five-point solver on n samples of 5 bearing pairs [n, 5, 3] (validation aid).
    -> dict(E [n, 10, 3, 3], n_models [n]): the first n_models[s] matrices of sample s are its real solutions."""
    b1 = np.ascontiguousarray(b1, np.float64).reshape(-1, 5, 3); b2 = np.ascontiguousarray(b2, np.float64).reshape(-1, 5, 3)
    n = len(b1); assert len(b2) == n
    E = np.zeros((max(n, 1), 10, 9)); k = np.zeros(max(n, 1), np.int32)
    p = lambda a: a.ctypes.data_as(_vp)   # noqa: E731
    check(lib().omvg_geom_debug_five_point(int(device), ctypes.c_uint32(n), p(b1), p(b2), p(E), p(k)))
    return dict(E=E[:n].reshape(n, 10, 3, 3).copy(), n_models=k[:n].copy())


ESSENTIAL_ANGULAR, ESSENTIAL_UPRIGHT = 3, 4


def angular_essential_acransac(offsets, bI, bJ, upright: bool = False, precision_deg: float = 4.0, max_iterations: int = 2048,
                               device: int = 0):
    """GeometricFilter_ESphericalMatrix_AC_Angular<upright>::Robust_estimation per pair (E_ACRobust_Angular.hpp:52-160)
    over a CSR of putative matches given as bearing vectors bI, bJ [n_matches, 3] ((*cam)(x) of each view).  Eight-point
    (`-g a`) or, with upright=True, upright three-point (`-g u`) AC-RANSAC, then RelativePoseFromEssential.
    -> list of dicts per pair: inliers (after the cheirality step: what the filter keeps), ransac_inliers (the AC-RANSAC
    list before it), F [3,3] (holds E), error_max (radians), min_nfa.  The reference keeps a pair iff it has more than
    20 (eight-point) or 7.5 (upright) inliers."""
    off = np.ascontiguousarray(offsets, np.uint64); n_pairs = len(off) - 1
    bI = np.ascontiguousarray(bI, np.float64).reshape(-1, 3); bJ = np.ascontiguousarray(bJ, np.float64).reshape(-1, 3)
    nm = int(off[-1]); assert len(bI) == nm == len(bJ)
    inl = np.zeros(max(nm, 1), np.uint32); ninl = np.zeros(max(n_pairs, 1), np.uint32); nr = np.zeros(max(n_pairs, 1), np.uint32)
    rinl = np.zeros(max(nm, 1), np.uint32); E = np.zeros((max(n_pairs, 1), 9)); st = np.zeros((max(n_pairs, 1), 2))
    p = lambda a: a.ctypes.data_as(_vp)   # noqa: E731
    check(lib().omvg_geom_angular_acransac(int(device), ESSENTIAL_UPRIGHT if upright else ESSENTIAL_ANGULAR, ctypes.c_uint64(n_pairs), p(off),
                                           p(bI), p(bJ), ctypes.c_double(precision_deg), ctypes.c_uint32(max_iterations),
                                           p(inl), p(ninl), p(E), p(st), p(nr), p(rinl)))
    out = []
    for q in range(n_pairs):
        a = int(off[q])
        out.append(dict(inliers=inl[a:a + int(ninl[q])].copy(), ransac_inliers=rinl[a:a + int(nr[q])].copy(), F=E[q].reshape(3, 3).copy(),
                        error_max=float(st[q, 0]), min_nfa=float(st[q, 1])))
    return out


def debug_angular_solver(b1, b2, upright: bool = False, device: int = 0):
    """The device eight-point (or upright three-point) solver on n samples of 8 (3) bearing pairs [n, ms, 3] (validation
    aid).  -> E [n, 3, 3]"""
    ms = 3 if upright else 8
    b1 = np.ascontiguousarray(b1, np.float64).reshape(-1, ms, 3); b2 = np.ascontiguousarray(b2, np.float64).reshape(-1, ms, 3)
    n = len(b1); assert len(b2) == n
    E = np.zeros((max(n, 1), 9))
    p = lambda a: a.ctypes.data_as(_vp)   # noqa: E731
    check(lib().omvg_geom_debug_angular_solver(int(device), ESSENTIAL_UPRIGHT if upright else ESSENTIAL_ANGULAR, ctypes.c_uint32(n), p(b1), p(b2), p(E)))
    return E[:n].reshape(n, 3, 3).copy()


def debug_relative_pose(E, b1, b2, index, device: int = 0):
    """RelativePoseFromEssential(b1, b2, E, index) as the device filter runs it (validation aid).
    -> dict(counts [4] (cheirality count per pose of MotionFromEssential), selected (the chosen pose's list), ok)"""
    E = np.ascontiguousarray(E, np.float64).reshape(9)
    b1 = np.ascontiguousarray(b1, np.float64).reshape(-1, 3); b2 = np.ascontiguousarray(b2, np.float64).reshape(-1, 3)
    idx = np.ascontiguousarray(index, np.uint32).reshape(-1)
    assert len(b1) == len(b2)
    counts = np.zeros(4, np.int32); sel = np.zeros(max(len(idx), 1), np.uint32); ns = np.zeros(1, np.uint32); ok = np.zeros(1, np.int32)
    p = lambda a: a.ctypes.data_as(_vp)   # noqa: E731
    check(lib().omvg_geom_debug_relative_pose(int(device), p(E), ctypes.c_uint32(len(b1)), p(b1), p(b2), ctypes.c_uint32(len(idx)), p(idx),
                                              p(counts), p(sel), p(ns), p(ok)))
    return dict(counts=counts, selected=sel[:int(ns[0])].copy(), ok=bool(ok[0]))
