"""Seeded synthetic inputs for the two hot paths (SURVEY.md §8d).

Shared by tests/ and bench.py so the CUDA path, the oracle and the compiled reference all see
byte-identical inputs.  Nothing here is on the product path.

* :func:`ba_scene` — the BA scene family of BASELINE.json configs 1/2/5: cameras on a radius-1.5
  ring (0.2·sin 3θ wobble) looking at the origin (openMVG ``LookAt``, numeric/numeric.cpp:65-74),
  points uniform in [-0.6,0.6]^3, each point seen by ``obs_per_point`` cameras of a strided window,
  one shared pinhole intrinsic f=1000, pp=(500,500) (as in every reference BA test,
  sfm/sfm_data_BA_test.cpp:361), pixel noise N(0,0.5), perturbed initial poses/points.
* :func:`descriptors` — 128-D uint8 SIFT-like descriptors: bytes u·v/255 (right-skewed like
  root-SIFT); image k re-uses 30 % of image k-1's rows ±8 noise so the ratio test passes for a
  realistic fraction.
"""
from __future__ import annotations

import numpy as np

# cameras::EINTRINSIC (reference: cameras/Camera_Common.hpp:39-49)
PINHOLE_CAMERA = 1
PINHOLE_CAMERA_RADIAL1 = 2
PINHOLE_CAMERA_RADIAL3 = 3
PINHOLE_CAMERA_BROWN = 4
PINHOLE_CAMERA_FISHEYE = 5
CAMERA_SPHERICAL = 7          # no parameter block; the intrinsic slot carries the image size {w, h}
INTR_NPARAMS = {1: 3, 2: 4, 3: 6, 4: 8, 5: 7, 7: 0}
INTR_STRIDE = 8


def _look_at(center: np.ndarray, up=np.array([0.0, 1.0, 0.0])) -> np.ndarray:
    zc = center / np.linalg.norm(center)
    xc = np.cross(up, zc)
    xc /= np.linalg.norm(xc)
    yc = np.cross(zc, xc)
    return np.stack([xc, yc, zc])


def _rodrigues(aa: np.ndarray) -> np.ndarray:
    th = np.linalg.norm(aa)
    if th < 1e-300:
        return np.eye(3)
    k = aa / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)


def _log_so3(R: np.ndarray) -> np.ndarray:
    """Rotation matrix -> angle-axis (generic branch; scenes here never sit at theta≈pi)."""
    c = np.clip((np.trace(R) - 1.0) / 2.0, -1.0, 1.0)
    th = np.arccos(c)
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    s = np.linalg.norm(v)
    if s < 1e-300:
        return np.zeros(3)
    return v / s * th


def ba_scene(n_cams: int, n_points: int, obs_per_point: int, seed: int = 42,
             model: int = PINHOLE_CAMERA, n_intrinsics: int = 1, noise_px: float = 0.5,
             outlier_frac: float = 0.0) -> dict:
    """Flat BA problem in the include/omvg_b200.h layout (all float64 / int32, C-contiguous)."""
    rng = np.random.default_rng(seed)
    f, cx, cy = 1000.0, 500.0, 500.0
    gtR = np.zeros((n_cams, 3, 3))
    gtC = np.zeros((n_cams, 3))
    poses = np.zeros((n_cams, 6))
    for i in range(n_cams):
        th = i * 2 * np.pi / n_cams
        c = np.array([1.5 * np.sin(th), 0.2 * np.sin(3 * th), 1.5 * np.cos(th)])
        R = _look_at(-c)
        gtR[i], gtC[i] = R, c
        dR = _rodrigues(rng.normal(0, 0.005, 3))
        Ri = dR @ R
        Ci = c + rng.normal(0, 0.005, 3)
        poses[i, :3] = _log_so3(Ri)
        poses[i, 3:] = -Ri @ Ci
    intr = np.zeros((n_intrinsics, INTR_STRIDE))
    intr[:, 0], intr[:, 1], intr[:, 2] = f, cx, cy
    gt_dist = np.zeros(INTR_STRIDE)
    if model == PINHOLE_CAMERA_RADIAL1:
        gt_dist[3] = 0.05
    elif model == PINHOLE_CAMERA_RADIAL3:
        gt_dist[3:6] = [0.05, -0.01, 0.002]
    elif model == PINHOLE_CAMERA_BROWN:
        gt_dist[3:8] = [0.05, -0.01, 0.002, 0.001, -0.0005]
    elif model == PINHOLE_CAMERA_FISHEYE:
        gt_dist[3:7] = [0.02, -0.005, 0.001, 0.0]
    intr_model = np.full(n_intrinsics, model, np.int32)
    view_pose = np.arange(n_cams, dtype=np.int32)
    view_intr = (np.arange(n_cams) % n_intrinsics).astype(np.int32)

    X = rng.uniform(-0.6, 0.6, (n_points, 3))
    s0 = rng.integers(0, n_cams, n_points)
    k = np.arange(obs_per_point)
    stride = 1 + (np.arange(n_points) % 3)
    cam = (s0[:, None] + k[None, :] * stride[:, None]) % n_cams          # [P, K]
    # a point cannot be observed twice by the same view (Observations is keyed by view id)
    if obs_per_point * 3 > n_cams:
        cam = (s0[:, None] + k[None, :]) % n_cams
    assert obs_per_point <= n_cams
    obs_point = np.repeat(np.arange(n_points, dtype=np.int32), obs_per_point)
    obs_view = cam.reshape(-1).astype(np.int32)
    Xc = np.einsum('oij,oj->oi', gtR[obs_view], X[obs_point] - gtC[obs_view])
    if model == CAMERA_SPHERICAL:
        # Camera_Spherical.hpp / functor.hpp:700-712: lon = atan2(x, z), lat = atan2(-y, |(x, z)|), pixel = (lon, -lat) / 2pi * max(w, h) + (w, h) / 2
        w_img, h_img = 4000.0, 2000.0
        intr[:, 0], intr[:, 1], intr[:, 2] = w_img, h_img, 0.0
        lon = np.arctan2(Xc[:, 0], Xc[:, 2]); lat = np.arctan2(-Xc[:, 1], np.hypot(Xc[:, 0], Xc[:, 2]))
        size = max(w_img, h_img)
        xy = np.stack([lon / (2 * np.pi) * size + w_img / 2, -lat / (2 * np.pi) * size + h_img / 2], 1) + rng.normal(0, noise_px, (len(obs_view), 2))
    else:
        u = Xc[:, :2] / Xc[:, 2:3]
        u = _distort(u, model, gt_dist)
        xy = np.stack([cx + f * u[:, 0], cy + f * u[:, 1]], 1) + rng.normal(0, noise_px, (len(obs_view), 2))
    if outlier_frac > 0:
        bad = rng.random(len(obs_view)) < outlier_frac
        xy[bad] += rng.normal(0, 60.0, (int(bad.sum()), 2))
    points = X + rng.normal(0, 0.01, X.shape)
    return dict(
        poses=np.ascontiguousarray(poses), intrinsics=np.ascontiguousarray(intr),
        intr_model=intr_model, points=np.ascontiguousarray(points),
        view_pose=view_pose, view_intr=view_intr,
        obs_view=np.ascontiguousarray(obs_view), obs_point=np.ascontiguousarray(obs_point),
        obs_xy=np.ascontiguousarray(xy), gt_dist=gt_dist, gt_R=gtR, gt_C=gtC)


def add_gcp(scene: dict, n_gcp: int, weight: float = 20.0, views_per_gcp: int = 4, seed: int = 7) -> dict:
    """Ground control points as Adjust adds them (sfm_data_BA_ceres.cpp:398-452): landmarks held
    constant at their surveyed position, observed with residuals multiplied by ``weight`` and no
    robust loss.  In the flat layout they are extra points (``point_fixed`` = 1) whose observations
    carry ``obs_weight`` = weight and ``obs_no_loss`` = 1; appended after the regular ones."""
    rng = np.random.default_rng(seed)
    s = dict(scene)
    n_cams = len(s["poses"]); n_pts = len(s["points"]); n_obs = len(s["obs_view"])
    Xg = rng.uniform(-0.5, 0.5, (n_gcp, 3))
    first = rng.integers(0, n_cams, n_gcp)
    cam = ((first[:, None] + np.arange(views_per_gcp)[None, :] * max(1, n_cams // (2 * views_per_gcp))) % n_cams).astype(np.int32)
    ov = cam.reshape(-1)
    op = np.repeat(np.arange(n_gcp, dtype=np.int32), views_per_gcp)
    Xc = np.einsum('oij,oj->oi', s["gt_R"][ov], Xg[op] - s["gt_C"][ov])
    u = _distort(Xc[:, :2] / Xc[:, 2:3], int(s["intr_model"][0]), s["gt_dist"])
    f, cx, cy = 1000.0, 500.0, 500.0
    xy = np.stack([cx + f * u[:, 0], cy + f * u[:, 1]], 1) + rng.normal(0, 0.3, (len(ov), 2))
    s["points"] = np.ascontiguousarray(np.concatenate([s["points"], Xg]))
    s["obs_view"] = np.ascontiguousarray(np.concatenate([s["obs_view"], ov]).astype(np.int32))
    s["obs_point"] = np.ascontiguousarray(np.concatenate([s["obs_point"], op + n_pts]).astype(np.int32))
    s["obs_xy"] = np.ascontiguousarray(np.concatenate([s["obs_xy"], xy]))
    s["obs_weight"] = np.concatenate([np.ones(n_obs), np.full(len(ov), float(weight))])
    s["obs_no_loss"] = np.concatenate([np.zeros(n_obs, np.uint8), np.ones(len(ov), np.uint8)])
    s["point_fixed"] = np.concatenate([np.zeros(n_pts, np.uint8), np.ones(n_gcp, np.uint8)])
    return s


def add_priors(scene: dict, sigma: float = 0.01, weight=(1.0, 1.0, 1.0), seed: int = 11,
               offset=(0.0, 0.0, 0.0), scale: float = 1.0) -> dict:
    """Pose-centre (GPS) priors on every view (sfm_view_priors.hpp:27-80): prior centre =
    scale * ground-truth centre + offset + N(0, sigma), per-axis weight.  ``prior_huber_a`` is the
    squared median fitting error and is filled by the registration step (host-side geometry, done by
    the C++ shim with openMVG's own functions)."""
    rng = np.random.default_rng(seed)
    s = dict(scene)
    n = len(s["poses"])
    s["prior_pose"] = np.arange(n, dtype=np.int32)
    s["prior_center"] = np.ascontiguousarray(scale * s["gt_C"] + np.asarray(offset) + rng.normal(0, sigma, (n, 3)))
    s["prior_weight"] = np.ascontiguousarray(np.tile(np.asarray(weight, np.float64), (n, 1)))
    s["prior_huber_a"] = 0.0
    return s


def _distort(u: np.ndarray, model: int, d: np.ndarray) -> np.ndarray:
    """Forward distortion of normalised coordinates, per camera model
    (sfm/sfm_data_BA_ceres_camera_functor.hpp:262-267, 372-379, 489-500, 609-626)."""
    if model == PINHOLE_CAMERA:
        return u
    r2 = (u * u).sum(1, keepdims=True)
    if model == PINHOLE_CAMERA_RADIAL1:
        return u * (1 + d[3] * r2)
    if model == PINHOLE_CAMERA_RADIAL3:
        return u * (1 + d[3] * r2 + d[4] * r2 ** 2 + d[5] * r2 ** 3)
    if model == PINHOLE_CAMERA_BROWN:
        k1, k2, k3, t1, t2 = d[3:8]
        rc = 1 + k1 * r2 + k2 * r2 ** 2 + k3 * r2 ** 3
        x, y = u[:, :1], u[:, 1:]
        tx = t2 * (r2 + 2 * x * x) + 2 * t1 * x * y
        ty = t1 * (r2 + 2 * y * y) + 2 * t2 * x * y
        return np.concatenate([x * rc + tx, y * rc + ty], 1)
    if model == PINHOLE_CAMERA_FISHEYE:
        r = np.sqrt(r2)
        th = np.arctan(r)
        thd = th * (1 + d[3] * th ** 2 + d[4] * th ** 4 + d[5] * th ** 6 + d[6] * th ** 8)
        scale = np.where(r > 1e-8, thd / np.maximum(r, 1e-300), 1.0)
        return u * scale
    raise ValueError(model)


def descriptors(n_images: int, n_desc, seed: int = 7, inlier_frac: float = 0.3) -> list:
    """List of [n_k,128] uint8 arrays; ``n_desc`` is an int or a per-image sequence."""
    rng = np.random.default_rng(seed)
    counts = [int(n_desc)] * n_images if np.isscalar(n_desc) else [int(x) for x in n_desc]
    out = []
    for k, n in enumerate(counts):
        u = rng.integers(0, 256, (n, 128), dtype=np.int32)
        v = rng.integers(0, 256, (n, 128), dtype=np.int32)
        d = (u * v // 255).astype(np.uint8)
        if k > 0 and n > 0 and len(out[-1]) > 0:
            m = min(n, len(out[-1]))
            sel = rng.random(m) < inlier_frac
            noise = rng.integers(-8, 9, (m, 128), dtype=np.int32)
            base = out[-1][:m].astype(np.int32)
            d[:m][sel] = np.clip(base[sel] + noise[sel], 0, 255).astype(np.uint8)
        out.append(np.ascontiguousarray(d))
    return out


def descriptor_collection(n_images: int, n_desc: int = 5000, seed: int = 1000, block: int = 25, lo: int = 0, hi=None) -> list:
    """The M1 / M2 collections of BASELINE.json configs[2]/[3] (200 / 1000 images x 5000): blocks of ``block``
    images, block b drawn by :func:`descriptors` with seed ``seed + b``.  Any [lo, hi) slice can be generated
    without the rest (each rank of a sharded run draws only its own images) and M1 is a prefix of M2."""
    hi = n_images if hi is None else min(hi, n_images)
    out = []
    for b in range(lo // block, (max(hi, lo + 1) - 1) // block + 1):
        if hi <= lo:
            break
        n_b = min(block, n_images - b * block)
        blk = descriptors(n_b, n_desc, seed=seed + b)
        a0 = max(lo, b * block) - b * block; a1 = min(hi, (b + 1) * block) - b * block
        out.extend(blk[a0:a1])
    return out


def sampled_pairs(n_images: int, n_pairs: int, seed: int = 5):
    """A seeded sample of distinct (I<J) pairs in Pair_Set (lexicographic) order."""
    rng = np.random.default_rng(seed)
    total = n_images * (n_images - 1) // 2
    pick = np.sort(rng.choice(total, size=min(n_pairs, total), replace=False))
    i, j = np.triu_indices(n_images, 1)
    return np.ascontiguousarray(i[pick].astype(np.uint32)), np.ascontiguousarray(j[pick].astype(np.uint32))


def exhaustive_pairs(n_images: int):
    """Pair_Builder.hpp:25-33 — all (I,J) with I<J in lexicographic order."""
    i, j = np.triu_indices(n_images, 1)
    return np.ascontiguousarray(i.astype(np.uint32)), np.ascontiguousarray(j.astype(np.uint32))


def two_view_matches(n: int, outlier_frac: float = 0.3, noise_px: float = 0.5, seed: int = 3, wh=(1000, 1000), planar: bool = False):
    """Putative matches of one image pair for the geometric filter (SURVEY §8f N4): n correspondences, a fraction
    of them gross outliers, the rest projections of a 3-D point cloud in two pinhole views + pixel noise.
    Positions are rounded to float32 as openMVG features store them (features/feature.hpp: PointFeature x, y are float).
    planar=True puts the points on a plane (homography model).
    -> (xI [n,2], xJ [n,2]) float64, inlier mask [n]"""
    rng = np.random.default_rng(seed)
    w, h = wh
    f = 1.1 * max(w, h)
    X = np.stack([rng.uniform(-1.5, 1.5, n), rng.uniform(-1.2, 1.2, n), rng.uniform(4.0, 9.0, n)], 1)
    if planar:                                                 # a plane: the two views are related by a homography
        X[:, 2] = 6.0 + 0.3 * X[:, 0] - 0.2 * X[:, 1]
    R2 = _rodrigues(np.array([0.03, -0.25, 0.02])); C2 = np.array([1.2, 0.05, 0.3])

    def proj(R, C):
        Xc = (X - C) @ R.T
        return np.stack([w / 2 + f * Xc[:, 0] / Xc[:, 2], h / 2 + f * Xc[:, 1] / Xc[:, 2]], 1)
    xI = proj(np.eye(3), np.zeros(3)) + rng.normal(0, noise_px, (n, 2))
    xJ = proj(R2, C2) + rng.normal(0, noise_px, (n, 2))
    out = rng.random(n) < outlier_frac
    xJ[out] = np.stack([rng.uniform(0, w, int(out.sum())), rng.uniform(0, h, int(out.sum()))], 1)
    return xI.astype(np.float32).astype(np.float64), xJ.astype(np.float32).astype(np.float64), ~out


def calibrated_two_view_matches(n: int, outlier_frac: float = 0.3, seed: int = 3, wh=(1600, 1200), intr_I=None, intr_J=None,
                                noise_px: float = 0.5, motion: str = "general"):
    """Putative matches of one CALIBRATED image pair for the essential-matrix filter (DESIGN §3.8): like
    two_view_matches, but each view has its own pinhole intrinsic (f, ppx, ppy), by default with different focal
    lengths and principal points.  motion: "general" (sideways + rotation), "short" (a baseline of 2 % of the depth),
    "forward" (the camera moves along its optical axis), "planar" (the points lie close to a plane).
    -> (xI [n,2], xJ [n,2]) float64, inlier mask [n], intr_I (f, ppx, ppy), intr_J (f, ppx, ppy)"""
    rng = np.random.default_rng(seed)
    w, h = wh
    if intr_I is None:
        intr_I = (1.1 * max(w, h), w / 2 + 13.5, h / 2 - 7.25)
    if intr_J is None:
        intr_J = (0.9 * max(w, h), w / 2 - 21.0, h / 2 + 9.5)
    X = np.stack([rng.uniform(-1.5, 1.5, n), rng.uniform(-1.2, 1.2, n), rng.uniform(4.0, 9.0, n)], 1)
    if motion == "planar":
        X[:, 2] = 6.0 + 0.3 * X[:, 0] - 0.2 * X[:, 1] + rng.normal(0, 0.01, n)
    R2, C2 = {"general": (_rodrigues(np.array([0.03, -0.25, 0.02])), np.array([1.2, 0.05, 0.3])),
              "short": (_rodrigues(np.array([0.01, -0.02, 0.005])), np.array([0.12, 0.01, 0.02])),
              "forward": (_rodrigues(np.array([0.01, 0.02, -0.01])), np.array([0.02, -0.01, 1.5])),
              "planar": (_rodrigues(np.array([0.05, -0.2, 0.03])), np.array([1.0, 0.1, 0.2]))}[motion]

    def proj(R, C, k):
        Xc = (X - C) @ R.T
        return np.stack([k[1] + k[0] * Xc[:, 0] / Xc[:, 2], k[2] + k[0] * Xc[:, 1] / Xc[:, 2]], 1)
    xI = proj(np.eye(3), np.zeros(3), intr_I) + rng.normal(0, noise_px, (n, 2))
    xJ = proj(R2, C2, intr_J) + rng.normal(0, noise_px, (n, 2))
    out = rng.random(n) < outlier_frac
    xJ[out] = np.stack([rng.uniform(0, w, int(out.sum())), rng.uniform(0, h, int(out.sum()))], 1)
    return (xI.astype(np.float32).astype(np.float64), xJ.astype(np.float32).astype(np.float64), ~out,
            tuple(float(v) for v in intr_I), tuple(float(v) for v in intr_J))


def spherical_bearings(xy: np.ndarray, wh=(2000, 1000)) -> np.ndarray:
    """Bearing vectors of equirectangular pixel positions [n, 2], as Camera_Spherical::operator() forms them
    (cameras/Camera_Spherical.hpp:115-131), with numpy's sin / cos."""
    w, h = wh
    size = float(max(w, h))
    lon = (xy[:, 0] - w / 2.0) / size * 2 * np.pi
    lat = -((xy[:, 1] - h / 2.0) / size) * 2 * np.pi
    return np.stack([np.cos(lat) * np.sin(lon), -np.sin(lat), np.cos(lat) * np.cos(lon)], 1)


ANGULAR_MOTIONS = ("general", "short", "forward", "full", "upright", "upright_tilt", "rotation")


def spherical_two_view_matches(n: int, outlier_frac: float = 0.3, seed: int = 3, motion: str = "general", wh=(2000, 1000),
                               noise_px: float = 0.3):
    """Putative matches of one pair of 360° (equirectangular) views for the angular essential-matrix filters (DESIGN
    §3.10).  motion: "general" (sideways + rotation), "short" (a baseline of 1 % of the depth), "forward" (along the
    optical axis), "full" (general motion, points all around the camera, half of them behind it: bearing z < 0),
    "upright" (a rotation about y and a translation with t_y = 0, the upright solver's model), "upright_tilt" (the same
    with a small t_y and a small tilt, off that model), "rotation" (a baseline of 1e-6 of the depth: the cheirality test
    is ambiguous).  Pixel positions are rounded to float32, as openMVG stores features, and the bearings are formed
    from them.  -> (xy_I [n,2], xy_J [n,2], bI [n,3], bJ [n,3], inlier mask [n])"""
    rng = np.random.default_rng(seed)
    w, h = wh
    if motion == "full":
        d = rng.normal(size=(n, 3))
    else:
        d = np.stack([rng.uniform(-1.2, 1.2, n), rng.uniform(-0.8, 0.8, n), np.ones(n)], 1)
    X = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(3.0, 10.0, (n, 1))
    R2, C2 = {"general": (_rodrigues(np.array([0.03, -0.25, 0.02])), np.array([1.2, 0.05, 0.3])),
              "short": (_rodrigues(np.array([0.01, -0.02, 0.005])), np.array([0.06, 0.01, 0.02])),
              "forward": (_rodrigues(np.array([0.01, 0.02, -0.01])), np.array([0.02, -0.01, 1.5])),
              "full": (_rodrigues(np.array([0.2, 0.9, -0.1])), np.array([0.9, -0.3, -0.6])),
              "upright": (_rodrigues(np.array([0.0, 0.35, 0.0])), np.array([0.8, 0.0, 0.5])),
              "upright_tilt": (_rodrigues(np.array([0.02, 0.35, -0.015])), np.array([0.8, 0.04, 0.5])),
              "rotation": (_rodrigues(np.array([0.05, 0.3, -0.02])), np.array([1e-6, 0.0, 0.0]))}[motion]

    def pix(b):
        b = b / np.linalg.norm(b, axis=1, keepdims=True)
        lon = np.arctan2(b[:, 0], b[:, 2]); lat = -np.arcsin(np.clip(b[:, 1], -1, 1))
        size = float(max(w, h))
        return np.stack([lon / (2 * np.pi) * size + w / 2.0, -lat / (2 * np.pi) * size + h / 2.0], 1)
    xI = pix(X) + rng.normal(0, noise_px, (n, 2))
    xJ = pix((X - C2) @ R2.T) + rng.normal(0, noise_px, (n, 2))
    out = rng.random(n) < outlier_frac
    xJ[out] = np.stack([rng.uniform(0, w, int(out.sum())), rng.uniform(0, h, int(out.sum()))], 1)
    xI = np.mod(xI, [w, h]).astype(np.float32).astype(np.float64)
    xJ = np.mod(xJ, [w, h]).astype(np.float32).astype(np.float64)
    return xI, xJ, spherical_bearings(xI, wh), spherical_bearings(xJ, wh), ~out


def guided_scene(n_views: int, n_feat, seed: int = 9, wh=(1600, 1200), planar: bool = False, shared_frac: float = 0.6,
                 n_dup: int = 0, desc_noise: int = 8, noise_px: float = 0.5):
    """Per-view feature positions and SIFT-like descriptors of one 3-D scene for guided matching (DESIGN §3.9).
    n_feat: features per view (int or list).  About shared_frac of each view's features are projections of shared
    3-D points (one base descriptor per point, +-desc_noise per view, 0.5 px position noise); the rest are distractors
    with their own random descriptors and positions.  planar: the points lie on one plane (homography scenes).
    n_dup: that many features per view repeat the position of another feature of the view (different descriptor).
    Views look at the scene from a short arc with different pinhole intrinsics; feature order is shuffled.
    Positions are float32 values (openMVG keeps feature coordinates in float).
    -> dict xy [list of [n,2] float64], desc [list of [n,128] uint8], point [list of [n] int, -1 = distractor],
       K [list of 3x3], R, C [lists], plane (n, d) or None, wh."""
    rng = np.random.default_rng(seed)
    w, h = wh
    counts = [int(n_feat)] * n_views if np.isscalar(n_feat) else [int(v) for v in n_feat]
    n_pts = max(1, int(shared_frac * max(counts + [1]) * 1.6))
    X = np.stack([rng.uniform(-2.0, 2.0, n_pts), rng.uniform(-1.5, 1.5, n_pts), rng.uniform(5.0, 9.0, n_pts)], 1)
    plane = None
    if planar:
        nrm = np.array([0.1, -0.15, 1.0]); nrm /= np.linalg.norm(nrm)
        plane = (nrm, 7.0)
        X[:, 2] = (7.0 - nrm[0] * X[:, 0] - nrm[1] * X[:, 1]) / nrm[2]
    base = rng.integers(0, 140, (n_pts, 128), dtype=np.int32)
    Ks, Rs, Cs, xys, descs, pids = [], [], [], [], [], []
    for v in range(n_views):
        f = max(w, h) * (0.9 + 0.25 * rng.random())
        K = np.array([[f, 0, w / 2 + rng.uniform(-20, 20)], [0, f, h / 2 + rng.uniform(-20, 20)], [0, 0, 1.0]])
        ang = 0.35 * (v / max(1, n_views - 1) - 0.5)
        C = np.array([7.0 * np.sin(ang), 0.2 * rng.normal(), 7.0 - 7.0 * np.cos(ang)])
        R = _rodrigues(np.array([0.02 * rng.normal(), -ang, 0.02 * rng.normal()]))
        Xc = (X - C) @ R.T
        uv = np.stack([K[0, 2] + f * Xc[:, 0] / Xc[:, 2], K[1, 2] + f * Xc[:, 1] / Xc[:, 2]], 1) + rng.normal(0, noise_px, (n_pts, 2))
        vis = np.flatnonzero((Xc[:, 2] > 0) & (uv[:, 0] >= 0) & (uv[:, 0] < w) & (uv[:, 1] >= 0) & (uv[:, 1] < h))
        n = counts[v]
        ns = min(len(vis), int(round(shared_frac * n)), n)
        sel = rng.choice(vis, ns, replace=False) if ns else np.zeros(0, np.int64)
        nd = n - ns
        xy = np.concatenate([uv[sel], np.stack([rng.uniform(0, w, nd), rng.uniform(0, h, nd)], 1)])
        d = np.concatenate([base[sel] + rng.integers(-desc_noise, desc_noise + 1, (ns, 128)), rng.integers(0, 140, (nd, 128))])
        pid = np.concatenate([sel, -np.ones(nd, np.int64)])
        perm = rng.permutation(n)
        xy, d, pid = xy[perm], d[perm], pid[perm]
        if n_dup and n > 1:
            src = rng.choice(n, min(n_dup, n - 1), replace=False)
            dst = (src + 1 + rng.integers(0, n - 1, len(src))) % n
            xy[dst] = xy[src]
        Ks.append(K); Rs.append(R); Cs.append(C)
        xys.append(xy.astype(np.float32).astype(np.float64))
        descs.append(np.clip(d, 0, 255).astype(np.uint8))
        pids.append(pid)
    return dict(xy=xys, desc=descs, point=pids, K=Ks, R=Rs, C=Cs, plane=plane, wh=(w, h))


def scene_fundamental(scene: dict, a: int, b: int) -> np.ndarray:
    """F with x_b^T F x_a = 0 for the views a, b of guided_scene (the epipolar line of x_a in view b is F x_a)."""
    R = scene["R"][b] @ scene["R"][a].T
    t = scene["R"][b] @ (scene["C"][a] - scene["C"][b])
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    F = np.linalg.inv(scene["K"][b]).T @ tx @ R @ np.linalg.inv(scene["K"][a])
    return F / np.linalg.norm(F)


def scene_homography(scene: dict, a: int, b: int) -> np.ndarray:
    """The homography x_b ~ H x_a induced by the plane of a planar guided_scene (by the plane at infinity otherwise)."""
    R = scene["R"][b] @ scene["R"][a].T
    G = R
    if scene["plane"] is not None:
        nrm, d = scene["plane"]
        t = scene["R"][b] @ (scene["C"][a] - scene["C"][b])
        G = R + np.outer(t, scene["R"][a] @ nrm) / (d - nrm @ scene["C"][a])
    H = scene["K"][b] @ G @ np.linalg.inv(scene["K"][a])
    return H / H[2, 2]
