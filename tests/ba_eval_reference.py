"""Extended-precision reference of one BA evaluation: residuals, Jacobian blocks, cost and pixel residual norms
(numpy, np.longdouble), with an error scale for every entry.

The expressions are the reference's own, differentiated forward-mode (ceres/jet.h) over the lanes
[intrinsics (8) | pose (6) | point (3)], as oracle/ba_oracle.cpp restates them:
    AngleAxisRotatePoint (rotation.h:563-622), both branches, the branch decided on the float64 theta^2 as Ceres does;
    hnormalized; the five pinhole functors and the spherical one (sfm_data_BA_ceres_camera_functor.hpp:103-717),
    the fisheye r > 1e-8 switch included; WeightedCostFunction (:35-90); HuberLoss (loss_function.cc:47-61) with
    Ceres' Corrector (corrector.cc:41-155; Huber has rho'' <= 0, so r and J are scaled by sqrt(rho')), or no loss;
    the option masks (free_masks of ba_step_reference.py); PoseCenterConstraintCostFunction
    (sfm_data_BA_ceres.cpp:44-80) under HuberLoss(prior_huber_a).
Every value and derivative carries a magnitude m: the first-order error scale of the expression that forms it,
    m(a +- b) = m(a) + m(b),  m(a b) = m(a) |b| + |a| m(b),  m(a / b) = (m(a) + |a / b| m(b)) / |b|,
    m(f(a)) = |f(a)| + |f'(a)| m(a) for sqrt, sin, cos, atan, atan2,
seeded with |x| for every input, so that m >= |value| and a rounding error of eps relative in any term of an entry
moves it by at most eps m.  "Sum of the absolute values of the terms": where an entry cancels (a landmark far from
the origin seen from nearby, a small-angle rotation derivative) its bar grows with the terms, not with the result.
Outputs are in the layout of omvg_ba_debug_eval / oracle_ba_eval: r[n][2], J_intr[n][2][8], J_pose[n][2][6],
J_point[n][2][3], NOT Jacobi-scaled."""
import numpy as np

from ba_step_reference import KI, free_masks

LD = np.longdouble
assert np.finfo(LD).eps < 1e-18, "long double is not an extended type on this platform"
NJ = KI + 6 + 3
DBL_EPSILON = float(np.finfo(np.float64).eps)
DBL_MIN = float(np.finfo(np.float64).tiny)


class Jet:
    """A value a[n] with derivatives v[n][NJ], and their magnitudes ma[n], mv[n][NJ] (see the module docstring)."""
    __slots__ = ("a", "v", "ma", "mv")

    def __init__(self, a, v, ma, mv):
        self.a, self.v, self.ma, self.mv = a, v, ma, mv

    @staticmethod
    def const(c, n):
        c = np.broadcast_to(np.asarray(c, LD), (n,)).copy()
        z = np.zeros((n, NJ), LD)
        return Jet(c, z, np.abs(c), z.copy())

    @staticmethod
    def var(x, lane):
        j = Jet.const(x, len(x)); j.v[:, lane] = 1; j.mv[:, lane] = 1
        return j

    def __add__(f, g):
        g = _lift(g, f)
        return Jet(f.a + g.a, f.v + g.v, f.ma + g.ma, f.mv + g.mv)

    __radd__ = __add__

    def __sub__(f, g):
        g = _lift(g, f)
        return Jet(f.a - g.a, f.v - g.v, f.ma + g.ma, f.mv + g.mv)

    def __rsub__(f, g):
        return _lift(g, f) - f

    def __neg__(f):
        return Jet(-f.a, -f.v, f.ma, f.mv)

    def __mul__(f, g):
        g = _lift(g, f)
        fa, ga, fma, gma = f.a[:, None], g.a[:, None], f.ma[:, None], g.ma[:, None]
        return Jet(f.a * g.a, fa * g.v + f.v * ga, f.ma * np.abs(g.a) + np.abs(f.a) * g.ma,
                   fma * np.abs(g.v) + np.abs(fa) * g.mv + f.mv * np.abs(ga) + np.abs(f.v) * gma)

    __rmul__ = __mul__

    def __truediv__(f, g):          # jet.h: q = f.a / g.a, (f.v - q g.v) / g.a
        g = _lift(g, f)
        q = f.a / g.a
        mq = (f.ma + np.abs(q) * g.ma) / np.abs(g.a)
        num = f.v - q[:, None] * g.v
        mnum = f.mv + mq[:, None] * np.abs(g.v) + np.abs(q)[:, None] * g.mv
        v = num / g.a[:, None]
        return Jet(q, v, mq, (mnum + np.abs(v) * g.ma[:, None]) / np.abs(g.a)[:, None])

    def __rtruediv__(f, g):
        return _lift(g, f) / f

    def _unary(f, y, d1, d2):
        """f(a) with f' = d1, f'' = d2 at a."""
        md1 = np.abs(d1) + np.abs(d2) * f.ma
        return Jet(y, d1[:, None] * f.v, np.abs(y) + np.abs(d1) * f.ma,
                   md1[:, None] * np.abs(f.v) + np.abs(d1)[:, None] * f.mv)

    def sqrt(f):
        y = np.sqrt(f.a)
        return f._unary(y, 1 / (2 * y), -1 / (4 * y * f.a))

    def sin(f):
        return f._unary(np.sin(f.a), np.cos(f.a), -np.sin(f.a))

    def cos(f):
        return f._unary(np.cos(f.a), -np.sin(f.a), -np.cos(f.a))

    def atan(f):
        t = 1 / (1 + f.a * f.a)
        return f._unary(np.arctan(f.a), t, -2 * f.a * t * t)

    def take(f, idx):
        return Jet(f.a[idx], f.v[idx], f.ma[idx], f.mv[idx])


def _lift(g, like):
    return g if isinstance(g, Jet) else Jet.const(g, len(like.a))


def atan2(y, x):
    """jet.h:682-695: atan2(y, x) + (x dy - y dx) / (x^2 + y^2)."""
    t = 1 / (x.a * x.a + y.a * y.a)
    mt = t * t * 2 * (np.abs(x.a) * x.ma + np.abs(y.a) * y.ma)
    inner = x.a[:, None] * y.v - y.a[:, None] * x.v
    minner = x.ma[:, None] * np.abs(y.v) + np.abs(x.a)[:, None] * y.mv + y.ma[:, None] * np.abs(x.v) + np.abs(y.a)[:, None] * x.mv
    val = np.arctan2(y.a, x.a)
    return Jet(val, t[:, None] * inner, np.abs(val) + t * (np.abs(x.a) * y.ma + np.abs(y.a) * x.ma),
               t[:, None] * minner + mt[:, None] * np.abs(inner))


def where(c, f, g):
    c1 = c[:, None]
    return Jet(np.where(c, f.a, g.a), np.where(c1, f.v, g.v), np.where(c, f.ma, g.ma), np.where(c1, f.mv, g.mv))


def taylor_branch(aa):
    """AngleAxisRotatePoint's branch: theta^2 <= DBL_EPSILON, theta^2 formed in float64 as Ceres forms it."""
    aa = np.asarray(aa, np.float64)
    t2 = aa[..., 0] * aa[..., 0] + aa[..., 1] * aa[..., 1] + aa[..., 2] * aa[..., 2]
    return ~(t2 > DBL_EPSILON)


def rotate(aa, pt, taylor):
    """rotation.h:563-622 for jets aa[3], pt[3]; taylor[n] selects the branch."""
    theta2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2]
    with np.errstate(all="ignore"):
        theta = theta2.sqrt(); c = theta.cos(); s = theta.sin(); ti = 1.0 / theta
        w = [aa[0] * ti, aa[1] * ti, aa[2] * ti]
        wxp = [w[1] * pt[2] - w[2] * pt[1], w[2] * pt[0] - w[0] * pt[2], w[0] * pt[1] - w[1] * pt[0]]
        tmp = (w[0] * pt[0] + w[1] * pt[1] + w[2] * pt[2]) * (1.0 - c)
        full = [pt[i] * c + wxp[i] * s + w[i] * tmp for i in range(3)]
    axp = [aa[1] * pt[2] - aa[2] * pt[1], aa[2] * pt[0] - aa[0] * pt[2], aa[0] * pt[1] - aa[1] * pt[0]]
    small = [pt[i] + axp[i] for i in range(3)]
    return [where(taylor, small[i], full[i]) for i in range(3)]


def _functor(model, K, E, X, xy, taylor):
    """sfm_data_BA_ceres_camera_functor.hpp, one model for all rows given (jets K[8], E[6], X[3])."""
    n = len(xy)
    p = rotate(E[:3], X, taylor)
    p = [p[i] + E[3 + i] for i in range(3)]
    if model == 7:                              # :662-717; K[0], K[1] are the image size, constants
        lon = atan2(p[0], p[2])
        lat = atan2(-p[1], (p[0] * p[0] + p[2] * p[2]).sqrt())
        wi, hi = K[0].a, K[1].a
        size = Jet.const(np.maximum(wi, hi), n)
        two_pi = LD(2 * np.pi)                  # T(2 * M_PI): the float64 constant
        return (lon / two_pi * size + Jet.const(wi / 2, n) - Jet.const(xy[:, 0], n),
                (-lat) / two_pi * size + Jet.const(hi / 2, n) - Jet.const(xy[:, 1], n))
    x, y = p[0] / p[2], p[1] / p[2]
    f, ppx, ppy = K[0], K[1], K[2]
    if model == 1:
        dx, dy = x, y
    elif model in (2, 3, 4):
        r2 = x * x + y * y
        if model == 2:
            rc = 1.0 + K[3] * r2
        else:
            r4 = r2 * r2; r6 = r4 * r2
            rc = 1.0 + K[3] * r2 + K[4] * r4 + K[5] * r6
        dx, dy = x * rc, y * rc
        if model == 4:
            t1, t2 = K[6], K[7]
            dx = dx + (t2 * (r2 + 2.0 * x * x) + 2.0 * t1 * x * y)
            dy = dy + (t1 * (r2 + 2.0 * y * y) + 2.0 * t2 * x * y)
    elif model == 5:                            # :580-627
        r2 = x * x + y * y
        with np.errstate(all="ignore"):
            r = r2.sqrt()
            th = r.atan(); th2 = th * th; th3 = th2 * th; th4 = th2 * th2; th5 = th4 * th; th7 = th3 * th3 * th
            th8 = th4 * th4; th9 = th8 * th
            thd = th + K[3] * th3 + K[4] * th5 + K[5] * th7 + K[6] * th9
            cd = thd * (1.0 / r)
        cd = where(r.a > LD(1e-8), cd, Jet.const(1.0, n))
        dx, dy = x * cd, y * cd
    else:
        raise ValueError(f"camera model {model}")
    return ppx + dx * f - Jet.const(xy[:, 0], n), ppy + dy * f - Jet.const(xy[:, 1], n)


def _huber(s, ms, a, lossy):
    """(rho0, m(rho0), sqrt(rho1), its relative magnitude) of HuberLoss(a) at s = |r|^2 (TrivialLoss where not lossy).
    In the tail sqrt(rho1) = sqrt(a / |r|) inherits half the relative error of |r|."""
    b = LD(a) * LD(a)
    tail = lossy & (s > b)
    with np.errstate(all="ignore"):
        rr = np.sqrt(s); mrr = rr + ms / (2 * rr)
        rho0 = np.where(tail, 2 * LD(a) * rr - b, s)
        mrho0 = np.where(tail, 2 * LD(a) * mrr + b, ms)
        sr = np.sqrt(np.where(tail, np.maximum(LD(DBL_MIN), LD(a) / rr), LD(1)))
        rel = np.where(tail, 1 + mrr / (2 * rr), 0)
    return rho0, mrho0, sr, rel


def _sq(r):
    """s = sum r_i^2 and its magnitude, from residual jets."""
    s = sum(x.a * x.a for x in r)
    return s, s + sum(2 * np.abs(x.a) * x.ma for x in r)


def evaluate(s, use_loss=1, huber_a=16.0, intrinsics_opt=14, extrinsics_opt=6, structure_opt=1):
    """One evaluation of scene s.  Returns a dict of long double arrays:
    r, J_intr, J_pose, J_point (as omvg_ba_debug_eval), cost (1/2 sum rho, observations only), norms (|r| in pixels,
    unweighted and without loss: omvg_ba_residual_norms), and m_<name> for each: their magnitudes (m_cost is the
    sum over observations of the magnitude of 1/2 rho).  Taylor-branch poses: `taylor` [n_obs]."""
    ov = np.asarray(s["obs_view"]); op = np.asarray(s["obs_point"])
    pose = np.asarray(s["view_pose"])[ov]; intr = np.asarray(s["view_intr"])[ov]
    poses = np.asarray(s["poses"], np.float64); K8 = np.asarray(s["intrinsics"], np.float64); pts = np.asarray(s["points"], np.float64)
    model = np.asarray(s["intr_model"])[intr]
    xy = np.asarray(s["obs_xy"], LD)
    n = len(ov)
    taylor = taylor_branch(poses[pose])
    out = {k: np.zeros(sh, LD) for k, sh in (("r", (n, 2)), ("J_intr", (n, 2, KI)), ("J_pose", (n, 2, 6)), ("J_point", (n, 2, 3)))}
    out.update({"m_" + k: np.zeros_like(v) for k, v in list(out.items())})
    out.update(norms=np.zeros(n, LD), m_norms=np.zeros(n, LD), obs_cost=np.zeros(n, LD), m_obs_cost=np.zeros(n, LD))
    w = np.ones(n, LD) if s.get("obs_weight") is None else np.asarray(s["obs_weight"], LD)
    lossy = np.full(n, bool(use_loss))
    if s.get("obs_no_loss") is not None:
        lossy &= ~np.asarray(s["obs_no_loss"]).astype(bool)
    for mdl in np.unique(model):
        idx = np.flatnonzero(model == mdl)
        K = [Jet.var(K8[intr[idx], k], k) for k in range(KI)]
        E = [Jet.var(poses[pose[idx], k], KI + k) for k in range(6)]
        X = [Jet.var(pts[op[idx], k], KI + 6 + k) for k in range(3)]
        R = _functor(int(mdl), K, E, X, xy[idx], taylor[idx])
        nrm2, mnrm2 = _sq(R)
        out["norms"][idx] = np.sqrt(nrm2); out["m_norms"][idx] = R[0].ma + R[1].ma
        wi = w[idx]
        R = [Jet(x.a * wi, x.v * wi[:, None], x.ma * np.abs(wi), x.mv * np.abs(wi)[:, None]) for x in R]
        sq, msq = _sq(R)
        rho0, mrho0, sr, rel = _huber(sq, msq, huber_a, lossy[idx])
        out["obs_cost"][idx] = rho0 / 2; out["m_obs_cost"][idx] = mrho0 / 2
        for row in range(2):
            out["r"][idx, row] = sr * R[row].a; out["m_r"][idx, row] = sr * (R[row].ma + rel * np.abs(R[row].a))
            for name, lo, hi in (("J_intr", 0, KI), ("J_pose", KI, KI + 6), ("J_point", KI + 6, NJ)):
                out[name][idx, row] = sr[:, None] * R[row].v[:, lo:hi]
                out["m_" + name][idx, row] = sr[:, None] * (R[row].mv[:, lo:hi] + rel[:, None] * np.abs(R[row].v[:, lo:hi]))
    fp, fc, fi = free_masks(s, intrinsics_opt, extrinsics_opt, structure_opt)
    for name, mask in (("J_point", fp[op]), ("J_pose", fc[pose]), ("J_intr", fi[intr])):
        out[name] = out[name] * mask[:, None, :]; out["m_" + name] = out["m_" + name] * mask[:, None, :]
    out["cost"] = out["obs_cost"].sum(); out["m_cost"] = out["m_obs_cost"].sum()
    out["taylor"] = taylor
    return out


def evaluate_priors(s, extrinsics_opt=6):
    """The pose-centre prior rows: r = w .* (-AngleAxisRotatePoint(-aa, t) - c0) under HuberLoss(prior_huber_a), with
    Ceres' correction.  Returns r [n][3], J [n][3][6] (pose columns, masked), cost, and m_r, m_J, m_cost."""
    pp = np.asarray(s["prior_pose"]); n = len(pp)
    poses = np.asarray(s["poses"], np.float64)[pp]
    c0 = np.asarray(s["prior_center"], LD); w = np.asarray(s["prior_weight"], LD)
    E = [Jet.var(poses[:, k], KI + k) for k in range(6)]
    c = rotate([-E[0], -E[1], -E[2]], E[3:], taylor_branch(-poses[:, :3]))
    R = [(c[i] * -1.0 - Jet.const(c0[:, i], n)) * Jet.const(w[:, i], n) for i in range(3)]
    sq, msq = _sq(R)
    rho0, mrho0, sr, rel = _huber(sq, msq, float(s["prior_huber_a"]), np.ones(n, bool))
    fc = free_masks(s, 14, extrinsics_opt, 1)[1][pp]
    out = dict(r=np.stack([sr * x.a for x in R], 1), m_r=np.stack([sr * (x.ma + rel * np.abs(x.a)) for x in R], 1),
               J=np.stack([sr[:, None] * x.v[:, KI:KI + 6] for x in R], 1) * fc[:, None, :],
               m_J=np.stack([sr[:, None] * (x.mv[:, KI:KI + 6] + rel[:, None] * np.abs(x.v[:, KI:KI + 6])) for x in R], 1) * fc[:, None, :],
               cost=(rho0 / 2).sum(), m_cost=(mrho0 / 2).sum())
    return out


def record_model(aa, fixed):
    """numpy model (float64) of cam_prep_kernel's compact pose record and of how eval_kernel forms dR_k X from it:
    returns a function X[3] -> [3][3] (column k = dR_k X).  R and dR_k are Ceres' (exact here); Jr column k =
    vee(skew(R' dR_k)), and dR_k X = R (j_k x X).  fixed=True: Taylor-branch poses take e_k x X instead."""
    aa = np.asarray(aa, np.float64)
    taylor = bool(taylor_branch(aa))
    E = [Jet.var(np.array([aa[k]]), KI + k) for k in range(3)]
    # R e_j and dR/daa_k e_j from the jets of rotate() (the record's cam_prep uses the same duals)
    R = np.zeros((3, 3)); dR = np.zeros((3, 3, 3))
    for j in range(3):
        e = [Jet.const(float(i == j), 1) for i in range(3)]
        col = rotate(E, e, np.array([taylor]))
        for i in range(3):
            R[i, j] = float(col[i].a[0])
            for k in range(3):
                dR[k, i, j] = float(col[i].v[0, KI + k])
    Jr = np.zeros((3, 3))
    for k in range(3):
        M = R.T @ dR[k]
        Jr[:, k] = 0.5 * np.array([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]])

    def dRX(X):
        X = np.asarray(X, np.float64)
        if fixed and taylor:
            return np.stack([np.cross(np.eye(3)[k], X) for k in range(3)], 1)
        return np.stack([R @ np.cross(Jr[:, k], X) for k in range(3)], 1)
    return dRX


# ------------------------------------------------------------------------------------------------ edge scenes
# Each scene is built from camera-frame points: the landmark is R'(pc - t), so depth, angle and image position are
# chosen on purpose; obs_xy = the reference's pixel - the residual asked for.
ROT_ANGLES = (0.0, 1e-12, 1e-10, 1e-9, 1.2e-8, 1.5e-8, 1e-7, 1e-4, np.pi - 1e-9, np.pi, 4.0, 2 * np.pi - 1e-6, 7.0)
TAYLOR_ANGLES = tuple(t for t in ROT_ANGLES if t * t <= DBL_EPSILON)
PINHOLE = [800.0, 500.0, 400.0]
BROWN = [900.0, 510.0, 390.0, 0.05, -0.01, 0.002, 0.01, -0.02]
FISHEYE = [600.0, 500.0, 400.0, 0.02, -0.005, 0.001, 0.0003]
SPHERICAL = [4000.0, 2000.0]


def rodrigues(aa):
    """Exact rotation matrix of an angle-axis vector (long double)."""
    aa = np.asarray(aa, LD); th = np.sqrt((aa * aa).sum())
    if th == 0:
        return np.eye(3, dtype=LD)
    k = aa / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]], LD)
    return np.eye(3, dtype=LD) + np.sin(th) * Kx + (1 - np.cos(th)) * (Kx @ Kx)


class SceneBuilder:
    def __init__(self, seed=0):
        self.rng = np.random.default_rng(seed)
        self.poses, self.intr, self.models, self.views = [], [], [], {}
        self.obs = []          # (view, point rows [m][3], resid [m][2], weight [m], no_loss [m], fixed [m])

    def pose(self, aa, t=None, center=None):
        aa = np.asarray(aa, np.float64)
        R = rodrigues(aa)
        if center is not None:
            t = -(R @ np.asarray(center, LD))
        self.poses.append(np.concatenate([aa, np.asarray(t, LD).astype(np.float64)]))
        return len(self.poses) - 1

    def axis_pose(self, theta, t_scale=1.0):
        a = self.rng.normal(size=3); a /= np.linalg.norm(a)
        return self.pose(theta * a, self.rng.normal(0, t_scale, 3))

    def camera(self, model, params):
        k = np.zeros(KI); k[:len(params)] = params
        self.intr.append(k); self.models.append(model)
        return len(self.intr) - 1

    def add(self, pose, cam, pc, resid=None, weight=None, no_loss=None, fixed=None):
        pc = np.atleast_2d(np.asarray(pc, np.float64)); m = len(pc)
        v = self.views.setdefault((pose, cam), len(self.views))
        P = np.asarray(self.poses[pose], LD); R = rodrigues(self.poses[pose][:3])
        X = ((pc.astype(LD) - P[3:]) @ R).astype(np.float64)            # R'(pc - t), row by row
        resid = self.rng.normal(0, 0.5, (m, 2)) if resid is None else np.broadcast_to(np.asarray(resid, np.float64), (m, 2))
        f = lambda a, d: np.broadcast_to(np.asarray(d if a is None else a), (m,))   # noqa: E731
        self.obs.append((v, X, resid, f(weight, 1.0), f(no_loss, 0), f(fixed, 0)))

    def cone(self, m, half_angle=0.5, depth=(1.0, 20.0)):
        """m camera-frame points inside a cone about the optical axis."""
        z = self.rng.uniform(*depth, m)
        return np.stack([self.rng.uniform(-half_angle, half_angle, m) * z, self.rng.uniform(-half_angle, half_angle, m) * z, z], 1)

    def build(self, ext=False):
        vp = np.array([k[0] for k in sorted(self.views, key=self.views.get)], np.int32)
        vi = np.array([k[1] for k in sorted(self.views, key=self.views.get)], np.int32)
        ov = np.concatenate([np.full(len(o[1]), o[0], np.int32) for o in self.obs])
        X = np.concatenate([o[1] for o in self.obs])
        s = dict(poses=np.ascontiguousarray(self.poses, np.float64), intrinsics=np.ascontiguousarray(self.intr, np.float64),
                 intr_model=np.asarray(self.models, np.int32), points=np.ascontiguousarray(X), view_pose=vp, view_intr=vi,
                 obs_view=np.ascontiguousarray(ov), obs_point=np.arange(len(X), dtype=np.int32), obs_xy=np.zeros((len(X), 2)))
        pixel = evaluate(s, use_loss=0)["r"]
        s["obs_xy"] = np.ascontiguousarray((pixel - np.concatenate([o[2] for o in self.obs])).astype(np.float64))
        if ext:
            s["obs_weight"] = np.concatenate([o[3] for o in self.obs]).astype(np.float64)
            s["obs_no_loss"] = np.concatenate([o[4] for o in self.obs]).astype(np.uint8)
            s["point_fixed"] = np.concatenate([o[5] for o in self.obs]).astype(np.uint8)
        return s


def _huber_edge(rng, a, m):
    """m residual vectors with |r|^2 = a^2 (1 +- 1e-9), alternating sides."""
    d = rng.normal(size=(m, 2)); d /= np.linalg.norm(d, axis=1)[:, None]
    return d * (a * np.sqrt(1 + 1e-9 * np.where(np.arange(m) % 2, 1, -1)))[:, None]


def scene_rotations(seed=1):
    b = SceneBuilder(seed)
    cams = [b.camera(1, PINHOLE), b.camera(4, BROWN)]
    for th in ROT_ANGLES:
        p = b.axis_pose(th)
        for c in cams:
            b.add(p, c, b.cone(10))
            b.add(p, c, b.cone(2), resid=[[40.0, -30.0], [-5.0, 25.0]])          # Huber tail
    return b.build()


def scene_depth(seed=2):
    b = SceneBuilder(seed)
    c = b.camera(3, [700.0, 480.0, 360.0, 0.05, -0.01, 0.002])
    for th in (1e-10, 0.7):
        p = b.axis_pose(th)
        for z in (1e-3, 1e-2, 1.0, 1e2, 1e4):
            b.add(p, c, b.cone(4, 0.4, (z, z * 1.1)))
        b.add(p, c, [[0.3, -0.2, -1.0], [-40.0, 10.0, -100.0]])                    # behind the camera
    for th in (1e-9, 1e-3, 2.5):                                                   # landmarks 1e4 from the origin, seen from 1..10
        a = b.rng.normal(size=3); a /= np.linalg.norm(a)
        p = b.pose(th * a, center=1e4 * a[::-1] / np.linalg.norm(a))
        b.add(p, c, b.cone(6, 0.4, (1.0, 10.0)))
    return b.build()


def scene_fisheye(seed=3):
    b = SceneBuilder(seed)
    c = b.camera(5, FISHEYE)
    p0 = b.pose(np.zeros(3), np.zeros(3))                                        # identity: p = X exactly
    r0 = 1e-8
    b.add(p0, c, [[0.0, 0.0, 2.0], [0.0, 0.0, 7.0],
                  [r0 * (1 + 1e-6) * 2, 0.0, 2.0], [0.0, -r0 * (1 + 1e-6) * 3, 3.0],
                  [r0 * (1 - 1e-6) * 2, 0.0, 2.0], [0.0, r0 * (1 - 1e-6) * 5, 5.0],
                  [r0 * 0.6 * 4, r0 * 0.8 * 4 * (1 + 1e-6), 4.0]])
    for th in (1e-9, 0.3):
        p = b.axis_pose(th)
        ang = np.linspace(0.05, 1.4, 12); phi = b.rng.uniform(0, 2 * np.pi, 12); z = b.rng.uniform(1, 10, 12)
        r = np.tan(ang)
        b.add(p, c, np.stack([r * np.cos(phi) * z, r * np.sin(phi) * z, z], 1))
    return b.build()


def scene_radial(seed=4):
    b = SceneBuilder(seed)
    cams = [b.camera(2, [750.0, 500.0, 400.0, 0.08]), b.camera(3, [700.0, 480.0, 360.0, 0.05, -0.01, 0.002]), b.camera(4, BROWN)]
    for th in (1e-9, 0.4):
        p = b.axis_pose(th)
        for c in cams:
            phi = b.rng.uniform(0, 2 * np.pi, 8); rr = b.rng.uniform(0.95, 1.05, 8); z = b.rng.uniform(1, 10, 8)
            b.add(p, c, np.stack([rr * np.cos(phi) * z, rr * np.sin(phi) * z, z], 1))
    return b.build()


def scene_spherical(seed=5):
    b = SceneBuilder(seed)
    c = b.camera(7, SPHERICAL)
    for th in (1e-10, 0.2):
        p = b.axis_pose(th)
        poles = [[1e-6, 1.0, 2e-6], [-3e-6, -1.0, 1e-6], [1e-3, -2.0, -1e-3], [2e-4, 3.0, 5e-4]]
        seam = [[1e-4, 0.2, -1.0], [-1e-4, 0.2, -1.0], [1e-7, -0.3, -2.0], [-1e-7, -0.3, -2.0], [0.5, 0.1, -1.0], [-0.5, 0.1, -1.0]]
        b.add(p, c, poles + seam)
        b.add(p, c, b.cone(6, 1.5))
    return b.build()


def scene_loss(seed=6, huber=(16.0, 3.5)):
    b = SceneBuilder(seed)
    c = b.camera(1, PINHOLE)
    for th in (1e-9, 0.5):
        p = b.axis_pose(th)
        for a in huber:
            b.add(p, c, b.cone(8), resid=_huber_edge(b.rng, a, 8))
        b.add(p, c, b.cone(4), resid=[[1e4, -3e3], [-2e4, 5e3], [7e3, 7e3], [0.0, 1e5]])   # far into the tail
        b.add(p, c, b.cone(4), resid=[[0.0, 0.0], [1e-3, 0.0], [0.0, -2.0], [3.0, 1.0]])
    return b.build()


def scene_weights(seed=7):
    b = SceneBuilder(seed)
    cams = [b.camera(1, PINHOLE), b.camera(4, BROWN)]
    for th in (1e-10, 0.6):
        p = b.axis_pose(th)
        for c in cams:
            for w in (0.0, 1e-3, 7.0, 1e3):
                b.add(p, c, b.cone(3), weight=w)
                b.add(p, c, b.cone(2), resid=[[30.0, 5.0], [2.0, -1.0]], weight=w, no_loss=1)
                b.add(p, c, b.cone(2), resid=[[3.0, 1.0], [0.5, 0.5]], weight=w, fixed=1)
            b.add(p, c, [[0.2, 0.1, -3.0]], resid=[[50.0, 50.0]], weight=0.0)       # removed, behind the camera
    return b.build(ext=True)


def scene_mixed(seed=8, per=6):
    b = SceneBuilder(seed)
    cams = [b.camera(1, PINHOLE), b.camera(4, BROWN), b.camera(5, FISHEYE), b.camera(7, SPHERICAL)]
    for th in (0.0, 1e-10, 1e-9, 0.3, 2.0):
        p = b.axis_pose(th)
        for c in cams:
            b.add(p, c, b.cone(per, 1.2 if c == 3 else 0.5))
            b.add(p, c, b.cone(1), resid=[[35.0, -20.0]])
    return b.build()


def scene_grid(seed=9, n_obs=60001):
    """>= 60 000 observations (not a multiple of 128) over poses of every angle of ROT_ANGLES and four camera models."""
    b = SceneBuilder(seed)
    cams = [b.camera(1, PINHOLE), b.camera(4, BROWN), b.camera(5, FISHEYE), b.camera(7, SPHERICAL)]
    poses = [b.axis_pose(th) for th in ROT_ANGLES] + [b.axis_pose(b.rng.uniform(0, 3)) for _ in range(27)]
    k = 0; i = 0
    while k < n_obs:
        m = min(97, n_obs - k)
        b.add(poses[i % len(poses)], cams[i % len(cams)], b.cone(m, 0.5), resid=b.rng.standard_t(2, (m, 2)) * 3)
        k += m; i += 1
    return b.build()


def scene_priors(seed=10):
    b = SceneBuilder(seed)
    c = b.camera(1, PINHOLE)
    ps = [b.axis_pose(th, 3.0) for th in ROT_ANGLES]
    for p in ps:
        b.add(p, c, b.cone(2))
    s = b.build()
    rng = np.random.default_rng(seed)
    P = np.asarray(s["poses"], LD)
    C = np.stack([-(rodrigues(P[k, :3].astype(np.float64)).T @ P[k, 3:]) for k in range(len(P))]).astype(np.float64)
    n = len(ps)
    s["prior_pose"] = np.arange(n, dtype=np.int32)
    off = rng.normal(size=(n, 3)); off *= (np.where(np.arange(n) % 2, 2.0, 0.05) / np.linalg.norm(off, axis=1))[:, None]
    s["prior_center"] = np.ascontiguousarray(C + off)
    s["prior_weight"] = np.ascontiguousarray(rng.uniform(0.5, 4.0, (n, 3)))
    s["prior_huber_a"] = 0.4
    return s
