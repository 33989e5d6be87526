"""Extended-precision reference of one LM step of the BA solve, stage by stage (numpy, np.longdouble).

Input is a residual vector r[n_obs][2] and the unscaled Jacobian blocks J_intr[n_obs][2][8], J_pose[n_obs][2][6],
J_point[n_obs][2][3] (Huber-corrected, weighted), as omvg_ba_debug_eval and oracle_ba_eval return them.  The
conventions are Ceres' (trust_region_minimizer.cc, levenberg_marquardt_strategy.cc, schur_eliminator), as the oracle
follows them (oracle/ba_oracle.cpp, solve_impl):
    scale = 1 / (1 + sqrt(sum J^2))  per column;   Js = J scale;   D^2 = clamp(sum Js^2, min_lm_diagonal, max_lm_diagonal) / radius
    S = A_rr + D_r^2 - A_rp (A_pp + D_p^2)^-1 A_pr,   b = g_r - A_rp (A_pp + D_p^2)^-1 g_p,   g = Js' r
    delta_r = -z,   delta_p = -(A_pp + D_p^2)^-1 (g_p - A_pr z),   model change = -sum (Js delta) . (r + Js delta / 2)
Vectors over all columns are ordered points (3 n_points), poses (6 n_poses), intrinsic slots (8 n_intrinsics); S, b
and z cover the last two (the reduced system, nd = 6 n_poses + 8 n_intrinsics unknowns).  Constant coordinates (option
masks, fixed or removed landmarks) are not unknowns: their Jacobian columns are dropped, and in the reduced system they
are identity rows with a zero right-hand side.  Every sum runs in long double; the 3x3 landmark inverses are the
explicit adjugate."""
import numpy as np

LD = np.longdouble
assert np.finfo(LD).eps < 1e-18, "long double is not an extended type on this platform"

KI = 8
NPARAMS = {1: 3, 2: 4, 3: 6, 4: 8, 5: 7, 7: 0}
OPTS = dict(intrinsics_opt=14, extrinsics_opt=6, structure_opt=1, min_lm_diagonal=1e-6, max_lm_diagonal=1e32)


def free_masks(s, intrinsics_opt=14, extrinsics_opt=6, structure_opt=1, point_constant=None):
    """Free coordinates: points [n_points][3], poses [n_poses][6], intrinsic slots [n_intr][8] (sfm_data_BA_ceres.cpp
    option masks, as make_masks in ba.cu).  point_constant: landmarks held constant besides point_fixed (removed tracks)."""
    npt, nc, ni = len(s["points"]), len(s["poses"]), len(s["intrinsics"])
    fp = np.zeros((npt, 3), bool)
    if structure_opt:
        live = np.bincount(s["obs_point"], minlength=npt) > 0
        if s.get("point_fixed") is not None:
            live &= ~np.asarray(s["point_fixed"]).astype(bool)
        if point_constant is not None:
            live &= ~np.asarray(point_constant).astype(bool)
        fp[live] = True
    fc = np.zeros((nc, 6), bool)
    fc[:, {1: [], 4: [3, 4, 5], 2: [0, 1, 2]}.get(extrinsics_opt, list(range(6)))] = True
    fi = np.zeros((ni, KI), bool)
    if not intrinsics_opt & 1:
        for q in range(ni):
            for i in range(NPARAMS[int(s["intr_model"][q])]):
                fi[q, i] = bool(intrinsics_opt & (2 if i == 0 else 4 if i <= 2 else 8))
    return fp, fc, fi


def solve_refined(S, b, rounds=3):
    """The solution of S z = b: a float64 LAPACK solve, then `rounds` rounds of iterative refinement with the residual
    formed in long double."""
    S = np.asarray(S, LD); b = np.asarray(b, LD)
    S64 = S.astype(np.float64)
    z = np.linalg.solve(S64, b.astype(np.float64)).astype(LD)
    for _ in range(rounds):
        res = b - S @ z
        z = z + np.linalg.solve(S64, res.astype(np.float64)).astype(LD)
    return z


class StepReference:
    """One LM step of the scene `s` from (r, J) at trust-region radius `radius` (see the module docstring)."""

    def __init__(self, s, r, J_intr, J_pose, J_point, radius, point_constant=None, **opts):
        o = dict(OPTS); o.update({k: v for k, v in opts.items() if k in OPTS})
        self.s = s
        npt, nc, ni = len(s["points"]), len(s["poses"]), len(s["intrinsics"])
        self.npt, self.nc, self.ni = npt, nc, ni
        self.nd = nd = 6 * nc + KI * ni
        op = np.asarray(s["obs_point"]); ov = np.asarray(s["obs_view"])
        pose = np.asarray(s["view_pose"])[ov]; intr = np.asarray(s["view_intr"])[ov]
        self.op, self.pose, self.intr = op, pose, intr
        fp, fc, fi = free_masks(s, o["intrinsics_opt"], o["extrinsics_opt"], o["structure_opt"], point_constant)
        self.fp, self.fc, self.fi = fp, fc, fi
        self.free = np.concatenate([fp.ravel(), fc.ravel(), fi.ravel()])
        self.free_r = self.free[3 * npt:]
        # masked, unscaled J: constant columns are not part of the reduced program
        Jp = np.asarray(J_point, LD) * fp[op][:, None, :]
        Jc = np.asarray(J_pose, LD) * fc[pose][:, None, :]
        Ji = np.asarray(J_intr, LD) * fi[intr][:, None, :]
        self.r = r = np.asarray(r, LD)
        # Jacobi scaling from the unscaled column norms (trust_region_minimizer.cc:239-253)
        n2p = np.zeros((npt, 3), LD); n2c = np.zeros((nc, 6), LD); n2i = np.zeros((ni, KI), LD)
        np.add.at(n2p, op, (Jp ** 2).sum(1)); np.add.at(n2c, pose, (Jc ** 2).sum(1)); np.add.at(n2i, intr, (Ji ** 2).sum(1))
        sp, scc, si = (1 / (1 + np.sqrt(n)) for n in (n2p, n2c, n2i))
        self.scale = np.concatenate([sp.ravel(), scc.ravel(), si.ravel()])
        Jp = Jp * sp[op][:, None, :]; Jc = Jc * scc[pose][:, None, :]; Ji = Ji * si[intr][:, None, :]
        self.Jp = Jp
        # LM diagonal (levenberg_marquardt_strategy.cc:75-87)
        dp = np.zeros((npt, 3), LD); dc = np.zeros((nc, 6), LD); di = np.zeros((ni, KI), LD)
        np.add.at(dp, op, (Jp ** 2).sum(1)); np.add.at(dc, pose, (Jc ** 2).sum(1)); np.add.at(di, intr, (Ji ** 2).sum(1))
        diag = np.concatenate([dp.ravel(), dc.ravel(), di.ravel()])
        D2 = np.minimum(np.maximum(diag, LD(o["min_lm_diagonal"])), LD(o["max_lm_diagonal"])) / LD(radius)
        self.lm_diag = np.sqrt(D2)
        D2p, D2r = D2[:3 * npt].reshape(npt, 3), D2[3 * npt:]
        # per observation: F = [Jc | Ji] on the reduced columns idx
        F = np.concatenate([Jc, Ji], axis=2)                                           # [n][2][14]
        self.F = F
        self.idx = idx = np.concatenate([6 * pose[:, None] + np.arange(6), 6 * nc + KI * intr[:, None] + np.arange(KI)], axis=1)
        S = np.zeros((nd, nd), LD); b = np.zeros(nd, LD)
        Smag = np.zeros((nd, nd), LD); bmag = np.zeros(nd, LD)                          # sums of |terms| of S and b
        FtF = np.einsum("nra,nrb->nab", F, F)
        np.add.at(S, (idx[:, :, None], idx[:, None, :]), FtF)
        np.add.at(Smag, (idx[:, :, None], idx[:, None, :]), np.abs(FtF))
        gr = np.einsum("nra,nr->na", F, r)
        np.add.at(b, idx, gr); np.add.at(bmag, idx, np.abs(gr))
        # landmark blocks A_pp + D_p^2, their adjugate inverses, g_p
        App = np.zeros((npt, 3, 3), LD); gp = np.zeros((npt, 3), LD)
        np.add.at(App, op, np.einsum("nra,nrb->nab", Jp, Jp)); np.add.at(gp, op, np.einsum("nra,nr->na", Jp, r))
        App[:, [0, 1, 2], [0, 1, 2]] += D2p
        pf = fp.any(1)
        self.Ainv = np.zeros((npt, 3, 3), LD)
        self.Ainv[pf] = _inv3(App[pf])
        self.gp = gp
        self.W = W = np.einsum("nra,nrb->nab", Jp, F)                                  # Jp' F  [n][3][14]
        if pf.any():
            v = np.einsum("jab,jb->ja", self.Ainv, gp)
            e = np.einsum("nab,na->nb", W, v[op])
            np.add.at(b, idx, -e); np.add.at(bmag, idx, np.abs(e))
            V = np.einsum("nab,nbc->nac", self.Ainv[op], W)                            # Ainv_j W_u
            oi, ui = _pairs(op, pf)
            for c0 in range(0, len(oi), 20000):
                a, u = oi[c0:c0 + 20000], ui[c0:c0 + 20000]
                T = np.einsum("pab,pac->pbc", W[a], V[u])
                np.add.at(S, (idx[a][:, :, None], idx[u][:, None, :]), -T)
                np.add.at(Smag, (idx[a][:, :, None], idx[u][:, None, :]), np.abs(T))
        S[np.arange(nd), np.arange(nd)] += np.where(self.free_r, D2r, 0)
        Smag[np.arange(nd), np.arange(nd)] += np.where(self.free_r, D2r, 0)
        const = np.flatnonzero(~self.free_r)
        S[const, :] = 0; S[:, const] = 0; S[const, const] = 1; b[const] = 0
        Smag[const, :] = 0; Smag[:, const] = 0; Smag[const, const] = 1; bmag[const] = 0
        self.S, self.b, self.Smag, self.bmag = S, b, Smag, bmag

    def back_substitute(self, z):
        """delta_p = -(A_pp + D_p^2)^-1 (g_p - A_pr z) per landmark, for a reduced solution z (the step is -z there)."""
        z = np.asarray(z, LD)
        Az = np.zeros((self.npt, 3), LD)
        np.add.at(Az, self.op, np.einsum("nab,nb->na", self.W, z[self.idx]))
        return -np.einsum("jab,jb->ja", self.Ainv, self.gp - Az)

    def model_change(self, delta_point, delta_red):
        """-sum m . (r + m / 2), m = Js delta (trust_region_minimizer.cc:402-405)."""
        dp = np.asarray(delta_point, LD).reshape(-1, 3); dr = np.asarray(delta_red, LD)
        m = np.einsum("nra,na->nr", self.Jp, dp[self.op]) + np.einsum("nra,na->nr", self.F, dr[self.idx])
        return -(m * (self.r + m / 2)).sum()

    def step(self):
        """The exact step of this reference: (delta_point [n_points][3], delta_red [nd], z*)."""
        z = solve_refined(self.S, self.b)
        return self.back_substitute(z), -z, z

    def candidate(self, delta_point, delta_red):
        """x + scale . delta on the free coordinates: (poses, intrinsics, points) as float64 arrays."""
        s, npt, nc = self.s, self.npt, self.nc
        d = np.concatenate([np.asarray(delta_point, LD).ravel(), np.asarray(delta_red, LD)]) * self.scale * self.free
        pts = (np.asarray(s["points"], LD) + d[:3 * npt].reshape(npt, 3)).astype(np.float64)
        poses = (np.asarray(s["poses"], LD) + d[3 * npt:3 * npt + 6 * nc].reshape(nc, 6)).astype(np.float64)
        intr = (np.asarray(s["intrinsics"], LD) + d[3 * npt + 6 * nc:].reshape(-1, KI)).astype(np.float64)
        return np.ascontiguousarray(poses), np.ascontiguousarray(intr), np.ascontiguousarray(pts)


def _inv3(A):
    """Inverse of 3x3 blocks [m][3][3] by the adjugate."""
    a, b, c = A[:, 0, 0], A[:, 0, 1], A[:, 0, 2]
    d, e, f = A[:, 1, 0], A[:, 1, 1], A[:, 1, 2]
    g, h, i = A[:, 2, 0], A[:, 2, 1], A[:, 2, 2]
    adj = np.stack([np.stack([e * i - f * h, c * h - b * i, b * f - c * e], -1),
                    np.stack([f * g - d * i, a * i - c * g, c * d - a * f], -1),
                    np.stack([d * h - e * g, b * g - a * h, a * e - b * d], -1)], 1)
    det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g)
    return adj / det[:, None, None]


def _pairs(op, point_free):
    """All ordered observation pairs (o, u) of the same free landmark."""
    keep = np.flatnonzero(point_free[op])
    order = keep[np.argsort(op[keep], kind="stable")]
    ps = op[order]
    cnt = np.bincount(ps, minlength=len(point_free))
    start = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    rep = cnt[ps]
    oi = np.repeat(order, rep)
    k = np.arange(rep.sum()) - np.repeat(np.cumsum(rep) - rep, rep)
    ui = order[np.repeat(start[ps], rep) + k]
    return oi, ui


def unreduced_step(ref):
    """The same step from the unreduced system (Js'Js + D^2) delta = -Js' r over the free columns, solved densely
    (float64 solve, long double refinement): (delta_point [n_points][3], delta_red [nd])."""
    npt, nd = ref.npt, ref.nd
    n = 3 * npt + nd
    cols = np.concatenate([3 * ref.op[:, None] + np.arange(3), 3 * npt + ref.idx], axis=1)      # [n_obs][17]
    Jo = np.concatenate([ref.Jp, ref.F], axis=2)                                                  # [n_obs][2][17]
    A = np.zeros((n, n), LD); g = np.zeros(n, LD)
    np.add.at(A, (cols[:, :, None], cols[:, None, :]), np.einsum("nra,nrb->nab", Jo, Jo))
    np.add.at(g, cols, np.einsum("nra,nr->na", Jo, ref.r))
    A[np.arange(n), np.arange(n)] += ref.lm_diag ** 2
    f = np.flatnonzero(ref.free)
    d = np.zeros(n, LD)
    d[f] = -solve_refined(A[np.ix_(f, f)], g[f])
    return d[:3 * npt].reshape(npt, 3), d[3 * npt:]
