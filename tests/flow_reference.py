"""Plain numpy reference of the first step of the per-frame flow / pose LM (vdo_pose_opt_flow2, oracle/flow_lm.c), in long double.

From the float inputs of one problem it forms the world points as the kernels do (Twl = Tcw_last^-1 with its translation rounded to
float), the state from T_init through the same quaternion normalisation, and from these the Jacobians J (2x6 per point), the Huber
weights, H_pp, b_p and per point h = w + w_prior and b_l.  For the first trial (lambda = 1e-5 * max(max h, max |diag H_pp|)):

  quirk 0  the full damped (6 + 2n)^2 system [[H_pp + lam I, H_pl], [H_lp, (h + lam) I]] [x; df] = [b_p; b_l] with lam on every
           diagonal entry, as g2o adds it; `solve_full` solves it as one sparse system, without a Schur elimination, so the kernels'
           elimination is checked independently; `backward_error` recovers df from x by back-substitution.
  quirk 1  S and g from the D^-1 = [[1/p, -h/(p lam)], [0, 1/lam]] (p = h + lam) of the 2-D flow vertex inside BlockSolver_6_3's
           3x3 blocks (SURVEY.md H1); the solve reads S's lower triangle.  `scale` includes the c_u/lam spill of the back-substitution.

Each operator comes with its magnitude: the same sum over absolute values, which is what a rounding error is measured against.
"""
import numpy as np

LD = np.longdouble
W_REP = 0.1


def _rot_to_quat(R):
    """Eigen::Quaternion(Matrix3) on a row-major 3x3; q = (x, y, z, w)."""
    t = R[0, 0] + R[1, 1] + R[2, 2]
    q = np.zeros(4, LD)
    if t > 0:
        t = np.sqrt(t + LD(1)); q[3] = t / 2; t = LD(0.5) / t
        q[0] = (R[2, 1] - R[1, 2]) * t; q[1] = (R[0, 2] - R[2, 0]) * t; q[2] = (R[1, 0] - R[0, 1]) * t
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(R[i, i] - R[j, j] - R[k, k] + LD(1))
        q[i] = t / 2; t = LD(0.5) / t
        q[3] = (R[k, j] - R[j, k]) * t; q[j] = (R[j, i] + R[i, j]) * t; q[k] = (R[k, i] + R[i, k]) * t
    return q


def _quat_to_rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], LD)


class FlowStep:
    """The first linearisation and the first trial's linear system of one problem (a synth.make_flow_problem dict)."""

    def __init__(self, p, mode, quirk):
        self.quirk = quirk
        f32 = lambda a: np.asarray(a, np.float32)
        fx, fy, cx, cy = f32(p["K"]).astype(LD)
        Tl, Ti = f32(p["Tcw_last"]), f32(p["T_init"])
        pts, depth, flow = f32(p["pts"]).astype(LD), f32(p["depth"]).astype(LD), f32(p["flow"]).astype(LD)
        self.n = n = len(depth)
        w_prior = LD(0.5 if mode else 0.3)
        # Twl: R^T exactly, t = -R^T t summed in double and rounded to float (the cv::Mat expression of the reference)
        Rwl = Tl[:3, :3].T.astype(LD)
        twl = np.array([np.float32(-sum(np.float64(Tl[c, r]) * np.float64(Tl[c, 3]) for c in range(3))) for r in range(3)], LD)
        Xc = np.stack([(pts[:, 0] - cx) * depth / fx, (pts[:, 1] - cy) * depth / fy, depth], -1)
        Xw = Xc @ Rwl.T + twl
        q = _rot_to_quat(Ti[:3, :3].astype(LD))
        if q[3] < 0:
            q = -q
        q = q / np.sqrt((q * q).sum())
        R, t = _quat_to_rot(q), Ti[:3, 3].astype(LD)
        X = Xw @ R.T + t
        x, y, z = X[:, 0], X[:, 1], X[:, 2]
        proj = np.stack([x / z * fx + cx, y / z * fy + cy], -1)
        e = pts + flow - proj                                              # f = the measured flow at the first linearisation
        delta = np.float64(np.float32(np.sqrt(np.float64(np.float32(0.04)))))
        dsqr = LD(np.float64(np.float32(delta * delta)))
        e2 = W_REP * (e * e).sum(1)
        hub = np.where(e2 <= dsqr, LD(1), LD(delta) / np.sqrt(np.maximum(e2, dsqr)))
        w = W_REP * hub
        z2 = z * z
        J = np.zeros((n, 2, 6), LD)
        J[:, 0] = np.stack([x * y / z2 * fx, -(1 + x * x / z2) * fx, y / z * fx, -1 / z * fx, 0 * z, x / z2 * fx], -1)
        J[:, 1] = np.stack([(1 + y * y / z2) * fy, -x * y / z2 * fy, -x / z * fy, 0 * z, -1 / z * fy, y / z2 * fy], -1)
        aJ = np.abs(J)
        self.J, self.w, self.h, self.e = J, w, w + w_prior, e
        self.bl = -(w[:, None] * e)                                       # - (w e + w_prior (f - f_hat)), f = f_hat
        self.bl_mag = w[:, None] * (np.abs(pts) + np.abs(flow) + np.abs(proj))
        self.Hpp = np.einsum("i,iar,iac->rc", w, J, J)
        self.Hpp_mag = np.einsum("i,iar,iac->rc", w, aJ, aJ)
        self.bp = -np.einsum("i,iar,ia->r", w, J, e)
        self.bp_mag = np.einsum("i,iar,ia->r", w, aJ, self.bl_mag / w[:, None])
        self.lam = LD(1e-5) * max(self.h.max(), np.abs(np.diag(self.Hpp)).max())
        self._schur()

    def _schur(self):
        lam, h, w = self.lam, self.h, self.w
        B = w[:, None, None] * self.J                                     # H_lp per point: rows u, v of the flow vertex
        p = h + lam
        if not self.quirk:
            a, b, c = 1 / p, 0 * p, 1 / p
        else:
            a, b, c = 1 / p, -h / (p * lam), 1 / lam + 0 * p
        aB = np.abs(B)
        # H_pl D^-1 H_lp with D^-1 = [[a, b], [0, c]]
        BDB = (np.einsum("i,ir,ic->rc", a, B[:, 0], B[:, 0]) + np.einsum("i,ir,ic->rc", b, B[:, 0], B[:, 1])
               + np.einsum("i,ir,ic->rc", c, B[:, 1], B[:, 1]))
        BDB_mag = (np.einsum("i,ir,ic->rc", a, aB[:, 0], aB[:, 0]) + np.einsum("i,ir,ic->rc", np.abs(b), aB[:, 0], aB[:, 1])
                   + np.einsum("i,ir,ic->rc", c, aB[:, 1], aB[:, 1]))
        d0, d1 = a * self.bl[:, 0] + b * self.bl[:, 1], c * self.bl[:, 1]
        d0m, d1m = a * self.bl_mag[:, 0] + np.abs(b) * self.bl_mag[:, 1], c * self.bl_mag[:, 1]
        I = np.eye(6, dtype=LD)
        self.S = self.Hpp + lam * I - BDB
        self.S_mag = self.Hpp_mag + lam * I + BDB_mag
        self.g = self.bp - (B[:, 0] * d0[:, None] + B[:, 1] * d1[:, None]).sum(0)
        self.g_mag = self.bp_mag + (aB[:, 0] * d0m[:, None] + aB[:, 1] * d1m[:, None]).sum(0)
        self.B, self.Dinv = B, (a, b, c)

    def back_substitute(self, x):
        """Flow increments of the first trial for the pose increment x (the kernels' back-substitution, with the spill in quirk 1)."""
        x = np.asarray(x, LD)
        cu = self.bl[:, 0] - self.B[:, 0] @ x
        cv = self.bl[:, 1] - self.B[:, 1] @ x
        p = self.h + self.lam
        if not self.quirk:
            return np.stack([cu / p, cv / p], -1)
        du = cu / p - self.h * cv / (p * self.lam)
        du[1:] += cu[1:] / self.lam
        return np.stack([du, cv / self.lam], -1)

    def backward_error(self, x):
        """quirk 0: normwise backward error of [x; df(x)] on the full damped system; quirk 1: of x on the symmetric matrix given by
        S's lower triangle (what the solve reads)."""
        x = np.asarray(x, LD)
        ax = np.abs(x)
        if self.quirk:
            Ssym = np.tril(self.S) + np.tril(self.S, -1).T
            r = Ssym @ x - self.g
            mag = np.abs(Ssym) @ ax + np.abs(self.g)
            return float(np.abs(r).max() / mag.max())
        df = self.back_substitute(x)
        lam, I = self.lam, np.eye(6, dtype=LD)
        A = self.Hpp + lam * I
        r_p = A @ x + np.einsum("iar,ia->r", self.B, df) - self.bp
        m_p = np.abs(A) @ ax + np.einsum("iar,ia->r", np.abs(self.B), np.abs(df)) + np.abs(self.bp)
        r_l = np.einsum("iar,r->ia", self.B, x) + (self.h + lam)[:, None] * df - self.bl
        m_l = np.einsum("iar,r->ia", np.abs(self.B), ax) + (self.h + lam)[:, None] * np.abs(df) + np.abs(self.bl)
        return float(max(np.abs(r_p).max(), np.abs(r_l).max()) / max(m_p.max(), m_l.max()))

    def full_system(self):
        """The damped (6 + 2n)^2 system of quirk 0 (scipy.sparse CSC, float64) and its right-hand side: pose first, then u, v per point."""
        import scipy.sparse as sp
        n, lam = self.n, self.lam
        A_pp = (self.Hpp + lam * np.eye(6, dtype=LD)).astype(np.float64)
        B = self.B.astype(np.float64).reshape(2 * n, 6)                   # H_lp, row 2i + a
        D = sp.diags(np.repeat((self.h + lam).astype(np.float64), 2))
        A = sp.bmat([[sp.csc_matrix(A_pp), sp.csc_matrix(B.T)], [sp.csc_matrix(B), D]], format="csc")
        rhs = np.concatenate([self.bp.astype(np.float64), self.bl.astype(np.float64).reshape(-1)])
        return A, rhs

    def solve_full(self):
        """x of the first trial from the full system (quirk 0), one sparse LU solve, no Schur elimination."""
        import scipy.sparse.linalg as spl
        A, rhs = self.full_system()
        return spl.spsolve(A, rhs)[:6]

    def scale(self, x):
        """The first trial's predicted decrease for pose increment x (the sum the kernels form, flow part with the spill) and its
        magnitude."""
        x = np.asarray(x, LD)
        df = self.back_substitute(x)
        a, b, c = self.Dinv
        lam = self.lam
        s = (df * (lam * df + self.bl)).sum() + (x * (lam * x + self.bp)).sum()
        cmag = self.bl_mag + np.abs(self.B) @ np.abs(x)                  # magnitude of c_u, c_v
        dfm = cmag * (np.abs(a) + np.abs(b) + np.abs(c) + (1 / lam if self.quirk else 0))[:, None]
        mag = (dfm * (2 * lam * dfm + self.bl_mag)).sum() + (np.abs(x) * (2 * lam * np.abs(x) + self.bp_mag)).sum()
        return float(s), float(mag)
