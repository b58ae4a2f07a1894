"""TEST INFRASTRUCTURE ONLY — numpy restatement of the reference's iterative path for K >= 2 grouped random effects with a Gaussian
likelihood (Woodbury identity on the random-effect scale, M = Sigma^-1 + Z^T Z, SSOR preconditioner). Probe vectors come from
`orc_gen_rand_normal`, the reference's GenRandVecNormalParallel. `dense_negll` is the exact likelihood from Psi = I + Z Sigma Z^T
(small n), for the comparison with the reference's Cholesky values."""
import numpy as np
import scipy.sparse as sp
from scipy.sparse.linalg import spsolve_triangular

from .laplace import _optimal_c, gen_rand_normal, logdet_tridiag

DEFAULTS = dict(cg_max_num_it=1000, cg_max_num_it_tridiag=1000, cg_delta_conv=1e-2, num_rand_vec_trace=50, seed_rand_vec_trace=1)


def level_index(group):
    """Per column, levels numbered by first appearance of the label string (what GPB_CreateREModel receives)."""
    group = np.asarray(group)
    if group.ndim == 1:
        group = group.reshape(-1, 1)
    cols = []
    for k in range(group.shape[1]):
        seen = {}
        cols.append(np.array([seen.setdefault(str(v), len(seen)) for v in group[:, k]], dtype=np.int64))
    return cols


class Structure:
    """Z (n x G, components in cum_num_rand_eff order), Z^T Z, level counts; fixed by the data."""

    def __init__(self, group):
        self.idx = level_index(group)
        self.K = len(self.idx)
        self.levels = [int(i.max()) + 1 for i in self.idx]
        self.cum = np.concatenate([[0], np.cumsum(self.levels)]).astype(np.int64)
        self.G = int(self.cum[-1])
        n = self.idx[0].shape[0]
        rows = np.concatenate([np.arange(n)] * self.K)
        cols = np.concatenate([self.idx[k] + self.cum[k] for k in range(self.K)])
        self.Z = sp.csr_matrix((np.ones(rows.shape[0]), (rows, cols)), shape=(n, self.G))
        self.ZtZ = (self.Z.T @ self.Z).tocsr()
        self.comp = np.repeat(np.arange(self.K), self.levels)

    def M(self, v):
        """Sigma^-1 + Z^T Z at variance ratios v (CalcCovFactor, re_model_template.h:9422-9429)."""
        return (self.ZtZ + sp.diags(1. / np.asarray(v, dtype=np.float64)[self.comp])).tocsr()


class SSOR:
    """P = L D^-1 L^T through L D^-1/2 (re_model_template.h:9433-9438)."""

    def __init__(self, M):
        self.M = M
        self.Dinv = 1. / M.diagonal()
        self.LD = (sp.tril(M, format="csr") @ sp.diags(np.sqrt(self.Dinv))).tocsr()
        self.LDt = self.LD.T.tocsr()

    def solve(self, R):
        """P^-1 R = (L D^-1/2)^-T (L D^-1/2)^-1 R."""
        W = spsolve_triangular(self.LD, R, lower=True)
        return spsolve_triangular(self.LDt, W, lower=False)


def cg_vec(M, pc, rhs, u0, p, delta_conv):
    """CGRandomEffectsVec (CG_utils.cpp:1147-1281); u0 = None starts from zero. Returns (u, iterations)."""
    p = min(p, rhs.shape[0])
    if np.sum(np.abs(rhs)) < 1e-100:
        return np.zeros_like(rhs), 0
    u = np.zeros_like(rhs) if u0 is None else u0.copy()
    r = rhs - M @ u if u0 is not None and np.any(u0 != 0) else rhs.copy()
    z = pc.solve(r)
    h = z.copy()
    for j in range(p):
        v = M @ h
        a = (r @ z) / (h @ v)
        u += a * h
        r_old, z_old = r, z
        r = r - a * v
        rn = np.linalg.norm(r)
        if not np.isfinite(rn):
            raise FloatingPointError("NaN or Inf in the conjugate gradient method")
        if rn < delta_conv:
            return u, j + 1
        z = pc.solve(r)
        b = (r @ z) / (r_old @ z_old)
        h = z + b * h
    return u, p


def cg_tridiag(M, pc, rhs, p, delta_conv):
    """CGTridiagRandomEffects (CG_utils.cpp:1283-1473): U = M^-1 rhs (t columns), Lanczos tridiagonals, iterations."""
    G, t = rhs.shape
    p = min(p, G)
    U = np.zeros_like(rhs)
    R = rhs.copy()
    Z = pc.solve(R)
    H = Z.copy()
    a, b = np.ones(t), np.zeros(t)
    Td, Ts = [], []
    for j in range(p):
        V = M @ H
        a_old = a
        a = np.sum(R * Z, axis=0) / np.sum(H * V, axis=0)
        U += H * a
        R_old, Z_old = R, Z
        R = R - V * a
        mean_norm = np.mean(np.linalg.norm(R, axis=0))
        if not np.isfinite(mean_norm):
            raise FloatingPointError("NaN or Inf in the conjugate gradient method")
        early = mean_norm < delta_conv
        Z = pc.solve(R)
        b_old = b
        b = np.sum(R * Z, axis=0) / np.sum(R_old * Z_old, axis=0)
        H = Z + H * b
        Td.append(1. / a + b_old / a_old)
        if j > 0:
            Ts.append(np.sqrt(b_old) / a_old)
        if early:
            return U, np.array(Td), np.array(Ts).reshape(-1, t), j + 1
    return U, np.array(Td), np.array(Ts).reshape(-1, t), p


def probes(st, t=50, seed=1, run_id=0):
    """rand_vec_probe_ (re_model_template.h:3039-3047): G x t, N(0, I)."""
    return gen_rand_normal(seed, run_id, st.G, t)


def evaluate(st, y, v, sigma2=None, r=None, x_prev=None, with_grad=False, **kw):
    """Negative log-likelihood pieces at variance ratios v (and error variance sigma2, default: profiled y^T Psi^-1 y / n).
    Returns a dict: quad, logdet, ldet_slq, negll, its, its_tridiag, x, and with_grad the gradient w.r.t. log v_k
    (CalcGradPars_Only_Grouped_REs_Woodbury_GaussLikelihood_Cluster_i, iterative / SSOR branch, re_model_template.h:2530-2619)."""
    cfg = dict(DEFAULTS, **kw)
    y = np.asarray(y, dtype=np.float64)
    v = np.asarray(v, dtype=np.float64)
    n = y.shape[0]
    M = st.M(v)
    pc = SSOR(M)
    Zty = st.Z.T @ y
    x, its = cg_vec(M, pc, Zty, x_prev, cfg["cg_max_num_it"], cfg["cg_delta_conv"])      # CalcYAux, iterative branch
    yaux = y - st.Z @ x
    quad = float(y @ yaux)
    if r is None:
        r = probes(st, cfg["num_rand_vec_trace"], cfg["seed_rand_vec_trace"])
    t = r.shape[1]
    u = pc.LD @ r                                                                           # u = L D^-1/2 r ~ N(0, P)
    U, Td, Ts, its_tri = cg_tridiag(M, pc, u, cfg["cg_max_num_it_tridiag"], cfg["cg_delta_conv"])
    ldet = logdet_tridiag(Td, Ts, st.G)
    logdet = ldet + 2. * np.sum(np.log(pc.LD.diagonal())) + float(np.sum(np.asarray(st.levels) * np.log(v)))
    s2 = quad / n if sigma2 is None else float(sigma2)
    out = dict(quad=quad, logdet=logdet, ldet_slq=ldet, its=its, its_tridiag=its_tri, x=x, yaux=yaux, u=u, U=U,
               negll=quad / 2. / s2 + logdet / 2. + n / 2. * (np.log(s2) + np.log(2 * np.pi)), sigma2=s2)
    if with_grad:
        PI = pc.solve(u)
        W = pc.Dinv[:, None] * (sp.triu(M, format="csr") @ PI)
        d = st.Z.T @ yaux
        grad = np.zeros(st.K)
        for k in range(st.K):
            sl = slice(st.cum[k], st.cum[k + 1])
            iv = 1. / v[k]
            q = v[k] * float(d[sl] @ d[sl])
            zA = -iv * np.sum(U[sl] * PI[sl], axis=0)
            zP = -2. * iv * np.sum(PI[sl] * W[sl], axis=0) + iv * np.sum(W[sl] * W[sl], axis=0)
            tr, trP = zA.mean(), zP.mean()
            trD = -iv * np.sum(pc.Dinv[sl])
            tr += _optimal_c(zA, zP, tr, trP) * (trD - trP)
            tr += st.levels[k]
            grad[k] = -q / s2 / 2. + tr / 2.
        out["grad"] = grad
    return out


def dense_negll(group, y, cov_pars):
    """Exact negative log-likelihood from Psi = sigma^2 (I + Z diag(v) Z^T) (small n): log|Psi / sigma^2|, y^T (Psi / sigma^2)^-1 y."""
    st = Structure(group)
    y = np.asarray(y, dtype=np.float64)
    n = y.shape[0]
    s2 = float(cov_pars[0])
    v = np.asarray(cov_pars[1:], dtype=np.float64) / s2
    Z = st.Z.toarray()
    Psi = np.eye(n) + (Z * v[st.comp]) @ Z.T
    L = np.linalg.cholesky(Psi)
    logdet = 2. * np.sum(np.log(np.diag(L)))
    w = np.linalg.solve(L, y)
    quad = float(w @ w)
    return dict(quad=quad, logdet=logdet, negll=quad / 2. / s2 + logdet / 2. + n / 2. * (np.log(s2) + np.log(2 * np.pi)))
