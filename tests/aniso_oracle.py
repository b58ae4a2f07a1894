"""Restatement of the reference's anisotropic Vecchia GP (matern_ard, gaussian_ard, matern_space_time) on top of the oracle's C
factor (oracle/vecchia.py), for the tests: ordering, scaled coordinates (ScaleCoordinates, cov_fcts.h:280-313), neighbour sets
searched on them, the likelihood at range 1, and the gradient written from the per-coordinate element formulas of the kernels (not
from the coordinate-share identity the device uses), plus the seeded data and the case grid shared by the golden generator and the
tests."""
import numpy as np

from oracle import vecchia as ov

MULT = {0.5: 1., 1.5: np.sqrt(3.), 2.5: np.sqrt(5.)}
ALIASES = {"exponential_ard": ("matern_ard", 0.5), "Matern_ard": ("matern_ard", 0.5),
           "exponential_space_time": ("matern_space_time", 0.5), "Matern_space_time": ("matern_space_time", 0.5)}


def parse(cov_function, shape):
    return ALIASES.get(cov_function, (cov_function, float(shape)))


def groups(cov_function, d):
    """coordinate -> group (ARD: identity; space-time: time 0, space 1)"""
    return np.array([0] + [1] * (d - 1) if cov_function == "matern_space_time" else list(range(d)), dtype=np.int32)


def cid(cov_function, shape):
    return 3 if cov_function == "gaussian_ard" else ov.cov_id("matern", shape)


def transform(cov_pars, cov_function, shape):
    """(sigma2, sigma1^2, rho_1..rho_C) -> sigma2, var ratio, lambda_1..lambda_C (cov_fcts.h:523-545)"""
    cp = np.asarray(cov_pars, dtype=np.float64)
    rho = cp[2:]
    lam = 1. / (rho * rho) if cov_function == "gaussian_ard" else MULT[shape] / rho
    return cp[0], cp[1] / cp[0], lam


def scale_factors(lam, cov_function, d):
    g = groups(cov_function, d)
    s = lam[g]
    return np.sqrt(s) if cov_function == "gaussian_ard" else s


def order(coords, ordering, seed):
    n = coords.shape[0]
    perm = ov.random_order(n, seed) if ordering in ("random", "time_random_space") else np.arange(n, dtype=np.int32)
    if ordering in ("time", "time_random_space"):
        perm = perm[ov.sort_indices(coords[perm, 0])]
    return perm


def kernel_and_grads(dx, cov_function, shape, lam):
    """Covariance at var 1 and its derivatives w.r.t. log(lambda_c) for coordinate differences dx (..., d), from the element
    formulas of the kernels in the original coordinates: ARD matern r = |lambda o dx|, gaussian_ard exp(-sum lambda_j dx_j^2)."""
    d = dx.shape[-1]
    g = groups(cov_function, d)
    C = int(g.max()) + 1
    lj = lam[g]
    if cov_function == "gaussian_ard":
        q = (lj * dx * dx).sum(-1)
        k = np.exp(-q)
        dk = np.stack([-(lj * dx * dx)[..., g == c].sum(-1) * k for c in range(C)], -1)
        return k, dk
    t = (lj * dx) ** 2                          # lambda_j^2 dx_j^2
    r = np.sqrt(t.sum(-1))
    e = np.exp(-r)
    tc = np.stack([t[..., g == c].sum(-1) for c in range(C)], -1)
    if shape == 0.5:
        k = e
        with np.errstate(invalid="ignore", divide="ignore"):
            dk = np.where(r[..., None] > 0, -e[..., None] * tc / r[..., None], 0.)
    elif shape == 1.5:
        k = (1. + r) * e
        dk = -e[..., None] * tc
    else:
        k = (1. + r + r * r / 3.) * e
        dk = -((1. + r) / 3. * e)[..., None] * tc
    return k, dk


class AnisoOracle:
    """Neighbour sets searched in the space scaled by the parameters of every likelihood evaluation, as the reference does outside a
    fit; `grad_profiled` uses the sets of the last search."""

    def __init__(self, coords, num_neighbors, cov_function, shape, ordering, seed):
        self.cov_function, self.shape = parse(cov_function, shape)
        coords = np.asarray(coords, dtype=np.float64)
        self.n, self.d = coords.shape
        self.m = min(int(num_neighbors), self.n - 1)
        self.perm = order(coords, ordering, seed)
        self.coords = np.ascontiguousarray(coords[self.perm])
        self.cid = cid(self.cov_function, self.shape)
        self.nn = None
        self.searches = 0

    def scaled(self, cov_pars):
        _, _, lam = transform(cov_pars, self.cov_function, self.shape)
        return self.coords * scale_factors(lam, self.cov_function, self.d)

    def search(self, cov_pars):
        self.nn = ov.knn(self.scaled(cov_pars), self.m)
        self.searches += 1

    def neg_log_likelihood(self, cov_pars, y):
        self.search(cov_pars)
        s2, var, _ = transform(cov_pars, self.cov_function, self.shape)
        A, Dinv, _, _, _ = ov.factor(self.scaled(cov_pars), self.nn, self.cid, np.array([var, 1.]))
        return ov.nll_from_factor(self.nn, A, Dinv, np.asarray(y, dtype=np.float64)[self.perm], s2)[0]

    def grad_profiled(self, cov_pars, y):
        """(negll, gradient w.r.t. log(var ratio), log(lambda_1..C)) with the error variance profiled out, at the current sets"""
        _, var, lam = transform(cov_pars, self.cov_function, self.shape)
        yo = np.asarray(y, dtype=np.float64)[self.perm]
        C = lam.shape[0]
        n = self.n
        quad = logdet = 0.
        uk = np.zeros(1 + C); udu = np.zeros(1 + C); tr = np.zeros(1 + C)
        for i in range(n):
            nb = self.nn[i][self.nn[i] >= 0][: min(i, self.m)]
            pts = np.vstack([self.coords[nb], self.coords[i:i + 1]])
            dx = pts[:, None, :] - pts[None, :, :]
            k, dk = kernel_and_grads(dx, self.cov_function, self.shape, lam)
            q = len(nb)
            Sig = var * k + np.eye(q + 1)          # nugget 1 on the transformed scale
            dS = [var * k] + [var * dk[..., c] for c in range(C)]  # log(var): d Sigma~ = Sigma~ without the nugget
            S = Sig[:q, :q]
            s = Sig[:q, q]
            A = np.linalg.solve(S, s) if q else np.zeros(0)
            D = Sig[q, q] - A @ s
            b = np.concatenate([-A, [1.]])
            By = yo[i] - A @ yo[nb]
            u = By / D
            w = np.linalg.solve(S, yo[nb]) if q else np.zeros(0)
            wt = np.concatenate([w, [0.]])
            quad += By * By / D
            logdet += np.log(D)
            for kk, G in enumerate(dS):
                dD = b @ G @ b
                dBy = -(b @ G @ wt)
                uk[kk] += dBy * u
                udu[kk] += u * u * dD
                tr[kk] += dD / D
        s2 = quad / n
        negll = quad / 2. / s2 + logdet / 2. + n / 2. * (np.log(s2) + np.log(2 * np.pi))
        return negll, (uk - 0.5 * udu) / s2 + 0.5 * tr


def init_cov_pars(coords_ordered, y, cov_function, shape):
    """FindInitCovPar for n <= 1000 (no sub-sample): (sigma2, sigma1^2, rho_1..C) on the original scale (cov_fcts.h:1440-1670)"""
    n, d = coords_ordered.shape
    var = np.var(y, ddof=1)
    mult = 2. * 3. if shape <= 1. else (2. * 4.7 if shape <= 2. else 2. * 5.9)
    iu = np.triu_indices(n, 1)

    def med(v):
        mv = np.median(v)
        return mv if mv >= 1e-10 else v.mean()
    if cov_function == "matern_space_time":
        sp = coords_ordered[:, 1:]
        dsp = np.sqrt(((sp[:, None, :] - sp[None, :, :]) ** 2).sum(-1))[iu]
        dt = np.abs(coords_ordered[:, None, 0] - coords_ordered[None, :, 0])[iu]
        lam = np.array([mult / med(dt), mult / med(dsp)])
    else:
        lam = np.zeros(d)
        for k in range(d):
            nu = len(np.unique(coords_ordered[:, k]))
            if nu == 1:
                raise ValueError("constant coordinate %d" % (k + 1))
            mk = (nu * nu - 1) / 3. / nu if nu <= 10 else med(np.abs(coords_ordered[:, None, k] - coords_ordered[None, :, k])[iu])
            lam[k] = 3. / (mk / 2.) ** 2 if cov_function == "gaussian_ard" else mult / mk
    rho = 1. / np.sqrt(lam) if cov_function == "gaussian_ard" else MULT[shape] / lam
    s2 = var / 2.
    return np.concatenate([[s2, s2], rho])


# ---- seeded data and the case grid (tests/golden/make_aniso_golden.py, tests/test_aniso_*.py)

def simulate(n, d, ranges, seed, cov_function="matern_ard", shape=1.5, kind="uniform", few_unique_col=None):
    """Anisotropic GP (variance 1, ranges per coordinate group) plus noise of variance 0.1 at seeded locations"""
    rng = np.random.default_rng(seed)
    if kind == "ties":   # 20 time points x n/20 sites
        sites = rng.uniform(0., 1., (n // 20, d - 1))
        t = np.repeat(np.arange(20.) / 20., n // 20)
        X = np.column_stack([t, np.tile(sites, (20, 1))])
    else:
        X = rng.uniform(0., 1., (n, d))
    if few_unique_col is not None:
        X[:, few_unique_col] = rng.integers(0, 6, n).astype(np.float64)
    cf, sh = parse(cov_function, shape)
    pars = np.concatenate([[0.1, 1.], ranges])
    _, _, lam = transform(pars, cf, sh)
    dx = X[:, None, :] - X[None, :, :]
    k, _ = kernel_and_grads(dx, cf, sh, lam)
    L = np.linalg.cholesky(k + 1e-8 * np.eye(n))
    y = L @ rng.standard_normal(n) + np.sqrt(0.1) * rng.standard_normal(n)
    return X, y


CASES = [
    dict(name="ard_exp_d1_m10", cov="matern_ard", shape=0.5, d=1, n=1500, m=10, ordering="random", ranges=[0.2], seed=1),
    dict(name="ard_m15_d2_m20", cov="matern_ard", shape=1.5, d=2, n=2000, m=20, ordering="random", ranges=[0.3, 0.08], seed=2),
    dict(name="ard_m25_d3_m30", cov="matern_ard", shape=2.5, d=3, n=2000, m=30, ordering="random", ranges=[0.2, 0.1, 0.4], seed=3),
    dict(name="ard_m15_d5_m45", cov="matern_ard", shape=1.5, d=5, n=1500, m=45, ordering="random", ranges=[0.5, 0.3, 0.8, 0.4, 1.0],
         seed=4),
    dict(name="ard_exp_d2_m60", cov="exponential_ard", shape=0.5, d=2, n=1500, m=60, ordering="random", ranges=[0.4, 0.1], seed=5),
    dict(name="gard_d2_m10", cov="gaussian_ard", shape=0., d=2, n=1500, m=10, ordering="random", ranges=[0.2, 0.1], seed=6,
         init=[0.1, 1.0, 0.15, 0.15]),
    dict(name="st_m15_d3_time_m20", cov="matern_space_time", shape=1.5, d=3, n=2000, m=20, ordering="time", ranges=[0.3, 0.1],
         seed=7),
    dict(name="st_exp_d2_trs_m30", cov="exponential_space_time", shape=0.5, d=2, n=2000, m=30, ordering="time_random_space",
         ranges=[0.2, 0.1], seed=8),
    dict(name="st_ties_m15_d3_m10", cov="matern_space_time", shape=1.5, d=3, n=2000, m=10, ordering="time", ranges=[0.3, 0.2],
         seed=9, kind="ties"),
    dict(name="ard_fewunique_init", cov="matern_ard", shape=1.5, d=2, n=1000, m=20, ordering="none", ranges=[2., 0.2], seed=10,
         few_unique_col=0, maxit=0),
]


def case_data(c):
    ranges = c["ranges"]
    X, y = simulate(c["n"], c["d"], ranges, c["seed"], c["cov"], c["shape"], c.get("kind", "uniform"), c.get("few_unique_col"))
    rng = np.random.default_rng(c["seed"] + 1000)
    Xp = rng.uniform(0., 1., (100, c["d"]))
    return X, y, Xp


def thetas(c):
    cf, _ = parse(c["cov"], c["shape"])
    C = 2 if cf == "matern_space_time" else c["d"]
    r = np.asarray(c["ranges"], dtype=np.float64)
    t1 = np.concatenate([[0.1, 1.0], r])
    t2 = np.concatenate([[0.15, 0.8], r * np.where(np.arange(C) % 2 == 0, 5.0, 0.25)])
    return t1, t2


def make_model(GPModel, c, X, lib=None):
    kw = {} if lib is None else dict(_lib=lib)
    return GPModel(gp_coords=X, cov_function=c["cov"], cov_fct_shape=c["shape"], gp_approx="vecchia", num_neighbors=c["m"],
                   vecchia_ordering=c["ordering"], seed=c["seed"], **kw)


def run_case(GPModel, c, lib=None):
    """The call sequence whose results the goldens record: NLL at theta1 then theta2 on one model (frozen sets), theta2 on a fresh
    model, a fit, and the prediction at the fitted parameters"""
    X, y, Xp = case_data(c)
    t1, t2 = thetas(c)
    m1 = make_model(GPModel, c, X, lib)
    out = dict(name=c["name"], nll_t1=m1.neg_log_likelihood(t1, y), nll_t2_same=m1.neg_log_likelihood(t2, y))
    m2 = make_model(GPModel, c, X, lib)
    out["nll_t2_fresh"] = m2.neg_log_likelihood(t2, y)
    m3 = make_model(GPModel, c, X, lib)
    params = dict(maxit=c.get("maxit", 1000))
    if c.get("init") is not None:
        params["init_cov_pars"] = np.array(c["init"])
    m3.fit(y, params=params)
    cp = np.asarray(m3.get_cov_pars()).reshape(-1)
    out.update(cov_pars=cp.tolist(), num_it=m3._get_num_optim_iter(), names=list(m3.cov_par_names))
    if c.get("maxit", 1000) > 0:
        out["nll_fit"] = m3.get_current_neg_log_likelihood()
    if c.get("maxit", 1000) > 0 and 2 * c["m"] <= 60:  # the default prediction neighbour count 2 m; the device engine takes <= 60
        p = m3.predict(y, Xp, cp, predict_var=True, predict_response=True)
        out.update(pred_mu=p["mu"].tolist(), pred_var=p["var"].tolist())
    return out, m3
