"""Deterministic count data for the Poisson Laplace-Vecchia tests, the golden-vector script and the benchmark.

`count_synth` draws coords U[0,1]^d, a smooth latent surface and Poisson(exp(eta)) counts (numpy PCG64, seeded), with
eta = log_mean + latent (+ offset). log_mean = -2.5 gives mostly zeros, log(1000) counts around 1e3; with `offset_is_mean`
the constant log_mean is handed to the model as a fixed-effect offset instead of being left for the GP to absorb."""
import numpy as np


def count_synth(n, seed=1, with_offset=False, log_mean=0., offset_is_mean=False, d=2):
    rng = np.random.default_rng(seed)
    coords = rng.random((n, d))
    latent = 0.8 * np.sin(5 * coords[:, 0]) * np.cos(3 * coords[:, -1]) + 0.2 * rng.standard_normal(n)
    offset = 0.4 * np.cos(3 * coords[:, 0]) - 0.1 if with_offset else None
    if offset_is_mean:
        offset = (offset if offset is not None else np.zeros(n)) + log_mean
    eta = latent + (log_mean if not offset_is_mean else 0.) + (offset if offset is not None else 0.)
    y = rng.poisson(np.exp(eta)).astype(np.float64)
    return coords, y, offset


def case_data(c):
    return count_synth(c["n"], c["dseed"], c.get("offset", False), c.get("log_mean", 0.), c.get("offset_is_mean", False))


# the unmodified reference Python package fitting counts (fills `out`; tests/dropin.py runs it against a chosen library)
DROPIN_SCRIPT = """
rng = np.random.default_rng(17)
n = 800
coords = rng.random((n, 2))
lat = 0.7 * np.sin(5 * coords[:, 0]) * np.cos(3 * coords[:, 1])
y = rng.poisson(np.exp(lat)).astype(np.float64)
m = gpb.GPModel(gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=10,
                vecchia_ordering="random", seed=1, likelihood="poisson")
m.fit(y=y)
out["cov_pars"] = np.asarray(m.get_cov_pars()).reshape(-1).tolist()
out["negll_opt"] = float(m.get_current_neg_log_likelihood())
out["negll_at"] = float(m.neg_log_likelihood(cov_pars=np.array([0.5, 0.1]), y=y))
"""
