"""Deterministic test data shared by the oracle-pinning tests, the GPU parity tests and the golden-vector script.

`sim_rand_unif` restates the pure-arithmetic LCG the reference's R tests use to build their data
(R-package/tests/testthat/test_GPModel_gaussian_process.R:37-43), in float64 like R."""
import numpy as np


def sim_rand_unif(n, init_c, mod=2.0 ** 32, a=22695477.0, c=1.0):
    s = np.empty(n)
    s[0] = np.floor(init_c * mod)
    for i in range(1, n):
        s[i] = (a * s[i - 1] + c) % mod
    return s / mod


def r_test_data():
    """n=100 coordinates and response of test_GPModel_gaussian_process.R:46-66."""
    from scipy.stats import norm
    n, d = 100, 2
    coords = sim_rand_unif(n * d, 0.1).reshape((n, d), order="F")
    D = np.sqrt(((coords[:, None, :] - coords[None, :, :]) ** 2).sum(-1))
    eps = np.linalg.cholesky(np.exp(-D / 0.1) + 1e-20 * np.eye(n)) @ norm.ppf(sim_rand_unif(n, 0.8))
    xi = norm.ppf(sim_rand_unif(n, 0.1)) / 5
    return coords, eps + xi


def synth(n, d=2, seed=1, smooth=True):
    """Synthetic coords U[0,1]^d and a response with spatial structure + noise (seeded, numpy PCG64)."""
    rng = np.random.default_rng(seed)
    coords = rng.random((n, d))
    y = rng.standard_normal(n) * 0.5
    if smooth:
        y = y + np.sin(4 * coords[:, 0]) + np.cos(3 * coords[:, -1]) * coords[:, 0]
    return coords, y


def lattice(k):
    """k x k regular lattice: ubiquitous distance ties — the neighbour tie-break rules matter here."""
    g = np.arange(k) / k
    xx, yy = np.meshgrid(g, g, indexing="ij")
    return np.stack([xx.ravel(), yy.ravel()], axis=1)


def r_grouped_test_data():
    """n=1000 single-level grouped data of test_GPModel_grouped_random_effects.R:27-41,62 (LCG modulus 134456)."""
    from scipy.stats import norm
    lcg = lambda n, c: sim_rand_unif(n, c, mod=134456.0, a=8121.0, c=28411.0)
    n, m = 1000, 100
    group = np.repeat(np.arange(1, m + 1), n // m)
    b1 = norm.ppf(lcg(m, 0.546))
    xi = np.sqrt(0.5) * norm.ppf(lcg(n, 0.1))
    return group, b1[group - 1] + xi


def grouped_synth(n, G, seed, balanced=False):
    rng = np.random.default_rng(seed)
    if balanced:
        group = rng.permutation(np.arange(n) % G)
    else:  # unbalanced group sizes
        p = rng.dirichlet(np.full(G, 0.7))
        group = rng.choice(G, size=n, p=p)
    b = rng.standard_normal(G) * 0.8
    y = b[group] + 0.6 * rng.standard_normal(n)
    return group, y


def r_binary_test_data():
    """n=100 coordinates and binary response of test_GPModel_non_Gaussian_data.R:38-47, 2512-2513 (logit link)."""
    from scipy.stats import norm
    n, d = 100, 2
    coords = sim_rand_unif(n * d, 0.1).reshape((n, d), order="F")
    D = np.sqrt(((coords[:, None, :] - coords[None, :, :]) ** 2).sum(-1))
    latent = np.linalg.cholesky(np.exp(-D / 0.1) + 1e-20 * np.eye(n)) @ norm.ppf(sim_rand_unif(n, 0.8))
    probs = 1. / (1. + np.exp(-latent))
    return coords, (sim_rand_unif(n, 0.2341) < probs).astype(np.float64)


def binary_synth(n, seed=1, with_offset=False, d=2):
    """Synthetic coords U[0,1]^d, a smooth latent surface and Bernoulli(logit) labels; optional fixed-effect offset.
    The surface depends on the first and the last coordinate; at d = 2 these are the data the Laplace goldens were made from."""
    rng = np.random.default_rng(seed)
    coords = rng.random((n, d))
    latent = 1.5 * np.sin(6 * coords[:, 0]) * np.cos(4 * coords[:, -1]) + 0.3 * rng.standard_normal(n)
    offset = 0.5 * np.cos(3 * coords[:, 0]) - 0.2 if with_offset else None
    eta = latent + (offset if with_offset else 0.)
    y = (rng.random(n) < 1. / (1. + np.exp(-eta))).astype(np.float64)
    return coords, y, offset
