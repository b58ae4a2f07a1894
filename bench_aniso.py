"""Anisotropic covariance functions of the Gaussian Vecchia GP on one GPU: matern_ard (d = 2) and matern_space_time (d = 3) at
n = 1e6, m = 30, and matern_ard at d = 5, n = 1e5, where the device neighbour search is brute force (O(n^2)).

Reports per model, in ms of wall clock around work that ends in a device synchronise (median of the timed repetitions):
  scale      gpbdev_vecchia_set_coord_scale (coordinates times the per-column factors)
  search     gpbdev_vecchia_search_neighbors on the scaled coordinates
  nll        likelihood pass at range 1 (the isotropic kernel: for d = 2 the headline two-observation kernel)
  grad_iso   isotropic gradient pass on the same coordinates (one range derivative)
  grad_aniso gradient pass with one range derivative per coordinate group
and the wall time of a full fit (GPModel.fit) with its iterations and neighbour searches. Prints the card name and power limit and
one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from gpboost_b200 import GPModel, load_lib  # noqa: E402


def P(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


def chk(lib, rc):
    if rc != 0:
        raise RuntimeError(lib.gpbdev_last_error().decode())


def timed(lib, h, fn, reps):
    out = []
    for _ in range(reps):
        chk(lib, lib.gpbdev_vecchia_sync(h))
        t0 = time.perf_counter()
        fn()
        chk(lib, lib.gpbdev_vecchia_sync(h))
        out.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(out))


def run(lib, name, cov, d, n, m, reps, fit):
    rng = np.random.default_rng(d)
    X = rng.uniform(0., 1., (n, d))
    y = np.sin(6. * X[:, 0]) + np.cos(3. * X[:, -1]) + 0.3 * rng.standard_normal(n)
    space_time = cov == "matern_space_time"
    groups = np.array([0] + [1] * (d - 1) if space_time else list(range(d)), dtype=np.int32)
    lam = np.sqrt(3.) / np.linspace(0.1, 0.3, int(groups.max()) + 1)
    scale = np.ascontiguousarray(lam[groups])
    perm = np.arange(n, dtype=np.int32)
    h = C.c_void_p()
    chk(lib, lib.gpbdev_vecchia_create_unsearched(C.byref(h), 0, C.c_int64(n), d, m, P(np.ascontiguousarray(X)), P(perm, C.c_int32),
                                                  C.c_int64(0), C.c_int64(n)))
    chk(lib, lib.gpbdev_vecchia_set_y(h, P(y)))
    res = {"model": name, "cov_function": cov, "n": n, "d": d, "m": m}
    res["scale_ms"] = timed(lib, h, lambda: chk(lib, lib.gpbdev_vecchia_set_coord_scale(h, P(scale))), reps)
    res["search_ms"] = timed(lib, h, lambda: chk(lib, lib.gpbdev_vecchia_search_neighbors(h)), max(1, reps // 4))
    sums = np.empty(9)
    out = np.empty(3 + 3 * (1 + int(groups.max()) + 1))
    ev = lambda mode: chk(lib, lib.gpbdev_vecchia_eval(h, 1, C.c_double(2.), C.c_double(1.), mode, P(sums)))  # noqa: E731
    ga = lambda: chk(lib, lib.gpbdev_vecchia_eval_grad_aniso(h, 1, C.c_double(2.), P(groups, C.c_int32), int(groups.max()) + 1, P(out)))  # noqa: E731
    for f in (lambda: ev(0), lambda: ev(2), ga):  # warm-up
        f()
    res["nll_ms"] = timed(lib, h, lambda: ev(0), reps)
    res["grad_iso_ms"] = timed(lib, h, lambda: ev(2), reps)
    res["grad_aniso_ms"] = timed(lib, h, ga, reps)
    lib.gpbdev_vecchia_free(h)
    if fit:
        mdl = GPModel(gp_coords=X, cov_function=cov, cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=m, vecchia_ordering="random",
                      seed=1)
        t0 = time.perf_counter()
        mdl.fit(y)
        res["fit_s"] = time.perf_counter() - t0
        res["fit_iters"] = mdl._get_num_optim_iter()
        res["fit_searches"] = mdl._get_num_neighbor_searches()
        res["fit_cov_pars"] = [float(v) for v in np.asarray(mdl.get_cov_pars()).reshape(-1)]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--n-d5", type=int, default=100000)
    args = ap.parse_args()
    lib = load_lib()
    if lib.gpbdev_device_count() < 1:
        raise SystemExit("bench_aniso.py needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    results = [run(lib, "ard_d2", "matern_ard", 2, args.n, 30, args.reps, True),
               run(lib, "space_time_d3", "matern_space_time", 3, args.n, 30, args.reps, True),
               run(lib, "ard_d5", "matern_ard", 5, args.n_d5, 30, max(2, args.reps // 4), False)]
    print(json.dumps({"metric": "aniso_vecchia", "card": card, "results": results}))


if __name__ == "__main__":
    main()
