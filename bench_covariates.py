"""Cost of linear regression covariates in the Gaussian Vecchia fit (gpboost_b200/csrc/dev/covariates.cuh) on one GPU, at n = 1e6,
m = 30 (Matern 1.5, d = 2, random ordering), p in {1, 8, 32}. Prints one JSON line:
  * gram_ms: device time of the GLS Gram pass (kernel + chunk reduction + the p^2 + p doubles to the host), CUDA events on the
    engine's stream, L2 flushed before every call; median of 20.
  * achieved bytes/s against two algorithmic traffic counts per row: perfect reuse of the neighbours' rows, 12 m + 16 + 8 p bytes
    (A, nn, D^-1, y - offset, the row's own X), and no reuse, plus 8 (p + 1) m bytes of gathered neighbour rows.
  * eval_ms: one profiled objective + gradient evaluation (STORE pass, Gram pass, p x p solve, residual pass, GRAD pass) against the
    evaluation without covariates (one GRAD pass), host wall time around synchronous calls, alternated in the same process; medians.
  * fit: a full fit (GPModel.fit(y, X)), wall time and L-BFGS iterations.
Writes nothing. Usage: python bench_covariates.py [--n 1000000] [--reps 20]"""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

M = 30
COV_MATERN15 = 1
MODE_STORE, MODE_GRAD = 1, 2


def P(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        return out[0].strip(), out[1].strip()
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import datagen
    from gpboost_b200 import GPModel
    from gpboost_b200.libpath import load_lib
    lib = load_lib()
    if lib.gpbdev_device_count() < 1:
        raise SystemExit("bench_covariates.py needs a CUDA device")

    def chk(rc):
        if rc != 0:
            raise RuntimeError(lib.gpbdev_last_error().decode())

    n = args.n
    coords, y = datagen.synth(n, 2, 1)
    rng = np.random.default_rng(2)
    var, range_t = 1.0, np.sqrt(3.) / 0.1
    name, plimit = gpu_info()
    res = {"bench": "covariates_gls", "gpu": name, "power_limit": plimit, "n": n, "m": M, "cov": "matern1.5", "d": 2, "p": {}}
    for p in (1, 8, 32):
        X = np.ones((n, p))
        X[:, 1:] = rng.standard_normal((n, p - 1))
        yy = y + X @ rng.uniform(-1., 1., p)
        mdl = GPModel(gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=M,
                      vecchia_ordering="random", seed=1)
        t0 = time.perf_counter()
        mdl.fit(yy, X=X)
        fit_s = time.perf_counter() - t0
        h = mdl.device_engine()
        sums = np.zeros(9)
        G = np.empty((p, p)); r = np.empty(p); o3 = np.empty(3)
        chk(lib.gpbdev_vecchia_eval(h, COV_MATERN15, C.c_double(var), C.c_double(range_t), MODE_STORE, P(sums)))
        chk(lib.gpbdev_vecchia_gls_gram(h, P(G), P(r)))  # warm-up
        times = []
        for _ in range(args.reps):
            chk(lib.gpbdev_vecchia_flush_l2(h))
            chk(lib.gpbdev_vecchia_timer_start(h))
            chk(lib.gpbdev_vecchia_gls_gram(h, P(G), P(r)))
            ms = C.c_float(0)
            chk(lib.gpbdev_vecchia_timer_stop(h, C.byref(ms)))
            times.append(ms.value)
        gram_ms = float(np.median(times))
        b_reuse = n * (12 * M + 16 + 8 * p)
        b_noreuse = b_reuse + n * 8 * (p + 1) * M

        def eval_cov():
            chk(lib.gpbdev_vecchia_eval(h, COV_MATERN15, C.c_double(var), C.c_double(range_t), MODE_STORE, P(sums)))
            chk(lib.gpbdev_vecchia_gls_gram(h, P(G), P(r)))
            beta = np.linalg.solve(G, r)
            chk(lib.gpbdev_vecchia_gls_residual(h, P(np.ascontiguousarray(beta)), P(o3)))
            chk(lib.gpbdev_vecchia_eval(h, COV_MATERN15, C.c_double(var), C.c_double(range_t), MODE_GRAD, P(sums)))

        def eval_plain():
            chk(lib.gpbdev_vecchia_eval(h, COV_MATERN15, C.c_double(var), C.c_double(range_t), MODE_GRAD, P(sums)))

        tc, tp = [], []
        eval_cov(); eval_plain()
        for _ in range(args.reps):
            # distinct parameters each time: no pass is answered from the stored factor
            range_t *= 1.0001
            t0 = time.perf_counter(); eval_cov(); tc.append((time.perf_counter() - t0) * 1e3)
            range_t *= 1.0001
            t0 = time.perf_counter(); eval_plain(); tp.append((time.perf_counter() - t0) * 1e3)
        res["p"][str(p)] = {
            "gram_ms": round(gram_ms, 4),
            "bytes_perfect_reuse": b_reuse, "bytes_no_reuse": b_noreuse,
            "gbps_vs_perfect_reuse": round(b_reuse / (gram_ms * 1e-3) / 1e9, 1),
            "gbps_vs_no_reuse": round(b_noreuse / (gram_ms * 1e-3) / 1e9, 1),
            "eval_ms_with_covariates": round(float(np.median(tc)), 3), "eval_ms_without": round(float(np.median(tp)), 3),
            "fit_s": round(fit_s, 3), "fit_iterations": mdl._get_num_optim_iter(),
        }
        del mdl
    print(json.dumps(res))


if __name__ == "__main__":
    main()
