"""Cost of the poisson likelihood in the Laplace-Vecchia engine (gpboost_b200/csrc/dev/laplace.cuh) next to bernoulli_logit, on one GPU,
at n = 1e6, m = 30 (Matern 1.5, d = 2, random ordering), 50 probe vectors, on the same coordinates (tests/poisson_data.py: counts
drawn from a smooth latent surface; the bernoulli labels are 1{count > 0} of the same draw). Prints one JSON line with, per likelihood:
  * eval_s: one Laplace likelihood evaluation (Newton mode finding + SLQ log-determinant), host wall time around the synchronous
    call, median of --reps; newton_it, cg_it (all Newton PCG iterations), slq_it of that evaluation;
  * op_ms / precond_ms at t = 1 and t = 50: device time (CUDA events) of one operator (B^T D^-1 B + W) X and one VADU preconditioner
    application, i.e. the cost of one CG iteration's two big steps, at the W of the mode;
  * grad_s: one evaluation with its gradient (GPB200_EvalLaplaceGradient) minus eval_s;
  * fit_s, fit_iterations, fit_cov_pars of one fit from the default initial values on the first --fit-n points (default 2e5; poisson
    only unless --fit names both).
Progress goes to stderr. Writes nothing. Usage:
  python bench_laplace_poisson.py [--n 1000000] [--reps 3] [--fit poisson|bernoulli_logit,poisson|none] [--fit-n 200000]"""
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
T = 50


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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--fit", default="poisson", help="likelihoods to fit, comma-separated, or 'none'")
    ap.add_argument("--fit-n", type=int, default=200_000, help="size of the fit's sub-problem (the first fit_n points)")
    args = ap.parse_args()
    import poisson_data
    from gpboost_b200 import GPModel
    from gpboost_b200.libpath import load_lib
    lib = load_lib()
    if lib.gpbdev_device_count() < 1:
        raise SystemExit("bench_laplace_poisson.py needs a CUDA device")
    lib.gpbdev_last_error.restype = C.c_char_p

    def chk(rc, err=lambda: lib.LGBM_GetLastError().decode()):
        if rc != 0:
            raise RuntimeError(err())

    n = args.n
    coords, counts, _ = poisson_data.count_synth(n, 7)
    labels = {"poisson": counts, "bernoulli_logit": (counts > 0).astype(np.float64)}
    cp = np.array([1.0, 0.1])
    name, plimit = gpu_info()
    res = {"bench": "laplace_poisson", "gpu": name, "power_limit": plimit, "n": n, "m": M, "cov": "matern1.5", "d": 2,
           "num_rand_vec_trace": T, "mean_count": float(counts.mean()), "lik": {}}

    def model(lik):
        mdl = GPModel(likelihood=lik, gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia",
                      num_neighbors=M, vecchia_ordering="random", seed=1)
        mdl.set_optim_params(dict(num_rand_vec_trace=T))
        return mdl

    log = lambda *a: print("[bench_laplace_poisson]", *a, file=sys.stderr, flush=True)
    for lik in ("bernoulli_logit", "poisson"):
        y = labels[lik]
        mdl = model(lik)
        mdl.neg_log_likelihood(cp, y)  # warm-up
        log(lik, "warm-up done")
        ev = []
        for _ in range(args.reps):
            t0 = time.perf_counter(); v = mdl.neg_log_likelihood(cp, y); ev.append(time.perf_counter() - t0)
        info = mdl.laplace_info()
        h = mdl.device_engine()
        ops = {}
        for t in (1, T):
            ms = np.zeros(2, dtype=np.float32)
            chk(lib.gpbdev_vecchia_laplace_time_ops(h, t, 10, ms.ctypes.data_as(C.POINTER(C.c_float))), lambda: lib.gpbdev_last_error().decode())
            ops["t%d" % t] = {"op_ms": round(float(ms[0]), 4), "precond_ms": round(float(ms[1]), 4)}
        gr = []
        g = np.zeros(2); nl = C.c_double(0.)
        for _ in range(args.reps):
            t0 = time.perf_counter()
            chk(lib.GPB200_EvalLaplaceGradient(mdl.handle, P(np.ascontiguousarray(y)), P(cp), None, C.byref(nl), P(g)))
            gr.append(time.perf_counter() - t0)
        r = {"negll": v, "eval_s": round(float(np.median(ev)), 4), "newton_it": int(info[1]), "cg_it": int(info[2]), "slq_it": int(info[3]),
             "ops": ops, "grad_s": round(float(np.median(gr)) - float(np.median(ev)), 4), "grad": g.tolist()}
        log(lik, r)
        if lik in args.fit.split(","):
            nf = min(n, args.fit_n)
            fm = GPModel(likelihood=lik, gp_coords=coords[:nf], cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia",
                         num_neighbors=M, vecchia_ordering="random", seed=1)
            fm.set_optim_params(dict(num_rand_vec_trace=T))
            t0 = time.perf_counter(); fm.fit(y[:nf]); r["fit_s"] = round(time.perf_counter() - t0, 3)
            r["fit_n"] = nf; r["fit_iterations"] = fm._get_num_optim_iter(); r["fit_cov_pars"] = fm.get_cov_pars().tolist()
            r["fit_negll"] = fm.get_current_neg_log_likelihood()
            log(lik, "fit", r)
            del fm
        res["lik"][lik] = r
        del mdl
    print(json.dumps(res))


if __name__ == "__main__":
    main()
