"""Cost of two crossed grouped random effects (gpboost_b200/csrc/dev/grouped_multi.cuh) on one GPU: n = 1e6 observations, factors with
1e4 and 1e3 levels, Gaussian likelihood, the reference's default iterative method (SSOR preconditioner, 50 probe vectors). Prints one
JSON line with
  * create_s: model creation (host level maps and Z^T Z pattern, device upload);
  * eval_s / grad_s: one likelihood evaluation (CG for M x = Z^T y, probe map, CG with Lanczos over 50 columns, SLQ) and one gradient
    after it, host wall time around the synchronous engine call, median of --reps; cg_it / slq_it of that evaluation;
  * spmm_ms / precond_ms: device time (CUDA events) of one M X and one P^-1 X on the 50 probe columns;
  * fit_s, fit_iterations, fit_cov_pars: one fit from the default initial values;
  * gpboost_it_per_s: boosting iterations per second with 50 features, 31 leaves, covariance parameters trained every iteration.
With --impl reference the same model calls run on the reference library (oracle/_ref): eval_s (GPModel.neg_log_likelihood), fit_s and
gpboost_it_per_s. Writes nothing. Usage: python bench_grouped_multi.py [--n 1000000] [--reps 3] [--boost-iters 5] [--impl cuda|reference]"""
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


def P(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip().split(",")
        return out[0].strip(), out[1].strip()
    except Exception:
        return None, None


def data(n, G1, G2, seed=0):
    rng = np.random.default_rng(seed)
    g1 = rng.integers(0, G1, size=n)
    g2 = rng.integers(0, G2, size=n)
    y = 0.5 * rng.standard_normal(n) + rng.standard_normal(G1)[g1] + 0.7 * rng.standard_normal(G2)[g2]
    return np.c_[g1, g2], y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--levels", default="10000,1000")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--boost-iters", type=int, default=5)
    ap.add_argument("--impl", default="cuda", choices=["cuda", "reference"])
    args = ap.parse_args()
    from gpboost_b200 import GPModel
    from gpboost_b200.booster import Booster, Dataset
    from gpboost_b200.libpath import load_lib
    log = lambda *a: print("[bench_grouped_multi]", *a, file=sys.stderr, flush=True)
    G1, G2 = (int(s) for s in args.levels.split(","))
    group, y = data(args.n, G1, G2)
    name, plimit = gpu_info()
    res = {"bench": "grouped_multi", "impl": args.impl, "gpu": name, "power_limit": plimit, "n": args.n, "levels": [G1, G2],
           "num_rand_vec_trace": 50}
    cp = np.array([0.25, 1.0, 0.5])
    if args.impl == "reference":
        from oracle import ref_lib_path
        lib = load_lib(ref_lib_path())
    else:
        lib = load_lib()
        if lib.gpbdev_device_count() < 1:
            raise SystemExit("bench_grouped_multi.py needs a CUDA device")
        lib.gpbdev_grouped_last_error.restype = C.c_char_p
    t0 = time.perf_counter()
    m = GPModel(group_data=group, _lib=lib)
    res["create_s"] = round(time.perf_counter() - t0, 3)
    res["negll"] = m.neg_log_likelihood(cp, y)  # warm-up (probe draw)
    ev = []
    for _ in range(args.reps):
        t0 = time.perf_counter(); m.neg_log_likelihood(cp, y); ev.append(time.perf_counter() - t0)
    res["model_eval_s"] = round(float(np.median(ev)), 4)
    if args.impl == "cuda":
        info = m.laplace_info()
        res["cg_it"], res["slq_it"] = int(info[2]), int(info[3])
        # the engine alone, driven as the optimiser drives it
        from oracle import grouped_multi as gm
        st = gm.Structure(group[:, :])
        idx = np.ascontiguousarray(np.concatenate(st.idx).astype(np.int32))
        lv = np.array(st.levels, dtype=np.int32)
        h = C.c_void_p()

        def chk(rc):
            if rc != 0:
                raise RuntimeError(lib.gpbdev_grouped_last_error().decode())
        chk(lib.gpbdev_grouped_multi_create(C.byref(h), 0, C.c_int64(args.n), 2, P(idx, C.c_int32), P(lv, C.c_int)))
        chk(lib.gpbdev_grouped_multi_set_y(h, P(np.ascontiguousarray(y))))
        r = np.asfortranarray(gm.probes(st, 50))
        chk(lib.gpbdev_grouped_multi_set_probes(h, P(r.reshape(-1, order="F")), 50))
        v = cp[1:] / cp[0]
        cfg = np.array([1000., 1000., 1e-2, 0.])
        out = np.zeros(5)
        g = np.zeros(2)
        chk(lib.gpbdev_grouped_multi_eval(h, P(v), P(cfg), P(out)))
        chk(lib.gpbdev_grouped_multi_grad(h, C.c_double(cp[0]), P(g)))
        ev, gr = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter(); chk(lib.gpbdev_grouped_multi_eval(h, P(v), P(cfg), P(out))); ev.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); chk(lib.gpbdev_grouped_multi_grad(h, C.c_double(cp[0]), P(g))); gr.append(time.perf_counter() - t0)
        res["eval_s"] = round(float(np.median(ev)), 4)
        res["grad_s"] = round(float(np.median(gr)), 4)
        res["engine_cg_it"], res["engine_slq_it"] = int(out[2]), int(out[3])
        chk(lib.gpbdev_grouped_multi_eval(h, P(v), P(cfg), P(out)))
        ms = np.zeros(2, dtype=np.float32)
        chk(lib.gpbdev_grouped_multi_time_ops(h, 10, P(ms, C.c_float)))
        res["spmm_ms"], res["precond_ms"] = round(float(ms[0]), 4), round(float(ms[1]), 4)
        nfo = np.zeros(2, dtype=np.int64)
        chk(lib.gpbdev_grouped_multi_info(h, P(nfo, C.c_int64)))
        res["G"], res["nnz_offdiag"] = int(nfo[0]), int(nfo[1])
        lib.gpbdev_grouped_multi_free(h)
    log(res)
    fm = GPModel(group_data=group, _lib=lib)
    t0 = time.perf_counter(); fm.fit(y); res["fit_s"] = round(time.perf_counter() - t0, 3)
    res["fit_iterations"] = fm._get_num_optim_iter()
    res["fit_cov_pars"] = fm.get_cov_pars().tolist()
    log(res)
    if args.boost_iters > 0:
        rng = np.random.default_rng(1)
        X = rng.random((args.n, 50))
        yb = y + 2 * np.sin(3 * X[:, 0]) + X[:, 1] ** 2
        params = {"objective": "regression", "num_leaves": 31, "learning_rate": 0.1, "max_bin": 255, "verbose": -1}
        gp = GPModel(group_data=group, _lib=lib)
        b = Booster(params, Dataset(X, yb, params=params, _lib=lib), gp_model=gp, _lib=lib)
        b.update()  # first iteration: initial values, host path
        t0 = time.perf_counter()
        for _ in range(args.boost_iters):
            b.update()
        res["gpboost_it_per_s"] = round(args.boost_iters / (time.perf_counter() - t0), 3)
        res["gpboost_cov_pars"] = gp.get_cov_pars().tolist()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
