"""Gaussian Vecchia GP with K independent realizations (cluster_ids) on one GPU: n = 1e6, m = 30, Matern 1.5, d = 2, random ordering;
K = 1, 100 and 10^4 equal clusters with interleaved labels, and K = 2 with a second cluster of 10 points.

Reports per K:
  create_s   model creation (ordering and the device neighbour search within every cluster), wall clock
  nll_ms     likelihood pass (gpbdev_vecchia_eval_async, NLL mode), device time from CUDA events on the engine's stream with the L2
             flushed before every pass, median of the repetitions
  grad_ms    gradient pass (GRAD mode), the same way
  fit_s      a full fit (GPModel.fit), wall clock, with its iterations
K = 1 is the model without cluster_ids (one label runs the unclustered code). K = 2 runs the clustered code on the same points, with
10 of them in a second cluster: its likelihood pass is alternated round by round with the pass of the same data without cluster_ids
(the headline pass), which measures what the clustered layout costs. With --reference (and oracle/_ref built) the reference library's
likelihood evaluation is timed on the CPU for each K. Prints the card name and power limit and one JSON line."""
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

COV_PARS = np.array([0.3, 1.0, 0.05])


def chk(lib, rc):
    if rc != 0:
        raise RuntimeError(lib.gpbdev_last_error().decode())


def eval_ms(lib, h, mode, reps):
    """median device time (CUDA events on the engine's stream, L2 flushed before each) of `reps` passes"""
    sums = np.empty(9)
    pt = (COV_PARS[1] / COV_PARS[0], np.sqrt(3.) / COV_PARS[2])
    out = []
    for _ in range(reps):
        chk(lib, lib.gpbdev_vecchia_flush_l2(h))
        chk(lib, lib.gpbdev_vecchia_sync(h))
        chk(lib, lib.gpbdev_vecchia_timer_start(h))
        chk(lib, lib.gpbdev_vecchia_eval_async(h, 1, C.c_double(pt[0]), C.c_double(pt[1]), mode))
        ms = C.c_float()
        chk(lib, lib.gpbdev_vecchia_timer_stop(h, C.byref(ms)))
        out.append(ms.value)
    chk(lib, lib.gpbdev_vecchia_last_sums(h, sums.ctypes.data_as(C.POINTER(C.c_double))))
    return float(np.median(out)), float(sums[0])


def data(n, K, seed=1):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0., 1., (n, 2))
    y = np.sin(6. * X[:, 0]) + np.cos(3. * X[:, 1]) + 0.3 * rng.standard_normal(n)
    if K == 2:  # one small second cluster
        lab = np.full(n, 3, dtype=np.int32)
        lab[rng.permutation(n)[:10]] = 10
    else:
        lab = (rng.permutation(n) % K).astype(np.int32) * 7 + 3  # K labels, interleaved
    return X, y, lab


def model(X, lab):
    return GPModel(gp_coords=X, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=30, vecchia_ordering="random",
                   seed=1, cluster_ids=lab)


def run(lib, n, K, reps, rounds, fit, ref):
    X, y, lab = data(n, K)
    res = {"K": K, "n": n, "m": 30}
    t0 = time.perf_counter()
    mdl = model(X, lab)
    res["create_s"] = time.perf_counter() - t0
    mdl.neg_log_likelihood(COV_PARS, y)
    h = mdl.device_engine()
    eval_ms(lib, h, 0, 2); eval_ms(lib, h, 2, 2)  # warm-up
    if K == 2:
        base = model(X, None)
        base.neg_log_likelihood(COV_PARS, y)
        hb = base.device_engine()
        eval_ms(lib, hb, 0, 2)
        a, b = [], []
        for _ in range(rounds):
            a.append(eval_ms(lib, h, 0, reps)[0])
            b.append(eval_ms(lib, hb, 0, reps)[0])
        res["nll_ms_rounds"] = a
        res["headline_nll_ms_rounds"] = b
        res["nll_ms"] = float(np.median(a))
        res["headline_nll_ms"] = float(np.median(b))
        del base
    else:
        res["nll_ms"] = eval_ms(lib, h, 0, reps)[0]
    res["grad_ms"] = eval_ms(lib, h, 2, reps)[0]
    if fit:
        t0 = time.perf_counter()
        mdl.fit(y)
        res["fit_s"] = time.perf_counter() - t0
        res["fit_iters"] = mdl._get_num_optim_iter()
        res["fit_cov_pars"] = [float(v) for v in np.asarray(mdl.get_cov_pars()).reshape(-1)]
    if ref is not None:
        rm = GPModel(gp_coords=X, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=30,
                     vecchia_ordering="random", seed=1, cluster_ids=lab, _lib=ref)
        rm.neg_log_likelihood(COV_PARS, y)
        t0 = time.perf_counter()
        rm.neg_log_likelihood(COV_PARS, y)
        res["reference_cpu_nll_s"] = time.perf_counter() - t0
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-fit", action="store_true")
    ap.add_argument("--reference", action="store_true", help="time the reference library's likelihood on the CPU (oracle/_ref)")
    args = ap.parse_args()
    lib = load_lib()
    if lib.gpbdev_device_count() < 1:
        raise SystemExit("bench_cluster_ids.py needs a CUDA device")
    ref = None
    if args.reference:
        from gpboost_b200.libpath import load_lib as load_any
        from oracle import ref_lib_path
        if os.path.exists(ref_lib_path()):
            ref = load_any(ref_lib_path())
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    results = [run(lib, args.n, K, args.reps, args.rounds, not args.no_fit, ref) for K in (1, 2, 100, 10000)]
    print(json.dumps({"metric": "cluster_ids_vecchia", "card": card, "reference": ref is not None, "results": results}))


if __name__ == "__main__":
    main()
