"""Cost of validation data in the GPBoost-Vecchia boosting loop (n = 1e6 x 50 features, Vecchia m = 30, a 1e5-row validation set,
num_neighbors_pred = 60, use_gp_model_for_validation = True, metric test_neg_log_likelihood).

Measures, alternating the two boosters round by round so that clock drift affects both alike:
  * one boosting iteration without validation data and one with it (update + eval_valid);
  * the parts of one validation step: the update's extra cost (the new tree's walk over the validation rows), the GP prediction from
    the cached prediction set (gpbdev_vecchia_predset_eval, CUDA events on the engine's stream) and the rest of eval_valid (the metric
    kernel and the host round trip);
  * the same GP prediction through the uncached GPB_PredictREModel path (coordinates copied, neighbour search rerun, results to the host).
Prints one JSON line. Usage: python bench_validation.py [--n 1000000] [--nv 100000] [--rounds 10]"""
import argparse
import ctypes
import json
import subprocess
import time

import numpy as np

from gpboost_b200 import GPModel, load_lib
from gpboost_b200.booster import Booster, Dataset


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().split("\n")[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception:
        return "unknown", "unknown"


def make_data(n, nv, F, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2., 2., size=(n + nv, F))
    coords = rng.uniform(0., 1., size=(n + nv, 2))
    y = np.sin(2. * X[:, 0]) + 0.5 * (X[:, 1] > 0.3) + np.sin(4. * coords[:, 0]) * np.cos(3. * coords[:, 1]) + 0.4 * rng.standard_normal(n + nv)
    return X[:n], y[:n], coords[:n], X[n:], y[n:], coords[n:]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--nv", type=int, default=100000)
    ap.add_argument("--F", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    lib = load_lib()
    X, y, coords, Xv, yv, cv = make_data(a.n, a.nv, a.F, 1)
    params = dict(objective="regression", num_leaves=31, learning_rate=0.1, max_bin=255, min_data_in_leaf=20, verbose=-1,
                  train_gp_model_cov_pars=True, use_gp_model_for_validation=True)
    boosters = []
    for with_valid in (False, True):
        dtrain = Dataset(X, y, params=params)
        gp = GPModel(gp_coords=coords, cov_function="exponential", gp_approx="vecchia", num_neighbors=30, vecchia_ordering="random", seed=1)
        bst = Booster(params, dtrain, gp_model=gp)
        if with_valid:
            gp.set_prediction_data(gp_coords_pred=cv, num_neighbors_pred=60)
            bst.add_valid(Dataset(Xv, yv, params=params, reference=dtrain), "valid")
        boosters.append((bst, gp, dtrain))
    t_plain, t_update_v, t_eval = [], [], []
    for r in range(a.warmup + a.rounds):
        bst, _, _ = boosters[0]
        t0 = time.perf_counter(); bst.update(); t1 = time.perf_counter()
        bstv, _, _ = boosters[1]
        t2 = time.perf_counter(); bstv.update(); t3 = time.perf_counter(); ev = bstv.eval_valid(); t4 = time.perf_counter()
        if r >= a.warmup:
            t_plain.append(t1 - t0); t_update_v.append(t3 - t2); t_eval.append(t4 - t3)
    # the GP prediction alone: cached prediction set (CUDA events on the engine's stream) vs the uncached C API path
    _, gpv, _ = boosters[1]
    eng = gpv.device_engine()
    lib.gpbdev_vecchia_predset_create.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_double), ctypes.c_int64, ctypes.c_int,
                                                  ctypes.POINTER(ctypes.c_void_p)]
    lib.gpbdev_vecchia_predset_eval.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_double,
                                                ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_void_p)]
    lib.gpbdev_vecchia_predset_free.argtypes = [ctypes.c_void_p]
    cv_rm = np.ascontiguousarray(cv)
    ps = ctypes.c_void_p()
    assert lib.gpbdev_vecchia_predset_create(eng, cv_rm.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), a.nv, 60, ctypes.byref(ps)) == 0
    cp = gpv.get_cov_pars()
    var, rng_t = cp[1] / cp[0], 1. / cp[2]  # exponential: transformed range = 1 / rho (cov_fcts.h)
    t_cached = []
    m_ptr, v_ptr = ctypes.c_void_p(), ctypes.c_void_p()
    for r in range(a.warmup + a.rounds):
        assert lib.gpbdev_vecchia_timer_start(eng) == 0
        assert lib.gpbdev_vecchia_predset_eval(ps, 0, var, rng_t, ctypes.byref(m_ptr), ctypes.byref(v_ptr)) == 0
        ms = ctypes.c_float(0.)
        assert lib.gpbdev_vecchia_timer_stop(eng, ctypes.byref(ms)) == 0
        if r >= a.warmup:
            t_cached.append(ms.value * 1e-3)
    lib.gpbdev_vecchia_predset_free(ps)
    resid = boosters[1][0].inner_predict(0) - y.astype(np.float32).astype(np.float64)
    t_uncached = []
    for r in range(a.warmup + a.rounds):
        t0 = time.perf_counter()
        gpv.predict(y=resid, gp_coords_pred=cv, cov_pars=cp, predict_var=True, predict_response=True, num_neighbors_pred=60)
        if r >= a.warmup:
            t_uncached.append(time.perf_counter() - t0)
    med = lambda v: float(np.median(v)) * 1e3  # noqa: E731
    name, power = gpu_info()
    print(json.dumps(dict(
        bench="validation", gpu=name, power_limit=power, n=a.n, n_valid=a.nv, features=a.F, num_neighbors=30, num_neighbors_pred=60,
        rounds=a.rounds, metric=ev[0][1],
        iteration_ms_without_validation=med(t_plain), iteration_ms_with_validation=med(np.add(t_update_v, t_eval)),
        update_ms_with_validation=med(t_update_v), eval_valid_ms=med(t_eval),
        gp_prediction_cached_ms_cuda_events=med(t_cached), gp_prediction_uncached_c_api_ms=med(t_uncached),
        eval_valid_minus_gp_prediction_ms=med(t_eval) - med(t_cached),
        tree_score_update_ms_estimate=med(t_update_v) - med(t_plain))))


if __name__ == "__main__":
    main()
