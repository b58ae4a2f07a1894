"""Prediction with a trained GPBoost model (n = 1e6 x 50 features, 100 trees of 31 leaves, Gaussian Vecchia GP with m = 15 at fixed
covariance parameters). One seeded model, one command, after warm-up:
  (a) the ensemble-prediction kernel alone: CUDA events over `--reps` launches on the training matrix held in HBM; algorithmic bytes
      nrow * ncol * 8 + nrow * 8 over the kernel time, as a share of the H100's 3.35 TB/s HBM figure (the bound this kernel would hit
      if the walk were free: it is reported as what it is, a share of the bandwidth bound);
  (b) LGBM_BoosterPredictForMat end to end on the training matrix in pageable host memory (wall clock, the call returns synchronised):
      the host walk (GPB200_BoosterPredictForMatHost) and the device path alternated in the same run, outputs compared bitwise;
  (c) Booster.predict with the GP model at `--n-test` new rows, and its three parts: ensemble prediction of the training matrix,
      GP prediction from the residual, ensemble prediction of the new rows.
Needs a CUDA device (there is no fallback). Prints one JSON line. Usage: python bench_predict.py [--n 1000000] [--n-test 100000]"""
import argparse
import ctypes as C
import json
import subprocess
import time

import numpy as np

from gpboost_b200 import GPModel, load_lib
from gpboost_b200.booster import Booster, Dataset, C_API_PREDICT_RAW_SCORE

HBM_BYTES_PER_S = 3.35e12  # NVIDIA data sheet, H100 SXM


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30).stdout.strip().split("\n")[0]
    name, power = [x.strip() for x in q.split(",")]
    return name, power


def make_data(n, F, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2., 2., size=(n, F))
    coords = rng.uniform(0., 1., size=(n, 2))
    y = np.sin(2. * X[:, 0]) + 0.5 * (X[:, 1] > 0.3) + 0.3 * X[:, 2] * X[:, 3] + np.sin(4. * coords[:, 0]) * np.cos(3. * coords[:, 1]) + \
        0.4 * rng.standard_normal(n)
    return X, y, coords


def predict_for_mat(lib, fn, bst, X):
    n = C.c_int64(0)
    out = np.empty(X.shape[0])
    t0 = time.perf_counter()
    rc = fn(bst.handle, X.ctypes.data_as(C.c_void_p), C.c_int(1), C.c_int32(X.shape[0]), C.c_int32(X.shape[1]), C.c_int(1),
            C.c_int(C_API_PREDICT_RAW_SCORE), C.c_int(0), C.c_int(-1), b"", C.byref(n), out.ctypes.data_as(C.POINTER(C.c_double)))
    t = time.perf_counter() - t0
    if rc != 0:
        raise RuntimeError(lib.LGBM_GetLastError().decode())
    return out, t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--n-test", type=int, default=100000)
    ap.add_argument("--F", type=int, default=50)
    ap.add_argument("--trees", type=int, default=100)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--host-rounds", type=int, default=2)
    a = ap.parse_args()
    lib = load_lib()
    if lib.gpbdev_device_count() < 1:
        raise SystemExit("bench_predict.py needs a CUDA device")
    name, power = gpu_info()
    X, y, coords = make_data(a.n, a.F, 1)
    Xt, _, coords_t = make_data(a.n_test, a.F, 2)
    params = dict(objective="regression", num_leaves=31, learning_rate=0.1, max_bin=255, min_data_in_leaf=20, verbose=-1,
                  train_gp_model_cov_pars=False)
    cov_pars = np.array([0.16, 0.25, 0.2])
    gp = GPModel(gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=15, vecchia_ordering="random",
                 seed=1)
    gp.set_optim_params(dict(init_cov_pars=cov_pars))
    dtrain = Dataset(X, y, params=params, free_raw_data=False)
    bst = Booster(params, dtrain, gp_model=gp)
    for _ in range(a.trees):
        bst.update()
    num_trees = bst.current_iteration()
    # (a) kernel alone
    ms = C.c_float(0.)
    for _ in range(2):  # the first call loads the module and fills the buffers
        rc = lib.GPB200_BoosterTimePredictKernel(bst.handle, X.ctypes.data_as(C.c_void_p), C.c_int(1), C.c_int32(a.n), C.c_int32(a.F), C.c_int(1),
                                                 C.c_int(0), C.c_int(-1), C.c_int(a.reps), C.byref(ms))
        if rc != 0:
            raise RuntimeError(lib.LGBM_GetLastError().decode())
    kernel_ms = float(ms.value)
    kernel_bytes = a.n * a.F * 8 + a.n * 8
    # (b) end to end, host walk and device path alternated
    t_host, t_dev = [], []
    predict_for_mat(lib, lib.LGBM_BoosterPredictForMat, bst, X)  # warm-up: staging buffers
    for r in range(a.rounds):
        if r < a.host_rounds:
            want, t = predict_for_mat(lib, lib.GPB200_BoosterPredictForMatHost, bst, X)
            t_host.append(t)
        got, t = predict_for_mat(lib, lib.LGBM_BoosterPredictForMat, bst, X)
        t_dev.append(t)
        if not np.array_equal(got, want):
            raise RuntimeError("device and host predictions differ")
    # (c) Booster.predict with the GP model
    kw = dict(gp_coords_pred=coords_t, predict_var=True, pred_latent=False, cov_pars=cov_pars)
    bst.predict(Xt, **kw)
    t_all, t_train, t_gp, t_test = [], [], [], []
    for _ in range(a.rounds):
        t0 = time.perf_counter()
        whole = bst.predict(Xt, **kw)
        t1 = time.perf_counter()
        f_train = bst._predict_for_mat(X, C_API_PREDICT_RAW_SCORE, 0, -1)
        t2 = time.perf_counter()
        re = gp.predict(y=dtrain.label - f_train, gp_coords_pred=coords_t, cov_pars=cov_pars, predict_var=True, predict_response=True)
        t3 = time.perf_counter()
        f_test = bst._predict_for_mat(Xt, C_API_PREDICT_RAW_SCORE, 0, -1)
        t4 = time.perf_counter()
        if not np.array_equal(whole["response_mean"], re["mu"] + f_test):
            raise RuntimeError("Booster.predict differs from its parts")
        t_all.append(t1 - t0); t_train.append(t2 - t1); t_gp.append(t3 - t2); t_test.append(t4 - t3)
    med = lambda v: float(np.median(v)) * 1e3  # noqa: E731
    print(json.dumps(dict(
        bench="predict", gpu=name, power_limit=power, n=a.n, features=a.F, num_trees=num_trees, num_leaves=31, n_test=a.n_test,
        kernel_ms_cuda_events=kernel_ms, kernel_launches=a.reps, kernel_algorithmic_bytes=kernel_bytes,
        kernel_bytes_per_s=kernel_bytes / (kernel_ms * 1e-3), kernel_share_of_hbm_bandwidth_bound=kernel_bytes / (kernel_ms * 1e-3) / HBM_BYTES_PER_S,
        predict_for_mat_device_ms=med(t_dev), predict_for_mat_device_ms_all=[round(t * 1e3, 3) for t in t_dev],
        predict_for_mat_host_walk_ms=med(t_host), host_walk_over_device=med(t_host) / med(t_dev), outputs_bitwise_equal=True,
        matrix_bytes=a.n * a.F * 8, device_path_host_bytes_per_s=a.n * a.F * 8 / (med(t_dev) * 1e-3),
        booster_predict_gp_ms=med(t_all), train_matrix_prediction_ms=med(t_train), gp_prediction_ms=med(t_gp), test_matrix_prediction_ms=med(t_test))))


if __name__ == "__main__":
    main()
