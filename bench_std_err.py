"""Standard errors of the Gaussian Vecchia covariance parameters at scale: GPModel.get_cov_pars(std_err=True) at n = 1e6, m = 30,
t = 50 probe vectors (the reference's default num_rand_vec_trace), Matern 1.5, d = 2, on one GPU.

Reports, with the card's name and power limit (nvidia-smi):
  first_call_s   wall clock of the first get_cov_pars(std_err=True) after a fit: the host draw of the n x t probe block
                 (GenRandVecNormalParallel), one-time engine set-up (CSC view of B, processing order) and the Fisher pass
  refit_call_s   the same after a refit (probes reused, set-up done): what every later fit's standard errors cost
  cached_call_s  a repeated call (cached, no kernel)
  fisher_pass_ms CUDA events around gpbdev_vecchia_fisher_info alone (median of --reps), probes upload included
Every timed call ends in a device synchronisation (the call returns after its results reached the host)."""
import argparse
import ctypes as C
import json
import subprocess
import time

import numpy as np


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=60).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
        return name, pl
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--m", type=int, default=30)
    ap.add_argument("--t", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import __graft_entry__  # noqa: F401
    from gpboost_b200 import GPModel
    from gpboost_b200.libpath import load_lib
    lib = load_lib()
    rng = np.random.default_rng(1)
    coords = rng.random((a.n, 2))
    y = np.sin(4 * coords[:, 0]) + np.cos(3 * coords[:, 1]) + 0.5 * rng.standard_normal(a.n)
    cov_pars = np.array([0.25, 1.0, 0.05])
    g = GPModel(gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=a.m,
                vecchia_ordering="random", seed=1)
    params = dict(init_cov_pars=cov_pars, maxit=0, num_rand_vec_trace=a.t)
    g.fit(y, params=params)
    t0 = time.perf_counter()
    tab = g.get_cov_pars(std_err=True)
    first = time.perf_counter() - t0
    t0 = time.perf_counter()
    g.get_cov_pars(std_err=True)
    cached = time.perf_counter() - t0
    refit = []
    for _ in range(a.reps):
        g.fit(y, params=params)
        t0 = time.perf_counter()
        tab2 = g.get_cov_pars(std_err=True)
        refit.append(time.perf_counter() - t0)
    assert np.array_equal(tab, tab2)
    # the Fisher pass alone (CUDA events on the engine's stream)
    eng = C.c_void_p()
    g._safe_call(lib.GPB200_GetDeviceEngine(g.handle, C.byref(eng)))
    Z = np.asfortranarray(rng.standard_normal((a.n, a.t)))
    s2, var, rt = cov_pars[0], cov_pars[1] / cov_pars[0], np.sqrt(3.) / cov_pars[2]
    FI = np.zeros(9)
    ms = []
    for _ in range(a.reps + 1):
        ev = C.c_float(0.)
        assert lib.gpbdev_vecchia_timer_start(eng) == 0
        rc = lib.gpbdev_vecchia_fisher_info(eng, 1, C.c_double(s2), C.c_double(var), C.c_double(rt),
                                            Z.ctypes.data_as(C.POINTER(C.c_double)), a.t, FI.ctypes.data_as(C.POINTER(C.c_double)))
        assert rc == 0, lib.gpbdev_last_error()
        assert lib.gpbdev_vecchia_timer_stop(eng, C.byref(ev)) == 0
        ms.append(ev.value)
    name, pl = card()
    print(json.dumps({"bench": "std_err", "gpu": name, "power_limit": pl, "n": a.n, "m": a.m, "t": a.t,
                      "first_call_s": round(first, 4), "refit_call_s": round(float(np.median(refit)), 4),
                      "cached_call_s": round(cached, 6), "fisher_pass_ms": round(float(np.median(ms[1:])), 2),
                      "std_err": tab[1].tolist()}))


if __name__ == "__main__":
    main()
