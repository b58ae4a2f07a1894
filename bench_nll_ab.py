#!/usr/bin/env python
"""bench_nll_ab.py — A/B of the two-observation Vecchia likelihood pass between two builds of the library.

Loads the product library and a second build of the same C API (--base, e.g. an earlier commit built with
`gpboost_b200.build.build(out_name=...)`), builds one engine per library on the same data and neighbour sets, and
  * checks that both return bitwise the same 9 sums for every covariance type and for the NLL, STORE and GRAD passes
    (headline size, and a small odd n evaluated whole and as row shards whose last warp pair is half real);
  * times gpbdev_vecchia_eval_async like bench.py does (L2 flushed before every pass, CUDA events on the engine's stream),
    `--passes` passes per library and round, the two libraries alternated for `--rounds` rounds in one process.
Prints one JSON line: the per-round medians of each library, their spread, and the card's name and power limit.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

COV_PARS = np.array([0.5, 1.0, 0.1])  # bench.py's (sigma^2, sigma_1^2, rho)
COVS = {"exponential": 0, "matern15": 1, "matern25": 2, "gaussian": 3}
MODES = {"nll": 0, "store": 1, "grad": 2}


def make_data(n, seed=1):
    rng = np.random.default_rng(seed)
    return rng.random((n, 2)), rng.standard_normal(n)


class Engine:
    def __init__(self, lib, coords, y, m, nn=None, rows=None):
        self.lib = lib
        n = coords.shape[0]
        lo, hi = rows if rows is not None else (0, n)
        self.h = C.c_void_p()
        c = np.ascontiguousarray(coords, dtype=np.float64)
        perm = np.arange(n, dtype=np.int32)
        nnp = None if nn is None else np.ascontiguousarray(nn, dtype=np.int32).ctypes.data_as(C.POINTER(C.c_int32))
        self.chk(lib.gpbdev_vecchia_create(C.byref(self.h), 0, C.c_int64(n), 2, m, c.ctypes.data_as(C.POINTER(C.c_double)),
                                           perm.ctypes.data_as(C.POINTER(C.c_int32)), nnp, C.c_int64(lo), C.c_int64(hi)))
        yy = np.ascontiguousarray(y, dtype=np.float64)
        self.chk(lib.gpbdev_vecchia_set_y(self.h, yy.ctypes.data_as(C.POINTER(C.c_double))))
        self.n, self.m = n, m

    def chk(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.gpbdev_last_error().decode())

    def nn(self):
        out = np.zeros((self.n, self.m), dtype=np.int32)
        self.chk(self.lib.gpbdev_vecchia_get_nn(self.h, out.ctypes.data_as(C.POINTER(C.c_int32))))
        return out

    def sums(self, cov, mode, var, rng):
        out = np.zeros(9)
        self.chk(self.lib.gpbdev_vecchia_eval(self.h, cov, C.c_double(var), C.c_double(rng), mode,
                                              out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def time_passes(self, cov, mode, var, rng, passes):
        ms, out = C.c_float(0), []
        for _ in range(passes):
            self.chk(self.lib.gpbdev_vecchia_flush_l2(self.h))
            self.chk(self.lib.gpbdev_vecchia_timer_start(self.h))
            self.chk(self.lib.gpbdev_vecchia_eval_async(self.h, cov, C.c_double(var), C.c_double(rng), mode))
            self.chk(self.lib.gpbdev_vecchia_timer_stop(self.h, C.byref(ms)))
            out.append(ms.value)
        self.chk(self.lib.gpbdev_vecchia_sync(self.h))
        return out

    def free(self):
        self.lib.gpbdev_vecchia_free(self.h)


def load(path):
    lib = C.CDLL(path)
    lib.gpbdev_last_error.restype = C.c_char_p
    return lib


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        name, plim, clk = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": plim, "sm_max_clock": clk}
    except Exception as e:  # the timing stands without it, but say so
        return {"unavailable": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="second build of the library (shared object) to compare against")
    ap.add_argument("--lib", default=os.path.join(ROOT, "gpboost_b200", "lib_gpboost_b200.so"))
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--m", type=int, default=30)
    ap.add_argument("--passes", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--modes", default="nll,grad", help="passes to time (comma separated: nll, store, grad)")
    args = ap.parse_args()
    libs = {"new": load(args.lib), "base": load(args.base)}
    var_t, range_t = COV_PARS[1] / COV_PARS[0], np.sqrt(3.) / COV_PARS[2]
    res = {"card": card(), "n": args.n, "m": args.m, "passes": args.passes, "rounds": args.rounds}

    # ---- identical sums: small odd n (whole and row shards) for every covariance type and pass, then the headline size
    mismatch = []
    n_small = 20001
    cs, ys = make_data(n_small, seed=7)
    first = Engine(libs["base"], cs, ys, args.m)
    nn_small = first.nn()
    first.free()
    shards = [None, (0, 10001), (10001, n_small), (3, 4004)]
    for rows in shards:
        eng = {k: Engine(lib, cs, ys, args.m, nn_small, rows) for k, lib in libs.items()}
        for cname, cov in COVS.items():
            for mname, mode in MODES.items():
                a, b = eng["new"].sums(cov, mode, var_t, range_t), eng["base"].sums(cov, mode, var_t, range_t)
                if a.tobytes() != b.tobytes():
                    mismatch.append({"n": n_small, "rows": rows, "cov": cname, "mode": mname, "new": a.tolist(), "base": b.tolist()})
        for e in eng.values():
            e.free()
    coords, y = make_data(args.n)
    eng = {"base": Engine(libs["base"], coords, y, args.m)}
    nn = eng["base"].nn()
    eng["new"] = Engine(libs["new"], coords, y, args.m, nn)
    for mname in ("nll", "grad"):
        a = eng["new"].sums(COVS["matern15"], MODES[mname], var_t, range_t)
        b = eng["base"].sums(COVS["matern15"], MODES[mname], var_t, range_t)
        res["sums_" + mname] = a.tolist()
        if a.tobytes() != b.tobytes():
            mismatch.append({"n": args.n, "rows": None, "cov": "matern15", "mode": mname, "new": a.tolist(), "base": b.tolist()})
    res["bitwise_equal"] = not mismatch
    res["mismatches"] = mismatch

    # ---- timing, alternated
    for mname in args.modes.split(","):
        mode = MODES[mname]
        for e in eng.values():  # warm-up
            e.time_passes(COVS["matern15"], mode, var_t, range_t, 3)
        med = {"new": [], "base": []}
        for _ in range(args.rounds):
            for k in ("base", "new"):
                med[k].append(float(np.median(eng[k].time_passes(COVS["matern15"], mode, var_t, range_t, args.passes))))
        out = {}
        for k, v in med.items():
            out[k] = {"round_medians_ms": [round(x, 4) for x in v], "median_ms": float(np.median(v)),
                      "spread_ms": float(max(v) - min(v))}
        out["speedup"] = out["base"]["median_ms"] / out["new"]["median_ms"]
        res[mname] = out
    for e in eng.values():
        e.free()
    print(json.dumps(res))
    return 0 if not mismatch else 1


if __name__ == "__main__":
    sys.exit(main())
