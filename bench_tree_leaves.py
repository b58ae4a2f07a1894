"""Per-tree time of the device tree learner (gpbdev_tree_train) at n = 1e6 rows x 50 features x 255 bins, for leaf budgets on
both sides of the 256-leaf graph and across several batches of splits, with device and with host gradients.

    python bench_tree_leaves.py [--trees 12] [--warmup 2] [--dump trees.npz]
    python bench_tree_leaves.py --compare a.npz b.npz

Prints one JSON line per (num_leaves, gradient location): the median wall time of one gpbdev_tree_train call (it ends with a
stream synchronise) over --trees trees after --warmup trees, all grown from the same gradient. The library is the product build,
or the one GPB200_LIB names. --dump writes every output of the last tree of each configuration; --compare checks two dumps for
bit-identity, e.g. this build against another commit's (gpboost_b200.build.build(out_name=...) in a checkout of that commit).
Nothing is written except the --dump file."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

OUTPUTS = ("split_feature", "threshold_bin", "left_child", "right_child", "split_gain", "leaf_value", "leaf_count")


class TreeCfg(C.Structure):  # gpbdev_tree_config
    _fields_ = [("num_leaves", C.c_int), ("min_data_in_leaf", C.c_int), ("min_sum_hessian_in_leaf", C.c_double),
                ("lambda_l2", C.c_double), ("min_gain_to_split", C.c_double), ("max_depth", C.c_int)]


def P(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def make_data(n, F, seed=5):
    rng = np.random.default_rng(seed)
    bins = rng.integers(0, 255, size=(F, n), dtype=np.uint8)
    grad = rng.standard_normal(n)
    for f in range(12):
        grad += (bins[f] > 40 + 15 * f) * (0.3 if f % 2 else -0.25)
    return bins, np.full(F, 255, np.int32), grad


def run(lib, bins, num_bin, grad, L, on_device, trees, warmup):
    F, n = bins.shape
    chk = lambda rc: rc == 0 or sys.exit("gpbdev: " + lib.gpbdev_tree_last_error().decode())
    h = C.c_void_p()
    cfg = TreeCfg(L, 20, 1e-3, 0., 0., -1)
    chk(lib.gpbdev_tree_create(C.byref(h), 0, C.c_int64(n), F, P(bins, C.c_uint8), P(num_bin, C.c_int32), C.byref(cfg)))
    g = P(grad, C.c_double)
    if on_device:
        g = C.c_void_p()
        chk(lib.gpbdev_vec_alloc(h, C.byref(g), C.c_int64(n)))
        chk(lib.gpbdev_vec_upload(h, g, P(grad, C.c_double), C.c_int64(n)))
    out = {k: np.zeros(L, np.float32 if k == "split_gain" else (np.float64 if k == "leaf_value" else np.int32)) for k in OUTPUTS}
    ptrs = [P(out[k], {np.dtype(np.int32): C.c_int, np.dtype(np.float32): C.c_float, np.dtype(np.float64): C.c_double}[out[k].dtype])
            for k in OUTPUTS]
    nl = C.c_int(0)
    times = []
    for t in range(warmup + trees):
        t0 = time.perf_counter()
        chk(lib.gpbdev_tree_train(h, g, 1 if on_device else 0, C.c_double(1.0), C.byref(nl), *ptrs))
        if t >= warmup:
            times.append(time.perf_counter() - t0)
    if on_device:
        lib.gpbdev_vec_free(h, g)
    lib.gpbdev_tree_free(h)
    k = nl.value
    res = {key: (v[:k - 1] if key in OUTPUTS[:5] else v[:k]).copy() for key, v in out.items()}
    res["num_leaves"] = np.array([k])
    return res, float(np.median(times)) * 1e3, float(np.min(times)) * 1e3


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    assert sorted(a.files) == sorted(b.files), (a.files, b.files)
    bad = [k for k in sorted(a.files) if a[k].dtype != b[k].dtype or not np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8))]
    print(json.dumps({"compared": len(a.files), "differ": bad}))
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--F", type=int, default=50)
    ap.add_argument("--leaves", default="31,256,257,1024,4096")
    ap.add_argument("--trees", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--dump", default=None)
    ap.add_argument("--compare", nargs=2, default=None)
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    from gpboost_b200 import libpath
    lib = libpath.load_lib()
    lib.gpbdev_tree_last_error.restype = C.c_char_p
    bins, num_bin, grad = make_data(args.n, args.F)
    dump = {}
    for L in [int(x) for x in args.leaves.split(",")]:
        for on_device in (True, False):
            res, med, best = run(lib, bins, num_bin, grad, L, on_device, args.trees, args.warmup)
            tag = "L%d_%s" % (L, "dev" if on_device else "host")
            dump.update({"%s_%s" % (tag, k): v for k, v in res.items()})
            print(json.dumps({"lib": os.path.basename(libpath.find_lib_path()), "num_leaves": L, "grad": "device" if on_device else "host",
                              "leaves_grown": int(res["num_leaves"][0]), "ms_per_tree_median": round(med, 3), "ms_per_tree_min": round(best, 3),
                              "trees": args.trees, "n": args.n, "F": args.F}), flush=True)
    if args.dump:
        np.savez(args.dump, **dump)


if __name__ == "__main__":
    main()
