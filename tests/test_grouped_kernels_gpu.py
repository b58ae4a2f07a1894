"""The grouped random-effect engine (gpboost_b200/csrc/dev/grouped_api.cu) against an extended-precision reference, at the
edges of its two reductions.

group_sums_kernel  one warp per group, lanes stride through the group's rows by 32 (group sizes 31 / 32 / 33 / 65, a group
                   of 2^20 rows), then a shuffle reduction
group_eval_kernel  one CTA of 256 threads; thread t sums the contiguous slice [t per, (t+1) per) of groups, per = ceil(G / 256)
                   (G = 255 / 256 / 257, and G = 1, where all but one thread is idle), then a tree reduction
group_yaux_kernel  y_aux = (y - s_g / (1/v + n_g)) scale, scattered back to the original row order

Reference: the five sums and y_aux from per-group sums taken in np.longdouble. Bars: each sum is a sum of products of the y_i;
it is held to bar x (the same sum over the magnitudes of those products), with bar = 8 eps (ceil(max n_g / 32) + ceil(G / 256)
+ 16), the longest fp64 summation chain either kernel runs, plus a few roundings per term. log(1 + v n_g) is taken of the
rounded 1 + v n_g, so each of its terms carries an absolute error of order eps: that sum is held against sum(1 + log(1 + v n_g)).
y_aux is compared elementwise against max |y_i| + |s_g| / (1/v + n_g) over the rows."""
import ctypes as C
import math

import numpy as np
import pytest

import datagen

LD = np.longdouble
EPS = np.finfo(np.float64).eps
VS = (1e-8, 1e-2, 1., 1e2, 1e8)
GS = (1, 2, 31, 255, 256, 257, 1000, 100000)
SIZES = ("ones", "32", "mixed", "big", "dirichlet")
# (G, sizes, num_groups - G: empty groups above the largest index used)
CASES = [(G, s, 0) for G in GS for s in SIZES]
CASES += [(255, "mixed", 3), (256, "32", 1), (1000, "dirichlet", 24), (1, "ones", 2)]

RATIOS = {}


def case_id(c):
    G, s, extra = c
    return "G%d-%s%s" % (G, s, "-empty%d" % extra if extra else "")


def make_case(c, seed=0):
    """group index (rows scrambled) and response"""
    G, sizes, extra = c
    rng = np.random.default_rng(seed + 7 * G + SIZES.index(sizes))
    if sizes == "dirichlet":
        group, y = datagen.grouped_synth(20 * G, G, seed + G)
        return group.astype(np.int32), y
    if sizes == "ones":
        ng = np.ones(G, dtype=np.int64)
    elif sizes == "32":
        ng = np.full(G, 32)
    elif sizes == "mixed":
        ng = np.array([31, 32, 33, 65])[np.arange(G) % 4]
    else:
        ng = np.ones(G, dtype=np.int64)
        ng[G // 2] = 1 << 20
    group = np.repeat(np.arange(G, dtype=np.int32), ng)[rng.permutation(int(ng.sum()))]
    b = rng.standard_normal(G) * 0.8
    y = b[group] + 0.6 * rng.standard_normal(group.shape[0]) + 0.3
    return group, y


def group_stats(group, y, num_groups):
    yl = y.astype(LD)
    ng = np.bincount(group, minlength=num_groups).astype(LD)
    s = np.zeros(num_groups, dtype=LD)
    a = np.zeros(num_groups, dtype=LD)   # sum of |y_i| per group: the magnitude of the terms of s_g
    np.add.at(s, group, yl)
    np.add.at(a, group, np.abs(yl))
    return group, yl, ng, s, a


def reference(group, y, num_groups, v, stats=None):
    group, yl, ng, s, a = stats or group_stats(group, y, num_groups)
    v = LD(v)
    d, opn = 1 / v + ng, 1 + v * ng
    lg = np.log(opn)
    yy = (yl * yl).sum()
    out = np.array([yy, (s * s / d).sum(), lg.sum(), (s * s * v / (opn * opn)).sum(), (v * ng / opn).sum()])
    scale = np.array([yy, (a * a / d).sum(), (1 + lg).sum(), (a * a * v / (opn * opn)).sum(), (v * ng / opn).sum()])
    m = s / d
    yaux = yl - m[group]
    yaux_scale = np.max(np.abs(yl) + (a / d)[group])
    return out, scale, yaux, yaux_scale


def bar(group, num_groups):
    max_ng = int(np.bincount(group, minlength=num_groups).max())
    return 8 * EPS * (math.ceil(max_ng / 32) + math.ceil(num_groups / 256) + 16)


def record(qty, err, scale, b, what):
    err, scale = float(err), float(scale)
    ratio = err / (b * scale) if scale > 0 else (0. if err == 0 else math.inf)
    if ratio > RATIOS.get(qty, (0., ""))[0]:
        RATIOS[qty] = (ratio, what)
    assert ratio <= 1., "%s: error %.3e > bar %.3e x scale %.3e (%s)" % (qty, err, b, scale, what)


@pytest.fixture(scope="module", autouse=True)
def report_ratios():
    yield
    if RATIOS:
        print("\nworst error / bar per quantity:")
        for k in sorted(RATIOS):
            print("  %-8s %.3e  %s" % (k, RATIOS[k][0], RATIOS[k][1]))


def P_(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


@pytest.fixture(scope="module")
def lib(product_lib):
    product_lib.gpbdev_grouped_last_error.restype = C.c_char_p
    return product_lib


@pytest.fixture(scope="module")
def gpu(lib):
    assert lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    return lib


def chk(lib, rc):
    assert rc == 0, lib.gpbdev_grouped_last_error().decode()


def refused(lib, rc, msg):
    assert rc == -1
    assert msg in lib.gpbdev_grouped_last_error().decode()


def create(lib, group, num_groups):
    h = C.c_void_p()
    g = np.ascontiguousarray(group, dtype=np.int32)
    chk(lib, lib.gpbdev_grouped_create(C.byref(h), 0, C.c_int64(g.shape[0]), P_(g, C.c_int32), num_groups))
    return h


def ev(lib, h, v):
    o = np.zeros(5)
    chk(lib, lib.gpbdev_grouped_eval(h, C.c_double(v), P_(o)))
    return o


def yaux(lib, h, v, scale, n):
    o = np.zeros(n)
    chk(lib, lib.gpbdev_grouped_yaux(h, C.c_double(v), C.c_double(scale), P_(o)))
    return o


def check_sums(out, ref, b, what):
    want, scale = ref[0], ref[1]
    for k, name in enumerate(("yy", "s2/d", "logdet", "dquad", "dlogdet")):
        record(name, abs(LD(out[k]) - want[k]), scale[k], b, what)


def check_yaux(got, ref, scale, b, what):
    record("yaux", np.max(np.abs(got.astype(LD) - ref[2] * LD(scale))), ref[3] * abs(scale), b, what)


# ---------------------------------------------------------------------------------------------------------- CPU-only
def test_cases_reach_every_reduction_edge():
    """group_eval_kernel's slices: one group per thread with idle threads (G < 256), exactly one (256), two for some threads
    (257); group_sums_kernel's lane loop: 1, 31, 32, 33, 65 and 2^20 rows per group"""
    per = {G: math.ceil(G / 256) for G, _, _ in CASES}
    assert {1, 2} <= set(per.values()) and max(per.values()) > 256
    assert {G for G, _, _ in CASES} >= {255, 256, 257}
    sizes = set()
    for c in CASES:
        if c[1] != "dirichlet" and c[0] <= 257:
            group, _ = make_case(c)
            sizes |= set(np.bincount(group).tolist())
    assert {1, 31, 32, 33, 65, 1 << 20} <= sizes
    group, _ = make_case((1000, "dirichlet", 0))
    ng = np.bincount(group, minlength=1000)
    assert ng.max() > 4 * ng.mean()   # unbalanced
    assert any(c[2] > 0 for c in CASES)


def test_create_refuses_out_of_range_index(lib):
    """checked on the host before any device resource is taken, so no GPU is needed"""
    h = C.c_void_p()
    for g, G in (([0, 1, -1], 2), ([0, 2, 1], 2), ([5], 5)):
        g = np.array(g, dtype=np.int32)
        refused(lib, lib.gpbdev_grouped_create(C.byref(h), 0, C.c_int64(g.shape[0]), P_(g, C.c_int32), G), "group index out of range")
    g = np.zeros(3, dtype=np.int32)
    refused(lib, lib.gpbdev_grouped_create(C.byref(h), 0, C.c_int64(3), P_(g, C.c_int32), 0), "at least one group")


# ---------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_grouped_engine_against_extended_reference(gpu, case):
    lib = gpu
    G, sizes, extra = case
    num_groups = G + extra
    group, y = make_case(case)
    n = group.shape[0]
    b = bar(group, num_groups)
    h = create(lib, group, num_groups)
    try:
        chk(lib, lib.gpbdev_grouped_set_y(h, P_(np.ascontiguousarray(y))))
        stats = group_stats(group, y, num_groups)
        for v in VS:
            ref = reference(group, y, num_groups, v, stats)
            check_sums(ev(lib, h, v), ref, b, "%s v=%g" % (case_id(case), v))
            for s in (1., 0.37):
                check_yaux(yaux(lib, h, v, s, n), ref, s, b, "%s v=%g scale=%g" % (case_id(case), v, s))
    finally:
        lib.gpbdev_grouped_free(h)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [(257, "mixed", 0), (256, "big", 0), (1000, "dirichlet", 5)], ids=case_id)
def test_device_resident_response(gpu, case):
    """set_y_device gives the sums of set_y bit for bit; yaux_device writes in place into the buffer it was given"""
    import torch
    lib = gpu
    G, sizes, extra = case
    num_groups = G + extra
    group, y = make_case(case)
    n = group.shape[0]
    v, scale = 0.7, 1. / 0.45
    h = create(lib, group, num_groups)
    try:
        chk(lib, lib.gpbdev_grouped_set_y(h, P_(np.ascontiguousarray(y))))
        want_sums = ev(lib, h, v)
        want_yaux = yaux(lib, h, v, scale, n)
        yd = torch.from_numpy(y).to("cuda:0")
        torch.cuda.synchronize()   # the engine's stream does not wait for torch's
        chk(lib, lib.gpbdev_grouped_set_y_device(h, C.c_void_p(yd.data_ptr())))
        assert np.array_equal(ev(lib, h, v), want_sums)
        chk(lib, lib.gpbdev_grouped_yaux_device(h, C.c_double(v), C.c_double(scale), C.c_void_p(yd.data_ptr())))
        assert np.array_equal(yd.cpu().numpy(), want_yaux)
        # the device response is a copy: overwriting the caller's buffer changed nothing
        assert np.array_equal(ev(lib, h, v), want_sums)
        ref = reference(group, y, num_groups, v)
        check_sums(want_sums, ref, bar(group, num_groups), case_id(case) + " device")
        check_yaux(want_yaux, ref, scale, bar(group, num_groups), case_id(case) + " device")
    finally:
        lib.gpbdev_grouped_free(h)


@pytest.mark.gpu
def test_new_response_replaces_the_sums(gpu):
    lib = gpu
    group, y = make_case((257, "mixed", 0))
    y2 = np.cos(np.arange(y.shape[0]) * 0.01) + 0.1 * y
    b = bar(group, 257)
    h = create(lib, group, 257)
    try:
        chk(lib, lib.gpbdev_grouped_set_y(h, P_(np.ascontiguousarray(y))))
        o1 = ev(lib, h, 2.)
        check_sums(o1, reference(group, y, 257, 2.), b, "first y")
        chk(lib, lib.gpbdev_grouped_set_y(h, P_(np.ascontiguousarray(y2))))
        o2 = ev(lib, h, 2.)
        assert not np.array_equal(o1[[0, 1, 3]], o2[[0, 1, 3]])
        ref2 = reference(group, y2, 257, 2.)
        check_sums(o2, ref2, b, "second y")
        check_yaux(yaux(lib, h, 2., 1., y.shape[0]), ref2, 1., b, "second y")
    finally:
        lib.gpbdev_grouped_free(h)


@pytest.mark.gpu
def test_error_paths(gpu):
    import torch
    lib = gpu
    group, y = make_case((31, "mixed", 0))
    n = group.shape[0]
    h = create(lib, group, 31)
    try:
        o, buf, buf_dev = np.zeros(5), np.zeros(n), torch.zeros(n, dtype=torch.float64, device="cuda:0")
        torch.cuda.synchronize()
        msg = "call gpbdev_grouped_set_y first"
        refused(lib, lib.gpbdev_grouped_eval(h, C.c_double(1.), P_(o)), msg)
        refused(lib, lib.gpbdev_grouped_yaux(h, C.c_double(1.), C.c_double(1.), P_(buf)), msg)
        refused(lib, lib.gpbdev_grouped_yaux_device(h, C.c_double(1.), C.c_double(1.), C.c_void_p(buf_dev.data_ptr())), msg)
        chk(lib, lib.gpbdev_grouped_set_y(h, P_(np.ascontiguousarray(y))))
        for v in (0., -1., float("nan")):
            refused(lib, lib.gpbdev_grouped_eval(h, C.c_double(v), P_(o)), "variance ratio must be positive")
        check_sums(ev(lib, h, 1.), reference(group, y, 31, 1.), bar(group, 31), "after refusals")
    finally:
        lib.gpbdev_grouped_free(h)


@pytest.mark.gpu
def test_gpmodel_string_labels_against_extended_reference(gpu):
    """GPModel(group_data=...) with string labels at G = 257: the host's level map, TransformCovPars and the
    Woodbury negative log-likelihood; response_gradient = y_aux / sigma^2"""
    from gpboost_b200 import GPModel
    group, y = make_case((257, "mixed", 0))
    labels = np.array(["lvl-%03d" % g for g in group])
    n = y.shape[0]
    s2, s1 = 0.45, 0.8
    v = s1 / s2
    out, scale, yaux_ref, yaux_scale = reference(group, y, 257, v)
    b = bar(group, 257)
    quad, logdet = out[0] - out[1], out[2]
    const = n / 2 * (np.log(LD(s2)) + np.log(2 * np.pi, dtype=LD))
    want = quad / 2 / LD(s2) + logdet / 2 + const
    mag = (out[0] + scale[1]) / 2 / LD(s2) + scale[2] / 2 + abs(const)
    m = GPModel(group_data=labels)
    record("negll", abs(LD(m.neg_log_likelihood(np.array([s2, s1]), y)) - want), mag, b, "GPModel G=257")
    m.set_optim_params({"init_cov_pars": np.array([s2, s1]), "maxit": 0})
    m.fit(y)
    g = m.response_gradient(y)
    record("resp_grad", np.max(np.abs(g.astype(LD) - yaux_ref / LD(s2))), yaux_scale / s2, b, "GPModel G=257")
