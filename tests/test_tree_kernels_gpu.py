"""Every path of the device tree learner against the tree oracle, at kernel level (C ABI only).

`gpbdev_tree_train` (gpboost_b200/csrc/dev/tree_api.cu) grows every tree through one leaf loop on the device (hist3_kernel,
reduce_scan2_kernel, tree_advance_kernel, part_count_kernel + part_scatter_kernel per split). It enqueues that loop in one of three
ways, picked from num_leaves, from where the gradient lives and from whether a collective is installed:

  graph    device gradients and num_leaves <= 256 (one batch of splits): captured once per (gradient buffer, hessian), replayed
  eager    host gradients, or num_leaves > 256: enqueued in batches of 255 splits; between batches the host reads whether the
           tree is finished and stops
  sharded  a data-parallel learner, here one GPU with an identity collective (gpbdev_tree_set_allreduce): the same loop enqueued
           eagerly with hist_reduce_kernel into the staging histogram, the all-reduce, reduce_scan2_kernel from the stage and the
           children's local ranges set after the partition (tree_local_ranges_kernel)

test_cases_reach_every_kernel_path checks, without a GPU, that the runs below reach every path with one batch and with several,
and a tree that stops in a later batch.

Pass bars against oracle/tree_oracle.c: number of leaves, split features, threshold bins, children, leaf counts and the leaf
of every row bit-exact; leaf values <= 1e-10 of the largest one (the device merges per-chunk partial sums, the oracle adds row
by row); split gains within one float32 rounding. Integer-valued gradients, and gradients on a grid of 2^-16, make every sum
exact in any order, so there the leaf values and gains must agree to the last bit as well.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import tree as ot

SPLIT_BATCH = 255  # kSplitBatch: splits enqueued between two reads of the finished flag; the graph holds one batch
KEPS = float(np.float32(1e-15))  # kEpsilon


def path(kind, L, on_device):
    """(leaf loop, batches of splits enqueued for a full tree) that gpbdev_tree_train runs on one GPU; kind "sharded" = an
    identity collective is installed. Restates the choice in tree_grow."""
    batches = -(-(L - 1) // SPLIT_BATCH)
    if kind == "sharded":
        return "sharded", batches
    return ("graph" if on_device and batches == 1 else "eager"), batches


# ---------------------------------------------------------------------------------------------------------------- data
# per-feature bin counts, cycled over the features: 1 = a constant feature, 256 = bin value 255 present
NB_CYCLE = (256, 2, 17, 1, 255, 3, 40, 256, 9, 128)


def make_bins(n, F, seed, dup=False):
    """Feature-major (F, n) uint8 bins with mixed num_bin. Feature 6 (mod 10) uses every third of its 40 bins (empty bins
    between occupied ones: equal-gain thresholds), feature 8 (mod 10) has ~95 % of the rows in one bin. dup: the last
    feature repeats feature 0 and the middle one feature 1 (equal-gain features: the smaller index must win)."""
    rng = np.random.default_rng(seed)
    num_bin = np.array([NB_CYCLE[f % len(NB_CYCLE)] for f in range(F)], np.int32)
    bins = np.empty((F, n), np.uint8)
    for f in range(F):
        nb = int(num_bin[f])
        b = rng.integers(0, nb, n)
        if f % 10 == 6:
            b = b // 3 * 3
        if f % 10 == 8:
            b = np.where(rng.random(n) < 0.95, nb // 2, b)
        if nb == 256:
            b[0] = 255
        bins[f] = b
    if dup and F >= 3:
        for dst, src in ((F - 1, 0), (F // 2, 1)):
            bins[dst] = bins[src]
            num_bin[dst] = num_bin[src]
    return bins, num_bin


def make_grad(kind, bins, num_bin, seed):
    """continuous (a step in each of the first ten features plus noise), scaled by 1e-6 / 1e6, the same on a grid of 2^-16 or
    integer-valued in {-1, 0} / {-2..2} (exact sums in any order: gain ties are exact ties), or all zero.

    Continuous gradients and tiny leaves do not go together in these tests: two features can split a leaf of two or three rows into
    the same rows with the sides swapped, and the two gains then differ only by rounding, in a way that depends on the last bit
    of the leaf's gradient sum. That sum descends from the root sum, which the device adds in a fixed tree order and the oracle
    row by row (the reference uses an OpenMP reduction, LeafSplits::Init): either choice is right, and which feature wins is
    decided by noise. On the grid every sum is exact, the two gains are equal in both and the feature tie rule decides."""
    F, n = bins.shape
    rng = np.random.default_rng(seed + 1)
    g = rng.standard_normal(n)
    for f in range(min(F, 10)):
        nb = int(num_bin[f])
        if nb > 1:
            g += (bins[f] > nb // 2) * (0.9 if f % 2 else -0.7)
    if kind == "cont":
        return g
    if kind == "tiny":
        return 1e-6 * g
    if kind == "huge":
        return 1e6 * g
    if kind == "zero":
        return np.zeros(n)
    if kind == "grid":
        return np.round(g * 65536.) / 65536.
    if kind == "int1":
        return -(g > 0.3).astype(np.float64)
    if kind == "int2":
        return np.clip(np.round(g), -2., 2.)
    raise ValueError(kind)


# one case: (n, F, num_leaves, gradient kind, dup, knobs); knobs are gpbdev_tree_config fields, "hess" the constant hessian
def case_id(c):
    n, F, L, kind, dup, knobs = c
    return "n%d-F%d-L%d-%s%s%s" % (n, F, L, kind, "-dup" if dup else "", "".join("-%s=%s" % (k, v) for k, v in sorted(knobs.items())))


# run on every bucket
CORE = [(4097, 33, 31, "cont", False, {}),
        (257, 9, 31, "int2", True, {"min_data_in_leaf": 1}),
        (50, 4, 8, "int1", False, {"min_data_in_leaf": 1}),
        (30000, 65, 63, "cont", False, {"min_data_in_leaf": 5})]
# feature counts around the 32-byte row padding (Fpad), the 64-feature CTA groups of hist2/hist3 and past 128; row counts
# from a pair of rows to several histogram chunks per SM
SHAPES = [(2, 1, 31, "grid", False, {"min_data_in_leaf": 1}),
          (7, 4, 31, "int2", False, {"min_data_in_leaf": 1}),
          (9, 31, 31, "grid", False, {"min_data_in_leaf": 1}),
          (50, 32, 31, "grid", False, {"min_data_in_leaf": 1}),
          (257, 33, 31, "grid", False, {"min_data_in_leaf": 3}),
          (4097, 64, 31, "cont", False, {}),
          (4097, 65, 31, "int1", True, {"min_data_in_leaf": 2}),
          (30000, 96, 31, "cont", False, {}),
          (4097, 129, 31, "cont", True, {}),
          (30000, 200, 31, "cont", False, {}),
          (9, 129, 31, "int2", False, {"min_data_in_leaf": 1}),
          (257, 200, 31, "grid", False, {"min_data_in_leaf": 2})]
# split knobs (each binds: test_knob_cases_bind) and gradient kinds; both run on every scan implementation
KNOBS = [(4097, 31, 31, "cont", False, {"max_depth": 1}),
         (4097, 31, 31, "cont", False, {"max_depth": 2}),
         (4097, 31, 31, "cont", False, {"max_depth": 5}),
         (257, 9, 31, "grid", False, {"min_data_in_leaf": 1, "lambda_l2": 1.5}),
         (257, 9, 31, "grid", False, {"min_data_in_leaf": 1, "lambda_l2": 100.}),
         (257, 9, 31, "int1", False, {"min_data_in_leaf": 1, "min_gain_to_split": 0.5}),
         (4097, 31, 31, "cont", False, {"min_gain_to_split": "stump"}),
         (257, 9, 31, "cont", False, {"min_data_in_leaf": 1, "min_sum_hessian_in_leaf": 15.5}),
         (257, 9, 31, "int2", False, {"min_data_in_leaf": 1, "min_sum_hessian_in_leaf": 3., "hess": 0.25}),
         (50, 4, 31, "cont", False, {"min_data_in_leaf": 20}),
         (50, 4, 31, "cont", False, {"min_data_in_leaf": 26}),
         (50, 9, 31, "int1", False, {"min_data_in_leaf": 0, "min_sum_hessian_in_leaf": 0.})]
GRADS = [(4097, 33, 31, "tiny", False, {}),
         (4097, 33, 31, "huge", False, {}),
         (4097, 33, 31, "zero", False, {}),
         (4097, 33, 31, "int1", True, {"min_data_in_leaf": 1}),
         (4097, 33, 31, "int2", True, {"min_data_in_leaf": 1}),
         (4097, 33, 31, "cont", True, {})]
SPLIT = KNOBS + GRADS
# leaf budgets around the batches of 255 splits (256 leaves: the last graph), and one the data cannot fill (the tree stops in a
# later batch)
FILLED = (2, 3, 31, 255, 256, 257, 300, 511, 512, 513, 766)
EARLY_STOP = 2000
LEAVES = [(4097, 33, L, "grid", False, {"min_data_in_leaf": 3}) for L in FILLED + (EARLY_STOP,)]


def stump_gain(bins, num_bin, grad):
    """a min_gain_to_split between the root's gain and every later one: the tree stops at one split"""
    t = ot.train_tree(bins, num_bin, grad, ot.make_config(num_leaves=31))
    g = np.asarray(t["split_gain"], np.float64)
    assert g[0] > 1.5 * g[1:].max()
    return float(0.5 * (g[0] + g[1:].max()))


_DATA = {}


def case_data(c):
    """bins, num_bin, grad, config, hess_const, oracle tree (cached: one oracle run per case)"""
    key = case_id(c)
    if key not in _DATA:
        n, F, L, kind, dup, knobs = c
        bins, num_bin = make_bins(n, F, n + F, dup)
        grad = make_grad(kind, bins, num_bin, n + F)
        k = dict(knobs)
        hess = k.pop("hess", 1.0)
        if k.get("min_gain_to_split") == "stump":
            k["min_gain_to_split"] = stump_gain(bins, num_bin, grad)
        cfg = ot.make_config(num_leaves=L, **k)
        _DATA[key] = (bins, num_bin, grad, cfg, hess, ot.train_tree(bins, num_bin, grad, oracle_config(cfg), hess_const=hess))
    return _DATA[key]


def oracle_config(cfg):
    """the reference raises min_data_in_leaf to 1 when it and min_sum_hessian_in_leaf are both 0 (Config::CheckParamConflict,
    io/config.cpp:400-405); the learner applies the same rule at creation, the oracle (a restatement of the tree learner
    alone) gets the adjusted config"""
    if cfg.min_data_in_leaf <= 0 and cfg.min_sum_hessian_in_leaf <= KEPS:
        return ot.make_config(cfg.num_leaves, 1, cfg.min_sum_hessian_in_leaf, cfg.lambda_l2, cfg.min_gain_to_split, cfg.max_depth)
    return cfg


# ---------------------------------------------------------------------------------------------------------------- runs
# (kind, gradient on the device, case): every case set on every kind. "graph" passes device gradients (budgets above 256 leaves
# then run eagerly from device gradients), "eager" host gradients.
KINDS = (("graph", 1), ("eager", 0), ("sharded", 1))
RUNS = [(kind, god, c) for kind, god in KINDS for cases in (CORE, SHAPES, SPLIT, LEAVES) for c in cases]


def run_id(r):
    kind, god, c = r
    return "%s-%s-%s" % (kind, "devgrad" if god else "hostgrad", case_id(c))


# ---------------------------------------------------------------------------------------------------------------- C ABI
def P(a, t):
    return a.ctypes.data_as(C.POINTER(t))


@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    product_lib.gpbdev_tree_last_error.restype = C.c_char_p
    product_lib.gpbdev_bin_last_error.restype = C.c_char_p
    return product_lib


def chk(lib, rc):
    assert rc == 0, lib.gpbdev_tree_last_error().decode()


# the identity collective of a one-rank data-parallel learner (module level: the callback must outlive every learner using it)
NOOP_ALLREDUCE = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_double), C.c_int64, C.c_void_p)(lambda ctx, buf, count, stream: 0)


def create(lib, bins, num_bin, cfg, sharded=False):
    F, n = bins.shape
    h = C.c_void_p()
    nb = np.ascontiguousarray(num_bin, dtype=np.int32)
    chk(lib, lib.gpbdev_tree_create(C.byref(h), 0, C.c_int64(n), F, P(np.ascontiguousarray(bins), C.c_uint8), P(nb, C.c_int32),
                                    C.byref(cfg)))
    if sharded:
        chk(lib, lib.gpbdev_tree_set_allreduce(h, NOOP_ALLREDUCE, None, C.c_int64(n)))
    return h


def dev_vec(lib, h, x):
    p = C.c_void_p()
    chk(lib, lib.gpbdev_vec_alloc(h, C.byref(p), C.c_int64(len(x))))
    chk(lib, lib.gpbdev_vec_upload(h, p, P(np.ascontiguousarray(x, dtype=np.float64), C.c_double), C.c_int64(len(x))))
    return p


def download(lib, h, p, n):
    out = np.empty(n)
    chk(lib, lib.gpbdev_vec_download(h, P(out, C.c_double), p, C.c_int64(n)))
    return out


def leaf_of_row(lib, h, n, num_leaves):
    """leaf of every row of the last tree through the product ABI: score = 0 + (leaf + 1) on a zeroed vector, so a row that no
    leaf claims reads -1"""
    s = C.c_void_p()
    chk(lib, lib.gpbdev_vec_alloc(h, C.byref(s), C.c_int64(n)))
    try:
        ids = np.arange(1, num_leaves + 1, dtype=np.float64)
        chk(lib, lib.gpbdev_tree_add_score(h, P(ids, C.c_double), num_leaves, s, None))
        return download(lib, h, s, n) - 1.
    finally:
        lib.gpbdev_vec_free(h, s)


def train(lib, h, n, L, grad, on_device, hess_const=1.0):
    """one tree; grad is a host float64 array, or a device pointer when on_device"""
    nl = C.c_int(0)
    sf = np.zeros(L, np.int32); tb = np.zeros(L, np.int32); lc = np.zeros(L, np.int32); rc = np.zeros(L, np.int32)
    sg = np.zeros(L, np.float32); lv = np.zeros(L, np.float64); cnt = np.zeros(L, np.int32)
    g = grad if on_device else P(np.ascontiguousarray(grad, dtype=np.float64), C.c_double)
    chk(lib, lib.gpbdev_tree_train(h, g, 1 if on_device else 0, C.c_double(hess_const), C.byref(nl), P(sf, C.c_int), P(tb, C.c_int),
                                   P(lc, C.c_int), P(rc, C.c_int), P(sg, C.c_float), P(lv, C.c_double), P(cnt, C.c_int)))
    k = nl.value
    return {"num_leaves": k, "split_feature": sf[:k - 1], "threshold_bin": tb[:k - 1], "left_child": lc[:k - 1], "right_child": rc[:k - 1],
            "split_gain": sg[:k - 1], "leaf_value": lv[:k], "leaf_count": cnt[:k], "leaf_of_row": leaf_of_row(lib, h, n, k)}


def check_tree(d, a, exact, what=""):
    assert d["num_leaves"] == a["num_leaves"], what
    for k in ("split_feature", "threshold_bin", "left_child", "right_child", "leaf_count"):
        assert np.array_equal(d[k], a[k]), (what, k)
    assert np.array_equal(d["leaf_of_row"], a["leaf_of_row"].astype(np.float64)), (what, "leaf_of_row")
    if exact:
        assert np.array_equal(d["leaf_value"], a["leaf_value"]), (what, "leaf_value")
        assert np.array_equal(d["split_gain"], a["split_gain"]), (what, "split_gain")
    else:
        assert np.max(np.abs(d["leaf_value"] - a["leaf_value"])) <= 1e-10 * np.max(np.abs(a["leaf_value"])), (what, "leaf_value")
        assert np.all(np.abs(d["split_gain"] - a["split_gain"]) <= np.spacing(np.abs(a["split_gain"]))), (what, "split_gain")


def run_case(lib, c, on_device, sharded):
    bins, num_bin, grad, cfg, hess, want = case_data(c)
    n = bins.shape[1]
    h = create(lib, bins, num_bin, cfg, sharded)
    g = None
    try:
        if on_device:
            g = dev_vec(lib, h, grad)
        got = train(lib, h, n, cfg.num_leaves, g if on_device else grad, on_device, hess)
    finally:
        if g is not None:
            lib.gpbdev_vec_free(h, g)
        lib.gpbdev_tree_free(h)
    check_tree(got, want, c[3] in ("int1", "int2", "grid", "zero"), case_id(c))


# ---------------------------------------------------------------------------------------------------------------- B
@pytest.mark.gpu
@pytest.mark.parametrize("run", RUNS, ids=[run_id(r) for r in RUNS])
def test_tree_matches_oracle(lib, run):
    kind, on_device, c = run
    run_case(lib, c, on_device, kind == "sharded")


# ---------------------------------------------------------------------------------------------------------------- C
def boost_data(n, L, min_data, max_bin):
    bins, num_bin = make_bins(n, 33, 11)
    if max_bin:
        num_bin = np.minimum(num_bin, max_bin).astype(np.int32)
        bins = (bins % num_bin[:, None]).astype(np.uint8)
    label = (make_grad("cont", bins, num_bin, 11) + 3.).astype(np.float32)
    return bins, num_bin, label, ot.make_config(num_leaves=L, min_data_in_leaf=min_data)


# (num_leaves, rows, min_data_in_leaf, bins per feature at most, sharded): 31 leaves = the graph, 300 = eager batches, and the
# data-parallel sequence. Boosting gradients are continuous, and in a big tree many leaves leave bins empty: larger = parent - smaller
# then holds a rounding residual instead of 0 there, which decides between thresholds of equal partition by noise (see make_grad).
# At 300 leaves, leaves of >= 50 rows on <= 8 bins per feature keep every bin occupied.
BOOST = [(31, 4097, 5, 0, False), (300, 100000, 50, 8, False), (31, 4097, 5, 0, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("L,n,min_data,max_bin,sharded", BOOST, ids=["L31", "L300", "L31-sharded"])
def test_boosting_rounds_on_one_learner(lib, L, n, min_data, max_bin, sharded):
    """Five rounds of L2 boosting on ONE learner (ot.boost_l2 at kernel level): the gradient score - label is formed on the
    device into one fixed buffer, every tree grows from it, the shrunk leaf values are added to the device score. State carried
    from tree to tree (histogram slots, splittable flags, the row-index buffers; on the graph the graph captured by the first
    tree and replayed by the others) must give the oracle's trees. Then a second gradient buffer and a new hessian constant,
    each of which must re-capture the graph, and the first buffer once more."""
    bins, num_bin, label, cfg = boost_data(n, L, min_data, max_bin)
    n, lr = bins.shape[1], 0.1
    trees, score_o, init = ot.boost_l2(bins, num_bin, label, cfg, lr, 5)
    assert len(trees) == 5
    h = create(lib, bins, num_bin, cfg, sharded)
    bufs = []
    try:
        score = dev_vec(lib, h, np.full(n, init)); lab = dev_vec(lib, h, label.astype(np.float64)); grad = dev_vec(lib, h, np.zeros(n))
        bufs += [score, lab, grad]
        for k, want in enumerate(trees):
            chk(lib, lib.gpbdev_vec_sub(h, score, lab, grad, C.c_int64(n)))
            got = train(lib, h, n, cfg.num_leaves, grad, True)
            got["leaf_value"] = got["leaf_value"] * lr
            check_tree(got, want, False, "tree %d" % k)
            chk(lib, lib.gpbdev_tree_add_score(h, P(np.ascontiguousarray(got["leaf_value"]), C.c_double), got["num_leaves"], score, None))
        s = download(lib, h, score, n)
        assert np.max(np.abs(s - score_o)) <= 1e-10 * np.max(np.abs(score_o))
        g1 = download(lib, h, grad, n)
        g2 = make_grad("cont", bins, num_bin, 12)
        grad2 = dev_vec(lib, h, g2)
        bufs.append(grad2)
        for buf, g, hess in ((grad2, g2, 1.0), (grad, g1, 0.25), (grad, g1, 1.0)):
            got = train(lib, h, n, cfg.num_leaves, buf, True, hess)
            check_tree(got, ot.train_tree(bins, num_bin, g, cfg, hess_const=hess), False, "hess %g" % hess)
    finally:
        for b in bufs:
            lib.gpbdev_vec_free(h, b)
        lib.gpbdev_tree_free(h)


# (num_leaves, rows, min_data_in_leaf, gradient on the device): the graph, and the eager batches from host gradients
LOOPS = [(31, 4097, 5, True), (300, 100000, 50, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("L,n,min_data,on_device", LOOPS, ids=["L31", "L300"])
def test_device_bins_constructor_matches_host_constructor(lib, L, n, min_data, on_device):
    """The Booster's learner reads the bin matrix gpbdev_bin_matrix wrote (gpbdev_tree_create_on_device_bins); the kernel-level
    one transposes host bins itself (gpbdev_tree_create). Integer-valued columns with bin upper bounds k + 0.5 give the same bins,
    and both learners must grow the same tree, row for row."""
    F = 40
    Fpad = (F + 31) // 32 * 32
    bins, num_bin = make_bins(n, F, 21)
    grad = make_grad("cont", bins, num_bin, 21)
    cfg = ot.make_config(num_leaves=L, min_data_in_leaf=min_data)
    X = np.ascontiguousarray(bins.T, dtype=np.float64)
    ub = np.full((F, 256), np.inf)
    for f in range(F):
        ub[f, :num_bin[f] - 1] = np.arange(num_bin[f] - 1) + 0.5
    bins_dev = C.c_void_p()
    rc = lib.gpbdev_bin_matrix(0, P(X, C.c_double), 1, C.c_int64(n), F, 1, F, P(np.arange(F, dtype=np.int32), C.c_int32),
                               P(num_bin, C.c_int32), P(ub, C.c_double), 256, Fpad, C.byref(bins_dev))
    assert rc == 0, lib.gpbdev_bin_last_error().decode()
    h_dev = C.c_void_p()
    h_host = None
    trees = []
    try:
        rm = np.empty((n, Fpad), np.uint8)
        assert lib.gpbdev_bin_download(0, bins_dev, C.c_int64(n), Fpad, P(rm, C.c_uint8)) == 0
        assert np.array_equal(rm[:, :F], bins.T) and not rm[:, F:].any()
        chk(lib, lib.gpbdev_tree_create_on_device_bins(C.byref(h_dev), 0, C.c_int64(n), F, Fpad, bins_dev, P(num_bin, C.c_int32),
                                                       C.byref(cfg)))
        h_host = create(lib, bins, num_bin, cfg)
        for h in (h_dev, h_host):
            if not on_device:
                trees.append(train(lib, h, n, cfg.num_leaves, grad, False))
                continue
            g = dev_vec(lib, h, grad)
            try:
                trees.append(train(lib, h, n, cfg.num_leaves, g, True))
            finally:
                lib.gpbdev_vec_free(h, g)
    finally:
        lib.gpbdev_tree_free(h_dev)
        if h_host is not None:
            lib.gpbdev_tree_free(h_host)
        lib.gpbdev_bin_free(0, bins_dev)
    want = ot.train_tree(bins, num_bin, grad, cfg)
    assert want["num_leaves"] == L
    for k in trees[0]:
        assert np.array_equal(trees[0][k], trees[1][k]), k
    check_tree(trees[0], want, False)


@pytest.mark.gpu
def test_config_checks_at_creation(lib):
    """min_data_in_leaf < 0 is refused (the reference's CHECK_GE); both limits at 0 become min_data_in_leaf = 1 as in the
    reference, instead of admitting splits with an empty child (test_zero_limits_admit_empty_children)"""
    bins, num_bin = make_bins(50, 4, 1)
    h = C.c_void_p()
    rc = lib.gpbdev_tree_create(C.byref(h), 0, C.c_int64(50), 4, P(bins, C.c_uint8), P(num_bin, C.c_int32),
                                C.byref(ot.make_config(num_leaves=8, min_data_in_leaf=-1)))
    assert rc != 0 and "min_data_in_leaf" in lib.gpbdev_tree_last_error().decode()


# ---------------------------------------------------------------------------------------------------------------- D
@pytest.fixture(scope="module")
def full_size():
    n, F = 1000000, 50
    rng = np.random.default_rng(5)
    bins = rng.integers(0, 255, size=(F, n), dtype=np.uint8)
    num_bin = np.full(F, 255, np.int32)
    grad = rng.standard_normal(n)
    for f in range(12):
        grad += (bins[f] > 40 + 15 * f) * (0.3 if f % 2 else -0.25)
    return bins, num_bin, grad


@pytest.mark.gpu
@pytest.mark.parametrize("L,on_device", [(31, True), (300, False)], ids=["L31", "L300"])
def test_full_size_tree_matches_oracle(lib, full_size, L, on_device):
    """n = 1e6 x 50 features x 255 bins: deep leaves still span several partition segments (max_seg = 4 x SMs of >= 1024 rows)
    and several histogram chunks; 31 leaves on the graph, 300 eagerly from host gradients"""
    bins, num_bin, grad = full_size
    cfg = ot.make_config(num_leaves=L, min_data_in_leaf=20)
    want = ot.train_tree(bins, num_bin, grad, cfg)
    assert want["num_leaves"] == L
    n = bins.shape[1]
    h = create(lib, bins, num_bin, cfg)
    g = None
    try:
        if on_device:
            g = dev_vec(lib, h, grad)
        got = train(lib, h, n, cfg.num_leaves, g if on_device else grad, on_device)
    finally:
        if g is not None:
            lib.gpbdev_vec_free(h, g)
        lib.gpbdev_tree_free(h)
    check_tree(got, want, False)


# ---------------------------------------------------------------------------------------------------------------- no GPU
def test_cases_reach_every_kernel_path():
    """Every path is run with one batch of splits and with several (the graph holds one batch by construction), so trimming RUNS
    cannot silently drop one; every case set runs on every path; a tree that stops early stops in a later batch."""
    reached = {(p, min(b, 2)) for p, b in (path(kind, c[2], god) for kind, god, c in RUNS)}
    assert reached == {("graph", 1), ("eager", 1), ("eager", 2), ("sharded", 1), ("sharded", 2)}
    for cases in (CORE, SHAPES, SPLIT, LEAVES):
        assert {path(kind, c[2], god)[0] for kind, god, c in RUNS if c in cases} == {"graph", "eager", "sharded"}
    assert {path("graph", L, 1)[0] for L in (256, 257)} == {"graph", "eager"}
    assert {c[0] for c in CORE + SHAPES} >= {2, 7, 9, 50, 257, 4097, 30000}
    assert {c[1] for c in CORE + SHAPES} >= {1, 4, 31, 32, 33, 64, 65, 96, 129, 200}
    assert {c[2] for c in LEAVES} == set(FILLED) | {EARLY_STOP}
    early = [c for c in LEAVES if c[2] == EARLY_STOP]
    assert len(early) == 1
    grown = case_data(early[0])[5]["num_leaves"]
    assert SPLIT_BATCH + 1 < grown < EARLY_STOP - SPLIT_BATCH, grown  # stops inside a batch after the first, before the last


def test_leaf_budget_cases_fill_their_budget():
    for c in LEAVES:
        if c[2] in FILLED:
            assert case_data(c)[5]["num_leaves"] == c[2], case_id(c)


def test_knob_cases_bind():
    """every knob case grows a different tree (structure or values) than the same data with that knob at its default"""
    # min_data_in_leaf is compared with 1; next to another knob it only sets the stage
    defaults = {"max_depth": -1, "lambda_l2": 0., "min_gain_to_split": 0., "min_sum_hessian_in_leaf": 1e-3, "min_data_in_leaf": 1}
    for c in KNOBS:
        n, F, L, kind, dup, knobs = c
        if knobs.get("min_data_in_leaf") == 0:  # test_zero_limits_admit_empty_children
            continue
        bins, num_bin, grad, cfg, hess, want = case_data(c)
        for k in knobs:
            if k == "hess" or (k == "min_data_in_leaf" and len(knobs) > 1):
                continue
            base = ot.make_config(cfg.num_leaves, cfg.min_data_in_leaf, cfg.min_sum_hessian_in_leaf, cfg.lambda_l2, cfg.min_gain_to_split,
                                  cfg.max_depth)
            setattr(base, k, defaults[k])
            other = ot.train_tree(bins, num_bin, grad, base, hess_const=hess)
            same = other["num_leaves"] == want["num_leaves"] and all(
                np.array_equal(other[x], want[x]) for x in ("split_feature", "threshold_bin", "leaf_value", "leaf_count"))
            assert not same, (case_id(c), k)
        if knobs.get("min_gain_to_split") == "stump":
            assert want["num_leaves"] == 2
    # the gradient kinds: all-zero gradients leave one leaf, the others a full tree
    for c in GRADS:
        if c[5] == {}:
            assert case_data(c)[5]["num_leaves"] == (1 if c[3] == "zero" else c[2]), case_id(c)


def test_zero_limits_admit_empty_children():
    """Why the learner raises min_data_in_leaf to 1 when both limits are 0: the tree learner alone (the oracle) then splits off
    children with no rows, since a threshold past a leaf's last occupied bin gains (sum g)^2 (1/(H + eps) - 1/(H + 2 eps)) > 0
    for a small hessian sum H. Such a split has no partition on the device."""
    for c in KNOBS:
        if c[5].get("min_data_in_leaf") == 0:
            bins, num_bin, grad, cfg, hess, want = case_data(c)
            raw = ot.train_tree(bins, num_bin, grad, cfg, hess_const=hess)
            assert (raw["leaf_count"] == 0).any()
            assert (want["leaf_count"] > 0).all()
