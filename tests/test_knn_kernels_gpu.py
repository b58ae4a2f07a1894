"""Every path of the device neighbour search (gpboost_b200/csrc/dev/knn.cuh) against the reference's walk, for model and
prediction queries.

The search must return the reference's neighbour sets bit for bit, in the same order. `knn_vecchia_device_ks` runs:

  knn_brute_kernel<KS>          queries below 4096, every query when there are at most 4096 candidates, every query when d > 3
  cell list + knn_grid_kernel   d <= 3 and more than 4096 candidates: knn_cell_id_kernel -> CUB sort -> knn_cell_start_kernel
  knn_walk_kernel<KS>           exact replay of the "risky" queries, whose pruning test smd > d T the rounding can decide
  KS = 1 / 2                    m <= 32 / 33 <= m <= 60
  model queries                 gpbdev_vecchia_create: q_begin = 0, end_search_at = n - 2
  prediction queries            gpbdev_vecchia_predict: q_begin = n_obs, end_search_at = n_obs - 1, over observed + prediction points

`gpbdev_knn_search` runs the same search from host coordinates and reports what it did. Three references, all exact:

  (a) the oracle's restatement of the reference's driver and walk (oracle.vecchia.knn_range): equal bit for bit, always;
  (b) an independent numpy brute force ordering every candidate by (sed, visit rank): sed summed in coordinate order from
      t = a - b; s = s + t*t (numpy rounds each operation, as __dsub_rn / __dmul_rn / __dadd_rn do), rank
      2|pos_j - pos_i| + (pos_j > pos_i) with pos from the same std::sort the reference uses (oracle.vecchia.sort_indices);
      the device must equal it on every query that is not risky (n <= 20 000);
  (c) the replay count: a query is risky when its m-th sed is T and one of its top m (from (b)) has
      fl(fl(csum_j - csum_i)^2) > fl(d T). The device's count (info[0], gpbdev_vecchia_knn_replayed) must equal it exactly.

In one dimension smd and sed are the same rounded number, so no 1-D query can be risky: the replay cannot run behind the 1-D
grid, and the bucket check below leaves that combination out. Integer lattices are exact as well; the lattices here have
spacing 1/k, whose rounding makes diagonal neighbours at the m-th distance risky.

CPU-only tests restate the dispatch and the grid sizing, check that the cases reach every bucket, that every grid case has at
most 2^d n / 8 cells and a short ring walk (a case that could run away is caught before it reaches a GPU), that the declared
replay flags hold for the reference, and that the entry's refusals fire."""
import ctypes as C
import functools
import math

import numpy as np
import pytest

import datagen
from oracle import predict as op
from oracle import vecchia as ov

BRUTE_REF_MAX_N = 20000  # the numpy brute force (b) runs up to this many points


def P(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


# ---------------------------------------------------------------------------------------------- restated dispatch (knn.cuh)
def brute_end(n, d, end_search_at):
    """knn_brute_end: first query of the cell-list search"""
    if d > 3 or end_search_at + 1 <= 4096:
        return n
    return min(n, 4096)


def grid_setup(coords):
    """knn_grid_setup: (g[3], h, ncell). Axes thinner than the cell edge are single slabs."""
    n, d = coords.shape
    lo, hi = coords.min(0), coords.max(0)
    sliced = [bool(hi[k] > lo[k]) for k in range(d)]
    target = max(1.0, n / 8.0)
    while True:
        vol, active = 1.0, 0
        for k in range(d):
            if sliced[k]:
                vol *= float(hi[k] - lo[k])
                active += 1
        h = math.pow(vol / target, 1.0 / active) if active else 1.0
        if not h > 0.:
            h = 1.0
        dropped = [k for k in range(d) if sliced[k] and float(hi[k] - lo[k]) < h]
        for k in dropped:
            sliced[k] = False
        if not dropped:
            break
    g = [1, 1, 1]
    for k in range(d):
        if sliced[k]:
            g[k] = max(int(min(math.ceil(float(hi[k] - lo[k]) / h), 1 << 20)), 1)
    return g, h, g[0] * g[1] * g[2]


def ks_of(m):
    return 1 if m <= 32 else 2


# ---------------------------------------------------------------------------------------------- cases
# (kind, data, n, np, d, m, ordering, replay): kind "model" (n points) or "pred" (n observed + np prediction points, m =
# num_neighbors_pred before the clip); replay = whether the reference makes some query risky (checked without a GPU below).
MODEL_CASES = []
for m in (1, 2, 31, 32, 33, 59, 60):  # n = 2, m + 1, m + 2 at every KS edge
    MODEL_CASES += [("model", "unif", 2, 0, 2, m, "random", False), ("model", "unif", m + 1, 0, 2, m, "random", False),
                    ("model", "unif", m + 2, 0, 2, m, "none", False)]
MODEL_CASES += [
    ("model", "unif", 33, 0, 3, 5, "random", False),
    ("model", "unif", 66, 0, 2, 2, "random", False),  # brute chunks of 32, 33, 64 and 65 candidates
    ("model", "unif", 66, 0, 1, 31, "none", False),
    ("model", "unif", 4096, 0, 2, 30, "random", False),  # brute / grid switch: 4097 candidates make the grid run
    ("model", "unif", 4097, 0, 2, 10, "random", False),
    ("model", "unif", 4098, 0, 2, 10, "random", False),
    ("model", "unif", 4099, 0, 3, 33, "random", False),
    ("model", "lat2_30", 900, 0, 2, 12, "random", True),  # brute force behind the replay
    ("model", "lat2_40", 1600, 0, 2, 48, "random", True),
    ("model", "unif", 20000, 0, 4, 20, "random", False),  # d > 3: brute force at every size
    ("model", "unif", 6000, 0, 5, 40, "none", False),
    ("model", "unif", 3000, 0, 10, 60, "random", False),
    ("model", "lat1", 10000, 0, 1, 10, "random", False),  # grid d = 1
    ("model", "unif", 8000, 0, 1, 40, "random", False),
    ("model", "unif", 20000, 0, 2, 20, "random", False),  # grid d = 2
    ("model", "unif", 10000, 0, 2, 45, "none", False),
    ("model", "lat2_65", 4225, 0, 2, 12, "random", True),
    ("model", "lat2_100", 10000, 0, 2, 48, "none", True),
    ("model", "lat2_100", 10000, 0, 2, 20, "random", True),
    ("model", "unif", 10000, 0, 3, 15, "random", False),  # grid d = 3
    ("model", "unif", 8000, 0, 3, 50, "none", False),
    ("model", "lat3_17", 4913, 0, 3, 26, "random", True),
    ("model", "lat3_17", 4913, 0, 3, 45, "random", True),
    ("model", "dup2", 6000, 0, 2, 10, "random", False),  # duplicates, one cell of > 1000 coincident points
    ("model", "dup3", 6000, 0, 3, 33, "random", False),
    ("model", "xconst", 6000, 0, 2, 15, "random", False),  # degenerate axes
    ("model", "zconst", 6000, 0, 3, 40, "random", False),
    ("model", "off_lat2_70", 4900, 0, 2, 20, "random", True),  # offset by 1e6
    ("model", "off_lat3_17", 4913, 0, 3, 10, "random", True),
    ("model", "flat_1e-3", 5000, 0, 3, 10, "random", False),  # nearly flat 3-D clouds
    ("model", "flat_1e-6", 5000, 0, 3, 10, "random", False),
    ("model", "flat_1e-9", 5000, 0, 3, 10, "random", False),
    ("model", "flat_1e-12", 5000, 0, 3, 10, "random", False),
    ("model", "unif", 100000, 0, 2, 20, "random", None),  # oracle walk only
    ("model", "unif", 100000, 0, 3, 33, "random", None),
]
PRED_CASES = [
    ("pred", "unif", 1, 3, 2, 5, "random", False),  # m clipped to n_obs
    ("pred", "unif", 5, 33, 2, 5, "random", False),  # num_neighbors_pred = n_obs: only the first query is in index order
    ("pred", "unif", 59, 31, 2, 59, "random", False),
    ("pred", "unif", 60, 32, 3, 60, "none", False),
    ("pred", "unif", 61, 1, 2, 60, "random", False),
    ("pred", "unif", 60, 33, 2, 31, "random", False),
    ("pred", "unif", 59, 32, 1, 33, "random", False),
    ("pred", "unif", 32, 8, 2, 10, "random", False),  # brute chunks of 32, 33, 64 and 65 candidates
    ("pred", "unif", 33, 8, 2, 10, "random", False),
    ("pred", "unif", 64, 8, 2, 10, "random", False),
    ("pred", "unif", 65, 8, 2, 10, "random", False),
    ("pred", "unif", 4096, 31, 2, 30, "random", False),  # last size with brute force only
    ("pred", "unif", 4097, 33, 2, 40, "random", False),  # first size on the grid
    ("pred", "lat2_30", 900, 200, 2, 12, "random", True),  # lattice midpoints: ties at the m-th distance
    ("pred", "lat2_30", 900, 200, 2, 40, "none", True),
    ("pred", "unif", 5000, 200, 1, 10, "random", False),  # grid d = 1
    ("pred", "lat1", 5000, 200, 1, 40, "random", False),
    ("pred", "unif", 20000, 500, 2, 20, "random", False),  # grid d = 2
    ("pred", "unif", 8000, 300, 2, 45, "none", False),
    ("pred", "lat2_65", 4225, 300, 2, 12, "random", True),
    ("pred", "lat2_100", 10000, 300, 2, 40, "random", True),
    ("pred", "out2", 6000, 400, 2, 20, "random", False),  # out of the observed box, and on observed points
    ("pred", "unif", 6000, 200, 3, 15, "random", False),  # grid d = 3
    ("pred", "unif", 6000, 200, 3, 50, "random", False),
    ("pred", "lat3_17", 4913, 300, 3, 7, "random", True),
    ("pred", "lat3_17", 4913, 300, 3, 45, "none", True),
    ("pred", "out3", 6000, 300, 3, 33, "random", False),
    ("pred", "unif", 6000, 200, 5, 20, "random", False),  # d > 3
    ("pred", "unif", 50000, 1000, 2, 30, "random", None),  # oracle walk only
]
CASES = MODEL_CASES + PRED_CASES


def case_id(c):
    kind, data, n, npred, d, m, order, _ = c
    return "%s-%s-d%d-n%d%s-m%d-%s" % (kind, data, d, n, "+%d" % npred if kind == "pred" else "", m, order)


def _lattice(k, d):
    g = np.arange(k) / k
    return np.stack([a.ravel() for a in np.meshgrid(*([g] * d), indexing="ij")], axis=1)


def _data(name, n, d, rng):
    if name == "unif":
        return rng.random((n, d))
    if name == "lat1":
        return np.arange(n, dtype=np.float64)[:, None]
    if name.startswith("lat2_") or name.startswith("lat3_"):
        c = _lattice(int(name[5:]), int(name[3]))
        assert c.shape == (n, d)
        return c
    if name.startswith("off_"):
        return _data(name[4:], n, d, rng) + 1e6
    if name in ("dup2", "dup3"):
        base = rng.random((n - 2000, d))
        return np.concatenate([base, base[:800], np.tile(base[7], (1200, 1))])[rng.permutation(n)]
    if name == "xconst":
        return np.stack([np.full(n, 0.5), rng.random(n)], axis=1)
    if name == "zconst":
        return np.concatenate([rng.random((n, 2)), np.full((n, 1), 0.25)], axis=1)
    if name.startswith("flat_"):
        return rng.random((n, 3)) * np.array([1., 1., float(name[5:])])
    if name in ("out2", "out3"):
        return rng.random((n, d))
    raise ValueError(name)


def _pred_points(c, obs, rng):
    kind, data, n, npred, d, m, order, _ = c
    if data == "lat1":  # midpoints between lattice points
        return rng.integers(0, n - 1, size=(npred, 1)) + 0.5
    if data.startswith("lat"):  # cell midpoints of the lattice: ties at the m-th distance
        k = int(data[5:])
        return (rng.integers(0, k - 1, size=(npred, d)) + 0.5) / k
    if data in ("out2", "out3"):  # a third outside the observed box, a third on observed points
        a, b = npred // 3, npred // 3
        return np.concatenate([rng.random((a, d)) * 1.6 - 0.3, obs[rng.integers(0, n, size=b)], rng.random((npred - a - b, d))])
    return rng.random((npred, d))


@functools.lru_cache(maxsize=None)
def points_of(c):
    """(coords in search order, q_begin, end_search_at, m clipped, perm of the observed points)"""
    kind, data, n, npred, d, m, order, _ = c
    rng = np.random.default_rng(sum(map(ord, case_id(c))))
    obs = _data(data, n, d, rng)
    perm = ov.random_order(n, 7) if order == "random" else np.arange(n, dtype=np.int32)
    obs = np.ascontiguousarray(obs[perm])
    if kind == "model":
        return obs, 0, n - 2, min(m, n - 1), perm
    allp = np.ascontiguousarray(np.concatenate([obs, _pred_points(c, obs, rng)]))
    return allp, n, n - 1, min(m, n), perm


def csums(X):
    s = np.zeros(X.shape[0])
    for k in range(X.shape[1]):
        s = s + X[:, k]
    return s


@functools.lru_cache(maxsize=None)
def brute_reference(c):
    """(b) and (c): (nn rows for the queries, risky flag per query). Rows i <= m take the predecessors in index order."""
    X, q0, esa, m, _ = points_of(c)
    n, d = X.shape
    cs = csums(X)
    pos = np.empty(n, dtype=np.int64)
    pos[ov.sort_indices(cs)] = np.arange(n)
    nn = np.full((n - q0, m), -1, dtype=np.int32)
    risky = np.zeros(n - q0, dtype=bool)
    ncand_max = esa + 1
    for i in range(q0, min(n, m + 1)):
        k = min(i, ncand_max)
        nn[i - q0, :k] = np.arange(k)
    first = max(q0, m + 1)
    chunk = max(1, (1 << 22) // max(ncand_max, 1))
    for a in range(first, n, chunk):
        b = min(n, a + chunk)
        nc = min(b - 1, ncand_max)
        s = np.zeros((b - a, nc))
        for k in range(d):
            t = X[None, :nc, k] - X[a:b, None, k]
            s = s + t * t
        q = np.arange(a, b)
        s[np.arange(nc)[None, :] >= np.minimum(q, ncand_max)[:, None]] = np.inf
        T = np.partition(s, m - 1, axis=1)[:, m - 1]
        for r, i in enumerate(q):
            idx = np.flatnonzero(s[r] <= T[r])
            rk = 2 * np.abs(pos[idx] - pos[i]) + (pos[idx] > pos[i])
            top = idx[np.lexsort((rk, s[r, idx]))[:m]]
            nn[i - q0] = top
            dd = cs[top] - cs[i]
            risky[i - q0] = bool(np.any(dd * dd > float(d) * T[r]))
    return nn, risky


def buckets_of(c, risky_any):
    """(path, KS, kind, replay) buckets a case reaches; path "brute" or "grid<d>"."""
    kind, data, n, npred, d, m, order, _ = c
    X, q0, esa, mc, _ = points_of(c)
    be = brute_end(X.shape[0], d, esa)
    paths = []
    if be > q0:
        paths.append("brute")
    if be < X.shape[0]:
        paths.append("grid%d" % d)
    return {(p, ks_of(mc), kind, bool(risky_any)) for p in paths}


REQUIRED_BUCKETS = {(p, ks, kind, rep) for p in ("brute", "grid1", "grid2", "grid3") for ks in (1, 2) for kind in ("model", "pred")
                    for rep in (False, True) if not (p == "grid1" and rep)}


# ---------------------------------------------------------------------------------------------- CPU-only checks
def test_cases_reach_every_bucket_and_edge():
    got = set()
    for c in CASES:
        if c[7] is not None:
            got |= buckets_of(c, c[7])
    assert REQUIRED_BUCKETS <= got, sorted(REQUIRED_BUCKETS - got)
    model_n = {c[2] for c in MODEL_CASES}
    assert {2, 33, 4096, 4097, 4098, 4099} <= model_n
    assert {m + 1 for m in (1, 2, 31, 32, 33, 59, 60)} <= model_n and {m + 2 for m in (1, 2, 31, 32, 33, 59, 60)} <= model_n
    assert {1, 5, 59, 60, 61, 4096, 4097} <= {c[2] for c in PRED_CASES}
    assert {1, 31, 32, 33} <= {c[3] for c in PRED_CASES}
    assert {1, 2, 31, 32, 33, 59, 60} <= {c[5] for c in CASES}
    # num_neighbors_pred = n_obs with at least three prediction points (rows after the first take the walk)
    assert {5, 59, 60} <= {c[2] for c in PRED_CASES if c[5] == c[2] and c[3] >= 3}
    assert {4, 5, 10} <= {c[4] for c in CASES}
    # brute-force chunks whose candidate count is 32, 33, 64 or 65, behind the index-order rows
    for k in (32, 33, 64, 65):
        assert any(brute_end(points_of(c)[0].shape[0], c[4], points_of(c)[2]) > k and
                   ((c[0] == "model" and c[2] > k > points_of(c)[3]) or (c[0] == "pred" and c[2] == k and c[5] < k))
                   for c in CASES), k
    # the switch: 4097 points are all brute force, 4098 put one query on the grid
    assert brute_end(4097, 2, 4095) == 4097 and brute_end(4098, 2, 4096) == 4096
    assert brute_end(4096 + 1 + 5, 2, 4096) == 4096 and brute_end(20000, 4, 19998) == 20000
    assert {o for c in CASES for o in [c[6]]} == {"random", "none"}


def test_restated_grid_sizing():
    rng = np.random.default_rng(0)
    # unchanged where no axis is thin: the benchmark's 2-D uniform workload, one cell edge h = sqrt(area / (n / 8))
    X = rng.random((200000, 2))
    g, h, ncell = grid_setup(X)
    ext = X.max(0) - X.min(0)
    h0 = math.pow(float(ext[0]) * float(ext[1]) / 25000.0, 0.5)
    assert h == h0 and g[:2] == [math.ceil(float(ext[0]) / h0), math.ceil(float(ext[1]) / h0)] and g[2] == 1
    # a thin axis becomes one slab, and h comes from the other two
    for eps in (1e-3, 1e-6, 1e-9, 1e-12):
        Y = rng.random((5000, 3)) * np.array([1., 1., eps])
        g, h, ncell = grid_setup(Y)
        assert g[2] == 1 and ncell <= 4 * 5000 / 8 and h > 1e-2, (eps, g, h)
    # a zero-extent axis as well
    assert grid_setup(np.stack([np.full(5000, 3.), rng.random(5000)], 1))[0][0] == 1


def _ring_cells(d, r):
    if d == 1:
        return 2 * r + 1
    if d == 2:
        return 1 if r == 0 else 8 * r
    return (2 * r + 1) ** 3


@pytest.mark.parametrize("c", [c for c in CASES], ids=case_id)
def test_grid_is_small_and_the_ring_walk_short(c):
    """At most 2^d n / 8 cells, and a bound on the rings each grid query walks: the m-th distance among the candidates every grid
    query has (the first brute_end points, or all observed points) over the cell edge."""
    from scipy.spatial import cKDTree
    X, q0, esa, m, _ = points_of(c)
    n, d = X.shape
    be = brute_end(n, d, esa)
    if be >= n:
        return
    g, h, ncell = grid_setup(X)
    assert ncell <= 2 ** d * max(1., n / 8.), (g, ncell)
    base = X[:min(be, esa + 1)]
    queries = X[max(be, q0):]
    dist = cKDTree(base).query(queries, k=m)[0]
    dist = dist if dist.ndim == 1 else dist[:, -1]
    r = np.minimum(np.floor(dist / (h * (1. - 1e-9))).astype(np.int64) + 1, max(g))
    cum = np.cumsum([_ring_cells(d, rr) for rr in range(int(r.max()) + 1)])
    work = int(cum[r].sum())  # cells the grid kernel enumerates over all queries
    assert r.max() <= 40 and work <= 5e8, (int(r.max()), work)


@pytest.mark.parametrize("c", [c for c in CASES if c[7] is not None], ids=case_id)
def test_declared_replay_holds_for_the_reference(c):
    """The brute force (b) agrees with the oracle's walk on every query that is not risky, and the case makes some query risky
    exactly when it says so (lattices and offsets do, so the replay runs behind both the brute force and the grid)."""
    X, q0, esa, m, _ = points_of(c)
    assert X.shape[0] <= BRUTE_REF_MAX_N + 1000
    nn_b, risky = brute_reference(c)
    nn_a = ov.knn_range(X, c[5], q0, esa)
    assert np.array_equal(nn_a[~risky], nn_b[~risky])
    assert bool(risky.any()) == c[7], int(risky.sum())


def test_oracle_walk_generalises_the_model_search():
    X = np.random.default_rng(3).random((700, 2))
    assert np.array_equal(ov.knn_range(X, 15, 0, 698), ov.knn(X, 15))
    # prediction: the first query takes all observed points in index order only when m = n_obs; the others are in distance order
    nb = ov.knn_range(X[:60], 5, 5, 4)
    assert np.array_equal(nb[0], np.arange(5))
    d = ((X[:5, None, :] - X[None, 6:60, :]) ** 2).sum(-1)
    assert np.array_equal(nb[1:], np.argsort(d.T, axis=1, kind="stable"))
    assert ov.knn_range(X[:10], 9, 3, 2).shape == (7, 3)


def test_entry_refusals(product_lib):
    lib = product_lib
    lib.gpbdev_last_error.restype = C.c_char_p
    X = np.random.default_rng(1).random((50, 2))
    nn = np.empty((50, 60), dtype=np.int32)
    info = np.empty(7, dtype=np.int64)

    def call(coords=X, n=50, d=2, m=5, q0=0, esa=48, out=nn, inf=info):
        return lib.gpbdev_knn_search(0, P(coords) if coords is not None else None, C.c_int64(n), d, m, C.c_int64(q0),
                                     C.c_int64(esa), P(out, C.c_int32) if out is not None else None,
                                     P(inf, C.c_int64) if inf is not None else None)

    for kw, msg in [(dict(coords=None), "null"), (dict(out=None), "null"), (dict(inf=None), "null"), (dict(d=0), "dim"),
                    (dict(m=0), "num_neighbors"), (dict(m=61), "num_neighbors"), (dict(q0=-1, esa=-2), "q_begin"),
                    (dict(q0=50, esa=49), "q_begin"), (dict(esa=47), "end_search_at"), (dict(q0=20, esa=20), "end_search_at"),
                    (dict(q0=20, esa=48), "end_search_at"), (dict(n=1, esa=-1), "n >= 2")]:
        assert call(**kw) != 0, kw
        assert msg in lib.gpbdev_last_error().decode(), (kw, lib.gpbdev_last_error())


# ---------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    product_lib.gpbdev_last_error.restype = C.c_char_p
    return product_lib


def chk(lib, rc):
    assert rc == 0, lib.gpbdev_last_error().decode()


def search(lib, X, m, q0, esa):
    n, d = X.shape
    mc = min(m, esa + 1)
    nn = np.full((n - q0, mc), -7, dtype=np.int32)
    info = np.zeros(7, dtype=np.int64)
    chk(lib, lib.gpbdev_knn_search(0, P(X), C.c_int64(n), d, m, C.c_int64(q0), C.c_int64(esa), P(nn, C.c_int32), P(info, C.c_int64)))
    return nn, info


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_device_search_matches_the_reference(lib, c):
    kind, data, n, npred, d, m, order, replay = c
    X, q0, esa, mc, perm = points_of(c)
    na = X.shape[0]
    nn, info = search(lib, X, m, q0, esa)
    nn2, info2 = search(lib, X, m, q0, esa)
    assert np.array_equal(nn, nn2) and np.array_equal(info, info2), "a repeated search differs"
    # what ran: the restated dispatch
    be = brute_end(na, d, esa)
    assert info[2] == be
    launches = int(be > q0) + 1
    if be < na:
        g, h, ncell = grid_setup(X)
        assert list(info[4:7]) == g and info[3] == ncell
        launches += 7
    else:
        assert info[3] == 0
    assert info[1] == launches
    # (a) the reference's walk
    want = ov.knn_range(X, m, q0, esa)
    bad = np.flatnonzero((nn != want).any(1))
    assert bad.size == 0, "%d rows differ from the walk, first query %d: %s vs %s" % (
        bad.size, bad[0] + q0, nn[bad[0]].tolist(), want[bad[0]].tolist())
    if replay is not None:
        # (b) the brute force on every query that is not risky, (c) the replay count
        nn_b, risky = brute_reference(c)
        assert np.array_equal(nn[~risky], nn_b[~risky])
        assert info[0] == int(risky.sum())
        assert (info[0] > 0) == replay
    if kind == "model":
        h = C.c_void_p()
        chk(lib, lib.gpbdev_vecchia_create(C.byref(h), 0, C.c_int64(n), d, mc, P(X), P(np.arange(n, dtype=np.int32), C.c_int32),
                                           None, C.c_int64(0), C.c_int64(n)))
        try:
            got = np.empty((n, mc), dtype=np.int32)
            chk(lib, lib.gpbdev_vecchia_get_nn(h, P(got, C.c_int32)))
            assert np.array_equal(got, nn)
            assert lib.gpbdev_vecchia_knn_replayed(h) == info[0]
        finally:
            lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
def test_prediction_on_a_tied_lattice_end_to_end():
    """GPModel.predict at lattice midpoints (distance ties at the m-th neighbour) against the oracle with the reference's walk,
    the observed points in the model's Vecchia order."""
    from gpboost_b200 import GPModel
    X = datagen.lattice(30)
    y = np.random.default_rng(4).standard_normal(X.shape[0])
    Xp = (np.random.default_rng(5).integers(0, 29, size=(150, 2)) + 0.5) / 30
    cp = np.array([0.3, 1.2, 0.1])
    mdl = GPModel(gp_coords=X, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=10,
                  vecchia_ordering="random", seed=3)
    perm = ov.random_order(X.shape[0], 3)
    for nnp in (12, 20, 40):
        r = mdl.predict(y, Xp, cp, predict_var=True, predict_response=False, num_neighbors_pred=nnp)
        mu, var = op.predict_gaussian(X[perm], y[perm], Xp, cp, "matern", 1.5, 10, predict_response=False, num_neighbors_pred=nnp)
        assert np.abs(r["mu"] - mu).max() <= 1e-8 * np.abs(mu).max(), nnp
        assert np.abs(r["var"] - var).max() <= 1e-8 * np.abs(var).max(), nnp


@pytest.mark.gpu
def test_prediction_on_the_grid_path_end_to_end():
    """20 000 observed points: the prediction queries run on the cell grid with q_begin > 0"""
    from gpboost_b200 import GPModel
    X, y = datagen.synth(20000, 2, 8)
    Xp = np.concatenate([np.random.default_rng(6).random((200, 2)), X[:20]])
    cp = np.array([0.25, 1.0, 0.08])
    mdl = GPModel(gp_coords=X, cov_function="exponential", cov_fct_shape=0.5, gp_approx="vecchia", num_neighbors=15,
                  vecchia_ordering="random", seed=2)
    r = mdl.predict(y, Xp, cp, predict_var=True, predict_response=True)
    mu, var = op.predict_gaussian(X, y, Xp, cp, "exponential", 0.5, 15, predict_response=True)
    assert np.abs(r["mu"] - mu).max() <= 1e-8 * np.abs(mu).max()
    assert np.abs(r["var"] - var).max() <= 1e-8 * np.abs(var).max()
