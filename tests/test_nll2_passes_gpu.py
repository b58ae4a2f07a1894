"""The likelihood pass (vecchia_nll2_kernel<COV, MODE_NLL>) and the store pass (MODE_STORE) of the two-observation kernel share
the pair-covariance stage and the elimination: every pair value is formed by the same expressions and written to the same matrix
slot at a lane-affine address, and the factorisation runs in the same order. Their likelihood sums must agree bit for bit.

The cases reach what that addressing has to get right beyond the headline run:
  * every covariance type at every neighbour count the kernel serves (m = 21 ... 30);
  * n odd, and row shards with an odd number of rows: the last pair of a warp is half real;
  * warps whose first pair has dummy slots (rows i < m) and whose next pair has none, and supplied neighbour sets padded with -1
    at rows i >= m: the keep masks that zero the pairs of dummy slots, with partners that wrap around the circulant schedule.
n is large enough that every warp of the persistent grid runs several pairs."""
import ctypes as C

import numpy as np
import pytest

COVS = {"exponential": 0, "matern1.5": 1, "matern2.5": 2, "gaussian": 3}
MODE_NLL, MODE_STORE = 0, 1
N = 20001


def P(a, t=C.c_double):
    return a.ctypes.data_as(C.POINTER(t))


@pytest.fixture(scope="module")
def lib(product_lib):
    assert product_lib.gpbdev_device_count() > 0, "no CUDA device visible — GPU tests need an H100"
    return product_lib


def chk(lib, rc):
    assert rc == 0, lib.gpbdev_last_error().decode()


def engine(lib, coords, y, m, nn=None, rows=None):
    n = coords.shape[0]
    lo, hi = rows if rows is not None else (0, n)
    h = C.c_void_p()
    c = np.ascontiguousarray(coords)
    perm = np.arange(n, dtype=np.int32)
    nnp = None if nn is None else P(np.ascontiguousarray(nn, dtype=np.int32), C.c_int32)
    chk(lib, lib.gpbdev_vecchia_create(C.byref(h), 0, C.c_int64(n), 2, m, P(c), P(perm, C.c_int32), nnp, C.c_int64(lo), C.c_int64(hi)))
    chk(lib, lib.gpbdev_vecchia_set_y(h, P(np.ascontiguousarray(y))))
    return h


def sums(lib, h, cov, mode, var, rng):
    out = np.zeros(9)
    chk(lib, lib.gpbdev_vecchia_eval(h, cov, C.c_double(var), C.c_double(rng), mode, P(out)))
    return out


def data(seed=5):
    r = np.random.default_rng(seed)
    return r.random((N, 2)), r.standard_normal(N)


def range_for(cov):
    # neighbour distances ~ 0.01 at n = 2e4: covariances between neighbours neither ~1 nor ~0
    return 30. if cov != "gaussian" else 900.


def assert_nll_equals_store(lib, h, cov):
    a = sums(lib, h, COVS[cov], MODE_NLL, 1.7, range_for(cov))
    b = sums(lib, h, COVS[cov], MODE_STORE, 1.7, range_for(cov))
    assert np.isfinite(a[:3]).all() and a[1] != 0.
    assert a[:3].tobytes() == b[:3].tobytes(), (a[:3], b[:3])


@pytest.mark.gpu
@pytest.mark.parametrize("m", list(range(21, 31)))
@pytest.mark.parametrize("cov", list(COVS))
def test_nll_pass_equals_store_pass(lib, cov, m):
    coords, y = data()
    h = engine(lib, coords, y, m)
    try:
        assert_nll_equals_store(lib, h, cov)
    finally:
        lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [(0, 10001), (3, 10004), (10001, N), (N - 4001, N)])
@pytest.mark.parametrize("cov", ["matern1.5", "gaussian"])
def test_row_shards_with_a_half_real_last_pair(lib, cov, rows):
    coords, y = data()
    h = engine(lib, coords, y, 30, rows=rows)
    try:
        assert_nll_equals_store(lib, h, cov)
    finally:
        lib.gpbdev_vecchia_free(h)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [21, 30])
@pytest.mark.parametrize("cov", list(COVS))
def test_supplied_sets_padded_beyond_row_m(lib, cov, m):
    """Rows i >= m with dummy slots scattered over the run: a warp's next pair is sometimes not free of dummy slots while the
    current one is, and the other way round."""
    coords, y = data()
    h0 = engine(lib, coords, y, m)
    nn = np.zeros((N, m), dtype=np.int32)
    chk(lib, lib.gpbdev_vecchia_get_nn(h0, P(nn, C.c_int32)))
    lib.gpbdev_vecchia_free(h0)
    r = np.random.default_rng(11)
    rows = r.choice(np.arange(m, N), size=N // 7, replace=False)
    for i in rows:
        nn[i, r.integers(1, m):] = -1  # keep at least one neighbour, pad the tail
    h = engine(lib, coords, y, m, nn=nn)
    try:
        assert_nll_equals_store(lib, h, cov)
    finally:
        lib.gpbdev_vecchia_free(h)
