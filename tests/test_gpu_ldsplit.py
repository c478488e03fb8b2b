"""snp_ldsplit, get_L and get_C on the device against the CPU oracle (tests/ldsplit_oracle.c, tests/ldsplit_ref.py): C
(with +Inf), best_ind (with NA), the get_L triplets and the whole result table byte for byte."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import bigsnpr_b200 as B
from bigsnpr_b200 import _lib, api
from tests import ldsplit_ref as R
from tests.test_ldsplit_oracle import outer4, spmat

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
INF = np.inf


def lower_of(A):
    return api.ldsplit_lower(sp.csc_matrix(A))


def same_table(got, want):
    if want is None:
        assert got is None
        return
    assert got is not None
    for k in ("max_size", "n_block"):
        assert np.array_equal(got[k], want[k]), k
    for k in ("cost", "cost2", "perc_kept"):
        assert got[k].tobytes() == np.asarray(want[k], dtype=np.float64).tobytes(), k
    assert len(got["all_last"]) == len(want["all_last"])
    for a, b, c, d in zip(got["all_last"], want["all_last"], got["all_size"], want["all_size"]):
        assert np.array_equal(a, b) and np.array_equal(c, d)


def check_split(low, thr_r2, min_size, max_size, handle=None, **kw):
    want = R.snp_ldsplit(low, thr_r2, min_size, max_size, **kw)
    h = handle or api.LDCorr(sp.csc_matrix((low[2], low[1], low[0])), upper=False)
    try:
        got = api.snp_ldsplit(h, thr_r2, min_size, max_size, **kw)
    finally:
        if handle is None:
            h.close()
    same_table(got, want)
    return got


def check_get_C(low, thr_r2, max_r2, min_size, max_size, max_K, max_cost, pos):
    m = len(low[0]) - 1
    L = R.L_csc(R.get_L(low, thr_r2, max_r2), m)
    Cw, bw = R.get_C(L, m, min_size, max_size, max_K, max_cost, pos)
    got = api.get_C(sp.csc_matrix((L[2], L[1], L[0]), shape=(m, m + 1)), min_size, max_size, max_K, max_cost, pos)
    assert got["C"].tobytes() == Cw.tobytes() and np.array_equal(got["best_ind"], bw)
    return got


def check_get_L(low, thr_r2, max_r2):
    want = R.get_L(low, thr_r2, max_r2)
    got = api.get_L(low[0], low[1], low[2], thr_r2, max_r2)
    for k, w in zip("ijx", want):
        assert got[k].tobytes() == w.tobytes(), k
    return got


def test_outer4_cases():
    low = lower_of(outer4())
    check_get_L(low, 0, 1)
    got = check_get_C(low, 0, 1, 1, 4, 5, INF, np.zeros(4))
    assert np.isinf(got["C"][:, 4]).all() and (got["best_ind"][:, 4] == api.NA_INTEGER).all()
    check_get_C(low, 0, 1, 2, 2, 3, INF, np.ones(4))
    check_get_C(low, 0, 1, 1, 3, 3, INF, np.linspace(0, 1, 4))
    check_get_C(low, 0, 1, 1, 3, 4, INF, np.arange(1, 5) * 2.0)
    # max_size == m: the block ending at the last SNP never wins a layer k >= 1
    got = check_get_C(low, 0, 1, 1, 4, 4, INF, np.zeros(4))
    assert not np.any(got["best_ind"][:, 1:] == 4)
    assert check_split(low, 0, 1, 3, max_K=3, max_r2=1, max_cost=INF, pos_scaled=np.arange(1, 5) * 2.0) is None
    check_split(low, 0, 1, 3, max_K=4, max_r2=1, max_cost=INF, pos_scaled=np.arange(1, 5) * 2.0)
    t = check_split(low, 0, 1, 2, max_K=4, max_r2=1, max_cost=INF)
    assert np.array_equal(t["perc_kept"], np.array([8, 6, 4]) / 16)


@pytest.fixture(scope="module")
def spm():
    A, _, _ = spmat()
    return lower_of(A + sp.triu(A, 1).T)


def test_spmat_reference_parameter_sets(spm):
    check_get_L(spm, 0.02, 1)
    check_get_L(spm, 0.02, 0.25)
    t = check_split(spm, 0.02, 10, 30, max_K=50, max_r2=1, max_cost=INF)
    assert np.array_equal(t["n_block"], np.arange(14, 41))
    check_split(spm, 0.1, 20, 40, max_K=50, max_r2=1, max_cost=INF)
    check_split(spm, 0.05, 20, 40, max_K=15, max_r2=1, max_cost=INF)
    check_split(spm, 0.02, 10, 30, max_K=50, max_r2=1, max_cost=float(np.median(t["cost"])))
    check_split(spm, 0.02, 10, 50, max_K=100, max_r2=0.25, max_cost=INF)
    check_split(spm, 0.02, 10, [40, 30, 30, 12, 401], max_K=50, max_r2=0.6, max_cost=INF)  # unsorted, repeated, == m
    check_split(spm, 0, 10, 30, max_K=50)  # thr_r2 = 0, default max_r2 and max_cost
    check_split(spm, 0.02, 20, 20, max_K=30, max_r2=1, max_cost=INF)  # min_size == max_size
    pos = np.arange(401) / 40.0  # a block spans at most 40 SNPs
    check_split(spm, 0.02, 10, [30, 60], max_K=50, max_r2=1, max_cost=INF, pos_scaled=pos)
    check_get_C(spm, 0.02, 1, 10, 60, 50, INF, pos)
    got = check_get_C(spm, 0.02, 0.1, 5, 401, 120, INF, np.zeros(401))  # max_r2 gives +Inf entries
    assert np.isinf(got["C"]).any()
    assert check_split(spm, 0.02, 200, 200, max_K=10, max_r2=1, max_cost=INF) is None  # 401 is not a multiple of 200


def test_max_cost_stops_at_several_layers(spm):
    layers = []
    full = R.snp_ldsplit(spm, 0.02, 10, 30, max_K=50, max_r2=1, max_cost=INF)
    for q in (0.1, 0.5, 0.9):
        mc = float(np.quantile(full["cost"], q))
        nl = []
        R.snp_ldsplit(spm, 0.02, 10, 30, max_K=50, max_r2=1, max_cost=mc, layers=nl)
        h = api.LDCorr(sp.csc_matrix((spm[2], spm[1], spm[0])), upper=False)
        got, lay, secs = h.split(0.02, 10, 30, max_K=50, max_r2=1, max_cost=mc)
        h.close()
        same_table(got, R.snp_ldsplit(spm, 0.02, 10, 30, max_K=50, max_r2=1, max_cost=mc))
        assert list(lay) == nl and nl[0] < 50
        layers.append(nl[0])
    assert len(set(layers)) == 3


def bed_corr(name):
    g = B.Bed(os.path.join(GOLD, name), device=0)
    G = B.read_bed(g, g.rows_along(), g.cols_along(), na_val=3)
    poly = (np.flatnonzero(np.nanstd(np.where(G == 3, np.nan, G), 0) > 0) + 1).astype(np.int32)
    corr = B.bed_cor(g, ind_col=poly, size=500)
    g.close()
    return corr


@pytest.mark.parametrize("name", ["example.bed", "example-missing.bed"])
def test_bed_cor_matrices(name):
    corr = bed_corr(name)
    low = api.ldsplit_lower(corr)
    m = len(low[0]) - 1
    check_get_L(low, 0.02, 0.3)
    sizes = [m // 30, m // 10, m // 5]
    want = R.snp_ldsplit(low, 0.02, 10, sizes, max_K=100)
    same_table(B.snp_ldsplit(corr, 0.02, 10, sizes, max_K=100), want)


def test_synth_20000():
    n, m = 2000, 20000
    g = B.Bed.synthetic(n, m, seed=11, ld_rho=0.9, ld_block=50)
    G = B.read_bed(g, g.rows_along(), g.cols_along(), na_val=3)
    keep = (np.flatnonzero(G.std(0) > 0) + 1).astype(np.int32)
    del G
    corr = B.bed_cor(g, ind_col=keep, size=100)
    g.close()
    low = api.ldsplit_lower(corr)
    mk = len(low[0]) - 1
    h = api.LDCorr(corr)
    try:
        for thr, sizes, K in ((0.02, [500, 1000], 200), (0, [300], 100)):
            same_table(api.snp_ldsplit(h, thr, 100, sizes, max_K=K), R.snp_ldsplit(low, thr, 100, sizes, max_K=K))
    finally:
        h.close()
    assert mk > 19000


def test_two_calls_identical_and_one_handle_serves_several(spm):
    h = api.LDCorr(sp.csc_matrix((spm[2], spm[1], spm[0])), upper=False)
    try:
        a = check_split(spm, 0.02, 10, [30, 40], handle=h, max_K=50, max_r2=1, max_cost=INF)
        b = check_split(spm, 0.02, 10, [30, 40], handle=h, max_K=50, max_r2=1, max_cost=INF)
        same_table(a, b)
        check_split(spm, 0.05, 20, 40, handle=h, max_K=15, max_r2=1, max_cost=INF)
        g = h.get_L(0.02, 1)
        w = R.get_L(spm, 0.02, 1)
        assert g["x"].tobytes() == w[2].tobytes()
    finally:
        h.close()


def test_abi_errors():
    lib = _lib.lib()
    low = lower_of(outer4())
    h = api.LDCorr(sp.csc_matrix(outer4()))
    out = [np.empty(4), np.empty(4), np.empty(4)]
    kept, path, lay = np.empty(4, dtype=np.int32), np.empty(10, dtype=np.int32), np.empty(1, dtype=np.int32)

    def call(min_size, S, K, pos=np.zeros(4)):
        return lib.bsg_ldsplit(h._h, 0.0, min_size, api._pi(np.array(S, dtype=np.int32)), len(S), K, 1.0, INF, api._pd(pos),
                               api._pi(kept), *(api._pd(o) for o in out), api._pi(path), api._pi(lay), None)

    assert call(1, [2], 4) == 0
    for args in ((0, [2], 4), (1, [5], 4), (3, [2], 4), (1, [2], 0), (1, [2], 4, np.array([0, 0, np.nan, 0]))):
        assert call(*args) == 9  # BSG_ERR_ARG
    h.close()
    # an empty column, a zero on the diagonal, rows out of order
    bad = (np.array([0, 2, 2, 3, 4], dtype=np.int64), np.array([0, 1, 2, 3], dtype=np.int32), np.ones(4))
    hh = _lib.vp()
    for p, i, x in (bad, (low[0], low[1], np.where(np.arange(low[2].size) == 4, 0.0, low[2])),
                    (low[0], low[1][[0, 2, 1, 3, 4, 5, 6, 7, 8, 9]], low[2])):
        rc = lib.bsg_ldcorr_open(4, p.ctypes.data_as(_lib.c_i64_p), api._pi(np.ascontiguousarray(i)), api._pd(x), 0,
                                 _lib.C.byref(hh))
        assert rc == 9
    # E for a 300,000-SNP diagonal matrix with blocks of 1 .. m SNPs needs ~1.8e11 bytes: refused from the size alone
    m = 300000
    lp = np.zeros(m + 2, dtype=np.int64)
    C = np.empty(1)
    rc = lib.bsg_ldsplit_costs(m, lp.ctypes.data_as(_lib.c_i64_p), None, None, 1, m, 1, INF, api._pd(np.zeros(m)), 0,
                               api._pd(C), api._pi(np.empty(1, dtype=np.int32)))
    assert rc == 7 and b"needs" in lib.bsg_last_error()  # BSG_ERR_ALLOC
    with pytest.raises(_lib.BsgError):
        api.get_C(sp.csc_matrix((4, 5)), 1, 2, 0, INF, np.zeros(4))


def test_shim_entry_points_equal_the_c_abi(spm, tmp_path):
    """_bigsnpr_get_L (5 arguments) and _bigsnpr_get_C (6) through the R shim, linked against the stand-in for R's C API:
    the results equal the C ABI's; a matrix that is not a dgCMatrix is refused."""
    import ctypes as C

    from tests.test_abi import build_shim_with_minir
    from tests.test_gpu_shim import MiniR

    Rm = MiniR(build_shim_with_minir(tmp_path))
    p, i, x = spm
    m = len(p) - 1
    res = Rm.call("_bigsnpr_get_L", Rm.ints(p), Rm.ints(i), Rm.reals(x), Rm.reals([0.02]), Rm.reals([0.5]))
    want = api.get_L(p, i, x, 0.02, 0.5)
    for k in "ijx":
        assert Rm.vec(Rm.named(res, k)).tobytes() == want[k].tobytes()
    L = R.L_csc((want["i"], want["j"], want["x"]), m)
    Ls = Rm.L
    Ls.Rf_allocVector.restype, Ls.Rf_allocVector.argtypes = C.c_void_p, [C.c_uint, C.c_long]
    Ls.Rf_install.restype, Ls.Rf_install.argtypes = C.c_void_p, [C.c_char_p]
    Ls.Rf_setAttrib.restype, Ls.Rf_setAttrib.argtypes = C.c_void_p, [C.c_void_p, C.c_void_p, C.c_void_p]
    Lobj = Ls.Rf_allocVector(19, 0)
    for name, v in (("p", Rm.ints(L[0])), ("i", Rm.ints(L[1])), ("x", Rm.reals(L[2])), ("Dim", Rm.ints([m, m + 1]))):
        Ls.Rf_setAttrib(Lobj, Ls.Rf_install(name.encode()), v)
    pos = np.arange(m) / 40.0
    args = (Rm.ints([10]), Rm.ints([60]), Rm.ints([50]), Rm.reals([3.0]), Rm.reals(pos))
    with pytest.raises(RuntimeError, match="dgCMatrix"):
        Rm.call("_bigsnpr_get_C", Lobj, *args)
    Ls.Rf_setAttrib(Lobj, Ls.Rf_install(b"class"), Rm.s("dgCMatrix"))
    res = Rm.call("_bigsnpr_get_C", Lobj, *args)
    got = api.get_C(sp.csc_matrix((L[2], L[1], L[0]), shape=(m, m + 1)), 10, 60, 50, 3.0, pos)
    assert Rm.vec(Rm.named(res, "C")).tobytes(order="F") == got["C"].tobytes(order="F")
    assert np.array_equal(Rm.vec(Rm.named(res, "best_ind")), got["best_ind"])
