"""bed_cor, bed_ld_scores and the clumping pair bands on the device against tests/cor_ref.py, byte for byte.

The pair sums are exact integers and the epilogues have one rounding sequence, so every case compares bytes: p, i, x of
the CSC (NaN where the model has NaN) and the LD scores.  The cases reach the edges of the tiling: row counts around the
64-code chunks and the 512-code (identity) / 256-code (compacted) line strides; column counts and windows around the
128-column blocks and the four B tiles of a work item; empty windows, ties, non-integer positions; missing values in one
column only (a 256-row A pair with one missing-free half), in the last row, everywhere; index multisets; nonzero pad bits;
and a 1.6-million-column band that the bound on the tile sums splits into several batches.  tests/cor_ref.py's Plan
asserts which of those paths a case reaches.  Every case runs again with BSG_GRAM_TMA=0 (in-kernel expansion, k_gram5).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import cor_ref as R

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_PLINK = np.array([3, 2, 0, 1], dtype=np.uint8)  # .bed codes: g0 -> 11, g1 -> 10, g2 -> 00, NA -> 01


def pack(G, pad_codes=None):
    """.bed bytes (m x ceil(n / 4)) of G (n x m, 3 = NA); pad slots get genotype 0 unless pad_codes (0..3) says otherwise."""
    n, m = G.shape
    nb = (n + 3) // 4
    codes = np.full((4 * nb, m), 3, dtype=np.uint8)
    codes[:n] = _PLINK[G]
    if pad_codes is not None and 4 * nb > n:
        codes[n:] = np.asarray(pad_codes, dtype=np.uint8)[: 4 * nb - n, None]
    by = codes[0::4] | (codes[1::4] << 2) | (codes[2::4] << 4) | (codes[3::4] << 6)
    return np.ascontiguousarray(by.T)


def _geno(rng, n, m, na=0.0):
    G = rng.integers(0, 3, size=(n, m)).astype(np.uint8)
    # neighbours copy each other's rows in runs, so r spans the whole range and thresholds prune
    for j in range(1, m):
        cp = rng.random(n) < 0.7
        G[cp, j] = G[cp, j - 1]
    if na > 0:
        G[rng.random((n, m)) < na] = 3
    return G


# ---- the case table ---------------------------------------------------------------------------------------------------------
def _case(name, G, ir=None, ic=None, size=500, pos=None, pad=None, fbm=False, cor_kw=({},)):
    return dict(name=name, G=G, ir=ir, ic=ic, size=size, pos=pos, pad=pad, fbm=fbm, cor_kw=cor_kw)


def cases():
    out = []
    rng = np.random.default_rng(11)
    for nr in (1, 2, 3, 4, 5, 63, 64, 65, 255, 256, 257, 511, 512, 513):
        G = _geno(rng, nr, 300, na=0.01)
        out.append(_case("rows%d_identity" % nr, G, size=129))
        Gb = _geno(rng, nr + 37, 300, na=0.01)
        ir = np.sort(rng.choice(nr + 37, nr, replace=False)) + 1
        out.append(_case("rows%d_subset" % nr, Gb, ir=ir, size=129))
    for nc in (1, 2, 127, 128, 129, 255, 256, 257, 383, 384, 385, 640, 1025):
        G = _geno(rng, 97, nc)
        G[40, nc // 2] = 3  # one column block with a missing value: mixed tiles
        sizes = (1, 127, 128, 129, 511, 512, 513, 700, 10**6) if nc >= 640 else (129, 10**6)
        for w in sizes:
            out.append(_case("cols%d_win%d" % (nc, w), G, size=w, fbm=(nc == 1025 and w == 513)))
    # positions: ties at size 0, non-integer positions, gaps that leave whole row blocks without pairs
    G = _geno(rng, 150, 700, na=0.005)
    pos = np.floor(np.arange(700) / 3.0) * 1000.0
    out.append(_case("tied_size0", G, size=0, pos=pos))
    pos = np.cumsum(rng.choice([0.0, 250.5, 1000.25, 3333.3], size=700))
    out.append(_case("nonint_pos", G, size=2.7, pos=pos))
    pos = np.r_[np.arange(200) * 1000.0, 1e9 + np.arange(300) * 1e6, 2e9 + np.arange(200) * 1000.0]
    out.append(_case("gaps", G, size=150, pos=pos, fbm=True))
    # missing-value patterns on one shape
    base = _geno(rng, 300, 400)
    out.append(_case("na_none", base.copy(), size=200))
    G = base.copy()
    G[17, 300] = 3
    out.append(_case("na_single", G, size=200, fbm=True))
    G = base.copy()
    G[-1, ::7] = 3
    out.append(_case("na_last_row", G, size=200))
    G = base.copy()
    G[:, 130] = 3  # all missing: nona = 0, r NaN and kept
    G[:, 260] = 3
    G[5, 260] = 2  # one non-missing value
    G[:, 261] = 1  # constant: deno 0
    G[:, 262] = 0
    G[:, 300] = G[:, 299]  # identical and negated: r at +-1 (clamped)
    G[:, 301] = 2 - G[:, 299]
    out.append(_case("na_edges", G, size=200, fbm=True))
    out.append(_case("na_1pct", _geno(rng, 300, 400, na=0.01), size=200,
                     cor_kw=tuple(dict(alpha=a, thr_r2=t, fill_diag=f) for a in (1.0, 0.05) for t in (0.0, 0.2)
                                  for f in (True, False))))
    # index forms
    G = _geno(rng, 260, 500, na=0.01)
    out.append(_case("idx_explicit", G, ir=np.arange(1, 261), ic=np.arange(1, 501), size=150))
    out.append(_case("idx_row_subset", G, ir=rng.choice(260, 130, replace=False) + 1, size=150))
    out.append(_case("idx_col_subset", G, ic=np.sort(rng.choice(500, 300, replace=False)) + 1, size=150))
    out.append(_case("idx_multisets", G, ir=rng.integers(1, 261, 300), ic=np.sort(rng.integers(1, 501, 450)), size=150))
    out.append(_case("idx_unsorted_cols", G, ic=rng.permutation(500)[:400] + 1, size=150,
                     pos=1000.0 * np.arange(1, 401)))
    # pad bits: nonzero codes in the pad slots of each column's last byte
    for nr in (61, 130, 257):
        out.append(_case("pad_bits_%d" % nr, _geno(rng, nr, 300, na=0.01), size=100, pad=[1, 2, 1]))
    return out


def batch_case():
    """64 rows x 1,600,000 columns, one-SNP window, missing values in every column block except three isolated ones: the
    tile sums split into four batches, one boundary at an odd row block."""
    rng = np.random.default_rng(5)
    n, m = 64, 1_600_000
    G = rng.integers(0, 3, size=(n, m), dtype=np.uint8)
    G[:, 1::2] = np.where(rng.random((n, m // 2)) < 0.8, G[:, 0::2], G[:, 1::2])
    blocks = np.arange(m // R.CTN)
    na_blocks = np.setdiff1d(blocks, [10, 20, 30])
    G[rng.integers(0, n, na_blocks.size), na_blocks * R.CTN + rng.integers(0, R.CTN, na_blocks.size)] = 3
    return _case("batches_1p6M", G, size=1)


def _select(c):
    G = c["G"]
    ir = np.arange(1, G.shape[0] + 1) if c["ir"] is None else np.asarray(c["ir"])
    ic = np.arange(1, G.shape[1] + 1) if c["ic"] is None else np.asarray(c["ic"])
    return G[ir - 1][:, ic - 1]


def run_case(B, c):
    """Device results of one case: {key: array}."""
    G = c["G"]
    n, m = G.shape
    handles = [("bed", B.Bed.from_packed(pack(G, c["pad"]), n, m))]
    if c["fbm"]:
        handles.append(("fbm", B.Bed.from_fbm(G)))
    ir = ... if c["ir"] is None else np.asarray(c["ir"], dtype=np.int32)
    ic = ... if c["ic"] is None else np.asarray(c["ic"], dtype=np.int32)
    res = {}
    for hn, g in handles:
        for q, kw in enumerate(c["cor_kw"]):
            import warnings

            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                p, i, x = B.bed_cor(g, ir, ic, size=c["size"], infos_pos=c["pos"], **kw)
            res["%s_cor%d_p" % (hn, q)], res["%s_cor%d_i" % (hn, q)], res["%s_cor%d_x" % (hn, q)] = p, i, np.array(x)
        res["%s_ld" % hn] = B.bed_ld_scores(g, ir, ic, size=c["size"], infos_pos=c["pos"])
        g.close()
    return res


def model_case(c):
    G = _select(c)
    nr, nc = G.shape
    pos = 1000.0 * np.arange(1, nc + 1) if c["pos"] is None else np.asarray(c["pos"], dtype=np.float64)
    band = R.Band(pos, c["size"] * 1000.0)
    S = R.pair_sums(G, band)
    res = {}
    for q, kw in enumerate(c["cor_kw"]):
        from bigsnpr_b200.api import cor_thresholds

        thr = cor_thresholds(nr, kw.get("alpha", 1.0), kw.get("thr_r2", 0.0))
        r, keep = R.cor_epilogue(S, thr)
        res["cor%d" % q] = R.csc(band, S, r, keep, kw.get("fill_diag", True))
    res["ld"] = R.ld_reduce(band, R.ld_epilogue(S))
    return res, R.Plan(G, band), band


def _assert_same(got, want, c):
    for key in [k for k in got if k.endswith("_p")]:
        hn, q = key.split("_")[0], key.split("_")[1]
        p, i, x = want[q]
        tag = (c["name"], hn, q)
        assert np.array_equal(got[key], p), tag
        assert np.array_equal(got["%s_%s_i" % (hn, q)], i), tag
        gx = got["%s_%s_x" % (hn, q)]
        assert np.array_equal(np.isnan(gx), np.isnan(x)), tag
        ok = ~np.isnan(x)
        assert np.array_equal(gx[ok].view(np.int64), x[ok].view(np.int64)), tag
    for key in [k for k in got if k.endswith("_ld")]:
        assert np.array_equal(got[key].view(np.int64), want["ld"].view(np.int64)), (c["name"], key)


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as b
    from bigsnpr_b200 import build

    build.build()
    return b


_MODELS = {}


def _model(c):
    if c["name"] not in _MODELS:
        _MODELS[c["name"]] = model_case(c)
    return _MODELS[c["name"]]


def test_case_table_bytes(B):
    cs = cases()
    mixed = 0
    for c in cs:
        want, plan, _ = _model(c)
        mixed += len(plan.mixed_pairs()) > 0
        _assert_same(run_case(B, c), want, c)
    by = {c["name"]: c for c in cs}
    assert R.Plan(_select(by["na_single"]), R.Band(1000.0 * np.arange(1, 401), 2e5)).mixed_pairs()
    assert mixed >= 10
    assert max(_model(by["cols1025_win700"])[1].ntiles) > 4  # wider than the four B tiles of a work item
    assert (_model(by["gaps"])[1].ntiles == 0).any()  # row blocks without a tile


def test_multi_batch_band_bytes(B):
    c = batch_case()
    want, plan, band = _model(c)
    assert plan.nbatches >= 3 and plan.split_pairs(), (plan.nbatches, plan.boundaries())
    _assert_same(run_case(B, c), want, c)


def test_determinism(B):
    c = [c for c in cases() if c["name"] == "na_1pct"][0]
    a, b = run_case(B, c), run_case(B, c)
    for k in a:
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k


_GRAM5_RUN = """
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import bigsnpr_b200 as B
from tests import test_gpu_cor as T
out = {}
for c in T.cases() + [T.batch_case()]:
    for k, v in T.run_case(B, c).items():
        out[c["name"] + "/" + k] = v
np.savez(sys.argv[2], **out)
"""


def test_in_kernel_expansion_bytes(B, tmp_path):
    """The same table through k_gram5 (BSG_GRAM_TMA=0 is read once per process, hence the subprocess)."""
    res = tmp_path / "gram5.npz"
    r = subprocess.run([sys.executable, "-c", _GRAM5_RUN, ROOT, str(res)], capture_output=True, text=True,
                       env=dict(os.environ, BSG_GRAM_TMA="0"), timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(res)
    for c in cases() + [batch_case()]:
        g = {k.split("/", 1)[1]: got[k] for k in got.files if k.startswith(c["name"] + "/")}
        assert g, c["name"]
        _assert_same(g, _model(c)[0], c)


# ---- thresholds -----------------------------------------------------------------------------------------------------------
def test_cormat_threshold_equality(B):
    rng = np.random.default_rng(3)
    G = _geno(rng, 90, 6, na=0.05)
    n, m = G.shape
    g = B.Bed.from_packed(pack(G), n, m)
    pos = np.arange(1.0, m + 1)
    band = R.Band(pos, 10.0)
    S = R.pair_sums(G, band)
    r, _ = R.cor_epilogue(S, np.zeros(n))
    q = int(np.argmax(np.abs(r)))  # the strongest pair, away from the clamp
    assert 0.2 < abs(r[q]) < 1
    nona = int(S["nona"][q])
    for t, kept in ((abs(r[q]), False), (np.nextafter(abs(r[q]), 0), True)):
        thr = np.full(n, 2.0)
        thr[nona - 1] = t
        p, i, x = B.corMat(g, np.arange(1, n + 1), np.arange(1, m + 1), 10.0, thr, pos, fill_diag=False)
        col = np.repeat(np.arange(m), np.diff(p))
        hit = (col == S["j0"][q]) & (i == S["j"][q])
        assert hit.any() == kept
        pm, im, xm = R.csc(band, S, *R.cor_epilogue(S, thr), fill_diag=False)
        assert np.array_equal(p, pm) and np.array_equal(i, im) and np.array_equal(x, xm)
    g.close()


# ---- clumping kinds -------------------------------------------------------------------------------------------------------
def _bed_stats(G):
    valid = G != 3
    gv = np.where(valid, G, 0).astype(np.float64)
    cnt = valid.sum(0)
    sumX = gv.sum(0)
    with np.errstate(all="ignore"):
        center = sumX / cnt
        denoX = (gv * gv).sum(0) - sumX * sumX / cnt
    return center, np.sqrt(denoX), sumX, denoX


def _clump_model(G, center, scale, pos, size, thr, ordv):
    band = R.Band(pos, size, both=True)
    flag = R.clump_epilogue(R.pair_sums(G, band), center, scale, thr)
    return R.clump_sweep(band, flag, pos, size, ordv)


def _levels_model(G, sumX, denoX, pos, size, levels, ti, ordv, band=None, S=None):
    band = R.Band(pos, size, both=True) if band is None else band
    S = R.pair_sums(G, band) if S is None else S
    lev = R.levels_epilogue(S, G.shape[0], sumX, denoX, levels, (G == 3).any(axis=0))
    return R.clump_sweep(band, lev > ti, pos, size, ordv)


def test_clumping_kinds_against_model_sweeps(B):
    rng = np.random.default_rng(19)
    by = {c["name"]: c for c in cases()}
    for name in ("rows257_subset", "cols1025_win513", "na_edges", "nonint_pos", "idx_multisets"):
        c = by[name]
        G = _select(c)
        n, m = G.shape
        pos = 1000.0 * np.arange(1, m + 1) if c["pos"] is None else np.asarray(c["pos"], dtype=np.float64)
        if name == "idx_multisets":
            pos = np.sort(rng.uniform(0, 1e5, m))
        size = float(c["size"]) * 1000.0
        center, scale, sumX, denoX = _bed_stats(G)
        ordv = (np.argsort(-rng.random(m), kind="stable") + 1).astype(np.int32)
        g = B.Bed.from_packed(pack(G), n, m)
        for thr in (0.05, 0.2):
            k = B.bed_clumping_chr(g, np.arange(1, n + 1), np.arange(1, m + 1), center, scale, ordv, None, pos, size, thr)
            assert np.array_equal(k, _clump_model(G, center, scale, pos, size, thr, ordv)), (name, thr)
        g.close()
        f = B.Bed.from_fbm(G)
        for thr in (0.05, 0.2):
            k = B.clumping_chr(f, np.arange(1, n + 1), np.arange(1, m + 1), ordv, None, pos, sumX, denoX, size, thr)
            assert np.array_equal(k, _levels_model(G, sumX, denoX, pos, size, [thr], 0, ordv)), (name, thr)
        f.close()


def test_grid_clumping_levels_against_model(B):
    rng = np.random.default_rng(23)
    G = _geno(rng, 400, 900, na=0.0)
    G[7, 450] = 3  # missing value: level 0 for its pairs
    n, m = G.shape
    pos = np.sort(rng.uniform(0, 5e5, m)).round(1)
    lpS = rng.random(m)
    thr_r2, base = (0.01, 0.1, 0.5, 0.95), (20, 50)
    f = B.Bed.from_fbm(G)
    res = B.snp_grid_clumping(f, np.ones(m, dtype=int), pos, lpS, grid_thr_r2=thr_r2, grid_base_size=base)
    f.close()
    st = {"sumX": np.where(G == 3, 0, G).sum(0).astype(np.float64)}
    with np.errstate(all="ignore"):
        gv = np.where(G == 3, 0, G).astype(np.float64)
        st["denoX"] = (gv * gv).sum(0) - st["sumX"] ** 2 / n
    levels = np.array(thr_r2)
    sizes = [1000.0 * b / t for t in thr_r2 for b in base]
    band = R.Band(pos, max(sizes), both=True)
    S = R.pair_sums(G, band)
    ordv = (np.argsort(-lpS, kind="stable") + 1).astype(np.int32)
    want = []
    for t in thr_r2:
        for b in base:
            ti = int(np.searchsorted(levels, t))
            keep = _levels_model(G, st["sumX"], st["denoX"], pos, 1000.0 * b / t, levels, ti, ordv, band, S)
            want.append(np.flatnonzero(keep == 1) + 1)
    assert len(res) == 1 and len(res[0]) == len(want)
    for got, w in zip(res[0], want):
        assert np.array_equal(np.sort(got), w)


def _clump_r2_chains(H, center, scale):
    """r^2 of the pair (owner 1, partner 0) by the pinned chain, and by the four chains a compiler could have chosen
    instead (each of the three fused steps rounded twice, or all of them)."""
    from tests.fixedpoint_ref import fma

    S = R.pair_sums(H, R.Band(np.array([1.0, 2.0]), 10.0, both=True))
    cx, cy, xs, ys, xy, nona = center[1], center[0], *(float(S[k][0]) for k in ("xs", "ys", "xy", "nona"))
    den = scale[1] * scale[0]
    f1, f2, f3 = (lambda c: fma(cy, -xs, c)), (lambda c: fma(cx, -ys, c)), (lambda c: fma(cx * cy, nona, c))
    u1, u2, u3 = (lambda c: c - cy * xs), (lambda c: c - cx * ys), (lambda c: c + cx * cy * nona)
    chains = [(f1, f2, f3), (u1, f2, f3), (f1, u2, f3), (f1, f2, u3), (u1, u2, u3)]
    out = []
    for a, b, c in chains:
        r = np.float64(c(b(a(xy)))) / den
        out.append(float(r * r))
    return out


def test_clumping_threshold_equality(B):
    """Two columns, thr_r2 set to the model's r^2 of the pair (no conflict: both kept) and to the double just below it
    (conflict: the lower-priority one goes), for the CLUMP chain and for LEVELS.  The CLUMP pairs are chosen so that every
    other rounding sequence of the numerator gives another r^2: each of them would flip one of the two decisions."""
    rng = np.random.default_rng(29)
    pos = np.array([1.0, 2.0])
    ordv = np.array([2, 1], dtype=np.int32)
    picked, missing = [], set(range(1, 5))
    for _ in range(2000):
        H = _geno(rng, 333, 2, na=0.03)
        center, scale, _, _ = _bed_stats(H)
        r2s = _clump_r2_chains(H, center, scale)
        hit = {q for q in missing if r2s[q] != r2s[0]}
        if hit:
            picked.append((H, center, scale, r2s[0]))
            missing -= hit
        if not missing:
            break
    assert not missing
    for H, center, scale, r2 in picked:
        n, m = H.shape
        S = R.pair_sums(H, R.Band(pos, 10.0, both=True))
        g = B.Bed.from_packed(pack(H), n, m)
        for thr, keep in ((r2, [1, 1]), (float(np.nextafter(r2, 0)), [0, 1])):
            assert R.clump_epilogue(S, center, scale, thr).tolist() == [keep == [0, 1]]
            k = B.bed_clumping_chr(g, np.arange(1, n + 1), np.arange(1, m + 1), center, scale, ordv, None, pos, 10.0, thr)
            assert k.tolist() == keep, (thr, r2)
        g.close()
    band = R.Band(pos, 10.0, both=True)
    # LEVELS on a missing-free pair
    H = _geno(rng, 333, 2)
    n, m = H.shape
    sx = H.sum(0).astype(np.float64)
    dX = (H.astype(np.float64) ** 2).sum(0) - sx * sx / n
    S2 = R.pair_sums(H, band)
    nm = float(S2["xy"][0]) - sx[0] * sx[1] / n
    r2 = nm * nm / (dX[0] * dX[1])
    f = B.Bed.from_fbm(H)
    for thr, keep in ((r2, [1, 1]), (float(np.nextafter(r2, 0)), [0, 1])):
        k = B.clumping_chr(f, np.arange(1, n + 1), np.arange(1, m + 1), ordv, None, pos, sx, dX, 10.0, thr)
        assert k.tolist() == keep, (thr, r2)
    f.close()


def test_multi_batch_clumping(B):
    c = batch_case()
    G = c["G"]
    n, m = G.shape
    pos = np.arange(1.0, m + 1)
    center, scale, _, _ = _bed_stats(G)
    ordv = (np.argsort(-np.random.default_rng(1).random(m), kind="stable") + 1).astype(np.int32)
    g = B.Bed.from_packed(pack(G), n, m)
    k = B.bed_clumping_chr(g, np.arange(1, n + 1), np.arange(1, m + 1), center, scale, ordv, None, pos, 1.0, 0.2)
    g.close()
    want = _clump_model(G, center, scale, pos, 1.0, 0.2, ordv)
    assert np.array_equal(k, want) and 0 < (want == 0).sum() < m


def _owner_csc(p, i, x, owners):
    """(column, row, value) of the CSC entries of the given columns, in storage order."""
    lens = p[owners + 1] - p[owners]
    idx = np.repeat(p[owners], lens) + np.arange(lens.sum()) - np.repeat(np.cumsum(lens) - lens, lens)
    return np.repeat(owners, lens), i[idx], x[idx]


def test_cfg2_shape_band_bytes():
    """configs[2]'s shape: 100,000 x 200,000 LD-structured synthetic, 0.5 % missing, 500-SNP window.  A row block then needs
    five six-product tiles (491,520 ints), so all 1,563 row blocks fit one batch (767,262,720 of the 805,306,368
    ints the bound allows); the multi-batch path is test_multi_batch_band_bytes'.  The last 1,024 owners (band offsets near
    1e8) and eight random row blocks are checked against the model, which generates only the columns their windows need."""
    import torch

    if torch.cuda.mem_get_info()[0] / 1e9 < 30:
        pytest.skip("needs ~20 GB of HBM")
    import bigsnpr_b200 as B
    from bigsnpr_b200 import build
    from oracle import ref

    build.build()
    ref.build()
    n, m, w = 100_000, 200_000, 500
    kw = dict(seed=37, na_rate=0.005, ld_rho=0.9, ld_block=50)
    g = B.Bed.synthetic(n, m, **kw)
    p, i, x = B.bed_cor(g, size=w, thr_r2=0.0)
    g.close()
    pos = 1000.0 * np.arange(1, m + 1)
    band = R.Band(pos, w * 1000.0)
    # with 100,000 rows at 0.5 %, a column without a missing value has probability 0.995^100000: every tile takes mode 1
    plan = R.Plan(np.ones(m, dtype=bool), band)
    assert plan.nbatches == 1 and max(plan.ntiles) == 5 and plan.batches[0][3] == 767_262_720
    rng = np.random.default_rng(2)
    blocks = [(m - 1024, m)] + [(b * R.TM, b * R.TM + R.TM) for b in rng.choice(m // R.TM, 8, replace=False)]
    thr = B.cor_thresholds(n, 1.0, 0.0)
    for lo, hi in blocks:
        c0 = max(0, lo - w)
        o = ref.synth_bed(n, hi - c0, col_offset=c0, **kw)
        G = ref.decode_dense(o)
        assert (G == 3).any(axis=0).all()
        owners = np.arange(lo, hi)
        S = R.pair_sums(G, band, owners, col0=c0)
        r, keep = R.cor_epilogue(S, thr)
        col = np.r_[S["j0"][keep], owners]
        row = np.r_[S["j"][keep], owners]
        val = np.r_[r[keep], np.ones(owners.size)]
        order = np.lexsort((row, col))
        gc, gi, gx = _owner_csc(p, i, x, owners)
        assert np.array_equal(gc, col[order]) and np.array_equal(gi, row[order]), (lo, hi)
        assert np.array_equal(gx.view(np.int64), val[order].view(np.int64)), (lo, hi)
