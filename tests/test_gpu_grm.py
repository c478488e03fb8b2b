"""bed_tcrossprodSelf on the device against the exact model of its arithmetic (tests/grm_ref.py), byte for byte, and
against the oracle where the weights span orders of magnitude.

K is a sum of exact integer Grams of base-128 weight digits folded into fp64 in a fixed order, plus vector terms from
the matvec engine, so a kernel, tile edge, k-block split, weight class or index form that changes any integer changes
the bytes here.  Shapes cross the 128- and 256-row tiles, the 8 x 8 super-tile order and the 262,144-code k-blocks;
missing values come as none, one code, 1 % spread and a whole row; the columns are all of them (the resident copy),
subsets, and unsorted multisets (the compacted copy).  Every process-wide switch runs in its own subprocess.

The missing-value lists of the matvec engine split an unscaled sum into 32-bit halves along the row layout they build,
which the model does not restate (tests/fixedpoint_ref.py); the byte comparisons therefore run with BSG_NA_LISTS=0.
The accuracy cases against the oracle run with the library's defaults.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests import grm_ref as gr  # noqa: E402

pytestmark = pytest.mark.gpu

ROWS = [1, 2, 127, 128, 129, 255, 256, 257, 513]
COLS = [1, 15, 16, 17, 127, 128, 129, 5000]
NA_MODES = ["none", "one", "spread", "row"]
FORMS = ["all", "subset", "multiset"]
PATHS = {
    "default": {},
    "no_tma": {"BSG_GRAM_TMA": "0"},
    "k_wgram": {"BSG_GRAM_TMA": "0", "BSG_GRM_TCGEN05": "0"},
    "slices2": {"BSG_GRM_SLICES": "2"},
    "slices3": {"BSG_GRM_SLICES": "3"},
    "slices5": {"BSG_GRM_SLICES": "5"},
    "slices9": {"BSG_GRM_SLICES": "9"},
}


def _model_args(env):
    ns = int(env.get("BSG_GRM_SLICES", "4"))
    tma = env.get("BSG_GRAM_TMA", "1") != "0"
    return ns, ("gramt" if tma and ns <= 4 else "wgram")


def _same(got, want, what=""):
    got, want = np.ascontiguousarray(got, dtype=np.float64), np.ascontiguousarray(want, dtype=np.float64)
    assert got.shape == want.shape, what
    if got.tobytes() != want.tobytes():
        bad = np.nonzero(got.reshape(-1).view(np.int64) != want.reshape(-1).view(np.int64))[0]
        k = bad[0]
        raise AssertionError("%s: %d of %d differ, first at %d: %r vs model %r (max |diff| %.3g)"
                             % (what, bad.size, got.size, k, got.reshape(-1)[k], want.reshape(-1)[k],
                                np.max(np.abs(got - want))))


def _handle(B, G):
    from oracle import ref

    n, m = G.shape
    return B.Bed.from_packed(ref.write_bed_bytes(G), n, m)


def _case(rng, nr, nc, na, form, skew):
    """(G, ir, ic, center, scale): a file and a selection of nr rows and nc columns."""
    if form == "all":
        n, m = nr, nc
    elif form == "subset":
        n, m = nr + 7, nc + 5
    else:
        n, m = nr // 2 + 3, nc // 2 + 3
    G = rng.integers(0, 3, size=(n, m)).astype(np.uint8)
    if form == "all":
        ir, ic = None, None
    elif form == "subset":
        ir, ic = np.sort(rng.choice(n, nr, replace=False)) + 1, np.sort(rng.choice(m, nc, replace=False)) + 1
    else:
        ir, ic = rng.integers(1, n + 1, nr), rng.integers(1, m + 1, nc)
    r0 = np.arange(n) if ir is None else ir - 1
    c0 = np.arange(m) if ic is None else ic - 1
    if na == "one":
        G[r0[nr // 2], c0[nc // 3]] = 3
    elif na == "spread":
        G[rng.random((n, m)) < 0.01] = 3
        G[r0[0], c0[0]] = 3
    elif na == "row":
        G[r0[nr - 1], :] = 3
    center = rng.uniform(0.2, 1.8, size=nc)
    scale = rng.uniform(0.45, 1.2, size=nc)  # W1 within a factor 16: one class
    if skew and nc > 1:  # a few rare-variant weights: two or three classes
        k = rng.choice(nc, min(3, nc - 1), replace=False)
        center[k], scale[k] = 2e-4, np.sqrt(2e-4 * (1 - 1e-4))
    return G, ir, ic, center, scale


def _grm(B, g, ir, ic, c, s):
    sel = lambda ind: ... if ind is None else ind  # noqa: E731
    return B.bed_tcrossprodSelf(g, lambda *a, **k: {"center": c, "scale": s}, sel(ir), sel(ic))[0]


def _cases():
    """(nr, nc, na, form, skew): every row count at 129 columns, every column count at 257 rows, missing-value modes
    and index forms rotated over them, and the shapes past 2,048 rows and past two k-blocks."""
    out = []
    i = 0
    for nr in ROWS:
        out.append((nr, 129, NA_MODES[i % 4], FORMS[i % 3], i % 2 == 1))
        i += 1
    for nc in COLS:
        out.append((257, nc, NA_MODES[i % 4], FORMS[(i + 1) % 3], i % 2 == 0))
        i += 1
    for na in NA_MODES:
        for form in FORMS:
            out.append((130, 300, na, form, (NA_MODES.index(na) + FORMS.index(form)) % 2 == 0))
    out += [(2100, 40, "spread", "all", False), (2100, 40, "one", "multiset", True)]
    return out


def run_cases(env, big=True):
    """Every case of _cases() on the device against the model; returns a list of failures."""
    import bigsnpr_b200 as B

    ns, path = _model_args(env)
    rng = np.random.default_rng(20261017)
    cases = list(_cases())
    if big:
        cases.append((5, 2 * 262144 + 300, "spread", "all", True))  # three k-blocks per class
    fails = []
    for nr, nc, na, form, skew in cases:
        G, ir, ic, c, s = _case(rng, nr, nc, na, form, skew)
        what = "%s nr=%d nc=%d na=%s %s classes=%d" % (env, nr, nc, na, form, gr.n_classes(c, s))
        g = _handle(B, G)
        try:
            _same(_grm(B, g, ir, ic, c, s), gr.tcrossprod(G, c, s, ir, ic, nslices=ns, path=path), what)
        except AssertionError as e:
            fails.append(str(e))
        g.close()
    return fails


_RUN = """
import sys, json
sys.path.insert(0, sys.argv[1])
from tests import test_gpu_grm as t
import os
fails = t.run_cases({k: v for k, v in os.environ.items() if k.startswith("BSG_GRM") or k.startswith("BSG_GRAM")},
                    big=sys.argv[3] == "1")
open(sys.argv[2], "w").write(json.dumps(fails))
"""


@pytest.fixture(scope="module")
def B():
    import bigsnpr_b200 as b

    from bigsnpr_b200 import build

    build.build()
    return b


@pytest.mark.parametrize("path", sorted(PATHS))
def test_every_path_matches_the_model(B, tmp_path, path):
    """Each switch is read once per process: one subprocess per kernel path."""
    import json

    res = tmp_path / "fails.json"
    env = dict(os.environ, BSG_NA_LISTS="0", **PATHS[path])
    for k in ("BSG_GRM_DSYRK",):
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-c", _RUN, ROOT, str(res), "1" if path in ("default", "k_wgram") else "0"],
                       capture_output=True, text=True, env=env, timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    fails = json.loads(res.read_text())
    assert not fails, "\n".join(fails[:10])


def test_device_entry_point_gives_the_same_bytes(B, rng, monkeypatch):
    import torch

    from bigsnpr_b200 import _lib

    monkeypatch.setenv("BSG_NA_LISTS", "0")
    for skew in (False, True):
        G, ir, ic, c, s = _case(rng, 300, 700, "spread", "multiset", skew)
        g = _handle(B, G)
        want = _grm(B, g, ir, ic, c, s)
        Kd = torch.empty((300, 300), dtype=torch.float64, device="cuda")
        ip = lambda a: np.ascontiguousarray(a, dtype=np.int32)  # noqa: E731
        irr, icc = ip(ir), ip(ic)
        cc, ss = np.ascontiguousarray(c), np.ascontiguousarray(s)
        _lib.check(_lib.lib().bsg_tcrossprod_dev(g._h, irr.ctypes.data_as(_lib.c_int_p), 300, icc.ctypes.data_as(_lib.c_int_p),
                                                 700, cc.ctypes.data_as(_lib.c_dbl_p), ss.ctypes.data_as(_lib.c_dbl_p),
                                                 ctypes.c_void_p(Kd.data_ptr())))
        torch.cuda.synchronize()
        _same(Kd.cpu().numpy().T, want, "bsg_tcrossprod_dev skew=%s" % skew)
        _same(want, gr.tcrossprod(G, c, s, ir, ic), "model")
        g.close()


# ---- accuracy where the weights span orders of magnitude ---------------------------------------------------------------------
def _oracle_K(oracle, G, c, s):
    n, m = G.shape
    o = oracle.OracleBed.from_packed(oracle.write_bed_bytes(G), n, m)
    return oracle.bed_tcrossprodSelf(o, lambda *a, **k: {"center": c, "scale": s}, block_size=m)[0]


def _skewed(rng):
    out = []
    for mac in (1, 2):
        for na in (0.0, 0.01):
            p = rng.uniform(0.02, 0.5, size=3000)
            G = rng.binomial(2, p[None, :], size=(2000, 3000)).astype(np.uint8)
            G[:, 11] = 0
            G[:mac, 11] = 1
            if na:
                G[rng.random(G.shape) < na] = 3
                G[:, 11] = np.where(G[:, 11] == 3, 0, G[:, 11])
            out.append(("MAC-%d na=%g" % (mac, na), G, None))
    for pc in (2e-6, 1 - 2e-6):
        for na in (0.0, 0.01):
            p = rng.uniform(0.02, 0.5, size=3000)
            G = rng.binomial(2, p[None, :], size=(1000, 3000)).astype(np.uint8)
            if na:
                G[rng.random(G.shape) < na] = 3
            out.append(("cohort p=%g na=%g" % (pc, na), G, pc))
    return out


def test_skewed_weights_stay_within_1e8_of_the_oracle(B, oracle, rng):
    """A MAC-1 or MAC-2 column under bed_scaleBinom, or a caller's cohort allele frequency of 2e-6 or 1 - 2e-6 on three
    columns, with and without 1 % missing values, on the path the library selects by itself."""
    report, worst = [], 0.0
    for name, G, pc in _skewed(rng):
        g = _handle(B, G)
        sc = B.bed_scaleBinom(g)
        c, s = np.array(sc["center"]), np.array(sc["scale"])
        if pc is not None:
            c[[0, 1500, 2999]] = 2 * pc
            s[[0, 1500, 2999]] = np.sqrt(2 * pc * (1 - pc))
        K = _grm(B, g, None, None, c, s)
        K0 = _oracle_K(oracle, G, c, s)
        err = float(np.max(np.abs(K - K0)) / np.max(np.abs(K0)))
        report.append("%s: %.3g (%d classes)" % (name, err, gr.n_classes(c, s)))
        worst = max(worst, err)
        g.close()
    assert worst < 1e-8, "\n".join(report)


# ---- DSYRK -------------------------------------------------------------------------------------------------------------------------
_DSYRK = """
import sys, json
sys.path.insert(0, sys.argv[1])
import numpy as np
from tests import test_gpu_grm as t
open(sys.argv[2], "w").write(json.dumps(t.dsyrk_errors()))
"""


def dsyrk_errors():
    import bigsnpr_b200 as B

    from oracle import ref

    ref.build()
    rng = np.random.default_rng(7)
    out = {}
    G = rng.integers(0, 3, size=(300, 900)).astype(np.uint8)
    G[rng.random(G.shape) < 0.01] = 3
    g = _handle(B, G)
    for name, c, s in (("binom", None, None),
                       ("negative center", rng.uniform(-1.0, 1.8, 900), rng.uniform(0.4, 1.2, 900))):
        if c is None:
            sc = B.bed_scaleBinom(g)
            c, s = np.array(sc["center"]), np.array(sc["scale"])
        K, K0 = _grm(B, g, None, None, c, s), _oracle_K(ref, G, c, s)
        out[name] = float(np.max(np.abs(K - K0)) / np.max(np.abs(K0)))
    g.close()
    return out


def test_dsyrk_path_matches_the_oracle(B, tmp_path):
    import json

    res = tmp_path / "dsyrk.json"
    env = dict(os.environ, BSG_GRM_DSYRK="1")
    r = subprocess.run([sys.executable, "-c", _DSYRK, ROOT, str(res)], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    errs = json.loads(res.read_text())
    assert all(v < 1e-12 for v in errs.values()), errs


def test_degenerate_scaling_falls_back_to_dsyrk(B, oracle, rng):
    """A negative center (W2' < 0) agrees with the oracle to 1e-12; a zero scale and a monomorphic column under
    bed_scaleBinom give the oracle's pattern of finite and non-finite entries."""
    G = rng.integers(0, 3, size=(200, 500)).astype(np.uint8)
    G[rng.random(G.shape) < 0.01] = 3
    G[:, 7] = 0  # monomorphic
    g = _handle(B, G)
    c, s = rng.uniform(-0.5, 1.8, 500), rng.uniform(0.4, 1.2, 500)
    K, K0 = _grm(B, g, None, None, c, s), _oracle_K(oracle, G, c, s)
    assert np.max(np.abs(K - K0)) / np.max(np.abs(K0)) < 1e-12
    sc = B.bed_scaleBinom(g)
    for c, s in ((np.array(sc["center"]), np.array(sc["scale"])), (np.ones(500), np.r_[np.ones(499), 0.0])):
        K, K0 = _grm(B, g, None, None, c, s), _oracle_K(oracle, G, c, s)
        assert np.array_equal(np.isfinite(K), np.isfinite(K0))
        assert np.array_equal(np.isnan(K), np.isnan(K0))
        fin = np.isfinite(K0)
        if fin.any():
            assert np.max(np.abs(K[fin] - K0[fin])) <= 1e-12 * np.max(np.abs(K0[fin]))
    g.close()
