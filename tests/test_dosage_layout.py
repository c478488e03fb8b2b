"""CPU checks of the dosage path (bigsnpr_b200/csrc/bsg_dosage.cu): the rule that decides which FBM.code256 tables
qualify (bsg_code256_dosage_scale), and lane-level NumPy models of the two byte-operand kernels.

k_dmvT (X.y): the CTA stage as either producer leaves it -- four 128-byte-swizzled TMA boxes (identity selection) or one
unswizzled 528-byte row per line filled by a 512-byte bulk copy (column list) -- the consumer's reads with the q >= 2 row
rotation, the PRMT transpose, the m16n8k32 fragments and the sample each accumulator goes to.  k_dmv (Xt.y): the lane's
16-byte line and digit words and the two IMMAs per 64-sample chunk.  Both are checked against exact integer dot products
with a partial last step and a segment reaching past the line stride, and every shared-memory load of k_dmvT must hit
32 distinct banks.
"""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_pmv_layout import mma_m16n8k32  # noqa: E402
from test_pmvt_layout import prmt, quant_digits  # noqa: E402
from test_pmvt_stage_layout import TRD, lds32_warp, tma_stage  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODE_DOSAGE = np.concatenate([[0, 1, 2, np.nan, 0, 1, 2], np.arange(201) * 0.01, np.full(48, np.nan)])

TW, TL, TB = 8, 32, 512
TBOX = 32 * 128
ROWP = 528
STG = 4 * TBOX + 1024
DIG_T, DIG_L = 4 * TBOX, TL * ROWP


# ---- eligibility --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def B():
    from bigsnpr_b200 import build

    build.build()
    import bigsnpr_b200

    return bigsnpr_b200


def test_dosage_scale_rule(B):
    f = B.code256_dosage_scale
    assert f(CODE_DOSAGE) == 100
    code = np.full(256, np.nan)
    code[:201] = np.arange(201) / 100.0
    assert f(code) == 100
    assert f(np.linspace(0, 2, 256)) == 0  # multiples of 2/255: D = 255 would need codes up to 510
    neg = CODE_DOSAGE.copy()
    neg[250] = -0.01
    assert f(neg) == 0
    big = np.full(256, np.nan)
    big[:3] = [0, 0.5, 128.0]  # D = 2 makes 256 > 255
    assert f(big) == 0
    big[2] = 127.5
    assert f(big) == 2
    inf = CODE_DOSAGE.copy()
    inf[255] = np.inf
    assert f(inf) == 0
    assert f(np.r_[[0.0, 0.25, 0.5], np.full(253, np.nan)]) == 4
    with pytest.raises(ValueError):
        f(np.zeros(10))


def test_int32_cap_of_a_ksplit():
    """q <= 255 and |digit| <= 128: an int32 accumulator holds 2^31 / 32,640 = 65,793 worst-case products, so both
    kernels cap a k-split at 65,536 contraction indices."""
    worst = 255 * 128
    assert 65536 * worst < 2**31 <= 65794 * worst
    acc = np.int64(0)
    for _ in range(65536 // 1024):
        acc += np.int64(1024) * 255 * (-128)  # the most negative product, 65,536 times
    assert -(2**31) <= acc and acc == -65536 * worst
    src = open(os.path.join(ROOT, "bigsnpr_b200", "csrc", "bsg_dosage.cu")).read()
    assert re.search(r"constexpr int MAX_LINES = 65536;", src)
    assert re.search(r"constexpr int DMAX_CHUNKS = 65536 / DCH;", src)


# ---- k_dmvT ---------------------------------------------------------------------------------------------------------------
def line_stage(vals_ext, lines, l0, x0, dig, step):
    """k_dmvT with a column list: row R = 512 bytes of line lines[min(l0 + R, last)] at R * ROWP, digits at DIG_L."""
    st = np.zeros(STG, dtype=np.uint8)
    for R in range(TL):
        t = min(l0 + R, len(lines) - 1)
        st[R * ROWP:R * ROWP + TB] = vals_ext[lines[t], x0:x0 + TB]
    block = dig[step * 256:(step + 1) * 256].view(np.uint8)
    st[DIG_L:DIG_L + 128] = block[:128]
    st[DIG_L + 144:DIG_L + 272] = block[128:]
    return st


def run_dmvT(vals, Q, n, stride, lines=None, garbage=None):
    """vals: (m, stride) value bytes; the CTA's segment starts at byte 0.  lines: selected physical lines (None: all, TMA
    stage).  garbage: bytes a bulk copy reads past the line stride (the next line / the slack).  Returns exact sums of
    samples < min(n, 512)."""
    m = vals.shape[0]
    sel = list(range(m)) if lines is None else list(lines)
    nsel = len(sel)
    nsteps = (nsel + TL - 1) // TL
    dig = quant_digits(Q, nsteps)
    ext = np.concatenate([vals, garbage if garbage is not None else np.zeros((m, TB), np.uint8)], axis=1)
    acc = np.zeros((TW, 4, 32, 4), dtype=np.int64)
    for step in range(nsteps):
        if lines is None:
            st = tma_stage(vals, stride, m, step * TL, 0, dig, step)
            dbase = DIG_T
        else:
            st = line_stage(ext, sel, step * TL, 0, dig, step)
            dbase = DIG_L
        for w in range(TW):
            lanes = [(lane >> 2, lane & 3) for lane in range(32)]
            dg = [dbase + g * 32 + 16 * (g >> 2) + 4 * q for g, q in lanes]
            b0, b1 = lds32_warp(st, dg), lds32_warp(st, [a + 16 for a in dg])
            rsw = [2 * (q >> 1) for g, q in lanes]
            W = np.zeros((32, 2, 2, 4), dtype=np.uint64)
            for sl in range(2):
                for hf in range(2):
                    x = []
                    for i in range(4):
                        if lines is None:
                            addrs = []
                            for (g, q), s in zip(lanes, rsw):
                                chunk0 = (4 * (w & 1) + (g >> 2)) ^ (4 * (q & 1) + s)
                                rd = (w >> 1) * TBOX + q * 512 + (s << 7) + chunk0 * 16 + 4 * (g & 3)
                                addrs.append((rd ^ TRD(i, sl)) + hf * 2048)
                        else:
                            addrs = [(16 * hf + 4 * q + (i ^ s)) * ROWP + (16 * w + 8 * sl + g) * 4
                                     for (g, q), s in zip(lanes, rsw)]
                        x.append(lds32_warp(st, addrs))
                    for lane in range(32):
                        lo, hi = (0x1054, 0x3276) if rsw[lane] else (0x5410, 0x7632)
                        x0, x1, x2, x3 = (x[i][lane] for i in range(4))
                        t0, t1 = prmt(x0, x1, 0x5140), prmt(x2, x3, 0x5140)
                        t2, t3 = prmt(x0, x1, 0x7362), prmt(x2, x3, 0x7362)
                        W[lane, sl, hf] = [prmt(t0, t1, lo), prmt(t0, t1, hi), prmt(t2, t3, lo), prmt(t2, t3, hi)]
            b = np.array([[b0[lane], b1[lane]] for lane in range(32)], dtype=np.uint64)
            for j in range(4):
                a = np.array([[W[lane, 0, 0, j], W[lane, 1, 0, j], W[lane, 0, 1, j], W[lane, 1, 1, j]]
                              for lane in range(32)], dtype=np.uint64)
                mma_m16n8k32(acc[w][j], a, b)
    nout = min(n, TB)
    part = np.zeros((TB, 8), dtype=object)
    part[:] = 0
    for w in range(TW):
        for lane in range(32):
            g, q = lane >> 2, lane & 3
            for j in range(4):
                for sl in range(2):
                    sample = 64 * w + 4 * (8 * sl + g) + j
                    if sample < nout:
                        for k in range(2):
                            part[sample, 2 * q + k] += int(acc[w][j][lane][2 * sl + k])
    return np.array([sum(int(part[i, s]) << (8 * s) for s in range(8)) for i in range(nout)], dtype=object)


def exact_cols(vals, Q, lines, n):
    sel = range(vals.shape[0]) if lines is None else lines
    return np.array([sum(int(vals[l, i]) * int(Qt) for l, Qt in zip(sel, Q)) for i in range(n)], dtype=object)


def test_kdmvT_tma_stage_exact_and_conflict_free():
    rng = np.random.default_rng(21)
    m = 45  # two steps, the second partial: rows past the map read as zero, their digits are zero
    vals = rng.integers(0, 256, size=(m, TB)).astype(np.uint8)
    Q = [int(v) for v in rng.integers(-2**59, 2**59, size=m)]
    assert np.array_equal(run_dmvT(vals, Q, TB, TB), exact_cols(vals, Q, None, TB))


def test_kdmvT_tma_segment_past_the_stride():
    rng = np.random.default_rng(22)
    m, stride, n = 40, 384, 301  # box 3 is out of bounds; samples n..stride are zero pads
    vals = rng.integers(0, 256, size=(m, stride)).astype(np.uint8)
    vals[:, n:] = 0
    Q = [int(v) for v in rng.integers(-2**59, 2**59, size=m)]
    assert np.array_equal(run_dmvT(vals, Q, n, stride), exact_cols(vals, Q, None, n))


def test_kdmvT_line_list_exact_and_conflict_free():
    rng = np.random.default_rng(23)
    m, stride, n = 70, 384, 333
    vals = rng.integers(0, 256, size=(m, stride)).astype(np.uint8)
    vals[:, n:] = 0
    garbage = rng.integers(1, 256, size=(m, TB)).astype(np.uint8)  # what a 512-byte copy reads past the stride
    lines = [int(v) for v in rng.integers(0, m, size=37)]  # duplicates, any order; the second step is partial
    Q = [int(v) for v in rng.integers(-2**59, 2**59, size=len(lines))]
    assert np.array_equal(run_dmvT(vals, Q, n, stride, lines, garbage), exact_cols(vals, Q, lines, n))


# ---- k_dmv ----------------------------------------------------------------------------------------------------------------
def test_kdmv_fragments_exact():
    """One warp, 32 lines, a stride of 3 chunks of 64 samples with n inside the last one."""
    rng = np.random.default_rng(24)
    stride, n = 192, 150
    vals = rng.integers(0, 256, size=(32, stride)).astype(np.uint8)
    vals[:, n:] = 0
    Q = [int(v) for v in rng.integers(-2**59, 2**59, size=n)] + [0] * (stride - n)
    dig = quant_digits(Q, stride // 32).view(np.uint8)
    acc = np.zeros((2, 2, 32, 4), dtype=np.int64)

    def words(b16):
        return [int.from_bytes(b16[4 * i:4 * i + 4].tobytes(), "little") for i in range(4)]

    for c in range(stride // 64):
        A = np.zeros((2, 2, 32, 4), dtype=np.uint64)
        Bw = np.zeros((32, 4), dtype=np.uint64)
        for lane in range(32):
            g, q = lane >> 2, lane & 3
            for t in range(2):
                for hh in range(2):
                    A[t, hh, lane] = words(vals[16 * t + 8 * hh + g, 64 * c + 16 * q:64 * c + 16 * q + 16])
            off = (2 * c + (q >> 1)) * 256 + g * 32 + 16 * (q & 1)
            Bw[lane] = words(dig[off:off + 16])
        for t in range(2):
            r0, r1 = A[t, 0], A[t, 1]
            mma_m16n8k32(acc[t][0], np.stack([r0[:, 0], r1[:, 0], r0[:, 1], r1[:, 1]], 1), Bw[:, 0:2])
            mma_m16n8k32(acc[t][1], np.stack([r0[:, 2], r1[:, 2], r0[:, 3], r1[:, 3]], 1), Bw[:, 2:4])
    part = np.zeros((32, 8), dtype=object)
    part[:] = 0
    for lane in range(32):
        g, q = lane >> 2, lane & 3
        for t in range(2):
            for hh in range(2):
                for k in range(2):
                    part[16 * t + 8 * hh + g, 2 * q + k] += int(acc[t][0][lane][2 * hh + k]) + int(acc[t][1][lane][2 * hh + k])
    got = [sum(int(part[l, s]) << (8 * s) for s in range(8)) for l in range(32)]
    want = [sum(int(vals[l, i]) * Q[i] for i in range(n)) for l in range(32)]
    assert got == want
