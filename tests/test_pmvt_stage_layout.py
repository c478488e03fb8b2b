"""Lane-level NumPy model of k_pmvT's CTA-wide TMA stage (bigsnpr_b200/csrc/bsg_pmv.cu): the four 128-byte-swizzled
boxes of 32 lines x 128 B and the split digit block a stage holds, the XOR-addressed reads of the eight consumer warps
(lanes with q >= 2 read a line quad as rows 2, 3, 0, 1), the PRMT transpose with the lane's own last selectors, the
mma.sync.m16n8k32 fragments and the sample each accumulator is added to.  It checks the plane sums against exact integer
dot products, with a partial last step and a segment reaching past the line stride (both zero-filled by the TMA unit),
and that every shared-memory load of a warp hits 32 distinct banks.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_pmv_layout import mma_m16n8k32  # noqa: E402
from test_pmvt_layout import exact, prmt, quant_digits  # noqa: E402

TWARPS, TLINES, TBYTES = 8, 32, 512
TBOX = 32 * 128
TDIG_OFF = 4 * TBOX
TSTAGE_BYTES = 4 * TBOX + 1024


def TRD(i, sl):
    return (i << 7) ^ (i << 4) ^ (sl << 5)


def tma_stage(packed, stride, rows, l0, x0, dig, step):
    """Bytes of one stage as the producer's copies leave them.  packed: (lines, stride) bytes of copy A; the tensor map
    spans `rows` lines x `stride` bytes, anything outside reads as zero.  Box j, row R, 16-byte chunk c -> chunk c ^ (R & 7)."""
    st = np.zeros(TSTAGE_BYTES, dtype=np.uint8)
    for j in range(4):
        for R in range(32):
            line = l0 + R
            for c in range(8):
                col = x0 + 128 * j + 16 * c
                src = np.zeros(16, dtype=np.uint8)
                if line < rows:
                    seg = packed[line, col:min(col + 16, stride)]
                    src[:seg.size] = seg
                dst = j * TBOX + R * 128 + (c ^ (R & 7)) * 16
                st[dst:dst + 16] = src
    block = dig[step * 256:(step + 1) * 256].view(np.uint8)
    st[TDIG_OFF:TDIG_OFF + 128] = block[:128]  # slices 0..3
    st[TDIG_OFF + 144:TDIG_OFF + 272] = block[128:]  # slices 4..7, 16 B further
    return st


def lds32_warp(st, addrs):
    """one warp-wide LDS.32: 32 lane addresses -> values; the addresses must fall in 32 distinct banks"""
    assert len({(a >> 2) & 31 for a in addrs}) == 32, sorted((a >> 2) & 31 for a in addrs)
    return [int.from_bytes(st[a:a + 4].tobytes(), "little") for a in addrs]


def run_cta(codes, Q, n, stride, plane=0):
    """codes: (nlines, 4 * stride) values 0..3 of one CTA's lines (its segment starts at byte 0); returns the exact
    per-sample sums of the CTA's 2048 samples (only samples < n are stored)."""
    nlines = codes.shape[0]
    nsteps = (nlines + TLINES - 1) // TLINES
    packed = np.zeros((nlines, stride), dtype=np.uint8)
    for c in range(4):
        packed |= (codes[:, c::4] << (2 * c)).astype(np.uint8)
    dig = quant_digits(Q, nsteps)
    assert TSTAGE_BYTES % 1024 == 0  # the XOR addressing needs 1 KB aligned boxes in every stage
    acc = np.zeros((TWARPS, 4, 4, 32, 4), dtype=np.int64)  # [warp][byte j][field c][lane][fragment]
    for step in range(nsteps):
        st = tma_stage(packed, stride, nlines, step * TLINES, 0, dig, step)
        for w in range(TWARPS):
            lanes = [(lane >> 2, lane & 3) for lane in range(32)]
            dg = [TDIG_OFF + g * 32 + 16 * (g >> 2) + 4 * q for g, q in lanes]
            b0, b1 = lds32_warp(st, dg), lds32_warp(st, [a + 16 for a in dg])
            rsw = [2 * (q >> 1) for g, q in lanes]
            rd = []
            for (g, q), s in zip(lanes, rsw):
                chunk0 = (4 * (w & 1) + (g >> 2)) ^ (4 * (q & 1) + s)
                rd.append((w >> 1) * TBOX + q * 512 + (s << 7) + chunk0 * 16 + 4 * (g & 3))
            W = np.zeros((32, 2, 2, 4), dtype=np.uint64)
            for sl in range(2):
                for hf in range(2):
                    x = [lds32_warp(st, [(a ^ TRD(i, sl)) + hf * 2048 for a in rd]) for i in range(4)]
                    for lane in range(32):
                        lo, hi = (0x1054, 0x3276) if rsw[lane] else (0x5410, 0x7632)
                        x0, x1, x2, x3 = (x[i][lane] for i in range(4))
                        t0, t1 = prmt(x0, x1, 0x5140), prmt(x2, x3, 0x5140)
                        t2, t3 = prmt(x0, x1, 0x7362), prmt(x2, x3, 0x7362)
                        W[lane, sl, hf] = [prmt(t0, t1, lo), prmt(t0, t1, hi), prmt(t2, t3, lo), prmt(t2, t3, hi)]
            b = np.array([[b0[lane], b1[lane]] for lane in range(32)], dtype=np.uint64)
            for j in range(4):
                for c in range(4):
                    mask = 0x03030303 << (2 * c)
                    a = np.zeros((32, 4), dtype=np.uint64)
                    for lane in range(32):
                        v4 = [int(W[lane, 0, 0, j]), int(W[lane, 1, 0, j]), int(W[lane, 0, 1, j]), int(W[lane, 1, 1, j])]
                        if plane == 1:
                            v4 = [v & (v >> 1) & 0x55555555 for v in v4]
                        elif plane == 2:
                            v4 = [(v >> 1) & 0x55555555 for v in v4]
                        a[lane] = [v & mask for v in v4]
                    mma_m16n8k32(acc[w][j][c], a, b)
    part = np.zeros((TBYTES * 4, 8), dtype=np.int64)
    for w in range(TWARPS):
        for lane in range(32):
            g, q = lane >> 2, lane & 3
            for j in range(4):
                for c in range(4):
                    for sl in range(2):
                        sample = 4 * (64 * w + 4 * (8 * sl + g) + j) + c
                        if sample >= n:
                            continue
                        for k in range(2):
                            v = int(acc[w][j][c][lane][2 * sl + k])
                            assert v % (4 ** c) == 0
                            part[sample, 2 * q + k] += v >> (2 * c)
    return np.array([sum(int(part[i, s]) << (8 * s) for s in range(8)) for i in range(n)], dtype=object)


def test_kpmvT_stage_model_matches_exact_sums():
    rng = np.random.default_rng(11)
    nlines = 45  # two steps, the second one partial: rows past the map read as zero, their digits are zero
    codes = rng.integers(0, 4, size=(nlines, 4 * TBYTES))
    Q = [int(v) for v in rng.integers(-2**59, 2**59, size=nlines)]
    for plane in (0, 1):
        got = run_cta(codes, Q, 4 * TBYTES, TBYTES, plane)
        assert np.array_equal(got, exact(codes, Q, plane)), plane


def test_kpmvT_stage_model_segment_past_the_stride():
    # the last CTA of a line: 384 of its 512 bytes exist (box 3 is out of bounds), 1,517 samples
    rng = np.random.default_rng(12)
    nlines, stride, n = 40, 384, 1517
    codes = rng.integers(0, 4, size=(nlines, 4 * stride))
    Q = [int(v) for v in rng.integers(-2**59, 2**59, size=nlines)]
    got = run_cta(codes, Q, n, stride)
    assert np.array_equal(got, exact(codes[:, :n], Q, 0))

