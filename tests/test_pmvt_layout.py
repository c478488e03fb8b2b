"""Lane-level NumPy model of the single-copy matvec kernels (bigsnpr_b200/csrc/bsg_pmv.cu: k_pmvT, k_pmvT2, k_quantT).
It replays the index arithmetic of the CUDA code on the CPU -- the cp.async destination layout of a warp's strip,
the four-line word reads, the PRMT byte transpose, the 2-bit field masks (field c enters as 4^c x code), the
mma.sync.m16n8k32 fragment ownership, the digit layout [step][slice][32 lines] and the sample each accumulator
belongs to -- and checks the plane sums against exact integer dot products.  It guards the layout contract between
the loader lanes, the reader lanes and the epilogue.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_pmv_layout import digits_of, mma_m16n8k32  # noqa: E402

TLINES = 32


def prmt(a, b, sel):
    """PTX prmt.b32 (default mode): result byte i = byte (sel >> 4i) & 7 of the 8-byte pool {a: 0-3, b: 4-7}."""
    pool = [(a >> (8 * i)) & 0xFF for i in range(4)] + [(b >> (8 * i)) & 0xFF for i in range(4)]
    return sum(pool[(sel >> (4 * i)) & 7] << (8 * i) for i in range(4))


def transpose4(x0, x1, x2, x3):
    t0, t1 = prmt(x0, x1, 0x5140), prmt(x2, x3, 0x5140)
    t2, t3 = prmt(x0, x1, 0x7362), prmt(x2, x3, 0x7362)
    return [prmt(t0, t1, 0x5410), prmt(t0, t1, 0x7632), prmt(t2, t3, 0x5410), prmt(t2, t3, 0x7632)]


def test_prmt_transpose_is_a_byte_transpose():
    rng = np.random.default_rng(0)
    x = [int(v) for v in rng.integers(0, 2**32, size=4, dtype=np.uint64)]
    W = transpose4(*x)
    for j in range(4):
        for r in range(4):
            assert (W[j] >> (8 * r)) & 0xFF == (x[r] >> (8 * j)) & 0xFF  # byte r of W_j = byte j of line r


def stage_strip(lines64, width):
    """cp.async destinations of one warp stage.  lines64: (32, width) bytes (width = 64 for k_pmvT_lines, 32 for k_pmvT2).
    k_pmvT_lines: word (row = 16 hf + 4 qq + r, column wc = 8 sl + gg) at word ((((r 2 + hf) 2 + sl) 4 + qq) 8 + gg)
    k_pmvT2:      word (row, column gg)                                 at word  (((r 2 + hf) 4 + qq) 8 + gg)"""
    smem = np.zeros(32 * width // 4, dtype=np.uint32)
    words = lines64.reshape(32, width // 4, 4)
    for lane in range(32):  # loader role: 4 (or 2) granules of 16 B per lane
        if width == 64:
            lrow, lch = lane >> 2, lane & 3
            for i in range(4):
                row = 8 * i + lrow
                hf, qq, r, sl, hc = row >> 4, (row >> 2) & 3, row & 3, lch >> 1, lch & 1
                dst = ((((r * 2 + hf) * 2 + sl) * 4 + qq) * 8) + 4 * hc
                for k in range(4):
                    b = words[row, 4 * lch + k]
                    smem[dst + k] = int(b[0]) | int(b[1]) << 8 | int(b[2]) << 16 | int(b[3]) << 24
        else:
            lrow, lch = lane >> 1, lane & 1
            for i in range(2):
                row = 16 * i + lrow
                hf, qq, r = row >> 4, (row >> 2) & 3, row & 3
                dst = (((r * 2 + hf) * 4 + qq) * 8) + 4 * lch
                for k in range(4):
                    b = words[row, 4 * lch + k]
                    smem[dst + k] = int(b[0]) | int(b[1]) << 8 | int(b[2]) << 16 | int(b[3]) << 24
    return smem


def quant_digits(Q, nsteps):
    """k_quantT: dig[(t / 32) * 256 + slice * 32 + (t % 32)]"""
    dig = np.zeros(nsteps * 256, dtype=np.int8)
    for t, q in enumerate(Q):
        for s, d in enumerate(digits_of(q)):
            dig[(t >> 5) * 256 + s * 32 + (t & 31)] = d
    return dig


def b_regs_of(dig, step):
    regs = np.zeros((32, 2), dtype=np.uint64)
    for lane in range(32):
        g, q = lane >> 2, lane & 3
        for h in range(2):
            base = step * 256 + g * 32 + 4 * q + 16 * h
            regs[lane][h] = sum((int(dig[base + i]) & 0xFF) << (8 * i) for i in range(4))
    return regs


def combine(part_row):
    return sum(int(part_row[s]) << (8 * s) for s in range(8))


def run_kpmvT(codes, Q, plane):
    """codes: (nlines, 256) values 0..3 for the 256 samples of one warp strip of k_pmvT (64 bytes per line)."""
    nlines = codes.shape[0]
    nsteps = (nlines + 31) // 32
    packed = np.zeros((nsteps * 32, 64), dtype=np.uint8)
    for c in range(4):
        packed[:nlines] |= (codes[:, c::4] << (2 * c)).astype(np.uint8)
    dig = quant_digits(Q, nsteps)
    acc = np.zeros((4, 4, 32, 4), dtype=np.int64)  # [byte j][field c][lane][fragment]
    for step in range(nsteps):
        smem = stage_strip(packed[32 * step:32 * step + 32], 64)
        b = b_regs_of(dig, step)
        W = np.zeros((32, 2, 2, 4), dtype=np.uint64)
        for lane in range(32):
            g, q = lane >> 2, lane & 3
            for sl in range(2):
                for hf in range(2):
                    x = [int(smem[((r * 2 + hf) * 2 + sl) * 32 + q * 8 + g]) for r in range(4)]
                    W[lane, sl, hf] = transpose4(*x)
        for j in range(4):
            for c in range(4):
                mask = 0x03030303 << (2 * c)
                a = np.zeros((32, 4), dtype=np.uint64)
                for lane in range(32):
                    w = [int(W[lane, 0, 0, j]), int(W[lane, 1, 0, j]), int(W[lane, 0, 1, j]), int(W[lane, 1, 1, j])]
                    if plane == 1:
                        w = [v & (v >> 1) & 0x55555555 for v in w]
                    elif plane == 2:
                        w = [(v >> 1) & 0x55555555 for v in w]
                    a[lane] = [v & mask for v in w]
                mma_m16n8k32(acc[j][c], a, b)
    part = np.zeros((256, 8), dtype=np.int64)
    for lane in range(32):
        g, q = lane >> 2, lane & 3
        for j in range(4):
            for c in range(4):
                for sl in range(2):
                    sample = 4 * (4 * (8 * sl + g) + j) + c
                    for k in range(2):
                        v = int(acc[j][c][lane][2 * sl + k])
                        assert v % (4 ** c) == 0
                        part[sample, 2 * q + k] += v >> (2 * c)
    return np.array([combine(part[i]) for i in range(256)], dtype=object)


def run_kpmvT2(codes, Q1, Q2, pl):
    """codes: (nlines, 128) values for the 128 samples of one warp strip of k_pmvT2 (32 bytes per line)."""
    nlines = codes.shape[0]
    nsteps = (nlines + 31) // 32
    packed = np.zeros((nsteps * 32, 32), dtype=np.uint8)
    for c in range(4):
        packed[:nlines] |= (codes[:, c::4] << (2 * c)).astype(np.uint8)
    d1, d2 = quant_digits(Q1, nsteps), quant_digits(Q2, nsteps)
    acc = np.zeros((2, 2, 4, 32, 4), dtype=np.int64)  # [plane][unit][field][lane][fragment]
    for step in range(nsteps):
        smem = stage_strip(packed[32 * step:32 * step + 32], 32)
        b1, b2 = b_regs_of(d1, step), b_regs_of(d2, step)
        W = np.zeros((32, 2, 4), dtype=np.uint64)
        for lane in range(32):
            g, q = lane >> 2, lane & 3
            for hf in range(2):
                x = [int(smem[(r * 2 + hf) * 32 + q * 8 + g]) for r in range(4)]
                W[lane, hf] = transpose4(*x)
        for u in range(2):
            for c in range(4):
                a0 = np.zeros((32, 4), dtype=np.uint64)
                a1 = np.zeros((32, 4), dtype=np.uint64)
                for lane in range(32):
                    w = [int(W[lane, 0, u]), int(W[lane, 0, u + 2]), int(W[lane, 1, u]), int(W[lane, 1, u + 2])]
                    f = [(v & (v >> 1)) if pl == 1 else (v >> 1) for v in w]
                    a0[lane] = [v & (0x03030303 << (2 * c)) for v in w]
                    a1[lane] = [v & (0x01010101 << (2 * c)) for v in f]
                mma_m16n8k32(acc[0][u][c], a0, b1)
                mma_m16n8k32(acc[1][u][c], a1, b2)
    out = []
    for p in range(2):
        part = np.zeros((128, 8), dtype=np.int64)
        for lane in range(32):
            g, q = lane >> 2, lane & 3
            for u in range(2):
                for c in range(4):
                    for sl in range(2):
                        sample = 4 * (4 * g + u + 2 * sl) + c
                        for k in range(2):
                            part[sample, 2 * q + k] += int(acc[p][u][c][lane][2 * sl + k]) >> (2 * c)
        out.append(np.array([combine(part[i]) for i in range(128)], dtype=object))
    return out


def exact(codes, Q, plane):
    X = codes.astype(object)
    if plane == 1:
        X = (codes == 3).astype(object)
    elif plane == 2:
        X = (codes >= 2).astype(object)
    return np.array([sum(int(X[t, i]) * int(Q[t]) for t in range(codes.shape[0])) for i in range(codes.shape[1])],
                    dtype=object)


def test_kpmvT_model_matches_exact_sums():
    rng = np.random.default_rng(1)
    nlines = 45  # two steps, the second one partial (digits of the missing lines are zero)
    codes = rng.integers(0, 4, size=(nlines, 256))
    Q = [int(v) for v in rng.integers(-2**59, 2**59, size=nlines)]
    for plane in (0, 1, 2):
        got = run_kpmvT(codes, Q, plane)
        assert np.array_equal(got, exact(codes, Q, plane)), plane


def test_kpmvT2_model_matches_exact_sums():
    rng = np.random.default_rng(2)
    nlines = 40
    codes = rng.integers(0, 4, size=(nlines, 128))
    Q1 = [int(v) for v in rng.integers(-2**59, 2**59, size=nlines)]
    Q2 = [int(v) for v in rng.integers(-2**59, 2**59, size=nlines)]
    for pl in (1, 2):
        raw, flag = run_kpmvT2(codes, Q1, Q2, pl)
        assert np.array_equal(raw, exact(codes, Q1, 0))
        assert np.array_equal(flag, exact(codes, Q2, pl))
