"""Lane-level NumPy model of the tensor-pipe matvec kernel (bigsnpr_b200/csrc/bsg_pmv.cu: k_prep2 digit layout,
k_pmv fragments and epilogue, combine).  It replays the exact index arithmetic of the CUDA code -- digit layout in shared
memory, mask decode of the packed words, mma.sync.m16n8k32 fragment ownership (PTX ISA: A row = groupID(+8),
col = 4*tid_in_group + i (+16); B row = 4*tid_in_group + i (+16), col = groupID; C row = groupID(+8),
col = 2*tid_in_group + i) -- and checks the result against exact integer dot products.  Runs on CPU: it
guards the layout contract between the quantiser and the consumer warps.
"""
import numpy as np

CODES, DIG = 512, 4096


def digits_of(Q):
    """signed base-256 digits, as peel() takes them off"""
    out = []
    v = int(Q)
    for _ in range(8):
        d = ((v & 0xFF) ^ 0x80) - 0x80
        out.append(d)
        v = (v - d) >> 8
    assert v == 0
    return out


def make_digit_chunk(Qchunk):
    """k_prep2: unit (w, s, q) at ((w*8+s)*4+q)*16, byte c*4+r <-> code
    t = (64q + 16w if w < 4 else 256 + 64q + 16(w-4)) + 4r + c  (word w of lane q, see k_pmv slot_load)."""
    buf = np.zeros(DIG, dtype=np.int8)
    D = np.array([digits_of(q) for q in Qchunk], dtype=np.int64)  # (512, 8)
    for w in range(8):
        for s in range(8):
            for q in range(4):
                base = ((w * 8 + s) * 4 + q) * 16
                for c in range(4):
                    for r in range(4):
                        buf[base + c * 4 + r] = D[(64 * q + 16 * w if w < 4 else 256 + 64 * q + 16 * (w - 4)) + 4 * r + c, s]
    return buf


def mma_m16n8k32(acc, a_regs, b_regs):
    """acc[lane][4] += A(16x32, u8) * B(32x8, s8) with the PTX fragment ownership; regs are uint32 arrays [32][4|2]."""
    A = np.zeros((16, 32), dtype=np.int64)
    B = np.zeros((32, 8), dtype=np.int64)
    for lane in range(32):
        g, q = lane >> 2, lane & 3
        for i in range(4):
            A[g, 4 * q + i] = (int(a_regs[lane][0]) >> (8 * i)) & 0xFF
            A[g + 8, 4 * q + i] = (int(a_regs[lane][1]) >> (8 * i)) & 0xFF
            A[g, 16 + 4 * q + i] = (int(a_regs[lane][2]) >> (8 * i)) & 0xFF
            A[g + 8, 16 + 4 * q + i] = (int(a_regs[lane][3]) >> (8 * i)) & 0xFF
            for h in range(2):
                byte = (int(b_regs[lane][h]) >> (8 * i)) & 0xFF
                B[16 * h + 4 * q + i, g] = (byte ^ 0x80) - 0x80
    Cm = A @ B
    for lane in range(32):
        g, q = lane >> 2, lane & 3
        acc[lane][0] += Cm[g, 2 * q]
        acc[lane][1] += Cm[g, 2 * q + 1]
        acc[lane][2] += Cm[g + 8, 2 * q]
        acc[lane][3] += Cm[g + 8, 2 * q + 1]


def run_subtile(lines_words, dig_chunks, with_na):
    """lines_words: [16][nchunks][32] uint32 packed words of 16 lines; returns (raw[16][8], na[16][8]) slice sums."""
    nchunks = len(dig_chunks)
    acc1 = np.zeros((32, 4), dtype=np.int64); acc16 = np.zeros((32, 4), dtype=np.int64)
    accn1 = np.zeros((32, 4), dtype=np.int64); accn16 = np.zeros((32, 4), dtype=np.int64)
    for c in range(nchunks):
        dig = dig_chunks[c].view(np.uint8)
        for w in range(8):
            a1 = np.zeros((32, 4), dtype=np.uint32); a16 = np.zeros((32, 4), dtype=np.uint32)
            n1 = np.zeros((32, 4), dtype=np.uint32); n16 = np.zeros((32, 4), dtype=np.uint32)
            bA = np.zeros((32, 2), dtype=np.uint32); bB = np.zeros((32, 2), dtype=np.uint32)
            for lane in range(32):
                g, q = lane >> 2, lane & 3
                # lane owns bytes [16q, 16q+16) (words 4q..4q+3) and [64+16q, 64+16q+16) (words 16+4q..) of the chunk
                wi = 4 * q + w if w < 4 else 16 + 4 * q + (w - 4)
                a = int(lines_words[g][c][wi]); b = int(lines_words[g + 8][c][wi])
                at, bt = a >> 2, b >> 2
                a1[lane] = [a & 0x03030303, b & 0x03030303, at & 0x03030303, bt & 0x03030303]
                a16[lane] = [a & 0x30303030, b & 0x30303030, at & 0x30303030, bt & 0x30303030]
                an, bn, ant, bnt = a & (a >> 1), b & (b >> 1), at & (at >> 1), bt & (bt >> 1)
                n1[lane] = [an & 0x01010101, bn & 0x01010101, ant & 0x01010101, bnt & 0x01010101]
                n16[lane] = [an & 0x10101010, bn & 0x10101010, ant & 0x10101010, bnt & 0x10101010]
                base = w * 512 + (g * 4 + q) * 16  # dbase + w*512
                regs = dig[base:base + 16].view(np.uint32)
                bA[lane] = regs[0:2]; bB[lane] = regs[2:4]
            mma_m16n8k32(acc1, a1, bA); mma_m16n8k32(acc16, a16, bB)
            if with_na:
                mma_m16n8k32(accn1, n1, bA); mma_m16n8k32(accn16, n16, bB)
    raw = np.zeros((16, 8), dtype=np.int64); na = np.zeros((16, 8), dtype=np.int64)
    for lane in range(32):
        g, q = lane >> 2, lane & 3
        for hrow in range(2):
            for i in range(2):
                raw[g + 8 * hrow, 2 * q + i] = acc1[lane][2 * hrow + i] + (acc16[lane][2 * hrow + i] >> 4)
                na[g + 8 * hrow, 2 * q + i] = accn1[lane][2 * hrow + i] + (accn16[lane][2 * hrow + i] >> 4)
    return raw, na


def test_pmv_layout_exact():
    rng = np.random.default_rng(5)
    L, nchunks = 1000, 2  # 1000 codes -> 2 chunks of 512 (pads are code 0)
    codes = rng.integers(0, 4, size=(16, nchunks * CODES))
    codes[:, L:] = 0
    Q = np.array([int(x) for x in rng.integers(-(1 << 59), 1 << 59, size=nchunks * CODES)], dtype=object)
    Q[L:] = 0
    words = np.zeros((16, nchunks, 32), dtype=np.uint32)
    for l in range(16):
        for c in range(nchunks):
            for wq in range(32):
                v = 0
                for p in range(16):
                    v |= int(codes[l, c * CODES + wq * 16 + p]) << (2 * p)
                words[l, c, wq] = v
    dig = [make_digit_chunk(Q[c * CODES:(c + 1) * CODES]) for c in range(nchunks)]
    raw, na = run_subtile(words, dig, with_na=True)
    for l in range(16):
        want_raw = sum(int(codes[l, k]) * int(Q[k]) for k in range(nchunks * CODES))
        want_na = sum(int(Q[k]) for k in range(nchunks * CODES) if codes[l, k] == 3)
        got_raw = sum(int(raw[l, s]) << (8 * s) for s in range(8))
        got_na = sum(int(na[l, s]) << (8 * s) for s in range(8))
        assert got_raw == want_raw and got_na == want_na


def test_combine8_is_fp64_exact_enough():
    """combine<8>: top-down fp64 sum of slice sums == exact integer / 2^e to 1 ulp."""
    rng = np.random.default_rng(6)
    for _ in range(50):
        v = [int(x) for x in rng.integers(-(1 << 33), 1 << 33, size=8)]
        e = int(rng.integers(-20, 80))
        exact = sum(vs << (8 * s) for s, vs in enumerate(v))
        acc = 0.0
        for s in range(7, -1, -1):
            acc += np.ldexp(float(v[s]), 8 * s - e)
        want = float(np.ldexp(np.float64(exact >> 40), 40 - e)) if abs(exact) > (1 << 100) else exact / 2.0 ** e
        assert abs(acc - want) <= 4 * np.spacing(abs(want)) + 0.0
