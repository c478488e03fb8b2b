// bsg_naell.cu -- missing values of the matvecs as blocked-ELL lists (DESIGN.md "Missing values").
//
// With missing values X.y and Xt.y need, per output line l, the sum N_l = sum_{t : code(l, t) missing} v[t] of the quantised
// vector over the line's missing entries (src/bed-acc.h:98-111: a missing genotype contributes 0 after centering).  Round 1
// had two ways to get it: a second plane of IMMAs over the whole matrix (X.y 1.68 ms instead of 1.07 ms at configs[1] with
// 1 % missing: the kernel becomes issue-bound) or CSR lists gathered warp-per-line from global memory, which cost one L1
// tag lookup per missing value (0.9 ms per 1 %) and lost to the plane above 0.5 %.
//
// Here the positions are stored so that the gather runs out of SHARED memory with coalesced index loads:
//   * the contraction index is cut into chunks of 4096; the quantised vector of one chunk (4096 x int64 = 32 KB) sits in
//     shared memory while every line group consumes its entries of that chunk (double-buffered: the next chunk's slice
//     streams in with cp.async meanwhile);
//   * lines are grouped by 32; a block (group g, chunk c) stores its entries ELL style in rows of 8 entries per line -- row r
//     holds slots 8r..8r+7 of the 32 lines, lane after lane, 16-bit byte offsets into the chunk's slice, padded to the block's
//     slot count -- so one warp load is 512 contiguous bytes (a uint4 = 8 entries per lane) and each lane adds the gathered
//     values to its own line's exact sum (row sums in int64, |Q| < 2^60, then split into 32-bit halves: no overflow, order
//     free);
//   * a warp keeps the sums of its group(s) in registers across its chunks; with few groups the chunks are split over CTAs and
//     the partial sums are combined with 64-bit integer atomics (exact, order free), for X.y straight into `part`;
//   * the ORDER of a line's entries is free (integer sums), so each block is re-ordered once at build time such that the 16
//     lanes of a half-warp hit 16 different shared-memory bank pairs in every slot: a greedy edge colouring of the bipartite
//     multigraph (lane, bank = index mod 16) with slots as colours (k_recolor).  Arrival order costs 2.66 wavefronts per
//     ideal one (ncu, profiles/r02_kcorr_ncu_before.txt); the colouring needs ~4 % more slots than the longest line and
//     makes the gathers conflict free (1.01, profiles/r02_kcorr_ncu_after.txt).  The idle slots of a half-warp all read ONE
//     zero word behind the slice, the one of a bank no entry of that slot uses, so the gather loop has no predicates and no
//     per-line counts.
// ~3.1 bytes per missing value and side including padding, built once per handle from the SNP-major copy.  The matvec
// kernels then always run in their no-missing mode.  Results equal the flag-plane path up to fp64 rounding of the last
// combination (the sums themselves are exact integers).
#include <stdint.h>
#include <stdlib.h>

#include <algorithm>

#include <cub/device/device_scan.cuh>

#include "bsg_internal.cuh"

namespace bsg {
namespace naell {

constexpr int CH = 4096;      // contraction indices per chunk (16-bit local index, 32 KB of int64 in shared memory)
constexpr int GW = 4;         // line groups per warp and pass (register accumulators)
constexpr int CORR_WARPS = 16;  // two CTAs per SM
constexpr int PAD0 = CH;      // unused slots: index CH + (lane & 15) -> 16 zero words, one per 64-bit bank
constexpr int SLACK = 3;      // slots beyond the longest line of a block that the colouring may use
constexpr int RC_MAX_ROWS = 32;  // blocks with more rows of 8 keep their arrival order (padding is still rewritten)
constexpr int RC_WARPS = 4;
constexpr int RC_WARP_SMEM = RC_MAX_ROWS * 8 * 32 * 3 + (32 + 32) * 4 * 8 + 2 * RC_MAX_ROWS * 8;  // see k_recolor

__device__ __forceinline__ uint32_t na_flags(uint32_t x) { return x & (x >> 1) & 0x55555555u; }

// ---- side 1: lines = SNPs (rows of the SNP-major copy), contraction over samples ------------------------------------
// warp per (line j, chunk c): the chunk is 1024 bytes = 256 words of the line
__global__ void k_cnt_lines(const uint8_t *__restrict__ A, int64_t stride, int n, int m, int nchunks, uint16_t *__restrict__ cnt) {
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int wpl = (int)(stride / 4);
  for (int64_t it = warp; it < (int64_t)m * nchunks; it += nw) {
    const int j = (int)(it / nchunks), c = (int)(it - (int64_t)j * nchunks);
    const uint32_t *line = reinterpret_cast<const uint32_t *>(A + (int64_t)j * stride);
    int k = 0;
#pragma unroll
    for (int r = 0; r < 8; r++) {
      const int w = c * (CH / 16) + r * 32 + lane;
      k += __popc(w < wpl ? na_flags(line[w]) : 0u);  // pad slots are code 0, never missing
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) k += __shfl_xor_sync(0xffffffffu, k, o);
    if (lane == 0) cnt[((int64_t)(j >> 5) * nchunks + c) * 32 + (j & 31)] = (uint16_t)k;
  }
}
__global__ void k_fill_lines(const uint8_t *__restrict__ A, int64_t stride, int n, int m, int nchunks,
                             const long long *__restrict__ off, uint16_t *__restrict__ ent) {
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int wpl = (int)(stride / 4);
  for (int64_t it = warp; it < (int64_t)m * nchunks; it += nw) {
    const int j = (int)(it / nchunks), c = (int)(it - (int64_t)j * nchunks);
    const uint32_t *line = reinterpret_cast<const uint32_t *>(A + (int64_t)j * stride);
    uint16_t *dst = ent + (off[(int64_t)(j >> 5) * nchunks + c] * 32 + (j & 31)) * 8;  // row r of this lane at + r * 256
    int base = 0;
    for (int r = 0; r < 8; r++) {
      const int w = c * (CH / 16) + r * 32 + lane;
      uint32_t f = w < wpl ? na_flags(line[w]) : 0u;
      const int k = __popc(f);
      int pre = k;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, pre, o);
        if (lane >= o) pre += v;
      }
      const int tot = __shfl_sync(0xffffffffu, pre, 31);
      int t = base + pre - k;
      while (f) {
        const int b = __ffs(f) - 1;
        f &= f - 1;
        dst[(int64_t)(t >> 3) * 256 + (t & 7)] = (uint16_t)(((r * 32 + lane) * 16 + (b >> 1)) * 8);  // byte offset in the slice
        t++;
      }
      base += tot;
    }
  }
}

// ---- side 0: lines = samples, contraction over SNPs: a CTA owns 512 samples (32 words) x the 4096 SNP lines of a chunk ----
__global__ void __launch_bounds__(256) k_cnt_samples(const uint8_t *__restrict__ A, int64_t stride, int n, int m, int nchunks,
                                                     uint16_t *__restrict__ cnt) {
  __shared__ unsigned int sc[512];
  const int c = blockIdx.x, wb = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t = threadIdx.x; t < 512; t += 256) sc[t] = 0;
  __syncthreads();
  const int64_t byte = ((int64_t)wb * 32 + lane) * 4;
  const int j1 = min(m, (c + 1) * CH);
  if (byte + 4 <= stride) {
    for (int j = c * CH + warp; j < j1; j += 8) {
      uint32_t f = na_flags(*reinterpret_cast<const uint32_t *>(A + (int64_t)j * stride + byte));
      while (f) {
        const int b = __ffs(f) - 1;
        f &= f - 1;
        atomicAdd(&sc[lane * 16 + (b >> 1)], 1u);
      }
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < 512; t += 256) {
    const int64_t i = (int64_t)wb * 512 + t;
    if (i < n) cnt[((i >> 5) * nchunks + c) * 32 + (i & 31)] = (uint16_t)sc[t];
  }
}
__global__ void __launch_bounds__(256) k_fill_samples(const uint8_t *__restrict__ A, int64_t stride, int n, int m, int nchunks,
                                                      const long long *__restrict__ off, uint16_t *__restrict__ ent) {
  __shared__ unsigned int cur[512];
  const int c = blockIdx.x, wb = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t = threadIdx.x; t < 512; t += 256) cur[t] = 0;
  __syncthreads();
  const int64_t byte = ((int64_t)wb * 32 + lane) * 4;
  const int j1 = min(m, (c + 1) * CH);
  if (byte + 4 <= stride) {
    for (int j = c * CH + warp; j < j1; j += 8) {
      uint32_t f = na_flags(*reinterpret_cast<const uint32_t *>(A + (int64_t)j * stride + byte));
      while (f) {
        const int b = __ffs(f) - 1;
        f &= f - 1;
        const int sl = lane * 16 + (b >> 1);
        const int64_t i = (int64_t)wb * 512 + sl;
        if (i < n) {
          const unsigned int t = atomicAdd(&cur[sl], 1u);  // any order: the sums are integers
          ent[((off[(i >> 5) * nchunks + c] + (t >> 3)) * 32 + (i & 31)) * 8 + (t & 7)] = (uint16_t)((j - c * CH) * 8);
        }
      }
    }
  }
}

// rows of 8 entries needed by the longest line of every block (32 lines x one chunk)
__global__ void k_block_max(const uint16_t *__restrict__ cnt, int64_t nblocks, long long *__restrict__ blk) {
  for (int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; b <= nblocks; b += (int64_t)gridDim.x * blockDim.x) {
    int mx = 0;
    if (b < nblocks)
      for (int r = 0; r < 32; r++) mx = max(mx, (int)cnt[b * 32 + r]);
    blk[b] = mx ? (mx + SLACK + 7) >> 3 : 0;
  }
}

__device__ __forceinline__ unsigned long long slot_mask(int S, int w4) {  // slots w4 * 64 .. w4 * 64 + 63 that exist (< S)
  const int nb = S - w4 * 64;
  return nb >= 64 ? ~0ull : (nb > 0 ? ((1ull << nb) - 1ull) : 0ull);
}

// Re-order the entries of every block (32 lines x one chunk), one warp per block: slot c of lane l gets an entry whose
// bank (index mod 16: the 64-bit word's bank pair) differs from the banks the other 15 lanes of the half-warp use in slot c.
// Greedy edge colouring: entries are taken line by line, k-th entry of lane 0, 1, .., 15 in turn (the two half-warps run
// side by side), each takes the smallest slot free for its lane and its bank; if none is left below the block's slot
// count, any slot free for the lane (a conflict, never an error).  Unused slots are rewritten to the zero words.
__global__ void __launch_bounds__(RC_WARPS * 32)
    k_recolor(const uint16_t *__restrict__ cnt, const long long *__restrict__ off, uint16_t *__restrict__ ent, int64_t nblocks,
              int recolor) {
  extern __shared__ __align__(16) unsigned char rc_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, half = lane >> 4, l16 = lane & 15;
  // per warp: entries [RC_MAX_ROWS * 8][32] u16, slot of entry [RC_MAX_ROWS * 8][32] u8, masks lane_used[32][4],
  // bank_used[2][16][4], free bank of every slot padf[2][RC_MAX_ROWS * 8] u8
  constexpr int S_MAX = RC_MAX_ROWS * 8;
  unsigned char *base = rc_smem + (size_t)warp * RC_WARP_SMEM;
  uint16_t *e = reinterpret_cast<uint16_t *>(base);
  uint8_t *col = base + S_MAX * 32 * 2;
  unsigned long long *lane_used = reinterpret_cast<unsigned long long *>(base + S_MAX * 32 * 3);
  unsigned long long *bank_used = lane_used + 32 * 4;
  uint8_t *padf = reinterpret_cast<uint8_t *>(bank_used + 32 * 4);
  for (int64_t b = (int64_t)blockIdx.x * RC_WARPS + warp; b < nblocks; b += (int64_t)gridDim.x * RC_WARPS) {
    const long long o0 = off[b];
    const int nrows = (int)(off[b + 1] - o0);
    if (nrows == 0) continue;
    const int S = nrows * 8, deg = cnt[b * 32 + lane];
    uint4 *rows = reinterpret_cast<uint4 *>(ent) + o0 * 32 + lane;
    if (nrows > RC_MAX_ROWS || !recolor) {  // too long for the staging buffers: arrival order, padding rewritten
      for (int r = 0; r < nrows; r++) {
        uint4 v = rows[(int64_t)r * 32];
        uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int q8 = 0; q8 < 8; q8++)
          if (r * 8 + q8 >= deg) {
            const uint32_t m = 0xFFFFu << (16 * (q8 & 1));
            w[q8 >> 1] = (w[q8 >> 1] & ~m) | ((uint32_t)((PAD0 + l16) * 8) << (16 * (q8 & 1)));
          }
        rows[(int64_t)r * 32] = make_uint4(w[0], w[1], w[2], w[3]);
      }
      continue;
    }
    __syncwarp();
    for (int r = 0; r < nrows; r++) {
      const uint4 v = rows[(int64_t)r * 32];
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int q8 = 0; q8 < 8; q8++) e[(r * 8 + q8) * 32 + lane] = (uint16_t)((w[q8 >> 1] >> (16 * (q8 & 1))) & 0xFFFFu);
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
      lane_used[lane * 4 + k] = 0;
      bank_used[lane * 4 + k] = 0;  // 2 halves x 16 banks = 32 mask rows
    }
    int maxdeg = deg;
#pragma unroll
    for (int o = 16; o; o >>= 1) maxdeg = max(maxdeg, __shfl_xor_sync(0xffffffffu, maxdeg, o));
    __syncwarp();
    for (int k = 0; k < maxdeg; k++) {
      for (int turn = 0; turn < 16; turn++) {
        if (l16 == turn && k < deg) {
          const int bank = (e[k * 32 + lane] >> 3) & 15;
          unsigned long long *lu = lane_used + lane * 4, *bu = bank_used + (half * 16 + bank) * 4;
          int c = -1;
          for (int w4 = 0; w4 < 4 && c < 0; w4++) {
            const unsigned long long freem = ~(lu[w4] | bu[w4]) & slot_mask(S, w4);
            if (freem) c = w4 * 64 + __ffsll((long long)freem) - 1;
          }
          if (c < 0) {  // no conflict-free slot left: any slot of the lane (deg <= S - SLACK, so one exists)
            for (int w4 = 0; w4 < 4 && c < 0; w4++) {
              const unsigned long long freem = ~lu[w4] & slot_mask(S, w4);
              if (freem) c = w4 * 64 + __ffsll((long long)freem) - 1;
            }
          }
          lu[c >> 6] |= 1ull << (c & 63);
          bu[c >> 6] |= 1ull << (c & 63);
          col[k * 32 + lane] = (uint8_t)c;
        }
        __syncwarp();
      }
    }
    // unused slots: all lanes of a half-warp that idle in slot c read the SAME zero word (a broadcast), the one of a bank no
    // entry of the slot uses -- a slot with an idle lane has at most 15 entries, so a free bank exists
    for (int c = l16; c < S; c += 16) {
      int f = 0;
      for (int bk = 0; bk < 16; bk++)
        if (!((bank_used[(half * 16 + bk) * 4 + (c >> 6)] >> (c & 63)) & 1ull)) {
          f = bk;
          break;
        }
      padf[half * S_MAX + c] = (uint8_t)f;
    }
    __syncwarp();
    for (int r = 0; r < nrows; r++) {
      uint32_t w[4];
#pragma unroll
      for (int q8 = 0; q8 < 8; q8 += 2)
        w[q8 >> 1] = (uint32_t)((PAD0 + padf[half * S_MAX + r * 8 + q8]) * 8) | ((uint32_t)((PAD0 + padf[half * S_MAX + r * 8 + q8 + 1]) * 8) << 16);
      rows[(int64_t)r * 32] = make_uint4(w[0], w[1], w[2], w[3]);
    }
    __syncwarp();
    uint16_t *mine = ent + (o0 * 32 + lane) * 8;  // slot c of this lane: mine[(c >> 3) * 256 + (c & 7)]
    for (int k = 0; k < deg; k++) {
      const int c = col[k * 32 + lane];
      mine[(int64_t)(c >> 3) * 256 + (c & 7)] = e[k * 32 + lane];
    }
    __syncwarp();
  }
}

// N[line] = sum of Q over the line's missing entries, as (low 32-bit halves, high halves) exact 64-bit sums.
// grid = (group CTAs, chunk splits), two CTAs of 16 warps per SM: a CTA walks its range of chunks -- the 32 KB vector slice
// of chunk c + 1 streams into the second shared-memory buffer (cp.async) while every warp consumes the block(s) of its line
// group(s) for chunk c; one barrier per chunk.  A warp's blocks of consecutive chunks are contiguous in memory, so it reads
// one sequential stream of index rows and asks L2 for the next 4 KB ahead of use.  With few groups the chunks are split
// over several CTAs (the partial sums are then combined with 64-bit integer atomics: exact, order free).
// Every slot of a block is gathered (unused ones read a zero word): no per-line counts, no predicates.
// dst_stride = 2: outN[line][2] (k_apply places them); dst_stride = 16: straight into part[line][8], part[line][12]
// (identity line order, `part` zeroed by the matvec launcher), always with atomics.
constexpr int SQ_WORDS = CH + 16;
constexpr int CORR_SMEM = 2 * SQ_WORDS * (int)sizeof(long long);

template <int GWT>
__global__ void __launch_bounds__(CORR_WARPS * 32, 2)
    k_corr(const long long *__restrict__ off, const uint16_t *__restrict__ ent, int nchunks, int ngroups, int gw,
           const long long *__restrict__ Q, int64_t qlen, long long *__restrict__ outN, int dst_stride, int dst_hi, int nlines) {
  extern __shared__ __align__(16) long long sq_all[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t W = (int64_t)blockIdx.x * CORR_WARPS + warp, TW = (int64_t)gridDim.x * CORR_WARPS;
  const int cper = (nchunks + gridDim.y - 1) / gridDim.y;
  const int c0 = blockIdx.y * cper, c1 = min(nchunks, c0 + cper);
  const bool atomic = gridDim.y > 1 || dst_stride != 2;
  const int npass = (int)((ngroups + TW * gw - 1) / (TW * gw));
  if (threadIdx.x < 32) sq_all[(threadIdx.x >> 4) * SQ_WORDS + CH + (threadIdx.x & 15)] = 0;
  const uint32_t sq_base = (uint32_t)__cvta_generic_to_shared(sq_all);
  auto stage = [&](int c, int buf) {  // vector slice of chunk c -> buffer buf; entries past the end are zero-filled
    if ((int64_t)(c + 1) * CH <= qlen) {  // whole chunk inside the vector: plain 16-byte copies
      const long long *src = Q + (int64_t)c * CH + 2 * threadIdx.x;
      const uint32_t dst = sq_base + (uint32_t)((buf * SQ_WORDS + 2 * threadIdx.x) * 8);
#pragma unroll
      for (int u = 0; u < CH / 2 / (CORR_WARPS * 32); u++)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + u * CORR_WARPS * 32 * 16), "l"(src + u * CORR_WARPS * 32 * 2)
                     : "memory");
      asm volatile("cp.async.commit_group;" ::: "memory");
      return;
    }
    for (int t = threadIdx.x; t < CH / 2; t += CORR_WARPS * 32) {
      const int64_t q = (int64_t)c * CH + 2 * t;
      const int64_t left = (qlen - q) * 8;
      const int bytes = left >= 16 ? 16 : (left > 0 ? (int)left : 0);
      const long long *src = bytes > 0 ? Q + q : Q;
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(sq_base + (uint32_t)((buf * SQ_WORDS + 2 * t) * 8)), "l"(src),
                   "r"(bytes)
                   : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  for (int pass = 0; pass < npass; pass++) {
    // groups are dealt round-robin over the warps of the grid: group (pass * gw + k) * TW + W
    long long lo[GWT], hi[GWT];
#pragma unroll
    for (int k = 0; k < GWT; k++) lo[k] = hi[k] = 0;
    __syncthreads();  // the buffers of the previous pass are no longer read
    if (c0 < c1) stage(c0, 0);
    for (int c = c0; c < c1; c++) {
      const int buf = (c - c0) & 1;
      const unsigned char *sq = reinterpret_cast<const unsigned char *>(sq_all + buf * SQ_WORDS);
      // entries are byte offsets into the slice.  |Q| < 2^60, so the 8 values of a row add up without overflow; the row
      // sum is then split into its 32-bit halves (exact over any number of rows)
      auto consume = [&](const uint4 &v, long long &l, long long &hh) {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        long long q[8];
#pragma unroll
        for (int q8 = 0; q8 < 8; q8++)
          q[q8] = *reinterpret_cast<const long long *>(sq + ((q8 & 1) ? (w[q8 >> 1] >> 16) : (w[q8 >> 1] & 0xFFFFu)));
        const long long rs = ((q[0] + q[1]) + (q[2] + q[3])) + ((q[4] + q[5]) + (q[6] + q[7]));
        l += (long long)(unsigned int)(rs & 0xFFFFFFFFll);
        hh += rs >> 32;
      };
      // GWT == 1 (few groups): the block's offsets and first 8 rows are requested BEFORE the wait for the vector slice
      uint4 pre[GWT == 1 ? 8 : 1];
      int pre_nrows = 0;
      const uint4 *pre_e = nullptr;
      if (GWT == 1) {
        const int64_t g = (int64_t)pass * TW + W;
        if (g < ngroups) {
          const int64_t blk = g * nchunks + c;
          const long long o0 = off[blk];
          pre_nrows = (int)(off[blk + 1] - o0);
          pre_e = reinterpret_cast<const uint4 *>(ent) + o0 * 32 + lane;
#pragma unroll
          for (int u = 0; u < 8; u++) pre[u] = (u < pre_nrows) ? __ldg(pre_e + (int64_t)u * 32) : make_uint4(0, 0, 0, 0);
          if (c + 1 < c1)  // the rows of the next chunk follow directly: 4 KB ahead into L2
            asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char *>(ent) + (o0 + pre_nrows) * 512 + lane * 128));
        }
      }
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncthreads();  // slice c is complete for every thread, and nobody still reads the other buffer (slice c - 1)
      if (c + 1 < c1) stage(c + 1, buf ^ 1);
      if (GWT == 1) {
#pragma unroll
        for (int u = 0; u < 8; u++)
          if (u < pre_nrows) consume(pre[u], lo[0], hi[0]);
        for (int r0 = 8; r0 < pre_nrows; r0 += 4) {
          uint4 v[4];
#pragma unroll
          for (int u = 0; u < 4; u++) v[u] = (r0 + u < pre_nrows) ? __ldg(pre_e + (int64_t)(r0 + u) * 32) : make_uint4(0, 0, 0, 0);
#pragma unroll
          for (int u = 0; u < 4; u++)
            if (r0 + u < pre_nrows) consume(v[u], lo[0], hi[0]);
        }
        continue;
      }
#pragma unroll
      for (int k = 0; k < GWT; k++) {
        const int64_t g = ((int64_t)pass * gw + k) * TW + W;
        if (k < gw && g < ngroups) {  // warp-uniform
          const int64_t blk = g * nchunks + c;
          const long long o0 = off[blk];
          const int nrows = (int)(off[blk + 1] - o0);  // rows of 8 entries per line (warp-uniform)
          const uint4 *e = reinterpret_cast<const uint4 *>(ent) + o0 * 32 + lane;
          for (int r0 = 0; r0 < nrows; r0 += 4) {  // up to 4 rows = 2 KB per warp in flight
            uint4 v[4];
#pragma unroll
            for (int u = 0; u < 4; u++) v[u] = (r0 + u < nrows) ? __ldg(e + (int64_t)(r0 + u) * 32) : make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int u = 0; u < 4; u++)
              if (r0 + u < nrows) consume(v[u], lo[k], hi[k]);
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < GWT; k++) {
      const int64_t g = ((int64_t)pass * gw + k) * TW + W;
      if (k < gw && g < ngroups && g * 32 + lane < nlines) {
        long long *dst = outN + (g * 32 + lane) * dst_stride;
        if (atomic) {
          if (lo[k]) atomicAdd(reinterpret_cast<unsigned long long *>(dst), (unsigned long long)lo[k]);
          if (hi[k]) atomicAdd(reinterpret_cast<unsigned long long *>(dst + dst_hi), (unsigned long long)hi[k]);
        } else {
          dst[0] = lo[k];
          dst[dst_hi] = hi[k];
        }
      }
    }
  }
}

// part[l][8] = low sum, part[l][12] = high sum (x 2^32 = 256^4): the finish kernels read the eight NA slices as
// sum_s part[l][8 + s] * 256^s, which this representation satisfies exactly
__global__ void k_apply(const long long *__restrict__ outN, const int *__restrict__ lines, int nlines, long long *__restrict__ part) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= nlines) return;
  const int64_t phys = lines ? lines[l] : l;
  part[(int64_t)l * 16 + 8] = outN[phys * 2];
  part[(int64_t)l * 16 + 12] = outN[phys * 2 + 1];
}

static int grid_cap(int64_t work, int block) { return (int)std::max<int64_t>(1, std::min<int64_t>((work + block - 1) / block, 132 * 32)); }

}  // namespace naell

// Build (once) the blocked-ELL lists of both sides.  Returns true when resident; false = use the flag-plane kernels
// (no missing value, rate above BSG_NA_LIST_MAX_RATE, not enough memory, BSG_NA_LISTS=0).
bool na_ell_ready(bsg_bed *h) {
  using namespace naell;
  if (h->na_ell != 0) return h->na_ell == 1;
  h->na_ell = -1;
  if (!h->has_na) return false;
  const char *ev = getenv("BSG_NA_LISTS");
  if (ev && ev[0] == '0') return false;
  double max_rate = 0.04;  // above ~4 % the lists (2 x 2 bytes x 1.3 per missing value) approach the size of the matrix itself
  if (const char *er = getenv("BSG_NA_LIST_MAX_RATE")) max_rate = atof(er);
  cudaStream_t s = h->stream;
  const int n = h->n, m = h->m;
  // missing values in total (exact counts cached at staging)
  long long nnz = 0;
  {
    std::vector<int32_t> c4((size_t)m * 4);
    if (cudaMemcpyAsync(c4.data(), h->cntA, c4.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
        cudaStreamSynchronize(s) != cudaSuccess) {
      cudaGetLastError();
      return false;
    }
    for (int j = 0; j < m; j++) nnz += c4[4 * (size_t)j + 3];
  }
  if (nnz <= 0 || (double)nnz > max_rate * (double)n * (double)m) return false;
  bool ok = true;
  for (int side = 0; side < 2 && ok; side++) {
    const int nlines = side == 0 ? n : m, qlen = side == 0 ? m : n;
    const int nchunks = (qlen + CH - 1) / CH, ngroups = (nlines + 31) / 32;
    const int64_t nblocks = (int64_t)ngroups * nchunks;
    uint16_t *cnt = nullptr, *ent = nullptr;
    long long *blk = nullptr, *off = nullptr, *outN = nullptr;
    void *tmp = nullptr;
    do {
      ok = false;
      size_t fr = 0, tot = 0;
      cudaMemGetInfo(&fr, &tot);
      const size_t meta = (size_t)nblocks * 64 + (size_t)(nblocks + 1) * 16 + (size_t)ngroups * 32 * 16;
      if (meta + (size_t)(3.2 * (double)nnz) + ((size_t)2 << 30) > fr) break;  // expected entries incl. padding
      if (cudaMalloc((void **)&cnt, (size_t)nblocks * 32 * sizeof(uint16_t)) != cudaSuccess ||
          cudaMalloc((void **)&blk, (size_t)(nblocks + 1) * sizeof(long long)) != cudaSuccess ||
          cudaMalloc((void **)&off, (size_t)(nblocks + 1) * sizeof(long long)) != cudaSuccess ||
          cudaMalloc((void **)&outN, (size_t)ngroups * 32 * 2 * sizeof(long long)) != cudaSuccess)
        break;
      if (cudaMemsetAsync(cnt, 0, (size_t)nblocks * 32 * sizeof(uint16_t), s) != cudaSuccess) break;
      if (side == 1) {
        k_cnt_lines<<<grid_cap((int64_t)m * nchunks * 32, 256), 256, 0, s>>>(h->A, h->strideA, n, m, nchunks, cnt);
      } else {
        dim3 grid((unsigned)nchunks, (unsigned)((h->strideA / 4 + 31) / 32));
        k_cnt_samples<<<grid, 256, 0, s>>>(h->A, h->strideA, n, m, nchunks, cnt);
      }
      k_block_max<<<grid_cap(nblocks + 1, 256), 256, 0, s>>>(cnt, nblocks, blk);
      size_t tb = 0;
      cub::DeviceScan::ExclusiveSum(nullptr, tb, blk, off, (int)(nblocks + 1), s);
      if (cudaMalloc(&tmp, tb ? tb : 16) != cudaSuccess) break;
      cub::DeviceScan::ExclusiveSum(tmp, tb, blk, off, (int)(nblocks + 1), s);
      long long rows = 0;
      if (cudaMemcpyAsync(&rows, off + nblocks, sizeof rows, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
          cudaStreamSynchronize(s) != cudaSuccess)
        break;
      cudaMemGetInfo(&fr, &tot);
      if ((size_t)rows * 512 + ((size_t)2 << 30) > fr) break;
      if (cudaMalloc((void **)&ent, std::max<size_t>((size_t)rows * 512, 512) + 4096) != cudaSuccess) break;  // + the L2 look-ahead of k_corr
      if (cudaMemsetAsync(ent, 0, std::max<size_t>((size_t)rows * 512, 512), s) != cudaSuccess) break;
      if (side == 1) {
        k_fill_lines<<<grid_cap((int64_t)m * nchunks * 32, 256), 256, 0, s>>>(h->A, h->strideA, n, m, nchunks, off, ent);
      } else {
        dim3 grid((unsigned)nchunks, (unsigned)((h->strideA / 4 + 31) / 32));
        k_fill_samples<<<grid, 256, 0, s>>>(h->A, h->strideA, n, m, nchunks, off, ent);
      }
      {
        const char *er = getenv("BSG_NA_RECOLOR");  // 0: keep the arrival order (measurement switch); padding is rewritten either way
        const size_t smem = (size_t)RC_WARPS * RC_WARP_SMEM;
        if (cudaFuncSetAttribute(k_recolor, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) break;
        k_recolor<<<grid_cap(nblocks * 32, RC_WARPS * 32), RC_WARPS * 32, smem, s>>>(cnt, off, ent, nblocks, (er && er[0] == '0') ? 0 : 1);
      }
      count_launch(5);
      if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) break;
      ok = true;
    } while (0);
    cudaGetLastError();
    cudaFree(tmp);
    cudaFree(blk);
    if (!ok) {
      cudaFree(cnt);
      cudaFree(off);
      cudaFree(ent);
      cudaFree(outN);
      break;
    }
    cudaFree(cnt);  // only the build needs the per-line counts
    h->ellCnt[side] = nullptr;
    h->ellOff[side] = off;
    h->ellEnt[side] = ent;
    h->ellOut[side] = outN;
    h->ellChunks[side] = nchunks;
    h->ellGroups[side] = ngroups;
  }
  if (!ok) {
    for (int side = 0; side < 2; side++) {
      cudaFree(h->ellCnt[side]);
      cudaFree(h->ellOff[side]);
      cudaFree(h->ellEnt[side]);
      cudaFree(h->ellOut[side]);
      h->ellCnt[side] = nullptr;
      h->ellOff[side] = nullptr;
      h->ellEnt[side] = nullptr;
      h->ellOut[side] = nullptr;
    }
    return false;
  }
  h->na_nnz = nnz;
  h->na_ell = 1;
  return true;
}

// NA-plane sums of `nlines` output lines (side 0: lines = samples, Q over the SNPs; side 1: lines = SNPs, Q over the
// samples; lines[l] = physical line of output l, null = identity) written into part[l][8 ..]
int na_ell_correction(bsg_bed *h, int side, const int *lines, int nlines, const long long *Q, long long *part, cudaStream_t s) {
  using namespace naell;
  if (nlines <= 0) return BSG_OK;
  int nsm = 132;
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, h->device);
  const int ngroups = h->ellGroups[side], nchunks = h->ellChunks[side];
  // two CTAs of 16 warps per SM: few groups -> one group per warp and the chunks split over several CTAs (one resident
  // wave, at least ~8 chunks each); many groups -> up to GW groups per warp
  const int64_t cta_slots = 2 * (int64_t)nsm, warp_slots = cta_slots * CORR_WARPS;
  int gw = (int)std::min<int64_t>(GW, std::max<int64_t>(1, (ngroups + warp_slots - 1) / warp_slots));
  int gctas = (int)std::min<int64_t>(cta_slots, ((int64_t)ngroups + (int64_t)CORR_WARPS * gw - 1) / ((int64_t)CORR_WARPS * gw));
  gctas = std::max(gctas, 1);
  int nsplit = std::max(1, std::min(std::max(1, nchunks / 8), (int)(cta_slots / gctas)));
  BSG_CUDA(cudaFuncSetAttribute(k_corr<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, CORR_SMEM));  // per device
  BSG_CUDA(cudaFuncSetAttribute(k_corr<GW>, cudaFuncAttributeMaxDynamicSharedMemorySize, CORR_SMEM));
  // identity line order (X.y: every sample): the sums go straight into part[line][8] / [12] (zeroed by the launcher of the
  // matvec kernel) with integer atomics; otherwise into outN and k_apply places the selected lines
  const bool direct = lines == nullptr;
  long long *dst = direct ? part + 8 : h->ellOut[side];
  const int dst_stride = direct ? 16 : 2, dst_hi = direct ? 4 : 1;
  const int dst_lines = direct ? nlines : ngroups * 32;
  if (!direct && nsplit > 1) BSG_CUDA(cudaMemsetAsync(h->ellOut[side], 0, (size_t)ngroups * 32 * 2 * sizeof(long long), s));
  dim3 grid((unsigned)gctas, (unsigned)nsplit);
  if (gw == 1)
    k_corr<1><<<grid, CORR_WARPS * 32, CORR_SMEM, s>>>(h->ellOff[side], h->ellEnt[side], nchunks, ngroups, gw, Q,
                                               side == 0 ? h->m : h->n, dst, dst_stride, dst_hi, dst_lines);
  else
    k_corr<GW><<<grid, CORR_WARPS * 32, CORR_SMEM, s>>>(h->ellOff[side], h->ellEnt[side], nchunks, ngroups, gw, Q,
                                                side == 0 ? h->m : h->n, dst, dst_stride, dst_hi, dst_lines);
  if (!direct) k_apply<<<(nlines + 255) / 256, 256, 0, s>>>(h->ellOut[side], lines, nlines, part);
  count_launch(2);
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

}  // namespace bsg
