// bsg_grid.cu -- the greedy clumping passes: bed_clumping_chr (src/clumping-bed.cpp:11-91), clumping_chr
// (src/clumping.cpp:10-91) and snp_grid_clumping (R/SCT.R:32-151), every clumping_chr_cached call of one chromosome in one call.
//
// Each pass reads one byte per pair of the band (bsg_cor.cu's pair_band): a conflict flag, or the number of the call's sorted
// distinct thresholds the pair's r2 exceeds (r2 > thr_t  <=>  level > t).  One instance is a (subset, size, threshold index);
// k_grid_round resolves every instance of a call in the same device rounds, the instance on the grid's y dimension and a
// subset -> band column map.  The clumpings of one chromosome are the one instance of the identity subset.
//
// The grid: the reference runs clumping_chr_cached (src/clumping-cached.cpp:11-110) once per (thr.imp, group) subset and grid
// point (thr.r2, base.size), with windows of 1000 * base.size / thr.r2 bp and a sparse r2 cache passed between the calls.  The
// statistic of a pair depends only on the two columns and their sumX / denoX, so here it is computed once per pair of the
// chromosome, over the union window (build_window(.., both = true)) at the largest size.
//
// Dosage handles (bsg_dosage_scale D > 0) get the grid's pair sums as exact integers on the tensor pipe: with q = D * value in
// 0..255 (NA codes 0), S = sum_i q_i q'_i comes from IMMA.16832.U8.U8 tiles and xySum = S / D^2.  A product reaches
// 255^2 = 65,025, so the int32 accumulators are drained into int64 every 32,768 samples (32,768 * 65,025 < 2^31): exact for
// any n (S < 2^53 up to 1.3e11 samples).
#include <math.h>

#include <algorithm>
#include <vector>

#include "bsg_gram.cuh"
#include "bsg_internal.cuh"

namespace bsg {
namespace grid {

constexpr int DTM = 128, DTN = 64;  // line pairs per CTA: 8 warps (4 x 2) of 32 x 32
constexpr int DCH = 64;             // bytes (samples) per line per step: one LDG.128 per lane
constexpr int DRAIN = 512;          // steps per int32 span: 512 * 64 = 32,768 samples
constexpr int SMEM = 256 * 32 * (int)sizeof(long long);

struct DTile {
  int i0, j0;  // first window owner j0, first partner j
};

// Q line c = the D-scaled bytes of (rows, cols[c]), pads 0; na[c] = the line holds an NA code in the selected rows
__global__ void k_dos_compact(const uint8_t *__restrict__ raw, int64_t n_tot, const uint8_t *__restrict__ lut,
                              const int *__restrict__ rows, int nr, const int *__restrict__ cols, int nc,
                              uint8_t *__restrict__ Q, int64_t stride, uint8_t *__restrict__ na) {
  __shared__ uint8_t sl[512];  // [0, 256): q of each code, [256, 512): 1 for an NA code
  for (int i = threadIdx.x; i < 512; i += blockDim.x) sl[i] = lut[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; c < nc; c += nw) {
    const uint8_t *col = raw + (int64_t)(cols ? cols[c] : (int)c) * n_tot;
    uint32_t *out = reinterpret_cast<uint32_t *>(Q + c * stride);
    int bad = 0;
    for (int64_t w = lane; w < stride / 4; w += 32) {
      uint32_t v = 0;
#pragma unroll
      for (int p = 0; p < 4; p++) {
        const int64_t i = 4 * w + p;
        if (i < nr) {
          const uint8_t b = col[rows ? rows[i] : (int)i];
          v |= (uint32_t)sl[b] << (8 * p);
          bad |= sl[256 + b];
        }
      }
      out[w] = v;
    }
    bad = __any_sync(0xffffffffu, bad);
    if (lane == 0) na[c] = (uint8_t)bad;
  }
}

// One 128 x 64 tile of line pairs (j0 = i0 + row, j = j0 + col) over all samples, then the level of every pair of the tile
// that lies in the band: j < j0 and j0 - 1 - j < wlen[j0].  Fragments come straight from global memory: lane (g, q) holds
// bytes 16 q .. 16 q + 15 of a 64-byte step of its lines, words (0, 1) feed one MMA and words (2, 3) the next; A and B use
// the same byte -> k-slot map, so the sum over the step is complete.
__global__ void __launch_bounds__(256, 2) k_dos_pairs(const uint8_t *__restrict__ Q, int64_t stride, int nc, int nsteps,
                                                       const DTile *__restrict__ tiles, const int *__restrict__ wlen,
                                                       const long long *__restrict__ boff, const uint8_t *__restrict__ na,
                                                       const double *__restrict__ sumX, const double *__restrict__ denoX,
                                                       int nr, double d2, const double *__restrict__ levels, int nlev,
                                                       uint8_t *__restrict__ lev) {
  extern __shared__ long long s64[];  // [32][256]: element e of thread t at e * 256 + t
  const DTile t = tiles[blockIdx.x];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int wm = warp >> 1, wn = warp & 1;
  const uint8_t *pa[4], *pb[4];
#pragma unroll
  for (int l = 0; l < 4; l++) {
    const int la = min(t.i0 + wm * 32 + (l >> 1) * 16 + g + 8 * (l & 1), nc - 1);
    const int lb = min(t.j0 + wn * 32 + l * 8 + g, nc - 1);
    pa[l] = Q + (int64_t)la * stride + 16 * q;
    pb[l] = Q + (int64_t)lb * stride + 16 * q;
  }
#pragma unroll
  for (int e = 0; e < 32; e++) s64[e * 256 + threadIdx.x] = 0;
  for (int c0 = 0; c0 < nsteps; c0 += DRAIN) {
    int acc[2][4][4];
#pragma unroll
    for (int mt = 0; mt < 2; mt++)
#pragma unroll
      for (int nt = 0; nt < 4; nt++)
#pragma unroll
        for (int k = 0; k < 4; k++) acc[mt][nt][k] = 0;
    const int c1 = min(nsteps, c0 + DRAIN);
#pragma unroll 2
    for (int c = c0; c < c1; c++) {
      const int64_t off = (int64_t)c * DCH;
      uint4 a[4], b[4];
#pragma unroll
      for (int l = 0; l < 4; l++) a[l] = gram::ldg128(pa[l] + off);
#pragma unroll
      for (int l = 0; l < 4; l++) b[l] = gram::ldg128(pb[l] + off);
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const uint32_t w0 = h ? 2 : 0;
#pragma unroll
        for (int mt = 0; mt < 2; mt++) {
          const uint32_t *r0 = &a[2 * mt].x, *r1 = &a[2 * mt + 1].x;
#pragma unroll
          for (int nt = 0; nt < 4; nt++) {
            const uint32_t *bw = &b[nt].x;
            gram::mma_u8u8(acc[mt][nt], r0[w0], r1[w0], r0[w0 + 1], r1[w0 + 1], bw[w0], bw[w0 + 1]);
          }
        }
      }
    }
#pragma unroll
    for (int mt = 0; mt < 2; mt++)
#pragma unroll
      for (int nt = 0; nt < 4; nt++)
#pragma unroll
        for (int k = 0; k < 4; k++) s64[(mt * 16 + nt * 4 + k) * 256 + threadIdx.x] += acc[mt][nt][k];
  }
#pragma unroll
  for (int mt = 0; mt < 2; mt++)
#pragma unroll
    for (int nt = 0; nt < 4; nt++)
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int j0 = t.i0 + wm * 32 + mt * 16 + g + 8 * (k >> 1);
        const int j = t.j0 + wn * 32 + nt * 8 + 2 * q + (k & 1);
        if (j0 >= nc || j >= j0 || j0 - 1 - j >= wlen[j0]) continue;
        // src/clumping.cpp:66-73 with the exact xySum; an NA code makes the reference's r2 NA, never > thr
        const double xySum = (double)s64[(mt * 16 + nt * 4 + k) * 256 + threadIdx.x] / d2;
        const double num = xySum - sumX[j] * sumX[j0] / nr;
        const double r2 = num * num / (denoX[j] * denoX[j0]);
        int l = 0;
        if (!na[j] && !na[j0])
          for (int u = 0; u < nlev; u++) l += r2 > levels[u];
        lev[boff[j0] + (j0 - 1 - j)] = (uint8_t)l;
      }
}

// One round of every instance's greedy pass, one warp per undecided subset column; instance in0 + blockIdx.y (subset, size,
// threshold index).  Without a loop over instances the kernel fits 32 registers, so 8 blocks of 256 threads share an SM:
// the rounds are latency bound and need those warps.  The sequential pass (src/clumping-bed.cpp:37-88) visits the variants by decreasing
// priority and keeps c0 unless an ALREADY KEPT variant of its window conflicts with it.  Only higher-priority neighbours
// matter, so c0's fate is known as soon as theirs is: REMOVED if one of its conflicting higher-priority neighbours is KEPT,
// KEPT if all of them are REMOVED (or there is none), otherwise undecided for this round.  By induction on the rank this
// gives the sequential result; the highest-ranked undecided variant is decided in every round, dense LD blocks resolve in
// two or three rounds.  Neighbours follow which_to_check (src/clumping-utils.h:12-43) literally on the subset's positions at
// the instance's size: left while pos[j] >= pos[j0] - size, right while pos[j] <= pos[j0] + size, each scan stopping at its
// first failure like the `break` of the sequential loops.  A pair conflicts at threshold index ti when its level exceeds ti.
// col == nullptr: the identity column map (one subset of every band column).
__global__ void k_grid_round(const uint8_t *__restrict__ lev, const long long *__restrict__ boff, const int *__restrict__ wlen,
                             const double *__restrict__ pos, const int *__restrict__ sub_off, const int *__restrict__ col,
                             const int *__restrict__ rank, const int *__restrict__ inst_sub, const double *__restrict__ inst_size,
                             const int *__restrict__ inst_lev, const long long *__restrict__ inst_state, int in0, int *state,
                             int *n_undecided) {
  const int lane = threadIdx.x & 31;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  const int in = in0 + blockIdx.y;
  const int s = inst_sub[in], base = sub_off[s], L = sub_off[s + 1] - base, ti = inst_lev[in];
  const double size = inst_size[in];
  int *st = state + inst_state[in];
  for (int c0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c0 < L; c0 += nw) {
    if (st[c0] != -1) continue;  // warp-uniform
    const int j0 = col ? col[base + c0] : c0, k = rank[base + c0], wl = wlen[j0];
    const long long b0 = boff[j0];
    const double pos_min = pos[j0] - size, pos_max = pos[j0] + size;
    int kept = 0, undec = 0;
    for (int c1 = c0 - 1; c1 >= 0; c1 -= 32) {  // left: pairs of j0's own window
      const int c = c1 - lane;
      bool ok = c >= 0;
      int j = 0;
      if (ok) {
        j = col ? col[base + c] : c;
        ok = pos[j] >= pos_min && j0 - 1 - j < wl;
      }
      const unsigned stop = __ballot_sync(0xffffffffu, !ok);
      const bool live = stop ? lane < __ffs(stop) - 1 : true;
      if (live && rank[base + c] < k && lev[b0 + (j0 - 1 - j)] > ti) {
        const int v = st[c];
        kept |= v == 1;
        undec |= v == -1;
      }
      if (stop) break;
    }
    for (int c1 = c0 + 1; c1 < L; c1 += 32) {  // right: j0 sits in the window of j
      const int c = c1 + lane;
      bool ok = c < L;
      int j = 0;
      if (ok) {
        j = col ? col[base + c] : c;
        ok = pos[j] <= pos_max && j - 1 - j0 < wlen[j];
      }
      const unsigned stop = __ballot_sync(0xffffffffu, !ok);
      const bool live = stop ? lane < __ffs(stop) - 1 : true;
      if (live && rank[base + c] < k && lev[boff[j] + (j - 1 - j0)] > ti) {
        const int v = st[c];
        kept |= v == 1;
        undec |= v == -1;
      }
      if (stop) break;
    }
    kept = __any_sync(0xffffffffu, kept);
    undec = __any_sync(0xffffffffu, undec);
    if (lane == 0) {
      if (kept)
        st[c0] = 0;
      else if (!undec)
        st[c0] = 1;
      else
        atomicAdd(n_undecided, 1);
    }
  }
}

}  // namespace grid

int dosage_pair_levels(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, int nlev, const PairBand &band) {
  using namespace grid;
  if (nc <= 0 || band.total == 0) return BSG_OK;
  cudaStream_t s = h->stream;
  std::vector<uint8_t> lut(512, 0);
  for (int b = 0; b < 256; b++) {
    const double v = h->code256[b];
    if (v != v)
      lut[256 + b] = 1;
    else
      lut[b] = (uint8_t)nearbyint(h->dos_scale * v);
  }
  const int64_t stride = round_up(std::max(nr, 1), 128);
  std::vector<DTile> tiles;
  for (int r0 = 0; r0 < nc; r0 += DTM) {
    int jb0, jb1;
    if (band.col_blocks(r0, std::min(nc, r0 + DTM), DTN, jb0, jb1))
      for (int jb = jb0; jb <= jb1; jb++) tiles.push_back(DTile{r0, jb * DTN});
  }
  Bufs b;
  uint8_t *d_lut = nullptr, *d_Q = nullptr, *d_na = nullptr;
  DTile *d_tiles = nullptr;
  BSG_CUDA(b.up(&d_lut, lut, s));
  BSG_CUDA(b.up(&d_tiles, tiles, s));
  BSG_CUDA(b.alloc(&d_na, (size_t)nc));
  cudaError_t e = b.alloc(&d_Q, (size_t)nc * stride);
  if (e != cudaSuccess) return cuda_fail(e, "dosage pair operand (nc x round_up(nr, 128) bytes)");
  const int cg = (int)std::min<int64_t>(((int64_t)nc * 32 + 255) / 256, 132 * 16);
  k_dos_compact<<<cg, 256, 0, s>>>(h->raw, h->n, d_lut, d_row, nr, d_col, nc, d_Q, stride, d_na);
  BSG_CUDA(cudaFuncSetAttribute(k_dos_pairs, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  k_dos_pairs<<<(unsigned)tiles.size(), 256, SMEM, s>>>(d_Q, stride, nc, (int)(stride / DCH), d_tiles, band.d_wlen, band.d_boff,
                                                         d_na, band.d_center, band.d_scale, nr,
                                                         (double)h->dos_scale * (double)h->dos_scale, band.d_thr, nlev,
                                                         band.d_keep);
  count_launch(2);
  BSG_CUDA(cudaGetLastError());
  BSG_CUDA(cudaStreamSynchronize(s));  // the scratch above is freed on return
  return BSG_OK;
}

// rank[c] = k for ord[k] = c + 1: ord lists the positions 1..L by decreasing priority, each once
static int ranks_of(const int *ord, int L, int *rank) {
  for (int c = 0; c < L; c++) rank[c] = -1;
  for (int k = 0; k < L; k++) {
    const int c = ord[k] - 1;
    if (c < 0 || c >= L || rank[c] != -1) return fail(BSG_ERR_BOUNDS, "Tested subscript out of bounds (ordInd).");
    rank[c] = k;
  }
  return BSG_OK;
}

// The greedy passes of every instance over one band of levels (or conflict flags), resolved together in device rounds.
// Subset s is the band columns col[sub_off[s] .. sub_off[s + 1]) with their ranks (col empty: the identity, one subset of
// all nc columns); instance i runs subset inst_sub[i] at size inst_size[i] and threshold index inst_lev[i].  keep receives
// each instance's 0 / 1 per subset column, instance after instance.
static int clump_rounds(bsg_bed *h, const PairBand &band, const double *pos, int nc, const std::vector<int> &sub_off,
                        const std::vector<int> &col, const std::vector<int> &rank, const std::vector<int> &inst_sub,
                        const std::vector<double> &inst_size, const std::vector<int> &inst_lev, int *keep) {
  using namespace grid;
  const int ninst = (int)inst_sub.size();
  std::vector<long long> inst_state(ninst);
  long long nstate = 0;
  int maxL = 0;
  for (int in = 0; in < ninst; in++) {
    const int L = sub_off[inst_sub[in] + 1] - sub_off[inst_sub[in]];
    inst_state[in] = nstate;
    nstate += L;
    maxL = std::max(maxL, L);
  }
  if (nstate == 0) return BSG_OK;
  cudaStream_t st = h->stream;
  const int dev = h->device;
  Bufs b;
  int *d_off = nullptr, *d_col = nullptr, *d_rank = nullptr, *d_isub = nullptr, *d_ilev = nullptr, *d_state = nullptr,
      *d_cnt = nullptr;
  double *d_pos = nullptr, *d_isize = nullptr;
  long long *d_ist = nullptr;
  BSG_CUDA(b.up(&d_off, sub_off, st, dev));
  if (!col.empty()) BSG_CUDA(b.up(&d_col, col, st, dev));
  BSG_CUDA(b.up(&d_rank, rank, st, dev));
  BSG_CUDA(b.up(&d_isub, inst_sub, st, dev));
  BSG_CUDA(b.up(&d_ilev, inst_lev, st, dev));
  BSG_CUDA(b.up(&d_isize, inst_size, st, dev));
  BSG_CUDA(b.up(&d_ist, inst_state, st, dev));
  BSG_CUDA(b.up(&d_pos, pos, (size_t)nc, st, dev));
  BSG_CUDA(b.alloc(&d_state, (size_t)nstate, dev, st));
  const int BATCH = 4;  // rounds per host round trip
  BSG_CUDA(b.alloc(&d_cnt, BATCH, dev, st));
  BSG_CUDA(cudaMemsetAsync(d_state, 0xFF, (size_t)nstate * sizeof(int), st));  // -1: undecided
  // instances on the grid's y dimension, at most 65,535 per launch
  const int gy = std::min(ninst, 65535), nlaunch = (ninst + gy - 1) / gy;
  const int gx = (int)std::max<int64_t>(1, std::min<int64_t>(((int64_t)maxL * 32 + 255) / 256, std::max(1, 132 * 16 / gy)));
  int left[BATCH] = {0};
  for (int64_t round = 0; round < (int64_t)maxL + BATCH; round += BATCH) {
    BSG_CUDA(cudaMemsetAsync(d_cnt, 0, BATCH * sizeof(int), st));
    for (int k = 0; k < BATCH; k++)
      for (int in0 = 0; in0 < ninst; in0 += gy)
        k_grid_round<<<dim3(gx, std::min(gy, ninst - in0)), 256, 0, st>>>(band.d_keep, band.d_boff, band.d_wlen, d_pos, d_off,
                                                                         d_col, d_rank, d_isub, d_isize, d_ilev, d_ist, in0,
                                                                         d_state, d_cnt + k);
    count_launch(BATCH * nlaunch);
    BSG_CUDA(cudaMemcpyAsync(left, d_cnt, BATCH * sizeof(int), cudaMemcpyDeviceToHost, st));
    BSG_CUDA(cudaStreamSynchronize(st));
    if (left[BATCH - 1] == 0) break;
  }
  BSG_CUDA(cudaMemcpyAsync(keep, d_state, (size_t)nstate * sizeof(int), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaStreamSynchronize(st));
  for (long long i = 0; i < nstate; i++)
    if (keep[i] != 0 && keep[i] != 1) return fail(BSG_ERR_CUDA, "clumping rounds did not converge.");
  return BSG_OK;
}

// bed_clumping_chr (src/clumping-bed.cpp:11-91, kind BAND_CLUMP) and clumping_chr (src/clumping.cpp:10-91, BAND_LEVELS with
// the one level thr; a NaN thr keeps every variant): one instance over every selected column at threshold index 0.
static int clumping_chr(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                        const double *scale, const int *ordInd, const double *pos, double size, double thr, int *keep,
                        int kind) {
  if (!h || !center || !scale || !ordInd || !pos || !keep) return fail(BSG_ERR_ARG, "null argument");
  BSG_TRY(bind_device(h));
  if (!ind_row) nr = h->n;
  if (!ind_col) nc = h->m;
  std::vector<int> rank(nc);
  BSG_TRY(ranks_of(ordInd, nc, rank.data()));
  PairBand band;
  BSG_TRY(pair_band(h, ind_row, nr, ind_col, nc, size, pos, kind, &thr, 1, center, scale, false, band));
  return clump_rounds(h, band, pos, nc, {0, nc}, {}, rank, {0}, {size}, {0}, keep);
}

}  // namespace bsg

using namespace bsg;

extern "C" {

int bsg_clumping_chr(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                     const double *scale, const int *ordInd, const double *pos, double size, double thr, int *keep) {
  return clumping_chr(h, ind_row, nr, ind_col, nc, center, scale, ordInd, pos, size, thr, keep, BAND_CLUMP);
}

int bsg_clumping_chr_fbm(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *sumX,
                         const double *denoX, const int *ordInd, const double *pos, double size, double thr,
                         int *keep) {
  return clumping_chr(h, ind_row, nr, ind_col, nc, sumX, denoX, ordInd, pos, size, thr, keep, BAND_LEVELS);
}

int bsg_grid_clumping_chr(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *pos,
                          const double *sumX, const double *denoX, int nsub, const int *sub_len, const int *sub_col,
                          const int *sub_ord, int npt, const double *thr_r2, const double *size_bp, int *keep) {
  if (!h || (nc > 0 && (!pos || !sumX || !denoX)) || nsub < 0 || npt < 0 || (nsub > 0 && !sub_len) ||
      (npt > 0 && (!thr_r2 || !size_bp)))
    return fail(BSG_ERR_ARG, "null argument");
  BSG_TRY(bind_device(h));
  if (!ind_row) nr = h->n;
  if (!ind_col) nc = h->m;
  for (int j = 1; j < nc; j++)
    if (pos[j] < pos[j - 1]) return fail(BSG_ERR_ARG, "'pos' is not sorted.");
  // subsets: 0-based chromosome columns and ranks, concatenated
  std::vector<int> sub_off(nsub + 1, 0), col, rank;
  for (int s = 0; s < nsub; s++) {
    if (sub_len[s] < 0 || sub_len[s] > nc) return fail(BSG_ERR_ARG, "subset %d: bad length.", s + 1);
    sub_off[s + 1] = sub_off[s] + sub_len[s];
  }
  const int ntot = sub_off[nsub];
  if (ntot > 0 && (!sub_col || !sub_ord || !keep)) return fail(BSG_ERR_ARG, "null argument");
  col.resize(ntot);
  rank.resize(ntot);
  for (int s = 0; s < nsub; s++) {
    const int o = sub_off[s], L = sub_len[s];
    for (int c = 0; c < L; c++) {
      const int j = sub_col[o + c] - 1;
      if (j < 0 || j >= nc || (c > 0 && j <= col[o + c - 1]))
        return fail(BSG_ERR_ARG, "subset %d: positions must be strictly ascending within 1..nc.", s + 1);
      col[o + c] = j;
    }
    BSG_TRY(ranks_of(sub_ord + o, L, rank.data() + o));
  }
  // distinct thresholds, ascending; point p conflicts when a pair's level exceeds its index
  std::vector<double> levels(thr_r2, thr_r2 + npt);
  double size_max = 0;
  for (int p = 0; p < npt; p++) {
    if (thr_r2[p] != thr_r2[p] || size_bp[p] != size_bp[p]) return fail(BSG_ERR_ARG, "grid points must not be NA.");
    size_max = std::max(size_max, size_bp[p]);
  }
  std::sort(levels.begin(), levels.end());
  levels.erase(std::unique(levels.begin(), levels.end()), levels.end());
  if (levels.size() > 255) return fail(BSG_ERR_ARG, "at most 255 distinct thresholds per call.");
  if (ntot == 0 || npt == 0) return BSG_OK;
  // instances (subset, point) in output order
  std::vector<int> inst_sub, inst_lev;
  std::vector<double> inst_size;
  for (int s = 0; s < nsub; s++)
    for (int p = 0; p < npt; p++) {
      inst_sub.push_back(s);
      inst_size.push_back(size_bp[p]);
      inst_lev.push_back((int)(std::lower_bound(levels.begin(), levels.end(), thr_r2[p]) - levels.begin()));
    }
  PairBand band;
  BSG_TRY(pair_band(h, ind_row, nr, ind_col, nc, size_max, pos, BAND_LEVELS, levels.data(), (int)levels.size(), sumX, denoX,
                    true, band));
  return clump_rounds(h, band, pos, nc, sub_off, col, rank, inst_sub, inst_size, inst_lev, keep);
}

}  // extern "C"
