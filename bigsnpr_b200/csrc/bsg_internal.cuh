// bsg_internal.cuh -- shared declarations of libbsgpu (not part of the public ABI).
//
// HBM layout of a staged genotype matrix (see DESIGN.md "Data layout"):
//   * "staged code": 2 bits per genotype, value = genotype for 0/1/2 and 3 for missing.  It is a
//     bijective recode of the .bed code of the reference (src/bed-acc.h:22-37: 00->2, 01->NA,
//     10->1, 11->0), done once at staging, so that the packed value IS the number the kernels
//     multiply with.  Padding slots (samples >= n of the last byte, bytes up to the line stride)
//     hold code 0: they add nothing to any sum and are never missing.
//   * copy A (SNP-major): line j = SNP column j, n codes, lowest bits = first sample -- the .bed
//     orientation.  Line stride = round_up(ceil(n/4), 128) bytes.
//   * copy B (sample-major), optional: line i = sample i, m codes.  Line stride = round_up(ceil(m/4), 128).
//     Built on request or on first use by the GRM; every other kernel runs from copy A alone.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>

#include "bsgpu.h"

#define BSG_KIND_BED 0
#define BSG_KIND_FBM 1

namespace bsg {

extern thread_local std::string g_err;
int fail(int code, const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what);
void count_launch(int n = 1);

#define BSG_CUDA(call)                                   \
  do {                                                   \
    cudaError_t e__ = (call);                            \
    if (e__ != cudaSuccess) return bsg::cuda_fail(e__, #call); \
  } while (0)

#define BSG_TRY(call)        \
  do {                       \
    int rc__ = (call);       \
    if (rc__) return rc__;   \
  } while (0)

inline int64_t round_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// growable device scratch buffer
struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes);
  void release();
  template <class T> T *as() { return reinterpret_cast<T *>(p); }
};

}  // namespace bsg

#define BSG_MAX_PEERS 16

// One rank's end of a group of GPUs that exchange data through each other's memory over NVLink / NVSwitch (peer access
// inside one process, CUDA IPC between processes).  Region layout (same on every rank):
//   [0, 1024)        push flags: flag[q] = last epoch whose data rank q has finished writing into THIS region
//   [1024, 2048)     barrier flags, same convention
//   [2048, 2112)     block counter of the fused kernels (+ padding)
//   [4096, ...)      slots: 2 parities x world x slot_elems doubles; slot (p, q) receives rank q's vector of epoch parity p
struct bsg_comm {
  int rank = 0, world = 1, device = 0;
  size_t slot_elems = 0;
  uint8_t *region = nullptr;
  size_t region_bytes = 0;
  uint8_t *peer[BSG_MAX_PEERS] = {nullptr};  // peer[q]: rank q's region mapped into this device's address space
  bool peer_ipc[BSG_MAX_PEERS] = {false};    // opened with cudaIpcOpenMemHandle (to be closed)
  unsigned long long epoch = 0, bar_epoch = 0;
  int *d_err = nullptr;                      // set by a kernel whose wait timed out
  bool connected = false;
};

struct bsg_bed {
  int kind = BSG_KIND_BED;
  int device = 0;
  int n = 0, m = 0;          // samples, SNP columns held by this handle
  int64_t n_byte = 0;        // ceil(n/4): bytes per column in the .bed file
  int64_t strideA = 0, strideB = 0;
  uint8_t *A = nullptr;      // m lines of strideA bytes
  uint8_t *B = nullptr;      // n lines of strideB bytes (may be null)
  int layouts = 0;
  int has_na = 0;
  int32_t *cntA = nullptr;   // [m][4] counts of codes 0,1,2,3 per SNP over all n samples
  int32_t *cntB = nullptr;   // [n][4] counts per sample over all m SNPs (only with copy B)
  uint8_t *naA = nullptr;    // [m] 1 if the SNP line has a missing value
  uint8_t *naB = nullptr;    // [n]
  // missing-value positions as blocked-ELL lists (bsg_naell.cu), built on first use; side 0: lines = samples, 1: lines = SNPs
  uint16_t *ellCnt[2] = {nullptr, nullptr}, *ellEnt[2] = {nullptr, nullptr};
  long long *ellOff[2] = {nullptr, nullptr}, *ellOut[2] = {nullptr, nullptr};
  int ellChunks[2] = {0, 0}, ellGroups[2] = {0, 0};
  int64_t na_nnz = 0;
  int na_ell = 0;            // 0 not tried yet, 1 resident, -1 not used (rate too high, no memory, disabled)
  double code256[256];       // FBM handles: value of each raw byte code (bigstatsr code256)
  int fbm_generic = 0;       // FBM whose codes are not {0,1,2,NA} (dosages ...): served by the fp64 kernels of bsg_generic.cu
  uint8_t *raw = nullptr;    // generic FBM: the n x m code bytes, column-major, as in the .bk file
  double *d_code = nullptr;  // generic FBM: code256 on the device [0,256) and the same with NA -> 3 [256,512)
  // dosage FBM (generic, every finite code a multiple of 1 / dos_scale: bsg_code256_dosage_scale): the byte-operand
  // products of bsg_dosage.cu read a value copy built on first use.  dosV: m lines of dosStride = round_up(n, 128) bytes,
  // byte = round(dos_scale * code256[raw]) in 0..255, NA codes and pads 0 (+ 512 bytes of slack for the last line's
  // segment loads); dosNaCnt[m]: NA codes per line; dosNa: the dosNaTotal (line, sample) positions of NA codes, in line
  // order, used only to set the outputs they touch to NaN.
  int dos_scale = 0;
  uint8_t *dosV = nullptr;
  int64_t dosStride = 0;
  int32_t *dosNaCnt = nullptr;
  int2 *dosNa = nullptr;
  int64_t dosNaTotal = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaStream_t copy_stream = nullptr;  // created on first use: host -> device uploads that run under the kernels of `stream`
  cudaEvent_t copy_ev[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // view cached for the 9-argument drop-in matvec calls (bsg_prodvec / bsg_cprodvec)
  struct bsg_view *cv = nullptr;
  std::vector<int> cv_row, cv_col;
  // fingerprint of the center / scale vectors last uploaded into the cached view (address, length, strided sample of the
  // values): an unchanged scaling is not uploaded again by the next 9-argument call
  const double *cv_center_ptr = nullptr, *cv_scale_ptr = nullptr;
  std::vector<double> cv_scal_sample;
  // scratch reused across calls
  bsg::DevBuf w_idx_row, w_idx_col, w_center, w_scale, w_x, w_out, w_tmp0, w_tmp1, w_tmp2, w_tmp3,
      w_part, w_dig1, w_dig2, w_misc;
  bsg::DevBuf w_proj[8];  // projection / multLinReg work arrays (grow-only, reused across calls)
};

namespace bsg {

// ---- bsg_core.cu -----------------------------------------------------------------------------
int stage_finish(bsg_bed *h);  // counts and NA flags from copy A; copy B only when requested
int build_copy_B(bsg_bed *h);  // sample-major copy on demand (no-op when resident)
int bind_device(const bsg_bed *h);
void prefault_pages(void *p, size_t bytes);  // parallel first touch of a host output buffer (bsg_core.cu)
cudaError_t pool_alloc(void **p, size_t bytes, int device, cudaStream_t s);  // stream-ordered pool, freed with cudaFree

// A failed device allocation or upload: BSG_ERR_ALLOC when the device is out of memory, else BSG_ERR_CUDA, with the
// message "<what> (<CUDA error>)".  Clears the sticky CUDA error.
int alloc_fail(cudaError_t e, const char *what);

// Device arrays of one call, freed together (cudaFree also returns pool_alloc memory to its pool).  The first failed
// alloc / up is kept in `err` and makes every later one a no-op, so a run of them is checked once, by status().
struct Bufs {
  std::vector<void *> p;
  cudaError_t err = cudaSuccess;
  Bufs() = default;
  Bufs(const Bufs &) = delete;
  Bufs &operator=(const Bufs &) = delete;
  ~Bufs() {
    for (void *q : p) cudaFree(q);
  }
  // count elements (at least one): cudaMalloc, or the stream-ordered pool of `device` when device >= 0
  template <class T>
  cudaError_t alloc(T **dst, size_t count, int device = -1, cudaStream_t s = nullptr) {
    if (err != cudaSuccess) return err;
    const size_t bytes = (count ? count : 1) * sizeof(T);
    err = device >= 0 ? pool_alloc((void **)dst, bytes, device, s) : cudaMalloc((void **)dst, bytes);
    if (err == cudaSuccess) p.push_back(*dst);
    return err;
  }
  // alloc, then copy count host elements on s
  template <class T>
  cudaError_t up(T **dst, const T *v, size_t count, cudaStream_t s, int device = -1) {
    if (alloc(dst, count, device, s) != cudaSuccess || !count) return err;
    return err = cudaMemcpyAsync(*dst, v, count * sizeof(T), cudaMemcpyHostToDevice, s);
  }
  template <class T>
  cudaError_t up(T **dst, const std::vector<T> &v, cudaStream_t s, int device = -1) {
    return up(dst, v.data(), v.size(), s, device);
  }
  // BSG_OK, or alloc_fail of the first failed alloc / up
  int status(const char *what) const { return err == cudaSuccess ? BSG_OK : alloc_fail(err, what); }
};

// Device time of a call between start(s) and stop(s): elapsed() waits for stop and reports a failure, ms() is 0 then.
struct CallTimer {
  cudaEvent_t ev[2] = {nullptr, nullptr};
  CallTimer() = default;
  CallTimer(const CallTimer &) = delete;
  CallTimer &operator=(const CallTimer &) = delete;
  ~CallTimer() {
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
  }
  cudaError_t start(cudaStream_t s);
  cudaError_t stop(cudaStream_t s);
  cudaError_t elapsed(float *ms) const;
  float ms() const {
    float t = 0;
    elapsed(&t);
    return t;
  }
};

// ---- index helpers (bsg_core.cu) -------------------------------------------------------------
// 1-based host indices checked against `limit` (src/bed-acc.h:64-65) into 0-based `out`; ind == NULL is the identity of
// length `len`.  label names the index in the bounds message ("", "row ", "column ").  maxmult: the largest number of
// times one index occurs (1 for an empty or identity index).
int host_index(const int *ind, int len, int limit, const char *label, std::vector<int> &out, int *maxmult = nullptr);
// host_index, uploaded into buf; ind == NULL -> *dev = nullptr.
int upload_index(bsg_bed *h, const int *ind, int len, int limit, DevBuf &buf, const int **dev);

// Head-room bits for sums of up to `maxmult` quantised values: with e = 60 - ex - hb every |v 2^e| < 2^(60 - hb), and
// while 60 - hb >= 53 that double is already an integer, so |rint(v 2^e)| < 2^(60 - hb) and the sum stays below 2^60.
// From hb = 8 on, rint may round an entry just below the binade up to 2^(60 - hb) itself and 2^hb of them reach 2^60:
// one more bit there keeps every sum below 2^60 (k_corr adds 8 of them in int64).
inline int hb_bits(int maxmult) {
  int b = 0;
  while ((1 << b) < maxmult) b++;
  return b >= 8 ? b + 1 : b;
}

// ---- the genotypes a per-call driver reads (bsg_core.cu) ---------------------------------------
// Hard calls: copy A.  Dosage FBM: the value copy dosV (byte = round(D * value), NA codes 0), the raw code bytes and
// lut, their values times D as ints (-1 for NA codes, dosage_lut).
struct Genotypes {
  const uint8_t *P = nullptr;
  int64_t stride = 0;
  double D = 0;                // dos_scale, 0 for hard calls
  const uint8_t *raw = nullptr;
  const int *lut = nullptr;    // device [256], in the caller's Bufs
  bool dosage = false;
};
// BSG_ERR_TYPE for an FBM whose codes are neither hard calls nor dosages; who: the message's subject, e.g.
// "big_univLinReg on the device needs"
int genotypes_check(const bsg_bed *h, const char *who);
// the operand of a handle that passed genotypes_check: builds the value copy of a dosage handle and uploads lut into b
// (a failed upload is left in b.err for the caller's b.status)
int genotypes(bsg_bed *h, Bufs &b, Genotypes *g);
// lut of a dosage handle uploaded into b, for drivers that read the raw code bytes only (no value copy)
int *dosage_lut(const bsg_bed *h, Bufs &b);

// ---- bsg_simple.cu: generic accessor-style kernels (any index multiset) ----------------------
int simple_prodvec(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, const double *d_center,
                   const double *d_scale, const double *d_x, double *d_out, cudaStream_t s);
int simple_cprodvec(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, const double *d_center,
                    const double *d_scale, const double *d_x, double *d_out, cudaStream_t s);
int counts_cols(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, int32_t *d_out4, cudaStream_t s);
int counts_rows(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, int32_t *d_out4, cudaStream_t s);
int read_dense(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, int na_val, int *d_out, cudaStream_t s);
int read_bytes(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, uint8_t *d_out, cudaStream_t s);
int pack_bed(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, uint8_t *d_out, cudaStream_t s);
int read_dense_scaled(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, const double *d_center,
                      const double *d_scale, double *d_out, cudaStream_t s);

// ---- bsg_pmv.cu: 4 x nr code counts per sample from the plane sums of the X-side kernels (device array)
int row_counts_planes(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, int32_t *d_out4);

// ---- bsg_stats.cu: 4 x nc code counts of (ind_row, ind_col) on the device (h->w_tmp0), on h->stream
int col_counts_dev(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, int32_t **d_out);
int simple_rowsumssq(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, const double *d_center,
                     const double *d_scale, double *d_out, cudaStream_t s);

// ---- bsg_cor.cu: dense sub-matrix of a packed matrix, per-line code counts ------------------------
int compact_lines(const uint8_t *src, int64_t src_stride, const int *code_idx, int ncodes, const int *line_idx,
                  int nlines, uint8_t *out, int64_t out_stride, cudaStream_t s);
int line_counts(const uint8_t *P, int64_t stride, int nlines, int L, int32_t *cnt, uint8_t *na, cudaStream_t s);

// ---- bsg_gram5.cu: 128 x 128 integer Gram tiles on wgmma (tiles = gram::Tile array on the device)
int gram5_launch(const uint8_t *P, int64_t stride, int nlines, int64_t line_bytes, const void *d_tiles, int ntiles,
                 int *d_sums, bool any_clean, bool any_na, cudaStream_t s);

// weighted Gram for the GRM on wgmma: tiles = (i0, j0, mode) int triplets on the host, K pre-zeroed, fills i >= j
int wgram5_launch(const uint8_t *P, int64_t stride, int nlines, int nslices, const uint8_t *const dig[3],
                  int64_t dig_stride, const double (*scale)[10], const int *h_tiles, int ntiles, double *K,
                  int64_t ldk, cudaStream_t s);

// ---- bsg_naell.cu: missing values of the matvecs as blocked-ELL lists gathered from shared memory -------------------
bool na_ell_ready(bsg_bed *h);
int na_ell_correction(bsg_bed *h, int side, const int *lines, int nlines, const long long *Q, long long *part, cudaStream_t s);

// ---- bsg_generic.cu: fp64 fallback for FBM.code256 handles whose codes are not 0 / 1 / 2 / NA (dosages) --------------
#define BSG_PACKED_ONLY(h, what)                                                                                          \
  do {                                                                                                                    \
    if ((h)->fbm_generic)                                                                                                 \
      return bsg::fail(BSG_ERR_TYPE, "%s needs hard calls (codes 0 / 1 / 2 / NA); this FBM.code256 holds other values "    \
                                     "(dosages): snp_colstats, snp_cor, snp_ld_scores, snp_clumping and snp_pcadapt are served " \
                                     "by the fp64 kernels, the packed engine is not.", what);                             \
  } while (0)
int generic_colstats(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, double *d_sumX, double *d_denoX,
                     cudaStream_t s);
// pair statistics of the windowed correlations straight from the code bytes; kind BAND_COR, BAND_LD or BAND_LEVELS
// (clumping_chr's statistic, src/clumping.cpp:66-73, with the caller's sumX / denoX: how many of the nlev sorted
// thresholds d_thr[] it exceeds)
int generic_pairs(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, int kind, const int *d_wlen,
                  const long long *d_boff, long long total, const double *d_thr, int nlev, double *d_band, uint8_t *d_keep,
                  const double *d_sumX, const double *d_denoX, cudaStream_t s);
int dosage_scale_of(const double *code256);  // the D of bsg_code256_dosage_scale (0: not a dosage table)
int generic_multlinreg(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, const double *d_U, int K,
                       double *d_out, cudaStream_t s);

// ---- bsg_cor.cu: the windowed pair band of bsg_cor, bsg_ld_scores and the clumpings (bsg_grid.cu) ------------------------
// Pair (j0, j0 - 1 - k) of the selected columns, k < wlen[j0], sits at boff[j0] + k.  The kind is the epilogue's template
// argument (k_cor_from_sums, gen::k_pairs):
enum BandKind {
  BAND_COR = 0,     // band = r, keep = r is NaN or |r| > thr[nona - 1] (src/corr.cpp:77-80)
  BAND_LD = 1,      // band = r^2 (src/ld-scores.cpp:63-66)
  BAND_CLUMP = 2,   // keep = bed_clumping_chr's conflict flag, r^2 > thr[0] (src/clumping-bed.cpp:62-78)
  BAND_LEVELS = 4,  // keep = how many of the sorted thresholds thr[] clumping_chr's r^2 exceeds (src/clumping.cpp:66-73)
};
struct PairBand {
  std::vector<int> wlen, reach;  // reach[j]: largest j0 whose window holds j
  std::vector<long long> boff;   // nc + 1 offsets
  long long total = 0;
  int *d_wlen = nullptr;
  long long *d_boff = nullptr;
  double *d_band = nullptr;      // BAND_COR, BAND_LD
  uint8_t *d_keep = nullptr;     // BAND_COR, BAND_CLUMP, BAND_LEVELS
  double *d_thr = nullptr;       // BAND_COR: by nona; BAND_LEVELS: sorted levels
  double *d_center = nullptr, *d_scale = nullptr;  // clumping kinds: per selected column (clumping_chr: sumX / denoX)
  Bufs mem;                      // owns the device arrays above
  // column blocks [jb0, jb1] of width tn holding the pairs of the window owners j0 in [r0, r1); false when they have none
  bool col_blocks(int r0, int r1, int tn, int &jb0, int &jb1) const;
};
// The band of ind_col over ind_row at `size`; the clumping kinds use the union of the two window tests.  thr: nthr host
// values (BAND_COR: nr thresholds by nona, BAND_CLUMP: one, BAND_LEVELS: sorted levels); center / scale: nc host values
// (clumping kinds).  Pair source: hard calls on the Gram tiles, other FBM tables on generic_pairs, except that dosage
// handles take dosage_pair_levels when `dosage_tiles` is set (BAND_LEVELS only).
int pair_band(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, double size, const double *pos, int kind,
              const double *thr, int nthr, const double *center, const double *scale, bool dosage_tiles, PairBand &b);
// bsg_grid.cu: BAND_LEVELS of a dosage handle with xySum = S / D^2, S the exact integer sum of the D-scaled bytes, on the
// tensor pipe
int dosage_pair_levels(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, int nlev, const PairBand &b);

// ---- bsg_gramt.cu: integer Gram tiles fed by TMA, wgmma MMAs (GRM and windowed correlations) ----------
namespace gram { struct Tile; }
bool gramt_enabled();  // BSG_GRAM_TMA=0 selects the round-1 kernels (in-kernel expansion) for cross-checks
int gramt_grm(const uint8_t *P, int64_t stride, int nr, int nc, const double *const Ws[3], const double wmax[3],
              const uint8_t *na, int nslices, double *K, int64_t ldk, int device, cudaStream_t s, int64_t klo, int64_t khi);
int gramt_cor(const uint8_t *M, int64_t stride, int nlines, const gram::Tile *tiles, int ntiles, int *d_sums, int device,
              cudaStream_t s, bool *done);
// TMA map over rows x pitch bytes: 128 B x box_rows boxes, 128-byte swizzle, zero fill out of bounds
int make_map(CUtensorMap *m, const uint8_t *base, int64_t rows, int64_t pitch, int box_rows);

// ---- bsg_pmv.cu: packed matrix x vector on the integer tensor pipe ----------------------------
struct PmvPlan;  // opaque, owned by a view
namespace pmv { struct Scal; }
// X~ x enqueued on `s`; with a communicator the partial n-vectors of the column shards are summed (fused epilogue)
int view_prodvec_comm(bsg_view *v, const double *x_dev, double *out_dev, cudaStream_t s, bsg_comm *comm);

// ---- bsg_dosage.cu: X.y / Xt.y of dosage FBM handles on the integer tensor pipe, from the value copy ----------------
int dosage_build(bsg_bed *h);           // value copy + NA list (no-op when resident)
int dosage_view_masks(bsg_view *v);     // selected-row / selected-column flags (only when the matrix has NA codes)
int dosage_prodvec(bsg_view *v, const double *x_dev, double *out_dev, cudaStream_t s);
int dosage_cprodvec(bsg_view *v, const double *x_dev, double *out_dev, cudaStream_t s);
int dosage_literal(bsg_view *v, bool cprod, const double *x_dev, double *out_dev, cudaStream_t s);  // per-element fp64
// prod_and_rowSumsSq2 of an FBM handle (dosage or hard calls) as the reference's loop: rss, per-row NA flag and, for K > 0,
// XV += (pre-zeroed); then XV rows holding an NA code set to NaN
int fbm_proj_literal(bsg_view *v, const double *d_V, int K, double *d_XV, double *d_rss, uint8_t *d_na, cudaStream_t s);
int fbm_nan_rows(const uint8_t *d_na, int nr, int K, double *d_XV, cudaStream_t s);
// bsg_pmv.cu: the vector preparation these kernels share with the 2-bit ones
int dosage_prep_cols(bsg_view *v, const double *x_dev, cudaStream_t s);
int dosage_prep_rows(bsg_view *v, const double *x_dev, long long *Q, cudaStream_t s);
// bsg_prs.cu: digits of one keep set's weights x[len] (len a multiple of 32) in k_pmvT's step order, exponent into *sc
int prs_prep(const double *x_dev, int len, pmv::Scal *sc, uint8_t *dig, cudaStream_t s);

// ---- bsg_la.cu: the Lanczos driver over one or several column shards (one replica of the recurrence per shard) ----
struct SvdShard {
  bsg_bed *h;
  const int *ind_col;              // local 1-based columns of this shard (null = all)
  int nc;
  const double *center, *scale;    // per local column, or null (bed_scaleBinom computed on the device)
  bsg_comm *comm;                  // null: single shard
  double *v_out;                   // host, receives this shard's rows of v (null: not wanted)
  int64_t v_ld;                    // leading dimension of v_out
  const int *v_pos;                // row of v_out per local column (null: 0..nc-1)
  double *center_out, *scale_out;  // optional, indexed like the rows of v_out
};
int lanczos_svd(std::vector<SvdShard> &sh, const int *ind_row, int nr, int ncol_total, int k, double tol, int maxit, double *d,
                double *u, int *niter, int *nops, double *z_dev, bsg_reduce_cb reduce_cb, void *cb_ctx);

// ---- bsg_comm.cu: collectives over NVLink peer memory ------------------------------------------------
// epilogue of X.y (integer slice sums -> fp64) fused with the all-reduce over the shards: one kernel
int comm_finish_prod_allreduce(bsg_comm *c, const long long *part, int nlines, const pmv::Scal *sc, int has_scaling,
                               int use_na, double *out_dev, cudaStream_t s);
// in-place sum of `count` doubles over the ranks (one-shot: push to every peer, sum in rank order)
int comm_allreduce_oneshot(bsg_comm *c, double *buf_dev, int64_t count, cudaStream_t s);
}  // namespace bsg

struct bsg_view {
  bsg_bed *h = nullptr;
  int nr = 0, nc = 0;
  int row_identity = 1, col_identity = 1;
  int row_maxmult = 1, col_maxmult = 1;
  int has_scaling = 0;       // center/scale given (else 0 / 1)
  // device arrays (owned)
  int *d_row = nullptr;      // [nr] 0-based rows (null if identity)
  int *d_col = nullptr;      // [nc] 0-based cols (null if identity)
  double *d_center = nullptr, *d_scale = nullptr;  // [nc] (null if !has_scaling)
  // prodvec over copy B: distinct rows to compute and the gather map back to ind_row order
  int *d_rows_unique = nullptr;  // [nru] sorted distinct rows (null if identity)
  int *d_row_gather = nullptr;   // [nr] position of each requested row in d_rows_unique
  int nru = 0;
  // scratch owned by the view (so device-pointer calls are allocation free)
  bsg::DevBuf s_vec0, s_vec1, s_q0, s_q1, s_dig1, s_dig2, s_part, s_scal, s_full;
  // dosage handles with NA codes: 1 per selected sample [n] / SNP column [m] (null if identity or no NA code)
  uint8_t *d_rowsel = nullptr, *d_colsel = nullptr;
};
