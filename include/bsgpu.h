/*
 * bsgpu.h -- C ABI of libbsgpu, the H100 (sm_90a) engine for bigsnpr's packed-genotype hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no R / torch types.  Every entry point
 * replaces one `.Call` target of privefl/bigsnpr 1.12.21 (file:line of the bigsnpr sources cited per
 * function); the R-side shim that binds them under the original `_bigsnpr_*` names is r_shim/ and
 * is documented in INTEGRATION.md.
 *
 * Conventions (kept from the reference so the shim is a pass-through):
 *   - ind_row / ind_col are 1-based int32 (R integer vectors); duplicates and any order are allowed
 *     (src/bed-acc.h:64-65).  NULL means "all rows" / "all columns" (rows_along / cols_along).
 *   - matrices are column-major; vectors are double (REALSXP) or int32 (INTSXP).
 *   - all pointers are HOST pointers unless the name ends in _dev.
 *   - every function returns 0 on success, else a BSG_ERR_* code; bsg_last_error() returns the message
 *     (the text the reference raises, e.g. "Incompatibility between dimensions.").
 *   - `ncores` of the reference is accepted by the shim and ignored: the GPU path has no thread knob.
 *   - there is no CPU fallback: without a CUDA device every compute entry point fails with
 *     BSG_ERR_CUDA.
 */
#ifndef BSGPU_H
#define BSGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BSG_OK 0
#define BSG_ERR_DIM 1     /* "Incompatibility between dimensions."  src/bed-acc.h:95-96 */
#define BSG_ERR_BOUNDS 2  /* subscript out of bounds                  src/bed-acc.h:64-65 */
#define BSG_ERR_MAGIC 3   /* "File is not a binary PED file."         src/bed-acc-xptr.cpp:21-22 */
#define BSG_ERR_MODE 4    /* "Variant-major is the only mode supported."  src/bed-acc-xptr.cpp:29-30 */
#define BSG_ERR_SIZE 5    /* "n or p does not match the dimensions of the file."  :33-34 */
#define BSG_ERR_IO 6      /* "Error when mapping file"                 src/bed-acc-xptr.cpp:19 */
#define BSG_ERR_ALLOC 7
#define BSG_ERR_CUDA 8
#define BSG_ERR_ARG 9
#define BSG_ERR_TYPE 10   /* "Unknown object type."                    src/corr.cpp:124 */

/* layouts kept resident in HBM (bit mask) */
#define BSG_LAYOUT_SNP_MAJOR 1    /* variant-major, the .bed orientation: serves every entry point at full speed */
#define BSG_LAYOUT_SAMPLE_MAJOR 2 /* also keep the 2-bit transpose (what the GRM tiles read; X.y 1-3 % faster on it) */
#define BSG_LAYOUT_AUTO 0         /* SNP-major only; the transpose is built on first use by bsg_tcrossprod */

typedef struct bsg_bed bsg_bed;   /* replaces class bed + XPtr<bed>: src/bed-acc.h:18-48, src/bed-acc-xptr.cpp:40-55 */
typedef struct bsg_comm bsg_comm;   /* one rank's end of a GPU group exchanging data over NVLink peer memory (no reference twin: the
                                       reference has no multi-device path; SURVEY.md section 8e) */
typedef struct bsg_group bsg_group; /* several GPUs driven by ONE host process: column shards of one matrix + their communicators */
typedef struct bsg_view bsg_view; /* replaces bedAccScaled: (ind_row, ind_col, center, scale) resident on device, src/bed-acc.h:86-115 */

const char *bsg_last_error(void);
int bsg_version(void);
int bsg_device_count(void);

/* ---- handles ------------------------------------------------------------------------------ */
/* bedXPtr(path, n, p): src/bed-acc-xptr.cpp:14-55.  Validates the header and size exactly as the
 * reference, then stages the packed bytes to HBM once (columns [col_begin, col_end), 0-based; pass
 * 0, m for the whole file -- the range is how SNP columns are sharded across GPUs / ranks). */
int bsg_open_bed(const char *path, int n, int m, int col_begin, int col_end, int device, int layouts,
                 bsg_bed **out);
/* same, from packed bytes in host memory (m * ceil(n/4) bytes, .bed bit layout, no header) */
int bsg_open_packed(const uint8_t *packed, int n, int m, int device, int layouts, bsg_bed **out);
/* synthetic .bed generated on the device (SURVEY.md section 8d): per-SNP maf ~ U(0.02,0.5),
 * g ~ Binomial(2, maf), missing with probability na_rate; counter-based RNG keyed by (seed, global
 * column = col_offset + j), so column shards of one matrix are reproducible on any rank. */
int bsg_open_synth(int n, int m, uint64_t seed, double na_rate, int64_t col_offset, int device,
                   int layouts, bsg_bed **out);
/* LD-structured variant of the generator (SURVEY.md section 8d, AR(1)-like haplotype blocks): within every block of
 * `ld_block` consecutive global columns a haplotype's allele uniform is copied from the previous SNP with probability
 * `rho`, so neighbouring SNPs are correlated (r2 well above 0) and the clumping / r2-threshold paths have something to
 * prune.  rho = 0 reproduces bsg_open_synth bit for bit.  Same (seed, global column) keying: shards are reproducible. */
int bsg_open_synth_ld(int n, int m, uint64_t seed, double na_rate, int64_t col_offset, double rho, int ld_block,
                      int device, int layouts, bsg_bed **out);
/* FBM.code256 (bigstatsr, R/bigSNP-class.R:7,13): n x m bytes column-major + 256 doubles.  Codes
 * that round to 0/1/2/NA are repacked to 2 bits at staging and share every kernel (snp_* twins:
 * src/colstats.cpp:8-35, src/corr.cpp:113-118, src/ld-scores.cpp:93-96). */
int bsg_open_fbm256(const uint8_t *bytes, int n, int m, const double *code256, int device, int layouts,
                    bsg_bed **out);
/* Dosage tables.  An FBM.code256 whose codes are not 0 / 1 / 2 / NA stages as a generic handle.  It is also a DOSAGE
 * handle when some integer D in 1..255 makes D * v an integer in 0..255 (within 1e-9) for every finite code value v, and
 * every other code value is NaN: CODE_DOSAGE (R/bigSNP-class.R:13: 0, 1, 2, NA, 0, 1, 2, seq(0, 2, by = 0.01), NA x 48)
 * gives D = 100.  bsg_code256_dosage_scale returns the smallest such D, or 0.  Dosage handles also serve X.y and Xt.y
 * (bsg_prodvec, bsg_cprodvec, views), bsg_prod_and_rowsumssq2 and bsg_randomsvd with explicit center / scale
 * (bsg_colstats, behind the NULL default, needs hard calls), on the integer tensor pipe: round(D v) is an exact byte, the sums are exact integers.
 *   - Element (bigstatsr's SubBMCode256Acc and scaling, [bigstatsr, unvendored]): (code256[b] - c_j) / s_j.
 *   - An NA code is NA_real and poisons every output it touches, even against a zero weight: X.y rows holding an NA in a
 *     selected column and Xt.y columns holding an NA in a selected row are NaN.  (.bed handles differ: there a missing
 *     value counts as 0 after centering, src/bed-acc.h:98-111.)
 *   - Non-finite x, center or 1/scale: as for .bed handles, the _dev forms return all NaN and the host forms re-run a
 *     literal per-element fp64 loop that propagates Inf / NaN element by element.
 *   - Footprint: the first product builds a value copy (round_up(n, 128) bytes per SNP) next to the raw bytes and the
 *     2-bit copy: about 2 n m + n m / 4 bytes in all (50,000 x 600,000: 67 GB).  One device; no column shards.
 * bsg_dosage_scale(h) is the handle's D (0: hard calls, or a table that does not qualify). */
int bsg_code256_dosage_scale(const double code256[256]);
int bsg_dosage_scale(const bsg_bed *h);
void bsg_close(bsg_bed *h);
int bsg_nrow(const bsg_bed *h);
int bsg_ncol(const bsg_bed *h);
int bsg_layouts(const bsg_bed *h);
int bsg_has_na(const bsg_bed *h);
/* bytes of packed genotypes one full pass reads (ceil(n/4) * m): the roofline numerator */
int64_t bsg_packed_bytes(const bsg_bed *h);
/* copy the staged matrix back in .bed bit layout (m * ceil(n/4) bytes): round-trip check */
int bsg_export_packed(const bsg_bed *h, uint8_t *out);

/* ---- X.y and Xt.y ---------------------------------------------------------------------------- */
/* The accessor state of a call (index vectors, center, scale) is cached on the handle: a following call with the same
 * index vectors (compared by content) re-uses it; center / scale are uploaded with every call, like the reference
 * re-reads them (src/bed-prod-vec.cpp:22-23).  bsg_set_scaling_reuse(1) (or BSG_SCALING_REUSE=1) lets a call skip that
 * upload when address, length and a strided sample of 2,048 values of each vector equal the previous call's -- the shape
 * of big_randomSVD's closures (R/autoSVD.R:216-218: ~1,000 calls with identical scaling vectors).  Opt-in because a vector
 * edited in place at an unsampled position would go unnoticed. */
int bsg_set_scaling_reuse(int on);
/* bed_pMatVec4: src/bed-prod-vec.cpp:15-54.  out[nr] = X~[ind_row, ind_col] %*% x[nc] */
int bsg_prodvec(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc,
                const double *center, const double *scale, const double *x, double *out);
/* bed_cpMatVec4: src/bed-prod-vec.cpp:59-97.  out[nc] = t(X~[ind_row, ind_col]) %*% x[nr] */
int bsg_cprodvec(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc,
                 const double *center, const double *scale, const double *x, double *out);

/* views: the accessor state of bedAccScaled kept on the device across calls (what big_randomSVD's
 * closures re-create on every operator call in the reference, R/autoSVD.R:216-218) */
int bsg_view_create(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc,
                    const double *center, const double *scale, bsg_view **out);
void bsg_view_destroy(bsg_view *v);
int bsg_view_prodvec(bsg_view *v, const double *x, double *out);   /* host vectors */
int bsg_view_cprodvec(bsg_view *v, const double *x, double *out);  /* host vectors */
/* device-resident vectors, enqueued on `stream` (a cudaStream_t; NULL = the legacy default stream, i.e. ordered with
 * everything the caller enqueued on stream 0 -- torch's default stream included); no sync.
 * Non-finite input: the host-vector forms above reproduce the reference's per-element Inf / NaN propagation (a zero scale
 * makes only that column's Xt.y entry NaN, src/bed-acc.h:98-111) by re-running through the accessor kernels.  The _dev
 * forms cannot look at their result: ANY non-finite x, center or 1/scale entry makes the WHOLE output NaN.  The SVD
 * drivers built on them return BSG_ERR_ARG in that case instead of iterating on NaNs. */
int bsg_view_prodvec_dev(bsg_view *v, const double *x_dev, double *out_dev, void *stream);
int bsg_view_cprodvec_dev(bsg_view *v, const double *x_dev, double *out_dev, void *stream);

/* ---- column / row statistics ------------------------------------------------------------------ */
/* bed_colstats: src/bed-fun.cpp:9-46.  n_bad = count behind the ">50% missing values" warning */
int bsg_colstats(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, double *sumX,
                 double *denoX, int *nb_nona_col, int *n_bad);
/* bed_col_counts_cpp / bed_row_counts_cpp: src/bed-fun.cpp:51-69, :72-98.  out is 4 x nc (4 x nr) */
int bsg_col_counts(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, int *out);
int bsg_row_counts(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, int *out);
/* snp_colstats: src/colstats.cpp:8-35 (FBM.code256 handles; NA handling as the reference: none) */
int bsg_snp_colstats(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, double *sumX,
                     double *denoX);

/* ---- dense decode ------------------------------------------------------------------------------ */
/* read_bed: src/bed-mat-acc.cpp:8-26 (NA -> na_val; R passes NA_INTEGER) */
int bsg_read_bed(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, int na_val,
                 int *out);
/* read_bed_scaled: src/bed-mat-acc.cpp:30-49 */
int bsg_read_bed_scaled(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc,
                        const double *center, const double *scale, double *out);

/* ---- windowed correlations ---------------------------------------------------------------------- */
/* corMat: src/corr.cpp:11-97,102-126.  CSC pieces: p[nc+1], *i (0-based rows, ascending, diagonal
 * last), *x; the caller releases *i and *x with bsg_free.  thr has nr entries, pos has nc. */
int bsg_cor(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, double size,
            const double *thr, const double *pos, int fill_diag, int64_t *p, int **i, double **x);
/* ld_scores: src/ld-scores.cpp:11-78,83-105 */
int bsg_ld_scores(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, double size,
                  const double *pos, double *out);
void bsg_free(void *ptr);
/* bed_clumping_chr: src/clumping-bed.cpp:11-91.  ordInd = 1-based positions (within ind_col) by decreasing
 * priority; center / scale / pos per selected column; keep[nc] receives 0 / 1.  Pair statistics come from the same
 * Gram tiles as bsg_cor; the greedy sweep in rank order is resolved on the device in rounds.  An ordInd that is not a
 * permutation of 1..nc (an entry out of range or repeated): BSG_ERR_BOUNDS. */
int bsg_clumping_chr(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                     const double *scale, const int *ordInd, const double *pos, double size, double thr,
                     int *keep);

/* ---- FBM.code256 <-> .bed conversion (SURVEY.md section 8f row 3) ----------------------------------- */
/* _bigsnpr_readbina2: src/read-plink.cpp:61-80 (snp_readBed2, R/read-plink.R:72-111).  out = nr x nc bytes column-major, the
 * FBM.code256 codes 0 / 1 / 2 / 3 (NA) of X[ind_row, ind_col] -- what the reference writes into the .bk file. */
int bsg_readbina2(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, unsigned char *out);
/* _bigsnpr_writebina: src/write-plink.cpp:13-52 (snp_writeBed, R/write-plink.R:15-45).  Writes X[ind_row, ind_col] of a
 * bed- or FBM-staged handle as a PLINK .bed: magic bytes, then ceil(nr/4) bytes per column, byte for byte the
 * reference's output (unused slots of a column's last byte hold genotype 0). */
int bsg_writebina(bsg_bed *h, const char *path, const int *ind_row, int nr, const int *ind_col, int nc);

/* Which kernel serves the X-side products (bsg_prodvec, bsg_view_prodvec*, XV and row sums of squares):
 * 0 = automatic -- the sample-major kernel when that copy is resident, else the SNP-major kernel (k_pmvT), which
 * needs only the copy every handle has; 1 = always the SNP-major kernel.  Process-wide; no reference twin
 * (bed_prodVec has one code path, src/bed-prod-vec.cpp:15-54). */
int bsg_set_prodvec_path(int path);

/* ---- PCA projection / pcadapt (SURVEY.md section 8f row 2) ------------------------------------------- */
/* _bigsnpr_prod_and_rowSumsSq: src/bed-fun.cpp:103-133 (R: part_prod, R/bed-projectPCA.R:45-58).
 * V is nc x K column-major; XV (nr x K column-major) = X~ V and rowSumsSq[nr] = sum_j X~_ij^2 with the
 * bedAccScaled semantics (missing value -> 0).  center / scale length nc, else
 * "Incompatibility between dimensions." */
int bsg_prod_and_rowsumssq(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc,
                           const double *center, const double *scale, const double *V, int K,
                           double *XV, double *rowSumsSq);
/* _bigsnpr_prod_and_rowSumsSq2: src/project-utils.cpp:11-43 (R: part_prod2 of snp_projectSelfPCA, R/bed-projectPCA.R:252-281).
 * Same outputs for an FBM.code256 handle (hard calls or a dosage table, bsg_dosage_scale > 0) with the accessor's literal
 * semantics: x = (code256[b] - c_j) / s_j and an NA code is NA_real, so a row holding an NA code in a selected column
 * has NaN in XV and in rowSumsSq.  XV runs on the integer tensor pipe (K single-vector X.y passes); rowSumsSq is one
 * literal fp64 pass over the codes (x^2 is not linear in the code), not a tuned path.  Other handles: BSG_ERR_TYPE. */
int bsg_prod_and_rowsumssq2(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc,
                            const double *center, const double *scale, const double *V, int K,
                            double *XV, double *rowSumsSq);
/* _bigsnpr_multLinReg: src/multLinReg.cpp:8-88 (R: pcadapt0, R/pcadapt.R:3-27).  U is nr x K column-major;
 * tscores is nc x K column-major (the reference returns transpose(res)); NA_REAL is written as NaN.
 * Works on .bed handles and on FBM.code256 handles alike (the reference dispatches on the class, :72-92). */
int bsg_multlinreg(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *U, int K,
                   double *tscores);

/* _bigsnpr_clumping_chr: src/clumping.cpp:10-91 (snp_clumping on an FBM.code256, R/clumping.R:93-137).  Same
 * greedy sweep; the statistic is r2 = (xySum - sumX_j sumX_j0 / n)^2 / (denoX_j denoX_j0) with the caller's
 * snp_colstats vectors and no missing-value handling (a missing genotype never prunes, like the reference's NA). */
int bsg_clumping_chr_fbm(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *sumX,
                         const double *denoX, const int *ordInd, const double *pos, double size, double thr,
                         int *keep);

/* snp_grid_clumping, one chromosome (R/SCT.R:32-151): every clumping_chr_cached call of the chromosome in one call.
 * ind_col (nc columns after `exclude`) with sorted pos and the snp_colstats vectors sumX / denoX over ind_row.
 * nsub subsets, concatenated: subset s has sub_len[s] entries of sub_col (1-based positions within ind_col, strictly
 * ascending) and of sub_ord (1-based positions within the subset by decreasing priority: order(S, decreasing = TRUE)).
 * npt grid points (thr_r2[p], size_bp[p]); size_bp is the reference's 1000 * base.size / thr.r2, in bp.
 * keep (sum_s npt * sub_len[s] ints) receives, subset by subset, point by point, 0 / 1 per subset column: the keep
 * vector of clumping_chr on that subset with that size and threshold.  The pair statistic of clumping_chr (bsg_clumping_chr_fbm)
 * is computed once per pair at the largest size: hard calls on the Gram tiles, dosage handles (bsg_dosage_scale D > 0)
 * as exact integer sums of D-scaled bytes on the tensor pipe (xySum = S / D^2), other tables by the fp64 kernels.
 * At most 255 distinct thresholds; unsorted pos, a subset out of order or out of range: BSG_ERR_ARG. */
int bsg_grid_clumping_chr(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *pos,
                          const double *sumX, const double *denoX, int nsub, const int *sub_len, const int *sub_col,
                          const int *sub_ord, int npt, const double *thr_r2, const double *size_bp, int *keep);

/* snp_PRS with thresholding (R/PRS.R:36-76) for nsets keep sets at once: what snp_grid_PRS (R/SCT.R:201-246) computes
 * for one chromosome.  Set c has set_len[c] entries, concatenated over the sets in cols (1-based columns, repeats
 * allowed), beta, same (NULL = all TRUE; 0 / 1) and lpS.  Thresholds are visited in stable decreasing order; an entry
 * joins at the first one its lpS exceeds (strict >), and column c * nthr + t of out (nr x nsets * nthr, column-major,
 * float rounded to nearest when out_double = 0, else double) is set c at thr[t]: prodVecRev summed over every entry
 * joined so far.  thr = NULL with nthr = 1 disables thresholding (one column over all entries, lpS unused).
 * The scores are exact integer sums of the codes times the 61-bit fixed-point weights (one quantisation per set,
 * reversed alleles as (g - 2) Q), with one fp64 sum of 8 digit slices per output.  A row holding an NA code in a
 * column joined so far is NaN (R: last + NA stays NA).  A set holding a non-finite beta is computed by R's loop in
 * fp64 instead (sum(betas[!same]) in double, R sums in long double).  ind_row: 1-based, repeats allowed, NULL = all.
 * A NaN or negative lpS of an entry, a NaN threshold, same not in {0, 1} or bad lengths: BSG_ERR_ARG (R's result for a
 * NaN lpS is an NA index, deliberately refused here); columns or rows out of range: BSG_ERR_BOUNDS.  Dosage tables
 * (bsg_dosage_scale D > 0) use the value bytes D x code and divide the slice sum by D once; other FBM.code256 tables:
 * BSG_ERR_TYPE; scratch and output larger than the free device memory:
 * BSG_ERR_ALLOC with the bytes needed, before any allocation. */
int bsg_prs_grid(bsg_bed *h, const int *ind_row, int nr, int nsets, const int *set_len, const int *cols,
                 const double *beta, const int *same, const double *lpS, int nthr, const double *thr, int out_double,
                 void *out);
/* device time in ms (CUDA events) of the last bsg_prs_grid, quantisation to the gathered output, copies excluded */
double bsg_prs_last_ms(void);

/* big_univLinReg (bigstatsr's univLinReg5 and its R glue; bigstatsr is not vendored in the reference): linear regression of
 * y on [C, X[ind_row, j]] for every selected column j, C = the covariates with the intercept.  U is nr x K column-major,
 * orthonormal, spanning the intercept (the first K left singular vectors of cbind(1, covar.train) the glue keeps);
 * y[nr] is y.train.  ind_row: 1-based, repeats allowed (a repeated row counts as often as it appears), NULL = all;
 * ind_col: 1-based, repeats in any order, NULL = all.  estim / std_err (nc each, in ind_col order):
 *   x2 = x - U U'x,  y2 = y - U U'y,  estim = x2'y2 / x2'x2,  std.err = sqrt((y2'y2 - estim x2'y2) / (nr - K - 1) / x2'x2),
 * evaluated as x2'x2 = SSx_c - |U'x_c|^2 with SSx_c from exact integer sums of x and x^2 and x_c, y_c centred (DESIGN.md
 * section 4.16).  The V = K + 1 products x'y_c, x'U are exact integer sums of the codes times fixed-point digits (y_c 61
 * bits, U 30 bits) from one read of the matrix per group of at most 64 digit slices.  NaN for a column with an NA code
 * on an ind_row row, a constant column, or x2'x2 <= 0.  Dosage tables (bsg_dosage_scale D > 0): the same sums over the
 * value bytes D x code, divided by D once per sum; other FBM.code256 tables: BSG_ERR_TYPE.  K < 1, nr - K - 1 < 1, a
 * non-finite y or U entry, or a U whose span misses the intercept: BSG_ERR_ARG; indices out of range: BSG_ERR_BOUNDS;
 * scratch larger than the free device memory: BSG_ERR_ALLOC with the bytes needed, before any allocation. */
int bsg_univlinreg(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *U, int K,
                   const double *y, double *estim, double *std_err);
/* device time in ms (CUDA events) of the last bsg_univlinreg: vector upload to the statistics, copies back excluded */
double bsg_univlinreg_last_ms(void);

/* big_univLogReg's per-SNP IRLS (bigstatsr's IRLS; not vendored in the reference): logistic regression of y01 on
 * A = [U, X[ind_row, j]] for every selected column j.  U is nr x K column-major (the orthonormal basis of cbind(1,
 * covar.train) big_univLinReg's glue keeps; any finite basis is accepted), gamma0[K] the null model's coefficients on U
 * (glm.fit of y01 on U), y01[nr] 0 / 1.  ind_row: 1-based, repeats allowed (each entry is one observation), NULL = all;
 * ind_col: 1-based, repeats in any order, NULL = all.  Per SNP, from beta = (gamma0, 0):
 *   eta = A beta, p = 1 / (1 + e^-eta), w = p (1 - p), H = A'WA, r = A'W z with W z = w eta + (y - p),
 *   beta_new = H^-1 r, until max |beta_new - beta| < tol or maxiter steps.
 * estim = beta_x, std_err = sqrt((H^-1)_xx) = 1 / L_xx of the last H solved (Cholesky, x last), niter = the steps taken,
 * or -maxiter when tol was not met in maxiter steps (the caller refits those; estim / std_err then hold the last step).
 * Every sum over observations runs in an order fixed by (nr, K) alone (DESIGN.md section 4.17): a SNP's bytes do not
 * depend on the other columns of the call, their order or repeats.  NaN estim / std_err and niter = 0 for a column with an
 * NA code on an ind_row row, a column constant over the rows, or an H whose factorisation meets a pivot <= 0 or a
 * non-finite value.  Dosage tables (bsg_dosage_scale D > 0) read x = byte / D from the value copy; other FBM.code256
 * tables: BSG_ERR_TYPE.  K < 1 or K > 80, nr < 1, tol <= 0, maxiter < 1, a y01 entry other than 0 / 1, non-finite U or
 * gamma0: BSG_ERR_ARG; indices out of range: BSG_ERR_BOUNDS; scratch larger than the free device memory: BSG_ERR_ALLOC
 * with the bytes needed, before any allocation. */
int bsg_univlogreg(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *U, int K,
                   const double *gamma0, const double *y01, double tol, int maxiter, double *estim, double *std_err,
                   int *niter);
/* device time in ms (CUDA events) of the last bsg_univlogreg: column checks to the last IRLS step, copies excluded */
double bsg_univlogreg_last_ms(void);

/* big_spLinReg (family 0) / big_spLogReg (family 1) with power_scale = 1, power_adaptive = 0 (bigstatsr's penalised
 * regression, not vendored in the reference; DESIGN.md section 4.19, restated in tests/splreg_ref.py).  Every fit
 * f = ia * K + k (alpha alphas[ia], fold k) runs on one 8-CTA thread-block cluster over the whole lambda path, state
 * kept on the device; nr <= 1,048,576.
 *   - Observations: ind_row (1-based, repeats allowed, NULL = all) with y[nr] (family 1: 0 / 1), covar nr x Kc
 *     column-major, base[nr] offset (NULL = 0), ind_sets[nr] fold of each observation in 1..K (K >= 2; every fold leaves
 *     at least two training observations and holds at least one).
 *   - Columns: ind_col (1-based, NULL = all) then the Kc covariates.  center / scale [nc + Kc] are the mean and sd (divisor
 *     nr) over all observations; genotype columns with scale <= 1e-8 are dropped (kept[nc] 0), the fit's J columns are the
 *     kept ones in ind_col order, then the covariates (a constant covariate: BSG_ERR_ARG).  Fits use x~ = (x - c) / s.
 *   - Penalty factors pf_X[nc], pf_covar[Kc] (NULL = 1); alphas in (0, 1].
 *   - Per fit: the null fit of the intercept and pf = 0 columns, lambda_max = max |z_j| / (alpha pf_j) over pf_j > 0,
 *     then nlambda values lambda_max * step^k, step = lambda_min_ratio^(1 / (nlambda - 1)), each from the previous
 *     solution: sequential strong rule, coordinate-descent passes over the working set until
 *     max |delta| <= eps * max |coef| (intercept included) or max_iter passes, a full KKT pass, repeat while a column
 *     violates.  Stops at the first of: more than dfmax nonzero coefficients (message 2), the best validation loss
 *     n_abort steps behind with at least nlam_min steps run (message 1), the end of the path (message 0).
 * Outputs, J = (kept genotype columns) + Kc: beta [F][J] and intercept [F] at each fit's best lambda (standardised
 * scale), best / length / message [F], lambda / loss (validation MSE or mean binomial deviance) / nnz / npass
 * [F][nlambda] (entries past length are 0), path_beta [F][nlambda][J] and path_b0 [F][nlambda] when not NULL.
 * Every sum over observations has one fixed order (8,192-position segments of 256-slot sums, added in order), so each
 * fit's bytes depend on its problem alone.
 * Refusals: power_scale != 1, power_adaptive != 0, alpha outside (0, 1], y01 not 0 / 1, non-finite y / covar / base,
 * negative or non-finite penalty factors, invalid path parameters: BSG_ERR_ARG; indices out of range: BSG_ERR_BOUNDS;
 * other FBM.code256 tables than hard calls and dosages: BSG_ERR_TYPE; scratch beyond free memory: BSG_ERR_ALLOC; all
 * before any allocation.  An NA code on a selected (row, column) pair: BSG_ERR_ARG after the column-statistics pass. */
int bsg_splreg(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, int family, const double *y,
               const double *covar, int Kc, const double *base, const double *pf_X, const double *pf_covar,
               const double *alphas, int nalpha, const int *ind_sets, int K, int nlambda, double lambda_min_ratio,
               int nlam_min, int n_abort, int dfmax, double eps, int max_iter, double power_scale, double power_adaptive,
               double *center, double *scale, uint8_t *kept, double *beta, double *intercept, int *best, int *length,
               int *message, double *lambda, double *loss, int *nnz, int *npass, double *path_beta, double *path_b0);
/* bsg_splreg over a dense host matrix instead of a handle: X is column-major with leading dimension ld >= nrow, nrow x ncol
 * elements of float (dtype 0) or double (dtype 1); ind_row / ind_col index it (1-based, repeats allowed, NULL = all).
 * X[ind_row, ind_col] is gathered through bounded pinned buffers and uploaded once to `device` (nr x nc elements of the
 * same type); each element is widened to double exactly when read, so the fit is bsg_splreg's on X converted to double:
 * same arguments after ind_col, same outputs, same arithmetic and summation order.  Coordinate descent visits the kept
 * columns by increasing column index (ties in ind_col order), then the covariates.  Refusals: those of bsg_splreg; a
 * dtype other than 0 / 1: BSG_ERR_TYPE; ld < nrow, negative sizes or a null X: BSG_ERR_DIM; a non-finite value on a
 * selected (row, column) pair: BSG_ERR_ARG naming the column, after the column-statistics pass; the staged block plus the
 * fits' state beyond free device memory: BSG_ERR_ALLOC with the bytes needed, before any allocation. */
int bsg_splreg_dense(const void *X, int dtype, int64_t ld, int nrow, int ncol, const int *ind_row, int nr,
                     const int *ind_col, int nc, int device, int family, const double *y, const double *covar, int Kc,
                     const double *base, const double *pf_X, const double *pf_covar, const double *alphas, int nalpha,
                     const int *ind_sets, int K, int nlambda, double lambda_min_ratio, int nlam_min, int n_abort,
                     int dfmax, double eps, int max_iter, double power_scale, double power_adaptive, double *center,
                     double *scale, uint8_t *kept, double *beta, double *intercept, int *best, int *length,
                     int *message, double *lambda, double *loss, int *nnz, int *npass, double *path_beta,
                     double *path_b0);
/* device time in ms (CUDA events) of the last bsg_splreg / bsg_splreg_dense: column statistics to the end of the last
 * fit */
double bsg_splreg_last_ms(void);
/* host time in ms of the last call's staging: the dense gather and upload, or the dosage value copy when it is built */
double bsg_splreg_last_stage_ms(void);

/* ---- sparse LD matrix (bigsparser's SFBM) and summary-statistics PRS -------------------------------------- */
/* as_SFBM(corr[, compact]) staged to HBM once, in bigsparser's storage as bigsnpr reads it (src/ld-scores-sfbm.cpp:14-66):
 *   - p: ncol + 1 doubles, non-decreasing integers starting at 0 (X$p);
 *   - first_i == NULL (non-compact): data interleaves (row, value) doubles, column j at data[2 p[j] .. 2 p[j + 1]), rows
 *     0-based integers in [0, nrow), each at most once per column;
 *   - first_i != NULL (compact): data holds values only, column j at data[p[j] .. p[j + 1]) for the contiguous rows
 *     first_i[j], first_i[j] + 1, ..., which must stay below nrow.
 * Columns hold the full symmetric matrix (both triangles and the diagonal).  The device keeps either form as given: int32
 * rows or first_i, fp64 values.  Malformed storage: BSG_ERR_ARG; not enough device memory: BSG_ERR_ALLOC. */
typedef struct bsg_sfbm bsg_sfbm;
int bsg_sfbm_open(int nrow, int ncol, const double *p, const double *data, const int *first_i, int device, bsg_sfbm **out);
void bsg_sfbm_close(bsg_sfbm *s);
int bsg_sfbm_nrow(const bsg_sfbm *s);
int bsg_sfbm_ncol(const bsg_sfbm *s);
/* ld_scores_sfbm: src/ld-scores-sfbm.cpp:9-69.  ind_sub: m 0-based columns (as the .Call target receives them); out[j] =
 * sum of x^2 over the stored entries of column ind_sub[j] whose row is in ind_sub.  ind_sub out of range: BSG_ERR_BOUNDS. */
int bsg_sfbm_ld_scores(bsg_sfbm *s, const int *ind_sub, int m, double *out);
/* lassosum2: src/lassosum2.cpp:20-70 for ngrid grid points in one launch (one CTA per point, every sweep in the kernel).
 * lambda and delta_plus_one are m x ngrid column-major: column g is what R/lassosum2.R:58-67 passes for ic = g.
 * beta_est (m x ngrid) and num_iter[ngrid] are bit-identical to the sequential loop; a diverged point (gap > gap0) gets
 * NA_real in its whole column; num_iter is maxiter + 1 when maxiter sweeps did not stop it.  seconds[ngrid] (NULL
 * allowed): device time of each point.  ind_sub: m 0-based columns, any order, repeats allowed (BSG_ERR_BOUNDS out of
 * range); the matrix must be square (BSG_ERR_DIM). */
int bsg_lassosum2(bsg_sfbm *corr, const double *beta_hat, int m, const int *ind_sub, int ngrid, const double *lambda,
                  const double *delta_plus_one, double dfmax, int maxiter, double tol, double *beta_est, int *num_iter,
                  double *seconds);
/* bigsparser::sp_solve_sym (called at R/LDpred2.R:38-39): x solving (A + diag(d)) x = b, A the n x n SFBM as stored, by
 * Eigen's ConjugateGradient with the identity preconditioner from x = 0, every sum in one fixed order (DESIGN.md §4.13).
 * d has length diag_len, 1 or n.  iters and error are Eigen's ConjugateGradient::iterations() / error(): the iteration
 * that reached |r|^2 < max(tol^2 |b|^2, DBL_MIN) (not counted) or maxiter, and sqrt(|r|^2 / |b|^2); b = 0 gives x = 0,
 * iters 0 and error 0.  A singular or indefinite system is not special-cased (error may be NaN).  A non-square handle or
 * diag_len not in {1, n}: BSG_ERR_DIM; tol < 0, maxiter < 0 or a null pointer: BSG_ERR_ARG. */
int bsg_sfbm_solve(bsg_sfbm *A, const double *b, const double *add_to_diag, int diag_len, double tol, int maxiter,
                   double *x, int *iters, double *error);
/* device time in ms (CUDA events) of the iterations of the last bsg_sfbm_solve on this handle, no-op launches after
 * convergence included; 0 when it ran none */
double bsg_sfbm_last_solve_ms(const bsg_sfbm *A);
/* LDpred2-auto: src/ldpred2-auto.cpp:56-202 (ldpred2_gibbs_auto) for nchain chains in one launch, one CTA per chain.
 * beta_hat, n_vec, log_var: m values (R/LDpred2.R:238-255 passes beta * sd, n_eff and 2 log sd); ind_sub: m 0-based
 * columns of corr, any order, repeats allowed (BSG_ERR_BOUNDS out of range).  Chain c starts from p_init[c] and draws
 * from the MRG32k3a state rng_state[6 c .. 6 c + 5] (as R's .Random.seed[2:7] for L'Ecuyer-CMRG, as unsigned words);
 * p_bounds[2], alpha_bounds[2] (alpha + 1, as the .Call receives them), mean_ld as the .Call takes them.  The draws are
 * the ones of DESIGN.md §4.15 (one uniform per coordinate, a normal when it is selected, rbeta, then the bootstrap), and
 * the MLE step returns the minimiser of MLE_alpha's objective over its box (golden-section search in alpha + 1 over
 * the objective profiled in sigma2), where the reference returns the point L-BFGS-B stops at.  Every output of a chain
 * depends only on the inputs and its own state: bit-identical to the sequential CPU restatement.
 * Outputs, column-major with one column per chain: beta_est, postp_est, corr_est (m x nchain: the averages over the
 * num_iter sweeps after burn_in, divided by num_iter; NA_real on divergence); path_p, path_h2, path_alpha ((burn_in +
 * num_iter) x nchain, NA_real past a divergence, and path_alpha all NA_real without use_mle); sample_beta (NULL allowed)
 * m x (num_iter / report_step) x nchain, dense, the causal effects at every report_step-th sweep after burn_in;
 * seconds[nchain] (NULL allowed) the device time of each chain.  m < 1, burn_in < 0, num_iter < 1, report_step < 1,
 * p_bounds not 0 < lo <= hi, alpha_bounds not finite lo <= hi, mean_ld <= 0, an invalid state or a null pointer:
 * BSG_ERR_ARG; a non-square corr: BSG_ERR_DIM. */
int bsg_ldpred2_auto(bsg_sfbm *corr, const double *beta_hat, const double *n_vec, const double *log_var, int m,
                     const int *ind_sub, int nchain, const double *p_init, double h2_init, int burn_in, int num_iter,
                     int report_step, int no_jump_sign, double shrink_corr, int use_mle, const double *p_bounds,
                     const double *alpha_bounds, double mean_ld, const unsigned *rng_state, double *beta_est,
                     double *postp_est, double *corr_est, double *path_p, double *path_h2, double *path_alpha,
                     double *sample_beta, double *seconds);
/* bsg_ldpred2_auto, and rng_out (NULL allowed) receives each chain's MRG32k3a state after its last sweep (6 words per
 * chain, after the last sweep's rbeta and bootstrap, or after the diverging sweep): the state R/LDpred2.R:266-279 continues
 * from in the same %dorng% iteration.  bsg_ldpred2_auto is this call with rng_out NULL. */
int bsg_ldpred2_auto_ex(bsg_sfbm *corr, const double *beta_hat, const double *n_vec, const double *log_var, int m,
                        const int *ind_sub, int nchain, const double *p_init, double h2_init, int burn_in, int num_iter,
                        int report_step, int no_jump_sign, double shrink_corr, int use_mle, const double *p_bounds,
                        const double *alpha_bounds, double mean_ld, const unsigned *rng_state, double *beta_est,
                        double *postp_est, double *corr_est, double *path_p, double *path_h2, double *path_alpha,
                        double *sample_beta, double *seconds, unsigned *rng_out);
/* LDpred2-grid: src/ldpred2.cpp:9-69 (ldpred2_gibbs_one) for npoint grid points in one launch, one CTA per point, or with
 * sampling, src/ldpred2-sampling.cpp:9-59 (ldpred2_gibbs_one_sampling) for one point.  beta_hat, n_vec: m values
 * (R/LDpred2.R:89-91 passes beta / scale and n_eff); ind_sub: m 0-based columns of corr, any order, repeats allowed
 * (BSG_ERR_BOUNDS out of range).  Point g runs with p[g], h2[g], sparse[g] (0 or not) and draws from the MRG32k3a state
 * rng_state[6 g .. 6 g + 5]: one uniform per coordinate, none for a coordinate a sparse point zeroes (postp < p), and a
 * normal by inversion when it is selected (DESIGN.md §4.18).  Every output of a point depends only on the inputs and its
 * own state: bit-identical to the sequential CPU restatement.  Outputs: beta_est (m x npoint, column-major, without
 * sampling): the average of C3 postp over the num_iter sweeps after burn_in, divided by num_iter, NA_real in the whole
 * column when a sweep's sum of squared draws exceeds 2 sum(beta_hat^2); sample_beta (m x num_iter, with sampling): the
 * coefficients after each sweep past burn_in; seconds[npoint] (NULL allowed): each point's device time.  m < 1,
 * burn_in < 0, num_iter < 1, sampling with npoint != 1, an invalid state or a null pointer: BSG_ERR_ARG; a non-square
 * corr: BSG_ERR_DIM; state larger than the free device memory (ncol + 3 m doubles per point, plus m x num_iter):
 * BSG_ERR_ALLOC, with the bytes needed. */
int bsg_ldpred2_grid(bsg_sfbm *corr, const double *beta_hat, const double *n_vec, int m, const int *ind_sub, int npoint,
                     const double *p, const double *h2, const int *sparse, int burn_in, int num_iter, int sampling,
                     const unsigned *rng_state, double *beta_est, double *sample_beta, double *seconds);

/* ---- near-independent LD blocks (snp_ldsplit, R/split-LD.R:99-138) -------------------------------------------------- */
/* Matrix::tril(corr) staged to HBM once: m x m lower triangle in CSC, p[m + 1] (non-decreasing, p[0] = 0), rows i
 * increasing within each column and in [column, m), the diagonal stored first and non-zero (R/split-LD.R:108-109),
 * values x.  Malformed input or a zero / missing diagonal: BSG_ERR_ARG.  sumsq2: 2 * sum(x^2), folded in storage order
 * (R computes it with BLAS crossprod, R/split-LD.R:111, which can differ in the last bit). */
typedef struct bsg_ldcorr bsg_ldcorr;
int bsg_ldcorr_open(int m, const long long *p, const int *i, const double *x, int device, bsg_ldcorr **out);
void bsg_ldcorr_close(bsg_ldcorr *c);
int bsg_ldcorr_m(const bsg_ldcorr *c);
double bsg_ldcorr_sumsq2(const bsg_ldcorr *c);
/* get_L: src/split-LD.cpp:15-61.  *count receives the number of triplets; with cap >= *count, li / lj / lx (0-based
 * column of corr, row, value) are filled in the reference's order (by column, row descending).  cap = 0: count only. */
int bsg_ldcorr_l_triplets(bsg_ldcorr *c, double thr_r2, double max_r2, long long *count, long long cap, int *li, int *lj,
                     double *lx);
/* The whole snp_ldsplit grid in one call: get_L, get_C (src/split-LD.cpp:65-145) for every max_size value in one pass
 * over E per layer, reconstruct_paths (R/split-LD.R:3-40) and get_perc (src/split-LD.cpp:149-182), bit-identical to
 * them.  max_size[n_max_size] in any order, repeats allowed; results are laid out by position t in the sorted list:
 * row t max_K + K - 1 of kept (1 when the row is part of the result), cost, cost2, perc_kept; the path of (t, K) at
 * all_last + t max_K (max_K + 1) / 2 + K (K - 1) / 2, K 1-based last indices.  max_cost is capped at sumsq2.  layers
 * (NULL allowed): the layers get_C ran per t; seconds[3] (NULL allowed): device time of building E, of the layers, of
 * the paths and perc_kept.  min_size < 1, max_size > m or < min_size, max_K < 1, a missing pos_scaled: BSG_ERR_ARG;
 * E and the layer state larger than the free device memory: BSG_ERR_ALLOC, with the bytes needed. */
int bsg_ldsplit(bsg_ldcorr *c, double thr_r2, int min_size, const int *max_size, int n_max_size, int max_K, double max_r2,
                double max_cost, const double *pos_scaled, int *kept, double *cost, double *cost2, double *perc_kept,
                int *all_last, int *layers, double *seconds);
/* get_C: src/split-LD.cpp:65-145 from L in CSC (m x (m + 1): lp[m + 2], rows li increasing within each column, lx), as
 * R passes it.  C (m x max_K doubles) and best_ind (m x max_K, 1-based, NA_integer_ where unset), column-major.  Same
 * argument checks and BSG_ERR_ALLOC rule as bsg_ldsplit. */
int bsg_ldsplit_costs(int m, const long long *lp, const int *li, const double *lx, int min_size, int max_size, int max_K,
                      double max_cost, const double *pos_scaled, int device, double *C, int *best_ind);

/* ---- Gram product --------------------------------------------------------------------------------- */
/* bed_tcrossprodSelf's block loop collapsed into one call: R/bed-tcrossprodSelf.R:38-49 +
 * src/bed-mat-acc.cpp:30-49.  K is nr x nr; center/scale are the per-column scaling (length nc). */
int bsg_tcrossprod(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc,
                   const double *center, const double *scale, double *K);
/* Same product, result left in the caller's DEVICE buffer K_dev (nr x nr doubles, full symmetric matrix) so
 * column shards can be summed in place by one all-reduce (SURVEY.md section 8e: GRM row). */
int bsg_tcrossprod_dev(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc,
                       const double *center, const double *scale, double *K_dev);

/* ---- truncated SVD ----------------------------------------------------------------------------------- */
/* bed_randomSVD: R/autoSVD.R:205-219 -> bigstatsr::big_randomSVD -> RSpectra::svds.  The Lanczos
 * iteration runs on the device over the two products above.  center/scale NULL = bed_scaleBinom
 * (R/binom-scaling.R:133-142) computed on the device and returned in center_out/scale_out.
 * d[k], u[nr x k], v[nc x k] column-major. */
int bsg_randomsvd(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc,
                  const double *center, const double *scale, int k, double tol, int maxit, double *d,
                  double *u, double *v, double *center_out, double *scale_out, int *niter, int *nops);

/* Ritz values that met the stopping rule in the last bsg_randomsvd / bsg_randomsvd_ex call of this thread (k when it
 * converged; fewer when `maxit` restarts were not enough -- RSpectra::svds warns in that case and so does the host
 * wrapper); -1 before any call. */
int bsg_randomsvd_nconv(void);

/* Same iteration for a matrix whose SNP columns are sharded over several handles (one per GPU / rank):
 * every rank calls it with its own shard and the same (ind_row, k, tol).  z_dev is a device buffer of nr
 * doubles owned by the caller; after each local A (A^T x) the library synchronises its stream and calls
 * reduce_cb(ctx), which must sum z_dev over the ranks (NCCL all-reduce) and return when the sum is visible
 * to the device.  ncol_total = number of columns of the whole matrix.  u is replicated, v is this rank's
 * rows. */
typedef void (*bsg_reduce_cb)(void *ctx);
int bsg_randomsvd_ex(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc,
                     const double *center, const double *scale, int k, double tol, int maxit, double *d,
                     double *u, double *v, double *center_out, double *scale_out, int *niter, int *nops,
                     double *z_dev, bsg_reduce_cb reduce_cb, void *ctx, int ncol_total);

/* ---- several GPUs (SURVEY.md section 8e; the reference has no multi-device path) ---------------------------------------
 * SNP columns are sharded contiguously over the GPUs (shard g = columns [g*m/G, (g+1)*m/G), first m % G shards one longer).
 * X.y ends in a sum of partial n-vectors over the shards, done INSIDE the product's epilogue kernel over NVLink peer memory;
 * Xt.y, column statistics and v need no exchange; Gram partials are summed by a two-shot all-reduce over peer memory.
 *
 * (1) one host process driving all GPUs -- what an R session is: bsg_group_*.  ind_col is a GLOBAL 1-based multiset. */
int bsg_group_open_bed(const char *path, int n, int m, const int *devices, int ndev, int layouts, bsg_group **out);
int bsg_group_open_synth(int n, int m, uint64_t seed, double na_rate, double ld_rho, int ld_block, const int *devices,
                         int ndev, int layouts, bsg_group **out);
void bsg_group_close(bsg_group *g);
int bsg_group_ndev(const bsg_group *g);
int bsg_group_nrow(const bsg_group *g);
int bsg_group_ncol(const bsg_group *g);
bsg_bed *bsg_group_shard(bsg_group *g, int i);          /* the per-device handle (statistics, counts, decode per shard) */
int bsg_group_shard_begin(const bsg_group *g, int i);   /* first global column (0-based) of shard i; i = ndev gives m */
/* bed_pMatVec4 / bed_cpMatVec4 (src/bed-prod-vec.cpp:15-54, :59-97) over the shards, host vectors, the 9-argument form */
int bsg_group_prodvec(bsg_group *g, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                      const double *scale, const double *x, double *out);
int bsg_group_cprodvec(bsg_group *g, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                       const double *scale, const double *x, double *out);
/* bed_randomSVD (R/autoSVD.R:205-219) over the shards: u[nr x k], v[nc x k] in the caller's column order */
int bsg_group_randomsvd(bsg_group *g, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                        const double *scale, int k, double tol, int maxit, double *d, double *u, double *v,
                        double *center_out, double *scale_out, int *niter, int *nops);
/* bed_tcrossprodSelf (R/bed-tcrossprodSelf.R:21-52) over the shards: K[nr x nr] on the host */
int bsg_group_tcrossprod(bsg_group *g, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                         const double *scale, double *K);

/* (2) one process per GPU (torchrun): every rank creates its end of the communicator (the 64-byte CUDA IPC handle of its
 * region comes back in handle64), the ranks exchange the handles by any means (torch.distributed all_gather) and connect.
 * max_elems = longest vector that will be reduced (n).  After that no host-side exchange happens on the data path. */
int bsg_comm_create(int rank, int world, int device, int64_t max_elems, bsg_comm **out, unsigned char *handle64);
int bsg_comm_connect(bsg_comm *c, const unsigned char *handles /* world x 64 bytes in rank order */);
void bsg_comm_destroy(bsg_comm *c);
int bsg_comm_rank(const bsg_comm *c);
int bsg_comm_world(const bsg_comm *c);
int bsg_comm_check(bsg_comm *c); /* error if a wait inside a collective timed out (a peer never arrived) */
/* in-place sum of count doubles over the ranks, enqueued on `stream`; same bits on every rank */
int bsg_comm_allreduce_dev(bsg_comm *c, double *buf_dev, int64_t count, void *stream);
/* X~ x over this rank's column shard with the sum over the ranks fused into the epilogue kernel: out_dev = full n-vector */
int bsg_view_prodvec_allreduce_dev(bsg_view *v, bsg_comm *c, const double *x_dev, double *out_dev, void *stream);
/* bed_randomSVD on a column-sharded matrix, every rank passing its shard: u, d replicated, v = this rank's rows */
int bsg_randomsvd_comm(bsg_bed *h, bsg_comm *c, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                       const double *scale, int ncol_total, int k, double tol, int maxit, double *d, double *u, double *v,
                       double *center_out, double *scale_out, int *niter, int *nops);

/* ---- instrumentation --------------------------------------------------------------------------------- */
/* kernels launched by this library since load (the bench's gpu_launches claim) */
int64_t bsg_launch_count(void);
/* CUDA-event timing of the matvecs' dominant kernel (k_pmv), recorded on the launching stream:
 * enable with bsg_set_kernel_timing(1); after a stream synchronise bsg_last_kernel_ms() is the device
 * time of the last launch. */
int bsg_set_kernel_timing(int on);
double bsg_last_kernel_ms(void);
/* number of k_pmv launches timed since bsg_set_kernel_timing(1) (at most the last 128) and their summed
 * device time in ms; call after synchronising */
int bsg_kernel_time_stats(int *count, double *total_ms);

#ifdef __cplusplus
}
#endif
#endif /* BSGPU_H */
