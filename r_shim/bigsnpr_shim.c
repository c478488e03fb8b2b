/*
 * bigsnpr_shim.c -- the R side of the drop-in boundary (see INTEGRATION.md).
 *
 * Replaces, inside the bigsnpr package, the generated src/RcppExports.cpp entries of the hot path and the
 * C++ files behind them (src/bed-acc-xptr.cpp, src/bed-prod-vec.cpp, src/bed-fun.cpp, src/bed-mat-acc.cpp,
 * src/corr.cpp, src/ld-scores.cpp, src/colstats.cpp).  Every function keeps the registered name and arity
 * of the reference (src/RcppExports.cpp:597-640), pulls plain pointers out of the SEXPs and calls libbsgpu
 * (include/bsgpu.h).  R's own wrappers (R/RcppExports.R, R/bed-mult-vec.R, R/binom-scaling.R, R/corr.R,
 * R/ld-scores.R) run unchanged.  `ncores` is accepted and ignored.
 *
 * Build (inside the package, needs R headers -- not available in the CUDA build image, so this file is
 * not compiled there):   PKG_LIBS = -L<dir> -lbsgpu     PKG_CPPFLAGS = -I<repo>/include
 */
#include <R.h>
#include <Rinternals.h>
#include <R_ext/Rdynload.h>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include "bsgpu.h"

static void chk(int rc) {
  if (rc) Rf_error("%s", bsg_last_error()); /* same texts as the reference, e.g. "Incompatibility between dimensions." */
}

/* obj$name for RefClass objects / environments (active bindings are evaluated, R/bed-class.R:105-110) */
static SEXP field(SEXP obj, const char *name) {
  SEXP call = PROTECT(Rf_lang3(Rf_install("$"), obj, Rf_mkString(name)));
  SEXP val = Rf_eval(call, R_GlobalEnv);
  UNPROTECT(1);
  return val;
}

static void bed_finalizer(SEXP xp) {
  bsg_bed *h = (bsg_bed *)R_ExternalPtrAddr(xp);
  if (h) bsg_close(h);
  R_ClearExternalPtr(xp);
}

static int gpu_device(void) {
  /* options(bigsnpr.gpu.device = k), default 0 */
  SEXP o = Rf_GetOption1(Rf_install("bigsnpr.gpu.device"));
  return (o == R_NilValue) ? 0 : Rf_asInteger(o);
}

/* options(bigsnpr.gpu.scaling.reuse = TRUE): an unchanged center / scale pair (same R vectors as in the previous call,
 * the pattern of big_randomSVD's closures) is not uploaded again -- include/bsgpu.h, bsg_set_scaling_reuse.  Default off. */
static void apply_scaling_option(void) {
  SEXP o = Rf_GetOption1(Rf_install("bigsnpr.gpu.scaling.reuse"));
  chk(bsg_set_scaling_reuse((o == R_NilValue) ? 0 : (Rf_asInteger(o) != 0)));
}

/* _bigsnpr_bedXPtr(path, n, p): src/bed-acc-xptr.cpp:40-55.  Validation + staging to HBM. */
SEXP _bigsnpr_bedXPtr(SEXP path, SEXP n, SEXP p) {
  bsg_bed *h = NULL;
  int m = Rf_asInteger(p);
  chk(bsg_open_bed(CHAR(STRING_ELT(path, 0)), Rf_asInteger(n), m, 0, m, gpu_device(), BSG_LAYOUT_AUTO, &h));
  SEXP xp = PROTECT(R_MakeExternalPtr(h, R_NilValue, R_NilValue));
  R_RegisterCFinalizerEx(xp, bed_finalizer, TRUE);
  UNPROTECT(1);
  return xp;
}

static bsg_bed *handle_of(SEXP obj_bed) {
  SEXP xp = field(obj_bed, "address"); /* lazily re-opens in PSOCK workers, R/bed-class.R:187-192 */
  bsg_bed *h = (bsg_bed *)R_ExternalPtrAddr(xp);
  if (!h) Rf_error("external pointer is not valid");
  return h;
}

/* _bigsnpr_bed_pMatVec4: src/bed-prod-vec.cpp:15-54 */
SEXP _bigsnpr_bed_pMatVec4(SEXP obj_bed, SEXP ind_row, SEXP ind_col, SEXP center, SEXP scale, SEXP x, SEXP ncores) {
  bsg_bed *h = handle_of(obj_bed);
  apply_scaling_option();
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col);
  if (LENGTH(center) != nc || LENGTH(scale) != nc) Rf_error("Incompatibility between dimensions.");
  SEXP out = PROTECT(Rf_allocVector(REALSXP, nr));
  chk(bsg_prodvec(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, REAL(center), REAL(scale), REAL(x), REAL(out)));
  UNPROTECT(1);
  return out;
}

/* _bigsnpr_bed_cpMatVec4: src/bed-prod-vec.cpp:59-97 */
SEXP _bigsnpr_bed_cpMatVec4(SEXP obj_bed, SEXP ind_row, SEXP ind_col, SEXP center, SEXP scale, SEXP x, SEXP ncores) {
  bsg_bed *h = handle_of(obj_bed);
  apply_scaling_option();
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col);
  if (LENGTH(center) != nc || LENGTH(scale) != nc) Rf_error("Incompatibility between dimensions.");
  SEXP out = PROTECT(Rf_allocVector(REALSXP, nc));
  chk(bsg_cprodvec(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, REAL(center), REAL(scale), REAL(x), REAL(out)));
  UNPROTECT(1);
  return out;
}

/* _bigsnpr_bed_colstats: src/bed-fun.cpp:9-46 -> list(sumX, denoX, nb_nona_col) + the >50% warning */
SEXP _bigsnpr_bed_colstats(SEXP obj_bed, SEXP ind_row, SEXP ind_col, SEXP ncores) {
  bsg_bed *h = handle_of(obj_bed);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col), n_bad = 0;
  SEXP sumX = PROTECT(Rf_allocVector(REALSXP, nc)), denoX = PROTECT(Rf_allocVector(REALSXP, nc));
  SEXP nona = PROTECT(Rf_allocVector(INTSXP, nc));
  chk(bsg_colstats(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, REAL(sumX), REAL(denoX), INTEGER(nona), &n_bad));
  if (n_bad > 0) Rf_warning("%d variants have >50%% missing values.", n_bad);
  SEXP res = PROTECT(Rf_allocVector(VECSXP, 3)), nm = PROTECT(Rf_allocVector(STRSXP, 3));
  SET_VECTOR_ELT(res, 0, sumX); SET_VECTOR_ELT(res, 1, denoX); SET_VECTOR_ELT(res, 2, nona);
  SET_STRING_ELT(nm, 0, Rf_mkChar("sumX")); SET_STRING_ELT(nm, 1, Rf_mkChar("denoX"));
  SET_STRING_ELT(nm, 2, Rf_mkChar("nb_nona_col"));
  Rf_setAttrib(res, R_NamesSymbol, nm);
  UNPROTECT(5);
  return res;
}

/* _bigsnpr_bed_col_counts_cpp / _bigsnpr_bed_row_counts_cpp: src/bed-fun.cpp:51-69, :72-98 */
static SEXP counts(SEXP obj_bed, SEXP ind_row, SEXP ind_col, int byrow) {
  bsg_bed *h = handle_of(obj_bed);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col), k = byrow ? nr : nc;
  SEXP res = PROTECT(Rf_allocMatrix(INTSXP, 4, k));
  chk((byrow ? bsg_row_counts : bsg_col_counts)(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, INTEGER(res)));
  UNPROTECT(1);
  return res;
}
SEXP _bigsnpr_bed_col_counts_cpp(SEXP o, SEXP r, SEXP c, SEXP ncores) { return counts(o, r, c, 0); }
SEXP _bigsnpr_bed_row_counts_cpp(SEXP o, SEXP r, SEXP c, SEXP ncores) { return counts(o, r, c, 1); }

/* _bigsnpr_read_bed: src/bed-mat-acc.cpp:8-26 */
SEXP _bigsnpr_read_bed(SEXP obj_bed, SEXP ind_row, SEXP ind_col) {
  bsg_bed *h = handle_of(obj_bed);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col);
  SEXP res = PROTECT(Rf_allocMatrix(INTSXP, nr, nc));
  chk(bsg_read_bed(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, NA_INTEGER, INTEGER(res)));
  UNPROTECT(1);
  return res;
}

/* _bigsnpr_read_bed_scaled: src/bed-mat-acc.cpp:30-49 */
SEXP _bigsnpr_read_bed_scaled(SEXP obj_bed, SEXP ind_row, SEXP ind_col, SEXP center, SEXP scale) {
  bsg_bed *h = handle_of(obj_bed);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col);
  if (LENGTH(center) != nc || LENGTH(scale) != nc) Rf_error("Incompatibility between dimensions.");
  SEXP res = PROTECT(Rf_allocMatrix(REALSXP, nr, nc));
  chk(bsg_read_bed_scaled(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, REAL(center), REAL(scale), REAL(res)));
  UNPROTECT(1);
  return res;
}

/* bigstatsr's FBM objects (RefClass environments) expose `$backingfile` (the .bk file: nrow x ncol elements of the FBM's
 * type, column-major, no header), `$nrow`, `$ncol` and, for FBM.code256, `$code256`.  The shim maps that file itself
 * (the reference reaches the same bytes through bigstatsr's C++ accessor, src/corr.cpp:113-118), so it depends on no
 * bigstatsr header or symbol.  Writable maps serve the in-place outputs of the reference: the integer FBM `keep` of the
 * clumping routines (R/clumping.R:115, R/bed-clumping.R:51) and the FBM.code256 filled by readbina2. */
static void *fbm_map(SEXP obj, size_t elt_size, int writable, size_t *bytes_out) {
  SEXP bf = field(obj, "backingfile");
  if (TYPEOF(bf) != STRSXP || LENGTH(bf) < 1) Rf_error("object has no backing file");
  const char *path = CHAR(STRING_ELT(bf, 0));
  size_t want = (size_t)Rf_asInteger(field(obj, "nrow")) * (size_t)Rf_asInteger(field(obj, "ncol")) * elt_size;
  int fd = open(path, writable ? O_RDWR : O_RDONLY);
  if (fd < 0) Rf_error("Error when mapping file:\n  %s.\n", path);
  struct stat st;
  if (fstat(fd, &st) != 0 || (size_t)st.st_size < want) {
    close(fd);
    Rf_error("Inconsistency between size of backingfile and dimensions.");
  }
  void *p = want ? mmap(NULL, want, writable ? (PROT_READ | PROT_WRITE) : PROT_READ, MAP_SHARED, fd, 0) : NULL;
  close(fd);
  if (want && p == MAP_FAILED) Rf_error("Error when mapping file:\n  %s.\n", path);
  *bytes_out = want;
  return p;
}
static void fbm_unmap(void *p, size_t bytes, int writable) {
  if (!p || !bytes) return;
  if (writable) msync(p, bytes, MS_SYNC); /* R reads the result through its own mapping of the same file */
  munmap(p, bytes);
}

/* FBM.code256 objects (snp_cor / snp_ld_scores / snp_colstats / snp_clumping / snp_pcadapt / snp_writeBed): the n x m
 * bytes are staged to HBM once per object; the handle is cached in the environment (variable ".bsg"). */
static bsg_bed *fbm_handle_of(SEXP obj) {
  SEXP cached = Rf_findVarInFrame(obj, Rf_install(".bsg"));
  if (cached != R_UnboundValue && TYPEOF(cached) == EXTPTRSXP && R_ExternalPtrAddr(cached))
    return (bsg_bed *)R_ExternalPtrAddr(cached);
  int n = Rf_asInteger(field(obj, "nrow")), m = Rf_asInteger(field(obj, "ncol"));
  SEXP code = PROTECT(Rf_coerceVector(field(obj, "code256"), REALSXP));
  if (LENGTH(code) != 256) Rf_error("'code256' must have 256 values.");
  size_t bytes = 0;
  void *raw = fbm_map(obj, 1, 0, &bytes);
  bsg_bed *h = NULL;
  int rc = bsg_open_fbm256((const uint8_t *)raw, n, m, REAL(code), gpu_device(), BSG_LAYOUT_SNP_MAJOR, &h);
  fbm_unmap(raw, bytes, 0);
  chk(rc);
  SEXP xp = PROTECT(R_MakeExternalPtr(h, R_NilValue, R_NilValue));
  R_RegisterCFinalizerEx(xp, bed_finalizer, TRUE);
  Rf_defineVar(Rf_install(".bsg"), xp, obj);
  UNPROTECT(2);
  return h;
}

static int has_field(SEXP obj, const char *name) { return Rf_findVarInFrame(obj, Rf_install(name)) != R_UnboundValue; }

/* dispatch of src/corr.cpp:113-125: "code256" -> FBM, "bedfile" -> bed, else "Unknown object type." */
static bsg_bed *any_handle(SEXP obj) {
  if (has_field(obj, "code256")) return fbm_handle_of(obj);
  if (has_field(obj, "bedfile")) return handle_of(obj);
  Rf_error("Unknown object type.");
  return NULL;
}

/* _bigsnpr_snp_colstats: src/colstats.cpp:8-35 */
SEXP _bigsnpr_snp_colstats(SEXP BM, SEXP rowInd, SEXP colInd, SEXP ncores) {
  bsg_bed *h = fbm_handle_of(BM);
  int nr = LENGTH(rowInd), nc = LENGTH(colInd);
  SEXP sumX = PROTECT(Rf_allocVector(REALSXP, nc)), denoX = PROTECT(Rf_allocVector(REALSXP, nc));
  chk(bsg_snp_colstats(h, INTEGER(rowInd), nr, INTEGER(colInd), nc, REAL(sumX), REAL(denoX)));
  SEXP res = PROTECT(Rf_allocVector(VECSXP, 2)), nm = PROTECT(Rf_allocVector(STRSXP, 2));
  SET_VECTOR_ELT(res, 0, sumX); SET_VECTOR_ELT(res, 1, denoX);
  SET_STRING_ELT(nm, 0, Rf_mkChar("sumX")); SET_STRING_ELT(nm, 1, Rf_mkChar("denoX"));
  Rf_setAttrib(res, R_NamesSymbol, nm);
  UNPROTECT(4);
  return res;
}

/* _bigsnpr_corMat: src/corr.cpp:102-126 -> list of m lists {i, x} (R/corr.R:43-47 assembles the dsCMatrix) */
SEXP _bigsnpr_corMat(SEXP obj, SEXP rowInd, SEXP colInd, SEXP size, SEXP thr, SEXP pos, SEXP fill_diag, SEXP ncores) {
  int nr = LENGTH(rowInd), nc = LENGTH(colInd);
  if (LENGTH(pos) != nc) Rf_error("Incompatibility between dimensions.");
  bsg_bed *h = any_handle(obj);
  int64_t *p = (int64_t *)R_alloc((size_t)nc + 1, sizeof(int64_t));
  int *ci = NULL;
  double *cx = NULL;
  chk(bsg_cor(h, INTEGER(rowInd), nr, INTEGER(colInd), nc, Rf_asReal(size), REAL(thr), REAL(pos), Rf_asLogical(fill_diag),
              p, &ci, &cx));
  SEXP res = PROTECT(Rf_allocVector(VECSXP, nc));
  SEXP nm = PROTECT(Rf_allocVector(STRSXP, 2));
  SET_STRING_ELT(nm, 0, Rf_mkChar("i")); SET_STRING_ELT(nm, 1, Rf_mkChar("x"));
  for (int j = 0; j < nc; j++) {
    int len = (int)(p[j + 1] - p[j]);
    SEXP el = PROTECT(Rf_allocVector(VECSXP, 2)), vi = PROTECT(Rf_allocVector(INTSXP, len));
    SEXP vx = PROTECT(Rf_allocVector(REALSXP, len));
    for (int k = 0; k < len; k++) { INTEGER(vi)[k] = ci[p[j] + k]; REAL(vx)[k] = cx[p[j] + k]; }
    SET_VECTOR_ELT(el, 0, vi); SET_VECTOR_ELT(el, 1, vx);
    Rf_setAttrib(el, R_NamesSymbol, nm);
    SET_VECTOR_ELT(res, j, el);
    UNPROTECT(3);
  }
  bsg_free(ci); bsg_free(cx);
  UNPROTECT(2);
  return res;
}

/* _bigsnpr_ld_scores: src/ld-scores.cpp:83-105 */
SEXP _bigsnpr_ld_scores(SEXP obj, SEXP rowInd, SEXP colInd, SEXP size, SEXP pos, SEXP ncores) {
  int nr = LENGTH(rowInd), nc = LENGTH(colInd);
  if (LENGTH(pos) != nc) Rf_error("Incompatibility between dimensions.");
  bsg_bed *h = any_handle(obj);
  SEXP out = PROTECT(Rf_allocVector(REALSXP, nc));
  chk(bsg_ld_scores(h, INTEGER(rowInd), nr, INTEGER(colInd), nc, Rf_asReal(size), REAL(pos), REAL(out)));
  UNPROTECT(1);
  return out;
}

/* _bigsnpr_bed_clumping_chr: src/clumping-bed.cpp:11-91 (12 arguments).  BM2 is the 1 x nc integer FBM `keep`
 * (R/bed-clumping.R:51), written in place through its backing file; rankInd is implied by ordInd. */
SEXP _bigsnpr_bed_clumping_chr(SEXP obj_bed, SEXP BM2, SEXP ind_row, SEXP ind_col, SEXP center, SEXP scale, SEXP ordInd,
                               SEXP rankInd, SEXP pos, SEXP size, SEXP thr, SEXP ncores) {
  bsg_bed *h = handle_of(obj_bed);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col);
  if (LENGTH(center) != nc || LENGTH(scale) != nc || LENGTH(pos) != nc || LENGTH(ordInd) != nc)
    Rf_error("Incompatibility between dimensions.");
  size_t bytes = 0;
  int *keep = (int *)fbm_map(BM2, sizeof(int), 1, &bytes);
  if (bytes < (size_t)nc * sizeof(int)) { fbm_unmap(keep, bytes, 1); Rf_error("Incompatibility between dimensions."); }
  int rc = bsg_clumping_chr(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, REAL(center), REAL(scale), INTEGER(ordInd), REAL(pos),
                            Rf_asReal(size), Rf_asReal(thr), keep);
  fbm_unmap(keep, bytes, 1);
  chk(rc);
  return R_NilValue;
}

/* _bigsnpr_clumping_chr: src/clumping.cpp:10-91 (12 arguments; BM is the FBM.code256 environment, src/clumping.cpp:24-25) */
SEXP _bigsnpr_clumping_chr(SEXP BM, SEXP BM2, SEXP rowInd, SEXP colInd, SEXP ordInd, SEXP rankInd, SEXP pos, SEXP sumX,
                           SEXP denoX, SEXP size, SEXP thr, SEXP ncores) {
  bsg_bed *h = fbm_handle_of(BM);
  int nr = LENGTH(rowInd), nc = LENGTH(colInd);
  if (LENGTH(sumX) != nc || LENGTH(denoX) != nc || LENGTH(pos) != nc || LENGTH(ordInd) != nc)
    Rf_error("Incompatibility between dimensions.");
  size_t bytes = 0;
  int *keep = (int *)fbm_map(BM2, sizeof(int), 1, &bytes);
  if (bytes < (size_t)nc * sizeof(int)) { fbm_unmap(keep, bytes, 1); Rf_error("Incompatibility between dimensions."); }
  int rc = bsg_clumping_chr_fbm(h, INTEGER(rowInd), nr, INTEGER(colInd), nc, REAL(sumX), REAL(denoX), INTEGER(ordInd), REAL(pos),
                                Rf_asReal(size), Rf_asReal(thr), keep);
  fbm_unmap(keep, bytes, 1);
  chk(rc);
  return R_NilValue;
}

/* _bigsnpr_clumping_chr_cached: src/clumping-cached.cpp:11-110 (14 arguments; one grid point of snp_grid_clumping,
 * R/SCT.R:121-135).  keep goes into BM2 as for _bigsnpr_clumping_chr.  The reference's sparse r2 cache never changes a
 * decision (a pair's r2 is the same whenever it is computed), so sqcor is returned as passed: R/SCT.R subsets it and hands it
 * back, which is valid for any cache value.  spInd and rankInd (implied by ordInd) are not needed. */
SEXP _bigsnpr_clumping_chr_cached(SEXP BM, SEXP BM2, SEXP sqcor, SEXP spInd, SEXP rowInd, SEXP colInd, SEXP ordInd,
                                  SEXP rankInd, SEXP pos, SEXP sumX, SEXP denoX, SEXP size, SEXP thr, SEXP ncores) {
  bsg_bed *h = fbm_handle_of(BM);
  int nr = LENGTH(rowInd), nc = LENGTH(colInd);
  if (LENGTH(spInd) != nc) Rf_error("Incompatibility between dimensions.");  /* myassert_size(spInd.size(), m) */
  if (LENGTH(sumX) != nc || LENGTH(denoX) != nc || LENGTH(pos) != nc || LENGTH(ordInd) != nc)
    Rf_error("Incompatibility between dimensions.");
  size_t bytes = 0;
  int *keep = (int *)fbm_map(BM2, sizeof(int), 1, &bytes);
  if (bytes < (size_t)nc * sizeof(int)) { fbm_unmap(keep, bytes, 1); Rf_error("Incompatibility between dimensions."); }
  int rc = bsg_clumping_chr_fbm(h, INTEGER(rowInd), nr, INTEGER(colInd), nc, REAL(sumX), REAL(denoX), INTEGER(ordInd), REAL(pos),
                                Rf_asReal(size), Rf_asReal(thr), keep);
  fbm_unmap(keep, bytes, 1);
  chk(rc);
  return sqcor;
}

/* _bigsnpr_readbina2: src/read-plink.cpp:61-80 (5 arguments; BM is the destination FBM.code256, filled in place; the R
 * wrapper creates it with exactly length(ind_row) x length(ind_col) bytes, R/read-plink.R:93-100) */
SEXP _bigsnpr_readbina2(SEXP BM, SEXP obj_bed, SEXP ind_row, SEXP ind_col, SEXP ncores) {
  bsg_bed *h = handle_of(obj_bed);
  size_t bytes = 0, want = (size_t)LENGTH(ind_row) * (size_t)LENGTH(ind_col);
  unsigned char *dst = (unsigned char *)fbm_map(BM, 1, 1, &bytes);
  if (bytes != want) { fbm_unmap(dst, bytes, 1); Rf_error("Incompatibility between dimensions."); }
  int rc = bsg_readbina2(h, INTEGER(ind_row), LENGTH(ind_row), INTEGER(ind_col), LENGTH(ind_col), dst);
  fbm_unmap(dst, bytes, 1);
  chk(rc);
  return R_NilValue;
}

/* _bigsnpr_writebina: src/write-plink.cpp:13-52 (5 arguments; BM is the FBM.code256 of the bigSNP, src/write-plink.cpp:19-20;
 * `tab` = getInverseCode() is implied by the library) */
SEXP _bigsnpr_writebina(SEXP filename, SEXP BM, SEXP tab, SEXP rowInd, SEXP colInd) {
  bsg_bed *h = fbm_handle_of(BM);
  chk(bsg_writebina(h, CHAR(STRING_ELT(filename, 0)), INTEGER(rowInd), LENGTH(rowInd), INTEGER(colInd), LENGTH(colInd)));
  return R_NilValue;
}

/* _bigsnpr_prod_and_rowSumsSq: src/bed-fun.cpp:103-133 (6 arguments) -> list(XV, rowSumsSq) */
SEXP _bigsnpr_prod_and_rowSumsSq(SEXP obj_bed, SEXP ind_row, SEXP ind_col, SEXP center, SEXP scale, SEXP V) {
  bsg_bed *h = handle_of(obj_bed);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col), K = Rf_ncols(V);
  if (LENGTH(center) != nc || LENGTH(scale) != nc || Rf_nrows(V) != nc) Rf_error("Incompatibility between dimensions.");
  SEXP XV = PROTECT(Rf_allocMatrix(REALSXP, nr, K)), rss = PROTECT(Rf_allocVector(REALSXP, nr));
  chk(bsg_prod_and_rowsumssq(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, REAL(center), REAL(scale), REAL(V), K, REAL(XV),
                             REAL(rss)));
  SEXP res = PROTECT(Rf_allocVector(VECSXP, 2));
  SET_VECTOR_ELT(res, 0, XV);
  SET_VECTOR_ELT(res, 1, rss);
  UNPROTECT(3);
  return res;
}

/* _bigsnpr_prod_and_rowSumsSq2: src/project-utils.cpp:11-43 (6 arguments; `BM` is an FBM.code256 environment, hard calls
 * or a dosage table) -> list(XV, rowSumsSq); a row holding an NA code in a selected column is NaN (NA_real in the reference) */
SEXP _bigsnpr_prod_and_rowSumsSq2(SEXP BM, SEXP ind_row, SEXP ind_col, SEXP center, SEXP scale, SEXP V) {
  bsg_bed *h = fbm_handle_of(BM);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col), K = Rf_ncols(V);
  if (LENGTH(center) != nc || LENGTH(scale) != nc || Rf_nrows(V) != nc) Rf_error("Incompatibility between dimensions.");
  SEXP XV = PROTECT(Rf_allocMatrix(REALSXP, nr, K)), rss = PROTECT(Rf_allocVector(REALSXP, nr));
  chk(bsg_prod_and_rowsumssq2(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, REAL(center), REAL(scale), REAL(V), K,
                              REAL(XV), REAL(rss)));
  SEXP res = PROTECT(Rf_allocVector(VECSXP, 2));
  SET_VECTOR_ELT(res, 0, XV);
  SET_VECTOR_ELT(res, 1, rss);
  UNPROTECT(3);
  return res;
}

/* _bigsnpr_multLinReg: src/multLinReg.cpp:64-88 (5 arguments; `obj` is a bed or an FBM.code256 environment) */
SEXP _bigsnpr_multLinReg(SEXP obj, SEXP ind_row, SEXP ind_col, SEXP U, SEXP ncores) {
  bsg_bed *h = any_handle(obj); /* src/multLinReg.cpp:72-78: FBM.code256 or bed, else "Unknown object type." */
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col), K = Rf_ncols(U);
  if (Rf_nrows(U) != nr) Rf_error("Incompatibility between dimensions.");
  SEXP t = PROTECT(Rf_allocMatrix(REALSXP, nc, K));
  chk(bsg_multlinreg(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, REAL(U), K, REAL(t)));
  for (R_xlen_t i = 0; i < XLENGTH(t); i++)
    if (ISNAN(REAL(t)[i])) REAL(t)[i] = NA_REAL; /* the library writes NaN where the reference writes NA_REAL */
  UNPROTECT(1);
  return t;
}

/* new entry points: R/bed-tcrossprodSelf.R's block loop and R/autoSVD.R's bed_randomSVD collapse to one call each */
SEXP _bigsnpr_bed_tcrossprod_gpu(SEXP obj_bed, SEXP ind_row, SEXP ind_col, SEXP center, SEXP scale) {
  bsg_bed *h = handle_of(obj_bed);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col);
  SEXP K = PROTECT(Rf_allocMatrix(REALSXP, nr, nr));
  chk(bsg_tcrossprod(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, REAL(center), REAL(scale), REAL(K)));
  UNPROTECT(1);
  return K;
}

/* `obj_bed` may also be an FBM.code256 environment (big_randomSVD's branch of snp_autoSVD passes G): a dosage table needs
 * center / scale (snp_scaleBinom); NULL scaling (bed_scaleBinom) needs hard calls */
SEXP _bigsnpr_bed_randomSVD_gpu(SEXP obj_bed, SEXP ind_row, SEXP ind_col, SEXP center, SEXP scale, SEXP k, SEXP tol) {
  bsg_bed *h = any_handle(obj_bed);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col), kk = Rf_asInteger(k), niter = 0, nops = 0;
  SEXP d = PROTECT(Rf_allocVector(REALSXP, kk)), u = PROTECT(Rf_allocMatrix(REALSXP, nr, kk));
  SEXP v = PROTECT(Rf_allocMatrix(REALSXP, nc, kk));
  SEXP co = PROTECT(Rf_allocVector(REALSXP, nc)), so = PROTECT(Rf_allocVector(REALSXP, nc));
  const double *cen = (center == R_NilValue) ? NULL : REAL(center), *sca = (scale == R_NilValue) ? NULL : REAL(scale);
  chk(bsg_randomsvd(h, INTEGER(ind_row), nr, INTEGER(ind_col), nc, cen, sca, kk, Rf_asReal(tol), 1000, REAL(d), REAL(u),
                    REAL(v), REAL(co), REAL(so), &niter, &nops));
  const char *names[] = {"d", "u", "v", "niter", "nops", "center", "scale", ""};
  SEXP res = PROTECT(Rf_mkNamed(VECSXP, names));
  SET_VECTOR_ELT(res, 0, d); SET_VECTOR_ELT(res, 1, u); SET_VECTOR_ELT(res, 2, v);
  SET_VECTOR_ELT(res, 3, Rf_ScalarInteger(niter)); SET_VECTOR_ELT(res, 4, Rf_ScalarInteger(nops));
  SET_VECTOR_ELT(res, 5, co); SET_VECTOR_ELT(res, 6, so);
  Rf_setAttrib(res, R_ClassSymbol, Rf_mkString("big_SVD"));
  UNPROTECT(6);
  return res;
}

/* ---- several GPUs from the one R process (SURVEY.md section 8e): options(bigsnpr.gpu.devices = c(0, 1, ...)) --------------
 * A group handle shards the file's SNP columns over the listed devices; the two new symbols mirror the single-GPU ones. */
static void group_finalizer(SEXP xp) {
  bsg_group *g = (bsg_group *)R_ExternalPtrAddr(xp);
  if (g) bsg_group_close(g);
  R_ClearExternalPtr(xp);
}
SEXP _bigsnpr_bed_group_gpu(SEXP path, SEXP n, SEXP p, SEXP devices) {
  bsg_group *g = NULL;
  chk(bsg_group_open_bed(CHAR(STRING_ELT(path, 0)), Rf_asInteger(n), Rf_asInteger(p), INTEGER(devices), LENGTH(devices),
                         BSG_LAYOUT_AUTO, &g));
  SEXP xp = PROTECT(R_MakeExternalPtr(g, R_NilValue, R_NilValue));
  R_RegisterCFinalizerEx(xp, group_finalizer, TRUE);
  UNPROTECT(1);
  return xp;
}
static bsg_group *group_of(SEXP xp) {
  bsg_group *g = (TYPEOF(xp) == EXTPTRSXP) ? (bsg_group *)R_ExternalPtrAddr(xp) : NULL;
  if (!g) Rf_error("external pointer is not valid");
  return g;
}
SEXP _bigsnpr_group_pMatVec4_gpu(SEXP grp, SEXP ind_row, SEXP ind_col, SEXP center, SEXP scale, SEXP x, SEXP transpose) {
  bsg_group *g = group_of(grp);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col), tr = Rf_asLogical(transpose);
  if (LENGTH(center) != nc || LENGTH(scale) != nc || LENGTH(x) != (tr ? nr : nc)) Rf_error("Incompatibility between dimensions.");
  SEXP out = PROTECT(Rf_allocVector(REALSXP, tr ? nc : nr));
  chk((tr ? bsg_group_cprodvec : bsg_group_prodvec)(g, INTEGER(ind_row), nr, INTEGER(ind_col), nc, REAL(center), REAL(scale),
                                                    REAL(x), REAL(out)));
  UNPROTECT(1);
  return out;
}
SEXP _bigsnpr_group_randomSVD_gpu(SEXP grp, SEXP ind_row, SEXP ind_col, SEXP center, SEXP scale, SEXP k, SEXP tol) {
  bsg_group *g = group_of(grp);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col), kk = Rf_asInteger(k), niter = 0, nops = 0;
  SEXP d = PROTECT(Rf_allocVector(REALSXP, kk)), u = PROTECT(Rf_allocMatrix(REALSXP, nr, kk));
  SEXP v = PROTECT(Rf_allocMatrix(REALSXP, nc, kk));
  SEXP co = PROTECT(Rf_allocVector(REALSXP, nc)), so = PROTECT(Rf_allocVector(REALSXP, nc));
  const double *cen = (center == R_NilValue) ? NULL : REAL(center), *sca = (scale == R_NilValue) ? NULL : REAL(scale);
  chk(bsg_group_randomsvd(g, INTEGER(ind_row), nr, INTEGER(ind_col), nc, cen, sca, kk, Rf_asReal(tol), 1000, REAL(d), REAL(u),
                          REAL(v), REAL(co), REAL(so), &niter, &nops));
  const char *names[] = {"d", "u", "v", "niter", "nops", "center", "scale", ""};
  SEXP res = PROTECT(Rf_mkNamed(VECSXP, names));
  SET_VECTOR_ELT(res, 0, d); SET_VECTOR_ELT(res, 1, u); SET_VECTOR_ELT(res, 2, v);
  SET_VECTOR_ELT(res, 3, Rf_ScalarInteger(niter)); SET_VECTOR_ELT(res, 4, Rf_ScalarInteger(nops));
  SET_VECTOR_ELT(res, 5, co); SET_VECTOR_ELT(res, 6, so);
  Rf_setAttrib(res, R_ClassSymbol, Rf_mkString("big_SVD"));
  UNPROTECT(6);
  return res;
}
SEXP _bigsnpr_group_tcrossprod_gpu(SEXP grp, SEXP ind_row, SEXP ind_col, SEXP center, SEXP scale) {
  bsg_group *g = group_of(grp);
  int nr = LENGTH(ind_row), nc = LENGTH(ind_col);
  if (LENGTH(center) != nc || LENGTH(scale) != nc) Rf_error("Incompatibility between dimensions.");
  SEXP K = PROTECT(Rf_allocMatrix(REALSXP, nr, nr));
  chk(bsg_group_tcrossprod(g, INTEGER(ind_row), nr, INTEGER(ind_col), nc, REAL(center), REAL(scale), REAL(K)));
  UNPROTECT(1);
  return K;
}

/* ---- sparse LD matrix (bigsparser's SFBM) ----------------------------------------------------------------------------
 * An SFBM environment carries $p (ncol + 1 doubles), $nrow, $ncol and, in the compact form, $first_i (ncol integers); the
 * reference reads $p and $first_i the same way (src/ld-scores-sfbm.cpp:18,29).  The stored doubles live in a data file:
 * interleaved (row, value) pairs, 2 p[ncol] doubles, or p[ncol] values when compact.  The field naming that file is taken
 * to be $sbk; bigsparser is not vendored, so this name is unconfirmed until the shim runs under R (INTEGRATION.md).  The
 * file is mapped once, staged to HBM, and the handle is cached in the environment (variable ".bsg_sfbm"). */
static void sfbm_finalizer(SEXP xp) {
  bsg_sfbm *s = (bsg_sfbm *)R_ExternalPtrAddr(xp);
  if (s) bsg_sfbm_close(s);
  R_ClearExternalPtr(xp);
}
static bsg_sfbm *sfbm_handle_of(SEXP obj) {
  SEXP cached = Rf_findVarInFrame(obj, Rf_install(".bsg_sfbm"));
  if (cached != R_UnboundValue && TYPEOF(cached) == EXTPTRSXP && R_ExternalPtrAddr(cached))
    return (bsg_sfbm *)R_ExternalPtrAddr(cached);
  int nrow = Rf_asInteger(field(obj, "nrow")), ncol = Rf_asInteger(field(obj, "ncol"));
  SEXP p = PROTECT(Rf_coerceVector(field(obj, "p"), REALSXP));
  if (ncol < 0 || LENGTH(p) != ncol + 1) Rf_error("Incompatibility between dimensions.");
  SEXP fi = has_field(obj, "first_i") ? field(obj, "first_i") : R_NilValue;
  const int compact = fi != R_NilValue && LENGTH(fi) == ncol && ncol > 0;
  if (compact) fi = Rf_coerceVector(fi, INTSXP);
  PROTECT(fi);
  const double nval = ncol > 0 ? REAL(p)[ncol] : 0;
  if (!(nval >= 0) || nval > 4e15) Rf_error("Inconsistency between size of backingfile and dimensions.");
  const size_t want = (size_t)nval * (compact ? 1 : 2) * sizeof(double);
  SEXP bf = field(obj, "sbk");
  if (TYPEOF(bf) != STRSXP || LENGTH(bf) < 1) Rf_error("object has no backing file");
  const char *path = CHAR(STRING_ELT(bf, 0));
  int fd = open(path, O_RDONLY);
  if (fd < 0) Rf_error("Error when mapping file:\n  %s.\n", path);
  struct stat st;
  if (fstat(fd, &st) != 0 || (size_t)st.st_size < want) {
    close(fd);
    Rf_error("Inconsistency between size of backingfile and dimensions.");
  }
  void *data = want ? mmap(NULL, want, PROT_READ, MAP_SHARED, fd, 0) : NULL;
  close(fd);
  if (want && data == MAP_FAILED) Rf_error("Error when mapping file:\n  %s.\n", path);
  bsg_sfbm *s = NULL;
  int rc = bsg_sfbm_open(nrow, ncol, REAL(p), (const double *)data, compact ? INTEGER(fi) : NULL, gpu_device(), &s);
  if (data) munmap(data, want);
  chk(rc);
  SEXP xp = PROTECT(R_MakeExternalPtr(s, R_NilValue, R_NilValue));
  R_RegisterCFinalizerEx(xp, sfbm_finalizer, TRUE);
  Rf_defineVar(Rf_install(".bsg_sfbm"), xp, obj);
  UNPROTECT(3);
  return s;
}

/* _bigsnpr_lassosum2: src/lassosum2.cpp:20-70, one grid point per call (R/lassosum2.R:56-69 loops over the grid with
 * foreach, so each call takes one SM); the batched grid is bsg_lassosum2 with ngrid > 1 (C ABI, Python mirror) */
SEXP _bigsnpr_lassosum2(SEXP corr, SEXP beta_hat, SEXP lambda, SEXP delta_plus_one, SEXP ind_sub, SEXP dfmax, SEXP maxiter,
                        SEXP tol) {
  bsg_sfbm *s = sfbm_handle_of(corr);
  SEXP bh = PROTECT(Rf_coerceVector(beta_hat, REALSXP)), lam = PROTECT(Rf_coerceVector(lambda, REALSXP));
  SEXP dp1 = PROTECT(Rf_coerceVector(delta_plus_one, REALSXP)), sub = PROTECT(Rf_coerceVector(ind_sub, INTSXP));
  int m = LENGTH(bh), it = 0;
  if (LENGTH(lam) != m || LENGTH(dp1) != m || LENGTH(sub) != m) Rf_error("Incompatibility between dimensions.");
  SEXP beta = PROTECT(Rf_allocVector(REALSXP, m));
  chk(bsg_lassosum2(s, REAL(bh), m, INTEGER(sub), 1, REAL(lam), REAL(dp1), Rf_asReal(dfmax), Rf_asInteger(maxiter),
                    Rf_asReal(tol), REAL(beta), &it, NULL));
  const char *names[] = {"beta_est", "num_iter", ""};
  SEXP res = PROTECT(Rf_mkNamed(VECSXP, names));
  SET_VECTOR_ELT(res, 0, beta);
  SET_VECTOR_ELT(res, 1, Rf_ScalarInteger(it));
  UNPROTECT(6);
  return res;
}

/* _bigsnpr_ld_scores_sfbm: src/ld-scores-sfbm.cpp:9-69 (ind_sub 0-based, as R/LDpred2.R:228-229 passes it) */
SEXP _bigsnpr_ld_scores_sfbm(SEXP X, SEXP ind_sub, SEXP ncores) {
  bsg_sfbm *s = sfbm_handle_of(X);
  SEXP sub = PROTECT(Rf_coerceVector(ind_sub, INTSXP));
  int m = LENGTH(sub);
  SEXP out = PROTECT(Rf_allocVector(REALSXP, m));
  chk(bsg_sfbm_ld_scores(s, INTEGER(sub), m, REAL(out)));
  UNPROTECT(2);
  return out;
}

/* p of a CSC matrix (integer, or double for very large ones, as R/split-LD.R:127 passes it) as 64-bit offsets */
static long long *csc_offsets(SEXP p) {
  SEXP pd = PROTECT(Rf_coerceVector(p, REALSXP));
  R_xlen_t n = XLENGTH(pd);
  long long *out = (long long *)R_alloc(n ? n : 1, sizeof(long long));
  for (R_xlen_t k = 0; k < n; k++) out[k] = (long long)REAL(pd)[k];
  UNPROTECT(1);
  return out;
}

/* _bigsnpr_get_L: src/split-LD.cpp:15-61 on Matrix::tril(corr)'s p, i, x (R/split-LD.R:116-117); list of 0-based i, j,
 * x triplets in the reference's order.  The matrix is staged for this call only. */
SEXP _bigsnpr_get_L(SEXP p, SEXP i, SEXP x, SEXP thr_r2, SEXP max_r2) {
  SEXP ii = PROTECT(Rf_coerceVector(i, INTSXP)), xx = PROTECT(Rf_coerceVector(x, REALSXP));
  long long *pp = csc_offsets(p);
  int m = (int)XLENGTH(p) - 1;
  if (m < 1 || pp[m] != XLENGTH(ii) || XLENGTH(xx) != XLENGTH(ii)) Rf_error("Incompatibility between dimensions.");
  bsg_ldcorr *c = NULL;
  chk(bsg_ldcorr_open(m, pp, INTEGER(ii), REAL(xx), gpu_device(), &c));
  long long n = 0;
  int rc = bsg_ldcorr_l_triplets(c, Rf_asReal(thr_r2), Rf_asReal(max_r2), &n, 0, NULL, NULL, NULL);
  if (rc) {
    bsg_ldcorr_close(c);
    chk(rc);
  }
  const char *names[] = {"i", "j", "x", ""};
  SEXP res = PROTECT(Rf_mkNamed(VECSXP, names));
  SEXP ri = PROTECT(Rf_allocVector(INTSXP, n)), rj = PROTECT(Rf_allocVector(INTSXP, n)), rx = PROTECT(Rf_allocVector(REALSXP, n));
  rc = bsg_ldcorr_l_triplets(c, Rf_asReal(thr_r2), Rf_asReal(max_r2), &n, n, INTEGER(ri), INTEGER(rj), REAL(rx));
  bsg_ldcorr_close(c);
  chk(rc);
  SET_VECTOR_ELT(res, 0, ri);
  SET_VECTOR_ELT(res, 1, rj);
  SET_VECTOR_ELT(res, 2, rx);
  UNPROTECT(6);
  return res;
}

/* _bigsnpr_get_C: src/split-LD.cpp:65-145 on the m x (m + 1) dgCMatrix L that R/split-LD.R:118-120 builds (its p, i, x
 * and Dim slots); list of C (m x max_K) and best_ind.  Any other matrix class is refused. */
SEXP _bigsnpr_get_C(SEXP L, SEXP min_size, SEXP max_size, SEXP max_K, SEXP max_cost, SEXP pos_scaled) {
  if (!Rf_inherits(L, "dgCMatrix")) Rf_error("'L' must be a dgCMatrix.");
  SEXP dim = PROTECT(Rf_coerceVector(Rf_getAttrib(L, Rf_install("Dim")), INTSXP));
  SEXP li = PROTECT(Rf_coerceVector(Rf_getAttrib(L, Rf_install("i")), INTSXP));
  SEXP lx = PROTECT(Rf_coerceVector(Rf_getAttrib(L, Rf_install("x")), REALSXP));
  SEXP pos = PROTECT(Rf_coerceVector(pos_scaled, REALSXP));
  SEXP lpv = Rf_getAttrib(L, Rf_install("p"));
  if (XLENGTH(dim) != 2) Rf_error("Incompatibility between dimensions.");
  int m = INTEGER(dim)[0], K = Rf_asInteger(max_K);
  if (INTEGER(dim)[1] != m + 1 || XLENGTH(lpv) != (R_xlen_t)m + 2 || XLENGTH(pos) != m || XLENGTH(li) != XLENGTH(lx))
    Rf_error("Incompatibility between dimensions.");
  long long *lp = csc_offsets(lpv);
  if (lp[m + 1] != XLENGTH(li)) Rf_error("Incompatibility between dimensions.");
  if (K < 1) Rf_error("max_K must be at least 1.");
  const char *names[] = {"C", "best_ind", ""};
  SEXP res = PROTECT(Rf_mkNamed(VECSXP, names));
  SEXP C = PROTECT(Rf_allocMatrix(REALSXP, m, K)), best = PROTECT(Rf_allocMatrix(INTSXP, m, K));
  chk(bsg_ldsplit_costs(m, lp, INTEGER(li), REAL(lx), Rf_asInteger(min_size), Rf_asInteger(max_size), K,
                        Rf_asReal(max_cost), REAL(pos), gpu_device(), REAL(C), INTEGER(best)));
  SET_VECTOR_ELT(res, 0, C);
  SET_VECTOR_ELT(res, 1, best);
  UNPROTECT(7);
  return res;
}

/* registration: same table shape as src/RcppExports.cpp:597-640 (only the hot-path rows shown; the other
 * entries of the reference stay as generated) */
static const R_CallMethodDef CallEntries[] = {
    {"_bigsnpr_bedXPtr", (DL_FUNC)&_bigsnpr_bedXPtr, 3},
    {"_bigsnpr_bed_colstats", (DL_FUNC)&_bigsnpr_bed_colstats, 4},
    {"_bigsnpr_bed_col_counts_cpp", (DL_FUNC)&_bigsnpr_bed_col_counts_cpp, 4},
    {"_bigsnpr_bed_row_counts_cpp", (DL_FUNC)&_bigsnpr_bed_row_counts_cpp, 4},
    {"_bigsnpr_read_bed", (DL_FUNC)&_bigsnpr_read_bed, 3},
    {"_bigsnpr_read_bed_scaled", (DL_FUNC)&_bigsnpr_read_bed_scaled, 5},
    {"_bigsnpr_bed_pMatVec4", (DL_FUNC)&_bigsnpr_bed_pMatVec4, 7},
    {"_bigsnpr_bed_cpMatVec4", (DL_FUNC)&_bigsnpr_bed_cpMatVec4, 7},
    {"_bigsnpr_snp_colstats", (DL_FUNC)&_bigsnpr_snp_colstats, 4},
    {"_bigsnpr_corMat", (DL_FUNC)&_bigsnpr_corMat, 8},
    {"_bigsnpr_ld_scores", (DL_FUNC)&_bigsnpr_ld_scores, 6},
    {"_bigsnpr_bed_clumping_chr", (DL_FUNC)&_bigsnpr_bed_clumping_chr, 12},
    {"_bigsnpr_clumping_chr", (DL_FUNC)&_bigsnpr_clumping_chr, 12},
    {"_bigsnpr_clumping_chr_cached", (DL_FUNC)&_bigsnpr_clumping_chr_cached, 14},
    {"_bigsnpr_readbina2", (DL_FUNC)&_bigsnpr_readbina2, 5},
    {"_bigsnpr_writebina", (DL_FUNC)&_bigsnpr_writebina, 5},
    {"_bigsnpr_prod_and_rowSumsSq", (DL_FUNC)&_bigsnpr_prod_and_rowSumsSq, 6},
    {"_bigsnpr_prod_and_rowSumsSq2", (DL_FUNC)&_bigsnpr_prod_and_rowSumsSq2, 6},
    {"_bigsnpr_multLinReg", (DL_FUNC)&_bigsnpr_multLinReg, 5},
    {"_bigsnpr_lassosum2", (DL_FUNC)&_bigsnpr_lassosum2, 8},
    {"_bigsnpr_ld_scores_sfbm", (DL_FUNC)&_bigsnpr_ld_scores_sfbm, 3},
    {"_bigsnpr_get_L", (DL_FUNC)&_bigsnpr_get_L, 5},
    {"_bigsnpr_get_C", (DL_FUNC)&_bigsnpr_get_C, 6},
    {"_bigsnpr_bed_tcrossprod_gpu", (DL_FUNC)&_bigsnpr_bed_tcrossprod_gpu, 5},
    {"_bigsnpr_bed_randomSVD_gpu", (DL_FUNC)&_bigsnpr_bed_randomSVD_gpu, 7},
    {"_bigsnpr_bed_group_gpu", (DL_FUNC)&_bigsnpr_bed_group_gpu, 4},
    {"_bigsnpr_group_pMatVec4_gpu", (DL_FUNC)&_bigsnpr_group_pMatVec4_gpu, 7},
    {"_bigsnpr_group_randomSVD_gpu", (DL_FUNC)&_bigsnpr_group_randomSVD_gpu, 7},
    {"_bigsnpr_group_tcrossprod_gpu", (DL_FUNC)&_bigsnpr_group_tcrossprod_gpu, 5},
    {NULL, NULL, 0}};

void R_init_bigsnpr_hotpath(DllInfo *dll) {
  /* in the package this table is merged into R_init_bigsnpr (src/RcppExports.cpp:637-640) */
  R_registerRoutines(dll, NULL, CallEntries, NULL, NULL);
  R_useDynamicSymbols(dll, FALSE);
}
