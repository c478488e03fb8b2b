/*
 * bsg_oracle.c -- CPU restatement of the bigsnpr hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  This file is the parity oracle and the CPU baseline
 * ("cpu_baseline.kind = port") for the H100 engine.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product
 * (libbsgpu.so) never links, loads or calls anything in this directory.
 *
 * The reference itself (privefl/bigsnpr 1.12.21) cannot be compiled in this image: it needs
 * R, Rcpp, RcppArmadillo, bigstatsr and rmio headers (SURVEY.md section 8c).  Each function below
 * restates one reference loop, scalar and literal (same operation order, same parenthesisation,
 * same OpenMP work split), citing the file:line it follows under /root/reference.
 * Parity of this oracle is pinned against the reference's own fixtures in tests/test_oracle.py:
 * inst/extdata/example.bed, example-missing.bed and tests/testthat/testdata/example.ld.
 *
 * Conventions kept from the reference: ind_row / ind_col are 1-based int32 (R integer vectors),
 * matrices are column-major, `bed` points at the first genotype byte (file offset 3).
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#else
static int omp_get_thread_num(void) { return 0; }
#endif

#define ORC_OK 0
#define ORC_ERR_DIM 1      /* "Incompatibility between dimensions." (src/bed-acc.h:95-96) */
#define ORC_ERR_BOUNDS 2   /* subscript out of bounds (bigstatsr vec_int_to_size, src/bed-acc.h:64-65) */
#define ORC_ERR_MAGIC 3    /* "File is not a binary PED file." (src/bed-acc-xptr.cpp:21-22) */
#define ORC_ERR_MODE 4     /* "Variant-major is the only mode supported." (src/bed-acc-xptr.cpp:29-30) */
#define ORC_ERR_SIZE 5     /* "n or p does not match the dimensions of the file." (src/bed-acc-xptr.cpp:33-34) */
#define ORC_ERR_IO 6
#define ORC_ERR_ALLOC 7

/* ------------------------------------------------------------------------------------------ */
/* src/bed-acc.h:22-37  bed::get_code : 4 x 256 table, num = {2, NA, 1, 0} indexed by the 2-bit  */
/* code, row i = sample slot within the byte (lowest bits first).                               */
static int g_lookup_byte[4][256];
static int g_lookup_ready = 0;

static void build_lookup(void) {
  static const int num[4] = {2, 3, 1, 0};
  int coeff = 1;
  for (int i = 0; i < 4; i++) {
    for (int k = 0; k < 256; k++) {
      int k2 = k / coeff;
      g_lookup_byte[i][k] = num[k2 % 4];
    }
    coeff *= 4;
  }
  g_lookup_ready = 1;
}

void orc_get_code(int na_val, int *out /* 4 x 256 column-major, as IntegerMatrix(4,256) */) {
  if (!g_lookup_ready) build_lookup();
  for (int k = 0; k < 256; k++)
    for (int i = 0; i < 4; i++) {
      int v = g_lookup_byte[i][k];
      out[i + 4 * k] = (v == 3) ? na_val : v;
    }
}

/* src/bed-acc-xptr.cpp:14-34  bed::bed : header and size validation. */
int orc_bed_validate(const char *path, int n, int m) {
  FILE *f = fopen(path, "rb");
  if (!f) return ORC_ERR_IO;
  unsigned char hdr[3];
  if (fread(hdr, 1, 3, f) != 3) { fclose(f); return ORC_ERR_MAGIC; }
  fseek(f, 0, SEEK_END);
  long long sz = ftell(f);
  fclose(f);
  if (!(hdr[0] == 0x6C && hdr[1] == 0x1B)) return ORC_ERR_MAGIC;
  if (hdr[2] != 0x01) return ORC_ERR_MODE;
  long long n_byte = ((long long)n + 3) / 4;
  if (3 + n_byte * (long long)m != sz) return ORC_ERR_SIZE;
  return ORC_OK;
}

/* ------------------------------------------------------------------------------------------ */
/* Accessors.  kind 0: bedAcc over a .bed (src/bed-acc.h:52-82).                               */
/*             kind 1: SubBMCode256Acc over an FBM.code256 backing file [bigstatsr, unvendored] */
/*                     value = code256[byte], matrix is n_tot x m_tot bytes, column-major.      */
typedef struct {
  int kind;
  const uint8_t *mat;
  size_t n_tot, m_tot, n_byte;
  const double *code256; /* kind 1 */
  size_t nr, nc;
  size_t *ind_row, *ind_col; /* 0-based */
} acc_t;

static int acc_init(acc_t *a, int kind, const uint8_t *mat, size_t n_tot, size_t m_tot,
                    const double *code256, const int *ind_row, size_t nr, const int *ind_col,
                    size_t nc) {
  if (!g_lookup_ready) build_lookup();
  a->kind = kind;
  a->mat = mat;
  a->n_tot = n_tot;
  a->m_tot = m_tot;
  a->n_byte = (n_tot + 3) / 4;
  a->code256 = code256;
  a->nr = nr;
  a->nc = nc;
  a->ind_row = (size_t *)malloc((nr ? nr : 1) * sizeof(size_t));
  a->ind_col = (size_t *)malloc((nc ? nc : 1) * sizeof(size_t));
  if (!a->ind_row || !a->ind_col) return ORC_ERR_ALLOC;
  /* vec_int_to_size(ind, limit, 1): 1-based -> 0-based with bounds check (src/bed-acc.h:64-65) */
  for (size_t i = 0; i < nr; i++) {
    long long v = (long long)ind_row[i] - 1;
    if (v < 0 || (size_t)v >= n_tot) return ORC_ERR_BOUNDS;
    a->ind_row[i] = (size_t)v;
  }
  for (size_t j = 0; j < nc; j++) {
    long long v = (long long)ind_col[j] - 1;
    if (v < 0 || (size_t)v >= m_tot) return ORC_ERR_BOUNDS;
    a->ind_col[j] = (size_t)v;
  }
  return ORC_OK;
}

static void acc_free(acc_t *a) {
  free(a->ind_row);
  free(a->ind_col);
}

/* src/bed-acc.h:71-75  bedAcc::operator() */
static inline int bed_get(const acc_t *a, size_t i, size_t j) {
  size_t i2 = a->ind_row[i];
  unsigned char byte = a->mat[i2 / 4 + a->ind_col[j] * a->n_byte];
  return g_lookup_byte[i2 % 4][byte];
}

/* generic "value with NA == 3" accessor used by corMat0 / ld_scores0 (src/corr.cpp:113-122) */
static inline double acc_get3(const acc_t *a, size_t i, size_t j) {
  if (a->kind == 0) return (double)bed_get(a, i, j);
  unsigned char byte = a->mat[a->ind_row[i] + a->ind_col[j] * a->n_tot];
  double v = a->code256[byte];
  return isnan(v) ? 3.0 : v; /* code[is_na(code)] = 3  (src/corr.cpp:115) */
}

/* src/bed-acc.h:86-115  bedAccScaled : per-column 4-entry table, NA -> 0. */
static double *build_lookup_scale(size_t p, const double *center, const double *scale) {
  double *t = (double *)malloc((p ? p : 1) * 4 * sizeof(double));
  if (!t) return NULL;
  for (size_t j = 0; j < p; j++) {
    for (size_t i = 0; i < 3; i++) t[i + 4 * j] = ((double)i - center[j]) / scale[j];
    t[3 + 4 * j] = 0.0;
  }
  return t;
}

/* ------------------------------------------------------------------------------------------ */
/* src/bed-prod-vec.cpp:15-54  bed_pMatVec4 :  out = X~ x ; per-thread partial vectors then      */
/* rowSums, 4-column unrolling with the reference's parenthesisation.                           */
int orc_pMatVec4(const uint8_t *bed, int n_tot, int m_tot, const int *ind_row, int nr,
                 const int *ind_col, int nc, const double *center, const double *scale,
                 const double *x, int ncores, double *out) {
  acc_t a;
  int rc = acc_init(&a, 0, bed, n_tot, m_tot, NULL, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  double *ls = build_lookup_scale(nc, center, scale);
  if (ncores < 1) ncores = 1;
  double *res = (double *)calloc((size_t)(nr ? nr : 1) * ncores, sizeof(double));
  if (!ls || !res) { free(ls); free(res); acc_free(&a); return ORC_ERR_ALLOC; }

#pragma omp parallel num_threads(ncores)
  {
    int id = omp_get_thread_num();
    double *r = res + (size_t)id * nr;
    int n2 = nr;
    int m = nc;
    int m2 = m - 3;
    int i, j;
#pragma omp for nowait
    for (j = 0; j < m2; j += 4) {
      for (i = 0; i < n2; i++) {
        r[i] += (x[j] * ls[bed_get(&a, i, j) + 4 * (size_t)j] +
                 x[j + 1] * ls[bed_get(&a, i, j + 1) + 4 * (size_t)(j + 1)]) +
                (x[j + 2] * ls[bed_get(&a, i, j + 2) + 4 * (size_t)(j + 2)] +
                 x[j + 3] * ls[bed_get(&a, i, j + 3) + 4 * (size_t)(j + 3)]);
      }
    }
#pragma omp for
    for (j = m - m % 4; j < m; j++) {
      for (i = 0; i < n2; i++) r[i] += x[j] * ls[bed_get(&a, i, j) + 4 * (size_t)j];
    }
  }
  /* rowSums(res) (src/bed-prod-vec.cpp:53): thread partials summed left to right */
  for (int i = 0; i < nr; i++) {
    double s = 0;
    for (int t = 0; t < ncores; t++) s += res[(size_t)t * nr + i];
    out[i] = s;
  }
  free(ls);
  free(res);
  acc_free(&a);
  return ORC_OK;
}

/* src/bed-prod-vec.cpp:59-97  bed_cpMatVec4 :  out = t(X~) x ; 4-row unrolling, fixed order. */
int orc_cpMatVec4(const uint8_t *bed, int n_tot, int m_tot, const int *ind_row, int nr,
                  const int *ind_col, int nc, const double *center, const double *scale,
                  const double *x, int ncores, double *out) {
  acc_t a;
  int rc = acc_init(&a, 0, bed, n_tot, m_tot, NULL, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  double *ls = build_lookup_scale(nc, center, scale);
  if (!ls) { acc_free(&a); return ORC_ERR_ALLOC; }
  if (ncores < 1) ncores = 1;
  int m = nc;
#pragma omp parallel num_threads(ncores)
  {
    int n = nr;
    int n2 = n - 3;
#pragma omp for
    for (int j = 0; j < m; j++) {
      const double *lj = ls + 4 * (size_t)j;
      double tmp = 0;
      int i = 0;
      for (; i < n2; i += 4) {
        tmp += (lj[bed_get(&a, i, j)] * x[i] + lj[bed_get(&a, i + 1, j)] * x[i + 1]) +
               (lj[bed_get(&a, i + 2, j)] * x[i + 2] + lj[bed_get(&a, i + 3, j)] * x[i + 3]);
      }
      for (; i < n; i++) tmp += lj[bed_get(&a, i, j)] * x[i];
      out[j] = tmp;
    }
  }
  free(ls);
  acc_free(&a);
  return ORC_OK;
}

/* src/bed-fun.cpp:9-46  bed_colstats : sumX, denoX = sum x^2 - (sum x)^2 / c, nb_nona_col = c.  */
/* returns in *n_bad the count behind the ">50% missing values" warning (:40-41).              */
int orc_bed_colstats(const uint8_t *bed, int n_tot, int m_tot, const int *ind_row, int nr,
                     const int *ind_col, int nc, int ncores, double *sumX, double *denoX,
                     int *nb_nona_col, int *n_bad) {
  acc_t a;
  int rc = acc_init(&a, 0, bed, n_tot, m_tot, NULL, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  if (ncores < 1) ncores = 1;
  int n = nr, m = nc;
#pragma omp parallel for num_threads(ncores)
  for (int j = 0; j < m; j++) {
    double xSum = 0, xxSum = 0;
    int c = n;
    for (int i = 0; i < n; i++) {
      double x = bed_get(&a, i, j);
      if (x != 3) {
        xSum += x;
        xxSum += x * x;
      } else {
        c--;
      }
    }
    sumX[j] = xSum;
    denoX[j] = xxSum - xSum * xSum / c;
    nb_nona_col[j] = c;
  }
  int bad = 0;
  for (int j = 0; j < m; j++) bad += (2 * nb_nona_col[j] < n);
  if (n_bad) *n_bad = bad;
  acc_free(&a);
  return ORC_OK;
}

/* src/bed-fun.cpp:51-69  bed_col_counts_cpp : 4 x nc counts of {0,1,2,NA}, column-major. */
int orc_bed_col_counts(const uint8_t *bed, int n_tot, int m_tot, const int *ind_row, int nr,
                       const int *ind_col, int nc, int ncores, int *res /* 4 x nc */) {
  acc_t a;
  int rc = acc_init(&a, 0, bed, n_tot, m_tot, NULL, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  if (ncores < 1) ncores = 1;
  size_t n = nr, m = nc;
  memset(res, 0, 4 * m * sizeof(int));
#pragma omp parallel for num_threads(ncores)
  for (size_t j = 0; j < m; j++)
    for (size_t i = 0; i < n; i++) res[bed_get(&a, i, j) + 4 * j]++;
  acc_free(&a);
  return ORC_OK;
}

/* src/bed-fun.cpp:72-98  bed_row_counts_cpp : 4 x nr counts, thread-local then merged. */
int orc_bed_row_counts(const uint8_t *bed, int n_tot, int m_tot, const int *ind_row, int nr,
                       const int *ind_col, int nc, int ncores, int *res /* 4 x nr */) {
  acc_t a;
  int rc = acc_init(&a, 0, bed, n_tot, m_tot, NULL, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  if (ncores < 1) ncores = 1;
  size_t n = nr, m = nc;
  memset(res, 0, 4 * n * sizeof(int));
#pragma omp parallel num_threads(ncores)
  {
    int *loc = (int *)calloc(4 * (n ? n : 1), sizeof(int));
#pragma omp for
    for (size_t j = 0; j < m; j++)
      for (size_t i = 0; i < n; i++) loc[bed_get(&a, i, j) + 4 * i]++;
#pragma omp critical
    for (size_t k = 0; k < 4 * n; k++) res[k] += loc[k];
    free(loc);
  }
  acc_free(&a);
  return ORC_OK;
}

/* src/bed-mat-acc.cpp:8-26  read_bed : dense decode, NA -> na_val (R: NA_INTEGER). */
int orc_read_bed(const uint8_t *bed, int n_tot, int m_tot, const int *ind_row, int nr,
                 const int *ind_col, int nc, int na_val, int *res /* nr x nc */) {
  acc_t a;
  int rc = acc_init(&a, 0, bed, n_tot, m_tot, NULL, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  for (size_t j = 0; j < (size_t)nc; j++)
    for (size_t i = 0; i < (size_t)nr; i++) {
      int g = bed_get(&a, i, j);
      res[i + (size_t)nr * j] = (g == 3) ? na_val : g;
    }
  acc_free(&a);
  return ORC_OK;
}

/* src/bed-mat-acc.cpp:30-49  read_bed_scaled : dense (g - center_j) / scale_j, NA -> 0. */
int orc_read_bed_scaled(const uint8_t *bed, int n_tot, int m_tot, const int *ind_row, int nr,
                        const int *ind_col, int nc, const double *center, const double *scale,
                        double *res /* nr x nc */) {
  acc_t a;
  int rc = acc_init(&a, 0, bed, n_tot, m_tot, NULL, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  double *ls = build_lookup_scale(nc, center, scale);
  if (!ls) { acc_free(&a); return ORC_ERR_ALLOC; }
  for (size_t j = 0; j < (size_t)nc; j++)
    for (size_t i = 0; i < (size_t)nr; i++)
      res[i + (size_t)nr * j] = ls[bed_get(&a, i, j) + 4 * j];
  free(ls);
  acc_free(&a);
  return ORC_OK;
}

/* src/bed-fun.cpp:103-133  prod_and_rowSumsSq : XV (nr x K) and row sums of squares. */
int orc_prod_and_rowSumsSq(const uint8_t *bed, int n_tot, int m_tot, const int *ind_row, int nr,
                           const int *ind_col, int nc, const double *center, const double *scale,
                           const double *V /* nc x K */, int K, double *XV /* nr x K */,
                           double *rowSumsSq /* nr */) {
  acc_t a;
  int rc = acc_init(&a, 0, bed, n_tot, m_tot, NULL, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  double *ls = build_lookup_scale(nc, center, scale);
  if (!ls) { acc_free(&a); return ORC_ERR_ALLOC; }
  size_t n = nr, m = nc;
  memset(XV, 0, n * (size_t)K * sizeof(double));
  memset(rowSumsSq, 0, n * sizeof(double));
  for (size_t j = 0; j < m; j++)
    for (size_t i = 0; i < n; i++) {
      double x = ls[bed_get(&a, i, j) + 4 * j];
      rowSumsSq[i] += x * x;
      for (size_t k = 0; k < (size_t)K; k++) XV[i + n * k] += x * V[j + m * k];
    }
  free(ls);
  acc_free(&a);
  return ORC_OK;
}

/* src/multLinReg.cpp:8-60  multLinReg : per SNP and per column k of U, the t-score of the simple linear
 * regression of the genotype on U[,k] over the samples where the genotype is present.  The sums run in sample
 * order in fp64 like the reference; the statistic is written with the reference's operation order (:44-51).
 * `tscores` is nc x K column-major (the reference returns transpose(res), :56).  NA_REAL is written as NaN. */
int orc_multLinReg(int kind, const uint8_t *mat, int n_tot, int m_tot, const double *code256,
                   const int *ind_row, int nr, const int *ind_col, int nc, const double *U /* nr x K */,
                   int K, int ncores, double *tscores /* nc x K */) {
  acc_t a;
  int rc = acc_init(&a, kind, mat, n_tot, m_tot, code256, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  if (ncores < 1) ncores = 1;
  const size_t n = nr, m = nc;
  int failed = 0;
#pragma omp parallel num_threads(ncores)
  {
    double *sums = (double *)malloc((size_t)(K > 0 ? K : 1) * 3 * sizeof(double));
    if (!sums) {
#pragma omp atomic write
      failed = 1;
    }
#pragma omp for
    for (size_t j = 0; j < m; j++) {
      if (!sums) continue;
      double *xy = sums, *ys = sums + K, *yy = sums + 2 * (size_t)K;
      for (int k = 0; k < 3 * K; k++) sums[k] = 0;
      int nona = (int)n;
      double xSum = 0, xxSum = 0;
      for (size_t i = 0; i < n; i++) {
        const double x = acc_get3(&a, i, j);
        if (x == 3) { nona--; continue; }
        xSum += x;
        xxSum += x * x;
        for (int k = 0; k < K; k++) {
          const double y = U[i + n * (size_t)k];
          xy[k] += x * y;
          ys[k] += y;
          yy[k] += y * y;
        }
      }
      const double deno_x = xxSum - xSum * xSum / nona;
      for (int k = 0; k < K; k++) {
        const double num = xy[k] - xSum * ys[k] / nona;
        const double deno_y = yy[k] - ys[k] * ys[k] / nona;
        const double deno = deno_x * deno_y - num * num;
        tscores[j + m * (size_t)k] = (deno == 0 || nona < 2) ? NAN : num * sqrt((nona - 2) / deno);
      }
    }
    free(sums);
  }
  acc_free(&a);
  return failed ? ORC_ERR_ALLOC : ORC_OK;
}

/* src/colstats.cpp:8-35  snp_colstats : FBM.code256 column sums, no NA handling. */
int orc_snp_colstats(const uint8_t *bk, int n_tot, int m_tot, const double *code256,
                     const int *ind_row, int nr, const int *ind_col, int nc, int ncores,
                     double *sumX, double *denoX) {
  acc_t a;
  int rc = acc_init(&a, 1, bk, n_tot, m_tot, code256, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  if (ncores < 1) ncores = 1;
  size_t n = nr, m = nc;
#pragma omp parallel for num_threads(ncores)
  for (size_t j = 0; j < m; j++) {
    double xSum = 0, xxSum = 0;
    for (size_t i = 0; i < n; i++) {
      double x = a.code256[a.mat[a.ind_row[i] + a.ind_col[j] * a.n_tot]];
      xSum += x;
      xxSum += x * x;
    }
    sumX[j] = xSum;
    denoX[j] = xxSum - xSum * xSum / n;
  }
  acc_free(&a);
  return ORC_OK;
}

/* ------------------------------------------------------------------------------------------ */
/* src/corr.cpp:11-97  corMat0 : windowed pairwise-complete Pearson r.                          */
/* Output as CSC pieces: p (nc+1), i (0-based, ascending, diagonal last), x.  Caller frees      */
/* *pi / *px with orc_free.  kind 0 = bed, kind 1 = FBM.code256 (src/corr.cpp:102-126).         */
typedef struct { int *ind; double *val; size_t len, cap; } colbuf_t;

static int colbuf_push(colbuf_t *b, int i, double v) {
  if (b->len == b->cap) {
    size_t nc = b->cap ? 2 * b->cap : 16;
    int *ni = (int *)realloc(b->ind, nc * sizeof(int));
    double *nv = (double *)realloc(b->val, nc * sizeof(double));
    if (!ni || !nv) return 1;
    b->ind = ni; b->val = nv; b->cap = nc;
  }
  b->ind[b->len] = i;
  b->val[b->len] = v;
  b->len++;
  return 0;
}

int orc_corMat(int kind, const uint8_t *mat, int n_tot, int m_tot, const double *code256,
               const int *ind_row, int nr, const int *ind_col, int nc, double size,
               const double *thr /* nr */, const double *pos /* nc */, int fill_diag, int ncores,
               long long *p /* nc+1 */, int **pi, double **px) {
  acc_t a;
  int rc = acc_init(&a, kind, mat, n_tot, m_tot, code256, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  if (ncores < 1) ncores = 1;
  int n = nr, m = nc;
  colbuf_t *cols = (colbuf_t *)calloc(m ? m : 1, sizeof(colbuf_t));
  int chunk_size = (int)ceil(m / (10.0 * ncores));
  if (chunk_size < 1) chunk_size = 1;
  int fail = 0;

#pragma omp parallel for schedule(dynamic, chunk_size) num_threads(ncores)
  for (int j0 = 0; j0 < m; j0++) {
    colbuf_t *cb = &cols[j0];
    if (fill_diag) fail |= colbuf_push(cb, j0, 1.0);

    double xSum0 = 0, xxSum0 = 0;
    for (int i = 0; i < n; i++) {
      double x = acc_get3(&a, i, j0);
      if (x != 3) {
        xSum0 += x;
        xxSum0 += x * x;
      }
    }

    double pos_min = pos[j0] - size;
    for (int j = j0 - 1; (j >= 0) && (pos[j] >= pos_min); j--) {
      int nona = 0;
      double xSum = xSum0, xxSum = xxSum0;
      double ySum = 0, yySum = 0, xySum = 0;
      for (int i = 0; i < n; i++) {
        double x = acc_get3(&a, i, j0);
        if (x == 3) continue;
        double y = acc_get3(&a, i, j);
        if (y == 3) {
          xSum -= x;
          xxSum -= x * x;
        } else {
          nona++;
          ySum += y;
          yySum += y * y;
          xySum += x * y;
        }
      }
      double num = xySum - xSum * ySum / nona;
      double deno_x = xxSum - xSum * xSum / nona;
      double deno_y = yySum - ySum * ySum / nona;
      double r = num / sqrt(deno_x * deno_y);

      /* thr[nona - 1] with nona == 0 reads thr[-1] in the reference (undefined); r is NaN
         there anyway (0/0), so the ISNAN branch decides. */
      if (isnan(r) || fabs(r) > thr[nona > 0 ? nona - 1 : 0]) {
        if (r > 1) r = 1; else if (r < -1) r = -1;
        fail |= colbuf_push(cb, j, r);
      }
    }
  }

  long long tot = 0;
  for (int j = 0; j < m; j++) { p[j] = tot; tot += (long long)cols[j].len; }
  p[m] = tot;
  int *oi = (int *)malloc((tot ? tot : 1) * sizeof(int));
  double *ox = (double *)malloc((tot ? tot : 1) * sizeof(double));
  if (!oi || !ox || fail) {
    for (int j = 0; j < m; j++) { free(cols[j].ind); free(cols[j].val); }
    free(cols); free(oi); free(ox); acc_free(&a);
    return ORC_ERR_ALLOC;
  }
  /* rev(ind), rev(val) (src/corr.cpp:90-92): ascending row index, diagonal last */
  for (int j = 0; j < m; j++) {
    size_t len = cols[j].len;
    for (size_t k = 0; k < len; k++) {
      oi[p[j] + k] = cols[j].ind[len - 1 - k];
      ox[p[j] + k] = cols[j].val[len - 1 - k];
    }
    free(cols[j].ind);
    free(cols[j].val);
  }
  free(cols);
  *pi = oi;
  *px = ox;
  acc_free(&a);
  return ORC_OK;
}

void orc_free(void *ptr) { free(ptr); }

/* src/ld-scores.cpp:11-78  ld_scores0 : res = 1 + sum r^2 over both members of each pair. */
int orc_ld_scores(int kind, const uint8_t *mat, int n_tot, int m_tot, const double *code256,
                  const int *ind_row, int nr, const int *ind_col, int nc, double size,
                  const double *pos, int ncores, double *res) {
  acc_t a;
  int rc = acc_init(&a, kind, mat, n_tot, m_tot, code256, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  if (ncores < 1) ncores = 1;
  int n = nr, m = nc;
  for (int j = 0; j < m; j++) res[j] = 1;
  int chunk_size = (int)ceil(m / (10.0 * ncores));
  if (chunk_size < 1) chunk_size = 1;

#pragma omp parallel for schedule(dynamic, chunk_size) num_threads(ncores)
  for (int j0 = 0; j0 < m; j0++) {
    double xSum0 = 0, xxSum0 = 0;
    for (int i = 0; i < n; i++) {
      double x = acc_get3(&a, i, j0);
      if (x != 3) {
        xSum0 += x;
        xxSum0 += x * x;
      }
    }
    double pos_min = pos[j0] - size;
    for (int j = j0 - 1; (j >= 0) && (pos[j] >= pos_min); j--) {
      int nona = 0;
      double xSum = xSum0, xxSum = xxSum0;
      double ySum = 0, yySum = 0, xySum = 0;
      for (int i = 0; i < n; i++) {
        double x = acc_get3(&a, i, j0);
        if (x == 3) continue;
        double y = acc_get3(&a, i, j);
        if (y == 3) {
          xSum -= x;
          xxSum -= x * x;
        } else {
          nona++;
          ySum += y;
          yySum += y * y;
          xySum += x * y;
        }
      }
      double num = xySum - xSum * ySum / nona;
      double deno_x = xxSum - xSum * xSum / nona;
      double deno_y = yySum - ySum * ySum / nona;
      double r2 = num * num / (deno_x * deno_y);
      if (!isnan(r2)) {
#pragma omp atomic
        res[j0] += r2;
#pragma omp atomic
        res[j] += r2;
      }
    }
  }
  acc_free(&a);
  return ORC_OK;
}

/* src/clumping-utils.h:12-43  which_to_check : neighbours of j0 inside the window with a better rank that are
 * not (yet) pruned, alternating right / left by increasing distance. */
static int which_to_check(int j0, const int *keep, const int *rankInd, const double *pos, int m, double size,
                          int *out) {
  int cnt = 0;
  double pos_min = pos[j0] - size, pos_max = pos[j0] + size;
  int not_min = 1, not_max = 1;
  for (int k = 1; not_max || not_min; k++) {
    if (not_max) {
      int j = j0 + k;
      not_max = (j < m) && (pos[j] <= pos_max);
      if (not_max && (rankInd[j0] > rankInd[j]) && (keep[j] != 0)) out[cnt++] = j;
    }
    if (not_min) {
      int j = j0 - k;
      not_min = (j >= 0) && (pos[j] >= pos_min);
      if (not_min && (rankInd[j0] > rankInd[j]) && (keep[j] != 0)) out[cnt++] = j;
    }
  }
  return cnt;
}

/* src/clumping-bed.cpp:11-91  bed_clumping_chr : greedy clumping in rank order on scaled dot products
 * r = sum_i macc(i, j) * macc(i, j0) (missing -> 0 after scaling).  Restated for one thread: the reference's
 * OpenMP version spin-waits on keep[] so that its result is the same for any ncores
 * (tests/testthat/test-2-bed-clumping-SVD.R:83). keep must come in filled with -1. */
int orc_bed_clumping_chr(const uint8_t *bed, int n_tot, int m_tot, const int *ind_row, int nr, const int *ind_col,
                         int nc, const double *center, const double *scale, const int *ordInd,
                         const int *rankInd, const double *pos, double size, double thr, int *keep) {
  acc_t a;
  int rc = acc_init(&a, 0, bed, n_tot, m_tot, NULL, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  double *ls = build_lookup_scale(nc, center, scale);
  int *chk = (int *)malloc((size_t)(nc ? nc : 1) * sizeof(int));
  if (!ls || !chk) { free(ls); free(chk); acc_free(&a); return ORC_ERR_ALLOC; }
  size_t n = nr, m = nc;
  for (size_t k = 0; k < m; k++) {
    size_t j0 = (size_t)ordInd[k] - 1;
    int nb_check = which_to_check((int)j0, keep, rankInd, pos, (int)m, size, chk);
    int keep_j0 = 1;
    for (int k2 = 0; k2 < nb_check; k2++) {
      int jk = chk[k2];
      if (keep[jk] == 0) continue; /* pruned: nothing to check (one thread: never -1 here) */
      size_t j = (size_t)jk;
      double r = 0;
      for (size_t i = 0; i < n; i++)
        r += ls[bed_get(&a, i, j) + 4 * j] * ls[bed_get(&a, i, j0) + 4 * j0];
      double r2 = r * r;
      if (r2 > thr) {
        keep_j0 = 0;
        break;
      }
    }
    keep[j0] = keep_j0;
  }
  free(ls);
  free(chk);
  acc_free(&a);
  return ORC_OK;
}

/* src/clumping.cpp:10-91  clumping_chr : the FBM.code256 twin.  Statistic (:66-73):
 *   xySum = sum_i macc(i, j) * macc(i, j0);  num = xySum - sumX[j] * sumX[j0] / n;
 *   r2 = num * num / (denoX[j] * denoX[j0])
 * with the accessor's code256 values (NA_real for a missing code, so r2 is NA and never > thr).  One thread, same
 * remark as above.  keep must come in filled with -1. */
int orc_clumping_chr(int kind, const uint8_t *mat, int n_tot, int m_tot, const double *code256, const int *ind_row,
                     int nr, const int *ind_col, int nc, const int *ordInd, const int *rankInd, const double *pos,
                     const double *sumX, const double *denoX, double size, double thr, int *keep) {
  acc_t a;
  int rc = acc_init(&a, kind, mat, n_tot, m_tot, code256, ind_row, nr, ind_col, nc);
  if (rc) { acc_free(&a); return rc; }
  int *chk = (int *)malloc((size_t)(nc ? nc : 1) * sizeof(int));
  if (!chk) { acc_free(&a); return ORC_ERR_ALLOC; }
  size_t n = nr, m = nc;
  for (size_t k = 0; k < m; k++) {
    size_t j0 = (size_t)ordInd[k] - 1;
    int nb_check = which_to_check((int)j0, keep, rankInd, pos, (int)m, size, chk);
    int keep_j0 = 1;
    for (int k2 = 0; k2 < nb_check; k2++) {
      int jk = chk[k2];
      if (keep[jk] == 0) continue;
      size_t j = (size_t)jk;
      double xySum = 0;
      for (size_t i = 0; i < n; i++) {
        double xa = acc_get3(&a, i, j), xb = acc_get3(&a, i, j0);
        if (xa == 3) xa = NAN; /* SubBMCode256Acc returns the code itself: NA_real for a missing genotype */
        if (xb == 3) xb = NAN;
        xySum += xa * xb;
      }
      double num = xySum - sumX[j] * sumX[j0] / n;
      double r2 = num * num / (denoX[j] * denoX[j0]);
      if (r2 > thr) {
        keep_j0 = 0;
        break;
      }
    }
    keep[j0] = keep_j0;
  }
  free(chk);
  acc_free(&a);
  return ORC_OK;
}

/* Synthetic .bed generator (SURVEY.md section 8d), the CPU twin of the device generator
 * (bigsnpr_b200/csrc/bsg_core.cu: k_synth): per-SNP maf ~ U(0.02, 0.5), g ~ Binomial(2, maf), missing with
 * probability na_rate; written in the .bed bit layout of src/write-plink.cpp:29-47 (pads = 00). */
static inline uint64_t orc_mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

void orc_synth_packed(int n, int m, uint64_t seed, double na_rate, long long col_offset, uint8_t *out) {
  static const uint8_t bedcode[4] = {3, 2, 0, 1}; /* genotype 0,1,2,NA -> .bed code 11,10,00,01 */
  size_t n_byte = ((size_t)n + 3) / 4;
  uint32_t na_thr = (uint32_t)(na_rate * 65536.0);
#pragma omp parallel for schedule(static)
  for (int j = 0; j < m; j++) {
    uint64_t kj = orc_mix64(seed ^ orc_mix64((uint64_t)(col_offset + j)));
    double maf = 0.02 + 0.48 * ((double)(kj >> 11) * (1.0 / 9007199254740992.0));
    uint32_t thr = (uint32_t)(maf * 16777216.0);
    uint8_t *col = out + (size_t)j * n_byte;
    memset(col, 0, n_byte);
    for (int i = 0; i < n; i++) {
      uint64_t hs = orc_mix64(kj + (uint64_t)i * 0xD1342543DE82EF95ull);
      uint32_t g = ((uint32_t)(hs & 0xFFFFFFu) < thr) + ((uint32_t)((hs >> 24) & 0xFFFFFFu) < thr);
      if ((uint32_t)((hs >> 48) & 0xFFFFu) < na_thr) g = 3;
      col[i >> 2] |= (uint8_t)(bedcode[g] << (2 * (i & 3)));
    }
  }
}

/* LD-structured twin of the device generator k_synth_ld (bigsnpr_b200/csrc/bsg_core.cu): inside every block of
 * `ld_block` global columns a haplotype's 24-bit allele uniform is copied from the previous SNP with probability rho
 * (16 bits of a second hash per haplotype).  Integer arithmetic only -> the same bytes as the device. */
void orc_synth_packed_ld(int n, int m, uint64_t seed, double na_rate, long long col_offset, double rho, int ld_block,
                         uint8_t *out) {
  static const uint8_t bedcode[4] = {3, 2, 0, 1};
  size_t n_byte = ((size_t)n + 3) / 4;
  uint32_t na_thr = (uint32_t)(na_rate * 65536.0), rho_thr = (uint32_t)(rho * 65536.0);
  long long gb0 = col_offset / ld_block, nblk = (col_offset + m + ld_block - 1) / ld_block - gb0;
#pragma omp parallel
  {
    uint32_t *u = (uint32_t *)malloc((size_t)2 * (n > 0 ? n : 1) * sizeof(uint32_t));
#pragma omp for schedule(dynamic, 1)
    for (long long b = 0; b < nblk; b++) {
      long long g0 = (gb0 + b) * ld_block, g1 = g0 + ld_block;
      if (g1 > col_offset + m) g1 = col_offset + m;
      for (long long gj = g0; gj < g1; gj++) {
        uint64_t kj = orc_mix64(seed ^ orc_mix64((uint64_t)gj));
        double maf = 0.02 + 0.48 * ((double)(kj >> 11) * (1.0 / 9007199254740992.0));
        uint32_t thr = (uint32_t)(maf * 16777216.0);
        int first = gj == g0;
        uint8_t *col = gj >= col_offset ? out + (size_t)(gj - col_offset) * n_byte : NULL;
        if (col) memset(col, 0, n_byte);
        for (int i = 0; i < n; i++) {
          uint64_t hs = orc_mix64(kj + (uint64_t)i * 0xD1342543DE82EF95ull);
          uint64_t h2 = orc_mix64(hs ^ 0xA5A5A5A5A5A5A5A5ull);
          int c0 = !first && (uint32_t)(h2 & 0xFFFFu) < rho_thr;
          int c1 = !first && (uint32_t)((h2 >> 16) & 0xFFFFu) < rho_thr;
          if (!c0) u[2 * i] = (uint32_t)(hs & 0xFFFFFFu);
          if (!c1) u[2 * i + 1] = (uint32_t)((hs >> 24) & 0xFFFFFFu);
          uint32_t g = (u[2 * i] < thr) + (u[2 * i + 1] < thr);
          if ((uint32_t)((hs >> 48) & 0xFFFFu) < na_thr) g = 3;
          if (col) col[i >> 2] |= (uint8_t)(bedcode[g] << (2 * (i & 3)));
        }
      }
    }
    free(u);
  }
}

int orc_max_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
