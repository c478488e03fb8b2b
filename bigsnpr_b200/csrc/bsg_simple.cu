// bsg_simple.cu -- generic accessor-style kernels over copy A.
//
// These follow the accessor semantics of the reference literally (bedAcc / bedAccScaled,
// src/bed-acc.h:52-115): arbitrary row / column index multisets, per-column 4-entry table
// {(0-c)/s, (1-c)/s, (2-c)/s, 0}, missing -> 0.  They serve (a) index patterns and inputs the
// tensor-pipe path does not take (non-finite vectors, zero scales), (b) the dense decodes and the
// count tables, (c) an on-device cross-check of the fast path in the GPU tests.
#include "bsg_internal.cuh"

namespace bsg {

__device__ __forceinline__ int code_at(const uint8_t *__restrict__ A, int64_t strideA, int row, int col) {
  return (A[(int64_t)col * strideA + (row >> 2)] >> (2 * (row & 3))) & 3;
}

// out[j] = sum_i T_j[code(row_i, col_j)] * x[i]     (src/bed-prod-vec.cpp:59-97)
// one warp per output column, lanes stride over the row list, fp64 warp reduction.
__global__ void k_cprodvec_simple(const uint8_t *__restrict__ A, int64_t strideA, const int *__restrict__ rows,
                                  int nr, const int *__restrict__ cols, int nc, const double *__restrict__ center,
                                  const double *__restrict__ scale, const double *__restrict__ x,
                                  double *__restrict__ out) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  int nw = (gridDim.x * blockDim.x) >> 5;
  for (int j = warp; j < nc; j += nw) {
    int col = cols ? cols[j] : j;
    double c = center ? center[j] : 0.0, s = scale ? scale[j] : 1.0;
    double t0 = (0.0 - c) / s, t1 = (1.0 - c) / s, t2 = (2.0 - c) / s;
    const uint8_t *line = A + (int64_t)col * strideA;
    double acc = 0;
    for (int i = lane; i < nr; i += 32) {
      int r = rows ? rows[i] : i;
      int g = (line[r >> 2] >> (2 * (r & 3))) & 3;
      double v = g == 0 ? t0 : (g == 1 ? t1 : (g == 2 ? t2 : 0.0));
      acc += v * x[i];
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) out[j] = acc;
  }
}

// out[i] = sum_j T_j[code(row_i, col_j)] * x[j]     (src/bed-prod-vec.cpp:15-54)
// thread per output row, blockIdx.y splits the column list; per-split partials are written to
// part[split][nr] and summed in split order by k_sum_splits (deterministic).
__global__ void k_prodvec_simple(const uint8_t *__restrict__ A, int64_t strideA, const int *__restrict__ rows,
                                 int nr, const int *__restrict__ cols, int nc, const double *__restrict__ center,
                                 const double *__restrict__ scale, const double *__restrict__ x,
                                 double *__restrict__ part, int cols_per_split, int square) {
  __shared__ double tab[128][4];
  __shared__ int scol[128];
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int r = (i < nr) ? (rows ? rows[i] : i) : 0;
  int j0 = blockIdx.y * cols_per_split;
  int j1 = min(nc, j0 + cols_per_split);
  double acc = 0;
  for (int jb = j0; jb < j1; jb += 128) {
    int nb = min(128, j1 - jb);
    __syncthreads();
    if (threadIdx.x < nb) {
      int j = jb + threadIdx.x;
      double c = center ? center[j] : 0.0, s = scale ? scale[j] : 1.0;
      const double t0 = (0.0 - c) / s, t1 = (1.0 - c) / s, t2 = (2.0 - c) / s;
      if (square) {  // row sums of squares (src/bed-fun.cpp:126)
        tab[threadIdx.x][0] = t0 * t0;
        tab[threadIdx.x][1] = t1 * t1;
        tab[threadIdx.x][2] = t2 * t2;
        tab[threadIdx.x][3] = 0.0;
      } else {
        const double xv = x[j];
        tab[threadIdx.x][0] = xv * t0;
        tab[threadIdx.x][1] = xv * t1;
        tab[threadIdx.x][2] = xv * t2;
        tab[threadIdx.x][3] = xv * 0.0;
      }
      scol[threadIdx.x] = cols ? cols[j] : j;
    }
    __syncthreads();
    if (i < nr) {
      for (int k = 0; k < nb; k++) {
        int g = (A[(int64_t)scol[k] * strideA + (r >> 2)] >> (2 * (r & 3))) & 3;
        acc += tab[k][g];
      }
    }
  }
  if (i < nr) part[(int64_t)blockIdx.y * nr + i] = acc;
}

__global__ void k_sum_splits(const double *__restrict__ part, int nr, int nsplit, double *__restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nr) return;
  double s = 0;
  for (int k = 0; k < nsplit; k++) s += part[(int64_t)k * nr + i];
  out[i] = s;
}

// 4 x nc counts (src/bed-fun.cpp:51-69): warp per column over the row multiset.
__global__ void k_counts_cols(const uint8_t *__restrict__ A, int64_t strideA, const int *__restrict__ rows, int nr,
                              const int *__restrict__ cols, int nc, int32_t *__restrict__ out) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  int nw = (gridDim.x * blockDim.x) >> 5;
  for (int j = warp; j < nc; j += nw) {
    int col = cols ? cols[j] : j;
    const uint8_t *line = A + (int64_t)col * strideA;
    int c1 = 0, c2 = 0, c3 = 0;
    for (int i = lane; i < nr; i += 32) {
      int r = rows ? rows[i] : i;
      int g = (line[r >> 2] >> (2 * (r & 3))) & 3;
      c1 += g == 1;
      c2 += g == 2;
      c3 += g == 3;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      c1 += __shfl_xor_sync(0xffffffffu, c1, o);
      c2 += __shfl_xor_sync(0xffffffffu, c2, o);
      c3 += __shfl_xor_sync(0xffffffffu, c3, o);
    }
    if (lane == 0) {
      out[4 * (int64_t)j + 0] = nr - c1 - c2 - c3;
      out[4 * (int64_t)j + 1] = c1;
      out[4 * (int64_t)j + 2] = c2;
      out[4 * (int64_t)j + 3] = c3;
    }
  }
}

// 4 x nr counts (src/bed-fun.cpp:72-98): thread per row over the column multiset (coalesced along rows).
__global__ void k_counts_rows(const uint8_t *__restrict__ A, int64_t strideA, const int *__restrict__ rows, int nr,
                              const int *__restrict__ cols, int nc, int32_t *__restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nr) return;
  int r = rows ? rows[i] : i;
  int c1 = 0, c2 = 0, c3 = 0;
  for (int j = 0; j < nc; j++) {
    int col = cols ? cols[j] : j;
    int g = (A[(int64_t)col * strideA + (r >> 2)] >> (2 * (r & 3))) & 3;
    c1 += g == 1;
    c2 += g == 2;
    c3 += g == 3;
  }
  out[4 * (int64_t)i + 0] = nc - c1 - c2 - c3;
  out[4 * (int64_t)i + 1] = c1;
  out[4 * (int64_t)i + 2] = c2;
  out[4 * (int64_t)i + 3] = c3;
}

__global__ void k_read_dense(const uint8_t *__restrict__ A, int64_t strideA, const int *__restrict__ rows, int nr,
                             const int *__restrict__ cols, int nc, int na_val, int *__restrict__ out) {
  int64_t total = (int64_t)nr * nc;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int j = (int)(t / nr), i = (int)(t - (int64_t)j * nr);
    int g = code_at(A, strideA, rows ? rows[i] : i, cols ? cols[j] : j);
    out[t] = g == 3 ? na_val : g;
  }
}

__global__ void k_read_dense_scaled(const uint8_t *__restrict__ A, int64_t strideA, const int *__restrict__ rows,
                                    int nr, const int *__restrict__ cols, int nc, const double *__restrict__ center,
                                    const double *__restrict__ scale, double *__restrict__ out) {
  int64_t total = (int64_t)nr * nc;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int j = (int)(t / nr), i = (int)(t - (int64_t)j * nr);
    int g = code_at(A, strideA, rows ? rows[i] : i, cols ? cols[j] : j);
    double c = center ? center[j] : 0.0, s = scale ? scale[j] : 1.0;
    out[t] = g == 3 ? 0.0 : ((double)g - c) / s;
  }
}

// FBM.code256 bytes of the sub-matrix (readbina2, src/read-plink.cpp:61-80): out[i + nr j] = code 0 / 1 / 2 / 3 (NA)
__global__ void k_read_bytes(const uint8_t *__restrict__ A, int64_t strideA, const int *__restrict__ rows, int nr,
                             const int *__restrict__ cols, int nc, uint8_t *__restrict__ out) {
  int64_t total = (int64_t)nr * nc;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int j = (int)(t / nr), i = (int)(t - (int64_t)j * nr);
    out[t] = (uint8_t)code_at(A, strideA, rows ? rows[i] : i, cols ? cols[j] : j);
  }
}

// .bed bytes of the sub-matrix as writebina lays them out (src/write-plink.cpp:29-47 with tab = getInverseCode(),
// R/utils.R:35-45): genotype 0 -> 11, 1 -> 10, 2 -> 00, NA -> 01; the unused slots of the last byte of a column hold
// genotype 0 (code 11), like the reference's `ind` built from zeros.  One thread per output byte.
__global__ void k_pack_bed(const uint8_t *__restrict__ A, int64_t strideA, const int *__restrict__ rows, int nr,
                           const int *__restrict__ cols, int nc, int nbytes, uint8_t *__restrict__ out) {
  int64_t total = (int64_t)nbytes * nc;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int j = (int)(t / nbytes), k = (int)(t - (int64_t)j * nbytes);
    const int col = cols ? cols[j] : j;
    uint32_t byte = 0;
#pragma unroll
    for (int c = 0; c < 4; c++) {
      const int i = 4 * k + c;
      const int g = i < nr ? code_at(A, strideA, rows ? rows[i] : i, col) : 0;
      const uint32_t bed2 = g == 0 ? 3u : (g == 1 ? 2u : (g == 2 ? 0u : 1u));
      byte |= bed2 << (2 * c);
    }
    out[t] = (uint8_t)byte;
  }
}

static int grid1(int64_t work, int block, int cap = 132 * 16) {
  int64_t g = (work + block - 1) / block;
  if (g < 1) g = 1;
  if (g > cap) g = cap;
  return (int)g;
}

int simple_cprodvec(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, const double *d_center,
                    const double *d_scale, const double *d_x, double *d_out, cudaStream_t s) {
  k_cprodvec_simple<<<grid1((int64_t)nc * 32, 256), 256, 0, s>>>(h->A, h->strideA, d_row, nr, d_col, nc, d_center,
                                                                d_scale, d_x, d_out);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

static int simple_prodvec_any(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, const double *d_center,
                              const double *d_scale, const double *d_x, double *d_out, cudaStream_t s, int square) {
  int gx = (nr + 255) / 256;
  int nsplit = (132 * 8 + gx - 1) / gx;
  int max_split = (nc + 127) / 128;
  if (nsplit > max_split) nsplit = max_split;
  if (nsplit < 1) nsplit = 1;
  int cps = ((nc + nsplit - 1) / nsplit + 127) / 128 * 128;
  if (cps < 128) cps = 128;
  nsplit = (nc + cps - 1) / cps;
  if (nsplit < 1) nsplit = 1;
  BSG_TRY(h->w_part.ensure((size_t)nsplit * (nr > 0 ? nr : 1) * sizeof(double)));
  if (nr == 0) return BSG_OK;
  dim3 grid(gx, nsplit);
  k_prodvec_simple<<<grid, 256, 0, s>>>(h->A, h->strideA, d_row, nr, d_col, nc, d_center, d_scale, d_x,
                                        h->w_part.as<double>(), cps, square);
  k_sum_splits<<<gx, 256, 0, s>>>(h->w_part.as<double>(), nr, nsplit, d_out);
  count_launch(2);
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

int simple_prodvec(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, const double *d_center,
                   const double *d_scale, const double *d_x, double *d_out, cudaStream_t s) {
  return simple_prodvec_any(h, d_row, nr, d_col, nc, d_center, d_scale, d_x, d_out, s, 0);
}

// rowSumsSq[i] = sum_j X~[i, j]^2  (src/bed-fun.cpp:123-127) with the same accessor kernel
int simple_rowsumssq(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, const double *d_center,
                     const double *d_scale, double *d_out, cudaStream_t s) {
  return simple_prodvec_any(h, d_row, nr, d_col, nc, d_center, d_scale, nullptr, d_out, s, 1);
}

int counts_cols(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, int32_t *d_out4, cudaStream_t s) {
  if (nc == 0) return BSG_OK;
  k_counts_cols<<<grid1((int64_t)nc * 32, 256), 256, 0, s>>>(h->A, h->strideA, d_row, nr, d_col, nc, d_out4);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

int counts_rows(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, int32_t *d_out4, cudaStream_t s) {
  if (nr == 0) return BSG_OK;
  k_counts_rows<<<(nr + 127) / 128, 128, 0, s>>>(h->A, h->strideA, d_row, nr, d_col, nc, d_out4);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

int read_dense(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, int na_val, int *d_out, cudaStream_t s) {
  if ((int64_t)nr * nc == 0) return BSG_OK;
  k_read_dense<<<grid1((int64_t)nr * nc, 256), 256, 0, s>>>(h->A, h->strideA, d_row, nr, d_col, nc, na_val, d_out);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

int read_bytes(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, uint8_t *d_out, cudaStream_t s) {
  if ((int64_t)nr * nc == 0) return BSG_OK;
  k_read_bytes<<<grid1((int64_t)nr * nc, 256), 256, 0, s>>>(h->A, h->strideA, d_row, nr, d_col, nc, d_out);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

int pack_bed(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, uint8_t *d_out, cudaStream_t s) {
  const int nbytes = (nr + 3) / 4;
  if ((int64_t)nbytes * nc == 0) return BSG_OK;
  k_pack_bed<<<grid1((int64_t)nbytes * nc, 256), 256, 0, s>>>(h->A, h->strideA, d_row, nr, d_col, nc, nbytes, d_out);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

int read_dense_scaled(bsg_bed *h, const int *d_row, int nr, const int *d_col, int nc, const double *d_center,
                      const double *d_scale, double *d_out, cudaStream_t s) {
  if ((int64_t)nr * nc == 0) return BSG_OK;
  k_read_dense_scaled<<<grid1((int64_t)nr * nc, 256), 256, 0, s>>>(h->A, h->strideA, d_row, nr, d_col, nc, d_center,
                                                                   d_scale, d_out);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

}  // namespace bsg
