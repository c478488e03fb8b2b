// bsg_comm.cu -- the multi-GPU side of the path (SURVEY.md section 8e): SNP columns sharded over the GPUs of one node,
// X.y partial n-vectors summed over the shards, Gram partials summed over the shards.  The reference has no multi-device
// code; the exchange steps are designed for NVLink 5 / NVSwitch peer memory:
//
//   * every rank owns a "region" of device memory that all its peers map (cudaDeviceEnablePeerAccess inside one process,
//     CUDA IPC handles between the processes of a torchrun job);
//   * X.y + all-reduce is ONE kernel (k_ar_oneshot<true>): the fp64 epilogue of the integer slice sums writes each value
//     straight into slot [rank] of every peer's region (remote stores over NVLink), a release flag per peer publishes the
//     block of stores, and once the flags of all peers have arrived each rank adds the `world` slots in rank order.
//     The sum order is fixed, so every rank holds the SAME bits (the Lanczos recurrences of the ranks cannot drift apart),
//     and no host thread, NCCL launch or stream synchronisation sits between the product and its reduction;
//   * large buffers (the n x n Gram partials) use the bandwidth-optimal two-shot form: reduce-scatter by peer reads of the
//     rank's own slice, then all-gather by peer reads of the reduced slices, separated by flag barriers.
//
// bsg_group_* drives several GPUs from ONE host process (the shape an R session has); bsg_comm_* + the *_comm entry points
// serve one-process-per-GPU launches (torchrun), where the only host-side exchange is the 64-byte IPC handle at set-up.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <thread>
#include <vector>

#include "bsg_internal.cuh"
#include "bsg_pmv_shared.cuh"

namespace bsg {

constexpr size_t REGION_FLAGS = 0, REGION_BAR = 1024, REGION_COUNTER = 2048, REGION_SLOTS = 4096;
constexpr unsigned long long WAIT_TIMEOUT_NS = 20ull * 1000ull * 1000ull * 1000ull;

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ double ld_relaxed_sys_f64(const double *p) {  // written by a peer: must not come from a stale L1 line
  double v;
  asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// spin until flag[q] >= epoch for every q < world (one thread); a peer that never arrives trips the timeout instead of
// hanging the device
__device__ __forceinline__ void wait_flags(const unsigned long long *flags, int world, unsigned long long epoch, int *err) {
  const unsigned long long t0 = globaltimer_ns();
  for (int q = 0; q < world; q++) {
    while (ld_acquire_sys(flags + q) < epoch) {
      if (globaltimer_ns() - t0 > WAIT_TIMEOUT_NS) {
        *err = 1;
        return;
      }
      __nanosleep(64);
    }
  }
}

struct ArArgs {
  double *push[BSG_MAX_PEERS];              // slot [parity][my rank] inside peer q's region
  unsigned long long *flag[BSG_MAX_PEERS];  // &flags[my rank] inside peer q's region
  const double *my_slots;                   // slot [parity][0] of my region (slot q at + q * slot_elems)
  const unsigned long long *my_flags;
  unsigned int *counter;
  unsigned long long epoch;
  size_t slot_elems;
  int world, rank;
  int *err;
};

// One-shot all-reduce, optionally fused with the X.y epilogue (FUSED: the value of element l is computed from the
// integer slice sums instead of read from `src`).  The grid is at most one wave, so every block is resident while it
// waits for the peers.
template <bool FUSED>
__global__ void __launch_bounds__(256) k_ar_oneshot(const ArArgs a, int64_t len, const double *src,
                                                    const long long *__restrict__ part, const pmv::Scal *sc, int has_scaling,
                                                    int use_na, double *out) {  // src may alias out (in-place form)
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t l = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; l < len; l += stride) {
    const double v = FUSED ? pmv::finish_prod_value(part, l, sc, has_scaling, use_na) : src[l];
#pragma unroll 1
    for (int q = 0; q < a.world; q++) a.push[q][l] = v;  // remote stores (own slot included), coalesced per warp
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(a.counter, 1u);
    if (prev == gridDim.x - 1) {  // last block of this rank: every store of the rank is fenced -> publish
      *a.counter = 0;
      __threadfence_system();
      for (int q = 0; q < a.world; q++) st_release_sys(a.flag[q], a.epoch);
    }
    wait_flags(a.my_flags, a.world, a.epoch, a.err);
  }
  __syncthreads();
  for (int64_t l = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; l < len; l += stride) {
    double acc = 0;
#pragma unroll 1
    for (int q = 0; q < a.world; q++) acc += ld_relaxed_sys_f64(a.my_slots + (size_t)q * a.slot_elems + l);
    out[l] = acc;  // rank order: identical bits on every rank
  }
}

// flag barrier over the group (one block): everything enqueued before it on the streams of all ranks has completed
// when the kernels enqueued after it start
struct BarArgs {
  unsigned long long *flag[BSG_MAX_PEERS];
  const unsigned long long *my_flags;
  unsigned long long epoch;
  int world;
  int *err;
};
__global__ void k_group_barrier(const BarArgs a) {
  __threadfence_system();
  if (threadIdx.x < a.world) st_release_sys(a.flag[threadIdx.x], a.epoch);
  if (threadIdx.x == 0) wait_flags(a.my_flags, a.world, a.epoch, a.err);
}

struct BufArgs {
  double *buf[BSG_MAX_PEERS];
  int world, rank;
};
// reduce-scatter: this rank sums its own slice over all ranks' buffers (peer reads), result in its own buffer
__global__ void k_ar2_reduce(const BufArgs a, int64_t count) {
  const int64_t chunk = (count + a.world - 1) / a.world;
  const int64_t i0 = (int64_t)a.rank * chunk, i1 = min(count, i0 + chunk);
  for (int64_t i = i0 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < i1; i += (int64_t)gridDim.x * blockDim.x) {
    double acc = 0;
#pragma unroll 1
    for (int q = 0; q < a.world; q++) acc += a.buf[q][i];
    a.buf[a.rank][i] = acc;
  }
}
// all-gather: fetch the reduced slices of the other ranks
__global__ void k_ar2_gather(const BufArgs a, int64_t count) {
  const int64_t chunk = (count + a.world - 1) / a.world;
  for (int q = 0; q < a.world; q++) {
    if (q == a.rank) continue;
    const int64_t i0 = (int64_t)q * chunk, i1 = min(count, i0 + chunk);
    for (int64_t i = i0 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < i1; i += (int64_t)gridDim.x * blockDim.x)
      a.buf[a.rank][i] = ld_relaxed_sys_f64(a.buf[q] + i);
  }
}

static size_t region_size(int world, size_t slot_elems) { return REGION_SLOTS + (size_t)2 * world * slot_elems * sizeof(double); }

static int comm_alloc(int rank, int world, int device, size_t slot_elems, bsg_comm **out) {
  if (world < 1 || world > BSG_MAX_PEERS || rank < 0 || rank >= world) return fail(BSG_ERR_ARG, "rank / world out of range (max %d ranks).", BSG_MAX_PEERS);
  BSG_CUDA(cudaSetDevice(device));
  bsg_comm *c = new bsg_comm();
  c->rank = rank;
  c->world = world;
  c->device = device;
  c->slot_elems = (slot_elems + 31) / 32 * 32;
  c->region_bytes = region_size(world, c->slot_elems);
  cudaError_t e = cudaMalloc((void **)&c->region, c->region_bytes);
  if (e == cudaSuccess) e = cudaMemset(c->region, 0, REGION_SLOTS);
  if (e == cudaSuccess) e = cudaMalloc((void **)&c->d_err, sizeof(int));
  if (e == cudaSuccess) e = cudaMemset(c->d_err, 0, sizeof(int));
  if (e != cudaSuccess) {
    cudaFree(c->region);
    delete c;
    return cuda_fail(e, "communicator region");
  }
  c->peer[rank] = c->region;
  *out = c;
  return BSG_OK;
}

static ArArgs ar_args(bsg_comm *c) {
  ArArgs a;
  const unsigned long long ep = ++c->epoch;
  const size_t par = (size_t)(ep & 1ull) * c->world * c->slot_elems;
  for (int q = 0; q < c->world; q++) {
    a.push[q] = reinterpret_cast<double *>(c->peer[q] + REGION_SLOTS) + par + (size_t)c->rank * c->slot_elems;
    a.flag[q] = reinterpret_cast<unsigned long long *>(c->peer[q] + REGION_FLAGS) + c->rank;
  }
  a.my_slots = reinterpret_cast<const double *>(c->region + REGION_SLOTS) + par;
  a.my_flags = reinterpret_cast<const unsigned long long *>(c->region + REGION_FLAGS);
  a.counter = reinterpret_cast<unsigned int *>(c->region + REGION_COUNTER);
  a.epoch = ep;
  a.slot_elems = c->slot_elems;
  a.world = c->world;
  a.rank = c->rank;
  a.err = c->d_err;
  return a;
}

static int ar_grid(int64_t len, int device) {
  int nsm = 132;
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device);
  return (int)std::max<int64_t>(1, std::min<int64_t>((len + 255) / 256, 2 * nsm));  // <= one resident wave
}

int comm_finish_prod_allreduce(bsg_comm *c, const long long *part, int nlines, const pmv::Scal *sc, int has_scaling,
                               int use_na, double *out_dev, cudaStream_t s) {
  if (!c->connected) return fail(BSG_ERR_ARG, "communicator is not connected.");
  if ((size_t)nlines > c->slot_elems) return fail(BSG_ERR_ARG, "vector longer than the communicator's slots (%d > %zu).", nlines, c->slot_elems);
  if (nlines <= 0) return BSG_OK;
  const ArArgs a = ar_args(c);
  k_ar_oneshot<true><<<ar_grid(nlines, c->device), 256, 0, s>>>(a, nlines, nullptr, part, sc, has_scaling, use_na, out_dev);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

int comm_allreduce_oneshot(bsg_comm *c, double *buf_dev, int64_t count, cudaStream_t s) {
  if (!c->connected) return fail(BSG_ERR_ARG, "communicator is not connected.");
  for (int64_t off = 0; off < count; off += (int64_t)c->slot_elems) {  // longer vectors go through in slot-sized pieces
    const int64_t len = std::min<int64_t>(c->slot_elems, count - off);
    const ArArgs a = ar_args(c);
    k_ar_oneshot<false><<<ar_grid(len, c->device), 256, 0, s>>>(a, len, buf_dev + off, nullptr, nullptr, 0, 0, buf_dev + off);
    count_launch();
  }
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

static int comm_barrier(bsg_comm *c, cudaStream_t s) {
  BarArgs b;
  b.epoch = ++c->bar_epoch;
  for (int q = 0; q < c->world; q++) b.flag[q] = reinterpret_cast<unsigned long long *>(c->peer[q] + REGION_BAR) + c->rank;
  b.my_flags = reinterpret_cast<const unsigned long long *>(c->region + REGION_BAR);
  b.world = c->world;
  b.err = c->d_err;
  k_group_barrier<<<1, 32, 0, s>>>(b);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

// in-place sum of `count` doubles over the ranks; bufs[q] = rank q's buffer as addressable from this device
static int comm_allreduce_twoshot(bsg_comm *c, double *const *bufs, int64_t count, cudaStream_t s) {
  BufArgs a;
  a.world = c->world;
  a.rank = c->rank;
  for (int q = 0; q < c->world; q++) a.buf[q] = bufs[q];
  const int grid = 4 * 132;
  BSG_TRY(comm_barrier(c, s));  // every partial is complete
  k_ar2_reduce<<<grid, 256, 0, s>>>(a, count);
  BSG_TRY(comm_barrier(c, s));  // every slice is reduced
  k_ar2_gather<<<grid, 256, 0, s>>>(a, count);
  count_launch(2);
  BSG_TRY(comm_barrier(c, s));  // nobody still reads a buffer its owner may now reuse
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

static int comm_check(bsg_comm *c) {
  int err = 0;
  BSG_CUDA(cudaMemcpy(&err, c->d_err, sizeof(int), cudaMemcpyDeviceToHost));
  if (err) return fail(BSG_ERR_CUDA, "a peer GPU did not reach the collective within %d s (rank %d of %d).",
                       (int)(WAIT_TIMEOUT_NS / 1000000000ull), c->rank, c->world);
  return BSG_OK;
}

}  // namespace bsg

using namespace bsg;

struct bsg_group {
  int ndev = 0, n = 0, m = 0;
  std::vector<int> devices, col0;  // col0[g] = first global column (0-based) of shard g; col0[ndev] = m
  std::vector<bsg_bed *> shard;
  std::vector<bsg_comm *> comm;
  // cached accessor state of the last (ind_row, ind_col): per-shard views + where each selected column went
  std::vector<int> cv_row, cv_col;
  bool cv_valid = false, cv_scaled = false;
  int cv_nr = 0, cv_nc = 0;
  std::vector<bsg_view *> view;
  std::vector<std::vector<int>> loc, pos;  // per shard: local 1-based column / position in the caller's ind_col
  std::vector<double *> d_x, d_out;        // per shard device vectors (grow-only)
  std::vector<size_t> cap_x, cap_out;
};

static void shard_range(int m, int world, int rank, int *b, int *e) {  // same rule as dist.shard_bounds
  const int base = m / world, rem = m % world;
  *b = rank * base + std::min(rank, rem);
  *e = *b + base + (rank < rem ? 1 : 0);
}

static int group_enable_peers(const std::vector<int> &devices) {
  for (int a : devices)
    for (int b : devices) {
      if (a == b) continue;
      int can = 0;
      BSG_CUDA(cudaDeviceCanAccessPeer(&can, a, b));
      if (!can) return fail(BSG_ERR_CUDA, "GPU %d cannot access GPU %d's memory (no NVLink / P2P path).", a, b);
      BSG_CUDA(cudaSetDevice(a));
      cudaError_t e = cudaDeviceEnablePeerAccess(b, 0);
      if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
      else if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceEnablePeerAccess");
    }
  return BSG_OK;
}

template <class OpenFn>
static int group_open_common(int n, int m, const int *devices, int ndev, bsg_group **out, OpenFn open_shard) {
  if (!out || !devices) return fail(BSG_ERR_ARG, "null argument");
  *out = nullptr;
  if (ndev < 1 || ndev > BSG_MAX_PEERS) return fail(BSG_ERR_ARG, "1..%d devices.", BSG_MAX_PEERS);
  if (m < ndev) return fail(BSG_ERR_ARG, "fewer columns than devices.");
  bsg_group *g = new bsg_group();
  g->ndev = ndev;
  g->n = n;
  g->m = m;
  g->devices.assign(devices, devices + ndev);
  g->col0.resize(ndev + 1);
  g->shard.assign(ndev, nullptr);
  g->comm.assign(ndev, nullptr);
  g->view.assign(ndev, nullptr);
  g->loc.resize(ndev);
  g->pos.resize(ndev);
  g->d_x.assign(ndev, nullptr);
  g->d_out.assign(ndev, nullptr);
  g->cap_x.assign(ndev, 0);
  g->cap_out.assign(ndev, 0);
  int rc = ndev > 1 ? group_enable_peers(g->devices) : BSG_OK;
  std::vector<int> rcs(ndev, 0);
  std::vector<std::string> errs(ndev);
  if (!rc) {
    // staging is per device and synchronous inside: one host thread per shard so the devices fill in parallel
    std::vector<std::thread> th;
    for (int i = 0; i < ndev; i++) {
      int b, e;
      shard_range(m, ndev, i, &b, &e);
      g->col0[i] = b;
      th.emplace_back([&, i, b, e] {
        rcs[i] = open_shard(i, b, e, &g->shard[i]);
        if (rcs[i]) errs[i] = g_err;
      });
    }
    g->col0[ndev] = m;
    for (auto &t : th) t.join();
    for (int i = 0; i < ndev && !rc; i++)
      if (rcs[i]) rc = fail(rcs[i], "%s", errs[i].c_str());
  }
  for (int i = 0; i < ndev && !rc; i++) rc = comm_alloc(i, ndev, g->devices[i], (size_t)n, &g->comm[i]);
  if (!rc)
    for (int i = 0; i < ndev; i++) {
      for (int q = 0; q < ndev; q++) g->comm[i]->peer[q] = g->comm[q]->region;  // one address space: peers are plain pointers
      g->comm[i]->connected = true;
    }
  if (rc) {
    std::string keep = g_err;
    bsg_group_close(g);
    g_err = keep;
    return rc;
  }
  *out = g;
  return BSG_OK;
}

static void group_drop_views(bsg_group *g) {
  for (auto &v : g->view) {
    if (v) bsg_view_destroy(v);
    v = nullptr;
  }
  g->cv_valid = false;
}

// (ind_row, ind_col) -> per-shard views.  ind_col is a GLOBAL 1-based multiset in any order; every entry goes to the shard
// that owns the column, in the caller's order (SURVEY.md section 8e "staging": bucketed by owner per call).
static int group_views(bsg_group *g, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                       const double *scale) {
  if (!ind_row) nr = g->n;
  if (!ind_col) nc = g->m;
  if (nr < 0 || nc < 0) return fail(BSG_ERR_ARG, "negative length");
  if ((center == nullptr) != (scale == nullptr)) return fail(BSG_ERR_ARG, "center and scale must be given together");
  bool hit = g->cv_valid && g->cv_nr == nr && g->cv_nc == nc && g->cv_scaled == (center != nullptr) &&
             (ind_row ? ((int)g->cv_row.size() == nr && memcmp(g->cv_row.data(), ind_row, (size_t)nr * sizeof(int)) == 0) : g->cv_row.empty()) &&
             (ind_col ? ((int)g->cv_col.size() == nc && memcmp(g->cv_col.data(), ind_col, (size_t)nc * sizeof(int)) == 0) : g->cv_col.empty());
  if (!hit) {
    group_drop_views(g);
    for (int i = 0; i < g->ndev; i++) {
      g->loc[i].clear();
      g->pos[i].clear();
    }
    if (ind_col) {
      std::vector<int> col0;
      BSG_TRY(host_index(ind_col, nc, g->m, "column ", col0));
      for (int t = 0; t < nc; t++) {
        const int c = col0[t];
        const int own = (int)(std::upper_bound(g->col0.begin(), g->col0.begin() + g->ndev, c) - g->col0.begin()) - 1;
        g->loc[own].push_back(c - g->col0[own] + 1);
        g->pos[own].push_back(t);
      }
    } else {
      for (int i = 0; i < g->ndev; i++)
        for (int c = g->col0[i]; c < g->col0[i + 1]; c++) g->pos[i].push_back(c);  // loc stays empty = identity
    }
  }
  std::vector<double> cs, ss;
  for (int i = 0; i < g->ndev; i++) {
    const int nci = (int)g->pos[i].size();
    const double *ci = nullptr, *si = nullptr;
    if (center) {
      cs.resize(std::max(nci, 1));
      ss.resize(std::max(nci, 1));
      for (int t = 0; t < nci; t++) {
        cs[t] = center[g->pos[i][t]];
        ss[t] = scale[g->pos[i][t]];
      }
      ci = cs.data();
      si = ss.data();
    }
    if (hit && g->view[i] && (!center || g->view[i]->d_center)) {
      if (center && nci > 0) {  // same index sets: only the scaling is refreshed (the reference rebuilds its accessor per call)
        BSG_CUDA(cudaSetDevice(g->devices[i]));
        cudaStream_t s = g->shard[i]->stream;
        BSG_CUDA(cudaMemcpyAsync(g->view[i]->d_center, ci, (size_t)nci * sizeof(double), cudaMemcpyHostToDevice, s));
        BSG_CUDA(cudaMemcpyAsync(g->view[i]->d_scale, si, (size_t)nci * sizeof(double), cudaMemcpyHostToDevice, s));
        BSG_CUDA(cudaStreamSynchronize(s));  // cs / ss are reused for the next shard
      }
      continue;
    }
    if (g->view[i]) bsg_view_destroy(g->view[i]);
    g->view[i] = nullptr;
    BSG_TRY(bsg_view_create(g->shard[i], ind_row, nr, ind_col ? g->loc[i].data() : nullptr, nci, ci, si, &g->view[i]));
  }
  g->cv_row.assign(ind_row ? ind_row : nullptr, ind_row ? ind_row + nr : nullptr);
  g->cv_col.assign(ind_col ? ind_col : nullptr, ind_col ? ind_col + nc : nullptr);
  g->cv_nr = nr;
  g->cv_nc = nc;
  g->cv_scaled = center != nullptr;
  g->cv_valid = true;
  return BSG_OK;
}

static int group_vec(bsg_group *g, int i, size_t nx, size_t nout) {
  BSG_CUDA(cudaSetDevice(g->devices[i]));
  if (nx > g->cap_x[i]) {
    if (g->d_x[i]) cudaFree(g->d_x[i]);
    g->d_x[i] = nullptr;
    BSG_CUDA(cudaMalloc((void **)&g->d_x[i], std::max<size_t>(nx, 1) * sizeof(double)));
    g->cap_x[i] = nx;
  }
  if (nout > g->cap_out[i]) {
    if (g->d_out[i]) cudaFree(g->d_out[i]);
    g->d_out[i] = nullptr;
    BSG_CUDA(cudaMalloc((void **)&g->d_out[i], std::max<size_t>(nout, 1) * sizeof(double)));
    g->cap_out[i] = nout;
  }
  return BSG_OK;
}

extern "C" {

// ---- communicators for one-process-per-GPU launches ---------------------------------------------------------------
int bsg_comm_create(int rank, int world, int device, int64_t max_elems, bsg_comm **out, unsigned char *handle64) {
  if (!out || !handle64 || max_elems < 1) return fail(BSG_ERR_ARG, "null argument");
  *out = nullptr;
  bsg_comm *c = nullptr;
  BSG_TRY(comm_alloc(rank, world, device, (size_t)max_elems, &c));
  cudaIpcMemHandle_t hd;
  static_assert(sizeof(hd) == 64, "IPC handle is 64 bytes");
  cudaError_t e = cudaIpcGetMemHandle(&hd, c->region);
  if (e != cudaSuccess) {
    bsg_comm_destroy(c);
    return cuda_fail(e, "cudaIpcGetMemHandle");
  }
  memcpy(handle64, &hd, 64);
  if (world == 1) c->connected = true;
  *out = c;
  return BSG_OK;
}

int bsg_comm_connect(bsg_comm *c, const unsigned char *handles /* world x 64 bytes, rank order */) {
  if (!c || !handles) return fail(BSG_ERR_ARG, "null argument");
  BSG_CUDA(cudaSetDevice(c->device));
  for (int q = 0; q < c->world; q++) {
    if (q == c->rank || c->peer[q]) continue;
    cudaIpcMemHandle_t hd;
    memcpy(&hd, handles + (size_t)q * 64, 64);
    void *p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, hd, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return cuda_fail(e, "cudaIpcOpenMemHandle (peer region)");
    c->peer[q] = (uint8_t *)p;
    c->peer_ipc[q] = true;
  }
  c->connected = true;
  return BSG_OK;
}

void bsg_comm_destroy(bsg_comm *c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  for (int q = 0; q < c->world; q++)
    if (c->peer_ipc[q] && c->peer[q]) cudaIpcCloseMemHandle(c->peer[q]);
  if (c->region) cudaFree(c->region);
  if (c->d_err) cudaFree(c->d_err);
  delete c;
}

int bsg_comm_rank(const bsg_comm *c) { return c ? c->rank : -1; }
int bsg_comm_world(const bsg_comm *c) { return c ? c->world : 0; }

int bsg_comm_check(bsg_comm *c) {
  if (!c) return fail(BSG_ERR_ARG, "null argument");
  BSG_CUDA(cudaSetDevice(c->device));
  return comm_check(c);
}

int bsg_comm_allreduce_dev(bsg_comm *c, double *buf_dev, int64_t count, void *stream) {
  if (!c || !buf_dev) return fail(BSG_ERR_ARG, "null argument");
  BSG_CUDA(cudaSetDevice(c->device));
  return comm_allreduce_oneshot(c, buf_dev, count, stream ? (cudaStream_t)stream : cudaStreamLegacy);
}

int bsg_view_prodvec_allreduce_dev(bsg_view *v, bsg_comm *c, const double *x_dev, double *out_dev, void *stream) {
  if (!c) return fail(BSG_ERR_ARG, "null argument");
  return view_prodvec_comm(v, x_dev, out_dev, stream ? (cudaStream_t)stream : cudaStreamLegacy, c);
}

int bsg_randomsvd_comm(bsg_bed *h, bsg_comm *c, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                       const double *scale, int ncol_total, int k, double tol, int maxit, double *d, double *u, double *v,
                       double *center_out, double *scale_out, int *niter, int *nops) {
  if (!h || !c || !d) return fail(BSG_ERR_ARG, "null argument");
  if (!ind_col) nc = h->m;
  std::vector<SvdShard> sh(1);
  sh[0] = SvdShard{h, ind_col, nc, center, scale, c->world > 1 ? c : nullptr, v, nc, nullptr, center_out, scale_out};
  BSG_TRY(lanczos_svd(sh, ind_row, nr, ncol_total, k, tol, maxit, d, u, niter, nops, nullptr, nullptr, nullptr));
  return comm_check(c);
}

// ---- one host process, several GPUs ------------------------------------------------------------------------------------
int bsg_group_open_bed(const char *path, int n, int m, const int *devices, int ndev, int layouts, bsg_group **out) {
  if (!path) return fail(BSG_ERR_ARG, "null argument");
  return group_open_common(n, m, devices, ndev, out, [&](int i, int b, int e, bsg_bed **h) {
    return bsg_open_bed(path, n, m, b, e, devices[i], layouts, h);
  });
}

int bsg_group_open_synth(int n, int m, uint64_t seed, double na_rate, double ld_rho, int ld_block, const int *devices, int ndev,
                         int layouts, bsg_group **out) {
  return group_open_common(n, m, devices, ndev, out, [&](int i, int b, int e, bsg_bed **h) {
    if (ld_rho > 0) return bsg_open_synth_ld(n, e - b, seed, na_rate, b, ld_rho, ld_block, devices[i], layouts, h);
    return bsg_open_synth(n, e - b, seed, na_rate, b, devices[i], layouts, h);
  });
}

void bsg_group_close(bsg_group *g) {
  if (!g) return;
  group_drop_views(g);
  for (int i = 0; i < g->ndev; i++) {
    cudaSetDevice(g->devices[i]);
    cudaDeviceSynchronize();
    if (g->d_x[i]) cudaFree(g->d_x[i]);
    if (g->d_out[i]) cudaFree(g->d_out[i]);
  }
  for (auto *c : g->comm)
    if (c) bsg_comm_destroy(c);
  for (auto *h : g->shard)
    if (h) bsg_close(h);
  delete g;
}

int bsg_group_ndev(const bsg_group *g) { return g ? g->ndev : 0; }
int bsg_group_nrow(const bsg_group *g) { return g ? g->n : 0; }
int bsg_group_ncol(const bsg_group *g) { return g ? g->m : 0; }
bsg_bed *bsg_group_shard(bsg_group *g, int i) { return (g && i >= 0 && i < g->ndev) ? g->shard[i] : nullptr; }
int bsg_group_shard_begin(const bsg_group *g, int i) { return (g && i >= 0 && i <= g->ndev) ? g->col0[i] : -1; }

// bed_pMatVec4 over the shards: out[nr] = X~[ind_row, ind_col] x.  Every device multiplies its own columns and the fused
// epilogue sums the partial vectors over NVLink; the host reads the result from the first device.
int bsg_group_prodvec(bsg_group *g, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                      const double *scale, const double *x, double *out) {
  if (!g || !x || !out) return fail(BSG_ERR_ARG, "null argument");
  BSG_TRY(group_views(g, ind_row, nr, ind_col, nc, center, scale));
  nr = g->cv_nr;
  std::vector<double> xs;
  for (int i = 0; i < g->ndev; i++) {  // phase 1: inputs
    const int nci = (int)g->pos[i].size();
    BSG_TRY(group_vec(g, i, nci, nr));
    xs.resize(std::max(nci, 1));
    for (int t = 0; t < nci; t++) xs[t] = x[g->pos[i][t]];
    BSG_CUDA(cudaMemcpyAsync(g->d_x[i], xs.data(), (size_t)nci * sizeof(double), cudaMemcpyHostToDevice, g->shard[i]->stream));
    BSG_CUDA(cudaStreamSynchronize(g->shard[i]->stream));  // xs is reused
  }
  for (int i = 0; i < g->ndev; i++) {  // phase 2: products + fused reduction, nothing on the host in between
    BSG_CUDA(cudaSetDevice(g->devices[i]));
    if (nr > 0 && (int)g->pos[i].size() == 0) BSG_CUDA(cudaMemsetAsync(g->d_out[i], 0, (size_t)nr * sizeof(double), g->shard[i]->stream));
    if ((int)g->pos[i].size() == 0) {
      if (g->ndev > 1) BSG_TRY(comm_allreduce_oneshot(g->comm[i], g->d_out[i], nr, g->shard[i]->stream));
    } else {
      BSG_TRY(view_prodvec_comm(g->view[i], g->d_x[i], g->d_out[i], g->shard[i]->stream, g->ndev > 1 ? g->comm[i] : nullptr));
    }
  }
  BSG_CUDA(cudaSetDevice(g->devices[0]));
  BSG_CUDA(cudaMemcpyAsync(out, g->d_out[0], (size_t)nr * sizeof(double), cudaMemcpyDeviceToHost, g->shard[0]->stream));
  for (int i = 0; i < g->ndev; i++) {
    BSG_CUDA(cudaSetDevice(g->devices[i]));
    BSG_CUDA(cudaStreamSynchronize(g->shard[i]->stream));
  }
  for (int i = 0; i < g->ndev && g->ndev > 1; i++) BSG_TRY(bsg_comm_check(g->comm[i]));
  return BSG_OK;
}

// bed_cpMatVec4 over the shards: every device produces the entries of its own columns (no reduction), scattered into the
// caller's order.
int bsg_group_cprodvec(bsg_group *g, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                       const double *scale, const double *x, double *out) {
  if (!g || !x || !out) return fail(BSG_ERR_ARG, "null argument");
  BSG_TRY(group_views(g, ind_row, nr, ind_col, nc, center, scale));
  nr = g->cv_nr;
  for (int i = 0; i < g->ndev; i++) {
    const int nci = (int)g->pos[i].size();
    BSG_TRY(group_vec(g, i, nr, nci));
    BSG_CUDA(cudaMemcpyAsync(g->d_x[i], x, (size_t)nr * sizeof(double), cudaMemcpyHostToDevice, g->shard[i]->stream));
    if (nci > 0) BSG_TRY(bsg_view_cprodvec_dev(g->view[i], g->d_x[i], g->d_out[i], g->shard[i]->stream));
  }
  std::vector<double> part;
  for (int i = 0; i < g->ndev; i++) {
    const int nci = (int)g->pos[i].size();
    BSG_CUDA(cudaSetDevice(g->devices[i]));
    part.resize(std::max(nci, 1));
    BSG_CUDA(cudaMemcpyAsync(part.data(), g->d_out[i], (size_t)nci * sizeof(double), cudaMemcpyDeviceToHost, g->shard[i]->stream));
    BSG_CUDA(cudaStreamSynchronize(g->shard[i]->stream));
    for (int t = 0; t < nci; t++) out[g->pos[i][t]] = part[t];
  }
  return BSG_OK;
}

// bed_randomSVD over the shards (R/autoSVD.R:205-219): the sync-free Lanczos iteration of bsg_la.cu with one replica of the
// recurrence per device, the fused X.y + all-reduce as the only exchange.  v comes back in the caller's column order.
int bsg_group_randomsvd(bsg_group *g, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                        const double *scale, int k, double tol, int maxit, double *d, double *u, double *v,
                        double *center_out, double *scale_out, int *niter, int *nops) {
  if (!g || !d) return fail(BSG_ERR_ARG, "null argument");
  if (!ind_row) nr = g->n;
  if (!ind_col) nc = g->m;
  if ((center == nullptr) != (scale == nullptr)) return fail(BSG_ERR_ARG, "center and scale must be given together");
  // bucket the columns (same rule as group_views, without building product views: the driver owns its own)
  std::vector<std::vector<int>> loc(g->ndev), pos(g->ndev);
  std::vector<int> col0;
  BSG_TRY(host_index(ind_col, nc, g->m, "column ", col0));
  for (int t = 0; t < nc; t++) {
    const int c = col0[t];
    const int own = (int)(std::upper_bound(g->col0.begin(), g->col0.begin() + g->ndev, c) - g->col0.begin()) - 1;
    loc[own].push_back(c - g->col0[own] + 1);
    pos[own].push_back(t);
  }
  std::vector<std::vector<double>> cs(g->ndev), ss(g->ndev);
  std::vector<SvdShard> sh;
  for (int i = 0; i < g->ndev; i++) {
    const int nci = (int)pos[i].size();
    if (center) {
      cs[i].resize(std::max(nci, 1));
      ss[i].resize(std::max(nci, 1));
      for (int t = 0; t < nci; t++) {
        cs[i][t] = center[pos[i][t]];
        ss[i][t] = scale[pos[i][t]];
      }
    }
    sh.push_back(SvdShard{g->shard[i], loc[i].data(), nci, center ? cs[i].data() : nullptr, center ? ss[i].data() : nullptr,
                          g->ndev > 1 ? g->comm[i] : nullptr, v, nc, pos[i].data(), center_out, scale_out});
  }
  BSG_TRY(lanczos_svd(sh, ind_row, nr, nc, k, tol, maxit, d, u, niter, nops, nullptr, nullptr, nullptr));
  for (int i = 0; i < g->ndev && g->ndev > 1; i++) BSG_TRY(bsg_comm_check(g->comm[i]));
  return BSG_OK;
}

// bed_tcrossprodSelf over the shards: K = sum_g X~_g X~_g^T.  One host thread per device runs the shard's Gram product
// (wgmma tiles, bsg_la.cu) into a device buffer; the partials are summed in place by the two-shot all-reduce over
// peer memory and the first device's copy goes back to the host.
int bsg_group_tcrossprod(bsg_group *g, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                         const double *scale, double *K) {
  if (!g || !K) return fail(BSG_ERR_ARG, "null argument");
  if (!center || !scale) return fail(BSG_ERR_DIM, "Incompatibility between dimensions.");
  if (!ind_row) nr = g->n;
  if (!ind_col) nc = g->m;
  std::vector<std::vector<int>> loc(g->ndev);
  std::vector<std::vector<double>> cs(g->ndev), ss(g->ndev);
  std::vector<int> col0;
  BSG_TRY(host_index(ind_col, nc, g->m, "column ", col0));
  for (int t = 0; t < nc; t++) {
    const int c = col0[t];
    const int own = (int)(std::upper_bound(g->col0.begin(), g->col0.begin() + g->ndev, c) - g->col0.begin()) - 1;
    loc[own].push_back(c - g->col0[own] + 1);
    cs[own].push_back(center[t]);
    ss[own].push_back(scale[t]);
  }
  const size_t nn = (size_t)std::max(nr, 1) * std::max(nr, 1);
  std::vector<double *> dK(g->ndev, nullptr);
  int rc = BSG_OK;
  for (int i = 0; i < g->ndev && !rc; i++) {
    cudaSetDevice(g->devices[i]);
    cudaError_t e = cudaMalloc((void **)&dK[i], nn * sizeof(double));
    if (e != cudaSuccess) rc = cuda_fail(e, "GRM partial");
  }
  std::vector<int> rcs(g->ndev, 0);
  std::vector<std::string> errs(g->ndev);
  if (!rc) {
    std::vector<std::thread> th;
    for (int i = 0; i < g->ndev; i++)
      th.emplace_back([&, i] {
        cudaSetDevice(g->devices[i]);
        if (loc[i].empty()) {
          if (cudaMemset(dK[i], 0, nn * sizeof(double)) != cudaSuccess) rcs[i] = BSG_ERR_CUDA;
        } else {
          rcs[i] = bsg_tcrossprod_dev(g->shard[i], ind_row, nr, loc[i].data(), (int)loc[i].size(), cs[i].data(), ss[i].data(), dK[i]);
        }
        if (rcs[i]) errs[i] = g_err;
      });
    for (auto &t : th) t.join();
    for (int i = 0; i < g->ndev && !rc; i++)
      if (rcs[i]) rc = fail(rcs[i], "%s", errs[i].c_str());
  }
  if (!rc && g->ndev > 1) {
    for (int i = 0; i < g->ndev && !rc; i++) {
      cudaSetDevice(g->devices[i]);
      rc = comm_allreduce_twoshot(g->comm[i], dK.data(), (int64_t)nr * nr, g->shard[i]->stream);
    }
  }
  if (!rc) {
    cudaSetDevice(g->devices[0]);
    prefault_pages(K, (size_t)nr * nr * sizeof(double));  // while the devices reduce
    cudaError_t e = cudaMemcpyAsync(K, dK[0], (size_t)nr * nr * sizeof(double), cudaMemcpyDeviceToHost, g->shard[0]->stream);
    if (e != cudaSuccess) rc = cuda_fail(e, "GRM download");
  }
  for (int i = 0; i < g->ndev; i++) {
    cudaSetDevice(g->devices[i]);
    cudaError_t e = cudaStreamSynchronize(g->shard[i]->stream);
    if (e != cudaSuccess && !rc) rc = cuda_fail(e, "GRM all-reduce");
  }
  for (int i = 0; i < g->ndev && g->ndev > 1 && !rc; i++) rc = bsg_comm_check(g->comm[i]);
  for (int i = 0; i < g->ndev; i++) {
    cudaSetDevice(g->devices[i]);
    if (dK[i]) cudaFree(dK[i]);
  }
  return rc;
}

}  // extern "C"
