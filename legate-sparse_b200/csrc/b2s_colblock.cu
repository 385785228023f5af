// b2s_colblock.cu — column-blocked copy of a CSR matrix for SpMV with an x vector that does not
// stay resident in L2.
//
// An x that does not stay resident in L2 next to the streamed matrix turns every gather into a
// DRAM access.  So the matrix is split once into `nblocks` column blocks A = [A_0 | A_1 | ...]
// (each a self-contained CSR with global column ids, stable within a row) and y = A x is evaluated as
//     y  = A_0 x ;  y += A_1 x ; ...
// by the same TMA pipe kernel (accumulate flag), one launch per block, so that every launch
// gathers from one <= ~20 MB slice of x.  Extra traffic: one more pass over indptr and y per block.
// Measured on an H100 SXM (50 MB L2, 700 W), 10M x 10M / 50 nnz per row fp64 (x = 80 MB), ms per
// SpMV: 40 MB slices (2 blocks) 8.60, 27 MB (3) 5.64, 20 MB (4) 4.89, 13 MB (6) 4.86.
//
// Replaces nothing in the reference by itself: it is a plan-time layout of the operand of
// legate_sparse's CSR SpMV task body (src/sparse/array/csr/spmv.cu:30-163): the reference hands the
// whole row block to one cusparseSpMV call (spmv.cu:117-152) and has no operand preparation of its own.
#include "b2s_common.cuh"

#include <cstdlib>

namespace b2s {

constexpr int kMaxColBlocks = 32;   // one lane of a warp per block in the split kernels

struct ColBlockHeader {
  b2s_dtype vt;
  b2s_itype it;
  int64_t nrows, ncols, nnz;
  int nblocks;
  int64_t block_cols;
  int64_t blk_nnz[kMaxColBlocks];
  int64_t* indptr[kMaxColBlocks];   // device, [nrows+1] each, starting at 0
  void* cols[kMaxColBlocks];        // device, 256-byte aligned segments
  void* vals[kMaxColBlocks];
  b2s_spmv_plan* plan[kMaxColBlocks];
};

}  // namespace b2s

struct b2s_colblock : b2s::ColBlockHeader {};

namespace b2s {

struct SplitOut {
  void* cols[kMaxColBlocks];
  void* vals[kMaxColBlocks];
};

template <typename I>
__device__ __forceinline__ int block_of(I c, int64_t bw) {
  if constexpr (sizeof(I) == 4) return (int)((uint32_t)c / (uint32_t)bw);
  else return (int)((uint64_t)c / (uint64_t)bw);
}

// cnt[b*stride + 1 + r] = number of entries of row r in column block b   (warp per row)
template <typename I>
__global__ void __launch_bounds__(256)
colblock_count_kernel(int64_t nrows, const int64_t* __restrict__ indptr, const I* __restrict__ cols,
                      int64_t bw, int nb, int64_t stride, int64_t* __restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < nrows; r += nwarps) {
    const int64_t lo = indptr[r], hi = indptr[r + 1];
    int mine = 0;   // lane k counts block k
    for (int64_t p0 = lo; p0 < hi; p0 += 32) {
      const int64_t p = p0 + lane;
      const int b = p < hi ? block_of<I>(cols[p], bw) : -1;
      for (int k = 0; k < nb; ++k) {
        const unsigned m = __ballot_sync(0xffffffffu, b == k);
        if (lane == k) mine += __popc(m);
      }
    }
    if (lane < nb) cnt[(int64_t)lane * stride + 1 + r] = mine;
  }
}

// stable scatter of every row's entries into their block's CSR (warp per row)
template <typename V, typename I>
__global__ void __launch_bounds__(256)
colblock_scatter_kernel(int64_t nrows, const int64_t* __restrict__ indptr, const I* __restrict__ cols,
                        const V* __restrict__ vals, int64_t bw, int nb, int64_t stride,
                        const int64_t* __restrict__ blk_indptr /* [nb][stride] */, const SplitOut out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < nrows; r += nwarps) {
    const int64_t lo = indptr[r], hi = indptr[r + 1];
    int64_t off = lane < nb ? blk_indptr[(int64_t)lane * stride + r] : 0;   // lane k: next slot in block k
    for (int64_t p0 = lo; p0 < hi; p0 += 32) {
      const int64_t p = p0 + lane;
      I c = 0;
      V v{};
      int b = -1;
      if (p < hi) { c = cols[p]; v = vals[p]; b = block_of<I>(c, bw); }
      for (int k = 0; k < nb; ++k) {
        const unsigned m = __ballot_sync(0xffffffffu, b == k);
        const int64_t o = __shfl_sync(0xffffffffu, off, k);
        if (b == k) {
          const int64_t dst = o + __popc(m & ((1u << lane) - 1u));
          reinterpret_cast<I*>(out.cols[k])[dst] = c;
          reinterpret_cast<V*>(out.vals[k])[dst] = v;
        }
        if (lane == k) off += __popc(m);
      }
    }
  }
}

// sampled rows: how many span more columns than one block would hold?
template <typename I>
__global__ void colblock_sample_kernel(int64_t nrows, const int64_t* __restrict__ indptr,
                                       const I* __restrict__ cols, int64_t nsamples, int64_t span_thr,
                                       unsigned long long* __restrict__ counters) {
  int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nsamples) return;
  const int64_t r = (int64_t)((__int128)s * nrows / nsamples);
  const int64_t lo = indptr[r], hi = indptr[r + 1];
  if (hi <= lo) return;
  int64_t mn = INT64_MAX, mx = INT64_MIN;
  for (int64_t p = lo; p < hi; ++p) {
    const int64_t c = (int64_t)cols[p];
    mn = min(mn, c); mx = max(mx, c);
  }
  atomicAdd(&counters[1], 1ull);
  if (mx - mn > span_thr) atomicAdd(&counters[0], 1ull);
}

static int64_t block_bytes_target() {
  const char* e = getenv("B2S_COLBLOCK_MB");
  int64_t mb = e ? atoll(e) : 20;
  if (mb < 1) mb = 20;
  return mb << 20;
}

static int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

static int64_t plan_ws_total(int64_t nrows, int64_t nnz, int nb) {
  // sum_b ws(nnz_b) <= ws(nnz) + nb * ws(1024)   (ws is affine in ceil(nnz_b/1024)); + alignment slack
  return b2s_spmv_plan_workspace_bytes(nrows, nnz) + (int64_t)nb * (b2s_spmv_plan_workspace_bytes(nrows, 1024) + 256);
}

}  // namespace b2s

using namespace b2s;

// =================================================================== C ABI
extern "C" int b2s_csr_colblock_suggest(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols,
                                        int64_t nnz, const int64_t* indptr, const void* indices,
                                        b2s_stream_t stream, int* out_nblocks) {
  B2S_REQUIRE(out_nblocks != nullptr, "out_nblocks is null");
  *out_nblocks = 1;
  B2S_REQUIRE(nrows >= 0 && ncols >= 0 && nnz >= 0, "negative size");
  B2S_REQUIRE(it == B2S_I32 || it == B2S_I64, "bad itype");
  const int64_t vbytes = (int64_t)dtype_size(vt);
  B2S_REQUIRE(vbytes > 0, "bad dtype");
  if (const char* e = getenv("B2S_SPMV_COLBLOCK")) {   // 0/1: never, N>1: always N blocks
    int f = atoi(e);
    if (f <= 1) return B2S_OK;
    *out_nblocks = f > kMaxColBlocks ? kMaxColBlocks : f;
    if ((int64_t)*out_nblocks > ncols) *out_nblocks = 1;
    return B2S_OK;
  }
  const int64_t target = block_bytes_target();
  if (nnz < (int64_t)4 << 20 || nrows < 1024) return B2S_OK;        // launch-bound anyway
  if (ncols * vbytes <= target + target / 4) return B2S_OK;          // x already L2 resident
  int64_t nb = ceil_div(ncols * vbytes, target);
  if (nb > kMaxColBlocks) nb = kMaxColBlocks;
  if (nnz / nrows < 2 * nb) return B2S_OK;   // < 2 entries per row and block: the extra indptr/y passes dominate
  B2S_REQUIRE(indptr && indices, "null matrix arrays");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* d = nullptr;
  B2S_CUDA_TRY(cudaMallocAsync((void**)&d, 16, st));
  B2S_CUDA_TRY(cudaMemsetAsync(d, 0, 16, st));
  const int64_t nsamples = nrows < 4096 ? nrows : 4096;
  const int64_t bw = ceil_div(ncols, nb);
  if (it == B2S_I32)
    colblock_sample_kernel<int32_t><<<(unsigned)ceil_div(nsamples, 128), 128, 0, st>>>(
        nrows, indptr, (const int32_t*)indices, nsamples, bw, d);
  else
    colblock_sample_kernel<int64_t><<<(unsigned)ceil_div(nsamples, 128), 128, 0, st>>>(
        nrows, indptr, (const int64_t*)indices, nsamples, bw, d);
  B2S_CHECK_LAUNCH();
  unsigned long long h[2] = {0, 0};
  B2S_CUDA_TRY(cudaMemcpyAsync(h, d, 16, cudaMemcpyDeviceToHost, st));
  B2S_CUDA_TRY(cudaStreamSynchronize(st));
  B2S_CUDA_TRY(cudaFreeAsync(d, st));
  // rows that reach across more than one block's worth of x: their gathers have no L2 locality
  if (h[1] > 0 && h[0] * 2 >= h[1]) *out_nblocks = (int)nb;
  return B2S_OK;
}

extern "C" int64_t b2s_csr_colblock_workspace_bytes(b2s_dtype vt, b2s_itype it, int64_t nrows,
                                                    int64_t nnz, int nblocks) {
  if (nrows < 0 || nnz < 0 || nblocks < 1 || nblocks > kMaxColBlocks) return -1;
  const int64_t vb = (int64_t)dtype_size(vt), ib = it == B2S_I32 ? 4 : 8;
  if (vb <= 0) return -1;
  int64_t b = 256;
  b += (int64_t)nblocks * align_up(nrows + 1, 32) * 8;   // per-block indptr, 256-byte aligned each
  b += align_up((ceil_div(nrows > 0 ? nrows : 1, 1024) + 1) * 8, 256);
  b += align_up(nnz * ib, 256) + (int64_t)nblocks * 256;
  b += align_up(nnz * vb, 256) + (int64_t)nblocks * 256;
  b += plan_ws_total(nrows, nnz, nblocks);
  return b;
}

extern "C" int b2s_csr_colblock_create(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols,
                                       int64_t nnz, const int64_t* indptr, const void* indices,
                                       const void* data, int nblocks, void* workspace,
                                       int64_t workspace_bytes, b2s_stream_t stream,
                                       b2s_colblock** out) {
  B2S_REQUIRE(out != nullptr, "out is null");
  *out = nullptr;
  B2S_REQUIRE(nrows > 0 && ncols > 0 && nnz > 0, "column blocking needs a non-empty matrix");
  B2S_REQUIRE(nblocks >= 2 && nblocks <= kMaxColBlocks, "nblocks must be in [2,32]");
  B2S_REQUIRE((int64_t)nblocks <= ncols, "more blocks than columns");
  B2S_REQUIRE(indptr && indices && data && workspace, "null argument");
  B2S_REQUIRE(it == B2S_I32 || it == B2S_I64, "bad itype");
  const int64_t need = b2s_csr_colblock_workspace_bytes(vt, it, nrows, nnz, nblocks);
  B2S_REQUIRE(need > 0, "bad dtype");
  if (workspace_bytes < need) {
    set_error("colblock workspace too small: %lld < %lld", (long long)workspace_bytes, (long long)need);
    return B2S_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t vb = (int64_t)dtype_size(vt), ib = it == B2S_I32 ? 4 : 8;
  const int nb = nblocks;
  // block width: multiple of 32 columns so that slices of x start on 256-byte lines
  int64_t bw = align_up(ceil_div(ncols, nb), 32);
  uintptr_t base = ((uintptr_t)workspace + 255) & ~(uintptr_t)255;
  const int64_t stride = align_up(nrows + 1, 32);   // keeps every block's indptr 256-byte aligned (TMA source)
  int64_t* blk_indptr = reinterpret_cast<int64_t*>(base);   base += (int64_t)nb * stride * 8;
  int64_t* blocksum = reinterpret_cast<int64_t*>(base);     base += align_up((ceil_div(nrows, 1024) + 1) * 8, 256);
  unsigned char* cols_base = reinterpret_cast<unsigned char*>(base);  base += align_up(nnz * ib, 256) + (int64_t)nb * 256;
  unsigned char* vals_base = reinterpret_cast<unsigned char*>(base);  base += align_up(nnz * vb, 256) + (int64_t)nb * 256;
  unsigned char* plan_base = reinterpret_cast<unsigned char*>(base);
  const unsigned char* ws_end = reinterpret_cast<unsigned char*>(workspace) + workspace_bytes;

  int64_t warps = nrows;
  int64_t grid = ceil_div(warps, 8);
  if (grid > (int64_t)kNumSMs * 32) grid = (int64_t)kNumSMs * 32;
  if (it == B2S_I32)
    colblock_count_kernel<int32_t><<<(unsigned)grid, 256, 0, st>>>(nrows, indptr, (const int32_t*)indices, bw, nb, stride, blk_indptr);
  else
    colblock_count_kernel<int64_t><<<(unsigned)grid, 256, 0, st>>>(nrows, indptr, (const int64_t*)indices, bw, nb, stride, blk_indptr);
  B2S_CHECK_LAUNCH();
  auto* C = new b2s_colblock();
  C->vt = vt; C->it = it; C->nrows = nrows; C->ncols = ncols; C->nnz = nnz; C->nblocks = nb; C->block_cols = bw;
  for (int b = 0; b < kMaxColBlocks; ++b) { C->plan[b] = nullptr; C->blk_nnz[b] = 0; }
  for (int b = 0; b < nb; ++b) {
    int64_t* ip = blk_indptr + (int64_t)b * stride;
    C->indptr[b] = ip;
    int rc = scan_inclusive_i64(nrows, ip + 1, ip, blocksum, st);
    if (rc) { delete C; return rc; }
    cudaError_t e = cudaMemcpyAsync(&C->blk_nnz[b], ip + nrows, 8, cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) { delete C; set_error("memcpy failed: %s", cudaGetErrorString(e)); return B2S_ERR_CUDA; }
  }
  {
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { delete C; set_error("colblock count failed: %s", cudaGetErrorString(e)); return B2S_ERR_CUDA; }
  }
  SplitOut so{};
  int64_t tot = 0, coff = 0, voff = 0;
  for (int b = 0; b < nb; ++b) {
    C->cols[b] = cols_base + coff;  coff += align_up(C->blk_nnz[b] * ib, 256);
    C->vals[b] = vals_base + voff;  voff += align_up(C->blk_nnz[b] * vb, 256);
    so.cols[b] = C->cols[b]; so.vals[b] = C->vals[b];
    tot += C->blk_nnz[b];
  }
  if (tot != nnz) {
    delete C;
    set_error("column ids outside [0, ncols): %lld of %lld entries fell into the blocks", (long long)tot, (long long)nnz);
    return B2S_ERR_ARG;
  }
  int rc = B2S_OK;
  B2S_DISPATCH_VT(vt, V, {
    if (it == B2S_I32)
      colblock_scatter_kernel<V, int32_t><<<(unsigned)grid, 256, 0, st>>>(
          nrows, indptr, (const int32_t*)indices, (const V*)data, bw, nb, stride, blk_indptr, so);
    else
      colblock_scatter_kernel<V, int64_t><<<(unsigned)grid, 256, 0, st>>>(
          nrows, indptr, (const int64_t*)indices, (const V*)data, bw, nb, stride, blk_indptr, so);
  });
  {
    g_launch_count.fetch_add(1);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { delete C; set_error("colblock scatter failed: %s", cudaGetErrorString(e)); return B2S_ERR_CUDA; }
  }
  // one SpMV plan per block, 1024-nnz tiles: the two ping-pong consumer groups of the pipe kernel
  // measured fastest with them (against 2048-nnz tiles on C2)
  for (int b = 0; b < nb && rc == B2S_OK; ++b) {
    if (C->blk_nnz[b] == 0) continue;
    const int64_t wsb = b2s_spmv_plan_workspace_bytes(nrows, C->blk_nnz[b]);
    uintptr_t pb = ((uintptr_t)plan_base + 255) & ~(uintptr_t)255;
    if (reinterpret_cast<unsigned char*>(pb) + wsb > ws_end) { set_error("colblock workspace carve overflow"); rc = B2S_ERR_WORKSPACE; break; }
    const int64_t tile = 1024;
    rc = plan_create_impl(it, nrows, ncols, C->blk_nnz[b], C->indptr[b], C->cols[b], reinterpret_cast<void*>(pb), wsb,
                          stream, tile, &C->plan[b]);
    plan_base = reinterpret_cast<unsigned char*>(pb) + wsb;
  }
  if (rc != B2S_OK) {
    for (int b = 0; b < nb; ++b) if (C->plan[b]) b2s_spmv_plan_destroy(C->plan[b]);
    delete C;
    return rc;
  }
  *out = C;
  return B2S_OK;
}

extern "C" void b2s_csr_colblock_destroy(b2s_colblock* cb) {
  if (!cb) return;
  for (int b = 0; b < cb->nblocks; ++b) if (cb->plan[b]) b2s_spmv_plan_destroy(cb->plan[b]);
  delete cb;
}

extern "C" int b2s_csr_colblock_info(const b2s_colblock* cb, int* nblocks, int64_t* block_cols,
                                     int64_t* blk_nnz /* [nblocks] or NULL */) {
  B2S_REQUIRE(cb != nullptr, "colblock is null");
  if (nblocks) *nblocks = cb->nblocks;
  if (block_cols) *block_cols = cb->block_cols;
  if (blk_nnz) for (int b = 0; b < cb->nblocks; ++b) blk_nnz[b] = cb->blk_nnz[b];
  return B2S_OK;
}

extern "C" int b2s_spmv_colblock(const b2s_colblock* cb, const void* x, void* y, const void* w,
                                 void* dot_out, void* const* y_peers, int npeers, b2s_stream_t stream) {
  B2S_REQUIRE(cb != nullptr, "colblock is null");
  B2S_REQUIRE(x != nullptr && y != nullptr, "null vector");
  B2S_REQUIRE(dot_out == nullptr || w != nullptr, "w null");
  int first = -1, last = -1;
  for (int b = 0; b < cb->nblocks; ++b)
    if (cb->blk_nnz[b] > 0) { if (first < 0) first = b; last = b; }
  B2S_REQUIRE(first >= 0, "empty colblock");
  for (int b = first; b <= last; ++b) {
    if (cb->blk_nnz[b] == 0) continue;
    const bool fin = b == last;
    int rc = spmv_entry(cb->vt, cb->it, cb->nrows, cb->ncols, cb->blk_nnz[b], cb->indptr[b], cb->cols[b],
                        cb->vals[b], x, y, cb->plan[b], B2S_SPMV_PIPE, fin ? dot_out : nullptr,
                        fin && dot_out ? plan_dot_partials(cb->plan[b]) : nullptr, fin ? w : nullptr,
                        fin ? y_peers : nullptr, fin ? npeers : 0, b != first, stream);
    if (rc) return rc;
  }
  return B2S_OK;
}

// One block of the sequence above (block `b` only): lets the caller overlap the host->device copy
// of x slice b+1 with the launch of block b (the slice [b*block_cols, (b+1)*block_cols) of x is
// all that block b reads).  Call for b = 0..nblocks-1 in order.  `block | (1 << 30)` forces the
// accumulating form (y += A_b x) for callers that computed the earlier blocks with another operand
// of the same rows (the 2-D host pipeline).
extern "C" int b2s_spmv_colblock_part(const b2s_colblock* cb, int block, const void* x, void* y,
                                      b2s_stream_t stream) {
  B2S_REQUIRE(cb != nullptr, "colblock is null");
  const bool force_acc = (block & (1 << 30)) != 0;   // bit 30: y += A_b x whatever the block's position
  block &= ~(1 << 30);
  B2S_REQUIRE(block >= 0 && block < cb->nblocks, "block out of range");
  B2S_REQUIRE(x != nullptr && y != nullptr, "null vector");
  if (cb->blk_nnz[block] == 0) return B2S_OK;
  int first = 0;
  while (cb->blk_nnz[first] == 0) ++first;
  return spmv_entry(cb->vt, cb->it, cb->nrows, cb->ncols, cb->blk_nnz[block], cb->indptr[block],
                    cb->cols[block], cb->vals[block], x, y, cb->plan[block], B2S_SPMV_PIPE, nullptr,
                    nullptr, nullptr, nullptr, 0, (block != first || force_acc) ? 1 : 0, stream);
}
