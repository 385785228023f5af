// tools/spmv_sweep.cu — standalone (no torch) micro-benchmark used to tune the SpMV kernels.
// Links against libb200sparse.so through the public C ABI; also measures two ceilings:
//   stream : read (col,val) arrays only           → HBM streaming ceiling for this access shape
//   gather : read col + gather x[col] (no vals)   → L2/L1tex gather ceiling
// Usage: spmv_sweep [rows=10000000] [k=50] [iters=20] [mode=random|banded|poisson]   (poisson: rows = grid side N)
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <algorithm>
#include <string>
#include <vector>
#include "../include/b200sparse.h"

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1);} } while (0)

__device__ __forceinline__ uint64_t mix64(uint64_t t) {
  t = (t ^ (t >> 30)) * 0xBF58476D1CE4E5B9ull;
  t = (t ^ (t >> 27)) * 0x94D049BB133111EBull;
  return t ^ (t >> 31);
}

template <typename I>
__global__ void gen_random(int64_t n, int64_t m, int k, I* cols, double* vals, int64_t* indptr) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t total = n * k;
  int64_t stride = m / k;
  for (; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = idx / k, j = idx % k;
    uint64_t h = mix64((uint64_t)idx + 1234567ull);
    cols[idx] = (I)(j * stride + (int64_t)(h % (uint64_t)stride));
    vals[idx] = 2.0 * ((double)(mix64(h + 99) >> 11) / 9007199254740992.0) - 1.0;
    if (j == 0) indptr[i] = i * k;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) indptr[n] = n * k;
}

template <typename I>
__global__ void gen_banded(int64_t n, int k, I* cols, double* vals, const int64_t* indptr) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  int half = k / 2;
  int64_t lo = r - half < 0 ? 0 : r - half;
  int64_t p = indptr[r];
  int64_t cnt = indptr[r + 1] - p;
  for (int64_t t = 0; t < cnt; ++t) { cols[p + t] = (I)(lo + t); vals[p + t] = 1.0; }
}

__global__ void banded_counts(int64_t n, int k, int64_t* cnt) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  int half = k / 2;
  int64_t lo = r - half < 0 ? 0 : r - half, hi = r + half > n - 1 ? n - 1 : r + half;
  cnt[r] = hi - lo + 1;
}

// 5-point Laplacian on an N x N grid (BASELINE config 3): row i has columns i-N, i-1, i, i+1, i+N inside the grid
__global__ void poisson_counts(int64_t N, int64_t* cnt) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * N) return;
  int64_t gi = i / N, gj = i % N;
  cnt[i] = 1 + (gi > 0) + (gi < N - 1) + (gj > 0) + (gj < N - 1);
}
template <typename I>
__global__ void gen_poisson(int64_t N, I* cols, double* vals, const int64_t* indptr) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * N) return;
  int64_t gi = i / N, gj = i % N, p = indptr[i];
  if (gi > 0)     { cols[p] = (I)(i - N); vals[p++] = -1.0; }
  if (gj > 0)     { cols[p] = (I)(i - 1); vals[p++] = -1.0; }
  cols[p] = (I)i; vals[p++] = 4.0;
  if (gj < N - 1) { cols[p] = (I)(i + 1); vals[p++] = -1.0; }
  if (gi < N - 1) { cols[p] = (I)(i + N); vals[p++] = -1.0; }
}

__global__ void fill_x(int64_t n, double* x) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = (double)(mix64(i + 7) >> 11) / 9007199254740992.0;
}

// ceilings
template <typename I>
__global__ void stream_kernel(int64_t nnz, const I* __restrict__ cols, const double* __restrict__ vals, double* out) {
  int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  double acc = 0;
  for (; i + 3 < nnz; i += (int64_t)gridDim.x * blockDim.x * 4) {
    int4 c = *reinterpret_cast<const int4*>(cols + i);
    double2 a = *reinterpret_cast<const double2*>(vals + i);
    double2 b = *reinterpret_cast<const double2*>(vals + i + 2);
    acc += a.x + a.y + b.x + b.y + (double)(c.x ^ c.y ^ c.z ^ c.w);
  }
  if (acc == 1.2345e-300) out[0] = acc;
}

template <int UNROLL>
__global__ void gather_kernel(int64_t nnz, const int* __restrict__ cols, const double* __restrict__ x, double* out) {
  int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  double acc = 0;
  for (; i + 3 < nnz; i += (int64_t)gridDim.x * blockDim.x * 4) {
    int4 c = *reinterpret_cast<const int4*>(cols + i);
    acc += __ldg(x + c.x) + __ldg(x + c.y) + __ldg(x + c.z) + __ldg(x + c.w);
  }
  if (acc == 1.2345e-300) out[0] = acc;
}

struct Timer {
  cudaEvent_t a, b;
  Timer() { cudaEventCreate(&a); cudaEventCreate(&b); }
  void start() { cudaEventRecord(a); }
  float stop() { cudaEventRecord(b); cudaEventSynchronize(b); float ms; cudaEventElapsedTime(&ms, a, b); return ms; }
};

template <typename I>
double run_case(const char* name, b2s_itype it, int64_t n, int64_t m, int64_t nnz, const int64_t* indptr,
                const I* cols, const double* vals, const double* x, double* y, int variant, int tile, int iters,
                bool nowin) {
  if (tile) { char buf[32]; snprintf(buf, sizeof buf, "%d", tile); setenv("B2S_SPMV_TILE_NNZ", buf, 1); }
  else if (!getenv("SWEEP_COLBLOCK")) unsetenv("B2S_SPMV_TILE_NNZ");
  if (getenv("SWEEP_COLBLOCK")) {   // column-blocked operand: SWEEP_COLBLOCK=N blocks (0 = library heuristic)
    int nb = atoi(getenv("SWEEP_COLBLOCK"));
    if (nb == 0) {
      if (b2s_csr_colblock_suggest(B2S_F64, it, n, m, nnz, indptr, cols, nullptr, &nb)) { printf("suggest failed\n"); exit(1); }
      printf("suggested blocks: %d\n", nb);
      if (nb < 2) return 0;
    }
    int64_t wb = b2s_csr_colblock_workspace_bytes(B2S_F64, it, n, nnz, nb);
    void* ws = nullptr; CK(cudaMalloc(&ws, wb));
    b2s_colblock* cb = nullptr;
    Timer tc; tc.start();
    if (b2s_csr_colblock_create(B2S_F64, it, n, m, nnz, indptr, cols, vals, nb, ws, wb, nullptr, &cb)) {
      printf("colblock_create failed: %s\n", b2s_last_error_string()); exit(1);
    }
    float cms = tc.stop();
    for (int i = 0; i < 3; ++i)
      if (b2s_spmv_colblock(cb, x, y, nullptr, nullptr, nullptr, 0, nullptr)) { printf("spmv failed: %s\n", b2s_last_error_string()); exit(1); }
    CK(cudaDeviceSynchronize());
    Timer t; t.start();
    for (int i = 0; i < iters; ++i) b2s_spmv_colblock(cb, x, y, nullptr, nullptr, nullptr, 0, nullptr);
    float ms = t.stop() / iters;
    double bytes = (double)nnz * (8 + sizeof(I)) + (double)(n + 1) * 8 + (double)m * 8 + (double)n * 8;
    printf("%-22s colblock=%d (build %.1f ms) idx%zu : %8.3f ms  %8.1f GFLOP/s  %7.1f GB/s (algorithmic)\n", name, nb, cms,
           sizeof(I) * 8, ms, 2.0 * nnz / ms / 1e6, bytes / ms / 1e6);
    // cross-check against the plain path
    double* y2; CK(cudaMalloc(&y2, n * 8));
    if (b2s_spmv_csr(B2S_F64, it, n, m, nnz, indptr, cols, vals, x, y2, nullptr, B2S_SPMV_ROWVEC, nullptr)) { printf("ref spmv failed\n"); exit(1); }
    std::vector<double> a(1 << 16), b(1 << 16);
    CK(cudaMemcpy(a.data(), y, a.size() * 8, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(b.data(), y2, b.size() * 8, cudaMemcpyDeviceToHost));
    double md = 0; for (size_t i = 0; i < a.size() && (int64_t)i < n; ++i) md = std::max(md, std::abs(a[i] - b[i]));
    printf("  max |colblock - rowvec| over first rows: %.3e\n", md);
    cudaFree(y2); b2s_csr_colblock_destroy(cb); cudaFree(ws);
    return ms;
  }
  if (nowin) setenv("B2S_SPMV_NO_WINDOW", "1", 1); else unsetenv("B2S_SPMV_NO_WINDOW");
  b2s_spmv_plan* plan = nullptr;
  void* ws = nullptr;
  if (variant != B2S_SPMV_ROWVEC) {
    int64_t wb = b2s_spmv_plan_workspace_bytes(n, nnz);
    CK(cudaMalloc(&ws, wb));
    int rc = b2s_spmv_plan_create(it, n, m, nnz, indptr, cols, ws, wb, nullptr, &plan);
    if (rc) { printf("plan_create failed: %s\n", b2s_last_error_string()); exit(1); }
  }
  for (int i = 0; i < 3; ++i) {
    int rc = b2s_spmv_csr(B2S_F64, it, n, m, nnz, indptr, cols, vals, x, y, plan, variant, nullptr);
    if (rc) { printf("spmv failed: %s\n", b2s_last_error_string()); exit(1); }
  }
  CK(cudaDeviceSynchronize());
  Timer t; t.start();
  for (int i = 0; i < iters; ++i) b2s_spmv_csr(B2S_F64, it, n, m, nnz, indptr, cols, vals, x, y, plan, variant, nullptr);
  float ms = t.stop() / iters;
  CK(cudaDeviceSynchronize());
  int64_t nt = 0, tn = 0, wt = 0;
  if (plan) b2s_spmv_plan_info(plan, &nt, &tn, &wt);
  double bytes = (double)nnz * (8 + sizeof(I)) + (double)(n + 1) * 8 + (double)m * 8 + (double)n * 8;
  printf("%-34s idx%zu tile=%5lld win=%lld/%lld : %8.3f ms  %8.1f GFLOP/s  %7.1f GB/s (algorithmic)\n", name,
         sizeof(I) * 8, (long long)tn, (long long)wt, (long long)nt, ms, 2.0 * nnz / ms / 1e6, bytes / ms / 1e6);
  if (plan) b2s_spmv_plan_destroy(plan);
  if (ws) cudaFree(ws);
  return ms;
}

int main(int argc, char** argv) {
  int64_t n = argc > 1 ? atoll(argv[1]) : 10000000;
  const int64_t gridN = n;   // mode=poisson: argv[1] is the grid side N, the matrix has N*N rows
  if (argc > 4 && std::string(argv[4]) == "poisson") n = gridN * gridN;
  int k = argc > 2 ? atoi(argv[2]) : 50;
  int iters = argc > 3 ? atoi(argv[3]) : 20;
  std::string mode = argc > 4 ? argv[4] : "random";
  int64_t m = getenv("SWEEP_NCOLS") ? atoll(getenv("SWEEP_NCOLS")) : n;  // rectangular: one column block
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  if (getenv("SWEEP_L2_PERSIST")) {
    size_t want = (size_t)atoll(getenv("SWEEP_L2_PERSIST")) << 20;
    if (want == 0 || want > (size_t)prop.persistingL2CacheMaxSize) want = prop.persistingL2CacheMaxSize;
    CK(cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want));
    printf("persisting L2 set-aside: %zu MB (max %d MB, window max %d MB)\n", want >> 20,
           prop.persistingL2CacheMaxSize >> 20, prop.accessPolicyMaxWindowSize >> 20);
  }
  printf("device %s, %d SMs, L2 %d MB; n=%lld k=%d mode=%s\n", prop.name, prop.multiProcessorCount,
         prop.l2CacheSize >> 20, (long long)n, k, mode.c_str());
  int64_t* indptr; CK(cudaMalloc(&indptr, (n + 1) * 8));
  int64_t nnz;
  if (mode == "banded") {
    int64_t* cnt; CK(cudaMalloc(&cnt, n * 8));
    banded_counts<<<(unsigned)((n + 255) / 256), 256>>>(n, k, cnt);
    std::vector<int64_t> h(n + 1, 0), hc(n);
    CK(cudaMemcpy(hc.data(), cnt, n * 8, cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n; ++i) h[i + 1] = h[i] + hc[i];
    CK(cudaMemcpy(indptr, h.data(), (n + 1) * 8, cudaMemcpyHostToDevice));
    nnz = h[n]; cudaFree(cnt);
  } else if (mode == "poisson") {
    int64_t* cnt; CK(cudaMalloc(&cnt, n * 8));
    poisson_counts<<<(unsigned)((n + 255) / 256), 256>>>(gridN, cnt);
    std::vector<int64_t> h(n + 1, 0), hc(n);
    CK(cudaMemcpy(hc.data(), cnt, n * 8, cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < n; ++i) h[i + 1] = h[i] + hc[i];
    CK(cudaMemcpy(indptr, h.data(), (n + 1) * 8, cudaMemcpyHostToDevice));
    nnz = h[n]; cudaFree(cnt);
  } else nnz = n * k;
  int32_t* c32; int64_t* c64; double *vals, *x, *y, *sink;
  CK(cudaMalloc(&c32, nnz * 4)); CK(cudaMalloc(&c64, nnz * 8)); CK(cudaMalloc(&vals, nnz * 8));
  CK(cudaMalloc(&x, m * 8)); CK(cudaMalloc(&y, n * 8)); CK(cudaMalloc(&sink, 64));
  if (mode == "banded") {
    gen_banded<int32_t><<<(unsigned)((n + 255) / 256), 256>>>(n, k, c32, vals, indptr);
    gen_banded<int64_t><<<(unsigned)((n + 255) / 256), 256>>>(n, k, c64, vals, indptr);
  } else if (mode == "poisson") {
    gen_poisson<int32_t><<<(unsigned)((n + 255) / 256), 256>>>(gridN, c32, vals, indptr);
    gen_poisson<int64_t><<<(unsigned)((n + 255) / 256), 256>>>(gridN, c64, vals, indptr);
  } else {
    gen_random<int32_t><<<prop.multiProcessorCount * 16, 256>>>(n, m, k, c32, vals, indptr);
    gen_random<int64_t><<<prop.multiProcessorCount * 16, 256>>>(n, m, k, c64, vals, indptr);
  }
  fill_x<<<(unsigned)((m + 255) / 256), 256>>>(m, x);
  CK(cudaDeviceSynchronize());

  // single-config mode (for ncu): spmv_sweep n k iters mode single <variant 1|2|3> <tile> <unused> [i64]
  if (argc > 8 && std::string(argv[5]) == "single") {
    int variant = atoi(argv[6]), tile = atoi(argv[7]);
    bool i64 = argc > 9 && std::string(argv[9]) == "i64";
    if (i64) run_case<int64_t>("single", B2S_I64, n, m, nnz, indptr, c64, vals, x, y, variant, tile, iters, false);
    else     run_case<int32_t>("single", B2S_I32, n, m, nnz, indptr, c32, vals, x, y, variant, tile, iters, false);
    return 0;
  }
  // ceilings
  {
    Timer t;
    for (int w = 0; w < 2; ++w) stream_kernel<int32_t><<<prop.multiProcessorCount * 32, 256>>>(nnz, c32, vals, sink);
    t.start();
    for (int i = 0; i < iters; ++i) stream_kernel<int32_t><<<prop.multiProcessorCount * 32, 256>>>(nnz, c32, vals, sink);
    float ms = t.stop() / iters;
    printf("ceiling stream (col32+val)            : %8.3f ms  %7.1f GB/s\n", ms, nnz * 12.0 / ms / 1e6);
    for (int w = 0; w < 2; ++w) gather_kernel<1><<<prop.multiProcessorCount * 32, 256>>>(nnz, c32, x, sink);
    t.start();
    for (int i = 0; i < iters; ++i) gather_kernel<1><<<prop.multiProcessorCount * 32, 256>>>(nnz, c32, x, sink);
    ms = t.stop() / iters;
    printf("ceiling gather (col32 + x[col])       : %8.3f ms  %7.1f Ggather/s\n", ms, nnz / ms / 1e6);
    CK(cudaDeviceSynchronize());
  }
  if (getenv("SWEEP_COLBLOCK")) {   // column-blocked operand: one measurement with the current environment
    run_case<int32_t>("colblock", B2S_I32, n, m, nnz, indptr, c32, vals, x, y, B2S_SPMV_PIPE, 0, iters, false);
    return 0;
  }
  int tiles[2] = {1024, 2048};
  for (int ti = 0; ti < 2; ++ti) {
    run_case<int32_t>("pipe", B2S_I32, n, m, nnz, indptr, c32, vals, x, y, B2S_SPMV_PIPE, tiles[ti], iters, false);
    if (mode == "banded")
      run_case<int32_t>("pipe (no x window)", B2S_I32, n, m, nnz, indptr, c32, vals, x, y, B2S_SPMV_PIPE, tiles[ti], iters, true);
  }
  run_case<int64_t>("pipe", B2S_I64, n, m, nnz, indptr, c64, vals, x, y, B2S_SPMV_PIPE, 2048, iters, false);
  run_case<int32_t>("tile", B2S_I32, n, m, nnz, indptr, c32, vals, x, y, B2S_SPMV_TILE, 1024, iters, true);
  run_case<int32_t>("rowvec", B2S_I32, n, m, nnz, indptr, c32, vals, x, y, B2S_SPMV_ROWVEC, 0, iters, false);
  return 0;
}
