// tools/gather_paths.cu — which on-chip path can gather 8-byte elements of an L2-resident vector
// fastest on sm_90a?  Standalone micro-benchmark (no torch, no libb200sparse) behind the claim in
// DESIGN.md §3.1b that config-2 SpMV (uniformly random columns) is bound by the per-request rate of
// the gather path and not by HBM.  Every mode performs the SAME work: for `nnz` random int32 column
// ids (read once from HBM, 4 B each) fetch x[col] (fp64) from an x of `xmb` MB and add it up; modes
// differ only in the hardware path that performs the gather:
//
//   lsu        ld.global.nc.f64 per element (what spmv_pipe_kernel's products consumer does)
//   lsu16      ld.global.nc.v2.f64 of the aligned 16-byte pair holding the element
//   bulk16     one 16-byte cp.async.bulk (UBLKCP) per element
//   mixb16     8 LSU warps gather (2048-TM) elements of every 2048-element tile themselves while a
//              producer warp stages the other TM through bulk16 — both request paths at once
//   ldgsts     cp.async.ca.shared.global 8-byte gathers (LDGSTS): the LSU request path, but the data lands in
//              shared memory without holding a destination register while in flight
//   dsmem      x slice spread over the shared memory of a thread-block cluster (8 or 16 CTAs),
//              ld.shared::cluster gathers (no L1TEX tag stage, no L2)
//
// Output: G gathers/s per mode + gathers per clock per SM (at the SM clock measured in-kernel),
// and a checksum against the lsu mode.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo tools/gather_paths.cu -o tools/gather_paths
// Usage: gather_paths [xmb=40] [nnz_millions=256] [iters=5]
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <vector>
#include <string>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1);} } while (0)

__device__ __forceinline__ uint64_t mix64(uint64_t t) {
  t = (t ^ (t >> 30)) * 0xBF58476D1CE4E5B9ull;
  t = (t ^ (t >> 27)) * 0x94D049BB133111EBull;
  return t ^ (t >> 31);
}
__global__ void gen_cols(int64_t nnz, int64_t ncols, int* cols) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += (int64_t)gridDim.x * blockDim.x)
    cols[i] = (int)(mix64((uint64_t)i + 0x1234567ull) % (uint64_t)ncols);
}
__global__ void gen_x(int64_t n, double* x) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    x[i] = (double)(mix64((uint64_t)i + 7) >> 11) / 9007199254740992.0;
}

// ---------------------------------------------------------------- helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint64_t* bar, uint32_t phase) {
  uint32_t ok;
  asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(phase) : "memory");
  return ok != 0;
}
// bounded wait: a mis-programmed TMA must not hang the box
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t phase, int* err) {
  for (int i = 0; i < (1 << 20); ++i) if (mbar_try(bar, phase)) return true;
  atomicExch(err, 1);
  return false;
}
__device__ __forceinline__ void bulk16(void* dst, const void* src, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], 16, [%2];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ double ldg_nc(const double* p) {
  double r; asm("ld.global.nc.f64 %0, [%1];" : "=d"(r) : "l"(p)); return r;
}
__device__ __forceinline__ double ldg_na(const double* p) {
  double r; asm("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(r) : "l"(p)); return r;
}
__device__ __forceinline__ double ldg_cg(const double* p) {
  double r; asm("ld.global.cg.f64 %0, [%1];" : "=d"(r) : "l"(p)); return r;
}
__device__ __forceinline__ double2 ldg_nc2(const double* p) {
  double2 r; asm("ld.global.nc.v2.f64 {%0,%1}, [%2];" : "=d"(r.x), "=d"(r.y) : "l"(p)); return r;
}
__device__ __forceinline__ int4 ldg_stream4(const int* p) {
  int4 r; asm("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p)); return r;
}
__device__ __forceinline__ double block_sum_to(double acc, double* out) {
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
  return acc;
}

// ---------------------------------------------------------------- lsu / lsu16
template <int UNROLL, bool WIDE>
__global__ void __launch_bounds__(256) k_lsu(int64_t nnz, const int* __restrict__ cols, const double* __restrict__ x, double* out) {
  double acc = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
  int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  for (; i + (UNROLL - 1) * stride + 3 < nnz; i += stride * UNROLL) {
    int4 c[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) c[u] = ldg_stream4(cols + i + u * stride);
    double v[UNROLL][4];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      if (WIDE) {
        double2 a = ldg_nc2(x + (c[u].x & ~1)), b = ldg_nc2(x + (c[u].y & ~1)), d = ldg_nc2(x + (c[u].z & ~1)), e = ldg_nc2(x + (c[u].w & ~1));
        v[u][0] = (c[u].x & 1) ? a.y : a.x; v[u][1] = (c[u].y & 1) ? b.y : b.x;
        v[u][2] = (c[u].z & 1) ? d.y : d.x; v[u][3] = (c[u].w & 1) ? e.y : e.x;
      } else {
        v[u][0] = ldg_nc(x + c[u].x); v[u][1] = ldg_nc(x + c[u].y); v[u][2] = ldg_nc(x + c[u].z); v[u][3] = ldg_nc(x + c[u].w);
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) acc += (v[u][0] + v[u][1]) + (v[u][2] + v[u][3]);
  }
  for (; i + 3 < nnz; i += stride) {
    int4 c = ldg_stream4(cols + i);
    acc += ldg_nc(x + c.x) + ldg_nc(x + c.y) + ldg_nc(x + c.z) + ldg_nc(x + c.w);
  }
  block_sum_to(acc, out);
}

// load flavours of the LSU path: MODE 0 = ld.global.nc, 1 = nc + L1::no_allocate, 2 = ld.global.cg
template <int MODE, int INFLIGHT>
__global__ void __launch_bounds__(256) k_lsu_mode(int64_t nnz, const int* __restrict__ cols, const double* __restrict__ x, double* out) {
  double acc = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
  constexpr int U = INFLIGHT / 4;
  int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  for (; i + (U - 1) * stride + 3 < nnz; i += stride * U) {
    int4 c[U];
#pragma unroll
    for (int u = 0; u < U; ++u) c[u] = ldg_stream4(cols + i + u * stride);
    double v[U][4];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int cc[4] = {c[u].x, c[u].y, c[u].z, c[u].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) v[u][k] = MODE == 0 ? ldg_nc(x + cc[k]) : (MODE == 1 ? ldg_na(x + cc[k]) : ldg_cg(x + cc[k]));
    }
#pragma unroll
    for (int u = 0; u < U; ++u) acc += (v[u][0] + v[u][1]) + (v[u][2] + v[u][3]);
  }
  block_sum_to(acc, out);
}

// ---------------------------------------------------------------- ldgsts: cp.async (LDGSTS) 8-byte gathers straight into shared memory
// No destination register is held while the gather is in flight: DEPTH commit groups of 4 gathers per
// thread are outstanding, the thread reads its own 4 slots back (2 x LDS.128) once the oldest group landed.
template <int DEPTH, bool CG16>
__global__ void __launch_bounds__(256) k_ldgsts(int64_t nnz, const int* __restrict__ cols, const double* __restrict__ x, double* out) {
  // CG16: cp.async.cg 16 bytes (LDGSTS.E.BYPASS.128) of the aligned pair that holds the element — the only
  // cp.async form that does not allocate an L1 line per request in flight; the 8-byte form is .ca only
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr int SL = CG16 ? 2 : 1;                          // doubles per slot
  double* ring = reinterpret_cast<double*>(smem);          // [DEPTH][1024 * SL]
  double acc = 0;
  const int tid = threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
  int64_t i = ((int64_t)blockIdx.x * blockDim.x + tid) * 4;
  int it = 0;
  unsigned par[DEPTH];
#pragma unroll
  for (int d = 0; d < DEPTH; ++d) par[d] = 0;
  auto consume = [&](int k) {
    const double* r = ring + ((k % DEPTH) * 1024 + tid * 4) * SL;
    if (CG16) {
      unsigned pm = 0;
#pragma unroll
      for (int d = 0; d < DEPTH; ++d) if (d == k % DEPTH) pm = par[d];
      acc += (r[0 + (pm & 1)] + r[2 + ((pm >> 1) & 1)]) + (r[4 + ((pm >> 2) & 1)] + r[6 + ((pm >> 3) & 1)]);
    } else {
      const double2 a = *reinterpret_cast<const double2*>(r), b = *reinterpret_cast<const double2*>(r + 2);
      acc += (a.x + a.y) + (b.x + b.y);
    }
  };
  for (; i + 3 < nnz; i += stride, ++it) {
    const int4 c = ldg_stream4(cols + i);
    double* slot = ring + ((it % DEPTH) * 1024 + tid * 4) * SL;
    const uint32_t d = smem_u32(slot);
    if (CG16) {
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(x + (c.x & ~1)) : "memory");
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 16), "l"(x + (c.y & ~1)) : "memory");
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 32), "l"(x + (c.z & ~1)) : "memory");
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d + 48), "l"(x + (c.w & ~1)) : "memory");
      const unsigned pm = (c.x & 1) | ((c.y & 1) << 1) | ((c.z & 1) << 2) | ((c.w & 1) << 3);
#pragma unroll
      for (int q = 0; q < DEPTH; ++q) if (q == it % DEPTH) par[q] = pm;
    } else {
      asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(x + c.x) : "memory");
      asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d + 8), "l"(x + c.y) : "memory");
      asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d + 16), "l"(x + c.z) : "memory");
      asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d + 24), "l"(x + c.w) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    if (it >= DEPTH - 1) {
      asm volatile("cp.async.wait_group %0;" ::"n"(DEPTH - 1) : "memory");
      // the group consumed here was issued DEPTH-1 iterations ago; its parity mask is still in par[]
      // only when DEPTH > 1 slots are distinct — consume before this iteration's mask overwrote it
      consume(it - (DEPTH - 1));
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  for (int k = (it >= DEPTH - 1 ? it - (DEPTH - 1) : 0); k < it; ++k) consume(k);
  block_sum_to(acc, out);
}

// ---------------------------------------------------------------- bulk16 (optionally mixed with LSU gathers)
// CTA = NCW consumer warps + 1 producer warp.  A tile = 2048 consecutive column ids.  The LAST TM of
// them are fetched by the producer warp into a ring stage (TM*16 bytes: every element arrives as the
// aligned 16-byte pair that holds it) together with the tile's TM column ids; consumers read them
// out of shared memory.  The first 2048-TM are gathered by the consumers through the LSU.
template <int NCW, int TILE, int TM, int STAGES>
__global__ void __launch_bounds__((NCW + 1) * 32)
k_tma(int64_t ntiles, const int* __restrict__ cols, const double* __restrict__ x,
      double* out, int consume, int* err) {
  constexpr int NCT = NCW * 32;
  constexpr int SLOT = 16;   // bytes per element
  constexpr int STAGE_BYTES = TM * SLOT + TM * 4;
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)STAGE_BYTES * STAGES);
  uint64_t* empty = full + STAGES;
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], NCT); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid >= NCT) {
    if (TM == 0) return;
    const int lane = tid - NCT;
    int64_t it = 0;
    for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
      const int s = (int)(it % STAGES);
      const uint32_t ph = (uint32_t)((it / STAGES) & 1);
      if (!mbar_wait(&empty[s], ph ^ 1u, err)) return;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // consumers' generic reads before the async-proxy refill
      unsigned char* st = smem + (size_t)STAGE_BYTES * s;
      int* scol = reinterpret_cast<int*>(st + TM * SLOT);
      const int* src = cols + t * TILE + (TILE - TM);
      // lane handles column ids [q*128 + lane*4, +4) for q = 0 .. TM/128-1
      int4 c[TM / 128 > 0 ? TM / 128 : 1];
#pragma unroll
      for (int q = 0; q < TM / 128; ++q) {
        c[q] = ldg_stream4(src + q * 128 + lane * 4);
        *reinterpret_cast<int4*>(scol + q * 128 + lane * 4) = c[q];
      }
      __syncwarp();
      if (lane == 0) mbar_expect_tx(&full[s], TM * 16);
      __syncwarp();
#pragma unroll
      for (int q = 0; q < TM / 128; ++q) {
        unsigned char* dst = st + (size_t)(q * 128 + lane * 4) * SLOT;
        bulk16(dst, x + (c[q].x & ~1), &full[s]);
        bulk16(dst + 16, x + (c[q].y & ~1), &full[s]);
        bulk16(dst + 32, x + (c[q].z & ~1), &full[s]);
        bulk16(dst + 48, x + (c[q].w & ~1), &full[s]);
      }
    }
    return;
  }
  double acc = 0;
  int64_t it = 0;
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
    // LSU share first (its latency overlaps the producer's work on this tile)
    constexpr int NL = TILE - TM;
    constexpr int NQ = (NL + NCT * 4 - 1) / (NCT * 4);
    const int* src = cols + t * TILE;
    int4 c[NQ > 0 ? NQ : 1];
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
      const int e = (q * NCT + tid) * 4;
      c[q] = e < NL ? ldg_stream4(src + e) : make_int4(-1, -1, -1, -1);
    }
#pragma unroll
    for (int q = 0; q < NQ; ++q)
      if (c[q].x >= 0) acc += (ldg_nc(x + c[q].x) + ldg_nc(x + c[q].y)) + (ldg_nc(x + c[q].z) + ldg_nc(x + c[q].w));
    if (TM > 0) {
      const int s = (int)(it % STAGES);
      const uint32_t ph = (uint32_t)((it / STAGES) & 1);
      if (!mbar_wait(&full[s], ph, err)) return;
      if (consume) {
        const unsigned char* st = smem + (size_t)STAGE_BYTES * s;
        const int* scol = reinterpret_cast<const int*>(st + TM * SLOT);
        const double* sd = reinterpret_cast<const double*>(st);
        for (int e = tid; e < TM; e += NCT) acc += sd[(e >> 2) * (SLOT / 2) + (e & 3) * 2 + (scol[e] & 1)];
      }
      mbar_arrive(&empty[s]);
    }
  }
  block_sum_to(acc, out);
}

// ---------------------------------------------------------------- DSMEM
// Cluster of CS CTAs, each holds SLICE doubles of x in shared memory; every thread gathers elements
// with ids uniform in [0, CS*SLICE) through ld.shared::cluster (mapa to the owning CTA).
template <int SLICE>
__global__ void __launch_bounds__(256) k_dsmem(int64_t nnz_per_cluster, const int* __restrict__ cols, const double* __restrict__ x,
                                               double* out, int cs) {
  extern __shared__ __align__(128) unsigned char smem[];
  double* sx = reinterpret_cast<double*>(smem);
  uint32_t rank, cid;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(cid));
  for (int i = threadIdx.x; i < SLICE; i += blockDim.x) sx[i] = x[(int64_t)rank * SLICE + i];
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  const uint32_t base = smem_u32(sx);
  const uint32_t total = (uint32_t)cs * SLICE;
  double acc = 0;
  const int* src = cols + (int64_t)cid * nnz_per_cluster;
  const int64_t stride = (int64_t)cs * 256 * 4;
  for (int64_t i = ((int64_t)rank * 256 + threadIdx.x) * 4; i + 3 < nnz_per_cluster; i += stride) {
    int4 c = ldg_stream4(src + i);
    uint32_t id[4] = {(uint32_t)c.x % total, (uint32_t)c.y % total, (uint32_t)c.z % total, (uint32_t)c.w % total};
    double v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint32_t owner = id[k] / SLICE, off = id[k] % SLICE, addr;
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(addr) : "r"(base + off * 8), "r"(owner));
      asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v[k]) : "r"(addr));
    }
    acc += (v[0] + v[1]) + (v[2] + v[3]);
  }
  asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  block_sum_to(acc, out);
}

__global__ void k_mod_ref(int64_t n, const int* __restrict__ cols, const double* __restrict__ x, uint32_t total, double* out) {
  double acc = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    acc += x[(uint32_t)cols[i] % total];
  block_sum_to(acc, out);
}

// SM clock during a memory-bound kernel: clock64 delta / globaltimer delta on one thread
__global__ void k_clock(double* mhz) {
  uint64_t t0, t1; long long c0 = clock64();
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  do { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); } while (t1 - t0 < 2000000ull);
  long long c1 = clock64();
  *mhz = (double)(c1 - c0) / (double)(t1 - t0) * 1e3;
}

struct Timer {
  cudaEvent_t a, b;
  Timer() { cudaEventCreate(&a); cudaEventCreate(&b); }
  void start() { cudaEventRecord(a); }
  float stop() { cudaEventRecord(b); cudaEventSynchronize(b); float ms; cudaEventElapsedTime(&ms, a, b); return ms; }
};

static double g_mhz = 1000.0;   // replaced by the in-kernel measurement
static int g_sms = 1;
static double* d_out;
static int* d_err;
static double ref_sum = 0;

static void report(const char* name, float ms, int64_t nnz, double sum, double expect) {
  int err = 0; CK(cudaMemcpy(&err, d_err, 4, cudaMemcpyDeviceToHost));
  double rate = nnz / (ms * 1e-3) / 1e9;
  double rel = expect > 0 ? fabs(sum - expect) / fabs(expect) : 0;
  printf("%-44s %8.3f ms  %7.1f Ggather/s  %5.2f /clk/SM   checksum relerr %.1e%s\n", name, ms, rate,
         rate * 1e9 / (g_mhz * 1e6) / g_sms, rel, err ? "  [TIMEOUT FLAG SET]" : "");
  fflush(stdout);
  CK(cudaMemset(d_err, 0, 4));
}

template <typename F>
static void run(const char* name, int64_t nnz, int iters, double expect, F launch) {
  Timer t;
  CK(cudaMemset(d_out, 0, 8));
  launch();
  CK(cudaDeviceSynchronize());
  double sum; CK(cudaMemcpy(&sum, d_out, 8, cudaMemcpyDeviceToHost));
  launch();
  t.start();
  for (int i = 0; i < iters; ++i) launch();
  float ms = t.stop() / iters;
  CK(cudaGetLastError());
  report(name, ms, nnz, sum, expect);
  if (expect == 0 && ref_sum == 0) ref_sum = sum;
}

template <int NCW, int TILE, int TM, int STAGES>
static void run_tma(const char* label, int64_t nnz, const int* cols, const double* x, int iters, int ctas_per_sm,
                    int consume, double expect) {
  auto kern = k_tma<NCW, TILE, TM, STAGES>;
  size_t smem = (size_t)(TM * (16 + 4)) * STAGES + 16 * STAGES + 128;
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int occ = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, (NCW + 1) * 32, smem));
  int per = ctas_per_sm < occ ? ctas_per_sm : occ;
  int64_t ntiles = nnz / TILE;
  char name[128];
  snprintf(name, sizeof name, "%s TMA %d of %d, warps=%d+1, CTAs/SM=%d%s", label, TM, TILE, NCW, per, consume ? "" : " (no read-out)");
  run(name, ntiles * TILE, iters, consume ? expect : -1.0, [&] { kern<<<per * g_sms, (NCW + 1) * 32, smem>>>(ntiles, cols, x, d_out, consume, d_err); });
}

int main(int argc, char** argv) {
  int xmb = argc > 1 ? atoi(argv[1]) : 40;
  int64_t nnz = (int64_t)(argc > 2 ? atoi(argv[2]) : 256) << 20;
  int iters = argc > 3 ? atoi(argv[3]) : 5;
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  g_sms = prop.multiProcessorCount;
  nnz = nnz / (2048 * g_sms * 8) * (2048 * g_sms * 8);
  int64_t ncols = ((int64_t)xmb << 20) / 8;
  printf("device %s, %d SMs, L2 %d MB; x = %d MB (%lld fp64), %lld gathers per pass\n", prop.name, prop.multiProcessorCount,
         prop.l2CacheSize >> 20, xmb, (long long)ncols, (long long)nnz);
  int* cols; double* x; double* d_mhz;
  CK(cudaMalloc(&cols, nnz * 4)); CK(cudaMalloc(&x, ncols * 8)); CK(cudaMalloc(&d_out, 64 * 8)); CK(cudaMalloc(&d_err, 4));
  CK(cudaMalloc(&d_mhz, 8)); CK(cudaMemset(d_err, 0, 4));
  gen_cols<<<g_sms * 8, 256>>>(nnz, ncols, cols);
  gen_x<<<g_sms * 8, 256>>>(ncols, x);
  CK(cudaDeviceSynchronize());

  // ---- LSU paths
  run("lsu   ld.global.nc.f64  unroll 1 (4 in flight)", nnz, iters, 0, [&] { k_lsu<1, false><<<g_sms * 8, 256>>>(nnz, cols, x, d_out); });
  // SM clock right after a loaded kernel
  k_clock<<<1, 1>>>(d_mhz); CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(&g_mhz, d_mhz, 8, cudaMemcpyDeviceToHost));
  printf("SM clock measured in-kernel: %.0f MHz (1 gather/clk/SM = %.1f Ggather/s)\n", g_mhz, g_mhz * g_sms / 1e3);
  run("lsu   ld.global.nc.f64  unroll 1", nnz, iters, ref_sum, [&] { k_lsu<1, false><<<g_sms * 8, 256>>>(nnz, cols, x, d_out); });
  run("lsu   ld.global.nc.f64  unroll 2 (8 in flight)", nnz, iters, ref_sum, [&] { k_lsu<2, false><<<g_sms * 8, 256>>>(nnz, cols, x, d_out); });
  run("lsu   ld.global.nc.f64  unroll 4 (16 in flight)", nnz, iters, ref_sum, [&] { k_lsu<4, false><<<g_sms * 8, 256>>>(nnz, cols, x, d_out); });
  run("lsu   unroll 2, 4 CTAs/SM", nnz, iters, ref_sum, [&] { k_lsu<2, false><<<g_sms * 4, 256>>>(nnz, cols, x, d_out); });
  run("lsu16 ld.global.nc.v2.f64 unroll 2", nnz, iters, ref_sum, [&] { k_lsu<2, true><<<g_sms * 8, 256>>>(nnz, cols, x, d_out); });

  // ---- cp.async (LDGSTS) gathers into shared memory: DEPTH x 4 gathers per thread in flight, no registers held.
  // `smem KB/SM` is what the resident CTAs allocate: the driver sizes the L1 with what is left of 256 KB, and the
  // 8-byte form (.ca) needs an L1 line per request in flight, the 16-byte form (.cg) does not.
  {
    auto go = [&](auto kern, const char* what, int depth, int ctas, size_t pad_kb) {
      size_t sm = (size_t)depth * 8192 * (strstr(what, "cg") ? 2 : 1) + pad_kb * 1024;
      CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
      CK(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
      char name[128]; snprintf(name, sizeof name, "ldgsts %s, %2d in flight/thread, CTAs/SM=%d, smem %3zu KB/SM", what, depth * 4, ctas, sm * ctas / 1024);
      run(name, nnz, iters, ref_sum, [&] { kern<<<g_sms * ctas, 256, sm>>>(nnz, cols, x, d_out); });
    };
    for (int ctas : {2, 4}) {
      for (size_t pad : {(size_t)0, (size_t)32}) {
        go(k_ldgsts<2, false>, "ca  8 B", 2, ctas, pad);
        go(k_ldgsts<2, true>,  "cg 16 B", 2, ctas, pad);
      }
    }
    go(k_ldgsts<1, false>, "ca  8 B", 1, 4, 0);
    go(k_ldgsts<1, true>,  "cg 16 B", 1, 4, 0);
    if (getenv("GATHER_LDGSTS_ONLY")) return 0;
  }

  // ---- load flavours x requests in flight x CTAs/SM (matters when x misses L2: run with xmb = 64 / 160)
  if (getenv("GATHER_FLAVOURS")) {
    const char* fl[3] = {"nc", "nc.L1::no_allocate", "cg"};
    for (int ctas : {4, 8}) {
      run((std::string("lsu ") + fl[0] + "  4 in flight, CTAs/SM=" + std::to_string(ctas)).c_str(), nnz, iters, ref_sum, [&] { k_lsu_mode<0, 4><<<g_sms * ctas, 256>>>(nnz, cols, x, d_out); });
      run((std::string("lsu ") + fl[1] + "  4 in flight, CTAs/SM=" + std::to_string(ctas)).c_str(), nnz, iters, ref_sum, [&] { k_lsu_mode<1, 4><<<g_sms * ctas, 256>>>(nnz, cols, x, d_out); });
      run((std::string("lsu ") + fl[2] + "  4 in flight, CTAs/SM=" + std::to_string(ctas)).c_str(), nnz, iters, ref_sum, [&] { k_lsu_mode<2, 4><<<g_sms * ctas, 256>>>(nnz, cols, x, d_out); });
      run((std::string("lsu ") + fl[0] + " 16 in flight, CTAs/SM=" + std::to_string(ctas)).c_str(), nnz, iters, ref_sum, [&] { k_lsu_mode<0, 16><<<g_sms * ctas, 256>>>(nnz, cols, x, d_out); });
      run((std::string("lsu ") + fl[1] + " 16 in flight, CTAs/SM=" + std::to_string(ctas)).c_str(), nnz, iters, ref_sum, [&] { k_lsu_mode<1, 16><<<g_sms * ctas, 256>>>(nnz, cols, x, d_out); });
      run((std::string("lsu ") + fl[2] + " 16 in flight, CTAs/SM=" + std::to_string(ctas)).c_str(), nnz, iters, ref_sum, [&] { k_lsu_mode<2, 16><<<g_sms * ctas, 256>>>(nnz, cols, x, d_out); });
    }
    return 0;
  }

  // ---- bulk16: producer warp stages the gathers with 16-byte cp.async.bulk copies
  run_tma<2, 512, 512, 4>("bulk16", nnz, cols, x, iters, 1, 1, ref_sum);
  run_tma<2, 512, 512, 4>("bulk16", nnz, cols, x, iters, 4, 1, ref_sum);
  run_tma<2, 256, 256, 4>("bulk16", nnz, cols, x, iters, 8, 1, ref_sum);
  run_tma<2, 512, 512, 4>("bulk16", nnz, cols, x, iters, 4, 0, ref_sum);
  // both paths at once: 8 LSU warps + 1 bulk-copy producer warp per CTA
  run_tma<8, 2048, 256, 2>("mixb16", nnz, cols, x, iters, 2, 1, ref_sum);
  run_tma<8, 2048, 512, 2>("mixb16", nnz, cols, x, iters, 2, 1, ref_sum);

  // ---- DSMEM: x slice in the shared memory of a cluster
  {
    constexpr int SLICE = 24 * 1024;   // 192 KB of fp64 per CTA
    auto kern = k_dsmem<SLICE>;
    size_t smem = (size_t)SLICE * 8;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    for (int cs : {1, 2, 4, 8, 16}) {
      cudaLaunchConfig_t cfg = {};
      cfg.blockDim = dim3(256);
      cfg.dynamicSmemBytes = smem;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      cfg.attrs = at; cfg.numAttrs = 1;
      int nclusters = 0;
      cfg.gridDim = dim3(cs);
      cudaError_t e = cudaOccupancyMaxActiveClusters(&nclusters, kern, &cfg);
      if (e != cudaSuccess || nclusters < 1) { printf("dsmem cluster=%d: not launchable (%s)\n", cs, cudaGetErrorString(e)); cudaGetLastError(); continue; }
      cfg.gridDim = dim3(nclusters * cs);
      int64_t per_cluster = nnz / 4 / nclusters / (cs * 1024) * (cs * 1024);   // a quarter of the gathers is plenty
      char name[96]; snprintf(name, sizeof name, "dsmem cluster=%d (%d clusters, %d SMs, %.1f MB of x each)", cs, nclusters, nclusters * cs,
                              cs * SLICE * 8.0 / 1048576.0);
      const int* ccols = cols; const double* cx = x; int ccs = cs;
      Timer t;
      CK(cudaMemset(d_out, 0, 8));
      CK(cudaLaunchKernelEx(&cfg, kern, per_cluster, ccols, cx, d_out, ccs));
      CK(cudaDeviceSynchronize());
      double got, want; CK(cudaMemcpy(&got, d_out, 8, cudaMemcpyDeviceToHost));
      CK(cudaMemset(d_out, 0, 8));
      k_mod_ref<<<g_sms * 8, 256>>>(per_cluster * nclusters, cols, x, (uint32_t)(cs * SLICE), d_out);
      CK(cudaDeviceSynchronize());
      CK(cudaMemcpy(&want, d_out, 8, cudaMemcpyDeviceToHost));
      t.start();
      for (int i = 0; i < iters; ++i) CK(cudaLaunchKernelEx(&cfg, kern, per_cluster, ccols, cx, d_out, ccs));
      float ms = t.stop() / iters;
      double rate = (double)per_cluster * nclusters / (ms * 1e-3) / 1e9;
      printf("%-60s %8.3f ms  %7.1f Ggather/s  %5.2f /clk/SM-in-use   checksum relerr %.1e\n", name, ms, rate,
             rate * 1e9 / (g_mhz * 1e6) / (nclusters * cs), fabs(got - want) / fabs(want));
    }
  }
  return 0;
}
