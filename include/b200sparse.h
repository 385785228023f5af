/*
 * b200sparse.h — C ABI of libb200sparse.so, the H100 (sm_90a) sparse hot path.
 *
 * This header is the drop-in boundary (SURVEY.md §8b).  The reference
 * (nv-legate/legate-sparse @ 49271fa) exports exactly one C symbol,
 *   void legate_sparse_perform_registration(void)      src/sparse/sparse_c.h:26
 * and moves everything else through Legate task contexts, i.e. there is no
 * per-operation C ABI upstream.  The entry points below are what the
 * reference's per-op task variants would bind if they were plain C calls;
 * each one cites the task (file:line) it replaces.
 *
 * Conventions (all entry points):
 *   - plain C types only: raw DEVICE pointers, sizes, an opaque stream handle
 *     (a cudaStream_t passed as void*; NULL = legacy default stream);
 *   - every call is asynchronous on `stream` unless stated otherwise and
 *     returns 0 on success or a non-zero B2S_ERR_* code (never aborts; the
 *     reference aborts via assert(false), src/sparse/util/cuda_help.h:51-74);
 *   - the caller owns every buffer (matrix arrays, vectors, workspaces);
 *   - matrices are scipy-layout CSR: indptr[nrows+1] (int64), indices[nnz]
 *     (int32 or int64, see b2s_itype), data[nnz].  The reference's
 *     Rect<1>{lo,hi} `pos` packing (legate_sparse/csr.py:238-251) is a Legion
 *     artifact and is not part of this boundary.
 */
#ifndef B200SPARSE_H
#define B200SPARSE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2S_VERSION 100 /* 0.1.0 */

/* value types = the reference's supported set (legate_sparse/utils.py:28-33,
 * src/sparse/util/dispatch.h:33-48) */
typedef enum { B2S_F32 = 0, B2S_F64 = 1, B2S_C64 = 2, B2S_C128 = 3 } b2s_dtype;
/* column-index width (reference: int64 `coord_ty`, legate_sparse/types.py:20;
 * dispatch.h:56-77 also instantiates int32) */
typedef enum { B2S_I32 = 0, B2S_I64 = 1 } b2s_itype;

enum {
  B2S_OK              = 0,
  B2S_ERR_ARG         = 1, /* bad argument (null pointer, negative size, bad enum) */
  B2S_ERR_CUDA        = 2, /* a CUDA runtime call / launch failed */
  B2S_ERR_WORKSPACE   = 3, /* caller workspace too small */
  B2S_ERR_UNSUPPORTED = 4, /* dtype/itype combination not built */
  B2S_ERR_OVERFLOW    = 5  /* hash table / size overflow */
};

typedef void* b2s_stream_t; /* cudaStream_t */

int         b2s_version(void);
const char* b2s_last_error_string(void); /* thread-local, valid until next call */
/* number of kernels launched by this library in this process (bench `gpu_launches`) */
int64_t     b2s_launch_count(void);

/* ------------------------------------------------------------------------
 * CSR SpMV  y = A x.          replaces CSRSpMVRowSplit::gpu_variant
 *   src/sparse/array/csr/spmv.cu:30-163 (cuSPARSE SpMV) and the CPU/OMP loops
 *   spmv.cc:36-43 / spmv_omp.cc:36-44.
 *
 * The local row block is [0,nrows); `x` is addressed with GLOBAL column ids
 * (the reference shifts the x base pointer instead, spmv.cu:75-90).
 *
 * Plan = cached per-matrix tiling (the analogue of Legate's cached image
 * partitions, csr.py:587-591): nnz-balanced tiles, the row that each tile
 * starts in, and the [min col, max col] x-window of each tile (the
 * reference's MIN_MAX image of crd→x).  Building a plan synchronises the
 * stream once.  `plan` may be NULL: then the plan-free row-vector kernel runs.
 * ---------------------------------------------------------------------- */
typedef struct b2s_spmv_plan b2s_spmv_plan; /* opaque, host object */

/* AUTO: PIPE when a plan is given and the arrays are 16-byte aligned, else TILE, else ROWVEC.
 * PIPE   = persistent kernel, (col,val,indptr[,x window]) streamed by TMA bulk copies into a shared-
 *          memory ring by a producer warp; consumers: row-walk (window matrices) or two ping-pong
 *          groups doing products + row reduction (x gathered from L2).  nnz-balanced tiles, rows
 *          that straddle tiles are completed by a fix-up pass (merge-path style decomposition).
 *          Matrices with skewed row lengths (plan statistic: longest row > 64 and > 8 x the mean; BASELINE
 *          config 5) run the async-gather kernel instead for plain y = A x / y += A x: x gathered by
 *          L1-bypassing cp.async one tile ahead, segmented sum in nnz order (b2s_spmv_agather.cuh).
 *          Same results contract: no floating-point atomics, bit-reproducible run to run.
 * TILE   = one CTA per tile, register-staged 128-bit loads (fallback for unaligned slices)
 * ROWVEC = plan-free 2..32 lanes per row */
enum { B2S_SPMV_AUTO = 0, B2S_SPMV_ROWVEC = 1, B2S_SPMV_TILE = 2, B2S_SPMV_PIPE = 3 };

/* bytes of device workspace a plan for this matrix needs */
int64_t b2s_spmv_plan_workspace_bytes(int64_t nrows, int64_t nnz);

int b2s_spmv_plan_create(b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                         const int64_t* indptr, const void* indices,
                         void* workspace, int64_t workspace_bytes,
                         b2s_stream_t stream, b2s_spmv_plan** out_plan);
void b2s_spmv_plan_destroy(b2s_spmv_plan* plan);
/* introspection (tests / bench): number of tiles, nnz per tile, and how many
 * tiles stage their x window in shared memory through the TMA bulk copy */
int b2s_spmv_plan_info(const b2s_spmv_plan* plan, int64_t* ntiles, int64_t* tile_nnz,
                       int64_t* window_tiles);

int b2s_spmv_csr(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                 const int64_t* indptr, const void* indices, const void* data,
                 const void* x, void* y, const b2s_spmv_plan* plan, int variant,
                 b2s_stream_t stream);

/* SpMV fused with the all-gather of y (multi-GPU, SURVEY §8e): besides the local `y` (this rank's
 * row block) every y[r] is also stored into `y_peers[g][r]`, g < npeers <= 7 — the same row block
 * inside the replicated result buffers of the OTHER ranks (peer device memory mapped with CUDA
 * IPC / symmetric memory; pointers already offset to this rank's first row).  The gather rides on
 * the kernel's own stores over NVLink/NVSwitch instead of a separate ncclAllGather; the caller
 * brackets the call with a cross-rank barrier.  Needs a plan and 16-byte aligned arrays.
 * npeers == -1: y_peers[0] is an NVSwitch MULTICAST address (NVLS) covering every rank's buffer —
 * each value is stored once with multimem.st and replicated by the switch. */
int b2s_spmv_csr_bcast(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                       const int64_t* indptr, const void* indices, const void* data,
                       const void* x, void* y, void* const* y_peers, int npeers,
                       const b2s_spmv_plan* plan, b2s_stream_t stream);

/* SpMV fused with a dot product:  y = A x;  dot_out[0] = sum_r w[r] * y[r]  (no conjugation).
 * With w = x (+ the row offset of the block) this is the CG pair q=A.matvec(p); pq=p.dot(q)
 * (linalg.py:519-520) in one pass.  `w` has nrows entries, `dot_out` is one device scalar of
 * the value type.  Requires a plan (per-tile partials live in the plan workspace). */
int b2s_spmv_csr_dot(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                     const int64_t* indptr, const void* indices, const void* data,
                     const void* x, void* y, const void* w, const b2s_spmv_plan* plan,
                     void* dot_out, b2s_stream_t stream);

/* ------------------------------------------------------------------------
 * Column-blocked operand for SpMV when x does not stay L2-resident (ncols * sizeof(value) well
 * above ~40 MB and rows that reach across all of x — the random C2 matrix of BASELINE.json).
 * A one-time layout of the operand of the reference's SpMV task body
 * (src/sparse/array/csr/spmv.cu:30-163, which only sizes a cuSPARSE buffer —
 * cusparseSpMV_bufferSize, spmv.cu:117-135 — and has no operand preparation), cached next to the plan.
 * A = [A_0 | A_1 | ...] by column ranges of `block_cols`; y = A_0 x; y += A_1 x; ... — one pipe
 * kernel launch per block, each gathering from one slice of x.  The object keeps device
 * pointers into `workspace` (caller-owned, must outlive it) and a COPY of the values: rebuild it
 * when the matrix values change.
 * ------------------------------------------------------------------------ */
typedef struct b2s_colblock b2s_colblock; /* opaque, host object */

/* Heuristic: *out_nblocks = 1 → not worthwhile; otherwise the number of blocks to build.
 * Samples row spans on the device (synchronises the stream).  B2S_SPMV_COLBLOCK=0 disables,
 * =N forces N blocks; B2S_COLBLOCK_MB sets the x-slice size (default 40). */
int b2s_csr_colblock_suggest(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                             const int64_t* indptr, const void* indices, b2s_stream_t stream,
                             int* out_nblocks);
int64_t b2s_csr_colblock_workspace_bytes(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t nnz,
                                         int nblocks);
/* nblocks in [2,32].  Entries keep their order within a row (stable split). */
int b2s_csr_colblock_create(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                            const int64_t* indptr, const void* indices, const void* data,
                            int nblocks, void* workspace, int64_t workspace_bytes,
                            b2s_stream_t stream, b2s_colblock** out);
void b2s_csr_colblock_destroy(b2s_colblock* cb);
int b2s_csr_colblock_info(const b2s_colblock* cb, int* nblocks, int64_t* block_cols,
                          int64_t* blk_nnz /* [nblocks] or NULL */);
/* y = A x over the blocks.  Optional fused dot (w, dot_out as in b2s_spmv_csr_dot) and peer
 * broadcast (y_peers, npeers as in b2s_spmv_csr_bcast) are applied by the last block's launch. */
int b2s_spmv_colblock(const b2s_colblock* cb, const void* x, void* y, const void* w, void* dot_out,
                      void* const* y_peers, int npeers, b2s_stream_t stream);
/* Block `block` of that sequence only (call for 0..nblocks-1 in order).  Block b reads only
 * x[b*block_cols, (b+1)*block_cols), so a host caller can overlap the H2D copy of the next slice
 * of x with this launch.  `block | (1 << 30)` forces the accumulating form y += A_b x (for a caller
 * that computed the earlier blocks of the same rows with another operand: 2-D row x column blocks). */
int b2s_spmv_colblock_part(const b2s_colblock* cb, int block, const void* x, void* y,
                           b2s_stream_t stream);

/* ------------------------------------------------------------------------
 * Dense vector kernels of the CG/GMRES loop.
 * ---------------------------------------------------------------------- */
/* AXPBY task: src/sparse/linalg/axpby.cu:25-66, axpby_template.inl:30-71.
 *   val = a[0]/b[0] (device scalars), negated if `negate`;
 *   isalpha: y = val*x + y   else: y = x + val*y                          */
int b2s_axpby(b2s_dtype vt, int64_t n, void* y, const void* x, const void* a, const void* b,
              int isalpha, int negate, b2s_stream_t stream);

int64_t b2s_reduce_workspace_bytes(void);
/* out[0] = sum_i conj?(x_i) * y_i  — numpy `x.dot(y)` semantics (NO conjugation),
 * the reference calls cupynumeric r.dot(z) (linalg.py:510,520); conj=1 gives vdot. */
int b2s_dot(b2s_dtype vt, int64_t n, const void* x, const void* y, int conj, void* out,
            void* partials, b2s_stream_t stream);
/* out[0] = ||x||_2 as the REAL type of vt (np.linalg.norm, linalg.py:482,529) */
int b2s_nrm2(b2s_dtype vt, int64_t n, const void* x, void* out, void* partials,
             b2s_stream_t stream);

/* Fused CG vector update (identity preconditioner), one pass over x,r,p,q:
 *   alpha = rho/pq;  x += alpha p;  r -= alpha q;  rr_out = <r,r>
 * = the two cg_axpby calls + the next r.dot(z) of linalg.py:523-525,510.      */
int b2s_cg_update(b2s_dtype vt, int64_t n, void* x, void* r, const void* p, const void* q,
                  const void* rho, const void* pq, void* rr_out, void* partials,
                  b2s_stream_t stream);
/* p = r + (rho/rho1) p   (linalg.py:516-518 with z == r); rho1[0]==0 ⇒ p = r */
int b2s_cg_pupdate(b2s_dtype vt, int64_t n, void* p, const void* r, const void* rho,
                   const void* rho1, b2s_stream_t stream);
/* same, and the new p block is also stored into the replicated p of every peer rank (fuses the
 * per-iteration all-gather of p of the row-partitioned CG into the update kernel) */
int b2s_cg_pupdate_bcast(b2s_dtype vt, int64_t n, void* p, const void* r, const void* rho,
                         const void* rho1, void* const* p_peers, int npeers, b2s_stream_t stream);
/* halo variant: peer g only receives the elements [lo[g], hi[g]) of this block (host arrays,
 * relative to the block) — the [min col, max col] image of the peer's rows, i.e. the reference's
 * image(crd→x, MIN_MAX) window (csr.py:591); an empty range (hi<=lo) sends nothing.  For banded /
 * stencil matrices this turns the all-gather of p into a nearest-neighbour halo exchange. */
int b2s_cg_pupdate_halo(b2s_dtype vt, int64_t n, void* p, const void* r, const void* rho,
                        const void* rho1, void* const* p_peers, int npeers, const int64_t* lo,
                        const int64_t* hi, b2s_stream_t stream);

/* ------------------------------------------------------------------------
 * Restarted GMRES, classical Gram-Schmidt (legate_sparse/linalg.py:607-640,655-657): the
 * tall-skinny products  h = V^H u,  u -= V h,  ||u||,  v = u/||u||,  x += V y  that upstream are
 * cupynumeric GEMVs on an (n, restart) array.  The Krylov basis is stored basis-vector-major:
 * vector c is basis[c*ldv .. c*ldv+n), ldv >= n (ldv*sizeof(value) a multiple of 16 enables the
 * 128-bit path).  `workspace`: b2s_cgs_workspace_bytes() bytes, zero-initialised once, reusable.
 * ------------------------------------------------------------------------ */
int64_t b2s_cgs_workspace_bytes(void);
/* h[c] = sum_i conj(basis[c][i]) * u[i],  c < k   (device output, k values) */
int b2s_cgs_project(b2s_dtype vt, int64_t n, int k, const void* basis, int64_t ldv, const void* u,
                    void* h, void* workspace, b2s_stream_t stream);
/* u[i] += s * sum_c h[c] * basis[c][i]  with s = -1 if negate else +1 (k <= 1024);
 * nrm_out (optional, device REAL scalar) = ||u_new||_2 in the same pass. */
int b2s_cgs_update(b2s_dtype vt, int64_t n, int k, const void* basis, int64_t ldv, const void* h,
                   int negate, void* u, void* nrm_out, void* workspace, b2s_stream_t stream);
/* out[i] = x[i] / s[0]   (s: device REAL scalar; out may be a basis row) */
int b2s_vscale_inv(b2s_dtype vt, int64_t n, const void* x, const void* s, void* out,
                   b2s_stream_t stream);

/* ------------------------------------------------------------------------
 * Cross-GPU all-reduce(sum) of one device scalar per rank through peer-mapped "boards" (NVLink P2P
 * stores + sequence flags inside a one-warp kernel; summed in rank order → bit-identical on every
 * rank).  The CG iteration's replacement for NCCL all-reduces of rho / p.q — the reference reduces
 * the same scalars as Legate futures (legate_sparse/linalg.py:519-526).
 *   boards[g]    device address of rank g's board (b2s_board_bytes() bytes, zero-initialised,
 *                symmetric memory; own board included)
 *   seq_counters >= 4 local device uint64, zeroed once;  err: optional local device int, set when
 *                a peer does not answer within ~8 s (the kernel never hangs)
 *   cur_out/prev_out (optional): prev_out[0] = cur_out[0]; cur_out[0] = sum
 * ---------------------------------------------------------------------- */
int64_t b2s_board_bytes(void);
int b2s_allreduce_board(b2s_dtype vt, void* inout, void* const* boards, int rank, int nranks,
                        int channel, void* seq_counters, void* cur_out, void* prev_out, void* err,
                        b2s_stream_t stream);
/* The same exchange folded into the final reduction of the producing kernel (one launch less per
 * exchange): b2s_cg_update whose r.r, and b2s_spmv_csr_dot whose w.y, come out summed over the ranks. */
int b2s_cg_update_allreduce(b2s_dtype vt, int64_t n, void* x, void* r, const void* p, const void* q,
                            const void* rho, const void* pq, void* rr_out, void* partials,
                            void* const* boards, int rank, int nranks, int channel, void* seq_counters,
                            void* cur_out, void* prev_out, void* err, b2s_stream_t stream);
int b2s_spmv_csr_dot_allreduce(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                               const int64_t* indptr, const void* indices, const void* data,
                               const void* x, void* y, const void* w, const b2s_spmv_plan* plan,
                               void* dot_out, void* const* boards, int rank, int nranks, int channel,
                               void* seq_counters, void* err, b2s_stream_t stream);

/* ------------------------------------------------------------------------
 * CSR x CSR SpGEMM  C = A B.   replaces SpGEMMCSRxCSRxCSRGPU
 *   src/sparse/array/csr/spgemm_csr_csr_csr.cu:64-487 (cuSPARSE SpGEMM) and the
 *   two-task CPU shape (NNZ task + numeric task, csr.py:687-744,
 *   spgemm_csr_csr_csr.cc:62-87,134-158).
 *
 * Two phases because C is caller-allocated:
 *   symbolic: row_nnz → c_indptr[nrowsA+1] (exclusive scan, c_indptr[nrowsA]=nnz(C)),
 *             also returns nnz(C) and the number of intermediate products on the host
 *             (synchronises the stream);
 *   numeric : fills c_indices (sorted within each row, like cuSPARSE) and c_data.
 * A block of rows of A may be passed (row-block partition); B is whole.
 * Reproducibility: the structure (c_indptr, c_indices) is deterministic; the VALUES are accumulated
 * with floating-point atomics (hash tables in shared memory, dense accumulators in HBM), so their
 * summation order — and the last bits of c_data — may differ from run to run (SpMV and the CG /
 * GMRES kernels have no such atomics and are bit-reproducible).
 * ---------------------------------------------------------------------- */
int64_t b2s_spgemm_workspace_bytes(int64_t nrowsA, int64_t nnzA, int64_t ncolsB);

int b2s_spgemm_symbolic(b2s_itype it, int64_t nrowsA, int64_t ncolsA, int64_t ncolsB,
                        const int64_t* a_indptr, const void* a_indices, int64_t nnzA,
                        const int64_t* b_indptr, const void* b_indices, int64_t nnzB,
                        int64_t* c_indptr, void* workspace, int64_t workspace_bytes,
                        int64_t* out_nnzC, int64_t* out_products, b2s_stream_t stream);

int b2s_spgemm_numeric(b2s_dtype vt, b2s_itype it, int64_t nrowsA, int64_t ncolsA,
                       int64_t ncolsB, const int64_t* a_indptr, const void* a_indices,
                       const void* a_data, int64_t nnzA, const int64_t* b_indptr,
                       const void* b_indices, const void* b_data, int64_t nnzB,
                       const int64_t* c_indptr, void* c_indices, void* c_data,
                       void* workspace, int64_t workspace_bytes, b2s_stream_t stream);

/* ------------------------------------------------------------------------
 * Small CSR helpers on the path's edges (SURVEY §8f "next" rows).
 * ---------------------------------------------------------------------- */
/* GetCSRDiagonal: src/sparse/array/csr/get_diagonal.cu:25-44 */
int b2s_csr_diagonal(b2s_dtype vt, b2s_itype it, int64_t nrows, const int64_t* indptr,
                     const void* indices, const void* data, void* diag, b2s_stream_t stream);
/* ExpandPosToCoordinates: src/sparse/array/conv/pos_to_coordinates_template.inl:46-112
 * rows_out[j] = i for indptr[i] <= j < indptr[i+1] (int64) */
int b2s_csr_expand_rows(int64_t nrows, int64_t nnz, const int64_t* indptr, int64_t* rows_out,
                        b2s_stream_t stream);
/* index width conversion (reference `cast` kernels, util/cusparse_utils.h:260-268) */
int b2s_cast_i64_to_i32(int64_t n, const int64_t* src, int32_t* dst, b2s_stream_t stream);
int b2s_cast_i32_to_i64(int64_t n, const int32_t* src, int64_t* dst, b2s_stream_t stream);
/* CSRToDense (csr_to_dense.cu:25-47): out is row-major nrows x ncols, pre-zeroed by callee */
int b2s_csr_to_dense(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols,
                     const int64_t* indptr, const void* indices, const void* data, void* out,
                     b2s_stream_t stream);


/* ------------------------------------------------------------------------
 * Device-side constructors (SURVEY §8 row f4) and the random generator north_star names.
 * Two-pass shape like the reference's count + fill tasks: the count pass writes per-row counts
 * into indptr[1..nrows] (pass `indptr + 1`), b2s_scan_i64 turns them into indptr, the caller
 * reads nnz = indptr[nrows], allocates indices/data and runs the fill pass.
 * ---------------------------------------------------------------------- */
int64_t b2s_scan_workspace_bytes(int64_t n);
/* indptr[0] = 0, indptr[i+1] = counts[0] + .. + counts[i], counts = indptr[1..n] on entry */
int b2s_scan_i64(int64_t n, int64_t* indptr, void* workspace, int64_t workspace_bytes,
                 b2s_stream_t stream);
/* DenseToCSRNNZ / DenseToCSR: src/sparse/array/conv/dense_to_csr.cu:25-43,128-149 (`!= 0` test,
 * CPU loops dense_to_csr.cc:32-40,55-64).  dense is row-major with leading dimension ld. */
int b2s_dense_to_csr_count(b2s_dtype vt, int64_t nrows, int64_t ncols, int64_t ld,
                           const void* dense, int64_t* row_nnz, b2s_stream_t stream);
int b2s_dense_to_csr_fill(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t ld,
                          const void* dense, const int64_t* indptr, void* indices, void* data,
                          b2s_stream_t stream);
/* dia_array.tocsr: legate_sparse/dia.py:159-190 (cupynumeric ops upstream).  data[d*ld + j] is
 * A[j - offsets[d], j] for j < width; `order` lists the diagonals by ascending offset (columns
 * come out sorted); explicit zeros are dropped (dia.py:171). */
int b2s_dia_to_csr_count(b2s_dtype vt, int64_t nrows, int64_t ncols, int ndiag, int64_t width,
                         int64_t ld, const void* data, const int64_t* offsets, const int* order,
                         int64_t* row_nnz, b2s_stream_t stream);
int b2s_dia_to_csr_fill(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int ndiag,
                        int64_t width, int64_t ld, const void* data, const int64_t* offsets,
                        const int* order, const int64_t* indptr, void* indices, void* out_data,
                        b2s_stream_t stream);
/* legate_sparse.random (no upstream counterpart: the reference's tests densify cupynumeric
 * random arrays, tests/integration/utils/sample.py:21-45).  Counter-based: rows [r0, r1) of an
 * m x n matrix with exactly nnz_total entries, k_i = nnz_total/m (+1 for nnz_total%m rows) per
 * row, the j-th entry of a row in the j-th of k_i equal strata of [0, n) (sorted, distinct),
 * values uniform in [lo, hi).  Entry (i, j) depends only on (seed, i, j). */
int b2s_random_csr_rowptr(int64_t m, int64_t nnz_total, uint64_t seed, int64_t r0, int64_t r1,
                          int64_t* indptr_local, b2s_stream_t stream);
int64_t b2s_random_csr_block_nnz(int64_t m, int64_t nnz_total, uint64_t seed, int64_t r0, int64_t r1);
int b2s_random_csr_fill(b2s_dtype vt, b2s_itype it, int64_t m, int64_t n, int64_t nnz_total,
                        uint64_t seed, int64_t r0, int64_t r1, double lo, double hi, void* indices,
                        void* data, b2s_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200SPARSE_H */
