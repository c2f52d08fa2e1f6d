/*
 * b200krylov.h — C-ABI of the H100-native Krylov inner-loop engine (libb200krylov.so).
 *
 * This is the drop-in boundary behind KrylovKit.jl's `apply` + VectorInterface +
 * `Orthogonalizer`/`OrthonormalBasis` plug-in surface (SURVEY.md §8b).  Every entry
 * point replaces one generic function that KrylovKit dispatches on the vector /
 * operator type; the reference file:line it replaces is cited on each declaration
 * (paths relative to the KrylovKit.jl source tree, v0.10.4).
 *
 * Conventions
 *   - plain C: pointers, sizes, scalars.  No torch / C++ types cross this boundary.
 *   - every call returns `int32_t` status: 0 = ok, <0 = error class (see B2K_E*); the
 *     Julia shim maps them to ArgumentError / DimensionMismatch / ErrorException.
 *     `b2k_last_error(ctx)` gives the message.
 *   - all device work is enqueued on ONE stream owned by the context; calls that
 *     return scalars block until the scalars are in the caller's host buffer
 *     (KrylovKit uses every inner/norm result immediately in host control flow).
 *   - vectors live in device "slabs": column-major n_local x ncols panels.  A vector
 *     handle (`b2k_vec`) is (space << 20 | column).  KrylovKit's OrthonormalBasis (a
 *     Julia Vector of independently allocated vectors, src/orthonormal.jl:26-28) maps
 *     to a list of handles; when the handles are consecutive columns the basis is a
 *     contiguous tall-skinny panel, which is what the fused kernels stream.
 *   - scalars cross the ABI as double regardless of the context dtype.
 *   - one context per process per GPU; multi-GPU = one process per GPU, rows sharded,
 *     coefficient reductions over NCCL inside the calls (b2k_ctx_create_dist).
 */
#ifndef B200KRYLOV_H
#define B200KRYLOV_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2K_ABI_VERSION 1

/* status codes */
#define B2K_OK            0
#define B2K_EINVAL       -1  /* -> ArgumentError   (e.g. zero start vector, lanczos.jl:184) */
#define B2K_EDIM         -2  /* -> DimensionMismatch (orthonormal.jl:93,140,158-161)        */
#define B2K_ECUDA        -3  /* CUDA runtime failure                                        */
#define B2K_ENOMEM       -4  /* slab has no free column / device allocation failed           */
#define B2K_ENCCL        -5  /* multi-GPU transport failure: NCCL, the NVLink peer-window
                                * rendezvous, or the watchdog of an in-kernel wait for another
                                * rank (B2K_PEER_TIMEOUT_S, default 120 s): a peer died or left
                                * the SPMD call order; destroy the context                  */
#define B2K_ENOTSUP      -6  /* combination not supported by this build                      */

/* dtypes (real only; KrylovKit also supports complex — out of scope, SURVEY App. A.12) */
#define B2K_F64 0
#define B2K_F32 1

/* Orthogonalizer tags — src/algorithms.jl:17-80 */
#define B2K_CGS   0  /* ClassicalGramSchmidt    */
#define B2K_MGS   1  /* ModifiedGramSchmidt     */
#define B2K_CGS2  2  /* ClassicalGramSchmidt2   */
#define B2K_MGS2  3  /* ModifiedGramSchmidt2 (KrylovDefaults.orth, algorithms.jl:558) */
#define B2K_CGSIR 4  /* ClassicalGramSchmidtIR(eta) */
#define B2K_MGSIR 5  /* ModifiedGramSchmidtIR(eta)  */
/* Engine-specific, FLAGGED (not a KrylovKit orthogonalizer): ModifiedGramSchmidt2 with every sweep over the whole
 * basis applied as ONE classical block (projection coefficients of a sweep all taken from the same vector)
 * instead of k sequential modified steps.  In the Lanczos recurrence (lanczos.jl:325-338) the first, two-vector
 * part stays exactly the reference's (w -= beta v_prev; alpha = <v, w>; w -= alpha v); only the second sweep over
 * all of V is blocked.  Same O(eps) orthogonality (both are "twice is enough"), coefficients differ at rounding
 * level.  Runs at the speed of ClassicalGramSchmidt2. */
#define B2K_MGS2B 6

typedef struct b2k_ctx b2k_ctx;   /* opaque: device, stream, slabs, scratch, NCCL comm */
typedef struct b2k_op  b2k_op;    /* opaque: CSR / dense operator resident in HBM        */
typedef int32_t b2k_vec;          /* (space << 20) | column                               */

#define B2K_VEC(space, col) ((b2k_vec)(((space) << 20) | (col)))
#define B2K_VEC_SPACE(v)    ((int32_t)((v) >> 20))
#define B2K_VEC_COL(v)      ((int32_t)((v) & 0xFFFFF))

/* ------------------------------------------------------------------ context ---- */

int32_t b2k_abi_version(void);
const char* b2k_last_error(const b2k_ctx* ctx);   /* ctx may be NULL: last create error */

/* Single-GPU context.  Creates space 0: an n_local x ncols slab of `dtype`. */
int32_t b2k_ctx_create(b2k_ctx** out, int32_t device, int64_t n_local, int32_t ncols,
                       int32_t dtype);
/* Row-sharded context: this process owns rows [row_offset, row_offset + n_local) of
 * n_global.  `nccl_uid` = the 128-byte ncclUniqueId obtained on rank 0
 * (b2k_nccl_unique_id) and broadcast by the host.  All inner products / norms /
 * projection coefficients are summed over ranks inside the calls (SURVEY §8e). */
int32_t b2k_ctx_create_dist(b2k_ctx** out, int32_t device, int64_t n_local, int32_t ncols,
                            int32_t dtype, int32_t rank, int32_t nranks,
                            const void* nccl_uid, int64_t n_global, int64_t row_offset);
int32_t b2k_nccl_unique_id(void* uid128);
int32_t b2k_ctx_destroy(b2k_ctx* ctx);
/* Additional vector space (e.g. the short right space of GKL, gkl.jl:31-38).
 * `sharded` = 0 means the space is replicated on every rank (no reduction). */
int32_t b2k_space_create(b2k_ctx* ctx, int64_t n_local, int32_t ncols, int32_t sharded,
                         int32_t* space_out);
int32_t b2k_ctx_sync(b2k_ctx* ctx);
/* number of kernels this library launched on the context since creation */
int64_t b2k_ctx_launch_count(const b2k_ctx* ctx);
/* raw CUDA stream (cudaStream_t) for event timing by the caller */
void*   b2k_ctx_stream(b2k_ctx* ctx);

/* Instrumentation (not part of the KrylovKit contract): per-kernel-class device timing with
 * CUDA events on the context stream.  class 0 = CSR SpMV, 1 = fused Gram-Schmidt sweep,
 * 2 = basis transform, 3 = project, 4 = unproject.  `bytes` = algorithmic bytes
 * (SURVEY §8d figures) summed over the recorded launches, `ms` their summed duration. */
int32_t b2k_prof_enable(b2k_ctx* ctx, int32_t on);
int32_t b2k_prof_reset(b2k_ctx* ctx);
int32_t b2k_prof_read(b2k_ctx* ctx, int32_t cls, int64_t* count, double* ms, double* bytes);
/* CUDA-event stopwatch on the context stream (start synchronises the stream first). */
int32_t b2k_timer_start(b2k_ctx* ctx);
int32_t b2k_timer_stop(b2k_ctx* ctx, double* ms);
/* page-locked host memory for fast uploads / downloads, and a whole-device sync */
int32_t b2k_pinned_alloc(size_t bytes, void** out);
int32_t b2k_pinned_free(void* p);
int32_t b2k_device_sync(void);
/* Device memory is drawn from the CUDA stream-ordered pool and kept for reuse (context and
 * operator creation become O(us) after first use); this returns the cached memory. */
int32_t b2k_cache_release(void);

/* ------------------------------------------------- vectors (VectorInterface) ---- */
/* zerovector / similar: src/innerproductvec.jl:82-137 is the reference's own list of
 * what a vector type must provide. */
int32_t b2k_vec_alloc(b2k_ctx* ctx, int32_t space, b2k_vec* out);
int32_t b2k_vec_alloc_range(b2k_ctx* ctx, int32_t space, int32_t count, b2k_vec* first);
int32_t b2k_vec_free(b2k_ctx* ctx, b2k_vec v);
int32_t b2k_vec_upload(b2k_ctx* ctx, b2k_vec v, const void* host);   /* host: n_local elems of dtype */
int32_t b2k_vec_download(b2k_ctx* ctx, b2k_vec v, void* host);
int32_t b2k_vec_copy(b2k_ctx* ctx, b2k_vec dst, b2k_vec src);         /* scale(v, One()) / copy */
int32_t b2k_vec_zero(b2k_ctx* ctx, b2k_vec v);                        /* zerovector!!          */
/* deterministic start vector: x[i] = (splitmix64(seed + gi) >> 11) * 2^-53, gi = global row */
int32_t b2k_vec_fill_splitmix(b2k_ctx* ctx, b2k_vec v, uint64_t seed);
int32_t b2k_vec_fill(b2k_ctx* ctx, b2k_vec v, double value);
/* inner(x,y) — VectorInterface.inner; call sites orthonormal.jl:99-112,418,461-486 */
int32_t b2k_vec_inner(b2k_ctx* ctx, b2k_vec x, b2k_vec y, double* out);
/* norm(x) — lanczos.jl:183,197,199,204 … */
int32_t b2k_vec_norm(b2k_ctx* ctx, b2k_vec x, double* out);
/* add!!(y, x, alpha, beta): y <- beta*y + alpha*x — orthonormal.jl:147,419; lanczos.jl:298-299 */
int32_t b2k_vec_axpby(b2k_ctx* ctx, b2k_vec y, b2k_vec x, double alpha, double beta);
/* scale!!(y, x, alpha): y <- alpha*x (y may alias x) — lanczos.jl:257, arnoldi.jl:209 */
int32_t b2k_vec_scale(b2k_ctx* ctx, b2k_vec y, b2k_vec x, double alpha);
/* y <- y + a1*x1 + a2*x2 in one sweep (the Lanczos 3-term update, lanczos.jl:298-299, 316-317) */
int32_t b2k_vec_axpy2(b2k_ctx* ctx, b2k_vec y, b2k_vec x1, double a1, b2k_vec x2, double a2);

/* ------------------------------------------------------------- operators ---- */
/* apply(A::AbstractMatrix, x) = A*x — src/apply.jl:1.  CSR, 0-based, int32 indices on
 * device.  rowptr/colidx given as int64 or int32 host arrays (idx_bytes = 8 or 4),
 * `index_base` 0 or 1.  vals are of the context dtype.  In a dist context the rows are
 * the local rows and colidx are GLOBAL columns; the halo plan is built here.  The stored
 * order is kept (unsorted and repeated columns included).  Refused, with *out left
 * untouched: idx_bytes not 4 / 8 or index_base not 0 / 1 (B2K_EINVAL); a negative n_rows,
 * n_cols or nnz (B2K_EINVAL); local n_rows or nnz >= 2^31, or on a single GPU n_cols
 * >= 2^31 (B2K_ENOTSUP; a dist context's n_cols is the global column count, which may
 * be larger); n_rows that is not the length of space 0 (dist) or of any space
 * (B2K_EDIM); rowptr[0] != base,
 * rowptr[n_rows] != nnz + base, an entry outside [base, nnz + base] or a decreasing
 * rowptr (B2K_EINVAL); a column outside [base, n_cols + base) (B2K_EINVAL; n_global in
 * a dist context). */
int32_t b2k_op_create_csr(b2k_ctx* ctx, b2k_op** out, int64_t n_rows, int64_t n_cols,
                          int64_t nnz, const void* rowptr, const void* colidx,
                          const void* vals, int32_t idx_bytes, int32_t index_base);
/* Julia SparseMatrixCSC (colptr, rowval, nzval; 1-based Int64) — converted to CSR of A
 * (transposed on the host once: within a row, columns ascending, a repeated entry in
 * colptr order).  rowval / nzval may be longer than nnz; the entries past nnz are never
 * read.  Single-GPU contexts only (B2K_ENOTSUP).  Refused, with *out left untouched:
 * idx_bytes / index_base as for CSR; the sizes and rows as for CSR; colptr[0] != base,
 * colptr[n_cols] != nnz + base or a decreasing colptr (B2K_EINVAL); a row outside
 * [base, n_rows + base) (B2K_EINVAL). */
int32_t b2k_op_create_csc(b2k_ctx* ctx, b2k_op** out, int64_t n_rows, int64_t n_cols,
                          int64_t nnz, const void* colptr, const void* rowval,
                          const void* nzval, int32_t idx_bytes, int32_t index_base);
/* Synthetic stencil operator assembled ON DEVICE as a genuine CSR matrix (benchmarks,
 * SURVEY §8d): grid nx*ny*nz (x fastest), Dirichlet boundaries, coefficients
 * c[0]=centre, c[1]=west(-x), c[2]=east(+x), c[3]=south(-y), c[4]=north(+y),
 * c[5]=down(-z), c[6]=up(+z).  nz = 1 gives the 5-point stencil (down/up ignored).
 * In a dist context rows [row_offset, row_offset+n_local) are assembled. */
int32_t b2k_op_create_stencil(b2k_ctx* ctx, b2k_op** out, int64_t nx, int64_t ny,
                              int64_t nz, const double c[7]);
/* Dense column-major m x n matrix (apply_normal / apply_adjoint, src/apply.jl:14-15).
 * x in `space_in` (length n), y in `space_out` (length m, row-sharded in dist mode). */
/* Matrix-free form of b2k_op_create_stencil (SURVEY §8f-4): nothing is assembled, every apply evaluates the
 * 5-/7-point stencil from the vector itself — 16 n bytes instead of 12 nnz + 20 n per apply — with the products
 * rounded and summed in the assembled operator's order (bit-identical results).  Works with every call that takes
 * a b2k_op (apply, shifted apply, fused dot, the device-chained Lanczos steps, CG / BiCGStab steps); row-sharded
 * contexts must shard by whole grid lines (2-D) / planes (3-D). */
int32_t b2k_op_create_stencil_free(b2k_ctx* ctx, b2k_op** out, int64_t nx, int64_t ny, int64_t nz,
                                   const double c[7]);
int32_t b2k_op_create_dense(b2k_ctx* ctx, b2k_op** out, int64_t m_local, int64_t n,
                            const void* host_colmajor, int64_t ld);
/* Dense m x n with entries uniform(-0.5,0.5) from the counter RNG, generated on device:
 * A[i,j] = (splitmix64(seed + gi + j*m_global) >> 11) * 2^-53 - 0.5 */
int32_t b2k_op_create_dense_splitmix(b2k_ctx* ctx, b2k_op** out, int64_t m_local, int64_t n,
                                     uint64_t seed);
int32_t b2k_op_destroy(b2k_ctx* ctx, b2k_op* op);
int32_t b2k_op_info(const b2k_op* op, int64_t* n_rows, int64_t* n_cols, int64_t* nnz,
                    int32_t* kind);
/* *out = a new CSR operator holding A' (n_cols x n_rows), built on the device from op's arrays (the matrix never
 * goes through the host).  Row c of A' lists its columns in ascending order (a stable sort by column of CSR(A)), so
 * the arrays are those b2k_op_create_csr builds from scipy's sorted A.T.tocsr(), and SpMV with the result gives the
 * same bits.  Any shape; n_cols must be the length of a vector space of the context.  Assembled stencils included:
 * the transpose of stencil(c) is stencil(c) with west/east, south/north and down/up swapped.  Matrix-free stencils,
 * dense operators (use b2k_op_apply_adjoint) and row-sharded contexts: B2K_ENOTSUP.  Destroy with b2k_op_destroy. */
int32_t b2k_op_create_transpose(b2k_ctx* ctx, b2k_op** out, const b2k_op* op);
/* Copy the device CSR back (test support): arrays sized n_rows+1 / nnz / nnz. */
int32_t b2k_op_csr_download(b2k_ctx* ctx, const b2k_op* op, int32_t* rowptr,
                            int32_t* colidx, void* vals);
/* y = A x — apply.jl:1 (never mutates x; y must differ from x) */
int32_t b2k_op_apply(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec y);
/* y = a1*A x + a0*x — apply.jl:4-11 */
int32_t b2k_op_apply_shifted(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec y,
                             double a0, double a1);
/* y = A' x — apply_adjoint, apply.jl:15 (dense: x in space_out, y in space_in;
 * CSR: transposed product) */
int32_t b2k_op_apply_adjoint(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec y);
/* y = A x AND z = A'(A x) from ONE pass over a dense A (SURVEY §8f-4; the flagged one-pass mode of the
 * Golub-Kahan-Lanczos step: gkl.jl:308-323 reads A twice per step, `apply_adjoint` then `apply_normal`; with z
 * the host recovers A'u_{k+1} = (z - sum_j c_j A'u_j) / beta_k without the second pass).  x, z: length n_cols
 * (z must not alias x); y: length n_rows.  Dense operators with at most 1700 (Float32) / 846 (Float64) columns;
 * B2K_ENOTSUP otherwise.  Row-sharded contexts sum z over the ranks. */
int32_t b2k_op_apply_normal_gram(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec y, b2k_vec z);
/* y = A x and dot = <v, y> in the same pass (lanczos.jl:297-298 `w = apply; α = inner(v,w)`) */
int32_t b2k_op_apply_dot(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec y, b2k_vec v,
                         double* dot);

/* Pencil (A, B) of geneigsolve / Golub-Ye (src/eigsolve/golubye.jl): two square operators of one context, of one
 * size.  Keeps references to A and B (destroy the pencil first).  Compares the CSR patterns ON THE DEVICE once
 * (rowptr and colidx equal) to pick the fused path, one pass over both matrices per call; any other pair
 * (different patterns, matrix-free stencil, dense) takes the composed path of b2k_op_apply / b2k_vec_axpby /
 * b2k_vec_inner.  Row-sharded contexts: B2K_ENOTSUP.  Different sizes / non-square: B2K_EDIM.  A == B or an
 * operator of another context: B2K_EINVAL.  The handle is opaque (struct b2k_pencil) and travels as a void*. */
int32_t b2k_pencil_create(b2k_ctx* ctx, void** out, const b2k_op* A, const b2k_op* B);
int32_t b2k_pencil_destroy(b2k_ctx* ctx, void* P);
/* golubyerecurrence's product, golubye.jl:198-199 (+202/211 when vprev >= 0):
 *   bx = B x;  w = add!!(A x, bx, -rho)  i.e. w[r] = fma(-rho, bx[r], (A x)[r]);
 *   if vprev >= 0:  w[r] = fma(-beta, vprev[r], w[r])          (add!!(w, V[end-1], -β), MGS order)
 *   if dot != NULL: *dot = <x, w>  (of the final w)
 * w and bx are bit-identical on both paths to b2k_op_apply with A and B followed by b2k_vec_axpby(w, bx, -rho, 1) and
 * b2k_vec_axpby(w, vprev, -beta, 1).  The dot of the fused path is a deterministic per-CTA sum (as b2k_op_apply_dot)
 * and may differ from b2k_vec_inner in the last bits.  w, bx, x, vprev pairwise distinct; a refused call writes
 * nothing. */
int32_t b2k_pencil_apply(b2k_ctx* ctx, const void* P, b2k_vec x, b2k_vec w, b2k_vec bx, double rho,
                         b2k_vec vprev, double beta, double* dot);
/* genapply and both Rayleigh inner products in one pass (golubye.jl:9-14, 112-114): ax = A x, bx = B x,
 * *xax = <x, ax>, *xbx = <x, bx> (each pointer may be NULL: that dot is not returned).  Same rounding contract as
 * b2k_pencil_apply; x, ax, bx pairwise distinct. */
int32_t b2k_pencil_rayleigh(b2k_ctx* ctx, const void* P, b2k_vec x, b2k_vec ax, b2k_vec bx,
                            double* xax, double* xbx);

/* One conjugate-gradient iteration (SURVEY §8f-2, src/linsolve/cg.jl:62-67) with one host round trip:
 * p <- beta*p + r; q <- (a0 + a1*A) p fused with <p,q>; alpha = rho/<p,q> (on the device);
 * x += alpha*p; r -= alpha*q; returns <p,q> and ||r||.  beta = 0 is the first iteration (p = r). */
int32_t b2k_cg_step(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec r, b2k_vec p, b2k_vec q,
                    double a0, double a1, double beta, double rho, double* pq_out, double* normr_out);

/* Up to `nsteps` CG iterations (every iteration after the first, cg.jl:62-101) enqueued back to back with rho,
 * beta, <p,q>, ||r|| kept on the device — three launches per iteration, ONE host synchronisation per call.  The
 * last kernel of an iteration tests ||r|| < tol like the reference does; launches behind a hit do nothing.
 * pq_out / normr_out: one entry per completed iteration (*steps_done of them); the iteration that reported
 * ||r|| < tol, if any, is the last one.  Same iterates as b2k_cg_step called *steps_done times.  Single GPU. */
int32_t b2k_cg_chain(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec r, b2k_vec p, b2k_vec q,
                     double a0, double a1, double beta, double rho, double tol, int32_t nsteps,
                     double* pq_out, double* normr_out, int32_t* steps_done);

/* One BiCGStab iteration (SURVEY §8f-2, src/linsolve/bicgstab.jl:95-171) as two calls, one host round trip
 * each, with the half-step convergence test (:118) between them on the host as in the reference.
 * half (:97-116): p <- r + beta*(p - omega*v) [first != 0: p <- r]; v <- (a0 + a1*A) p with
 *   sigma = <rs, v> taken from the SpMV pass; alpha = rho/sigma (on the device); s <- r - alpha*v; ||s||.
 * full (:139-150, :98): t <- (a0 + a1*A) s with <t,s> from the SpMV pass; <t,t>; omega = <t,s>/<t,t> (on the
 *   device); x <- x + alpha*p + omega*s; r <- s - omega*t; ||r|| and the next rho = <rs, r>.
 * Every elementwise update uses the rounding sequence of the add!! calls it replaces. */
int32_t b2k_bicgstab_half(b2k_ctx* ctx, const b2k_op* op, b2k_vec rs, b2k_vec r, b2k_vec p, b2k_vec v,
                          b2k_vec s, double a0, double a1, double beta, double omega, double rho,
                          int32_t first, double* sigma_out, double* norms_out);
int32_t b2k_bicgstab_full(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec r, b2k_vec rs, b2k_vec p,
                          b2k_vec s, b2k_vec t, double a0, double a1, double alpha, double* omega_out,
                          double* normr_out, double* rho_out);

/* Up to `nsteps` BiCGStab iterations (every iteration after the first, bicgstab.jl:95-171) enqueued back to back:
 * rho, rho_old, alpha, omega stay on the device, the kernels that produce ||s|| and ||r|| make the reference's two
 * convergence tests (:118, :152) and launches behind a hit do nothing — ONE host synchronisation per call instead
 * of two per iteration.  rho = <rs, r> of the current residual, rho_old / alpha / omega from the previous iteration.
 * rec_out: 8 doubles per completed iteration {rho, sigma, alpha, ||s||, omega, ||r||, next rho, stop code}; stop
 * code 1 = ||s|| < tol (the full step of that iteration has not run), 2 = ||r|| < tol; the stopping iteration is
 * the last of *steps_done.  Same iterates as b2k_bicgstab_half/_full called in turn.  Single GPU, CSR operator. */
int32_t b2k_bicgstab_chain(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec r, b2k_vec rs, b2k_vec p,
                           b2k_vec v, b2k_vec s, b2k_vec t, double a0, double a1, double rho, double rho_old,
                           double alpha, double omega, double tol, int32_t nsteps, double* rec_out,
                           int32_t* steps_done);

/* Up to `nsteps` MINRES iterations (Paige & Saunders 1975: Lanczos + Givens QR, unpreconditioned) for the symmetric
 * system (a0 + a1*A) x = b, enqueued back to back with ONE host synchronisation per call.  Two launches per iteration k:
 *   q <- (a0 + a1*A) v_k with v_k = p_cur/beta_k formed while gathering (p_cur stays unnormalised) and
 *        alpha = <v_k, q> in the epilogue;
 *   one streaming pass (9 vector sweeps): p_{k} = q - alpha v_k - beta_k v_{k-1} over p_prev, beta_{k+1} = ||p_k||, and
 *        the direction / solution update of iteration k-1, d = (v_{k-1} - delta d1 - eps d2)/gamma over d2,
 *        x += phi d (it needs gamma_{k-1}, hence beta_k: one iteration late); the scalar recurrence (delta, gamma,
 *        c, s, phi, phibar) follows in the same kernel, in Float64.
 * A last launch applies the update still pending, so on return x is the iterate of the last recorded iteration.
 * After the call the roles have rotated *steps_done times: if *steps_done is odd, p_prev / p_cur have swapped and
 * so have d1 / d2 (p_cur is again the latest Lanczos vector, d1 the latest direction).
 * state_in / state_out, 8 doubles: {beta_k, 1/beta_k, 1/beta_{k-1}, c, s, deltabar, eps, phibar}; a process
 * started from the residual r (p_cur = r, p_prev = d1 = d2 = 0) has {||r||, 1/||r||, 0, -1, 0, 0, 0, ||r||}.
 * Handing state_out to the next call continues the same process bit for bit.
 * rec_out: 8 doubles per completed iteration {alpha, beta_{k+1}, gamma, phi, |phibar|, stop code, delta, eps};
 * stop code 1 = |phibar| < tol, 2 = gamma == 0 (singular on the Krylov space; that iteration leaves x unchanged and
 * sets d to zero), 3 = beta_{k+1} == 0; the stopping iteration is the last of *steps_done and the launches behind
 * it do nothing.  Vectors are rounded exactly as the scale!! / add!! sequence they replace; alpha and beta are
 * deterministic per-CTA sums (as b2k_op_apply_dot).  nsteps is capped at 511.
 * Single GPU, CSR and stencil operators: B2K_ENOTSUP for dense operators and row-sharded contexts; B2K_EDIM when a
 * length differs; B2K_EINVAL when two vectors are the same.  A refused call writes nothing. */
int32_t b2k_minres_chain(b2k_ctx* ctx, const b2k_op* op, b2k_vec x, b2k_vec p_prev, b2k_vec p_cur, b2k_vec q,
                         b2k_vec d1, b2k_vec d2, double a0, double a1, const double* state_in, double tol,
                         int32_t nsteps, double* rec_out, double* state_out, int32_t* steps_done);

/* Up to `nsteps` (1 <= nsteps <= B2K_MAX_CHAIN - 1) LSMR iterations (src/lssolve/lsmr.jl:61-149, with lambda) for
 * min ||b - A x||^2 + lambda^2 ||x||^2, A a stored CSR matrix (m x n) and At its exact transpose
 * (b2k_op_create_transpose), enqueued back to back with ONE host synchronisation per call.  Per iteration: the A
 * SpMV (gathering v = v~/alpha), one streaming pass over the m-vectors (Ah-bar, r, Ah, u~, beta), the A' SpMV
 * (gathering u = u~/beta; skipped when beta <= tol), one streaming pass over the n-vectors (v into its ring slot,
 * h-bar, x, h, v~ = A'u - beta v); with krylovdim > 1 the reorthogonalisation of v~ against the ring in slot order
 * (ModifiedGramSchmidt / ModifiedGramSchmidt2: the pipelined MGS sweep once / twice; ClassicalGramSchmidt2 /
 * ModifiedGramSchmidt2Blocked: two passes of the cooperative classical sweep) and a norm pass.  The scalar recurrence runs on the device
 * in Float64; the updates it drives are applied one iteration late, and two flush launches apply the last ones.
 * Vectors: x, h, hbar, spare (length n); r, Ah, Ahbar, u, av (length m; av is work space); ring: max(krylovdim, 1)
 * columns of the spare column's space, in slot order.  ON ENTRY AND ON RETURN the vectors are those of the
 * reference loop at the top of iteration iter0 + 1: u normalised, v_{iter0+1} normalised in ring slot
 * iter0 % max(krylovdim, 1), no update pending.  After a call that ran d = *steps_done iterations, iter0 + d is the
 * next call's iter0.  The last iteration's stop code moves v (the reference's `v`): code 2 (beta <= tol) keeps
 * v_k in its slot and leaves u unnormalised; code 3 (alpha <= tol) leaves v unnormalised in the SPARE column and
 * the ring untouched; otherwise v is in slot (iter0 + d) % max(krylovdim, 1).
 * state_in / state_out, 10 doubles: {alpha, beta, alphabar, rho, rhobar, cbar, sbar, theta, zetabar, lambda}; the
 * reference's loop starts from {alpha, beta, alpha, 1, 1, 1, 0, 0, alpha*beta, lambda}.  Handing state_out to the
 * next call continues the same process bit for bit.
 * rec_out: 16 doubles per completed iteration {alpha, beta, rho, rhobar, theta, zeta, |zetabar|, stop code,
 * A' applied (0 / 1), alphabar, cbar, sbar, g, zeta/(rho rhobar), 0, 0}; stop code 1 = |zetabar| <= tol, 2 = beta <=
 * tol, 3 = alpha <= tol, 4 = a non-finite scalar.  A beta / alpha breakdown is completed as the reference completes
 * it, and the chain stops after it; the stopping iteration is the last of *steps_done.
 * Rounding: every vector is rounded exactly like the scale!! / add!! it replaces, given the same scalars; beta and
 * (krylovdim <= 1) alpha are CTA-ordered sums, which may differ from b2k_vec_norm in the last bits, and the three
 * rotations spell hypot out as sqrt(a*a + b*b) with every operation rounded on its own (it overflows once an
 * argument exceeds about 1.3e154).  The chained and the step-by-step loop therefore agree to rounding, not bit for
 * bit.  A refused call writes nothing: B2K_ENOTSUP for a row-sharded context, an operator that is not a stored CSR
 * matrix, krylovdim > 1 with another orthogonalizer, krylovdim > 128 or (CGS2 / MGS2B) more ring columns than the
 * sweep's panel ring holds; B2K_EDIM when At is not A's shape transposed, a vector has the wrong length, or the m-vectors (r, Ah, Ahbar,
 * u, av) or the n-vectors (x, h, hbar, spare, ring) are not columns of one space each;
 * B2K_EINVAL for null pointers, two handles of one vector, nsteps outside 1 .. B2K_MAX_CHAIN - 1 or iter0 < 0. */
int32_t b2k_lsmr_chain(b2k_ctx* ctx, const b2k_op* A, const b2k_op* At, b2k_vec x, b2k_vec h, b2k_vec hbar,
                       b2k_vec r, b2k_vec Ah, b2k_vec Ahbar, b2k_vec u, b2k_vec av, const b2k_vec* ring,
                       int32_t krylovdim, b2k_vec spare, int32_t alg, int32_t iter0, const double* state_in,
                       double tol, int32_t nsteps, double* rec_out, double* state_out, int32_t* steps_done);

/* ---------------------------------------------- basis (OrthonormalBasis) ---- */
/* project!!(y, b, x, alpha, beta, r): h[j] = beta*h[j] + alpha*<b[cols[j]], x>
 * — src/orthonormal.jl:88-118.  h is a HOST vector (orthonormal.jl:374, arnoldi.jl:212). */
int32_t b2k_basis_project(b2k_ctx* ctx, const b2k_vec* cols, int32_t k, b2k_vec x,
                          double alpha, double beta, double* h_host);
/* G[i,j] = <X[i], Y[j]> for i < p, j < q, except the leading p0 x q0 block, which is not written (64 x 64 column
 * blocks wholly inside it are not swept).  G_host column-major, leading dimension ldg >= p.  1 <= p, q <= 256,
 * 0 <= p0 <= p, 0 <= q0 <= q.
 * The cross Gram matrix of two bases (the oblique projection W'V of BiArnoldi, src/factorizations/biarnoldi.jl)
 * in ONE sweep over the rows of both lists for p, q <= 64; larger lists are swept in 64 x 64 column blocks
 * (each block reads its own X and Y columns).  Handles may be in any order, in any spaces of one length, and may
 * repeat between X and Y.  Deterministic: per-thread fma chains in the vector type, then threads and CTAs summed
 * in double in a fixed order (basis.cu).  One host synchronisation.  Bad sizes / null pointers: B2K_EINVAL;
 * columns of different lengths: B2K_EDIM; row-sharded contexts: B2K_ENOTSUP.  A refused call writes nothing. */
int32_t b2k_basis_cross_inner(b2k_ctx* ctx, const b2k_vec* X, int32_t p, const b2k_vec* Y, int32_t q,
                              int32_t p0, int32_t q0, double* G_host, int32_t ldg);
/* unproject!!(y, b, c, alpha, beta, r): y = beta*y + alpha*sum_j b[cols[j]]*c[j]
 * — src/orthonormal.jl:132-196; also Base.:*(b, x) orthonormal.jl:57-60, the GMRES
 * x-update gmres.jl:105-108 and Ritz vectors eigsolve/lanczos.jl:131-133.
 * beta == 0 produces a hard zero before accumulation (orthonormal.jl:141-142). */
int32_t b2k_basis_unproject(b2k_ctx* ctx, b2k_vec y, const b2k_vec* cols, int32_t k,
                            const double* c_host, double alpha, double beta);
/* orthogonalize!!(v, b, h, alg) for every Orthogonalizer tag — src/orthonormal.jl:378-452.
 * Also returns norm(v) after orthogonalisation in *nrm_out (arnoldi.jl:243, orthonormal.jl:524)
 * and, for the IR variants, the number of passes in *passes_out (may be NULL).
 * CGS2 runs as ONE fused three-sweep cooperative kernel on a single GPU. */
int32_t b2k_basis_orthogonalize(b2k_ctx* ctx, b2k_vec v, const b2k_vec* cols, int32_t k,
                                double* h_host, int32_t alg, double eta, double* nrm_out,
                                int32_t* passes_out);
/* orthogonalize!!(v, q, alg) against ONE normalised vector — orthonormal.jl:455-489 */
int32_t b2k_vec_orthogonalize(b2k_ctx* ctx, b2k_vec v, b2k_vec q, int32_t alg, double eta,
                              double* s_out, double* nrm_out);
/* One whole Lanczos expansion step, expand! + lanczosrecurrence —
 * src/factorizations/lanczos.jl:250-272, 295-376 — enqueued without host round trips:
 *   cols[k] <- r / beta_old (the residual's storage becomes basis column k+1, :257);
 *   w = A*cols[k]; three-term recurrence and (re)orthogonalisation per `alg`;
 * on return r holds the new residual, *alpha_out / *beta_out the new coefficients.
 * cols has k+1 entries: the k current basis vectors followed by the handle that will
 * hold the new basis vector (must equal r's handle on entry when in_place != 0; then a
 * fresh column `w` receives the new residual). */
int32_t b2k_lanczos_expand(b2k_ctx* ctx, const b2k_op* op, const b2k_vec* cols, int32_t k,
                           b2k_vec r, b2k_vec w, double beta_old, int32_t alg, double eta,
                           double* alpha_out, double* beta_out);
/* Up to `nsteps` consecutive expand! steps — the inner loop of src/eigsolve/lanczos.jl:33-78
 * while K < krylovdim and beta > tol — without returning to the caller in between.  `cols` has
 * capacity k + nsteps + 1: on entry the k basis handles followed by the residual handle; new
 * residual columns are allocated from the slab.  On return cols[0 .. k + *steps_done) is the basis,
 * *r_out the residual; alphas_out/betas_out hold one entry per step.  Stops early once beta <= tol.
 *
 * HANDLES: the d = *steps_done new basis vectors are cols[k .. k + d).  cols[k] may or may not be the residual
 * handle that was passed in: with ClassicalGramSchmidt2 on a square CSR operator the steps are chained on the
 * device (SpMV with the normalisation r/beta fused into its gather + ONE cooperative Gram-Schmidt launch per
 * step, scalars kept in device records, a single host synchronisation per call) and the normalised vector is
 * written to a column of its own; the library then RELEASES the residual handle passed in (the caller must
 * not free it again).  If cols[k] still equals it on return the caller keeps owning it.  Steps enqueued
 * behind a beta <= tol are skipped on the device, so the returned factorization is the one of the
 * step-by-step loop bit for bit.  A non-zero status can come with *steps_done > 0: those steps are valid. */
int32_t b2k_lanczos_expand_many(b2k_ctx* ctx, const b2k_op* op, b2k_vec* cols, int32_t k,
                                int32_t nsteps, double beta_old, double tol, int32_t alg, double eta,
                                double* alphas_out, double* betas_out, int32_t* steps_done,
                                b2k_vec* r_out);
/* Up to `nsteps` (<= B2K_MAX_CHAIN = 512) consecutive GKL expand! steps — src/factorizations/gkl.jl:246-269 with
 * gklrecurrence :308-323 — for a CSR matrix A (m x n) and its exact transpose At (n x m, b2k_op_create_transpose),
 * chained on the device with ONE host synchronisation per call: three launches per ClassicalGramSchmidt2 step (At
 * SpMV, A SpMV, one cooperative Gram-Schmidt sweep over U), one more with ModifiedGramSchmidt2Blocked (the same sweep
 * over V), and one flush launch per call.  ucols (capacity k + nsteps + 1) holds U in [0, k) and the residual r in
 * [k]; vcols (capacity k + nsteps) holds V in [0, k).  On return the d = *steps_done new vectors are ucols[k .. k+d)
 * and vcols[k .. k+d), *r_out (= ucols[k + d]) is the new residual, alphas_out / betas_out hold one entry per step.
 * HANDLES as b2k_lanczos_expand_many's chained path: the new columns are allocated by the library and the residual
 * handle passed in is RELEASED when d > 0.  Stops early after a step with beta <= tol or a non-finite alpha or beta
 * (its beta is reported as NaN when alpha is not finite); the steps enqueued behind it do nothing.  A non-zero status
 * can come with *steps_done > 0: those steps are valid.  Vectors are rounded exactly like the scale!! / add!! they
 * replace, given the same scalars; alpha and beta are deterministic per-CTA sums (as b2k_op_apply_dot) and may differ
 * from b2k_vec_norm in the last bits.  A refused call writes nothing: B2K_ENOTSUP for alg other than CGS2 / MGS2B, a
 * dense or matrix-free operator, a row-sharded context, or more columns than the sweep's panel ring holds; B2K_EDIM
 * when At's shape is not A's transposed or a column is not in one space of the right length (U, r: m; V: n). */
int32_t b2k_gkl_expand_many(b2k_ctx* ctx, const b2k_op* A, const b2k_op* At, b2k_vec* ucols, b2k_vec* vcols,
                            int32_t k, int32_t nsteps, double beta_old, double tol, int32_t alg,
                            double* alphas_out, double* betas_out, int32_t* steps_done, b2k_vec* r_out);
/* basistransform!(b, U): b[j] <- sum_i b[i]*U[i,j], j < keep — src/orthonormal.jl:291-354.
 * U is host column-major m x keep (ldu).  In place on cols[0..keep) (row-tile resident). */
int32_t b2k_basis_transform(b2k_ctx* ctx, const b2k_vec* cols, int32_t m,
                            const double* U_host, int32_t ldu, int32_t keep);
/* rank1update!(b, y, x, alpha, beta, r): b[cols[i]] = beta*b[cols[i]] + alpha*y*conj(x[i])
 * — src/orthonormal.jl:210-275 */
int32_t b2k_basis_rank1update(b2k_ctx* ctx, const b2k_vec* cols, int32_t k, b2k_vec y,
                              const double* x_host, double alpha, double beta);
/* rmul!(b, G::Givens) — src/dense/givens.jl:12-36: (q1,q2) <- (c*q1 - s*q2, s*q1 + c*q2) */
int32_t b2k_basis_givens(b2k_ctx* ctx, b2k_vec q1, b2k_vec q2, double c, double s);
/* rmul!(b, H::Householder) — src/dense/reflector.jl:143-154:
 * w = sum_i b[cols[i]]*v[i]; b[cols[i]] -= beta*w*conj(v[i]).  `work` is a scratch vector. */
int32_t b2k_basis_householder(b2k_ctx* ctx, const b2k_vec* cols, int32_t k,
                              const double* v_host, double beta, b2k_vec work);

/* Host-only helper (no device work): restore tridiagonal form after a thick restart —
 * src/eigsolve/lanczos.jl:88-105 with the Householder conventions of dense/reflector.jl.
 * D: sorted Ritz values, f: residual weights, U: K x K column-major (updated in place by the
 * reflectors); alphas/betas get the new T entries.  In Julia this loop stays in Julia. */
int32_t b2k_host_lanczos_restart(int32_t K, int32_t keep, const double* D, const double* f,
                                 double* U, int32_t ldu, double* alphas, double* betas);

/* ------------------------------------------------------- block (BlockLanczos) ---- */
/* block_inner(X, Y): M[i,j] = <X[i], Y[j]> — src/factorizations/blocklanczos.jl:43-52.
 * M host column-major p x q. */
int32_t b2k_block_inner(b2k_ctx* ctx, const b2k_vec* X, int32_t p, const b2k_vec* Y,
                        int32_t q, double* M_host);
/* Y[j] <- Y[j] - sum_i X[i]*M[i,j] (blocklanczos.jl:253-260), M host col-major p x q */
int32_t b2k_block_axpy(b2k_ctx* ctx, const b2k_vec* Y, int32_t q, const b2k_vec* X,
                       int32_t p, const double* M_host, int32_t ldm);
/* block_reorthogonalize!(R, V): every R[i] MGS-orthogonalised against V — blocklanczos.jl:277-284 */
int32_t b2k_block_reorthogonalize(b2k_ctx* ctx, const b2k_vec* R, int32_t p,
                                  const b2k_vec* V, int32_t k);
/* block_qr!(block, tol) — blocklanczos.jl:312-353: MGS-QR with rank detection and the
 * DGKS drift pass.  R_host col-major p x p (full, rows of dropped vectors zero),
 * good[i] = 1 if vector i survived, *drift = is_drift. */
int32_t b2k_block_qr(b2k_ctx* ctx, const b2k_vec* X, int32_t p, double tol, double* R_host,
                     int32_t* good, int32_t* drift);

/* apply(A, X::Block) — blocklanczos.jl:38: Y[i] = A X[i], i < p.  A single-GPU CSR operator reads the matrix once
 * per 8 vectors (SpMM); bit-identical to p calls of b2k_op_apply. */
int32_t b2k_op_apply_block(b2k_ctx* ctx, const b2k_op* op, const b2k_vec* X, const b2k_vec* Y, int32_t p);
/* Flagged replacement of block_reorthogonalize! (FLAGGED mode of the host driver, not the reference's
 * arithmetic): block classical Gram-Schmidt of the p <= 8 vectors R against V, `passes` (1 or 2) times, the
 * basis read once per pass for the whole block.  H_host (k x p col-major, may be NULL) = summed coefficients
 * V'R, G_host (p x p, may be NULL) = Gram matrix of the orthogonalised block.  One host synchronisation. */
int32_t b2k_block_orthogonalize(b2k_ctx* ctx, const b2k_vec* R, int32_t p, const b2k_vec* V, int32_t k,
                                int32_t passes, double* H_host, double* G_host);
/* block_qr! (FLAGGED): CholeskyQR2 of p <= 8 vectors, in place.  G0_host (may be NULL) = the Gram
 * matrix X'X if the caller already has it.  R_host (p x p col-major) = the upper-triangular factor with positive
 * diagonal (the factor block_qr!'s modified Gram-Schmidt produces, to rounding).  *ok = 0: the block is
 * numerically rank deficient at the scale block_qr! drops vectors (100 tol) — X is untouched, call b2k_block_qr. */
int32_t b2k_block_cholqr(b2k_ctx* ctx, const b2k_vec* X, int32_t p, double tol, const double* G0_host,
                         double* R_host, int32_t* ok);

#ifdef __cplusplus
}
#endif
#endif /* B200KRYLOV_H */
