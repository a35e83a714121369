// slu_solve.cu -- triangular solves on the device-resident factors (SURVEY 8f row N2: the consumer of pdgstrf3d).
//
// The reference solves with pdgstrs3d (SRC/double/pdgstrs3d.c:6604): per supernode a dense triangular solve with the
// diagonal block and a GEMV-like update of the dependent rows, messages along the process grid, and along Z the
// ancestor contributions reduced pairwise / the ancestor solution broadcast back (dbroadcastAncestor3d,
// pd3dcomm.c:1145).  Here the factors never leave HBM: the same level batches that drove the factorization drive
//   forward   for every level, bottom-up:   x_k <- L_kk^-1 x_k ;  x[rows below] -= L(below,k) x_k     (atomic adds)
//   backward  for every level, top-down:    x_k <- x_k - U(k,:) x[cols] ;  x_k <- U_kk^-1 x_k
// with four small kernels per level; one right-hand side streams L and U once (HBM-bound: 8 bytes per stored entry,
// 16 in doublecomplex).
// x is a device vector in the ordering of the factored matrix (the caller applies the permutations, as pdgssvx3d does
// around pdgstrs3d).  The transposed and conjugate-transposed solves (A^T x = b, A^H x = b) run over the same levels with
// U^T forward and L^T backward (below solve_update_u_kernel); pdgstrs3d itself has no such mode.
//
// Compiled twice, like slu_api.cu: as is for double, and through slu_solve_z.cu with SLU_COMPLEX for doublecomplex
// (pzgstrs3d, SRC/complex16/pzgstrs3d.c).  The element arithmetic goes through the val_t helpers of slu_scalar.cuh;
// complex pivots are applied through the Smith-scaled reciprocal the complex factorization uses, and a complex atomic
// update is two double atomics.  Buffers are sized by MAX_NS_HELD (512 columns in double, 256 in doublecomplex).
#include "slu_device.cuh"
#define SLU_COMMON_HELPERS_ONLY
#include "slu_kernels_common.cuh"
#include "slu_scalar.cuh"

#include <type_traits>

namespace SLU_NS {

constexpr int SOLVE_ROWS = 256;   // rows of an L panel / columns of a U panel per CTA in the update kernels
// __launch_bounds__ minimum of CTAs per SM for solve_diag / solve_update_u: 4 (64 registers) for the batched doublecomplex
// instantiations, which ptxas otherwise compiles with a spill; 0 (no minimum) for every other one, which compile as before
template <class LU>
constexpr int SOLVE_MIN_CTAS = (VAL_DOUBLES == 2 && std::is_same<LU, BatchedLU>::value) ? 4 : 0;

// x_k <- L_kk^-1 x_k (unit lower) or U_kk^-1 x_k (upper, non-unit): one CTA per supernode, column sweep in shared
// memory.  16-column blocks: warp 0 finishes the block's 16 unknowns with shuffles, then all threads apply them.
template <bool UPPER, class LU>
__global__ void __launch_bounds__(256, SOLVE_MIN_CTAS<LU>) solve_diag_kernel(LU dd, const int32_t *nodes, val_t *x, int n, int nrhs)
{
    __shared__ val_t xs[MAX_NS_HELD];
    const DeviceLU &d = member_view(dd);
    x = member_ptr(dd, x, (uint32_t)(n * nrhs));   // the host keeps n * nrhs < 2^31
    const NodeDesc nd = d.nodes[nodes[blockIdx.x]];
    const int ns = nd.ns, lda = nd.nsupr, tid = threadIdx.x;
    const val_t *A = d.val + nd.lval;
    for (int rhs = 0; rhs < nrhs; ++rhs) {
        val_t *xk = x + (size_t)rhs * n + nd.fsupc;
        for (int r = tid; r < ns; r += 256) xs[r] = xk[r];
        __syncthreads();
        if (!UPPER) {
            for (int c0 = 0; c0 < ns; c0 += 16) {
                const int cb = min(16, ns - c0);
                if (tid < 32) {   // the 16 x 16 unit-lower block, lane r owns unknown c0 + r
                    val_t v = (tid < cb) ? xs[c0 + tid] : vzero();
                    for (int c = 0; c < cb; ++c) {
                        const val_t xc = vshfl(0xffffffffu, v, c);
                        if (tid > c && tid < cb) vsubmul(v, A[(size_t)(c0 + c) * lda + c0 + tid], xc);
                    }
                    if (tid < cb) xs[c0 + tid] = v;
                }
                __syncthreads();
                for (int r = c0 + cb + tid; r < ns; r += 256) {
                    val_t acc = vzero();
                    for (int c = 0; c < cb; ++c) vaddmul(acc, A[(size_t)(c0 + c) * lda + r], xs[c0 + c]);
                    xs[r] = vsub(xs[r], acc);
                }
                __syncthreads();
            }
        } else {
            for (int c1 = ns; c1 > 0; c1 -= 16) {
                const int c0 = max(0, c1 - 16), cb = c1 - c0;
                if (tid < 32) {   // upper block, solved from its last unknown up
                    val_t v = (tid < cb) ? xs[c0 + tid] : vzero();
                    for (int c = cb - 1; c >= 0; --c) {
                        const val_t piv = A[(size_t)(c0 + c) * lda + c0 + c];
                        val_t xc = vshfl(0xffffffffu, v, c);
                        xc = vdiv(xc, piv);
                        if (tid == c) v = xc;
                        if (tid < c) vsubmul(v, A[(size_t)(c0 + c) * lda + c0 + tid], xc);
                    }
                    if (tid < cb) xs[c0 + tid] = v;
                }
                __syncthreads();
                for (int r = tid; r < c0; r += 256) {
                    val_t acc = vzero();
                    for (int c = 0; c < cb; ++c) vaddmul(acc, A[(size_t)(c0 + c) * lda + r], xs[c0 + c]);
                    xs[r] = vsub(xs[r], acc);
                }
                __syncthreads();
            }
        }
        for (int r = tid; r < ns; r += 256) xk[r] = xs[r];
        __syncthreads();
    }
}

// x[rows below] -= L(below, k) x_k: CTA = 256 rows of one panel, thread = row (coalesced down the columns)
template <class LU>
__global__ void __launch_bounds__(SOLVE_ROWS) solve_update_l_kernel(LU dd, Batch b, val_t *x, int n, int nrhs)
{
    __shared__ val_t xs[MAX_NS_HELD];
    const DeviceLU &d = member_view(dd);
    x = member_ptr(dd, x, (uint32_t)(n * nrhs));   // the host keeps n * nrhs < 2^31
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const NodeDesc nd = d.nodes[b.nodes[slot]];
    const int i = (int)(blockIdx.x - b.prefix[slot]) * SOLVE_ROWS + threadIdx.x;
    const int ns = nd.ns, lda = nd.nsupr;
    const val_t *L = d.val + nd.lval + ns;
    const int row = i < nd.m ? d.lrows[nd.lrow + ns + i] : 0;
    for (int rhs = 0; rhs < nrhs; ++rhs) {
        __syncthreads();
        for (int c = threadIdx.x; c < ns; c += SOLVE_ROWS) xs[c] = x[(size_t)rhs * n + nd.fsupc + c];
        __syncthreads();
        if (i < nd.m) {
            val_t acc = vzero();
#pragma unroll 8
            for (int c = 0; c < ns; ++c) vaddmul(acc, L[(size_t)c * lda + i], xs[c]);
            vatomic_sub(x + (size_t)rhs * n + row, acc);
        }
    }
}

// x_k -= U(k, cols) x[cols]: CTA = 256 packed columns of one U panel; warp w sweeps columns w, w+8, ..., lanes over rows
template <class LU>
__global__ void __launch_bounds__(256, SOLVE_MIN_CTAS<LU>) solve_update_u_kernel(LU dd, Batch b, val_t *x, int n, int nrhs)
{
    __shared__ val_t part[8][MAX_NS_HELD];
    const DeviceLU &d = member_view(dd);
    x = member_ptr(dd, x, (uint32_t)(n * nrhs));   // the host keeps n * nrhs < 2^31
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const NodeDesc nd = d.nodes[b.nodes[slot]];
    const int j0 = (int)(blockIdx.x - b.prefix[slot]) * SOLVE_ROWS, j1 = min(nd.ncols, j0 + SOLVE_ROWS);
    const int ns = nd.ns, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const val_t *U = d.val + nd.uval;
    const int32_t *cols = d.ucols + nd.ucol;
    for (int rhs = 0; rhs < nrhs; ++rhs) {
        val_t acc[MAX_NS_HELD / 32];
#pragma unroll
        for (int t = 0; t < MAX_NS_HELD / 32; ++t) acc[t] = vzero();
        for (int j = j0 + warp; j < j1; j += 8) {
            const val_t xj = x[(size_t)rhs * n + cols[j]];
            const val_t *col = U + (size_t)j * ns;
#pragma unroll
            for (int t = 0; t < MAX_NS_HELD / 32; ++t) {
                const int r = t * 32 + lane;
                if (r < ns) vaddmul(acc[t], col[r], xj);
            }
        }
#pragma unroll
        for (int t = 0; t < MAX_NS_HELD / 32; ++t) {
            const int r = t * 32 + lane;
            if (r < ns) part[warp][r] = acc[t];
        }
        __syncthreads();
        for (int r = threadIdx.x; r < ns; r += 256) {
            val_t sum = vzero();
#pragma unroll
            for (int w = 0; w < 8; ++w) sum = vadd(sum, part[w][r]);
            vatomic_sub(x + (size_t)rhs * n + nd.fsupc + r, sum);
        }
        __syncthreads();
    }
}

// ---- transposed solves: A^T x = b as U^T y = b, then L^T x = y, over the same level plan and in the same directions as
// the plain solve, because both the targets of the forward scatter (the packed U columns) and the sources of the backward
// gather (the L rows) are ancestor supernodes:
//   forward   for every level, bottom-up:   y_k <- U_kk^-T x_k ;  x[ucols(k)] -= U(k,:)^T y_k       (atomic adds)
//   backward  for every level, top-down:    x_k <- x_k - L(below,k)^T x[rows below] ;  x_k <- L_kk^-T x_k
// CONJ (doublecomplex only) reads every factor entry conjugated, the pivots included: A^H = U^H L^H.  The zero padding
// above the skyline segments of a packed U column adds nothing to its dot product.

__device__ __forceinline__ val_t warp_sum(val_t v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = vadd(v, vshfl(0xffffffffu, v, (threadIdx.x & 31) ^ o));
    return v;
}

// y_k <- U_kk^-T x_k (forward: lower, non-unit) or x_k <- L_kk^-T x_k (backward: upper, unit): one CTA per supernode.
// Row r of the transposed triangle is column r of the diagonal block, contiguous in memory.  Per 16-unknown block: one
// warp per unknown gathers the unknowns solved before it along that column, and the 16 x 16 block is staged in shared
// memory (blk[i][j] = block(c0 + i, c0 + j)) so that warp 0 solves it with shuffles, lane r owning unknown c0 + r.  The
// forward pass multiplies by the pivots' reciprocals, taken in parallel while the block is staged.  In doublecomplex a
// minimum of 4 CTAs per SM (64 registers): without it ptxas spills around the division of the unbatched forward kernel.
template <bool BACKWARD, bool CONJ, class LU>
__global__ void __launch_bounds__(256, VAL_DOUBLES == 2 ? 4 : 0) solve_diag_trans_kernel(LU dd, const int32_t *nodes, val_t *x, int n, int nrhs)
{
    __shared__ val_t xs[MAX_NS_HELD];
    __shared__ val_t blk[16][17], rpiv[16];
    const DeviceLU &d = member_view(dd);
    x = member_ptr(dd, x, (uint32_t)(n * nrhs));   // the host keeps n * nrhs < 2^31
    const NodeDesc nd = d.nodes[nodes[blockIdx.x]];
    const int ns = nd.ns, lda = nd.nsupr, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const val_t *A = d.val + nd.lval;
    for (int rhs = 0; rhs < nrhs; ++rhs) {
        val_t *xk = x + (size_t)rhs * n + nd.fsupc;
        for (int r = tid; r < ns; r += 256) xs[r] = xk[r];
        __syncthreads();
        for (int b = 0; b < ns; b += 16) {
            const int c0 = BACKWARD ? max(0, ns - b - 16) : b, cb = BACKWARD ? ns - b - c0 : min(16, ns - b);
            const int lo = BACKWARD ? c0 + cb : 0, hi = BACKWARD ? ns : c0;   // the unknowns solved so far
            for (int rr = warp; rr < cb; rr += 8) {
                const val_t *col = A + (size_t)(c0 + rr) * lda;
                val_t acc = vzero();
                for (int c = lo + lane; c < hi; c += 32) vaddmul(acc, vconj<CONJ>(col[c]), xs[c]);
                acc = warp_sum(acc);
                if (lane == 0) xs[c0 + rr] = vsub(xs[c0 + rr], acc);
            }
            {
                const int i = tid & 15, j = tid >> 4;
                blk[i][j] = (i < cb && j < cb) ? vconj<CONJ>(A[(size_t)(c0 + j) * lda + c0 + i]) : vzero();
                if (!BACKWARD && tid < cb) rpiv[tid] = vrecip(vconj<CONJ>(A[(size_t)(c0 + tid) * lda + c0 + tid]));
            }
            __syncthreads();
            if (tid < 32) {   // transposed triangle: entry (r, c) = blk[c][r]
                val_t v = (tid < cb) ? xs[c0 + tid] : vzero();
                if (!BACKWARD) {
                    for (int c = 0; c < cb; ++c) {
                        const val_t xc = vmul(vshfl(0xffffffffu, v, c), rpiv[c]);
                        if (tid == c) v = xc;
                        if (tid > c && tid < cb) vsubmul(v, blk[c][tid], xc);
                    }
                } else {
                    for (int c = cb - 1; c > 0; --c) {
                        const val_t xc = vshfl(0xffffffffu, v, c);
                        if (tid < c) vsubmul(v, blk[c][tid], xc);
                    }
                }
                if (tid < cb) xs[c0 + tid] = v;
            }
            __syncthreads();
        }
        for (int r = tid; r < ns; r += 256) xk[r] = xs[r];
        __syncthreads();
    }
}

// x[ucols(k)] -= U(k, :)^T y_k: CTA = 256 packed columns of one U panel; warp w takes columns w, w+8, ..., one dot
// product per column with the lanes along its ns contiguous entries
template <bool CONJ, class LU>
__global__ void __launch_bounds__(256, SOLVE_MIN_CTAS<LU>) solve_scatter_ut_kernel(LU dd, Batch b, val_t *x, int n, int nrhs)
{
    __shared__ val_t ys[MAX_NS_HELD];
    const DeviceLU &d = member_view(dd);
    x = member_ptr(dd, x, (uint32_t)(n * nrhs));   // the host keeps n * nrhs < 2^31
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const NodeDesc nd = d.nodes[b.nodes[slot]];
    const int j0 = (int)(blockIdx.x - b.prefix[slot]) * SOLVE_ROWS, j1 = min(nd.ncols, j0 + SOLVE_ROWS);
    const int ns = nd.ns, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const val_t *U = d.val + nd.uval;
    const int32_t *cols = d.ucols + nd.ucol;
    for (int rhs = 0; rhs < nrhs; ++rhs) {
        __syncthreads();
        for (int r = threadIdx.x; r < ns; r += 256) ys[r] = x[(size_t)rhs * n + nd.fsupc + r];
        __syncthreads();
        for (int j = j0 + warp; j < j1; j += 8) {
            const val_t *col = U + (size_t)j * ns;
            val_t acc = vzero();
            for (int r = lane; r < ns; r += 32) vaddmul(acc, vconj<CONJ>(col[r]), ys[r]);
            acc = warp_sum(acc);
            if (lane == 0) vatomic_sub(x + (size_t)rhs * n + cols[j], acc);
        }
    }
}

// x_k -= L(below, k)^T x[rows below]: CTA = 256 rows of one L panel, warp w = rows 32w ... 32w+31 of them, lane = row
// (coalesced down each column); a warp sum per column into part[w][c], then the CTA's sums go to x_k with atomic adds
template <bool CONJ, class LU>
__global__ void __launch_bounds__(SOLVE_ROWS, SOLVE_MIN_CTAS<LU>) solve_gather_lt_kernel(LU dd, Batch b, val_t *x, int n, int nrhs)
{
    __shared__ val_t part[SOLVE_ROWS / 32][MAX_NS_HELD];
    const DeviceLU &d = member_view(dd);
    x = member_ptr(dd, x, (uint32_t)(n * nrhs));   // the host keeps n * nrhs < 2^31
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const NodeDesc nd = d.nodes[b.nodes[slot]];
    const int i0 = (int)(blockIdx.x - b.prefix[slot]) * SOLVE_ROWS, i = i0 + threadIdx.x;
    const int ns = nd.ns, lda = nd.nsupr, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nwarps = min(SOLVE_ROWS / 32, (nd.m - i0 + 31) / 32);   // warps with at least one row of the panel
    const val_t *L = d.val + nd.lval + ns;
    const int row = i < nd.m ? d.lrows[nd.lrow + ns + i] : 0;
    for (int rhs = 0; rhs < nrhs; ++rhs) {
        if (warp < nwarps) {
            const val_t xr = i < nd.m ? x[(size_t)rhs * n + row] : vzero();
            for (int c = 0; c < ns; ++c) {
                const val_t v = warp_sum(i < nd.m ? vmul(vconj<CONJ>(L[(size_t)c * lda + i]), xr) : vzero());
                if (lane == 0) part[warp][c] = v;
            }
        }
        __syncthreads();
        for (int c = threadIdx.x; c < ns; c += SOLVE_ROWS) {
            val_t sum = part[0][c];
            for (int w = 1; w < nwarps; ++w) sum = vadd(sum, part[w][c]);
            vatomic_sub(x + (size_t)rhs * n + nd.fsupc + c, sum);
        }
        __syncthreads();
    }
}

// keep / zero the entries of the supernodes in a node list (multi-GPU ownership masks)
__global__ void solve_mask_kernel(DeviceLU d, const int32_t *nodes, int count, val_t *x, int n, int nrhs, const val_t *src)
{
    for (int t = blockIdx.x; t < count; t += gridDim.x) {
        const NodeDesc nd = d.nodes[nodes[t]];
        for (int rhs = 0; rhs < nrhs; ++rhs)
            for (int r = threadIdx.x; r < nd.ns; r += blockDim.x)
                x[(size_t)rhs * n + nd.fsupc + r] = src ? src[(size_t)rhs * n + nd.fsupc + r] : vzero();
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Device-side distribution (SURVEY 8f row N1): scatter P A P^T from a CSR copy in HBM straight into the L / U panels
// of the arena -- the job pddistribute3d (SRC/double/pddistribute3d.c:1357) does on the host, without the 8-bytes-per-
// factor-entry host arrays and their H2D.  One thread per row of A; an entry (i, j) of the permuted matrix belongs to
// the L panel of supno(j) if i is at or below that supernode's first row, else to the U panel of supno(i).
// `active[k]` = 0 for panels this rank does not hold or holds as zero-initialised replicated ancestors.
// Batched: member blockIdx.y scatters its own nnz values (aval + member * nnz) into its own arena.
template <class LU>
__global__ void fill_csr_kernel(LU dd, int n, const int32_t *__restrict__ rowptr, const int32_t *__restrict__ colind,
                                const val_t *__restrict__ aval, const int32_t *__restrict__ perm, const int8_t *__restrict__ active,
                                int *err)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const DeviceLU &d = member_view(dd);
    if constexpr (std::is_same<LU, BatchedLU>::value) aval += (int64_t)blockIdx.y * rowptr[n];
    const int pi = perm[r];
    for (int p = rowptr[r]; p < rowptr[r + 1]; ++p) {
        const int pj = perm[colind[p]];
        const int ks = d.supno[pj];
        if (pi >= d.xsup[ks]) {                       // L panel of block column ks (diagonal block included)
            if (!active[ks]) continue;
            const NodeDesc *nd = d.nodes + ks;
            const int32_t *srow = d.lsrow + nd->lrow;
            const int q = lower_bound_i32(srow, nd->nsupr, pi);
            if (q >= nd->nsupr || srow[q] != pi) { atomicAdd(err, 1); continue; }
            d.val[nd->lval + (int64_t)(pj - nd->fsupc) * nd->nsupr + d.lspos[nd->lrow + q]] = aval[p];
        } else {                                      // U panel of block row supno(i)
            const int kr = d.supno[pi];
            if (!active[kr]) continue;
            const NodeDesc *nd = d.nodes + kr;
            const int32_t *uc = d.ucols + nd->ucol;
            const int q = lower_bound_i32(uc, nd->ncols, pj);
            // above the column's skyline start is dense-packed padding, not a slot
            if (q >= nd->ncols || uc[q] != pj || pi < d.ufst[nd->ucol + q]) { atomicAdd(err, 1); continue; }
            d.val[nd->uval + (int64_t)q * nd->ns + (pi - nd->fsupc)] = aval[p];
        }
    }
}

// ---- affine fill (slu_b200_batch_fill_affine) ----
// csr_slot: the arena offset of entry (pi, pj) of the permuted matrix; -1 in a panel `active` leaves out, -2 without a slot.
// The search of fill_csr_kernel, which keeps its own copy: written through this helper, that kernel compiles to other code.
__device__ __forceinline__ int64_t csr_slot(const DeviceLU &d, int pi, int pj, const int8_t *__restrict__ active)
{
    const int ks = d.supno[pj];
    if (pi >= d.xsup[ks]) {                       // L panel of block column ks (diagonal block included)
        if (!active[ks]) return -1;
        const NodeDesc *nd = d.nodes + ks;
        const int32_t *srow = d.lsrow + nd->lrow;
        const int q = lower_bound_i32(srow, nd->nsupr, pi);
        if (q >= nd->nsupr || srow[q] != pi) return -2;
        return nd->lval + (int64_t)(pj - nd->fsupc) * nd->nsupr + d.lspos[nd->lrow + q];
    }
    const int kr = d.supno[pi];                   // U panel of block row supno(i)
    if (!active[kr]) return -1;
    const NodeDesc *nd = d.nodes + kr;
    const int32_t *uc = d.ucols + nd->ucol;
    const int q = lower_bound_i32(uc, nd->ncols, pj);
    // above the column's skyline start is dense-packed padding, not a slot
    if (q >= nd->ncols || uc[q] != pj || pi < d.ufst[nd->ucol + q]) return -2;
    return nd->uval + (int64_t)q * nd->ns + (pi - nd->fsupc);
}

// dst[p] = csr_slot of entry p (-1 where it has none, counted in *err): one thread per row, as fill_csr_kernel.  A batched
// handle fills every panel, so no entry is left out as inactive.
__global__ void fill_affine_slot_kernel(DeviceLU d, int n, const int32_t *__restrict__ rowptr, const int32_t *__restrict__ colind,
                                        const int32_t *__restrict__ perm, const int8_t *__restrict__ active, int64_t *__restrict__ dst,
                                        int *err)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int pi = perm[r];
    for (int p = rowptr[r]; p < rowptr[r + 1]; ++p) {
        const int64_t o = csr_slot(d, pi, perm[colind[p]], active);
        if (o == -2) atomicAdd(err, 1);
        dst[p] = o < 0 ? -1 : o;
    }
}

// grid (entry tiles, members): thread = one entry of member blockIdx.y, v = c_0 V_0 then v = fma(c_t, V_t, v) for t = 1, 2, ...;
// the member's coefficients are staged in shared memory FA_THREADS at a time, each term is read coalesced, each slot written
// once with a plain store
constexpr int FA_THREADS = 256;
__global__ void __launch_bounds__(FA_THREADS) fill_affine_kernel(BatchedLU dd, int64_t nnz, int nterms, const val_t *__restrict__ terms,
                                                                 const val_t *__restrict__ coef, const int64_t *__restrict__ dst)
{
    __shared__ val_t cs[FA_THREADS];
    const DeviceLU d = member_view(dd);
    coef += (int64_t)blockIdx.y * nterms;
    const int64_t p = (int64_t)blockIdx.x * FA_THREADS + threadIdx.x;
    val_t v = vzero();
    for (int t0 = 0; t0 < nterms; t0 += FA_THREADS) {
        __syncthreads();
        if (t0 + (int)threadIdx.x < nterms) cs[threadIdx.x] = coef[t0 + threadIdx.x];
        __syncthreads();
        if (p >= nnz) continue;
        const int tn = min(FA_THREADS, nterms - t0);
        int t = 0;
        if (t0 == 0) { v = vmul(cs[0], terms[p]); t = 1; }
        for (; t < tn; ++t) v = vfma(cs[t], terms[(int64_t)(t0 + t) * nnz + p], v);
    }
    if (p < nnz) {
        const int64_t o = dst[p];
        if (o >= 0) d.val[o] = v;
    }
}

int launch_fill_affine(const BatchedLU &d, int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm, const int8_t *active,
                       int64_t *dst, int64_t nnz, int nterms, const val_t *terms, const val_t *coef, int *err, cudaStream_t s)
{
    if (n <= 0) return 0;
    fill_affine_slot_kernel<<<(n + 127) / 128, 128, 0, s>>>(d, n, rowptr, colind, perm, active, dst, err);
    if (nnz <= 0) return 1;
    fill_affine_kernel<<<member_grid(d, (unsigned)((nnz + FA_THREADS - 1) / FA_THREADS)), FA_THREADS, 0, s>>>(d, nnz, nterms, terms, coef, dst);
    return 2;
}
// ---- scaled, row-permuted fill (slu_b200_fill_csr_scaled) ----
// M = Pr Dr A Dc with the caller's R, C; its equilibration follows dgsequ_dist / dlaqgs_dist (SRC/double/dgsequ_dist.c,
// dlaqgs_dist.c) with the magnitude of slud_z_abs1 (|re| + |im|) in doublecomplex.  The maxima are order-independent, so
// the atomics on their bit patterns give the same R and C on every run.  Thread = row i of A (row rmap[i] of F), member
// blockIdx.y.
constexpr double EQ_SMLNUM = 2.2250738585072014e-308;           // dmach_dist("S") = DBL_MIN
constexpr double EQ_BIGNUM = 1.0 / EQ_SMLNUM;
constexpr double EQ_SMALL = EQ_SMLNUM / 2.220446049250313e-16;  // dlaqgs: dmach("Safe minimum") / dmach("Precision")
constexpr double EQ_LARGE = 1.0 / EQ_SMALL;
constexpr double EQ_THRESH = 0.1;

__device__ __forceinline__ double eq_abs1(double v) { return fabs(v); }
__device__ __forceinline__ double eq_abs1(double2 v) { return fabs(v.x) + fabs(v.y); }
__device__ __forceinline__ double eq_mod(double v) { return fabs(v); }
__device__ __forceinline__ double eq_mod(double2 v) { return hypot(v.x, v.y); }
__device__ __forceinline__ double vscale_d(double s, double v) { return s * v; }
__device__ __forceinline__ double2 vscale_d(double s, double2 v) { return make_double2(s * v.x, s * v.y); }
__device__ __forceinline__ unsigned long long dbits(double v) { return (unsigned long long)__double_as_longlong(v); }
__device__ __forceinline__ double bitsd(unsigned long long b) { return __longlong_as_double((long long)b); }
// entry p of row i, scaled: (R[i] a) C[j], in that order
__device__ __forceinline__ val_t scaled_entry(const ScaledFill &f, const val_t *aval, const double *R, const double *C, int i, int64_t p)
{
    const double ri = R ? R[i] : 1.0, cj = C ? C[f.colind[p]] : 1.0;
    return vscale_d(cj, vscale_d(ri, aval[p]));
}

// row maxima r_i of |M| (stat rmin / rmax / zrow), then the column maxima of |M_ij| / clamp(r_i) into ccol
__global__ void equil_rows_kernel(ScaledFill f)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
    if (i >= f.n) return;
    const int64_t nnz = f.rowptr[f.n];
    const val_t *aval = f.aval + (int64_t)m * nnz;
    const double *R = f.R_in ? f.R_in + m * f.rc_stride : nullptr, *C = f.C_in ? f.C_in + m * f.rc_stride : nullptr;
    double rm = 0.0;
    for (int64_t p = f.rowptr[i]; p < f.rowptr[i + 1]; ++p) rm = fmax(rm, eq_abs1(scaled_entry(f, aval, R, C, i, p)));
    EquilStat *st = f.st + m;
    atomicMin(&st->rmin, dbits(rm));
    atomicMax(&st->rmax, dbits(rm));
    if (rm == 0.0) atomicMin(&st->zrow, i);
    const double r = 1.0 / fmin(fmax(rm, EQ_SMLNUM), EQ_BIGNUM);
    f.rinv[(int64_t)m * f.n + i] = r;
    unsigned long long *ccol = f.ccol + (int64_t)m * f.n;
    for (int64_t p = f.rowptr[i]; p < f.rowptr[i + 1]; ++p)
        atomicMax(ccol + f.colind[p], dbits(eq_abs1(scaled_entry(f, aval, R, C, i, p)) * r));
}

// thread = column j: stat cmin / cmax / zcol
__global__ void equil_cols_kernel(ScaledFill f)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
    if (j >= f.n) return;
    const unsigned long long c = f.ccol[(int64_t)m * f.n + j];
    EquilStat *st = f.st + m;
    atomicMin(&st->cmin, c);
    atomicMax(&st->cmax, c);
    if (c == 0) atomicMin(&st->zcol, j);
}

// thread = index t: the final R[t] and C[t] of the member.  equil: dgsequ's rowcnd / colcnd / amax and dlaqgs's choice
// (THRESH, SMALL, LARGE), the chosen factors folded into the caller's; the member's out[0..3].  Else a copy (ones for nullptr).
template <bool EQUIL>
__global__ void equil_apply_kernel(ScaledFill f)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
    if (t >= f.n) return;
    const double rin = f.R_in ? f.R_in[m * f.rc_stride + t] : 1.0, cin = f.C_in ? f.C_in[m * f.rc_stride + t] : 1.0;
    const int64_t o = (int64_t)m * f.n + t;
    if (!EQUIL) {
        f.R[o] = rin;
        f.C[o] = cin;
        return;
    }
    const EquilStat st = f.st[m];
    const double amax = bitsd(st.rmax);
    const double rowcnd = fmax(bitsd(st.rmin), EQ_SMLNUM) / fmin(amax, EQ_BIGNUM);
    const double colcnd = fmax(bitsd(st.cmin), EQ_SMLNUM) / fmin(bitsd(st.cmax), EQ_BIGNUM);
    int equed;   // 0 none, 1 rows, 2 columns, 3 both
    if (rowcnd >= EQ_THRESH && amax >= EQ_SMALL && amax <= EQ_LARGE) equed = colcnd >= EQ_THRESH ? 0 : 2;
    else equed = colcnd >= EQ_THRESH ? 1 : 3;
    f.R[o] = (equed & 1) ? rin * f.rinv[o] : rin;
    f.C[o] = (equed & 2) ? cin * (1.0 / fmin(fmax(bitsd(f.ccol[o]), EQ_SMLNUM), EQ_BIGNUM)) : cin;
    if (t == 0) {
        double *out = f.out + (int64_t)m * 6;
        out[0] = rowcnd;
        out[1] = colcnd;
        out[2] = amax;
        out[3] = equed;
    }
}

// the scatter into the zeroed arena, one plain store per slot; the row's sum of |f_ij| in CSR order (fixed) and its max
// go to the member's fnorm / fmax
template <class LU>
__global__ void fill_scaled_kernel(LU dd, ScaledFill f)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
    if (i >= f.n) return;
    const DeviceLU &d = member_view(dd);
    const int64_t nnz = f.rowptr[f.n];
    const val_t *aval = f.aval + (int64_t)m * nnz;
    const double *R = f.R + (int64_t)m * f.n, *C = f.C + (int64_t)m * f.n;
    const int pi = f.rmap[i];
    double sum = 0.0, mx = 0.0;
    for (int64_t p = f.rowptr[i]; p < f.rowptr[i + 1]; ++p) {
        const val_t v = scaled_entry(f, aval, R, C, i, p);
        const double a = eq_mod(v);
        sum += a;
        mx = fmax(mx, a);
        const int64_t o = csr_slot(d, pi, f.perm[f.colind[p]], f.active);
        if (o >= 0) d.val[o] = v;
        else if (o == -2 && m == 0) atomicAdd(f.err, 1);
    }
    atomicMax(&f.st[m].fnorm, dbits(sum));
    atomicMax(&f.st[m].fmax, dbits(mx));
}

template <class LU>
static int launch_fill_scaled_t(const LU &d, const ScaledFill &f, bool equil, cudaStream_t s)
{
    if (f.n <= 0) return 0;
    const dim3 g = member_grid(d, (unsigned)((f.n + 127) / 128));
    if (equil) {
        equil_rows_kernel<<<g, 128, 0, s>>>(f);
        equil_cols_kernel<<<g, 128, 0, s>>>(f);
        equil_apply_kernel<true><<<g, 128, 0, s>>>(f);
    } else {
        equil_apply_kernel<false><<<g, 128, 0, s>>>(f);
    }
    fill_scaled_kernel<LU><<<g, 128, 0, s>>>(d, f);
    return equil ? 4 : 2;
}
int launch_fill_scaled(const DeviceLU &d, const ScaledFill &f, bool equil, cudaStream_t s) { return launch_fill_scaled_t(d, f, equil, s); }
int launch_fill_scaled(const BatchedLU &d, const ScaledFill &f, bool equil, cudaStream_t s) { return launch_fill_scaled_t(d, f, equil, s); }

// thread = entry i of the member blockIdx.y, every right-hand side
template <bool SCATTER>
__global__ void permute_scale_kernel(val_t *__restrict__ dst, const val_t *__restrict__ src, const int32_t *__restrict__ map,
                                     const double *__restrict__ scale, int n, int nrhs)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t base = (int64_t)blockIdx.y * n * nrhs;
    const double sc = scale[(int64_t)blockIdx.y * n + i];
    const int k = map[i];
    for (int r = 0; r < nrhs; ++r) {
        const int64_t c = base + (int64_t)r * n;
        if (SCATTER) dst[c + k] = vscale_d(sc, src[c + i]);
        else dst[c + i] = vscale_d(sc, src[c + k]);
    }
}

int launch_permute_scale(val_t *dst, const val_t *src, const int32_t *map, const double *scale, int n, int nrhs, int members,
                         bool scatter, cudaStream_t s)
{
    if (n <= 0) return 0;
    const dim3 g((unsigned)((n + 255) / 256), (unsigned)members);
    if (scatter) permute_scale_kernel<true><<<g, 256, 0, s>>>(dst, src, map, scale, n, nrhs);
    else permute_scale_kernel<false><<<g, 256, 0, s>>>(dst, src, map, scale, n, nrhs);
    return 1;
}

template <class LU>
static int launch_fill_csr_t(const LU &d, int n, const int32_t *rowptr, const int32_t *colind, const val_t *aval, const int32_t *perm,
                             const int8_t *active, int *err, cudaStream_t s)
{
    fill_csr_kernel<LU><<<member_grid(d, (n + 127) / 128), 128, 0, s>>>(d, n, rowptr, colind, aval, perm, active, err);
    return 1;
}
template <bool CONJ, class LU>
static void launch_solve_trans_c(const LU &d, const int32_t *nodes, const Batch *b, unsigned ctas, bool backward, val_t *x, int n,
                                 int nrhs, cudaStream_t s)
{
    if (!b && backward) solve_diag_trans_kernel<true, CONJ, LU><<<member_grid(d, ctas), 256, 0, s>>>(d, nodes, x, n, nrhs);
    else if (!b) solve_diag_trans_kernel<false, CONJ, LU><<<member_grid(d, ctas), 256, 0, s>>>(d, nodes, x, n, nrhs);
    else if (backward) solve_gather_lt_kernel<CONJ, LU><<<member_grid(d, ctas), SOLVE_ROWS, 0, s>>>(d, *b, x, n, nrhs);
    else solve_scatter_ut_kernel<CONJ, LU><<<member_grid(d, ctas), 256, 0, s>>>(d, *b, x, n, nrhs);
}
// trans 1 / 2: the transposed kernels, conjugating in doublecomplex for 2 (in double 2 is 1)
template <class LU>
static void launch_solve_trans(const LU &d, const int32_t *nodes, const Batch *b, unsigned ctas, bool backward, int trans, val_t *x,
                               int n, int nrhs, cudaStream_t s)
{
    if constexpr (VAL_DOUBLES == 2)
        if (trans == 2) return launch_solve_trans_c<true>(d, nodes, b, ctas, backward, x, n, nrhs, s);
    launch_solve_trans_c<false>(d, nodes, b, ctas, backward, x, n, nrhs, s);
}
template <class LU>
static int launch_solve_diag_t(const LU &d, const int32_t *nodes, int count, bool backward, int trans, val_t *x, int n, int nrhs,
                               cudaStream_t s)
{
    if (count <= 0) return 0;
    if (trans) launch_solve_trans(d, nodes, nullptr, (unsigned)count, backward, trans, x, n, nrhs, s);
    else if (backward) solve_diag_kernel<true, LU><<<member_grid(d, count), 256, 0, s>>>(d, nodes, x, n, nrhs);
    else solve_diag_kernel<false, LU><<<member_grid(d, count), 256, 0, s>>>(d, nodes, x, n, nrhs);
    return 1;
}
template <class LU>
static int launch_solve_update_t(const LU &d, const Batch &b, int64_t ctas, bool backward, int trans, val_t *x, int n, int nrhs,
                                 cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    if (trans) launch_solve_trans(d, b.nodes, &b, (unsigned)ctas, backward, trans, x, n, nrhs, s);
    else if (backward) solve_update_u_kernel<LU><<<member_grid(d, (unsigned)ctas), 256, 0, s>>>(d, b, x, n, nrhs);
    else solve_update_l_kernel<LU><<<member_grid(d, (unsigned)ctas), SOLVE_ROWS, 0, s>>>(d, b, x, n, nrhs);
    return 1;
}
int launch_fill_csr(const DeviceLU &d, int n, const int32_t *rowptr, const int32_t *colind, const val_t *aval, const int32_t *perm,
                    const int8_t *active, int *err, cudaStream_t s)
{
    return launch_fill_csr_t(d, n, rowptr, colind, aval, perm, active, err, s);
}
int launch_solve_diag(const DeviceLU &d, const int32_t *nodes, int count, bool backward, int trans, val_t *x, int n, int nrhs,
                      cudaStream_t s)
{
    return launch_solve_diag_t(d, nodes, count, backward, trans, x, n, nrhs, s);
}
int launch_solve_update(const DeviceLU &d, const Batch &b, int64_t ctas, bool backward, int trans, val_t *x, int n, int nrhs,
                        cudaStream_t s)
{
    return launch_solve_update_t(d, b, ctas, backward, trans, x, n, nrhs, s);
}
int launch_fill_csr(const BatchedLU &d, int n, const int32_t *rowptr, const int32_t *colind, const val_t *aval, const int32_t *perm,
                    const int8_t *active, int *err, cudaStream_t s)
{
    return launch_fill_csr_t(d, n, rowptr, colind, aval, perm, active, err, s);
}
int launch_solve_diag(const BatchedLU &d, const int32_t *nodes, int count, bool backward, int trans, val_t *x, int n, int nrhs,
                      cudaStream_t s)
{
    return launch_solve_diag_t(d, nodes, count, backward, trans, x, n, nrhs, s);
}
int launch_solve_update(const BatchedLU &d, const Batch &b, int64_t ctas, bool backward, int trans, val_t *x, int n, int nrhs,
                        cudaStream_t s)
{
    return launch_solve_update_t(d, b, ctas, backward, trans, x, n, nrhs, s);
}
int launch_solve_mask(const DeviceLU &d, const int32_t *nodes, int count, val_t *x, int n, int nrhs, const val_t *src, cudaStream_t s)
{
    if (count <= 0) return 0;
    solve_mask_kernel<<<std::min(count, 132 * 8), 128, 0, s>>>(d, nodes, count, x, n, nrhs, src);
    return 1;
}

}  // namespace SLU_NS
