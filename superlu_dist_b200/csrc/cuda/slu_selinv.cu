// slu_selinv.cu -- selected inversion on the resident factors (slu_b200_selinv, slu_b200_selinv_get, slu_b200_logdet).
// Double only.
//
// H = F^-T on every stored position of L + U, in a second arena laid out exactly as the factors (L panels nsupr x ns,
// dense-packed U panels ns x ncols, the same NodeDesc offsets).  For supernode K with sub-diagonal rows R and packed
// columns C, and M = H(R, C) (the values at the Schur-update destinations of K, already final in the supernodes of later
// levels), the host walks the level plan top-down and per level runs:
//   selinv_gemm_kernel<0>  H(R,K) <- -M U_KC^T                       (m x ns, inner ncols; M gathered in the loader)
//   selinv_gemm_kernel<1>  H(K,C) <- -L_RK^T M                       (ns x ncols, inner m)
//   selinv_gemm_kernel<2>  H(K,K) <- I - L_RK^T H(R,K)               (ns x ns, inner m; H(R,K) as the first kernel left it)
//   selinv_trsm_kernel<0>  every row x of L panel K of H:    x <- x U_KK^-T
//   selinv_trsm_kernel<1>  every column y of [H(K,K) H(K,C)]: y <- L_KK^-T y
// The last two give H(R,K) = -M U_KC^T U_KK^-T, H(K,C) = -L_KK^-T L_RK^T M and
// H(K,K) = L_KK^-T (I - L_RK^T (-M U_KC^T)) U_KK^-T = L_KK^-T (U_KK^-T - L_RK^T H(R,K)).
// Every entry of H is owned by one thread of each kernel and written with plain stores; the factors are only read.
#include "slu_device.cuh"
#define SLU_COMMON_HELPERS_ONLY
#include "slu_kernels_common.cuh"

#include <cmath>

namespace slu {

// ------------------------------------------------------------------------------------------------
// GEMM tiles on DMMA m16n8k8: 64 x 64 output tiles, 4 warps of 32 x 32, k-steps of 16.  Operands are staged through
// registers (the M operand is a gather through the destination maps, so cp.async does not apply): the next k-step is
// loaded while the current one is multiplied.
// ------------------------------------------------------------------------------------------------
constexpr int SI_BM = SELINV_TILE, SI_BN = SELINV_TILE, SI_BK = 16, SI_NT = 128;
constexpr int SI_LDA = SI_BM + 4, SI_LDB = SI_BK + 4;
constexpr int SI_PER = SI_BK * SI_BM / SI_NT;   // operand elements per thread and k-step (A and B alike)

// H(R, C) of supernode nd at (i, j): the destination of L(i) U(j) in the Schur update of nd, addressed as schur_kernel's
// epilogue addresses it
__device__ __forceinline__ double gather_m(const DeviceLU &d, const NodeDesc &nd, const double *__restrict__ hv, int i, int j)
{
    const RowInfo ri = d.rowinfo[nd.ws_row + i];
    const ColInfo cj = d.colinfo[nd.ws_col + j];
    if (ri.ib >= cj.jb) {
        const int p = d.lrel[cj.lrel_off + i];
        return p >= 0 ? hv[cj.lbase + p] : 0.0;
    }
    const int q = d.urel[ri.urel_off + j];
    return q >= 0 ? hv[ri.ubase + (int64_t)q * ri.ldu] : 0.0;
}

// MODE 0: out(i, p) = H(R,K), A(i, j) = M, B(j, p) = U_KC(p, j), inner ncols
// MODE 1: out(p, j) = H(K,C), A(p, i) = L_RK(i, p), B(i, j) = M, inner m
// MODE 2: out(p, q) = H(K,K), A(p, i) = L_RK(i, p), B(i, q) = H(R,K)(i, q), inner m
template <int MODE>
__global__ void __launch_bounds__(SI_NT) selinv_gemm_kernel(DeviceLU d, Batch b, double *__restrict__ hv)
{
    __shared__ __align__(16) double As[SI_BK * SI_LDA];
    __shared__ __align__(16) double Bs[SI_BN * SI_LDB];
    if (blockIdx.x >= b.prefix[b.count]) return;
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const NodeDesc nd = d.nodes[b.nodes[slot]];
    const int ns = nd.ns, m = nd.m, nc = nd.ncols, lda = nd.nsupr;
    const int rows = MODE == 0 ? m : ns, cols = MODE == 1 ? nc : ns, K = MODE == 0 ? nc : m;
    const int tiles_r = (rows + SI_BM - 1) / SI_BM;
    const int tile = (int)(blockIdx.x - b.prefix[slot]);
    const int r0 = (tile % tiles_r) * SI_BM, c0 = (tile / tiles_r) * SI_BN;
    const double *__restrict__ val = d.val;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;

    // A(r, k) and B(k, c) of the product; zero outside the operand
    auto a_at = [&](int r, int k) -> double {
        if (r >= rows || k >= K) return 0.0;
        if (MODE == 0) return gather_m(d, nd, hv, r, k);
        return val[nd.lval + (int64_t)r * lda + ns + k];
    };
    auto b_at = [&](int k, int c) -> double {
        if (k >= K || c >= cols) return 0.0;
        if (MODE == 0) return val[nd.uval + (int64_t)k * ns + c];
        if (MODE == 1) return gather_m(d, nd, hv, k, c);
        return hv[nd.lval + (int64_t)c * lda + ns + k];
    };
    // element e of a k-step: the index that is contiguous in memory runs fastest over the threads
    constexpr bool A_RFAST = MODE == 0, B_CFAST = MODE == 0;
    double ra[SI_PER], rb[SI_PER];
    auto fetch = [&](int k0) {
#pragma unroll
        for (int s = 0; s < SI_PER; ++s) {
            const int e = tid + s * SI_NT;
            const int ar = A_RFAST ? e % SI_BM : e / SI_BK, ak = A_RFAST ? e / SI_BM : e % SI_BK;
            ra[s] = a_at(r0 + ar, k0 + ak);
            const int bc = B_CFAST ? e % SI_BN : e / SI_BK, bk = B_CFAST ? e / SI_BN : e % SI_BK;
            rb[s] = b_at(k0 + bk, c0 + bc);
        }
    };
    auto stash = [&]() {
#pragma unroll
        for (int s = 0; s < SI_PER; ++s) {
            const int e = tid + s * SI_NT;
            const int ar = A_RFAST ? e % SI_BM : e / SI_BK, ak = A_RFAST ? e / SI_BM : e % SI_BK;
            As[ak * SI_LDA + ar] = ra[s];
            const int bc = B_CFAST ? e % SI_BN : e / SI_BK, bk = B_CFAST ? e / SI_BN : e % SI_BK;
            Bs[bc * SI_LDB + bk] = rb[s];
        }
    };

    double acc[2][4][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) acc[mt][nt][0] = acc[mt][nt][1] = acc[mt][nt][2] = acc[mt][nt][3] = 0.0;
    const int KT = (K + SI_BK - 1) / SI_BK;
    if (KT > 0) fetch(0);
    for (int kt = 0; kt < KT; ++kt) {
        stash();
        __syncthreads();
        if (kt + 1 < KT) fetch((kt + 1) * SI_BK);
#pragma unroll
        for (int k8 = 0; k8 < SI_BK; k8 += 8) {
            double a[2][4], bb[4][2];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                const double *p = As + (k8 + t) * SI_LDA + wm + 16 * mt + g;
                a[mt][0] = p[0]; a[mt][1] = p[8]; a[mt][2] = p[4 * SI_LDA]; a[mt][3] = p[4 * SI_LDA + 8];
            }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const double *p = Bs + (wn + 8 * nt + g) * SI_LDB + k8 + t;
                bb[nt][0] = p[0]; bb[nt][1] = p[4];
            }
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) dmma1688(acc[mt][nt], a[mt], bb[nt]);
        }
        __syncthreads();
    }
    // lane (g, t) holds rows g, g + 8 and columns 2t, 2t + 1 of each 16 x 8 piece
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = r0 + wm + 16 * mt + g + 8 * (e >> 1), c = c0 + wn + 8 * nt + 2 * t + (e & 1);
                if (r >= rows || c >= cols) continue;
                const double v = -acc[mt][nt][e];
                if (MODE == 0) hv[nd.lval + (int64_t)c * lda + ns + r] = v;
                else if (MODE == 1) hv[nd.uval + (int64_t)c * ns + r] = v;
                else hv[nd.lval + (int64_t)c * lda + r] = (r == c ? 1.0 : 0.0) + v;
            }
}

// ------------------------------------------------------------------------------------------------
// In-place back substitution with an upper triangular T of the supernode's diagonal block, one vector per thread, 16
// unknowns at a time: the already solved unknowns are subtracted, then the 16 x 16 block inverse of diag_inv_kernel is
// applied.  COLS = 0: the rows x of L panel K of H, T = U_KK (x <- x U_KK^-T, i.e. U_KK x^T = x^T); COLS = 1: the ns
// columns of H(K,K) and the ncols columns of H(K,C), T = L_KK^T (unit; its block inverse is inv(L_bb) read transposed).
// ------------------------------------------------------------------------------------------------
template <int COLS>
__global__ void __launch_bounds__(SELINV_VECS) selinv_trsm_kernel(DeviceLU d, Batch b, const double *__restrict__ dinv,
                                                                   double *__restrict__ hv)
{
    if (blockIdx.x >= b.prefix[b.count]) return;
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const NodeDesc nd = d.nodes[b.nodes[slot]];
    const int ns = nd.ns, lda = nd.nsupr;
    const int v = (int)(blockIdx.x - b.prefix[slot]) * SELINV_VECS + threadIdx.x;
    if (v >= (COLS ? ns + nd.ncols : lda)) return;
    double *x;
    int64_t stride;
    if (!COLS) { x = hv + nd.lval + v; stride = lda; }
    else if (v < ns) { x = hv + nd.lval + (int64_t)v * lda; stride = 1; }
    else { x = hv + nd.uval + (int64_t)(v - ns) * ns; stride = 1; }
    const double *__restrict__ D = d.val + nd.lval;          // the diagonal block, column-major with lda
    const double *__restrict__ inv = dinv + nd.ws_inv;
    for (int blk = (ns - 1) / 16; blk >= 0; --blk) {
        const int p0 = blk * 16, w = min(16, ns - p0);
        double acc[16];
#pragma unroll
        for (int r = 0; r < 16; ++r) acc[r] = r < w ? x[(int64_t)(p0 + r) * stride] : 0.0;
        for (int q = p0 + w; q < ns; ++q) {
            const double z = x[(int64_t)q * stride];
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                if (r >= w) break;
                const double tv = COLS ? D[(int64_t)(p0 + r) * lda + q] : D[(int64_t)q * lda + p0 + r];
                acc[r] = fma(-tv, z, acc[r]);
            }
        }
        const double *bi = inv + (size_t)blk * 512 + (COLS ? 256 : 0);
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            if (r >= w) break;
            double y = 0.0;
#pragma unroll
            for (int c = 0; c < 16; ++c) y = fma(COLS ? bi[r * 16 + c] : bi[c * 16 + r], acc[c], y);
            x[(int64_t)(p0 + r) * stride] = y;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// log |det| and the number of negative pivots: one supernode per thread, fixed-order reductions (no float atomics)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void si_block_reduce(double &s, int &neg)
{
    __shared__ double ss[SELINV_VECS / 32];
    __shared__ int sn[SELINV_VECS / 32];
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_down_sync(0xffffffffu, s, o);
        neg += __shfl_down_sync(0xffffffffu, neg, o);
    }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { ss[w] = s; sn[w] = neg; }
    __syncthreads();
    if (threadIdx.x == 0) {
        s = 0.0; neg = 0;
        for (int i = 0; i < SELINV_VECS / 32; ++i) { s += ss[i]; neg += sn[i]; }
    }
}

__global__ void __launch_bounds__(SELINV_VECS) selinv_logdet_partial_kernel(DeviceLU d, const int32_t *nodes, int count, double *part,
                                                                            int *pneg)
{
    const int t = blockIdx.x * SELINV_VECS + threadIdx.x;
    double s = 0.0;
    int neg = 0;
    if (t < count) {
        const NodeDesc nd = d.nodes[nodes[t]];
        const double *D = d.val + nd.lval;
        for (int i = 0; i < nd.ns; ++i) {
            const double p = D[(int64_t)i * nd.nsupr + i];
            s += log(fabs(p));
            neg += p < 0.0;
        }
    }
    si_block_reduce(s, neg);
    if (threadIdx.x == 0) { part[blockIdx.x] = s; pneg[blockIdx.x] = neg; }
}

__global__ void __launch_bounds__(SELINV_VECS) selinv_logdet_final_kernel(const double *part, const int *pneg, int nparts, double *out)
{
    double s = 0.0;
    int neg = 0;
    for (int i = threadIdx.x; i < nparts; i += SELINV_VECS) { s += part[i]; neg += pneg[i]; }
    si_block_reduce(s, neg);
    if (threadIdx.x == 0) { out[0] = s; out[1] = (neg & 1) ? -1.0 : 1.0; }
}

// ------------------------------------------------------------------------------------------------
// out[p] = A^-1(i, colind[p]) = H(perm[colind[p]], perm[i]): the slot search of fill_csr_kernel with the roles of row and
// column swapped, reading instead of writing.  One thread per row of the pattern.
// ------------------------------------------------------------------------------------------------
__global__ void selinv_get_kernel(DeviceLU d, const double *__restrict__ hv, int n, const int32_t *__restrict__ rowptr,
                                  const int32_t *__restrict__ colind, const int32_t *__restrict__ perm, double *__restrict__ out,
                                  int *err)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int pj = perm[i];                       // column of H
    const int ks = d.supno[pj];
    for (int p = rowptr[i]; p < rowptr[i + 1]; ++p) {
        const int pi = perm[colind[p]];           // row of H
        double v = NAN;
        if (pi >= d.xsup[ks]) {                   // L panel of block column supno(pj), diagonal block included
            const NodeDesc *nd = d.nodes + ks;
            const int32_t *srow = d.lsrow + nd->lrow;
            const int q = lower_bound_i32(srow, nd->nsupr, pi);
            if (q < nd->nsupr && srow[q] == pi) v = hv[nd->lval + (int64_t)(pj - nd->fsupc) * nd->nsupr + d.lspos[nd->lrow + q]];
            else atomicAdd(err, 1);
        } else {                                  // U panel of block row supno(pi)
            const NodeDesc *nd = d.nodes + d.supno[pi];
            const int32_t *uc = d.ucols + nd->ucol;
            const int q = lower_bound_i32(uc, nd->ncols, pj);
            if (q < nd->ncols && uc[q] == pj) v = hv[nd->uval + (int64_t)q * nd->ns + (pi - nd->fsupc)];
            else atomicAdd(err, 1);
        }
        out[p] = v;
    }
}

// ------------------------------------------------------------------------------------------------
int launch_selinv_gemm(const DeviceLU &d, const Batch &b, int64_t ctas, int mode, double *hv, cudaStream_t s)
{
    if (b.count <= 0) return 0;
    const unsigned grid = (unsigned)(ctas > 0 ? ctas : 1);   // an empty batch still makes its launch: the count stays fixed
    if (mode == 0) selinv_gemm_kernel<0><<<grid, SI_NT, 0, s>>>(d, b, hv);
    else if (mode == 1) selinv_gemm_kernel<1><<<grid, SI_NT, 0, s>>>(d, b, hv);
    else selinv_gemm_kernel<2><<<grid, SI_NT, 0, s>>>(d, b, hv);
    return 1;
}

int launch_selinv_trsm(const DeviceLU &d, const Batch &b, int64_t ctas, int cols, const double *dinv, double *hv, cudaStream_t s)
{
    if (b.count <= 0) return 0;
    const unsigned grid = (unsigned)(ctas > 0 ? ctas : 1);
    if (cols) selinv_trsm_kernel<1><<<grid, SELINV_VECS, 0, s>>>(d, b, dinv, hv);
    else selinv_trsm_kernel<0><<<grid, SELINV_VECS, 0, s>>>(d, b, dinv, hv);
    return 1;
}

int launch_selinv_logdet(const DeviceLU &d, const int32_t *nodes, int count, double *part, int *pneg, double *out, cudaStream_t s)
{
    const int nparts = (count + SELINV_VECS - 1) / SELINV_VECS;
    if (nparts <= 0) return 0;
    selinv_logdet_partial_kernel<<<nparts, SELINV_VECS, 0, s>>>(d, nodes, count, part, pneg);
    selinv_logdet_final_kernel<<<1, SELINV_VECS, 0, s>>>(part, pneg, nparts, out);
    return 2;
}

int launch_selinv_get(const DeviceLU &d, const double *hv, int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm,
                      double *out, int *err, cudaStream_t s)
{
    if (n <= 0) return 0;
    selinv_get_kernel<<<(n + 127) / 128, 128, 0, s>>>(d, hv, n, rowptr, colind, perm, out, err);
    return 1;
}

}  // namespace slu
