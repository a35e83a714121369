// slu_kernels_z.cu -- the sm_90a kernels of the doublecomplex hot path (pzgstrf3d, SURVEY 8a row a15:
// SRC/complex16/pzgstrf3d.c:120, Local_Zgstrf2 pzgstrf2.c:508-601, zscatter_l/zblock_gemm_scatter).
// Same batched level-synchronous structure and HBM layout as slu_kernels.cu; elements are (re, im) pairs.
//
//   diag_lu_kernel   unpivoted complex LU of the diagonal block, reciprocal pivots (slud_z_div), tiny-pivot rule
//                    of pzgstrf2.c:545-560 (|re|+|im| < thresh, replacement +-thresh + 0i)
//   diag_inv_kernel  inverse of every 16x16 diagonal block of U_kk and L_kk
//   trsm_kernel      left-looking panel solves on 32-vector strips held in shared memory
//   schur_kernel     V = L(below,k) U(k,:) as a REAL product on the FP64 tensor cores (DMMA m8n8k4):
//                    [Ar Ai] (m x 2k, the interleaved storage read as a real matrix) times
//                    [[Br Bi] [-Bi Br]] (2k x 2n) gives the interleaved (re, im) of V with exactly the 4 real
//                    multiply-adds per complex one; the second factor is never built -- each lane reads the raw
//                    (re, im) pair of U with a lane-constant swap and sign.  Subtract-scatter fused in the epilogue.
//   u_convert / axpy as in the real build.
// diag_lu, diag_inv, trsm and schur are templated on their DeviceLU type, as in slu_kernels.cu: the BatchedLU
// instantiations serve the batched handles (slu_b200_z_batch_*, member = blockIdx.y).
#define SLU_COMPLEX 1
#include "slu_device.cuh"
#include "slu_kernels_common.cuh"
#include "slu_scalar.cuh"   // zd, zmul, zsubmul, zrecip ...

#include <climits>

namespace sluz {

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem, bool pred)
{
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    int sz = pred ? 16 : 0;  // src-size 0 => the 16 bytes are zero-filled
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(sa), "l"(gmem), "r"(sz));
}

// ------------------------------------------------------------------------------------------------
// diagonal block LU (same schedule as the real kernel: 16-column panels in shared memory)
// ------------------------------------------------------------------------------------------------
template <class LU>
__global__ void __launch_bounds__(512) diag_lu_kernel(LU dd, Batch b, int replace_tiny, double thresh)
{
    extern __shared__ double2 smz[];
    const DeviceLU &d = member_view(dd);
    constexpr int NB = DIAG_NB;
    const int k = b.nodes[blockIdx.x];
    const NodeDesc nd = d.nodes[k];
    const int ns = nd.ns, lda = nd.nsupr, tid = threadIdx.x, nt = blockDim.x;
    zd *A = d.val + nd.lval;
    zd *Ps = smz;            // panel  Ps[c*rem + i]
    zd *Us = smz + NB * ns;  // U12    Us[c*NB + p]

    for (int j0 = 0; j0 < ns; j0 += NB) {
        const int jb = min(NB, ns - j0), rem = ns - j0;
        for (int idx = tid; idx < jb * rem; idx += nt) {
            int c = idx / rem, i = idx - c * rem;
            Ps[c * rem + i] = A[(size_t)(j0 + c) * lda + j0 + i];
        }
        __syncthreads();
        // (1) warp 0 factors the jb x jb diagonal block (lane r owns row r)
        if (tid < 32) {
            const int r = tid;
            for (int c = 0; c < jb; ++c) {
                if (r == 0) {
                    zd p = Ps[c * rem + c];
                    // pzgstrf2.c:545-560 as written: fires only when both parts are non-zero
                    if (replace_tiny && fabs(p.x) + fabs(p.y) < thresh && p.x != 0.0 && p.y != 0.0) {
                        p = zmake((p.x < 0) ? -thresh : thresh, 0.0);
                        Ps[c * rem + c] = p;
                        if (replace_tiny == 1) atomicAdd(d.tiny, 1ULL);  // 2: replicated copy, counted by its owner
                    }
                    if (zzero(p)) atomicMin(d.info, nd.fsupc + j0 + c + 1);  // pzgstrf2.c:568-571
                }
                __syncwarp();
                const zd p = Ps[c * rem + c];
                if (r > c && r < jb) {
                    zd l = Ps[c * rem + r];
                    if (!zzero(p)) l = zmul(l, zrecip(p));
                    Ps[c * rem + r] = l;
                    for (int cc = c + 1; cc < jb; ++cc) {
                        zd t = Ps[cc * rem + r];
                        zsubmul(t, l, Ps[cc * rem + c]);
                        Ps[cc * rem + r] = t;
                    }
                }
                __syncwarp();
            }
        }
        __syncthreads();
        // (2) rows below the diagonal block: x U11 = a, one row per thread
        for (int i = jb + tid; i < rem; i += nt) {
            zd x[NB];
#pragma unroll
            for (int c = 0; c < NB; ++c) x[c] = (c < jb) ? Ps[c * rem + i] : zmake(0.0, 0.0);
#pragma unroll
            for (int c = 0; c < NB; ++c) {
                if (c < jb) {
                    zd v = x[c];
#pragma unroll
                    for (int p = 0; p < NB; ++p)
                        if (p < c) zsubmul(v, x[p], Ps[c * rem + p]);
                    const zd pv = Ps[c * rem + c];
                    x[c] = zzero(pv) ? v : zmul(v, zrecip(pv));
                }
            }
#pragma unroll
            for (int c = 0; c < NB; ++c)
                if (c < jb) Ps[c * rem + i] = x[c];
        }
        __syncthreads();
        for (int idx = tid; idx < jb * rem; idx += nt) {
            int c = idx / rem, i = idx - c * rem;
            A[(size_t)(j0 + c) * lda + j0 + i] = Ps[c * rem + i];
        }
        const int r2 = rem - jb;
        if (r2 > 0) {
            // U12 = L11^-1 A12 (unit lower), one trailing column per thread
            for (int c = tid; c < r2; c += nt) {
                zd x[NB];
                zd *col = A + (size_t)(j0 + jb + c) * lda + j0;
#pragma unroll
                for (int p = 0; p < NB; ++p) x[p] = (p < jb) ? col[p] : zmake(0.0, 0.0);
#pragma unroll
                for (int p = 0; p < NB; ++p)
#pragma unroll
                    for (int q = p + 1; q < NB; ++q)
                        if (q < jb) zsubmul(x[q], Ps[p * rem + q], x[p]);
#pragma unroll
                for (int p = 0; p < NB; ++p) {
                    if (p < jb) col[p] = x[p];
                    Us[c * NB + p] = x[p];
                }
            }
            __syncthreads();
            // A22 -= L21 U12
            for (int idx = tid; idx < r2 * r2; idx += nt) {
                int c = idx / r2, i = idx - c * r2;
                zd acc = zmake(0.0, 0.0);
#pragma unroll
                for (int p = 0; p < NB; ++p)
                    if (p < jb) zaddmul(acc, Ps[p * rem + jb + i], Us[c * NB + p]);
                zd *dst = A + (size_t)(j0 + jb + c) * lda + j0 + jb + i;
                zd t = *dst;
                t.x -= acc.x; t.y -= acc.y;
                *dst = t;
            }
        }
        __syncthreads();
    }
}

template <class LU>
static int launch_diag_lu_t(const LU &d, const Batch &b, int max_ns, int replace_tiny, double thresh, cudaStream_t s)
{
    if (b.count <= 0) return 0;
    size_t smem = sizeof(zd) * 2 * DIAG_NB * (size_t)max_ns;
    static std::atomic<unsigned long long> attr_0{0};
    ensure_dyn_smem(diag_lu_kernel<LU>, (int)(sizeof(zd) * 2 * DIAG_NB * MAX_NS_HELD), attr_0);
    int threads = max_ns <= 32 ? 128 : (max_ns <= 128 ? 256 : 512);
    diag_lu_kernel<LU><<<member_grid(d, b.count), threads, smem, s>>>(d, b, replace_tiny, thresh);
    return 1;
}
int launch_diag_lu(const DeviceLU &d, const Batch &b, int max_ns, int replace_tiny, double thresh, cudaStream_t s)
{
    return launch_diag_lu_t(d, b, max_ns, replace_tiny, thresh, s);
}
int launch_diag_lu(const BatchedLU &d, const Batch &b, int max_ns, int replace_tiny, double thresh, cudaStream_t s)
{
    return launch_diag_lu_t(d, b, max_ns, replace_tiny, thresh, s);
}

// ------------------------------------------------------------------------------------------------
// inverse of the 16x16 diagonal blocks: dinv[ws_inv + blk*512 + {0: inv U (column-major 16x16), 256: inv L}]
// ------------------------------------------------------------------------------------------------
template <class LU>
__global__ void __launch_bounds__(64) diag_inv_kernel(LU dd, Batch b, zd *dinv)
{
    __shared__ zd M[16 * 17];
    const DeviceLU &d = member_view(dd);
    dinv = member_inv(dd, dinv);
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const int k = b.nodes[slot];
    const NodeDesc nd = d.nodes[k];
    const int blk = (int)(blockIdx.x - b.prefix[slot]);
    const int j0 = blk * 16, jb = min(16, nd.ns - j0), lda = nd.nsupr, tid = threadIdx.x;
    const zd *A = d.val + nd.lval;
    for (int idx = tid; idx < 256; idx += 64) {
        int c = idx >> 4, r = idx & 15;
        zd v = zmake((r == c) ? 1.0 : 0.0, 0.0);
        if (r < jb && c < jb) v = A[(size_t)(j0 + c) * lda + j0 + r];
        M[c * 17 + r] = v;
    }
    __syncthreads();
    zd *out = dinv + nd.ws_inv + (size_t)blk * 512;
    const int c = tid & 31;
    if (tid < 32) {  // column c of inv(U), U = upper triangle of M (non-unit)
        if (c < 16) {
            zd x[16];
#pragma unroll
            for (int r = 0; r < 16; ++r) x[r] = zmake(0.0, 0.0);
            for (int r = c; r >= 0; --r) {
                zd sacc = zmake((r == c) ? 1.0 : 0.0, 0.0);
                for (int q = r + 1; q <= c; ++q) zsubmul(sacc, M[q * 17 + r], x[q]);
                const zd piv = M[r * 17 + r];
                x[r] = zzero(piv) ? sacc : zmul(sacc, zrecip(piv));
            }
#pragma unroll
            for (int r = 0; r < 16; ++r) out[c * 16 + r] = x[r];
        }
    } else if (c < 16) {  // column c of inv(L), L = unit lower triangle of M
        zd x[16];
#pragma unroll
        for (int r = 0; r < 16; ++r) x[r] = zmake(0.0, 0.0);
        x[c] = zmake(1.0, 0.0);
        for (int r = c + 1; r < 16; ++r) {
            zd sacc = zmake(0.0, 0.0);
            for (int q = c; q < r; ++q) zsubmul(sacc, M[q * 17 + r], x[q]);
            x[r] = sacc;
        }
#pragma unroll
        for (int r = 0; r < 16; ++r) out[256 + c * 16 + r] = x[r];
    }
}

template <class LU>
static int launch_diag_inv_t(const LU &d, const Batch &b, int64_t ctas, zd *dinv, cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    diag_inv_kernel<LU><<<member_grid(d, (unsigned)ctas), 64, 0, s>>>(d, b, dinv);
    return 1;
}
int launch_diag_inv(const DeviceLU &d, const Batch &b, int64_t ctas, zd *dinv, cudaStream_t s)
{
    return launch_diag_inv_t(d, b, ctas, dinv, s);
}
int launch_diag_inv(const BatchedLU &d, const Batch &b, int64_t ctas, zd *dinv, cudaStream_t s)
{
    return launch_diag_inv_t(d, b, ctas, dinv, s);
}

// ------------------------------------------------------------------------------------------------
// panel triangular solves:  Y <- Y T^-1, T upper triangular ns x ns, blocked by 16 columns (left-looking)
//   L case: vectors = sub-diagonal rows of panel k, T(p,c) = U_kk(p,c)            (non-unit)
//   U case: vectors = packed columns of U(k,:),    T(p,c) = L_kk(c,p) (transposed, unit)
// A CTA keeps a strip of 32 vectors in shared memory (Ys[c][s]); 256 threads = 32 vectors x 8 column lanes, each
// thread owns columns cl and cl + 8 of the current 16-column block.  Each block is multiplied by the inverse of
// T_jj and corrected once with it, as in slu_kernels.cu.
// ------------------------------------------------------------------------------------------------
constexpr int TZ_LD = TRSM_STRIP + 1;

template <bool UCASE, class LU>
__global__ void __launch_bounds__(256) trsm_kernel(LU dd, Batch b, const zd *dinv)
{
    extern __shared__ double2 smz[];
    const DeviceLU &d = member_view(dd);
    dinv = member_inv(dd, dinv);
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const int k = b.nodes[slot];
    const NodeDesc nd = d.nodes[k];
    const int strip = (int)(blockIdx.x - b.prefix[slot]);
    const int ns = nd.ns, lda = nd.nsupr, tid = threadIdx.x;
    const int nvec = UCASE ? nd.ncols : nd.m;
    const int v0 = strip * TRSM_STRIP, nv = min(TRSM_STRIP, nvec - v0);
    if (nv <= 0) return;
    const zd *T = d.val + nd.lval;                // diagonal block (LU in place), lda = nsupr
    const zd *inv = dinv + nd.ws_inv;
    zd *X = UCASE ? d.val + nd.uval + (size_t)v0 * ns : d.val + nd.lval + ns + v0;
    zd *Ys = smz;                                  // Ys[c * TZ_LD + s], c < ns
    zd *Tmp = smz + (size_t)ns * TZ_LD;            // Tmp[q * TZ_LD + s], q < 16

    if (!UCASE) {
        for (int idx = tid; idx < ns * TRSM_STRIP; idx += 256) {
            int c = idx / TRSM_STRIP, s = idx - c * TRSM_STRIP;
            Ys[c * TZ_LD + s] = (s < nv) ? X[(size_t)c * lda + s] : zmake(0.0, 0.0);
        }
    } else {
        for (int idx = tid; idx < ns * TRSM_STRIP; idx += 256) {
            int s = idx / ns, c = idx - s * ns;
            Ys[c * TZ_LD + s] = (s < nv) ? X[(size_t)s * ns + c] : zmake(0.0, 0.0);
        }
    }
    __syncthreads();

    const int s = tid & 31, cl = tid >> 5;  // vector, column lane (0..7)
    for (int j0 = 0; j0 < ns; j0 += 16) {
        // (1) tmp(s, c) = Y(s, j0 + c) - sum_{p < j0} Y(s, p) T(p, j0 + c)
        zd acc[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int c = j0 + cl + 8 * h;
            acc[h] = (c < ns) ? Ys[c * TZ_LD + s] : zmake(0.0, 0.0);
        }
        for (int p = 0; p < j0; ++p) {
            const zd y = Ys[p * TZ_LD + s];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = j0 + cl + 8 * h;
                if (c < ns) {
                    const zd t = UCASE ? __ldg(T + (size_t)p * lda + c) : __ldg(T + (size_t)c * lda + p);
                    zsubmul(acc[h], y, t);
                }
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) Tmp[(cl + 8 * h) * TZ_LD + s] = acc[h];
        __syncthreads();
        // (2) x(s, c) = sum_q tmp(s, q) Inv(q, c), then one correction step x += (tmp - x T_jj) Inv: the product with
        // an explicit inverse alone has a backward error that grows with cond(T_jj) on consistent right-hand sides
        const zd *ib = inv + (size_t)(j0 >> 4) * 512;
        const int jb = min(16, ns - j0);
        zd out[2] = {zmake(0.0, 0.0), zmake(0.0, 0.0)};
        auto mul_inv = [&]() {
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const zd y = Tmp[q * TZ_LD + s];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int c = cl + 8 * h;
                    const zd t = UCASE ? __ldg(ib + 256 + q * 16 + c) : __ldg(ib + c * 16 + q);
                    zaddmul(out[h], y, t);
                }
            }
        };
        mul_inv();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int c = j0 + cl + 8 * h;
            if (c < ns) Ys[c * TZ_LD + s] = out[h];
        }
        __syncthreads();
        // tmp - x T_jj, T_jj(q, c) for q <= c < jb; in the U case its diagonal is 1 (the stored one holds U's pivots)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int c = cl + 8 * h;
            zd r = zmake(0.0, 0.0);
            if (c < jb) {
                r = acc[h];
                for (int q = 0; q <= c; ++q) {
                    const zd x = Ys[(j0 + q) * TZ_LD + s];
                    if (UCASE && q == c) r = zmake(r.x - x.x, r.y - x.y);
                    else zsubmul(r, x, UCASE ? __ldg(T + (size_t)(j0 + q) * lda + j0 + c)
                                             : __ldg(T + (size_t)(j0 + c) * lda + j0 + q));
                }
            }
            Tmp[c * TZ_LD + s] = r;   // every thread read its tmp in (2), before the barrier above
        }
        __syncthreads();
        mul_inv();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int c = j0 + cl + 8 * h;
            if (c < ns) Ys[c * TZ_LD + s] = out[h];
        }
        __syncthreads();
    }
    if (!UCASE) {
        for (int idx = tid; idx < ns * TRSM_STRIP; idx += 256) {
            int c = idx / TRSM_STRIP, ss = idx - c * TRSM_STRIP;
            if (ss < nv) X[(size_t)c * lda + ss] = Ys[c * TZ_LD + ss];
        }
    } else {
        for (int idx = tid; idx < ns * TRSM_STRIP; idx += 256) {
            int ss = idx / ns, c = idx - ss * ns;
            if (ss < nv) X[(size_t)ss * ns + c] = Ys[c * TZ_LD + ss];
        }
    }
}

template <bool UCASE, class LU>
static int launch_trsm(const LU &d, const Batch &b, int64_t ctas, int max_ns, const zd *dinv, cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    static std::atomic<unsigned long long> attr_0{0};
    ensure_dyn_smem(trsm_kernel<UCASE, LU>, (int)(sizeof(zd) * (MAX_NS_HELD + 16) * TZ_LD), attr_0);
    const size_t smem = sizeof(zd) * ((size_t)max_ns + 16) * TZ_LD;
    trsm_kernel<UCASE, LU><<<member_grid(d, (unsigned)ctas), 256, smem, s>>>(d, b, dinv);
    return 1;
}
int launch_trsm_l(const DeviceLU &d, const Batch &b, int64_t ctas, int max_ns, const zd *dinv, cudaStream_t s)
{
    return launch_trsm<false>(d, b, ctas, max_ns, dinv, s);
}
int launch_trsm_u(const DeviceLU &d, const Batch &b, int64_t ctas, int max_ns, const zd *dinv, cudaStream_t s)
{
    return launch_trsm<true>(d, b, ctas, max_ns, dinv, s);
}
int launch_trsm_l(const BatchedLU &d, const Batch &b, int64_t ctas, int max_ns, const zd *dinv, cudaStream_t s)
{
    return launch_trsm<false>(d, b, ctas, max_ns, dinv, s);
}
int launch_trsm_u(const BatchedLU &d, const Batch &b, int64_t ctas, int max_ns, const zd *dinv, cudaStream_t s)
{
    return launch_trsm<true>(d, b, ctas, max_ns, dinv, s);
}

// ------------------------------------------------------------------------------------------------
// complex tile product on DMMA: acc (BM rows x BNC complex columns, interleaved) += A(m0.., :) B(:, n0..)
// A is M x K complex (lda), B is K x N complex (ldb); BKC complex k per pipeline stage.
// Shared memory keeps the RAW interleaved tiles: As[p][2*row + c], Bs[col][2*p + c].
// ------------------------------------------------------------------------------------------------
template <int BM, int BNC, int WARPS_M, int WARPS_N, int BKC = 8, int STAGES = 3>
struct ZCfg {
    static constexpr int NT = 32 * WARPS_M * WARPS_N;
    static constexpr int WTM = BM / WARPS_M, WTN = 2 * BNC / WARPS_N;  // warp tile in REAL columns
    static constexpr int MI = WTM / 8, NI = WTN / 8;
    static constexpr int LDA2 = 2 * BM, LDB2 = 2 * BKC + 4;            // doubles; LDB2 = 4 (mod 16): conflict-free
    static constexpr int A_STAGE = BKC * LDA2, B_STAGE = BNC * LDB2;
    static constexpr size_t SMEM = sizeof(double) * STAGES * (A_STAGE + B_STAGE);
};

template <int BM, int BNC, int WARPS_M, int WARPS_N, int BKC = 8, int STAGES = 3>
__device__ __forceinline__ void zgemm_tile(const zd *__restrict__ A, int lda, const zd *__restrict__ B, int ldb, int M,
                                           int N, int K, int m0, int n0, double *sm,
                                           double (&acc)[BM / WARPS_M / 8][2 * BNC / WARPS_N / 8][2])
{
    using C = ZCfg<BM, BNC, WARPS_M, WARPS_N, BKC, STAGES>;
    static_assert((BKC * BM) % C::NT == 0 && (BNC * BKC) % C::NT == 0 && BKC % 2 == 0, "loader mapping");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm0 = (warp % WARPS_M) * C::WTM, wn0 = (warp / WARPS_M) * C::WTN;
    double *As = sm, *Bs = sm + STAGES * C::A_STAGE;
    const int KT = (K + BKC - 1) / BKC;

    auto load = [&](int st, int kt) {
        const int k0 = kt * BKC;
        double *as = As + st * C::A_STAGE, *bs = Bs + st * C::B_STAGE;
#pragma unroll
        for (int idx = tid; idx < BKC * BM; idx += C::NT) {       // one complex element (16 B) per copy
            const int p = idx / BM, mm = idx - p * BM;
            const bool ok = (m0 + mm < M) && (k0 + p < K);
            const zd *src = ok ? A + (size_t)(k0 + p) * lda + m0 + mm : A;
            cp_async16(as + p * C::LDA2 + 2 * mm, src, ok);
        }
#pragma unroll
        for (int idx = tid; idx < BNC * BKC; idx += C::NT) {
            const int j = idx / BKC, p = idx - j * BKC;
            const bool ok = (n0 + j < N) && (k0 + p < K);
            const zd *src = ok ? B + (size_t)(n0 + j) * ldb + k0 + p : B;
            cp_async16(bs + j * C::LDB2 + 2 * p, src, ok);
        }
    };

    // lane constants of the fragment reads (see the header comment): A^(i, 2p+c) = As[p][2i+c];
    // B~(2p+c, 2j+e) = sgn * Bs[j][2p + (c^e)], sgn = -1 iff e == 0 and c == 1
    const int lr = lane >> 2, lk = lane & 3;
    const int pa = lk >> 1, ca = lk & 1;
    const int eb = lr & 1, jb = lr >> 1;
    const int cb = ca ^ eb;
    const int flip = (eb == 0 && ca == 1) ? (int)0x80000000 : 0;

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < KT) load(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < KT; ++kt) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        if (kt + STAGES - 1 < KT) load((kt + STAGES - 1) % STAGES, kt + STAGES - 1);
        cp_async_commit();
        const double *as = As + (kt % STAGES) * C::A_STAGE, *bs = Bs + (kt % STAGES) * C::B_STAGE;
#pragma unroll
        for (int k4 = 0; k4 < BKC / 2; ++k4) {  // 4 real k = 2 complex k per DMMA step
            double a[C::MI], bb[C::NI];
#pragma unroll
            for (int mi = 0; mi < C::MI; ++mi) a[mi] = as[(k4 * 2 + pa) * C::LDA2 + 2 * (wm0 + mi * 8 + lr) + ca];
#pragma unroll
            for (int ni = 0; ni < C::NI; ++ni) {
                const double v = bs[((wn0 >> 1) + ni * 4 + jb) * C::LDB2 + 2 * (k4 * 2 + pa) + cb];
                bb[ni] = __hiloint2double(__double2hiint(v) ^ flip, __double2loint(v));
            }
#pragma unroll
            for (int mi = 0; mi < C::MI; ++mi)
#pragma unroll
                for (int ni = 0; ni < C::NI; ++ni) dmma884(acc[mi][ni][0], acc[mi][ni][1], a[mi], bb[ni]);
        }
    }
    cp_async_wait<0>();
}

// ------------------------------------------------------------------------------------------------
// Schur-complement update of a batch of supernodes: complex tile product + fused subtract-scatter
// ------------------------------------------------------------------------------------------------
template <int BM, int BNC, int WARPS_M, int WARPS_N, class LU = DeviceLU>
__global__ void __launch_bounds__(32 * WARPS_M * WARPS_N, 2)
    schur_kernel(LU dd, Batch b, int mode, int split_n, int split_i)
{
    using C = ZCfg<BM, BNC, WARPS_M, WARPS_N>;
    extern __shared__ double smd[];
    const DeviceLU &d = member_view(dd);
    const int64_t gt = (int64_t)blockIdx.x * split_n + split_i;
    if (gt >= b.prefix[b.count]) return;
    const int slot = find_slot(b.prefix, b.count, gt);
    const int k = b.nodes[slot];
    const NodeDesc nd = d.nodes[k];
    const int tile = (int)(gt - b.prefix[slot]);
    const int tiles_m = (nd.m + BM - 1) / BM;
    int tm, tn;
    if (mode == 0) {
        tm = tile % tiles_m; tn = tile / tiles_m;
    } else {
        const int tru = (nd.urg_rows + BM - 1) / BM, tcu = (nd.urg_cols + BNC - 1) / BNC;
        if (mode == 1) {
            if (tile < tiles_m * tcu) { tm = tile % tiles_m; tn = tile / tiles_m; }
            else { const int t = tile - tiles_m * tcu; tm = t % tru; tn = tcu + t / tru; }
        } else {
            const int rm = tiles_m - tru;
            tm = tru + tile % rm; tn = tcu + tile / rm;
        }
    }
    const int m0 = tm * BM, n0 = tn * BNC;

    double acc[C::MI][C::NI][2];
#pragma unroll
    for (int mi = 0; mi < C::MI; ++mi)
#pragma unroll
        for (int ni = 0; ni < C::NI; ++ni) acc[mi][ni][0] = acc[mi][ni][1] = 0.0;

    zgemm_tile<BM, BNC, WARPS_M, WARPS_N>(d.val + nd.lval + nd.ns, nd.nsupr, d.val + nd.uval, nd.ns, nd.m, nd.ncols,
                                          nd.ns, m0, n0, smd, acc);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm0 = m0 + (warp % WARPS_M) * C::WTM;
    const int wn0c = n0 + (((warp / WARPS_M) * C::WTN) >> 1);  // first complex column of the warp tile
    const RowInfo *rinfo = d.rowinfo + nd.ws_row;
    const ColInfo *cinfo = d.colinfo + nd.ws_col;
    RowInfo ri[C::MI];
    bool rok[C::MI];
#pragma unroll
    for (int mi = 0; mi < C::MI; ++mi) {
        const int i = wm0 + mi * 8 + (lane >> 2);
        rok[mi] = i < nd.m;
        if (rok[mi]) ri[mi] = rinfo[i];
    }
#pragma unroll
    for (int ni = 0; ni < C::NI; ++ni) {
        const int j = wn0c + ni * 4 + (lane & 3);  // this lane holds (re, im) of complex column j
        const bool cok = j < nd.ncols;
        ColInfo cj;
        if (cok) cj = cinfo[j];
        int64_t idx[C::MI];
#pragma unroll
        for (int mi = 0; mi < C::MI; ++mi) {
            idx[mi] = -1;
            if (!cok || !rok[mi]) continue;
            const int i = wm0 + mi * 8 + (lane >> 2);
            if (ri[mi].ib >= cj.jb) {
                const int p = d.lrel[cj.lrel_off + i];
                if (p >= 0) idx[mi] = cj.lbase + p;
            } else {
                const int q = d.urel[ri[mi].urel_off + j];
                if (q >= 0) idx[mi] = ri[mi].ubase + (int64_t)q * ri[mi].ldu;
            }
        }
#pragma unroll
        for (int mi = 0; mi < C::MI; ++mi)
            if (idx[mi] >= 0) {
                double *dst = reinterpret_cast<double *>(d.val + idx[mi]);
                atomicAdd(dst, flip_sign(acc[mi][ni][0]));
                atomicAdd(dst + 1, flip_sign(acc[mi][ni][1]));
            }
    }
}

template <int BM, int BNC, int WARPS_M, int WARPS_N, class LU = DeviceLU>
static int launch_schur_t(const LU &d, const Batch &b, int64_t ctas, int mode, int split_n, int split_i, cudaStream_t s)
{
    using C = ZCfg<BM, BNC, WARPS_M, WARPS_N>;
    static std::atomic<unsigned long long> attr_0{0};
    ensure_dyn_smem(schur_kernel<BM, BNC, WARPS_M, WARPS_N, LU>, (int)C::SMEM, attr_0);
    const int64_t grid = (ctas + split_n - 1) / split_n;
    schur_kernel<BM, BNC, WARPS_M, WARPS_N, LU><<<member_grid(d, (unsigned)grid), C::NT, C::SMEM, s>>>(d, b, mode, split_n, split_i);
    return 1;
}

int launch_schur(const DeviceLU &d, const Batch &b, int64_t ctas, int big, int mode, int split_n, int split_i, cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    if (big) return launch_schur_t<SCHUR_BM_BIG, SCHUR_BN_TILE, 4, 2>(d, b, ctas, mode, split_n, split_i, s);
    return launch_schur_t<SCHUR_BM_SMALL, SCHUR_BN_SMALL, 2, 2>(d, b, ctas, mode, split_n, split_i, s);
}

// batched: the default tiles of the launcher above, no Z split
int launch_schur(const BatchedLU &d, const Batch &b, int64_t ctas, int big, int mode, cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    if (big) return launch_schur_t<SCHUR_BM_BIG, SCHUR_BN_TILE, 4, 2>(d, b, ctas, mode, 1, 0, s);
    return launch_schur_t<SCHUR_BM_SMALL, SCHUR_BN_SMALL, 2, 2>(d, b, ctas, mode, 1, 0, s);
}

// plain C -= A*B with the same main loop (kernel-level test)
template <int BM, int BNC, int WARPS_M, int WARPS_N>
__global__ void __launch_bounds__(32 * WARPS_M * WARPS_N, 2)
    gemm_sub_kernel(int M, int N, int K, const zd *A, int lda, const zd *B, int ldb, zd *Cm, int ldc)
{
    using C = ZCfg<BM, BNC, WARPS_M, WARPS_N>;
    extern __shared__ double smd[];
    const int tiles_m = (M + BM - 1) / BM;
    const int m0 = (blockIdx.x % tiles_m) * BM, n0 = (blockIdx.x / tiles_m) * BNC;
    double acc[C::MI][C::NI][2];
#pragma unroll
    for (int mi = 0; mi < C::MI; ++mi)
#pragma unroll
        for (int ni = 0; ni < C::NI; ++ni) acc[mi][ni][0] = acc[mi][ni][1] = 0.0;
    zgemm_tile<BM, BNC, WARPS_M, WARPS_N>(A, lda, B, ldb, M, N, K, m0, n0, smd, acc);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm0 = m0 + (warp % WARPS_M) * C::WTM;
    const int wn0c = n0 + (((warp / WARPS_M) * C::WTN) >> 1);
#pragma unroll
    for (int ni = 0; ni < C::NI; ++ni) {
        const int j = wn0c + ni * 4 + (lane & 3);
        if (j >= N) continue;
#pragma unroll
        for (int mi = 0; mi < C::MI; ++mi) {
            const int i = wm0 + mi * 8 + (lane >> 2);
            if (i < M) {
                double *dst = reinterpret_cast<double *>(Cm + (size_t)j * ldc + i);
                atomicAdd(dst, flip_sign(acc[mi][ni][0]));
                atomicAdd(dst + 1, flip_sign(acc[mi][ni][1]));
            }
        }
    }
}

template <int BM, int BNC, int WARPS_M, int WARPS_N>
static int launch_gemm_sub_t(int m, int n, int k, const zd *a, int lda, const zd *b, int ldb, zd *c, int ldc, cudaStream_t s)
{
    using C = ZCfg<BM, BNC, WARPS_M, WARPS_N>;
    static std::atomic<unsigned long long> attr_0{0};
    ensure_dyn_smem(gemm_sub_kernel<BM, BNC, WARPS_M, WARPS_N>, (int)C::SMEM, attr_0);
    int64_t ctas = (int64_t)((m + BM - 1) / BM) * ((n + BNC - 1) / BNC);
    gemm_sub_kernel<BM, BNC, WARPS_M, WARPS_N><<<(unsigned)ctas, C::NT, C::SMEM, s>>>(m, n, k, a, lda, b, ldb, c, ldc);
    return 1;
}

int launch_gemm_sub(int m, int n, int k, const zd *a, int lda, const zd *b, int ldb, zd *c, int ldc, int variant,
                    cudaStream_t s)
{
    if (m <= 0 || n <= 0) return 0;
    if (variant != 7 && m >= 96 && n >= 96) return launch_gemm_sub_t<SCHUR_BM_BIG, SCHUR_BN_TILE, 4, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    return launch_gemm_sub_t<SCHUR_BM_SMALL, SCHUR_BN_SMALL, 2, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
}

// ------------------------------------------------------------------------------------------------
// skyline <-> dense-packed U (boundary conversions), ancestor-reduction add
// ------------------------------------------------------------------------------------------------
template <bool PACK>
__global__ void __launch_bounds__(256) u_convert_kernel(DeviceLU d, Batch b, zd *sky, const int64_t *sky_off)
{
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const int k = b.nodes[slot];
    const NodeDesc nd = d.nodes[k];
    const int chunk = (int)(blockIdx.x - b.prefix[slot]);
    const int ns = nd.ns, klst = nd.fsupc + ns;
    zd *sk = sky + sky_off[slot];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int j = chunk * 32 + warp; j < min(nd.ncols, chunk * 32 + 32); j += 8) {
        const int fst = d.ufst[nd.ucol + j], len = klst - fst, top = ns - len;
        const int64_t seg = d.useg[nd.ucol + j];
        zd *col = d.val + nd.uval + (size_t)j * ns;
        for (int r = lane; r < ns; r += 32) {
            if (PACK) { if (r >= top) sk[seg + (r - top)] = col[r]; }
            else col[r] = (r >= top) ? sk[seg + (r - top)] : zmake(0.0, 0.0);
        }
    }
}
int launch_u_convert(const DeviceLU &d, const Batch &b, int64_t ctas, int pack, zd *sky, const int64_t *sky_off,
                     cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    if (pack) u_convert_kernel<true><<<(unsigned)ctas, 256, 0, s>>>(d, b, sky, sky_off);
    else u_convert_kernel<false><<<(unsigned)ctas, 256, 0, s>>>(d, b, sky, sky_off);
    return 1;
}

__global__ void axpy_kernel(double *__restrict__ dst, const double *__restrict__ src, int64_t n)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) dst[i] += src[i];
}
int launch_axpy(zd *dst, const zd *src, int64_t n, cudaStream_t s)
{
    if (n <= 0) return 0;
    const int64_t nd2 = 2 * n;  // (re, im) pairs add component-wise
    int64_t blocks = (nd2 + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    axpy_kernel<<<(unsigned)blocks, 256, 0, s>>>(reinterpret_cast<double *>(dst), reinterpret_cast<const double *>(src), nd2);
    return 1;
}

__global__ void axpy_atomic_kernel(double *__restrict__ dst, const double *__restrict__ src, int64_t n)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) atomicAdd(dst + i, src[i]);
}
int launch_axpy_atomic(zd *dst, const zd *src, int64_t n, cudaStream_t s)
{
    if (n <= 0) return 0;
    const int64_t nd2 = 2 * n;
    int64_t blocks = (nd2 + 255) / 256;
    if (blocks > 132 * 4) blocks = 132 * 4;
    axpy_atomic_kernel<<<(unsigned)blocks, 256, 0, s>>>(reinterpret_cast<double *>(dst), reinterpret_cast<const double *>(src), nd2);
    return 1;
}

}  // namespace sluz
