// slu_selinv.cu -- selected inversion on the resident factors (slu_b200_selinv, slu_b200_selinv_get, slu_b200_logdet).
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
//
// Compiled twice, like slu_solve.cu: as is for double, and through slu_selinv_z.cu with SLU_COMPLEX for doublecomplex
// (slu_b200_z_selinv ...).  The transpose is plain in both: H = F^-T, not F^-H, so A^-1(i, j) = H(perm[j], perm[i]) holds
// unchanged.  Element arithmetic goes through the val_t helpers of slu_scalar.cuh; the complex products stay on the FP64
// DMMA pipe through the real embedding of zgemm_tile (slu_kernels_z.cu): [Ar Ai] times [[Br Bi] [-Bi Br]], the second
// factor read from the raw interleaved tile with a lane-constant swap and sign.
//
// Every kernel is templated on its DeviceLU type, as the factorization and the solve are: the BatchedLU instantiations
// (slu_b200_batch_selinv ...) run the same body over every member of a batched handle, the member in blockIdx.y.  A
// member's H arena has exactly its factors' layout, so the members' H arenas are val_stride elements apart as their
// factors are.
#include "slu_device.cuh"
#define SLU_COMMON_HELPERS_ONLY
#include "slu_kernels_common.cuh"
#include "slu_scalar.cuh"

#include <cmath>
#include <type_traits>

namespace SLU_NS {

// the member's H arena (the identity for a plain DeviceLU)
template <class T> __device__ __forceinline__ T *member_h(const DeviceLU &, T *hv) { return hv; }
template <class T> __device__ __forceinline__ T *member_h(const BatchedLU &d, T *hv) { return hv + (int64_t)blockIdx.y * d.val_stride; }

// ------------------------------------------------------------------------------------------------
// GEMM tiles on DMMA m16n8k8: 64 x 64 real output tiles (SELINV_TILE_M rows x SELINV_TILE_N val_t columns: 64 complex
// columns are 128 real ones, so the complex tile has 32), 4 warps of 32 x 32 real, k-steps of 16 real (8 complex).
// Operands are staged through registers (the M operand is a gather through the destination maps, so cp.async does not
// apply): the next k-step is loaded while the current one is multiplied.  Shared memory holds the real embedding of A
// (As[real k][row]: the real part of A(row, p) at real k = 2p, the imaginary part at 2p + 1) and B as it is stored
// (Bs[column][real k]: interleaved (re, im) in doublecomplex).
// ------------------------------------------------------------------------------------------------
constexpr int SI_RK = 16;                                  // real k per k-step
constexpr int SI_BM = SELINV_TILE_M, SI_BN = SELINV_TILE_N, SI_BK = SI_RK / VAL_DOUBLES, SI_NT = 128;
constexpr int SI_LDA = SI_BM + 4, SI_LDB = SI_RK + 4;     // doubles
constexpr int SI_PA = SI_BK * SI_BM / SI_NT, SI_PB = SI_BK * SI_BN / SI_NT;   // val_t of A / B per thread and k-step
static_assert(SI_PB <= SI_PA, "fetch / stash loop over the A elements");
static_assert(SI_BN * VAL_DOUBLES == 64 && SI_BM == 64, "4 warps of 32 x 32 real outputs");

// H(R, C) of supernode nd at (i, j): the destination of L(i) U(j) in the Schur update of nd, addressed as schur_kernel's
// epilogue addresses it
__device__ __forceinline__ val_t gather_m(const DeviceLU &d, const NodeDesc &nd, const val_t *__restrict__ hv, int i, int j)
{
    const RowInfo ri = d.rowinfo[nd.ws_row + i];
    const ColInfo cj = d.colinfo[nd.ws_col + j];
    if (ri.ib >= cj.jb) {
        const int p = d.lrel[cj.lrel_off + i];
        return p >= 0 ? hv[cj.lbase + p] : vzero();
    }
    const int q = d.urel[ri.urel_off + j];
    return q >= 0 ? hv[ri.ubase + (int64_t)q * ri.ldu] : vzero();
}

// A(r, k) into the real embedding, B(k, c) as stored
__device__ __forceinline__ void si_put_a(double *As, int k, int r, val_t v)
{
#ifdef SLU_COMPLEX
    As[(2 * k) * SI_LDA + r] = v.x;
    As[(2 * k + 1) * SI_LDA + r] = v.y;
#else
    As[k * SI_LDA + r] = v;
#endif
}
__device__ __forceinline__ void si_put_b(double *Bs, int k, int c, val_t v)
{
#ifdef SLU_COMPLEX
    *reinterpret_cast<double2 *>(Bs + c * SI_LDB + 2 * k) = v;
#else
    Bs[c * SI_LDB + k] = v;
#endif
}

// __launch_bounds__ minimum of CTAs per SM: 2 for the batched instantiations, 0 (no minimum) for the unbatched ones, which
// compile as before.  Two 128-thread CTAs leave the 255-register cap as it is; without the hint ptxas compiles the batched
// doublecomplex mode 1 at 168 registers with a 12-byte spill in the k-loop, and with it no batched product spills.
template <class LU>
constexpr int SELINV_MIN_CTAS = std::is_same<LU, BatchedLU>::value ? 2 : 0;

// MODE 0: out(i, p) = H(R,K), A(i, j) = M, B(j, p) = U_KC(p, j), inner ncols
// MODE 1: out(p, j) = H(K,C), A(p, i) = L_RK(i, p), B(i, j) = M, inner m
// MODE 2: out(p, q) = H(K,K), A(p, i) = L_RK(i, p), B(i, q) = H(R,K)(i, q), inner m
template <int MODE, class LU>
__global__ void __launch_bounds__(SI_NT, SELINV_MIN_CTAS<LU>) selinv_gemm_kernel(LU dd, Batch b, val_t *__restrict__ hv)
{
    __shared__ __align__(16) double As[SI_RK * SI_LDA];
    __shared__ __align__(16) double Bs[SI_BN * SI_LDB];
    if (blockIdx.x >= b.prefix[b.count]) return;
    const DeviceLU &d = member_view(dd);
    hv = member_h(dd, hv);
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const NodeDesc nd = d.nodes[b.nodes[slot]];
    const int ns = nd.ns, m = nd.m, nc = nd.ncols, lda = nd.nsupr;
    const int rows = MODE == 0 ? m : ns, cols = MODE == 1 ? nc : ns, K = MODE == 0 ? nc : m;
    const int tiles_r = (rows + SI_BM - 1) / SI_BM;
    const int tile = (int)(blockIdx.x - b.prefix[slot]);
    const int r0 = (tile % tiles_r) * SI_BM, c0 = (tile / tiles_r) * SI_BN;
    const val_t *__restrict__ val = d.val;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int wm = (warp & 1) * 32, wn = (warp >> 1) * 32;   // real columns

    // A(r, k) and B(k, c) of the product; zero outside the operand
    auto a_at = [&](int r, int k) -> val_t {
        if (r >= rows || k >= K) return vzero();
        if (MODE == 0) return gather_m(d, nd, hv, r, k);
        return val[nd.lval + (int64_t)r * lda + ns + k];
    };
    auto b_at = [&](int k, int c) -> val_t {
        if (k >= K || c >= cols) return vzero();
        if (MODE == 0) return val[nd.uval + (int64_t)k * ns + c];
        if (MODE == 1) return gather_m(d, nd, hv, k, c);
        return hv[nd.lval + (int64_t)c * lda + ns + k];
    };
    // element e of a k-step: the index that is contiguous in memory runs fastest over the threads
    constexpr bool A_RFAST = MODE == 0, B_CFAST = MODE == 0;
    val_t ra[SI_PA], rb[SI_PB];
    auto fetch = [&](int k0) {
#pragma unroll
        for (int s = 0; s < SI_PA; ++s) {
            const int e = tid + s * SI_NT;
            const int ar = A_RFAST ? e % SI_BM : e / SI_BK, ak = A_RFAST ? e / SI_BM : e % SI_BK;
            ra[s] = a_at(r0 + ar, k0 + ak);
            if (s >= SI_PB) continue;
            const int bc = B_CFAST ? e % SI_BN : e / SI_BK, bk = B_CFAST ? e / SI_BN : e % SI_BK;
            rb[s] = b_at(k0 + bk, c0 + bc);
        }
    };
    auto stash = [&]() {
#pragma unroll
        for (int s = 0; s < SI_PA; ++s) {
            const int e = tid + s * SI_NT;
            const int ar = A_RFAST ? e % SI_BM : e / SI_BK, ak = A_RFAST ? e / SI_BM : e % SI_BK;
            si_put_a(As, ak, ar, ra[s]);
            if (s >= SI_PB) continue;
            const int bc = B_CFAST ? e % SI_BN : e / SI_BK, bk = B_CFAST ? e / SI_BN : e % SI_BK;
            si_put_b(Bs, bk, bc, rb[s]);
        }
    };
#ifdef SLU_COMPLEX
    // the embedded B~(2p + c, 2j + e) = sgn * Bs[j][2p + (c ^ e)], sgn = -1 iff e == 0 and c == 1; this lane reads real
    // k = k8 + t (+ 4), c = t & 1, at real column 2j + e = wn + 8 nt + g, e = g & 1
    const int bsw = (t & 2) + ((t ^ g) & 1);
    const int flip = ((g & 1) == 0 && (t & 1) == 1) ? (int)0x80000000 : 0;
    auto bsgn = [&](double v) { return __hiloint2double(__double2hiint(v) ^ flip, __double2loint(v)); };
#endif

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
        for (int k8 = 0; k8 < SI_RK; k8 += 8) {
            double a[2][4], bb[4][2];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                const double *p = As + (k8 + t) * SI_LDA + wm + 16 * mt + g;
                a[mt][0] = p[0]; a[mt][1] = p[8]; a[mt][2] = p[4 * SI_LDA]; a[mt][3] = p[4 * SI_LDA + 8];
            }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
#ifdef SLU_COMPLEX
                const double *p = Bs + (((wn + 8 * nt + g) >> 1) * SI_LDB) + k8 + bsw;
                bb[nt][0] = bsgn(p[0]); bb[nt][1] = bsgn(p[4]);
#else
                const double *p = Bs + (wn + 8 * nt + g) * SI_LDB + k8 + t;
                bb[nt][0] = p[0]; bb[nt][1] = p[4];
#endif
            }
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) dmma1688(acc[mt][nt], a[mt], bb[nt]);
        }
        __syncthreads();
    }
    // lane (g, t) holds rows g, g + 8 and real columns 2t, 2t + 1 of each 16 x 8 piece: in doublecomplex the (re, im) of
    // complex column t of its 16 x 4 piece
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#ifdef SLU_COMPLEX
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = r0 + wm + 16 * mt + g + 8 * h, c = c0 + (wn >> 1) + 4 * nt + t;
                if (r >= rows || c >= cols) continue;
                const val_t v = zmake(-acc[mt][nt][2 * h], -acc[mt][nt][2 * h + 1]);
                if (MODE == 0) hv[nd.lval + (int64_t)c * lda + ns + r] = v;
                else if (MODE == 1) hv[nd.uval + (int64_t)c * ns + r] = v;
                else hv[nd.lval + (int64_t)c * lda + r] = zmake((r == c ? 1.0 : 0.0) + v.x, v.y);
            }
#else
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = r0 + wm + 16 * mt + g + 8 * (e >> 1), c = c0 + wn + 8 * nt + 2 * t + (e & 1);
                if (r >= rows || c >= cols) continue;
                const double v = -acc[mt][nt][e];
                if (MODE == 0) hv[nd.lval + (int64_t)c * lda + ns + r] = v;
                else if (MODE == 1) hv[nd.uval + (int64_t)c * ns + r] = v;
                else hv[nd.lval + (int64_t)c * lda + r] = (r == c ? 1.0 : 0.0) + v;
            }
#endif
}

// ------------------------------------------------------------------------------------------------
// In-place back substitution with an upper triangular T of the supernode's diagonal block, one vector per thread, 16
// unknowns at a time: the already solved unknowns are subtracted, giving R, then the 16 x 16 block inverse of
// diag_inv_kernel is applied and corrected once, Z = inv R + inv (R - T_jj (inv R)), as trsm_kernel does.  COLS = 0: the
// rows x of L panel K of H, T = U_KK (x <- x U_KK^-T, i.e. U_KK x^T = x^T); COLS = 1: the ns columns of H(K,K) and the
// ncols columns of H(K,C), T = L_KK^T (unit; its block inverse is inv(L_bb) read transposed).  In doublecomplex the
// block inverses and T_jj are read transposed exactly as in double, never conjugated.
// ------------------------------------------------------------------------------------------------
// The minimum of one CTA per SM only changes ptxas's register target: without it the correction step's 32 live values
// spilled in the batched double COLS = 0 and doublecomplex COLS = 1 instantiations.
template <int COLS, class LU>
__global__ void __launch_bounds__(SELINV_VECS, 1) selinv_trsm_kernel(LU dd, Batch b, const val_t *__restrict__ dinv,
                                                                   val_t *__restrict__ hv)
{
    if (blockIdx.x >= b.prefix[b.count]) return;
    const DeviceLU &d = member_view(dd);
    dinv = member_inv(dd, dinv);
    hv = member_h(dd, hv);
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const NodeDesc nd = d.nodes[b.nodes[slot]];
    const int ns = nd.ns, lda = nd.nsupr;
    const int v = (int)(blockIdx.x - b.prefix[slot]) * SELINV_VECS + threadIdx.x;
    if (v >= (COLS ? ns + nd.ncols : lda)) return;
    val_t *x;
    int64_t stride;
    if (!COLS) { x = hv + nd.lval + v; stride = lda; }
    else if (v < ns) { x = hv + nd.lval + (int64_t)v * lda; stride = 1; }
    else { x = hv + nd.uval + (int64_t)(v - ns) * ns; stride = 1; }
    const val_t *__restrict__ D = d.val + nd.lval;          // the diagonal block, column-major with lda
    const val_t *__restrict__ inv = dinv + nd.ws_inv;
    for (int blk = (ns - 1) / 16; blk >= 0; --blk) {
        const int p0 = blk * 16, w = min(16, ns - p0);
        val_t acc[16];
#pragma unroll
        for (int r = 0; r < 16; ++r) acc[r] = r < w ? x[(int64_t)(p0 + r) * stride] : vzero();
        for (int q = p0 + w; q < ns; ++q) {
            const val_t z = x[(int64_t)q * stride];
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                if (r >= w) break;
                const val_t tv = COLS ? D[(int64_t)(p0 + r) * lda + q] : D[(int64_t)q * lda + p0 + r];
                acc[r] = vfnma(tv, z, acc[r]);
            }
        }
        // Z = inv R, then one correction step Z += inv (R - T_jj Z) with the block's own entries (unit diagonal for
        // L_KK^T): the product with the explicit inverse alone has a backward error that grows with cond(T_jj)
        const val_t *bi = inv + (size_t)blk * 512 + (COLS ? 256 : 0);
        auto tjj = [&](int r, int c) -> val_t {      // T_jj(r, c), c > r
            return COLS ? D[(int64_t)(p0 + r) * lda + p0 + c] : D[(int64_t)(p0 + c) * lda + p0 + r];
        };
        val_t z[16];
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            z[r] = vzero();
            if (r >= w) continue;
#pragma unroll
            for (int c = 0; c < 16; ++c) z[r] = vfma(COLS ? bi[r * 16 + c] : bi[c * 16 + r], acc[c], z[r]);
        }
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            if (r >= w) break;
            val_t s = COLS ? vsub(acc[r], z[r]) : vfnma(D[(int64_t)(p0 + r) * lda + p0 + r], z[r], acc[r]);
#pragma unroll
            for (int c = r + 1; c < 16; ++c) {
                if (c >= w) break;
                s = vfnma(tjj(r, c), z[c], s);
            }
            acc[r] = s;
        }
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            if (r >= w) break;
            val_t y = z[r];
#pragma unroll
            for (int c = 0; c < 16; ++c) y = vfma(COLS ? bi[r * 16 + c] : bi[c * 16 + r], acc[c], y);
            x[(int64_t)(p0 + r) * stride] = y;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// log |det| and its phase: one supernode per thread, fixed-order reductions (no float atomics).  The phase is the number
// of negative pivots in double and the sum of the pivots' arguments in doublecomplex, kept reduced modulo 2 pi.
// ------------------------------------------------------------------------------------------------
#ifdef SLU_COMPLEX
constexpr double SI_TWO_PI = 6.283185307179586;
__device__ __forceinline__ double si_wrap(double th) { return remainder(th, SI_TWO_PI); }
#endif

__device__ __forceinline__ void si_block_reduce(double &s, phase_t &ph)
{
    __shared__ double ss[SELINV_VECS / 32];
    __shared__ phase_t sn[SELINV_VECS / 32];
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_down_sync(0xffffffffu, s, o);
        ph += __shfl_down_sync(0xffffffffu, ph, o);
    }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { ss[w] = s; sn[w] = ph; }
    __syncthreads();
    if (threadIdx.x == 0) {
        s = 0.0; ph = 0;
        for (int i = 0; i < SELINV_VECS / 32; ++i) { s += ss[i]; ph += sn[i]; }
    }
}

// batched: grid (nparts, members), member j's partials at j * nparts
template <class LU>
__global__ void __launch_bounds__(SELINV_VECS) selinv_logdet_partial_kernel(LU dd, const int32_t *nodes, int count, double *part,
                                                                            phase_t *pph)
{
    const DeviceLU &d = member_view(dd);
    part = member_ptr(dd, part, gridDim.x);
    pph = member_ptr(dd, pph, gridDim.x);
    const int t = blockIdx.x * SELINV_VECS + threadIdx.x;
    double s = 0.0;
    phase_t ph = 0;
    if (t < count) {
        const NodeDesc nd = d.nodes[nodes[t]];
        const val_t *D = d.val + nd.lval;
        for (int i = 0; i < nd.ns; ++i) {
            const val_t p = D[(int64_t)i * nd.nsupr + i];
#ifdef SLU_COMPLEX
            s += log(hypot(p.x, p.y));
            ph += atan2(p.y, p.x);
#else
            s += log(fabs(p));
            ph += p < 0.0;
#endif
        }
#ifdef SLU_COMPLEX
        ph = si_wrap(ph);
#endif
    }
    si_block_reduce(s, ph);
#ifdef SLU_COMPLEX
    ph = si_wrap(ph);
#endif
    if (threadIdx.x == 0) { part[blockIdx.x] = s; pph[blockIdx.x] = ph; }
}

// out[0] = log |det|; double: out[1] = the sign; doublecomplex: out[1], out[2] = exp(i theta).  MEMBERS: grid (1, members),
// member j's partials at j * nparts and its result at out + j * (1 + VAL_DOUBLES)
template <bool MEMBERS>
__global__ void __launch_bounds__(SELINV_VECS) selinv_logdet_final_kernel(const double *part, const phase_t *pph, int nparts, double *out)
{
    if (MEMBERS) {
        part += (size_t)blockIdx.y * nparts;
        pph += (size_t)blockIdx.y * nparts;
        out += (size_t)blockIdx.y * (1 + VAL_DOUBLES);
    }
    double s = 0.0;
    phase_t ph = 0;
    for (int i = threadIdx.x; i < nparts; i += SELINV_VECS) { s += part[i]; ph += pph[i]; }
    si_block_reduce(s, ph);
#ifdef SLU_COMPLEX
    if (threadIdx.x == 0) {
        const double th = si_wrap(ph);
        out[0] = s; out[1] = cos(th); out[2] = sin(th);
    }
#else
    if (threadIdx.x == 0) { out[0] = s; out[1] = (ph & 1) ? -1.0 : 1.0; }
#endif
}

// ------------------------------------------------------------------------------------------------
// Inertia: the signs of the pivots, one supernode per thread as in the logdet reduction.  Integer counts (negative real
// part, the others, |u_ii| <= thresh) and the max of |Im u_ii| / |u_ii|, reduced in a fixed order without atomics.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void inertia_block_reduce(long long (&c)[3], double &def)
{
    __shared__ long long sc[SELINV_VECS / 32][3];
    __shared__ double sd[SELINV_VECS / 32];
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int q = 0; q < 3; ++q) c[q] += __shfl_down_sync(0xffffffffu, c[q], o);
        def = fmax(def, __shfl_down_sync(0xffffffffu, def, o));
    }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
        for (int q = 0; q < 3; ++q) sc[w][q] = c[q];
        sd[w] = def;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        c[0] = c[1] = c[2] = 0;
        def = 0.0;
        for (int i = 0; i < SELINV_VECS / 32; ++i) {
            for (int q = 0; q < 3; ++q) c[q] += sc[i][q];
            def = fmax(def, sd[i]);
        }
    }
}

// batched: grid (nparts, members), member j's partials at j * nparts (counts: 3 per partial)
template <class LU>
__global__ void __launch_bounds__(SELINV_VECS) inertia_partial_kernel(LU dd, const int32_t *nodes, int count, double thresh,
                                                                      long long *pcnt, double *pdef)
{
    const DeviceLU &d = member_view(dd);
    pcnt = member_ptr(dd, pcnt, 3 * gridDim.x);
    pdef = member_ptr(dd, pdef, gridDim.x);
    const int t = blockIdx.x * SELINV_VECS + threadIdx.x;
    long long c[3] = {0, 0, 0};
    double def = 0.0;
    if (t < count) {
        const NodeDesc nd = d.nodes[nodes[t]];
        const val_t *D = d.val + nd.lval;
        for (int i = 0; i < nd.ns; ++i) {
            const val_t p = D[(int64_t)i * nd.nsupr + i];
#ifdef SLU_COMPLEX
            const double a = hypot(p.x, p.y), re = p.x;
            if (a > 0.0) def = fmax(def, fabs(p.y) / a);
#else
            const double a = fabs(p), re = p;
#endif
            c[0] += re < 0.0;
            c[2] += a <= thresh;
        }
        c[1] = nd.ns - c[0];
    }
    inertia_block_reduce(c, def);
    if (threadIdx.x == 0) {
        for (int q = 0; q < 3; ++q) pcnt[3 * blockIdx.x + q] = c[q];
        pdef[blockIdx.x] = def;
    }
}

// grid (1, members): member j's partials at j * nparts, its counts at cnt + 3 j and its defect at def[j]
__global__ void __launch_bounds__(SELINV_VECS) inertia_final_kernel(const long long *pcnt, const double *pdef, int nparts,
                                                                    long long *cnt, double *def)
{
    pcnt += (size_t)blockIdx.y * 3 * nparts;
    pdef += (size_t)blockIdx.y * nparts;
    long long c[3] = {0, 0, 0};
    double m = 0.0;
    for (int i = threadIdx.x; i < nparts; i += SELINV_VECS) {
        for (int q = 0; q < 3; ++q) c[q] += pcnt[3 * i + q];
        m = fmax(m, pdef[i]);
    }
    inertia_block_reduce(c, m);
    if (threadIdx.x == 0) {
        for (int q = 0; q < 3; ++q) cnt[3 * blockIdx.y + q] = c[q];
        def[blockIdx.y] = m;
    }
}

// ------------------------------------------------------------------------------------------------
// out[p] = A^-1(i, colind[p]) = H(perm[colind[p]], perm[i]): the slot search of fill_csr_kernel with the roles of row and
// column swapped, reading instead of writing.  One thread per row of the pattern.  Batched: member j's values at
// out + j * nnz; a missing slot depends on the structure only, so only member 0 counts it.
// ------------------------------------------------------------------------------------------------
template <class LU>
__global__ void selinv_get_kernel(LU dd, const val_t *__restrict__ hv, int n, const int32_t *__restrict__ rowptr,
                                  const int32_t *__restrict__ colind, const int32_t *__restrict__ perm, val_t *__restrict__ out,
                                  int *err)
{
    constexpr bool BATCHED = std::is_same<LU, BatchedLU>::value;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const DeviceLU &d = member_view(dd);
    hv = member_h(dd, hv);
    if (BATCHED) out += (int64_t)blockIdx.y * rowptr[n];
    const bool count = !BATCHED || blockIdx.y == 0;
    const int pj = perm[i];                       // column of H
    const int ks = d.supno[pj];
    for (int p = rowptr[i]; p < rowptr[i + 1]; ++p) {
        const int pi = perm[colind[p]];           // row of H
        val_t v = vnan();
        if (pi >= d.xsup[ks]) {                   // L panel of block column supno(pj), diagonal block included
            const NodeDesc *nd = d.nodes + ks;
            const int32_t *srow = d.lsrow + nd->lrow;
            const int q = lower_bound_i32(srow, nd->nsupr, pi);
            if (q < nd->nsupr && srow[q] == pi) v = hv[nd->lval + (int64_t)(pj - nd->fsupc) * nd->nsupr + d.lspos[nd->lrow + q]];
            else if (count) atomicAdd(err, 1);
        } else {                                  // U panel of block row supno(pi)
            const NodeDesc *nd = d.nodes + d.supno[pi];
            const int32_t *uc = d.ucols + nd->ucol;
            const int q = lower_bound_i32(uc, nd->ncols, pj);
            if (q < nd->ncols && uc[q] == pj) v = hv[nd->uval + (int64_t)q * nd->ns + (pi - nd->fsupc)];
            else if (count) atomicAdd(err, 1);
        }
        out[p] = v;
    }
}

// ------------------------------------------------------------------------------------------------
// The batched launchers make exactly the launches of the unbatched ones, with gridDim.y = members.
template <class LU>
static int launch_selinv_gemm_t(const LU &d, const Batch &b, int64_t ctas, int mode, val_t *hv, cudaStream_t s)
{
    if (b.count <= 0) return 0;
    const dim3 grid = member_grid(d, (unsigned)(ctas > 0 ? ctas : 1));   // an empty batch still makes its launch: the count stays fixed
    if (mode == 0) selinv_gemm_kernel<0, LU><<<grid, SI_NT, 0, s>>>(d, b, hv);
    else if (mode == 1) selinv_gemm_kernel<1, LU><<<grid, SI_NT, 0, s>>>(d, b, hv);
    else selinv_gemm_kernel<2, LU><<<grid, SI_NT, 0, s>>>(d, b, hv);
    return 1;
}

template <class LU>
static int launch_selinv_trsm_t(const LU &d, const Batch &b, int64_t ctas, int cols, const val_t *dinv, val_t *hv, cudaStream_t s)
{
    if (b.count <= 0) return 0;
    const dim3 grid = member_grid(d, (unsigned)(ctas > 0 ? ctas : 1));
    if (cols) selinv_trsm_kernel<1, LU><<<grid, SELINV_VECS, 0, s>>>(d, b, dinv, hv);
    else selinv_trsm_kernel<0, LU><<<grid, SELINV_VECS, 0, s>>>(d, b, dinv, hv);
    return 1;
}

template <class LU>
static int launch_selinv_logdet_t(const LU &d, const int32_t *nodes, int count, double *part, phase_t *pph, double *out, cudaStream_t s)
{
    const int nparts = (count + SELINV_VECS - 1) / SELINV_VECS;
    if (nparts <= 0) return 0;
    selinv_logdet_partial_kernel<LU><<<member_grid(d, nparts), SELINV_VECS, 0, s>>>(d, nodes, count, part, pph);
    selinv_logdet_final_kernel<std::is_same<LU, BatchedLU>::value><<<member_grid(d, 1), SELINV_VECS, 0, s>>>(part, pph, nparts, out);
    return 2;
}

template <class LU>
static int launch_inertia_t(const LU &d, const int32_t *nodes, int count, double thresh, long long *pcnt, double *pdef,
                            long long *cnt, double *def, cudaStream_t s)
{
    const int nparts = (count + SELINV_VECS - 1) / SELINV_VECS;
    if (nparts <= 0) return 0;
    inertia_partial_kernel<LU><<<member_grid(d, nparts), SELINV_VECS, 0, s>>>(d, nodes, count, thresh, pcnt, pdef);
    inertia_final_kernel<<<member_grid(d, 1), SELINV_VECS, 0, s>>>(pcnt, pdef, nparts, cnt, def);
    return 2;
}

template <class LU>
static int launch_selinv_get_t(const LU &d, const val_t *hv, int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm,
                               val_t *out, int *err, cudaStream_t s)
{
    if (n <= 0) return 0;
    selinv_get_kernel<LU><<<member_grid(d, (n + 127) / 128), 128, 0, s>>>(d, hv, n, rowptr, colind, perm, out, err);
    return 1;
}

int launch_selinv_gemm(const DeviceLU &d, const Batch &b, int64_t ctas, int mode, val_t *hv, cudaStream_t s)
{
    return launch_selinv_gemm_t(d, b, ctas, mode, hv, s);
}
int launch_selinv_trsm(const DeviceLU &d, const Batch &b, int64_t ctas, int cols, const val_t *dinv, val_t *hv, cudaStream_t s)
{
    return launch_selinv_trsm_t(d, b, ctas, cols, dinv, hv, s);
}
int launch_selinv_logdet(const DeviceLU &d, const int32_t *nodes, int count, double *part, phase_t *pph, double *out, cudaStream_t s)
{
    return launch_selinv_logdet_t(d, nodes, count, part, pph, out, s);
}
int launch_selinv_get(const DeviceLU &d, const val_t *hv, int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm,
                      val_t *out, int *err, cudaStream_t s)
{
    return launch_selinv_get_t(d, hv, n, rowptr, colind, perm, out, err, s);
}
int launch_selinv_gemm(const BatchedLU &d, const Batch &b, int64_t ctas, int mode, val_t *hv, cudaStream_t s)
{
    return launch_selinv_gemm_t(d, b, ctas, mode, hv, s);
}
int launch_selinv_trsm(const BatchedLU &d, const Batch &b, int64_t ctas, int cols, const val_t *dinv, val_t *hv, cudaStream_t s)
{
    return launch_selinv_trsm_t(d, b, ctas, cols, dinv, hv, s);
}
int launch_selinv_logdet(const BatchedLU &d, const int32_t *nodes, int count, double *part, phase_t *pph, double *out, cudaStream_t s)
{
    return launch_selinv_logdet_t(d, nodes, count, part, pph, out, s);
}
int launch_selinv_get(const BatchedLU &d, const val_t *hv, int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm,
                      val_t *out, int *err, cudaStream_t s)
{
    return launch_selinv_get_t(d, hv, n, rowptr, colind, perm, out, err, s);
}
int launch_inertia(const DeviceLU &d, const int32_t *nodes, int count, double thresh, long long *pcnt, double *pdef, long long *cnt,
                   double *def, cudaStream_t s)
{
    return launch_inertia_t(d, nodes, count, thresh, pcnt, pdef, cnt, def, s);
}
int launch_inertia(const BatchedLU &d, const int32_t *nodes, int count, double thresh, long long *pcnt, double *pdef, long long *cnt,
                   double *def, cudaStream_t s)
{
    return launch_inertia_t(d, nodes, count, thresh, pcnt, pdef, cnt, def, s);
}

}  // namespace SLU_NS
