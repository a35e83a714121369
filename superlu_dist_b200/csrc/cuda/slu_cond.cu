// slu_cond.cu -- 1-norm condition estimation on the resident factors (slu_b200_gscon and its twins): the device side of
// LAPACK's dlacn2 / zlacn2 reverse-communication estimator, as dgecon / zgecon and sequential SuperLU's dgscon / zgscon
// drive it.  The host runs one solve (slu_api.cu) per round and then the three step kernels below; every n-vector stays
// in HBM.  gridDim.y = member: a batched handle estimates all its members in lock-step, and a member whose next kase is
// not the one of the round keeps its pending vector (CondState::kase tells which members consume the round's result).
//
// Deterministic by construction, so that every run and every rank of a Z group takes the same decisions: per-CTA
// partials in a fixed order (cond_partials_kernel), then one CTA per member reduces them in a fixed order
// (cond_finalize_kernel); no floating-point atomics.
//
// Compiled twice, like slu_solve.cu: as is for double, and through slu_cond_z.cu with SLU_COMPLEX for doublecomplex
// (zlacn2: |x_i| is the modulus, the sign vector is x_i / |x_i|, and there is no repeated-sign test).
#include "slu_device.cuh"
#include "slu_scalar.cuh"

#include <cfloat>
#include <climits>

namespace SLU_NS {

constexpr int COND_THREADS = 256;
constexpr int COND_PER_THREAD = COND_CHUNK / COND_THREADS;
constexpr int COND_ITMAX = 5;   // dlacn2 ITMAX

#ifdef SLU_COMPLEX
__device__ __forceinline__ double cabs_(val_t a) { return hypot(a.x, a.y); }
__device__ __forceinline__ val_t cond_sign(val_t a)      // zlacn2: x / |x|, or 1 where |x| <= safmin
{
    const double r = cabs_(a);
    return r > DBL_MIN ? zmake(a.x / r, a.y / r) : zmake(1.0, 0.0);
}
__device__ __forceinline__ val_t cond_real(double r) { return zmake(r, 0.0); }
#else
__device__ __forceinline__ double cabs_(val_t a) { return fabs(a); }
__device__ __forceinline__ val_t cond_sign(val_t a) { return a >= 0.0 ? 1.0 : -1.0; }   // dlacn2: x >= 0 -> +1
__device__ __forceinline__ val_t cond_real(double r) { return r; }
#endif

// the larger |x_i|; on a tie the lower index (idamax / izmax1)
__device__ __forceinline__ void cond_max(double &v, int &i, double v2, int i2)
{
    if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}

// block-wide reduction in a fixed order: warp shuffles, then warp 0 over the warps' results
__device__ __forceinline__ void cond_block_reduce(double &sum, double &mv, int &mi, int &diff)
{
    __shared__ double s_sum[COND_THREADS / 32], s_mv[COND_THREADS / 32];
    __shared__ int s_mi[COND_THREADS / 32], s_diff[COND_THREADS / 32];
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_down_sync(0xffffffffu, sum, o);
        diff += __shfl_down_sync(0xffffffffu, diff, o);
        cond_max(mv, mi, __shfl_down_sync(0xffffffffu, mv, o), __shfl_down_sync(0xffffffffu, mi, o));
    }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { s_sum[w] = sum; s_mv[w] = mv; s_mi[w] = mi; s_diff[w] = diff; }
    __syncthreads();
    if (w == 0) {
        const bool on = lane < COND_THREADS / 32;
        sum = on ? s_sum[lane] : 0.0;
        mv = on ? s_mv[lane] : -1.0;
        mi = on ? s_mi[lane] : INT_MAX;
        diff = on ? s_diff[lane] : 0;
        for (int o = 16; o > 0; o >>= 1) {
            sum += __shfl_down_sync(0xffffffffu, sum, o);
            diff += __shfl_down_sync(0xffffffffu, diff, o);
            cond_max(mv, mi, __shfl_down_sync(0xffffffffu, mv, o), __shfl_down_sync(0xffffffffu, mi, o));
        }
    }
}

// dlacn2's first call: x = (1/n, ..., 1/n), kase 1
__global__ void __launch_bounds__(COND_THREADS) cond_init_kernel(CondState *st, val_t *v, int n)
{
    const int m = blockIdx.y;
    val_t *vm = v + (size_t)m * n;
    const int i0 = blockIdx.x * COND_CHUNK + threadIdx.x;
    for (int k = 0; k < COND_PER_THREAD; ++k) {
        const int i = i0 + k * COND_THREADS;
        if (i < n) vm[i] = cond_real(1.0 / n);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        CondState s{};
        s.phase = 1;
        s.kase = 1;
        st[m] = s;
    }
}

// per chunk of the result of the members that consume this round: sum |x_i|, max |x_i| with its lowest index, and (real,
// after an e_j solve) how many signs differ from the last sign vector
__global__ void __launch_bounds__(COND_THREADS) cond_partials_kernel(const CondState *st, int kase, const val_t *x, const val_t *sgn,
                                                                      int n, CondPart *part)
{
    const int m = blockIdx.y;
    const CondState s = st[m];
    if (s.kase != kase) return;
    const val_t *xm = x + (size_t)m * n;
#ifndef SLU_COMPLEX
    const val_t *sm = sgn + (size_t)m * n;
#endif
    double sum = 0.0, mv = -1.0;
    int mi = INT_MAX, diff = 0;
    const int i0 = blockIdx.x * COND_CHUNK + threadIdx.x;
    for (int k = 0; k < COND_PER_THREAD; ++k) {
        const int i = i0 + k * COND_THREADS;
        if (i >= n) break;
        const val_t xi = xm[i];
        const double a = cabs_(xi);
        sum += a;
        cond_max(mv, mi, a, i);
#ifndef SLU_COMPLEX
        if (s.phase == 3) diff += cond_sign(xi) != sm[i];
#endif
    }
    cond_block_reduce(sum, mv, mi, diff);
    if (threadIdx.x == 0) part[(size_t)m * gridDim.x + blockIdx.x] = CondPart{sum, mv, mi, diff};
}

// one CTA per member: reduce its partials in chunk order, then one step of dlacn2 / zlacn2 (thread 0).  Every member
// counts the kase it waits for into counts[0] / counts[1] (integer atomics).
__global__ void __launch_bounds__(COND_THREADS) cond_finalize_kernel(CondState *st, int kase, const val_t *x, int n, const CondPart *part,
                                                                      int nchunks, int *counts)
{
    const int m = blockIdx.x;
    CondState s = st[m];
    const bool mine = s.kase == kase;
    double sum = 0.0, mv = -1.0;
    int mi = INT_MAX, diff = 0;
    if (mine)
        for (int c = threadIdx.x; c < nchunks; c += COND_THREADS) {
            const CondPart p = part[(size_t)m * nchunks + c];
            sum += p.sum;
            diff += p.diff;
            cond_max(mv, mi, p.maxv, p.maxi);
        }
    cond_block_reduce(sum, mv, mi, diff);
    if (threadIdx.x != 0) return;
    s.act = COND_NONE;
    if (mine) {
        const int j = mi < n ? mi : 0;          // NaN everywhere: no maximum (the estimate is not finite anyway)
        bool alt = false;
        switch (s.phase) {
        case 1:                                 // x = B (1/n): the first estimate
            if (n == 1) { s.est = sum; s.kase = 0; break; }
            s.est = sum;
            s.act = COND_SIGN; s.kase = 2; s.phase = 2;
            break;
        case 2:                                 // x = B^T sign(B (1/n))
            s.j = j; s.iter = 2;
            s.act = COND_EJ; s.kase = 1; s.phase = 3;
            break;
        case 3:                                 // x = B e_j
            s.estold = s.est;
            s.est = sum;
#ifndef SLU_COMPLEX
            if (diff == 0) { alt = true; break; }   // repeated sign vector: converged
#endif
            if (s.est <= s.estold) { alt = true; break; }   // no increase: cycling
            s.act = COND_SIGN; s.kase = 2; s.phase = 4;
            break;
        case 4: {                               // x = B^T sign(B e_j)
            const int jlast = s.j;
            s.j = j;
#ifdef SLU_COMPLEX
            const double xl = cabs_(x[(size_t)m * n + jlast]);
#else
            const double xl = x[(size_t)m * n + jlast];   // dlacn2 compares the signed entry with the maximum
#endif
            if (xl != mv && s.iter < COND_ITMAX) {
                ++s.iter;
                s.act = COND_EJ; s.kase = 1; s.phase = 3;
            } else {
                alt = true;
            }
            break;
        }
        case 5: {                               // x = B (alternating vector)
            const double t = 2.0 * (sum / (3.0 * n));
            if (t > s.est) s.est = t;
            s.kase = 0;
            break;
        }
        }
        if (alt) { s.act = COND_ALT; s.kase = 1; s.phase = 5; }
    }
    st[m] = s;                                  // act = COND_NONE for a member that waits: cond_next leaves its vector alone
    if (s.kase) atomicAdd(counts + s.kase - 1, 1);
}

// the next vector of every member that consumed this round: e_j, the sign vector of x (kept in sgn for the real
// repeated-sign test) or the alternating vector (-1)^i (1 + i / (n - 1))
__global__ void __launch_bounds__(COND_THREADS) cond_next_kernel(const CondState *st, const val_t *x, val_t *v, val_t *sgn, int n)
{
    const int m = blockIdx.y;
    const CondState s = st[m];
    if (s.act == COND_NONE) return;
    const size_t off = (size_t)m * n;
    const int i0 = blockIdx.x * COND_CHUNK + threadIdx.x;
    for (int k = 0; k < COND_PER_THREAD; ++k) {
        const int i = i0 + k * COND_THREADS;
        if (i >= n) break;
        val_t r;
        if (s.act == COND_EJ) {
            r = cond_real(i == s.j ? 1.0 : 0.0);
        } else if (s.act == COND_SIGN) {
            r = cond_sign(x[off + i]);
#ifndef SLU_COMPLEX
            sgn[off + i] = r;
#endif
        } else {
            r = cond_real((i & 1 ? -1.0 : 1.0) * (1.0 + (double)i / (double)(n - 1)));
        }
        v[off + i] = r;
    }
}

// ---- the loop on the device (gscon_device, gsrfs_device's ferr): conditional graph nodes in place of the host's reads ----

// after a round (first = 0): the next kase by the host loop's rule (the other kase if a member waits for it, else the same
// one if a member waits for it, else 0) and one round more; first = 1: kase 1, 0 rounds.  The WHILE handle w continues while
// a kase is left and fewer than max_rounds rounds ran (the host loop fails there; the members still waiting get NaN).
__global__ void cond_continue_kernel(const int *counts, int *loop, int first, int max_rounds, cudaGraphConditionalHandle w)
{
    int kase = 1, rounds = 0;
    if (!first) {
        kase = loop[0];
        rounds = loop[1] + 1;
        if (counts[2 - kase] > 0) kase = 3 - kase;
        else if (counts[kase - 1] == 0) kase = 0;
    }
    loop[0] = kase;
    loop[1] = rounds;
    cudaGraphSetConditional(w, kase != 0 && rounds < max_rounds ? 1u : 0u);
}

// at the head of each round: the IF node of the round's kase runs
__global__ void cond_select_kernel(const int *loop, cudaGraphConditionalHandle k1, cudaGraphConditionalHandle k2)
{
    cudaGraphSetConditional(k1, loop[0] == 1 ? 1u : 0u);
    cudaGraphSetConditional(k2, loop[0] == 2 ? 1u : 0u);
}

// one thread per member: rcond as gscon's host side: anorm 0 or +inf -> 0, (1 / est) / anorm where est is finite and not 0,
// else 0.  NaN where the member's status is not 0, anorm is negative or NaN (which the host call refuses), or the estimate
// stopped at the round cap.
__global__ void __launch_bounds__(COND_THREADS) cond_rcond_kernel(const CondState *st, const double *anorm, const int32_t *status, int members,
                                                                  double *rcond)
{
    const int m = blockIdx.x * COND_THREADS + threadIdx.x;
    if (m >= members) return;
    const double a = anorm[m], q = __longlong_as_double(0x7ff8000000000000LL);
    const CondState s = st[m];
    double r;
    if (status[m] != 0 || !(a >= 0.0)) r = q;
    else if (a == 0.0 || isinf(a)) r = 0.0;
    else if (s.kase != 0) r = q;
    else r = isfinite(s.est) && s.est != 0.0 ? (1.0 / s.est) / a : 0.0;
    rcond[m] = r;
}

int launch_cond_continue(const int *counts, int *loop, int first, int max_rounds, cudaGraphConditionalHandle w, cudaStream_t s)
{
    cond_continue_kernel<<<1, 1, 0, s>>>(counts, loop, first, max_rounds, w);
    return 1;
}

int launch_cond_select(const int *loop, cudaGraphConditionalHandle k1, cudaGraphConditionalHandle k2, cudaStream_t s)
{
    cond_select_kernel<<<1, 1, 0, s>>>(loop, k1, k2);
    return 1;
}

int launch_cond_rcond(const CondState *st, const double *anorm, const int32_t *status, int members, double *rcond, cudaStream_t s)
{
    cond_rcond_kernel<<<(members + COND_THREADS - 1) / COND_THREADS, COND_THREADS, 0, s>>>(st, anorm, status, members, rcond);
    return 1;
}

int launch_cond_init(CondState *st, val_t *v, int n, int members, cudaStream_t s)
{
    cond_init_kernel<<<dim3((n + COND_CHUNK - 1) / COND_CHUNK, members), COND_THREADS, 0, s>>>(st, v, n);
    return 1;
}

int launch_cond_step(CondState *st, int kase, const val_t *x, val_t *v, val_t *sgn, CondPart *part, int *counts, int n, int members,
                     cudaStream_t s)
{
    const int nchunks = (n + COND_CHUNK - 1) / COND_CHUNK;
    const dim3 grid(nchunks, members);
    cond_partials_kernel<<<grid, COND_THREADS, 0, s>>>(st, kase, x, sgn, n, part);
    cond_finalize_kernel<<<members, COND_THREADS, 0, s>>>(st, kase, x, n, part, nchunks, counts);
    cond_next_kernel<<<grid, COND_THREADS, 0, s>>>(st, x, v, sgn, n);
    return 3;
}

}  // namespace SLU_NS
