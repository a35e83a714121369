// slu_refine.cu -- iterative refinement with error bounds on the resident factors (slu_b200_gsrfs and its twins): the
// device side of pdgsrfs's loop (SRC/double/pdgsrfs.c:198-251) and of the forward error bound of LAPACK dgerfs.  The host
// (slu_api.cu) runs the scaled solve of the residual between the residual / decide kernels and the update; the stopping
// state of every column stays in HBM.  Every kernel runs over (rows, members) with gridDim.y = member; a member's nrhs
// columns are consecutive blocks of n elements, so column c = member * nrhs + j of the state arrays is block c of a vector.
//
// The residual is deterministic: one thread per (row, column, member) walks the row's entries in CSR order with unfused,
// rounded multiplies and adds, and the per-column maximum is an integer atomicMax on the bit patterns of non-negative
// doubles (as the equilibration's maxima).  berr is therefore a pure function of (A, b, x).
//
// Compiled twice, like slu_cond.cu: as is for double, and through slu_refine_z.cu with SLU_COMPLEX for doublecomplex,
// where |.| is cabs1 = |re| + |im| (pzgsrfs, zgerfs).
#include "slu_device.cuh"
#include "slu_scalar.cuh"

#include <cfloat>

namespace SLU_NS {

constexpr int REF_THREADS = 256;
constexpr double REF_EPS = DBL_EPSILON / 2;   // dmach("Epsilon"): the unit roundoff 2^-53

__device__ __forceinline__ unsigned long long ref_bits(double v) { return (unsigned long long)__double_as_longlong(v); }

#ifdef SLU_COMPLEX
__device__ __forceinline__ double ref_abs1(val_t a) { return __dadd_rn(fabs(a.x), fabs(a.y)); }
// acc + a * x: four rounded products, two rounded sums for the product, then two rounded sums into acc
__device__ __forceinline__ val_t ref_addmul(val_t acc, val_t a, val_t x)
{
    const double re = __dsub_rn(__dmul_rn(a.x, x.x), __dmul_rn(a.y, x.y));
    const double im = __dadd_rn(__dmul_rn(a.x, x.y), __dmul_rn(a.y, x.x));
    return make_double2(__dadd_rn(acc.x, re), __dadd_rn(acc.y, im));
}
__device__ __forceinline__ val_t ref_sub(val_t a, val_t b) { return make_double2(__dsub_rn(a.x, b.x), __dsub_rn(a.y, b.y)); }
__device__ __forceinline__ val_t ref_add(val_t a, val_t b) { return make_double2(__dadd_rn(a.x, b.x), __dadd_rn(a.y, b.y)); }
__device__ __forceinline__ val_t ref_scale(double s, val_t a) { return make_double2(__dmul_rn(s, a.x), __dmul_rn(s, a.y)); }
#else
__device__ __forceinline__ double ref_abs1(val_t a) { return fabs(a); }
__device__ __forceinline__ val_t ref_addmul(val_t acc, val_t a, val_t x) { return __dadd_rn(acc, __dmul_rn(a, x)); }
__device__ __forceinline__ val_t ref_sub(val_t a, val_t b) { return __dsub_rn(a, b); }
__device__ __forceinline__ val_t ref_add(val_t a, val_t b) { return __dadd_rn(a, b); }
__device__ __forceinline__ val_t ref_scale(double s, val_t a) { return __dmul_rn(s, a); }
#endif

// r = b - A x and w = |A| |x| + |b| for row i of column j of member blockIdx.y; inactive columns get r = 0.  Active columns:
// berr bits of max_i |r_i| / w_i (safe1 + |r_i| where w_i <= safe2, rows with w_i = 0 skipped) and, with W, dgerfs's
// W_i = |r_i| + (n + 1) eps w_i (+ safe1 where w_i <= safe2)
__global__ void __launch_bounds__(REF_THREADS) refine_residual_kernel(RefineArgs a, const val_t *__restrict__ x, val_t *__restrict__ r)
{
    const int t = blockIdx.x * REF_THREADS + threadIdx.x, m = blockIdx.y, n = a.n;
    if (t >= n * a.nrhs) return;
    const int j = t / n, i = t - j * n;
    const int64_t c = (int64_t)m * a.nrhs + j, o = c * n + i;
    if (!a.st[c].active) {
        r[o] = vzero();
        return;
    }
    const val_t *av = a.aval + (int64_t)m * a.nnz, *xc = x + c * n;
    val_t ax = vzero();
    double w = 0.0;
    for (int p = a.rowptr[i]; p < a.rowptr[i + 1]; ++p) {
        const val_t aij = av[p], xk = xc[a.colind[p]];
        ax = ref_addmul(ax, aij, xk);
        w = __dadd_rn(w, __dmul_rn(ref_abs1(aij), ref_abs1(xk)));
    }
    const val_t bi = a.b[o];
    const val_t ri = ref_sub(bi, ax);
    w = __dadd_rn(w, ref_abs1(bi));
    r[o] = ri;
    const double ar = ref_abs1(ri), safe1 = (n + 1) * DBL_MIN, safe2 = safe1 / REF_EPS;
    if (a.W) {
        const double wi = __dadd_rn(ar, __dmul_rn((n + 1) * REF_EPS, w));
        a.W[o] = w > safe2 ? wi : __dadd_rn(wi, safe1);
    }
    if (w == 0.0) return;
    const double s = w > safe2 ? __ddiv_rn(ar, w) : __ddiv_rn(__dadd_rn(safe1, ar), w);
    atomicMax(&a.st[c].berr_bits, ref_bits(s));
}

// one thread per column of member blockIdx.y: berr of this step, then pdgsrfs's test; a column that continues counts
// itself into *active
__global__ void __launch_bounds__(REF_THREADS) refine_decide_kernel(RefineArgs a, int *active)
{
    const int j = blockIdx.x * REF_THREADS + threadIdx.x;
    if (j >= a.nrhs) return;
    RefineState s = a.st[(int64_t)blockIdx.y * a.nrhs + j];
    if (!s.active) return;
    s.berr = __longlong_as_double((long long)s.berr_bits);
    s.berr_bits = 0;
    if (s.berr > REF_EPS && 2.0 * s.berr <= s.lstres && s.count < REFINE_ITMAX) {
        s.lstres = s.berr;
        ++s.count;
        atomicAdd(active, 1);
    } else {
        s.active = 0;
    }
    a.st[(int64_t)blockIdx.y * a.nrhs + j] = s;
}

// x += dx on the columns still active
__global__ void __launch_bounds__(REF_THREADS) refine_update_kernel(RefineArgs a, val_t *__restrict__ x, const val_t *__restrict__ dx)
{
    const int t = blockIdx.x * REF_THREADS + threadIdx.x, m = blockIdx.y, n = a.n;
    if (t >= n * a.nrhs) return;
    const int64_t c = (int64_t)m * a.nrhs + t / n, o = (int64_t)m * n * a.nrhs + t;
    if (a.st[c].active) x[o] = ref_add(x[o], dx[o]);
}

// dst = W src elementwise over members blocks of n x nrhs (the diag(W) of the forward error estimate)
__global__ void __launch_bounds__(REF_THREADS) refine_scale_kernel(val_t *dst, const val_t *src, const double *W, int64_t len)
{
    const int64_t t = (int64_t)blockIdx.x * REF_THREADS + threadIdx.x;
    if (t < len) dst[t] = ref_scale(W[t], src[t]);
}

// ---- the loop on the device (slu_b200_gsrfs_device): the host reads nothing between steps, conditional graph nodes loop --

constexpr int XMAX_PER_THREAD = 8;

__device__ __forceinline__ double ref_nan() { return __longlong_as_double(0x7ff8000000000000LL); }

// pdgsrfs's start (lstres = 3, count = 0) for every column; the columns of a member whose status is not 0 start inactive
__global__ void __launch_bounds__(REF_THREADS) refine_init_kernel(RefineState *st, const int32_t *status, int nrhs, int cols)
{
    const int c = blockIdx.x * REF_THREADS + threadIdx.x;
    if (c < cols) st[c] = RefineState{3.0, 0.0, 0ull, 0, status[c / nrhs] == 0};
}

// the refinement's WHILE node runs another step while a column is active
__global__ void refine_continue_kernel(const int *active, cudaGraphConditionalHandle h)
{
    cudaGraphSetConditional(h, *active > 0 ? 1u : 0u);
}

// max_i |x_i| per column: a CTA reduces XMAX_PER_THREAD * REF_THREADS rows of column blockIdx.y, then one integer atomicMax
// on the bits of the non-negative result, so the maximum does not depend on the order
__global__ void __launch_bounds__(REF_THREADS) refine_xmax_kernel(int n, const val_t *__restrict__ x, unsigned long long *xmax)
{
    const int64_t c = blockIdx.y;
    const val_t *xc = x + c * n;
    unsigned long long m = 0;
    for (int k = 0; k < XMAX_PER_THREAD; ++k) {
        const int i = (blockIdx.x * XMAX_PER_THREAD + k) * REF_THREADS + threadIdx.x;
        if (i < n) m = max(m, ref_bits(ref_abs1(xc[i])));
    }
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_down_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(xmax + c, m);
}

// per column: berr and steps of the loop, and dgerfs's ferr = est / max_i |x_i| (est where x = 0), as gsrfs's host side.
// A member whose status is not 0: NaN berr and ferr, 0 steps; a column whose estimate stopped at the round cap: NaN ferr.
__global__ void __launch_bounds__(REF_THREADS) refine_finish_kernel(RefineArgs a, const CondState *est, const unsigned long long *xmax,
                                                                     const int32_t *status, double *berr, double *ferr, int32_t *steps)
{
    const int c = blockIdx.x * REF_THREADS + threadIdx.x;
    if (c >= a.nrhs * a.members) return;
    const RefineState s = a.st[c];
    const bool ok = status[c / a.nrhs] == 0;
    berr[c] = ok ? s.berr : ref_nan();
    steps[c] = ok ? s.count : 0;
    if (!ferr) return;
    const CondState e = est[c];
    const double xm = __longlong_as_double((long long)xmax[c]);
    ferr[c] = !ok || e.kase != 0 ? ref_nan() : xm != 0.0 ? e.est / xm : e.est;
}

static dim3 refine_grid(const RefineArgs &a) { return dim3((unsigned)(((int64_t)a.n * a.nrhs + REF_THREADS - 1) / REF_THREADS), (unsigned)a.members); }

int launch_refine_residual(const RefineArgs &a, const val_t *x, val_t *r, cudaStream_t s)
{
    refine_residual_kernel<<<refine_grid(a), REF_THREADS, 0, s>>>(a, x, r);
    return 1;
}

int launch_refine_decide(const RefineArgs &a, int *active, cudaStream_t s)
{
    refine_decide_kernel<<<dim3((unsigned)((a.nrhs + REF_THREADS - 1) / REF_THREADS), (unsigned)a.members), REF_THREADS, 0, s>>>(a, active);
    return 1;
}

int launch_refine_update(const RefineArgs &a, val_t *x, const val_t *dx, cudaStream_t s)
{
    refine_update_kernel<<<refine_grid(a), REF_THREADS, 0, s>>>(a, x, dx);
    return 1;
}

int launch_refine_scale(val_t *dst, const val_t *src, const double *W, int64_t len, cudaStream_t s)
{
    if (len <= 0) return 0;
    refine_scale_kernel<<<(unsigned)((len + REF_THREADS - 1) / REF_THREADS), REF_THREADS, 0, s>>>(dst, src, W, len);
    return 1;
}

int launch_refine_init(RefineState *st, const int32_t *status, int nrhs, int members, cudaStream_t s)
{
    const int cols = nrhs * members;
    refine_init_kernel<<<(cols + REF_THREADS - 1) / REF_THREADS, REF_THREADS, 0, s>>>(st, status, nrhs, cols);
    return 1;
}

int launch_refine_continue(const int *active, cudaGraphConditionalHandle h, cudaStream_t s)
{
    refine_continue_kernel<<<1, 1, 0, s>>>(active, h);
    return 1;
}

int launch_refine_xmax(const RefineArgs &a, const val_t *x, unsigned long long *xmax, cudaStream_t s)
{
    const int per = XMAX_PER_THREAD * REF_THREADS;
    refine_xmax_kernel<<<dim3((unsigned)((a.n + per - 1) / per), (unsigned)(a.nrhs * a.members)), REF_THREADS, 0, s>>>(a.n, x, xmax);
    return 1;
}

int launch_refine_finish(const RefineArgs &a, const CondState *est, const unsigned long long *xmax, const int32_t *status, double *berr,
                         double *ferr, int32_t *steps, cudaStream_t s)
{
    const int cols = a.nrhs * a.members;
    refine_finish_kernel<<<(cols + REF_THREADS - 1) / REF_THREADS, REF_THREADS, 0, s>>>(a, est, xmax, status, berr, ferr, steps);
    return 1;
}

}  // namespace SLU_NS
