// slu_grad.cu -- the gradient kernels of the device-resident factors (slu_b200_solve_grad_device, _logdet_grad_device,
// _selinv_device and _logdet_device, with their batched twins): sampled products on the kept A's pattern, the gather of the
// selected inverse through the refill's slot map, and the device status of a selected inversion.  Every kernel runs over
// (entry or row tiles, members) with gridDim.y = member; a member whose status is not 0 gets NaN.
//
// Compiled twice, like slu_refine.cu: as is for double, and through slu_grad_z.cu with SLU_COMPLEX for doublecomplex, where
// the solve gradient conjugates x and the log-determinant gradient conjugates H.
#include "slu_device.cuh"
#include "slu_scalar.cuh"

namespace SLU_NS {

constexpr int GRAD_THREADS = 256;
constexpr int GRAD_TILE = 32;          // the staging transpose: 32 x 32 tiles, 32 x 8 threads

__device__ __forceinline__ val_t grad_nan()
{
    const double q = __longlong_as_double(0x7ff8000000000000LL);
#ifdef SLU_COMPLEX
    return make_double2(q, q);
#else
    return q;
#endif
}

// dst[(m n + i) nrhs + k] = src[(m nrhs + k) ld + i]: the members' n x nrhs column-major blocks (ld apart per column) to
// row-major rows of nrhs values, so that the gradient reads the nrhs values of one row as one contiguous run.  grid (row
// tiles, right-hand-side tiles, members); coalesced reads along i, coalesced writes along (i, k)
__global__ void __launch_bounds__(GRAD_TILE * 8) grad_stage_kernel(val_t *__restrict__ dst, const val_t *__restrict__ src, int n, int nrhs,
                                                                int ld)
{
    __shared__ val_t tile[GRAD_TILE][GRAD_TILE + 1];
    const int64_t m = blockIdx.z;
    const int i0 = blockIdx.x * GRAD_TILE, k0 = blockIdx.y * GRAD_TILE;
    for (int r = threadIdx.y; r < GRAD_TILE; r += 8) {
        const int i = i0 + threadIdx.x, k = k0 + r;
        if (i < n && k < nrhs) tile[r][threadIdx.x] = src[(m * nrhs + k) * ld + i];
    }
    __syncthreads();
    for (int r = threadIdx.y; r < GRAD_TILE; r += 8) {
        const int i = i0 + r, k = k0 + threadIdx.x;
        if (i < n && k < nrhs) dst[(m * n + i) * nrhs + k] = tile[threadIdx.x][r];
    }
}

int launch_grad_stage(val_t *dst, const val_t *src, int n, int nrhs, int ld, int members, cudaStream_t s)
{
    if (n <= 0 || nrhs <= 0 || members <= 0) return 0;
    const dim3 g((unsigned)((n + GRAD_TILE - 1) / GRAD_TILE), (unsigned)((nrhs + GRAD_TILE - 1) / GRAD_TILE), (unsigned)members);
    grad_stage_kernel<<<g, dim3(GRAD_TILE, 8), 0, s>>>(dst, src, n, nrhs, ld);
    return 1;
}

// g[m nnz + e] = -sum over k = 0 .. nrhs-1 of lam(row[e], k) conj(x(colind[e], k)), accumulated in that order with one fused
// multiply-add per term (four in complex).  thread = entry e of member blockIdx.y; element (i, k) of member m at
// p[m ms + i rs + k].  Coalesced reads of row and colind; the lam reads of one row fall on one run, the x reads are gathered.
__global__ void __launch_bounds__(GRAD_THREADS) solve_grad_kernel(SolveGrad a)
{
    const int64_t e = (int64_t)blockIdx.x * GRAD_THREADS + threadIdx.x;
    if (e >= a.nnz) return;
    const int64_t m = blockIdx.y;
    if (a.status[m] != 0) {
        a.grad[m * a.nnz + e] = grad_nan();
        return;
    }
    const val_t *l = a.lam + m * a.lms + (int64_t)a.row[e] * a.rs;
    const val_t *x = a.x + m * a.xms + (int64_t)a.colind[e] * a.rs;
#ifdef SLU_COMPLEX
    double re = 0.0, im = 0.0;
    for (int k = 0; k < a.nrhs; ++k) {
        const val_t u = l[k], v = x[k];
        re = fma(u.x, v.x, re);
        re = fma(u.y, v.y, re);
        im = fma(u.y, v.x, im);
        im = fma(-u.x, v.y, im);
    }
    a.grad[m * a.nnz + e] = make_double2(-re, -im);
#else
    double acc = 0.0;
    for (int k = 0; k < a.nrhs; ++k) acc = fma(l[k], x[k], acc);
    a.grad[m * a.nnz + e] = -acc;
#endif
}

int launch_solve_grad(const SolveGrad &a, int members, cudaStream_t s)
{
    if (a.nnz <= 0 || members <= 0) return 0;
    solve_grad_kernel<<<dim3((unsigned)((a.nnz + GRAD_THREADS - 1) / GRAD_THREADS), (unsigned)members), GRAD_THREADS, 0, s>>>(a);
    return 1;
}

// the member's H arena: hv for an unbatched handle, val_stride elements apart on a batched one (64-bit offset)
__device__ __forceinline__ int64_t grad_member_off(const DeviceLU &, int64_t) { return 0; }
__device__ __forceinline__ int64_t grad_member_off(const BatchedLU &d, int64_t m) { return m * d.val_stride; }

// g[m nnz + e] = c_m ((R_i h) C_j), h = H[slot[e]] of member m (conj(H) in complex), i = row[e], j = colind[e]: the scaling
// in refill_kernel's order, then the coefficient; in complex the product c u as (c.x u.x - c.y u.y, c.x u.y + c.y u.x) with
// every multiply and add rounded on its own.  Coalesced reads of slot, row and colind, one gathered read of H, one coalesced
// store.  An entry without a slot gets NaN.
template <class LU>
__global__ void __launch_bounds__(GRAD_THREADS) logdet_grad_kernel(LU d, LogdetGrad a)
{
    const int64_t e = (int64_t)blockIdx.x * GRAD_THREADS + threadIdx.x;
    if (e >= a.nnz) return;
    const int64_t m = blockIdx.y;
    const int64_t o = a.slot[e];
    if (a.status[m] != 0 || o < 0) {
        a.grad[m * a.nnz + e] = grad_nan();
        return;
    }
    const double r = a.R[m * a.n + a.row[e]], c = a.C[m * a.n + a.colind[e]];
    const val_t h = a.hv[grad_member_off(d, m) + o];
    const val_t k = a.coef[m];
#ifdef SLU_COMPLEX
    const double ux = __dmul_rn(__dmul_rn(r, h.x), c), uy = __dmul_rn(__dmul_rn(r, -h.y), c);
    a.grad[m * a.nnz + e] = make_double2(__dsub_rn(__dmul_rn(k.x, ux), __dmul_rn(k.y, uy)),
                                         __dadd_rn(__dmul_rn(k.x, uy), __dmul_rn(k.y, ux)));
#else
    a.grad[m * a.nnz + e] = __dmul_rn(k, __dmul_rn(__dmul_rn(r, h), c));
#endif
}

template <class LU>
static int launch_logdet_grad_t(const LU &d, const LogdetGrad &a, int members, cudaStream_t s)
{
    if (a.nnz <= 0 || members <= 0) return 0;
    logdet_grad_kernel<LU><<<dim3((unsigned)((a.nnz + GRAD_THREADS - 1) / GRAD_THREADS), (unsigned)members), GRAD_THREADS, 0, s>>>(d, a);
    return 1;
}
int launch_logdet_grad(const DeviceLU &d, const LogdetGrad &a, cudaStream_t s) { return launch_logdet_grad_t(d, a, 1, s); }
int launch_logdet_grad(const BatchedLU &d, const LogdetGrad &a, cudaStream_t s) { return launch_logdet_grad_t(d, a, d.members, s); }

// the status of a device selected inversion: status[j] = -1 where the sweep missed a destination (*err), else info[j]; rec =
// {the factorization count it inverted (*epoch), *err}.  One CTA.
__global__ void __launch_bounds__(GRAD_THREADS) selinv_status_kernel(const int *__restrict__ err, const int32_t *__restrict__ info, int members,
                                                                  const unsigned long long *__restrict__ epoch, int32_t *__restrict__ status,
                                                                  unsigned long long *__restrict__ rec)
{
    const int bad = *err;
    for (int j = threadIdx.x; j < members; j += GRAD_THREADS) status[j] = bad ? -1 : info[j];
    if (threadIdx.x == 0) {
        rec[0] = *epoch;
        rec[1] = (unsigned long long)bad;
    }
}

int launch_selinv_status(const int *err, const int32_t *info, int members, const unsigned long long *epoch, int32_t *status,
                         unsigned long long *rec, cudaStream_t s)
{
    selinv_status_kernel<<<1, GRAD_THREADS, 0, s>>>(err, info, members, epoch, status, rec);
    return 1;
}

// res holds members x (1 + VAL_DOUBLES) doubles as launch_selinv_logdet leaves them: logabs[j] and sign[j VAL_DOUBLES ...] of
// member j, copied as they are, or NaN where status[j] is not 0.  One CTA.
__global__ void __launch_bounds__(GRAD_THREADS) logdet_out_kernel(const double *__restrict__ res, const int32_t *__restrict__ status, int members,
                                                               double *__restrict__ logabs, double *__restrict__ sign)
{
    const double q = __longlong_as_double(0x7ff8000000000000LL);
    for (int j = threadIdx.x; j < members; j += GRAD_THREADS) {
        const bool ok = status[j] == 0;
        const double *r = res + (int64_t)j * (1 + VAL_DOUBLES);
        logabs[j] = ok ? r[0] : q;
        for (int c = 0; c < VAL_DOUBLES; ++c) sign[(int64_t)j * VAL_DOUBLES + c] = ok ? r[1 + c] : q;
    }
}

int launch_logdet_out(const double *res, const int32_t *status, int members, double *logabs, double *sign, cudaStream_t s)
{
    logdet_out_kernel<<<1, GRAD_THREADS, 0, s>>>(res, status, members, logabs, sign);
    return 1;
}

}  // namespace SLU_NS
