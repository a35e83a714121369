// slu_kernels_common.cuh -- device code shared by the double (slu_kernels.cu) and doublecomplex (slu_kernels_z.cu)
// kernels: batch slot search, cp.async / DMMA wrappers, and the destination maps of the Schur update, which only
// touch index arrays.  Compiled into namespace SLU_NS (slu_device.cuh).
#pragma once
#include "slu_device.cuh"

#include <atomic>

namespace SLU_NS {

// Opt a kernel in to more than 48 KB of dynamic shared memory.  The attribute is per device (context), and one
// process may hold handles on several GPUs (slu_b200_options_t.device), so the "already done" state is a per-device
// bit -- one atomic mask per call site -- not a process-wide flag.  Returns false (and leaves the bit clear) when
// the runtime refuses, so that the launch error is reported by the caller's cudaGetLastError.
template <class K>
inline bool ensure_dyn_smem(K kernel, int bytes, std::atomic<unsigned long long> &done)
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return false;
    const unsigned long long bit = dev < 64 ? 1ull << dev : 0;
    if (bit && (done.load(std::memory_order_acquire) & bit)) return true;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) return false;
    if (bit) done.fetch_or(bit, std::memory_order_release);
    return true;
}

// ------------------------------------------------------------------------------------------------
// batched launches (BatchedLU): the member of a CTA is blockIdx.y.  For a plain DeviceLU these are the identity, so
// the unbatched instantiations of a kernel templated on its DeviceLU type compile exactly as before.
__device__ __forceinline__ const DeviceLU &member_view(const DeviceLU &d) { return d; }
__device__ __forceinline__ DeviceLU member_view(const BatchedLU &d)
{
    DeviceLU m = d;
    m.val += (int64_t)blockIdx.y * d.val_stride;
    m.info += blockIdx.y;
    return m;
}
// a per-member buffer of `stride` (< 2^32) elements per member
template <class T> __device__ __forceinline__ T *member_ptr(const DeviceLU &, T *p, uint32_t) { return p; }
template <class T> __device__ __forceinline__ T *member_ptr(const BatchedLU &, T *p, uint32_t stride) { return p + (size_t)blockIdx.y * stride; }
template <class T> __device__ __forceinline__ T *member_inv(const DeviceLU &, T *dinv) { return dinv; }
template <class T> __device__ __forceinline__ T *member_inv(const BatchedLU &d, T *dinv) { return dinv + (int64_t)blockIdx.y * d.inv_stride; }
// launch grid: the unbatched x extent, one row per member
inline dim3 member_grid(const DeviceLU &, unsigned x) { return dim3(x); }
inline dim3 member_grid(const BatchedLU &d, unsigned x) { return dim3(x, (unsigned)d.members); }

// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int find_slot(const int64_t *prefix, int count, int64_t bid)
{
    int lo = 0, hi = count;  // prefix[lo] <= bid < prefix[hi]
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (prefix[mid] <= bid) lo = mid; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ void cp_async8(void *smem, const void *gmem, bool pred)
{
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    int sz = pred ? 8 : 0;  // src-size 0 => the 8 bytes are zero-filled
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(sa), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async8_plain(void *smem, const void *gmem)
{
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(sa), "l"(gmem));
}
// -x without the FP64 pipe (the DMMA pipe executes DADD too and is the busy unit of the Schur kernel)
__device__ __forceinline__ double flip_sign(double x)
{
    return __hiloint2double(__double2hiint(x) ^ (int)0x80000000, __double2loint(x));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void dmma884(double &d0, double &d1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(d0), "+d"(d1)
                 : "d"(a), "d"(b));
}
// d(16x8) += a(16x8) b(8x8), sm_90 (SASS DMMA.16x8x8: 8x the work of DMMA.8x8x4 per instruction).  Lane l with
// g = l/4, t = l%4 holds a = {A(g,t), A(g+8,t), A(g,t+4), A(g+8,t+4)}, b = {B(t,g), B(t+4,g)} and
// d = {D(g,2t), D(g,2t+1), D(g+8,2t), D(g+8,2t+1)}.
__device__ __forceinline__ void dmma1688(double (&d)[4], const double (&a)[4], const double (&b)[2])
{
    asm("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}

// ------------------------------------------------------------------------------------------------
// destination maps of the Schur update of supernode k
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int lower_bound_i32(const int32_t *a, int n, int key)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (a[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

#ifndef SLU_COMMON_HELPERS_ONLY   // one definition per precision: slu_kernels.cu / slu_kernels_z.cu
__global__ void __launch_bounds__(SETUP_THREADS) schur_setup_kernel(DeviceLU d, Batch b)
{
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const int k = b.nodes[slot];
    const NodeDesc nd = d.nodes[k];
    const int64_t t = (int64_t)(blockIdx.x - b.prefix[slot]) * SETUP_THREADS + threadIdx.x;
    const int m = nd.m, n = nd.ncols;
    const int32_t *rows = d.lrows + nd.lrow + nd.ns;  // sub-diagonal rows in panel order
    const int32_t *cols = d.ucols + nd.ucol;
    const LBlk *lb = d.lblk + nd.lblk;
    const UBlk *ub = d.ublk + nd.ublk;

    if (t < m) {  // RowInfo of source row i
        const int i = (int)t, r = rows[i], ib = d.supno[r];
        int lo = 0, hi = nd.nlb;  // block with row0 <= i
        while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (lb[mid].row0 <= i) lo = mid; else hi = mid; }
        const NodeDesc dst = d.nodes[ib];
        RowInfo ri;
        ri.ib = ib;
        ri.ldu = dst.ns;
        ri.ubase = dst.uval + (r - d.xsup[ib]);
        ri.urel_off = nd.ws_urel + lb[lo].urel_off - lb[lo].colstart;
        ri.shared = lb[lo].shared; ri.pad = 0;
        d.rowinfo[nd.ws_row + i] = ri;
        return;
    }
    int64_t u = t - m;
    if (u < n) {  // ColInfo of source column j
        const int j = (int)u, c = cols[j], jb = d.supno[c];
        int lo = 0, hi = nd.nub;
        while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (ub[mid].col0 <= j) lo = mid; else hi = mid; }
        const NodeDesc dst = d.nodes[jb];
        ColInfo ci;
        ci.jb = jb;
        ci.pad = ub[lo].shared;
        ci.lbase = dst.lval + (int64_t)(c - d.xsup[jb]) * dst.nsupr;
        ci.lrel_off = nd.ws_lrel + ub[lo].lrel_off - ub[lo].rowstart;
        d.colinfo[nd.ws_col + j] = ci;
        return;
    }
    u -= n;
    if (u < nd.lrel_total) {  // row position of source row i in destination L panel jb
        int lo = 0, hi = nd.nub;
        while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (ub[mid].lrel_off <= u) lo = mid; else hi = mid; }
        const int i = ub[lo].rowstart + (int)(u - ub[lo].lrel_off);
        const int r = rows[i];
        const NodeDesc dst = d.nodes[ub[lo].jb];
        const int32_t *srow = d.lsrow + dst.lrow;
        const int q = lower_bound_i32(srow, dst.nsupr, r);
        int pos = -1;
        if (dst.held && q < dst.nsupr && srow[q] == r) pos = d.lspos[dst.lrow + q];
        else atomicAdd(d.err, 1);
        d.lrel[nd.ws_lrel + u] = pos;
        return;
    }
    u -= nd.lrel_total;
    if (u < nd.urel_total) {  // packed column position of source column j in destination U panel ib
        int lo = 0, hi = nd.nlb;
        while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (lb[mid].urel_off <= u) lo = mid; else hi = mid; }
        const int j = lb[lo].colstart + (int)(u - lb[lo].urel_off);
        const int c = cols[j];
        const NodeDesc dst = d.nodes[lb[lo].ib];
        const int32_t *dc = d.ucols + dst.ucol;
        const int q = lower_bound_i32(dc, dst.ncols, c);
        int pos = -1;
        if (dst.held && q < dst.ncols && dc[q] == c) pos = q;
        else atomicAdd(d.err, 1);
        d.urel[nd.ws_urel + u] = pos;
    }
}

int launch_schur_setup(const DeviceLU &d, const Batch &b, int64_t ctas, cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    schur_setup_kernel<<<(unsigned)ctas, SETUP_THREADS, 0, s>>>(d, b);
    return 1;
}
#endif  // SLU_COMMON_HELPERS_ONLY

}  // namespace SLU_NS
