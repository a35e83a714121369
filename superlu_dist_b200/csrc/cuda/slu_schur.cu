// slu_schur.cu -- the Schur complement of a partial factorization (slu_b200_schur_get, slu_b200_batch_schur_get): after
// the eliminated supernodes are factored, the panels of the Schur supernodes (the last nschur columns, never factored)
// hold S = A22 - A21 A11^-1 A12 on the symbolic pattern.  One launch copies every stored entry of those panels into a
// dense, zeroed s x s column-major buffer: the L panels (diagonal block included) give the entries on and below each
// supernode's diagonal block, the skyline segments of the U panels the entries to the right of it.  The two sets are
// disjoint, so every entry is written exactly once with a plain store and the result does not depend on scheduling.
//
// The kernel is templated on its LU type, as the selinv kernels are: in the BatchedLU instantiation the member is
// blockIdx.y, reading its own value arena and writing its own s x s block of S (member * s * s elements in).
//
// Compiled twice, like slu_selinv.cu: as is for double, and through slu_schur_z.cu with SLU_COMPLEX for doublecomplex.
#include "slu_device.cuh"
#define SLU_COMMON_HELPERS_ONLY
#include "slu_kernels_common.cuh"

namespace SLU_NS {

constexpr int GATHER_THREADS = 128;
constexpr int GATHER_UNROLL = 4;     // loads in flight per thread before the stores

// the member's s x s block of S: S itself for a plain DeviceLU
__device__ __forceinline__ val_t *member_S(const DeviceLU &, val_t *S, int64_t) { return S; }
__device__ __forceinline__ val_t *member_S(const BatchedLU &, val_t *S, int64_t s) { return S + (int64_t)blockIdx.y * s * s; }

// one CTA per unit: unit (k, c) is column c of L panel k if c < ns, else packed column c - ns of U panel k
template <class LU>
__global__ void __launch_bounds__(GATHER_THREADS) schur_gather_kernel(LU dd, const int2 *__restrict__ units, int n0,
                                                                      int64_t s, val_t *__restrict__ S)
{
    const DeviceLU &d = member_view(dd);
    S = member_S(dd, S, s);
    const int2 u = units[blockIdx.x];
    const NodeDesc &nd = d.nodes[u.x];
    const int ns = nd.ns, f = nd.fsupc;
    if (u.y < ns) {
        const int len = nd.nsupr;
        const val_t *__restrict__ src = d.val + nd.lval + (int64_t)u.y * len;
        const int32_t *__restrict__ rows = d.lrows + nd.lrow;
        val_t *__restrict__ dst = S + (int64_t)(f + u.y - n0) * s - n0;       // dst[r] = S(r - n0, column)
        for (int i0 = threadIdx.x; i0 < len; i0 += GATHER_THREADS * GATHER_UNROLL) {
            val_t v[GATHER_UNROLL];
            int r[GATHER_UNROLL];
#pragma unroll
            for (int t = 0; t < GATHER_UNROLL; ++t) {
                const int i = i0 + t * GATHER_THREADS;
                if (i < len) { v[t] = src[i]; r[t] = rows[i]; }
            }
#pragma unroll
            for (int t = 0; t < GATHER_UNROLL; ++t)
                if (i0 + t * GATHER_THREADS < len) dst[r[t]] = v[t];
        }
    } else {
        const int64_t q = nd.ucol + (u.y - ns);
        const int col = d.ucols[q], fst = d.ufst[q], klst = f + ns;
        const val_t *__restrict__ src = d.val + nd.uval + (int64_t)(u.y - ns) * ns - f;   // src[r] = U(r, col)
        val_t *__restrict__ dst = S + (int64_t)(col - n0) * s - n0;
        for (int r = fst + threadIdx.x; r < klst; r += GATHER_THREADS) dst[r] = src[r];
    }
}

// one launch of nunits CTAs per member (gridDim.y = members on a BatchedLU)
template <class LU>
static int launch_schur_gather_t(const LU &d, const int2 *units, int64_t nunits, int n0, int s, val_t *S, cudaStream_t st)
{
    if (nunits <= 0) return 0;
    schur_gather_kernel<LU><<<member_grid(d, (unsigned)nunits), GATHER_THREADS, 0, st>>>(d, units, n0, (int64_t)s, S);
    return 1;
}

int launch_schur_gather(const DeviceLU &d, const int2 *units, int64_t nunits, int n0, int s, val_t *S, cudaStream_t st)
{
    return launch_schur_gather_t(d, units, nunits, n0, s, S, st);
}
int launch_schur_gather(const BatchedLU &d, const int2 *units, int64_t nunits, int n0, int s, val_t *S, cudaStream_t st)
{
    return launch_schur_gather_t(d, units, nunits, n0, s, S, st);
}

}  // namespace SLU_NS
