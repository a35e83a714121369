// slu_schur.cu -- the Schur complement of a partial factorization (slu_b200_schur_get): after the eliminated supernodes
// are factored, the panels of the Schur supernodes (the last nschur columns, never factored) hold
// S = A22 - A21 A11^-1 A12 on the symbolic pattern.  One launch copies every stored entry of those panels into a dense,
// zeroed s x s column-major buffer: the L panels (diagonal block included) give the entries on and below each supernode's
// diagonal block, the skyline segments of the U panels the entries to the right of it.  The two sets are disjoint, so
// every entry is written exactly once with a plain store and the result does not depend on scheduling.
//
// Compiled twice, like slu_selinv.cu: as is for double, and through slu_schur_z.cu with SLU_COMPLEX for doublecomplex.
#include "slu_device.cuh"

namespace SLU_NS {

constexpr int GATHER_THREADS = 128;
constexpr int GATHER_UNROLL = 4;     // loads in flight per thread before the stores

// one CTA per unit: unit (k, c) is column c of L panel k if c < ns, else packed column c - ns of U panel k
__global__ void __launch_bounds__(GATHER_THREADS) schur_gather_kernel(DeviceLU d, const int2 *__restrict__ units, int n0,
                                                                      int64_t s, val_t *__restrict__ S)
{
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

int launch_schur_gather(const DeviceLU &d, const int2 *units, int64_t nunits, int n0, int s, val_t *S, cudaStream_t st)
{
    if (nunits <= 0) return 0;
    schur_gather_kernel<<<(unsigned)nunits, GATHER_THREADS, 0, st>>>(d, units, n0, (int64_t)s, S);
    return 1;
}

}  // namespace SLU_NS
