// slu_kernels.cu -- the sm_90a kernels of the pdgstrf3d hot path.
//
//   diag_lu_kernel      unpivoted LU of the diagonal block      (Local_Dgstrf2, SRC/double/pdgstrf2.c:508-601)
//   trsm_kernel<false>  L(below,k) <- L(below,k) U_kk^-1         (dLPanelTrSolve, SRC/double/dtrfCommWrapper.c:120-223)
//   trsm_kernel<true>   U(k,:)     <- L_kk^-1 U(k,:)             (dUPanelTrSolve, dtrfCommWrapper.c:242-357)
//   schur_setup_kernel  destination maps of one supernode       (index work of dscatter_l/dscatter_u,
//                                                                 SRC/double/dscatter.c:138-174, 222-243)
//   schur_kernel_h      V = L(below,k) U(k,:) of the big tiles on FP64 tensor cores (mma.sync.m16n8k8.f64) with the
//   schur_kernel        (small tiles: mma.sync.m8n8k4.f64)
//                       subtract-scatter fused into the epilogue: no bigV buffer
//                                                                (dblock_gemm_scatter, SRC/double/dscatter3d.c:82-189)
//   u_expand / u_pack   skyline <-> dense-packed U at the boundary (dRgather_U, SRC/double/dgather.c:256-398)
//   axpy_kernel         ancestor reduction add                  (dzRecvLPanel/UPanel, SRC/double/pd3dcomm.c:224-331)
//
// wgmma has no f64 kind, so the native FP64 tensor path on
// sm_90a is the warp-level DMMA fed from shared memory; tiles are staged with cp.async (LDGSTS).
#include "slu_device.cuh"
#include "slu_kernels_common.cuh"

#include <climits>

namespace slu {

// ------------------------------------------------------------------------------------------------
// diagonal block LU: one CTA per supernode, right-looking with NB-wide panels in shared memory
// ------------------------------------------------------------------------------------------------
template <class LU>
__global__ void __launch_bounds__(512) diag_lu_kernel(LU dd, Batch b, int replace_tiny, double thresh, int skip_lo, int skip_hi)
{
    extern __shared__ double sm[];
    const DeviceLU &d = member_view(dd);
    constexpr int NB = DIAG_NB;
    const int k = b.nodes[blockIdx.x];
    const NodeDesc nd = d.nodes[k];
    if (nd.ns >= skip_lo && nd.ns <= skip_hi) return;   // taken by the cluster kernel
    const int ns = nd.ns, lda = nd.nsupr, tid = threadIdx.x, nt = blockDim.x;
    double *A = d.val + nd.lval;
    double *Ps = sm;            // panel  Ps[c*rem + i]
    double *Us = sm + NB * ns;  // U12    Us[c*NB + p]

    for (int j0 = 0; j0 < ns; j0 += NB) {
        const int jb = min(NB, ns - j0), rem = ns - j0;
        for (int idx = tid; idx < jb * rem; idx += nt) {
            int c = idx / rem, i = idx - c * rem;
            Ps[c * rem + i] = A[(size_t)(j0 + c) * lda + j0 + i];
        }
        __syncthreads();
        // (1) warp 0 factors the jb x jb diagonal block in place (lane r owns row r; warp-level steps only)
        if (tid < 32) {
            const int r = tid;
            for (int c = 0; c < jb; ++c) {
                if (r == 0) {
                    double p = Ps[c * rem + c];
                    if (replace_tiny && fabs(p) < thresh) {  // pdgstrf2.c:544-560
                        p = (p < 0) ? -thresh : thresh;
                        Ps[c * rem + c] = p;
                        if (replace_tiny == 1) atomicAdd(d.tiny, 1ULL);  // 2: replicated copy, counted by its owner
                    }
                    if (p == 0.0) atomicMin(d.info, nd.fsupc + j0 + c + 1);  // pdgstrf2.c:568-571
                }
                __syncwarp();
                const double p = Ps[c * rem + c];
                if (r > c && r < jb) {
                    double l = Ps[c * rem + r];
                    if (p != 0.0) l *= 1.0 / p;
                    Ps[c * rem + r] = l;
                    for (int cc = c + 1; cc < jb; ++cc) Ps[cc * rem + r] -= l * Ps[cc * rem + c];
                }
                __syncwarp();
            }
        }
        __syncthreads();
        // (2) rows below the diagonal block: x U11 = a, one row per thread, same operation order as the
        //     right-looking rank-1 sweep (scale by the reciprocal pivot, then update the columns to the right)
        for (int i = jb + tid; i < rem; i += nt) {
            double x[NB];
#pragma unroll
            for (int c = 0; c < NB; ++c) x[c] = (c < jb) ? Ps[c * rem + i] : 0.0;
#pragma unroll
            for (int c = 0; c < NB; ++c) {
                if (c < jb) {
                    double v = x[c];
#pragma unroll
                    for (int p = 0; p < NB; ++p)
                        if (p < c) v -= x[p] * Ps[c * rem + p];
                    const double pv = Ps[c * rem + c];
                    x[c] = (pv != 0.0) ? v * (1.0 / pv) : v;
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
                double x[NB];
                double *col = A + (size_t)(j0 + jb + c) * lda + j0;
#pragma unroll
                for (int p = 0; p < NB; ++p) x[p] = (p < jb) ? col[p] : 0.0;
#pragma unroll
                for (int p = 0; p < NB; ++p)
#pragma unroll
                    for (int q = p + 1; q < NB; ++q)
                        if (q < jb) x[q] -= Ps[p * rem + q] * x[p];
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
                double acc = 0.0;
#pragma unroll
                for (int p = 0; p < NB; ++p)
                    if (p < jb) acc += Ps[p * rem + jb + i] * Us[c * NB + p];
                A[(size_t)(j0 + jb + c) * lda + j0 + jb + i] -= acc;
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// diagonal block LU on a thread-block cluster (supernodes of 65..256 columns).  The one-CTA kernel above streams the
// block through L2 from ONE SM at every 16-column step: 0.54 ms for a 252-column block, at every level of the
// elimination tree and on every rank of a cooperative group -- the Amdahl term of the 8-GPU run (VERDICT r1).
// Here a cluster of 8 CTAs (8 SMs of one GPC) holds the whole block in shared memory, one 32-column slab per CTA:
//   step j:  CTA j factors its slab's rows [32j, ns) (right-looking rank-1 steps, one row per thread in registers, the
//            pivot row published through shared memory), writes the finished slab to HBM;
//            cluster barrier (release / acquire);
//            CTAs > j read the L panel back from L2, solve their 32 x 32 U12 block (unit lower) and update their slab
//            with DMMA m8n8k4 (A = L21 from shared memory, B = U12).
// 8 steps for 256 columns; every CTA touches HBM twice (load its slab, store it) plus one L-panel read per step.
// Arithmetic rules of the reference kept: reciprocal pivot, tiny-pivot replacement, zero pivot -> info
// (pdgstrf2.c:544-571); only the summation order differs.
// ------------------------------------------------------------------------------------------------
constexpr int DC_CL = 8, DC_W = 32, DC_MAX_NS = DC_CL * DC_W, DC_MIN_NS = 65;
constexpr int DC_LD = DC_MAX_NS + 4;     // column stride of the slab / panel in shared memory (== 4 mod 16 doubles)
constexpr size_t DC_SMEM = sizeof(double) * (2 * DC_W * DC_LD + 2 * 40 + DC_W * 36);

__device__ __forceinline__ void cluster_sync_all()
{
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned cluster_rank()
{
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}

template <class LU>
__global__ void __cluster_dims__(DC_CL, 1, 1) __launch_bounds__(256) diag_lu_cluster_kernel(LU dd, Batch b, int replace_tiny, double thresh)
{
    extern __shared__ double sm[];
    const DeviceLU &d = member_view(dd);
    double *S = sm;                        // my slab      S[c * DC_LD + r], r < ns, c < 32
    double *P = S + DC_W * DC_LD;          // L panel      P[c * DC_LD + i], i < rem (rows relative to j0)
    double *urow = P + DC_W * DC_LD;       // pivot rows, double buffered: urow[buf * 40 + c], [buf * 40 + 32] = 1 / pivot
    double *U12 = urow + 2 * 40;           // my solved 32 x 32 block: U12[c * 36 + p]
    const int k = b.nodes[blockIdx.x / DC_CL];
    const NodeDesc nd = d.nodes[k];
    const int ns = nd.ns;
    if (ns < DC_MIN_NS || ns > DC_MAX_NS) return;      // the whole cluster leaves: the one-CTA kernel takes these
    const int lda = nd.nsupr, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int me = (int)cluster_rank();
    const int nslab = (ns + DC_W - 1) / DC_W;
    const int c0 = me * DC_W, wc = min(DC_W, ns - c0);           // my columns [c0, c0 + wc); wc <= 0: no slab
    double *A = d.val + nd.lval;

    if (wc > 0)
        for (int idx = tid; idx < wc * ns; idx += 256) {
            const int c = idx / ns, r = idx - c * ns;
            S[c * DC_LD + r] = A[(size_t)(c0 + c) * lda + r];
        }
    __syncthreads();

    for (int j = 0; j < nslab; ++j) {
        const int j0 = j * DC_W, jb = min(DC_W, ns - j0), rem = ns - j0;
        if (me == j) {
            // ---- panel: rows [j0, ns) of my slab, thread t owns row j0 + t -------------------------------------------
            double x[DC_W];
            const bool mine = tid < rem;
#pragma unroll
            for (int c = 0; c < DC_W; ++c) x[c] = (mine && c < jb) ? S[c * DC_LD + j0 + tid] : 0.0;
#pragma unroll
            for (int c = 0; c < DC_W; ++c) {
                double *ur = urow + (c & 1) * 40;
                if (c < jb && tid == c) {
                    double pv = x[c];
                    if (replace_tiny && fabs(pv) < thresh) {  // pdgstrf2.c:544-560
                        pv = (pv < 0) ? -thresh : thresh;
                        x[c] = pv;
                        if (replace_tiny == 1) atomicAdd(d.tiny, 1ULL);
                    }
                    if (pv == 0.0) atomicMin(d.info, nd.fsupc + j0 + c + 1);  // pdgstrf2.c:568-571
#pragma unroll
                    for (int cc = 0; cc < DC_W; ++cc) ur[cc] = x[cc];
                    ur[32] = (pv != 0.0) ? 1.0 / pv : 1.0;
                }
                __syncthreads();
                if (c < jb && mine && tid > c) {
                    const double l = x[c] * ur[32];
                    x[c] = l;
#pragma unroll
                    for (int cc = c + 1; cc < DC_W; ++cc) x[cc] -= l * ur[cc];
                }
            }
            if (mine)
#pragma unroll
                for (int c = 0; c < DC_W; ++c)
                    if (c < jb) S[c * DC_LD + j0 + tid] = x[c];
            __syncthreads();
            // ---- the slab is final: rows < j0 are U, rows >= j0 were just factored -----------------------------------
            for (int idx = tid; idx < wc * ns; idx += 256) {
                const int c = idx / ns, r = idx - c * ns;
                A[(size_t)(c0 + c) * lda + r] = S[c * DC_LD + r];
            }
            __threadfence();
        }
        cluster_sync_all();
        if (me > j && wc > 0) {
            // ---- L panel of step j from L2 ---------------------------------------------------------------------------
            for (int idx = tid; idx < jb * rem; idx += 256) {
                const int c = idx / rem, i = idx - c * rem;
                P[c * DC_LD + i] = __ldcg(A + (size_t)(j0 + c) * lda + j0 + i);
            }
            __syncthreads();
            // ---- U12 = L11^-1 S[j0 : j0 + jb, :] (unit lower), one column per thread ---------------------------------
            if (tid < wc) {
                double x[DC_W];
#pragma unroll
                for (int p = 0; p < DC_W; ++p) x[p] = (p < jb) ? S[tid * DC_LD + j0 + p] : 0.0;
#pragma unroll
                for (int p = 0; p < DC_W; ++p)
#pragma unroll
                    for (int q = p + 1; q < DC_W; ++q)
                        if (q < jb) x[q] -= P[p * DC_LD + q] * x[p];
#pragma unroll
                for (int p = 0; p < DC_W; ++p) {
                    if (p < jb) S[tid * DC_LD + j0 + p] = x[p];
                    U12[tid * 36 + p] = x[p];
                }
            } else if (tid < DC_W) {
#pragma unroll
                for (int p = 0; p < DC_W; ++p) U12[tid * 36 + p] = 0.0;
            }
            __syncthreads();
            // ---- S[j0 + jb :, :] -= L21 U12 on DMMA: warp w takes the 8-row tiles w, w + 8, ...; K = 32 --------------
            const int r2 = rem - jb;   // > 0 implies jb == 32
            const int lr = lane >> 2, lk = lane & 3;
            for (int t = warp; t * 8 < r2; t += 8) {
                const int i = t * 8 + lr;             // row relative to j0 + jb
                const bool ok = i < r2;
                double acc[4][2];
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) acc[ni][0] = acc[ni][1] = 0.0;
#pragma unroll
                for (int p0 = 0; p0 < DC_W; p0 += 4) {
                    const double a = ok ? P[(p0 + lk) * DC_LD + jb + i] : 0.0;
#pragma unroll
                    for (int ni = 0; ni < 4; ++ni) dmma884(acc[ni][0], acc[ni][1], a, U12[(ni * 8 + lr) * 36 + p0 + lk]);
                }
#pragma unroll
                for (int ni = 0; ni < 4; ++ni)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int c = ni * 8 + 2 * lk + e;
                        if (ok && c < wc) S[c * DC_LD + j0 + jb + i] -= acc[ni][e];
                    }
            }
            __syncthreads();
        }
    }
}

template <class LU>
static int launch_diag_lu_t(const LU &d, const Batch &b, int max_ns, int replace_tiny, double thresh, cudaStream_t s)
{
    if (b.count <= 0) return 0;
    int launched = 0, skip_lo = 1, skip_hi = 0;    // empty range: the one-CTA kernel takes every supernode
    if (max_ns >= DC_MIN_NS) {
        static std::atomic<unsigned long long> attrc{0};
        ensure_dyn_smem(diag_lu_cluster_kernel<LU>, (int)DC_SMEM, attrc);
        diag_lu_cluster_kernel<LU><<<member_grid(d, b.count * DC_CL), 256, DC_SMEM, s>>>(d, b, replace_tiny, thresh);
        skip_lo = DC_MIN_NS; skip_hi = DC_MAX_NS;
        ++launched;
        if (b.count == 1 && max_ns <= DC_MAX_NS) return launched;   // the single supernode of a chain level went to the cluster
    }
    size_t smem = sizeof(double) * 2 * DIAG_NB * (size_t)max_ns;
    static std::atomic<unsigned long long> attr_0{0};
    ensure_dyn_smem(diag_lu_kernel<LU>, (int)(sizeof(double) * 2 * DIAG_NB * MAX_NS), attr_0);
    int threads = max_ns <= 32 ? 128 : (max_ns <= 128 ? 256 : 512);
    diag_lu_kernel<LU><<<member_grid(d, b.count), threads, smem, s>>>(d, b, replace_tiny, thresh, skip_lo, skip_hi);
    return launched + 1;
}
int launch_diag_lu(const DeviceLU &d, const Batch &b, int max_ns, int replace_tiny, double thresh, cudaStream_t s)
{
    return launch_diag_lu_t(d, b, max_ns, replace_tiny, thresh, s);
}
int launch_diag_lu(const BatchedLU &d, const Batch &b, int max_ns, int replace_tiny, double thresh, cudaStream_t s)
{
    return launch_diag_lu_t(d, b, max_ns, replace_tiny, thresh, s);
}

// Shared images of DMMA.16x8x8 operands (the Hopper main loop and the panel TRSM): rows g and g+8 of a 16-row block
// are adjacent (row r at prow(r)), and so are k and k+4 of an 8-deep slice (at pk(k)), so that each lane's fragment
// pairs are 16-byte loads.
__device__ __forceinline__ int prow(int r) { return (r & ~15) | ((r & 7) << 1) | ((r >> 3) & 1); }
__device__ __forceinline__ int pk(int k) { return (k & ~7) | ((k & 3) << 1) | ((k >> 2) & 1); }

// ------------------------------------------------------------------------------------------------
// panel triangular solves on the FP64 tensor cores.
//   Y <- Y T^-1, T upper triangular ns x ns, blocked by 16 columns (left-looking):
//       Y_j <- (Y_j - sum_{p<j} Y_p T_pj) inv(T_jj)
//   L case: vectors = sub-diagonal rows of panel k, T(p,c) = U_kk(p,c)            (non-unit)
//   U case: vectors = packed columns of U(k,:),    T(p,c) = L_kk(c,p) (transposed, unit)
// The 16x16 diagonal blocks are inverted once per supernode by diag_inv_kernel; everything else is
// substitution.  Inside a block, R = Y_j - sum is multiplied by the inverse and then corrected once,
// X = R inv + (R - (R inv) T_jj) inv: the product with an explicit inverse alone has a backward error that
// grows with cond(T_jj) on consistent right-hand sides, the correction brings it to substitution's.
// ------------------------------------------------------------------------------------------------
template <class LU>
__global__ void __launch_bounds__(64) diag_inv_kernel(LU dd, Batch b, double *dinv)
{
    __shared__ double M[16 * 17];
    const DeviceLU &d = member_view(dd);
    dinv = member_inv(dd, dinv);
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const int k = b.nodes[slot];
    const NodeDesc nd = d.nodes[k];
    const int blk = (int)(blockIdx.x - b.prefix[slot]);
    const int j0 = blk * 16, jb = min(16, nd.ns - j0), lda = nd.nsupr, tid = threadIdx.x;
    const double *A = d.val + nd.lval;
    for (int idx = tid; idx < 256; idx += 64) {
        int c = idx >> 4, r = idx & 15;
        double v = (r == c) ? 1.0 : 0.0;
        if (r < jb && c < jb) v = A[(size_t)(j0 + c) * lda + j0 + r];
        M[c * 17 + r] = v;
    }
    __syncthreads();
    double *out = dinv + nd.ws_inv + (size_t)blk * 512;
    const int c = tid & 31;
    if (tid < 32) {  // column c of inv(U), U = upper triangle of M (non-unit)
        if (c < 16) {
            double x[16];
#pragma unroll
            for (int r = 0; r < 16; ++r) x[r] = 0.0;
            for (int r = c; r >= 0; --r) {
                double sacc = (r == c) ? 1.0 : 0.0;
                for (int q = r + 1; q <= c; ++q) sacc -= M[q * 17 + r] * x[q];
                x[r] = sacc / M[r * 17 + r];
            }
#pragma unroll
            for (int r = 0; r < 16; ++r) out[c * 16 + r] = x[r];
        }
    } else if (c < 16) {  // column c of inv(L), L = unit lower triangle of M
        double x[16];
#pragma unroll
        for (int r = 0; r < 16; ++r) x[r] = 0.0;
        x[c] = 1.0;
        for (int r = c + 1; r < 16; ++r) {
            double sacc = 0.0;
            for (int q = c; q < r; ++q) sacc -= M[q * 17 + r] * x[q];
            x[r] = sacc;
        }
#pragma unroll
        for (int r = 0; r < 16; ++r) out[256 + c * 16 + r] = x[r];
    }
}

template <class LU>
static int launch_diag_inv_t(const LU &d, const Batch &b, int64_t ctas, double *dinv, cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    diag_inv_kernel<LU><<<member_grid(d, (unsigned)ctas), 64, 0, s>>>(d, b, dinv);
    return 1;
}
int launch_diag_inv(const DeviceLU &d, const Batch &b, int64_t ctas, double *dinv, cudaStream_t s)
{
    return launch_diag_inv_t(d, b, ctas, dinv, s);
}
int launch_diag_inv(const BatchedLU &d, const Batch &b, int64_t ctas, double *dinv, cudaStream_t s)
{
    return launch_diag_inv_t(d, b, ctas, dinv, s);
}

// trsm_kernel: one CTA of four warps per strip of TRSM_STRIP = 32 vectors, on DMMA.16x8x8.  Warp (mt, nt) owns vectors
// 16 mt .. 16 mt + 15 and columns 8 nt .. 8 nt + 7 of every 16-column block j; its sum over p < j0 runs in four
// independent accumulators (k8 slice q adds into acc[q % 4]), which are added before Y_j - sum is multiplied by
// inv(T_jj).  The strip stays in shared memory for the whole sweep, vector s at prow(s) of each column, so that A
// fragments are 16-byte loads; T streams through a double buffer of TRSM_KC x 16 chunks, row p at pk(p).  That is
// 90 KB of shared memory at ns = 256 (two CTAs per SM) and 162 KB at ns = 512.  Keep it there: with a third T stage
// (99 KB) or 128-row chunks (110 KB) the kernel was no faster alone and the look-ahead step, where it runs beside the
// Schur kernel's 88 KB CTAs, was 7 % slower (DESIGN §4d).
constexpr int TRSM_THREADS = 128, TRSM_KC = 64;
constexpr int TRSM_LD = TRSM_STRIP + 4;   // == 4 (mod 16) doubles: conflict-free A fragments
constexpr int TRSM_LDT = TRSM_KC + 8;     // == 8 (mod 16): conflict-free B fragments
static_assert(TRSM_STRIP == 32 && TRSM_THREADS == 128 && TRSM_KC % 16 == 0, "trsm_kernel thread mapping");
static_assert(2 * 16 * TRSM_LD <= 16 * TRSM_LDT, "X and R - X T_jj of a block fit in one T buffer");
static size_t trsm_smem(int max_ns)
{
    return sizeof(double) * ((size_t)((max_ns + 15) & ~15) * TRSM_LD + 2 * 16 * TRSM_LDT);
}

template <bool UCASE, class LU>
__global__ void __launch_bounds__(TRSM_THREADS, 2) trsm_kernel(LU dd, Batch b, const double *dinv)
{
    extern __shared__ __align__(16) double Ys[];   // [nsp][TRSM_LD], then Tb[2][16][TRSM_LDT]
    const DeviceLU &d = member_view(dd);
    dinv = member_inv(dd, dinv);
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const NodeDesc nd = d.nodes[b.nodes[slot]];
    const int strip = (int)(blockIdx.x - b.prefix[slot]);
    const int ns = nd.ns, lda = nd.nsupr, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nsp = (ns + 15) & ~15;
    const double *T = d.val + nd.lval;
    const double *inv = dinv + nd.ws_inv;
    const int nvec = UCASE ? nd.ncols : nd.m;
    const int v0 = strip * TRSM_STRIP, nv = min(TRSM_STRIP, nvec - v0);
    double *X = UCASE ? d.val + nd.uval + (size_t)v0 * ns : d.val + nd.lval + ns + v0;
    double *const Tb = Ys + (size_t)nsp * TRSM_LD;

    // the strip, zero beyond nv vectors and ns columns.  L: X(s, c) = X[c lda + s], lane = s and warp = c mod 4.
    // U: X(s, c) = X[s ns + c], 16 vectors x 2 columns per warp, so that the shared stores stay conflict-free.
    const int us = (lane & 15) | (warp & 1) << 4, uc = (lane >> 4) | (warp >> 1) << 1;
    if (!UCASE) {
        const bool sv = lane < nv;
        const double *x = X + (size_t)warp * lda + lane;
        const size_t step = (size_t)4 * lda;
        for (int c = warp; c < nsp; c += 4, x += step) {
            const bool ok = sv && c < ns;
            cp_async8(Ys + c * TRSM_LD + prow(lane), ok ? x : X, ok);
        }
    } else {
        const bool sv = us < nv;
        const double *x = X + (size_t)us * ns;
        for (int c = uc; c < nsp; c += 4) {
            const bool ok = sv && c < ns;
            cp_async8(Ys + c * TRSM_LD + prow(us), ok ? x + c : X, ok);
        }
    }

    // T chunks in sweep order: block j0 = 16, 32, .. takes rows pn = 0, TRSM_KC, .. < j0 of columns j0 .. j0 + 15.
    // L: T(p, c) = T[c lda + p], p = tid mod TRSM_KC.  U: T(p, c) = T[p lda + c], 8 rows x 4 columns per warp.
    int jn = 16, pn = 0;
    auto fetch = [&](int buf) {
        if (jn >= ns) return;
        double *dst = Tb + buf * 16 * TRSM_LDT;
        constexpr int PASSES = 16 * TRSM_KC / TRSM_THREADS;
        if (!UCASE) {
            constexpr int CS = TRSM_THREADS / TRSM_KC;   // columns per pass
            const int p = tid & (TRSM_KC - 1), c0 = tid / TRSM_KC;
            const bool pv = pn + p < jn;
            const double *src = T + (size_t)(jn + c0) * lda + pn + p;
            const size_t step = (size_t)CS * lda;
#pragma unroll
            for (int i = 0; i < PASSES; ++i, src += step) {
                const bool ok = pv && jn + c0 + CS * i < ns;
                cp_async8(dst + (c0 + CS * i) * TRSM_LDT + pk(p), ok ? src : T, ok);
            }
        } else {
            const int c = tid >> 3, p0 = tid & 7;
            const bool cv = jn + c < ns;
            const double *src = T + (size_t)(pn + p0) * lda + jn + c;
            const size_t step = (size_t)8 * lda;
#pragma unroll
            for (int i = 0; i < PASSES; ++i, src += step) {
                const bool ok = cv && pn + p0 + 8 * i < jn;
                cp_async8(dst + c * TRSM_LDT + pk(p0 + 8 * i), ok ? src : T, ok);
            }
        }
        pn += TRSM_KC;
        if (pn >= jn) { jn += 16; pn = 0; }
    };
    cp_async_commit();
    fetch(0);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();

    const int g = lane >> 2, t = lane & 3, mt = warp & 1, nt = warp >> 1;
    const double *const ya = Ys + t * TRSM_LD + 16 * mt + 2 * g;         // A fragment of columns p..p+7: ya + p LD
    double *const yd = Ys + (8 * nt + 2 * t) * TRSM_LD + 16 * mt + 2 * g;  // D tile of block j0: yd + (j0 + e) LD
    const double *const tb = Tb + (8 * nt + g) * TRSM_LDT + 2 * t;         // B fragment of k8 slice q: tb + 8 q
    int buf = 0;
    for (int j0 = 0; j0 < ns; j0 += 16) {
        // inv(T_jj) and T_jj itself, loaded ahead: the latency hides behind the update.  T_jj is padded with the
        // identity beyond jb as diag_inv_kernel pads it; in the U case its diagonal is 1 (the stored one holds U's pivots).
        const double *ib = inv + (size_t)(j0 >> 4) * 512;
        const int jb = min(16, ns - j0);
        double bi[2][2], bt[2][2];
#pragma unroll
        for (int kk = 0; kk < 2; ++kk)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int p = 8 * kk + 4 * h + t, c = 8 * nt + g;
                bi[kk][h] = UCASE ? ib[256 + p * 16 + c] : ib[c * 16 + p];
                double v = (p == c) ? 1.0 : 0.0;
                if (c < jb && (UCASE ? p < c : p <= c))
                    v = UCASE ? T[(size_t)(j0 + p) * lda + j0 + c] : T[(size_t)(j0 + c) * lda + j0 + p];
                bt[kk][h] = v;
            }
        double acc[4][4];
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.0;
        for (int pc = 0; pc < j0; pc += TRSM_KC) {
            cp_async_wait<0>();
            __syncthreads();
            fetch(buf ^ 1);
            cp_async_commit();
            const double *yc = ya + (size_t)pc * TRSM_LD, *tc = tb + buf * 16 * TRSM_LDT;
            const int nq = min(TRSM_KC, j0 - pc) >> 3;   // even: j0 - pc is a multiple of 16
#pragma unroll
            for (int q = 0; q < TRSM_KC / 8; ++q) {
                if (q < nq) {
                    const double2 lo = *reinterpret_cast<const double2 *>(yc + 8 * q * TRSM_LD);
                    const double2 hi = *reinterpret_cast<const double2 *>(yc + (8 * q + 4) * TRSM_LD);
                    const double2 v = *reinterpret_cast<const double2 *>(tc + 8 * q);
                    const double a[4] = {lo.x, lo.y, hi.x, hi.y}, bb[2] = {v.x, v.y};
                    dmma1688(acc[q & 3], a, bb);
                }
            }
            buf ^= 1;
        }
        // D = {D(g, 2t), D(g, 2t+1), D(g+8, 2t), D(g+8, 2t+1)}; rows g and g+8 are adjacent in the strip
        double2 *d0 = reinterpret_cast<double2 *>(yd + (size_t)j0 * TRSM_LD), *d1 = reinterpret_cast<double2 *>(yd + (size_t)(j0 + 1) * TRSM_LD);
        double sum[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) sum[e] = (acc[0][e] + acc[1][e]) + (acc[2][e] + acc[3][e]);
        const double2 y0 = *d0, y1 = *d1;
        const double r[4] = {y0.x - sum[0], y1.x - sum[1], y0.y - sum[2], y1.y - sum[3]};   // R = Y_j - sum, kept
        *d0 = make_double2(r[0], r[2]);
        *d1 = make_double2(r[1], r[3]);
        __syncthreads();   // each product with a 16-row right factor reads both column halves of the block
        // X = R inv, then the correction X += (R - X T_jj) inv; X and R - X T_jj pass between the warps through the
        // T buffer that the sweep is not fetching into (it is refilled only after the next block's first barrier).
        double *const xw = Tb + (buf ^ 1) * 16 * TRSM_LDT, *const cw = xw + 16 * TRSM_LD;
        const size_t dofs = (size_t)(8 * nt + 2 * t) * TRSM_LD + 16 * mt + 2 * g;
        const size_t aofs = (size_t)t * TRSM_LD + 16 * mt + 2 * g;
        auto mul16 = [&](double (&acc)[4], const double *a0, const double (&b)[2][2]) {
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                const double2 lo = *reinterpret_cast<const double2 *>(a0 + (size_t)(8 * kk) * TRSM_LD);
                const double2 hi = *reinterpret_cast<const double2 *>(a0 + (size_t)(8 * kk + 4) * TRSM_LD);
                const double a[4] = {lo.x, lo.y, hi.x, hi.y};
                dmma1688(acc, a, b[kk]);
            }
        };
        double o[4] = {0.0, 0.0, 0.0, 0.0};
        mul16(o, ya + (size_t)j0 * TRSM_LD, bi);
        *reinterpret_cast<double2 *>(xw + dofs) = make_double2(o[0], o[2]);
        *reinterpret_cast<double2 *>(xw + dofs + TRSM_LD) = make_double2(o[1], o[3]);
        __syncthreads();
        double xt[4] = {0.0, 0.0, 0.0, 0.0};
        mul16(xt, xw + aofs, bt);
        *reinterpret_cast<double2 *>(cw + dofs) = make_double2(r[0] - xt[0], r[2] - xt[2]);
        *reinterpret_cast<double2 *>(cw + dofs + TRSM_LD) = make_double2(r[1] - xt[1], r[3] - xt[3]);
        __syncthreads();
        mul16(o, cw + aofs, bi);
        *d0 = make_double2(o[0], o[2]);
        *d1 = make_double2(o[1], o[3]);
    }
    __syncthreads();
    if (!UCASE) {
        if (lane < nv) {
            double *x = X + (size_t)warp * lda + lane;
            const size_t step = (size_t)4 * lda;
            for (int c = warp; c < ns; c += 4, x += step) *x = Ys[c * TRSM_LD + prow(lane)];
        }
    } else if (us < nv) {
        double *x = X + (size_t)us * ns;
        for (int c = uc; c < ns; c += 4) x[c] = Ys[c * TRSM_LD + prow(us)];
    }
}

template <bool UCASE, class LU>
static int launch_trsm(const LU &d, const Batch &b, int64_t ctas, int max_ns, const double *dinv, cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    static std::atomic<unsigned long long> attr{0};
    ensure_dyn_smem(trsm_kernel<UCASE, LU>, (int)trsm_smem(MAX_NS), attr);
    trsm_kernel<UCASE, LU><<<member_grid(d, (unsigned)ctas), TRSM_THREADS, trsm_smem(max_ns), s>>>(d, b, dinv);
    return 1;
}
int launch_trsm_l(const DeviceLU &d, const Batch &b, int64_t ctas, int max_ns, const double *dinv, cudaStream_t s)
{
    return launch_trsm<false>(d, b, ctas, max_ns, dinv, s);
}
int launch_trsm_u(const DeviceLU &d, const Batch &b, int64_t ctas, int max_ns, const double *dinv, cudaStream_t s)
{
    return launch_trsm<true>(d, b, ctas, max_ns, dinv, s);
}
int launch_trsm_l(const BatchedLU &d, const Batch &b, int64_t ctas, int max_ns, const double *dinv, cudaStream_t s)
{
    return launch_trsm<false>(d, b, ctas, max_ns, dinv, s);
}
int launch_trsm_u(const BatchedLU &d, const Batch &b, int64_t ctas, int max_ns, const double *dinv, cudaStream_t s)
{
    return launch_trsm<true>(d, b, ctas, max_ns, dinv, s);
}

// ------------------------------------------------------------------------------------------------
// FP64 tensor-core GEMM tile (DMMA m8n8k4), cp.async multi-stage pipeline
// ------------------------------------------------------------------------------------------------
template <int BM, int BN, int WARPS_M, int WARPS_N>
struct GemmCfg {
    static constexpr int BK = 16, STAGES = 3;
    static constexpr int NT = 32 * WARPS_M * WARPS_N;
    static constexpr int WTM = BM / WARPS_M, WTN = BN / WARPS_N;
    static constexpr int MI = WTM / 8, NI = WTN / 8;
    static constexpr int LDA = BM + 4, LDB = BK + 4;  // strides == 4 (mod 16) doubles: conflict-free fragment loads
    static constexpr int A_STAGE = BK * LDA, B_STAGE = BN * LDB;
    static constexpr size_t SMEM = sizeof(double) * STAGES * (A_STAGE + B_STAGE);
};

// acc[mi][ni][2] += A(m0.., :) * B(:, n0..) for the CTA tile; A is M x K (lda), B is K x N (ldb).
// Interior tiles (no M/N edge) and full k-steps use running pointers: every warp copies whole 32-row column
// slices of A (row offsets become immediates) and the B slices advance by constant strides.  Edge tiles and the
// K tail take the general predicated loader, which spends ~300 instructions per k-step on 64-bit address arithmetic
// and predicates.
template <int BM, int BN, int WARPS_M, int WARPS_N>
__device__ __forceinline__ void gemm_tile(const double *__restrict__ A, int lda, const double *__restrict__ B,
                                          int ldb, int M, int N, int K, int m0, int n0, double *sm,
                                          double (&acc)[BM / WARPS_M / 8][BN / WARPS_N / 8][2])
{
    using C = GemmCfg<BM, BN, WARPS_M, WARPS_N>;
    constexpr int BK = C::BK, STAGES = C::STAGES;
    constexpr int NW = C::NT / 32;                  // warps
    constexpr int CA = BK / NW, RA = BM / 32;       // A: columns per warp and 32-row slices per column
    constexpr int CB = C::NT / BK, JB = BN / CB;    // B: columns per pass and passes
    static_assert(BK % NW == 0 && BM % 32 == 0 && C::NT % BK == 0 && BN % CB == 0, "tile shape vs loader mapping");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm0 = (warp % WARPS_M) * C::WTM, wn0 = (warp / WARPS_M) * C::WTN;
    double *As = sm, *Bs = sm + STAGES * C::A_STAGE;
    const int KT = (K + BK - 1) / BK;
    const int KF = ((m0 + BM <= M) && (n0 + BN <= N)) ? K / BK : 0;  // k-steps the fast loader serves

    auto load = [&](int st, int kt) {  // general: predicated, zero-filled
        const int k0 = kt * BK;
        double *as = As + st * C::A_STAGE, *bs = Bs + st * C::B_STAGE;
#pragma unroll
        for (int idx = tid; idx < BK * BM; idx += C::NT) {
            int kk = idx / BM, mm = idx - kk * BM;
            bool p = (m0 + mm < M) && (k0 + kk < K);
            const double *src = p ? A + (size_t)(k0 + kk) * lda + m0 + mm : A;
            cp_async8(as + kk * C::LDA + mm, src, p);
        }
#pragma unroll
        for (int idx = tid; idx < BK * BN; idx += C::NT) {
            int nn = idx / BK, kk = idx - nn * BK;
            bool p = (n0 + nn < N) && (k0 + kk < K);
            const double *src = p ? B + (size_t)(n0 + nn) * ldb + k0 + kk : B;
            cp_async8(bs + nn * C::LDB + kk, src, p);
        }
    };
    // running sources/destinations of the fast loader (k-steps are issued in increasing order)
    const double *pa = A + (size_t)warp * lda + m0 + lane;
    const double *pb = B + (size_t)(n0 + tid / BK) * ldb + (tid % BK);
    const size_t a_col = (size_t)NW * lda, a_step = (size_t)BK * lda, b_col = (size_t)CB * ldb;
    double *const sa = As + warp * C::LDA + lane, *const sb = Bs + (tid / BK) * C::LDB + (tid % BK);
    auto load_fast = [&](int st) {
        double *as = sa + st * C::A_STAGE, *bs = sb + st * C::B_STAGE;
        const double *p = pa;
#pragma unroll
        for (int c = 0; c < CA; ++c) {
#pragma unroll
            for (int r = 0; r < RA; ++r) cp_async8_plain(as + c * NW * C::LDA + 32 * r, p + 32 * r);
            p += a_col;
        }
        const double *q = pb;
#pragma unroll
        for (int j = 0; j < JB; ++j) {
            cp_async8_plain(bs + j * CB * C::LDB, q);
            q += b_col;
        }
        pa += a_step;
        pb += BK;
    };
    auto issue = [&](int st, int kt) {
        if (kt < KF) load_fast(st);
        else load(st, kt);
    };

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < KT) issue(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < KT; ++kt) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        if (kt + STAGES - 1 < KT) issue((kt + STAGES - 1) % STAGES, kt + STAGES - 1);
        cp_async_commit();
        const double *as = As + (kt % STAGES) * C::A_STAGE, *bs = Bs + (kt % STAGES) * C::B_STAGE;
#pragma unroll
        for (int k4 = 0; k4 < BK / 4; ++k4) {
            double a[C::MI], bb[C::NI];
#pragma unroll
            for (int mi = 0; mi < C::MI; ++mi) a[mi] = as[(k4 * 4 + (lane & 3)) * C::LDA + wm0 + mi * 8 + (lane >> 2)];
#pragma unroll
            for (int ni = 0; ni < C::NI; ++ni) bb[ni] = bs[(wn0 + ni * 8 + (lane >> 2)) * C::LDB + k4 * 4 + (lane & 3)];
#pragma unroll
            for (int mi = 0; mi < C::MI; ++mi)
#pragma unroll
                for (int ni = 0; ni < C::NI; ++ni) dmma884(acc[mi][ni][0], acc[mi][ni][1], a[mi], bb[ni]);
        }
    }
    cp_async_wait<0>();
}

// ------------------------------------------------------------------------------------------------
// Schur-complement update of a batch of supernodes: GEMM tile + fused subtract-scatter epilogue
// ------------------------------------------------------------------------------------------------
// Tile t of a rows x cols rectangle of tiles, in bands of SCHUR_BAND tile rows taken one after the other, column by
// column within a band.  CTAs start in tile order, so the ~2 per SM in flight at once share a few row tiles of A (L panel)
// and column tiles of B (U panel), a working set of about 6 MB.  Column by column over all rows of a tall update
// (m ~ 10^4: 80 row tiles, 21 MB of A at k = 256), the tiles in flight touch the whole L panel for every column tile.
constexpr int SCHUR_BAND = 16;
__device__ __forceinline__ void band_order(int t, int rows, int cols, int &r, int &c)
{
    const int per = SCHUR_BAND * cols, b = t / per, r0 = b * SCHUR_BAND, h = min(SCHUR_BAND, rows - r0), u = t - b * per;
    r = r0 + u % h; c = u / h;
}

// (tm, tn) of tile number `tile` of a supernode with BM x BN tiles.  mode 0: all tiles in bands; 1 (urgent): the
// first tcu tile columns entirely, then the first tru tile rows of the rest; 2 (bulk): the others, in bands
template <int BM, int BN>
__device__ __forceinline__ void schur_tile_of(const NodeDesc &nd, int tile, int mode, int &tm, int &tn)
{
    const int tiles_m = (nd.m + BM - 1) / BM, tiles_n = (nd.ncols + BN - 1) / BN;
    if (mode == 0) {
        band_order(tile, tiles_m, tiles_n, tm, tn);
    } else {
        const int tru = (nd.urg_rows + BM - 1) / BM, tcu = (nd.urg_cols + BN - 1) / BN;
        if (mode == 1) {
            if (tile < tiles_m * tcu) { tm = tile % tiles_m; tn = tile / tiles_m; }
            else { const int t = tile - tiles_m * tcu; tm = t % tru; tn = tcu + t / tru; }
        } else {
            band_order(tile, tiles_m - tru, tiles_n - tcu, tm, tn);
            tm += tru; tn += tcu;
        }
    }
}

template <int BM, int BN, int WARPS_M, int WARPS_N, class LU>
__global__ void __launch_bounds__(32 * WARPS_M * WARPS_N, (32 * WARPS_M * WARPS_N <= 256) ? 2 : 1)
    schur_kernel(LU dd, Batch b, int mode, int split_n, int split_i)
{
    using C = GemmCfg<BM, BN, WARPS_M, WARPS_N>;
    extern __shared__ double sm[];
    const DeviceLU &d = member_view(dd);
    // cooperative ancestors: the ranks of a Z group deal the tiles of the batch round-robin
    const int64_t gt = (int64_t)blockIdx.x * split_n + split_i;
    if (gt >= b.prefix[b.count]) return;
    const int slot = find_slot(b.prefix, b.count, gt);
    const int k = b.nodes[slot];
    const NodeDesc nd = d.nodes[k];
    int tm, tn;
    schur_tile_of<BM, BN>(nd, (int)(gt - b.prefix[slot]), mode, tm, tn);
    const int m0 = tm * BM, n0 = tn * BN;

    double acc[C::MI][C::NI][2];
#pragma unroll
    for (int mi = 0; mi < C::MI; ++mi)
#pragma unroll
        for (int ni = 0; ni < C::NI; ++ni) acc[mi][ni][0] = acc[mi][ni][1] = 0.0;

    gemm_tile<BM, BN, WARPS_M, WARPS_N>(d.val + nd.lval + nd.ns, nd.nsupr, d.val + nd.uval, nd.ns, nd.m, nd.ncols, nd.ns,
                                        m0, n0, sm, acc);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm0 = m0 + (warp % WARPS_M) * C::WTM, wn0 = n0 + (warp / WARPS_M) * C::WTN;
    const RowInfo *rinfo = d.rowinfo + nd.ws_row;
    const ColInfo *cinfo = d.colinfo + nd.ws_col;
    // per-thread row descriptors (MI rows), reused for every column
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
        // destination offsets of the 2 x MI elements of this 8-column slab, then one batch of independent REDs
        int64_t idx[2][C::MI];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int j = wn0 + ni * 8 + 2 * (lane & 3) + e;
            const bool cok = j < nd.ncols;
            ColInfo cj;
            if (cok) cj = cinfo[j];
#pragma unroll
            for (int mi = 0; mi < C::MI; ++mi) {
                idx[e][mi] = -1;
                if (!cok || !rok[mi]) continue;
                const int i = wm0 + mi * 8 + (lane >> 2);
                if (ri[mi].ib >= cj.jb) {
                    const int p = d.lrel[cj.lrel_off + i];
                    if (p >= 0) idx[e][mi] = cj.lbase + p;
                } else {
                    const int q = d.urel[ri[mi].urel_off + j];
                    if (q >= 0) idx[e][mi] = ri[mi].ubase + (int64_t)q * ri[mi].ldu;
                }
            }
        }
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
            for (int mi = 0; mi < C::MI; ++mi)
                if (idx[e][mi] >= 0) atomicAdd(d.val + idx[e][mi], flip_sign(acc[mi][ni][e]));
    }
}

// ------------------------------------------------------------------------------------------------
// The Hopper main loop: mma.sync.m16n8k8.f64 (DMMA.16x8x8) on 64 x 32 warp tiles.  Per k8 step a warp issues 16 MMAs
// fed by 12 16-byte shared loads (0.375 B of shared memory per FMA, against 0.5 with 32 x 32 tiles of DMMA.8x8x4).
// The loader permutes the shared image so that every lane's fragment pairs are adjacent: rows g and g+8 of a 16-row
// block of A (row r at prow(r)), k and k+4 of an 8-deep slice of B (at pk(k)).  A and B columns are only 8-byte
// aligned in global memory (lda = nsupr, ldb = ns), so the copies stay 8-byte cp.async.
// ------------------------------------------------------------------------------------------------
template <int BM, int BN, int WARPS_M, int WARPS_N, int BK, int STAGES>
struct HCfg {
    static constexpr int NT = 32 * WARPS_M * WARPS_N;
    static constexpr int WTM = BM / WARPS_M, WTN = BN / WARPS_N;
    static constexpr int MT = WTM / 16, NT8 = WTN / 8;
    static constexpr int LDA = BM + 4, LDB = BK + 8;  // == 4 and 8 (mod 16) doubles: conflict-free 16-byte fragment loads
    static constexpr int A_STAGE = BK * LDA, B_STAGE = BN * LDB;
    static constexpr size_t SMEM = sizeof(double) * STAGES * (A_STAGE + B_STAGE);
    static_assert(WTM % 16 == 0 && WTN % 8 == 0 && BK % 8 == 0, "tile shape vs m16n8k8");
};

template <int BM, int BN, int WARPS_M, int WARPS_N, int BK, int STAGES>
__device__ __forceinline__ void gemm_tile_h(const double *__restrict__ A, int lda, const double *__restrict__ B, int ldb,
                                            int M, int N, int K, int m0, int n0, double *sm,
                                            double (&acc)[BM / WARPS_M / 16][BN / WARPS_N / 8][4],
                                            const double *base = nullptr, const KSeg *seg = nullptr, int nseg = 0)
{
    using C = HCfg<BM, BN, WARPS_M, WARPS_N, BK, STAGES>;
    constexpr int NW = C::NT / 32;
    constexpr int CA = BK / NW, RA = BM / 32;       // A: columns per warp and 32-row slices per column
    constexpr int CB = C::NT / BK, JB = BN / CB;    // B: columns per pass and passes
    static_assert(BK % NW == 0 && BM % 32 == 0 && C::NT % BK == 0 && BN % CB == 0, "tile shape vs loader mapping");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int wm0 = (warp % WARPS_M) * C::WTM, wn0 = (warp / WARPS_M) * C::WTN;
    double *As = sm, *Bs = sm + STAGES * C::A_STAGE;
    // K runs over segments: (A, B, K) first, then seg[0 .. nseg) (A = base + a ...).  Each segment takes
    // ceil(k / BK) k-steps, its tail on the predicated loader; the pipeline runs straight across the boundaries.
    int KT = (K + BK - 1) / BK;
    for (int q = 0; q < nseg; ++q) KT += (seg[q].k + BK - 1) / BK;
    const bool full = (m0 + BM <= M) && (n0 + BN <= N);  // whole k-steps of a full tile take the unpredicated loader
    int k0 = 0, sg = 0;                                    // the loader is at depth k0 of segment sg (0: the first)

    auto load = [&](int st) {  // edge tiles and the K tail: predicated, zero-filled
        double *as = As + st * C::A_STAGE, *bs = Bs + st * C::B_STAGE;
#pragma unroll
        for (int idx = tid; idx < BK * BM; idx += C::NT) {
            const int kk = idx / BM, mm = idx - kk * BM;
            const bool p = (m0 + mm < M) && (k0 + kk < K);
            cp_async8(as + kk * C::LDA + prow(mm), p ? A + (size_t)(k0 + kk) * lda + m0 + mm : A, p);
        }
#pragma unroll
        for (int idx = tid; idx < BK * BN; idx += C::NT) {
            const int nn = idx / BK, kk = idx - nn * BK;
            const bool p = (n0 + nn < N) && (k0 + kk < K);
            cp_async8(bs + nn * C::LDB + pk(kk), p ? B + (size_t)(n0 + nn) * ldb + k0 + kk : B, p);
        }
    };
    // running sources of the unpredicated loader (k-steps are issued in increasing order); each warp copies whole
    // 32-row column slices of A, so the permuted destinations are a per-lane constant plus immediates
    const double *pa = A + (size_t)warp * lda + m0 + lane;
    const double *pb = B + (size_t)(n0 + tid / BK) * ldb + (tid % BK);
    double *const sa = As + warp * C::LDA + prow(lane), *const sb = Bs + (tid / BK) * C::LDB + pk(tid % BK);
    auto load_fast = [&](int st) {
        const size_t a_col = (size_t)NW * lda, a_step = (size_t)BK * lda, b_col = (size_t)CB * ldb;
        double *as = sa + st * C::A_STAGE, *bs = sb + st * C::B_STAGE;
        const double *p = pa;
#pragma unroll
        for (int c = 0; c < CA; ++c) {
#pragma unroll
            for (int r = 0; r < RA; ++r) cp_async8_plain(as + c * NW * C::LDA + 32 * r, p + 32 * r);
            p += a_col;
        }
        const double *q = pb;
#pragma unroll
        for (int j = 0; j < JB; ++j) {
            cp_async8_plain(bs + j * CB * C::LDB, q);
            q += b_col;
        }
        pa += a_step;
        pb += BK;
    };
    auto issue = [&](int st) {  // the next k-step (they are issued in order)
        if (k0 >= K) {          // re-seat the loader on the next segment
            const KSeg q = seg[sg++];
            A = base + q.a; lda = q.lda; B = base + q.b; ldb = q.ldb; K = q.k; k0 = 0;
            pa = A + (size_t)warp * lda + m0 + lane;
            pb = B + (size_t)(n0 + tid / BK) * ldb + (tid % BK);
        }
        if (full && k0 + BK <= K) load_fast(st);
        else load(st);
        k0 += BK;
    };

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < KT) issue(s);
        cp_async_commit();
    }
    for (int kt = 0; kt < KT; ++kt) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        if (kt + STAGES - 1 < KT) issue((kt + STAGES - 1) % STAGES);
        cp_async_commit();
        const double *as = As + (kt % STAGES) * C::A_STAGE + t * C::LDA + wm0 + 2 * g;
        const double *bs = Bs + (kt % STAGES) * C::B_STAGE + (wn0 + g) * C::LDB + 2 * t;
#pragma unroll
        for (int k8 = 0; k8 < BK / 8; ++k8) {
            double a[C::MT][4], bb[C::NT8][2];
#pragma unroll
            for (int mt = 0; mt < C::MT; ++mt) {
                const double2 lo = *reinterpret_cast<const double2 *>(as + k8 * 8 * C::LDA + 16 * mt);
                const double2 hi = *reinterpret_cast<const double2 *>(as + (k8 * 8 + 4) * C::LDA + 16 * mt);
                a[mt][0] = lo.x; a[mt][1] = lo.y; a[mt][2] = hi.x; a[mt][3] = hi.y;
            }
#pragma unroll
            for (int nt = 0; nt < C::NT8; ++nt) {
                const double2 v = *reinterpret_cast<const double2 *>(bs + 8 * nt * C::LDB + 8 * k8);
                bb[nt][0] = v.x; bb[nt][1] = v.y;
            }
#pragma unroll
            for (int mt = 0; mt < C::MT; ++mt)
#pragma unroll
                for (int nt = 0; nt < C::NT8; ++nt) dmma1688(acc[mt][nt], a[mt], bb[nt]);
        }
    }
    cp_async_wait<0>();
}

// Schur update on the Hopper main loop: the tile enumeration (modes, Z split) and destination maps of schur_kernel,
// atomic scatter.  Thread (g, t) of a warp holds rows 16 mt + g + 8 h and columns 8 nt + 2 t + e of its warp tile.
template <int BM, int BN, int WARPS_M, int WARPS_N, int BK, int STAGES, int MINB, class LU = DeviceLU>
__global__ void __launch_bounds__(32 * WARPS_M * WARPS_N, MINB)
    schur_kernel_h(LU dd, Batch b, int mode, int split_n, int split_i)
{
    using C = HCfg<BM, BN, WARPS_M, WARPS_N, BK, STAGES>;
    extern __shared__ __align__(16) double sm[];
    const DeviceLU &d = member_view(dd);
    const int64_t gt = (int64_t)blockIdx.x * split_n + split_i;
    if (gt >= b.prefix[b.count]) return;
    const int slot = find_slot(b.prefix, b.count, gt);
    const int k = b.nodes[slot];
    const NodeDesc nd = d.nodes[k];
    int tm, tn;
    // a deferred child has only its panel tiles (mode 1 with urg = its parent's columns), whatever the launch
    schur_tile_of<BM, BN>(nd, (int)(gt - b.prefix[slot]), nd.defer ? 1 : mode, tm, tn);
    const int m0 = tm * BM, n0 = tn * BN;

    double acc[C::MT][C::NT8][4];
#pragma unroll
    for (int mt = 0; mt < C::MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < C::NT8; ++nt) acc[mt][nt][0] = acc[mt][nt][1] = acc[mt][nt][2] = acc[mt][nt][3] = 0.0;
    gemm_tile_h<BM, BN, WARPS_M, WARPS_N, BK, STAGES>(d.val + nd.lval + nd.ns, nd.nsupr, d.val + nd.uval, nd.ns, nd.m,
                                                      nd.ncols, nd.ns, m0, n0, sm, acc, d.val, d.kseg + nd.kseg_off, nd.nkseg);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm0 = m0 + (warp % WARPS_M) * C::WTM + (lane >> 2), wn0 = n0 + (warp / WARPS_M) * C::WTN + 2 * (lane & 3);
    // a deferred child leaves the elements below and right of its parent's columns to its parent's update
    const int defer_i = nd.defer ? nd.urg_rows : nd.m, defer_j = nd.defer ? nd.urg_cols : nd.ncols;
    const RowInfo *rinfo = d.rowinfo + nd.ws_row;
    const ColInfo *cinfo = d.colinfo + nd.ws_col;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        RowInfo ri[C::MT];
        bool rok[C::MT];
#pragma unroll
        for (int mt = 0; mt < C::MT; ++mt) {
            const int i = wm0 + 16 * mt + 8 * h;
            rok[mt] = i < nd.m;
            if (rok[mt]) ri[mt] = rinfo[i];
        }
#pragma unroll
        for (int nt = 0; nt < C::NT8; ++nt) {
            int64_t idx[2][C::MT];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int j = wn0 + 8 * nt + e;
                const bool cok = j < nd.ncols;
                ColInfo cj;
                if (cok) cj = cinfo[j];
#pragma unroll
                for (int mt = 0; mt < C::MT; ++mt) {
                    idx[e][mt] = -1;
                    const int i = wm0 + 16 * mt + 8 * h;
                    if (!cok || !rok[mt] || (i >= defer_i && j >= defer_j)) continue;
                    if (ri[mt].ib >= cj.jb) {
                        const int p = d.lrel[cj.lrel_off + i];
                        if (p >= 0) idx[e][mt] = cj.lbase + p;
                    } else {
                        const int q = d.urel[ri[mt].urel_off + j];
                        if (q >= 0) idx[e][mt] = ri[mt].ubase + (int64_t)q * ri[mt].ldu;
                    }
                }
            }
#pragma unroll
            for (int e = 0; e < 2; ++e)
#pragma unroll
                for (int mt = 0; mt < C::MT; ++mt)
                    if (idx[e][mt] >= 0) atomicAdd(d.val + idx[e][mt], flip_sign(acc[mt][nt][2 * h + e]));
        }
    }
}

// the tile of schur_kernel_h on the Schur path (SCHUR_BM_BIG x SCHUR_BN_TILE: the host plan enumerates these tiles)
#define SCHUR_H_TILE SCHUR_BM_BIG, SCHUR_BN_TILE, 2, 2, 16, 3, 2
template <int BM, int BN, int WARPS_M, int WARPS_N, int BK, int STAGES, int MINB, class LU>
static int launch_schur_h(const LU &d, const Batch &b, int64_t ctas, int mode, int split_n, int split_i, cudaStream_t s)
{
    using C = HCfg<BM, BN, WARPS_M, WARPS_N, BK, STAGES>;
    static std::atomic<unsigned long long> attr_0{0};
    ensure_dyn_smem(schur_kernel_h<BM, BN, WARPS_M, WARPS_N, BK, STAGES, MINB, LU>, (int)C::SMEM, attr_0);
    const int64_t grid = (ctas + split_n - 1) / split_n;
    schur_kernel_h<BM, BN, WARPS_M, WARPS_N, BK, STAGES, MINB, LU><<<member_grid(d, (unsigned)grid), C::NT, C::SMEM, s>>>(d, b, mode, split_n, split_i);
    return 1;
}

// the small tiles (updates of fewer than 96 rows or columns): schur_kernel on mma.sync.m8n8k4.f64
template <class LU>
static int launch_schur_small(const LU &d, const Batch &b, int64_t ctas, int mode, int split_n, int split_i, cudaStream_t s)
{
    using C = GemmCfg<SCHUR_BM_SMALL, SCHUR_BN_SMALL, 2, 2>;
    static std::atomic<unsigned long long> attr_0{0};
    ensure_dyn_smem(schur_kernel<SCHUR_BM_SMALL, SCHUR_BN_SMALL, 2, 2, LU>, (int)C::SMEM, attr_0);
    const int64_t grid = (ctas + split_n - 1) / split_n;
    schur_kernel<SCHUR_BM_SMALL, SCHUR_BN_SMALL, 2, 2, LU><<<member_grid(d, (unsigned)grid), C::NT, C::SMEM, s>>>(d, b, mode, split_n, split_i);
    return 1;
}

int launch_schur(const DeviceLU &d, const Batch &b, int64_t ctas, int big, int mode, int split_n, int split_i, cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    if (big) return launch_schur_h<SCHUR_H_TILE>(d, b, ctas, mode, split_n, split_i, s);
    return launch_schur_small(d, b, ctas, mode, split_n, split_i, s);
}

// batched: the same two kernels, no Z split
int launch_schur(const BatchedLU &d, const Batch &b, int64_t ctas, int big, int mode, cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    if (big) return launch_schur_h<SCHUR_H_TILE>(d, b, ctas, mode, 1, 0, s);
    return launch_schur_small(d, b, ctas, mode, 1, 0, s);
}

// plain C -= A*B with the same main loop (kernel-level test and micro-benchmark of tile configurations)
template <int BM, int BN, int WARPS_M, int WARPS_N>
__global__ void __launch_bounds__(32 * WARPS_M * WARPS_N, 2)
    gemm_sub_kernel(int M, int N, int K, const double *A, int lda, const double *B, int ldb, double *Cm, int ldc)
{
    using C = GemmCfg<BM, BN, WARPS_M, WARPS_N>;
    extern __shared__ double sm[];
    const int tiles_m = (M + BM - 1) / BM;
    const int m0 = (blockIdx.x % tiles_m) * BM, n0 = (blockIdx.x / tiles_m) * BN;
    double acc[C::MI][C::NI][2];
#pragma unroll
    for (int mi = 0; mi < C::MI; ++mi)
#pragma unroll
        for (int ni = 0; ni < C::NI; ++ni) acc[mi][ni][0] = acc[mi][ni][1] = 0.0;
    gemm_tile<BM, BN, WARPS_M, WARPS_N>(A, lda, B, ldb, M, N, K, m0, n0, sm, acc);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm0 = m0 + (warp % WARPS_M) * C::WTM, wn0 = n0 + (warp / WARPS_M) * C::WTN;
#pragma unroll
    for (int ni = 0; ni < C::NI; ++ni)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int j = wn0 + ni * 8 + 2 * (lane & 3) + e;
            if (j >= N) continue;
#pragma unroll
            for (int mi = 0; mi < C::MI; ++mi) {
                const int i = wm0 + mi * 8 + (lane >> 2);
                if (i < M) atomicAdd(Cm + (size_t)j * ldc + i, flip_sign(acc[mi][ni][e]));
            }
        }
}

template <int BM, int BN, int WARPS_M, int WARPS_N>
static int launch_gemm_sub_t(int m, int n, int k, const double *a, int lda, const double *b, int ldb, double *c, int ldc,
                             cudaStream_t s)
{
    using C = GemmCfg<BM, BN, WARPS_M, WARPS_N>;
    static std::atomic<unsigned long long> attr_0{0};
    ensure_dyn_smem(gemm_sub_kernel<BM, BN, WARPS_M, WARPS_N>, (int)C::SMEM, attr_0);
    int64_t ctas = (int64_t)((m + BM - 1) / BM) * ((n + BN - 1) / BN);
    gemm_sub_kernel<BM, BN, WARPS_M, WARPS_N><<<(unsigned)ctas, C::NT, C::SMEM, s>>>(m, n, k, a, lda, b, ldb, c, ldc);
    return 1;
}

// the same on the Hopper main loop (gemm_tile_h)
template <int BM, int BN, int WARPS_M, int WARPS_N, int BK, int STAGES, int MINB>
__global__ void __launch_bounds__(32 * WARPS_M * WARPS_N, MINB)
    gemm_sub_kernel_h(int M, int N, int K, const double *A, int lda, const double *B, int ldb, double *Cm, int ldc,
                      const double *base, const KSeg *seg, int nseg)
{
    using C = HCfg<BM, BN, WARPS_M, WARPS_N, BK, STAGES>;
    extern __shared__ __align__(16) double sm[];
    const int tiles_m = (M + BM - 1) / BM;
    const int m0 = (blockIdx.x % tiles_m) * BM, n0 = (blockIdx.x / tiles_m) * BN;
    double acc[C::MT][C::NT8][4];
#pragma unroll
    for (int mt = 0; mt < C::MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < C::NT8; ++nt) acc[mt][nt][0] = acc[mt][nt][1] = acc[mt][nt][2] = acc[mt][nt][3] = 0.0;
    gemm_tile_h<BM, BN, WARPS_M, WARPS_N, BK, STAGES>(A, lda, B, ldb, M, N, K, m0, n0, sm, acc, base, seg, nseg);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm0 = m0 + (warp % WARPS_M) * C::WTM + (lane >> 2), wn0 = n0 + (warp / WARPS_M) * C::WTN + 2 * (lane & 3);
#pragma unroll
    for (int nt = 0; nt < C::NT8; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int j = wn0 + 8 * nt + e;
            if (j >= N) continue;
#pragma unroll
            for (int mt = 0; mt < C::MT; ++mt)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int i = wm0 + 16 * mt + 8 * h;
                    if (i < M) atomicAdd(Cm + (size_t)j * ldc + i, flip_sign(acc[mt][nt][2 * h + e]));
                }
        }
}

template <int BM, int BN, int WARPS_M, int WARPS_N, int BK, int STAGES, int MINB>
static int launch_gemm_sub_h(int m, int n, int k, const double *a, int lda, const double *b, int ldb, double *c, int ldc,
                             cudaStream_t s, const double *base = nullptr, const KSeg *seg = nullptr, int nseg = 0)
{
    using C = HCfg<BM, BN, WARPS_M, WARPS_N, BK, STAGES>;
    static std::atomic<unsigned long long> attr_0{0};
    ensure_dyn_smem(gemm_sub_kernel_h<BM, BN, WARPS_M, WARPS_N, BK, STAGES, MINB>, (int)C::SMEM, attr_0);
    const int64_t ctas = (int64_t)((m + BM - 1) / BM) * ((n + BN - 1) / BN);
    gemm_sub_kernel_h<BM, BN, WARPS_M, WARPS_N, BK, STAGES, MINB><<<(unsigned)ctas, C::NT, C::SMEM, s>>>(m, n, k, a, lda, b, ldb, c, ldc,
                                                                                                       base, seg, nseg);
    return 1;
}

int launch_gemm_sub_seg(int m, int n, int k, const double *a, int lda, const double *b, int ldb, const double *base, const KSeg *seg,
                        int nseg, double *c, int ldc, cudaStream_t s)
{
    if (m <= 0 || n <= 0) return 0;
    return launch_gemm_sub_h<SCHUR_H_TILE>(m, n, k, a, lda, b, ldb, c, ldc, s, base, seg, nseg);
}

int launch_gemm_sub(int m, int n, int k, const double *a, int lda, const double *b, int ldb, double *c, int ldc,
                    int variant, cudaStream_t s)
{
    if (m <= 0 || n <= 0) return 0;
    switch (variant) {
    // 30..: the Hopper main loop (gemm_tile_h, DMMA.16x8x8, 64 x 32 warp tiles)
    case 30: return launch_gemm_sub_h<128, 64, 2, 2, 16, 3, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 31: return launch_gemm_sub_h<128, 64, 2, 2, 32, 2, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 32: return launch_gemm_sub_h<128, 128, 2, 4, 16, 4, 1>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 33: return launch_gemm_sub_h<128, 128, 2, 4, 32, 3, 1>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 34: return launch_gemm_sub_h<64, 64, 1, 2, 16, 3, 3>(m, n, k, a, lda, b, ldb, c, ldc, s);    // 2 warps, 3 CTAs/SM
    default: break;
    }
    if (m >= 96 && n >= 96) return launch_gemm_sub_h<SCHUR_H_TILE>(m, n, k, a, lda, b, ldb, c, ldc, s);
    return launch_gemm_sub_t<SCHUR_BM_SMALL, SCHUR_BN_SMALL, 2, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
}

// ------------------------------------------------------------------------------------------------
// skyline <-> dense-packed U (boundary conversions), ancestor-reduction add
// ------------------------------------------------------------------------------------------------
template <bool PACK>
__global__ void __launch_bounds__(256) u_convert_kernel(DeviceLU d, Batch b, double *sky, const int64_t *sky_off)
{
    const int slot = find_slot(b.prefix, b.count, blockIdx.x);
    const int k = b.nodes[slot];
    const NodeDesc nd = d.nodes[k];
    const int chunk = (int)(blockIdx.x - b.prefix[slot]);
    const int ns = nd.ns, klst = nd.fsupc + ns;
    double *sk = sky + sky_off[slot];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int j = chunk * 32 + warp; j < min(nd.ncols, chunk * 32 + 32); j += 8) {
        const int fst = d.ufst[nd.ucol + j], len = klst - fst, top = ns - len;
        const int64_t seg = d.useg[nd.ucol + j];
        double *col = d.val + nd.uval + (size_t)j * ns;
        for (int r = lane; r < ns; r += 32) {
            if (PACK) { if (r >= top) sk[seg + (r - top)] = col[r]; }
            else col[r] = (r >= top) ? sk[seg + (r - top)] : 0.0;
        }
    }
}
int launch_u_convert(const DeviceLU &d, const Batch &b, int64_t ctas, int pack, double *sky,
                     const int64_t *sky_off, cudaStream_t s)
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
int launch_axpy(double *dst, const double *src, int64_t n, cudaStream_t s)
{
    if (n <= 0) return 0;
    int64_t blocks = (n + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    axpy_kernel<<<(unsigned)blocks, 256, 0, s>>>(dst, src, n);
    return 1;
}

__global__ void axpy_atomic_kernel(double *__restrict__ dst, const double *__restrict__ src, int64_t n)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) atomicAdd(dst + i, src[i]);
}
int launch_axpy_atomic(double *dst, const double *src, int64_t n, cudaStream_t s)
{
    if (n <= 0) return 0;
    int64_t blocks = (n + 255) / 256;
    if (blocks > 132 * 4) blocks = 132 * 4;  // a few CTAs per SM: it shares the GPU with the factorization
    axpy_atomic_kernel<<<(unsigned)blocks, 256, 0, s>>>(dst, src, n);
    return 1;
}

}  // namespace slu
