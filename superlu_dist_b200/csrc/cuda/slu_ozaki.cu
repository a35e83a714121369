// slu_ozaki.cu -- the Schur-complement GEMM of wide supernodes on the int8 tensor cores (Hopper wgmma).
//
// The tensor cores have no FP64 kind fast enough to matter beside int8, so V = L(below,k) * U(k,:) (dblock_gemm_scatter,
// SRC/double/dscatter3d.c:82-189) is computed EXACTLY-ROUNDED-EQUIVALENT from int8 slices (Ozaki scheme): every row i
// of the L operand is scaled by a power of two 2^-e_i so that |a| < 1 and cut into S signed base-128 digits
//        a = 2^e_i * sum_s d_s * 2^(-6-7s),   |d_s| <= 64            (S = 8: 55 bits >= the 53 of a double)
// and likewise every column j of the U operand (2^f_j, digits t).  Then
//        (A B)_ij = 2^(e_i+f_j-12) * sum_g 2^(-7g) * sum_{s+t=g} (A_s B_t)_ij
// where each A_s B_t is an int8 x int8 -> int32 product, exact on the tensor cores (|sum| <= 8*512*2^12 < 2^31).
// Products with s + t >= S are dropped: the result carries a NORMWISE error like a DGEMM's, at worst
// k * (S+2) * 2^(4-7S) * max_p|a_ip| * max_p|b_pj| (2.6e-13 for the default S = 7, 2.2e-15 for S = 8), typically one to two
// orders below -- bounds and cases in tests/test_gpu_ozaki.py.
//
// Mapping onto wgmma (one CTA = one 128 x NT tile of V; two consumer warpgroups, one per 64-row half, and one producer
// warpgroup that hands its registers to them with setmaxnreg):
//   * operands are pre-sliced ONCE per supernode by oz_slice_* into int8 tiles that already have the shared-memory
//     image wgmma wants (K-major "core matrices" of 8 rows x 16 bytes, no swizzle: LBO = 128 B between the two
//     16-byte K chunks, SBO = 256 B between 8-row groups), so a pipeline stage (all S slices of a 128-row x 32-k
//     A tile and of an NT-column x 32-k B tile) is TWO contiguous bulk copies (cp.async.bulk, the TMA engine's 1-D
//     mode) completing on an mbarrier;
//   * the S column-slices of B sit one under the other in shared memory, so ONE wgmma m64nNk32 of A_s against the
//     first (S-s)*NT rows of that stack yields A_s*B_t for every t <= S-1-s, landing in accumulator columns
//     [s*NT, S*NT): the accumulator of digit group g = s+t holds columns [g*NT, (g+1)*NT).  S instructions per
//     32-k step (N = S*NT ... NT) instead of S(S+1)/2;
//   * accumulators: S*NT/2 registers per consumer thread (112 for S = 7); the epilogue recombines the groups in FP64
//     (Horner in 2^-7), scales by 2^(e_i-6) * 2^(f_j-6) and subtract-scatters with RED.ADD.F64 exactly like the DMMA
//     kernel.
// One producer lane issues the bulk copies; the consumers release a stage (mbarrier arrive, one per warpgroup) once
// wgmma.wait_group shows the MMAs that read it are complete.  Every wait is bounded (trap after ~1 s) so a protocol
// bug cannot hang the GPU.
#include "slu_device.cuh"
#define SLU_COMMON_HELPERS_ONLY
#include "slu_kernels_common.cuh"
#include "slu_wgmma.cuh"

#include <cstdio>

namespace slu {
namespace oz {

constexpr int TM = 128;                 // rows of a tile: two wgmma M = 64 halves
constexpr int KSTEP = 32;               // int8 k per wgmma = k per pipeline stage
constexpr int A_SLICE_BYTES = TM * KSTEP;  // one slice of one A tile stage
constexpr int CONSUMERS = 256;          // two warpgroups: tile rows [0, 64) and [64, 128)
constexpr int THREADS = CONSUMERS + 128; // + the producer warpgroup (one lane issues the copies)

// ---------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    uint32_t done = 0;
    const long long t0 = clock64();
    while (true) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done)
                     : "r"(bar), "r"(parity)
                     : "memory");
        if (done) break;
        if (clock64() - t0 > 2000000000LL) __trap();  // ~1 s at 2 GHz: report, never hang
    }
}
// 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier (TMA engine; SASS UBLKCP)
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
// the same, landing at the same CTA-relative offset of every CTA in ctamask and signalling each one's mbarrier there
__device__ __forceinline__ void bulk_g2s_multicast(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar, uint16_t ctamask)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "h"(ctamask)
                 : "memory");
}
__device__ __forceinline__ void cluster_sync_all()
{
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank()
{
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// arrive on the mbarrier at the same CTA-relative offset in CTA `cta` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t cta)
{
    asm volatile("{\n\t.reg .b32 ra;\n\tmapa.shared::cluster.u32 ra, %0, %1;\n\t"
                 "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}" ::"r"(bar), "r"(cta)
                 : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// register budget of the 384-thread CTA: the producer warpgroup gives back what the accumulators of the consumers need
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory"); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory"); }

// shared-memory matrix descriptor, K-major, no swizzle: start >> 4 at [0,14), LBO >> 4 at [16,30) (128 B between the two
// 16-byte K chunks), SBO >> 4 at [32,46) (256 B between 8-row groups), base offset 0, layout type 0 at [62,64)
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr)
{
    return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)(128 >> 4) << 16) | ((uint64_t)(256 >> 4) << 32);
}


// ---------------------------------------------------------------------------------------------------------------
// slicing
// ---------------------------------------------------------------------------------------------------------------
// scale exponent of a row/column whose largest magnitude is mx: |x| < 2^e for every entry
__device__ __forceinline__ int scale_exp(double mx)
{
    if (!(mx > 0.0) || isinf(mx)) return 0;
    int e;
    frexp(mx, &e);  // mx = f * 2^e, 0.5 <= f < 1
    return e;
}
// digits of 16 consecutive k of one row/column -> one 16-byte word per slice.  x * p1 * p2 = x * 2^(7S-1-e) exactly.
template <int S>
__device__ __forceinline__ void slice16(const double (&x)[16], double p1, double p2, uint4 (&out)[S])
{
    uint32_t w[S][4];
#pragma unroll
    for (int s = 0; s < S; ++s) w[s][0] = w[s][1] = w[s][2] = w[s][3] = 0;
#pragma unroll
    for (int t = 0; t < 16; ++t) {
        long long M = __double2ll_rn(x[t] * p1 * p2);
#pragma unroll
        for (int s = S - 1; s >= 1; --s) {
            const int d = (int)((M + 64) & 127) - 64;  // balanced digit in [-64, 63]
            M = (M - d) >> 7;
            w[s][t >> 2] |= (uint32_t)(d & 0xFF) << (8 * (t & 3));
        }
        w[0][t >> 2] |= (uint32_t)((int)M & 0xFF) << (8 * (t & 3));  // |M| <= 64 here
    }
#pragma unroll
    for (int s = 0; s < S; ++s) out[s] = make_uint4(w[s][0], w[s][1], w[s][2], w[s][3]);
}
__device__ __forceinline__ void scale_factors(int e, int S, double &p1, double &p2, double &back)
{
    const int t = 7 * S - 1 - e;            // x * 2^t is an integer below 2^(7S-1)
    const int h = t / 2;
    p1 = ldexp(1.0, h);
    p2 = ldexp(1.0, t - h);
    back = ldexp(1.0, e - 6);               // the epilogue multiplies by 2^(e_i-6) * 2^(f_j-6)
}

// A operand: rows of a column-major m x k block (lda).  Pass 1: scale exponent per row.
__device__ __forceinline__ void a_rowmax(const double *__restrict__ A, int lda, int m, int k, int r, int *rexp)
{
    if (r >= m) return;
    double mx = 0.0;
    for (int p = 0; p < k; ++p) mx = fmax(mx, fabs(A[(size_t)p * lda + r]));
    rexp[r] = scale_exp(mx);
}
// Pass 2: thread = row r of tile rt, one 32-k step ks.  out is the tile array [rt][ks][s][4096 bytes].
template <int S>
__device__ __forceinline__ void a_slice_step(const double *__restrict__ A, int lda, int m, int k, int KS, int rt, int ks, int rl,
                                             const int *__restrict__ rexp, double *__restrict__ rscale, int8_t *__restrict__ out)
{
    const int r = rt * TM + rl;
    double p1 = 0, p2 = 0, back = 1.0;
    if (r < m) scale_factors(rexp[r], S, p1, p2, back);
    if (ks == 0 && r < m) rscale[r] = back;
    int8_t *base = out + ((size_t)(rt * KS + ks) * S) * A_SLICE_BYTES + (rl >> 3) * 256 + (rl & 7) * 16;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        double x[16];
#pragma unroll
        for (int t = 0; t < 16; ++t) {
            const int p = ks * KSTEP + half * 16 + t;
            x[t] = (r < m && p < k) ? A[(size_t)p * lda + r] : 0.0;
        }
        uint4 dg[S];
        slice16<S>(x, p1, p2, dg);
#pragma unroll
        for (int s = 0; s < S; ++s) *reinterpret_cast<uint4 *>(base + (size_t)s * A_SLICE_BYTES + half * 128) = dg[s];
    }
}
// B operand: columns of a column-major k x n block (ldb): K is contiguous.  One warp per column j (of the padded
// CT*NT columns); lane c covers k in [16c, 16c+16).  out is the tile array [ct][ks][t][NT*32 bytes].
template <int S, int NT>
__device__ __forceinline__ void b_slice_col(const double *__restrict__ B, int ldb, int k, int n, int KS, int j, int lane,
                                            double *__restrict__ cscale, int8_t *__restrict__ out)
{
    const int nchunk = 2 * KS;  // 16-k chunks, <= 32 for k <= 512
    double x[16];
    double mx = 0.0;
#pragma unroll
    for (int t = 0; t < 16; ++t) {
        const int p = lane * 16 + t;
        x[t] = (j < n && lane < nchunk && p < k) ? B[(size_t)j * ldb + p] : 0.0;
        mx = fmax(mx, fabs(x[t]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const int e = scale_exp(mx);
    double p1, p2, back;
    scale_factors(e, S, p1, p2, back);
    if (lane == 0 && j < n) cscale[j] = back;
    if (lane >= nchunk) return;
    uint4 dg[S];
    slice16<S>(x, p1, p2, dg);
    const int ct = j / NT, jl = j - ct * NT, ks = lane >> 1, half = lane & 1;
    int8_t *base = out + ((size_t)(ct * KS + ks) * S) * (NT * KSTEP) + (jl >> 3) * 256 + half * 128 + (jl & 7) * 16;
#pragma unroll
    for (int s = 0; s < S; ++s) *reinterpret_cast<uint4 *>(base + (size_t)s * (NT * KSTEP)) = dg[s];
}


// ---------------------------------------------------------------------------------------------------------------
// the tile product
// ---------------------------------------------------------------------------------------------------------------
template <int S, int NT, int STAGES>
struct TileCfg {
    static constexpr int A_STAGE = S * A_SLICE_BYTES, B_STAGE = S * NT * KSTEP, STAGE = A_STAGE + B_STAGE;
    static constexpr int ACC = S * NT / 2;   // accumulator registers per consumer thread
    static constexpr size_t SMEM = (size_t)STAGES * STAGE + 8 * 2 * STAGES + 1024;  // + alignment slack
    static_assert(S * NT <= 256, "accumulator groups exceed the widest wgmma (N = 256)");
    static_assert(NT % 32 == 0, "wgmma N of every slice instruction must be a multiple of 32");
};

// Stage ring at the 1 KB aligned start of dynamic shared memory: STAGES stages, then full[STAGES], empty[STAGES].
// CL > 1: the CL CTAs of a cluster work on CL neighbouring column tiles of the SAME row tile.  The A stage (S slices
// of 128 rows x 32 k, 4/5 of the operand bytes) is fetched from L2 once per cluster: CTA r copies the r-th 1/CL of it
// with a multicast bulk copy that lands in every CTA's shared memory and counts on every CTA's full barrier; a stage
// is re-used only when the MMAs of ALL CTAs have read it (empty barrier: 2 * CL arrivals, one per warpgroup of the
// cluster).
template <int S, int NT, int STAGES, int CL>
struct Pipe {
    using C = TileCfg<S, NT, STAGES>;
    uint32_t sbase;
    __device__ __forceinline__ explicit Pipe(uint8_t *smem_raw)
        : sbase(smem_u32(reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023))) {}
    __device__ __forceinline__ uint32_t full(int st) const { return sbase + STAGES * C::STAGE + 8 * st; }
    __device__ __forceinline__ uint32_t empty(int st) const { return sbase + STAGES * C::STAGE + 8 * (STAGES + st); }
    // thread 0; the caller then synchronises the CTA (CL > 1: the cluster) before anybody uses the barriers
    __device__ __forceinline__ void init() const
    {
        for (int st = 0; st < STAGES; ++st) { mbar_init(full(st), 1); mbar_init(empty(st), 2 * CL); }
        fence_barrier_init();
    }
    // producer lane: the ksteps stages of one tile; g counts k-steps over the CTA's life (ring slot and parity)
    __device__ __forceinline__ uint32_t load(const int8_t *ga, const int8_t *gb, int ksteps, uint32_t g) const
    {
        constexpr uint16_t MASK = (uint16_t)((1u << CL) - 1);
        constexpr int A_PART = C::A_STAGE / CL;
        static_assert(C::A_STAGE % (16 * CL) == 0, "A stage must split into 16-byte aligned parts");
        const uint32_t crank = CL > 1 ? cluster_ctarank() : 0;
        for (int ks = 0; ks < ksteps; ++ks, ++g) {
            const int st = g % STAGES;
            if (g >= (uint32_t)STAGES) mbar_wait(empty(st), ((g / STAGES) - 1) & 1);
            mbar_expect_tx(full(st), C::STAGE);
            const uint32_t a0 = sbase + st * C::STAGE;
            if (CL > 1)
                bulk_g2s_multicast(a0 + crank * A_PART, ga + (size_t)ks * C::A_STAGE + crank * A_PART, A_PART, full(st), MASK);
            else
                bulk_g2s(a0, ga + (size_t)ks * C::A_STAGE, C::A_STAGE, full(st));
            bulk_g2s(a0 + C::A_STAGE, gb + (size_t)ks * C::B_STAGE, C::B_STAGE, full(st));
        }
        return g;
    }
    __device__ __forceinline__ void release(int st) const
    {
        if ((threadIdx.x & 127) != 0) return;    // one arrival per warpgroup
        if (CL == 1) {
            mbar_arrive(empty(st));
        } else {
#pragma unroll
            for (int r = 0; r < CL; ++r) mbar_arrive_cluster(empty(st), r);
        }
    }
    // consumer warpgroups: acc = the S accumulator groups of this warpgroup's 64 x NT half of the tile
    __device__ __forceinline__ uint32_t mma(int ksteps, uint32_t g, uint32_t (&acc)[C::ACC]) const
    {
        const uint32_t half = (threadIdx.x >> 7) * (A_SLICE_BYTES / 2);   // rows [64 wg, 64 wg + 64) of each slice
        for (int ks = 0; ks < ksteps; ++ks, ++g) {
            const int st = g % STAGES;
            mbar_wait(full(st), (g / STAGES) & 1);
            const uint32_t a0 = sbase + st * C::STAGE;
            wgmma_fence();
            issue<0>(acc, smem_desc(a0 + half), smem_desc(a0 + C::A_STAGE), ks != 0);
            wgmma_commit();
            wgmma_wait<1>();                      // the previous k-step's MMAs are done: its stage is free
            if (ks > 0) release((g - 1) % STAGES);
        }
        wgmma_wait<0>();
        if (ksteps > 0) release((g - 1) % STAGES);
        return g;
    }
    template <int s>
    __device__ __forceinline__ static void issue(uint32_t (&acc)[C::ACC], uint64_t adesc, uint64_t bdesc, uint32_t accumulate)
    {
        if constexpr (s < S) {
            Wgmma<(S - s) * NT>::mma(acc + s * (NT / 2), adesc + (uint64_t)(s * (A_SLICE_BYTES >> 4)), bdesc, accumulate | s);
            issue<s + 1>(acc, adesc, bdesc, accumulate);
        }
    }
};

// Where a consumer thread's accumulator elements sit in the 128 x NT tile: register 4c + 2h + e of every group is
// (row tile_row(h), column 8c + 2 (lane % 4) + e).
__device__ __forceinline__ int tile_row(int h) { return ((threadIdx.x >> 5) << 4) + ((threadIdx.x & 31) >> 2) + 8 * h; }
__device__ __forceinline__ int tile_col(int c, int e) { return 8 * c + 2 * (threadIdx.x & 3) + e; }

// int32 -> double without the (slow) I2F.F64 path: 2^52 + 2^31 + x is exact in a double whose low word is x ^ 2^31
__device__ __forceinline__ double i2d(uint32_t x)
{
    return __hiloint2double(0x43300000, (int)(x ^ 0x80000000u)) - 4503601774854144.0;  // 2^52 + 2^31
}

// FP64 value (before the row/column scales) of accumulator element idx (0 <= idx < NT/2) of this thread.
// PAIRS (k-steps <= 8, i.e. supernodes <= 256 columns: |acc_g| <= 8*256*2^12 = 2^23): neighbouring groups are first
// combined exactly in int32 (acc_hi * 128 + acc_lo < 2^31), halving the conversions.
template <int S, int NT, bool PAIRS>
__device__ __forceinline__ double combine(const uint32_t *acc, int idx)
{
    auto r = [&](int g) { return acc[g * (NT / 2) + idx]; };
    if constexpr (PAIRS) {
        // sum_g acc_g 2^(-7g): pair (g-1, g), g odd, is P = acc_(g-1) * 128 + acc_g with weight 2^(-7g); Horner over
        // the pairs in 2^-14, a leading single group (S odd) pre-scaled by 2^7, the common 2^-7 applied last
        double acc_d;
        if constexpr (S % 2 == 1) acc_d = i2d(r(S - 1)) * 128.0;
        else acc_d = i2d((uint32_t)((int)r(S - 2) * 128 + (int)r(S - 1)));
#pragma unroll
        for (int g = (S % 2 == 1) ? S - 2 : S - 3; g >= 1; g -= 2)
            acc_d = fma(acc_d, 6.103515625e-05, i2d((uint32_t)((int)r(g - 1) * 128 + (int)r(g))));
        return acc_d * 0.0078125;
    } else {
        double acc_d = i2d(r(S - 1));
#pragma unroll
        for (int g = S - 2; g >= 0; --g) acc_d = fma(acc_d, 0.0078125, i2d(r(g)));
        return acc_d;
    }
}
template <int S, int NT>
__device__ __forceinline__ double combine(const uint32_t *acc, int idx, int ks)
{
    return ks <= 8 ? combine<S, NT, true>(acc, idx) : combine<S, NT, false>(acc, idx);
}

// ---------------------------------------------------------------------------------------------------------------
// dense C -= A * B (kernel-level test and micro-benchmark, slu_b200_k_gemm_sub variants >= 100)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) dense_rowmax_kernel(const double *A, int lda, int m, int k, int *rexp)
{
    a_rowmax(A, lda, m, k, blockIdx.x * 128 + threadIdx.x, rexp);
}
template <int S>
__global__ void __launch_bounds__(128) dense_slice_a_kernel(const double *A, int lda, int m, int k, int KS, const int *rexp,
                                                            double *rscale, int8_t *out)
{
    a_slice_step<S>(A, lda, m, k, KS, blockIdx.x, blockIdx.y, threadIdx.x, rexp, rscale, out);
}
template <int S, int NT>
__global__ void __launch_bounds__(128) dense_slice_b_kernel(const double *B, int ldb, int k, int n, int KS, int ncol_pad,
                                                            double *cscale, int8_t *out)
{
    const int j = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (j < ncol_pad) b_slice_col<S, NT>(B, ldb, k, n, KS, j, threadIdx.x & 31, cscale, out);
}


// EPI: 0 = subtract with RED.ADD.F64 (the real thing), 1 = plain store of -V (timing only), 2 = no output (timing only)
template <int S, int NT, int STAGES, int CL, int EPI>
__global__ void __launch_bounds__(THREADS, 1)
    dense_gemm_kernel(const int8_t *As, const int8_t *Bs, const double *rscale, const double *cscale, int M, int N, int KS,
                      double *Cm, int ldc)
{
    using C = TileCfg<S, NT, STAGES>;
    extern __shared__ uint8_t oz_smem[];
    const Pipe<S, NT, STAGES, CL> pipe(oz_smem);
    const int tiles_m = (M + TM - 1) / TM, tiles_n = (N + NT - 1) / NT;
    // a cluster takes CL neighbouring column tiles of one row tile
    const int cid = blockIdx.x / CL, cr = blockIdx.x % CL;
    const int tm = cid % tiles_m, tn = (cid / tiles_m) * CL + cr;
    const int tnb = min(tn, tiles_n - 1);          // a column tile past the edge still takes part in the cluster protocol
    if (threadIdx.x == 0) pipe.init();
    if (CL > 1) cluster_sync_all(); else __syncthreads();   // CL > 1: nobody multicasts before every barrier exists
    if (threadIdx.x >= CONSUMERS) {
        producer_regs();
        if (threadIdx.x == CONSUMERS) pipe.load(As + (size_t)tm * KS * C::A_STAGE, Bs + (size_t)tnb * KS * C::B_STAGE, KS, 0);
    } else {
        consumer_regs();
        uint32_t acc[C::ACC];
        pipe.mma(KS, 0, acc);
        if (EPI != 2 && tn < tiles_n) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = tm * TM + tile_row(h);
                if (i >= M) continue;
                const double rs = rscale[i];
#pragma unroll
                for (int c = 0; c < NT / 8; ++c)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int j = tn * NT + tile_col(c, e);
                        if (j >= N) continue;
                        const double v = combine<S, NT>(acc, 4 * c + 2 * h + e, KS) * rs * cscale[j];
                        if (EPI == 0) atomicAdd(Cm + (size_t)j * ldc + i, -v);
                        else Cm[(size_t)j * ldc + i] = -v;
                    }
            }
        }
    }
    if (CL > 1) cluster_sync_all();   // peers may still signal my barriers until they are done
}

struct DenseWs {          // scratch of the dense entry (per process, grows on demand)
    int8_t *a = nullptr, *b = nullptr;
    double *rs = nullptr, *cs = nullptr;
    int *rexp = nullptr;
    size_t na = 0, nb = 0, nr = 0, nc = 0;
};
static DenseWs g_dense;

template <class T>
static bool grow(T *&p, size_t &have, size_t need)
{
    if (need <= have) return true;
    if (p) cudaFree(p);
    p = nullptr;
    have = 0;
    if (cudaMalloc((void **)&p, need * sizeof(T)) != cudaSuccess) return false;
    have = need;
    return true;
}

template <class K>
static void launch_clustered(K kernel, dim3 grid, int threads, size_t smem, int cl, cudaStream_t s, void **args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cl; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    cudaLaunchKernelExC(&cfg, (const void *)kernel, args);
}

template <int S, int NT, int STAGES, int CL = 1, int EPI = 0>
static int launch_dense_t(int m, int n, int k, const double *a, int lda, const double *b, int ldb, double *c, int ldc, cudaStream_t s)
{
    using C = TileCfg<S, NT, STAGES>;
    const int KS = (k + KSTEP - 1) / KSTEP, RT = (m + TM - 1) / TM, CT = (n + NT - 1) / NT;
    if (k > 512) return 0;
    DenseWs &w = g_dense;
    size_t nrexp = w.nr;
    if (!grow(w.a, w.na, (size_t)RT * KS * C::A_STAGE) || !grow(w.b, w.nb, (size_t)CT * KS * C::B_STAGE) ||
        !grow(w.rs, w.nr, (size_t)RT * TM) || !grow(w.cs, w.nc, (size_t)CT * NT))
        return 0;
    if (nrexp != w.nr || !w.rexp) {
        if (w.rexp) cudaFree(w.rexp);
        if (cudaMalloc((void **)&w.rexp, w.nr * sizeof(int)) != cudaSuccess) return 0;
    }
    dense_rowmax_kernel<<<RT, 128, 0, s>>>(a, lda, m, k, w.rexp);
    dense_slice_a_kernel<S><<<dim3(RT, KS), 128, 0, s>>>(a, lda, m, k, KS, w.rexp, w.rs, w.a);
    dense_slice_b_kernel<S, NT><<<(CT * NT + 3) / 4, 128, 0, s>>>(b, ldb, k, n, KS, CT * NT, w.cs, w.b);
    static std::atomic<unsigned long long> attr{0};
    ensure_dyn_smem(dense_gemm_kernel<S, NT, STAGES, CL, EPI>, (int)C::SMEM, attr);
    const int grid = RT * ((CT + CL - 1) / CL) * CL;
    if (CL == 1) {
        dense_gemm_kernel<S, NT, STAGES, CL, EPI><<<grid, THREADS, C::SMEM, s>>>(w.a, w.b, w.rs, w.cs, m, n, KS, c, ldc);
    } else {
        const int8_t *pa = w.a, *pb = w.b;
        const double *prs = w.rs, *pcs = w.cs;
        int KSv = KS;
        void *args[] = {&pa, &pb, &prs, &pcs, &m, &n, &KSv, &c, &ldc};
        launch_clustered(dense_gemm_kernel<S, NT, STAGES, CL, EPI>, dim3(grid), THREADS, C::SMEM, CL, s, args);
    }
    return 4;
}

// ---------------------------------------------------------------------------------------------------------------
// the Schur update of a batch of wide supernodes (dblock_gemm_scatter + dscatter_l / dscatter_u, fused)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) schur_rowmax_kernel(DeviceLU d, const int32_t *nodes, const int64_t *p_rt, int count)
{
    const int slot = find_slot(p_rt, count, blockIdx.x);
    const NodeDesc nd = d.nodes[nodes[slot]];
    const int rt = (int)(blockIdx.x - p_rt[slot]);
    a_rowmax(d.val + nd.lval + nd.ns, nd.nsupr, nd.m, nd.ns, rt * TM + threadIdx.x, d.oz_rexp + nd.ws_ozs);
}
template <int S>
__global__ void __launch_bounds__(128) schur_slice_a_kernel(DeviceLU d, const int32_t *nodes, const int64_t *p_ak, int count)
{
    const int slot = find_slot(p_ak, count, blockIdx.x);
    const NodeDesc nd = d.nodes[nodes[slot]];
    const int idx = (int)(blockIdx.x - p_ak[slot]), KS = (nd.ns + KSTEP - 1) / KSTEP;
    a_slice_step<S>(d.val + nd.lval + nd.ns, nd.nsupr, nd.m, nd.ns, KS, idx / KS, idx % KS, threadIdx.x, d.oz_rexp + nd.ws_ozs,
                    d.oz_scale + nd.ws_ozs, d.oz_i8 + nd.ws_oza);
}
template <int S>
__global__ void __launch_bounds__(128) schur_slice_b_kernel(DeviceLU d, const int32_t *nodes, const int64_t *p_b, int count)
{
    const int slot = find_slot(p_b, count, blockIdx.x);
    const NodeDesc nd = d.nodes[nodes[slot]];
    const int j = (int)(blockIdx.x - p_b[slot]) * 4 + (threadIdx.x >> 5);
    const int npad = (nd.ncols + OZ_NT - 1) / OZ_NT * OZ_NT, mpad = (nd.m + TM - 1) / TM * TM;
    if (j < npad)
        b_slice_col<S, OZ_NT>(d.val + nd.uval, nd.ns, nd.ns, nd.ncols, (nd.ns + KSTEP - 1) / KSTEP, j, threadIdx.x & 31,
                              d.oz_scale + nd.ws_ozs + mpad, d.oz_i8 + nd.ws_ozb);
}

// Destinations of a consumer thread's 2 x NT/4 elements of tile (tm, tn) of supernode nd (column descriptors of the
// tile in shared memory: sc_*); off = -1: no destination.
struct Dest {
    long long off[2][OZ_NT / 4];
    double rs[2];
};
template <int NT>
__device__ __forceinline__ void dest_offsets(const DeviceLU &d, const NodeDesc &nd, int tm, int tn, bool tile_ok,
                                             const int *sc_jb, const long long *sc_lbase, const long long *sc_lrel, Dest &D)
{
    static_assert(NT == OZ_NT, "Dest holds OZ_NT / 4 columns per row");
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int i = tm * TM + tile_row(h);
        D.rs[h] = 0.0;
#pragma unroll
        for (int q = 0; q < NT / 4; ++q) D.off[h][q] = -1;
        if (!tile_ok || i >= nd.m) continue;
        const RowInfo ri = d.rowinfo[nd.ws_row + i];
        D.rs[h] = d.oz_scale[nd.ws_ozs + i];
        long long last_off = -1;
        int lpos = -1;
#pragma unroll
        for (int q = 0; q < NT / 4; ++q) {
            const int c = tile_col(q >> 1, q & 1), jb = sc_jb[c];
            if (jb < 0) continue;
            if (ri.ib >= jb) {   // destination in L panel jb: row position of my row there
                if (sc_lrel[c] != last_off) { last_off = sc_lrel[c]; lpos = d.lrel[last_off + i]; }
                if (lpos >= 0) D.off[h][q] = sc_lbase[c] + lpos;
            } else {             // destination in U panel ib: packed column position of column j there
                const int p = d.urel[ri.urel_off + tn * NT + c];
                if (p >= 0) D.off[h][q] = ri.ubase + (long long)p * ri.ldu;
            }
        }
    }
}
// recombine, scale, subtract-scatter
template <int S, int NT>
__device__ __forceinline__ void scatter(const DeviceLU &d, const uint32_t *acc, int ks, const Dest &D, const double *sc_scale)
{
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < NT / 4; ++q) {
            const long long o = D.off[h][q];
            if (o < 0) continue;
            const int c = tile_col(q >> 1, q & 1);
            const double val = flip_sign(combine<S, NT>(acc, 2 * (q >> 1) * 2 + 2 * h + (q & 1), ks) * D.rs[h] * sc_scale[c]);
            atomicAdd(d.val + o, val);
        }
}
template <int NT>
__device__ __forceinline__ void load_col_desc(const DeviceLU &d, const NodeDesc &nd, int tn, bool tile_ok, int c, int *sc_jb,
                                              long long *sc_lbase, long long *sc_lrel, double *sc_scale)
{
    const int j = tn * NT + c, mpad = (nd.m + TM - 1) / TM * TM;
    if (tile_ok && j < nd.ncols) {
        const ColInfo cj = d.colinfo[nd.ws_col + j];
        sc_jb[c] = cj.jb; sc_lbase[c] = cj.lbase; sc_lrel[c] = cj.lrel_off;
        sc_scale[c] = d.oz_scale[nd.ws_ozs + mpad + j];
    } else {
        sc_jb[c] = -1; sc_lbase[c] = 0; sc_lrel[c] = -1; sc_scale[c] = 0.0;
    }
}

// Tiles are enumerated in units of 128 x (CL * NT) "cluster tiles" (the host counts them with OZ_NT_HOST = CL * NT
// columns); the CL CTAs of a cluster take its CL column tiles and share the A operand through multicast.
// The destination offsets are worked out after the MMAs: held across the k-loop beside the S * NT / 2 accumulators
// they would spill.  Two consumer warpgroups per SM and the producer's prefetch cover part of that index chase.
template <int S, int NT, int STAGES, int CL>
__global__ void __launch_bounds__(THREADS, 1) schur_kernel_tc(DeviceLU d, Batch b, int mode, int split_n, int split_i)
{
    using C = TileCfg<S, NT, STAGES>;
    extern __shared__ uint8_t oz_smem[];
    __shared__ int sc_jb[NT];
    __shared__ long long sc_lbase[NT], sc_lrel[NT];
    __shared__ double sc_scale[NT];
    constexpr int NTC = NT * CL;
    const Pipe<S, NT, STAGES, CL> pipe(oz_smem);
    const int cr = blockIdx.x % CL;
    const int64_t gt = (int64_t)(blockIdx.x / CL) * split_n + split_i;  // cooperative ancestors: tiles dealt round-robin
    if (gt >= b.prefix[b.count]) return;                              // the whole cluster leaves
    const int slot = find_slot(b.prefix, b.count, gt);
    const int k = b.nodes[slot];
    const NodeDesc nd = d.nodes[k];
    const int tile = (int)(gt - b.prefix[slot]);
    const int tiles_m = (nd.m + TM - 1) / TM;
    int tm, tnc;
    if (mode == 0) {
        tm = tile % tiles_m; tnc = tile / tiles_m;
    } else {  // look-ahead split, same convention as schur_kernel (slu_kernels.cu)
        const int tru = (nd.urg_rows + TM - 1) / TM, tcu = (nd.urg_cols + NTC - 1) / NTC;
        if (mode == 1) {
            if (tile < tiles_m * tcu) { tm = tile % tiles_m; tnc = tile / tiles_m; }
            else { const int t = tile - tiles_m * tcu; tm = t % tru; tnc = tcu + t / tru; }
        } else {
            const int rm = tiles_m - tru;
            tm = tru + tile % rm; tnc = tcu + tile / rm;
        }
    }
    const int tiles_n = (nd.ncols + NT - 1) / NT;
    const int tn = tnc * CL + cr, tnb = min(tn, tiles_n - 1);   // a column tile past the edge still runs the protocol
    const int KS = (nd.ns + KSTEP - 1) / KSTEP;
    if (threadIdx.x == 0) pipe.init();
    if (threadIdx.x < NT) load_col_desc<NT>(d, nd, tn, tn < tiles_n, threadIdx.x, sc_jb, sc_lbase, sc_lrel, sc_scale);
    if (CL > 1) cluster_sync_all(); else __syncthreads();   // CL > 1: nobody multicasts before every barrier exists
    if (threadIdx.x >= CONSUMERS) {
        producer_regs();
        if (threadIdx.x == CONSUMERS)
            pipe.load(d.oz_i8 + nd.ws_oza + (size_t)tm * KS * C::A_STAGE, d.oz_i8 + nd.ws_ozb + (size_t)tnb * KS * C::B_STAGE, KS, 0);
    } else {
        consumer_regs();
        uint32_t acc[C::ACC];
        pipe.mma(KS, 0, acc);
        Dest D;
        dest_offsets<NT>(d, nd, tm, tn, tn < tiles_n, sc_jb, sc_lbase, sc_lrel, D);
        scatter<S, NT>(d, acc, KS, D, sc_scale);
    }
    if (CL > 1) cluster_sync_all();   // peers may still signal my barriers until they are done
}

template <int S>
static int launch_slice_t(const DeviceLU &d, const int32_t *nodes, int count, const int64_t *p_rt, int64_t n_rt, const int64_t *p_ak,
                          int64_t n_ak, const int64_t *p_b, int64_t n_b, cudaStream_t s)
{
    schur_rowmax_kernel<<<(unsigned)n_rt, 128, 0, s>>>(d, nodes, p_rt, count);
    schur_slice_a_kernel<S><<<(unsigned)n_ak, 128, 0, s>>>(d, nodes, p_ak, count);
    schur_slice_b_kernel<S><<<(unsigned)n_b, 128, 0, s>>>(d, nodes, p_b, count);
    return 3;
}
template <int S>
static int launch_schur_tc_t(const DeviceLU &d, const Batch &b, int64_t ctas, int mode, int split_n, int split_i, cudaStream_t s)
{
    // one CTA per SM (the S * NT / 2 accumulator registers per consumer thread rule out two): a four-deep ring
    constexpr int CL = OZ_CL, STAGES = 4;
    using C = TileCfg<S, OZ_NT, STAGES>;
    static std::atomic<unsigned long long> attr{0};
    ensure_dyn_smem(schur_kernel_tc<S, OZ_NT, STAGES, CL>, (int)C::SMEM, attr);
    const int64_t grid = (ctas + split_n - 1) / split_n * CL;
    if (CL == 1) {
        schur_kernel_tc<S, OZ_NT, STAGES, CL><<<(unsigned)grid, THREADS, C::SMEM, s>>>(d, b, mode, split_n, split_i);
    } else {
        DeviceLU dd = d;
        Batch bb = b;
        void *args[] = {&dd, &bb, &mode, &split_n, &split_i};
        launch_clustered(schur_kernel_tc<S, OZ_NT, STAGES, CL>, dim3((unsigned)grid), THREADS, C::SMEM, CL, s, args);
    }
    return 1;
}

}  // namespace oz

int launch_oz_slice(const DeviceLU &d, const int32_t *nodes, int count, const int64_t *p_rt, int64_t n_rt, const int64_t *p_ak,
                    int64_t n_ak, const int64_t *p_b, int64_t n_b, int S, cudaStream_t s)
{
    if (count <= 0 || n_rt <= 0) return 0;
    switch (S) {
    case 5: return oz::launch_slice_t<5>(d, nodes, count, p_rt, n_rt, p_ak, n_ak, p_b, n_b, s);
    case 6: return oz::launch_slice_t<6>(d, nodes, count, p_rt, n_rt, p_ak, n_ak, p_b, n_b, s);
    case 8: return oz::launch_slice_t<8>(d, nodes, count, p_rt, n_rt, p_ak, n_ak, p_b, n_b, s);
    default: return oz::launch_slice_t<7>(d, nodes, count, p_rt, n_rt, p_ak, n_ak, p_b, n_b, s);
    }
}
int launch_oz_schur(const DeviceLU &d, const Batch &b, int64_t ctas, int mode, int split_n, int split_i, int S, cudaStream_t s)
{
    if (b.count <= 0 || ctas <= 0) return 0;
    switch (S) {
    case 5: return oz::launch_schur_tc_t<5>(d, b, ctas, mode, split_n, split_i, s);
    case 6: return oz::launch_schur_tc_t<6>(d, b, ctas, mode, split_n, split_i, s);
    case 8: return oz::launch_schur_tc_t<8>(d, b, ctas, mode, split_n, split_i, s);
    default: return oz::launch_schur_tc_t<7>(d, b, ctas, mode, split_n, split_i, s);
    }
}

// variants 100 + 10*(S - 4) + {0: NT = 32, 1: NT = 64 (S <= 8), 2: NT = 32 with 3 stages}
int launch_gemm_sub_ozaki(int m, int n, int k, const double *a, int lda, const double *b, int ldb, double *c, int ldc, int variant,
                          cudaStream_t s)
{
    // 1xy: x = slices (1: 5, 2: 6, 3: 7, 4: 8), y = configuration:
    //   0: 2 stages, no cluster   1: 3 stages, no cluster   2: 2 stages, cluster 2   3: 3 stages, cluster 2   4: 3 stages, cluster 4
    //   8: as 1 with a plain store instead of RED (timing only)   9: as 1 without any output (timing only)
    switch (variant) {
    case 110: return oz::launch_dense_t<5, 32, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 120: return oz::launch_dense_t<6, 32, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 123: return oz::launch_dense_t<6, 32, 3, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 130: return oz::launch_dense_t<7, 32, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 131: return oz::launch_dense_t<7, 32, 3>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 132: return oz::launch_dense_t<7, 32, 2, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 133: return oz::launch_dense_t<7, 32, 3, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 134: return oz::launch_dense_t<7, 32, 3, 4>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 138: return oz::launch_dense_t<7, 32, 3, 1, 1>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 139: return oz::launch_dense_t<7, 32, 3, 1, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 140: return oz::launch_dense_t<8, 32, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 141: return oz::launch_dense_t<8, 32, 3>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 143: return oz::launch_dense_t<8, 32, 3, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 144: return oz::launch_dense_t<8, 32, 3, 4>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 148: return oz::launch_dense_t<7, 32, 3, 2, 1>(m, n, k, a, lda, b, ldb, c, ldc, s);
    case 149: return oz::launch_dense_t<7, 32, 3, 2, 2>(m, n, k, a, lda, b, ldb, c, ldc, s);
    default: return 0;
    }
}

}  // namespace slu
