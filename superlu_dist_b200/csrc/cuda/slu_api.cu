// slu_api.cu -- C-ABI (include/slu_b200.h) and host orchestration of the CUDA pdgstrf3d.
//
// The level loop mirrors pdgstrf3d (SRC/double/pdgstrf3d.c:333-385): for every Z-tree level this
// rank takes part in, factor its elimination sub-forest, combining the replicated ancestor copies
// along Z.  Inside a forest the reference walks supernodes one at a time with a look-ahead pipeline
// (dsparseTreeFactor_ASYNC, SRC/double/dtreeFactorization.c:295-716); here all supernodes of one
// topological level are processed by a handful of batched kernel launches (diagonal LU -> panel
// solves -> destination maps -> fused GEMM+scatter), the whole L/U resident in HBM, with
//   * look-ahead: panel work + "urgent" Schur tiles on a high-priority stream, the bulk on a second one;
//   * multi-GPU: either the reference's pairwise ancestor reduction, or (default) cooperative ancestors --
//     one NCCL all-reduce per topological level over the Z group, Schur tiles dealt round-robin;
//   * Pr x Pc > 1: block-cyclic pieces in, whole panels replicated per layer, same cooperative schedule;
//   * slu_b200_factor_host: D2H of every level overlapped with the factorization of the upper levels.
// No host compute touches the values.
//
// This file is compiled twice (see slu_device.cuh): as is for double, and through slu_api_z.cu with SLU_COMPLEX for
// doublecomplex, where the exported names become slu_b200_z_* / pzgstrf3d_b200 and the value pointers of the view
// are read as (re, im) pairs.
#include "slu_b200.h"
#include "slu_device.cuh"

#ifdef SLU_COMPLEX
#define slu_b200_handle_s slu_b200_zhandle_s
#define slu_b200_handle_t slu_b200_zhandle_t
#define slu_b200_create slu_b200_z_create
#define slu_b200_upload slu_b200_z_upload
#define slu_b200_factor slu_b200_z_factor
#define slu_b200_factor_host slu_b200_z_factor_host
#define slu_b200_download slu_b200_z_download
#define slu_b200_fill_csr slu_b200_z_fill_csr
#define slu_b200_solve slu_b200_z_solve
#define slu_b200_solve_trans slu_b200_z_solve_trans
#define slu_b200_get_stats slu_b200_z_get_stats
#define slu_b200_destroy slu_b200_z_destroy
#define slu_b200_plan slu_b200_z_plan
#define pdgstrf3d_b200 pzgstrf3d_b200
#define slu_b200_k_diag_lu slu_b200_z_k_diag_lu
#define slu_b200_k_trsm_l slu_b200_z_k_trsm_l
#define slu_b200_k_trsm_u slu_b200_z_k_trsm_u
#define slu_b200_k_gemm_sub slu_b200_z_k_gemm_sub
#define slu_b200_batch_create slu_b200_z_batch_create
#define slu_b200_batch_fill_csr slu_b200_z_batch_fill_csr
#define slu_b200_batch_factor slu_b200_z_batch_factor
#define slu_b200_batch_solve slu_b200_z_batch_solve
#define slu_b200_batch_solve_trans slu_b200_z_batch_solve_trans
#define slu_b200_batch_download slu_b200_z_batch_download
#define slu_b200_gscon slu_b200_z_gscon
#define slu_b200_batch_gscon slu_b200_z_batch_gscon
#define slu_b200_selinv slu_b200_z_selinv
#define slu_b200_selinv_get slu_b200_z_selinv_get
#define slu_b200_logdet slu_b200_z_logdet
#define slu_b200_batch_selinv slu_b200_z_batch_selinv
#define slu_b200_batch_selinv_get slu_b200_z_batch_selinv_get
#define slu_b200_batch_logdet slu_b200_z_batch_logdet
#define slu_b200_inertia slu_b200_z_inertia
#define slu_b200_batch_inertia slu_b200_z_batch_inertia
#define slu_b200_batch_fill_affine slu_b200_z_batch_fill_affine
#define slu_b200_schur_create slu_b200_z_schur_create
#define slu_b200_schur_get slu_b200_z_schur_get
#define slu_b200_schur_condense slu_b200_z_schur_condense
#define slu_b200_schur_expand slu_b200_z_schur_expand
#define slu_b200_batch_schur_create slu_b200_z_batch_schur_create
#define slu_b200_batch_schur_get slu_b200_z_batch_schur_get
#define slu_b200_batch_schur_condense slu_b200_z_batch_schur_condense
#define slu_b200_batch_schur_expand slu_b200_z_batch_schur_expand
#define slu_b200_fill_csr_scaled slu_b200_z_fill_csr_scaled
#define slu_b200_get_scaling slu_b200_z_get_scaling
#define slu_b200_solve_scaled slu_b200_z_solve_scaled
#define slu_b200_batch_fill_csr_scaled slu_b200_z_batch_fill_csr_scaled
#define slu_b200_batch_get_scaling slu_b200_z_batch_get_scaling
#define slu_b200_batch_solve_scaled slu_b200_z_batch_solve_scaled
#define slu_b200_gsrfs slu_b200_z_gsrfs
#define slu_b200_batch_gsrfs slu_b200_z_batch_gsrfs
#define slu_b200_refill slu_b200_z_refill
#define slu_b200_batch_refill slu_b200_z_batch_refill
#define slu_b200_solve_device slu_b200_z_solve_device
#define slu_b200_batch_solve_device slu_b200_z_batch_solve_device
#define slu_b200_solve_scaled_device slu_b200_z_solve_scaled_device
#define slu_b200_batch_solve_scaled_device slu_b200_z_batch_solve_scaled_device
#define slu_b200_factor_device slu_b200_z_factor_device
#define slu_b200_batch_factor_device slu_b200_z_batch_factor_device
#define slu_b200_get_device slu_b200_z_get_device
#define slu_b200_gsrfs_device slu_b200_z_gsrfs_device
#define slu_b200_batch_gsrfs_device slu_b200_z_batch_gsrfs_device
#define slu_b200_gscon_device slu_b200_z_gscon_device
#define slu_b200_batch_gscon_device slu_b200_z_batch_gscon_device
#define slu_b200_selinv_device slu_b200_z_selinv_device
#define slu_b200_batch_selinv_device slu_b200_z_batch_selinv_device
#define slu_b200_logdet_device slu_b200_z_logdet_device
#define slu_b200_batch_logdet_device slu_b200_z_batch_logdet_device
#define slu_b200_logdet_grad_device slu_b200_z_logdet_grad_device
#define slu_b200_batch_logdet_grad_device slu_b200_z_batch_logdet_grad_device
#define slu_b200_solve_grad_device slu_b200_z_solve_grad_device
#define slu_b200_batch_solve_grad_device slu_b200_z_batch_solve_grad_device
#define SLU_API "slu_b200_z_"     // name prefix of the exported calls, for error messages
#else
#define SLU_API "slu_b200_"
#endif

#include <dlfcn.h>
#include <omp.h>

#include <algorithm>
#include <array>
#include <map>
#include <mutex>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <functional>
#include <vector>

using namespace SLU_NS;

// one error string for both precisions (slu_b200_last_error)
#ifdef SLU_COMPLEX
extern thread_local std::string slu_b200_err_storage;
#else
thread_local std::string slu_b200_err_storage;
#endif
#define g_err slu_b200_err_storage

namespace {

int fail(const char *fmt, ...)
{
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return -1;
}
#define CU(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) return fail("%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
    } while (0)

double now_s()
{
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

constexpr int BC_HEADER = 2, LB_DESCRIPTOR = 2, BR_HEADER = 3, UB_DESCRIPTOR = 2;

// ---- NCCL through dlopen: no link-time dependency, the caller's (torch's) libnccl.so.2 is reused ---
}  // namespace

// the by-value ncclUniqueId argument of ncclCommInitRank needs a real 128-byte struct type
struct slu_nccl_id { char internal[128]; };

namespace {
struct NcclApi {
    void *so = nullptr;
    int (*GetUniqueId)(slu_nccl_id *) = nullptr;
    int (*CommInitRank)(void **, int, slu_nccl_id, int) = nullptr;
    int (*CommDestroy)(void *) = nullptr;
    int (*Send)(const void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*Recv)(void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*AllReduce)(const void *, void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*CommSplit)(void *, int, int, void **, void *) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, void *, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    bool load()
    {
        if (so) return true;
        const char *names[] = {getenv("SLU_B200_NCCL"), "libnccl.so.2", "libnccl.so"};
        for (const char *n : names) {
            if (!n) continue;
            so = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (so) break;
        }
        if (!so) return false;
        GetUniqueId = (decltype(GetUniqueId))dlsym(so, "ncclGetUniqueId");
        CommInitRank = (decltype(CommInitRank))dlsym(so, "ncclCommInitRank");
        CommDestroy = (decltype(CommDestroy))dlsym(so, "ncclCommDestroy");
        Send = (decltype(Send))dlsym(so, "ncclSend");
        Recv = (decltype(Recv))dlsym(so, "ncclRecv");
        AllReduce = (decltype(AllReduce))dlsym(so, "ncclAllReduce");
        CommSplit = (decltype(CommSplit))dlsym(so, "ncclCommSplit");
        AllGather = (decltype(AllGather))dlsym(so, "ncclAllGather");
        GetErrorString = (decltype(GetErrorString))dlsym(so, "ncclGetErrorString");
        return GetUniqueId && CommInitRank && CommDestroy && Send && Recv && AllReduce;
    }
} g_nccl;
constexpr int NCCL_INT32 = 2, NCCL_FLOAT64 = 8, NCCL_SUM = 0, NCCL_MIN = 3;
#define NC(call)                                                                                   \
    do {                                                                                           \
        int r_ = (call);                                                                           \
        if (r_ != 0) return fail("%s:%d %s: NCCL error %d %s", __FILE__, __LINE__, #call, r_,      \
                                 g_nccl.GetErrorString ? g_nccl.GetErrorString(r_) : "");          \
    } while (0)

// NCCL communicators outlive a factorization, as the reference's MPI communicators do (superlu_gridinit3d creates
// them once, pdgstrf3d only uses them): the 128-byte NCCL id names the clique, and the world communicator plus the
// per-Z-level group communicators built from it are cached per process under (id, grid shape, my coordinates).
// Repeated pdgstrf3d_b200 calls with the same id reuse them; slu_b200_comm_cache_clear() destroys them.
struct CommSet {
    void *comm = nullptr;
    std::vector<void *> gcomm;
};
std::mutex g_comm_mu;
std::map<std::string, CommSet> g_comm_cache;

// slu_b200_plan: run the analysis without touching a device -- buffers record their sizes only
thread_local bool g_plan_only = false;

template <class T>
struct DevBuf {
    T *p = nullptr;
    size_t n = 0;
    int alloc(size_t count)
    {
        release();
        n = count;
        if (g_plan_only) return 0;
        if (count == 0) count = 1;
        cudaError_t e = cudaMalloc((void **)&p, count * sizeof(T));
        if (e != cudaSuccess) return fail("cudaMalloc(%zu bytes): %s", count * sizeof(T), cudaGetErrorString(e));
        return 0;
    }
    int upload(const std::vector<T> &h)
    {
        if (alloc(h.size())) return -1;
        if (g_plan_only) return 0;
        if (!h.empty()) CU(cudaMemcpy(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
        return 0;
    }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
    size_t bytes() const { return n * sizeof(T); }
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }   // the CU()/NC() early returns must not leak HBM
};

struct EventSet {            // timing events with the same guarantee
    cudaEvent_t e[6] = {};
    int create() { for (auto &x : e) if (cudaEventCreate(&x) != cudaSuccess) return -1; return 0; }
    ~EventSet() { for (auto x : e) if (x) cudaEventDestroy(x); }
    cudaEvent_t &operator[](int i) { return e[i]; }
};

struct LevelPlan {
    int zlvl = 0, count = 0, max_ns = 0;
    int64_t nodes_off = 0;
    int64_t trsml_prefix = 0, trsml_ctas = 0, trsmu_prefix = 0, trsmu_ctas = 0, setup_prefix = 0, setup_ctas = 0;
    int64_t inv_prefix = 0, inv_ctas = 0;
    int64_t urg_prefix = 0, urg_ctas = 0, bulk_prefix = 0, bulk_ctas = 0;  // look-ahead split of the big batch
    int64_t slab_begin = 0, slab_end = 0;  // val range of this level's panels (contiguous in cooperative forests)
    int big_count = 0, small_count = 0;
    int64_t big_nodes = 0, big_prefix = 0, big_ctas = 0, small_nodes = 0, small_prefix = 0, small_ctas = 0;
    // int8 tensor-core path: the wide supernodes of the level (slu_ozaki.cu)
    int tc_count = 0;
    int64_t tc_nodes = 0, tc_prefix = 0, tc_ctas = 0, tc_urg_prefix = 0, tc_urg_ctas = 0, tc_bulk_prefix = 0, tc_bulk_ctas = 0;
    int64_t tc_p_rt = 0, tc_n_rt = 0, tc_p_ak = 0, tc_n_ak = 0, tc_p_b = 0, tc_n_b = 0;
    int64_t sl_prefix = 0, sl_ctas = 0, su_prefix = 0, su_ctas = 0;   // triangular solve: 256-row / 256-column tiles
};

// selected inversion (slu_b200_selinv): per level, offsets into d_si_pool of the CTA prefixes of the three products
// (gemm[0..2], slu_selinv.cu modes) and the two triangular solves (trsm[0]: rows, [1]: columns), and their CTA counts
struct SelinvLevel {
    int64_t gemm_prefix[3] = {0, 0, 0}, gemm_ctas[3] = {0, 0, 0};
    int64_t trsm_prefix[2] = {0, 0}, trsm_ctas[2] = {0, 0};
};

}  // namespace

struct slu_b200_handle_s {
    slu_b200_lu_view_t view;
    slu_b200_options_t opt;
    int nsupers = 0, n = 0, max_lvl = 1;
    std::vector<int32_t> xsup, my_tree, my_zero;
    std::vector<NodeDesc> nodes;          // host copy
    std::vector<std::vector<int32_t>> znodes;  // held nodes per Z level, arena order
    std::vector<int64_t> chunk_start;     // val offsets per Z level (L part, U part interleaved): [maxLvl+1]
    std::vector<int64_t> sky_len;         // skyline nnz of each held U panel (host side)
    std::vector<char> u_full;             // 1 if the skyline of U panel k equals its dense-packed form
    std::vector<LevelPlan> levels;
    // device
    DevBuf<val_t> val, stage, d_inv;
    DevBuf<NodeDesc> d_nodes;
    DevBuf<int32_t> d_xsup, d_supno, d_lrows, d_lsrow, d_lspos, d_ucols, d_ufst, d_useg, d_pool_i32, d_lrel, d_urel;
    DevBuf<int64_t> d_pool_i64;
    DevBuf<KSeg> d_kseg;                  // K segments of deferred child updates (NodeDesc.kseg_off)
    double merge[3] = {0, 0, 0};          // deferred children, destination REDs at depth 1 and at the planned depth
    DevBuf<LBlk> d_lblk;
    DevBuf<UBlk> d_ublk;
    DevBuf<RowInfo> d_rowinfo;
    DevBuf<ColInfo> d_colinfo;
    DevBuf<int8_t> d_oz_i8;               // int8 tensor-core path: int8 slice workspace (two level parities)
    DevBuf<double> d_oz_scale;
    DevBuf<int> d_oz_rexp;
    int tc_slices = 0, tc_min_ns = 0;     // 0 slices: int8 tensor-core path off
    int tc_max_m = 0;                     // > 0: only updates of fewer rows take the int8 path (SLU_B200_TC_MAX_M); 0: no limit
    bool tc_force_off = false, tc_alloc_failed = false;   // slice workspace did not fit: analysed again without the int8 tensor-core path
    DevBuf<val_t> d_x, d_x2;              // triangular solve: right-hand sides / solution
    std::vector<int64_t> z_nodes_off;     // [zl] offset into d_pool_i32 of the forest's node list (solve masks)
    DevBuf<int> d_flags;                  // [0]=info [1]=err
    DevBuf<unsigned long long> d_tiny;
    DeviceLU dev{};
    cudaStream_t stream = nullptr, stream2 = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::vector<cudaEvent_t> ev_panel, ev_bulk;
    cudaStream_t s_down = nullptr;                       // overlapped D2H (slu_b200_factor_host)
    cudaStream_t s_up = nullptr;                         // overlapped H2D (options.reserved[3])
    std::vector<cudaEvent_t> ev_up;                      // [li] level li's panels have arrived in the arena
    std::vector<int32_t> h_pool_i32;                     // host copy of the level node lists
    bool grouped = false;                                // every forest laid out level by level
    std::vector<UpSeg> h_segs;                           // download chunks (arena offset, -, length), by release level
    std::vector<val_t *> h_seg_host;                     // host address of each chunk
    std::vector<std::array<int64_t, 2>> lvl_segs;         // [li] -> [first, last) chunk released after level li
    bool pipe_ready = false;
    int64_t ws_max[4] = {0, 0, 0, 0};
    void *comm = nullptr;
    bool coop = false;                    // cooperative ancestors: all ranks of a Z group factor the shared forest
    int P2 = 1;                           // nprow * npcol: ranks of one layer (2D input: panels replicated per layer)
    void *lcomm = nullptr;                // communicator of my layer (structure exchange)
    std::vector<const slu_int *> Lidx, Uidx;        // [nsupers] index arrays of the FULL panels
    std::vector<std::vector<slu_int>> fullL, fullU; // their storage when merged from the 2D pieces
    struct Piece { int64_t dev; val_t *host; int64_t width, height, spitch, dpitch; };
    std::vector<Piece> pieces;            // my local blocks <-> their place in the replicated panels
    std::vector<LBlk> h_lblk;
    std::vector<UBlk> h_ublk;
    std::vector<void *> gcomm;            // [zl] communicator of my Z group at level zl (2^zl ranks)
    slu_b200_stats_t st{};
    bool uploaded = false;
    // batched handle (slu_b200_batch_create): `batch` members of one pattern share everything above except the value
    // arena, d_inv and the info flags, which hold `batch` consecutive copies
    int batch = 0;                        // 0: an ordinary handle
    int64_t member_len = 0, inv_len = 0;  // elements of one member's arena / diag-inverse workspace
    BatchedLU bdev{};
    // info of every member (one on an unbatched handle): -1 no factors since the last fill or upload, 0 factored, > 0 the
    // first zero pivot (1-based column)
    std::vector<int> member_info;
    // condition estimation (slu_b200_gscon): per member the pending vector (batched handles only), the last real sign
    // vector, the state; the reduction partials and the two kase counters
    DevBuf<val_t> d_cv, d_csgn;
    DevBuf<CondState> d_cstate;
    DevBuf<CondPart> d_cpart;
    DevBuf<int> d_ccount;
    // selected inversion (slu_b200_selinv / slu_b200_z_selinv): H = F^-T in a second arena of the factors' layout, its level plan,
    // and whether it describes the current factors (a later upload, fill_csr or factor clears it)
    DevBuf<val_t> d_hinv;
    DevBuf<int64_t> d_si_pool;
    std::vector<SelinvLevel> si_levels;
    bool si_ready = false;
    // partial factorization (slu_b200_schur_create): the supernodes from column schur_first = n - nschur on are in no level
    // of the plan, so factor, condense and expand stop at them; d_sunits lists the gather's (supernode, column) units and
    // d_S is the s x s buffer of slu_b200_schur_get, batch x s x s on a batched Schur handle (slu_b200_batch_schur_get;
    // allocated on first use, freed by destroy).  nschur = 0: not a Schur handle.
    int nschur = 0, schur_first = INT_MAX;
    DevBuf<int2> d_sunits;
    DevBuf<val_t> d_S;
    // static pivoting (slu_b200_fill_csr_scaled): the last scaled fill's perm_r, its composed row map perm[perm_r[i]], perm,
    // and the final R and C (batch x n on a batched handle).  `scaled`: they describe the values in the arena (a later
    // upload, fill_csr, batch_fill_csr or batch_fill_affine clears it).
    DevBuf<int32_t> d_perm_r, d_rmap, d_cperm;
    DevBuf<double> d_R, d_C;
    bool scaled = false;
    // iterative refinement (slu_b200_gsrfs): A as the last scaled fill received it (rowptr, colind, batch x nnz values; kept
    // and dropped with the scaling), the right-hand sides and the solution being refined, dgerfs's W and the per-column state
    DevBuf<int32_t> d_arp, d_aci;
    DevBuf<val_t> d_aval;
    DevBuf<val_t> d_rb, d_rx;
    DevBuf<double> d_rw;
    DevBuf<RefineState> d_rst;
    DevBuf<int> d_ract;
    // refill (slu_b200_refill): the arena offset and the row of every entry of the kept A, built by the first refill after a
    // scaled fill (amap_ready) and shared by the members; dropped with the scaling
    DevBuf<int64_t> d_amap;
    DevBuf<int32_t> d_arow;
    bool amap_ready = false;
    // the calls on the caller's stream: the handle's device, and the events that order the handle's stream after the caller's
    // work (ev_in) and the caller's stream after the handle's (ev_out)
    int device = 0;
    cudaEvent_t ev_in = nullptr, ev_out = nullptr;
    // factor_device: every member's info on the device, as member_info holds it (written by every factorization), and
    // whether member_info waits for it (status_on_device; settle)
    DevBuf<int32_t> d_info;
    bool status_on_device = false;
    // the device factorizations so far, counted by factor_info_kernel (a replay counts too): epoch is the count the last
    // settle read, si_epoch the count selinv inverted
    DevBuf<unsigned long long> d_epoch;
    unsigned long long epoch = 0, si_epoch = 0;
    // a call on the caller's stream has been captured into a CUDA graph: the buffers those calls use are pinned (grow)
    bool captured = false;
    bool loop_captured = false;           // one of them was gsrfs_device or gscon_device: their buffers are pinned too (grow_loop)
    // gsrfs_device / gscon_device: their outputs before the copies to the caller (berr then ferr, steps; rcond) and anorm,
    // max_i |x_i| per column as bits, the estimator loop's {kase, rounds}; the side streams the bodies of the conditional
    // nodes are captured on (one per nesting depth); the executable graphs of the eager calls, each with the key it was
    // captured for and the buffer addresses it holds (captured again when one of them moved)
    DevBuf<double> d_rout, d_canorm, d_crcond;
    DevBuf<int32_t> d_rsteps;
    DevBuf<unsigned long long> d_rxmax;
    DevBuf<int> d_cloop;
    cudaStream_t s_body[2] = {nullptr, nullptr};
    struct LoopGraph {
        std::array<int, 4> key;
        std::vector<uintptr_t> bufs;
        cudaGraph_t graph;
        cudaGraphExec_t exec;
        int launches;
    };
    std::vector<LoopGraph> loop_graphs;
    // the gradient calls (selinv_device, logdet_device, logdet_grad_device, solve_grad_device): the status of the last device
    // selected inversion per member and its record {factorization count inverted, missed destinations} (si_dev: the inverse
    // came from selinv_device, settle reads the record); logdet_device's partials and result; solve_grad_device's row-major
    // copies of lambda and x
    DevBuf<int32_t> d_si_status;
    DevBuf<unsigned long long> d_si_rec;
    bool si_dev = false;
    DevBuf<double> d_lpart, d_lres;
    DevBuf<phase_t> d_lph;
    DevBuf<val_t> d_gstage;
};

namespace {

// The handle's state in one place.  Every call that writes the arena first says so here, after its argument checks and
// before its first write, and sets the state it establishes only once it has succeeded: a call that fails on the way
// leaves a handle whose factors (and values, for a fill) the calls that read them refuse.

// member_info after a device factorization (factor_device) until settle reads the status it left on the device
constexpr int INFO_PENDING = INT_MIN;

// a factorization is about to overwrite the arena: no member has factors, and the inverse no longer describes them.  d_info
// says the same in the handle's stream order (a captured refill carries it into every replay).
int factors_replaced(slu_b200_handle_s *H)
{
    std::fill(H->member_info.begin(), H->member_info.end(), -1);
    H->status_on_device = false;
    H->si_ready = false;
    CU(cudaMemsetAsync(H->d_info.p, 0xff, H->d_info.bytes(), H->stream));
    return 0;
}

// an upload or a fill is about to overwrite the arena: no values to factor either, and the scaling no longer describes
// them.  The A kept for refinement and the refill's slot map go with the scaling, except on a scaled fill (keep_a), which
// reuses their buffers (the map is rebuilt by the next refill).
int values_replaced(slu_b200_handle_s *H, bool keep_a = false)
{
    const int rc = factors_replaced(H);
    H->uploaded = false;
    H->scaled = false;
    H->amap_ready = false;
    if (keep_a || H->captured) return rc;    // a captured refill reads them (grow)
    H->d_arp.release();
    H->d_aci.release();
    H->d_aval.release();
    H->d_amap.release();
    H->d_arow.release();
    return rc;
}

// What a call needs of the handle (check): one bit per condition
enum Need : unsigned {
    UNBATCHED = 1u << 0,      // kind: slu_b200_create / schur_create
    BATCHED = 1u << 1,        //       slu_b200_batch_create / batch_schur_create
    NOT_SCHUR = 1u << 2,      // complete factors: not a Schur handle
    SCHUR = 1u << 3,          // a Schur handle
    GRID_Z = 1u << 4,         // 1 x 1 x Pz
    GRID_SOLVE = 1u << 5,     // 1 x 1 x Pz, cooperative along Z
    GRID_1 = 1u << 6,         // 1 x 1 x 1, world_size 1
    UPLOADED = 1u << 7,       // values from a successful upload or fill
    SCALED = 1u << 8,         // the scaling of a successful scaled fill
    FACTORED = 1u << 9,       // every member factored with info 0
    SI_READY = 1u << 10,      // the inverse of selinv on the current factors
    DEVICE_ORDERED = 1u << 11, // with FACTORED: a call on the caller's stream, which takes a pending status as it is (and
                               // on a captured handle any status: a replay may have changed it, and the guard covers it)
};

// The status a device factorization left in d_info and d_tiny, read into member_info and stats.tiny_pivots once the handle's
// stream has drained: what a host-synchronous call sees, exactly as after slu_b200_factor.  On a captured handle it is read
// every time, since a replay of the graph may have rewritten it (every fill, refill and factorization writes d_info), and
// the inverse of selinv goes when a factorization has run since it (the epoch moved).  While the handle's stream is being
// captured nothing is read: a wait would end the capture.
int settle(slu_b200_handle_s *H)
{
    if (!H->status_on_device && !H->captured) return 0;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    CU(cudaStreamIsCapturing(H->stream, &cs));
    if (cs != cudaStreamCaptureStatusNone) return 0;
    std::vector<int32_t> info(H->member_info.size());
    unsigned long long tiny = 0;
    CU(cudaStreamSynchronize(H->stream));
    CU(cudaMemcpy(info.data(), H->d_info.p, info.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&tiny, H->d_tiny.p, sizeof tiny, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&H->epoch, H->d_epoch.p, sizeof H->epoch, cudaMemcpyDeviceToHost));
    std::copy(info.begin(), info.end(), H->member_info.begin());
    H->st.tiny_pivots = (int64_t)tiny;
    H->status_on_device = false;
    if (H->si_dev) {                       // the inverse of selinv_device: the count it inverted, and whether it missed destinations
        unsigned long long rec[2] = {0, 0};
        CU(cudaMemcpy(rec, H->d_si_rec.p, sizeof rec, cudaMemcpyDeviceToHost));
        H->si_epoch = rec[0];
        if (rec[1]) H->si_ready = false;
    }
    if (H->captured && H->epoch != H->si_epoch) H->si_ready = false;
    return 0;
}

// Refuses a call on a handle that does not give it what it needs, with a message that starts with fn, the call's exported
// name.  Kind, then Schur, then grid, then state; except that an unbatched schur_* call names a missing Schur handle first.
int check(slu_b200_handle_s *H, const char *fn, unsigned need)
{
    if ((need & SCHUR) && (need & UNBATCHED) && !H->nschur) return fail("%s needs a Schur handle (" SLU_API "schur_create)", fn);
    if ((need & UNBATCHED) && H->batch)
        return fail("%s on a batched handle (%d members): use the " SLU_API "batch_* calls", fn, H->batch);
    if ((need & BATCHED) && !H->batch) return fail("%s on an unbatched handle: use the " SLU_API "* calls without _batch", fn);
    if ((need & NOT_SCHUR) && H->nschur)
        return fail("%s on a Schur handle (partial factorization, nschur = %d): its factors are incomplete; use the %s calls", fn,
                    H->nschur, H->batch ? SLU_API "batch_schur_*" : SLU_API "schur_*");
    if ((need & SCHUR) && !H->nschur) return fail("%s needs a batched Schur handle (" SLU_API "batch_schur_create)", fn);
    if ((need & (GRID_Z | GRID_SOLVE)) && H->P2 > 1) return fail("%s handles 1 x 1 x Pz grids (Pr x Pc = %d)", fn, H->P2);
    if ((need & GRID_SOLVE) && H->comm && !H->coop)
        return fail("%s: the Z-distributed solve needs the cooperative schedule (options.reserved[1] = 0)", fn);
    if ((need & GRID_1) && (H->view.nprow * H->view.npcol * H->view.npdep != 1 || H->opt.world_size > 1))
        return fail("%s needs a 1 x 1 x 1 grid with world_size 1 (got %d x %d x %d, world_size %d)", fn, H->view.nprow, H->view.npcol,
                    H->view.npdep, H->opt.world_size);
    if ((need & UPLOADED) && !H->uploaded)
        return fail("%s before a successful %s", fn, H->batch ? SLU_API "batch_fill_csr" : SLU_API "upload or " SLU_API "fill_csr");
    if ((need & SCALED) && !H->scaled)
        return fail("%s needs a scaled fill on this handle first (a later upload or plain fill drops the scaling and the kept A)", fn);
    if ((need & FACTORED) && !(need & DEVICE_ORDERED) && settle(H)) return -1;
    if (need & FACTORED)
        for (size_t j = 0; j < H->member_info.size(); ++j) {
            const int info = H->member_info[j];
            if (info == 0 || ((need & DEVICE_ORDERED) && (info == INFO_PENDING || H->captured))) continue;
            if (!H->batch)
                return fail("%s needs a successful " SLU_API "factor %s", fn, (need & SCALED) ? "after the scaled fill" : "(info = 0) on this handle first");
            if (info < 0) return fail("%s needs a " SLU_API "batch_factor of the filled members first", fn);
            return fail("%s: member %zu has an exact zero pivot in column %d", fn, j, info);
        }
    if ((need & SI_READY) && !H->si_ready)
        return fail("%s needs %s on the current factors first (a later fill, upload or factorization invalidates it)", fn,
                    H->batch ? SLU_API "batch_selinv" : SLU_API "selinv");
    return 0;
}

// A CUDA graph captured from the calls on the caller's stream holds raw pointers to the buffers they use: d_x, d_x2, and the
// kept A and the slot map of the refill.  Once one of those calls has been captured (H->captured), none of them is freed
// or moved again until slu_b200_destroy; moves: the call would do so.
int pin_check(const slu_b200_handle_s *H, bool moves, const char *fn)
{
    if (moves && H->captured)
        return fail("%s would reallocate a buffer that a captured CUDA graph uses: after a capture the handle's buffers keep "
                    "their sizes until " SLU_API "destroy", fn);
    return 0;
}

// Every growth of those buffers (exact: resized to len, else grown to at least len).  capturing: the call is being captured,
// where an allocation is not allowed: it is refused before anything is enqueued.  A buffer never allocated is held by no
// graph: its first allocation is refused only under capture.
template <class T>
int grow(const slu_b200_handle_s *H, DevBuf<T> &b, size_t len, bool exact, bool capturing, const char *fn)
{
    if (exact ? b.n == len : b.n >= len) return 0;
    if (capturing)
        return fail("%s would allocate device buffers while the stream is capturing a CUDA graph: make this call once outside "
                    "capture first", fn);
    if (b.p && pin_check(H, true, fn)) return -1;
    return b.alloc(len);
}

// The growth of the buffers that only the graphs of gsrfs_device and gscon_device hold besides the host calls gsrfs and gscon
// (the refinement's and the estimator's): pinned once one of those calls was captured (loop_captured).
template <class T>
int grow_loop(const slu_b200_handle_s *H, DevBuf<T> &b, size_t len, bool capturing, const char *fn)
{
    if (b.n >= len) return 0;
    if (capturing || H->loop_captured) return grow(H, b, len, false, capturing, fn);
    return b.alloc(len);
}

int device_setup(const slu_b200_options_t *opt)
{
    if (opt->device >= 0) CU(cudaSetDevice(opt->device));
    CU(cudaFree(0));
    return 0;
}

// ------------------------------------------------------------------------------------------------
// analysis: parse the reference index arrays, lay out HBM, plan the level batches
// ------------------------------------------------------------------------------------------------
int analyze(slu_b200_handle_s *H)
{
    const slu_b200_lu_view_t &v = H->view;
    const int nsupers = v.nsupers, n = v.n;
    if (H->P2 > 1 && !H->coop)
        return fail("Pr x Pc > 1 needs the cooperative schedule (options.reserved[1] must be 0)");
    if (v.npdep < 1 || (v.npdep & (v.npdep - 1))) return fail("npdep must be a power of two");
    int max_lvl = 1;
    while ((1 << (max_lvl - 1)) < v.npdep) ++max_lvl;
    if (v.maxLvl != max_lvl) return fail("maxLvl %d does not match npdep %d", v.maxLvl, v.npdep);
    if (v.nforests != (1 << max_lvl) - 1) return fail("nforests must be 2^maxLvl - 1");
    H->nsupers = nsupers; H->n = n; H->max_lvl = max_lvl;
    H->xsup.assign(v.xsup, v.xsup + nsupers + 1);
    H->my_tree.assign(v.myTreeIdxs, v.myTreeIdxs + max_lvl);
    H->my_zero.assign(v.myZeroTrIdxs, v.myZeroTrIdxs + max_lvl);
    const std::vector<int32_t> &xsup = H->xsup;
    std::vector<int32_t> supno((size_t)n);
    for (int k = 0; k < nsupers; ++k) {
        if (xsup[k + 1] - xsup[k] > MAX_NS_HELD) return fail("supernode %d wider than %d columns is not supported", k, MAX_NS_HELD);
        for (int c = xsup[k]; c < xsup[k + 1]; ++c) supno[c] = k;
    }

    const bool timing = getenv("SLU_B200_TIMING") != nullptr;
    double tmark = now_s();
    auto lap = [&](const char *what) { if (timing) { double t = now_s(); fprintf(stderr, "analyze: %-28s %.3f s\n", what, t - tmark); tmark = t; } };
    H->nodes.assign(nsupers, NodeDesc{});
    H->znodes.assign(max_lvl, {});
    std::vector<int> forest_of(nsupers, -1), zl_of(nsupers, -1);
    for (int zl = 0; zl < max_lvl; ++zl) {
        const slu_b200_forest_t &f = v.forests[H->my_tree[zl]];
        for (int t = 0; t < f.nNodes; ++t) {
            int k = f.nodeList[t];
            if (k < 0 || k >= nsupers || zl_of[k] != -1) return fail("bad forest node list");
            zl_of[k] = zl;
            H->znodes[zl].push_back(k);
        }
    }

    // topological levels inside each forest (a supernode precedes every block it updates); the node lists are
    // valid elimination orders, so one sweep suffices
    std::vector<int> lev(nsupers, 0);
    for (int zl = 0; zl < max_lvl; ++zl)
        for (int k : H->znodes[zl]) {
            const slu_int *li = H->Lidx[k], *ui = H->Uidx[k];
            if (!li) return fail("supernode %d of my forest has no L panel", k);
            int w = BC_HEADER;
            for (int b = 0; b < li[0]; ++b) {
                int t = li[w];
                if (b > 0 && t >= 0 && t < nsupers && zl_of[t] == zl) lev[t] = std::max(lev[t], lev[k] + 1);
                w += LB_DESCRIPTOR + li[w + 1];
            }
            if (!ui) continue;
            int u = BR_HEADER;
            for (int b = 0; b < ui[0]; ++b) {
                int t = ui[u];
                if (t < 0 || t >= nsupers) return fail("U panel %d: bad block id", k);
                int jns = xsup[t + 1] - xsup[t];
                bool nonempty = false;
                for (int c = 0; c < jns && !nonempty; ++c) nonempty = ui[u + UB_DESCRIPTOR + c] < xsup[k + 1];
                if (nonempty && zl_of[t] == zl) lev[t] = std::max(lev[t], lev[k] + 1);
                u += UB_DESCRIPTOR + jns;
            }
        }
    lap("forests + topological levels");
    // cooperative ancestors (world_size > 1): every rank of a Z group factors the shared forest; its panels are
    // laid out level by level so that the panels due at one topological level are one contiguous slab
    const bool coop = H->coop;
    // options.reserved[3] (overlapped upload): the same level-by-level layout for every forest, so that the panels
    // are needed in arena order
    H->grouped = H->opt.reserved[3] && H->P2 == 1;
    if (coop || H->grouped)
        for (int zl = ((H->P2 > 1 || H->grouped) ? 0 : 1); zl < max_lvl; ++zl)
            std::stable_sort(H->znodes[zl].begin(), H->znodes[zl].end(), [&](int a, int b) { return lev[a] < lev[b]; });

    // pass 1: sizes and offsets.  Three sweeps over the held supernodes in arena order: (a) parallel -- count rows,
    // blocks and non-empty U columns of each panel; (b) serial -- prefix sums give every panel its place in the value
    // arena and in the index arenas; (c) parallel -- fill the index arenas, cross maps and flop counts.
    std::vector<int32_t> lrows, lsrow, lspos, ucols, ufst, useg;
    std::vector<LBlk> lblk;
    std::vector<UBlk> ublk;
    H->sky_len.assign(nsupers, 0);
    H->u_full.assign(nsupers, 1);
    H->chunk_start.assign(max_lvl + 1, 0);
    int64_t voff = 0;
    double ops = 0, ops_schur = 0, bytes_schur = 0;
    int64_t nnz_l = 0, nnz_u = 0;
    // arena order: per Z level, per group (the whole forest, or one topological level of a cooperatively factored /
    // grouped forest), first the L panels of the group, then its U panels
    std::vector<int32_t> order;                       // held supernodes in the order their L panels are laid out
    std::vector<std::pair<int64_t, int64_t>> groups;  // [begin, end) into order
    std::vector<int> group_zl;
    order.reserve(nsupers);
    for (int zl = 0; zl < max_lvl; ++zl) {
        const bool split = (coop && (zl >= 1 || H->P2 > 1)) || H->grouped;
        int64_t g0 = (int64_t)order.size();
        for (size_t t = 0; t < H->znodes[zl].size(); ++t) {
            const int k = H->znodes[zl][t];
            if (split && t > 0 && lev[H->znodes[zl][t - 1]] != lev[k]) {
                groups.emplace_back(g0, (int64_t)order.size()); group_zl.push_back(zl);
                g0 = (int64_t)order.size();
            }
            order.push_back(k);
        }
        if ((int64_t)order.size() > g0) { groups.emplace_back(g0, (int64_t)order.size()); group_zl.push_back(zl); }
    }
    const int64_t nheld = (int64_t)order.size();
    std::vector<int32_t> cnt_ucols(nheld, 0), cnt_ublk(nheld, 0);
    std::vector<char> bad(1, 0);
    std::string badmsg;
    auto flag = [&](const char *fmt, int a1, int a2 = 0, int a3 = 0) {
#pragma omp critical(slu_analyze_err)
        if (!bad[0]) { char buf[256]; snprintf(buf, sizeof buf, fmt, a1, a2, a3); badmsg = buf; bad[0] = 1; }
    };
    // a handful of threads is enough (and 8 ranks of one box share the cores)
    const int nth = std::max(1, std::min(omp_get_max_threads(), 16));
    // (a) counts
#pragma omp parallel for schedule(dynamic, 64) num_threads(nth)
    for (int64_t t = 0; t < nheld; ++t) {
        const int k = order[t];
        const slu_int *li = H->Lidx[k], *ui = H->Uidx[k];
        NodeDesc &nd = H->nodes[k];
        nd.held = 1; nd.fsupc = xsup[k]; nd.ns = xsup[k + 1] - xsup[k];
        nd.nsupr = li[1]; nd.m = nd.nsupr - nd.ns;
        const int nblk = li[0];
        if (nblk < 1 || li[BC_HEADER] != k || li[BC_HEADER + 1] != nd.ns) { flag("L panel %d: the diagonal block must come first and be full", k); continue; }
        nd.nlb = nblk - 1;
        if (!ui) continue;
        const int nb = ui[0], klst = xsup[k + 1];
        int u = BR_HEADER, ncols = 0, nub = 0;
        for (int bq = 0; bq < nb; ++bq) {
            const int jb = ui[u];
            if (jb < 0 || jb >= nsupers) { flag("U panel %d: bad block id", k); break; }
            const int jns = xsup[jb + 1] - xsup[jb];
            int c2 = 0;
            for (int c = 0; c < jns; ++c) c2 += ui[u + UB_DESCRIPTOR + c] < klst;
            ncols += c2; nub += c2 > 0;
            u += UB_DESCRIPTOR + jns;
        }
        cnt_ucols[t] = ncols; cnt_ublk[t] = nub;
    }
    if (bad[0]) return fail("%s", badmsg.c_str());
    // (b) offsets
    std::vector<int64_t> off_lrow(nheld + 1, 0), off_lblk(nheld + 1, 0), off_ucol(nheld + 1, 0), off_ublk(nheld + 1, 0);
    for (int64_t t = 0; t < nheld; ++t) {
        const NodeDesc &nd = H->nodes[order[t]];
        off_lrow[t + 1] = off_lrow[t] + nd.nsupr;
        off_lblk[t + 1] = off_lblk[t] + nd.nlb;
        off_ucol[t + 1] = off_ucol[t] + cnt_ucols[t];
        off_ublk[t + 1] = off_ublk[t] + cnt_ublk[t];
    }
    {
        int last_zl = -1;
        for (size_t g = 0; g < groups.size(); ++g) {
            if (group_zl[g] != last_zl) { for (int z = last_zl + 1; z <= group_zl[g]; ++z) H->chunk_start[z] = voff; last_zl = group_zl[g]; }
            for (int64_t t = groups[g].first; t < groups[g].second; ++t) {
                NodeDesc &nd = H->nodes[order[t]];
                nd.lval = voff; voff += (int64_t)nd.nsupr * nd.ns;
                nnz_l += (int64_t)nd.nsupr * nd.ns;
            }
            for (int64_t t = groups[g].first; t < groups[g].second; ++t) {
                NodeDesc &nd = H->nodes[order[t]];
                nd.ncols = cnt_ucols[t];
                nd.uval = voff; voff += (int64_t)nd.ns * nd.ncols;
                nnz_u += (int64_t)nd.ns * nd.ncols;
            }
        }
        for (int z = last_zl + 1; z < max_lvl; ++z) H->chunk_start[z] = voff;
    }
    lrows.resize((size_t)off_lrow[nheld]); lsrow.resize(lrows.size()); lspos.resize(lrows.size());
    ucols.resize((size_t)off_ucol[nheld]); ufst.resize(ucols.size()); useg.resize(ucols.size());
    lblk.resize((size_t)off_lblk[nheld]); ublk.resize((size_t)off_ublk[nheld]);
    // (c) fill
#pragma omp parallel reduction(+ : ops, ops_schur, bytes_schur) num_threads(nth)
    {
        std::vector<std::pair<int32_t, int32_t>> tmp;
#pragma omp for schedule(dynamic, 32)
        for (int64_t t = 0; t < nheld; ++t) {
            const int k = order[t];
            const int zl = zl_of[k];
            const slu_int *li = H->Lidx[k];
            NodeDesc &nd = H->nodes[k];
            nd.lrow = off_lrow[t]; nd.lblk = off_lblk[t]; nd.ucol = off_ucol[t]; nd.ublk = off_ublk[t];
            const int nblk = li[0];
            {
                int w = BC_HEADER, row0 = 0, last_ib = -1;
                int64_t lr = nd.lrow, lbq = nd.lblk;
                bool okp = true;
                tmp.clear();
                for (int bq = 0; bq < nblk && okp; ++bq) {
                    int ib = li[w], nb = li[w + 1];
                    if (ib <= last_ib) { flag("L panel %d: row blocks are not in ascending order", k); okp = false; break; }
                    last_ib = ib;
                    if (row0 + nb > nd.nsupr) { flag("L panel %d: row count mismatch", k); okp = false; break; }
                    for (int q = 0; q < nb; ++q) {
                        int r = li[w + 2 + q];
                        if (r < xsup[ib] || r >= xsup[ib + 1]) { flag("L panel %d: row %d outside block %d", k, r, ib); okp = false; break; }
                        if (bq == 0 && r != xsup[k] + q) { flag("L panel %d: diagonal block rows must be sorted", k); okp = false; break; }
                        tmp.emplace_back(r, row0 + q);
                        lrows[lr++] = r;
                    }
                    if (bq > 0) lblk[lbq++] = LBlk{ib, row0 - nd.ns, nb, 0, 0};
                    row0 += nb;
                    w += LB_DESCRIPTOR + nb;
                }
                if (!okp) continue;
                if (row0 != nd.nsupr) { flag("L panel %d: row count mismatch", k); continue; }
                std::sort(tmp.begin(), tmp.end());
                for (size_t q = 0; q < tmp.size(); ++q) { lsrow[nd.lrow + q] = tmp[q].first; lspos[nd.lrow + q] = tmp[q].second; }
            }
            const slu_int *ui = H->Uidx[k];
            int ldu = 0;
            double utrsm = 0;
            if (ui) {
                const int nb = ui[0], klst = xsup[k + 1];
                int u = BR_HEADER, seg = 0, last_jb = k, col = 0;
                int64_t uc = nd.ucol, ubq = nd.ublk;
                bool oku = true, full = true;
                for (int bq = 0; bq < nb && oku; ++bq) {
                    int jb = ui[u];
                    if (jb <= last_jb || jb >= nsupers) { flag("U panel %d: column blocks are not ascending", k); oku = false; break; }
                    last_jb = jb;
                    int jns = xsup[jb + 1] - xsup[jb], col0 = col, cnt = 0;
                    for (int c = 0; c < jns; ++c) {
                        int fst = ui[u + UB_DESCRIPTOR + c];
                        if (fst >= klst) continue;
                        if (fst < xsup[k]) { flag("U panel %d: fstnz below the supernode", k); oku = false; break; }
                        ucols[uc] = xsup[jb] + c; ufst[uc] = fst; useg[uc] = seg; ++uc;
                        int len = klst - fst;
                        seg += len; ldu = std::max(ldu, len);
                        utrsm += (double)len * (len + 1);
                        if (len != nd.ns) full = false;
                        ++cnt;
                    }
                    if (cnt) ublk[ubq++] = UBlk{jb, col0, cnt, 0, 0};
                    col += cnt;
                    u += UB_DESCRIPTOR + jns;
                }
                if (!oku) continue;
                if (seg != ui[1]) { flag("U panel %d: nnz mismatch (%d vs %d)", k, seg, ui[1]); continue; }
                H->sky_len[k] = seg;
                H->u_full[k] = full ? 1 : 0;
            }
            nd.nub = cnt_ublk[t];
            // cross maps: colstart per L block, rowstart per U block
            const int32_t *ucp = ucols.data() + nd.ucol;
            int64_t uoff = 0;
            for (int bq = 0; bq < nd.nlb; ++bq) {
                LBlk &lb = lblk[nd.lblk + bq];
                lb.colstart = (int)(std::lower_bound(ucp, ucp + nd.ncols, xsup[lb.ib + 1]) - ucp);
                lb.urel_off = uoff;
                uoff += nd.ncols - lb.colstart;
            }
            nd.urel_total = uoff;
            int64_t loff = 0;
            int q0 = 0;                                   // both block lists ascend: one merge sweep
            for (int bq = 0; bq < nd.nub; ++bq) {
                UBlk &ub = ublk[nd.ublk + bq];
                while (q0 < nd.nlb && lblk[nd.lblk + q0].ib < ub.jb) ++q0;
                ub.rowstart = q0 < nd.nlb ? lblk[nd.lblk + q0].row0 : nd.m;
                ub.lrel_off = loff;
                loff += nd.m - ub.rowstart;
            }
            nd.lrel_total = loff;
            // flops in the reference's accounting
            double diag = 0;
#ifdef SLU_COMPLEX
            for (int j = 0; j < nd.ns; ++j) { double r = nd.ns - j - 1; diag += (6 * r + 10) + 8 * r * r; }  // pzgstrf2.c:578,590
#else
            for (int j = 0; j < nd.ns; ++j) { double r = nd.ns - j - 1; diag += r + 2 * r * r; }
#endif
            double sch = 2.0 * nd.m * (double)ldu * nd.ncols;
            if (H->my_zero[zl]) continue;  // replicated ancestor copy: counted by its owner layer only
            if (nd.fsupc >= H->schur_first) continue;  // a Schur supernode of a partial factorization: not eliminated
            if (H->P2 > 1 && (k % v.nprow != v.myrow || k % v.npcol != v.mycol)) continue;  // ... and by the diagonal owner
            ops += diag + utrsm + sch;
            ops_schur += sch;
            bytes_schur += VAL_DOUBLES * (8.0 * ((double)nd.m * nd.ns + (double)nd.ns * nd.ncols) + 16.0 * nd.m * (double)nd.ncols) +
                           4.0 * (nd.m + nd.ncols);
        }
    }
    if (bad[0]) return fail("%s", badmsg.c_str());
    H->chunk_start[max_lvl] = voff;
    lap("pass 1 (index arrays)");

    // every destination of a held supernode must be held too
    for (int zl = 0; zl < max_lvl; ++zl)
        for (int k : H->znodes[zl]) {
            const NodeDesc &nd = H->nodes[k];
            for (int b = 0; b < nd.nlb; ++b)
                if (!H->nodes[lblk[nd.lblk + b].ib].held) return fail("supernode %d updates block row %d which this rank does not hold", k, lblk[nd.lblk + b].ib);
            for (int b = 0; b < nd.nub; ++b)
                if (!H->nodes[ublk[nd.ublk + b].jb].held) return fail("supernode %d updates block column %d which this rank does not hold", k, ublk[nd.ublk + b].jb);
        }

    // level batches
    std::vector<int32_t> seen_by(nsupers, -1), stamp(nsupers, -1), ndest(nsupers, 0);
    std::vector<int32_t> pool_i32;
    std::vector<int64_t> pool_i64;
    int64_t ws_row_max = 0, ws_col_max = 0, ws_lrel_max = 0, ws_urel_max = 0, ws_inv_max = 0;
    int64_t ws_oz_i8_max = 0, ws_oz_s_max = 0;
    double ops_tc = 0;
#ifndef SLU_COMPLEX
    // int8 tensor-core path (slu_ozaki.cu): options.reserved[4] = int8 slices per operand (0: default = off, < 0: off),
    // options.reserved[5] = narrowest supernode that takes it (0: default)
    H->tc_slices = H->opt.reserved[4] < 0 ? 0 : (H->opt.reserved[4] == 0 ? (OZ_DEFAULT_ON ? OZ_DEFAULT_SLICES : 0) : std::min(8, std::max(5, (int)H->opt.reserved[4])));
    H->tc_min_ns = H->opt.reserved[5] > 0 ? H->opt.reserved[5] : OZ_DEFAULT_MIN_NS;
    if (getenv("SLU_B200_TC_MAX_M")) H->tc_max_m = std::max(0, atoi(getenv("SLU_B200_TC_MAX_M")));
    if (getenv("SLU_B200_TC_SLICES")) { int v = atoi(getenv("SLU_B200_TC_SLICES")); H->tc_slices = v <= 0 ? 0 : std::min(8, std::max(5, v)); }
    if (getenv("SLU_B200_TC_MIN_NS")) H->tc_min_ns = std::max(1, atoi(getenv("SLU_B200_TC_MIN_NS")));
    if (H->tc_force_off) H->tc_slices = 0;
#endif
    // Deferred Schur updates along supernode chains (DESIGN 4a).  When the structure of supernode k is exactly the columns
    // of its parent p followed by the structure of p (L rows and packed U columns, position by position), the part of k's
    // update below and right of p's columns has p's region and destination maps: it runs inside p's update as more K
    // segments of one GEMM, and k keeps only its panel tiles (those that write p).  options.reserved[6] or
    // SLU_B200_SCHUR_DEPTH = the most panels one GEMM takes (1: off).
    int depth = H->opt.reserved[6] > 0 ? H->opt.reserved[6] : SCHUR_DEPTH_DEFAULT;
    if (getenv("SLU_B200_SCHUR_DEPTH")) depth = atoi(getenv("SLU_B200_SCHUR_DEPTH"));
    depth = std::min(SCHUR_DEPTH_MAX, std::max(1, depth));
#ifdef SLU_COMPLEX
    depth = 1;   // slu_kernels_z.cu has no segmented K loop
#endif
    if (H->tc_slices > 0 || H->P2 > 1 || max_lvl > 1) depth = 1;   // int8 route, 2D layers, Z-split tile dealing: DESIGN 8
    std::vector<KSeg> kseg;
    {
        std::vector<std::vector<KSeg>> carried(nsupers);   // segments of nested children each supernode's update carries
        std::vector<int32_t> panels(nsupers, 1);
        int64_t deferred = 0;
        double reds = 0, saved = 0;
        for (int k = 0; k < nsupers; ++k) {   // children before parents: a parent's id is larger
            NodeDesc &nd = H->nodes[k];
            if (!nd.held || xsup[k] >= H->schur_first || H->my_zero[zl_of[k]] || nd.m <= 0 || nd.ncols <= 0) continue;
            reds += (double)nd.m * nd.ncols;
            if (depth < 2 || nd.m < 96 || nd.ncols < 96) continue;
            const int p = supno[lrows[nd.lrow + nd.ns]];
            const NodeDesc &pd = H->nodes[p];
            if (!pd.held || zl_of[p] != zl_of[k] || xsup[p] >= H->schur_first || pd.m < 96 || pd.ncols < 96) continue;
            if (nd.m != pd.ns + pd.m || nd.ncols != pd.ns + pd.ncols || panels[k] + panels[p] > depth) continue;
            bool nest = true;
            for (int i = 0; i < nd.m && nest; ++i)
                nest = lrows[nd.lrow + nd.ns + i] == (i < pd.ns ? xsup[p] + i : lrows[pd.lrow + i]);
            for (int j = 0; j < nd.ncols && nest; ++j)
                nest = ucols[nd.ucol + j] == (j < pd.ns ? xsup[p] + j : ucols[pd.ucol + j - pd.ns]);
            if (!nest) continue;
            nd.defer = 1;
            panels[p] += panels[k];
            // row ns_p of k's update is row 0 of p's: every carried segment starts ns_p rows / packed columns further on
            carried[p].push_back(KSeg{nd.lval + nd.ns + pd.ns, nd.uval + (int64_t)pd.ns * nd.ns, nd.nsupr, nd.ns, nd.ns, 0});
            for (const KSeg &q : carried[k]) carried[p].push_back(KSeg{q.a + pd.ns, q.b + (int64_t)pd.ns * q.ldb, q.lda, q.ldb, q.k, 0});
            ++deferred;
            saved += (double)pd.m * pd.ncols;
        }
        for (int k = 0; k < nsupers; ++k)
            if (!carried[k].empty()) {
                H->nodes[k].kseg_off = (int64_t)kseg.size();
                H->nodes[k].nkseg = (int)carried[k].size();
                kseg.insert(kseg.end(), carried[k].begin(), carried[k].end());
            }
        H->merge[0] = (double)deferred; H->merge[1] = reds; H->merge[2] = reds - saved;
    }
    H->levels.clear();
    for (int zl = 0; zl < max_lvl; ++zl) {
        int maxlev = -1;
        for (int k : H->znodes[zl]) maxlev = std::max(maxlev, lev[k]);
        std::vector<std::vector<int32_t>> by(maxlev + 1);
        for (int k : H->znodes[zl])
            if (xsup[k] < H->schur_first) by[lev[k]].push_back(k);   // a partial factorization leaves its Schur supernodes out
        for (auto &nodes : by) {
            if (nodes.empty()) continue;
            LevelPlan L;
            L.zlvl = zl; L.count = (int)nodes.size();
            L.nodes_off = (int64_t)pool_i32.size();
            pool_i32.insert(pool_i32.end(), nodes.begin(), nodes.end());
            // which destination panels are updated by MORE than one supernode of this level?  (LBlk / UBlk.shared; an
            // exclusive destination is updated tile-disjointly by its single source.  Every scatter is a RED today.)
            for (int k : nodes) {
                const NodeDesc &nd = H->nodes[k];
                if (nd.m <= 0 || nd.ncols <= 0) continue;
                auto touch = [&](int t) {
                    if (seen_by[t] == k) return;
                    seen_by[t] = k;
                    if (stamp[t] != (int)H->levels.size()) { stamp[t] = (int)H->levels.size(); ndest[t] = 0; }
                    ++ndest[t];
                };
                for (int q = 0; q < nd.nlb; ++q) touch(lblk[nd.lblk + q].ib);
                for (int q = 0; q < nd.nub; ++q) touch(ublk[nd.ublk + q].jb);
            }
            for (int k : nodes) {
                const NodeDesc &nd = H->nodes[k];
                if (nd.m <= 0 || nd.ncols <= 0) continue;
                for (int q = 0; q < nd.nlb; ++q) { LBlk &lb = lblk[nd.lblk + q]; lb.shared = ndest[lb.ib] >= 2; }
                for (int q = 0; q < nd.nub; ++q) { UBlk &ub = ublk[nd.ublk + q]; ub.shared = ndest[ub.jb] >= 2; }
            }
            std::vector<int32_t> big, small, tc;
            std::vector<int64_t> p_l{0}, p_u{0}, p_s{0}, p_big{0}, p_small{0}, p_inv{0}, p_urg{0}, p_bulk{0};
            std::vector<int64_t> p_tc{0}, p_tc_urg{0}, p_tc_bulk{0}, p_tc_rt{0}, p_tc_ak{0}, p_tc_b{0}, p_sl{0}, p_su{0};
            int64_t wr = 0, wc = 0, wl = 0, wu = 0, woz = 0, wozs = 0;
            L.slab_begin = INT64_MAX;
            for (int k : nodes) {
                NodeDesc &nd = H->nodes[k];
                L.slab_begin = std::min(L.slab_begin, nd.lval);
                L.slab_end = std::max(L.slab_end, std::max(nd.lval + (int64_t)nd.nsupr * nd.ns, nd.uval + (int64_t)nd.ns * nd.ncols));
                L.max_ns = std::max(L.max_ns, nd.ns);
                p_l.push_back(p_l.back() + (nd.m + TRSM_STRIP - 1) / TRSM_STRIP);
                p_u.push_back(p_u.back() + (nd.ncols + TRSM_STRIP - 1) / TRSM_STRIP);
                p_sl.push_back(p_sl.back() + (nd.m + 255) / 256);
                p_su.push_back(p_su.back() + (nd.ncols + 255) / 256);
                nd.ws_inv = p_inv.back() * 512;
                p_inv.push_back(p_inv.back() + (nd.ns + 15) / 16);
                bool has_schur = nd.m > 0 && nd.ncols > 0;
                int64_t tasks = has_schur ? (int64_t)nd.m + nd.ncols + nd.lrel_total + nd.urel_total : 0;
                p_s.push_back(p_s.back() + (tasks + SETUP_THREADS - 1) / SETUP_THREADS);
                nd.ws_row = wr; nd.ws_col = wc; nd.ws_lrel = wl; nd.ws_urel = wu;
                if (has_schur) {
                    wr += nd.m; wc += nd.ncols; wl += nd.lrel_total; wu += nd.urel_total;
                    if (nd.m >= 96 && nd.ncols >= 96) {
                        bool use_tc = false;
                        int bn = SCHUR_BN_TILE;
#ifndef SLU_COMPLEX
                        use_tc = H->tc_slices > 0 && nd.ns >= H->tc_min_ns && nd.ns <= 512 && (H->tc_max_m <= 0 || nd.m < H->tc_max_m);
                        if (use_tc) bn = OZ_NT_HOST;
#endif
                        (use_tc ? tc : big).push_back(k);
                        const int64_t tiles_m = (nd.m + SCHUR_BM_BIG - 1) / SCHUR_BM_BIG, tiles_n = (nd.ncols + bn - 1) / bn;
                        if (nd.defer) {   // only the panel tiles (the kernel takes them as mode 1 in every launch)
                            const int np = H->nodes[supno[lrows[nd.lrow + nd.ns]]].ns;
                            const int64_t tru = (np + SCHUR_BM_BIG - 1) / SCHUR_BM_BIG, tcu = (np + bn - 1) / bn;
                            const int64_t urg = tiles_m * tcu + tru * (tiles_n - tcu);
                            nd.urg_rows = np; nd.urg_cols = np;
                            p_big.push_back(p_big.back() + urg);
                            p_urg.push_back(p_urg.back() + urg);
                            p_bulk.push_back(p_bulk.back());
                            continue;
                        }
                        p_big.push_back(p_big.back() + tiles_m * tiles_n);
                        // look-ahead: which destinations are factored at the very next level of this forest?
                        int r1 = 0, c1 = 0;
                        bool other = false;
                        for (int q = 0; q < nd.nlb; ++q) {
                            const LBlk &lb = lblk[nd.lblk + q];
                            if (zl_of[lb.ib] == zl && lev[lb.ib] == lev[k] + 1) { if (q == 0) r1 = lb.nrows; else other = true; }
                        }
                        for (int q = 0; q < nd.nub; ++q) {
                            const UBlk &ub = ublk[nd.ublk + q];
                            if (zl_of[ub.jb] == zl && lev[ub.jb] == lev[k] + 1) { if (q == 0) c1 = ub.ncols; else other = true; }
                        }
                        if (other) { r1 = nd.m; c1 = nd.ncols; }
                        nd.urg_rows = r1; nd.urg_cols = c1;
                        const int64_t tru = (r1 + SCHUR_BM_BIG - 1) / SCHUR_BM_BIG, tcu = (c1 + bn - 1) / bn;
                        if (use_tc) {
#ifndef SLU_COMPLEX
                            p_big.pop_back();
                            p_tc.push_back(p_tc.back() + tiles_m * tiles_n);
                            p_tc_urg.push_back(p_tc_urg.back() + tiles_m * tcu + tru * (tiles_n - tcu));
                            p_tc_bulk.push_back(p_tc_bulk.back() + (tiles_m - tru) * (tiles_n - tcu));
                            const int S = H->tc_slices, KS = (nd.ns + OZ_KSTEP - 1) / OZ_KSTEP;
                            p_tc_rt.push_back(p_tc_rt.back() + tiles_m);
                            p_tc_ak.push_back(p_tc_ak.back() + tiles_m * KS);
                            p_tc_b.push_back(p_tc_b.back() + ((nd.ncols + OZ_NT - 1) / OZ_NT * OZ_NT + 3) / 4);
                            nd.ws_oza = woz; woz += oz_a_bytes(nd.m, nd.ns, S);
                            nd.ws_ozb = woz; woz += oz_b_bytes(nd.ncols, nd.ns, S);
                            nd.ws_ozs = wozs; wozs += oz_scale_elems(nd.m, nd.ncols);
                            if (!H->my_zero[zl]) ops_tc += 2.0 * nd.m * (double)nd.ns * nd.ncols;
#endif
                            continue;
                        }
                        p_urg.push_back(p_urg.back() + tiles_m * tcu + tru * (tiles_n - tcu));
                        p_bulk.push_back(p_bulk.back() + (tiles_m - tru) * (tiles_n - tcu));
                    } else {
                        small.push_back(k);
                        p_small.push_back(p_small.back() + (int64_t)((nd.m + SCHUR_BM_SMALL - 1) / SCHUR_BM_SMALL) * ((nd.ncols + SCHUR_BN_SMALL - 1) / SCHUR_BN_SMALL));
                    }
                }
            }
            ws_row_max = std::max(ws_row_max, wr); ws_col_max = std::max(ws_col_max, wc);
            ws_lrel_max = std::max(ws_lrel_max, wl); ws_urel_max = std::max(ws_urel_max, wu);
            ws_inv_max = std::max(ws_inv_max, p_inv.back() * 512);
            ws_oz_i8_max = std::max(ws_oz_i8_max, woz); ws_oz_s_max = std::max(ws_oz_s_max, wozs);
            auto put64 = [&](const std::vector<int64_t> &p) { int64_t o = (int64_t)pool_i64.size(); pool_i64.insert(pool_i64.end(), p.begin(), p.end()); return o; };
            L.trsml_prefix = put64(p_l); L.trsml_ctas = p_l.back();
            L.trsmu_prefix = put64(p_u); L.trsmu_ctas = p_u.back();
            L.setup_prefix = put64(p_s); L.setup_ctas = p_s.back();
            L.inv_prefix = put64(p_inv); L.inv_ctas = p_inv.back();
            L.sl_prefix = put64(p_sl); L.sl_ctas = p_sl.back();
            L.su_prefix = put64(p_su); L.su_ctas = p_su.back();
            L.big_count = (int)big.size(); L.big_nodes = (int64_t)pool_i32.size();
            pool_i32.insert(pool_i32.end(), big.begin(), big.end());
            L.big_prefix = put64(p_big); L.big_ctas = p_big.back();
            L.urg_prefix = put64(p_urg); L.urg_ctas = p_urg.back();
            L.bulk_prefix = put64(p_bulk); L.bulk_ctas = p_bulk.back();
            L.tc_count = (int)tc.size(); L.tc_nodes = (int64_t)pool_i32.size();
            pool_i32.insert(pool_i32.end(), tc.begin(), tc.end());
            L.tc_prefix = put64(p_tc); L.tc_ctas = p_tc.back();
            L.tc_urg_prefix = put64(p_tc_urg); L.tc_urg_ctas = p_tc_urg.back();
            L.tc_bulk_prefix = put64(p_tc_bulk); L.tc_bulk_ctas = p_tc_bulk.back();
            L.tc_p_rt = put64(p_tc_rt); L.tc_n_rt = p_tc_rt.back();
            L.tc_p_ak = put64(p_tc_ak); L.tc_n_ak = p_tc_ak.back();
            L.tc_p_b = put64(p_tc_b); L.tc_n_b = p_tc_b.back();
            L.small_count = (int)small.size(); L.small_nodes = (int64_t)pool_i32.size();
            pool_i32.insert(pool_i32.end(), small.begin(), small.end());
            L.small_prefix = put64(p_small); L.small_ctas = p_small.back();
            const int64_t lim = 2147483647LL;
            if (L.trsml_ctas > lim || L.trsmu_ctas > lim || L.setup_ctas > lim || L.big_ctas > lim || L.small_ctas > lim)
                return fail("a level needs more than 2^31 CTAs in one launch");
            H->levels.push_back(L);
        }
    }

    H->z_nodes_off.assign(max_lvl, 0);
    for (int zl = 0; zl < max_lvl; ++zl) {
        H->z_nodes_off[zl] = (int64_t)pool_i32.size();
        pool_i32.insert(pool_i32.end(), H->znodes[zl].begin(), H->znodes[zl].end());
    }
    lap("level batches");
    // the Schur workspace is double-buffered by level parity: with look-ahead the bulk update of level l still
    // reads its maps while level l+1 builds its own
    H->ws_max[0] = ws_row_max; H->ws_max[1] = ws_col_max; H->ws_max[2] = ws_lrel_max; H->ws_max[3] = ws_urel_max;
    for (size_t li = 0; li < H->levels.size(); ++li) {
        if (!(li & 1)) continue;
        const LevelPlan &L = H->levels[li];
        for (int t = 0; t < L.count; ++t) {
            NodeDesc &nd = H->nodes[pool_i32[L.nodes_off + t]];
            nd.ws_row += ws_row_max; nd.ws_col += ws_col_max; nd.ws_lrel += ws_lrel_max; nd.ws_urel += ws_urel_max;
            nd.ws_oza += ws_oz_i8_max; nd.ws_ozb += ws_oz_i8_max; nd.ws_ozs += ws_oz_s_max;
        }
    }
    // upload the index structures
    const int members = std::max(1, H->batch);
    H->member_len = voff; H->inv_len = ws_inv_max;
    if (H->val.alloc((size_t)voff * members)) return -1;
    if (H->d_nodes.upload(H->nodes) || H->d_xsup.upload(H->xsup) || H->d_supno.upload(supno) ||
        H->d_lrows.upload(lrows) || H->d_lsrow.upload(lsrow) || H->d_lspos.upload(lspos) ||
        H->d_ucols.upload(ucols) || H->d_ufst.upload(ufst) || H->d_useg.upload(useg) ||
        H->d_lblk.upload(lblk) || H->d_ublk.upload(ublk) || H->d_pool_i32.upload(pool_i32) ||
        H->d_pool_i64.upload(pool_i64) || H->d_kseg.upload(kseg))
        return -1;
    if (H->d_rowinfo.alloc((size_t)ws_row_max * 2) || H->d_colinfo.alloc((size_t)ws_col_max * 2) ||
        H->d_lrel.alloc((size_t)ws_lrel_max * 2) || H->d_urel.alloc((size_t)ws_urel_max * 2) || H->d_flags.alloc((size_t)members + 1) ||
        H->d_inv.alloc((size_t)ws_inv_max * members) ||
        H->d_tiny.alloc(1))
        return -1;
    if (ws_oz_i8_max > 0 &&
        (H->d_oz_i8.alloc((size_t)ws_oz_i8_max * 2) || H->d_oz_scale.alloc((size_t)ws_oz_s_max * 2) || H->d_oz_rexp.alloc((size_t)ws_oz_s_max * 2))) {
        H->tc_alloc_failed = true;
        H->d_oz_i8.release(); H->d_oz_scale.release(); H->d_oz_rexp.release();
        return fail("int8 tensor-core path: cannot allocate %.1f GB of int8 slice workspace (options.reserved[4] = -1 turns the path off): %s",
                    2e-9 * ws_oz_i8_max, g_err.c_str());
    }
    lap("device alloc + index upload");
    H->h_lblk = lblk;
    H->h_ublk = ublk;
    H->h_pool_i32 = pool_i32;
    DeviceLU &d = H->dev;
    d.val = H->val.p; d.nodes = H->d_nodes.p; d.xsup = H->d_xsup.p; d.supno = H->d_supno.p;
    d.lrows = H->d_lrows.p; d.lsrow = H->d_lsrow.p; d.lspos = H->d_lspos.p;
    d.ucols = H->d_ucols.p; d.ufst = H->d_ufst.p; d.useg = H->d_useg.p;
    d.lblk = H->d_lblk.p; d.ublk = H->d_ublk.p; d.rowinfo = H->d_rowinfo.p; d.colinfo = H->d_colinfo.p;
    d.oz_i8 = H->d_oz_i8.p; d.oz_scale = H->d_oz_scale.p; d.oz_rexp = H->d_oz_rexp.p;
    d.lrel = H->d_lrel.p; d.urel = H->d_urel.p; d.info = H->d_flags.p; d.err = H->d_flags.p + members; d.tiny = H->d_tiny.p;
    d.kseg = H->d_kseg.p;

    slu_b200_stats_t &st = H->st;
    st.ops_fact = ops; st.ops_schur = ops_schur; st.schur_bytes = bytes_schur;
    st.nnz_l = nnz_l; st.nnz_u = nnz_u; st.nlevels = (int)H->levels.size();
    st.lu_device_bytes = (int64_t)H->val.bytes();
    st.reserved[1] = ops_tc;                                   // Schur flops taken by the int8 tensor-core path
    st.reserved[2] = (double)(H->d_oz_i8.bytes() + H->d_oz_scale.bytes() + H->d_oz_rexp.bytes());
    st.reserved[3] = (double)H->tc_slices;
    st.index_device_bytes = (int64_t)(H->d_nodes.bytes() + H->d_xsup.bytes() + H->d_supno.bytes() + H->d_lrows.bytes() * 3 +
                                      H->d_ucols.bytes() * 3 + H->d_lblk.bytes() + H->d_ublk.bytes() + H->d_pool_i32.bytes() +
                                      H->d_pool_i64.bytes() + H->d_rowinfo.bytes() + H->d_colinfo.bytes() + H->d_lrel.bytes() +
                                      H->d_urel.bytes() + H->d_oz_i8.bytes() + H->d_oz_scale.bytes() + H->d_oz_rexp.bytes());
    int mine = 0;
    for (int zl = 0; zl < max_lvl; ++zl)
        if (!H->my_zero[zl])
            for (int k : H->znodes[zl]) mine += xsup[k] < H->schur_first;
    st.my_supernodes = mine;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Pr x Pc > 1.  The caller's panels are block-cyclic pieces (block (I,J) on process (I mod Pr, J mod Pc),
// SRC/include/superlu_defs.h:270-279).  Here every rank of a layer keeps the WHOLE panels of the layer's forests
// and the cooperative schedule does the rest: each rank uploads only its own blocks into a zeroed arena, the
// per-level all-reduce makes the panels complete, the Schur tiles are dealt over the Pr*Pc*2^level ranks of the
// group, and the local blocks are copied back at the end.  What the reference does with per-supernode panel and
// diagonal broadcasts (dIBcast_LPanel/UPanel, dcommunication_aux.c:29-283) becomes one NVSwitch all-reduce per level.
// ------------------------------------------------------------------------------------------------
int gather_structure(slu_b200_handle_s *H)
{
    const slu_b200_lu_view_t &v = H->view;
    const int nsupers = v.nsupers;
    H->Lidx.assign(nsupers, nullptr);
    H->Uidx.assign(nsupers, nullptr);
    if (H->P2 == 1) {
        for (int k = 0; k < nsupers; ++k) { H->Lidx[k] = v.Lrowind_bc_ptr[k]; H->Uidx[k] = v.Ufstnz_br_ptr[k]; }
        return 0;
    }
    const slu_int *xsup = v.xsup;
    // serialise my pieces of the supernodes of my forests: [type, k, len, payload]
    std::vector<int32_t> mine;
    std::vector<char> inforest(nsupers, 0);
    for (int zl = 0; zl < v.maxLvl; ++zl) {
        const slu_b200_forest_t &f = v.forests[v.myTreeIdxs[zl]];
        for (int t = 0; t < f.nNodes; ++t) inforest[f.nodeList[t]] = 1;
    }
    for (int k = 0; k < nsupers; ++k) {
        if (!inforest[k]) continue;
        if (k % v.npcol == v.mycol) {
            const slu_int *li = v.Lrowind_bc_ptr[k / v.npcol];
            if (li) {
                int len = BC_HEADER + li[0] * LB_DESCRIPTOR + li[1];
                mine.push_back(0); mine.push_back(k); mine.push_back(len);
                mine.insert(mine.end(), li, li + len);
            }
        }
        if (k % v.nprow == v.myrow) {
            const slu_int *ui = v.Ufstnz_br_ptr[k / v.nprow];
            if (ui) {
                mine.push_back(1); mine.push_back(k); mine.push_back(ui[2]);
                mine.insert(mine.end(), ui, ui + ui[2]);
            }
        }
    }
    // all-gather over my layer
    if (!g_nccl.AllGather) return fail("this NCCL has no ncclAllGather");
    const int P2 = H->P2;
    DevBuf<int32_t> dsz, dall, dsend, drecv;
    std::vector<int32_t> sizes(P2, 0), one{(int32_t)mine.size()};
    if (dsz.upload(one) || dall.alloc(P2)) return -1;
    NC(g_nccl.AllGather(dsz.p, dall.p, 1, NCCL_INT32, H->lcomm, H->stream));
    CU(cudaStreamSynchronize(H->stream));
    CU(cudaMemcpy(sizes.data(), dall.p, P2 * sizeof(int32_t), cudaMemcpyDeviceToHost));
    size_t maxn = 1;
    for (int s2 : sizes) maxn = std::max(maxn, (size_t)s2);
    std::vector<int32_t> padded(maxn, 0), all(maxn * P2);
    std::copy(mine.begin(), mine.end(), padded.begin());
    if (dsend.upload(padded) || drecv.alloc(maxn * P2)) return -1;
    NC(g_nccl.AllGather(dsend.p, drecv.p, maxn, NCCL_INT32, H->lcomm, H->stream));
    CU(cudaStreamSynchronize(H->stream));
    CU(cudaMemcpy(all.data(), drecv.p, all.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
    dsz.release(); dall.release(); dsend.release(); drecv.release();
    // merge
    struct Blk { int id; const int32_t *body; int len; };
    std::vector<std::vector<Blk>> lb(nsupers), ub(nsupers);
    for (int r = 0; r < P2; ++r) {
        const int32_t *p = all.data() + (size_t)r * maxn, *e = p + sizes[r];
        while (p < e) {
            int type = p[0], k = p[1], len = p[2];
            const int32_t *idx = p + 3;
            if (k < 0 || k >= nsupers) return fail("bad structure message");
            if (type == 0) {
                int w = BC_HEADER;
                for (int b = 0; b < idx[0]; ++b) { lb[k].push_back(Blk{idx[w], idx + w, LB_DESCRIPTOR + idx[w + 1]}); w += LB_DESCRIPTOR + idx[w + 1]; }
            } else {
                int u = BR_HEADER;
                for (int b = 0; b < idx[0]; ++b) {
                    int jns = xsup[idx[u] + 1] - xsup[idx[u]];
                    ub[k].push_back(Blk{idx[u], idx + u, UB_DESCRIPTOR + jns});
                    u += UB_DESCRIPTOR + jns;
                }
            }
            p += 3 + len;
        }
    }
    H->fullL.assign(nsupers, {});
    H->fullU.assign(nsupers, {});
    auto byid = [](const Blk &a, const Blk &b) { return a.id < b.id; };
    for (int k = 0; k < nsupers; ++k) {
        if (!inforest[k]) continue;
        if (!lb[k].empty()) {
            std::sort(lb[k].begin(), lb[k].end(), byid);
            std::vector<slu_int> &f = H->fullL[k];
            f.assign(BC_HEADER, 0);
            int nrows = 0;
            for (auto &b : lb[k]) { f.insert(f.end(), b.body, b.body + b.len); nrows += b.body[1]; }
            f[0] = (slu_int)lb[k].size(); f[1] = nrows;
            H->Lidx[k] = f.data();
        }
        if (!ub[k].empty()) {
            std::sort(ub[k].begin(), ub[k].end(), byid);
            std::vector<slu_int> &f = H->fullU[k];
            f.assign(BR_HEADER, 0);
            int nnz = 0;
            for (auto &b : ub[k]) { f.insert(f.end(), b.body, b.body + b.len); nnz += b.body[1]; }
            f[0] = (slu_int)ub[k].size(); f[1] = nnz; f[2] = (slu_int)f.size();
            H->Uidx[k] = f.data();
        }
    }
    return 0;
}

// where my local blocks sit inside the replicated panels
int build_pieces(slu_b200_handle_s *H)
{
    const slu_b200_lu_view_t &v = H->view;
    H->pieces.clear();
    if (H->P2 == 1) return 0;
    const slu_int *xsup = v.xsup;
    for (auto &zn : H->znodes)
        for (int k : zn) {
            const NodeDesc &nd = H->nodes[k];
            if (k % v.npcol == v.mycol && v.Lrowind_bc_ptr[k / v.npcol]) {
                const slu_int *li = v.Lrowind_bc_ptr[k / v.npcol];
                val_t *lv = (val_t *)v.Lnzval_bc_ptr[k / v.npcol];
                if (!lv) return fail("L piece %d has no values", k);
                // row offset of every block of the full panel
                const slu_int *fi = H->Lidx[k];
                int w = BC_HEADER, lo = 0;
                for (int b = 0; b < li[0]; ++b) {
                    int ib = li[w], nb = li[w + 1], fw = BC_HEADER, fo = 0, found = 0;
                    for (int q = 0; q < fi[0]; ++q) {
                        if (fi[fw] == ib) { found = 1; break; }
                        fo += fi[fw + 1]; fw += LB_DESCRIPTOR + fi[fw + 1];
                    }
                    if (!found) return fail("L piece %d: block %d missing from the merged panel", k, ib);
                    H->pieces.push_back({nd.lval + fo, lv + lo, nb, nd.ns, li[1], nd.nsupr});
                    lo += nb; w += LB_DESCRIPTOR + nb;
                }
            }
            if (k % v.nprow == v.myrow && v.Ufstnz_br_ptr[k / v.nprow]) {
                const slu_int *ui = v.Ufstnz_br_ptr[k / v.nprow];
                val_t *uv = (val_t *)v.Unzval_br_ptr[k / v.nprow];
                const int klst = xsup[k + 1];
                int u = BR_HEADER;
                int64_t lo = 0;
                for (int b = 0; b < ui[0]; ++b) {
                    int jb = ui[u], jns = xsup[jb + 1] - xsup[jb], cnt = 0;
                    for (int c = 0; c < jns; ++c) {
                        int fst = ui[u + UB_DESCRIPTOR + c];
                        if (fst >= klst) continue;
                        if (klst - fst != nd.ns) return fail("Pr x Pc > 1 needs U panels whose skyline segments are all full");
                        ++cnt;
                    }
                    if (cnt) {
                        int64_t col0 = -1;
                        for (int q = 0; q < nd.nub; ++q)
                            if (H->h_ublk[nd.ublk + q].jb == jb) { col0 = H->h_ublk[nd.ublk + q].col0; break; }
                        if (col0 < 0) return fail("U piece %d: block %d missing from the merged panel", k, jb);
                        if (!uv) return fail("U piece %d has no values", k);
                        H->pieces.push_back({nd.uval + col0 * nd.ns, uv + lo, (int64_t)cnt * nd.ns, 1, (int64_t)cnt * nd.ns, (int64_t)cnt * nd.ns});
                        lo += (int64_t)cnt * nd.ns;
                    }
                    u += UB_DESCRIPTOR + jns;
                }
            }
        }
    return 0;
}

int transfer_2d(slu_b200_handle_s *H, bool to_device)
{
    if (to_device) CU(cudaMemsetAsync(H->val.p, 0, H->val.bytes(), H->stream));
    for (const auto &p : H->pieces) {
        if (to_device)
            CU(cudaMemcpy2DAsync(H->val.p + p.dev, (size_t)p.dpitch * sizeof(val_t), p.host, (size_t)p.spitch * sizeof(val_t), (size_t)p.width * sizeof(val_t),
                                 (size_t)p.height, cudaMemcpyHostToDevice, H->stream));
        else
            CU(cudaMemcpy2DAsync(p.host, (size_t)p.spitch * sizeof(val_t), H->val.p + p.dev, (size_t)p.dpitch * sizeof(val_t), (size_t)p.width * sizeof(val_t),
                                 (size_t)p.height, cudaMemcpyDeviceToHost, H->stream));
    }
    CU(cudaStreamSynchronize(H->stream));
    return 0;
}

// copy a list of (device offset, host pointer, length) runs, merging neighbours
struct Run { int64_t dev; val_t *host; int64_t len; };
int copy_runs(slu_b200_handle_s *H, std::vector<Run> &runs, bool to_device, val_t *arena)
{
    size_t i = 0;
    while (i < runs.size()) {
        Run r = runs[i];
        size_t j = i + 1;
        while (j < runs.size() && runs[j].dev == r.dev + r.len && runs[j].host == r.host + r.len) { r.len += runs[j].len; ++j; }
        if (r.len > 0) {
            if (to_device) CU(cudaMemcpyAsync(arena + r.dev, r.host, (size_t)r.len * sizeof(val_t), cudaMemcpyHostToDevice, H->stream));
            else CU(cudaMemcpyAsync(r.host, arena + r.dev, (size_t)r.len * sizeof(val_t), cudaMemcpyDeviceToHost, H->stream));
        }
        i = j;
    }
    return 0;
}

// skyline <-> dense-packed conversion of the U panels that are not already identical
int convert_u(slu_b200_handle_s *H, bool to_device, val_t *arena)
{
    DeviceLU d = H->dev;
    d.val = arena;
    const size_t STAGE = (size_t)32 << 20;  // elements (256 MB of doubles) per round
    std::vector<int32_t> pend;
    for (auto &zn : H->znodes)
        for (int k : zn)
            if (!H->u_full[k] && H->nodes[k].ncols > 0) pend.push_back(k);
    if (pend.empty()) return 0;
    size_t need = 0;
    for (int k : pend) need = std::max(need, (size_t)H->sky_len[k]);
    if (H->stage.n < std::max(need, std::min(STAGE, need * 64))) {
        if (H->stage.alloc(std::max(need, std::min(STAGE, need * 64)))) return -1;
    }
    size_t i = 0;
    DevBuf<int32_t> dn;
    DevBuf<int64_t> dp, ds;
    while (i < pend.size()) {
        std::vector<int32_t> nodes;
        std::vector<int64_t> prefix{0}, soff;
        size_t used = 0;
        while (i < pend.size() && used + (size_t)H->sky_len[pend[i]] <= H->stage.n) {
            int k = pend[i++];
            nodes.push_back(k);
            soff.push_back((int64_t)used);
            used += (size_t)H->sky_len[k];
            prefix.push_back(prefix.back() + (H->nodes[k].ncols + 31) / 32);
        }
        if (dn.upload(nodes) || dp.upload(prefix) || ds.upload(soff)) return -1;
        Batch b{dn.p, dp.p, (int)nodes.size()};
        if (to_device) {
            for (size_t t = 0; t < nodes.size(); ++t)
                CU(cudaMemcpyAsync(H->stage.p + soff[t], H->view.Unzval_br_ptr[nodes[t]], (size_t)H->sky_len[nodes[t]] * sizeof(val_t),
                                   cudaMemcpyHostToDevice, H->stream));
            launch_u_convert(d, b, prefix.back(), 0, H->stage.p, ds.p, H->stream);
        } else {
            launch_u_convert(d, b, prefix.back(), 1, H->stage.p, ds.p, H->stream);
            for (size_t t = 0; t < nodes.size(); ++t)
                CU(cudaMemcpyAsync(H->view.Unzval_br_ptr[nodes[t]], H->stage.p + soff[t], (size_t)H->sky_len[nodes[t]] * sizeof(val_t),
                                   cudaMemcpyDeviceToHost, H->stream));
        }
        CU(cudaStreamSynchronize(H->stream));
        CU(cudaGetLastError());
    }
    dn.release(); dp.release(); ds.release();
    return 0;
}

// member: which value arena of a batched handle (0 for an ordinary one)
int transfer(slu_b200_handle_s *H, bool to_device, int member = 0)
{
    if (H->P2 > 1) return transfer_2d(H, to_device);
    val_t *arena = H->val.p + (int64_t)member * H->member_len;
    std::vector<Run> runs;
    for (auto &zn : H->znodes) {
        for (int k : zn) {
            const NodeDesc &nd = H->nodes[k];
            runs.push_back(Run{nd.lval, (val_t *)H->view.Lnzval_bc_ptr[k], (int64_t)nd.nsupr * nd.ns});
        }
        for (int k : zn) {
            const NodeDesc &nd = H->nodes[k];
            if (H->u_full[k] && nd.ncols > 0) runs.push_back(Run{nd.uval, (val_t *)H->view.Unzval_br_ptr[k], (int64_t)nd.ns * nd.ncols});
        }
    }
    for (auto &r : runs)
        if (r.len > 0 && !r.host) return fail("a held panel has a NULL value pointer");
    if (copy_runs(H, runs, to_device, arena)) return -1;
    if (convert_u(H, to_device, arena)) return -1;
    CU(cudaStreamSynchronize(H->stream));
    return 0;
}

int reduce_ancestors(slu_b200_handle_s *H, int zl)
{
    // dreduceAllAncestors3d (pd3dcomm.c:1046-1081): layers with z % 2^(zl+1) != 0 send all their
    // ancestor panels to z - 2^zl, which adds them.  The ancestor forests are one contiguous slab.
    const int z = H->view.mydep;
    const int64_t begin = H->chunk_start[zl + 1], end = H->chunk_start[H->max_lvl];
    const int64_t total = end - begin;
    if (total <= 0) return 0;
    const size_t CH = (size_t)64 << 20;  // elements per message (512 MB of doubles)
    if (z % (1 << (zl + 1)) != 0) {
        const int peer = z - (1 << zl);
        for (int64_t o = 0; o < total; o += (int64_t)CH) {
            size_t len = (size_t)std::min<int64_t>(CH, total - o);
            NC(g_nccl.Send(H->val.p + begin + o, len * VAL_DOUBLES, NCCL_FLOAT64, peer, H->comm, H->stream));
        }
    } else {
        const int peer = z + (1 << zl);
        if (H->stage.n < std::min<size_t>(CH, (size_t)total))
            if (H->stage.alloc(std::min<size_t>(CH, (size_t)total))) return -1;
        for (int64_t o = 0; o < total; o += (int64_t)CH) {
            size_t len = (size_t)std::min<int64_t>(CH, total - o);
            NC(g_nccl.Recv(H->stage.p, len * VAL_DOUBLES, NCCL_FLOAT64, peer, H->comm, H->stream));
            H->st.gpu_launches += launch_axpy(H->val.p + begin + o, H->stage.p, (int64_t)len, H->stream);
        }
    }
    return 0;
}

// ---- overlapped download ------------------------------------------------------------------------------------
// A panel is final as soon as the panel work of its level is done (nothing updates a factored panel), so its D2H
// can run on a copy stream while the upper levels are still being factored.  The arena is cut into chunks that are
// contiguous on both sides (host arrays of consecutive supernodes are usually adjacent); a chunk is released after
// the last level any of its panels belongs to.
int pipe_prepare(slu_b200_handle_s *H)
{
    if (H->pipe_ready) return 0;
    if (H->P2 > 1) return fail("overlapped transfers are not available for Pr x Pc > 1");
    for (auto &zn : H->znodes)
        for (int k : zn)
            if (!H->u_full[k] && H->nodes[k].ncols > 0)
                return fail("overlapped transfers need U panels whose skyline segments are all full");
    std::vector<int32_t> pool(H->d_pool_i32.n);
    CU(cudaMemcpy(pool.data(), H->d_pool_i32.p, pool.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
    std::vector<int> level_of(H->nsupers, -1);
    for (size_t li = 0; li < H->levels.size(); ++li)
        for (int t = 0; t < H->levels[li].count; ++t) level_of[pool[H->levels[li].nodes_off + t]] = (int)li;
    // panels in arena order, merged into chunks of <= 32M elements (256 MB of doubles)
    const int64_t CH = (int64_t)32 << 20;
    H->h_segs.clear(); H->h_seg_host.clear();
    std::vector<int> seg_level;
    bool fresh = true;       // never merge across a Z-level boundary: with reference-style ancestors a layer with
                             // my_zero[zl+1] never runs that level, and a chunk spanning both would never be released
    auto add = [&](int64_t dev, val_t *host, int64_t len, int lvl) {
        if (len <= 0) return;
        if (!H->h_segs.empty() && !fresh) {
            UpSeg &b2 = H->h_segs.back();
            if (b2.dst + b2.len == dev && H->h_seg_host.back() + b2.len == host && b2.len + len <= CH) {
                b2.len += len;
                seg_level.back() = std::max(seg_level.back(), lvl);
                return;
            }
        }
        H->h_segs.push_back(UpSeg{dev, 0, len});
        H->h_seg_host.push_back(host);
        seg_level.push_back(lvl);
        fresh = false;
    };
    for (auto &zn : H->znodes) {
        fresh = true;
        for (int k : zn) add(H->nodes[k].lval, (val_t *)H->view.Lnzval_bc_ptr[k], (int64_t)H->nodes[k].nsupr * H->nodes[k].ns, level_of[k]);
        for (int k : zn) add(H->nodes[k].uval, (val_t *)H->view.Unzval_br_ptr[k], (int64_t)H->nodes[k].ns * H->nodes[k].ncols, level_of[k]);
    }
    // bucket the chunks by release level
    H->lvl_segs.assign(H->levels.size(), {0, 0});
    std::vector<size_t> order(H->h_segs.size());
    for (size_t i = 0; i < order.size(); ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) { return seg_level[x] < seg_level[y]; });
    std::vector<UpSeg> segs2;
    std::vector<val_t *> host2;
    for (size_t i : order) {
        if (seg_level[i] < 0) continue;
        segs2.push_back(H->h_segs[i]);
        host2.push_back(H->h_seg_host[i]);
        H->lvl_segs[seg_level[i]][1] = (int64_t)segs2.size();
    }
    int64_t prev = 0;
    for (auto &r : H->lvl_segs) { r[0] = prev; if (r[1] < prev) r[1] = prev; prev = r[1]; }
    H->h_segs.swap(segs2);
    H->h_seg_host.swap(host2);
    if (!H->s_down && cudaStreamCreateWithFlags(&H->s_down, cudaStreamNonBlocking) != cudaSuccess)
        return fail("cannot create the download stream");
    H->pipe_ready = true;
    return 0;
}

// D2H of the chunks whose panels are all final once level li's panel work is done
int pipe_download_level(slu_b200_handle_s *H, size_t li)
{
    const int64_t a = H->lvl_segs[li][0], b = H->lvl_segs[li][1];
    if (a >= b) return 0;
    CU(cudaStreamWaitEvent(H->s_down, H->ev_panel[li], 0));
    for (int64_t q = a; q < b; ++q)
        CU(cudaMemcpyAsync(H->h_seg_host[q], H->val.p + H->h_segs[q].dst, (size_t)H->h_segs[q].len * sizeof(val_t), cudaMemcpyDeviceToHost, H->s_down));
    return 0;
}

// ---- overlapped upload (options.reserved[3]) ---------------------------------------------------------------
// With the level-by-level layout the panels are needed in arena order.  The arena is zeroed, every level's host
// panels are copied through a staging buffer and ADDED to the arena with atomic adds on a copy stream (a Schur
// update scattered into an ancestor before that ancestor's A values arrive commutes with the addition), and the
// panel work of level li waits for the event of level li only: the H2D of the upper levels -- most of the bytes --
// runs under the factorization of the lower ones.
int upload_pipe_issue(slu_b200_handle_s *H)
{
    if (!H->grouped) return fail("overlapped upload needs options.reserved[3] at create time and Pr x Pc = 1");
    for (auto &zn : H->znodes)
        for (int k : zn)
            if (!H->u_full[k] && H->nodes[k].ncols > 0)
                return fail("overlapped transfers need U panels whose skyline segments are all full");
    const size_t CAP = (size_t)32 << 20;  // elements per staging round
    if (H->stage.n < CAP && H->stage.alloc(CAP)) return -1;
    if (!H->s_up && cudaStreamCreateWithFlags(&H->s_up, cudaStreamNonBlocking) != cudaSuccess)
        return fail("cannot create the upload stream");
    if (H->ev_up.size() != H->levels.size()) {
        for (auto e : H->ev_up) if (e) cudaEventDestroy(e);
        H->ev_up.assign(H->levels.size(), nullptr);
        for (auto &e : H->ev_up) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    }
    cudaStream_t su = H->s_up;
    CU(cudaMemsetAsync(H->val.p, 0, H->val.bytes(), su));
    for (size_t li = 0; li < H->levels.size(); ++li) {
        const LevelPlan &L = H->levels[li];
        const int32_t *nodes = H->h_pool_i32.data() + L.nodes_off;
        int64_t off = L.slab_begin;   // next arena element to receive
        size_t fill = 0;
        auto flush = [&]() -> int {
            if (!fill) return 0;
            H->st.gpu_launches += launch_axpy_atomic(H->val.p + off, H->stage.p, (int64_t)fill, su);
            off += (int64_t)fill;
            fill = 0;
            return 0;
        };
        for (int pass = 0; pass < 2; ++pass)  // the L panels of the level, then its U panels (arena order)
            for (int t = 0; t < L.count; ++t) {
                const int k = nodes[t];
                const NodeDesc &nd = H->nodes[k];
                const int64_t dev = pass ? nd.uval : nd.lval;
                const int64_t len = pass ? (int64_t)nd.ns * nd.ncols : (int64_t)nd.nsupr * nd.ns;
                const val_t *host = (const val_t *)(pass ? H->view.Unzval_br_ptr[k] : H->view.Lnzval_bc_ptr[k]);
                if (len <= 0) continue;
                if (dev != off + (int64_t)fill) return fail("internal: level %zu is not contiguous in the arena", li);
                if (!host) return fail("a held panel has a NULL value pointer");
                int64_t pos = 0;
                while (pos < len) {
                    const size_t take = (size_t)std::min<int64_t>(len - pos, (int64_t)(CAP - fill));
                    CU(cudaMemcpyAsync(H->stage.p + fill, host + pos, take * sizeof(val_t), cudaMemcpyHostToDevice, su));
                    fill += take; pos += (int64_t)take;
                    if (fill == CAP && flush()) return -1;
                }
            }
        if (flush()) return -1;
        CU(cudaEventRecord(H->ev_up[li], su));
    }
    return 0;
}

// The panel work of one level: diagonal LU, the inverses of the 16x16 diagonal blocks, the two panel solves and the
// destination maps of the Schur update (value-independent: built once on H->dev for every member).  marks: nullptr, or
// two profiling events recorded after the diagonal LU and after the panel solves.  Returns the kernel launches.
template <class LU>
int panel_work(const slu_b200_handle_s *H, const LU &d, const LevelPlan &L, int replace_tiny, cudaStream_t s,
               const cudaEvent_t *marks = nullptr)
{
    const int32_t *nodes = H->d_pool_i32.p + L.nodes_off;
    const int64_t *p64 = H->d_pool_i64.p;
    int launches = launch_diag_lu(d, Batch{nodes, p64 + L.trsml_prefix, L.count}, L.max_ns, replace_tiny, H->opt.thresh, s);
    if (marks) cudaEventRecord(marks[0], s);
    launches += launch_diag_inv(d, Batch{nodes, p64 + L.inv_prefix, L.count}, L.inv_ctas, H->d_inv.p, s);
    launches += launch_trsm_l(d, Batch{nodes, p64 + L.trsml_prefix, L.count}, L.trsml_ctas, L.max_ns, H->d_inv.p, s);
    launches += launch_trsm_u(d, Batch{nodes, p64 + L.trsmu_prefix, L.count}, L.trsmu_ctas, L.max_ns, H->d_inv.p, s);
    if (marks) cudaEventRecord(marks[1], s);
    launches += launch_schur_setup(H->dev, Batch{nodes, p64 + L.setup_prefix, L.count}, L.setup_ctas, s);
    return launches;
}

// the Schur launch of the level loop: the cooperative split of an unbatched handle; a batched handle has none
int schur_launch(const DeviceLU &d, const Batch &b, int64_t ctas, int big, int mode, int split_n, int split_i, cudaStream_t s)
{
    return launch_schur(d, b, ctas, big, mode, split_n, split_i, s);
}
int schur_launch(const BatchedLU &d, const Batch &b, int64_t ctas, int big, int mode, int, int, cudaStream_t s)
{
    return launch_schur(d, b, ctas, big, mode, s);
}

// The level loop of a factorization, enqueued on H->stream (the bulk Schur tiles on stream2 with look-ahead, joined back
// before it returns) after the caller has reset the info flags and d_tiny: slu_b200_factor, factor_host, batch_factor and
// the factor_device twins.  d = H->dev, or H->bdev with every launch over the members (a batched handle has a 1 x 1 x 1
// grid and no int8 levels: tc_count = 0).  prof: the per-level timings of options.verbose >= 2, which wait for every
// level; pipelined / up_pipe: factor_host's overlapped D2H / H2D.  Without them and on one rank, no host wait, no
// allocation and no host copy: the loop can be captured into a CUDA graph.  Returns the kernel launches, < 0 on an error.
template <class LU>
int64_t factor_levels(slu_b200_handle_s *H, const LU &d, bool prof, bool pipelined, bool up_pipe)
{
    float t_diag = 0, t_trsm = 0, t_setup = 0, t_schur = 0, t_red = 0;
    EventSet pe;
    if (prof && pe.create()) return fail("cannot create the profiling events");
    const cudaStream_t s = H->stream, s2 = H->stream2;
    int64_t launches = 0;
    // Look-ahead (the role of dsparseTreeFactor_ASYNC's pipeline, dtreeFactorization.c:430-454,598-706): the
    // critical path (panel work of level l, then the "urgent" Schur tiles that feed the panels of level l+1) runs on
    // a high-priority stream; the bulk of the Schur update of level l runs on a second stream, concurrently with the
    // panel work of level l+1.  All updates are atomic adds, so bulk(l) and anything of level l+1 commute; the only
    // ordering needed is panel(l) after bulk(l-2) (in-order stream: after every earlier bulk).
    const bool lookahead = !prof && !H->opt.reserved[0];
    size_t li = 0;
    for (int zl = 0; zl < H->max_lvl; ++zl) {
        const bool coopz = H->coop && (zl >= 1 || H->P2 > 1);
        if (H->my_zero[zl] && !coopz) continue;  // pdgstrf3d.c:336
        const int split_n = coopz ? (H->P2 << zl) : 1;
        const int split_i = coopz ? ((H->view.mydep & ((1 << zl) - 1)) * H->P2 + H->view.myrow * H->view.npcol + H->view.mycol) : 0;
        size_t first = (size_t)-1, last = (size_t)-1;
        for (; li < H->levels.size() && H->levels[li].zlvl <= zl; ++li) {
            const LevelPlan &L = H->levels[li];
            if (L.zlvl < zl) continue;
            if (first == (size_t)-1) first = li;
            last = li;
            const int64_t *p64 = H->d_pool_i64.p;
            if (lookahead && li >= first + 2) CU(cudaStreamWaitEvent(s, H->ev_bulk[li - 2], 0));
            if (up_pipe) CU(cudaStreamWaitEvent(s, H->ev_up[li], 0));  // this level's A values are in the arena
            if (coopz && L.slab_end > L.slab_begin) {
                // every rank of the Z group holds a partial sum of this level's panels (its own Schur contributions,
                // plus A on the group leader): one in-place all-reduce makes them complete and identical everywhere.
                // Replaces dreduceAllAncestors3d's pairwise Send/Recv (pd3dcomm.c:1046-1081) for this forest.
                if (prof) cudaEventRecord(pe[5], s);
                NC(g_nccl.AllReduce(H->val.p + L.slab_begin, H->val.p + L.slab_begin, (size_t)(L.slab_end - L.slab_begin) * VAL_DOUBLES,
                                    NCCL_FLOAT64, NCCL_SUM, H->gcomm[zl], s));
                if (prof) { cudaEventRecord(pe[0], s); cudaEventSynchronize(pe[0]); float ms; cudaEventElapsedTime(&ms, pe[5], pe[0]); t_red += ms; }
            }
            if (prof) cudaEventRecord(pe[0], s);
            // tiny-pivot replacements are counted once: by the layer that owns the forest (not by the replicated
            // copies of a cooperative group) and by one rank of its 2D grid (stat->TinyPivots is MPI_SUMmed there,
            // pdgssvx3d.c:1149)
            const bool count_tiny = !H->my_zero[zl] && (H->P2 == 1 || (H->view.myrow == 0 && H->view.mycol == 0));
            launches += panel_work(H, d, L, H->opt.replace_tiny_pivot ? (count_tiny ? 1 : 2) : 0, s, prof ? &pe[1] : nullptr);
#ifndef SLU_COMPLEX
            const int32_t *tcn = H->d_pool_i32.p + L.tc_nodes;
            if (L.tc_count > 0)      // int8 slices of the level's wide panels (final after the TRSMs above)
                launches += launch_oz_slice(d, tcn, L.tc_count, p64 + L.tc_p_rt, L.tc_n_rt, p64 + L.tc_p_ak, L.tc_n_ak,
                                            p64 + L.tc_p_b, L.tc_n_b, H->tc_slices, s);
#endif
            if (prof) cudaEventRecord(pe[3], s);
            const int32_t *bign = H->d_pool_i32.p + L.big_nodes;
            if (lookahead || pipelined) CU(cudaEventRecord(H->ev_panel[li], s));
            if (pipelined && pipe_download_level(H, li)) return -1;
            if (lookahead) {
                launches += schur_launch(d, Batch{bign, p64 + L.urg_prefix, L.big_count}, L.urg_ctas, 1, 1, split_n, split_i, s);
                launches += schur_launch(d, Batch{H->d_pool_i32.p + L.small_nodes, p64 + L.small_prefix, L.small_count}, L.small_ctas, 0, 0, split_n, split_i, s);
#ifndef SLU_COMPLEX
                launches += launch_oz_schur(d, Batch{tcn, p64 + L.tc_urg_prefix, L.tc_count}, L.tc_urg_ctas, 1, split_n, split_i, H->tc_slices, s);
#endif
                CU(cudaStreamWaitEvent(s2, H->ev_panel[li], 0));
#ifndef SLU_COMPLEX
                launches += launch_oz_schur(d, Batch{tcn, p64 + L.tc_bulk_prefix, L.tc_count}, L.tc_bulk_ctas, 2, split_n, split_i, H->tc_slices, s2);
#endif
                launches += schur_launch(d, Batch{bign, p64 + L.bulk_prefix, L.big_count}, L.bulk_ctas, 1, 2, split_n, split_i, s2);
                CU(cudaEventRecord(H->ev_bulk[li], s2));
            } else {
#ifndef SLU_COMPLEX
                launches += launch_oz_schur(d, Batch{tcn, p64 + L.tc_prefix, L.tc_count}, L.tc_ctas, 0, split_n, split_i, H->tc_slices, s);
#endif
                launches += schur_launch(d, Batch{bign, p64 + L.big_prefix, L.big_count}, L.big_ctas, 1, 0, split_n, split_i, s);
                launches += schur_launch(d, Batch{H->d_pool_i32.p + L.small_nodes, p64 + L.small_prefix, L.small_count}, L.small_ctas, 0, 0, split_n, split_i, s);
            }
            if (prof) {
                cudaEventRecord(pe[4], s);
                cudaEventSynchronize(pe[4]);
                float ms;
                cudaEventElapsedTime(&ms, pe[0], pe[1]); t_diag += ms;
                cudaEventElapsedTime(&ms, pe[1], pe[2]); t_trsm += ms;
                cudaEventElapsedTime(&ms, pe[2], pe[3]); t_setup += ms;
                cudaEventElapsedTime(&ms, pe[3], pe[4]); t_schur += ms;
            }
        }
        if (lookahead && last != (size_t)-1) {  // join the bulk stream before anything that reads the ancestors
            CU(cudaStreamWaitEvent(s, H->ev_bulk[last], 0));
            if (last > first) CU(cudaStreamWaitEvent(s, H->ev_bulk[last - 1], 0));
        }
        if (zl < H->max_lvl - 1 && !H->coop) {
            if (prof) cudaEventRecord(pe[0], s);
            // the pairwise reduction adds non-atomically: every upload into the ancestors must have landed
            if (up_pipe && !H->ev_up.empty()) CU(cudaStreamWaitEvent(s, H->ev_up.back(), 0));
            if (reduce_ancestors(H, zl)) return -1;
            if (prof) { cudaEventRecord(pe[1], s); cudaEventSynchronize(pe[1]); float ms; cudaEventElapsedTime(&ms, pe[0], pe[1]); t_red += ms; }
        }
    }
    if (prof) {
        H->st.t_diag_ms = t_diag; H->st.t_trsm_ms = t_trsm; H->st.t_schur_setup_ms = t_setup; H->st.t_schur_ms = t_schur; H->st.t_reduce_ms = t_red;
    }
    return launches;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// C-ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

#ifndef SLU_COMPLEX
int slu_b200_abi_version(void) { return SLU_B200_ABI_VERSION; }
void slu_b200_struct_sizes(int32_t out[4])
{
    out[0] = (int32_t)sizeof(slu_b200_forest_t); out[1] = (int32_t)sizeof(slu_b200_lu_view_t);
    out[2] = (int32_t)sizeof(slu_b200_options_t); out[3] = (int32_t)sizeof(slu_b200_stats_t);
}
const char *slu_b200_last_error(void) { return g_err.c_str(); }
int slu_b200_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int slu_b200_nccl_unique_id(unsigned char id[128])
{
    if (!g_nccl.load()) return fail("cannot load libnccl.so.2");
    slu_nccl_id u;
    NC(g_nccl.GetUniqueId(&u));
    memcpy(id, u.internal, 128);
    return 0;
}

void *slu_b200_host_alloc(size_t bytes)
{
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void slu_b200_host_free(void *p) { if (p) cudaFreeHost(p); }
#endif  // !SLU_COMPLEX

#ifdef SLU_COMPLEX
void slu_b200_z_comm_cache_clear(void)
#else
void slu_b200_z_comm_cache_clear(void);
static void comm_cache_clear_d(void)
#endif
{
    std::lock_guard<std::mutex> lock(g_comm_mu);
    for (auto &kv : g_comm_cache) {
        for (void *c : kv.second.gcomm) if (c && g_nccl.CommDestroy) g_nccl.CommDestroy(c);
        if (kv.second.comm && g_nccl.CommDestroy) g_nccl.CommDestroy(kv.second.comm);
    }
    g_comm_cache.clear();
}
#ifndef SLU_COMPLEX
void slu_b200_comm_cache_clear(void)
{
    comm_cache_clear_d();
    slu_b200_z_comm_cache_clear();
}
#endif

void slu_b200_destroy(slu_b200_handle_t H)
{
    if (!H) return;
    // the NCCL communicators belong to the per-process cache (slu_b200_comm_cache_clear)
    if (H->ev0) cudaEventDestroy(H->ev0);
    if (H->ev1) cudaEventDestroy(H->ev1);
    if (H->ev_in) cudaEventDestroy(H->ev_in);
    if (H->ev_out) cudaEventDestroy(H->ev_out);
    if (H->stream) cudaStreamDestroy(H->stream);
    if (H->stream2) cudaStreamDestroy(H->stream2);
    if (H->s_down) cudaStreamDestroy(H->s_down);
    if (H->s_up) cudaStreamDestroy(H->s_up);
    for (auto s : H->s_body) if (s) cudaStreamDestroy(s);
    for (auto &g : H->loop_graphs) {
        cudaGraphExecDestroy(g.exec);
        cudaGraphDestroy(g.graph);
    }
    for (auto e : H->ev_up) if (e) cudaEventDestroy(e);
    for (auto e : H->ev_panel) if (e) cudaEventDestroy(e);
    for (auto e : H->ev_bulk) if (e) cudaEventDestroy(e);
    delete H;                                   // every DevBuf frees its HBM
}

// batch > 0: a batched handle (slu_b200_batch_create), 1 x 1 x 1 grid, FP64 DMMA kernels only
// nschur > 0: a Schur handle (slu_b200_schur_create), 1 x 1 x 1 grid, FP64 DMMA kernels only; with batch > 0 a batched one
// (slu_b200_batch_schur_create)
static int create_impl(slu_b200_handle_t *out, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, int batch, int nschur = 0)
{
    if (!out || !lu || !opt) return fail("null argument");
    *out = nullptr;
    if (opt->schur_variant != 0) return fail("options.schur_variant is retired and must be 0 (got %d)", opt->schur_variant);
    if (nschur) {
        const char *fn = batch ? SLU_API "batch_schur_create" : SLU_API "schur_create";
        if (nschur < 1 || nschur >= lu->n) return fail("%s: nschur = %d, must satisfy 1 <= nschur < n = %d", fn, nschur, lu->n);
        if (lu->nprow != 1 || lu->npcol != 1 || lu->npdep != 1 || opt->world_size > 1)
            return fail("%s handles 1 x 1 x 1 grids (world_size 1)", fn);
        if (opt->reserved[4] > 0) return fail("%s: the int8 tensor-core path (options.reserved[4] = %d) is not available on a Schur handle", fn, opt->reserved[4]);
        const int n0 = lu->n - nschur;
        for (int k = 0; k < lu->nsupers; ++k)
            if (lu->xsup[k] < n0 && lu->xsup[k + 1] > n0)
                return fail("%s: column n - nschur = %d is not a supernode boundary: supernode %d spans columns %d..%d", fn, n0, k,
                            lu->xsup[k], lu->xsup[k + 1] - 1);
    }
    if (slu_b200_device_count() < 1) return fail("no CUDA device: libslu_b200 has no CPU fallback");
    if (device_setup(opt)) return -1;
    slu_b200_handle_s *H = new slu_b200_handle_s;
    H->view = *lu;
    H->opt = *opt;
    H->batch = batch;
    H->nschur = nschur;
    if (nschur) H->schur_first = lu->n - nschur;
    if (batch || nschur) {   // the int8 path and the overlapped upload are not batched, nor used by a partial factorization
        H->opt.reserved[3] = 0;
        H->opt.reserved[4] = -1;
        H->tc_force_off = true;
    }
    H->coop = opt->world_size > 1 && !opt->reserved[1];
    H->P2 = lu->nprow * lu->npcol;
    double t0 = now_s();
    if (lu->npdep < 1 || (lu->npdep & (lu->npdep - 1)) || H->P2 < 1) { slu_b200_destroy(H); return fail("bad process grid"); }
    H->max_lvl = 1;
    while ((1 << (H->max_lvl - 1)) < lu->npdep) ++H->max_lvl;
    if (cudaGetDevice(&H->device) != cudaSuccess || cudaStreamCreate(&H->stream) != cudaSuccess || cudaEventCreate(&H->ev0) != cudaSuccess ||
        cudaEventCreate(&H->ev1) != cudaSuccess || cudaEventCreateWithFlags(&H->ev_in, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&H->ev_out, cudaEventDisableTiming) != cudaSuccess) {
        slu_b200_destroy(H);
        return fail("cannot create stream/events");
    }
    if (opt->world_size > 1) {
        if (opt->world_size != lu->npdep * H->P2) { slu_b200_destroy(H); return fail("world_size does not match the process grid"); }
        if (!g_nccl.load()) { slu_b200_destroy(H); return fail("cannot load libnccl.so.2"); }
        std::string key((const char *)opt->nccl_id, 128);
        const int32_t shape[9] = {opt->world_size, opt->world_rank, lu->nprow, lu->npcol, lu->npdep, lu->myrow, lu->mycol, lu->mydep, (int32_t)H->coop};
        key.append((const char *)shape, sizeof shape);
        std::lock_guard<std::mutex> lock(g_comm_mu);
        CommSet &cs = g_comm_cache[key];
        if (!cs.comm) {
            slu_nccl_id id;
            memcpy(id.internal, opt->nccl_id, 128);
            int r = g_nccl.CommInitRank(&cs.comm, opt->world_size, id, opt->world_rank);
            if (r != 0) { g_comm_cache.erase(key); slu_b200_destroy(H); return fail("ncclCommInitRank failed: %d", r); }
            cs.gcomm.assign(H->max_lvl, nullptr);
            if (H->coop) {
                if (!g_nccl.CommSplit) { g_comm_cache.erase(key); slu_b200_destroy(H); return fail("this NCCL has no ncclCommSplit (need >= 2.18)"); }
                // my group at Z level zl: the Pr*Pc ranks of each of the 2^zl layers sharing forest my_tree[zl]
                for (int zl = (H->P2 > 1 ? 0 : 1); zl < H->max_lvl; ++zl) {
                    r = g_nccl.CommSplit(cs.comm, lu->mydep >> zl, opt->world_rank, &cs.gcomm[zl], nullptr);
                    if (r != 0) { g_comm_cache.erase(key); slu_b200_destroy(H); return fail("ncclCommSplit failed: %d", r); }
                }
            }
        }
        H->comm = cs.comm;
        H->gcomm = cs.gcomm;
        if (H->coop) H->lcomm = H->gcomm[0];
    } else if (lu->npdep > 1 || H->P2 > 1) {
        slu_b200_destroy(H);
        return fail("a process grid with more than one rank needs world_size == nprow*npcol*npdep and an NCCL id");
    }
    if (gather_structure(H)) { slu_b200_destroy(H); return -1; }
    if (analyze(H)) {
        // the int8 slice workspace of the int8 tensor-core path did not fit beside the L/U arena: plan again without it (FP64 DMMA only)
        if (!H->tc_alloc_failed) { slu_b200_destroy(H); return -1; }
        cudaGetLastError();
        H->tc_force_off = true;
        H->tc_alloc_failed = false;
        if (analyze(H)) { slu_b200_destroy(H); return -1; }
    }
    if (build_pieces(H)) { slu_b200_destroy(H); return -1; }
    if (nschur) {            // the gather units: every L column and every packed U column of the Schur supernodes
        std::vector<int2> units;
        for (int k = 0; k < H->nsupers; ++k) {
            if (H->xsup[k] < H->schur_first) continue;
            const NodeDesc &nd = H->nodes[k];
            for (int c = 0; c < nd.ns + nd.ncols; ++c) units.push_back(make_int2(k, c));
        }
        if (H->d_sunits.upload(units)) { slu_b200_destroy(H); return -1; }
    }
    if (batch) {             // the stats describe the whole handle: every member's work
        slu_b200_stats_t &st = H->st;
        st.ops_fact *= batch; st.ops_schur *= batch; st.schur_bytes *= batch;
        st.nnz_l *= batch; st.nnz_u *= batch;
        static_cast<DeviceLU &>(H->bdev) = H->dev;
        H->bdev.val_stride = H->member_len;
        H->bdev.inv_stride = H->inv_len;
        H->bdev.members = batch;
    }
    H->member_info.assign(batch ? batch : 1, -1);
    if (H->d_info.alloc(H->member_info.size()) || cudaMemset(H->d_info.p, 0xff, H->d_info.bytes()) != cudaSuccess ||
        H->d_epoch.alloc(1) || cudaMemset(H->d_epoch.p, 0, H->d_epoch.bytes()) != cudaSuccess) {
        slu_b200_destroy(H);
        return fail("cannot allocate the device status");
    }
    {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);  // hi = numerically lowest = highest priority
        cudaStreamDestroy(H->stream);
        H->stream = nullptr;
        if (cudaStreamCreateWithPriority(&H->stream, cudaStreamNonBlocking, hi) != cudaSuccess ||
            cudaStreamCreateWithPriority(&H->stream2, cudaStreamNonBlocking, lo) != cudaSuccess) {
            slu_b200_destroy(H);
            return fail("cannot create the look-ahead streams");
        }
        H->ev_panel.resize(H->levels.size());
        H->ev_bulk.resize(H->levels.size());
        for (size_t i = 0; i < H->levels.size(); ++i) {
            cudaEventCreateWithFlags(&H->ev_panel[i], cudaEventDisableTiming);
            cudaEventCreateWithFlags(&H->ev_bulk[i], cudaEventDisableTiming);
        }
    }
    H->st.t_analyze_s = now_s() - t0;
    *out = H;
    return 0;
}

int slu_b200_create(slu_b200_handle_t *out, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt)
{
    return create_impl(out, lu, opt, 0);
}

int slu_b200_upload(slu_b200_handle_t H)
{
    if (!H) return fail("null handle");
    if (check(H, SLU_API "upload", UNBATCHED)) return -1;
    double t0 = now_s();
    if (values_replaced(H)) return -1;
    if (transfer(H, true)) return -1;
    H->st.t_upload_s = now_s() - t0;
    H->uploaded = true;
    return 0;
}

int slu_b200_download(slu_b200_handle_t H)
{
    if (!H) return fail("null handle");
    if (check(H, SLU_API "download", UNBATCHED)) return -1;
    double t0 = now_s();
    if (transfer(H, false)) return -1;
    H->st.t_download_s = now_s() - t0;
    return 0;
}

static int factor_impl(slu_b200_handle_t H, int *info, bool pipelined, bool up_pipe = false)
{
    if (!H || !info) return fail("null argument");
    if (check(H, SLU_API "factor", UNBATCHED | UPLOADED)) return -1;
    if (factors_replaced(H)) return -1;
    if (pipelined && pipe_prepare(H)) return -1;
    cudaStream_t s = H->stream;
    int init[2] = {INT_MAX, 0};
    CU(cudaMemcpyAsync(H->d_flags.p, init, sizeof init, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(H->d_tiny.p, 0, sizeof(unsigned long long), s));
    H->st.gpu_launches = 0;                // the pairwise reduction of the level loop adds its launches here too
    const bool prof = H->opt.verbose >= 2 && !pipelined;
    CU(cudaEventRecord(H->ev0, s));
    const int64_t launches = factor_levels(H, H->dev, prof, pipelined, up_pipe);
    if (launches < 0) return -1;
    H->st.gpu_launches += launches;
    if (H->comm)  // pdgstrf3d.c:388-392: MPI_Allreduce(info, MIN) over the 3D grid
        NC(g_nccl.AllReduce(H->d_flags.p, H->d_flags.p, 1, NCCL_INT32, NCCL_MIN, H->comm, s));
    CU(cudaEventRecord(H->ev1, s));
    CU(cudaStreamSynchronize(s));
    if (pipelined) CU(cudaStreamSynchronize(H->s_down));
    if (up_pipe) CU(cudaStreamSynchronize(H->s_up));
    CU(cudaGetLastError());
    float ms = 0;
    CU(cudaEventElapsedTime(&ms, H->ev0, H->ev1));
    H->st.t_factor_s = ms * 1e-3;
    int flags[2];
    unsigned long long tiny = 0;
    CU(cudaMemcpy(flags, H->d_flags.p, sizeof flags, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&tiny, H->d_tiny.p, sizeof tiny, cudaMemcpyDeviceToHost));
    H->st.tiny_pivots = (int64_t)tiny;
    if (flags[1]) return fail("%d Schur-update destinations were not found in the L/U structure", flags[1]);
    *info = H->member_info[0] = flags[0] == INT_MAX ? 0 : flags[0];
    CU(cudaMemcpy(H->d_info.p, H->member_info.data(), sizeof(int32_t), cudaMemcpyHostToDevice));   // for the device solves
    return 0;
}

int slu_b200_factor(slu_b200_handle_t H, int *info) { return factor_impl(H, info, false); }

int slu_b200_factor_host(slu_b200_handle_t H, int *info)
{
    if (!H || !info) return fail("null argument");
    if (check(H, SLU_API "factor_host", UNBATCHED | NOT_SCHUR)) return -1;
    // The overlapped transfers move whole panels between the caller's arrays and the arena, which needs the U
    // skylines to equal their dense-packed form (symmetric patterns) and 1 x 1 x Pz pieces.  Anything else -- the
    // unsymmetric patterns SuperLU exists for, Pr x Pc pieces -- takes the plain path: upload (with the skyline
    // conversion), factor, download.  Same results, no overlap.
    bool overlappable = H->P2 == 1;
    for (size_t zl = 0; zl < H->znodes.size() && overlappable; ++zl)
        for (int k : H->znodes[zl])
            if (!H->u_full[k] && H->nodes[k].ncols > 0) { overlappable = false; break; }
    if (!overlappable) {
        if (slu_b200_upload(H)) return -1;
        int rc2 = factor_impl(H, info, false);
        return rc2 ? rc2 : slu_b200_download(H);
    }
    if (H->grouped) {                      // options.reserved[3]: H2D, factorization and D2H all overlapped
        if (values_replaced(H)) return -1;
        if (pipe_prepare(H) || upload_pipe_issue(H)) return -1;
        H->uploaded = true;
        H->st.t_upload_s = 0;
        int rc3 = factor_impl(H, info, true, true);
        H->st.t_download_s = 0;
        return rc3;
    }
    if (slu_b200_upload(H)) return -1;
    int rc = factor_impl(H, info, true);   // downloads every level as soon as it is final
    H->st.t_download_s = 0;
    return rc;
}

// Device-side distribution (SURVEY 8f row N1): A arrives as host CSR (the caller's matrix, perm[old] = new as
// ScalePermstruct->perm_c after sp_colorder), is copied to HBM once (12 bytes per nonzero instead of 8 bytes per FACTOR
// entry; 20 instead of 16 in doublecomplex, where val holds (re, im) pairs) and scattered into the panels by a kernel --
// what pddistribute3d does on the host.  Replicated ancestors of other layers start at zero (dinit3DLUstructForest,
// pdgssvx3d.c:948).  Replaces slu_b200_upload.  On a batched handle (slu_b200_batch_fill_csr) val holds batch x nnz values,
// member-major.
static int fill_csr_impl(slu_b200_handle_t H, bool batched, int n, const int32_t *rowptr, const int32_t *colind, const double *val,
                         const int32_t *perm, const char *fn)
{
    if (!H || !rowptr || !colind || !val || !perm) return fail("null argument");
    if (check(H, fn, batched ? BATCHED : (UNBATCHED | GRID_Z))) return -1;
    if (n != H->n) return fail("%s: matrix order %d does not match the handle's %d", fn, n, H->n);
    double t0 = now_s();
    const int B = batched ? H->batch : 1;
    const int64_t nnz = rowptr[n];
    DevBuf<int32_t> drp, dci, dperm;
    DevBuf<val_t> dv;
    DevBuf<int8_t> dact;
    std::vector<int8_t> act(H->nsupers, 0);
    for (int zl = 0; zl < H->max_lvl; ++zl)      // the panels this layer holds (a batched handle has one level: znodes[0])
        if (batched || !H->my_zero[zl])
            for (int k : H->znodes[zl]) act[k] = 1;
    if (drp.alloc((size_t)n + 1) || dci.alloc((size_t)nnz) || dv.alloc((size_t)nnz * B) || dperm.alloc((size_t)n) || dact.upload(act))
        return -1;
    cudaStream_t s = H->stream;
    CU(cudaMemcpyAsync(drp.p, rowptr, ((size_t)n + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dci.p, colind, (size_t)nnz * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dv.p, val, (size_t)nnz * B * sizeof(val_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dperm.p, perm, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    if (values_replaced(H)) return -1;
    CU(cudaMemsetAsync(H->val.p, 0, H->val.bytes(), s));
    CU(cudaMemsetAsync(H->dev.err, 0, sizeof(int), s));
    if (batched) launch_fill_csr(H->bdev, n, drp.p, dci.p, dv.p, dperm.p, dact.p, H->dev.err, s);
    else launch_fill_csr(H->dev, n, drp.p, dci.p, dv.p, dperm.p, dact.p, H->dev.err, s);
    int bad = 0;
    CU(cudaMemcpyAsync(&bad, H->dev.err, sizeof(int), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    if (bad)
        return fail("%s: %d entries of %s have no slot in the L/U structure (wrong permutation or symbolic structure)", fn, bad,
                    batched ? "the members" : "A");
    H->st.t_upload_s = now_s() - t0;
    H->uploaded = true;
    return 0;
}

int slu_b200_fill_csr(slu_b200_handle_t H, int n, const int32_t *rowptr, const int32_t *colind, const double *val, const int32_t *perm)
{
    return fill_csr_impl(H, false, n, rowptr, colind, val, perm, SLU_API "fill_csr");
}

// Triangular solves on the resident factors (the job of pdgstrs3d, SRC/double/pdgstrs3d.c:6604, for factors that never
// left HBM).  Along Z: forward, the partial vectors climb the Z tree -- an all-reduce over the group of each level,
// after which only the group's owner layer keeps the vector (the reference reduces the ancestor contributions
// pairwise); backward, the owner's solution is spread to its group the same way (dbroadcastAncestor3d,
// pd3dcomm.c:1145); a last all-reduce of the owned pieces gives every rank the full solution.  In doublecomplex xh holds
// (re, im) pairs and n, ldx count complex elements; the all-reduces sum 2 * len doubles (a componentwise sum is the
// complex sum).
// trans = 1 / 2 solves A^T x = b / A^H x = b on the same factors: U^T forward, L^T backward, in the same level order and with
// the same all-reduces along Z, because the forward scatter and the backward gather reach ancestors only, as in the plain
// solve.

// One level of one pass: the diagonal solve and the update, in the order of the pass (forward: diagonal first).  The update
// streams the L panel (plain forward, transposed backward) or the U panel, tiled by sl_prefix / su_prefix.  A template for
// both handle kinds, hence outside the extern "C" block.
}  // extern "C"
template <class LU>
static int solve_level(const slu_b200_handle_s *H, const LU &d, const LevelPlan &L, bool backward, int trans, val_t *x, int n, int nrhs,
                       cudaStream_t s)
{
    const int32_t *nodes = H->d_pool_i32.p + L.nodes_off;
    const int64_t *p64 = H->d_pool_i64.p;
    const bool upanel = backward == (trans == 0);
    const Batch b{nodes, p64 + (upanel ? L.su_prefix : L.sl_prefix), L.count};
    int launches = 0;
    if (!backward) launches += launch_solve_diag(d, nodes, L.count, false, trans, x, n, nrhs, s);
    launches += launch_solve_update(d, b, upanel ? L.su_ctas : L.sl_ctas, backward, trans, x, n, nrhs, s);
    if (backward) launches += launch_solve_diag(d, nodes, L.count, true, trans, x, n, nrhs, s);
    return launches;
}

// The passes of a solve over the whole level plan: both for a solve; on a Schur handle the forward one alone is condense, the
// backward one expand.
enum { PASS_FORWARD = 1, PASS_BACKWARD = 2, PASS_BOTH = 3 };

// The passes on device LU d (H->dev, or H->bdev for every member of a batched handle) of a 1 x 1 x 1 grid, in place in d_x
// (one n x nrhs block per member).  Enqueued on H->stream, not synchronised.  Returns the kernel launches.
template <class LU>
static int solve_passes(slu_b200_handle_t H, const LU &d, int nrhs, int trans, int passes = PASS_BOTH)
{
    val_t *x = H->d_x.p;
    int launches = 0;
    if (passes & PASS_FORWARD)
        for (size_t li = 0; li < H->levels.size(); ++li)        // forward: L y = b (U^T y = b)
            launches += solve_level(H, d, H->levels[li], false, trans, x, H->n, nrhs, H->stream);
    if (passes & PASS_BACKWARD)
        for (size_t li = H->levels.size(); li-- > 0;)           // backward: U x = y (L^T x = y)
            launches += solve_level(H, d, H->levels[li], true, trans, x, H->n, nrhs, H->stream);
    return launches;
}
extern "C" {

// The solve of an unbatched handle on device vectors: b in d_x2 (n x nrhs, both buffers hold n * nrhs elements), the
// solution in *result (d_x, or d_x2 along Z) on every rank.  Enqueued on H->stream, not synchronised.  Returns the kernel
// launches, < 0 on an error.
static int solve_dev(slu_b200_handle_t H, int nrhs, int trans, val_t **result)
{
    const int n = H->n;
    const size_t len = (size_t)n * nrhs;
    cudaStream_t s = H->stream;
    const DeviceLU &d = H->dev;
    val_t *x = H->d_x.p, *x2 = H->d_x2.p;
    const bool multi = H->comm != nullptr;
    int launches = 0;
    auto forest_nodes = [&](int zl) { return H->d_pool_i32.p + H->z_nodes_off[zl]; };
    if (multi) {      // start from the entries this rank owns: b on the owner layer of every forest, 0 elsewhere
        CU(cudaMemsetAsync(x, 0, len * sizeof(val_t), s));
        for (int zl = 0; zl < H->max_lvl; ++zl)
            if (!H->my_zero[zl]) launches += launch_solve_mask(d, forest_nodes(zl), (int)H->znodes[zl].size(), x, n, nrhs, x2, s);
    } else {
        CU(cudaMemcpyAsync(x, x2, len * sizeof(val_t), cudaMemcpyDeviceToDevice, s));
    }
    // forward: L y = b (U^T y = b)
    size_t li = 0;
    for (int zl = 0; zl < H->max_lvl; ++zl) {
        if (multi && zl >= 1) {
            NC(g_nccl.AllReduce(x, x, len * VAL_DOUBLES, NCCL_FLOAT64, NCCL_SUM, H->gcomm[zl], s));
            if (H->my_zero[zl]) CU(cudaMemsetAsync(x, 0, len * sizeof(val_t), s));
        }
        for (; li < H->levels.size() && H->levels[li].zlvl <= zl; ++li) {
            const LevelPlan &L = H->levels[li];
            if (L.zlvl < zl || H->my_zero[zl]) continue;
            launches += solve_level(H, d, L, false, trans, x, n, nrhs, s);
        }
    }
    // backward: U x = y (L^T x = y)
    li = H->levels.size();
    for (int zl = H->max_lvl - 1; zl >= 0; --zl) {
        size_t lo = li;
        while (lo > 0 && H->levels[lo - 1].zlvl >= zl) --lo;
        if (!H->my_zero[zl])
            for (size_t q = li; q-- > lo;) {
                const LevelPlan &L = H->levels[q];
                if (L.zlvl != zl) continue;
                launches += solve_level(H, d, L, true, trans, x, n, nrhs, s);
            }
        li = lo;
        if (multi && zl >= 1) {
            if (H->my_zero[zl]) CU(cudaMemsetAsync(x, 0, len * sizeof(val_t), s));
            NC(g_nccl.AllReduce(x, x, len * VAL_DOUBLES, NCCL_FLOAT64, NCCL_SUM, H->gcomm[zl], s));
        }
    }
    *result = x;
    if (multi) {      // every rank contributes the entries it owns: the full solution everywhere
        CU(cudaMemsetAsync(x2, 0, len * sizeof(val_t), s));
        for (int zl = 0; zl < H->max_lvl; ++zl)
            if (!H->my_zero[zl]) launches += launch_solve_mask(d, forest_nodes(zl), (int)H->znodes[zl].size(), x2, n, nrhs, x, s);
        NC(g_nccl.AllReduce(x2, x2, len * VAL_DOUBLES, NCCL_FLOAT64, NCCL_SUM, H->comm, s));
        *result = x2;
    }
    return launches;
}

// x in A's ordering: b' = the row-permuted, scaled b into the solve's input (one scatter launch), the plain solve, x = the
// scaled, permuted-back solution (one gather launch).  trans 0: b'[rmap[i]] = R[i] b[i], x[j] = C[j] y[perm[j]]; trans 1 / 2:
// b'[perm[j]] = C[j] b[j], x[i] = R[i] y[rmap[i]] (the scalings are real, so F^H needs nothing more than F^T).
// Where solve_scaled_dev takes b: d_x2 on a batched handle, d_x on an unbatched one (the scatter writes b' where the plain
// solve takes its right-hand side)
static val_t *scaled_in(slu_b200_handle_t H, bool batched) { return batched ? H->d_x2.p : H->d_x.p; }

// The device part of solve_scaled: b in scaled_in(H), x in d_x2 (both buffers hold batch x n x nrhs).  Enqueued on H->stream,
// not synchronised.  Returns the kernel launches, < 0 on an error.
static int solve_scaled_dev(slu_b200_handle_t H, bool batched, int nrhs, int trans)
{
    const int B = batched ? H->batch : 1, n = H->n;
    cudaStream_t s = H->stream;
    val_t *in = scaled_in(H, batched), *b = batched ? H->d_x.p : H->d_x2.p;
    int launches = launch_permute_scale(b, in, trans ? H->d_cperm.p : H->d_rmap.p, trans ? H->d_C.p : H->d_R.p, n, nrhs, B, true, s);
    val_t *y = H->d_x.p;
    if (batched) {
        launches += solve_passes(H, H->bdev, nrhs, trans);
    } else {
        const int l = solve_dev(H, nrhs, trans, &y);
        if (l < 0) return -1;
        launches += l;
    }
    launches += launch_permute_scale(H->d_x2.p, y, trans ? H->d_rmap.p : H->d_cperm.p, trans ? H->d_R.p : H->d_C.p, n, nrhs, B, false, s);
    return launches;
}

// The checks of every solve on x (ldx >= n, nrhs columns per member), after null pointers: what the call needs of the handle
// (check), trans, nrhs / ldx and, where limit, n * nrhs below 2^31 per member
static int solve_check(slu_b200_handle_t H, const char *fn, unsigned need, int trans, int nrhs, int ldx, bool limit)
{
    if (check(H, fn, need)) return -1;
    if (trans < 0 || trans > 2) return fail("%s: trans = %d, must be 0 (A x = b), 1 (A^T x = b) or 2 (A^H x = b)", fn, trans);
    if (nrhs < 1 || ldx < H->n) return fail("%s: bad nrhs / ldx", fn);
    if (limit && (int64_t)H->n * nrhs > INT_MAX) return fail("%s: n * nrhs must stay below 2^31 per member", fn);
    return 0;
}

// The buffers solve_enqueue uses for len elements in all
static int solve_buffers(slu_b200_handle_t H, bool batched, bool scaled, size_t len, bool capturing, const char *fn)
{
    return grow(H, H->d_x, len, false, capturing, fn) || ((scaled || !batched) && grow(H, H->d_x2, len, false, capturing, fn)) ? -1 : 0;
}

// Every solve: b (one n x nrhs block per member at pitch ldb, in memory of `kind`'s source) copied where the device solve
// takes it, then that solve on H->stream: scaled, solve_scaled_dev (b in scaled_in, x in d_x2); the complete unbatched solve,
// solve_dev (b in d_x2, x where it says); else the passes in place in d_x.  Returns the kernel launches and points *x at the
// solution, < 0 on an error.
static int solve_enqueue(slu_b200_handle_t H, bool batched, bool scaled, int passes, const double *b, int ldb, int nrhs, int trans,
                         cudaMemcpyKind kind, val_t **x)
{
    const bool full = !scaled && !batched && passes == PASS_BOTH;
    const size_t w = (size_t)H->n * sizeof(val_t), cols = (size_t)nrhs * (batched ? H->batch : 1);
    *x = scaled ? H->d_x2.p : H->d_x.p;
    CU(cudaMemcpy2DAsync(scaled ? scaled_in(H, batched) : full ? H->d_x2.p : H->d_x.p, w, b, (size_t)ldb * sizeof(val_t), w, cols, kind,
                         H->stream));
    if (scaled) return solve_scaled_dev(H, batched, nrhs, trans);
    if (full) return solve_dev(H, nrhs, trans, x);
    return batched ? solve_passes(H, H->bdev, nrhs, trans, passes) : solve_passes(H, H->dev, nrhs, trans, passes);
}

// Every solve on host vectors: solve, solve_trans, solve_scaled (need has SCALED), schur_condense / expand and their batched
// twins (fn, with what they need of the handle).  x: one n x nrhs block per member (ldx >= n), block j at x + j * ldx * nrhs:
// b on entry, the result on return.
static int solve_host(slu_b200_handle_t H, const char *fn, unsigned need, double *xh, int ldx, int nrhs, int trans, int passes)
{
    if (!H || !xh) return fail("null argument");
    const bool batched = H->batch > 0, scaled = (need & SCALED) != 0;
    if (solve_check(H, fn, need, trans, nrhs, ldx, batched || scaled)) return -1;
    const int B = batched ? H->batch : 1, n = H->n;
    if (solve_buffers(H, batched, scaled, (size_t)n * nrhs * B, false, fn)) return -1;
    cudaStream_t s = H->stream;
    double t0 = now_s();
    val_t *result = nullptr;
    // the blocks are B * nrhs columns at pitch ldx: one 2D copy each way
    const int launches = solve_enqueue(H, batched, scaled, passes, xh, ldx, nrhs, trans, cudaMemcpyHostToDevice, &result);
    if (launches < 0) return -1;
    CU(cudaMemcpy2DAsync(xh, (size_t)ldx * sizeof(val_t), result, (size_t)n * sizeof(val_t), (size_t)n * sizeof(val_t), (size_t)nrhs * B,
                         cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    H->st.reserved[4] = now_s() - t0;      // seconds of the last solve (H2D of b and D2H of x included)
    H->st.reserved[5] = (double)launches;
    return 0;
}

int slu_b200_solve(slu_b200_handle_t H, double *xh, int ldx, int nrhs)
{
    return solve_host(H, SLU_API "solve", UNBATCHED | NOT_SCHUR | GRID_SOLVE | FACTORED, xh, ldx, nrhs, 0, PASS_BOTH);
}

int slu_b200_solve_trans(slu_b200_handle_t H, double *xh, int ldx, int nrhs, int trans)
{
    return solve_host(H, SLU_API "solve_trans", UNBATCHED | NOT_SCHUR | GRID_SOLVE | FACTORED, xh, ldx, nrhs, trans, PASS_BOTH);
}

#ifndef SLU_COMPLEX
// ---- benchmark support (SURVEY 8a row a10: the reference's GPU Schur path is "to be beaten") ------------------------
// Export what an EXTERNAL baseline needs to redo one level's Schur updates on this handle's device data: the DeviceLU
// struct (device pointers) and the ids of the level's supernodes with a big (>= 96 x 96) update.  oracle/ref_gpu_schur.cu
// uses it to time cublasDgemm into a bigV buffer + a restatement of the reference's Scatter_GPU_kernel on exactly the
// same operands; slu_b200_k_rerun_schur times this library's fused kernel on them.
int slu_b200_k_level_export(slu_b200_handle_t H, int level, void *device_lu, int device_lu_bytes, int32_t *nodes, int max_nodes)
{
    if (!H || level < 0 || level >= (int)H->levels.size()) return fail("bad handle / level");
    if (check(H, "slu_b200_k_level_export", UNBATCHED | NOT_SCHUR)) return -1;
    if (device_lu && device_lu_bytes == (int)sizeof(DeviceLU)) memcpy(device_lu, &H->dev, sizeof(DeviceLU));
    else if (device_lu) return fail("DeviceLU is %d bytes", (int)sizeof(DeviceLU));
    const LevelPlan &L = H->levels[level];
    int cnt = 0;
    for (int pass = 0; pass < 2; ++pass) {
        const int64_t off = pass ? L.tc_nodes : L.big_nodes;
        const int c = pass ? L.tc_count : L.big_count;
        for (int t = 0; t < c; ++t, ++cnt)
            if (nodes && cnt < max_nodes) nodes[cnt] = H->h_pool_i32[off + t];
    }
    return cnt;
}
// Re-run the destination maps + the fused Schur kernels of one level `reps` times on whatever the arena holds (timing
// only: the values are updated again and again); *ms = mean device time of the Schur launches of the level.
int slu_b200_k_rerun_schur(slu_b200_handle_t H, int level, int reps, float *ms)
{
    if (!H || level < 0 || level >= (int)H->levels.size() || reps < 1 || !ms) return fail("bad argument");
    if (check(H, "slu_b200_k_rerun_schur", UNBATCHED | NOT_SCHUR)) return -1;
    const LevelPlan &L = H->levels[level];
    cudaStream_t s = H->stream;
    const DeviceLU &d = H->dev;
    const int32_t *nodes = H->d_pool_i32.p + L.nodes_off;
    const int64_t *p64 = H->d_pool_i64.p;
    EventSet ev;
    if (ev.create()) return fail("cannot create events");
    launch_schur_setup(d, Batch{nodes, p64 + L.setup_prefix, L.count}, L.setup_ctas, s);
    const int32_t *tcn = H->d_pool_i32.p + L.tc_nodes;
    if (L.tc_count > 0)
        launch_oz_slice(d, tcn, L.tc_count, p64 + L.tc_p_rt, L.tc_n_rt, p64 + L.tc_p_ak, L.tc_n_ak, p64 + L.tc_p_b, L.tc_n_b, H->tc_slices, s);
    for (int r = -1; r < reps; ++r) {
        if (r == 0) CU(cudaEventRecord(ev[0], s));
        launch_oz_schur(d, Batch{tcn, p64 + L.tc_prefix, L.tc_count}, L.tc_ctas, 0, 1, 0, H->tc_slices, s);
        launch_schur(d, Batch{H->d_pool_i32.p + L.big_nodes, p64 + L.big_prefix, L.big_count}, L.big_ctas, 1, 0, 1, 0, s);
    }
    CU(cudaEventRecord(ev[1], s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    float t = 0;
    CU(cudaEventElapsedTime(&t, ev[0], ev[1]));
    *ms = t / reps;
    return 0;
}
#endif  // !SLU_COMPLEX

// ---- selected inversion and log-determinant on the resident factors ------------------------------------------------
// slu_selinv.cu holds the kernels and the recurrences (slu_selinv_z.cu the doublecomplex build).  The sweep walks the
// level plan top-down (the backward solve's order): every Schur destination of a supernode lies in a supernode of a later
// level, so its gathered block M = H(R, C) is final.  Per level 7 launches: the destination maps and the 16x16
// diagonal-block inverses are rebuilt in the factorization's per-level workspaces, then three products and two
// triangular solves; a level with no Schur update (the root) has no maps to build and makes 6.

// CTA prefixes of the selinv kernels, from the level plan: built once per handle.  Product tiles are SELINV_TILE_M rows
// by SELINV_TILE_N val_t columns (64 x 64 real outputs: 32 complex columns in doublecomplex).
static int selinv_plan(slu_b200_handle_s *H)
{
    std::vector<int64_t> pool;
    H->si_levels.assign(H->levels.size(), SelinvLevel{});
    auto tr = [](int64_t a) { return (a + SELINV_TILE_M - 1) / SELINV_TILE_M; };
    auto tc = [](int64_t a) { return (a + SELINV_TILE_N - 1) / SELINV_TILE_N; };
    for (size_t li = 0; li < H->levels.size(); ++li) {
        const LevelPlan &L = H->levels[li];
        SelinvLevel &S = H->si_levels[li];
        std::vector<int64_t> p[5];
        for (auto &v : p) v.assign(1, 0);
        for (int t = 0; t < L.count; ++t) {
            const NodeDesc &nd = H->nodes[H->h_pool_i32[L.nodes_off + t]];
            p[0].push_back(p[0].back() + tr(nd.m) * tc(nd.ns));
            p[1].push_back(p[1].back() + tr(nd.ns) * tc(nd.ncols));
            p[2].push_back(p[2].back() + tr(nd.ns) * tc(nd.ns));
            p[3].push_back(p[3].back() + (nd.nsupr + SELINV_VECS - 1) / SELINV_VECS);
            p[4].push_back(p[4].back() + (nd.ns + nd.ncols + SELINV_VECS - 1) / SELINV_VECS);
        }
        for (int q = 0; q < 5; ++q) {
            if (p[q].back() > 2147483647LL) return fail(SLU_API "selinv: a level needs more than 2^31 CTAs in one launch");
            int64_t &off = q < 3 ? S.gemm_prefix[q] : S.trsm_prefix[q - 3];
            int64_t &ctas = q < 3 ? S.gemm_ctas[q] : S.trsm_ctas[q - 3];
            off = (int64_t)pool.size();
            ctas = p[q].back();
            pool.insert(pool.end(), p[q].begin(), p[q].end());
        }
    }
    return H->d_si_pool.upload(pool);
}

// The plan and the second arena, on the first selected inversion of the handle (allocates)
static int selinv_alloc(slu_b200_handle_t H, int members, const char *fn)
{
    if (H->si_levels.empty() && selinv_plan(H)) return -1;
    if (!H->d_hinv.p && H->d_hinv.alloc((size_t)H->member_len * members)) {
        cudaGetLastError();
        std::string why = g_err;
        H->d_hinv.release();
        return fail("%s: the inverse needs a second arena of %.2f GB beside the factors, which does not fit (%s); "
                    "the factors are unchanged", fn, 1e-9 * sizeof(val_t) * H->member_len * members, why.c_str());
    }
    return 0;
}
}  // extern "C"

// The sweep's launches on H->stream, dev.err counting the missed destinations -> the launches; *flops as selinv's out[1] for
// one member
template <class LU>
static int selinv_enqueue(slu_b200_handle_t H, const LU &d, double *flops)
{
    cudaStream_t s = H->stream;
    const int64_t *p64 = H->d_pool_i64.p, *sp = H->d_si_pool.p;
    val_t *hv = H->d_hinv.p;
    int launches = 0;
    CU(cudaMemsetAsync(H->dev.err, 0, sizeof(int), s));
    for (size_t li = H->levels.size(); li-- > 0;) {
        const LevelPlan &L = H->levels[li];
        const SelinvLevel &S = H->si_levels[li];
        const int32_t *nodes = H->d_pool_i32.p + L.nodes_off;
        launches += launch_schur_setup(H->dev, Batch{nodes, p64 + L.setup_prefix, L.count}, L.setup_ctas, s);
        launches += launch_diag_inv(d, Batch{nodes, p64 + L.inv_prefix, L.count}, L.inv_ctas, H->d_inv.p, s);
        for (int q = 0; q < 3; ++q) launches += launch_selinv_gemm(d, Batch{nodes, sp + S.gemm_prefix[q], L.count}, S.gemm_ctas[q], q, hv, s);
        for (int q = 0; q < 2; ++q)
            launches += launch_selinv_trsm(d, Batch{nodes, sp + S.trsm_prefix[q], L.count}, S.trsm_ctas[q], q, H->d_inv.p, hv, s);
        // 2 flops per multiply-add in both precisions (a complex multiply-add counts once, as ops_fact counts the complex
        // Schur update): 4x this in real flops in doublecomplex
        for (int t = 0; t < L.count; ++t) {
            const NodeDesc &nd = H->nodes[H->h_pool_i32[L.nodes_off + t]];
            const double m = nd.m, n = nd.ncols, ns = nd.ns;
            *flops += 4.0 * m * n * ns + 2.0 * m * ns * ns + (nd.nsupr + ns + n) * ns * ns;
        }
    }
    return launches;
}

// The sweep on device LU d (H->dev, or H->bdev for every member of a batched handle: the same launches with gridDim.y =
// members), then a wait for the missed-destination count.  The destination maps are value-independent and built on H->dev
// for all members, as in slu_b200_batch_factor.  fn names the call in the messages.
template <class LU>
static int selinv_sweep(slu_b200_handle_t H, const LU &d, int members, const char *fn, double out[4])
{
    H->si_ready = false;
    H->si_dev = false;
    if (selinv_alloc(H, members, fn)) return -1;
    cudaStream_t s = H->stream;
    double flops = 0;
    const double t0 = now_s();
    const int launches = selinv_enqueue(H, d, &flops);
    if (launches < 0) return -1;
    int bad = 0;
    CU(cudaMemcpyAsync(&bad, H->dev.err, sizeof(int), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    if (bad) return fail("%s: %d Schur-update destinations were not found in the L/U structure", fn, bad);
    H->si_ready = true;
    H->si_epoch = H->epoch;                // selinv's check settled the handle: the factorizations counted so far
    if (out) {
        out[0] = now_s() - t0;
        out[1] = flops * members;
        out[2] = (double)launches;
        out[3] = (double)(H->d_hinv.bytes() + H->d_si_pool.bytes());
    }
    return 0;
}
extern "C" {

int slu_b200_selinv(slu_b200_handle_t H, double out[4])
{
    if (!H) return fail("null handle");
    if (check(H, SLU_API "selinv", UNBATCHED | NOT_SCHUR | GRID_1 | FACTORED)) return -1;
    return selinv_sweep(H, H->dev, 1, SLU_API "selinv", out);
}

// The entries of A^-1 on A's pattern from the inverse of the last selinv, for every member (one on an unbatched handle):
// out holds members x nnz values, member j's at out + j * nnz.  need: what the call (fn) needs of the handle.
static int selinv_get_impl(slu_b200_handle_t H, const char *fn, unsigned need, int n, const int32_t *rowptr, const int32_t *colind,
                           const int32_t *perm, double *out)
{
    if (!H || !rowptr || !colind || !perm || !out) return fail("null argument");
    if (check(H, fn, need)) return -1;
    if (n != H->n) return fail("%s: matrix order %d does not match the handle's %d", fn, n, H->n);
    const int64_t nnz = rowptr[n];
    if (rowptr[0] != 0 || nnz < 0) return fail("%s: bad rowptr", fn);
    const int B = H->batch ? H->batch : 1;
    DevBuf<int32_t> drp, dci, dperm;
    DevBuf<val_t> dout;
    if (drp.alloc((size_t)n + 1) || dci.alloc((size_t)nnz) || dperm.alloc((size_t)n) || dout.alloc((size_t)nnz * B)) return -1;
    cudaStream_t s = H->stream;
    CU(cudaMemcpyAsync(drp.p, rowptr, ((size_t)n + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dci.p, colind, (size_t)nnz * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dperm.p, perm, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(H->dev.err, 0, sizeof(int), s));
    if (H->batch) launch_selinv_get(H->bdev, H->d_hinv.p, n, drp.p, dci.p, dperm.p, dout.p, H->dev.err, s);
    else launch_selinv_get(H->dev, H->d_hinv.p, n, drp.p, dci.p, dperm.p, dout.p, H->dev.err, s);
    int bad = 0;
    CU(cudaMemcpyAsync(out, dout.p, (size_t)nnz * B * sizeof(val_t), cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(&bad, H->dev.err, sizeof(int), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    if (bad) return fail("%s: %d entries have no slot in the L/U structure (A^-1 is known on the pattern of L+U only)", fn, bad);
    return 0;
}

int slu_b200_selinv_get(slu_b200_handle_t H, int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm, double *out)
{
    return selinv_get_impl(H, SLU_API "selinv_get", UNBATCHED | NOT_SCHUR | GRID_1 | FACTORED | SI_READY, n, rowptr, colind, perm, out);
}

// log |det| and the sign of every member (one on an unbatched handle): logabs[members]; sign[members] (double) or
// sign[2 * members] = exp(i theta_j) as (re, im) pairs (doublecomplex).  need: what the call (fn) needs of the handle.
static int logdet_impl(slu_b200_handle_t H, const char *fn, unsigned need, double *logabs, double *sign)
{
    if (!H || !logabs || !sign) return fail("null argument");
    if (check(H, fn, need)) return -1;
    const int B = H->batch ? H->batch : 1;
    const int count = (int)H->znodes[0].size();
    const int nparts = (count + SELINV_VECS - 1) / SELINV_VECS;
    DevBuf<double> part, res;
    DevBuf<phase_t> ph;
    if (part.alloc((size_t)nparts * B) || ph.alloc((size_t)nparts * B) || res.alloc((size_t)(1 + VAL_DOUBLES) * B)) return -1;
    cudaStream_t s = H->stream;
    const int32_t *nodes = H->d_pool_i32.p + H->z_nodes_off[0];
    if (H->batch) launch_selinv_logdet(H->bdev, nodes, count, part.p, ph.p, res.p, s);
    else launch_selinv_logdet(H->dev, nodes, count, part.p, ph.p, res.p, s);
    std::vector<double> r((size_t)(1 + VAL_DOUBLES) * B, 0.0);
    for (int j = 0; j < B; ++j) r[(size_t)j * (1 + VAL_DOUBLES) + 1] = 1.0;   // no supernode: log |det| 0, sign 1
    if (nparts > 0) CU(cudaMemcpyAsync(r.data(), res.p, r.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    for (int j = 0; j < B; ++j) {
        logabs[j] = r[(size_t)j * (1 + VAL_DOUBLES)];
        for (int c = 0; c < VAL_DOUBLES; ++c) sign[(size_t)j * VAL_DOUBLES + c] = r[(size_t)j * (1 + VAL_DOUBLES) + 1 + c];
    }
    return 0;
}

int slu_b200_logdet(slu_b200_handle_t H, double *logabs, double *sign)
{
    return logdet_impl(H, SLU_API "logdet", UNBATCHED | NOT_SCHUR | GRID_1 | FACTORED, logabs, sign);
}

// ---- partial factorization: the Schur complement and the two partial solves ------------------------------------------
// A Schur handle is an ordinary one whose level plan leaves out the supernodes of the last nschur columns (analyze).  The
// factorization then eliminates A11 only; every Schur update of the eliminated part still lands in the Schur panels, which
// start as A22 and end as S = A22 - A21 A11^-1 A12 on the symbolic pattern.  The forward pass of the solve over the same
// plan is condense (its update scatter subtracts L21 y1 from the Schur rows), the backward pass with x2 in the Schur
// positions is expand.
int slu_b200_schur_create(slu_b200_handle_t *out, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, int nschur)
{
    if (!out || !lu || !opt) return fail("null argument");
    *out = nullptr;
    if (nschur < 1 || nschur >= lu->n)
        return fail(SLU_API "schur_create: nschur = %d, must satisfy 1 <= nschur < n = %d", nschur, lu->n);
    return create_impl(out, lu, opt, 0, nschur);
}

// S of every member (one on an unbatched handle) into the host array S: member j's s x s block at S + j * lds * s.  The
// caller has checked the handle.
static int schur_get_impl(slu_b200_handle_t H, double *S, int lds, const char *fn)
{
    const int s = H->nschur, B = H->batch ? H->batch : 1;
    if (lds < s) return fail("%s: lds = %d, must be >= nschur = %d", fn, lds, s);
    const double t0 = now_s();
    const size_t elems = (size_t)s * s * B;
    if (!H->d_S.p && H->d_S.alloc(elems)) {
        const std::string why = g_err;
        H->d_S.release();
        cudaGetLastError();
        if (H->batch)
            return fail("%s: the %d Schur complements of %d x %d need %.2f GB of HBM: %s", fn, B, s, s,
                        1e-9 * (double)(elems * sizeof(val_t)), why.c_str());
        return fail("%s: the %d x %d Schur complement needs %.2f GB of HBM: %s", fn, s, s, 1e-9 * (double)(elems * sizeof(val_t)),
                    why.c_str());
    }
    EventSet ev;
    if (ev.create()) return fail("cannot create events");
    cudaStream_t st = H->stream;
    CU(cudaMemsetAsync(H->d_S.p, 0, elems * sizeof(val_t), st));
    CU(cudaEventRecord(ev[0], st));
    if (H->batch) launch_schur_gather(H->bdev, H->d_sunits.p, (int64_t)H->d_sunits.n, H->schur_first, s, H->d_S.p, st);
    else launch_schur_gather(H->dev, H->d_sunits.p, (int64_t)H->d_sunits.n, H->schur_first, s, H->d_S.p, st);
    CU(cudaEventRecord(ev[1], st));
    if (lds == s)   // one contiguous copy
        CU(cudaMemcpyAsync(S, H->d_S.p, elems * sizeof(val_t), cudaMemcpyDeviceToHost, st));
    else            // the B blocks are B * s columns at pitch lds
        CU(cudaMemcpy2DAsync(S, (size_t)lds * sizeof(val_t), H->d_S.p, (size_t)s * sizeof(val_t), (size_t)s * sizeof(val_t),
                             (size_t)s * B, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    float ms = 0;
    CU(cudaEventElapsedTime(&ms, ev[0], ev[1]));
    H->st.reserved[6] = now_s() - t0;      // seconds of the call
    H->st.reserved[7] = ms;                // device milliseconds of the gather kernel
    return 0;
}

int slu_b200_schur_get(slu_b200_handle_t H, double *S, int lds)
{
    if (!H || !S) return fail("null argument");
    const char *fn = SLU_API "schur_get";
    if (check(H, fn, UNBATCHED | SCHUR | FACTORED)) return -1;
    return schur_get_impl(H, S, lds, fn);
}

// condense: the forward pass over the plan; expand: the backward pass.  x: host, n x nrhs (ldx >= n), ordering of F.
int slu_b200_schur_condense(slu_b200_handle_t H, double *x, int ldx, int nrhs)
{
    return solve_host(H, SLU_API "schur_condense", UNBATCHED | SCHUR | FACTORED, x, ldx, nrhs, 0, PASS_FORWARD);
}

int slu_b200_schur_expand(slu_b200_handle_t H, double *x, int ldx, int nrhs)
{
    return solve_host(H, SLU_API "schur_expand", UNBATCHED | SCHUR | FACTORED, x, ldx, nrhs, 0, PASS_BACKWARD);
}

// ---- batched handles: many matrices of one sparsity pattern (pdgssvx3d_csc_batch, SRC/double/pdgssvx3d_csc_batch.c:81,
// and its doublecomplex twin pzgssvx3d_csc_batch, SRC/complex16/pzgssvx3d_csc_batch.c:80; dsparseTreeFactorBatchGPU,
// SRC/CplusplusFactor/batch_factorize.cu:801) ----------------------------------------------------------------------------
// Everything the analysis builds is value-independent and shared by the members: the level plan and CTA prefixes, NodeDesc,
// the LBlk/UBlk tables, the look-ahead split and the RowInfo/ColInfo/lrel/urel maps (built once per level by
// schur_setup_kernel).  Each member has its own value arena, d_inv slice and info flag; every batched launch is the
// unbatched one with gridDim.y = members, so a batched factorization takes exactly as many launches as one matrix.

// the checks of batch_create and batch_schur_create (fn) before create_impl
static int batch_create_check(const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, int batch, const char *fn)
{
    if (batch < 1 || batch > 65535) return fail("%s: batch = %d, must be 1 ... 65535", fn, batch);
    if (lu->nprow != 1 || lu->npcol != 1 || lu->npdep != 1)
        return fail("%s: batched handles need a 1 x 1 x 1 grid (got %d x %d x %d)", fn, lu->nprow, lu->npcol, lu->npdep);
    if (opt->world_size > 1) return fail("%s: batched handles are single-GPU (world_size = %d)", fn, opt->world_size);
    return 0;
}

int slu_b200_batch_create(slu_b200_handle_t *out, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, int batch)
{
    if (!out || !lu || !opt) return fail("null argument");
    *out = nullptr;
    if (batch_create_check(lu, opt, batch, SLU_API "batch_create")) return -1;
    return create_impl(out, lu, opt, batch);
}

// rowptr / colind / perm as slu_b200_fill_csr, shared by the members; val = batch x nnz values, member-major
int slu_b200_batch_fill_csr(slu_b200_handle_t H, int n, const int32_t *rowptr, const int32_t *colind, const double *val,
                            const int32_t *perm)
{
    return fill_csr_impl(H, true, n, rowptr, colind, val, perm, SLU_API "batch_fill_csr");
}

// factor_impl's level loop on a 1 x 1 x 1 grid, every launch over all members (look-ahead streams and events as there:
// the members advance in lockstep).  The destination maps are value-independent: one schur_setup launch per level.
int slu_b200_batch_factor(slu_b200_handle_t H, int *info)
{
    if (!H || !info) return fail("null argument");
    if (check(H, SLU_API "batch_factor", BATCHED | UPLOADED)) return -1;
    if (factors_replaced(H)) return -1;
    const int B = H->batch;
    cudaStream_t s = H->stream;
    std::vector<int> flags(B + 1, INT_MAX);
    flags[B] = 0;
    CU(cudaMemcpyAsync(H->d_flags.p, flags.data(), flags.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(H->d_tiny.p, 0, sizeof(unsigned long long), s));
    CU(cudaStreamSynchronize(s));   // `flags` is pageable host memory reused below
    CU(cudaEventRecord(H->ev0, s));
    const int64_t launches = factor_levels(H, H->bdev, false, false, false);
    if (launches < 0) return -1;
    CU(cudaEventRecord(H->ev1, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    float ms = 0;
    CU(cudaEventElapsedTime(&ms, H->ev0, H->ev1));
    H->st.t_factor_s = ms * 1e-3;
    H->st.gpu_launches = launches;
    unsigned long long tiny = 0;
    CU(cudaMemcpy(flags.data(), H->d_flags.p, flags.size() * sizeof(int), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&tiny, H->d_tiny.p, sizeof tiny, cudaMemcpyDeviceToHost));
    H->st.tiny_pivots = (int64_t)tiny;   // summed over the members
    if (flags[B]) return fail("%d Schur-update destinations were not found in the L/U structure", flags[B]);
    for (int j = 0; j < B; ++j) info[j] = H->member_info[j] = flags[j] == INT_MAX ? 0 : flags[j];
    CU(cudaMemcpy(H->d_info.p, H->member_info.data(), (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice));
    return 0;
}

int slu_b200_batch_solve(slu_b200_handle_t H, double *xh, int ldx, int nrhs)
{
    return solve_host(H, SLU_API "batch_solve", BATCHED | NOT_SCHUR | FACTORED, xh, ldx, nrhs, 0, PASS_BOTH);
}

int slu_b200_batch_solve_trans(slu_b200_handle_t H, double *xh, int ldx, int nrhs, int trans)
{
    return solve_host(H, SLU_API "batch_solve_trans", BATCHED | NOT_SCHUR | FACTORED, xh, ldx, nrhs, trans, PASS_BOTH);
}

// ---- condition estimation on the resident factors (LAPACK dgecon / zgecon, sequential SuperLU dgscon / zgscon) --------
// dlacn2 / zlacn2 estimate ||B||_1 for B = F^-1 (norm '1') or B = F^-T / F^-H (norm 'I'), F = P A P^T, by reverse
// communication: "kase 1" asks for B x, "kase 2" for B^T x (B^H x).  Each round here is one solve of every member on
// device vectors (solve_dev / solve_passes, exactly the launches of a solve) and the step kernels of slu_cond.cu; the
// host only reads back how many members wait for kase 1 and for kase 2.  The next round takes the kase other than the
// last one if any member waits for it, else the same one: with one member these are exactly dlacn2's solves, and in a
// batch no member waits more than one round.
// Where the next vectors live: a batched handle keeps every member's pending vector in d_cv, because a member whose kase
// is not the round's must keep it; each round copies d_cv into d_x, where the batched solve runs in place.  An unbatched
// handle's one member takes every round, so its step kernels write the next vector straight into d_x2, where solve_dev
// takes its right-hand side (in place over the solution along Z, where the solve ends in d_x2).
constexpr int COND_MAX_ROUNDS = 64;     // dlacn2 makes at most 11 solves; lock-step at most doubles that

}  // extern "C"
// The estimator's buffers for `members` vectors of n elements (pinned once a call on the caller's stream was captured: grow)
static int cond_buffers(slu_b200_handle_t H, int n, int members, bool capturing, const char *fn)
{
    const size_t len = (size_t)n * members;
    const size_t parts = (size_t)((n + COND_CHUNK - 1) / COND_CHUNK) * members;
    if (VAL_DOUBLES == 1 && grow_loop(H, H->d_csgn, len, capturing, fn)) return -1;     // the real repeated-sign test
    if (grow_loop(H, H->d_cstate, members, capturing, fn) || grow_loop(H, H->d_cpart, parts, capturing, fn) ||
        grow_loop(H, H->d_ccount, 2, capturing, fn))
        return -1;
    return 0;
}

// The rounds of dlacn2 / zlacn2 over `members` vectors of n elements, shared by gscon and the forward error bound of gsrfs:
// v holds the pending vectors; apply(kase, &x) enqueues the operator of kase on them, points x at the result and returns its
// launches (< 0 on an error).  Ends when no member waits; the estimates are then in d_cstate.  *rounds counts the
// applications.  Returns the launches of the applications, < 0 on an error.
template <class Apply>
static int cond_rounds(slu_b200_handle_t H, int n, int members, val_t *v, Apply apply, int *rounds, const char *fn)
{
    if (cond_buffers(H, n, members, false, fn)) return -1;
    cudaStream_t s = H->stream;
    launch_cond_init(H->d_cstate.p, v, n, members, s);
    int launches = 0;
    for (int kase = 1;;) {
        if (*rounds == COND_MAX_ROUNDS) return fail("%s: the estimator did not finish in %d solves", fn, *rounds);
        val_t *x = nullptr;
        const int l = apply(kase, &x);
        if (l < 0) return -1;
        launches += l;
        CU(cudaMemsetAsync(H->d_ccount.p, 0, 2 * sizeof(int), s));
        launch_cond_step(H->d_cstate.p, kase, x, v, H->d_csgn.p, H->d_cpart.p, H->d_ccount.p, n, members, s);
        int waiting[2] = {0, 0};                      // members waiting for kase 1 / kase 2
        CU(cudaMemcpyAsync(waiting, H->d_ccount.p, sizeof waiting, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        ++*rounds;
        if (waiting[2 - kase] > 0) kase = 3 - kase;
        else if (waiting[kase - 1] == 0) break;
    }
    CU(cudaGetLastError());
    return launches;
}

// gscon's buffers: the solve's, the pending vectors (gscon_v), the estimator's, anorm and rcond of every member
static int gscon_buffers(slu_b200_handle_t H, bool batched, bool capturing, const char *fn)
{
    const int B = batched ? H->batch : 1;
    const size_t len = (size_t)H->n * B;
    return grow(H, H->d_x, len, false, capturing, fn) || (batched ? grow_loop(H, H->d_cv, len, capturing, fn) : grow(H, H->d_x2, len, false, capturing, fn)) ||
           cond_buffers(H, H->n, B, capturing, fn) || grow_loop(H, H->d_canorm, B, capturing, fn) || grow_loop(H, H->d_crcond, B, capturing, fn) ? -1 : 0;
}

// gscon's pending vectors
static val_t *gscon_v(slu_b200_handle_t H, bool batched) { return batched ? H->d_cv.p : H->d_x2.p; }

// gscon's operator for cond_rounds and cond_loop: the solve of kase (kase 1 with F for norm '1', with F^T / F^H for 'I'; kase
// 2 the other) of every member's pending vector, the result in *x.  Returns the launches, < 0 on an error.
static int gscon_apply(slu_b200_handle_t H, bool batched, bool one, int kase, val_t **x)
{
    const int trans = (kase == 1) == one ? 0 : (VAL_DOUBLES == 2 ? 2 : 1);
    *x = H->d_x.p;
    if (!batched) return solve_dev(H, 1, trans, x);
    CU(cudaMemcpyAsync(*x, H->d_cv.p, (size_t)H->n * H->batch * sizeof(val_t), cudaMemcpyDeviceToDevice, H->stream));
    return solve_passes(H, H->bdev, 1, trans);
}
extern "C" {

// the preconditions of the matching solve are checked by the caller; B = 1 member on an unbatched handle.  rcond from
// cond_rcond_kernel, as gscon_device's.
static int gscon_impl(slu_b200_handle_t H, char norm, const double *anorm, double *rcond, const char *fn)
{
    const bool batched = H->batch > 0;
    const int B = batched ? H->batch : 1, n = H->n;
    const bool one = norm == '1' || norm == 'O' || norm == 'o';
    if (!one && norm != 'I' && norm != 'i')
        return fail("%s: norm must be '1', 'O' or 'I' (got character code %d)", fn, (int)(unsigned char)norm);
    for (int j = 0; j < B; ++j) {
        if (anorm[j] >= 0.0) continue;
        if (batched) return fail("%s: anorm[%d] = %g, must be >= 0", fn, j, anorm[j]);
        return fail("%s: anorm = %g, must be >= 0", fn, anorm[j]);
    }
    const double t0 = now_s();
    int rounds = 0;
    bool any = false;
    for (int j = 0; j < B; ++j) {
        rcond[j] = 0.0;                                   // anorm 0 or +inf: rcond 0 without a solve
        any = any || (anorm[j] > 0.0 && std::isfinite(anorm[j]));
    }
    if (any) {
        if (gscon_buffers(H, batched, false, fn)) return -1;
        cudaStream_t s = H->stream;
        CU(cudaMemcpyAsync(H->d_canorm.p, anorm, (size_t)B * sizeof(double), cudaMemcpyHostToDevice, s));
        auto apply = [&](int kase, val_t **x) { return gscon_apply(H, batched, one, kase, x); };
        if (cond_rounds(H, n, B, gscon_v(H, batched), apply, &rounds, fn) < 0) return -1;
        launch_cond_rcond(H->d_cstate.p, H->d_canorm.p, H->d_info.p, B, H->d_crcond.p, s);
        CU(cudaMemcpyAsync(rcond, H->d_crcond.p, (size_t)B * sizeof(double), cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        CU(cudaGetLastError());
    }
    H->st.reserved[6] = now_s() - t0;
    H->st.reserved[7] = (double)rounds;
    return 0;
}

int slu_b200_gscon(slu_b200_handle_t H, char norm, double anorm, double *rcond)
{
    if (!H || !rcond) return fail("null argument");
    if (check(H, SLU_API "gscon", UNBATCHED | NOT_SCHUR | GRID_SOLVE | FACTORED)) return -1;
    return gscon_impl(H, norm, &anorm, rcond, SLU_API "gscon");
}

int slu_b200_batch_gscon(slu_b200_handle_t H, char norm, const double *anorm, double *rcond)
{
    if (!H || !anorm || !rcond) return fail("null argument");
    if (check(H, SLU_API "batch_gscon", BATCHED | NOT_SCHUR | FACTORED)) return -1;
    return gscon_impl(H, norm, anorm, rcond, SLU_API "batch_gscon");
}

// D2H of member `member`'s L and U into the view's Lnzval / Unzval, as slu_b200_download
int slu_b200_batch_download(slu_b200_handle_t H, int member)
{
    if (!H) return fail("null handle");
    if (check(H, SLU_API "batch_download", BATCHED)) return -1;
    if (member < 0 || member >= H->batch) return fail(SLU_API "batch_download: member %d out of range (batch of %d)", member, H->batch);
    double t0 = now_s();
    if (transfer(H, false, member)) return -1;
    H->st.t_download_s = now_s() - t0;
    return 0;
}

// ---- selected inversion and log-determinants on batched handles: selinv_sweep over H->bdev, so the sweep makes exactly the
// launches of one unbatched sweep, each over every member (gridDim.y = member).  The H arena holds `batch` member arenas,
// member_len elements apart as the members' factors are.
int slu_b200_batch_selinv(slu_b200_handle_t H, double out[4])
{
    if (!H) return fail("null handle");
    if (check(H, SLU_API "batch_selinv", BATCHED | NOT_SCHUR | FACTORED)) return -1;
    return selinv_sweep(H, H->bdev, H->batch, SLU_API "batch_selinv", out);
}

int slu_b200_batch_selinv_get(slu_b200_handle_t H, int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm,
                              double *out)
{
    return selinv_get_impl(H, SLU_API "batch_selinv_get", BATCHED | NOT_SCHUR | FACTORED | SI_READY, n, rowptr, colind, perm, out);
}

int slu_b200_batch_logdet(slu_b200_handle_t H, double *logabs, double *sign)
{
    return logdet_impl(H, SLU_API "batch_logdet", BATCHED | NOT_SCHUR | FACTORED, logabs, sign);
}

// ---- inertia from the signs of the pivots (slu_b200_inertia, slu_b200_batch_inertia) --------------------------------------
// F = P A P^T = L U with a symmetric permutation, no row exchanges and a unit-diagonal L: for a real symmetric (complex
// Hermitian) A, U = D L^T (D L^H), so by Sylvester's law the signs of the u_ii are those of A's eigenvalues.  Two launches
// over the level plan's supernodes for all members (d = H->dev, or H->bdev with gridDim.y = members); counts[3 j + c] and
// defect[j] per member.  The checks are the caller's.
}  // extern "C"
template <class LU>
static int inertia_impl(slu_b200_handle_t H, const LU &d, int members, int64_t *counts, double *defect)
{
    const int count = (int)H->znodes[0].size();
    const int nparts = (count + SELINV_VECS - 1) / SELINV_VECS;
    DevBuf<long long> pcnt, cnt;
    DevBuf<double> pdef, def;
    if (pcnt.alloc((size_t)3 * nparts * members) || pdef.alloc((size_t)nparts * members) || cnt.alloc((size_t)3 * members) ||
        def.alloc((size_t)members))
        return -1;
    cudaStream_t s = H->stream;
    std::vector<long long> c((size_t)3 * members, 0);
    std::vector<double> m((size_t)members, 0.0);
    if (launch_inertia(d, H->d_pool_i32.p + H->z_nodes_off[0], count, H->opt.thresh, pcnt.p, pdef.p, cnt.p, def.p, s)) {
        CU(cudaMemcpyAsync(c.data(), cnt.p, c.size() * sizeof(long long), cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(m.data(), def.p, m.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    for (size_t i = 0; i < c.size(); ++i) counts[i] = (int64_t)c[i];
    for (int j = 0; j < members; ++j) defect[j] = m[j];
    return 0;
}
extern "C" {

int slu_b200_inertia(slu_b200_handle_t H, int64_t counts[3], double *defect)
{
    if (!H || !counts || !defect) return fail("null argument");
    if (check(H, SLU_API "inertia", UNBATCHED | NOT_SCHUR | GRID_1 | FACTORED)) return -1;
    return inertia_impl(H, H->dev, 1, counts, defect);
}

int slu_b200_batch_inertia(slu_b200_handle_t H, int64_t *counts, double *defect)
{
    if (!H || !counts || !defect) return fail("null argument");
    if (check(H, SLU_API "batch_inertia", BATCHED | NOT_SCHUR | FACTORED)) return -1;
    return inertia_impl(H, H->bdev, H->batch, counts, defect);
}

// ---- affine families (slu_b200_batch_fill_affine): member j = sum_t coef[j nterms + t] A_t on one pattern.  The T terms
// cross PCIe once instead of B member value arrays; the slot search runs once per entry, then one launch over (entries,
// members) combines and scatters.  Otherwise as slu_b200_batch_fill_csr: the arena is zeroed, the factors, inverse and
// member infos are invalidated.
int slu_b200_batch_fill_affine(slu_b200_handle_t H, int n, const int32_t *rowptr, const int32_t *colind, int nterms,
                               const double *terms, const double *coef, const int32_t *perm)
{
    if (!H || !rowptr || !colind || !terms || !coef || !perm) return fail("null argument");
    const char *fn = SLU_API "batch_fill_affine";
    if (check(H, fn, BATCHED)) return -1;
    if (n != H->n) return fail("%s: matrix order %d does not match the handle's %d", fn, n, H->n);
    if (nterms < 1) return fail("%s: nterms = %d, must be at least 1", fn, nterms);
    if (rowptr[0] != 0) return fail("%s: bad rowptr (rowptr[0] = %d, must be 0)", fn, rowptr[0]);
    for (int i = 0; i < n; ++i)
        if (rowptr[i + 1] < rowptr[i]) return fail("%s: bad rowptr (rowptr[%d] = %d < rowptr[%d] = %d)", fn, i + 1, rowptr[i + 1], i, rowptr[i]);
    const int64_t nnz = rowptr[n];
    for (int64_t p = 0; p < nnz; ++p)
        if (colind[p] < 0 || colind[p] >= n) return fail("%s: colind[%lld] = %d is outside 0 ... %d", fn, (long long)p, colind[p], n - 1);
    double t0 = now_s();
    const int B = H->batch;
    DevBuf<int32_t> drp, dci, dperm;
    DevBuf<int64_t> ddst;
    DevBuf<val_t> dterms, dcoef;
    DevBuf<int8_t> dact;
    std::vector<int8_t> act(H->nsupers, 0);
    for (int k : H->znodes[0]) act[k] = 1;
    if (drp.alloc((size_t)n + 1) || dci.alloc((size_t)nnz) || dperm.alloc((size_t)n) || ddst.alloc((size_t)nnz) ||
        dterms.alloc((size_t)nnz * nterms) || dcoef.alloc((size_t)B * nterms) || dact.upload(act))
        return -1;
    cudaStream_t s = H->stream;
    int *err = H->d_flags.p + B;
    CU(cudaMemcpyAsync(drp.p, rowptr, ((size_t)n + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dci.p, colind, (size_t)nnz * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dperm.p, perm, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dterms.p, terms, (size_t)nnz * nterms * sizeof(val_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dcoef.p, coef, (size_t)B * nterms * sizeof(val_t), cudaMemcpyHostToDevice, s));
    if (values_replaced(H)) return -1;
    CU(cudaMemsetAsync(H->val.p, 0, H->val.bytes(), s));
    CU(cudaMemsetAsync(err, 0, sizeof(int), s));
    launch_fill_affine(H->bdev, n, drp.p, dci.p, dperm.p, dact.p, ddst.p, nnz, nterms, dterms.p, dcoef.p, err, s);
    int bad = 0;
    CU(cudaMemcpyAsync(&bad, err, sizeof(int), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    if (bad) return fail("%s: %d entries of the pattern have no slot in the L/U structure (wrong permutation or symbolic structure)", fn, bad);
    H->st.t_upload_s = now_s() - t0;
    H->uploaded = true;
    return 0;
}

// ---- static pivoting: the row permutation and scalings of pdgssvx3d (pdgssvx3d.c:695-727) around the device routes.
// The matching runs once per pattern on the host (sluh_large_diag_perm); the scaled, row-permuted fill, the equilibration
// and the vector transforms of the solve run on the device, per fill and per member.
static int check_perm(const int32_t *p, int n, std::vector<char> &seen, const char *fn, const char *what)
{
    seen.assign(n, 0);
    for (int i = 0; i < n; ++i) {
        if (p[i] < 0 || p[i] >= n || seen[p[i]]) return fail("%s: %s is not a permutation of 0 ... %d (entry %d = %d)", fn, what, n - 1, i, p[i]);
        seen[p[i]] = 1;
    }
    return 0;
}

static int check_scale(const double *v, int64_t len, const char *fn, const char *what)
{
    for (int64_t t = 0; t < len; ++t)
        if (!(std::isfinite(v[t]) && v[t] > 0.0)) return fail("%s: %s[%lld] = %g, must be finite and > 0", fn, what, (long long)t, v[t]);
    return 0;
}

// what every scaled call needs of the handle: the kind its name says, no Schur handle, a 1 x 1 x 1 grid
static unsigned scaled_need(bool batched) { return (batched ? BATCHED : UNBATCHED) | NOT_SCHUR | GRID_1; }

// batched: every member's values (val: members x nnz), R / C shared (rc_per_member = 0) or per member; out: members x 6
static int fill_scaled_impl(slu_b200_handle_t H, bool batched, int n, const int32_t *rowptr, const int32_t *colind, const double *val,
                            const int32_t *perm_r, const int32_t *perm, const double *R, const double *C, int rc_per_member, int flags,
                            double *out, const char *fn)
{
    if (!H || !rowptr || !colind || !val || !perm) return fail("null argument");
    if (check(H, fn, scaled_need(batched))) return -1;
    if (n != H->n) return fail("%s: matrix order %d does not match the handle's %d", fn, n, H->n);
    if (flags & ~SLU_B200_FILL_EQUIL) return fail("%s: unknown flags 0x%x", fn, flags);
    if (rc_per_member != 0 && rc_per_member != 1) return fail("%s: rc_per_member = %d, must be 0 or 1", fn, rc_per_member);
    if (rowptr[0] != 0) return fail("%s: bad rowptr (rowptr[0] = %d, must be 0)", fn, rowptr[0]);
    for (int i = 0; i < n; ++i)
        if (rowptr[i + 1] < rowptr[i]) return fail("%s: bad rowptr (rowptr[%d] = %d < rowptr[%d] = %d)", fn, i + 1, rowptr[i + 1], i, rowptr[i]);
    const int64_t nnz = rowptr[n];
    for (int64_t p = 0; p < nnz; ++p)
        if (colind[p] < 0 || colind[p] >= n) return fail("%s: colind[%lld] = %d is outside 0 ... %d", fn, (long long)p, colind[p], n - 1);
    std::vector<char> seen;
    if ((perm_r && check_perm(perm_r, n, seen, fn, "perm_r")) || check_perm(perm, n, seen, fn, "perm")) return -1;
    const int B = batched ? H->batch : 1;
    const int64_t rc_len = (int64_t)n * (rc_per_member ? B : 1);
    if ((R && check_scale(R, rc_len, fn, "R")) || (C && check_scale(C, rc_len, fn, "C"))) return -1;
    if (pin_check(H, H->d_aci.n != (size_t)nnz || H->d_aval.n != (size_t)nnz * B, fn)) return -1;
    if (values_replaced(H, true)) return -1;   // before the buffers of the scaling and the kept A are resized
    const bool equil = flags & SLU_B200_FILL_EQUIL;
    double t0 = now_s();
    std::vector<int32_t> pr(n), rmap(n);
    for (int i = 0; i < n; ++i) {
        pr[i] = perm_r ? perm_r[i] : i;
        rmap[i] = perm[pr[i]];
    }
    // every panel of a 1 x 1 x 1 grid is held
    std::vector<int8_t> act(H->nsupers, 1);
    std::vector<EquilStat> st0(B, EquilStat{0, 0, 0, 0, 0, 0, INT_MAX, INT_MAX});
    for (auto &e : st0) {
        const double big = 1.0 / 2.2250738585072014e-308;   // dgsequ's initial rcmin: bignum = 1 / dmach("S")
        memcpy(&e.rmin, &big, sizeof big);
        e.cmin = e.rmin;
    }
    // A stays in HBM for slu_b200_gsrfs: 4 (n + 1) + 4 nnz + 8 nnz batch bytes (16 per value in complex), reused by the next
    // scaled fill of the same nnz
    DevBuf<int32_t> &drp = H->d_arp, &dci = H->d_aci;
    DevBuf<val_t> &dv = H->d_aval;
    DevBuf<double> dRin, dCin, drinv, dout;
    DevBuf<unsigned long long> dccol;
    DevBuf<EquilStat> dst;
    DevBuf<int8_t> dact;
    const size_t bn = (size_t)B * n;
    if ((drp.n != (size_t)n + 1 && drp.alloc((size_t)n + 1)) || grow(H, dci, (size_t)nnz, true, false, fn) ||
        grow(H, dv, (size_t)nnz * B, true, false, fn) || dact.upload(act) || dst.upload(st0) ||
        dout.alloc((size_t)B * 6) || (R && dRin.alloc((size_t)rc_len)) || (C && dCin.alloc((size_t)rc_len)) ||
        (equil && (drinv.alloc(bn) || dccol.alloc(bn))))
        return -1;
    if (H->d_R.n != bn && (H->d_R.alloc(bn) || H->d_C.alloc(bn))) return -1;
    if (H->d_perm_r.n != (size_t)n && (H->d_perm_r.alloc(n) || H->d_rmap.alloc(n) || H->d_cperm.alloc(n))) return -1;
    cudaStream_t s = H->stream;
    int *err = H->d_flags.p + (batched ? B : 1);
    CU(cudaMemcpyAsync(drp.p, rowptr, ((size_t)n + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dci.p, colind, (size_t)nnz * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(dv.p, val, (size_t)nnz * B * sizeof(val_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(H->d_perm_r.p, pr.data(), (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(H->d_rmap.p, rmap.data(), (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(H->d_cperm.p, perm, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    if (R) CU(cudaMemcpyAsync(dRin.p, R, (size_t)rc_len * sizeof(double), cudaMemcpyHostToDevice, s));
    if (C) CU(cudaMemcpyAsync(dCin.p, C, (size_t)rc_len * sizeof(double), cudaMemcpyHostToDevice, s));
    if (equil) CU(cudaMemsetAsync(dccol.p, 0, bn * sizeof(unsigned long long), s));
    CU(cudaMemsetAsync(H->val.p, 0, H->val.bytes(), s));
    CU(cudaMemsetAsync(err, 0, sizeof(int), s));
    ScaledFill f{};
    f.n = n;
    f.rowptr = drp.p; f.colind = dci.p; f.rmap = H->d_rmap.p; f.perm = H->d_cperm.p; f.aval = dv.p;
    f.R_in = R ? dRin.p : nullptr; f.C_in = C ? dCin.p : nullptr; f.rc_stride = rc_per_member ? n : 0;
    f.R = H->d_R.p; f.C = H->d_C.p; f.rinv = drinv.p; f.ccol = dccol.p; f.st = dst.p; f.out = dout.p;
    f.active = dact.p; f.err = err;
    if (batched) launch_fill_scaled(H->bdev, f, equil, s);
    else launch_fill_scaled(H->dev, f, equil, s);
    int bad = 0;
    std::vector<double> o(equil ? (size_t)B * 6 : 0);
    CU(cudaMemcpyAsync(&bad, err, sizeof(int), cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(st0.data(), dst.p, (size_t)B * sizeof(EquilStat), cudaMemcpyDeviceToHost, s));
    if (equil) CU(cudaMemcpyAsync(o.data(), dout.p, o.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    if (bad) return fail("%s: %d entries of A have no slot in the L/U structure (wrong permutation or symbolic structure)", fn, bad);
    for (int m = 0; equil && m < B; ++m) {   // dgsequ's info: the first exactly zero row, else the first zero column
        char mem[32] = "";
        if (batched) snprintf(mem, sizeof mem, " (member %d)", m);
        if (st0[m].zrow != INT_MAX) return fail("%s: row %d of A%s is exactly zero: cannot equilibrate", fn, st0[m].zrow, mem);
        if (st0[m].zcol != INT_MAX) return fail("%s: column %d of A%s is exactly zero: cannot equilibrate", fn, st0[m].zcol, mem);
    }
    if (out)
        for (int m = 0; m < B; ++m) {
            double *om = out + (size_t)m * 6, fn_, fm;
            memcpy(&fn_, &st0[m].fnorm, sizeof fn_);
            memcpy(&fm, &st0[m].fmax, sizeof fm);
            if (equil) for (int k = 0; k < 4; ++k) om[k] = o[(size_t)m * 6 + k];
            else { om[0] = om[1] = 1.0; om[2] = fm; om[3] = 0.0; }
            om[4] = fn_;
            om[5] = fm;
        }
    H->st.t_upload_s = now_s() - t0;
    H->uploaded = true;
    H->scaled = true;
    return 0;
}

static int get_scaling_impl(slu_b200_handle_t H, bool batched, int member, int32_t *perm_r, double *R, double *C, const char *fn)
{
    if (!H) return fail("null handle");
    if (check(H, fn, scaled_need(batched) | SCALED)) return -1;
    if (batched && (member < 0 || member >= H->batch)) return fail("%s: member %d is outside 0 ... %d", fn, member, H->batch - 1);
    const size_t n = (size_t)H->n, off = (size_t)member * n;
    if (perm_r) CU(cudaMemcpy(perm_r, H->d_perm_r.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (R) CU(cudaMemcpy(R, H->d_R.p + off, n * sizeof(double), cudaMemcpyDeviceToHost));
    if (C) CU(cudaMemcpy(C, H->d_C.p + off, n * sizeof(double), cudaMemcpyDeviceToHost));
    return 0;
}

int slu_b200_fill_csr_scaled(slu_b200_handle_t H, int n, const int32_t *rowptr, const int32_t *colind, const double *val,
                             const int32_t *perm_r, const int32_t *perm, const double *R, const double *C, int flags, double out[6])
{
    return fill_scaled_impl(H, false, n, rowptr, colind, val, perm_r, perm, R, C, 0, flags, out, SLU_API "fill_csr_scaled");
}

int slu_b200_get_scaling(slu_b200_handle_t H, int32_t *perm_r, double *R, double *C)
{
    return get_scaling_impl(H, false, 0, perm_r, R, C, SLU_API "get_scaling");
}

int slu_b200_solve_scaled(slu_b200_handle_t H, double *x, int ldx, int nrhs, int trans)
{
    return solve_host(H, SLU_API "solve_scaled", scaled_need(false) | SCALED | FACTORED, x, ldx, nrhs, trans, PASS_BOTH);
}

int slu_b200_batch_fill_csr_scaled(slu_b200_handle_t H, int n, const int32_t *rowptr, const int32_t *colind, const double *val,
                                   const int32_t *perm_r, const int32_t *perm, const double *R, const double *C, int rc_per_member,
                                   int flags, double *out)
{
    return fill_scaled_impl(H, true, n, rowptr, colind, val, perm_r, perm, R, C, rc_per_member, flags, out,
                            SLU_API "batch_fill_csr_scaled");
}

int slu_b200_batch_get_scaling(slu_b200_handle_t H, int member, double *R, double *C)
{
    return get_scaling_impl(H, true, member, nullptr, R, C, SLU_API "batch_get_scaling");
}

int slu_b200_batch_solve_scaled(slu_b200_handle_t H, double *x, int ldx, int nrhs, int trans)
{
    return solve_host(H, SLU_API "batch_solve_scaled", scaled_need(true) | SCALED | FACTORED, x, ldx, nrhs, trans, PASS_BOTH);
}

// ---- iterative refinement with error bounds: pdgsrfs (pdgsrfs.c:198-251) for op(A) = A in A's own ordering, on the factors
// and scalings of the last scaled fill and the A it kept; the forward error bound of LAPACK dgerfs.  Each step runs the
// residual kernel over every (row, column, member), the decide kernel and one read of the count of columns still active, then
// one scaled solve of the whole block of residuals and the update.  ferr: dlacn2 through cond_rounds, each (member, column)
// one estimator member: kase 1 solves with A^T (A^H) and multiplies by W, kase 2 multiplies by W and solves with A.

// The checks of gsrfs and gsrfs_device after null pointers: what they need of the handle, nrhs, ldb / ldx, n * nrhs
static int gsrfs_check(slu_b200_handle_t H, const char *fn, unsigned need, int ldb, int ldx, int nrhs)
{
    if (check(H, fn, need)) return -1;
    const int n = H->n;
    if (nrhs < 1) return fail("%s: nrhs = %d, must be >= 1", fn, nrhs);
    if (ldb < n || ldx < n) return fail("%s: ldb = %d and ldx = %d must be >= n = %d", fn, ldb, ldx, n);
    if ((int64_t)n * nrhs > INT_MAX) return fail("%s: n * nrhs must stay below 2^31 per member", fn);
    return 0;
}

// The refinement's buffers for cols columns of len elements in all, with ferr the estimator's (pinned after a capture: grow)
static int refine_buffers(slu_b200_handle_t H, size_t len, int cols, bool ferr, bool capturing, const char *fn)
{
    if (grow(H, H->d_x, len, false, capturing, fn) || grow(H, H->d_x2, len, false, capturing, fn) || grow_loop(H, H->d_rb, len, capturing, fn) ||
        grow_loop(H, H->d_rx, len, capturing, fn) || grow_loop(H, H->d_rst, cols, capturing, fn) || grow_loop(H, H->d_ract, 1, capturing, fn) ||
        grow_loop(H, H->d_rout, 2 * (size_t)cols, capturing, fn) || grow_loop(H, H->d_rsteps, cols, capturing, fn))
        return -1;
    return ferr && (grow_loop(H, H->d_rw, len, capturing, fn) || grow_loop(H, H->d_cv, len, capturing, fn) ||
                    cond_buffers(H, H->n, cols, capturing, fn) || grow_loop(H, H->d_rxmax, cols, capturing, fn)) ? -1 : 0;
}

// The pieces of the refinement of x in d_rx for b in d_rb, shared by gsrfs (the host reads d_ract between refine_check and
// refine_step) and gsrfs_loop (a WHILE node).  Each enqueues on H->stream and returns its launches, < 0 on an error.
static RefineArgs refine_args(slu_b200_handle_t H, bool batched, int nrhs, bool ferr)
{
    return RefineArgs{H->n, nrhs, batched ? H->batch : 1, (int64_t)H->d_aci.n, H->d_arp.p, H->d_aci.p, H->d_aval.p, H->d_rb.p, H->d_rst.p,
                      ferr ? H->d_rw.p : nullptr};
}

// pdgsrfs's start state of every column (lstres = 3, count = 0); inactive where the member's status is not 0
static int refine_init(slu_b200_handle_t H, const RefineArgs &a)
{
    return launch_refine_init(H->d_rst.p, H->d_info.p, a.nrhs, a.members, H->stream);
}

// the residual of every active column, then pdgsrfs's test: d_ract = the columns that take another step
static int refine_check(slu_b200_handle_t H, const RefineArgs &a, bool batched)
{
    const int l = launch_refine_residual(a, H->d_rx.p, scaled_in(H, batched), H->stream);
    CU(cudaMemsetAsync(H->d_ract.p, 0, sizeof(int), H->stream));
    return l + launch_refine_decide(a, H->d_ract.p, H->stream);
}

// one step: dx = A^-1 r in d_x2, x += dx on the active columns
static int refine_step(slu_b200_handle_t H, const RefineArgs &a, bool batched)
{
    const int l = solve_scaled_dev(H, batched, a.nrhs, 0);
    return l < 0 ? -1 : l + launch_refine_update(a, H->d_rx.p, H->d_x2.p, H->stream);
}

// dgerfs's operator for ferr on the pending vectors v in d_cv, the result in d_x2 (*res): kase 1 diag(W) A^-T v (A^-H in
// complex), kase 2 A^-1 diag(W) v
static int refine_ferr_apply(slu_b200_handle_t H, bool batched, int nrhs, int kase, val_t **res)
{
    const int64_t len = (int64_t)H->n * nrhs * (batched ? H->batch : 1);
    val_t *in = scaled_in(H, batched);
    *res = H->d_x2.p;
    if (kase == 2) {
        const int l = launch_refine_scale(in, H->d_cv.p, H->d_rw.p, len, H->stream);
        const int ls = solve_scaled_dev(H, batched, nrhs, 0);
        return ls < 0 ? -1 : l + ls;
    }
    CU(cudaMemcpyAsync(in, H->d_cv.p, (size_t)len * sizeof(val_t), cudaMemcpyDeviceToDevice, H->stream));
    const int l = solve_scaled_dev(H, batched, nrhs, VAL_DOUBLES == 2 ? 2 : 1);
    return l < 0 ? -1 : l + launch_refine_scale(*res, *res, H->d_rw.p, len, H->stream);
}

// berr, steps and (ferr, the estimate in d_cstate) dgerfs's ferr = est / max_i |x_i| per column into d_rout (berr, ferr), d_rsteps
static int refine_end(slu_b200_handle_t H, const RefineArgs &a, bool ferr)
{
    const int cols = a.nrhs * a.members;
    int launches = 0;
    if (ferr) {
        CU(cudaMemsetAsync(H->d_rxmax.p, 0, (size_t)cols * sizeof(unsigned long long), H->stream));
        launches += launch_refine_xmax(a, H->d_rx.p, H->d_rxmax.p, H->stream);
    }
    return launches + launch_refine_finish(a, H->d_cstate.p, H->d_rxmax.p, H->d_info.p, H->d_rout.p, ferr ? H->d_rout.p + cols : nullptr,
                                           H->d_rsteps.p, H->stream);
}

static int gsrfs_impl(slu_b200_handle_t H, bool batched, const double *bh, int ldb, double *xh, int ldx, int nrhs, double *berr,
                      double *ferr, int32_t *steps, const char *fn)
{
    if (!H || !bh || !xh || !berr) return fail("%s: null argument (b, x and berr are required)", fn);
    if (gsrfs_check(H, fn, scaled_need(batched) | SCALED | FACTORED, ldb, ldx, nrhs)) return -1;
    const int n = H->n, cols = (batched ? H->batch : 1) * nrhs;
    if (refine_buffers(H, (size_t)n * cols, cols, ferr != nullptr, false, fn)) return -1;
    cudaStream_t s = H->stream;
    const double t0 = now_s();
    const size_t w = (size_t)n * sizeof(val_t);
    CU(cudaMemcpy2DAsync(H->d_rb.p, w, bh, (size_t)ldb * sizeof(val_t), w, (size_t)cols, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpy2DAsync(H->d_rx.p, w, xh, (size_t)ldx * sizeof(val_t), w, (size_t)cols, cudaMemcpyHostToDevice, s));
    const RefineArgs a = refine_args(H, batched, nrhs, ferr != nullptr);
    int launches = refine_init(H, a);       // d_info is 0 for every member here (FACTORED)
    for (int step = 0;; ++step) {
        if (step > REFINE_ITMAX) return fail("%s: the refinement did not stop after %d steps", fn, REFINE_ITMAX);
        const int lc = refine_check(H, a, batched);
        if (lc < 0) return -1;
        launches += lc;
        int active = 0;
        CU(cudaMemcpyAsync(&active, H->d_ract.p, sizeof(int), cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        if (active == 0) break;
        const int ls = refine_step(H, a, batched);
        if (ls < 0) return -1;
        launches += ls;
    }
    if (ferr) {
        int rounds = 0;
        auto apply = [&](int kase, val_t **res) { return refine_ferr_apply(H, batched, nrhs, kase, res); };
        const int l = cond_rounds(H, n, cols, H->d_cv.p, apply, &rounds, fn);
        if (l < 0) return -1;
        launches += l;
    }
    const int le = refine_end(H, a, ferr != nullptr);
    if (le < 0) return -1;
    launches += le;
    CU(cudaMemcpy2DAsync(xh, (size_t)ldx * sizeof(val_t), H->d_rx.p, w, w, (size_t)cols, cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(berr, H->d_rout.p, (size_t)cols * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (ferr) CU(cudaMemcpyAsync(ferr, H->d_rout.p + cols, (size_t)cols * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (steps) CU(cudaMemcpyAsync(steps, H->d_rsteps.p, (size_t)cols * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    H->st.reserved[4] = now_s() - t0;
    H->st.reserved[5] = (double)launches;
    return 0;
}

int slu_b200_gsrfs(slu_b200_handle_t H, const double *b, int ldb, double *x, int ldx, int nrhs, double *berr, double *ferr, int32_t *steps)
{
    return gsrfs_impl(H, false, b, ldb, x, ldx, nrhs, berr, ferr, steps, SLU_API "gsrfs");
}

int slu_b200_batch_gsrfs(slu_b200_handle_t H, const double *b, int ldb, double *x, int ldx, int nrhs, double *berr, double *ferr,
                         int32_t *steps)
{
    return gsrfs_impl(H, true, b, ldb, x, ldx, nrhs, berr, ferr, steps, SLU_API "batch_gsrfs");
}

// ---- device-resident refill and solves on the caller's stream (pdgssvx3d's Fact = SamePattern_SameRowPerm for values that
// already live in HBM).  Every call checks its pointers before it enqueues anything, orders the handle's stream after the
// work already on the caller's stream, and the caller's stream after its own work, with events: no host wait, no PCIe copy.
static int check_device_ptr(slu_b200_handle_t H, const void *p, const char *fn, const char *what)
{
    cudaPointerAttributes a{};
    const cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail("%s: %s is not a pointer CUDA knows (%s)", fn, what, cudaGetErrorString(e));
    }
    if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged)
        return fail("%s: %s must point at device or managed memory on device %d, not at %s memory", fn, what, H->device,
                    a.type == cudaMemoryTypeHost ? "pinned host" : "host");
    if (a.device != H->device) return fail("%s: %s points at memory of device %d, the handle's device is %d", fn, what, a.device, H->device);
    return 0;
}

// cap: the call is being captured (capturing), which pins the handle's buffers from now on
static int stream_enter(slu_b200_handle_t H, cudaStream_t caller, bool cap)
{
    H->captured = H->captured || cap;
    CU(cudaEventRecord(H->ev_in, caller));
    CU(cudaStreamWaitEvent(H->stream, H->ev_in, 0));
    return 0;
}

static int stream_leave(slu_b200_handle_t H, cudaStream_t caller)
{
    CU(cudaGetLastError());
    CU(cudaEventRecord(H->ev_out, H->stream));
    CU(cudaStreamWaitEvent(caller, H->ev_out, 0));
    return 0;
}

// Whether the caller's stream is capturing a CUDA graph: 1 yes, 0 no, < 0 an error.  Every call on the caller's stream asks
// before it enqueues anything, refuses under capture what would allocate or wait on the host, and marks the handle as
// captured (pin_check) in stream_enter, once it is sure to enqueue.
static int capturing(slu_b200_handle_t H, cudaStream_t caller, const char *fn)
{
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    const cudaError_t e = cudaStreamIsCapturing(caller, &cs);
    if (e != cudaSuccess) return fail("%s: cudaStreamIsCapturing: %s", fn, cudaGetErrorString(e));
    return cs != cudaStreamCaptureStatusNone;
}

// The refill's slot map of the kept A (d_amap, d_arow), once per scaled fill: allocates and waits for it -> its launches
static int build_amap(slu_b200_handle_t H, const char *fn)
{
    if (H->amap_ready) return 0;
    const int64_t nnz = (int64_t)H->d_aci.n;
    const cudaStream_t s = H->stream;
    DevBuf<int8_t> act;                       // every panel of a 1 x 1 x 1 grid is held
    if (grow(H, H->d_amap, nnz, true, false, fn) || grow(H, H->d_arow, nnz, true, false, fn) || act.alloc(H->nsupers)) return -1;
    CU(cudaMemsetAsync(act.p, 1, act.bytes(), s));
    const int launches = launch_refill_slots(H->dev, H->n, H->d_arp.p, H->d_aci.p, H->d_rmap.p, H->d_cperm.p, act.p, H->d_amap.p,
                                             H->d_arow.p, s);
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    H->amap_ready = true;
    return launches;
}

// New values of the last scaled fill's pattern, val on the device (batch x nnz on a batched handle): the arena zeroed, then
// F = Pc Pr Dr A Dc Pc^T with the kept perm_r, perm, R and C, bit for bit the scaled fill's values; val also replaces the
// kept A.  The first refill after a scaled fill builds the slot map (allocates, and waits for it once).
static int refill_impl(slu_b200_handle_t H, bool batched, const double *val, void *stream, const char *fn)
{
    if (!H || !val) return fail("%s: null argument", fn);
    if (check(H, fn, scaled_need(batched) | SCALED)) return -1;
    if (check_device_ptr(H, val, fn, "val")) return -1;
    const cudaStream_t caller = (cudaStream_t)stream, s = H->stream;
    const int cap = capturing(H, caller, fn);
    if (cap < 0) return -1;
    if (cap && !H->amap_ready)
        return fail("%s: the first refill after a scaled fill builds the slot map and waits for it: make this call once outside "
                    "capture first", fn);
    const int n = H->n;
    const int64_t nnz = (int64_t)H->d_aci.n;
    int launches = build_amap(H, fn);
    if (launches < 0) return -1;
    if (stream_enter(H, caller, cap)) return -1;
    if (factors_replaced(H)) return -1;           // d_info's reset goes into the caller's stream order
    H->uploaded = false;
    CU(cudaMemsetAsync(H->val.p, 0, H->val.bytes(), s));
    const Refill r{n, nnz, (const val_t *)val, H->d_amap.p, H->d_arow.p, H->d_aci.p, H->d_R.p, H->d_C.p, H->d_aval.p};
    launches += batched ? launch_refill(H->bdev, r, s) : launch_refill(H->dev, r, s);
    if (stream_leave(H, caller)) return -1;
    H->st.t_upload_s = 0;
    H->st.reserved[4] = 0;
    H->st.reserved[5] = (double)launches;
    H->uploaded = true;
    return 0;
}

// factor / batch_factor on the caller's stream: the same level loop, with the info flags and d_tiny reset by a kernel and
// every member's info written to info (device memory) and d_info by another.  No host wait, copy or allocation: capturable.
// member_info stays INFO_PENDING until a host-synchronous call settles it.
static int factor_device_impl(slu_b200_handle_t H, bool batched, int32_t *info, void *stream, const char *fn)
{
    if (!H || !info) return fail("%s: null argument", fn);
    if (check(H, fn, scaled_need(batched) | UPLOADED)) return -1;
    if (check_device_ptr(H, info, fn, "info")) return -1;
    const cudaStream_t caller = (cudaStream_t)stream, s = H->stream;
    const int cap = capturing(H, caller, fn);
    if (cap < 0) return -1;
    const int B = batched ? H->batch : 1;
    if (stream_enter(H, caller, cap)) return -1;
    if (factors_replaced(H)) return -1;
    int64_t launches = launch_factor_begin(H->d_flags.p, B, H->d_tiny.p, s);
    const int64_t l = batched ? factor_levels(H, H->bdev, false, false, false) : factor_levels(H, H->dev, false, false, false);
    if (l < 0) return -1;
    launches += l + launch_factor_info(H->d_flags.p, B, info, H->d_info.p, H->d_epoch.p, s);
    if (stream_leave(H, caller)) return -1;
    H->st.t_factor_s = 0;
    H->st.gpu_launches = launches;
    std::fill(H->member_info.begin(), H->member_info.end(), INFO_PENDING);
    H->status_on_device = true;
    return 0;
}

// solve / solve_trans (scaled = false: F's ordering) and solve_scaled (A's ordering) on device x, with the host twins' layout
// and checks; the same device work, with device-to-device copies in place of the H2D and D2H ones.  1 x 1 x 1 grids.  After
// a device factorization the host has not seen the members' info: the guard turns the x of every member whose d_info is not
// 0 into NaN.
static int solve_device_impl(slu_b200_handle_t H, bool batched, bool scaled, double *xd, int ldx, int nrhs, int trans, void *stream,
                             const char *fn)
{
    if (!H || !xd) return fail("%s: null argument", fn);
    if (solve_check(H, fn, scaled_need(batched) | (scaled ? SCALED : 0) | FACTORED | DEVICE_ORDERED, trans, nrhs, ldx, true)) return -1;
    if (check_device_ptr(H, xd, fn, "x")) return -1;
    const int B = batched ? H->batch : 1, n = H->n;
    const cudaStream_t caller = (cudaStream_t)stream, s = H->stream;
    const int cap = capturing(H, caller, fn);
    if (cap < 0) return -1;
    if (solve_buffers(H, batched, scaled, (size_t)n * nrhs * B, cap, fn)) return -1;
    if (stream_enter(H, caller, cap)) return -1;
    val_t *result = nullptr;
    int launches = solve_enqueue(H, batched, scaled, PASS_BOTH, xd, ldx, nrhs, trans, cudaMemcpyDeviceToDevice, &result);
    if (launches < 0) return -1;
    launches += launch_solve_guard(result, H->d_info.p, (int64_t)n * nrhs, B, s);
    const size_t w = (size_t)n * sizeof(val_t);
    CU(cudaMemcpy2DAsync(xd, (size_t)ldx * sizeof(val_t), result, w, w, (size_t)nrhs * B, cudaMemcpyDeviceToDevice, s));
    if (stream_leave(H, caller)) return -1;
    H->st.reserved[4] = 0;
    H->st.reserved[5] = (double)launches;
    return 0;
}

// ---- gradients on the caller's stream (selinv_device, logdet_device, logdet_grad_device, solve_grad_device and their twins).
// The checks of solve_scaled_device; no host wait or PCIe copy, except in the allocating first calls (the second arena and the
// plan of the first selected inversion, the refill's slot map, the staging buffer of a wider solve_grad), which are refused
// under capture.  The result of a member whose status is not 0 (its factorization, or a selected inversion that missed a
// destination) is NaN.

// selinv's sweep ordered on the caller's stream.  The missed-destination count stays on the device: selinv_status_kernel
// turns it into the status logdet_grad_device reads, and the next host-synchronous call reads it (settle) before it trusts
// the inverse.
static int selinv_device_impl(slu_b200_handle_t H, bool batched, void *stream, const char *fn)
{
    if (!H) return fail("%s: null argument", fn);
    if (check(H, fn, scaled_need(batched) | SCALED | FACTORED | DEVICE_ORDERED)) return -1;
    const cudaStream_t caller = (cudaStream_t)stream, s = H->stream;
    const int cap = capturing(H, caller, fn);
    if (cap < 0) return -1;
    const int B = batched ? H->batch : 1;
    if (!H->d_hinv.p || H->si_levels.empty() || !H->d_si_status.p) {
        if (cap)
            return fail("%s: the first selected inversion on a handle allocates the inverse's arena and plan: make this call once "
                        "outside capture first", fn);
        if (selinv_alloc(H, B, fn) || H->d_si_status.alloc((size_t)B) || H->d_si_rec.alloc(2)) return -1;
    }
    if (stream_enter(H, caller, cap)) return -1;
    H->si_ready = false;
    double flops = 0;
    int launches = batched ? selinv_enqueue(H, H->bdev, &flops) : selinv_enqueue(H, H->dev, &flops);
    if (launches < 0) return -1;
    launches += launch_selinv_status(H->dev.err, H->d_info.p, B, H->d_epoch.p, H->d_si_status.p, H->d_si_rec.p, s);
    if (stream_leave(H, caller)) return -1;
    H->si_ready = true;
    H->si_dev = true;
    H->status_on_device = true;           // the next host-synchronous call settles the record before it reads the inverse
    H->st.reserved[4] = 0;
    H->st.reserved[5] = (double)launches;
    return 0;
}

// logdet's reduction into the handle's buffers, then logabs[members] and sign[members * VAL_DOUBLES] on the device
static int logdet_device_impl(slu_b200_handle_t H, bool batched, double *logabs, double *sign, void *stream, const char *fn)
{
    if (!H || !logabs || !sign) return fail("%s: null argument", fn);
    if (check(H, fn, scaled_need(batched) | SCALED | FACTORED | DEVICE_ORDERED)) return -1;
    if (check_device_ptr(H, logabs, fn, "logabs") || check_device_ptr(H, sign, fn, "sign")) return -1;
    const cudaStream_t caller = (cudaStream_t)stream, s = H->stream;
    const int cap = capturing(H, caller, fn);
    if (cap < 0) return -1;
    const int B = batched ? H->batch : 1;
    const int count = (int)H->znodes[0].size();
    const size_t nparts = (size_t)(count + SELINV_VECS - 1) / SELINV_VECS;
    if (grow(H, H->d_lpart, nparts * B, false, cap, fn) || grow(H, H->d_lph, nparts * B, false, cap, fn) ||
        grow(H, H->d_lres, (size_t)(1 + VAL_DOUBLES) * B, false, cap, fn))
        return -1;
    if (stream_enter(H, caller, cap)) return -1;
    const int32_t *nodes = H->d_pool_i32.p + H->z_nodes_off[0];
    int launches = batched ? launch_selinv_logdet(H->bdev, nodes, count, H->d_lpart.p, H->d_lph.p, H->d_lres.p, s)
                           : launch_selinv_logdet(H->dev, nodes, count, H->d_lpart.p, H->d_lph.p, H->d_lres.p, s);
    launches += launch_logdet_out(H->d_lres.p, H->d_info.p, B, logabs, sign, s);
    if (stream_leave(H, caller)) return -1;
    H->st.reserved[4] = 0;
    H->st.reserved[5] = (double)launches;
    return 0;
}

// grad[members x nnz] = coef[j] R_i C_j H(slot of entry (i, j)) (conj(H) in doublecomplex): the inverse of the last selinv or
// selinv_device gathered through the refill's slot map onto the kept A's pattern, in the scaled fill's entry order
static int logdet_grad_impl(slu_b200_handle_t H, bool batched, const double *coef, double *grad, void *stream, const char *fn)
{
    if (!H || !coef || !grad) return fail("%s: null argument", fn);
    if (check(H, fn, scaled_need(batched) | SCALED | FACTORED | DEVICE_ORDERED)) return -1;
    if (!H->si_ready)
        return fail("%s needs %s or %s on the current factors first (a later fill, refill, upload or factorization invalidates "
                    "the inverse)", fn, batched ? SLU_API "batch_selinv_device" : SLU_API "selinv_device",
                    batched ? SLU_API "batch_selinv" : SLU_API "selinv");
    if (check_device_ptr(H, coef, fn, "coef") || check_device_ptr(H, grad, fn, "grad")) return -1;
    const cudaStream_t caller = (cudaStream_t)stream, s = H->stream;
    const int cap = capturing(H, caller, fn);
    if (cap < 0) return -1;
    if (cap && !H->amap_ready)
        return fail("%s: the first gradient or refill after a scaled fill builds the slot map and waits for it: make this call "
                    "once outside capture first", fn);
    int launches = build_amap(H, fn);
    if (launches < 0) return -1;
    if (stream_enter(H, caller, cap)) return -1;
    const LogdetGrad a{H->n, (int64_t)H->d_aci.n, H->d_amap.p, H->d_arow.p, H->d_aci.p, H->d_R.p, H->d_C.p, H->d_hinv.p,
                       (const val_t *)coef, H->si_dev ? H->d_si_status.p : H->d_info.p, (val_t *)grad};
    launches += batched ? launch_logdet_grad(H->bdev, a, s) : launch_logdet_grad(H->dev, a, s);
    if (stream_leave(H, caller)) return -1;
    H->st.reserved[4] = 0;
    H->st.reserved[5] = (double)launches;
    return 0;
}

// grad[members x nnz] = -sum_k lam(i, k) conj(x(j, k)) on the kept A's pattern; lam and x: members blocks of n x nrhs
// column-major, ldl / ldx apart per column, as the device solves take them.  nrhs > 1 goes through row-major copies in
// d_gstage, so that each entry reads its nrhs values of lam and of x as two contiguous runs.
static int solve_grad_impl(slu_b200_handle_t H, bool batched, const double *lam, int ldl, const double *x, int ldx, int nrhs,
                           double *grad, void *stream, const char *fn)
{
    if (!H || !lam || !x || !grad) return fail("%s: null argument", fn);
    if (check(H, fn, scaled_need(batched) | SCALED | FACTORED | DEVICE_ORDERED)) return -1;
    const int B = batched ? H->batch : 1, n = H->n;
    if (nrhs < 1 || ldl < n || ldx < n) return fail("%s: bad nrhs / ldl / ldx", fn);
    if ((int64_t)n * nrhs > INT_MAX) return fail("%s: n * nrhs must stay below 2^31 per member", fn);
    if (check_device_ptr(H, lam, fn, "lam") || check_device_ptr(H, x, fn, "x") || check_device_ptr(H, grad, fn, "grad")) return -1;
    const cudaStream_t caller = (cudaStream_t)stream, s = H->stream;
    const int cap = capturing(H, caller, fn);
    if (cap < 0) return -1;
    if (cap && !H->amap_ready)
        return fail("%s: the first gradient or refill after a scaled fill builds the slot map and waits for it: make this call "
                    "once outside capture first", fn);
    const size_t len = (size_t)n * nrhs * B;
    if (nrhs > 1 && grow(H, H->d_gstage, 2 * len, false, cap, fn)) return -1;
    int launches = build_amap(H, fn);
    if (launches < 0) return -1;
    if (stream_enter(H, caller, cap)) return -1;
    SolveGrad a{(int64_t)H->d_aci.n, nrhs, 0, H->d_arow.p, H->d_aci.p, (const val_t *)lam, (const val_t *)x, ldl, ldx, 1,
                H->d_info.p, (val_t *)grad};
    if (nrhs > 1) {
        launches += launch_grad_stage(H->d_gstage.p, a.lam, n, nrhs, ldl, B, s);
        launches += launch_grad_stage(H->d_gstage.p + len, a.x, n, nrhs, ldx, B, s);
        a.lam = H->d_gstage.p;
        a.x = H->d_gstage.p + len;
        a.lms = a.xms = (int64_t)n * nrhs;
        a.rs = nrhs;
    }
    launches += launch_solve_grad(a, B, s);
    if (stream_leave(H, caller)) return -1;
    H->st.reserved[4] = 0;
    H->st.reserved[5] = (double)launches;
    return 0;
}

int slu_b200_selinv_device(slu_b200_handle_t H, void *stream)
{
    return selinv_device_impl(H, false, stream, SLU_API "selinv_device");
}

int slu_b200_batch_selinv_device(slu_b200_handle_t H, void *stream)
{
    return selinv_device_impl(H, true, stream, SLU_API "batch_selinv_device");
}

int slu_b200_logdet_device(slu_b200_handle_t H, double *logabs, double *sign, void *stream)
{
    return logdet_device_impl(H, false, logabs, sign, stream, SLU_API "logdet_device");
}

int slu_b200_batch_logdet_device(slu_b200_handle_t H, double *logabs, double *sign, void *stream)
{
    return logdet_device_impl(H, true, logabs, sign, stream, SLU_API "batch_logdet_device");
}

int slu_b200_logdet_grad_device(slu_b200_handle_t H, const double *coef, double *grad, void *stream)
{
    return logdet_grad_impl(H, false, coef, grad, stream, SLU_API "logdet_grad_device");
}

int slu_b200_batch_logdet_grad_device(slu_b200_handle_t H, const double *coef, double *grad, void *stream)
{
    return logdet_grad_impl(H, true, coef, grad, stream, SLU_API "batch_logdet_grad_device");
}

int slu_b200_solve_grad_device(slu_b200_handle_t H, const double *lam, int ldl, const double *x, int ldx, int nrhs, double *grad,
                               void *stream)
{
    return solve_grad_impl(H, false, lam, ldl, x, ldx, nrhs, grad, stream, SLU_API "solve_grad_device");
}

int slu_b200_batch_solve_grad_device(slu_b200_handle_t H, const double *lam, int ldl, const double *x, int ldx, int nrhs,
                                     double *grad, void *stream)
{
    return solve_grad_impl(H, true, lam, ldl, x, ldx, nrhs, grad, stream, SLU_API "batch_solve_grad_device");
}

// ---- iterative refinement and condition estimation on the caller's stream (gsrfs_device, gscon_device and their twins).
// The host loops of gsrfs and gscon read a counter back after every step or round to decide whether to go on.  Here the
// decision stays on the device: each loop is a conditional WHILE node whose body ends with a kernel that sets the node's
// handle from the same counter, and the estimator's body runs the solve of the round's kase in one of two IF nodes.  The
// residual, decide, update, solve and estimator-step kernels are those of the host loops, so the device loops take the same
// decisions on the same vectors.  One enqueue path serves both ways a call runs: under the caller's capture (the handle's
// stream joins it in stream_enter) the nodes go straight into the caller's graph; an eager call captures the same sequence
// on the handle's stream once, caches the executable graph and launches it, with only the copies of the caller's pointers
// outside it.  Conditional nodes cannot be children of a child graph node, hence the nodes are added to the capture itself:
// each body graph is captured on a side stream of the handle (one per nesting depth), swapped in for H->stream while the
// body's solves are enqueued.
}  // extern "C"

// conditional graph nodes need a driver of CUDA 12.4 or later; read once
static int conditional_nodes_check(const char *fn)
{
    static int version = 0;
    if (version == 0) CU(cudaDriverGetVersion(&version));
    if (version < 12040)
        return fail("%s needs a CUDA driver of version 12.4 or later for conditional graph nodes (this driver is %d.%d)", fn,
                    version / 1000, version % 1000 / 10);
    return 0;
}

// a new conditional handle in the graph being captured on H->stream
static int cond_handle(slu_b200_handle_t H, cudaGraphConditionalHandle *h)
{
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaGraph_t g = nullptr;
    CU(cudaStreamGetCaptureInfo(H->stream, &cs, nullptr, &g, nullptr, nullptr));
    if (cs != cudaStreamCaptureStatusActive) return fail("the handle's stream is not capturing a CUDA graph");
    CU(cudaGraphConditionalHandleCreate(h, g, 0, 0));
    return 0;
}

// A conditional node of `type` on handle h after the current dependencies of the capture on H->stream, its body captured from
// body() (which enqueues on H->stream and returns < 0 on an error) on side stream s_body[depth]; the node becomes the
// capture's next dependency.  H->stream is restored on every path.
template <class Body>
static int add_conditional(slu_b200_handle_t H, cudaGraphConditionalNodeType type, cudaGraphConditionalHandle h, int depth, Body body)
{
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaGraph_t g = nullptr;
    const cudaGraphNode_t *deps = nullptr;
    size_t ndeps = 0;
    CU(cudaStreamGetCaptureInfo(H->stream, &cs, nullptr, &g, &deps, &ndeps));
    cudaGraphNodeParams p{};
    p.type = cudaGraphNodeTypeConditional;
    p.conditional.handle = h;
    p.conditional.type = type;
    p.conditional.size = 1;
    cudaGraphNode_t node = nullptr;
    CU(cudaGraphAddNode(&node, g, deps, ndeps, &p));
    const cudaStream_t outer = H->stream, side = H->s_body[depth];
    CU(cudaStreamBeginCaptureToGraph(side, p.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    H->stream = side;
    const int rc = body();
    H->stream = outer;
    cudaGraph_t captured = nullptr;
    const cudaError_t e = cudaStreamEndCapture(side, &captured);
    if (rc < 0) return -1;
    if (e != cudaSuccess) return fail("cudaStreamEndCapture (conditional node body): %s", cudaGetErrorString(e));
    CU(cudaStreamUpdateCaptureDependencies(outer, &node, 1, cudaStreamSetCaptureDependencies));
    return 0;
}

// The rounds of cond_rounds as a WHILE node: cond_init, then per round the IF node of the round's kase (apply(kase, &x), the
// counter reset and the step kernels of that kase; launch_cond_step takes its kase as an argument) and the decision.  Enqueued
// on H->stream, which is capturing.  Returns the launches (each body counted once), < 0 on an error.
template <class Apply>
static int cond_loop(slu_b200_handle_t H, int n, int members, val_t *v, Apply apply)
{
    int launches = launch_cond_init(H->d_cstate.p, v, n, members, H->stream);
    cudaGraphConditionalHandle w;
    if (cond_handle(H, &w)) return -1;
    launches += launch_cond_continue(H->d_ccount.p, H->d_cloop.p, 1, COND_MAX_ROUNDS, w, H->stream);
    const int rc = add_conditional(H, cudaGraphCondTypeWhile, w, 0, [&]() -> int {
        cudaGraphConditionalHandle k[2];
        if (cond_handle(H, &k[0]) || cond_handle(H, &k[1])) return -1;
        launches += launch_cond_select(H->d_cloop.p, k[0], k[1], H->stream);
        for (int kase = 1; kase <= 2; ++kase)
            if (add_conditional(H, cudaGraphCondTypeIf, k[kase - 1], 1, [&]() -> int {
                    val_t *x = nullptr;
                    const int l = apply(kase, &x);
                    if (l < 0) return -1;
                    CU(cudaMemsetAsync(H->d_ccount.p, 0, 2 * sizeof(int), H->stream));
                    launches += l + launch_cond_step(H->d_cstate.p, kase, x, v, H->d_csgn.p, H->d_cpart.p, H->d_ccount.p, n, members, H->stream);
                    return 0;
                }))
                return -1;
        launches += launch_cond_continue(H->d_ccount.p, H->d_cloop.p, 0, COND_MAX_ROUNDS, w, H->stream);
        return 0;
    });
    return rc < 0 ? -1 : launches;
}

// Runs enqueue() (a call's device work on H->stream, returning its launches) after stream_enter.  Under the caller's capture
// (cap) it goes into the caller's graph.  Otherwise the graph captured from it for this key is launched on H->stream, captured
// and instantiated first if there is none or if one of the buffer addresses it holds (bufs) has changed since.
template <class Enqueue>
static int run_loop(slu_b200_handle_t H, bool cap, const std::array<int, 4> &key, const std::vector<uintptr_t> &bufs, Enqueue enqueue)
{
    if (cap) return enqueue();
    auto it = std::find_if(H->loop_graphs.begin(), H->loop_graphs.end(), [&](const slu_b200_handle_s::LoopGraph &g) { return g.key == key; });
    if (it != H->loop_graphs.end() && it->bufs != bufs) {        // a buffer moved: capture again
        cudaGraphExecDestroy(it->exec);
        cudaGraphDestroy(it->graph);
        H->loop_graphs.erase(it);
        it = H->loop_graphs.end();
    }
    if (it == H->loop_graphs.end()) {
        CU(cudaStreamBeginCapture(H->stream, cudaStreamCaptureModeThreadLocal));
        const int launches = enqueue();
        cudaGraph_t graph = nullptr;
        const cudaError_t e = cudaStreamEndCapture(H->stream, &graph);
        if (launches < 0 || e != cudaSuccess) {
            if (graph) cudaGraphDestroy(graph);
            return launches < 0 ? -1 : fail("cudaStreamEndCapture: %s", cudaGetErrorString(e));
        }
        cudaGraphExec_t exec = nullptr;
        const cudaError_t ei = cudaGraphInstantiate(&exec, graph, 0);
        if (ei != cudaSuccess) {
            cudaGraphDestroy(graph);
            return fail("cudaGraphInstantiate: %s", cudaGetErrorString(ei));
        }
        H->loop_graphs.push_back({key, bufs, graph, exec, launches});
        it = H->loop_graphs.end() - 1;
    }
    CU(cudaGraphLaunch(it->exec, H->stream));
    return it->launches;
}

// the side streams of the conditional bodies, created outside capture by a call's first use
static int body_streams(slu_b200_handle_t H, bool cap, const char *fn)
{
    if (H->s_body[0]) return 0;
    if (cap) return fail("%s would create streams while the stream is capturing a CUDA graph: make this call once outside capture first", fn);
    for (auto &s : H->s_body) CU(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    return 0;
}

// gsrfs's loop for x in d_rx and b in d_rb, results in d_rx, d_rout (berr, then ferr) and d_rsteps: gsrfs's pieces, the steps
// in a WHILE node and (ferr) dgerfs's estimate in cond_loop, then the guard of x.  Enqueued on H->stream, capturing.
static int gsrfs_loop(slu_b200_handle_t H, bool batched, int nrhs, bool ferr)
{
    const RefineArgs a = refine_args(H, batched, nrhs, ferr);
    int launches = refine_init(H, a);
    const int lc = refine_check(H, a, batched);
    if (lc < 0) return -1;
    launches += lc;
    cudaGraphConditionalHandle w;
    if (cond_handle(H, &w)) return -1;
    launches += launch_refine_continue(H->d_ract.p, w, H->stream);
    if (add_conditional(H, cudaGraphCondTypeWhile, w, 0, [&]() -> int {
            const int ls = refine_step(H, a, batched);
            const int l = ls < 0 ? -1 : refine_check(H, a, batched);
            if (l < 0) return -1;
            launches += ls + l + launch_refine_continue(H->d_ract.p, w, H->stream);
            return 0;
        }))
        return -1;
    if (ferr) {
        auto apply = [&](int kase, val_t **res) { return refine_ferr_apply(H, batched, nrhs, kase, res); };
        const int l = cond_loop(H, H->n, a.nrhs * a.members, H->d_cv.p, apply);
        if (l < 0) return -1;
        launches += l;
    }
    const int le = refine_end(H, a, ferr);
    if (le < 0) return -1;
    return launches + le + launch_solve_guard(H->d_rx.p, H->d_info.p, (int64_t)H->n * nrhs, a.members, H->stream);
}

// gscon's rounds for every member, anorm in d_canorm, rcond into d_crcond.  Capturing, on H->stream.
static int gscon_loop(slu_b200_handle_t H, bool batched, bool one)
{
    const int B = batched ? H->batch : 1;
    auto apply = [&](int kase, val_t **x) { return gscon_apply(H, batched, one, kase, x); };
    const int l = cond_loop(H, H->n, B, gscon_v(H, batched), apply);
    if (l < 0) return -1;
    return l + launch_cond_rcond(H->d_cstate.p, H->d_canorm.p, H->d_info.p, B, H->d_crcond.p, H->stream);
}
extern "C" {

// gsrfs / batch_gsrfs on device b, x and outputs, ordered on the caller's stream (see the section comment above)
static int gsrfs_device_impl(slu_b200_handle_t H, bool batched, const double *bd, int ldb, double *xd, int ldx, int nrhs, double *berr,
                             double *ferr, int32_t *steps, void *stream, const char *fn)
{
    if (!H || !bd || !xd || !berr) return fail("%s: null argument (b, x and berr are required)", fn);
    if (gsrfs_check(H, fn, scaled_need(batched) | SCALED | FACTORED | DEVICE_ORDERED, ldb, ldx, nrhs)) return -1;
    const int B = batched ? H->batch : 1, n = H->n;
    if (check_device_ptr(H, bd, fn, "b") || check_device_ptr(H, xd, fn, "x") || check_device_ptr(H, berr, fn, "berr") ||
        (ferr && check_device_ptr(H, ferr, fn, "ferr")) || (steps && check_device_ptr(H, steps, fn, "steps")))
        return -1;
    if (conditional_nodes_check(fn)) return -1;
    const cudaStream_t caller = (cudaStream_t)stream;
    const int cap = capturing(H, caller, fn);
    if (cap < 0) return -1;
    const int cols = B * nrhs;
    if (refine_buffers(H, (size_t)n * cols, cols, ferr != nullptr, cap, fn) || grow_loop(H, H->d_cloop, 2, cap, fn) || body_streams(H, cap, fn))
        return -1;
    H->loop_captured = H->loop_captured || cap;
    if (stream_enter(H, caller, cap)) return -1;
    const size_t w = (size_t)n * sizeof(val_t);
    CU(cudaMemcpy2DAsync(H->d_rb.p, w, bd, (size_t)ldb * sizeof(val_t), w, (size_t)cols, cudaMemcpyDeviceToDevice, H->stream));
    CU(cudaMemcpy2DAsync(H->d_rx.p, w, xd, (size_t)ldx * sizeof(val_t), w, (size_t)cols, cudaMemcpyDeviceToDevice, H->stream));
    const std::vector<uintptr_t> bufs = {
        (uintptr_t)H->d_x.p, (uintptr_t)H->d_x2.p, (uintptr_t)H->d_rb.p, (uintptr_t)H->d_rx.p, (uintptr_t)H->d_rst.p, (uintptr_t)H->d_ract.p,
        (uintptr_t)H->d_rw.p, (uintptr_t)H->d_cv.p, (uintptr_t)H->d_csgn.p, (uintptr_t)H->d_cstate.p, (uintptr_t)H->d_cpart.p,
        (uintptr_t)H->d_ccount.p, (uintptr_t)H->d_cloop.p, (uintptr_t)H->d_rout.p, (uintptr_t)H->d_rsteps.p, (uintptr_t)H->d_rxmax.p,
        (uintptr_t)H->d_arp.p, (uintptr_t)H->d_aci.p, (uintptr_t)H->d_aci.n, (uintptr_t)H->d_aval.p, (uintptr_t)H->d_R.p,
        (uintptr_t)H->d_C.p, (uintptr_t)H->d_rmap.p, (uintptr_t)H->d_cperm.p, (uintptr_t)H->d_info.p};
    const int launches = run_loop(H, cap, {0, batched, nrhs, ferr != nullptr}, bufs, [&] { return gsrfs_loop(H, batched, nrhs, ferr != nullptr); });
    if (launches < 0) return -1;
    cudaStream_t s = H->stream;
    CU(cudaMemcpy2DAsync(xd, (size_t)ldx * sizeof(val_t), H->d_rx.p, w, w, (size_t)cols, cudaMemcpyDeviceToDevice, s));
    CU(cudaMemcpyAsync(berr, H->d_rout.p, (size_t)cols * sizeof(double), cudaMemcpyDeviceToDevice, s));
    if (ferr) CU(cudaMemcpyAsync(ferr, H->d_rout.p + cols, (size_t)cols * sizeof(double), cudaMemcpyDeviceToDevice, s));
    if (steps) CU(cudaMemcpyAsync(steps, H->d_rsteps.p, (size_t)cols * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    if (stream_leave(H, caller)) return -1;
    H->st.reserved[4] = 0;
    H->st.reserved[5] = (double)launches;
    return 0;
}

// gscon / batch_gscon with device anorm and rcond (one per member), ordered on the caller's stream
static int gscon_device_impl(slu_b200_handle_t H, bool batched, char norm, const double *anorm, double *rcond, void *stream, const char *fn)
{
    if (!H || !anorm || !rcond) return fail("%s: null argument", fn);
    if (check(H, fn, scaled_need(batched) | FACTORED | DEVICE_ORDERED)) return -1;
    const bool one = norm == '1' || norm == 'O' || norm == 'o';
    if (!one && norm != 'I' && norm != 'i')
        return fail("%s: norm must be '1', 'O' or 'I' (got character code %d)", fn, (int)(unsigned char)norm);
    if (check_device_ptr(H, anorm, fn, "anorm") || check_device_ptr(H, rcond, fn, "rcond")) return -1;
    if (conditional_nodes_check(fn)) return -1;
    const cudaStream_t caller = (cudaStream_t)stream;
    const int cap = capturing(H, caller, fn);
    if (cap < 0) return -1;
    const int B = batched ? H->batch : 1;
    if (gscon_buffers(H, batched, cap, fn) || grow_loop(H, H->d_cloop, 2, cap, fn) || body_streams(H, cap, fn)) return -1;
    H->loop_captured = H->loop_captured || cap;
    if (stream_enter(H, caller, cap)) return -1;
    CU(cudaMemcpyAsync(H->d_canorm.p, anorm, (size_t)B * sizeof(double), cudaMemcpyDeviceToDevice, H->stream));
    const std::vector<uintptr_t> bufs = {
        (uintptr_t)H->d_x.p, (uintptr_t)H->d_x2.p, (uintptr_t)H->d_cv.p, (uintptr_t)H->d_csgn.p, (uintptr_t)H->d_cstate.p,
        (uintptr_t)H->d_cpart.p, (uintptr_t)H->d_ccount.p, (uintptr_t)H->d_cloop.p, (uintptr_t)H->d_canorm.p, (uintptr_t)H->d_crcond.p,
        (uintptr_t)H->d_info.p};
    const int launches = run_loop(H, cap, {1, batched, 1, one}, bufs, [&] { return gscon_loop(H, batched, one); });
    if (launches < 0) return -1;
    CU(cudaMemcpyAsync(rcond, H->d_crcond.p, (size_t)B * sizeof(double), cudaMemcpyDeviceToDevice, H->stream));
    if (stream_leave(H, caller)) return -1;
    H->st.reserved[4] = 0;
    H->st.reserved[5] = (double)launches;
    H->st.reserved[6] = 0;
    H->st.reserved[7] = 0;
    return 0;
}

int slu_b200_gsrfs_device(slu_b200_handle_t H, const double *b, int ldb, double *x, int ldx, int nrhs, double *berr, double *ferr,
                          int32_t *steps, void *stream)
{
    return gsrfs_device_impl(H, false, b, ldb, x, ldx, nrhs, berr, ferr, steps, stream, SLU_API "gsrfs_device");
}

int slu_b200_batch_gsrfs_device(slu_b200_handle_t H, const double *b, int ldb, double *x, int ldx, int nrhs, double *berr, double *ferr,
                                int32_t *steps, void *stream)
{
    return gsrfs_device_impl(H, true, b, ldb, x, ldx, nrhs, berr, ferr, steps, stream, SLU_API "batch_gsrfs_device");
}

int slu_b200_gscon_device(slu_b200_handle_t H, char norm, const double *anorm, double *rcond, void *stream)
{
    return gscon_device_impl(H, false, norm, anorm, rcond, stream, SLU_API "gscon_device");
}

int slu_b200_batch_gscon_device(slu_b200_handle_t H, char norm, const double *anorm, double *rcond, void *stream)
{
    return gscon_device_impl(H, true, norm, anorm, rcond, stream, SLU_API "batch_gscon_device");
}

int slu_b200_get_device(slu_b200_handle_t H, int *device)
{
    if (!H || !device) return fail(SLU_API "get_device: null argument");
    *device = H->device;
    return 0;
}

int slu_b200_factor_device(slu_b200_handle_t H, int32_t *info, void *stream)
{
    return factor_device_impl(H, false, info, stream, SLU_API "factor_device");
}

int slu_b200_batch_factor_device(slu_b200_handle_t H, int32_t *info, void *stream)
{
    return factor_device_impl(H, true, info, stream, SLU_API "batch_factor_device");
}

int slu_b200_refill(slu_b200_handle_t H, const double *val, void *stream)
{
    return refill_impl(H, false, val, stream, SLU_API "refill");
}

int slu_b200_batch_refill(slu_b200_handle_t H, const double *val, void *stream)
{
    return refill_impl(H, true, val, stream, SLU_API "batch_refill");
}

int slu_b200_solve_device(slu_b200_handle_t H, double *x, int ldx, int nrhs, int trans, void *stream)
{
    return solve_device_impl(H, false, false, x, ldx, nrhs, trans, stream, SLU_API "solve_device");
}

int slu_b200_batch_solve_device(slu_b200_handle_t H, double *x, int ldx, int nrhs, int trans, void *stream)
{
    return solve_device_impl(H, true, false, x, ldx, nrhs, trans, stream, SLU_API "batch_solve_device");
}

int slu_b200_solve_scaled_device(slu_b200_handle_t H, double *x, int ldx, int nrhs, int trans, void *stream)
{
    return solve_device_impl(H, false, true, x, ldx, nrhs, trans, stream, SLU_API "solve_scaled_device");
}

int slu_b200_batch_solve_scaled_device(slu_b200_handle_t H, double *x, int ldx, int nrhs, int trans, void *stream)
{
    return solve_device_impl(H, true, true, x, ldx, nrhs, trans, stream, SLU_API "batch_solve_scaled_device");
}

// ---- partial factorization on batched handles: a batched handle whose level plan leaves out the Schur supernodes, as an
// unbatched Schur handle's does.  batch_factor eliminates A11 of every member, the gather runs over (units, members), and
// condense / expand are the forward / backward pass of solve_host over the same plan.
int slu_b200_batch_schur_create(slu_b200_handle_t *out, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, int batch,
                                int nschur)
{
    if (!out || !lu || !opt) return fail("null argument");
    *out = nullptr;
    const char *fn = SLU_API "batch_schur_create";
    if (batch_create_check(lu, opt, batch, fn)) return -1;
    if (nschur < 1 || nschur >= lu->n) return fail("%s: nschur = %d, must satisfy 1 <= nschur < n = %d", fn, nschur, lu->n);
    return create_impl(out, lu, opt, batch, nschur);
}

// S: batch blocks of s x s, member j's at S + j * lds * s
int slu_b200_batch_schur_get(slu_b200_handle_t H, double *S, int lds)
{
    if (!H || !S) return fail("null argument");
    const char *fn = SLU_API "batch_schur_get";
    if (check(H, fn, BATCHED | SCHUR | FACTORED)) return -1;
    return schur_get_impl(H, S, lds, fn);
}

int slu_b200_batch_schur_condense(slu_b200_handle_t H, double *x, int ldx, int nrhs)
{
    return solve_host(H, SLU_API "batch_schur_condense", BATCHED | SCHUR | FACTORED, x, ldx, nrhs, 0, PASS_FORWARD);
}

int slu_b200_batch_schur_expand(slu_b200_handle_t H, double *x, int ldx, int nrhs)
{
    return solve_host(H, SLU_API "batch_schur_expand", BATCHED | SCHUR | FACTORED, x, ldx, nrhs, 0, PASS_BACKWARD);
}

int slu_b200_get_stats(slu_b200_handle_t H, slu_b200_stats_t *out)
{
    if (!H || !out) return fail("null argument");
    if (settle(H)) return -1;
    *out = H->st;
    return 0;
}

int pdgstrf3d_b200(const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, slu_b200_stats_t *stats, int *info)
{
    slu_b200_handle_t H = nullptr;
    if (slu_b200_create(&H, lu, opt)) return -1;
    int rc;
    if (opt->reserved[2]) {
        rc = slu_b200_factor_host(H, info);   // overlapped H2D / factor / D2H
    } else {
        rc = slu_b200_upload(H);
        if (!rc) rc = slu_b200_factor(H, info);
        if (!rc) rc = slu_b200_download(H);
    }
    if (stats) *stats = H->st;
    slu_b200_destroy(H);
    return rc;
}

// Analysis only, no device needed: HBM bytes, flops in the reference's accounting, level count ... for one rank of a
// 1 x 1 x Pz grid -- what a caller needs to size a run for 180 GB GPUs before it allocates them.  Also checks the
// level-by-level layout that the overlapped upload (options.reserved[3]) relies on.
static int plan_impl(const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, slu_b200_stats_t *stats, double *merge)
{
    if (!lu || !opt || !stats) return fail("null argument");
    if (opt->schur_variant != 0) return fail("options.schur_variant is retired and must be 0 (got %d)", opt->schur_variant);
    if (lu->nprow * lu->npcol != 1) return fail("slu_b200_plan handles 1 x 1 x Pz grids (a Pr x Pc layer needs its peers' index pieces)");
    struct Guard { Guard() { g_plan_only = true; } ~Guard() { g_plan_only = false; } } guard;
    slu_b200_handle_s *H = new slu_b200_handle_s;
    H->view = *lu;
    H->opt = *opt;
    H->coop = opt->world_size > 1 && !opt->reserved[1];
    H->P2 = 1;
    int rc = (gather_structure(H) || analyze(H)) ? -1 : 0;
    if (!rc && H->grouped)
        for (size_t li = 0; li < H->levels.size() && !rc; ++li) {
            const LevelPlan &L = H->levels[li];
            const int32_t *nodes = H->h_pool_i32.data() + L.nodes_off;
            int64_t off = L.slab_begin;
            for (int pass = 0; pass < 2 && !rc; ++pass)
                for (int t = 0; t < L.count; ++t) {
                    const NodeDesc &nd = H->nodes[nodes[t]];
                    const int64_t dev = pass ? nd.uval : nd.lval;
                    const int64_t len = pass ? (int64_t)nd.ns * nd.ncols : (int64_t)nd.nsupr * nd.ns;
                    if (len <= 0) continue;
                    if (dev != off) { rc = fail("level %zu is not contiguous in the arena", li); break; }
                    off += len;
                }
            if (!rc && off != L.slab_end) rc = fail("level %zu: slab end mismatch", li);
        }
    if (!rc) *stats = H->st;
    if (!rc && merge) std::copy(H->merge, H->merge + 3, merge);
    delete H;
    return rc;
}
int slu_b200_plan(const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, slu_b200_stats_t *stats)
{
    return plan_impl(lu, opt, stats, nullptr);
}
#ifndef SLU_COMPLEX
int slu_b200_k_schur_merge(const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, double out[3])
{
    if (!out) return fail("null argument");
    slu_b200_stats_t st{};
    return plan_impl(lu, opt, &st, out);
}
#endif

// ---- kernel-level entry points -----------------------------------------------------------------
namespace {
struct MiniLU {  // a one-supernode DeviceLU around a caller-provided block
    DevBuf<val_t> val;
    DevBuf<NodeDesc> nodes;
    DevBuf<int32_t> ids;
    DevBuf<int64_t> prefix;
    DevBuf<int> flags;
    DevBuf<unsigned long long> tiny;
    DevBuf<val_t> inv;
    DeviceLU d{};
    int init(const NodeDesc &nd, size_t nval, const std::vector<int64_t> &pre)
    {
        if (val.alloc(nval) || nodes.upload(std::vector<NodeDesc>{nd}) || ids.upload(std::vector<int32_t>{0}) ||
            prefix.upload(pre) || flags.alloc(2) || tiny.alloc(1))
            return -1;
        int init[2] = {INT_MAX, 0};
        cudaMemcpy(flags.p, init, sizeof init, cudaMemcpyHostToDevice);
        cudaMemset(tiny.p, 0, 8);
        d.val = val.p; d.nodes = nodes.p; d.info = flags.p; d.err = flags.p + 1; d.tiny = tiny.p;
        return 0;
    }
    ~MiniLU() { val.release(); nodes.release(); ids.release(); prefix.release(); flags.release(); tiny.release(); inv.release(); }
};
}  // namespace

int slu_b200_k_diag_lu(double *a, int ns, int lda, int replace_tiny, double thresh, int col0, int *info, int *tiny)
{
    if (slu_b200_device_count() < 1) return fail("no CUDA device");
    if (ns < 1 || ns > MAX_NS_HELD || lda < ns) return fail("bad size");
    MiniLU M;
    NodeDesc nd{}; nd.held = 1; nd.ns = ns; nd.nsupr = lda; nd.fsupc = col0; nd.lval = 0;
    if (M.init(nd, (size_t)lda * ns, {0, 1})) return -1;
    CU(cudaMemcpy(M.val.p, a, (size_t)lda * ns * sizeof(val_t), cudaMemcpyHostToDevice));
    launch_diag_lu(M.d, Batch{M.ids.p, M.prefix.p, 1}, ns, replace_tiny, thresh, 0);
    CU(cudaDeviceSynchronize());
    CU(cudaGetLastError());
    CU(cudaMemcpy(a, M.val.p, (size_t)lda * ns * sizeof(val_t), cudaMemcpyDeviceToHost));
    int flags[2]; unsigned long long t;
    CU(cudaMemcpy(flags, M.flags.p, sizeof flags, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&t, M.tiny.p, 8, cudaMemcpyDeviceToHost));
    if (info) *info = flags[0] == INT_MAX ? 0 : flags[0];
    if (tiny) *tiny = (int)t;
    return 0;
}

static int k_trsm(bool ucase, const double *lu_, int ldlu, int ns, double *x_, int nvec, int ldx)
{
    const val_t *lu = (const val_t *)lu_;
    val_t *x = (val_t *)x_;
    if (slu_b200_device_count() < 1) return fail("no CUDA device");
    if (ns < 1 || ns > MAX_NS_HELD || ldlu < ns || nvec < 0) return fail("bad size");
    // assemble a panel: L case [diag (ns rows) ; x (m rows)] with lda = ns + m; U case diag + packed U
    MiniLU M;
    NodeDesc nd{}; nd.held = 1; nd.ns = ns; nd.lval = 0;
    size_t nval;
    std::vector<val_t> h;
    if (!ucase) {
        nd.nsupr = ns + nvec; nd.m = nvec;
        nval = (size_t)nd.nsupr * ns;
        h.assign(nval, val_t{});
        for (int c = 0; c < ns; ++c) {
            for (int r = 0; r < ns; ++r) h[(size_t)c * nd.nsupr + r] = lu[(size_t)c * ldlu + r];
            for (int r = 0; r < nvec; ++r) h[(size_t)c * nd.nsupr + ns + r] = x[(size_t)c * ldx + r];
        }
    } else {
        nd.nsupr = ns; nd.m = 0; nd.ncols = nvec; nd.uval = (int64_t)ns * ns;
        nval = (size_t)ns * ns + (size_t)ns * nvec;
        h.assign(nval, val_t{});
        for (int c = 0; c < ns; ++c)
            for (int r = 0; r < ns; ++r) h[(size_t)c * ns + r] = lu[(size_t)c * ldlu + r];
        for (int c = 0; c < nvec; ++c)
            for (int r = 0; r < ns; ++r) h[(size_t)ns * ns + (size_t)c * ns + r] = x[(size_t)c * ldx + r];
    }
    int64_t ctas = (nvec + TRSM_STRIP - 1) / TRSM_STRIP;
    if (M.init(nd, nval, {0, ctas})) return -1;
    CU(cudaMemcpy(M.val.p, h.data(), nval * sizeof(val_t), cudaMemcpyHostToDevice));
    Batch b{M.ids.p, M.prefix.p, 1};
    const int nb16 = (ns + 15) / 16;
    DevBuf<int64_t> pinv;
    if (M.inv.alloc((size_t)nb16 * 512) || pinv.upload(std::vector<int64_t>{0, nb16})) return -1;
    launch_diag_inv(M.d, Batch{M.ids.p, pinv.p, 1}, nb16, M.inv.p, 0);
    if (ucase) launch_trsm_u(M.d, b, ctas, ns, M.inv.p, 0); else launch_trsm_l(M.d, b, ctas, ns, M.inv.p, 0);
    CU(cudaDeviceSynchronize());
    pinv.release();
    CU(cudaDeviceSynchronize());
    CU(cudaGetLastError());
    CU(cudaMemcpy(h.data(), M.val.p, nval * sizeof(val_t), cudaMemcpyDeviceToHost));
    if (!ucase) {
        for (int c = 0; c < ns; ++c)
            for (int r = 0; r < nvec; ++r) x[(size_t)c * ldx + r] = h[(size_t)c * nd.nsupr + ns + r];
    } else {
        for (int c = 0; c < nvec; ++c)
            for (int r = 0; r < ns; ++r) x[(size_t)c * ldx + r] = h[(size_t)ns * ns + (size_t)c * ns + r];
    }
    return 0;
}
int slu_b200_k_trsm_l(const double *lu, int ldlu, int ns, double *x, int m, int ldx) { return k_trsm(false, lu, ldlu, ns, x, m, ldx); }
int slu_b200_k_trsm_u(const double *lu, int ldlu, int ns, double *x, int ncols, int ldx) { return k_trsm(true, lu, ldlu, ns, x, ncols, ldx); }

int slu_b200_k_gemm_sub(int m, int n, int k, const double *a, int lda, const double *b, int ldb, double *c, int ldc,
                        int reps, float *ms)
{
    const int variant = getenv("SLU_B200_GEMM_VARIANT") ? atoi(getenv("SLU_B200_GEMM_VARIANT")) : 0;
    if (slu_b200_device_count() < 1) return fail("no CUDA device");
    DevBuf<val_t> da, db, dc;
    if (da.alloc((size_t)lda * k) || db.alloc((size_t)ldb * n) || dc.alloc((size_t)ldc * n)) return -1;
    CU(cudaMemcpy(da.p, a, (size_t)lda * k * sizeof(val_t), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(db.p, b, (size_t)ldb * n * sizeof(val_t), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(dc.p, c, (size_t)ldc * n * sizeof(val_t), cudaMemcpyHostToDevice));
    EventSet ev;
    if (ev.create()) return fail("cannot create events");
    cudaEvent_t e0 = ev[0], e1 = ev[1];
#ifndef SLU_COMPLEX
    std::function<int(int, int, int, const val_t *, int, const val_t *, int, val_t *, int, int, cudaStream_t)> launch_gemm_sub =
        [](int m_, int n_, int k_, const val_t *a_, int lda_, const val_t *b_, int ldb_, val_t *c_, int ldc_, int variant_, cudaStream_t s_) {
        if (variant_ >= 100) return launch_gemm_sub_ozaki(m_, n_, k_, a_, lda_, b_, ldb_, c_, ldc_, variant_, s_);
        return SLU_NS::launch_gemm_sub(m_, n_, k_, a_, lda_, b_, ldb_, c_, ldc_, variant_, s_);
    };
    if (variant >= 100 && k > 512) return fail("the int8 tensor-core path handles k <= 512 (MAX_SUPER_SIZE)");
    // variant 35: schur_kernel_h's segmented K loop; K cut into three segments (k1 = k / 3 | 1, k2 = k / 3, the rest), the
    // second and third repacked with leading dimensions lda + 2q + 1 and their own depth + q + 1 (operands after da / db)
    DevBuf<val_t> dseg;
    DevBuf<KSeg> dks;
    if (variant == 35) {
        const int k1 = std::min(k, (k / 3) | 1), k2 = std::min(k - k1, k / 3), kq[3] = {k1, k2, k - k1 - k2};
        std::vector<KSeg> ks;
        std::vector<val_t> h;
        int kstart = k1;
        for (int q = 1; q < 3; ++q) {
            const int la = lda + 2 * q + 1, lb = kq[q] + q + 1;
            if (kq[q] <= 0) continue;
            KSeg g{(int64_t)h.size(), 0, la, lb, kq[q], 0};
            h.resize(h.size() + (size_t)la * kq[q], 0.0);
            for (int c = 0; c < kq[q]; ++c)
                for (int r = 0; r < m; ++r) h[g.a + (size_t)c * la + r] = a[(size_t)(kstart + c) * lda + r];
            g.b = (int64_t)h.size();
            h.resize(h.size() + (size_t)lb * n, 0.0);
            for (int c = 0; c < n; ++c)
                for (int r = 0; r < kq[q]; ++r) h[g.b + (size_t)c * lb + r] = b[(size_t)c * ldb + kstart + r];
            ks.push_back(g);
            kstart += kq[q];
        }
        if (dseg.upload(h) || dks.upload(ks)) return -1;
        // k1 and the segment count by value: the launcher outlives this block (timed repetitions below)
        launch_gemm_sub = [k1, nks = (int)ks.size(), &dseg, &dks](int m_, int n_, int, const val_t *a_, int lda_, const val_t *b_, int ldb_,
                                                                 val_t *c_, int ldc_, int, cudaStream_t s_) {
            return launch_gemm_sub_seg(m_, n_, k1, a_, lda_, b_, ldb_, dseg.p, dks.p, nks, c_, ldc_, s_);
        };
    }
#endif
    launch_gemm_sub(m, n, k, da.p, lda, db.p, ldb, dc.p, ldc, variant, 0);
    CU(cudaDeviceSynchronize());
    CU(cudaGetLastError());
    CU(cudaMemcpy(c, dc.p, (size_t)ldc * n * sizeof(val_t), cudaMemcpyDeviceToHost));
    if (reps > 0) {
        cudaEventRecord(e0, 0);
        for (int r = 0; r < reps; ++r) launch_gemm_sub(m, n, k, da.p, lda, db.p, ldb, dc.p, ldc, variant, 0);
        cudaEventRecord(e1, 0);
        CU(cudaEventSynchronize(e1));
        float t = 0;
        cudaEventElapsedTime(&t, e0, e1);
        if (ms) *ms = t / reps;
    }
    return 0;
}

}  // extern "C"
