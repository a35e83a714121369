// slu_device.cuh -- data structures shared by the host orchestration (slu_api.cu) and the sm_90a
// kernels (slu_kernels.cu) of libslu_b200.so.
//
// HBM layout (DESIGN.md section 3).  One value arena `val` (double) holds, per Z-tree level of the
// forests this rank owns, first the L panels then the U panels of that forest:
//   L panel k : column-major nsupr x ns, lda = nsupr  -- byte-identical to Lnzval_bc_ptr[k]
//               (SRC/include/superlu_defs.h:156-178), so upload/download of L is a plain copy;
//   U panel k : DENSE-PACKED ns x ncols, ld = ns: only the columns with a non-empty skyline segment,
//               zero-padded above the segment.  This is the GEMM-ready form the reference re-creates
//               for every supernode in dRgather_U (SRC/double/dgather.c:256-398); here it is the
//               resident form and is converted from/to the skyline of Unzval_br_ptr[k] only at
//               upload/download.
// Index arenas (int32): per L panel the row ids in panel order (`lrows`) and a sorted copy with the
// panel position of each (`lsrow`,`lspos`) for destination lookups; per U panel the sorted global
// column ids of its packed columns (`ucols`) with first-nonzero row (`ufst`) and skyline offset
// (`useg`).
//
// The header (and slu_api.cu) is compiled twice: as is for double (namespace slu, pdgstrf3d) and with SLU_COMPLEX
// for doublecomplex (namespace sluz, pzgstrf3d; SURVEY 8a row a15: "identical algorithm on interleaved (r,i)
// pairs").  All offsets and lengths count ELEMENTS of val_t, so the host orchestration is the same source.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#ifdef SLU_COMPLEX
#define SLU_NS sluz
#else
#define SLU_NS slu
#endif

namespace SLU_NS {

#ifdef SLU_COMPLEX
typedef double2 val_t;       // (re, im) = the reference's doublecomplex, SRC/include/dcomplex.h:30
#else
typedef double val_t;
#endif
constexpr int VAL_DOUBLES = (int)(sizeof(val_t) / sizeof(double));

struct NodeDesc {            // one per supernode (indexed by global supernode id); zero if not held
    int32_t held, ns, nsupr, m, ncols, nlb, nub, fsupc;
    int64_t lval, uval;      // offsets into val (elements)
    int64_t lrow, ucol;      // offsets into lrows/lsrow/lspos and ucols/ufst/useg
    int64_t lblk, ublk;      // offsets into the LBlk / UBlk arrays
    int64_t ws_row, ws_col;  // offsets into the per-level rowinfo / colinfo workspace
    int64_t ws_lrel, ws_urel;
    int64_t lrel_total, urel_total;
    int64_t ws_inv;          // offset into the per-level workspace of inverted 16x16 diagonal blocks
    int32_t urg_rows, urg_cols;  // look-ahead: leading rows / packed columns whose destination is factored at
                                 // the NEXT level (the parent supernode); tiles touching them are "urgent"
    // int8 tensor-core path (slu_ozaki.cu): per-level workspace of this supernode's int8 slices and scales
    int64_t ws_oza, ws_ozb;      // byte offsets into oz_i8: A tiles [rt][ks][s][4096], B tiles [ct][ks][s][OZ_NT*32]
    int64_t ws_ozs;              // element offset into oz_scale / oz_rexp: row scales [0, 128*RT), column scales after
    // deferred Schur updates along supernode chains (DESIGN 4a): kseg[kseg_off ...] = the nkseg K segments of nested
    // children that this supernode's update carries after its own; defer = 1: this supernode's update beyond the first
    // urg_rows rows and urg_cols columns (its parent's columns) is carried by its parent's update
    int64_t kseg_off;
    int32_t nkseg, defer;
};

// deferred Schur updates (DESIGN 4a): panels per GEMM when options.reserved[6] is 0, and the most it accepts
constexpr int SCHUR_DEPTH_DEFAULT = 4, SCHUR_DEPTH_MAX = 4;

struct KSeg {                // one K segment of a Schur GEMM: A = val + a (lda), B = val + b (ldb), depth k
    int64_t a, b;
    int32_t lda, ldb, k, pad;
};

struct LBlk {                // an off-diagonal L block of panel k
    int32_t ib, row0, nrows; // rows [row0, row0+nrows) of the m sub-diagonal rows
    int32_t colstart;        // first packed U column j of panel k with supno(col) > ib (U-destinations)
    int64_t urel_off;        // offset (within the node's urel table) of this block's column map
    int32_t shared, pad;     // 1: another supernode of the same level also updates panel ib (scatter must be atomic)
};
struct UBlk {                // a U block (packed columns [col0, col0+ncols)) of block row k
    int32_t jb, col0, ncols;
    int32_t rowstart;        // first sub-diagonal row i of panel k with supno(row) >= jb (L-destinations)
    int64_t lrel_off;
    int32_t shared, pad;     // 1: another supernode of the same level also updates panel jb
};

struct RowInfo {             // built per supernode by schur_setup_kernel
    int32_t ib, ldu;         // destination block row and its leading dimension (SuperSize(ib))
    int64_t ubase;           // val offset of element (row, first packed column) of U panel ib
    int64_t urel_off;        // urel[urel_off + j] = packed column position of source column j
    int32_t shared, pad;     // destination U panel ib is also updated by another supernode of this level
};
struct ColInfo {
    int32_t jb, pad;         // pad: 1 if destination L panel jb is also updated by another supernode of this level
    int64_t lbase;           // val offset of the top of destination column in L panel jb
    int64_t lrel_off;        // lrel[lrel_off + i] = row position of source row i in L panel jb
};

struct DeviceLU {            // everything the kernels need, passed by value
    val_t *val;
    const NodeDesc *nodes;
    const int32_t *xsup, *supno;
    const int32_t *lrows, *lsrow, *lspos;
    const int32_t *ucols, *ufst, *useg;
    const LBlk *lblk;
    const UBlk *ublk;
    RowInfo *rowinfo;
    ColInfo *colinfo;
    int32_t *lrel, *urel;
    int8_t *oz_i8;           // int8 tensor-core path: int8 slice tiles of the level's wide supernodes
    double *oz_scale;        //   2^(e-6) back-scales of their rows / columns
    int *oz_rexp;            //   row exponents (between the two slicing passes)
    int *info;               // min over zero pivots of (1-based global column); INT_MAX if none
    unsigned long long *tiny;
    int *err;                // debug: count of destination lookups that failed
    const KSeg *kseg;        // the K segments of deferred child updates (NodeDesc.kseg_off)
};

// Several matrices of one sparsity pattern factored together (slu_b200_batch_*): every structure-only object of
// DeviceLU is shared, each member has its own value arena, diag-inverse workspace and info flag.  A batched launch
// has the grid of the unbatched one in x and the member in blockIdx.y (member_view, slu_kernels_common.cuh).
struct BatchedLU : DeviceLU {
    int64_t val_stride;      // elements between the value arenas of two members (val = member 0)
    int64_t inv_stride;      // elements between their diag-inverse workspaces
    int32_t members, pad;    // info = [members] flags
};

struct Batch {               // one kernel launch over several supernodes
    const int32_t *nodes;    // supernode ids
    const int64_t *prefix;   // [count+1] cumulative CTA counts
    int32_t count;
};

constexpr int DIAG_NB = 16;
constexpr int TRSM_NB = 16;
constexpr int MAX_NS = 512;  // MAX_SUPER_SIZE, SRC/include/superlu_defs.h:154
constexpr int TRSM_STRIP = 32;       // vectors per TRSM CTA, every ns (the CTA prefix of a level batch is built with this)
#ifdef SLU_COMPLEX
constexpr int MAX_NS_HELD = 256;    // widest supernode the kernels accept (the default superlu_maxsup)
constexpr int SCHUR_BN_TILE = 32;   // columns of a big Schur tile (complex columns: 64 real ones)
#else
constexpr int MAX_NS_HELD = MAX_NS;  // MAX_SUPER_SIZE
constexpr int SCHUR_BN_TILE = 64;
#endif

// launchers (slu_kernels.cu).  Every launcher returns the number of kernels it launched.
// replace_tiny: 0 off, 1 replace and count in d.tiny, 2 replace without counting (replicated copy of a shared forest)
int launch_diag_lu(const DeviceLU &d, const Batch &b, int max_ns, int replace_tiny, double thresh,
                   cudaStream_t s);
// inverse of every 16x16 diagonal block of U_kk and L_kk: dinv[ws_inv + blk*512 + {0: inv U, 256: inv L}]
int launch_diag_inv(const DeviceLU &d, const Batch &b, int64_t ctas, val_t *dinv, cudaStream_t s);
int launch_trsm_l(const DeviceLU &d, const Batch &b, int64_t ctas, int max_ns, const val_t *dinv, cudaStream_t s);
int launch_trsm_u(const DeviceLU &d, const Batch &b, int64_t ctas, int max_ns, const val_t *dinv, cudaStream_t s);
int launch_schur_setup(const DeviceLU &d, const Batch &b, int64_t ctas, cudaStream_t s);
// big: SCHUR_BM_BIG x SCHUR_BN_TILE tiles (double: schur_kernel_h, DMMA.16x8x8, 2 CTAs/SM), else SCHUR_BM_SMALL x SCHUR_BN_SMALL
// mode 0: every tile of each supernode; 1: only the urgent tiles (urg_rows/urg_cols); 2: only the others
// split_n/split_i: this rank takes tiles t with t % split_n == split_i (cooperative ancestor forests)
int launch_schur(const DeviceLU &d, const Batch &b, int64_t ctas, int big, int mode, int split_n, int split_i, cudaStream_t s);
// skyline (sky + sky_off[slot]) <-> dense-packed U panel of each node of the batch; 32 columns per CTA
int launch_u_convert(const DeviceLU &d, const Batch &b, int64_t ctas, int pack, val_t *sky,
                     const int64_t *sky_off, cudaStream_t s);
int launch_axpy(val_t *dst, const val_t *src, int64_t n, cudaStream_t s);
// dst += src with atomic adds (overlapped upload: races with the Schur scatter into the same panels)
int launch_axpy_atomic(val_t *dst, const val_t *src, int64_t n, cudaStream_t s);
struct UpSeg { int64_t dst, src, len; };  // a transfer chunk: arena offset, (unused), length in elements
// standalone kernel tests
int launch_gemm_sub(int m, int n, int k, const val_t *a, int lda, const val_t *b, int ldb, val_t *c,
                    int ldc, int variant, cudaStream_t s);
#ifndef SLU_COMPLEX
// C -= A B + sum over q of A_q B_q on schur_kernel_h's tile and segmented K loop (A_q = base + seg[q].a, device array seg)
int launch_gemm_sub_seg(int m, int n, int k, const double *a, int lda, const double *b, int ldb, const double *base, const KSeg *seg,
                        int nseg, double *c, int ldc, cudaStream_t s);
#endif

// slu_solve.cu (double) / slu_solve_z.cu (doublecomplex): triangular solves on the resident factors.
// x: device, n x nrhs elements of val_t, ordering of the factored matrix.  trans: 0 solves A x = b (forward pass with L,
// backward with U; the update takes the L / U panel tiles), 1 A^T x = b and 2 A^H x = b (forward with U^T, backward with
// L^T; the update takes the U / L panel tiles); 2 is 1 in double.
constexpr int SOLVE_TILE = 256;
int launch_solve_diag(const DeviceLU &d, const int32_t *nodes, int count, bool backward, int trans, val_t *x, int n, int nrhs,
                      cudaStream_t s);
int launch_solve_update(const DeviceLU &d, const Batch &b, int64_t ctas, bool backward, int trans, val_t *x, int n, int nrhs,
                        cudaStream_t s);
// x[entries of the listed supernodes] = src[...] (src == nullptr: 0)
int launch_solve_mask(const DeviceLU &d, const int32_t *nodes, int count, val_t *x, int n, int nrhs, const val_t *src, cudaStream_t s);
// device-side distribution of a CSR matrix (device arrays) into the arena; *err counts entries without a slot
int launch_fill_csr(const DeviceLU &d, int n, const int32_t *rowptr, const int32_t *colind, const val_t *aval, const int32_t *perm,
                    const int8_t *active, int *err, cudaStream_t s);

// batched launches (both precisions): the same kernels over d.members matrices of one pattern (gridDim.y = members).
// dinv = member 0's workspace; in the solve x holds the members' n x nrhs blocks back to back, in fill_csr aval their
// nnz values.  Always the FP64 DMMA path: the int8 path is not batched.
int launch_diag_lu(const BatchedLU &d, const Batch &b, int max_ns, int replace_tiny, double thresh, cudaStream_t s);
int launch_diag_inv(const BatchedLU &d, const Batch &b, int64_t ctas, val_t *dinv, cudaStream_t s);
int launch_trsm_l(const BatchedLU &d, const Batch &b, int64_t ctas, int max_ns, const val_t *dinv, cudaStream_t s);
int launch_trsm_u(const BatchedLU &d, const Batch &b, int64_t ctas, int max_ns, const val_t *dinv, cudaStream_t s);
int launch_schur(const BatchedLU &d, const Batch &b, int64_t ctas, int big, int mode, cudaStream_t s);
int launch_solve_diag(const BatchedLU &d, const int32_t *nodes, int count, bool backward, int trans, val_t *x, int n, int nrhs,
                      cudaStream_t s);
int launch_solve_update(const BatchedLU &d, const Batch &b, int64_t ctas, bool backward, int trans, val_t *x, int n, int nrhs,
                        cudaStream_t s);
int launch_fill_csr(const BatchedLU &d, int n, const int32_t *rowptr, const int32_t *colind, const val_t *aval, const int32_t *perm,
                    const int8_t *active, int *err, cudaStream_t s);
// affine fill (slu_b200_batch_fill_affine), 2 launches: dst[p] = the arena offset of CSR entry p (the slot search of fill_csr,
// once per entry; -1 and a count in *err where it has no slot, -1 in a panel `active` leaves out), then member j's value of
// entry p, coef[j nterms] terms[p] + sum over t >= 1 of coef[j nterms + t] terms[t nnz + p] in that order, goes to its arena
// at dst[p]
int launch_fill_affine(const BatchedLU &d, int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm, const int8_t *active,
                       int64_t *dst, int64_t nnz, int nterms, const val_t *terms, const val_t *coef, int *err, cudaStream_t s);

// scaled, row-permuted fill (slu_b200_fill_csr_scaled and its batched / z twins): F = Pc Pr Dr A Dc Pc^T, entry (i, j) of A to
// F(rmap[i], perm[j]) with rmap = perm o perm_r, value (R[i] a_ij) C[j].  Per member: the equilibration reductions (bit
// patterns of non-negative doubles, which order as unsigned integers) and the norms of F.
struct EquilStat {
    unsigned long long rmin, rmax;   // min / max of the row maxima of |Pr Dr A Dc| (rmin starts at bignum, as dgsequ's rcmin)
    unsigned long long cmin, cmax;   // min / max of the column maxima of the row-scaled matrix
    unsigned long long fnorm, fmax;  // ||F||_inf and max |f_ij|
    int zrow, zcol;                  // smallest row / column of A that is exactly zero (INT_MAX: none)
};
struct ScaledFill {
    int n;
    const int32_t *rowptr, *colind, *rmap, *perm;
    const val_t *aval;                 // members x nnz values, member-major
    const double *R_in, *C_in;         // nullptr: ones; else rc_stride elements apart per member (0: shared)
    int64_t rc_stride;
    double *R, *C;                     // members x n: the final scalings
    double *rinv;                      // members x n scratch: dgsequ's row factors
    unsigned long long *ccol;          // members x n scratch: column maxima (bits)
    EquilStat *st;                     // [members]
    double *out;                       // members x 6 (slu_b200_fill_csr_scaled's out[0..3])
    const int8_t *active;
    int *err;                          // entries without a slot (member 0's count)
};
// equil: 4 launches (row maxima and column maxima, column reductions, the dgsequ / dlaqgs decision folded into R and C, the
// scatter with the norms); else 2 (R and C copied, the scatter).  Over (rows, members).
int launch_fill_scaled(const DeviceLU &d, const ScaledFill &f, bool equil, cudaStream_t s);
int launch_fill_scaled(const BatchedLU &d, const ScaledFill &f, bool equil, cudaStream_t s);
// refill of a scaled fill's pattern with new values (slu_b200_refill and its batched / z twins).  The slot map, once per
// scaled fill: slot[p] = the arena offset of CSR entry p at (rmap[i], perm[colind[p]]) (-1 without one), row[p] = its row i;
// 1 launch over rows.  The refill: member j's value a of entry p goes to its arena at slot[p] as (R[i] a) C[j], exactly the
// value of launch_fill_scaled's scatter, and to aval; 1 launch over (entries, members), no search.
int launch_refill_slots(const DeviceLU &d, int n, const int32_t *rowptr, const int32_t *colind, const int32_t *rmap, const int32_t *perm,
                        const int8_t *active, int64_t *slot, int32_t *row, cudaStream_t s);
struct Refill {
    int n;
    int64_t nnz;
    const val_t *val;                  // members x nnz new values, member-major
    const int64_t *slot;
    const int32_t *row, *colind;
    const double *R, *C;               // members x n: the kept scalings
    val_t *aval;                       // members x nnz: the kept A, receives val
};
int launch_refill(const DeviceLU &d, const Refill &r, cudaStream_t s);
int launch_refill(const BatchedLU &d, const Refill &r, cudaStream_t s);
// the status of a factorization on the device (slu_b200_factor_device and its batched / z twins), 1 launch each.  begin:
// flags[0 .. members) = INT_MAX, the error slot flags[members] = 0, *tiny = 0.  info: out[j] = status[j] = -1 if the error
// slot is not 0, else 0 or member j's first zero pivot (flags[j], 1-based), and ++*epoch.  guard: x holds members blocks of len elements;
// the block of every member whose status is not 0 becomes quiet NaN.
int launch_factor_begin(int *flags, int members, unsigned long long *tiny, cudaStream_t s);
int launch_factor_info(const int *flags, int members, int32_t *out, int32_t *status, unsigned long long *epoch, cudaStream_t s);
int launch_solve_guard(val_t *x, const int32_t *status, int64_t len, int members, cudaStream_t s);
// the vector transforms of slu_b200_solve_scaled, over (entries, members) with members blocks of n x nrhs (scale: n per
// member): scatter dst[map[i]] = scale[i] src[i], else gather dst[i] = scale[i] src[map[i]]
int launch_permute_scale(val_t *dst, const val_t *src, const int32_t *map, const double *scale, int n, int nrhs, int members,
                         bool scatter, cudaStream_t s);

// slu_cond.cu (double) / slu_cond_z.cu (doublecomplex): the step kernels of the dlacn2 / zlacn2 1-norm estimator
// (slu_b200_gscon).  One CondState per member: dlacn2's EST, ESTOLD and ISAVE(1..3) as phase, j, iter; kase = the solve
// the member waits for (1: with B, 2: with B^T / B^H, 0: done); act = the next vector its last step wrote.
// Vectors: `members` blocks of n elements back to back.
constexpr int COND_CHUNK = 2048;      // elements per CTA of the per-member reductions
enum { COND_NONE = 0, COND_EJ = 1, COND_SIGN = 2, COND_ALT = 3 };
struct CondState {
    double est, estold;
    int32_t phase, kase, j, iter, act, pad;
};
struct CondPart { double sum, maxv; int32_t maxi, diff; };   // one chunk: sum |x_i|, max |x_i| at the lowest index, sign changes
// v = 1/n for every member, state reset (kase 1)
int launch_cond_init(CondState *st, val_t *v, int n, int members, cudaStream_t s);
// after a solve of kase `kase` whose results are x: the members waiting for it take one dlacn2 step and write their next
// vector into v; counts[0] / [1] (zeroed by the caller) receive how many members then wait for kase 1 / 2.  3 launches.
// part: members * ceil(n / COND_CHUNK) entries
int launch_cond_step(CondState *st, int kase, const val_t *x, val_t *v, val_t *sgn, CondPart *part, int *counts, int n, int members,
                     cudaStream_t s);
// The estimator loop on the device (gscon_device, gsrfs_device's ferr), in conditional graph nodes.  loop = {kase of the next
// round, rounds so far}.  continue: first = 1 starts the loop (kase 1, 0 rounds); else one round more and the next kase from
// counts as the host loop takes it; the WHILE handle w = a kase is left and fewer than max_rounds rounds ran.  select: the
// IF handles k1 / k2 = the round's kase.  rcond: (1 / est) / anorm per member, as gscon.  1 launch each.
int launch_cond_continue(const int *counts, int *loop, int first, int max_rounds, cudaGraphConditionalHandle w, cudaStream_t s);
int launch_cond_select(const int *loop, cudaGraphConditionalHandle k1, cudaGraphConditionalHandle k2, cudaStream_t s);
int launch_cond_rcond(const CondState *st, const double *anorm, const int32_t *status, int members, double *rcond, cudaStream_t s);

// slu_refine.cu (double) / slu_refine_z.cu (doublecomplex): the step kernels of iterative refinement (slu_b200_gsrfs), pdgsrfs's
// loop per column.  One RefineState per column, members x nrhs of them, member-major; vectors: members blocks of n x nrhs.
constexpr int REFINE_ITMAX = 20;      // pdgsrfs.c ITMAX
struct RefineState {
    double lstres, berr;              // pdgsrfs's lstres (3 at the start), the berr of the last residual
    unsigned long long berr_bits;     // this step's max_i |r_i| / w_i as bits (atomicMax; zeroed by the decide kernel)
    int32_t count, active;            // steps taken; 1 while the column is refined
};
struct RefineArgs {
    int n, nrhs, members;
    int64_t nnz;
    const int32_t *rowptr, *colind;
    const val_t *aval;                // members x nnz, member-major: A as the scaled fill received it
    const val_t *b;                   // right-hand sides
    RefineState *st;
    double *W;                        // nullptr, or dgerfs's W of every active column (the forward error estimate)
};
// r = b - A x for the active columns (0 elsewhere), their berr bits and W
int launch_refine_residual(const RefineArgs &a, const val_t *x, val_t *r, cudaStream_t s);
// berr of the step, pdgsrfs's test; *active (zeroed by the caller) receives the columns that take another step
int launch_refine_decide(const RefineArgs &a, int *active, cudaStream_t s);
// x += dx on the active columns
int launch_refine_update(const RefineArgs &a, val_t *x, const val_t *dx, cudaStream_t s);
// dst[t] = W[t] src[t], t < len
int launch_refine_scale(val_t *dst, const val_t *src, const double *W, int64_t len, cudaStream_t s);
// The refinement loop on the device (gsrfs_device), in conditional graph nodes.  init: pdgsrfs's start state of every column,
// inactive where the member's status is not 0.  continue: the WHILE handle h = *active > 0.  xmax: max_i |x_i| of every
// column as bits into xmax (zeroed by the caller).  finish: berr, steps and (ferr non-null) dgerfs's ferr per column.
int launch_refine_init(RefineState *st, const int32_t *status, int nrhs, int members, cudaStream_t s);
int launch_refine_continue(const int *active, cudaGraphConditionalHandle h, cudaStream_t s);
int launch_refine_xmax(const RefineArgs &a, const val_t *x, unsigned long long *xmax, cudaStream_t s);
int launch_refine_finish(const RefineArgs &a, const CondState *est, const unsigned long long *xmax, const int32_t *status, double *berr,
                         double *ferr, int32_t *steps, cudaStream_t s);

#ifndef SLU_COMPLEX
// slu_ozaki.cu: the Schur update of wide supernodes on wgmma (int8 slices, exact int32 accumulation in registers)
constexpr int OZ_NT = 32;             // columns of one CTA's int8 Schur tile (rows: 128)
constexpr int OZ_CL = 1;              // CTAs per cluster sharing the A operand by multicast
constexpr int OZ_NT_HOST = OZ_NT * OZ_CL;  // columns of the tile unit the host enumerates
constexpr int OZ_KSTEP = 32;          // int8 k per wgmma instruction and per pipeline stage
constexpr int OZ_DEFAULT_SLICES = 7;  // 48 bits per operand: error ~1e-15 * k * rowmax * colmax (scripts/ozaki_emulate.py)
constexpr int OZ_DEFAULT_MIN_NS = 128;
// Off by default: the slices are scaled per L row and per U column, not per k, so the error is relative to rowmax * colmax
// of each update and grows as (max / min pivot-row scale)^2 on a matrix that is not equilibrated (DESIGN 4b).  An
// explicit slice count (options.reserved[4] = 5..8, or SLU_B200_TC_SLICES) opts in; SLU_B200_TC_MAX_M limits it to
// updates of fewer rows (0: no limit).
constexpr bool OZ_DEFAULT_ON = false;
inline int64_t oz_a_bytes(int m, int ns, int S) { return (int64_t)((m + 127) / 128) * ((ns + OZ_KSTEP - 1) / OZ_KSTEP) * S * 4096; }
inline int64_t oz_b_bytes(int n, int ns, int S) { return (int64_t)((n + OZ_NT - 1) / OZ_NT) * ((ns + OZ_KSTEP - 1) / OZ_KSTEP) * S * OZ_NT * OZ_KSTEP; }
inline int64_t oz_scale_elems(int m, int n) { return (int64_t)((m + 127) / 128) * 128 + (int64_t)((n + OZ_NT - 1) / OZ_NT) * OZ_NT; }
// slice the L rows / U columns of the batch's supernodes (3 launches); prefixes: row tiles, row tiles x k-steps, 4-column groups
int launch_oz_slice(const DeviceLU &d, const int32_t *nodes, int count, const int64_t *p_rt, int64_t n_rt, const int64_t *p_ak,
                    int64_t n_ak, const int64_t *p_b, int64_t n_b, int S, cudaStream_t s);
// fused GEMM + scatter of the batch's 128 x OZ_NT tiles; mode / split as launch_schur
int launch_oz_schur(const DeviceLU &d, const Batch &b, int64_t ctas, int mode, int split_n, int split_i, int S, cudaStream_t s);
// slu_ozaki.cu: C -= A*B through int8 slices on wgmma (variants 110..149: slices, stages, cluster)
int launch_gemm_sub_ozaki(int m, int n, int k, const double *a, int lda, const double *b, int ldb, double *c, int ldc,
                          int variant, cudaStream_t s);
#endif

// slu_selinv.cu (double) / slu_selinv_z.cu (doublecomplex): selected inversion H = F^-T on the stored pattern of L + U into
// a second arena hv of the factors' layout (slu_b200_selinv).  Per level, top-down, after launch_schur_setup and
// launch_diag_inv of the level: the three products (mode 0: H(R,K) = -M U_KC^T, tiles of m x ns; 1: H(K,C) = -L_RK^T M,
// ns x ncols; 2: H(K,K) = I - L_RK^T H(R,K), ns x ns; SELINV_TILE_M rows x SELINV_TILE_N val_t columns per tile, 64 x 64
// real outputs in both precisions), then the triangular solves (cols 0: every row of L panel K of hv times U_KK^-T;
// 1: L_KK^-T times the ns + ncols columns of H(K,K) and H(K,C); SELINV_VECS vectors per CTA).  Each launcher makes one
// launch per call, even for an empty batch.
constexpr int SELINV_TILE_M = 64;
#ifdef SLU_COMPLEX
constexpr int SELINV_TILE_N = 32;   // complex columns: 64 real ones
typedef double phase_t;             // log-determinant phase: the sum of the pivots' arguments
#else
constexpr int SELINV_TILE_N = 64;
typedef int phase_t;                // log-determinant phase: the number of negative pivots
#endif
constexpr int SELINV_VECS = 128;
int launch_selinv_gemm(const DeviceLU &d, const Batch &b, int64_t ctas, int mode, val_t *hv, cudaStream_t s);
int launch_selinv_trsm(const DeviceLU &d, const Batch &b, int64_t ctas, int cols, const val_t *dinv, val_t *hv, cudaStream_t s);
// log |det| into out[0] and the phase after it, over the listed supernodes' pivots: double out[1] = the sign (+1 / -1),
// doublecomplex out[1], out[2] = exp(i theta), theta = sum of arg u_ii reduced modulo 2 pi; part / pph:
// ceil(count / SELINV_VECS) entries.  2 launches.
int launch_selinv_logdet(const DeviceLU &d, const int32_t *nodes, int count, double *part, phase_t *pph, double *out, cudaStream_t s);
// out[p] = H(perm[colind[p]], perm[i]) for the entries p of row i; *err counts entries without a slot (out = NaN there)
int launch_selinv_get(const DeviceLU &d, const val_t *hv, int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm,
                      val_t *out, int *err, cudaStream_t s);
// batched (slu_b200_batch_selinv ...): the same launches over d.members matrices of one pattern (gridDim.y = members).  hv =
// member 0's H arena, the members' arenas d.val_stride elements apart; dinv as launch_diag_inv.  logdet: part / pph hold
// members x ceil(count / SELINV_VECS) entries, out members x (1 + VAL_DOUBLES).  get: out holds members x nnz values,
// member-major; *err counts member 0's entries without a slot only (the count of the unbatched call).
int launch_selinv_gemm(const BatchedLU &d, const Batch &b, int64_t ctas, int mode, val_t *hv, cudaStream_t s);
int launch_selinv_trsm(const BatchedLU &d, const Batch &b, int64_t ctas, int cols, const val_t *dinv, val_t *hv, cudaStream_t s);
int launch_selinv_logdet(const BatchedLU &d, const int32_t *nodes, int count, double *part, phase_t *pph, double *out, cudaStream_t s);
int launch_selinv_get(const BatchedLU &d, const val_t *hv, int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm,
                      val_t *out, int *err, cudaStream_t s);
// slu_grad.cu (double) / slu_grad_z.cu (doublecomplex): the gradient kernels (slu_b200_solve_grad_device, _logdet_grad_device
// and their twins), 1 launch each.  stage: dst[(m n + i) nrhs + k] = src[(m nrhs + k) ld + i] for members blocks of n x nrhs
// column-major values.
int launch_grad_stage(val_t *dst, const val_t *src, int n, int nrhs, int ld, int members, cudaStream_t s);
// g[m nnz + e] = -sum_k lam_m(row[e], k) conj(x_m(colind[e], k)) on the kept A's pattern; element (i, k) of member m at
// lam[m lms + i rs + k] (x: xms); NaN for every entry of a member whose status is not 0.  members = gridDim.y
struct SolveGrad {
    int64_t nnz;
    int nrhs, pad;
    const int32_t *row, *colind;
    const val_t *lam, *x;
    int64_t lms, xms, rs;
    const int32_t *status;
    val_t *grad;                       // members x nnz, member-major
};
int launch_solve_grad(const SolveGrad &a, int members, cudaStream_t s);
// g[m nnz + e] = coef[m] ((R_i h) C_j), h = H[slot[e]] of member m (conj(H) in doublecomplex); NaN for every entry of a member
// whose status is not 0 and for an entry without a slot
struct LogdetGrad {
    int n;
    int64_t nnz;
    const int64_t *slot;
    const int32_t *row, *colind;
    const double *R, *C;               // members x n
    const val_t *hv;                   // member 0's H arena (the members' d.val_stride elements apart)
    const val_t *coef;                 // [members]
    const int32_t *status;
    val_t *grad;                       // members x nnz, member-major
};
int launch_logdet_grad(const DeviceLU &d, const LogdetGrad &a, cudaStream_t s);
int launch_logdet_grad(const BatchedLU &d, const LogdetGrad &a, cudaStream_t s);
// after a device selected inversion: status[j] = -1 if *err (missed destinations) is not 0, else info[j]; rec[0] = *epoch,
// rec[1] = *err
int launch_selinv_status(const int *err, const int32_t *info, int members, const unsigned long long *epoch, int32_t *status,
                         unsigned long long *rec, cudaStream_t s);
// logabs[j] and sign[j VAL_DOUBLES ...] from launch_selinv_logdet's out (members x (1 + VAL_DOUBLES)), NaN where status[j] is
// not 0
int launch_logdet_out(const double *res, const int32_t *status, int members, double *logabs, double *sign, cudaStream_t s);
// inertia (slu_b200_inertia, _batch_inertia) over the listed supernodes' pivots u_ii: per member cnt[3 j ...] = the pivots with
// Re u_ii < 0, the others, those with |u_ii| <= thresh; def[j] = max |Im u_ii| / |u_ii| (0 in double).  pcnt / pdef: members x
// ceil(count / SELINV_VECS) partials (3 counts each).  2 launches.
int launch_inertia(const DeviceLU &d, const int32_t *nodes, int count, double thresh, long long *pcnt, double *pdef, long long *cnt,
                   double *def, cudaStream_t s);
int launch_inertia(const BatchedLU &d, const int32_t *nodes, int count, double thresh, long long *pcnt, double *pdef, long long *cnt,
                   double *def, cudaStream_t s);

// slu_schur.cu (double) / slu_schur_z.cu (doublecomplex): the Schur complement of a partial factorization
// (slu_b200_schur_get).  S(r - n0, c - n0) = every stored entry (r, c) of the Schur supernodes' panels, into a zeroed s x s
// column-major buffer (ld s); units[u] = (supernode k, column c): c < ns is column c of L panel k (diagonal block included),
// c >= ns the skyline segment of packed column c - ns of U panel k.  One launch of nunits CTAs.
int launch_schur_gather(const DeviceLU &d, const int2 *units, int64_t nunits, int n0, int s, val_t *S, cudaStream_t st);
// batched (slu_b200_batch_schur_get): the same launch over d.members matrices of one pattern (gridDim.y = members); S holds
// members blocks of s x s, member j's at S + j * s * s
int launch_schur_gather(const BatchedLU &d, const int2 *units, int64_t nunits, int n0, int s, val_t *S, cudaStream_t st);

#ifdef SLU_COMPLEX
constexpr int SCHUR_BM_BIG = 128, SCHUR_BM_SMALL = 32, SCHUR_BN_SMALL = 16;
#else
constexpr int SCHUR_BM_BIG = 128, SCHUR_BM_SMALL = 32, SCHUR_BN_SMALL = 32;
#endif
constexpr int SETUP_THREADS = 256;

}  // namespace SLU_NS
