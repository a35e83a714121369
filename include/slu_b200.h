/*
 * slu_b200.h -- C-ABI of libslu_b200.so: an H100-native (sm_90a) implementation of
 * SuperLU_DIST's 3D supernodal numeric factorization hot path `pdgstrf3d`.
 *
 * Boundary.  The reference reaches a non-C factorization backend through an opaque handle
 * (SRC/include/superlu_upacked.h:17-28, called from SRC/double/pdgssvx3d.c:1013-1021):
 *
 *     dCreateLUgpuHandle(...)   -> slu_b200_create() + slu_b200_upload()
 *     pdgstrf3d_LUv1(handle)    -> slu_b200_factor()
 *     dCopyLUGPU2Host(handle,.) -> slu_b200_download()
 *     dDestroyLUgpuHandle(.)    -> slu_b200_destroy()
 *
 * and the plain CPU/“HALO” path through `pdgstrf3d(options, m, n, anorm, trf3Dpartition, SCT,
 * LUstruct, grid3d, stat, info)` (SRC/double/pdgstrf3d.c:121-124) -> pdgstrf3d_b200().
 *
 * No reference struct crosses this boundary.  The caller passes a flat *view* (plain pointers
 * and sizes) of the structures the reference already holds; the data those pointers address
 * keep the reference's exact layout (SRC/include/superlu_defs.h:156-204):
 *
 *   L block column k  (local index k / npcol):
 *     Lrowind_bc_ptr[lk] = [ nblk, nrows ; (ib, nbrow, row ids ...) x nblk ]   BC_HEADER=2, LB_DESCRIPTOR=2
 *     Lnzval_bc_ptr[lk]  = column-major nrows x SuperSize(k); diagonal block first on its owner
 *   U block row k     (local index k / nprow):
 *     Ufstnz_br_ptr[lk]  = [ nblk, nnz, indexlen ; (jb, nnz_blk, fstnz[SuperSize(jb)]) x nblk ]  BR_HEADER=3, UB_DESCRIPTOR=2
 *     Unzval_br_ptr[lk]  = concatenated skyline column segments [fstnz, xsup[k+1])
 *
 * The INTEGRATION.md shim (oracle/ref_build/pdgstrf3d_hook.c) shows the ~60 lines a reference
 * maintainer adds to fill this view from dLUstruct_t / dtrf3Dpartition_t / gridinfo3d_t.
 *
 * Error convention (mirrors pdgstrf3d.c:388-392): functions return 0 on success, <0 on an
 * argument/runtime error (message via slu_b200_last_error()); *info = 0, or the 1-based global
 * column of the first exactly-zero pivot, min-reduced over all ranks of the 3D grid.
 */
#ifndef SLU_B200_H
#define SLU_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SLU_B200_ABI_VERSION 1

/* int_t of the reference's default build (SRC/include/superlu_defs.h:126-129). */
typedef int32_t slu_int;

/* One sForest_t (SRC/include/superlu_defs.h:940-962): an elimination sub-forest. */
typedef struct {
    slu_int nNodes;               /* number of supernodes in the forest (0: empty)          */
    const slu_int *nodeList;      /* supernode ids in an order valid for factorization      */
    slu_int numLvl;               /* topoInfo.numLvl (informational)                        */
    const slu_int *eTreeTopLims;  /* topoInfo.eTreeTopLims[numLvl+1] (informational)        */
} slu_b200_forest_t;

/* Flat view of Glu_persist_t + gridinfo3d_t + dLocalLU_t + dtrf3Dpartition_t. */
typedef struct {
    /* Glu_persist_t (superlu_defs.h:454-457) */
    slu_int n;                    /* matrix order                                            */
    slu_int nsupers;              /* number of supernodes                                    */
    const slu_int *xsup;          /* [nsupers+1] first column of each supernode              */
    /* gridinfo3d_t (superlu_defs.h:417-438) */
    slu_int nprow, npcol, npdep;  /* process grid Pr x Pc x Pz (Pz a power of two)                */
    slu_int myrow, mycol, mydep;  /* my coordinates                                          */
    /* dLocalLU_t (superlu_ddefs.h:97-307): arrays of per-local-block pointers (host memory) */
    slu_int **Lrowind_bc_ptr;     /* [ceil(nsupers/npcol)]                                   */
    double **Lnzval_bc_ptr;       /* [ceil(nsupers/npcol)]  in: A / partial sums, out: L     */
    slu_int **Ufstnz_br_ptr;      /* [ceil(nsupers/nprow)]                                   */
    double **Unzval_br_ptr;       /* [ceil(nsupers/nprow)]  in: A / partial sums, out: U     */
    /* dtrf3Dpartition_t (superlu_ddefs.h:317-337) */
    slu_int maxLvl;               /* log2(npdep)+1                                           */
    const slu_int *myTreeIdxs;    /* [maxLvl] forest index I hold at each Z-tree level       */
    const slu_int *myZeroTrIdxs;  /* [maxLvl] 1 = my copy of that forest starts as zeros     */
    slu_int nforests;             /* 2^maxLvl - 1                                            */
    const slu_b200_forest_t *forests; /* [nforests]                                          */
} slu_b200_lu_view_t;

typedef struct {
    int32_t device;               /* CUDA device ordinal (-1: current device)                */
    int32_t replace_tiny_pivot;   /* options->ReplaceTinyPivot (superlu_defs.h:707)          */
    double thresh;                /* smach_dist("Epsilon")*anorm (pdgstrf3d.c:132-133)       */
    int32_t verbose;              /* 0 silent                                                */
    int32_t pinned_host;          /* 1: caller's nzval arrays are page-locked (faster copies) */
    /* multi-GPU (npdep*nprow*npcol > 1): one NCCL communicator over the 3D grid replaces   */
    /* grid3d->comm for the panel / ancestor traffic (pd3dcomm.c:1046-1081).                 */
    int32_t world_size;           /* ranks in the 3D grid (1: no communication)              */
    int32_t world_rank;           /* my rank: mydep*(nprow*npcol) + myrow*npcol + mycol      */
    unsigned char nccl_id[128];   /* ncclUniqueId from slu_b200_nccl_unique_id on rank 0     */
    int32_t schur_variant;        /* retired, must be 0: create and plan refuse any other value     */
    int32_t reserved[7];          /* [0] no look-ahead, [1] reference-style ancestors, [2] pdgstrf3d_b200 */
                                  /* uses slu_b200_factor_host (overlapped transfers), [3] level-by-  */
                                  /* level arena so that factor_host also overlaps the upload,        */
                                  /* [4] tcgen05 path for wide supernodes: int8 slices per operand    */
                                  /* (0 = default: off, 5..8 opt in, < 0 = off: FP64 DMMA only; needs  */
                                  /* balanced pivot-row scales, e.g. an equilibrated A), [5] narrowest */
                                  /* supernode that takes the tcgen05 path (0 = default 128), [6] the  */
                                  /* most supernode panels one Schur GEMM takes (0 = default 4, 1 =    */
                                  /* off, up to 4; DESIGN 4a): a child whose structure is its parent's */
                                  /* columns followed by its parent's structure leaves the rest of its */
                                  /* update to its parent's, as more K.  The environment variable      */
                                  /* SLU_B200_SCHUR_DEPTH overrides it.  Always 1 in doublecomplex, on */
                                  /* the int8 path, on Pr x Pc > 1 and on Pz > 1.  Results change only */
                                  /* in summation order; the flop counts do not change.                */
} slu_b200_options_t;

typedef struct {
    double ops_fact;              /* flops, reference accounting (stat->ops[FACT]): diag LU  */
                                  /* pdgstrf2.c:578,590; U-TRSM trfAux.c:2303; Schur         */
                                  /* sec_structs.c:692-693.  Local to this rank.             */
    double ops_schur;             /* the 2*m*n*k part of ops_fact                            */
    double schur_bytes;           /* algorithmic bytes of the Schur updates (DESIGN.md)      */
    int64_t tiny_pivots;          /* stat->TinyPivots                                        */
    int64_t gpu_launches;         /* kernels launched by the last slu_b200_factor()          */
    double t_analyze_s;           /* host: structure analysis + device index build           */
    double t_upload_s;            /* H2D of L/U values                                       */
    double t_factor_s;            /* device time of the last factor (CUDA events)            */
    double t_download_s;          /* D2H of L/U values                                       */
    double t_diag_ms, t_trsm_ms, t_schur_setup_ms, t_schur_ms, t_reduce_ms; /* phase sums,   */
                                  /* only filled when options.verbose >= 2 (adds syncs)      */
    int64_t lu_device_bytes;      /* HBM held by L/U values                                  */
    int64_t index_device_bytes;   /* HBM held by index structures + workspace                */
    int64_t nnz_l, nnz_u;         /* doubles stored in my L / U panels (device layout)       */
    int32_t nlevels;              /* level-synchronous steps executed                        */
    int32_t my_supernodes;        /* supernodes this rank factored                           */
    double reserved[8];           /* [0] ms spent slicing (verbose >= 2), [1] Schur flops taken by the */
                                  /* tcgen05 path, [2] bytes of its int8 workspace, [3] slices in use,  */
                                  /* [4] seconds of the last slu_b200_solve, _solve_trans, _solve_scaled */
                                  /* or _gsrfs, [5] its kernel launches, [6] seconds of the last slu_b200_gscon or         */
                                  /* _batch_gscon, [7] the solve rounds it ran                          */
} slu_b200_stats_t;

typedef struct slu_b200_handle_s *slu_b200_handle_t;

int slu_b200_abi_version(void);
/* sizeof of {slu_b200_forest_t, slu_b200_lu_view_t, slu_b200_options_t, slu_b200_stats_t}: lets a
 * foreign-function binding (cgo / ctypes / Fortran) verify its struct mirrors before the first call */
void slu_b200_struct_sizes(int32_t out[4]);
const char *slu_b200_last_error(void);
/* number of visible CUDA devices (0 if none / driver missing); never throws */
int slu_b200_device_count(void);

/* Analyse the structure, allocate HBM, build device index structures.  Values are not read.
 * Every handle call that writes the values in HBM (an upload, any fill, a factorization) first discards what the handle
 * knew about them: a call of these that fails leaves the handle with no factors (and, for an upload or fill, no values
 * to factor either).  The calls that read the factors then refuse, with a message, until a successful fill and
 * factorization. */
int slu_b200_create(slu_b200_handle_t *h, const slu_b200_lu_view_t *lu,
                    const slu_b200_options_t *opt);
/* H2D: copy the view's Lnzval/Unzval (for the supernodes of my forests) into HBM. */
int slu_b200_upload(slu_b200_handle_t h);
/* Factor in HBM.  Collective over the NCCL communicator when world_size > 1. */
int slu_b200_factor(slu_b200_handle_t h, int *info);
/* upload + factor + download in one call with the D2H overlapped with the factorization: a panel is
 * final once the panel work of its level is done, so it is copied back on a second stream while the
 * upper levels are still being factored.  Same result as the three separate calls; needs page-locked
 * host arrays to actually overlap.  Patterns whose U skylines are not all full (unsymmetric patterns) and
 * Pr x Pc pieces take the plain upload / factor / download path inside this call: same results, no overlap. */
int slu_b200_factor_host(slu_b200_handle_t h, int *info);
/* D2H: write L and U back into the view's Lnzval/Unzval in the reference layout. */
int slu_b200_download(slu_b200_handle_t h);
/* Device-side distribution (the job of pddistribute3d, SRC/double/pddistribute3d.c:1357, on the GPU): instead of
 * slu_b200_upload of the caller's Lnzval/Unzval arrays, scatter the matrix itself into the panels.  A: n x n host CSR
 * (int32 indices, no duplicate entries); perm[old] = new is the final permutation of the factored matrix
 * (P (A) P^T, rows and columns alike).  12 bytes per nonzero cross PCIe instead of 8 bytes per factor entry; the value
 * arrays of the view may then be NULL-backed (never read) if the caller also skips slu_b200_download.  1 x 1 x Pz.
 * An entry of a U column above that column's skyline start (Ufstnz) has no slot, as an entry outside the structure:
 * the call fails with the count of such entries rather than writing it into the zero padding above the segment. */
int slu_b200_fill_csr(slu_b200_handle_t h, int n, const int32_t *rowptr, const int32_t *colind, const double *val,
                      const int32_t *perm);
/* Solve L U x = b with the factors still resident in HBM (after a successful slu_b200_factor / _factor_host on this
 * handle) -- the consumer of pdgstrf3d, pdgstrs3d (SRC/double/pdgstrs3d.c:6604), without the D2H/H2D round trip.
 * x: host, n x nrhs column-major (ldx >= n), in the ordering of the factored matrix (the caller applies the
 * permutations / scalings, as pdgssvx3d does around pdgstrs3d); holds b on entry, the solution on return.
 * 1 x 1 x Pz grids: collective, every rank passes the same b and receives the full x (NCCL all-reduces along Z
 * replace the ancestor reduce / dbroadcastAncestor3d, pd3dcomm.c:1145).  stats.reserved[4] = seconds of the call. */
int slu_b200_solve(slu_b200_handle_t h, double *x, int ldx, int nrhs);
/* Solve op(A) x = b on the same resident factors, as LAPACK getrs(trans) / SuperLU dgstrs(trans): trans takes the values
 * of the reference's trans_t (SRC/include/superlu_enum_consts.h:34): 0 = NOTRANS (exactly slu_b200_solve), 1 = TRANS
 * (A^T x = b), 2 = CONJ (A^H x = b; the same as 1 in double).  A^T = U^T L^T is solved as U^T y = b, then L^T x = y, over
 * the level plan of the plain solve: no second analysis or factorization of A^T, no second copy of the factors.  Uses:
 * adjoint solves for gradients and sensitivities, 1-norm condition estimation.  x, ldx, nrhs, the restrictions (a
 * successful factorization, 1 x 1 x Pz, the cooperative schedule along Z) and stats.reserved[4] / [5] (the last solve of
 * either kind) are those of slu_b200_solve.  x uses the ordering of the factored matrix F = P A P^T; since
 * F^T = P A^T P^T, the caller permutes b and x exactly as for the plain solve.  trans outside {0, 1, 2} fails.
 * The reference's pdgstrs3d has no transposed mode. */
int slu_b200_solve_trans(slu_b200_handle_t h, double *x, int ldx, int nrhs, int trans);
/* Reciprocal condition number estimate on the resident factors, as LAPACK dgecon and sequential SuperLU dgscon:
 * *rcond = (1 / est) / anorm, where est estimates ||F^-1|| (= ||A^-1||) of the factored matrix F = P A P^T in the 1-norm
 * (norm '1' or 'O') or the infinity-norm (norm 'I'; 'o' and 'i' are accepted too), and anorm = ||A|| in the same norm,
 * computed by the caller (pdgssvx3d computes it with pdlangs).  est is LAPACK's dlacn2 (Hager / Higham) applied to F^-1
 * exactly as dgecon drives it: "kase 1" solves with F and "kase 2" with F^T (swapped for norm 'I'), from the start vector
 * (1/n, ..., 1/n), at most 5 iterations, the final alternating-sign vector; about 5 solves.  The whole iteration runs on
 * device vectors: per solve the host reads back two counters, no n-vector crosses PCIe.  est is a lower bound of the
 * norm and usually within a factor of 3 of it.
 * anorm < 0 or NaN fails; anorm = 0 or +inf gives *rcond = 0 without a solve; a non-finite estimate gives *rcond = 0.
 * The estimate describes L U as factored: where tiny pivots were replaced (options.replace_tiny_pivot), that is the
 * perturbed matrix, not A.  Restrictions as slu_b200_solve (a successful factorization, 1 x 1 x Pz, collective along Z:
 * every rank passes the same anorm and receives the same rcond).  stats.reserved[6] = seconds of the call,
 * stats.reserved[7] = the solves it ran; stats.reserved[4] / [5] keep describing the last slu_b200_solve*.  The
 * reference's pdgssvx3d has no condition estimator. */
int slu_b200_gscon(slu_b200_handle_t h, char norm, double anorm, double *rcond);
/* Selected inversion on the resident factors (SelInv / PSelInv): H = F^-T on the stored pattern of L+U, F = P A P^T = L U,
 * into a second HBM arena of the factors' layout (allocated on first use, freed by destroy).  One sweep over the level plan,
 * top-down, about twice the Schur-update flops; deterministic (every entry written once with plain stores: two calls on the
 * same factors give bit-identical H); the factors are only read.  A^-1(i, j) = H(perm[j], perm[i]): the entries of A^-1 on
 * the pattern of A^T, and of A where A is structurally symmetric.  Where tiny pivots were replaced the result describes
 * L U as factored, as for slu_b200_gscon.  If the second arena does not fit, the call fails and the handle stays usable for
 * solves.  Restrictions (all fail with a message): a successful factorization (info = 0), an unbatched handle (batched
 * handles: slu_b200_batch_selinv below), a 1 x 1 x 1 grid (world_size 1).  Doublecomplex through slu_b200_z_selinv below; the reference's pdgssvx3d has no selected inversion.
 * out (may be NULL): [0] seconds, [1] flops (accounting in DESIGN.md), [2] kernel launches, [3] HBM bytes it holds. */
int slu_b200_selinv(slu_b200_handle_t h, double out[4]);
/* out[p] = (A^-1)(i, colind[p]) for every entry p of row i of the CSR pattern; A = P^T F P, perm[old] = new as in
 * slu_b200_fill_csr.  Fails, with the count, if any (perm[colind[p]], perm[i]) has no slot in L+U.  Needs slu_b200_selinv
 * on the current factors: a later upload, fill_csr or factor invalidates the inverse; n must match the handle. */
int slu_b200_selinv_get(slu_b200_handle_t h, int n, const int32_t *rowptr, const int32_t *colind,
                        const int32_t *perm, double *out);
/* log|det A| and its sign (+1 / -1) from the resident factors: sum of log |U_kk(i,i)| in a fixed order (deterministic),
 * sign from the count of negative pivots; the symmetric permutation does not change det.  Restrictions of selinv. */
int slu_b200_logdet(slu_b200_handle_t h, double *logabs, double *sign);
/* Inertia of a real symmetric / complex Hermitian A from the resident factors (MUMPS INFOG(12), PARDISO iparm(22..23)):
 * F = P A P^T = L U uses a symmetric permutation, no row exchanges and a unit-diagonal L, so U = D L^T (D L^H) and by
 * Sylvester's law the signs of the pivots u_ii are those of A's eigenvalues; for A - sigma B with B positive definite,
 * counts[0] is the number of eigenvalues of the pencil below sigma (spectrum slicing, PEXSI's inertia counting, checking
 * the inertia of a KKT matrix).
 * counts[0] = pivots with u_ii < 0 (Re u_ii < 0 in doublecomplex), counts[1] = the others (counts[0] + counts[1] = n),
 * counts[2] = pivots with |u_ii| <= options.thresh (replaced tiny pivots land exactly there), counted in 0/1 as well.
 * *defect = max_i |Im u_ii| / |u_ii| in doublecomplex (0 for a Hermitian A up to rounding), 0 in double.
 * The library does not check symmetry: the caller asserts it, and defect is the diagnostic for complex input.  Two limits:
 * where a tiny pivot was replaced (options.replace_tiny_pivot) the counts describe L U as factored, not A, which is what
 * counts[2] is for; counts[2] uses options.thresh whether or not replacement is on, so a caller that wants that count must
 * pass a threshold.  Fixed-order integer reductions (deterministic), 2 kernel launches.  Restrictions and messages of
 * slu_b200_logdet: a successful factorization, an unbatched handle that is not a Schur handle, a 1 x 1 x 1 grid. */
int slu_b200_inertia(slu_b200_handle_t h, int64_t counts[3], double *defect);
/* Partial factorization with a Schur complement (MUMPS ICNTL(19), PARDISO iparm(36)): with F = P A P^T = [A11 A12; A21 A22]
 * and the s = nschur "Schur" unknowns last, eliminate A11 only and keep S = A22 - A21 A11^-1 A12.  Uses: domain
 * decomposition (S is the interface operator), sparse-dense block coupling, Kron reduction, static condensation, marginal
 * precision matrices.  The view must come from a symbolic factorization that keeps the Schur columns last in whole
 * supernodes (sluh_symbolic_schur; hostlib.schur_order orders a pattern so).
 * schur_create: as slu_b200_create, but the supernodes with xsup[k] >= n - nschur are left out of the level plan; their
 * panels keep their place in HBM and receive every Schur update of the eliminated part.  Fails with a message unless
 * 1 <= nschur < n, n - nschur is a supernode boundary (the message names the supernode across it), the grid is 1 x 1 x 1
 * with world_size 1 and the int8 tensor-core path is off (options.reserved[4] <= 0; FP64 DMMA only, as on batched handles).
 * A Schur handle takes slu_b200_upload, _fill_csr, _factor, _download, _get_stats, _destroy and the schur_* calls below;
 * factor_host, solve, solve_trans, gscon, selinv, selinv_get, logdet, the batch_* and kernel-export calls fail on it with
 * a message and leave it usable, and the schur_* calls fail on ordinary and batched handles (batched Schur handles:
 * slu_b200_batch_schur_create and the batch_schur_* calls below).  factor eliminates the
 * non-Schur supernodes only: info = 0 or the 1-based column of the first exact zero pivot among them; ops_fact, ops_schur,
 * nlevels and my_supernodes count the eliminated work.  download writes L11, U11, L21 and U12, and S in the Schur panels,
 * in the reference layout.
 * schur_get: S into the host array S, s x s column-major (lds >= s); row and column t are F's index n - s + t.  Every
 * stored entry of the Schur panels is written once by one gather kernel into a zeroed device buffer (kept by the handle
 * until destroy), then copied back: entries outside the stored pattern are exactly 0 and two calls on the same factors are
 * bit-identical.  If the s x s buffer does not fit, the call fails with its size.  Needs a successful factor (info = 0).
 * stats.reserved[6] = seconds of the call, stats.reserved[7] = device milliseconds of the gather kernel.
 * schur_condense: the forward pass of the solve over the eliminated supernodes: x holds b on entry, and y1 = L11^-1 b1 in
 * the eliminated positions and g = b2 - A21 A11^-1 b1 in the Schur positions on return.
 * schur_expand: the backward pass: x holds y1 (as condense left it) and x2 in the Schur positions on entry,
 * x1 = A11^-1 (b1 - A12 x2) and x2 on return.  So condense, x2 = S^-1 g (by the caller), expand solves A x = b.
 * Both: x, ldx and nrhs as slu_b200_solve (ordering of F), need a successful factor, set stats.reserved[4] / [5]. */
int slu_b200_schur_create(slu_b200_handle_t *h, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, int nschur);
int slu_b200_schur_get(slu_b200_handle_t h, double *S, int lds);
int slu_b200_schur_condense(slu_b200_handle_t h, double *x, int ldx, int nrhs);
int slu_b200_schur_expand(slu_b200_handle_t h, double *x, int ldx, int nrhs);
int slu_b200_get_stats(slu_b200_handle_t h, slu_b200_stats_t *out);
void slu_b200_destroy(slu_b200_handle_t h);

/* The one-call drop-in for pdgstrf3d (pdgstrf3d.c:121): create+upload+factor+download+destroy. */
int pdgstrf3d_b200(const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt,
                   slu_b200_stats_t *stats, int *info);

/* Fill `id` (128 bytes) with a fresh ncclUniqueId; rank 0 calls it and broadcasts the bytes. */
int slu_b200_nccl_unique_id(unsigned char id[128]);
/* The NCCL communicators (world + per-Z-level groups) built from an id are cached per process and reused by every
 * later create / pdgstrf3d_b200 with the same id and grid coordinates -- the counterpart of the MPI communicators
 * superlu_gridinit3d creates once (SRC/prec-independent/superlu_grid3d.c:47-63).  Destroy them explicitly: */
void slu_b200_comm_cache_clear(void);

/* Page-locked host allocation helpers for callers that want full-speed PCIe copies. */
void *slu_b200_host_alloc(size_t bytes);
void slu_b200_host_free(void *p);

/* Analysis only -- needs no device: fills stats (lu_device_bytes, index_device_bytes, ops_fact, nnz_l/u, nlevels,
 * my_supernodes) for this rank of a 1 x 1 x Pz grid, e.g. to size a run for 180 GB GPUs before allocating them
 * (the role of the reference's memory estimate dQuerySpace_dist, SRC/double/dmemory_dist.c). */
int slu_b200_plan(const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, slu_b200_stats_t *stats);

/* ---- kernel-level entry points (host pointers; used by tests and micro-benchmarks) ---------- */
/* In-place unpivoted LU of an ns x ns column-major block (Local_Dgstrf2, pdgstrf2.c:508-601). */
int slu_b200_k_diag_lu(double *a, int ns, int lda, int replace_tiny, double thresh, int col0,
                       int *info, int *tiny);
/* X <- X * U^-1, U = upper triangle (non-unit) of lu[ns x ns] (dLPanelTrSolve,
 * dtrfCommWrapper.c:120-223).  x is m x ns column-major. */
int slu_b200_k_trsm_l(const double *lu, int ldlu, int ns, double *x, int m, int ldx);
/* X <- L^-1 * X, L = unit lower triangle of lu (dUPanelTrSolve, dtrfCommWrapper.c:242-357).
 * x is ns x ncols column-major. */
int slu_b200_k_trsm_u(const double *lu, int ldlu, int ns, double *x, int ncols, int ldx);
/* C <- C - A*B with the Schur-update main loop (dblock_gemm_scatter, dscatter3d.c:82-189,
 * identity scatter).  Returns device milliseconds of the kernel in *ms if non-NULL. */
int slu_b200_k_gemm_sub(int m, int n, int k, const double *a, int lda, const double *b, int ldb,
                        double *c, int ldc, int reps, float *ms);
/* benchmark support (SURVEY 8a row a10): see slu_api.cu; device_lu receives the library's DeviceLU struct (device
 * pointers; layout in superlu_dist_b200/csrc/cuda/slu_device.cuh), nodes the level's supernodes with a big update.
 * Returns their count (< 0 on error). */
int slu_b200_k_level_export(slu_b200_handle_t h, int level, void *device_lu, int device_lu_bytes, int32_t *nodes, int max_nodes);
int slu_b200_k_rerun_schur(slu_b200_handle_t h, int level, int reps, float *ms);
/* the deferred Schur updates the analysis plans (options.reserved[6]), without a device: out[0] = supernodes whose update
 * is carried by their parent's, out[1] / out[2] = destination updates (RED.ADD.F64) of one factorization without and with
 * them.  variant 35 of slu_b200_k_gemm_sub (SLU_B200_GEMM_VARIANT) runs the same segmented K loop. */
int slu_b200_k_schur_merge(const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, double out[3]);

/* ---- batched handles: many matrices of ONE sparsity pattern (the reference's pdgssvx3d_csc_batch /
 * dsparseTreeFactorBatchGPU): per-cell implicit solves, parameter sweeps, ensemble members.  The structure analysis,
 * index arenas, level plan and Schur destination maps are built once and shared; every member has its own value arena
 * (stats.lu_device_bytes = batch x one member), diag-inverse workspace and info flag.  A batched factorization makes
 * exactly as many kernel launches as one unbatched factorization, each over batch x the CTAs (gridDim.y = member).
 * Double precision here and doublecomplex through the slu_b200_z_batch_* twins below; 1 x 1 x 1 grid, FP64 DMMA
 * kernels only (the int8 path is not used; stats.reserved[1] = 0).
 * A batched handle takes only these calls (create, fill_csr, fill_affine, factor, solve, solve_trans, gscon, selinv,
 * selinv_get, logdet, inertia and download, each with the batch_ prefix) plus slu_b200_get_stats and slu_b200_destroy; every other call on it
 * fails, and these fail on an unbatched handle.  Stats describe the whole handle: ops_fact, ops_schur, nnz_l, nnz_u and
 * lu_device_bytes are batch x the per-member values, tiny_pivots is summed over the members, t_factor_s is the device
 * time of the one batched call, stats.reserved[4] / [5] describe the last slu_b200_batch_solve or _batch_solve_trans.
 * Measured on an NVIDIA H100 80GB HBM3 at a 400 W power limit, per member, against one unbatched handle looping over
 * the members: Poisson 16^3, B = 64: factor 0.081 vs 1.337 ms (16.5x), solve (nrhs 1) 0.039 vs 0.872 ms; Poisson 32^3,
 * B = 64: factor 1.41 vs 5.53 ms (3.9x); more in README.md. */
/* batch >= 1 members sharing the structure of `lu`; nprow = npcol = npdep = 1, world_size = 1 */
int slu_b200_batch_create(slu_b200_handle_t *h, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, int batch);
/* one CSR pattern and one perm (as slu_b200_fill_csr); val = batch x nnz values, member-major */
int slu_b200_batch_fill_csr(slu_b200_handle_t h, int n, const int32_t *rowptr, const int32_t *colind,
                            const double *val, const int32_t *perm);
/* info[batch]: per member, 0 or the 1-based column of its first exact zero pivot */
int slu_b200_batch_factor(slu_b200_handle_t h, int *info);
/* x: batch blocks, block j at x + j*ldx*nrhs, each n x nrhs column-major (ldx >= n), ordering of the factored matrix;
 * b on entry, the solution on return.  Fails, naming the member, unless every member's last info was 0. */
int slu_b200_batch_solve(slu_b200_handle_t h, double *x, int ldx, int nrhs);
/* op(A_j) x_j = b_j for every member, trans as slu_b200_solve_trans; x and the restrictions as slu_b200_batch_solve */
int slu_b200_batch_solve_trans(slu_b200_handle_t h, double *x, int ldx, int nrhs, int trans);
/* rcond[j] for every member, as slu_b200_gscon with anorm[j] = ||A_j|| (both arrays hold batch entries).  The members
 * run dlacn2 in lock-step: each round is one batched solve of one kase for all members; only the members waiting for
 * that kase take its result, the others keep their pending vector.  The next round takes the other kase if any member
 * waits for it, else the same one, so no member waits more than one round and a batch takes at most twice the solves
 * of its slowest member.  stats.reserved[7] = the rounds.  Fails, naming the member, unless every member's last info
 * was 0. */
int slu_b200_batch_gscon(slu_b200_handle_t h, char norm, const double *anorm, double *rcond);
/* write member j's L/U into the view's Lnzval / Unzval arrays, in the reference layout (as slu_b200_download) */
int slu_b200_batch_download(slu_b200_handle_t h, int member);
/* Selected inversion of every member, as slu_b200_selinv: H_j = F_j^-T on the stored pattern of L+U, into a second HBM
 * arena of batch x one member's factors (allocated on first use, freed by destroy).  One sweep over the level plan for all
 * members: out[2] (kernel launches) equals an unbatched sweep's whatever the batch (7 per level, 6 at the root), each
 * launch over batch x the CTAs.  out[1] = batch x the per-member flops; out[0] and out[3] as slu_b200_selinv.
 * Deterministic, factors only read.  If the second arena does not fit, the call fails with its size and the handle stays
 * usable for batch_solve / batch_gscon.  Fails, naming the member, unless every member's last info was 0. */
int slu_b200_batch_selinv(slu_b200_handle_t h, double out[4]);
/* as slu_b200_selinv_get for every member, one CSR pattern and perm shared: out holds batch x nnz values, member-major
 * (member j's at out + j*nnz).  Needs slu_b200_batch_selinv on the current factors (a later batch_fill_csr or batch_factor
 * invalidates it); an entry with no slot fails with the count of one member, as the unbatched call. */
int slu_b200_batch_selinv_get(slu_b200_handle_t h, int n, const int32_t *rowptr, const int32_t *colind,
                              const int32_t *perm, double *out);
/* logabs[batch], sign[batch]: every member's log|det A_j| and sign, as slu_b200_logdet (needs no batch_selinv).  Fails,
 * naming the member, unless every member's last info was 0. */
int slu_b200_batch_logdet(slu_b200_handle_t h, double *logabs, double *sign);
/* every member's inertia, as slu_b200_inertia: member j's counts at counts[3*j + c], its defect at defect[j]; the same two
 * launches whatever the batch.  Fails, naming the member, unless every member's last info was 0; fails on Schur handles. */
int slu_b200_batch_inertia(slu_b200_handle_t h, int64_t *counts, double *defect);
/* Affine families (frequency sweeps K - w^2 M + i w C, shifted pencils A - sigma B, GMRF Q(theta) = sum_t theta_t Q_t):
 * member j, entry p: v = sum_t coef[j*nterms + t] * terms[t*nnz + p], t = 0 .. nterms-1 in order (v = c_0 V_0, then one
 * fused multiply-add per term; in doublecomplex the complex product of slu_scalar.cuh).  The nterms x nnz terms cross
 * PCIe once instead of batch x nnz values, and the slot search runs once per entry, not once per member.  Otherwise as
 * slu_b200_batch_fill_csr: one CSR pattern (rowptr, colind) and perm shared by all members, the arena zeroed first (fill-in
 * slots are 0), each slot written once with a plain store (deterministic); entries with no slot fail with their count;
 * the previous factors, selected inverse and member infos are invalidated (batch_solve fails until batch_factor).  Plain
 * and Schur batched handles; fails on unbatched handles, unless nterms >= 1, on a mismatched n, a rowptr that does not
 * start at 0 or decreases, and a colind outside 0 .. n-1.  Offsets are 64-bit. */
int slu_b200_batch_fill_affine(slu_b200_handle_t h, int n, const int32_t *rowptr, const int32_t *colind, int nterms,
                               const double *terms, const double *coef, const int32_t *perm);
/* Partial factorization on batched handles: the slu_b200_schur_* calls for `batch` matrices of one pattern (substructuring
 * with many same-mesh subdomains, static condensation of many element matrices, Kron reduction of network ensembles,
 * parameter sweeps of marginal precision matrices).
 * batch_schur_create: the checks of batch_create and of schur_create (1 <= batch <= 65535, 1 <= nschur < n, n - nschur a
 * supernode boundary, 1 x 1 x 1 grid with world_size 1, int8 path off), with messages that name batch_schur_create.  The
 * handle takes batch_fill_csr, batch_fill_affine, batch_factor, batch_download, get_stats, destroy and the four
 * batch_schur_* calls; batch_solve, batch_solve_trans, batch_gscon, batch_selinv, batch_selinv_get, batch_logdet and
 * batch_inertia fail on it with a message
 * ("Schur handle") and leave it usable, the unbatched schur_* calls fail on it ("batched handle"), and the batch_schur_*
 * calls fail on ordinary, plain batched and unbatched Schur handles.  batch_factor eliminates A11 of every member in one
 * launch sequence (the launches of one unbatched Schur factorization, each over batch x the CTAs): info[j] = 0 or the
 * 1-based column of member j's first exact zero pivot among the eliminated supernodes.  batch_download(j) writes member
 * j's L11, U11, L21, U12 and S.  Stats: batch x the per-member eliminated work (ops_fact, ops_schur); nlevels and
 * my_supernodes those of the eliminated part.
 * batch_schur_get: every member's S, member j's s x s block at S + j*lds*s (lds >= s), as schur_get: one gather launch
 * over (units, members) into a zeroed batch x s x s HBM buffer (allocated on first use, kept until destroy; if it does not
 * fit, the call fails with its size and the handle stays usable), then one copy; entries off the stored pattern are
 * exactly 0 and two calls are bit-identical.  stats.reserved[6] = seconds of the call, [7] = device ms of the gather.
 * batch_schur_condense / batch_schur_expand: the forward / backward pass of slu_b200_batch_solve over the eliminated
 * supernodes (as schur_condense / schur_expand for every member); x, ldx, nrhs and the checks as batch_solve (n * nrhs
 * below 2^31 per member); they set stats.reserved[4] / [5].
 * All but create fail, naming the member, unless every member's last info was 0. */
int slu_b200_batch_schur_create(slu_b200_handle_t *h, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt,
                                int batch, int nschur);
int slu_b200_batch_schur_get(slu_b200_handle_t h, double *S, int lds);
int slu_b200_batch_schur_condense(slu_b200_handle_t h, double *x, int ldx, int nrhs);
int slu_b200_batch_schur_expand(slu_b200_handle_t h, double *x, int ldx, int nrhs);

/* ---- static pivoting: row permutation and equilibration on the device fill (the pre-processing pdgssvx3d runs in front
 * of pdgstrf3d: pdgsequ / pdlaqgs, pdgssvx3d.c:695, and the large-diagonal row permutation with its scalings, dldperm_dist
 * job 5, pdgssvx3d.c:727).  The factorization pivots statically: a matrix with a zero or dominated diagonal (KKT /
 * saddle-point systems, circuit matrices) needs its large entries moved to the diagonal first.  The matching runs once per
 * pattern on the host (sluh_large_diag_perm, slu_b200_host.h); the fill, the equilibration and the vector transforms of the
 * solve run on the device, on every fill and every member.
 * fill_csr_scaled: as slu_b200_fill_csr, with F = Pc Pr Dr A Dc Pc^T: entry (i, j) of A goes to F(perm[perm_r[i]], perm[j])
 * with the value (R[i] * a_ij) * C[j], evaluated in that order.  perm_r (perm_r[i] = the row of Pr A that holds row i of
 * A), R and C may each be NULL (identity, ones); perm must be the final permutation of the pattern of Pr A (ordering and
 * symbolic factorization run on that pattern).  The arena is zeroed first, each slot gets one plain store (deterministic);
 * entries with no slot fail with their count.  flags & SLU_B200_FILL_EQUIL: equilibrate M = Pr Dr A Dc on the device with
 * dgsequ_dist / dlaqgs_dist semantics: row maxima of |M|, column maxima of the row-scaled matrix, smlnum = dmach("S")
 * clamping, and THRESH = 0.1 with the amax small / large tests choosing rows, columns, both or neither; the chosen factors
 * are folded into R and C.  The magnitude is slud_z_abs1 (|re| + |im|) in doublecomplex.  The maxima are taken with
 * integer atomics on the bit patterns, so R and C are bit-identical from run to run.  A zero row or column of A fails,
 * naming it (dgsequ's info).  4 kernel launches with EQUIL, 2 without.
 * out (nullable): [0] rowcnd, [1] colcnd, [2] amax, [3] equed (0 none, 1 rows, 2 columns, 3 both); without EQUIL 1, 1,
 * max |f_ij|, 0.  [4] ||F||_inf as fixed-order row sums (no float atomics), the anorm of slu_b200_gscon(h, 'I', ...); [5]
 * max |f_ij| ([4], [5] with the modulus).  The handle keeps perm_r, perm[perm_r[.]], perm and the final R and C in HBM until
 * a later upload, fill_csr, batch_fill_csr or batch_fill_affine, which drops them.  It keeps A as well, for slu_b200_gsrfs:
 * rowptr, colind and the values as given, 4 (n + 1) + 4 nnz + 8 nnz batch bytes (16 per value in doublecomplex), reused by
 * the next scaled fill of the same nnz and dropped with the scalings.
 * get_scaling: the kept perm_r, R and C (each nullable).
 * solve_scaled: solve op(A) x = b on the factors of F, x (n x nrhs, ldx >= n) in A's own ordering, b on entry.  trans 0:
 * b'[perm[perm_r[i]]] = R[i] b[i], F y = b', x[j] = C[j] y[perm[j]]; trans 1 / 2: b'[perm[j]] = C[j] b[j], F^T y = b' (F^H),
 * x[i] = R[i] y[perm[perm_r[i]]].  Two launches on top of the plain solve, no n-vector work on the host; stats.reserved[4] /
 * [5] as slu_b200_solve.  Fails unless the last fill was a scaled one and the factorization after it succeeded.
 * All fail with a message, leaving the handle as it was, on a perm_r or perm that is not a permutation, an R or C entry
 * that is not finite and > 0, Schur handles, and grids other than 1 x 1 x 1 with world_size 1.
 * slu_b200_gscon, selinv, logdet and inertia keep describing F: log|det A| = log|det F| - sum log R_i - sum log C_j, the
 * sign multiplied by sign(perm_r); inertia has no meaning once perm_r is not the identity. */
#define SLU_B200_FILL_EQUIL 1
int slu_b200_fill_csr_scaled(slu_b200_handle_t h, int n, const int32_t *rowptr, const int32_t *colind, const double *val,
                             const int32_t *perm_r, const int32_t *perm, const double *R, const double *C, int flags,
                             double out[6]);
int slu_b200_get_scaling(slu_b200_handle_t h, int32_t *perm_r, double *R, double *C);
int slu_b200_solve_scaled(slu_b200_handle_t h, double *x, int ldx, int nrhs, int trans);
/* Batched: one perm_r and perm for all members (the reference's SamePattern_SameRowPerm: match a representative member on
 * the host, equilibrate every member on the device).  val: batch x nnz, member-major; R and C shared (rc_per_member = 0:
 * n entries) or per member (1: batch x n); out: batch x 6 (nullable).  The equilibration is one launch sequence over (rows,
 * members), the launches of the unbatched call.  batch_get_scaling returns member `member`'s final R and C;
 * batch_solve_scaled takes batch_solve's x layout and its per-member info checks. */
int slu_b200_batch_fill_csr_scaled(slu_b200_handle_t h, int n, const int32_t *rowptr, const int32_t *colind, const double *val,
                                   const int32_t *perm_r, const int32_t *perm, const double *R, const double *C, int rc_per_member,
                                   int flags, double *out);
int slu_b200_batch_get_scaling(slu_b200_handle_t h, int member, double *R, double *C);
int slu_b200_batch_solve_scaled(slu_b200_handle_t h, double *x, int ldx, int nrhs, int trans);
/* ---- iterative refinement with error bounds on the factors of a scaled fill: pdgsrfs (pdgsrfs.c:198-251) for op(A) = A in
 * A's own ordering, the step static pivoting relies on to recover the accuracy lost to replaced tiny pivots.  The scaled
 * fill keeps A in HBM for it (see fill_csr_scaled); a plain fill_csr user gets the same fill from fill_csr_scaled with NULL
 * perm_r, R and C and no flags.
 * b (n x nrhs, ldb >= n): the right-hand sides.  x (ldx >= n): the caller's solution on entry (typically solve_scaled's),
 * the refined one on return.  Per column j and step: r = b - A x, w = |A| |x| + |b| with the kept A, berr = max_i |r_i| / w_i
 * ((safe1 + |r_i|) / w_i where w_i <= safe2, rows with w_i = 0 skipped; safe1 = (n + 1) dmach("S"), safe2 = safe1 / eps);
 * while berr > eps, 2 berr <= the last step's berr (3 at the start) and fewer than 20 steps: x += the scaled solve of r.
 * berr[j] (required) is the berr of the returned x, steps[j] (nullable) the steps taken.  The columns are independent, as in
 * the reference's per-column loop: each step solves the whole block, a column that has stopped is left exactly as it was.
 * ferr[j] (nullable): dgerfs's forward error bound, est ||A^-1 diag(W)||_inf / max_i |x_i| with W_i = |r_i| + (n + 1) eps w_i
 * (+ safe1 where w_i <= safe2) of the returned x, estimated by the dlacn2 of slu_b200_gscon (divided only where max |x_i| > 0).
 * In doublecomplex |.| is cabs1 (|re| + |im|), as pzgsrfs and zgerfs, and the estimate solves with A^H.
 * The residual walks each row's entries in CSR order with unfused multiplies and adds, and the maxima are integer atomics on
 * bit patterns: berr is a pure function of (A, b, x), bit for bit.  The solves sum with atomic adds, so the steps taken and
 * the refined x can differ between runs at the eps level.  b and x go up once and x comes back once; per step the host reads
 * the count of columns still active.  stats.reserved[4] / [5] = seconds and kernel launches of the whole call.
 * Fails with a message, leaving the handle usable, without a scaled fill (or after a later upload, fill_csr, batch_fill_csr
 * or batch_fill_affine) and a successful factor after it, on Schur handles, grids other than 1 x 1 x 1 with world_size 1,
 * ldb or ldx < n, nrhs < 1, n * nrhs >= 2^31, and null b, x or berr.
 * batch_gsrfs: b and x in batch_solve_scaled's layout (ldb / ldx apart, nrhs columns per member); berr, ferr and steps hold
 * batch x nrhs entries, member-major; fails, naming the member, unless every member's last info was 0. */
int slu_b200_gsrfs(slu_b200_handle_t h, const double *b, int ldb, double *x, int ldx, int nrhs, double *berr, double *ferr,
                   int32_t *steps);
int slu_b200_batch_gsrfs(slu_b200_handle_t h, const double *b, int ldb, double *x, int ldx, int nrhs, double *berr,
                         double *ferr, int32_t *steps);
/* ---- device-resident refill and solves on the caller's CUDA stream: the loop of pdgssvx3d's Fact = SamePattern_SameRowPerm
 * (Newton and time-stepping loops, parameter and shift sweeps) for values and right-hand sides that are already on the GPU.
 * stream: a cudaStream_t passed as void* (NULL = the legacy default stream).  val and x must be device or managed memory on
 * the handle's device (checked with cudaPointerGetAttributes before anything is enqueued; host memory or another device's
 * memory is refused, naming the argument); keeping x + ldx * nrhs (* batch) in bounds is the caller's job.  Each call makes
 * the handle's stream wait for the work already on `stream` before it reads val or x, and `stream` wait for the handle's
 * work before it returns, with events: the caller may overwrite or free val and read x in `stream` order right after the
 * call.  No host synchronisation and no PCIe copy, except where a buffer grows (a larger nrhs) and in the first refill after
 * each scaled fill, which builds the slot map and waits for it.  stats.reserved[5] = the call's kernel launches;
 * stats.reserved[4] (and t_upload_s for a refill) = 0: no host clock measures work that is not waited for.
 * refill: new values of the pattern of the handle's last successful scaled fill (fill_csr_scaled, batch_fill_csr_scaled),
 * val: nnz values in that fill's CSR entry order (batch x nnz, member-major, on a batched handle).  The arena is zeroed and
 * F = Pc Pr Dr A Dc Pc^T written with the kept perm_r, perm, R and C: (R[i] * a_ij) * C[j], one plain store per slot, bit
 * for bit what fill_csr_scaled writes with the same R and C and no EQUIL.  The equilibration is not redone (R and C stay
 * those of the scaled fill, per member).  val also replaces the kept A, so gsrfs refines against the new matrix.  The
 * first refill after a scaled fill builds the slot map: 8 bytes per entry for the arena offset and 4 for the row, shared by
 * the members, dropped with the scaling.  Then 1 launch: thread = entry, no search.  After it the handle has values and
 * its scaling and no factors: factor / batch_factor follow, on the handle's stream after the refill.  Fails with a message,
 * leaving the handle as it was, without a scaled fill (or after a later upload or plain fill, which drop it), on Schur
 * handles and on grids other than 1 x 1 x 1 with world_size 1.
 * solve_device / solve_scaled_device: slu_b200_solve and _solve_trans (trans 0, 1 or 2, F's ordering) and
 * slu_b200_solve_scaled (A's ordering) on device x, with their layout, ldx / nrhs checks (n * nrhs < 2^31) and state
 * checks; the same device work, with device-to-device 2D copies in place of the H2D and D2H ones.  1 x 1 x 1 grids only.
 * The batched twins take the batched layout (member j's block at x + j * ldx * nrhs) and check every member's info. */
int slu_b200_refill(slu_b200_handle_t h, const double *val, void *stream);
int slu_b200_batch_refill(slu_b200_handle_t h, const double *val, void *stream);
int slu_b200_solve_device(slu_b200_handle_t h, double *x, int ldx, int nrhs, int trans, void *stream);
int slu_b200_batch_solve_device(slu_b200_handle_t h, double *x, int ldx, int nrhs, int trans, void *stream);
int slu_b200_solve_scaled_device(slu_b200_handle_t h, double *x, int ldx, int nrhs, int trans, void *stream);
int slu_b200_batch_solve_scaled_device(slu_b200_handle_t h, double *x, int ldx, int nrhs, int trans, void *stream);
/* ---- factorization on the caller's CUDA stream, and CUDA graphs of refill -> factor -> solve.
 * factor_device / batch_factor_device: slu_b200_factor / _batch_factor (the same plan, kernels, look-ahead streams, deferred
 * chains and int8 route), ordered on `stream` as the calls above, for 1 x 1 x 1 grids and handles that are not Schur handles;
 * refused, with a message, before a successful fill, upload or refill.  No host wait, no host copy and no allocation.  info:
 * 1 (batch) int32 in device memory on the handle's device (checked as val / x above), written in `stream` order with each
 * member's status: 0 factored; > 0 the 1-based column of the first exact zero pivot, as slu_b200_factor's info; -1 when
 * Schur-update destinations were missing from the L/U structure (slu_b200_factor fails with a message there).  The handle
 * keeps the same status on the device.  stats.gpu_launches counts the call's kernels (2 more than slu_b200_factor: the status
 * reset and the status write); stats.t_factor_s = 0.
 * Deferred status: until the host has read it, the handle's factors are "pending".  The calls on `stream` (solve_device,
 * solve_scaled_device and their batched twins) take pending factors as they are, without a wait.  Every host-synchronous
 * call that needs factors (solve, solve_trans, solve_scaled, gscon, gsrfs, selinv, logdet, inertia and their batched
 * twins) and get_stats first synchronise the handle's stream and read the status: they then refuse, and report
 * stats.tiny_pivots, exactly as after slu_b200_factor.
 * get_stats while the handle's stream is being captured (after a captured call, before the capture ends) does not wait:
 * it returns the stats as the host last saw them.
 * Solves after a failed member: a device solve cannot refuse what the host has not seen.  solve_device and
 * solve_scaled_device (both precisions, batched or not) overwrite every column of x (rows 0 .. n-1) of each member whose
 * status is not 0 with quiet NaN (both parts in doublecomplex); the other members' x are the solutions.  On a handle
 * with a captured call, whose status a replay may change behind the host's back, the device solves accept any status and
 * leave it to this guard.
 * CUDA graphs: refill, factor_device, solve_device and solve_scaled_device (and their batched / z twins) may be captured
 * (cudaStreamBeginCapture on `stream`, any capture mode; torch.cuda.CUDAGraph).  Under capture a call that would allocate,
 * grow a buffer or wait on the host is refused before it enqueues anything, leaving the capture valid: the first refill
 * after a scaled fill, and a solve with more right-hand sides (nrhs * batch) than any solve before.  Make such a call once
 * outside capture first.  A graph holds the addresses of the handle's buffers: from the first captured call on, a call that
 * would reallocate one of them (a solve, gscon or gsrfs with more right-hand sides than any before, a scaled fill with
 * another nnz) is refused, naming the captured graph, until slu_b200_destroy; an upload or plain fill keeps the kept A's
 * buffers instead of freeing them.  A buffer that no call has allocated yet is in no graph: a later call outside capture
 * allocates it (gscon after a captured gsrfs_device without ferr, gsrfs after a captured gscon_device).  A replay runs on the stream it is launched on, not on the handle's stream: a
 * host-synchronous call after a replay needs the caller to have synchronised that stream first (the status it reads is
 * then the replay's, and a selinv inverse from before a replayed factorization is refused as after slu_b200_factor); a
 * call on the same stream is ordered after the replay without that.  Destroying the handle while
 * a graph that uses it is alive is the caller's error, as with any CUDA library workspace. */
int slu_b200_factor_device(slu_b200_handle_t h, int32_t *info, void *stream);
int slu_b200_batch_factor_device(slu_b200_handle_t h, int32_t *info, void *stream);
/* ---- iterative refinement and condition estimation on the caller's CUDA stream, capturable into the same graph.
 * gsrfs_device / batch_gsrfs_device: slu_b200_gsrfs / _batch_gsrfs (A x = b on the factors and scalings of the last scaled
 * fill or refill and the A it kept) with b, x, berr and the nullable ferr and steps in device memory, in the host twins'
 * layouts (outputs: one value per (member, column), member-major); they compute what the host twins compute.
 * gscon_device / batch_gscon_device: slu_b200_gscon / _batch_gscon (dlacn2 on F after a fill and a factorization) with anorm
 * and rcond in device memory, one value per member; norm '1', 'O' or 'I'.
 * Preconditions, pointer checks, stream order and refusals are those of solve_device / solve_scaled_device above: 1 x 1 x 1
 * grids, no Schur handles, gsrfs_device needs a scaled fill; factors pending from factor_device are taken as they are.  No
 * host wait, PCIe copy or allocation, except where a buffer grows: the first call of each kind, or a gsrfs_device with more
 * right-hand sides than any before, allocates and must be made once outside capture (under capture it is refused before
 * anything is enqueued, leaving the capture valid).  The loops run on the device: each is a conditional WHILE node of a CUDA
 * graph whose body decides, on the device, whether it runs again (the estimator's body runs its solve in one of two IF
 * nodes), with the host loops' kernels, so the device loops take the same decisions on the same vectors.  Called under
 * capture, the nodes go into the caller's graph; called eagerly, the handle launches a graph of the same sequence that it
 * captured at the first such call (one per kind, batched, nrhs and ferr; captured again when a buffer it holds moved).  That
 * first eager call of each kind, nrhs and ferr instantiates its graph, which may wait for the device once.
 * A member whose status is not 0 (a zero pivot from factor_device, which the host has not seen): x, berr, ferr and rcond
 * NaN, steps 0, its columns never refined; the other members are unaffected.  An estimate that does not finish in 64 solves
 * (where the host calls fail) gives NaN ferr / rcond for the members still waiting.  gscon_device: rcond 0 for anorm 0 or
 * +inf, NaN for a negative or NaN anorm (refused by the host call).  stats.reserved[4] = 0, [5] = the launches enqueued
 * outside the loops plus one pass of each loop body (both IF bodies); gscon_device sets [6] and [7] to 0.
 * Needs a CUDA driver of version 12.4 or later (conditional nodes); an older one is refused, naming its version. */
int slu_b200_gsrfs_device(slu_b200_handle_t h, const double *b, int ldb, double *x, int ldx, int nrhs, double *berr,
                          double *ferr, int32_t *steps, void *stream);
int slu_b200_batch_gsrfs_device(slu_b200_handle_t h, const double *b, int ldb, double *x, int ldx, int nrhs, double *berr,
                                double *ferr, int32_t *steps, void *stream);
int slu_b200_gscon_device(slu_b200_handle_t h, char norm, const double *anorm, double *rcond, void *stream);
int slu_b200_batch_gscon_device(slu_b200_handle_t h, char norm, const double *anorm, double *rcond, void *stream);
/* ---- gradients on the caller's CUDA stream, capturable into the same graph: the pieces of d log|det A| / dA and of the
 * adjoint of x = A^-1 b, in A's own ordering and on the pattern of the last scaled fill (the order refill takes).
 * selinv_device / batch_selinv_device: slu_b200_selinv / _batch_selinv ordered on the stream, with no host wait and no
 * timing.  The missed-destination check stays on the device: a member of a sweep that missed one gets NaN from
 * logdet_grad_device, and the next host-synchronous call reads the check before it lets selinv_get use the inverse.  The
 * first selected inversion on a handle allocates the second arena and uploads the plan (refused under capture); the arena is
 * never moved afterwards.
 * logdet_device / batch_logdet_device: slu_b200_logdet / _batch_logdet into logabs[members] and sign[members] in device
 * memory, bit for bit the host call's values.
 * logdet_grad_device / batch_logdet_grad_device: grad[j nnz + e] = coef[j] R_i C_j H(perm[perm_r[i]], perm[j]) for entry e =
 * (i, j) of the scaled fill's CSR pattern, H the inverse of the last selinv or selinv_device (F^-T), R and C member j's
 * scalings: coef[j] A_j^-T(i, j), the gradient of log |det A_j| times coef[j].  coef: one value per member in device memory.
 * Refused when the host knows the inverse is stale (a later fill, refill, upload or factorization).
 * solve_grad_device / batch_solve_grad_device: grad[j nnz + e] = -sum_k lam_j(i, k) x_j(col, k) for entry e = (i, col) of the
 * same pattern: the gradient of a loss with respect to A's values when x = A^-1 b and lam = A^-T dL/dx (solve_scaled_device
 * with trans 1).  lam and x: n x nrhs column-major per member, ldl / ldx elements apart per column, member-major.  A first
 * call with more right-hand sides than any before allocates a staging buffer (refused under capture).
 * Every call: the preconditions, pointer checks, stream order and refusals of solve_scaled_device (a scaled fill, factors from
 * factor or pending from factor_device, 1 x 1 x 1 grids, no Schur handles); the first gradient call after a scaled fill builds
 * the refill's slot map if no refill did (allocates and waits once; refused under capture).  A member whose status is not 0
 * gets NaN results; the other members are unaffected.  stats.reserved[4] = 0, [5] = the launches enqueued. */
int slu_b200_selinv_device(slu_b200_handle_t h, void *stream);
int slu_b200_batch_selinv_device(slu_b200_handle_t h, void *stream);
int slu_b200_logdet_device(slu_b200_handle_t h, double *logabs, double *sign, void *stream);
int slu_b200_batch_logdet_device(slu_b200_handle_t h, double *logabs, double *sign, void *stream);
int slu_b200_logdet_grad_device(slu_b200_handle_t h, const double *coef, double *grad, void *stream);
int slu_b200_batch_logdet_grad_device(slu_b200_handle_t h, const double *coef, double *grad, void *stream);
int slu_b200_solve_grad_device(slu_b200_handle_t h, const double *lam, int ldl, const double *x, int ldx, int nrhs,
                               double *grad, void *stream);
int slu_b200_batch_solve_grad_device(slu_b200_handle_t h, const double *lam, int ldl, const double *x, int ldx, int nrhs,
                                     double *grad, void *stream);
/* the CUDA device the handle was created on (options.device, or the current device when that was < 0): where the
 * device-memory arguments of the calls above must live */
int slu_b200_get_device(slu_b200_handle_t h, int *device);
/* ---- doublecomplex twins (SRC/complex16/pzgstrf3d.c:120; the reference's z* handle API,
 * SRC/include/superlu_upacked.h:84-97).  Same view/options/stats structs: the Lnzval_bc_ptr / Unzval_br_ptr
 * entries point at arrays of doublecomplex {double r, i} (SRC/include/dcomplex.h:30) and are declared double*
 * only to keep one struct; n, nsupr, lda ... count complex elements.  Supernodes up to 256 columns.
 * stats.ops_fact follows the reference's own complex accounting (pzgstrf2.c:578,590 for the diagonal blocks,
 * the precision-independent 2*m*n*k for the Schur update, sec_structs.c:692-693).
 * slu_b200_z_fill_csr and slu_b200_z_solve follow the same convention: val and x point at interleaved
 * doublecomplex, and n, ldx, nnz count complex elements.  The solve (the role of pzgstrs3d,
 * SRC/complex16/pzgstrs3d.c) has the restrictions of slu_b200_solve.  slu_b200_z_solve_trans solves A^T x = b (trans 1)
 * or A^H x = b (trans 2: every factor entry, the pivots included, is read conjugated), as slu_b200_solve_trans.
 * Checked on an H100 by tests/test_gpu_variants_complex.py: kernels vs NumPy, cg20 vs the reference's pzgstrf3d
 * factors, pzdrive3d drop-in; by tests/test_gpu_solve_complex.py: solves on the resident factors, device-side
 * distribution; and by tests/test_gpu_solve_trans.py: transposed and conjugate-transposed solves against SciPy. */
typedef struct slu_b200_zhandle_s *slu_b200_zhandle_t;
int slu_b200_z_create(slu_b200_zhandle_t *h, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt);
int slu_b200_z_upload(slu_b200_zhandle_t h);
int slu_b200_z_factor(slu_b200_zhandle_t h, int *info);
int slu_b200_z_factor_host(slu_b200_zhandle_t h, int *info);
int slu_b200_z_download(slu_b200_zhandle_t h);
int slu_b200_z_fill_csr(slu_b200_zhandle_t h, int n, const int32_t *rowptr, const int32_t *colind, const double *val,
                        const int32_t *perm);
int slu_b200_z_solve(slu_b200_zhandle_t h, double *x, int ldx, int nrhs);
int slu_b200_z_solve_trans(slu_b200_zhandle_t h, double *x, int ldx, int nrhs, int trans);
/* as slu_b200_gscon, with zgecon's zlacn2: "kase 2" solves with F^H, |x_i| is the modulus, the sign vector is x_i / |x_i|
 * (1 where |x_i| is below the safe minimum) and there is no repeated-sign test */
int slu_b200_z_gscon(slu_b200_zhandle_t h, char norm, double anorm, double *rcond);
/* as slu_b200_selinv / _selinv_get / _logdet, with the same restrictions, messages and invalidation.  H = F^-T with a
 * plain transpose, not the conjugate, so A^-1(i, j) = H(perm[j], perm[i]) holds unchanged (for a Hermitian A,
 * A^-1(j, i) = conj(A^-1(i, j))).  out[1] counts 2 flops per complex multiply-add, as ops_fact does: 4x that in real
 * flops.  selinv_get's out holds nnz interleaved doublecomplex (a complex NaN where a failed entry has no slot).
 * z_logdet: *logabs = log |det A| = sum of log |u_ii|; sign[0..1] = exp(i theta), theta = sum of arg u_ii reduced
 * modulo 2 pi (|sign| = 1), as complex numpy.linalg.slogdet returns it; fixed-order sums, deterministic. */
int slu_b200_z_selinv(slu_b200_zhandle_t h, double out[4]);
int slu_b200_z_selinv_get(slu_b200_zhandle_t h, int n, const int32_t *rowptr, const int32_t *colind,
                          const int32_t *perm, double *out);
int slu_b200_z_logdet(slu_b200_zhandle_t h, double *logabs, double *sign);
/* as slu_b200_schur_create / _schur_get / _schur_condense / _schur_expand, with the same restrictions and messages; S and
 * x hold interleaved doublecomplex (S: s x s complex), lds and ldx count complex elements. */
int slu_b200_z_schur_create(slu_b200_zhandle_t *h, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, int nschur);
int slu_b200_z_schur_get(slu_b200_zhandle_t h, double *S, int lds);
int slu_b200_z_schur_condense(slu_b200_zhandle_t h, double *x, int ldx, int nrhs);
int slu_b200_z_schur_expand(slu_b200_zhandle_t h, double *x, int ldx, int nrhs);
/* batched doublecomplex handles (the reference's pzgssvx3d_csc_batch, SRC/complex16/pzgssvx3d_csc_batch.c:80): the
 * slu_b200_batch_* calls above with the same semantics, restrictions and stats; val and x point at interleaved
 * doublecomplex, n, ldx and nnz count complex elements.  Stats through slu_b200_z_get_stats, slu_b200_z_destroy frees.
 * A batched z handle takes only these calls, and these fail on an unbatched z handle.  Measured on an NVIDIA H100 80GB
 * HBM3 at a 400 W power limit, per member, against one unbatched z handle looping over the members: Poisson 16^3,
 * B = 64: factor 0.203 vs 4.147 ms (20.5x), solve (nrhs 1) 0.056 vs 1.130 ms; more in README.md. */
int slu_b200_z_batch_create(slu_b200_zhandle_t *h, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, int batch);
int slu_b200_z_batch_fill_csr(slu_b200_zhandle_t h, int n, const int32_t *rowptr, const int32_t *colind,
                              const double *val, const int32_t *perm);
int slu_b200_z_batch_factor(slu_b200_zhandle_t h, int *info);
int slu_b200_z_batch_solve(slu_b200_zhandle_t h, double *x, int ldx, int nrhs);
int slu_b200_z_batch_solve_trans(slu_b200_zhandle_t h, double *x, int ldx, int nrhs, int trans);
int slu_b200_z_batch_gscon(slu_b200_zhandle_t h, char norm, const double *anorm, double *rcond);
int slu_b200_z_batch_download(slu_b200_zhandle_t h, int member);
/* as slu_b200_batch_selinv / _batch_selinv_get / _batch_logdet, with the z conventions of slu_b200_z_selinv: out of
 * z_batch_selinv_get holds batch x nnz interleaved doublecomplex, member-major; z_batch_logdet's sign holds 2 x batch
 * doubles, exp(i theta_j) as (re, im) pairs. */
int slu_b200_z_batch_selinv(slu_b200_zhandle_t h, double out[4]);
int slu_b200_z_batch_selinv_get(slu_b200_zhandle_t h, int n, const int32_t *rowptr, const int32_t *colind,
                                const int32_t *perm, double *out);
int slu_b200_z_batch_logdet(slu_b200_zhandle_t h, double *logabs, double *sign);
/* as slu_b200_inertia / _batch_inertia / _batch_fill_affine with the same restrictions and messages: the sign test is on
 * Re u_ii, |u_ii| is the modulus and defect the max of |Im u_ii| / |u_ii|; terms and coef of z_batch_fill_affine hold
 * interleaved doublecomplex, n and nnz count complex elements. */
int slu_b200_z_inertia(slu_b200_zhandle_t h, int64_t counts[3], double *defect);
int slu_b200_z_batch_inertia(slu_b200_zhandle_t h, int64_t *counts, double *defect);
int slu_b200_z_batch_fill_affine(slu_b200_zhandle_t h, int n, const int32_t *rowptr, const int32_t *colind, int nterms,
                                 const double *terms, const double *coef, const int32_t *perm);
/* as slu_b200_batch_schur_create / _get / _condense / _expand, with the same restrictions and messages; S and x hold
 * interleaved doublecomplex, lds and ldx count complex elements. */
int slu_b200_z_batch_schur_create(slu_b200_zhandle_t *h, const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt,
                                  int batch, int nschur);
int slu_b200_z_batch_schur_get(slu_b200_zhandle_t h, double *S, int lds);
int slu_b200_z_batch_schur_condense(slu_b200_zhandle_t h, double *x, int ldx, int nrhs);
int slu_b200_z_batch_schur_expand(slu_b200_zhandle_t h, double *x, int ldx, int nrhs);
/* as slu_b200_fill_csr_scaled / _get_scaling / _solve_scaled and their batched twins, with the same semantics and
 * messages: val and x hold interleaved doublecomplex, the scalings R and C are real; the equilibration uses slud_z_abs1. */
int slu_b200_z_fill_csr_scaled(slu_b200_zhandle_t h, int n, const int32_t *rowptr, const int32_t *colind, const double *val,
                               const int32_t *perm_r, const int32_t *perm, const double *R, const double *C, int flags,
                               double out[6]);
int slu_b200_z_get_scaling(slu_b200_zhandle_t h, int32_t *perm_r, double *R, double *C);
int slu_b200_z_solve_scaled(slu_b200_zhandle_t h, double *x, int ldx, int nrhs, int trans);
int slu_b200_z_batch_fill_csr_scaled(slu_b200_zhandle_t h, int n, const int32_t *rowptr, const int32_t *colind,
                                     const double *val, const int32_t *perm_r, const int32_t *perm, const double *R,
                                     const double *C, int rc_per_member, int flags, double *out);
int slu_b200_z_batch_get_scaling(slu_b200_zhandle_t h, int member, double *R, double *C);
int slu_b200_z_batch_solve_scaled(slu_b200_zhandle_t h, double *x, int ldx, int nrhs, int trans);
/* as slu_b200_gsrfs / _batch_gsrfs: b and x hold interleaved doublecomplex (ldb, ldx count complex elements), berr and ferr
 * are real; |.| is cabs1 and the forward error estimate solves with A^H */
int slu_b200_z_gsrfs(slu_b200_zhandle_t h, const double *b, int ldb, double *x, int ldx, int nrhs, double *berr, double *ferr,
                     int32_t *steps);
int slu_b200_z_batch_gsrfs(slu_b200_zhandle_t h, const double *b, int ldb, double *x, int ldx, int nrhs, double *berr,
                           double *ferr, int32_t *steps);
/* as slu_b200_refill / _solve_device / _solve_scaled_device and their batched twins: val and x point at interleaved
 * doublecomplex on the device, nnz and ldx count complex elements */
int slu_b200_z_refill(slu_b200_zhandle_t h, const double *val, void *stream);
int slu_b200_z_batch_refill(slu_b200_zhandle_t h, const double *val, void *stream);
int slu_b200_z_solve_device(slu_b200_zhandle_t h, double *x, int ldx, int nrhs, int trans, void *stream);
int slu_b200_z_batch_solve_device(slu_b200_zhandle_t h, double *x, int ldx, int nrhs, int trans, void *stream);
int slu_b200_z_solve_scaled_device(slu_b200_zhandle_t h, double *x, int ldx, int nrhs, int trans, void *stream);
int slu_b200_z_batch_solve_scaled_device(slu_b200_zhandle_t h, double *x, int ldx, int nrhs, int trans, void *stream);
int slu_b200_z_factor_device(slu_b200_zhandle_t h, int32_t *info, void *stream);
int slu_b200_z_batch_factor_device(slu_b200_zhandle_t h, int32_t *info, void *stream);
int slu_b200_z_get_device(slu_b200_zhandle_t h, int *device);
/* as slu_b200_gsrfs_device / _gscon_device and their batched twins: b and x interleaved doublecomplex on the device (ldb, ldx
 * count complex elements); berr, ferr, anorm and rcond real */
int slu_b200_z_gsrfs_device(slu_b200_zhandle_t h, const double *b, int ldb, double *x, int ldx, int nrhs, double *berr,
                            double *ferr, int32_t *steps, void *stream);
int slu_b200_z_batch_gsrfs_device(slu_b200_zhandle_t h, const double *b, int ldb, double *x, int ldx, int nrhs,
                                  double *berr, double *ferr, int32_t *steps, void *stream);
int slu_b200_z_gscon_device(slu_b200_zhandle_t h, char norm, const double *anorm, double *rcond, void *stream);
int slu_b200_z_batch_gscon_device(slu_b200_zhandle_t h, char norm, const double *anorm, double *rcond, void *stream);
/* as slu_b200_selinv_device / _logdet_device / _logdet_grad_device / _solve_grad_device and their batched twins: sign holds
 * 2 x members doubles (exp(i theta) as (re, im)); coef, grad, lam and x interleaved doublecomplex (ldl, ldx count complex
 * elements).  logdet_grad: grad = coef[j] R_i C_j conj(H(...)), coef[j] A_j^-H(i, j); solve_grad: grad = -sum_k lam_j(i, k)
 * conj(x_j(col, k)) with lam = A^-H dL/dx (trans 2) */
int slu_b200_z_selinv_device(slu_b200_zhandle_t h, void *stream);
int slu_b200_z_batch_selinv_device(slu_b200_zhandle_t h, void *stream);
int slu_b200_z_logdet_device(slu_b200_zhandle_t h, double *logabs, double *sign, void *stream);
int slu_b200_z_batch_logdet_device(slu_b200_zhandle_t h, double *logabs, double *sign, void *stream);
int slu_b200_z_logdet_grad_device(slu_b200_zhandle_t h, const double *coef, double *grad, void *stream);
int slu_b200_z_batch_logdet_grad_device(slu_b200_zhandle_t h, const double *coef, double *grad, void *stream);
int slu_b200_z_solve_grad_device(slu_b200_zhandle_t h, const double *lam, int ldl, const double *x, int ldx, int nrhs,
                                 double *grad, void *stream);
int slu_b200_z_batch_solve_grad_device(slu_b200_zhandle_t h, const double *lam, int ldl, const double *x, int ldx, int nrhs,
                                       double *grad, void *stream);
int slu_b200_z_get_stats(slu_b200_zhandle_t h, slu_b200_stats_t *out);
int slu_b200_z_plan(const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, slu_b200_stats_t *stats);
void slu_b200_z_destroy(slu_b200_zhandle_t h);
/* drop-in body of pzgstrf3d (complex16/pzgstrf3d.c:120-123): create + upload + factor + download + destroy */
int pzgstrf3d_b200(const slu_b200_lu_view_t *lu, const slu_b200_options_t *opt, slu_b200_stats_t *stats, int *info);
void slu_b200_z_comm_cache_clear(void);   /* called by slu_b200_comm_cache_clear */
/* kernel-level test entries; arrays are interleaved (re, im), sizes in complex elements */
int slu_b200_z_k_diag_lu(double *a, int ns, int lda, int replace_tiny, double thresh, int col0, int *info, int *tiny);
int slu_b200_z_k_trsm_l(const double *lu, int ldlu, int ns, double *x, int m, int ldx);
int slu_b200_z_k_trsm_u(const double *lu, int ldlu, int ns, double *x, int ncols, int ldx);
int slu_b200_z_k_gemm_sub(int m, int n, int k, const double *a, int lda, const double *b, int ldb, double *c, int ldc,
                          int reps, float *ms);

#ifdef __cplusplus
}
#endif
#endif /* SLU_B200_H */
