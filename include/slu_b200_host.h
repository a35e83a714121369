/*
 * slu_b200_host.h -- C-ABI of libslu_b200_host.so: host-side producers of the INPUT of the hot
 * path, in the reference's data layout.  On the GPU box /root/reference does not exist, so the
 * synthetic benchmark matrices of BASELINE.json (3D 7-pt Poisson, audikw_1-shaped FEM) need their
 * own ordering + symbolic factorization + "distribution" into dLocalLU_t-style block storage.
 * These play the role of (they are NOT ports of):
 *   get_perm_c_dist            SRC/prec-independent/get_perm_c.c:479      -> sluh_nd_order (geometric ND),
 *                                                                          sluh_nd_order_graph (any pattern)
 *   symbfact / sp_colorder     SRC/prec-independent/symbfact.c, sp_colorder.c -> sluh_symbolic
 *   pddistribute3d             SRC/double/pddistribute3d.c:1357           -> sluh_symb_export + sluh_fill_values
 *   getForests                 SRC/prec-independent/supernodalForest.c:29 -> sluh_forests
 * plus the ||LU - A||_F checker the reference lacks (BASELINE.md section 2).
 * Pure C++/OpenMP, no CUDA: usable in the CPU-only test-suite.
 */
#ifndef SLU_B200_HOST_H
#define SLU_B200_HOST_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- synthetic matrices (CSR, int32 indices) ------------------------------------------------ */
/* 7-point Laplacian on an nx x ny x nz grid, Dirichlet: a_ii = 6, a_ij = -1 (SURVEY 8d config 2). */
int64_t sluh_poisson3d_nnz(int nx, int ny, int nz);
void sluh_poisson3d(int nx, int ny, int nz, int32_t *rowptr, int32_t *colind, double *val);
/* audikw_1-shaped: `dof` unknowns per node of an nx x ny x nz grid coupled through the 27-point
 * stencil; off-diagonals uniform(-1,0) from a counter-based generator seeded with `seed`,
 * diagonal = sum |row| + 1 (strictly diagonally dominant, unsymmetric values, symmetric pattern). */
int64_t sluh_fem3d_nnz(int nx, int ny, int nz, int dof);
void sluh_fem3d(int nx, int ny, int nz, int dof, uint64_t seed, int32_t *rowptr, int32_t *colind,
                double *val);
/* Geometric nested dissection of the grid (dof unknowns per node kept adjacent):
 * perm[old] = new.  Boxes with <= leaf nodes are ordered lexicographically. */
void sluh_nd_order(int nx, int ny, int nz, int dof, int leaf, int32_t *perm);
/* Nested dissection of a GENERAL pattern (a matrix read from a file has no geometry): A + A^T of the n x n CSR pattern,
 * automatic nested dissection on breadth-first level structures with a greedy separator refinement, pieces of <= leaf
 * unknowns by reverse Cuthill-McKee; compress_dof != 0 merges indistinguishable vertices (the dof of one FEM node)
 * first.  The role of get_perm_c_dist with METIS_AT_PLUS_A (get_perm_c.c:479-560).  perm[old] = new; 0 on success. */
int sluh_nd_order_graph(int n, const int32_t *rowptr, const int32_t *colind, int leaf, int compress_dof, int32_t *perm);

/* ---- static-pivoting row permutation (the role of dldperm_dist job 5 / LargeDiag_MC64, pdgssvx3d.c:727) ----------- */
/* Maximum-product matching of the n x n CSR pattern with the scalings of MC64 job 5 (Duff & Koster 2001): absval[p] =
 * |a_p| (the caller passes the modulus for complex A); explicit zeros are not edges.  perm_r[i] = the row of Pr A that
 * holds row i of A, so that a_{i, perm_r[i]} lies on the diagonal of Pr A and the product of |diag| is maximal.
 * R[i] = exp(u_i), C[j] = exp(v_j) / colmax_j from the optimal duals: |R_i a_ij C_j| <= 1 everywhere, = 1 on the
 * matching (up to rounding).  Greedy start on the tight edges, then successive shortest augmenting paths (Dijkstra on
 * reduced costs, binary heap); ties go to the smallest row index, so two calls give identical results.
 * Returns 0; the structural rank r < n if A is structurally singular (perm_r, R, C then unwritten, out[0] = -inf);
 * -1 on bad input (rowptr not starting at 0 or decreasing, colind outside 0 .. n-1, a negative or non-finite absval).
 * out (nullable): [0] = sum_i log |a_{i, perm_r[i]}|, [1] = host seconds. */
int sluh_large_diag_perm(int n, const int32_t *rowptr, const int32_t *colind, const double *absval, int32_t *perm_r,
                         double *R, double *C, double out[2]);

/* ---- symbolic factorization of P (A + A^T) P^T ----------------------------------------------- */
typedef struct sluh_symb sluh_symb;
/* perm_in[old] = new (NULL: identity).  The final permutation is perm_in composed with an etree
 * postorder (what sp_colorder does).  relax: subtrees with <= relax columns become one (padded)
 * supernode; maxsup: maximum supernode width (sp_ienv_dist(2), (3)); amalg: a parent column joins
 * the supernode of its child chain while the explicit zeros stay below this fraction of the block
 * (0: exact fundamental supernodes). */
sluh_symb *sluh_symbolic(int n, const int32_t *rowptr, const int32_t *colind,
                         const int32_t *perm_in, int relax, int maxsup, double amalg);
/* Partial factorization (slu_b200_schur_create): as sluh_symbolic, but the nschur columns that perm_in sends to
 * n - nschur .. n - 1 (the Schur set) stay there in their relative order.  The other columns are postordered on their own
 * elimination forest and partitioned as by sluh_symbolic; the Schur block is cut into supernodes of maxsup columns, so
 * n - nschur is a supernode boundary.  nschur = 0 is sluh_symbolic.  NULL if nschur is outside [0, n]. */
sluh_symb *sluh_symbolic_schur(int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm_in,
                               int relax, int maxsup, double amalg, int nschur);
void sluh_symb_free(sluh_symb *s);
int32_t sluh_symb_nsupers(const sluh_symb *s);
/* sizes[0..3] = total lengths of the L index, L value, U index, U value arenas;
 * sizes[4] = flops in the reference's accounting (ops[FACT]); sizes[5] = Schur 2mnk flops part. */
void sluh_symb_sizes(const sluh_symb *s, double *sizes);
/* Copy out: perm[n] (old->new), xsup[nsupers+1], setree[nsupers] (parent, nsupers for roots),
 * offsets [nsupers+1] into each arena, and the two index arenas in the reference layout. */
void sluh_symb_export(const sluh_symb *s, int32_t *perm, int32_t *xsup, int32_t *setree,
                      int64_t *lidx_off, int32_t *lidx, int64_t *lval_off, int64_t *uidx_off,
                      int32_t *uidx, int64_t *uval_off);

/* Zero the value arenas and scatter P A P^T into them (the job of pddistribute3d).  active
 * (nullable, [nsupers]): entries whose destination panel has active == 0 are not written -- panels a
 * Z-layer does not hold (zero length in *_off) or holds as zero-initialised ancestor copies
 * (dinit3DLUstructForest, pdgssvx3d.c:948). */
void sluh_fill_values(int n, const int32_t *rowptr, const int32_t *colind, const double *val,
                      const int32_t *perm, int nsupers, const int32_t *xsup,
                      const int64_t *lidx_off, const int32_t *lidx, const int64_t *lval_off,
                      double *lval, const int64_t *uidx_off, const int32_t *uidx,
                      const int64_t *uval_off, double *uval, const int8_t *active);

/* Z-forest partition (heap numbering of getGridTrees, supernodal_etree.c:840-851):
 * forest_of[k] in [0, 2^maxLvl - 1).  weight[k] = cost estimate of supernode k. */
void sluh_forests(int nsupers, const int32_t *setree, const double *weight, int maxLvl,
                  int32_t *forest_of);

/* ---- checker: y = M x for nvec vectors, M held in the reference L/U block layout ------------- */
/* mode 0: the panels hold a plain matrix (the permuted A before factorization);
 * mode 1: the panels hold factors: y = L (U x), L unit lower.  x, y: n x nvec column-major.
 * Panels whose index pointer is NULL are skipped. */
void sluh_panel_matvec(int mode, int n, int nsupers, const int32_t *xsup,
                       const int32_t *const *lidx, const double *const *lval,
                       const int32_t *const *uidx, const double *const *uval, int nvec,
                       const double *x, double *y);

/* ---- matrix files (SURVEY 8f N4): the formats the reference's drivers read ---------------------- */
/* Harwell-Boeing (dreadhb_dist / zreadhb_dist, SRC/double/dreadhb.c), Matrix Market coordinate (dreadMM_dist,
 * SRC/double/dreadMM.c), Rutherford-Boeing (dreadrb.c), triplets with / without a header line (dreadtriple.c,
 * dreadtriple_noheader.c) and the reference's binary dump (dread_binary, SRC/double/dbinary_io.c).  format: "hb", "rb",
 * "mm", "bin", "dat", "datnh" or NULL (by file extension, the suffixes EXAMPLE/dcreate_matrix.c:108-123 dispatches on:
 * .mtx/.mm, .bin, .dat, .datnh, anything else Harwell- / Rutherford-Boeing).  Symmetric storage is
 * expanded; the result is compressed-column, rows sorted, like the reference's readers return it.
 * Returns NULL and fills err on failure. */
typedef struct sluh_matrix sluh_matrix;
sluh_matrix *sluh_read_matrix(const char *path, const char *format, char *err, int errlen);
void sluh_matrix_dims(const sluh_matrix *m, int32_t *nrow, int32_t *ncol, int64_t *nnz, int32_t *is_complex);
/* val: nnz doubles, or 2*nnz (re, im) for a complex matrix */
void sluh_matrix_export_csc(const sluh_matrix *m, int32_t *colptr, int32_t *rowind, double *val);
void sluh_matrix_export_csr(const sluh_matrix *m, int32_t *rowptr, int32_t *colind, double *val);
void sluh_matrix_free(sluh_matrix *m);
/* dwrite_binary's file layout (dbinary_io.c:24-42) at an arbitrary path; 0 on success */
int sluh_write_binary(const char *path, int32_t n, int32_t nnz, const int32_t *colptr, const int32_t *rowind,
                      const double *val);

#ifdef __cplusplus
}
#endif
#endif
