// slu_host.cpp -- host-side producers of the hot path's input (see include/slu_b200_host.h).
//
// Everything here is written from the published algorithms (Liu's elimination tree, the
// Gilbert-Ng-Peyton column counts, supernodal symbolic factorization, geometric nested
// dissection); the reference's own preprocessing (SRC/prec-independent/symbfact.c, sp_colorder.c,
// SRC/double/pddistribute3d.c) is only the specification of the OUTPUT layout
// (SRC/include/superlu_defs.h:156-204).
#include "slu_b200_host.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <vector>

#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

constexpr int BC_HEADER = 2, LB_DESCRIPTOR = 2, BR_HEADER = 3, UB_DESCRIPTOR = 2;

// ------------------------------------------------------------------------------------------------
// synthetic matrices
// ------------------------------------------------------------------------------------------------
inline uint64_t splitmix64(uint64_t x)
{
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
inline double u01(uint64_t seed, uint64_t a, uint64_t b)
{
    uint64_t h = splitmix64(seed ^ splitmix64(a * 0x100000001B3ull + b));
    return (double)(h >> 11) * (1.0 / 9007199254740992.0);
}

}  // namespace

extern "C" int64_t sluh_poisson3d_nnz(int nx, int ny, int nz)
{
    int64_t n = (int64_t)nx * ny * nz;
    return 7 * n - 2 * ((int64_t)ny * nz + (int64_t)nx * nz + (int64_t)nx * ny);
}

extern "C" void sluh_poisson3d(int nx, int ny, int nz, int32_t *rowptr, int32_t *colind, double *val)
{
    int64_t n = (int64_t)nx * ny * nz;
    // row lengths first (so that the fill can run in parallel)
    rowptr[0] = 0;
    for (int64_t i = 0; i < n; ++i) {
        int x = (int)(i % nx), y = (int)((i / nx) % ny), z = (int)(i / ((int64_t)nx * ny));
        int c = 1 + (x > 0) + (x < nx - 1) + (y > 0) + (y < ny - 1) + (z > 0) + (z < nz - 1);
        rowptr[i + 1] = rowptr[i] + c;
    }
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        int x = (int)(i % nx), y = (int)((i / nx) % ny), z = (int)(i / ((int64_t)nx * ny));
        int64_t p = rowptr[i];
        auto put = [&](int64_t j, double v) { colind[p] = (int32_t)j; val[p] = v; ++p; };
        if (z > 0) put(i - (int64_t)nx * ny, -1.0);
        if (y > 0) put(i - nx, -1.0);
        if (x > 0) put(i - 1, -1.0);
        put(i, 6.0);
        if (x < nx - 1) put(i + 1, -1.0);
        if (y < ny - 1) put(i + nx, -1.0);
        if (z < nz - 1) put(i + (int64_t)nx * ny, -1.0);
    }
}

extern "C" int64_t sluh_fem3d_nnz(int nx, int ny, int nz, int dof)
{
    int64_t nodes_pairs = 0;
    for (int z = 0; z < nz; ++z) {
        int cz = 1 + (z > 0) + (z < nz - 1);
        for (int y = 0; y < ny; ++y) {
            int cy = 1 + (y > 0) + (y < ny - 1);
            // sum over x of cx = 3*nx - 2
            nodes_pairs += (int64_t)cz * cy * (3 * (int64_t)nx - 2);
        }
    }
    return nodes_pairs * dof * dof;
}

extern "C" void sluh_fem3d(int nx, int ny, int nz, int dof, uint64_t seed, int32_t *rowptr,
                           int32_t *colind, double *val)
{
    int64_t nodes = (int64_t)nx * ny * nz;
    rowptr[0] = 0;
    for (int64_t v = 0; v < nodes; ++v) {
        int x = (int)(v % nx), y = (int)((v / nx) % ny), z = (int)(v / ((int64_t)nx * ny));
        int c = (1 + (x > 0) + (x < nx - 1)) * (1 + (y > 0) + (y < ny - 1)) *
                (1 + (z > 0) + (z < nz - 1)) * dof;
        for (int d = 0; d < dof; ++d) rowptr[v * dof + d + 1] = rowptr[v * dof + d] + c;
    }
#pragma omp parallel for schedule(static)
    for (int64_t v = 0; v < nodes; ++v) {
        int x = (int)(v % nx), y = (int)((v / nx) % ny), z = (int)(v / ((int64_t)nx * ny));
        for (int d = 0; d < dof; ++d) {
            int64_t row = v * dof + d, p = rowptr[row], pdiag = -1;
            double s = 0.0;
            for (int dz = -1; dz <= 1; ++dz) {
                if (z + dz < 0 || z + dz >= nz) continue;
                for (int dy = -1; dy <= 1; ++dy) {
                    if (y + dy < 0 || y + dy >= ny) continue;
                    for (int dx = -1; dx <= 1; ++dx) {
                        if (x + dx < 0 || x + dx >= nx) continue;
                        int64_t w = v + dx + (int64_t)dy * nx + (int64_t)dz * nx * ny;
                        for (int e = 0; e < dof; ++e) {
                            int64_t col = w * dof + e;
                            colind[p] = (int32_t)col;
                            if (col == row) {
                                pdiag = p;
                                val[p] = 0.0;
                            } else {
                                double a = -u01(seed, (uint64_t)row, (uint64_t)col);
                                val[p] = a;
                                s += std::fabs(a);
                            }
                            ++p;
                        }
                    }
                }
            }
            val[pdiag] = s + 1.0;
        }
    }
}

namespace {
struct NdCtx {
    int nx, ny, nz, dof, leaf;
    int32_t *perm;
    int64_t next;
};
void nd_emit(NdCtx &c, int x0, int x1, int y0, int y1, int z0, int z1)
{
    for (int z = z0; z < z1; ++z)
        for (int y = y0; y < y1; ++y)
            for (int x = x0; x < x1; ++x) {
                int64_t v = x + (int64_t)y * c.nx + (int64_t)z * c.nx * c.ny;
                for (int d = 0; d < c.dof; ++d) c.perm[v * c.dof + d] = (int32_t)(c.next++);
            }
}
void nd_rec(NdCtx &c, int x0, int x1, int y0, int y1, int z0, int z1)
{
    int lx = x1 - x0, ly = y1 - y0, lz = z1 - z0;
    if (lx <= 0 || ly <= 0 || lz <= 0) return;
    if ((int64_t)lx * ly * lz <= c.leaf || (lx <= 2 && ly <= 2 && lz <= 2)) {
        nd_emit(c, x0, x1, y0, y1, z0, z1);
        return;
    }
    if (lx >= ly && lx >= lz) {
        int m = x0 + lx / 2;
        nd_rec(c, x0, m, y0, y1, z0, z1);
        nd_rec(c, m + 1, x1, y0, y1, z0, z1);
        nd_emit(c, m, m + 1, y0, y1, z0, z1);
    } else if (ly >= lz) {
        int m = y0 + ly / 2;
        nd_rec(c, x0, x1, y0, m, z0, z1);
        nd_rec(c, x0, x1, m + 1, y1, z0, z1);
        nd_emit(c, x0, x1, m, m + 1, z0, z1);
    } else {
        int m = z0 + lz / 2;
        nd_rec(c, x0, x1, y0, y1, z0, m);
        nd_rec(c, x0, x1, y0, y1, m + 1, z1);
        nd_emit(c, x0, x1, y0, y1, m, m + 1);
    }
}
}  // namespace

extern "C" void sluh_nd_order(int nx, int ny, int nz, int dof, int leaf, int32_t *perm)
{
    NdCtx c{nx, ny, nz, dof, leaf < 1 ? 1 : leaf, perm, 0};
    nd_rec(c, 0, nx, 0, ny, 0, nz);
}

// ------------------------------------------------------------------------------------------------
// symbolic factorization
// ------------------------------------------------------------------------------------------------
struct sluh_symb {
    int n = 0, nsupers = 0;
    std::vector<int32_t> perm, xsup, supno, setree;
    std::vector<int64_t> sptr;   // [nsupers+1] into srow
    std::vector<int32_t> srow;   // sorted global rows of each supernode (own columns first)
    double ops_fact = 0, ops_schur = 0;
    double lidx_len = 0, lval_len = 0, uidx_len = 0, uval_len = 0;
};

namespace {

// strictly-lower pattern of P (A+A^T) P^T, CSC (column c -> sorted unique rows r > c)
void build_lower(int n, const int32_t *rowptr, const int32_t *colind, const int32_t *p,
                 std::vector<int64_t> &cp, std::vector<int32_t> &ri)
{
    cp.assign((size_t)n + 1, 0);
    for (int i = 0; i < n; ++i)
        for (int64_t q = rowptr[i]; q < rowptr[i + 1]; ++q) {
            int j = colind[q];
            if (i == j) continue;
            int r = p[i], c = p[j];
            ++cp[(size_t)std::min(r, c) + 1];
        }
    for (int c = 0; c < n; ++c) cp[c + 1] += cp[c];
    std::vector<int32_t> tmp((size_t)cp[n]);
    std::vector<int64_t> nxt(cp.begin(), cp.end() - 1);
    for (int i = 0; i < n; ++i)
        for (int64_t q = rowptr[i]; q < rowptr[i + 1]; ++q) {
            int j = colind[q];
            if (i == j) continue;
            int r = p[i], c = p[j];
            tmp[(size_t)nxt[std::min(r, c)]++] = std::max(r, c);
        }
    std::vector<int64_t> cnt((size_t)n + 1, 0);
#pragma omp parallel for schedule(dynamic, 4096)
    for (int c = 0; c < n; ++c) {
        auto b = tmp.begin() + cp[c], e = tmp.begin() + cp[c + 1];
        std::sort(b, e);
        cnt[c + 1] = std::unique(b, e) - b;
    }
    std::vector<int64_t> cp2((size_t)n + 1, 0);
    for (int c = 0; c < n; ++c) cp2[c + 1] = cp2[c] + cnt[c + 1];
    ri.resize((size_t)cp2[n]);
#pragma omp parallel for schedule(static)
    for (int c = 0; c < n; ++c)
        std::copy(tmp.begin() + cp[c], tmp.begin() + cp[c] + cnt[c + 1], ri.begin() + cp2[c]);
    cp.swap(cp2);
}

// transpose of a strictly-lower CSC: for each row r the sorted columns c < r
void transpose_lower(int n, const std::vector<int64_t> &cp, const std::vector<int32_t> &ri,
                     std::vector<int64_t> &rp, std::vector<int32_t> &ci)
{
    rp.assign((size_t)n + 1, 0);
    for (size_t q = 0; q < ri.size(); ++q) ++rp[(size_t)ri[q] + 1];
    for (int r = 0; r < n; ++r) rp[r + 1] += rp[r];
    ci.resize(ri.size());
    std::vector<int64_t> nxt(rp.begin(), rp.end() - 1);
    for (int c = 0; c < n; ++c)
        for (int64_t q = cp[c]; q < cp[c + 1]; ++q) ci[(size_t)nxt[ri[q]]++] = c;
}

// Liu's elimination-tree algorithm with path compression
void etree(int n, const std::vector<int64_t> &rp, const std::vector<int32_t> &ci,
           std::vector<int32_t> &parent)
{
    parent.assign(n, -1);
    std::vector<int32_t> anc(n, -1);
    for (int j = 0; j < n; ++j)
        for (int64_t q = rp[j]; q < rp[j + 1]; ++q) {
            int r = ci[q];
            while (anc[r] != -1 && anc[r] != j) {
                int t = anc[r];
                anc[r] = j;
                r = t;
            }
            if (anc[r] == -1) { anc[r] = j; parent[r] = j; }
        }
}

void postorder(int n, const std::vector<int32_t> &parent, std::vector<int32_t> &invpost)
{
    std::vector<int32_t> head(n, -1), next(n, -1), stack;
    for (int j = n - 1; j >= 0; --j)
        if (parent[j] != -1) { next[j] = head[parent[j]]; head[parent[j]] = j; }
    invpost.assign(n, -1);
    int k = 0;
    for (int root = 0; root < n; ++root) {
        if (parent[root] != -1) continue;
        stack.push_back(root);
        while (!stack.empty()) {
            int v = stack.back(), c = head[v];
            if (c == -1) { invpost[v] = k++; stack.pop_back(); }
            else { head[v] = next[c]; stack.push_back(c); }
        }
    }
}

}  // namespace

extern "C" sluh_symb *sluh_symbolic(int n, const int32_t *rowptr, const int32_t *colind,
                                    const int32_t *perm_in, int relax, int maxsup, double amalg)
{
    return sluh_symbolic_schur(n, rowptr, colind, perm_in, relax, maxsup, amalg, 0);
}

// nschur > 0: the columns perm_in sends to n - nschur .. n - 1 (the Schur set) stay there, in the caller's relative order.
// Every ancestor of a Schur column is a Schur column, so postordering only the elimination forest of the other columns (a
// column whose parent is a Schur column becomes a root) and appending the Schur columns keeps parent > child.  Column
// counts and the relaxed / amalgamated partition are computed on that postordered part alone; the Schur block is cut
// into supernodes of maxsup columns, so no supernode straddles column n - nschur.
extern "C" sluh_symb *sluh_symbolic_schur(int n, const int32_t *rowptr, const int32_t *colind, const int32_t *perm_in,
                                          int relax, int maxsup, double amalg, int nschur)
{
    if (nschur < 0 || nschur > n) return nullptr;
    sluh_symb *S = new sluh_symb;
    S->n = n;
    if (maxsup < 1) maxsup = 1;
    const int n1 = n - nschur;   // eliminated columns [0, n1)
    std::vector<int32_t> p((size_t)n);
    if (perm_in) std::copy(perm_in, perm_in + n, p.begin());
    else std::iota(p.begin(), p.end(), 0);

    std::vector<int64_t> cp, rp;
    std::vector<int32_t> ri, ci, parent, invpost;
    build_lower(n, rowptr, colind, p.data(), cp, ri);
    transpose_lower(n, cp, ri, rp, ci);
    etree(n, rp, ci, parent);
    if (nschur == 0) {
        postorder(n, parent, invpost);
    } else {
        std::vector<int32_t> par1(parent.begin(), parent.begin() + n1);
        for (int j = 0; j < n1; ++j)
            if (par1[j] >= n1) par1[j] = -1;
        postorder(n1, par1, invpost);
        invpost.resize(n);
        for (int j = n1; j < n; ++j) invpost[j] = j;
    }
    bool ident = true;
    for (int i = 0; i < n && ident; ++i) ident = invpost[i] == i;
    if (!ident) {
        for (int i = 0; i < n; ++i) p[i] = invpost[p[i]];
        build_lower(n, rowptr, colind, p.data(), cp, ri);
        transpose_lower(n, cp, ri, rp, ci);
        etree(n, rp, ci, parent);
    }
    { std::vector<int32_t>().swap(ci); std::vector<int64_t>().swap(rp); }
    S->perm = p;

    // subtree sizes / first descendants (labels [0, n1) are a postorder of their forest: parent[j] > j); the Schur
    // columns' values are not used
    std::vector<int32_t> size(n, 1), first(n);
    for (int j = 0; j < n; ++j)
        if (parent[j] != -1) size[parent[j]] += size[j];
    for (int j = 0; j < n; ++j) first[j] = j - size[j] + 1;

    // column counts of L (Gilbert, Ng & Peyton skeleton algorithm; post = identity) of the columns [0, n1): their subtrees
    // lie in [0, n1), and every count or least common ancestor the walk puts on a Schur column stays outside them
    std::vector<int32_t> cc(n), maxfirst(n, -1), prevleaf(n, -1), anc(n);
    for (int j = 0; j < n; ++j) { cc[j] = size[j] == 1 ? 1 : 0; anc[j] = j; }
    for (int j = 0; j < n1; ++j) {
        if (parent[j] != -1) --cc[parent[j]];
        for (int64_t q = cp[j]; q < cp[j + 1]; ++q) {
            int i = ri[q];  // i > j
            if (first[j] <= maxfirst[i]) continue;
            maxfirst[i] = first[j];
            int jprev = prevleaf[i];
            prevleaf[i] = j;
            ++cc[j];
            if (jprev != -1) {
                int qq = jprev;
                while (qq != anc[qq]) qq = anc[qq];
                for (int s = jprev; s != qq;) { int sp = anc[s]; anc[s] = qq; s = sp; }
                --cc[qq];
            }
        }
        if (parent[j] != -1) anc[j] = parent[j];
    }
    for (int j = 0; j < n1; ++j)
        if (parent[j] != -1) cc[parent[j]] += cc[j];

    // supernode partition: relaxed leaf subtrees + fundamental chains, capped at maxsup
    std::vector<int32_t> &xsup = S->xsup;
    xsup.clear();
    {
        int j = 0;
        while (j < n1) {
            // is j the first column of a maximal subtree with <= relax columns ?
            int root = -1;
            if (relax > 1) {
                // climb from j while the subtree still starts at j and stays small
                int r = j;
                if (first[r] == j) {
                    while (parent[r] != -1 && parent[r] < n1 && first[parent[r]] == j && size[parent[r]] <= relax) r = parent[r];
                    // need the maximal small subtree that STARTS at j: r's subtree is [j, r]
                    if (size[r] <= relax && size[r] > 1) root = r;
                }
            }
            if (root >= 0) {
                // the subtree [j, root] becomes supernode(s) of width <= maxsup
                int f = j, l = root;
                while (f <= l) { xsup.push_back(f); f += std::min(maxsup, l - f + 1); }
                j = root + 1;
                continue;
            }
            int f = j;
            xsup.push_back(f);
            ++j;
            // chain amalgamation: column j joins [f, j) when it is the parent of j-1 and the explicit
            // zeros this adds (every earlier column is padded to the structure of column j) stay below
            // the fraction `amalg` of the merged block; amalg = 0 gives exact fundamental supernodes.
            double ent = cc[f];
            while (j < n1 && j - f < maxsup && parent[j - 1] == j) {
                double w = j - f + 1;
                double merged = w * cc[j] + w * (w - 1) / 2, tru = ent + cc[j];
                if (merged - tru > amalg * merged + 1e-9) break;
                ent = tru;
                ++j;
            }
        }
        for (int f = n1; f < n; f += maxsup) xsup.push_back(f);
        xsup.push_back(n);
    }
    int nsupers = (int)xsup.size() - 1;
    S->nsupers = nsupers;
    S->supno.resize(n);
    for (int s = 0; s < nsupers; ++s)
        for (int c = xsup[s]; c < xsup[s + 1]; ++c) S->supno[c] = s;
    const std::vector<int32_t> &supno = S->supno;

    // supernodal symbolic: struct(s) = own cols + A-pattern + children's structs below s
    S->sptr.assign((size_t)nsupers + 1, 0);
    S->setree.assign(nsupers, nsupers);
    std::vector<int32_t> mark(n, -1), chead(nsupers, -1), cnext(nsupers, -1), others;
    double est = 0;
    for (int s = 0; s < nsupers; ++s) est += cc[xsup[s]];
    S->srow.reserve((size_t)(est * 1.05) + 1024);
    for (int s = 0; s < nsupers; ++s) {
        int f = xsup[s], l = xsup[s + 1] - 1;
        others.clear();
        for (int c = f; c <= l; ++c)
            for (int64_t q = cp[c]; q < cp[c + 1]; ++q) {
                int r = ri[q];
                if (r > l && mark[r] != s) { mark[r] = s; others.push_back(r); }
            }
        for (int ch = chead[s]; ch != -1; ch = cnext[ch]) {
            int64_t b = S->sptr[ch] + (xsup[ch + 1] - xsup[ch]), e = S->sptr[ch + 1];
            for (int64_t q = b; q < e; ++q) {
                int r = S->srow[(size_t)q];
                if (r > l && mark[r] != s) { mark[r] = s; others.push_back(r); }
            }
        }
        std::sort(others.begin(), others.end());
        for (int c = f; c <= l; ++c) S->srow.push_back(c);
        S->srow.insert(S->srow.end(), others.begin(), others.end());
        S->sptr[s + 1] = (int64_t)S->srow.size();
        if (!others.empty()) {
            int ps = supno[others[0]];
            S->setree[s] = ps;
            cnext[s] = chead[ps];
            chead[ps] = s;
        }
    }

    // arena sizes and the reference's flop accounting
    for (int s = 0; s < nsupers; ++s) {
        double ns = xsup[s + 1] - xsup[s];
        int64_t b = S->sptr[s], e = S->sptr[s + 1];
        double nsupr = (double)(e - b), m = nsupr - ns;
        int nblk = 0, last = -1, ufst = 0;
        for (int64_t q = b; q < e; ++q) {
            int ib = supno[S->srow[(size_t)q]];
            if (ib != last) { ++nblk; last = ib; if (ib != s) ufst += xsup[ib + 1] - xsup[ib]; }
        }
        S->lidx_len += BC_HEADER + nblk * LB_DESCRIPTOR + nsupr;
        S->lval_len += nsupr * ns;
        if (m > 0) {
            S->uidx_len += BR_HEADER + (nblk - 1) * UB_DESCRIPTOR + ufst;
            S->uval_len += m * ns;
        }
        double diag = 0;
        for (int j = 0; j < (int)ns; ++j) { double r = ns - j - 1; diag += r + 2 * r * r; }
        double schur = 2.0 * m * m * ns;
        S->ops_fact += diag + m * ns * (ns + 1) + schur;
        S->ops_schur += schur;
    }
    return S;
}

extern "C" void sluh_symb_free(sluh_symb *s) { delete s; }
extern "C" int32_t sluh_symb_nsupers(const sluh_symb *s) { return s->nsupers; }
extern "C" void sluh_symb_sizes(const sluh_symb *s, double *sizes)
{
    sizes[0] = s->lidx_len; sizes[1] = s->lval_len; sizes[2] = s->uidx_len; sizes[3] = s->uval_len;
    sizes[4] = s->ops_fact; sizes[5] = s->ops_schur;
}

extern "C" void sluh_symb_export(const sluh_symb *S, int32_t *perm, int32_t *xsup, int32_t *setree,
                                 int64_t *lidx_off, int32_t *lidx, int64_t *lval_off,
                                 int64_t *uidx_off, int32_t *uidx, int64_t *uval_off)
{
    int n = S->n, nsupers = S->nsupers;
    std::copy(S->perm.begin(), S->perm.end(), perm);
    std::copy(S->xsup.begin(), S->xsup.end(), xsup);
    std::copy(S->setree.begin(), S->setree.end(), setree);
    (void)n;
    const std::vector<int32_t> &supno = S->supno;
    lidx_off[0] = lval_off[0] = uidx_off[0] = uval_off[0] = 0;
    // pass 1: offsets
    for (int s = 0; s < nsupers; ++s) {
        int ns = S->xsup[s + 1] - S->xsup[s];
        int64_t b = S->sptr[s], e = S->sptr[s + 1], nsupr = e - b, m = nsupr - ns;
        int nblk = 0, last = -1;
        int64_t ufst = 0;
        for (int64_t q = b; q < e; ++q) {
            int ib = supno[S->srow[(size_t)q]];
            if (ib != last) { ++nblk; last = ib; if (ib != s) ufst += S->xsup[ib + 1] - S->xsup[ib]; }
        }
        lidx_off[s + 1] = lidx_off[s] + BC_HEADER + nblk * LB_DESCRIPTOR + nsupr;
        lval_off[s + 1] = lval_off[s] + nsupr * ns;
        uidx_off[s + 1] = uidx_off[s] + (m > 0 ? BR_HEADER + (nblk - 1) * UB_DESCRIPTOR + ufst : 0);
        uval_off[s + 1] = uval_off[s] + m * ns;
    }
    // pass 2: index arrays
#pragma omp parallel for schedule(dynamic, 64)
    for (int s = 0; s < nsupers; ++s) {
        int f = S->xsup[s], ns = S->xsup[s + 1] - f, klst = f + ns;
        int64_t b = S->sptr[s], e = S->sptr[s + 1], nsupr = e - b, m = nsupr - ns;
        int32_t *li = lidx + lidx_off[s];
        int nblk = 0;
        int64_t w = BC_HEADER;
        for (int64_t q = b; q < e;) {
            int ib = supno[S->srow[(size_t)q]];
            int64_t q2 = q;
            while (q2 < e && supno[S->srow[(size_t)q2]] == ib) ++q2;
            li[w++] = ib;
            li[w++] = (int32_t)(q2 - q);
            for (int64_t t = q; t < q2; ++t) li[w++] = S->srow[(size_t)t];
            ++nblk;
            q = q2;
        }
        li[0] = nblk;
        li[1] = (int32_t)nsupr;
        if (m <= 0) continue;
        int32_t *ui = uidx + uidx_off[s];
        int64_t u = BR_HEADER;
        int nub = 0;
        for (int64_t q = b + ns; q < e;) {
            int jb = supno[S->srow[(size_t)q]];
            int64_t q2 = q;
            while (q2 < e && supno[S->srow[(size_t)q2]] == jb) ++q2;
            int jf = S->xsup[jb], jns = S->xsup[jb + 1] - jf;
            ui[u++] = jb;
            ui[u++] = (int32_t)((q2 - q) * ns);
            for (int c = 0; c < jns; ++c) ui[u + c] = klst;       // empty segment
            for (int64_t t = q; t < q2; ++t) ui[u + (S->srow[(size_t)t] - jf)] = f;  // full segment
            u += jns;
            ++nub;
            q = q2;
        }
        ui[0] = nub;
        ui[1] = (int32_t)(m * ns);
        ui[2] = (int32_t)u;
    }
}

extern "C" void sluh_fill_values(int n, const int32_t *rowptr, const int32_t *colind,
                                 const double *val, const int32_t *perm, int nsupers,
                                 const int32_t *xsup, const int64_t *lidx_off, const int32_t *lidx,
                                 const int64_t *lval_off, double *lval, const int64_t *uidx_off,
                                 const int32_t *uidx, const int64_t *uval_off, double *uval,
                                 const int8_t *active)
{
    std::vector<int32_t> supno((size_t)n);
#pragma omp parallel for schedule(dynamic, 256)
    for (int s = 0; s < nsupers; ++s)
        for (int c = xsup[s]; c < xsup[s + 1]; ++c) supno[c] = s;
    // flat row lists of L panels, flat (column, first row, segment offset) lists of U panels; a U panel lists only the
    // columns with a non-empty skyline segment (fstnz < klst), as the device analysis does
    std::vector<int64_t> lro((size_t)nsupers + 1, 0), uco((size_t)nsupers + 1, 0);
    for (int s = 0; s < nsupers; ++s) {
        lro[s + 1] = lro[s] + lidx[lidx_off[s] + 1];
        int64_t nc = 0;
        if (uidx_off[s + 1] > uidx_off[s]) {
            const int32_t *ui = uidx + uidx_off[s];
            int klst = xsup[s + 1];
            int64_t u = BR_HEADER;
            for (int b = 0; b < ui[0]; ++b) {
                int jb = ui[u], jns = xsup[jb + 1] - xsup[jb];
                for (int c = 0; c < jns; ++c) nc += ui[u + UB_DESCRIPTOR + c] < klst;
                u += UB_DESCRIPTOR + jns;
            }
        }
        uco[s + 1] = uco[s] + nc;
    }
    std::vector<int32_t> lrows((size_t)lro[nsupers]), ucols((size_t)uco[nsupers]), ufst((size_t)uco[nsupers]),
        useg((size_t)uco[nsupers]);
#pragma omp parallel for schedule(dynamic, 64)
    for (int s = 0; s < nsupers; ++s) {
        const int32_t *li = lidx + lidx_off[s];
        int64_t w = BC_HEADER, o = lro[s];
        for (int b = 0; b < li[0]; ++b) {
            int nb = li[w + 1];
            for (int t = 0; t < nb; ++t) lrows[(size_t)o++] = li[w + 2 + t];
            w += LB_DESCRIPTOR + nb;
        }
        if (uidx_off[s + 1] == uidx_off[s]) continue;
        const int32_t *ui = uidx + uidx_off[s];
        int klst = xsup[s + 1];
        int64_t u = BR_HEADER, oc = uco[s];
        int32_t seg = 0;
        for (int b = 0; b < ui[0]; ++b) {
            int jb = ui[u], jf = xsup[jb], jns = xsup[jb + 1] - jf;
            for (int c = 0; c < jns; ++c) {
                int fst = ui[u + UB_DESCRIPTOR + c];
                if (fst < klst) { ucols[(size_t)oc] = jf + c; ufst[(size_t)oc] = fst; useg[(size_t)oc] = seg - (fst - xsup[s]); ++oc; seg += klst - fst; }
            }
            u += UB_DESCRIPTOR + jns;
        }
    }
    int64_t ltot = lval_off[nsupers], utot = uval_off[nsupers];
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < ltot; ++i) lval[i] = 0.0;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < utot; ++i) uval[i] = 0.0;
#pragma omp parallel for schedule(dynamic, 1024)
    for (int i = 0; i < n; ++i) {
        int r = perm[i], ib = supno[r];
        for (int64_t q = rowptr[i]; q < rowptr[i + 1]; ++q) {
            int c = perm[colind[q]], jb = supno[c];
            if (active && !active[ib >= jb ? jb : ib]) continue;
            if (ib >= jb) {
                const int32_t *b = lrows.data() + lro[jb], *e = lrows.data() + lro[jb + 1];
                const int32_t *it = std::lower_bound(b, e, r);
                if (it == e || *it != r) { fprintf(stderr, "sluh_fill_values: (%d,%d) not in L structure\n", r, c); abort(); }
                int64_t nsupr = e - b;
                lval[lval_off[jb] + (it - b) + (int64_t)(c - xsup[jb]) * nsupr] = val[q];
            } else {
                const int32_t *b = ucols.data() + uco[ib], *e = ucols.data() + uco[ib + 1];
                const int32_t *it = std::lower_bound(b, e, c);
                // an entry above its column's skyline start has no slot either
                if (it == e || *it != c || r < ufst[(size_t)(uco[ib] + (it - b))]) {
                    fprintf(stderr, "sluh_fill_values: (%d,%d) not in U structure\n", r, c);
                    abort();
                }
                uval[uval_off[ib] + useg[(size_t)(uco[ib] + (it - b))] + (r - xsup[ib])] = val[q];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Z-forest partition
// ------------------------------------------------------------------------------------------------
namespace {
struct ForestCtx {
    int nsupers;
    const int32_t *setree;
    std::vector<double> wsub;
    std::vector<int32_t> chead, cnext;
    int32_t *forest_of;
};
void assign_subtree(ForestCtx &c, int root, int f)
{
    std::vector<int32_t> st{root};
    while (!st.empty()) {
        int v = st.back();
        st.pop_back();
        c.forest_of[v] = f;
        for (int ch = c.chead[v]; ch != -1; ch = c.cnext[ch]) st.push_back(ch);
    }
}
void split_forest(ForestCtx &c, std::vector<int32_t> roots, int f, int levels_left)
{
    if (levels_left <= 1) {
        for (int r : roots) assign_subtree(c, r, f);
        return;
    }
    std::vector<int32_t> bin[2];
    double total0 = 0;
    for (int r : roots) total0 += c.wsub[r];
    for (int iter = 0;; ++iter) {
        std::sort(roots.begin(), roots.end(), [&](int a, int b) { return c.wsub[a] > c.wsub[b]; });
        double w[2] = {0, 0};
        bin[0].clear(); bin[1].clear();
        for (int r : roots) { int t = w[0] <= w[1] ? 0 : 1; bin[t].push_back(r); w[t] += c.wsub[r]; }
        double tot = w[0] + w[1];
        if (roots.empty()) break;
        bool balanced = roots.size() >= 2 && std::max(w[0], w[1]) <= 0.55 * tot;
        int heavy = roots[0];
        bool can_peel = c.chead[heavy] != -1 && c.wsub[heavy] > 0.02 * total0;
        if (balanced || !can_peel) break;
        c.forest_of[heavy] = f;  // becomes an ancestor shared by both halves
        roots.erase(roots.begin());
        for (int ch = c.chead[heavy]; ch != -1; ch = c.cnext[ch]) roots.push_back(ch);
    }
    split_forest(c, bin[0], 2 * f + 1, levels_left - 1);
    split_forest(c, bin[1], 2 * f + 2, levels_left - 1);
}
}  // namespace

extern "C" void sluh_forests(int nsupers, const int32_t *setree, const double *weight, int maxLvl,
                             int32_t *forest_of)
{
    ForestCtx c;
    c.nsupers = nsupers; c.setree = setree; c.forest_of = forest_of;
    c.wsub.assign(weight, weight + nsupers);
    c.chead.assign(nsupers, -1); c.cnext.assign(nsupers, -1);
    std::vector<int32_t> roots;
    for (int s = 0; s < nsupers; ++s) {  // parent > child, so one ascending sweep accumulates
        int p = setree[s];
        if (p >= 0 && p < nsupers) { c.wsub[p] += c.wsub[s]; }
    }
    for (int s = nsupers - 1; s >= 0; --s) {
        int p = setree[s];
        if (p >= 0 && p < nsupers) { c.cnext[s] = c.chead[p]; c.chead[p] = s; }
        else roots.push_back(s);
    }
    for (int s = 0; s < nsupers; ++s) forest_of[s] = -1;
    split_forest(c, roots, 0, maxLvl);
}

// ------------------------------------------------------------------------------------------------
// checker: y = M x with M in the reference block layout
// ------------------------------------------------------------------------------------------------
extern "C" void sluh_panel_matvec(int mode, int n, int nsupers, const int32_t *xsup,
                                  const int32_t *const *lidx, const double *const *lval,
                                  const int32_t *const *uidx, const double *const *uval, int nvec,
                                  const double *x, double *y)
{
    // mode 0: y = A x (panels hold A);  mode 1: y = L (U x) (panels hold the factors);
    // mode 2: y = U x only;  mode 3: y = L x only (unit lower) -- the two halves of mode 1, so that ranks holding
    // disjoint sets of factored supernodes can all-reduce the intermediate vector (bench.py, N > 1)
    std::vector<double> tbuf;
    const double *t = x;
    if (mode == 1 || mode == 2) {
        // t = U x : rows of supernode k are produced only by panel k -> no write conflicts
        tbuf.assign((size_t)n * nvec, 0.0);
#pragma omp parallel
        {
            std::vector<int32_t> pos;
#pragma omp for schedule(dynamic, 16)
            for (int k = 0; k < nsupers; ++k) {
                int f = xsup[k], ns = xsup[k + 1] - f, klst = f + ns;
                const int32_t *li = lidx[k];
                if (li) {
                    int nsupr = li[1];
                    if (li[BC_HEADER] != k || li[BC_HEADER + 1] != ns) { fprintf(stderr, "panel_matvec: diagonal block of %d missing\n", k); abort(); }
                    pos.assign(ns, 0);
                    for (int i = 0; i < ns; ++i) pos[li[BC_HEADER + LB_DESCRIPTOR + i] - f] = i;
                    const double *lv = lval[k];
                    for (int v = 0; v < nvec; ++v)
                        for (int c = 0; c < ns; ++c) {
                            double xc = x[(size_t)v * n + f + c];
                            const double *col = lv + (size_t)c * nsupr;
                            for (int r = 0; r <= c; ++r) tbuf[(size_t)v * n + f + r] += col[pos[r]] * xc;
                        }
                }
                const int32_t *ui = uidx[k];
                if (!ui) continue;
                const double *uv = uval[k];
                int64_t u = BR_HEADER, seg = 0;
                for (int b = 0; b < ui[0]; ++b) {
                    int jb = ui[u], jf = xsup[jb], jns = xsup[jb + 1] - jf;
                    for (int c = 0; c < jns; ++c) {
                        int fst = ui[u + UB_DESCRIPTOR + c];
                        if (fst >= klst) continue;
                        for (int v = 0; v < nvec; ++v) {
                            double xc = x[(size_t)v * n + jf + c];
                            for (int r = fst; r < klst; ++r) tbuf[(size_t)v * n + r] += uv[seg + (r - fst)] * xc;
                        }
                        seg += klst - fst;
                    }
                    u += UB_DESCRIPTOR + jns;
                }
            }
        }
        t = tbuf.data();
        if (mode == 2) {
            for (size_t i = 0; i < (size_t)n * nvec; ++i) y[i] = tbuf[i];
            return;
        }
    }
    if (mode == 3) mode = 1;
    for (size_t i = 0; i < (size_t)n * nvec; ++i) y[i] = 0.0;
#pragma omp parallel
    {
        std::vector<int32_t> rows;
        std::vector<double> acc;
#pragma omp for schedule(dynamic, 16)
        for (int k = 0; k < nsupers; ++k) {
            int f = xsup[k], ns = xsup[k + 1] - f, klst = f + ns;
            const int32_t *li = lidx[k];
            if (li) {
                int nsupr = li[1];
                rows.resize(nsupr);
                int64_t w = BC_HEADER, o = 0;
                for (int b = 0; b < li[0]; ++b) {
                    int nb = li[w + 1];
                    for (int q = 0; q < nb; ++q) rows[o++] = li[w + 2 + q];
                    w += LB_DESCRIPTOR + nb;
                }
                const double *lv = lval[k];
                acc.assign((size_t)nsupr, 0.0);
                for (int v = 0; v < nvec; ++v) {
                    std::fill(acc.begin(), acc.end(), 0.0);
                    for (int c = 0; c < ns; ++c) {
                        double tc = t[(size_t)v * n + f + c];
                        const double *col = lv + (size_t)c * nsupr;
                        if (mode == 0) {
                            for (int i = 0; i < nsupr; ++i) acc[i] += col[i] * tc;
                        } else {
                            for (int i = 0; i < nsupr; ++i) {
                                int r = rows[i];
                                if (r >= klst || r > f + c) acc[i] += col[i] * tc;  // strictly below the diagonal
                                else if (r == f + c) acc[i] += tc;                  // unit diagonal
                            }
                        }
                    }
                    for (int i = 0; i < nsupr; ++i) {
#pragma omp atomic
                        y[(size_t)v * n + rows[i]] += acc[i];
                    }
                }
            }
            if (mode == 1) continue;
            const int32_t *ui = uidx[k];
            if (!ui) continue;
            const double *uv = uval[k];
            int64_t u = BR_HEADER, seg = 0;
            for (int b = 0; b < ui[0]; ++b) {
                int jb = ui[u], jf = xsup[jb], jns = xsup[jb + 1] - jf;
                for (int c = 0; c < jns; ++c) {
                    int fst = ui[u + UB_DESCRIPTOR + c];
                    if (fst >= klst) continue;
                    for (int v = 0; v < nvec; ++v) {
                        double xc = x[(size_t)v * n + jf + c];
                        for (int r = fst; r < klst; ++r) {
#pragma omp atomic
                            y[(size_t)v * n + r] += uv[seg + (r - fst)] * xc;
                        }
                    }
                    seg += klst - fst;
                }
                u += UB_DESCRIPTOR + jns;
            }
        }
    }
}
