// slu_match.cpp -- maximum-product bipartite matching with its scalings (sluh_large_diag_perm): the row permutation that
// puts large entries on the diagonal, the role of MC64 job 5 in front of a static-pivoting factorization.
//
// Written from the literature (Duff & Koster, "On algorithms for permuting large entries to the diagonal of a sparse
// matrix", SIAM J. Matrix Anal. Appl. 22(4), 2001; the shortest augmenting path method of Jonker & Volgenant):
//   costs   c_ij = log colmax_j - log |a_ij| >= 0 on the nonzeros (explicit zeros are not edges);
//   start   u_i = min_j c_ij, v_j = min_i (c_ij - u_i), then a greedy matching on the tight edges (c_ij - u_i - v_j = 0);
//   finish  for every unmatched column, Dijkstra on the reduced costs c_ij - u_i - v_j >= 0 (binary heap, lazy deletion)
//           to the nearest free row, dual update, augmentation.
// The duals are optimal for the dual of the assignment problem, so R_i = exp(u_i), C_j = exp(v_j) / colmax_j give
// |R_i a_ij C_j| = exp(u_i + v_j - c_ij) <= 1, with equality on the matching.  Costs and duals are kept in long double
// (64-bit mantissa on x86-64) so that the rounding they accumulate over many augmentations stays far below one double
// ulp of the scaled entries.  Ties go to the smallest row index (heap order (distance, row), rows of a column ascending):
// the result is deterministic.
#include "slu_b200_host.h"

#include <chrono>
#include <cmath>
#include <functional>
#include <limits>
#include <queue>
#include <utility>
#include <vector>

namespace {
typedef long double ld;
}

extern "C" int sluh_large_diag_perm(int n, const int32_t *rowptr, const int32_t *colind, const double *absval, int32_t *perm_r,
                                    double *R, double *C, double out[2])
{
    const auto t0 = std::chrono::steady_clock::now();
    if (n < 0 || !rowptr || (n > 0 && (!colind || !absval || !perm_r || !R || !C))) return -1;
    if (rowptr[0] != 0) return -1;
    for (int i = 0; i < n; ++i)
        if (rowptr[i + 1] < rowptr[i]) return -1;
    const int64_t nnz = rowptr[n];
    // column-major copy of the edges (rows ascending within a column) and the column maxima
    std::vector<double> colmax(n, 0.0);
    std::vector<int64_t> cp(n + 1, 0);
    for (int64_t p = 0; p < nnz; ++p) {
        const int j = colind[p];
        const double a = absval[p];
        if (j < 0 || j >= n || !(a >= 0.0) || !std::isfinite(a)) return -1;
        if (a == 0.0) continue;
        ++cp[j + 1];
        if (a > colmax[j]) colmax[j] = a;
    }
    for (int j = 0; j < n; ++j) cp[j + 1] += cp[j];
    std::vector<int32_t> ri(cp[n]);
    std::vector<ld> cost(cp[n]);
    std::vector<double> aval(cp[n]);
    {
        std::vector<int64_t> pos(cp.begin(), cp.end() - 1);
        for (int i = 0; i < n; ++i)
            for (int64_t p = rowptr[i]; p < rowptr[i + 1]; ++p) {
                const double a = absval[p];
                if (a == 0.0) continue;
                const int j = colind[p];
                const int64_t q = pos[j]++;
                ri[q] = i;
                aval[q] = a;
                cost[q] = logl((ld)colmax[j]) - logl((ld)a);
            }
    }
    const ld INF = std::numeric_limits<ld>::infinity();
    std::vector<ld> u(n, INF), v(n, 0);
    for (int j = 0; j < n; ++j)
        for (int64_t q = cp[j]; q < cp[j + 1]; ++q)
            if (cost[q] < u[ri[q]]) u[ri[q]] = cost[q];
    for (int i = 0; i < n; ++i)
        if (u[i] == INF) u[i] = 0;   // an empty row: no edge constrains it (the matrix is structurally singular)
    for (int j = 0; j < n; ++j) {
        ld m = INF;
        for (int64_t q = cp[j]; q < cp[j + 1]; ++q) m = std::min(m, cost[q] - u[ri[q]]);
        v[j] = m == INF ? 0 : m;
    }
    std::vector<int32_t> row_match(n, -1), col_match(n, -1);
    for (int j = 0; j < n; ++j)   // greedy: the first free row on a tight edge
        for (int64_t q = cp[j]; q < cp[j + 1]; ++q) {
            const int i = ri[q];
            if (row_match[i] < 0 && (cost[q] - u[i]) - v[j] == 0) {
                row_match[i] = j;
                col_match[j] = i;
                break;
            }
        }

    // successive shortest augmenting paths from the unmatched columns
    std::vector<ld> d(n, INF);
    std::vector<int32_t> pred(n, -1);
    std::vector<char> done(n, 0);
    std::vector<int32_t> touched, final_rows;
    typedef std::pair<ld, int32_t> Item;
    std::priority_queue<Item, std::vector<Item>, std::greater<Item>> heap;
    int matched = 0;
    for (int j = 0; j < n; ++j) matched += col_match[j] >= 0;
    for (int j0 = 0; j0 < n; ++j0) {
        if (col_match[j0] >= 0) continue;
        touched.clear();
        final_rows.clear();
        heap = decltype(heap)();
        auto relax = [&](int j, ld dj) {
            for (int64_t q = cp[j]; q < cp[j + 1]; ++q) {
                const int i = ri[q];
                if (done[i]) continue;
                ld r = (cost[q] - u[i]) - v[j];
                if (r < 0) r = 0;   // rounding of a tight edge
                const ld nd = dj + r;
                if (nd < d[i]) {
                    if (d[i] == INF) touched.push_back(i);
                    d[i] = nd;
                    pred[i] = j;
                    heap.push(Item(nd, i));
                }
            }
        };
        relax(j0, 0);
        int iend = -1;
        ld D = 0;
        while (!heap.empty()) {
            const Item it = heap.top();
            heap.pop();
            const int i = it.second;
            if (done[i] || it.first > d[i]) continue;
            done[i] = 1;
            final_rows.push_back(i);
            if (row_match[i] < 0) { iend = i; D = it.first; break; }
            relax(row_match[i], it.first);
        }
        if (iend >= 0) {
            // dual update on the finalized part of the tree, then flip the path
            v[j0] += D;
            for (int i : final_rows) {
                const ld delta = D - d[i];
                if (i == iend || delta == 0) continue;
                u[i] -= delta;
                v[row_match[i]] += delta;
            }
            for (int i = iend;;) {
                const int j = pred[i], prev = col_match[j];
                col_match[j] = i;
                row_match[i] = j;
                if (j == j0) break;
                i = prev;
            }
            ++matched;
        }
        for (int i : touched) { d[i] = INF; done[i] = 0; pred[i] = -1; }
    }
    if (matched < n) {   // the largest product over perfect matchings is 0
        if (out) {
            out[0] = -INFINITY;
            out[1] = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        }
        return matched;
    }

    ld logprod = 0;
    for (int j = 0; j < n; ++j)
        for (int64_t q = cp[j]; q < cp[j + 1]; ++q)
            if (ri[q] == col_match[j]) { logprod += logl((ld)aval[q]); break; }
    for (int i = 0; i < n; ++i) {
        perm_r[i] = row_match[i];
        R[i] = (double)expl(u[i]);
    }
    for (int j = 0; j < n; ++j) C[j] = (double)(expl(v[j]) / (ld)colmax[j]);
    if (out) {
        out[0] = (double)logprod;
        out[1] = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    }
    return 0;
}
