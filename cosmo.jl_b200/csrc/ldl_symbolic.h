// ldl_symbolic.h -- host symbolic analysis of the quasi-definite KKT matrix K = [P + sigma I, A'; A, -diag(1/rho)] for
// the device LDL' plugin (ldl.cuh): fill-reducing ordering, elimination tree, the pattern of L in CSC and CSR form and
// the level schedules of the factorisation and of the two triangular solves.  Plain C++, no CUDA: it also backs
// cosmo_b200_ldl_symbolic, which runs without a GPU.
//
// Conventions: indices are in the permuted order unless named otherwise; L is unit lower triangular and stored
// without its diagonal; perm[k] is the original index (x: 0..n-1, y: n..n+m-1) of the k-th pivot.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <functional>
#include <queue>
#include <utility>
#include <vector>

namespace cosmo {
namespace ldl {

// K entry sources, summed in order by the device assembly: value of P_ (CSR index), value of At_ (CSR index),
// -1/rho_i, sigma
enum { SRC_P = 0, SRC_AT = 1, SRC_RHO = 2, SRC_SIGMA = 3 };
inline int64_t src_code(int64_t idx, int kind) { return (idx << 2) | kind; }

// a level (or a run of consecutive levels, each at most kRunWidth wide) that runs as one kernel launch; runs take one
// CTA and separate their levels with __syncthreads()
constexpr int kRunWidth = 8;
struct Segment { int l0, l1; bool run; };

struct Symbolic {
  int n = 0, m = 0, N = 0;
  std::vector<int> perm, iperm, parent, level, depth;
  // strictly lower triangle of the permuted K by columns (diagonal first), with the sources of every entry
  std::vector<int64_t> Kp, Ksp, Ksrc;
  std::vector<int> Ki;
  // L by columns (rows ascending) and by rows (columns ascending); Rmap[r] = CSC position of CSR entry r
  std::vector<int64_t> Lp, Rp, Rmap;
  std::vector<int> Li, Rj;
  // columns sorted by level (factorisation, forward solve) and by depth (backward solve)
  std::vector<int> fcols, fptr, bcols, bptr;
  std::vector<Segment> fseg, bseg;
  int64_t nnz_triu_K() const { return Kp.empty() ? 0 : Kp.back(); }
  int64_t nnz_L() const { return Lp.empty() ? 0 : Lp.back(); }
};

// Minimum degree on the quotient graph (George & Liu; Amestoy, Davis & Duff 1996 for the approximate degree): every
// eliminated pivot becomes an element whose member list replaces the fill clique; elements adjacent to the pivot are
// absorbed into it, and elements that become subsets of the new one are absorbed too.  The degree of a variable i is
// the approximate external degree |A_i| + |L_p \ i| + sum_e |L_e \ L_p|, capped at the number of uneliminated
// variables.  Ties go to the smaller index, so the ordering is deterministic.  No supervariable detection.
inline std::vector<int> min_degree_order(int N, const std::vector<int64_t>& ptr, const std::vector<int>& adj) {
  std::vector<std::vector<int>> A(N), E(N), L(N);
  for (int i = 0; i < N; ++i) A[i].assign(adj.begin() + ptr[i], adj.begin() + ptr[i + 1]);
  std::vector<int> deg(N), state(N, 0);   // 0: variable, 1: live element, 2: absorbed element
  std::vector<int> mark(N, -1), w(N, 0), wmark(N, -1);
  typedef std::pair<int, int> DI;
  std::priority_queue<DI, std::vector<DI>, std::greater<DI>> heap;
  for (int i = 0; i < N; ++i) { deg[i] = (int)A[i].size(); heap.push(DI(deg[i], i)); }
  std::vector<int> order;
  order.reserve(N);
  std::vector<int> Lnew;
  for (int k = 0; k < N; ++k) {
    int p = -1;
    while (!heap.empty()) {
      DI t = heap.top(); heap.pop();
      if (state[t.second] == 0 && deg[t.second] == t.first) { p = t.second; break; }
    }
    if (p < 0) break;   // cannot happen: every variable keeps one live heap entry
    order.push_back(p);
    state[p] = 1;
    // L_p = (A_p u union of the absorbed L_e) \ {p}
    Lnew.clear();
    mark[p] = k;
    for (int v : A[p]) if (state[v] == 0 && mark[v] != k) { mark[v] = k; Lnew.push_back(v); }
    for (int e : E[p]) {
      if (state[e] != 1) continue;
      for (int v : L[e]) if (state[v] == 0 && mark[v] != k) { mark[v] = k; Lnew.push_back(v); }
      state[e] = 2;
      std::vector<int>().swap(L[e]);
    }
    std::vector<int>().swap(A[p]);
    std::vector<int>().swap(E[p]);
    // |L_e \ L_p| for every live element next to L_p
    for (int i : Lnew)
      for (int e : E[i]) {
        if (state[e] != 1) continue;
        if (wmark[e] != k) { wmark[e] = k; w[e] = (int)L[e].size(); }
        w[e] -= 1;
      }
    const int remaining = N - k - 1;
    for (int i : Lnew) {
      long long d = (long long)Lnew.size() - 1;
      size_t o = 0;
      for (int e : E[i]) {
        if (state[e] != 1) continue;
        if (w[e] == 0) { state[e] = 2; std::vector<int>().swap(L[e]); continue; }   // L_e inside L_p: absorbed
        E[i][o++] = e;
        d += w[e];
      }
      E[i].resize(o);
      E[i].push_back(p);
      o = 0;
      for (int v : A[i]) if (state[v] == 0 && mark[v] != k) A[i][o++] = v;   // L_p now covers the pruned neighbours
      A[i].resize(o);
      d += (long long)o;
      deg[i] = (int)std::min<long long>(d, remaining - 1 < 0 ? 0 : remaining - 1);
      heap.push(DI(deg[i], i));
    }
    L[p] = Lnew;
  }
  return order;
}

// Full analysis.  P: CSR of the n x n P (both triangles stored; the upper one is read), At: CSR of A' (n rows, m
// columns).  Column indices are 0-based.
inline void analyze(int n, int m, const std::vector<int>& Prow, const std::vector<int>& Pcol, const std::vector<int>& Atrow,
                    const std::vector<int>& Atcol, Symbolic& S) {
  const int N = n + m;
  S.n = n; S.m = m; S.N = N;
  // upper-triangle entries (r < c) of K in the original order, with their sources; the diagonal comes separately
  struct Ent { int r, c; int64_t src; };
  std::vector<Ent> ent;
  ent.reserve((size_t)Pcol.size() / 2 + Atcol.size() + 1);
  for (int r = 0; r < n; ++r)
    for (int k = Prow[r]; k < Prow[r + 1]; ++k)
      if (Pcol[k] > r) ent.push_back(Ent{r, Pcol[k], src_code(k, SRC_P)});
  for (int c = 0; c < n; ++c)
    for (int k = Atrow[c]; k < Atrow[c + 1]; ++k) ent.push_back(Ent{c, n + Atcol[k], src_code(k, SRC_AT)});
  // symmetric adjacency (duplicates removed) for the ordering and the tree
  std::vector<int64_t> aptr(N + 1, 0);
  for (const Ent& e : ent) { aptr[e.r + 1]++; aptr[e.c + 1]++; }
  for (int i = 0; i < N; ++i) aptr[i + 1] += aptr[i];
  std::vector<int> adj(aptr[N]);
  {
    std::vector<int64_t> nx(aptr.begin(), aptr.end() - 1);
    for (const Ent& e : ent) { adj[nx[e.r]++] = e.c; adj[nx[e.c]++] = e.r; }
    std::vector<int64_t> np(N + 1, 0);
    int64_t o = 0;
    for (int i = 0; i < N; ++i) {
      std::sort(adj.begin() + aptr[i], adj.begin() + aptr[i + 1]);
      const int64_t b = o;
      for (int64_t k = aptr[i]; k < aptr[i + 1]; ++k)
        if (k == aptr[i] || adj[k] != adj[k - 1]) adj[o++] = adj[k];
      np[i] = b;
      np[i + 1] = o;
    }
    adj.resize(o);
    aptr.swap(np);
  }
  S.perm = min_degree_order(N, aptr, adj);
  S.iperm.assign(N, 0);
  for (int k = 0; k < N; ++k) S.iperm[S.perm[k]] = k;
  // lower triangle of the permuted K by columns: (col, row, src), diagonal sources first
  {
    struct T3 { int c, r; int64_t src; };
    std::vector<T3> t;
    t.reserve(ent.size() + N + n);
    for (int i = 0; i < N; ++i) {
      const int pi = S.iperm[i];
      if (i < n) t.push_back(T3{pi, pi, src_code(0, SRC_SIGMA)});
      else t.push_back(T3{pi, pi, src_code(i - n, SRC_RHO)});
    }
    for (int r = 0; r < n; ++r)
      for (int k = Prow[r]; k < Prow[r + 1]; ++k)
        if (Pcol[k] == r) t.push_back(T3{S.iperm[r], S.iperm[r], src_code(k, SRC_P)});
    for (const Ent& e : ent) {
      const int a = S.iperm[e.r], b = S.iperm[e.c];
      t.push_back(T3{std::min(a, b), std::max(a, b), e.src});
    }
    std::stable_sort(t.begin(), t.end(), [](const T3& x, const T3& y) { return x.c != y.c ? x.c < y.c : x.r < y.r; });
    S.Kp.assign(N + 1, 0);
    S.Ki.clear(); S.Ksp.assign(1, 0); S.Ksrc.clear();
    for (size_t k = 0; k < t.size(); ++k) {
      if (k == 0 || t[k].c != t[k - 1].c || t[k].r != t[k - 1].r) {
        if (k) S.Ksp.push_back((int64_t)S.Ksrc.size());
        S.Ki.push_back(t[k].r);
        S.Kp[t[k].c + 1]++;
      }
      S.Ksrc.push_back(t[k].src);
    }
    S.Ksp.push_back((int64_t)S.Ksrc.size());
    for (int j = 0; j < N; ++j) S.Kp[j + 1] += S.Kp[j];
  }
  // elimination tree (Liu's algorithm with path compression) over the upper triangle of the permuted K:
  // column j sees rows i < j, i.e. the entries (j, i) of the lower-triangle CSC of column i
  std::vector<std::vector<int>> upper(N);   // upper[j] = rows i < j with K(i, j) != 0
  for (int i = 0; i < N; ++i)
    for (int64_t k = S.Kp[i] + 1; k < S.Kp[i + 1]; ++k) upper[S.Ki[k]].push_back(i);
  S.parent.assign(N, -1);
  {
    std::vector<int> anc(N, -1);
    for (int j = 0; j < N; ++j)
      for (int i : upper[j]) {
        while (i != -1 && i < j) {
          const int nxt = anc[i];
          anc[i] = j;
          if (nxt == -1) { S.parent[i] = j; break; }
          i = nxt;
        }
      }
  }
  // row structure of L: the row subtree of row i is reached from every k with K(k, i) != 0, k < i
  S.Rp.assign(N + 1, 0);
  S.Rj.clear();
  std::vector<int64_t> cnt(N, 0);
  {
    std::vector<int> flag(N, -1), stack;
    for (int i = 0; i < N; ++i) {
      flag[i] = i;
      const size_t b = S.Rj.size();
      for (int k : upper[i])
        for (int t = k; t != -1 && flag[t] != i; t = S.parent[t]) { flag[t] = i; S.Rj.push_back(t); }
      std::sort(S.Rj.begin() + b, S.Rj.end());
      for (size_t r = b; r < S.Rj.size(); ++r) cnt[S.Rj[r]]++;
      S.Rp[i + 1] = (int64_t)S.Rj.size();
    }
  }
  S.Lp.assign(N + 1, 0);
  for (int j = 0; j < N; ++j) S.Lp[j + 1] = S.Lp[j] + cnt[j];
  S.Li.assign(S.Lp[N], 0);
  S.Rmap.assign(S.Rj.size(), 0);
  {
    std::vector<int64_t> nx(S.Lp.begin(), S.Lp.end() - 1);
    for (int i = 0; i < N; ++i)
      for (int64_t r = S.Rp[i]; r < S.Rp[i + 1]; ++r) {
        const int64_t q = nx[S.Rj[r]]++;
        S.Li[q] = i;
        S.Rmap[r] = q;
      }
  }
  // level = 1 + max level of the children (factorisation, forward solve); depth from the root (backward solve)
  S.level.assign(N, 0);
  S.depth.assign(N, 0);
  for (int j = 0; j < N; ++j)
    if (S.parent[j] >= 0) S.level[S.parent[j]] = std::max(S.level[S.parent[j]], S.level[j] + 1);
  for (int j = N - 1; j >= 0; --j) S.depth[j] = S.parent[j] < 0 ? 0 : S.depth[S.parent[j]] + 1;
  auto schedule = [&](const std::vector<int>& lv, std::vector<int>& cols, std::vector<int>& ptr, std::vector<Segment>& seg) {
    int nl = 0;
    for (int j = 0; j < N; ++j) nl = std::max(nl, lv[j] + 1);
    if (N == 0) nl = 0;
    ptr.assign(nl + 1, 0);
    for (int j = 0; j < N; ++j) ptr[lv[j] + 1]++;
    for (int l = 0; l < nl; ++l) ptr[l + 1] += ptr[l];
    cols.assign(N, 0);
    std::vector<int> nx(ptr.begin(), ptr.end() - 1);
    for (int j = 0; j < N; ++j) cols[nx[lv[j]]++] = j;
    seg.clear();
    for (int l = 0; l < nl;) {
      int e = l;
      while (e < nl && ptr[e + 1] - ptr[e] <= kRunWidth) ++e;
      if (e - l >= 2) { seg.push_back(Segment{l, e, true}); l = e; }
      else { seg.push_back(Segment{l, l + 1, false}); ++l; }
    }
  };
  schedule(S.level, S.fcols, S.fptr, S.fseg);
  schedule(S.depth, S.bcols, S.bptr, S.bseg);
}

}  // namespace ldl
}  // namespace cosmo
