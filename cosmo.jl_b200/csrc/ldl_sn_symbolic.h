// ldl_sn_symbolic.h -- host symbolic analysis of the supernodal LDL' KKT plugin (ldl_sn.cuh).  Plain C++, no CUDA: it
// also backs cosmo_b200_ldl_sn_symbolic, which runs without a GPU.
//
// It starts from the simplicial analysis (ldl::analyze: minimum-degree ordering, elimination tree, column counts, the
// entries of K and their sources) and renumbers the columns by a postorder of the elimination tree, so the factor is
// the simplicial plugin's up to a symmetric permutation.  On top of it:
//
//   supernodes   maximal runs j, j+1, ... with parent(j) = j+1 and |L(:,j)| = |L(:,j+1)| + 1 (fundamental, a column may
//                have other children), then relaxed amalgamation: the next run is merged in while it continues the
//                chain (parent(last) = first of the next run) and the explicit zeros stay under the rule of relax_ok
//   panels       supernode s with columns [c0, c1) (width w) and rows R_s = [c0, c1) u struct(L(:, c1-1)) (h of them)
//                is a dense h x w column-major panel: entry (i, j) at off[s] + i + h*j.  Diagonal D_j at (j, j), L
//                strictly below it; the upper triangle of the diagonal block is unused
//   K map        every entry of the permuted K goes to one panel position (Kpos), its sources as ldl::analyze lists them
//   updates      descendant d updates s when rows of d fall in [c0_s, c1_s); per s, the list (d, p0, p1) in ascending
//                d: rows p0..p1-1 of R_d are the columns of s it touches, rows p0..h_d-1 the rows it updates
//   forward      per row r, the segments (d, i) with R_d[i] = r outside r's own supernode (ascending d): the solved
//                columns row r gathers from
//   schedules    supernodal levels (leaves 0) order the factorisation and the forward solve, depths the backward solve
#pragma once
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "ldl_symbolic.h"

namespace cosmo {
namespace ldl_sn {

// Relaxed amalgamation (Ashcraft & Grimes, "The influence of relaxed supernode partitions on the multifrontal method",
// ACM TOMS 15, 1989), with the thresholds CHOLMOD made common: a merged supernode of width w may carry this share of
// explicit zeros among its stored entries.  No merge makes a supernode wider than kMaxRelaxedWidth; fundamental
// supernodes are never split.
constexpr int kMaxRelaxedWidth = 256;
inline bool relax_ok(int w, int64_t zeros, int64_t stored) {
  if (w > kMaxRelaxedWidth) return false;
  const double z = stored > 0 ? (double)zeros / (double)stored : 0.0;
  return w <= 4 || (w <= 16 && z <= 0.8) || (w <= 48 && z <= 0.1) || z <= 0.05;
}

struct Symbolic {
  int n = 0, m = 0, N = 0, ns = 0;
  std::vector<int> perm, parent;          // postordered pivots: perm[k] = original index, parent in this numbering
  std::vector<int64_t> colcount;          // |L(:, k)| below the diagonal, postordered
  std::vector<int> sptr, snode_of;        // columns of supernode s: [sptr[s], sptr[s+1])
  std::vector<int> sparent, slevel, sdepth;
  std::vector<int64_t> rptr;              // R_s = rows[rptr[s] .. rptr[s+1]), ascending, the w columns first
  std::vector<int> rows;
  std::vector<int64_t> off;               // panel offsets, off[ns] = total panel entries
  std::vector<int64_t> Ksp, Ksrc, Kpos;   // entries of K: sources (as ldl::analyze) and panel position
  std::vector<int64_t> uptr;              // updates of s: [uptr[s], uptr[s+1]) into ud, up0, up1
  std::vector<int> ud, up0, up1;
  std::vector<int64_t> gptr;              // forward gather of row r: segments [gptr[r], gptr[r+1]) into gd, gi
  std::vector<int> gd, gi;
  std::vector<int> lcols, lptr;           // supernodes by level
  std::vector<int> lrows, lrptr;          // their columns by level (the rows the forward gather runs over)
  std::vector<int> bcols, bptr;           // supernodes by depth
  int max_width = 0, levels = 0, simplicial_levels = 0;
  int64_t stored = 0, nnz_L = 0, nnz_K = 0;
  double update_flops = 0.0;              // multiply-adds x 2 of the descendant updates of one factorisation
  int64_t zeros() const { return stored - nnz_L; }
  int width(int s) const { return sptr[s + 1] - sptr[s]; }
  int height(int s) const { return (int)(rptr[s + 1] - rptr[s]); }
};

inline void analyze(int n, int m, const std::vector<int>& Prow, const std::vector<int>& Pcol, const std::vector<int>& Atrow,
                    const std::vector<int>& Atcol, Symbolic& S) {
  ldl::Symbolic B;
  ldl::analyze(n, m, Prow, Pcol, Atrow, Atcol, B);
  const int N = B.N;
  S.n = n; S.m = m; S.N = N;
  S.nnz_L = B.nnz_L();
  S.nnz_K = B.nnz_triu_K();
  S.simplicial_levels = (int)B.fptr.size() - 1;
  if (S.simplicial_levels < 0) S.simplicial_levels = 0;
  // postorder: children in ascending order, roots in ascending order
  std::vector<int> post, ipost(N), head(N, -1), next(N, -1);
  post.reserve(N);
  for (int j = N - 1; j >= 0; --j)
    if (B.parent[j] >= 0) { next[j] = head[B.parent[j]]; head[B.parent[j]] = j; }
  {
    std::vector<int> stack;
    for (int r = 0; r < N; ++r) {
      if (B.parent[r] >= 0) continue;
      stack.push_back(r);
      while (!stack.empty()) {
        const int j = stack.back();
        if (head[j] >= 0) { const int c = head[j]; head[j] = next[c]; stack.push_back(c); }
        else { stack.pop_back(); post.push_back(j); }
      }
    }
  }
  for (int k = 0; k < N; ++k) ipost[post[k]] = k;
  S.perm.resize(N); S.parent.resize(N); S.colcount.resize(N);
  for (int k = 0; k < N; ++k) {
    const int o = post[k];
    S.perm[k] = B.perm[o];
    S.parent[k] = B.parent[o] < 0 ? -1 : ipost[B.parent[o]];
    S.colcount[k] = B.Lp[o + 1] - B.Lp[o];
  }
  const std::vector<int64_t>& cc = S.colcount;
  // fundamental supernodes, then greedy amalgamation along chains
  std::vector<int> fund{0};
  for (int j = 0; j + 1 < N; ++j)
    if (!(S.parent[j] == j + 1 && cc[j] == cc[j + 1] + 1)) fund.push_back(j + 1);
  if (N > 0) fund.push_back(N);
  S.sptr.assign(1, 0);
  if (N > 0) {
    int a = 0, e = fund[1];
    for (size_t f = 1; f + 1 < fund.size(); ++f) {
      const int e2 = fund[f + 1];
      bool merge = S.parent[e - 1] == e;
      if (merge) {
        const int w = e2 - a;
        int64_t zeros = 0;
        for (int c = a; c < e2; ++c) zeros += (e2 - 1 - c) + cc[e2 - 1] - cc[c];
        merge = relax_ok(w, zeros, (int64_t)w * (w - 1) / 2 + (int64_t)w * cc[e2 - 1]);
      }
      if (merge) { e = e2; continue; }
      S.sptr.push_back(e);
      a = e; e = e2;
    }
    S.sptr.push_back(N);
  }
  const int ns = (int)S.sptr.size() - 1;
  S.ns = ns;
  S.snode_of.assign(N, 0);
  for (int s = 0; s < ns; ++s)
    for (int c = S.sptr[s]; c < S.sptr[s + 1]; ++c) S.snode_of[c] = s;
  // row structures, panels, supernodal tree
  S.rptr.assign(ns + 1, 0);
  S.off.assign(ns + 1, 0);
  S.rows.clear();
  S.sparent.assign(ns, -1);
  S.stored = 0; S.max_width = 0;
  for (int s = 0; s < ns; ++s) {
    const int c0 = S.sptr[s], c1 = S.sptr[s + 1], w = c1 - c0, o = post[c1 - 1];
    for (int c = c0; c < c1; ++c) S.rows.push_back(c);
    const size_t b = S.rows.size();
    for (int64_t q = B.Lp[o]; q < B.Lp[o + 1]; ++q) S.rows.push_back(ipost[B.Li[q]]);
    std::sort(S.rows.begin() + b, S.rows.end());
    S.rptr[s + 1] = (int64_t)S.rows.size();
    const int64_t h = S.rptr[s + 1] - S.rptr[s];
    S.off[s + 1] = S.off[s] + h * w;
    S.stored += (int64_t)w * (w - 1) / 2 + (int64_t)w * (h - w);
    S.max_width = std::max(S.max_width, w);
    if (S.parent[c1 - 1] >= 0) S.sparent[s] = S.snode_of[S.parent[c1 - 1]];
  }
  S.slevel.assign(ns, 0);
  S.sdepth.assign(ns, 0);
  for (int s = 0; s < ns; ++s)
    if (S.sparent[s] >= 0) S.slevel[S.sparent[s]] = std::max(S.slevel[S.sparent[s]], S.slevel[s] + 1);
  for (int s = ns - 1; s >= 0; --s) S.sdepth[s] = S.sparent[s] < 0 ? 0 : S.sdepth[S.sparent[s]] + 1;
  auto rel = [&](int s, int r) {   // position of row r in R_s
    return (int64_t)(std::lower_bound(S.rows.begin() + S.rptr[s], S.rows.begin() + S.rptr[s + 1], r) - S.rows.begin() - S.rptr[s]);
  };
  // K entries -> panel positions
  S.Ksp = B.Ksp;
  S.Ksrc = B.Ksrc;
  S.Kpos.assign(B.Ki.size(), 0);
  for (int c = 0; c < N; ++c)
    for (int64_t e = B.Kp[c]; e < B.Kp[c + 1]; ++e) {
      const int a = ipost[c], b = ipost[B.Ki[e]];
      const int lo = std::min(a, b), hi = std::max(a, b);
      const int s = S.snode_of[lo];
      S.Kpos[e] = S.off[s] + rel(s, hi) + (int64_t)S.height(s) * (lo - S.sptr[s]);
    }
  // descendant updates (ascending d per target) and the forward gather segments (ascending d per row)
  std::vector<int64_t> ucnt(ns + 1, 0), gcnt(N + 1, 0);
  struct Upd { int d, s, p0, p1; };
  std::vector<Upd> upd;
  S.update_flops = 0.0;
  for (int d = 0; d < ns; ++d) {
    const int w = S.width(d), h = S.height(d);
    const int* R = S.rows.data() + S.rptr[d];
    for (int i = w; i < h;) {
      const int s = S.snode_of[R[i]];
      int i1 = i;
      while (i1 < h && R[i1] < S.sptr[s + 1]) ++i1;
      upd.push_back(Upd{d, s, i, i1});
      ucnt[s + 1]++;
      const double nj = i1 - i, ni = h - i;
      S.update_flops += 2.0 * w * (nj * ni - nj * (nj - 1) / 2);
      i = i1;
    }
    for (int i = w; i < h; ++i) gcnt[R[i] + 1]++;
  }
  for (int s = 0; s < ns; ++s) ucnt[s + 1] += ucnt[s];
  S.uptr = ucnt;
  S.ud.resize(upd.size()); S.up0.resize(upd.size()); S.up1.resize(upd.size());
  {
    std::vector<int64_t> nx(ucnt.begin(), ucnt.end() - 1);
    for (const Upd& u : upd) {
      const int64_t k = nx[u.s]++;
      S.ud[k] = u.d; S.up0[k] = u.p0; S.up1[k] = u.p1;
    }
  }
  for (int r = 0; r < N; ++r) gcnt[r + 1] += gcnt[r];
  S.gptr = gcnt;
  S.gd.resize(gcnt[N]); S.gi.resize(gcnt[N]);
  {
    std::vector<int64_t> nx(gcnt.begin(), gcnt.end() - 1);
    for (int d = 0; d < ns; ++d) {
      const int* R = S.rows.data() + S.rptr[d];
      for (int i = S.width(d); i < S.height(d); ++i) {
        const int64_t k = nx[R[i]]++;
        S.gd[k] = d; S.gi[k] = i;
      }
    }
  }
  // schedules
  auto schedule = [&](const std::vector<int>& lv, std::vector<int>& cols, std::vector<int>& ptr) {
    int nl = 0;
    for (int s = 0; s < ns; ++s) nl = std::max(nl, lv[s] + 1);
    ptr.assign(nl + 1, 0);
    for (int s = 0; s < ns; ++s) ptr[lv[s] + 1]++;
    for (int l = 0; l < nl; ++l) ptr[l + 1] += ptr[l];
    cols.assign(ns, 0);
    std::vector<int> nx(ptr.begin(), ptr.end() - 1);
    for (int s = 0; s < ns; ++s) cols[nx[lv[s]]++] = s;
    return nl;
  };
  S.levels = schedule(S.slevel, S.lcols, S.lptr);
  schedule(S.sdepth, S.bcols, S.bptr);
  S.lrptr.assign(S.levels + 1, 0);
  S.lrows.clear();
  for (int l = 0; l < S.levels; ++l) {
    for (int k = S.lptr[l]; k < S.lptr[l + 1]; ++k)
      for (int c = S.sptr[S.lcols[k]]; c < S.sptr[S.lcols[k] + 1]; ++c) S.lrows.push_back(c);
    S.lrptr[l + 1] = (int)S.lrows.size();
  }
}

}  // namespace ldl_sn
}  // namespace cosmo
