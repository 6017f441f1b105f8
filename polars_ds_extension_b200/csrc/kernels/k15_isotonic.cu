// K15 — isotonic_regression: the least-squares monotone fit of pl_isotonic_regression by pool-adjacent-violators over
// partitions, with the partition solutions joined up a binary tree of merges.
//
// The reference (src/num_ext/isotonic_regression.rs, scipy's PAVA) runs one sequential loop.  The L2 isotonic solution
// does not depend on the order in which adjacent violators are pooled, so:
//   * leaf pass (one thread per partition of R = 32 rows): PAVA on the partition.  Its block stack goes to scratch as
//     per-block end row, leaf-local inclusive prefix sums of w and w y, and the block mean; each row's leaf-local fit
//     goes to the output;
//   * merge levels (one thread per node, one launch per level): node i of level l joins its children A (left) and B.
//     Both solutions are non-decreasing, so the joined solution keeps a prefix of A's blocks and a suffix of B's blocks
//     and pools the rest into one bridge [p, q) around the junction j.  The bridge is the common tangent of the two
//     convex chains of the cumulative-sum diagram: a tangent from B's end to A (a galloping binary search over A's rows)
//     and a tangent from A's end to B, alternated until neither moves.  A node stores its bridge (p, q, mean) and its
//     totals (sum w, sum w y);
//   * final pass (one warp per partition, one lane per row): a row covered by a bridge takes the mean of the highest
//     such bridge on its path to the root; every other row keeps its leaf-local value.
// A row's block in the solution of any node is found by walking down from that node (highest covering bridge, else the
// leaf block); the sum of rows [v, u) around a junction is a leaf-local prefix difference plus the totals of the
// sibling nodes below the junction, added bottom up.  So no value is formed from global prefix sums, every sum has a
// fixed order, no atomics touch data and a repeated call is bit-identical.  increasing = 0 fits -y and negates.
//
// Groups (pdsb_dev_grouped_isotonic_f64): every group is cut into partitions from its own first row and has its own
// tree over its own partitions, laid out exactly as a call on the group's rows alone lays out its tree, so every sum is
// formed in the same order and a group's output is bit for bit that call's.  Merges never join two groups.  The single
// column is the one-group case (ONE: the group terms are constants and no table is read).
// DESIGN.md "K15 in detail" has the byte count, the work bound and the choices.
//
// ptxas (-Xptxas -v, sm_90a, CUDA 12.9): see DESIGN.md "K15 in detail"; no stack frame and no spill in any kernel.
#include "../common.h"
#include "../host/host.h"
#include "kernels.h"
#include "segment_groups.h"
#include <cmath>
#include <cub/cub.cuh>
#include <vector>

namespace pdsb {
namespace {

constexpr int R = 32;          // rows per partition (= lanes of the final pass's warp)
constexpr int NT = 64;         // partitions per CTA in the leaf pass
constexpr int RP = R + 1;      // shared-memory row pitch (conflict-free column access)
constexpr int MAXL = 40;       // tree levels: up to 2^39 partitions in a group

// The leaf stacks are indexed by each partition's first row (a partition holds at most as many blocks as rows).  The
// nodes of each group's tree are stored group after group, level by level within a group: W / S hold every node, p / q
// / m the nodes of levels >= 1 only.
struct Tree {
  const double* pw;            // [n] leaf-local inclusive prefix of w over the blocks (slot: first row + b)
  const double* ps;            // [n] the same of w y
  const double* mean;          // [n] block mean
  const uint8_t* end;          // [n] block end row, local to the partition (exclusive)
  const int* nb;               // [P] blocks per partition
  const double* W;             // [nodes] node totals of w and w y (level 0 = the partitions)
  const double* S;
  const int64_t* p;            // [internal nodes] bridge [p, q) (p = q = -1: none) and its mean
  const int64_t* q;
  const double* m;
  // ONE only, tables in the parameters: W index and p index of each level's first node, and each level's p / q / m.
  // The final pass walks every level for every row and takes the level's own pointers: two instructions fewer per
  // level than base + index, which measured 0.3 ms of the final pass at 1e8 rows on the no-pooling shape
  int64_t lw[MAXL], li[MAXL];
  const int64_t* pl[MAXL];
  const int64_t* ql[MAXL];
  const double* ml[MAXL];
};

// The group a lookup stays in.  With x = partitions - 1, level l of the group has (x >> l) + 1 nodes and starts
// l + 2x - popc(x) - 2 (x >> l) + popc(x >> l) nodes into the group's tree, so node i of level l is W[wb + lv(l) + i]
// and (l >= 1) p[ib + lv(l) + i]: one base per group instead of a table of offsets per level.  A walk over the levels
// takes the closed form once and then steps by the level sizes.
struct Grp {
  int64_t r0, r1;              // rows [r0, r1)
  int64_t k0;                  // first partition
  int64_t x;                   // partitions - 1
  int64_t wb, ib;
  int64_t w0;                  // W index of the group's first node (= wb + lv(0))
};

__device__ __forceinline__ Grp make_grp(int64_t r0, int64_t r1, int64_t k0, int64_t i0, int64_t P) {
  const int64_t x = P - 1, c = 2 * x - __popcll(x);
  return {r0, r1, k0, x, k0 + i0 + c, i0 + c - P, k0 + i0};
}
__device__ __forceinline__ int64_t lv(const Grp& G, int l) {
  const int64_t y = G.x >> l;
  return l - 2 * y + __popcll(y);
}

// The call's groups.  ONE: one group of rows [0, n) and P partitions, and no table is read.
struct Groups {
  const int64_t* off;          // [G + 1] first row of each group
  const int64_t* pbase;        // [G + 1] first partition
  const int64_t* ibase;        // [G + 1] first internal node
  const int64_t* pgrp;         // [P] the group of each partition
  const int64_t* order;        // the groups by tree height, tallest first
  const int64_t* lnode;        // level l >= 1, entry lb + rank: the first node of the group of that rank (scanned)
  int64_t n, P;
};

template <bool ONE>
__device__ __forceinline__ Grp group_ctx(const Groups& Gs, int64_t g) {
  if (ONE) return make_grp(0, Gs.n, 0, 0, Gs.P);
  const int64_t k0 = __ldg(Gs.pbase + g);
  return make_grp(__ldg(Gs.off + g), __ldg(Gs.off + g + 1), k0, __ldg(Gs.ibase + g), __ldg(Gs.pbase + g + 1) - k0);
}

struct Blk { int64_t s, e; double m; };

// smallest block b of partition k (first row base) whose end is > t (t a local row)
__device__ __forceinline__ int leaf_find(const Tree& T, int64_t k, int64_t base, int t) {
  const uint8_t* E = T.end + base;
  int lo = 0, hi = __ldg(T.nb + k) - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if ((int)__ldg(E + mid) > t) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// the block that contains row r in the solution of the level-`lvl` node holding r
template <bool ONE>
__device__ Blk block_of(const Tree& T, const Grp& G, int lvl, int64_t r) {
  const int64_t r0 = ONE ? 0 : G.r0, k = (r - r0) / R;
  int64_t o = ONE ? 0 : G.ib + lv(G, lvl);       // first node of level l
  for (int l = lvl; l >= 1; --l) {
    const int64_t i = (ONE ? T.li[l] : o) + (k >> l);
    const int64_t p = __ldg(T.p + i), q = __ldg(T.q + i);
    if (p <= r && r < q) return {p, q, __ldg(T.m + i)};
    if (!ONE) o -= (G.x >> (l - 1)) + 1;
  }
  const int64_t base = r0 + k * R;
  const int b = leaf_find(T, (ONE ? 0 : G.k0) + k, base, (int)(r - base));
  return {base + (b ? __ldg(T.end + base + b - 1) : 0), base + __ldg(T.end + base + b), __ldg(T.mean + base + b)};
}

// sums of rows [x, end of the level-`lvl` node holding x); x a block start
template <bool ONE>
__device__ void suffix_sums(const Tree& T, const Grp& G, int lvl, int64_t x, double& W, double& S) {
  const int64_t r0 = ONE ? 0 : G.r0, k = (x - r0) / R, base = r0 + k * R, kg = (ONE ? 0 : G.k0) + k;
  const int b = leaf_find(T, kg, base, (int)(x - base));
  const int last = __ldg(T.nb + kg) - 1;
  W = __ldg(T.pw + base + last) - (b ? __ldg(T.pw + base + b - 1) : 0.0);
  S = __ldg(T.ps + base + last) - (b ? __ldg(T.ps + base + b - 1) : 0.0);
  int64_t o = ONE ? 0 : G.w0;                    // first node of level l - 1
  for (int l = 1; l <= lvl; ++l) {
    const int64_t c = k >> (l - 1), last = G.x >> (l - 1), i = (ONE ? T.lw[l - 1] : o) + c + 1;
    if (!(c & 1) && c < last) { W += __ldg(T.W + i); S += __ldg(T.S + i); }   // a right sibling
    if (!ONE) o += last + 1;
  }
}

// sums of rows [start of the level-`lvl` node holding y - 1, y); y a block end
template <bool ONE>
__device__ void prefix_sums(const Tree& T, const Grp& G, int lvl, int64_t y, double& W, double& S) {
  const int64_t r0 = ONE ? 0 : G.r0, k = (y - 1 - r0) / R, base = r0 + k * R;
  const int b = leaf_find(T, (ONE ? 0 : G.k0) + k, base, (int)(y - base) - 1);
  W = __ldg(T.pw + base + b);
  S = __ldg(T.ps + base + b);
  int64_t o = ONE ? 0 : G.w0;                    // first node of level l - 1
  for (int l = 1; l <= lvl; ++l) {
    const int64_t c = k >> (l - 1), i = (ONE ? T.lw[l - 1] : o) + c - 1;
    if (c & 1) { W += __ldg(T.W + i); S += __ldg(T.S + i); }
    if (!ONE) o += (G.x >> (l - 1)) + 1;
  }
}

// mean of the pool [v, u) around the junction of a level-(cl + 1) merge (v <= j <= u, v < u)
template <bool ONE>
__device__ __forceinline__ double pool_mean(const Tree& T, const Grp& G, int cl, int64_t v, int64_t j, int64_t u) {
  double wa = 0.0, sa = 0.0, wb = 0.0, sb = 0.0;
  if (v < j) suffix_sums<ONE>(T, G, cl, v, wa, sa);
  if (u > j) prefix_sums<ONE>(T, G, cl, u, wb, sb);
  return (sa + sb) / (wa + wb);
}

// Largest vertex v <= amax of A's chain from which the pool [v, b) takes no more of A: v == a0, or the block left of v
// has a mean below the pool's.  True for v up to the tangent point and false after it, so a galloping search from amax
// over A's rows (a row stands for the start of its block) finds it.
template <bool ONE>
__device__ int64_t left_tangent(const Tree& T, const Grp& G, int cl, int64_t a0, int64_t j, int64_t amax, int64_t b) {
  auto stops = [&](int64_t v) { return v == a0 || block_of<ONE>(T, G, cl, v - 1).m < pool_mean<ONE>(T, G, cl, v, j, b); };
  if (stops(amax)) return amax;
  int64_t lo = -1, hi = amax, best = a0;   // rows <= lo: true; rows >= hi: false
  for (int64_t d = 1;; d *= 2) {
    const Blk B = block_of<ONE>(T, G, cl, max(a0, amax - d));
    if (stops(B.s)) { lo = B.e - 1; best = B.s; break; }
    hi = B.s;
  }
  while (hi - lo > 1) {
    const Blk B = block_of<ONE>(T, G, cl, lo + (hi - lo) / 2);
    if (stops(B.s)) { lo = B.e - 1; best = B.s; } else { hi = B.s; }
  }
  return best;
}

// Smallest vertex u >= bmin of B's chain at which the pool [a, u) takes no more of B: u == b1, or the block right of u
// has a mean above the pool's.  The mirror image of left_tangent.
template <bool ONE>
__device__ int64_t right_tangent(const Tree& T, const Grp& G, int cl, int64_t j, int64_t b1, int64_t a, int64_t bmin) {
  auto stops = [&](int64_t u) { return u == b1 || block_of<ONE>(T, G, cl, u).m > pool_mean<ONE>(T, G, cl, a, j, u); };
  if (stops(bmin)) return bmin;
  int64_t lo = bmin - 1, hi = b1, best = b1;   // rows <= lo: false; rows >= hi: true
  for (int64_t d = 1;; d *= 2) {
    const Blk B = block_of<ONE>(T, G, cl, min(b1 - 1, bmin + d - 1));
    if (stops(B.e)) { hi = B.s; best = B.e; break; }
    lo = B.e - 1;
  }
  while (hi - lo > 1) {
    const Blk B = block_of<ONE>(T, G, cl, lo + (hi - lo) / 2);
    if (stops(B.e)) { hi = B.s; best = B.e; } else { lo = B.e - 1; }
  }
  return best;
}

// Partitions blockIdx.x * NT + [0, NT).  ONE: partition k is rows [k R, k R + R) of the column; otherwise rows
// [r0, r0 + len) of its group, so the CTA's rows are contiguous within a group with a gap after a group's short last
// partition.
template <bool HAS_W, bool ONE>
__global__ void __launch_bounds__(NT)
iso_leaf(const double* __restrict__ y, const double* __restrict__ w, Groups Gs, double sg, double* __restrict__ pw,
         double* __restrict__ ps, double* __restrict__ mean, uint8_t* __restrict__ end, int* __restrict__ nbo,
         double* __restrict__ W, double* __restrict__ S, double* __restrict__ out, int* status) {
  __shared__ double tS[NT * RP];     // rows, then the block stack (w y sums), then the fitted rows
  __shared__ double tW[NT * RP];     // weights, then the stack's weight sums
  __shared__ uint8_t tE[NT * RP];
  __shared__ int64_t r0s[ONE ? 1 : NT];
  __shared__ int lens[ONE ? 1 : NT];
  const int64_t row0 = (int64_t)blockIdx.x * NT * R;
  const int64_t k = (int64_t)blockIdx.x * NT + threadIdx.x;
  int64_t g = 0;
  Grp G{};
  if (k < Gs.P) {
    if (!ONE) g = __ldg(Gs.pgrp + k);
    G = group_ctx<ONE>(Gs, g);
  }
  if (!ONE) {
    r0s[threadIdx.x] = k < Gs.P ? G.r0 + (k - G.k0) * R : 0;
    lens[threadIdx.x] = k < Gs.P ? (int)min((int64_t)R, G.r1 - r0s[threadIdx.x]) : 0;
    __syncthreads();
  }
  auto row = [&](int i, int64_t& r) {           // the row of tile slot i, false if the slot holds none
    if (ONE) { r = row0 + i; return r < Gs.n; }
    r = r0s[i / R] + i % R;
    return i % R < lens[i / R];
  };
  for (int i = threadIdx.x; i < NT * R; i += NT) {
    int64_t r;
    double v = 0.0, wv = 1.0;
    if (row(i, r)) { v = __ldg(y + r); if (HAS_W) wv = __ldg(w + r); }
    tS[(i / R) * RP + i % R] = v;
    tW[(i / R) * RP + i % R] = wv;
  }
  __syncthreads();
  if (k < Gs.P) {
    double* Sr = tS + threadIdx.x * RP;
    double* Wt = tW + threadIdx.x * RP;
    uint8_t* E = tE + threadIdx.x * RP;
    const int64_t base = ONE ? k * R : r0s[threadIdx.x];
    const int len = ONE ? (int)min((int64_t)R, Gs.n - base) : lens[threadIdx.x];
    int bad = 0, nb = 0;
    for (int i = 0; i < len; ++i) {
      const double yi = Sr[i], wi = Wt[i];
      if (!isfinite(yi) || !isfinite(wi)) bad |= PDSB_ISO_NONFINITE;
      if (wi <= 0.0) bad |= PDSB_ISO_NONPOSITIVE_WEIGHT;
      double s = HAS_W ? wi * (sg * yi) : sg * yi, ws = wi;
      while (nb > 0 && Sr[nb - 1] / Wt[nb - 1] >= s / ws) {   // equal neighbours are pooled, as in the reference
        s += Sr[nb - 1];
        ws += Wt[nb - 1];
        --nb;
      }
      Sr[nb] = s; Wt[nb] = ws; E[nb] = (uint8_t)(i + 1); ++nb;
    }
    if (bad) atomicOr(status + g, bad);
    double cw = 0.0, cs = 0.0;
    for (int b = 0; b < nb; ++b) {
      cw += Wt[b]; cs += Sr[b];
      pw[base + b] = cw; ps[base + b] = cs;
      mean[base + b] = Sr[b] / Wt[b];
      end[base + b] = E[b];
    }
    const int64_t node = G.w0 + (k - G.k0);
    nbo[k] = nb; W[node] = cw; S[node] = cs;
    for (int b = nb - 1; b >= 0; --b) {            // rows of block b start at or after slot b: fill backwards
      const double v = sg * (Sr[b] / Wt[b]);
      for (int i = b ? E[b - 1] : 0; i < E[b]; ++i) Sr[i] = v;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NT * R; i += NT) {
    int64_t r;
    if (row(i, r)) out[r] = tS[(i / R) * RP + i % R];
  }
}

// Node i of level lvl (>= 1) of a group from its children 2i, 2i + 1 of level lvl - 1.  ONE: thread i is node i.
// Otherwise thread t is node lnode[lb] + t of the level: the groups of height > lvl are the first na of `order`, and
// lnode[lb + rank] is where the nodes of the group of that rank start.
template <bool ONE>
__global__ void iso_merge(Tree T, Groups Gs, int lvl, int64_t lb, int64_t na, double* __restrict__ Wo,
                          double* __restrict__ So, int64_t* __restrict__ po, int64_t* __restrict__ qo,
                          double* __restrict__ mo, const int* __restrict__ status) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t g = 0, i = t;
  if (!ONE) {
    const int64_t* L = Gs.lnode + lb;
    const int64_t u = __ldg(L) + t;
    if (u >= __ldg(L + na)) return;
    int64_t lo = 0, hi = na;                       // L[lo] <= u < L[hi]
    while (hi - lo > 1) { const int64_t mid = (lo + hi) >> 1; if (__ldg(L + mid) <= u) lo = mid; else hi = mid; }
    g = __ldg(Gs.order + lo);
    i = u - __ldg(L + lo);
  }
  const Grp G = group_ctx<ONE>(Gs, g);
  if (ONE && i > (G.x >> lvl)) return;
  const int cl = lvl - 1;
  const int64_t ia = 2 * i, ib = 2 * i + 1;
  const int64_t ca = (ONE ? T.lw[cl] : G.wb + lv(G, cl)) + ia, no = (ONE ? T.lw[lvl] : G.wb + lv(G, lvl)) + i,
                io = (ONE ? T.li[lvl] : G.ib + lv(G, lvl)) + i;
  int64_t p = -1, q = -1;
  double m = 0.0;
  if (ib > (G.x >> cl)) {                          // a lone left child: nothing to join
    Wo[no] = __ldg(T.W + ca); So[no] = __ldg(T.S + ca);
  } else {
    Wo[no] = __ldg(T.W + ca) + __ldg(T.W + ca + 1);
    So[no] = __ldg(T.S + ca) + __ldg(T.S + ca + 1);
    if (status[g] == 0) {
      const int64_t span = (int64_t)R << cl;
      const int64_t a0 = G.r0 + ia * span, j = G.r0 + ib * span, b1 = min(j + span, G.r1);
      const Blk L = block_of<ONE>(T, G, cl, j - 1), Rb = block_of<ONE>(T, G, cl, j);
      if (L.m >= Rb.m) {
        int64_t a = L.s, b = Rb.e;
        for (;;) {
          const int64_t a2 = left_tangent<ONE>(T, G, cl, a0, j, a, b);
          const int64_t b2 = right_tangent<ONE>(T, G, cl, j, b1, a2, b);
          if (a2 == a && b2 == b) break;
          a = a2; b = b2;
        }
        p = a; q = b;
        m = pool_mean<ONE>(T, G, cl, a, j, b);
      }
    }
  }
  po[io] = p; qo[io] = q; mo[io] = m;
}

// one warp per partition, one lane per row: the highest bridge covering the row, if any, replaces its leaf-local value.
// top: the tallest tree's top level (ONE: the tree's).
template <bool ONE>
__global__ void iso_final(Tree T, Groups Gs, int top, double sg, double* __restrict__ out, const int* __restrict__ status) {
  const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  if (ONE) {                                     // one tree: its level table in the parameters, nothing per group
    const int64_t r = k * R + (threadIdx.x & 31);
    if (k >= Gs.P || r >= Gs.n) return;
    if (*status != 0) { out[r] = NAN; return; }   // invalid input: all NaN (the host reports w <= 0 as an error)
    for (int l = top; l >= 1; --l) {
      const int64_t i = k >> l;
      const int64_t p = __ldg(T.pl[l] + i), q = __ldg(T.ql[l] + i);
      if (p <= r && r < q) { out[r] = sg * __ldg(T.ml[l] + i); return; }
    }
    return;
  }
  if (k >= Gs.P) return;
  const int64_t g = __ldg(Gs.pgrp + k);
  const Grp G = group_ctx<false>(Gs, g);
  const int64_t kl = k - G.k0;
  const int64_t r = G.r0 + kl * R + (threadIdx.x & 31);
  if (r >= G.r1) return;
  if (status[g] != 0) { out[r] = NAN; return; }
  const int gtop = G.x > 0 ? 64 - __clzll(G.x) : 0;
  int64_t o = G.ib + lv(G, gtop);                // first node of level l
  for (int l = gtop; l >= 1; --l) {
    const int64_t i = o + (kl >> l);
    const int64_t p = __ldg(T.p + i), q = __ldg(T.q + i);
    if (p <= r && r < q) { out[r] = sg * __ldg(T.m + i); return; }
    o -= (G.x >> (l - 1)) + 1;
  }
}

// ---------------- the group tables (grouped calls only) ----------------
// Per group: partitions P = ceil(len / R), tree height L (levels, 0 for an empty group) and internal nodes
// L - 1 + x - popc(x) (x = P - 1); a histogram of L.  pcnt / icnt have n_groups + 1 entries, the last 0.
__global__ void iso_plan(const int64_t* __restrict__ off, int64_t n_groups, int64_t* __restrict__ pcnt,
                         int64_t* __restrict__ icnt, int* __restrict__ height, int64_t* __restrict__ gid,
                         unsigned long long* __restrict__ hist) {
  __shared__ unsigned int h[MAXL + 2];
  for (int i = threadIdx.x; i <= MAXL + 1; i += blockDim.x) h[i] = 0;
  __syncthreads();
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g <= n_groups; g += (int64_t)gridDim.x * blockDim.x) {
    if (g == n_groups) { pcnt[g] = 0; icnt[g] = 0; continue; }
    const int64_t P = (off[g + 1] - off[g] + R - 1) / R, x = P - 1;
    const int L = P == 0 ? 0 : (x == 0 ? 1 : 65 - __clzll(x));
    pcnt[g] = P;
    icnt[g] = P == 0 ? 0 : L - 1 + x - __popcll(x);
    height[g] = L;
    gid[g] = g;
    atomicAdd(h + min(L, MAXL + 1), 1u);   // MAXL + 1: taller than supported
  }
  __syncthreads();
  for (int i = threadIdx.x; i <= MAXL + 1; i += blockDim.x)
    if (h[i]) atomicAdd(hist + i, (unsigned long long)h[i]);
}

struct LevelBases { int64_t lb[MAXL + 1]; int levels; };

// cnt[lb[l] + rank] = nodes at level l of the group of that rank (the groups of height > l are the first ranks); the
// entry after the last is 0, so an exclusive scan gives lnode
__global__ void iso_level_nodes(LevelBases B, const int64_t* __restrict__ order, const int64_t* __restrict__ pbase,
                                int64_t* __restrict__ cnt) {
  const int64_t F = B.lb[B.levels];
  for (int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; f <= F; f += (int64_t)gridDim.x * blockDim.x) {
    if (f == F) { cnt[f] = 0; continue; }
    int l = 1;
    while (B.lb[l + 1] <= f) ++l;
    const int64_t g = order[f - B.lb[l]];
    cnt[f] = ((pbase[g + 1] - pbase[g] - 1) >> l) + 1;
  }
}

// the fit's arrays, carved from one allocation (every sub-array 8-byte aligned); base == nullptr only sizes it
struct Bufs {
  double *pw, *ps, *mean, *W, *S, *m;
  int64_t *p, *q;
  int* nb;
  uint8_t* end;
};
int64_t carve(char* base, int64_t n, int64_t P, int64_t I, Bufs& B) {
  char* cur = base;
  int64_t used = 0;
  auto take = [&](int64_t bytes) { char* r = cur; bytes = (bytes + 7) & ~int64_t(7); used += bytes; if (cur) cur += bytes; return r; };
  B.pw = (double*)take(n * (int64_t)sizeof(double));
  B.ps = (double*)take(n * (int64_t)sizeof(double));
  B.mean = (double*)take(n * (int64_t)sizeof(double));
  B.W = (double*)take((P + I) * (int64_t)sizeof(double));
  B.S = (double*)take((P + I) * (int64_t)sizeof(double));
  B.p = (int64_t*)take(I * (int64_t)sizeof(int64_t));
  B.q = (int64_t*)take(I * (int64_t)sizeof(int64_t));
  B.m = (double*)take(I * (int64_t)sizeof(double));
  B.nb = (int*)take(P * (int64_t)sizeof(int));
  B.end = (uint8_t*)take(n);
  return used;
}
int64_t internal_nodes(int64_t P) {
  if (P <= 0) return 0;
  int64_t I = 0;
  for (int64_t c = P; c > 1;) { c = (c + 1) / 2; I += c; }
  return I;
}

// The leaf pass, the merge levels and the final pass over one group (ONE) or the planned groups.  levels: the tallest
// tree's height; A[l]: groups of height > l (grouped only).
int run_fit(const double* y, const double* w, const Groups& Gs, bool one, const int64_t* A, const LevelBases& LB,
            int levels, int64_t I, int increasing, double* out, int* status, DevBag& bag, cudaStream_t s) {
  Bufs B{};
  char* base = bag.alloc<char>((size_t)carve(nullptr, Gs.n, Gs.P, I, B));
  if (!base) return 1;
  carve(base, Gs.n, Gs.P, I, B);
  Tree T{B.pw, B.ps, B.mean, B.end, B.nb, B.W, B.S, B.p, B.q, B.m, {}, {}, {}, {}, {}};
  if (one)                                       // the one tree's level offsets: node i of level l is W[lw[l] + i]
    for (int l = 0; l < levels; ++l) {
      T.lw[l] = l ? T.lw[l - 1] + ((Gs.P - 1) >> (l - 1)) + 1 : 0;
      T.li[l] = T.lw[l] - Gs.P;
      T.pl[l] = B.p + T.li[l]; T.ql[l] = B.q + T.li[l]; T.ml[l] = B.m + T.li[l];
    }
  const double sg = increasing ? 1.0 : -1.0;
  int rc = 0;
  auto launched = [&]() { cudaError_t e = cudaGetLastError(); count_launch();
                          if (e != cudaSuccess) { set_error("isotonic_regression launch failed: %s", cudaGetErrorString(e)); rc = 1; }
                          return rc == 0; };
  const int gleaf = (int)ceil_div(Gs.P, NT);
#define PDSB_ISO_LEAF(HW, O) iso_leaf<HW, O><<<gleaf, NT, 0, s>>>(y, w, Gs, sg, B.pw, B.ps, B.mean, B.end, B.nb, B.W, B.S, out, status)
  if (one) { if (w) PDSB_ISO_LEAF(true, true); else PDSB_ISO_LEAF(false, true); }
  else     { if (w) PDSB_ISO_LEAF(true, false); else PDSB_ISO_LEAF(false, false); }
#undef PDSB_ISO_LEAF
  if (!launched()) return rc;
  for (int l = 1; l < levels; ++l) {
    if (one) {
      iso_merge<true><<<(int)ceil_div(((Gs.P - 1) >> l) + 1, 128), 128, 0, s>>>(T, Gs, l, 0, 0, B.W, B.S, B.p, B.q, B.m, status);
    } else {
      const int64_t bound = (Gs.P >> l) + A[l];      // sum over the groups of ((P_g - 1) >> l) + 1
      iso_merge<false><<<(int)ceil_div(bound, 128), 128, 0, s>>>(T, Gs, l, LB.lb[l], A[l], B.W, B.S, B.p, B.q, B.m, status);
    }
    if (!launched()) return rc;
  }
  if (one) iso_final<true><<<(int)ceil_div(Gs.P, 8), 256, 0, s>>>(T, Gs, levels - 1, sg, out, status);
  else iso_final<false><<<(int)ceil_div(Gs.P, 8), 256, 0, s>>>(T, Gs, levels - 1, sg, out, status);
  launched();
  return rc;
}

}  // namespace

int64_t isotonic_scratch_bytes(int64_t n) {
  if (n <= 0) return 0;
  const int64_t P = ceil_div(n, R);
  Bufs B{};
  return carve(nullptr, n, P, internal_nodes(P), B);
}

int isotonic_fit(const double* y, const double* w, int64_t n, int increasing, double* out, int* status,
                 cudaStream_t s) {
  PDSB_CUDA_OK(cudaMemsetAsync(status, 0, sizeof(int), s));
  if (n <= 0) return 0;
  const int64_t P = ceil_div(n, R);
  int levels = 1;
  for (int64_t c = P; c > 1; c = (c + 1) / 2) ++levels;
  if (levels > MAXL) { set_error("isotonic_regression: %lld rows is more than supported", (long long)n); return 1; }
  Groups Gs{};
  Gs.n = n; Gs.P = P;
  DevBag bag(s);
  return run_fit(y, w, Gs, true, nullptr, LevelBases{}, levels, internal_nodes(P), increasing, out, status, bag, s);
}

int grouped_isotonic_fit(const double* y, const double* w, const int64_t* offsets, int64_t n_groups, int64_t n,
                         int increasing, double* out, int* status, cudaStream_t s) {
  if (n_groups <= 0) return 0;
  PDSB_CUDA_OK(cudaMemsetAsync(status, 0, (size_t)n_groups * sizeof(int), s));
  if (n <= 0) return 0;
  const size_t G1 = (size_t)n_groups + 1;
  DevBag bag(s);
  int64_t* pcnt = bag.alloc<int64_t>(G1);
  int64_t* icnt = bag.alloc<int64_t>(G1);
  int64_t* pbase = bag.alloc<int64_t>(G1);
  int64_t* ibase = bag.alloc<int64_t>(G1);
  int* height = bag.alloc<int>((size_t)n_groups);
  int64_t* gid = bag.alloc<int64_t>((size_t)n_groups);
  unsigned long long* hist = bag.alloc<unsigned long long>(MAXL + 2);
  if (!pcnt || !icnt || !pbase || !ibase || !height || !gid || !hist) return 1;
  PDSB_CUDA_OK(cudaMemsetAsync(hist, 0, (MAXL + 2) * sizeof(unsigned long long), s));
  iso_plan<<<(int)std::min<int64_t>(ceil_div((int64_t)G1, 256), 4096), 256, 0, s>>>(offsets, n_groups, pcnt, icnt, height,
                                                                                      gid, hist);
  PDSB_LAUNCH_OK();
  count_launch();
  size_t tb = 0;
  PDSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, tb, pcnt, pbase, (int64_t)G1, s));
  void* tmp = bag.alloc<unsigned char>(std::max<size_t>(tb, 1));
  if (!tmp) return 1;
  PDSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(tmp, tb, pcnt, pbase, (int64_t)G1, s));
  PDSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(tmp, tb, icnt, ibase, (int64_t)G1, s));
  unsigned long long h[MAXL + 2];
  int64_t P = 0, I = 0;
  PDSB_CUDA_OK(cudaMemcpyAsync(h, hist, sizeof(h), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaMemcpyAsync(&P, pbase + n_groups, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaMemcpyAsync(&I, ibase + n_groups, sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  PDSB_CUDA_OK(cudaStreamSynchronize(s));
  if (h[MAXL + 1]) { set_error("isotonic_regression: a group has more rows than supported"); return 1; }
  int levels = 0;
  for (int l = 0; l <= MAXL; ++l) if (h[l]) levels = l;
  // A[l] = groups taller than l; level l >= 1 has entries lb[l] .. lb[l] + A[l] of lnode
  int64_t A[MAXL + 1] = {0};
  LevelBases LB{};
  LB.levels = std::max(levels, 1);
  for (int l = levels - 1; l >= 1; --l) A[l] = A[l + 1] + (int64_t)h[l + 1];
  LB.lb[1] = 0;
  for (int l = 1; l < LB.levels; ++l) LB.lb[l + 1] = LB.lb[l] + A[l];
  Groups Gs{offsets, pbase, ibase, nullptr, nullptr, nullptr, n, P};
  int64_t* pgrp = bag.alloc<int64_t>((size_t)P);
  if (!pgrp) return 1;
  segment_groups<<<(int)std::min<int64_t>(ceil_div(P, 256), 8192), 256, 0, s>>>(pbase, n_groups, P, pgrp);   // pgrp[k]: partition k's group
  PDSB_LAUNCH_OK();
  count_launch();
  Gs.pgrp = pgrp;
  if (levels >= 2) {                               // some group has merges: its nodes per level, tallest groups first
    const int64_t F = LB.lb[levels];
    int* hsorted = bag.alloc<int>((size_t)n_groups);
    int64_t* order = bag.alloc<int64_t>((size_t)n_groups);
    int64_t* cnt = bag.alloc<int64_t>((size_t)F + 1);
    int64_t* lnode = bag.alloc<int64_t>((size_t)F + 1);
    if (!hsorted || !order || !cnt || !lnode) return 1;
    size_t ts = 0, tc = 0;
    PDSB_CUDA_OK(cub::DeviceRadixSort::SortPairsDescending(nullptr, ts, height, hsorted, gid, order, n_groups, 0, 6, s));
    PDSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, tc, cnt, lnode, F + 1, s));
    void* tmp2 = bag.alloc<unsigned char>(std::max<size_t>(std::max(ts, tc), 1));
    if (!tmp2) return 1;
    PDSB_CUDA_OK(cub::DeviceRadixSort::SortPairsDescending(tmp2, ts, height, hsorted, gid, order, n_groups, 0, 6, s));
    iso_level_nodes<<<(int)std::min<int64_t>(ceil_div(F + 1, 256), 8192), 256, 0, s>>>(LB, order, pbase, cnt);
    PDSB_LAUNCH_OK();
    count_launch();
    PDSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(tmp2, tc, cnt, lnode, F + 1, s));
    Gs.order = order; Gs.lnode = lnode;
  }
  return run_fit(y, w, Gs, false, A, LB, levels, I, increasing, out, status, bag, s);
}

}  // namespace pdsb
