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
// DESIGN.md "K15 in detail" has the byte count, the work bound and the choices.
//
// ptxas (-Xptxas -v, sm_90a, CUDA 12.9): see DESIGN.md "K15 in detail"; no stack frame and no spill in any kernel.
#include "../common.h"
#include "kernels.h"
#include <cmath>
#include <vector>

namespace pdsb {
namespace {

constexpr int R = 32;          // rows per partition (= lanes of the final pass's warp)
constexpr int NT = 64;         // partitions per CTA in the leaf pass
constexpr int RP = R + 1;      // shared-memory row pitch (conflict-free column access)
constexpr int MAXL = 40;       // tree levels: up to 2^39 partitions

struct Tree {
  const double* pw;            // [P R] leaf-local inclusive prefix of w over the blocks (slot k R + b)
  const double* ps;            // [P R] the same of w y
  const double* mean;          // [P R] block mean
  const uint8_t* end;          // [P R] block end row, local to the partition (exclusive)
  const int* nb;               // [P] blocks per partition
  const double* W[MAXL];       // per level: node totals of w and w y (level 0 = the partitions)
  const double* S[MAXL];
  const int64_t* p[MAXL];      // per level >= 1: bridge [p, q) (p = q = -1: none) and its mean
  const int64_t* q[MAXL];
  const double* m[MAXL];
  int64_t cnt[MAXL];           // nodes per level
  int64_t n;
};

struct Blk { int64_t s, e; double m; };

// smallest block b of partition k whose end is > t (t a local row)
__device__ __forceinline__ int leaf_find(const Tree& T, int64_t k, int t) {
  const uint8_t* E = T.end + k * R;
  int lo = 0, hi = __ldg(T.nb + k) - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if ((int)__ldg(E + mid) > t) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// the block that contains row r in the solution of the level-`lvl` node holding r
__device__ Blk block_of(const Tree& T, int lvl, int64_t r) {
  const int64_t k = r / R;
  for (int l = lvl; l >= 1; --l) {
    const int64_t i = k >> l;
    const int64_t p = __ldg(T.p[l] + i), q = __ldg(T.q[l] + i);
    if (p <= r && r < q) return {p, q, __ldg(T.m[l] + i)};
  }
  const int b = leaf_find(T, k, (int)(r - k * R));
  const int64_t base = k * R;
  return {base + (b ? __ldg(T.end + base + b - 1) : 0), base + __ldg(T.end + base + b), __ldg(T.mean + base + b)};
}

// sums of rows [x, end of the level-`lvl` node holding x); x a block start
__device__ void suffix_sums(const Tree& T, int lvl, int64_t x, double& W, double& S) {
  const int64_t k = x / R, base = k * R;
  const int b = leaf_find(T, k, (int)(x - base));
  const int last = __ldg(T.nb + k) - 1;
  W = __ldg(T.pw + base + last) - (b ? __ldg(T.pw + base + b - 1) : 0.0);
  S = __ldg(T.ps + base + last) - (b ? __ldg(T.ps + base + b - 1) : 0.0);
  for (int l = 1; l <= lvl; ++l) {
    const int64_t c = k >> (l - 1);
    if (!(c & 1) && c + 1 < T.cnt[l - 1]) { W += __ldg(T.W[l - 1] + c + 1); S += __ldg(T.S[l - 1] + c + 1); }
  }
}

// sums of rows [start of the level-`lvl` node holding y - 1, y); y a block end
__device__ void prefix_sums(const Tree& T, int lvl, int64_t y, double& W, double& S) {
  const int64_t k = (y - 1) / R, base = k * R;
  const int b = leaf_find(T, k, (int)(y - base) - 1);
  W = __ldg(T.pw + base + b);
  S = __ldg(T.ps + base + b);
  for (int l = 1; l <= lvl; ++l) {
    const int64_t c = k >> (l - 1);
    if (c & 1) { W += __ldg(T.W[l - 1] + c - 1); S += __ldg(T.S[l - 1] + c - 1); }
  }
}

// mean of the pool [v, u) around the junction of a level-(cl + 1) merge (v <= j <= u, v < u)
__device__ __forceinline__ double pool_mean(const Tree& T, int cl, int64_t v, int64_t j, int64_t u) {
  double wa = 0.0, sa = 0.0, wb = 0.0, sb = 0.0;
  if (v < j) suffix_sums(T, cl, v, wa, sa);
  if (u > j) prefix_sums(T, cl, u, wb, sb);
  return (sa + sb) / (wa + wb);
}

// Largest vertex v <= amax of A's chain from which the pool [v, b) takes no more of A: v == a0, or the block left of v
// has a mean below the pool's.  True for v up to the tangent point and false after it, so a galloping search from amax
// over A's rows (a row stands for the start of its block) finds it.
__device__ int64_t left_tangent(const Tree& T, int cl, int64_t a0, int64_t j, int64_t amax, int64_t b) {
  auto stops = [&](int64_t v) { return v == a0 || block_of(T, cl, v - 1).m < pool_mean(T, cl, v, j, b); };
  if (stops(amax)) return amax;
  int64_t lo = -1, hi = amax, best = a0;   // rows <= lo: true; rows >= hi: false
  for (int64_t d = 1;; d *= 2) {
    const Blk B = block_of(T, cl, max(a0, amax - d));
    if (stops(B.s)) { lo = B.e - 1; best = B.s; break; }
    hi = B.s;
  }
  while (hi - lo > 1) {
    const Blk B = block_of(T, cl, lo + (hi - lo) / 2);
    if (stops(B.s)) { lo = B.e - 1; best = B.s; } else { hi = B.s; }
  }
  return best;
}

// Smallest vertex u >= bmin of B's chain at which the pool [a, u) takes no more of B: u == b1, or the block right of u
// has a mean above the pool's.  The mirror image of left_tangent.
__device__ int64_t right_tangent(const Tree& T, int cl, int64_t j, int64_t b1, int64_t a, int64_t bmin) {
  auto stops = [&](int64_t u) { return u == b1 || block_of(T, cl, u).m > pool_mean(T, cl, a, j, u); };
  if (stops(bmin)) return bmin;
  int64_t lo = bmin - 1, hi = b1, best = b1;   // rows <= lo: false; rows >= hi: true
  for (int64_t d = 1;; d *= 2) {
    const Blk B = block_of(T, cl, min(b1 - 1, bmin + d - 1));
    if (stops(B.e)) { hi = B.s; best = B.e; break; }
    lo = B.e - 1;
  }
  while (hi - lo > 1) {
    const Blk B = block_of(T, cl, lo + (hi - lo) / 2);
    if (stops(B.e)) { hi = B.s; best = B.e; } else { lo = B.e - 1; }
  }
  return best;
}

template <bool HAS_W>
__global__ void __launch_bounds__(NT)
iso_leaf(const double* __restrict__ y, const double* __restrict__ w, int64_t n, int64_t P, double sg,
         double* __restrict__ pw, double* __restrict__ ps, double* __restrict__ mean, uint8_t* __restrict__ end,
         int* __restrict__ nbo, double* __restrict__ W0, double* __restrict__ S0, double* __restrict__ out,
         int* status) {
  __shared__ double tS[NT * RP];     // rows, then the block stack (w y sums), then the fitted rows
  __shared__ double tW[NT * RP];     // weights, then the stack's weight sums
  __shared__ uint8_t tE[NT * RP];
  const int64_t row0 = (int64_t)blockIdx.x * NT * R;
  for (int i = threadIdx.x; i < NT * R; i += NT) {
    const int64_t r = row0 + i;
    double v = 0.0, wv = 1.0;
    if (r < n) { v = __ldg(y + r); if (HAS_W) wv = __ldg(w + r); }
    tS[(i / R) * RP + i % R] = v;
    tW[(i / R) * RP + i % R] = wv;
  }
  __syncthreads();
  const int64_t k = (int64_t)blockIdx.x * NT + threadIdx.x;
  if (k < P) {
    double* S = tS + threadIdx.x * RP;
    double* Wt = tW + threadIdx.x * RP;
    uint8_t* E = tE + threadIdx.x * RP;
    const int len = (int)min((int64_t)R, n - k * R);
    int bad = 0, nb = 0;
    for (int i = 0; i < len; ++i) {
      const double yi = S[i], wi = Wt[i];
      if (!isfinite(yi) || !isfinite(wi)) bad |= PDSB_ISO_NONFINITE;
      if (wi <= 0.0) bad |= PDSB_ISO_NONPOSITIVE_WEIGHT;
      double s = HAS_W ? wi * (sg * yi) : sg * yi, ws = wi;
      while (nb > 0 && S[nb - 1] / Wt[nb - 1] >= s / ws) {   // equal neighbours are pooled, as in the reference
        s += S[nb - 1];
        ws += Wt[nb - 1];
        --nb;
      }
      S[nb] = s; Wt[nb] = ws; E[nb] = (uint8_t)(i + 1); ++nb;
    }
    if (bad) atomicOr(status, bad);
    const int64_t base = k * R;
    double cw = 0.0, cs = 0.0;
    for (int b = 0; b < nb; ++b) {
      cw += Wt[b]; cs += S[b];
      pw[base + b] = cw; ps[base + b] = cs;
      mean[base + b] = S[b] / Wt[b];
      end[base + b] = E[b];
    }
    nbo[k] = nb; W0[k] = cw; S0[k] = cs;
    for (int b = nb - 1; b >= 0; --b) {            // rows of block b start at or after slot b: fill backwards
      const double v = sg * (S[b] / Wt[b]);
      for (int i = b ? E[b - 1] : 0; i < E[b]; ++i) S[i] = v;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < NT * R; i += NT) {
    const int64_t r = row0 + i;
    if (r < n) out[r] = tS[(i / R) * RP + i % R];
  }
}

// node i of level lvl (>= 1) from its children 2i, 2i + 1 of level lvl - 1
__global__ void iso_merge(Tree T, int lvl, double* __restrict__ Wo, double* __restrict__ So, int64_t* __restrict__ po,
                          int64_t* __restrict__ qo, double* __restrict__ mo, const int* __restrict__ status) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= T.cnt[lvl]) return;
  const int cl = lvl - 1;
  const int64_t ia = 2 * i, ib = 2 * i + 1;
  int64_t p = -1, q = -1;
  double m = 0.0;
  if (ib >= T.cnt[cl]) {                           // a lone left child: nothing to join
    Wo[i] = __ldg(T.W[cl] + ia); So[i] = __ldg(T.S[cl] + ia);
  } else {
    Wo[i] = __ldg(T.W[cl] + ia) + __ldg(T.W[cl] + ib);
    So[i] = __ldg(T.S[cl] + ia) + __ldg(T.S[cl] + ib);
    if (*status == 0) {
      const int64_t span = (int64_t)R << cl;
      const int64_t a0 = ia * span, j = ib * span, b1 = min(j + span, T.n);
      const Blk L = block_of(T, cl, j - 1), Rb = block_of(T, cl, j);
      if (L.m >= Rb.m) {
        int64_t a = L.s, b = Rb.e;
        for (;;) {
          const int64_t a2 = left_tangent(T, cl, a0, j, a, b);
          const int64_t b2 = right_tangent(T, cl, j, b1, a2, b);
          if (a2 == a && b2 == b) break;
          a = a2; b = b2;
        }
        p = a; q = b;
        m = pool_mean(T, cl, a, j, b);
      }
    }
  }
  po[i] = p; qo[i] = q; mo[i] = m;
}

// one warp per partition, one lane per row: the highest bridge covering the row, if any, replaces its leaf-local value
__global__ void iso_final(Tree T, int top, double sg, double* __restrict__ out, const int* __restrict__ status) {
  const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
  const int64_t r = k * R + (threadIdx.x & 31);
  if (k >= T.cnt[0] || r >= T.n) return;
  if (*status != 0) { out[r] = NAN; return; }     // invalid input: all NaN (the host reports w <= 0 as an error)
  for (int l = top; l >= 1; --l) {
    const int64_t i = k >> l;
    const int64_t p = __ldg(T.p[l] + i), q = __ldg(T.q[l] + i);
    if (p <= r && r < q) { out[r] = sg * __ldg(T.m[l] + i); return; }
  }
}

}  // namespace

int64_t isotonic_scratch_bytes(int64_t n) {
  if (n <= 0) return 0;
  const int64_t P = ceil_div(n, R);
  int64_t b = P * R * (3 * (int64_t)sizeof(double) + 1) + ((P * (int64_t)sizeof(int) + 7) & ~int64_t(7));
  for (int64_t c = P, l = 0;; ++l) {
    b += c * (2 * (int64_t)sizeof(double)) + (l ? c * (2 * (int64_t)sizeof(int64_t) + (int64_t)sizeof(double)) : 0);
    if (c == 1) break;
    c = (c + 1) / 2;
  }
  return b;
}

int isotonic_fit(const double* y, const double* w, int64_t n, int increasing, double* out, int* status,
                 cudaStream_t s) {
  PDSB_CUDA_OK(cudaMemsetAsync(status, 0, sizeof(int), s));
  if (n <= 0) return 0;
  const int64_t P = ceil_div(n, R);
  std::vector<int64_t> cnt;
  for (int64_t c = P;; c = (c + 1) / 2) { cnt.push_back(c); if (c == 1) break; }
  const int L = (int)cnt.size();
  if (L > MAXL) { set_error("isotonic_regression: %lld rows is more than supported", (long long)n); return 1; }
  char* base = nullptr;
  if (dev_alloc((void**)&base, (size_t)isotonic_scratch_bytes(n), s)) return 1;
  // doubles first, then the int64 bridge bounds, then the ints and bytes (every sub-array stays 8-byte aligned)
  char* cur = base;
  auto take = [&](size_t bytes) { char* p = cur; cur += (bytes + 7) & ~size_t(7); return p; };
  double* pw = (double*)take(P * R * sizeof(double));
  double* ps = (double*)take(P * R * sizeof(double));
  double* mean = (double*)take(P * R * sizeof(double));
  Tree T{};
  double* Wl[MAXL]; double* Sl[MAXL]; int64_t* pl[MAXL]; int64_t* ql[MAXL]; double* ml[MAXL];
  for (int l = 0; l < L; ++l) {
    Wl[l] = (double*)take(cnt[l] * sizeof(double));
    Sl[l] = (double*)take(cnt[l] * sizeof(double));
    if (l) {
      pl[l] = (int64_t*)take(cnt[l] * sizeof(int64_t));
      ql[l] = (int64_t*)take(cnt[l] * sizeof(int64_t));
      ml[l] = (double*)take(cnt[l] * sizeof(double));
    } else {
      pl[l] = ql[l] = nullptr; ml[l] = nullptr;
    }
    T.W[l] = Wl[l]; T.S[l] = Sl[l]; T.p[l] = pl[l]; T.q[l] = ql[l]; T.m[l] = ml[l]; T.cnt[l] = cnt[l];
  }
  int* nb = (int*)take(P * sizeof(int));
  uint8_t* end = (uint8_t*)take(P * R);
  T.pw = pw; T.ps = ps; T.mean = mean; T.end = end; T.nb = nb; T.n = n;
  const double sg = increasing ? 1.0 : -1.0;
  int rc = 0;
  auto launched = [&]() { cudaError_t e = cudaGetLastError(); count_launch();
                          if (e != cudaSuccess) { set_error("isotonic_regression launch failed: %s", cudaGetErrorString(e)); rc = 1; }
                          return rc == 0; };
  const int gleaf = (int)ceil_div(P, NT);
  if (w) iso_leaf<true><<<gleaf, NT, 0, s>>>(y, w, n, P, sg, pw, ps, mean, end, nb, Wl[0], Sl[0], out, status);
  else iso_leaf<false><<<gleaf, NT, 0, s>>>(y, w, n, P, sg, pw, ps, mean, end, nb, Wl[0], Sl[0], out, status);
  if (!launched()) goto done;
  for (int l = 1; l < L; ++l) {
    iso_merge<<<(int)ceil_div(cnt[l], 128), 128, 0, s>>>(T, l, Wl[l], Sl[l], pl[l], ql[l], ml[l], status);
    if (!launched()) goto done;
  }
  iso_final<<<(int)ceil_div(P, 8), 256, 0, s>>>(T, L - 1, sg, out, status);
  launched();
done:
  dev_free(base, s);
  return rc;
}

}  // namespace pdsb
