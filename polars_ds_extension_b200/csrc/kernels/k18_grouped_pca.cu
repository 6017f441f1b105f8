// K18 — group_by(key).agg(pds.singular_values / pds.pca) and pds.principal_components(...).over(key): every group's
// centred Gram, eigen-solve and projection in one launch sequence.
//
// Polars' loop makes one pl_singular_values / pl_pca / pl_principal_components call per group (K13: an upload, a K2a
// Gram, a one-CTA Jacobi, a synchronise, a download).  Here the frame stays in HBM in key order, as for pl_lr_by:
//   pass 0  K5's work list (build_work_list): a group of len rows is ceil(len / 8192) items of equal size;
//   pass 1  (center only) one warp per item: per column, the sum (f64) and the count of the non-null values;
//   pass 2  one warp per item: the group's means from the pass-1 partials (summed in item order), then the packed Gram of
//           [x - mu | 1] over the item's kept rows, products and sums in f64 (f32 is widened after centring), through a
//           [32][p + 2] shared tile and tile_triangle_sum;
//   pass 3  one 32-thread CTA per group: the item Grams summed in item order, jacobi.h's Jacobi with NT = 32, K13's stable
//           descending sort and svd_flip sign rule, sigma = sqrt(max(lambda, 0));
//   pass 4  (principal_components) one warp per item: mu and V[:, :k] of its group in shared memory, then one row per lane,
//           (x - mu) V[:, j] in f64 with K13's per-row arithmetic; rows of a group with fewer rows than k are NaN.
// Centring rule (the loop's `f - f.mean()`): a column's mean is taken over its non-null values in the group, in f64; a
// value is null when its row is masked and it is NaN (the host uploads nulls as NaN).  f32 columns subtract the mean
// rounded to f32 in f32 arithmetic; f64 columns subtract it in f64.  The Gram is that of the centred values, never
// S - n mu mu^T, which would lose (mu / sigma)^2 eps.  Only masked rows leave the Gram: a NaN or inf in a kept row reaches
// it and the group's status reads PDSB_PCA_NONFINITE.  Every partial is reduced in an order fixed by the group's own
// rows, so a group's sigma, V and components are bit for bit the same whatever the other groups hold.
// HBM bytes per row: p s in pass 1 (+ s for the mask), p s again in pass 2, and p s + 8 k in pass 4.
//
// ptxas (-Xptxas -v, sm_90a, CUDA 12.9), registers; no spill anywhere, and no stack frame except pca_gram_kernel's:
//   pca_sums_kernel f32 / f64 37 / 38; pca_gram_kernel f32 / f64 40 / 48 with a 560-byte stack frame (acc[PACKED_ACC],
//   indexed at run time by tile_triangle_sum, lives in local memory); grouped_eigen_kernel 64;
//   grouped_project_kernel<T, KT> for KT = 1 / 2 / 4 / 8: f32 32 / 32 / 40 / 48, f64 32 / 32 / 40 / 46.
#include "../common.h"
#include "kernels.h"
#include "../host/host.h"
#include "k5_solve.h"
#include <cmath>

namespace pdsb {

namespace {

constexpr int NT = 32;          // jacobi.h's CTA size: one warp per group in pass 3

}  // namespace
}  // namespace pdsb

#include "jacobi.h"

namespace pdsb {
namespace {

constexpr int GK_MAXP = 64;     // features per call
constexpr int SW_WARPS = 8;     // warps per CTA of pass 1
constexpr int GW_WARPS = 4;     // warps per CTA of pass 2
constexpr int PW_WARPS = 4;     // warps per CTA of pass 4

// x - mu by the loop's rule: f32 in f32 with the mean rounded to f32, everything else in f64
template <typename T>
__device__ __forceinline__ double centred(T x, double mu) {
  if constexpr (sizeof(T) == 4) return (double)(x - (float)mu);
  else return (double)x - mu;
}

// ---------------- pass 1: per-item column sums and non-null counts ----------------
// part1[c][it] = sum of column c's non-null values in item it, part1[p + c][it] = their number
template <typename T>
__global__ void __launch_bounds__(SW_WARPS * 32)
pca_sums_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ mask, const int64_t* __restrict__ rows,
                int64_t n_items, int p, double* __restrict__ part1, unsigned long long* __restrict__ queue) {
  const int lane = threadIdx.x & 31;
  for (int64_t item = pop_item(queue); item < n_items; item = pop_item(queue)) {
    const int64_t r0 = rows[2 * item], r1 = rows[2 * item + 1];
    for (int c = 0; c < p; ++c) {
      const T* xc = X + (int64_t)c * ldx;
      double s = 0.0, cnt = 0.0;
#pragma unroll 4
      for (int64_t r = r0 + lane; r < r1; r += 32) {
        const T x = xc[r];
        const bool null = mask && mask[r] == T(0) && isnan(x);
        if (!null) { s += (double)x; cnt += 1.0; }
      }
      for (int off = 16; off; off >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, off);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
      }
      if (lane == 0) {
        part1[(size_t)c * n_items + item] = s;
        part1[(size_t)(p + c) * n_items + item] = cnt;
      }
    }
  }
}

// the means of group g from the pass-1 partials, summed in item order, into mu[0..p) (shared); one lane per column
__device__ __forceinline__ void group_means(const double* __restrict__ part1, const int64_t* __restrict__ item_start,
                                            int64_t n_items, int64_t g, int p, double* mu) {
  for (int c = threadIdx.x & 31; c < p; c += 32) {
    double s = 0.0, cnt = 0.0;
    for (int64_t it = item_start[g]; it < item_start[g + 1]; ++it) {
      s += part1[(size_t)c * n_items + it];
      cnt += part1[(size_t)(p + c) * n_items + it];
    }
    mu[c] = s / cnt;        // 0 / 0 = NaN for a column without a value: every row of the group is masked then
  }
}

// ---------------- pass 2: per-item Gram of [x - mu | 1] over the kept rows ----------------
// part2[k][it], k = the packed upper triangle over q1 = p + 1 columns (the last one counts the kept rows).  mean
// (center only): [n_groups][p], written by the warp that takes the group's first item.
template <typename T>
__global__ void __launch_bounds__(GW_WARPS * 32)
pca_gram_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ mask, const int64_t* __restrict__ rows,
                const int64_t* __restrict__ group, const int64_t* __restrict__ item_start, int64_t n_items, int p,
                int center, const double* __restrict__ part1, double* __restrict__ mean, double* __restrict__ part2,
                unsigned long long* __restrict__ queue) {
  extern __shared__ __align__(16) double gsm[];
  const int lane = threadIdx.x & 31, q1 = p + 1, ld = q1 + 1, nm = q1 * (q1 + 1) / 2;
  double* tile = gsm + (size_t)(threadIdx.x >> 5) * (32 * ld + GK_MAXP);
  double* mu = tile + 32 * ld;
  double* my = tile + (size_t)lane * ld;
  const int per_lane = (nm + 31) / 32;
  for (int64_t item = pop_item(queue); item < n_items; item = pop_item(queue)) {
    const int64_t g = group[item];
    const int64_t r0 = rows[2 * item], r1 = rows[2 * item + 1];
    __syncwarp();                                  // the previous item's reads of mu are done
    if (center) {
      group_means(part1, item_start, n_items, g, p, mu);
      if (item == item_start[g])
        for (int c = lane; c < p; c += 32) mean[(size_t)g * p + c] = mu[c];
    }
    __syncwarp();
    double acc[PACKED_ACC];
    for (int m = 0; m < per_lane; ++m) acc[m] = 0.0;
    for (int64_t rb = r0; rb < r1; rb += 32) {
      const int64_t r = rb + lane;
      const bool keep = r < r1 && (!mask || mask[r] != T(0));
      for (int c = 0; c < p; ++c) {
        double v = 0.0;
        if (keep) {
          const T x = X[(int64_t)c * ldx + r];
          v = center ? centred<T>(x, mu[c]) : (double)x;
        }
        my[c] = v;
      }
      my[p] = keep ? 1.0 : 0.0;
      __syncwarp();
      tile_triangle_sum(tile, ld, q1, nullptr, 0, acc);
      __syncwarp();
    }
    for (int m = 0; m < per_lane; ++m) {
      const int k = lane + 32 * m;
      if (k < nm) part2[(size_t)k * n_items + item] = acc[m];
    }
  }
}

// ---------------- pass 3: one eigen-solve per group ----------------
// One 32-thread CTA per group, everything in shared memory: A and Vu [p x p], jacobi.h's rotation table, the sort.
// status[2g] = PDSB_PCA_OK or PDSB_PCA_NONFINITE (a NaN / inf in the summed Gram), status[2g + 1] = min(kept rows, p).
__host__ __device__ inline size_t eigen_smem(int p) {
  return (2 * (size_t)p * p + 4 * (size_t)(p / 2 + 2)) * sizeof(double) + (size_t)p * sizeof(int);
}

__global__ void __launch_bounds__(NT)
grouped_eigen_kernel(const double* __restrict__ part2, const int64_t* __restrict__ item_start, int64_t n_items, int p,
                     double* __restrict__ sigma, double* __restrict__ V, int* __restrict__ status) {
  extern __shared__ __align__(16) double esm[];
  const int64_t g = blockIdx.x;
  const int tid = threadIdx.x, q1 = p + 1, nm = q1 * (q1 + 1) / 2;
  double* A = esm;
  double* Vu = A + (size_t)p * p;
  double* cs = Vu + (size_t)p * p;
  int* perm = reinterpret_cast<int*>(cs + 4 * (size_t)(p / 2 + 2));
  const int64_t it0 = item_start[g], it1 = item_start[g + 1];
  bool bad = false;
  double count = 0.0;
  for (int k = tid; k < nm; k += NT) {
    double s = 0.0;
    for (int64_t it = it0; it < it1; ++it) s += part2[(size_t)k * n_items + it];
    bad |= !isfinite(s);
    int i, j;
    packed_pair(k, q1, i, j);
    if (j < p) { at(A, p, i, j) = s; at(A, p, j, i) = s; }
    else if (i == p) count = s;
  }
  bad = __any_sync(0xffffffffu, bad);
  count = __shfl_sync(0xffffffffu, count, (nm - 1) % NT);
  if (tid == 0) {
    status[2 * g] = bad ? PDSB_PCA_NONFINITE : PDSB_PCA_OK;
    status[2 * g + 1] = (int)fmin(fmax(rint(count), 0.0), (double)p);
  }
  if (bad) return;
  __syncthreads();
  jacobi_eigen(A, Vu, p, cs);
  // K13's stable descending order and sign rule (pca_eigen_kernel)
  for (int i = tid; i < p; i += NT) {
    const double li = at(A, p, i, i);
    int r = 0;
    for (int j = 0; j < p; ++j) {
      const double lj = at(A, p, j, j);
      r += (lj > li) || (lj == li && j < i);
    }
    perm[r] = i;
  }
  __syncthreads();
  double* Vg = V + (size_t)g * p * p;
  for (int r = tid; r < p; r += NT) {
    const int c = perm[r];
    int best = 0; double bmax = -1.0;
    for (int i = 0; i < p; ++i) { const double a = fabs(at(Vu, p, i, c)); if (a > bmax) { bmax = a; best = i; } }
    const double sgn = at(Vu, p, best, c) < 0.0 ? -1.0 : 1.0;
    for (int i = 0; i < p; ++i) Vg[i + (size_t)r * p] = sgn * at(Vu, p, i, c);
    sigma[(size_t)g * p + r] = sqrt(fmax(at(A, p, c, c), 0.0));
  }
}

// ---------------- pass 4: segmented projection ----------------
// out[j * ldo + r] = sum_c (x_rc - mu_c) V_g[c, j], j < k, in f64 with K13's order (one fma per feature in column order),
// KT outputs per lane at a time.  Per warp of shared memory: mu [p] and V_g[:, :k] as [p][k].
__host__ __device__ inline size_t project_warp_doubles(int p, int k) { return (size_t)p + (size_t)p * k; }

template <typename T, int KT>
__global__ void __launch_bounds__(PW_WARPS * 32)
grouped_project_kernel(const T* __restrict__ X, int64_t ldx, const int64_t* __restrict__ offsets,
                       const int64_t* __restrict__ rows, const int64_t* __restrict__ group, int64_t n_items, int p,
                       const double* __restrict__ mean, const double* __restrict__ V, int k, double* __restrict__ out,
                       int64_t ldo, unsigned long long* __restrict__ queue) {
  extern __shared__ __align__(16) double psm[];
  const int lane = threadIdx.x & 31;
  double* mu = psm + (size_t)(threadIdx.x >> 5) * project_warp_doubles(p, k);
  double* vs = mu + p;
  for (int64_t item = pop_item(queue); item < n_items; item = pop_item(queue)) {
    const int64_t r0 = rows[2 * item], r1 = rows[2 * item + 1];
    if (r0 >= r1) continue;
    const int64_t g = group[item];
    if (offsets[g + 1] - offsets[g] < k) {          // pca.rs:90-93: fewer rows than k
      for (int64_t r = r0 + lane; r < r1; r += 32)
        for (int j = 0; j < k; ++j) out[(int64_t)j * ldo + r] = nan("");
      continue;
    }
    __syncwarp();                                  // the previous item's reads of mu / vs are done
    for (int c = lane; c < p; c += 32) mu[c] = mean ? mean[(size_t)g * p + c] : 0.0;
    const double* Vg = V + (size_t)g * p * p;
    for (int e = lane; e < p * k; e += 32) { const int c = e / k, j = e - c * k; vs[e] = Vg[c + (size_t)j * p]; }
    __syncwarp();
    for (int64_t r = r0 + lane; r < r1; r += 32) {
      for (int j0 = 0; j0 < k; j0 += KT) {
        double acc[KT];
#pragma unroll
        for (int j = 0; j < KT; ++j) acc[j] = 0.0;
        for (int c = 0; c < p; ++c) {
          const T x = X[(int64_t)c * ldx + r];
          const double xc = mean ? centred<T>(x, mu[c]) : (double)x;
          const double* vc = vs + (size_t)c * k + j0;
#pragma unroll
          for (int j = 0; j < KT; ++j)
            if (j0 + j < k) acc[j] = fma(xc, vc[j], acc[j]);
        }
#pragma unroll
        for (int j = 0; j < KT; ++j)
          if (j0 + j < k) __stcs(out + (int64_t)(j0 + j) * ldo + r, acc[j]);
      }
    }
  }
}

template <typename T, int KT>
int launch_grouped_project(const T* X, int64_t ldx, const int64_t* offsets, const GroupWork& wl, int p,
                           const double* mean, const double* V, int k, double* out, int64_t ldo, cudaStream_t s) {
  auto kern = grouped_project_kernel<T, KT>;
  const size_t smem = (size_t)PW_WARPS * project_warp_doubles(p, k) * sizeof(double);
  const int grid = persistent_grid(kern, PW_WARPS * 32, smem, wl.n_items, 2);
  if (!grid) return 1;
  PDSB_CUDA_OK(cudaMemsetAsync(wl.queue, 0, sizeof(unsigned long long), s));
  kern<<<grid, PW_WARPS * 32, smem, s>>>(X, ldx, offsets, wl.rows, wl.group, wl.n_items, p, mean, V, k, out, ldo,
                                         wl.queue);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

}  // namespace

template <typename T>
int grouped_pca(const T* X, int64_t ldx, const T* mask, const int64_t* offsets, int64_t n_groups, int64_t n, int p,
                int center, double* mean, double* sigma, double* V, int* status, cudaStream_t s) {
  if (n_groups <= 0) return 0;
  if (p < 1 || p > GK_MAXP) { set_error("grouped pca: %d features; at most %d are supported", p, GK_MAXP); return 1; }
  if (!offsets || !sigma || !V || !status || (n > 0 && !X) || (center && !mean)) {
    set_error("grouped pca: null argument"); return 1;
  }
  DevBag bag(s);
  GroupWork wl;
  if (build_work_list(offsets, n_groups, n, ItemCount::EXACT, ItemMaps::ROWS_AND_GROUP, bag, wl, s)) return 1;
  const int64_t n_items = wl.n_items;
  // pass 1
  double* part1 = nullptr;
  if (center) {
    if (!(part1 = bag.alloc<double>((size_t)2 * p * n_items))) return 1;
    auto kern = pca_sums_kernel<T>;
    const int grid = persistent_grid(kern, SW_WARPS * 32, 0, n_items, 4);
    if (!grid) return 1;
    PDSB_CUDA_OK(cudaMemsetAsync(wl.queue, 0, sizeof(unsigned long long), s));
    kern<<<grid, SW_WARPS * 32, 0, s>>>(X, ldx, mask, wl.rows, n_items, p, part1, wl.queue);
    PDSB_LAUNCH_OK();
    count_launch();
  }
  // pass 2
  const int q1 = p + 1, nm = q1 * (q1 + 1) / 2;
  double* part2 = bag.alloc<double>((size_t)nm * n_items);
  if (!part2) return 1;
  {
    auto kern = pca_gram_kernel<T>;
    const size_t smem = (size_t)GW_WARPS * (32 * (q1 + 1) + GK_MAXP) * sizeof(double);
    const int grid = persistent_grid(kern, GW_WARPS * 32, smem, n_items, 1);
    if (!grid) return 1;
    PDSB_CUDA_OK(cudaMemsetAsync(wl.queue, 0, sizeof(unsigned long long), s));
    kern<<<grid, GW_WARPS * 32, smem, s>>>(X, ldx, mask, wl.rows, wl.group, wl.item_start, n_items, p, center, part1,
                                           mean, part2, wl.queue);
    PDSB_LAUNCH_OK();
    count_launch();
  }
  // pass 3
  const size_t esmem = eigen_smem(p);
  if (smem_opt_in(grouped_eigen_kernel, esmem)) return 1;
  grouped_eigen_kernel<<<(unsigned)n_groups, NT, esmem, s>>>(part2, wl.item_start, n_items, p, sigma, V, status);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

template <typename T>
int grouped_project(const T* X, int64_t ldx, const int64_t* offsets, int64_t n_groups, int64_t n, int p,
                    const double* mean, const double* V, int k, double* out, int64_t ldo, cudaStream_t s) {
  if (n_groups <= 0 || n <= 0) return 0;
  if (p < 1 || p > GK_MAXP) { set_error("grouped pca: %d features; at most %d are supported", p, GK_MAXP); return 1; }
  if (k < 1 || k > p) { set_error("grouped pca: k = %d outside [1, %d]", k, p); return 1; }
  if (!X || !offsets || !V || !out || ldo < n) { set_error("grouped pca: invalid projection arguments"); return 1; }
  DevBag bag(s);
  GroupWork wl;
  // each row's output depends only on its own values and its group, so the list need not be exact
  if (build_work_list(offsets, n_groups, n, ItemCount::BOUND, ItemMaps::ROWS_AND_GROUP, bag, wl, s)) return 1;
  if (k <= 1) return launch_grouped_project<T, 1>(X, ldx, offsets, wl, p, mean, V, k, out, ldo, s);
  if (k <= 2) return launch_grouped_project<T, 2>(X, ldx, offsets, wl, p, mean, V, k, out, ldo, s);
  if (k <= 4) return launch_grouped_project<T, 4>(X, ldx, offsets, wl, p, mean, V, k, out, ldo, s);
  return launch_grouped_project<T, 8>(X, ldx, offsets, wl, p, mean, V, k, out, ldo, s);   // chunks of 8 above 8
}

template int grouped_pca<float>(const float*, int64_t, const float*, const int64_t*, int64_t, int64_t, int, int, double*,
                                double*, double*, int*, cudaStream_t);
template int grouped_pca<double>(const double*, int64_t, const double*, const int64_t*, int64_t, int64_t, int, int,
                                 double*, double*, double*, int*, cudaStream_t);
template int grouped_project<float>(const float*, int64_t, const int64_t*, int64_t, int64_t, int, const double*,
                                    const double*, int, double*, int64_t, cudaStream_t);
template int grouped_project<double>(const double*, int64_t, const int64_t*, int64_t, int64_t, int, const double*,
                                     const double*, int, double*, int64_t, cudaStream_t);

}  // namespace pdsb
