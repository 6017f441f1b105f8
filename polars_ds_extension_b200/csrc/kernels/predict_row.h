// The per-row predict rule of K4 (predict_kernel, predict_frame_kernel) and K5's segmented predict
// (group_predict_kernel), and the row walk over one item of K5's work list.  All three go through these helpers, so a row's pred / resid are bit for bit the same
// whichever of them computes it:
//   beta rounded to T; the accumulator starts at the bias (0 without one); one fma per feature in ascending column
//   order; resid = y - pred; valid = the fit is OK and the row's mask is not 0.
// Each kernel keeps its own shared-memory layout of the [(p + 1) x t] beta table and its own loop over the slots.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <initializer_list>
#include <type_traits>

namespace pdsb {

// VEC consecutive rows of one column as one 16-byte access (VEC = 1: one element)
template <typename T, int VEC> struct VecT { using type = T; };
template <> struct VecT<float, 4> { using type = float4; };
template <> struct VecT<double, 2> { using type = double2; };

template <typename T, int VEC>
__device__ __forceinline__ void load_rows(const T* __restrict__ src, T (&v)[VEC]) {
  const typename VecT<T, VEC>::type t = *reinterpret_cast<const typename VecT<T, VEC>::type*>(src);
  memcpy(v, &t, sizeof(t));
}
template <typename T, int VEC>
__device__ __forceinline__ void store_rows(T* __restrict__ dst, const T (&v)[VEC]) {
  typename VecT<T, VEC>::type t;
  memcpy(&t, v, sizeof(t));
  *reinterpret_cast<typename VecT<T, VEC>::type*>(dst) = t;
}

// Slot r of the staged beta column of one fit (a target, or a group): feature r < p, slot p the bias (0 without one).
// The fit's p + add_bias coefficients start at beta[base]; a fit that is not OK stages 0.
template <typename T>
__device__ __forceinline__ T staged_beta(const double* __restrict__ beta, size_t base, int r, int p, int add_bias, bool ok) {
  double v = 0.0;
  if (ok) {
    if (r < p) v = beta[base + r];
    else if (add_bias) v = beta[base + p];
  }
  return (T)v;
}

// acc = pred of VEC rows from the staged column sb: sb[p], then fma(x_c, sb[c], acc) for c = 0 .. p-1.  load_x(c, xv)
// fills xv with the rows' values of feature c.  UNROLL > 0 unrolls the feature loop that many times; 0 leaves it to
// the compiler.
template <typename T, int VEC, int UNROLL = 0, typename LoadX>
__device__ __forceinline__ void predict_acc(const T* sb, int p, LoadX load_x, T (&acc)[VEC]) {
#pragma unroll
  for (int v = 0; v < VEC; ++v) acc[v] = sb[p];
  auto feature = [&](int c) {
    const T b = sb[c];
    T xv[VEC];
    load_x(c, xv);
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = fma(xv[v], b, acc[v]);
  };
  if constexpr (UNROLL > 0) {
#pragma unroll UNROLL
    for (int c = 0; c < p; ++c) feature(c);
  } else {
    for (int c = 0; c < p; ++c) feature(c);
  }
}

// Rows [r0, r1) of one work item, walked by the calling lane of a warp: rows [a0, a1) as whole VEC-row vectors from
// aligned addresses, VEC consecutive rows per lane and step, then the fewer than VEC rows on either side one per lane.
// body(row, std::integral_constant<int, V>()) handles rows [row, row + V).
template <int VEC, typename Body>
__device__ __forceinline__ void walk_item_rows(int64_t r0, int64_t r1, Body body) {
  const int lane = threadIdx.x & 31;
  const int64_t a0 = min((r0 + VEC - 1) / VEC * VEC, r1);
  const int64_t a1 = max(r1 / VEC * VEC, a0);
  for (int64_t r = a0 + (int64_t)lane * VEC; r < a1; r += 32 * VEC) body(r, std::integral_constant<int, VEC>());
  const int nh = (int)(a0 - r0);
  if (lane < nh) body(r0 + lane, std::integral_constant<int, 1>());
  else if (lane - nh < r1 - a1) body(a1 + (lane - nh), std::integral_constant<int, 1>());
}
// whether walk_item_rows may take 16-byte vectors of T: every non-null column 16-byte aligned, ld a multiple of VEC
template <typename T>
inline bool rows_vec_ok(int64_t ld, std::initializer_list<const void*> cols) {
  for (const void* c : cols)
    if (c && (reinterpret_cast<uintptr_t>(c) & 15) != 0) return false;
  return ld % (int64_t)(16 / sizeof(T)) == 0;
}

template <typename T>
__device__ __forceinline__ T resid_of(T y, T pred) { return y - pred; }

// m: the row's mask value (1 without a mask)
template <typename T>
__device__ __forceinline__ uint8_t valid_of(bool ok, T m) { return (ok && m != T(0)) ? 1 : 0; }

}  // namespace pdsb
