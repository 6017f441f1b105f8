// K1 — pack: Arrow column chunks (any numeric dtype, optional validity bitmap, arbitrary bit offset) -> one
// column of the column-major device design matrix in the compute dtype T.
//
// Reference: series_to_slice_inner (/root/reference/src/utils/mod.rs:101-206: cast to the target dtype :140-144,
// null -> NaN :146-154) and the null policies of series_to_mat_for_lr (src/num_ext/linear_regression.rs:192-248:
// skip = AND of validities then filter, fill = fill_null(x) on the features).  Here "filter" is replaced by a row
// mask: a dropped row is written as all-zero and its entry in the ones/mask column is 0, so it contributes
// nothing to X'X, X'y or the row count, and no compaction pass (read+write of the whole frame) is needed.
// The reference's physical ones column (:180-182) is never materialised.
// When a column already has the compute dtype and no nulls the host layer skips this kernel entirely and DMAs the
// Arrow buffer straight into its slot (the reference's own fast path, utils/mod.rs:118-132, is the same idea).
#include "../common.h"
#include "kernels.h"

namespace pdsb {

namespace {

// Every source value is converted straight to T with one rounding, as the reference's cast to the compute dtype does
// (polars `cast(Float32)` / `cast(Float64)`): (float)(long long) is cvt.rn.f32.s64.  Going through double first would
// round an integer of more than 53 significant bits twice in f32 mode.
template <typename T, typename S> __device__ __forceinline__ T load_as(const void* src, int64_t i) {
  return (T)reinterpret_cast<const S*>(src)[i];
}

template <typename T> __device__ __forceinline__ T load_any(const void* src, int dtype, int64_t i) {
  switch (dtype) {
    case PDSB_F32: return load_as<T, float>(src, i);
    case PDSB_F64: return load_as<T, double>(src, i);
    case PDSB_I8: return load_as<T, int8_t>(src, i);
    case PDSB_U8: return load_as<T, uint8_t>(src, i);
    case PDSB_I16: return load_as<T, int16_t>(src, i);
    case PDSB_U16: return load_as<T, uint16_t>(src, i);
    case PDSB_I32: return load_as<T, int32_t>(src, i);
    case PDSB_U32: return load_as<T, uint32_t>(src, i);
    case PDSB_I64: return load_as<T, long long>(src, i);
    case PDSB_U64: return load_as<T, unsigned long long>(src, i);
    case PDSB_BOOL: {
      const uint8_t* b = reinterpret_cast<const uint8_t*>(src);
      return (T)((b[i >> 3] >> (i & 7)) & 1);
    }
  }
  return T(0);
}

__device__ __forceinline__ bool bit_at(const uint8_t* bm, int64_t i) { return (bm[i >> 3] >> (i & 7)) & 1; }

template <typename T>
__global__ void pack_kernel(const void* __restrict__ src, int dtype, const uint8_t* __restrict__ validity,
                            int64_t bit_offset, int64_t len, T* __restrict__ dst, int mode, T fill,
                            int64_t bstride, int64_t row0) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (int64_t)gridDim.x * blockDim.x) {
    T v;
    // `src` is uploaded already offset to the chunk's first element for byte-addressable types; BOOL keeps the
    // bit offset because it is bit-packed.
    if (dtype == PDSB_BOOL) v = load_any<T>(src, dtype, i + bit_offset);
    else v = load_any<T>(src, dtype, i);
    if (validity && !bit_at(validity, i + bit_offset)) {
      if (mode == 0) v = (T)nan("");
      else if (mode == 1) v = fill;
      else v = T(0);
    }
    if (bstride) { const int64_t r = row0 + i; dst[(r >> 7) * bstride + (r & 127)] = v; }   // frame column
    else dst[i] = v;
  }
}

template <typename T>
__global__ void to_frame_kernel(const T* __restrict__ src, int64_t ld, int64_t n, int ncols, T* __restrict__ frame) {
  // scalar fallback (unaligned sources): one thread per (row, column), coalesced on both sides
  const int64_t nb = (n + 127) >> 7;
  const int64_t total = nb * 128 * ncols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t blk = i / ((int64_t)ncols * 128);
    const int64_t rem = i - blk * ncols * 128;
    const int c = (int)(rem >> 7);
    const int64_t row = (blk << 7) + (rem & 127);
    frame[i] = row < n ? src[(int64_t)c * ld + row] : T(0);
  }
}

// Column-major -> row-blocked frame, 16 bytes per lane.  A (block, column) segment is 128 rows = 512 B (f32) / 1 KB
// (f64) and is CONTIGUOUS on both sides, so this is a gather of whole segments, not a transpose: one warp moves one
// 512-byte piece per task (fully coalesced read and write), TPW consecutive tasks per trip with every load issued
// before the first store (TPW x 16 B in flight per lane).  Consecutive tasks are consecutive in the DESTINATION.
// Round 1's one-element-per-thread kernel reached 45 % of the HBM peak (8.9 ms for 26.4 GB, launches_r01_summary.csv).
template <typename T, int TPW>
__global__ void __launch_bounds__(256)
to_frame_vec_kernel(const T* __restrict__ src, int64_t ld, int64_t n, int ncols, T* __restrict__ frame) {
  constexpr int EPU = 16 / (int)sizeof(T);                // elements per 16-byte unit
  constexpr int PARTS = 128 / (32 * EPU);                 // 32-lane pieces per segment (1 for f32, 2 for f64)
  const int64_t nb = (n + 127) >> 7;
  const int64_t tasks = nb * ncols * PARTS;
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t per_blk = (int64_t)ncols * PARTS;
  for (int64_t t0 = warp0 * TPW; t0 < tasks; t0 += nwarps * TPW) {
    uint4 v[TPW];
#pragma unroll
    for (int k = 0; k < TPW; ++k) {
      const int64_t t = t0 + k;
      v[k] = make_uint4(0, 0, 0, 0);
      if (t < tasks) {
        const int64_t blk = t / per_blk;
        const int rem = (int)(t - blk * per_blk);
        const int c = rem / PARTS, part = rem - c * PARTS;
        const int64_t row = (blk << 7) + (int64_t)(part * 32 + lane) * EPU;
        const T* sp = src + (int64_t)c * ld + row;
        if (row + EPU <= n) v[k] = __ldcs(reinterpret_cast<const uint4*>(sp));     // streamed once: evict-first
        else {
          T e[EPU];
#pragma unroll
          for (int j = 0; j < EPU; ++j) e[j] = (row + j < n) ? sp[j] : T(0);
          v[k] = *reinterpret_cast<const uint4*>(e);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < TPW; ++k) {
      const int64_t t = t0 + k;
      if (t < tasks) reinterpret_cast<uint4*>(frame)[t * 32 + lane] = v[k];
    }
  }
}

template <typename T>
__global__ void and_validity_kernel(const uint8_t* __restrict__ validity, int64_t bit_offset, int64_t len,
                                    T* __restrict__ rowmask) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (int64_t)gridDim.x * blockDim.x)
    if (!bit_at(validity, i + bit_offset)) rowmask[i] = T(0);
}

template <typename T>
__global__ void fill_kernel(T* __restrict__ dst, int64_t len, T v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (int64_t)gridDim.x * blockDim.x) dst[i] = v;
}

template <typename T>
__global__ void zero_masked_kernel(T* __restrict__ col, const T* __restrict__ rowmask, int64_t len) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (int64_t)gridDim.x * blockDim.x)
    if (rowmask[i] == T(0)) col[i] = T(0);
}

// SUM = false: count of nonzeros; SUM = true: sum of the values divided by len (the mean)
template <typename T, bool SUM = false>
__global__ void count_mask_kernel(const T* __restrict__ rowmask, int64_t len, double* __restrict__ out) {
  // single block, deterministic
  __shared__ double red[32];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < len; i += blockDim.x) {
    if constexpr (SUM) s += (double)rowmask[i];
    else s += (rowmask[i] != T(0)) ? 1.0 : 0.0;
  }
  for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) v += red[i];
    *out = SUM ? v / (double)len : v;
  }
}

inline int grid_for(int64_t len) {
  int64_t g = ceil_div(len > 0 ? len : 1, 256);
  int64_t cap = (int64_t)sm_count() * 16;
  return (int)(g < cap ? g : cap);
}

}  // namespace

#define PDSB_AFTER_LAUNCH(name)                                                        \
  do {                                                                                 \
    cudaError_t e = cudaGetLastError();                                                \
    count_launch();                                                                    \
    if (e != cudaSuccess) { set_error(name " launch failed: %s", cudaGetErrorString(e)); return 1; } \
  } while (0)

template <typename T>
int pack_chunk(const void* src, int src_dtype, const uint8_t* validity, int64_t bit_offset, int64_t len,
               T* dst, int mode, T fill, cudaStream_t s, int64_t bstride, int64_t row0) {
  if (len <= 0) return 0;
  pack_kernel<T><<<grid_for(len), 256, 0, s>>>(src, src_dtype, validity, bit_offset, len, dst, mode, fill, bstride, row0);
  PDSB_AFTER_LAUNCH("pack");
  return 0;
}
template <typename T>
int to_frame(const T* src, int64_t ld, int64_t n, int ncols, T* frame, cudaStream_t s) {
  if (n <= 0) return 0;
  const int64_t total = ((n + 127) >> 7) * 128 * ncols;
  const bool aligned = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(frame)) & 15) == 0 &&
                       ((ld * (int64_t)sizeof(T)) & 15) == 0;
  if (aligned) {
    constexpr int TPW = 8;
    const int64_t tasks = total * (int64_t)sizeof(T) / 512;
    int64_t g = ceil_div(ceil_div(tasks, TPW), 8);                 // 8 warps per block
    const int64_t cap = (int64_t)sm_count() * 8;                   // 2048 threads per SM resident
    to_frame_vec_kernel<T, TPW><<<(int)(g < cap ? (g > 0 ? g : 1) : cap), 256, 0, s>>>(src, ld, n, ncols, frame);
  } else {
    to_frame_kernel<T><<<grid_for(total), 256, 0, s>>>(src, ld, n, ncols, frame);
  }
  PDSB_AFTER_LAUNCH("to_frame");
  return 0;
}
template <typename T>
int and_validity(const uint8_t* validity, int64_t bit_offset, int64_t len, T* rowmask, cudaStream_t s) {
  if (len <= 0) return 0;
  and_validity_kernel<T><<<grid_for(len), 256, 0, s>>>(validity, bit_offset, len, rowmask);
  PDSB_AFTER_LAUNCH("and_validity");
  return 0;
}
template <typename T>
int fill_value(T* dst, int64_t len, T v, cudaStream_t s) {
  if (len <= 0) return 0;
  fill_kernel<T><<<grid_for(len), 256, 0, s>>>(dst, len, v);
  PDSB_AFTER_LAUNCH("fill");
  return 0;
}
template <typename T>
int zero_masked(T* col, const T* rowmask, int64_t len, cudaStream_t s) {
  if (len <= 0) return 0;
  zero_masked_kernel<T><<<grid_for(len), 256, 0, s>>>(col, rowmask, len);
  PDSB_AFTER_LAUNCH("zero_masked");
  return 0;
}
template <typename T>
int count_mask(const T* rowmask, int64_t len, double* out, cudaStream_t s) {
  count_mask_kernel<T><<<1, 1024, 0, s>>>(rowmask, len, out);
  PDSB_AFTER_LAUNCH("count_mask");
  return 0;
}
template <typename T>
int mean_values(const T* v, int64_t len, double* out, cudaStream_t s) {
  count_mask_kernel<T, true><<<1, 1024, 0, s>>>(v, len, out);
  PDSB_AFTER_LAUNCH("mean_values");
  return 0;
}

#define INST(T)                                                                                              \
  template int pack_chunk<T>(const void*, int, const uint8_t*, int64_t, int64_t, T*, int, T, cudaStream_t, int64_t, int64_t); \
  template int to_frame<T>(const T*, int64_t, int64_t, int, T*, cudaStream_t);                                 \
  template int and_validity<T>(const uint8_t*, int64_t, int64_t, T*, cudaStream_t);                          \
  template int fill_value<T>(T*, int64_t, T, cudaStream_t);                                                  \
  template int zero_masked<T>(T*, const T*, int64_t, cudaStream_t);                                          \
  template int count_mask<T>(const T*, int64_t, double*, cudaStream_t);
INST(float)
INST(double)
template int mean_values<double>(const double*, int64_t, double*, cudaStream_t);

}  // namespace pdsb
