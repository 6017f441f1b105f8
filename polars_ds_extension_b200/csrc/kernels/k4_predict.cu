// K4 — streaming predict / residual / SSR:  pred = [X|1] beta, resid = Y - pred.
//
// Reference: `let pred = x * &coeffs; let resid = y - &pred;` (/root/reference/src/num_ext/linear_regression.rs:
// 782-785, 635-636) plus the mask re-insertion loop (:790-812) and the residual sums the report needs (:863-875,
// 1036-1038).  One coalesced, vectorised pass: each thread owns VEC consecutive rows (16-byte loads per column
// because X is column-major), beta lives in shared memory, pred and resid are written once; the optional SSR is
// reduced in f64 per block and summed in a fixed order by a second tiny kernel (bit-reproducible).
// HBM-bound: algorithmic bytes per row = (p + t) * s read + 2 t * s written.
// Row-blocked frames (the resident f32 layout) go through predict_frame_kernel below: same arithmetic order, so the
// same pred / resid bit for bit, but fed by a bulk-copy ring instead of per-thread loads.
#include "../common.h"
#include "kernels.h"
#include "mbarrier.h"

namespace pdsb {

namespace {

template <typename T, int VEC> struct VecT;
template <> struct VecT<float, 4> { using type = float4; };
template <> struct VecT<double, 2> { using type = double2; };
template <> struct VecT<float, 1> { using type = float; };
template <> struct VecT<double, 1> { using type = double; };

template <typename T, int VEC>
__global__ void __launch_bounds__(256)
predict_kernel(const T* __restrict__ X, int64_t ldx, const T* __restrict__ Y, int64_t ldy,
               const T* __restrict__ w, const T* __restrict__ mask, int64_t n, int p, int t, int add_bias,
               const double* __restrict__ beta, const int* __restrict__ status, T* __restrict__ pred,
               T* __restrict__ resid, int64_t ldo, uint8_t* __restrict__ valid, double* __restrict__ ssr_part) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sb = reinterpret_cast<T*>(smem_raw);  // [(p+1) x t]
  const int q = p + (add_bias ? 1 : 0);
  const bool gated = status && (*status != 0);
  for (int i = threadIdx.x; i < (p + 1) * t; i += blockDim.x) {
    int r = i % (p + 1), k = i / (p + 1);
    double v = 0.0;
    if (!gated) {
      if (r < p) v = beta[(size_t)k * q + r];
      else if (add_bias) v = beta[(size_t)k * q + p];
    }
    sb[i] = (T)v;
  }
  __syncthreads();
  using V = typename VecT<T, VEC>::type;
  double ssr_loc[4] = {0.0, 0.0, 0.0, 0.0};   // sum e^2   (up to 4 targets)
  double wssr_loc[4] = {0.0, 0.0, 0.0, 0.0};  // sum w e^2
  const int64_t nvec = (n + VEC - 1) / VEC;
  for (int64_t iv = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; iv < nvec; iv += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = iv * VEC;
    const bool full = (row + VEC <= n);
    for (int k0 = 0; k0 < t; ++k0) {
      T acc[VEC];
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc[v] = sb[k0 * (p + 1) + p];
      for (int c = 0; c < p; ++c) {
        const T b = sb[k0 * (p + 1) + c];
        const T* src = X + (int64_t)c * ldx + row;
        T xv[VEC];
        if (full) { V tmp = *reinterpret_cast<const V*>(src); memcpy(xv, &tmp, sizeof(V)); }
        else {
#pragma unroll
          for (int v = 0; v < VEC; ++v) xv[v] = (row + v < n) ? src[v] : T(0);
        }
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc[v] = fma(xv[v], b, acc[v]);
      }
      T yv[VEC], rv[VEC], mv[VEC], wv[VEC];
      const T* ys = Y + (int64_t)k0 * ldy + row;
#pragma unroll
      for (int v = 0; v < VEC; ++v) {
        bool in = row + v < n;
        yv[v] = in ? ys[v] : T(0);
        mv[v] = (in && mask) ? mask[row + v] : T(1);
        wv[v] = (in && w) ? w[row + v] : T(1);
        rv[v] = yv[v] - acc[v];
      }
      double sl = 0.0, swl = 0.0;
#pragma unroll
      for (int v = 0; v < VEC; ++v)
        if (row + v < n && mv[v] != T(0)) {
          double e2 = (double)rv[v] * (double)rv[v];
          sl += e2; swl += (double)wv[v] * e2;
        }
      if (k0 < 4) { ssr_loc[k0] += sl; wssr_loc[k0] += swl; }
      T* pd = pred + (int64_t)k0 * ldo + row;
      T* rd = resid + (int64_t)k0 * ldo + row;
      if (full) {
        V tp, tr; memcpy(&tp, acc, sizeof(V)); memcpy(&tr, rv, sizeof(V));
        *reinterpret_cast<V*>(pd) = tp; *reinterpret_cast<V*>(rd) = tr;
      } else {
#pragma unroll
        for (int v = 0; v < VEC; ++v) if (row + v < n) { pd[v] = acc[v]; rd[v] = rv[v]; }
      }
      if (valid && k0 == 0) {
#pragma unroll
        for (int v = 0; v < VEC; ++v)
          if (row + v < n) valid[row + v] = (!gated && mv[v] != T(0)) ? 1 : 0;
      }
    }
  }
  if (ssr_part) {
    __shared__ double red[8][8];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int k = 0; k < 8; ++k) {
      double v = (k < 4) ? ssr_loc[k] : wssr_loc[k - 4];
      for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if (lane == 0) red[k][wid] = v;
    }
    __syncthreads();
    if (threadIdx.x < 8) {
      double v = 0.0;
      for (int i = 0; i < (int)(blockDim.x >> 5); ++i) v += red[threadIdx.x][i];
      ssr_part[(size_t)blockIdx.x * 8 + threadIdx.x] = v;
    }
  }
}

// ------------------------------------------------------------------------------ K4 on the row-blocked frame ----------
// A 128-row block of the frame is one contiguous run of ncols x 512 bytes, so the frame kernel streams it the way the
// moments kernel does: a persistent grid (one CTA per SM, blocks dealt round-robin so the CTAs read adjacent DRAM), one
// producer lane that lands each block's X and Y columns in a shared-memory ring with 1-D bulk copies, and consumer
// warpgroups that take alternate ring slots, one thread per row.  Column c of a slot sits at tile[c * 128 + row]:
// conflict-free reads, and every warp writes pred / resid as contiguous runs.
constexpr int FR_NCW = 2;                              // consumer warpgroups
constexpr int FR_THREADS = FR_NCW * 128 + 32;          // + the producer warp
constexpr size_t FR_RING_BYTES = 200 * 1024;           // bytes in flight per SM that keep HBM busy

struct FrameArgs {
  const float* frame;
  int64_t n, nblocks, bstride;   // bstride = ncols * 128 elements per block
  int p, t, add_bias;
  int col0;                      // first frame column of the one copy (joined) or of X
  int ycol, joined;              // joined: X and Y are adjacent, one copy of (p + t) x 512 bytes carries both
  int xoff, yoff;                // slot column of the first feature / target
  int ring, ncw;                 // ring slots (a multiple of ncw) and consumer warpgroups in use
  uint32_t slot_bytes;
};

__global__ void __launch_bounds__(FR_THREADS, 1)
predict_frame_kernel(const FrameArgs a, const float* __restrict__ mask, const double* __restrict__ beta,
                     const int* __restrict__ status, float* __restrict__ pred, float* __restrict__ resid, int64_t ldo,
                     uint8_t* __restrict__ valid, double* __restrict__ ssr_part) {
  extern __shared__ __align__(128) unsigned char fr_smem[];
  // layout: ring slots | beta [(p+1) x t] f32 | full[ring], empty[ring]
  const int p = a.p, t = a.t;
  float* sb = reinterpret_cast<float*>(fr_smem + (size_t)a.ring * a.slot_bytes);
  uint64_t* full = reinterpret_cast<uint64_t*>(fr_smem + (((size_t)a.ring * a.slot_bytes + (size_t)(p + 1) * t * 4 + 7) & ~(size_t)7));
  uint64_t* empty = full + a.ring;
  const int q = p + (a.add_bias ? 1 : 0);
  const bool gated = status && (*status != 0);
  for (int i = threadIdx.x; i < (p + 1) * t; i += blockDim.x) {
    int r = i % (p + 1), k = i / (p + 1);
    double v = 0.0;
    if (!gated) {
      if (r < p) v = beta[(size_t)k * q + r];
      else if (a.add_bias) v = beta[(size_t)k * q + p];
    }
    sb[i] = (float)v;
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < a.ring; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t my_blocks = a.nblocks > (int64_t)blockIdx.x ? (uint32_t)((a.nblocks - 1 - blockIdx.x) / gridDim.x + 1) : 0u;
  double ssr_loc[4] = {0.0, 0.0, 0.0, 0.0};   // sum e^2 (up to 4 targets; the frame carries no weights)
  if (warp < 4 * FR_NCW) {
    // =============================== consumers: warpgroup wg takes slots wg, wg + ncw, ... (always the same slots,
    // because ring is a multiple of ncw: a slot's parity waits never run a phase ahead)
    const int wg = warp >> 2, r = threadIdx.x & 127;
    for (uint32_t i = wg; wg < a.ncw && i < my_blocks; i += a.ncw) {
      const uint32_t s = i % a.ring;
      const int64_t row = ((int64_t)i * gridDim.x + blockIdx.x) * FRAME_ROWS + r;
      const bool in = row < a.n;
      const float mv = (in && mask) ? mask[row] : 1.0f;
      mbar_wait(&full[s], (i / a.ring) & 1);
      const float* tile = reinterpret_cast<const float*>(fr_smem + (size_t)s * a.slot_bytes) + r;
      const float* xs = tile + a.xoff * FRAME_ROWS;
      for (int k0 = 0; k0 < t; ++k0) {
        // the order of predict_kernel: bias (or 0), then one fma per feature in ascending order, then y - pred
        const float* bk = sb + k0 * (p + 1);
        float acc = bk[p];
#pragma unroll 8
        for (int c = 0; c < p; ++c) acc = fmaf(xs[c * FRAME_ROWS], bk[c], acc);
        const float rv = tile[(a.yoff + k0) * FRAME_ROWS] - acc;
        if (ssr_part && in && mv != 0.0f) {
          const double e2 = (double)rv * (double)rv;
#pragma unroll
          for (int j = 0; j < 4; ++j) if (j == k0) ssr_loc[j] += e2;
        }
        if (in) { pred[(int64_t)k0 * ldo + row] = acc; resid[(int64_t)k0 * ldo + row] = rv; }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);               // this warp's reads of the slot are complete
      if (valid && in) valid[row] = (!gated && mv != 0.0f) ? 1 : 0;
    }
  } else {
    // =============================== producer (warp-uniform loop, one elected lane issues) ==========================
    for (uint32_t i = 0; i < my_blocks; ++i) {
      const uint32_t s = i % a.ring;
      mbar_wait(&empty[s], ((i / a.ring) & 1) ^ 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(&full[s], a.slot_bytes);
        const float* blk = a.frame + ((int64_t)i * gridDim.x + blockIdx.x) * a.bstride;
        unsigned char* dst = fr_smem + (size_t)s * a.slot_bytes;
        if (a.joined) {
          bulk_load(dst, blk + (size_t)a.col0 * FRAME_ROWS, a.slot_bytes, &full[s]);
        } else {
          bulk_load(dst, blk + (size_t)a.col0 * FRAME_ROWS, (uint32_t)p * FRAME_ROWS * 4, &full[s]);
          bulk_load(dst + (size_t)p * FRAME_ROWS * 4, blk + (size_t)a.ycol * FRAME_ROWS, (uint32_t)t * FRAME_ROWS * 4, &full[s]);
        }
      }
      __syncwarp();
    }
  }
  if (ssr_part) {
    // fixed order: xor tree inside each warp, then the consumer warps in index order (bit-reproducible run to run)
    __shared__ double red[4 * FR_NCW][4];
    if (warp < 4 * FR_NCW) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        double v = ssr_loc[k];
        for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0) red[warp][k] = v;
      }
    }
    __syncthreads();
    if (threadIdx.x < 8) {
      double v = 0.0;
      for (int i = 0; i < 4 * FR_NCW; ++i) v += red[i][threadIdx.x & 3];
      ssr_part[(size_t)blockIdx.x * 8 + threadIdx.x] = v;     // slots 4..7 (weighted SSR) equal 0..3: no weights
    }
  }
}

__global__ void ssr_reduce_kernel(const double* __restrict__ part, int nblocks, double* __restrict__ ssr) {
  int k = threadIdx.x;
  if (k >= 8) return;
  double s = 0.0;
  for (int b = 0; b < nblocks; ++b) s += part[(size_t)b * 8 + k];
  ssr[k] = s;
}

}  // namespace

template <typename T>
int predict_resid(const T* X, int64_t ldx, const T* Y, int64_t ldy, const T* w, const T* mask, int64_t n,
                  int p, int t, int add_bias, const double* beta, const int* status, T* pred, T* resid,
                  int64_t ldo, uint8_t* valid, double* ssr, cudaStream_t s) {
  if (n <= 0) return 0;
  if (ssr && t > 4) { set_error("predict: ssr supports at most 4 targets"); return 1; }
  constexpr int VEC = sizeof(T) == 4 ? 4 : 2;
  auto aligned = [&](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  bool vec_ok = aligned(X) && aligned(pred) && aligned(resid) && (ldx % VEC == 0) && (ldo % VEC == 0);
  const int64_t work = vec_ok ? ceil_div(n, VEC) : n;
  int grid = (int)std::min<int64_t>(ceil_div(work, 256), (int64_t)sm_count() * 8);
  if (grid < 1) grid = 1;
  size_t smem = (size_t)(p + 1) * t * sizeof(T);
  double* part = nullptr;
  if (ssr) { if (dev_alloc((void**)&part, (size_t)grid * 8 * sizeof(double), s)) return 1; }
  if (vec_ok) {
    auto k = predict_kernel<T, VEC>;
    if (smem > 48 * 1024) PDSB_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<grid, 256, smem, s>>>(X, ldx, Y, ldy, w, mask, n, p, t, add_bias, beta, status, pred, resid, ldo, valid, part);
  } else {
    auto k = predict_kernel<T, 1>;
    if (smem > 48 * 1024) PDSB_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<grid, 256, smem, s>>>(X, ldx, Y, ldy, w, mask, n, p, t, add_bias, beta, status, pred, resid, ldo, valid, part);
  }
  cudaError_t e = cudaGetLastError();
  count_launch();
  if (e == cudaSuccess && ssr) {
    ssr_reduce_kernel<<<1, 32, 0, s>>>(part, grid, ssr);
    e = cudaGetLastError();
    count_launch();
  }
  if (part) dev_free(part, s);
  if (e != cudaSuccess) { set_error("predict launch failed: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

template int predict_resid<float>(const float*, int64_t, const float*, int64_t, const float*, const float*,
                                  int64_t, int, int, int, const double*, const int*, float*, float*, int64_t,
                                  uint8_t*, double*, cudaStream_t);
template int predict_resid<double>(const double*, int64_t, const double*, int64_t, const double*, const double*,
                                   int64_t, int, int, int, const double*, const int*, double*, double*, int64_t,
                                   uint8_t*, double*, cudaStream_t);

int predict_frame_f32(const float* frame, int64_t n, int ncols, int xcol, int p, int ycol, int t, int add_bias,
                      const float* mask, const double* beta, const int* status, float* pred, float* resid, int64_t ldo,
                      uint8_t* valid, double* ssr, cudaStream_t s) {
  if (n <= 0 || t <= 0) return 0;
  if (ssr && t > 4) { set_error("predict: ssr supports at most 4 targets"); return 1; }
  if (p < 0 || xcol < 0 || ycol < 0 || xcol + p > ncols || ycol + t > ncols) { set_error("predict_frame: columns out of range"); return 1; }
  if (reinterpret_cast<uintptr_t>(frame) & 15) { set_error("predict_frame: the frame must be 16-byte aligned"); return 1; }
  FrameArgs a;
  a.frame = frame; a.n = n; a.nblocks = ceil_div(n, FRAME_ROWS); a.bstride = (int64_t)ncols * FRAME_ROWS;
  a.p = p; a.t = t; a.add_bias = add_bias; a.ycol = ycol;
  // one copy when the targets follow the features or the features follow the targets
  if (ycol == xcol + p) { a.joined = 1; a.col0 = xcol; a.xoff = 0; a.yoff = p; }
  else if (xcol == ycol + t) { a.joined = 1; a.col0 = ycol; a.xoff = t; a.yoff = 0; }
  else { a.joined = 0; a.col0 = xcol; a.xoff = 0; a.yoff = p; }
  a.slot_bytes = (uint32_t)(p + t) * FRAME_ROWS * sizeof(float);
  const size_t tail = (((size_t)(p + 1) * t * sizeof(float) + 7) & ~(size_t)7);      // beta, then the barriers
  const size_t smem_max = 227 * 1024 - 1024;                                          // sm_90 block limit, less static
  int ring = (int)std::min<size_t>(FR_RING_BYTES / a.slot_bytes, 64);
  ring -= ring % FR_NCW;
  if (ring >= FR_NCW) a.ncw = FR_NCW;
  else { ring = 1; a.ncw = 1; }                                                     // wide frames: one slot, one warpgroup
  a.ring = ring;
  const size_t smem = (size_t)ring * a.slot_bytes + tail + 2 * sizeof(uint64_t) * ring;
  if (smem > smem_max) { set_error("predict_frame: p + t = %d columns do not fit one shared-memory slot", p + t); return 1; }
  int grid = (int)std::min<int64_t>(a.nblocks, (int64_t)sm_count());
  PDSB_CUDA_OK(cudaFuncSetAttribute(predict_frame_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  double* part = nullptr;
  if (ssr) { if (dev_alloc((void**)&part, (size_t)grid * 8 * sizeof(double), s)) return 1; }
  predict_frame_kernel<<<grid, FR_THREADS, smem, s>>>(a, mask, beta, status, pred, resid, ldo, valid, part);
  cudaError_t e = cudaGetLastError();
  count_launch();
  if (e == cudaSuccess && ssr) {
    ssr_reduce_kernel<<<1, 32, 0, s>>>(part, grid, ssr);
    e = cudaGetLastError();
    count_launch();
  }
  if (part) dev_free(part, s);
  if (e != cudaSuccess) { set_error("predict_frame launch failed: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

}  // namespace pdsb
