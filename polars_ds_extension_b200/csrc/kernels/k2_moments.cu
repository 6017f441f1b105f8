// K2 — which kernel forms the moments M = [X | Y | 1]' diag(w) [X | Y | 1] of a call, for every caller in the library.
// Each kernel's own test says which calls it can take (moments_small_supported, moments_wgmma_supported,
// moments_dmma_supported; the tile kernel takes any); the order below and the caller's precision contract say which of
// those runs.
#include "../common.h"
#include "kernels.h"
#include <type_traits>

namespace pdsb {

static thread_local int t_last_moments_path = 0;
static std::atomic<int> g_forced_path{0};

int last_moments_path() { return t_last_moments_path; }
void force_moments_path(int path) { g_forced_path.store(path); }

// f32 operands that the DMMA kernels do not take, copied to f64 columns ([X | Y | w | mask], 128-byte aligned) and routed
// as f64 data: the tile kernel would form f32 products
static int moments_widened(const float* X, int64_t ldx, const float* Y, int64_t ldy, const float* w, const float* mask,
                           int64_t n, int p, int t, double* M, cudaStream_t s) {
  const int64_t ld = (n + 31) & ~int64_t(31);
  double* Z = nullptr;
  if (dev_alloc((void**)&Z, (size_t)std::max<int64_t>(ld, 1) * (p + t + 2) * sizeof(double), s)) return 1;
  double* Yd = Z + (size_t)p * ld;
  double* wd = w ? Yd + (size_t)t * ld : nullptr;
  double* md = mask ? Yd + (size_t)(t + 1) * ld : nullptr;
  int rc = widen_f32(X, ldx, n, p, Z, ld, s);
  if (!rc) rc = widen_f32(Y, ldy, n, t, Yd, ld, s);
  if (!rc && w) rc = widen_f32(w, n, n, 1, wd, ld, s);
  if (!rc && mask) rc = widen_f32(mask, n, n, 1, md, ld, s);
  if (!rc) rc = moments<double>(MomentsPrecision::F64_PRODUCTS, Z, ld, Yd, ld, wd, md, n, p, t, M, s);
  dev_free(Z, s);
  return rc;
}

template <typename T>
int moments(MomentsPrecision prec, const T* X, int64_t ldx, const T* Y, int64_t ldy, const T* w, const T* mask, int64_t n,
            int p, int t, double* M, cudaStream_t s, int64_t bstride) {
  constexpr bool F32 = std::is_same<T, float>::value;
  const bool tf32 = F32 && prec == MomentsPrecision::TF32_ALLOWED;
  if (tf32) t_last_moments_path = 0;
  const int q1 = p + t + 1;
  if (p < 0 || t < 0 || q1 > 260) { set_error("moments: p+t+1=%d out of range (max 260)", q1); return 1; }
  if constexpr (F32) {
    if (tf32) {
      // pdsb_set_moments_path: 1 skips the register and wgmma kernels, 2 makes wgmma the only choice
      const int forced = g_forced_path.load();
      // few features, one target, no mask / weights: the register kernel is HBM-bound where the tensor-core kernel is
      // bound by its per-stage cost (path 3)
      if (!w && !mask && forced == 0 && n >= 65536 && moments_small_supported(n, p, t, bstride)) {
        const int rc = moments_small<float>(X, ldx, Y, n, p, M, s);
        if (rc == 0) t_last_moments_path = 3;
        return rc;
      }
      if (!w && forced != 1 && moments_wgmma_supported(X, ldx, Y, ldy, n, p, t, bstride)) {
        const int rc = moments_wgmma_f32(X, ldx, Y, ldy, mask, n, p, t, M, s, bstride);
        if (rc == 0) t_last_moments_path = 1;
        if (rc >= 0) return rc;   // -1: the tensor maps could not be encoded; the next kernel takes the call
      }
      if (forced == 2) { set_error("moments: tensor-core path forced but shape/alignment unsupported"); return 1; }
    } else if (prec == MomentsPrecision::F64_PRODUCTS && !moments_dmma_supported(X, ldx, Y, ldy, w, mask, n, p, t, bstride)) {
      return moments_widened(X, ldx, Y, ldy, w, mask, n, p, t, M, s);
    }
  }
  if (moments_dmma_supported(X, ldx, Y, ldy, w, mask, n, p, t, bstride)) return moments_dmma(X, ldx, Y, ldy, w, mask, n, p, t, M, s);
  return moments_tile(X, ldx, Y, ldy, w, mask, n, p, t, M, s, bstride);
}

template int moments<float>(MomentsPrecision, const float*, int64_t, const float*, int64_t, const float*, const float*,
                            int64_t, int, int, double*, cudaStream_t, int64_t);
template int moments<double>(MomentsPrecision, const double*, int64_t, const double*, int64_t, const double*,
                             const double*, int64_t, int, int, double*, cudaStream_t, int64_t);

}  // namespace pdsb
