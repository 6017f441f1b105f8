// K13 — PCA: singular values and right singular vectors of X from its Gram matrix, and the projection X V[:, :k].
//
// Replaces the dense faer SVD of the whole n x p matrix that pl_singular_values / pl_pca / pl_principal_components run
// on the CPU (/root/reference/src/num_ext/pca.rs:39-182).  The right singular vectors of X are the eigenvectors of
// G = X'X and the singular values the square roots of its eigenvalues, so
//   * pass 1 is K2a's moments kernel (one read of X, f64 products and sums);
//   * pca_eigen_kernel: one CTA, K3's parallel-ordered Jacobi on G, stable descending sort, sign rule, sigma;
//   * pca_project_kernel (principal_components only): out[:, j] = X V[:, j], one more read of X.
// Accuracy (DESIGN.md "K13 PCA"): sigma_i to ~eps (sigma_1 / sigma_i)^2 relative, against eps sigma_1 / sigma_i for an SVD
// of X; values below ~sqrt(eps) sigma_1 are not resolved.
//
// ptxas (-Xptxas -v, sm_90a, CUDA 12.9), registers: pca_eigen_kernel 64 (__launch_bounds__(256, 1): at the default bound
// ptxas kept 40 and spilled 16 bytes around the division subroutines); pca_project_kernel<T, KT> for KT = 1 / 2 / 4 / 8 /
// 16 / 32 outputs per thread: f64 32 / 32 / 40 / 52 / 68 / 120, f32 31 / 32 / 40 / 48 / 66 / 122; widen_kernel 30.
// No stack frame and no spill in any of them.
#include "../common.h"
#include "kernels.h"
#include <cmath>

namespace pdsb {

namespace {

constexpr int NT = 256;

}  // namespace
}  // namespace pdsb

#include "jacobi.h"

namespace pdsb {
namespace {

// status[0]: PDSB_PCA_OK or PDSB_PCA_NONFINITE; status[1]: dim = min(rows counted in the moments, p)
__global__ void __launch_bounds__(NT, 1)
pca_eigen_kernel(const double* __restrict__ M, int q1, int p, double* Ag, double* Vu, double* cs, int* perm,
                 double* __restrict__ sigma, double* __restrict__ V, int* __restrict__ status, int use_smem) {
  extern __shared__ double eig_smem[];
  double* A = use_smem ? eig_smem : Ag;
  const int tid = threadIdx.x;
  __shared__ int sh_bad;
  if (tid == 0) sh_bad = 0;
  __syncthreads();
  for (int idx = tid; idx < p * p; idx += NT) {
    const int i = idx % p, j = idx / p;
    const double v = M[(size_t)i * q1 + j];
    if (!isfinite(v)) sh_bad = 1;
    A[idx] = v;
  }
  __syncthreads();
  if (tid == 0) {
    const double count = M[(size_t)(q1 - 1) * q1 + (q1 - 1)];
    status[0] = sh_bad ? PDSB_PCA_NONFINITE : PDSB_PCA_OK;
    status[1] = (int)fmin(fmax(rint(count), 0.0), (double)p);
  }
  if (sh_bad) return;
  jacobi_eigen(A, Vu, p, cs);
  // stable descending order: rank of i = #{j : lam_j > lam_i} + #{j < i : lam_j == lam_i}
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
  // column r of V = eigenvector perm[r], signed so that its largest-magnitude entry (the first one on ties) is positive:
  // sklearn's svd_flip(u_based_decision=False), the rule behind PCA.components_
  for (int r = tid; r < p; r += NT) {
    const int c = perm[r];
    int best = 0; double bmax = -1.0;
    for (int i = 0; i < p; ++i) { const double a = fabs(at(Vu, p, i, c)); if (a > bmax) { bmax = a; best = i; } }
    const double sgn = at(Vu, p, best, c) < 0.0 ? -1.0 : 1.0;
    for (int i = 0; i < p; ++i) V[i + (size_t)r * p] = sgn * at(Vu, p, i, c);
    sigma[r] = sqrt(fmax(at(A, p, c, c), 0.0));
  }
}

// out[j * ldo + r] = sum_c X[c * ldx + r] * V[c + (k0 + j) * p] for the KT columns k0 .. k0 + KT - 1 of this grid row
// (j < k - k0).  One row per thread and iteration; V's slice in shared memory ([p][KT], read as broadcasts).
template <typename T, int KT>
__global__ void __launch_bounds__(256)
pca_project_kernel(const T* __restrict__ X, int64_t ldx, int64_t n, int p, const double* __restrict__ V, int k,
                   double* __restrict__ out, int64_t ldo) {
  extern __shared__ __align__(16) double vs[];
  const int k0 = blockIdx.y * KT;
  const int kn = min(KT, k - k0);
  for (int e = threadIdx.x; e < p * KT; e += blockDim.x) {
    const int c = e / KT, j = e % KT;
    vs[e] = j < kn ? V[c + (size_t)(k0 + j) * p] : 0.0;
  }
  __syncthreads();
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    double acc[KT];
#pragma unroll
    for (int j = 0; j < KT; ++j) acc[j] = 0.0;
    const T* xr = X + r;
#pragma unroll 4
    for (int c = 0; c < p; ++c) {
      const double x = (double)__ldcs(xr + (int64_t)c * ldx);
      const double* vc = vs + c * KT;
      if constexpr (KT == 1) {
        acc[0] = fma(x, vc[0], acc[0]);
      } else {
#pragma unroll
        for (int j = 0; j < KT; j += 2) {
          const double2 v2 = *reinterpret_cast<const double2*>(vc + j);
          acc[j] = fma(x, v2.x, acc[j]);
          acc[j + 1] = fma(x, v2.y, acc[j + 1]);
        }
      }
    }
    double* o = out + (int64_t)k0 * ldo + r;
#pragma unroll
    for (int j = 0; j < KT; ++j)
      if (j < kn) __stcs(o + (int64_t)j * ldo, acc[j]);
  }
}

__global__ void widen_kernel(const float* __restrict__ X, int64_t ldx, int64_t n, int p, double* __restrict__ Y,
                             int64_t ldy) {
  const int64_t total = n * p;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = e / n, r = e - c * n;
    Y[c * ldy + r] = (double)X[c * ldx + r];
  }
}

template <typename T, int KT>
int launch_project(const T* X, int64_t ldx, int64_t n, int p, const double* V, int k, double* out, int64_t ldo,
                   cudaStream_t s) {
  auto kern = pca_project_kernel<T, KT>;
  const size_t smem = (size_t)p * KT * sizeof(double);
  if (smem > 48 * 1024) PDSB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem) != cudaSuccess || per_sm < 1) {
    (void)cudaGetLastError();
    per_sm = 1;
  }
  const int ky = (k + KT - 1) / KT;
  const int64_t want = ceil_div(n, 256);
  const int gx = (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)sm_count() * per_sm / ky + 1));
  kern<<<dim3(gx, ky), 256, smem, s>>>(X, ldx, n, p, V, k, out, ldo);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

}  // namespace

int widen_f32(const float* X, int64_t ldx, int64_t n, int p, double* Y, int64_t ldy, cudaStream_t s) {
  if (n * p == 0) return 0;
  const int grid = (int)std::min<int64_t>(ceil_div(n * p, 256), (int64_t)sm_count() * 8);
  widen_kernel<<<grid, 256, 0, s>>>(X, ldx, n, p, Y, ldy);
  PDSB_LAUNCH_OK();
  count_launch();
  return 0;
}

int pca_eigen(const double* M, int q1, int p, double* sigma, double* V, int* status, cudaStream_t s) {
  const size_t nd = 2 * (size_t)p * p + 4 * (size_t)(p / 2 + 2);
  char* base = nullptr;
  if (dev_alloc((void**)&base, nd * sizeof(double) + (size_t)p * sizeof(int) + 64, s)) return 1;
  double* A = reinterpret_cast<double*>(base);
  double* Vu = A + (size_t)p * p;
  double* cs = Vu + (size_t)p * p;
  int* perm = reinterpret_cast<int*>(cs + 4 * (size_t)(p / 2 + 2));
  const size_t hot = (size_t)p * p * sizeof(double);      // A on chip when it fits (p <= 160)
  const int use_smem = hot <= 200 * 1024;
  if (use_smem && hot > 48 * 1024) cudaFuncSetAttribute(pca_eigen_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hot);
  pca_eigen_kernel<<<1, NT, use_smem ? hot : 0, s>>>(M, q1, p, A, Vu, cs, perm, sigma, V, status, use_smem);
  cudaError_t e = cudaGetLastError();
  count_launch();
  dev_free(base, s);
  if (e != cudaSuccess) { set_error("pca eigen launch failed: %s", cudaGetErrorString(e)); return 1; }
  return 0;
}

template <typename T>
int pca_project(const T* X, int64_t ldx, int64_t n, int p, const double* V, int k, double* out, int64_t ldo,
                cudaStream_t s) {
  if (n == 0 || k == 0) return 0;
  if (k <= 1) return launch_project<T, 1>(X, ldx, n, p, V, k, out, ldo, s);
  if (k <= 2) return launch_project<T, 2>(X, ldx, n, p, V, k, out, ldo, s);
  if (k <= 4) return launch_project<T, 4>(X, ldx, n, p, V, k, out, ldo, s);
  if (k <= 8) return launch_project<T, 8>(X, ldx, n, p, V, k, out, ldo, s);
  if (k <= 16) return launch_project<T, 16>(X, ldx, n, p, V, k, out, ldo, s);
  return launch_project<T, 32>(X, ldx, n, p, V, k, out, ldo, s);     // more than 32 columns: grid rows of 32
}

template int pca_project<float>(const float*, int64_t, int64_t, int, const double*, int, double*, int64_t, cudaStream_t);
template int pca_project<double>(const double*, int64_t, int64_t, int, const double*, int, double*, int64_t, cudaStream_t);

}  // namespace pdsb
