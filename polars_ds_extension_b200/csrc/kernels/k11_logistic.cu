// K11 — logistic regression (pds.logistic_reg) and GLM.fit: the per-row pass of Newton / IRLS.  The probabilities of
// pl_logistic_pred are K10's predict_strided with the binomial inverse link.
//
// Reference: faer_logistic_reg (/root/reference/src/linear/logistic/logistic_solver.rs:107-146) minimises
//     cost(w) = mean_i stable_log_loss(y_i, x_i.w) + (l2 / 2) |w_features|^2           (:42-74)
// with argmin's L-BFGS (OWL-QN when l1 > 0) from a seeded random start; the expression bodies are pl_logistic_coeffs /
// pl_logistic_pred (src/num_ext/logistic_regression.rs:10-99).  The minimiser of that convex cost does not depend on the
// optimiser, so this path runs Newton's method in its IRLS form, which is built from the kernels of the linear path:
// at the current w every row gets
//     eta = x.w,  mu = sigmoid(eta),  weight = mu (1 - mu),  working response z = eta + (y - mu) / weight
// (this kernel, one coalesced pass that also returns the summed log-loss), then the WEIGHTED moments
// [X | z | 1]' diag(weight) [X | z | 1] (K2a) and the ridge solve on them (K3) give the next w; the gradient norm the
// reference stops on comes out of the same moments:  X' (mu - y) = (X' W X) w - X' W z.
// HBM-bound: (p + 1) s read + 2 s written per row and iteration here, (p + 2) s read by the moments pass.
//
// The same row pass serves GLM.fit (faer_irls, /root/reference/src/linear/glm/glm_solvers.rs:249-359) for the
// gaussian / poisson / binomial / gamma families: the kernel is a template over a family policy.  The skeleton (grid-
// stride rows, beta in dynamic shared memory, eta = x.beta, the w and z writes) is shared; the policy supplies
// mu = g^-1(eta), the weight and the working response, and whether a log-loss partial is summed.  The INIT variant is
// faer_irls's first iteration: mu_0 comes from y and mean(y) (precomputed on the device), eta_0 = g(mu_0), and
// X is not read.  One entry, irls_rows, launches every policy: PDSB_IRLS_LOGISTIC or a pdsb_glm_family.
#include "../common.h"
#include "glm_links.h"
#include "logistic_rows.h"
#include "kernels.h"

namespace pdsb {

namespace {

constexpr int IRLS_THREADS = 256;
using glm::GlmRows;          // logistic_rows.h, shared with K16
using glm::LogisticRows;

template <class F, bool INIT>
__global__ void __launch_bounds__(IRLS_THREADS)
irls_rows_kernel(const double* __restrict__ X, int64_t ldx, const double* __restrict__ y, const double* __restrict__ mask,
                 int64_t n, int p, int add_bias, const double* __restrict__ beta,
                 const double* __restrict__ ymean /* INIT: mean(y) */, double* __restrict__ w_out,
                 double* __restrict__ z_out, double* __restrict__ loss_parts /* [gridDim.x] */) {
  extern __shared__ double sb[];                // p + add_bias coefficients, bias last
  double ybar = 0.0;
  if constexpr (INIT) {
    ybar = *ymean;
  } else {
    for (int i = threadIdx.x; i < p + add_bias; i += blockDim.x) sb[i] = beta[i];
    __syncthreads();
  }
  double loss = 0.0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    double eta, mu;
    if constexpr (INIT) {
      mu = F::start(y[r], ybar);
      eta = F::link(mu);
    } else {
      eta = add_bias ? sb[p] : 0.0;
      for (int c = 0; c < p; ++c) eta = fma(X[(int64_t)c * ldx + r], sb[c], eta);
    }
    const bool use = !mask || mask[r] != 0.0;
    const double yv = y[r];
    if constexpr (!INIT) mu = F::inv(eta);
    double wt, z;
    F::weight_response(eta, mu, yv, wt, z);
    w_out[r] = use ? wt : 0.0;
    z_out[r] = use ? z : 0.0;
    if constexpr (F::kLoss) {
      if (use) loss += F::loss(yv, eta);
    }
  }
  if constexpr (F::kLoss) {
    // fixed-shape reduction -> one partial per block (summed in order by the host: reproducible)
    __shared__ double red[IRLS_THREADS / 32];
    for (int off = 16; off; off >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, off);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = loss;
    __syncthreads();
    if (threadIdx.x == 0) {
      double v = 0.0;
      for (int i = 0; i < IRLS_THREADS / 32; ++i) v += red[i];
      loss_parts[blockIdx.x] = v;
    }
  }
}

// The INIT instance reads ymean instead of X and beta, so it needs no shared memory.
template <class F, bool INIT>
void launch_rows(int grid, cudaStream_t s, const double* X, int64_t ldx, const double* y, const double* mask, int64_t n,
                 int p, int add_bias, const double* beta, const double* ymean, double* w, double* z, double* loss_parts) {
  const size_t smem = INIT ? 0 : (size_t)(p + add_bias) * sizeof(double);
  irls_rows_kernel<F, INIT><<<grid, IRLS_THREADS, smem, s>>>(X, ldx, y, mask, n, p, add_bias, beta, ymean, w, z,
                                                              loss_parts);
}

template <class L>
void launch_glm_rows(int grid, cudaStream_t s, const double* X, int64_t ldx, const double* y, const double* mask,
                     int64_t n, int p, int add_bias, const double* beta, const double* ymean, double* w, double* z) {
  if (ymean) launch_rows<GlmRows<L>, true>(grid, s, X, ldx, y, mask, n, p, add_bias, beta, ymean, w, z, nullptr);
  else launch_rows<GlmRows<L>, false>(grid, s, X, ldx, y, mask, n, p, add_bias, beta, ymean, w, z, nullptr);
}

}  // namespace

int irls_max_parts() { return sm_count() * 8; }

int irls_rows(int family, const double* X, int64_t ldx, const double* y, const double* mask, int64_t n, int p,
              int add_bias, const double* beta, const double* ymean, double* w, double* z, double* loss_parts,
              int* n_parts, cudaStream_t s) {
  if (n <= 0) return 0;
  const int grid = (int)std::min<int64_t>(ceil_div(n, (int64_t)IRLS_THREADS), irls_max_parts());
  switch (family) {
    case PDSB_IRLS_LOGISTIC:       // Newton on the log-loss starts from beta = 0: no INIT instance
      if (ymean) { set_error("irls_rows: the logistic pass has no start from mean(y)"); return 1; }
      launch_rows<LogisticRows, false>(grid, s, X, ldx, y, mask, n, p, add_bias, beta, nullptr, w, z, loss_parts);
      break;
    case PDSB_GLM_GAUSSIAN: launch_glm_rows<glm::Gaussian>(grid, s, X, ldx, y, mask, n, p, add_bias, beta, ymean, w, z); break;
    case PDSB_GLM_POISSON: launch_glm_rows<glm::Poisson>(grid, s, X, ldx, y, mask, n, p, add_bias, beta, ymean, w, z); break;
    case PDSB_GLM_BINOMIAL: launch_glm_rows<glm::Binomial>(grid, s, X, ldx, y, mask, n, p, add_bias, beta, ymean, w, z); break;
    case PDSB_GLM_GAMMA: launch_glm_rows<glm::Gamma>(grid, s, X, ldx, y, mask, n, p, add_bias, beta, ymean, w, z); break;
    default: set_error("irls_rows: unknown family %d", family); return 1;
  }
  PDSB_LAUNCH_OK();
  count_launch();
  if (n_parts) *n_parts = grid;
  return 0;
}

}  // namespace pdsb
