// The per-row rules of the Newton / IRLS passes: logistic_reg's and GLM.fit's.  K11's row pass (single fits) and K16's
// fused grouped pass both use them, so a row's weight, working response and log-loss are the same expressions in both.
#pragma once
#include <cuda_runtime.h>
#include "glm_links.h"

namespace pdsb {
namespace glm {

constexpr double IRLS_MIN_WEIGHT = 1e-12;     // keeps z finite when mu saturates (the row then carries no information)

// logistic_solver.rs:22-25
__device__ __forceinline__ double stable_log_loss(double y, double z) { return fmax(z, 0.0) - y * z + log1p(exp(-fabs(z))); }

// pds.logistic_reg: Newton on the mean log-loss; the weight is clamped so z stays finite, and the loss is summed.
struct LogisticRows {
  static constexpr bool kLoss = true;
  __device__ static double inv(double eta) { return stable_sigmoid(eta); }
  __device__ static void weight_response(double eta, double mu, double y, double& wt, double& z) {
    wt = fmax(mu * (1.0 - mu), IRLS_MIN_WEIGHT);
    z = eta + (y - mu) / wt;
  }
  __device__ static double loss(double y, double eta) { return stable_log_loss(y, eta); }
};

// GLM.fit, one family L (glm_links.h): d = g'(mu), w = 1 / (d^2 V(mu)), z = eta + d (y - mu)   (glm_solvers.rs:293-307).
// No clamp: like the reference, a non-finite row makes non-finite moments.  No loss.
template <class L>
struct GlmRows {
  static constexpr bool kLoss = false;
  __device__ static double inv(double eta) { return L::inv(eta); }
  __device__ static double link(double mu) { return L::link(mu); }
  __device__ static double start(double y, double ybar) { return L::start(y, ybar); }
  __device__ static void weight_response(double eta, double mu, double y, double& wt, double& z) {
    const double d = L::deriv(mu);
    wt = __drcp_rn(d * d * L::variance(mu));
    z = eta + d * (y - mu);
  }
  __device__ static double loss(double, double) { return 0.0; }
};

}  // namespace glm
}  // namespace pdsb
