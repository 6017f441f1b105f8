// The per-row rule of logistic_reg's Newton / IRLS pass: K11's row pass (single fit) and K16's fused grouped pass both
// use it, so a row's weight, working response and log-loss are the same expressions in both.
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

}  // namespace glm
}  // namespace pdsb
