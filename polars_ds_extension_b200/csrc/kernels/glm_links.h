// Link and variance functions of the GLM families, as device policies shared by the IRLS row pass (K11) and the
// strided predict (K10).
//
// Reference: LinkFunction / VarianceFunction (/root/reference/src/linear/glm/link_functions.rs:1-79) and the family
// table GLMFamily::{link_function, variance_function} (src/linear/glm/glm_solvers.rs:17-47).  Each policy restates the
// reference's expression in the same order (powi(2) is a product; recip is __drcp_rn, the correctly rounded 1 / x,
// which unlike the division operator needs no stack frame in the row pass), with one deliberate change: the logit
// inverse is the overflow-free sigmoid of logistic_solver.rs:10-18, where the reference's exp(eta) / (1 + exp(eta))
// turns NaN for eta above ~709 (DESIGN.md §5, deviation 8).
#pragma once
#include <cuda_runtime.h>

namespace pdsb {
namespace glm {

// logistic_solver.rs:10-18
__device__ __forceinline__ double stable_sigmoid(double x) {
  const double r = 1.0 / (1.0 + exp(-fabs(x)));
  return x >= 0.0 ? r : 1.0 - r;
}

// g, g^-1, g' and V of one family.  start(y, mean_y) is faer_irls's mu_0 (glm_solvers.rs:263-278).
struct Gaussian {                       // identity link, V = 1
  __device__ static double link(double mu) { return mu; }
  __device__ static double inv(double eta) { return eta; }
  __device__ static double deriv(double) { return 1.0; }
  __device__ static double variance(double) { return 1.0; }
  __device__ static double start(double y, double ybar) { return (y + ybar) * 0.5; }
};
struct Poisson {                        // log link, V = mu
  __device__ static double link(double mu) { return log(mu); }
  __device__ static double inv(double eta) { return exp(eta); }
  __device__ static double deriv(double mu) { return __drcp_rn(mu); }
  __device__ static double variance(double mu) { return mu; }
  __device__ static double start(double y, double ybar) { return (y + ybar) * 0.5; }
};
struct Binomial {                       // logit link, V = mu (1 - mu)
  __device__ static double link(double mu) { return log(mu / (1.0 - mu)); }
  __device__ static double inv(double eta) { return stable_sigmoid(eta); }
  __device__ static double deriv(double mu) { return 1.0 / (mu * (1.0 - mu)); }
  __device__ static double variance(double mu) { return mu * (1.0 - mu); }
  __device__ static double start(double y, double) { return (y + 0.5) * 0.5; }
};
struct Gamma {                          // inverse link, V = mu^2
  __device__ static double link(double mu) { return __drcp_rn(mu); }
  __device__ static double inv(double eta) { return __drcp_rn(eta); }
  __device__ static double deriv(double mu) { const double r = __drcp_rn(mu); return -(r * r); }
  __device__ static double variance(double mu) { return mu * mu; }
  __device__ static double start(double y, double ybar) { return (y + ybar) * 0.5; }
};

}  // namespace glm
}  // namespace pdsb
