// gemb200_jac.h — the rollout-Jacobian launch (gemb200_rollout_jacobians) as the host unit sees it.  The kernels live in
// gemb200_tangent.cuh and are instantiated per (motor family, real) in gemb200_jac_tu.cu.
#pragma once
#include <cuda_runtime.h>

#include "gemb200_params.h"

namespace gemb200 {

// Where the Jacobians of a rollout go: jac_x [K][N][n_x][n_x] and jac_u [K][N][n_x][n_u] in the handle's dtype (jac_u may be NULL and is
// never written when n_u == 0).  A second kernel argument next to StepParams, so that the step and rollout kernels keep their parameter block.
struct JacOut {
  void* jx;
  void* ju;
  int nu;  // caller-side action width (0: finite converter)
};

template <int FAM, typename real> cudaError_t launch_jac_f(bool finite, int nref, const StepParams<real>& p, const JacOut& jo, cudaStream_t st);

// Where the return gradients of gemb200_rollout_return_grads go, and how the reward reads the state row.  ws: the caller's workspace
// [K][N][W] (W = n_x (n_x + n_u) + n_x + n_u words: one [J_x | J_u | d(g^k r_k)/dx | d(g^k r_k)/da] row per env and step); grad_a [K][N][n_u];
// grad_x0 [N][n_x]; value_grad [N][n_x] or NULL.  ref_base / rw_base: the entry of the family's state vector (before the wrappers) that
// reward term r / t reads (StepParams::ref_state / rw_state index the row after the wrappers); wmask: the union of those entries.
struct GradOut {
  void* ws;
  void* grad_a;
  void* grad_x0;
  const void* value_grad;
  int nu;
  uint32_t wmask;
  int8_t ref_base[kMaxRef];
  int8_t rw_base[kMaxState];
};

template <int FAM, typename real> cudaError_t launch_grad_f(int nref, const StepParams<real>& p, const GradOut& go, cudaStream_t st);

}  // namespace gemb200
