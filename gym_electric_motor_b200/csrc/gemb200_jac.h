// gemb200_jac.h — the tangent-rollout launches as the host unit sees them: rollout Jacobians (gemb200_rollout_jacobians), return gradients
// and parameter sensitivities, one launch_tangent_f overload per output kind.  The kernels live in gemb200_tangent.cuh and are instantiated
// per (kind, motor family, real) from gemb200_tangent_tu.cu.
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

template <int FAM, typename real> cudaError_t launch_tangent_f(bool finite, int nref, const StepParams<real>& p, const JacOut& jo, cudaStream_t st);

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

// finite: ignored, return gradients cover continuous converters only (gemb200_rollout_return_grads refuses finite ones)
template <int FAM, typename real> cudaError_t launch_tangent_f(bool finite, int nref, const StepParams<real>& p, const GradOut& go, cudaStream_t st);

// Where the parameter sensitivities of gemb200_rollout_param_sens go, and with respect to what.  sio: S = d x / d theta [N][n_x][n_p], read
// at the start of the launch and overwritten with its value after the last step; sout: S after every step [K][N][n_x][n_p], or NULL; slot[c]:
// the parameter row slot of column c; raw: the configuration's parameter row (the envs' parameters when the handle has no per-env blocks).
constexpr int kMaxSensParams = 12;
struct PsOut {
  void* sio;
  void* sout;
  int np;
  int32_t slot[kMaxSensParams];
  double raw[kMaxDraw];
};

template <int FAM, typename real> cudaError_t launch_tangent_f(bool finite, int nref, const StepParams<real>& p, const PsOut& po, cudaStream_t st);

}  // namespace gemb200
