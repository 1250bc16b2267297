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

}  // namespace gemb200
