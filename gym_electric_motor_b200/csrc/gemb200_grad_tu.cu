// gemb200_grad_tu.cu — the return-gradient kernels of one (motor family, real): compiled once per pair by build.py with
//   -DGEMB200_JAC_FAM=<0..5> -DGEMB200_JAC_REAL=<float|double>
// 5 reference counts x {shared, per-env coefficients} = 10 kernels per unit (continuous converters only).
#ifndef GEMB200_JAC_FAM
#error "compile with -DGEMB200_JAC_FAM=<family> -DGEMB200_JAC_REAL=<float|double>"
#endif
#include "gemb200_tangent.cuh"

namespace gemb200 {

template <int FAM, typename real, int NREF>
static cudaError_t launch_grad_t(const StepParams<real>& p, const GradOut& go, cudaStream_t st) {
  constexpr int NX1 = Fam<FAM>::NX + (Fam<FAM>::EPS ? 1 : 0);
  // the stash row (W words) and the coefficient row of the reward tangent (NS words); odd: the lanes' rows fall into different banks
  const int jstride = (NX1 * (NX1 + go.nu) + NX1 + go.nu + Fam<FAM>::NS) | 1;
  const int range = p.env_end - p.env_begin;
  // the largest block whose staging rows fit the default 48 KB of dynamic shared memory
  int block = GEMB200_BLOCK;
  while (block > 32 && (size_t)block * (size_t)(p.row_stride + jstride) * sizeof(real) > 48 * 1024) block >>= 1;
  const size_t smem = (size_t)block * (size_t)(p.row_stride + jstride) * sizeof(real);
  const int grid = (range + block - 1) / block;
  if (p.envp) return_grad_kernel<FAM, real, NREF, true><<<grid, block, smem, st>>>(p, go, jstride);
  else return_grad_kernel<FAM, real, NREF, false><<<grid, block, smem, st>>>(p, go, jstride);
  return cudaGetLastError();
}

template <int FAM, typename real>
cudaError_t launch_grad_f(int nref, const StepParams<real>& p, const GradOut& go, cudaStream_t st) {
  switch (nref) {
    case 0: return launch_grad_t<FAM, real, 0>(p, go, st);
    case 1: return launch_grad_t<FAM, real, 1>(p, go, st);
    case 2: return launch_grad_t<FAM, real, 2>(p, go, st);
    case 3: return launch_grad_t<FAM, real, 3>(p, go, st);
    case 4: return launch_grad_t<FAM, real, 4>(p, go, st);
  }
  return cudaErrorInvalidValue;
}

template cudaError_t launch_grad_f<GEMB200_JAC_FAM, GEMB200_JAC_REAL>(int, const StepParams<GEMB200_JAC_REAL>&, const GradOut&, cudaStream_t);

}  // namespace gemb200
