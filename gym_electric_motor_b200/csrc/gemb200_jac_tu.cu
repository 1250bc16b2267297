// gemb200_jac_tu.cu — the rollout-Jacobian kernels of one (motor family, real): compiled once per pair by build.py with
//   -DGEMB200_JAC_FAM=<0..5> -DGEMB200_JAC_REAL=<float|double>
// 2 converter kinds x 5 reference counts x {shared, per-env coefficients} = 20 kernels per unit.
#ifndef GEMB200_JAC_FAM
#error "compile with -DGEMB200_JAC_FAM=<family> -DGEMB200_JAC_REAL=<float|double>"
#endif
#include "gemb200_tangent.cuh"

namespace gemb200 {

template <int FAM, bool FINITE, typename real, int NREF>
static cudaError_t launch_jac_t(const StepParams<real>& p, const JacOut& jo, cudaStream_t st) {
  constexpr int NX1 = Fam<FAM>::NX + (Fam<FAM>::EPS ? 1 : 0);
  const int nu = FINITE ? 0 : jo.nu;
  const int jstride = (NX1 * (NX1 + nu)) | 1;  // odd: the lanes' staging rows fall into different banks
  const int range = p.env_end - p.env_begin;
  // the largest block whose staging rows fit the default 48 KB of dynamic shared memory
  int block = GEMB200_BLOCK;
  while (block > 32 && (size_t)block * (size_t)(p.row_stride + jstride) * sizeof(real) > 48 * 1024) block >>= 1;
  const size_t smem = (size_t)block * (size_t)(p.row_stride + jstride) * sizeof(real);
  const int grid = (range + block - 1) / block;
  if (p.envp) jacobian_kernel<FAM, FINITE, real, NREF, true><<<grid, block, smem, st>>>(p, jo, jstride);
  else jacobian_kernel<FAM, FINITE, real, NREF, false><<<grid, block, smem, st>>>(p, jo, jstride);
  return cudaGetLastError();
}

template <int FAM, typename real>
cudaError_t launch_jac_f(bool finite, int nref, const StepParams<real>& p, const JacOut& jo, cudaStream_t st) {
#define GEMB200_JAC_NREF(R) \
  case R: return finite ? launch_jac_t<FAM, true, real, R>(p, jo, st) : launch_jac_t<FAM, false, real, R>(p, jo, st);
  switch (nref) {
    GEMB200_JAC_NREF(0)
    GEMB200_JAC_NREF(1)
    GEMB200_JAC_NREF(2)
    GEMB200_JAC_NREF(3)
    GEMB200_JAC_NREF(4)
  }
#undef GEMB200_JAC_NREF
  return cudaErrorInvalidValue;
}

template cudaError_t launch_jac_f<GEMB200_JAC_FAM, GEMB200_JAC_REAL>(bool, int, const StepParams<GEMB200_JAC_REAL>&, const JacOut&, cudaStream_t);

}  // namespace gemb200
