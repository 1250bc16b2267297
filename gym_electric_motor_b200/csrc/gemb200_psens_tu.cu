// gemb200_psens_tu.cu — the parameter-sensitivity kernels of one (motor family, real): compiled once per pair by build.py with
//   -DGEMB200_JAC_FAM=<0..5> -DGEMB200_JAC_REAL=<float|double>
// 2 converter kinds x 5 reference counts x {shared, per-env coefficients} = 20 kernels per unit.
#ifndef GEMB200_JAC_FAM
#error "compile with -DGEMB200_JAC_FAM=<family> -DGEMB200_JAC_REAL=<float|double>"
#endif
#include "gemb200_tangent.cuh"

namespace gemb200 {

template <int FAM, bool FINITE, typename real, int NREF>
static cudaError_t launch_psens_t(const StepParams<real>& p, const PsOut& po, cudaStream_t st) {
  constexpr int NX1 = Fam<FAM>::NX + (Fam<FAM>::EPS ? 1 : 0);
  const int jstride = (po.np * (NX1 + ps_words<FAM>())) | 1;  // odd: the lanes' staging rows fall into different banks
  const int range = p.env_end - p.env_begin;
  // the largest block whose staging rows fit the default 48 KB of dynamic shared memory; a 32-thread block that does not fit (fp64 with many
  // parameters) opts in to more
  int block = GEMB200_BLOCK;
  while (block > 32 && (size_t)block * (size_t)(p.row_stride + jstride) * sizeof(real) > 48 * 1024) block >>= 1;
  const size_t smem = (size_t)block * (size_t)(p.row_stride + jstride) * sizeof(real);
  const int grid = (range + block - 1) / block;
  auto kern = p.envp ? param_sens_kernel<FAM, FINITE, real, NREF, true> : param_sens_kernel<FAM, FINITE, real, NREF, false>;
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  kern<<<grid, block, smem, st>>>(p, po, jstride);
  return cudaGetLastError();
}

template <int FAM, typename real>
cudaError_t launch_psens_f(bool finite, int nref, const StepParams<real>& p, const PsOut& po, cudaStream_t st) {
#define GEMB200_PSENS_NREF(R) \
  case R: return finite ? launch_psens_t<FAM, true, real, R>(p, po, st) : launch_psens_t<FAM, false, real, R>(p, po, st);
  switch (nref) {
    GEMB200_PSENS_NREF(0)
    GEMB200_PSENS_NREF(1)
    GEMB200_PSENS_NREF(2)
    GEMB200_PSENS_NREF(3)
    GEMB200_PSENS_NREF(4)
  }
#undef GEMB200_PSENS_NREF
  return cudaErrorInvalidValue;
}

template cudaError_t launch_psens_f<GEMB200_JAC_FAM, GEMB200_JAC_REAL>(bool, int, const StepParams<GEMB200_JAC_REAL>&, const PsOut&, cudaStream_t);

}  // namespace gemb200
