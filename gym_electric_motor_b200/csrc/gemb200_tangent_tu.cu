// gemb200_tangent_tu.cu — the tangent-rollout kernels of one kind and one (motor family, real): compiled once per triple by build.py with
//   -DGEMB200_TAN_OUT=<JacOut: rollout Jacobians | GradOut: return gradients | PsOut: parameter sensitivities> -DGEMB200_JAC_FAM=<0..5>
//   -DGEMB200_JAC_REAL=<float|double>
// Per unit: 2 converter kinds (return gradients: continuous only) x 5 reference counts x {shared, per-env coefficients} kernels.
#if !defined(GEMB200_TAN_OUT) || !defined(GEMB200_JAC_FAM) || !defined(GEMB200_JAC_REAL)
#error "compile with -DGEMB200_TAN_OUT=<JacOut|GradOut|PsOut> -DGEMB200_JAC_FAM=<family> -DGEMB200_JAC_REAL=<float|double>"
#endif
#include "gemb200_tangent.cuh"

namespace gemb200 {

// The staging row of one env (jstride words, odd: the lanes' rows fall into different banks) and the kernel of each kind
template <int FAM, bool FINITE> static int tangent_stride(const JacOut& jo) {
  constexpr int NX1 = Fam<FAM>::NX + (Fam<FAM>::EPS ? 1 : 0);
  return (NX1 * (NX1 + (FINITE ? 0 : jo.nu))) | 1;
}
template <int FAM, bool FINITE> static int tangent_stride(const GradOut& go) {  // the stash row (W words) and the reward row (NS)
  constexpr int NX1 = Fam<FAM>::NX + (Fam<FAM>::EPS ? 1 : 0);
  return (NX1 * (NX1 + go.nu) + NX1 + go.nu + Fam<FAM>::NS) | 1;
}
template <int FAM, bool FINITE> static int tangent_stride(const PsOut& po) {  // S and the coefficient tangents
  constexpr int NX1 = Fam<FAM>::NX + (Fam<FAM>::EPS ? 1 : 0);
  return (po.np * (NX1 + ps_words<FAM>())) | 1;
}
template <int FAM, bool FINITE, typename real, int NREF, bool ENVP> static auto tangent_kernel(const JacOut&) { return jacobian_kernel<FAM, FINITE, real, NREF, ENVP>; }
template <int FAM, bool FINITE, typename real, int NREF, bool ENVP> static auto tangent_kernel(const GradOut&) { return return_grad_kernel<FAM, real, NREF, ENVP>; }
template <int FAM, bool FINITE, typename real, int NREF, bool ENVP> static auto tangent_kernel(const PsOut&) { return param_sens_kernel<FAM, FINITE, real, NREF, ENVP>; }

// The launch shape: the largest block of 128 / 64 / 32 threads whose staging rows fit the default 48 KB of dynamic shared memory; a 32-thread
// block that does not fit (parameter sensitivities in fp64 with many parameters) opts in to more
template <int FAM, bool FINITE, typename real, int NREF, typename O>
static cudaError_t launch_tangent_t(const StepParams<real>& p, const O& o, cudaStream_t st) {
  const int jstride = tangent_stride<FAM, FINITE>(o);
  const int range = p.env_end - p.env_begin;
  int block = kBlock;
  while (block > 32 && (size_t)block * (size_t)(p.row_stride + jstride) * sizeof(real) > 48 * 1024) block >>= 1;
  const size_t smem = (size_t)block * (size_t)(p.row_stride + jstride) * sizeof(real);
  const int grid = (range + block - 1) / block;
  auto kern = p.envp ? tangent_kernel<FAM, FINITE, real, NREF, true>(o) : tangent_kernel<FAM, FINITE, real, NREF, false>(o);
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  kern<<<grid, block, smem, st>>>(p, o, jstride);
  return cudaGetLastError();
}

template <int FAM, typename real>
cudaError_t launch_tangent_f(bool finite, int nref, const StepParams<real>& p, const GEMB200_TAN_OUT& o, cudaStream_t st) {
  constexpr bool kFinite = !std::is_same<GEMB200_TAN_OUT, GradOut>::value;  // return gradients: continuous converters only
#define GEMB200_TAN_NREF(R)                                                                  \
  case R:                                                                                    \
    if constexpr (kFinite) { if (finite) return launch_tangent_t<FAM, true, real, R>(p, o, st); } \
    return launch_tangent_t<FAM, false, real, R>(p, o, st);
  switch (nref) {
    GEMB200_TAN_NREF(0)
    GEMB200_TAN_NREF(1)
    GEMB200_TAN_NREF(2)
    GEMB200_TAN_NREF(3)
    GEMB200_TAN_NREF(4)
  }
#undef GEMB200_TAN_NREF
  return cudaErrorInvalidValue;
}

template cudaError_t launch_tangent_f<GEMB200_JAC_FAM, GEMB200_JAC_REAL>(bool, int, const StepParams<GEMB200_JAC_REAL>&, const GEMB200_TAN_OUT&, cudaStream_t);

}  // namespace gemb200
