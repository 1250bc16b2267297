// gemb200_launch.cuh — step/reset kernel dispatch for ONE (motor family, real) pair.
//
// The step kernel has 5 families x {cont, finite} x {fp32, fp64} x NREF 0..4 x {AoS, SoA} = 200 instantiations; each
// (family, real) pair is compiled in its own translation unit (gemb200_step_tu.cu with -DGEMB200_TU_FAM / -DGEMB200_TU_REAL) so that
// the library builds in parallel.  gemb200.cu only sees the declarations below.
#pragma once
#include "gemb200_kernels.cuh"

namespace gemb200 {

// p.roll_steps == 0: one step (step_kernel); >= 1: that many fused steps (rollout_kernel).  A launch with a reference feed (p.ref_feed)
// or with discounted returns (p.ret_out) takes the general or ENVP instantiation: the PLAIN kernels have neither.
template <int FAM, typename real> cudaError_t launch_step_f(bool finite, int nref, const StepParams<real>& p, cudaStream_t st);
template <int FAM, typename real> cudaError_t launch_reset_f(int nref, const StepParams<real>& p, cudaStream_t st);

#ifdef GEMB200_TU_FAM
// Block size of a launch: kBlock (128) threads, or — for batches too small to give every SM its share of 128-thread blocks — 64 or 32, so that
// the blocks spread evenly (N = 65 536: 512 blocks of 128 threads are 3.46 per SM, i.e. a 4-vs-3 imbalance; 2048 blocks of 32 are 13.8).  The
// kernels index with blockDim.x, so the choice is a launch parameter.
static int pick_block(int range) {
  static const int sms = [] { int dev = 0, n = 132; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); return n; }();
  int block = kBlock;
  while (block > 32 && (range + block - 1) / block < sms * 8) block >>= 1;
  return block;
}

template <int FAM, bool FINITE, typename real, int NREF, bool SOA, bool PLAIN = false, bool MECH = false, bool IL = false>
static cudaError_t launch_step_t(const StepParams<real>& p, cudaStream_t st) {
  const int range = p.env_end - p.env_begin;
  const int block = pick_block(range);
  const size_t smem = (size_t)block * (size_t)p.row_stride * sizeof(real);
  const int grid = (range + block - 1) / block;
  if constexpr (!PLAIN) {
    if (p.envp) {  // per-env parameter blocks: the ENVP instantiation of the general kernel (row-per-env I/O layout only, checked by the host)
      if constexpr (SOA) return cudaErrorInvalidValue;
      else {
      if (p.roll_steps > 0) rollout_kernel<FAM, FINITE, real, NREF, SOA, false, false, true><<<grid, block, smem, st>>>(p);
      else step_kernel<FAM, FINITE, real, NREF, SOA, false, false, true><<<grid, block, smem, st>>>(p);
      return cudaGetLastError();
      }
    }
  }
  if (p.roll_steps > 0) rollout_kernel<FAM, FINITE, real, NREF, SOA, PLAIN, MECH, false, IL><<<grid, block, smem, st>>>(p);
  else step_kernel<FAM, FINITE, real, NREF, SOA, PLAIN, MECH, false, IL><<<grid, block, smem, st>>>(p);
  return cudaGetLastError();
}
// PLAIN instantiations (fp32): {cont, finite, finite with interlocking time} x {constant speed, integrating load} x {AoS, SoA}
template <int FAM, typename real, int NREF>
static cudaError_t launch_plain_t(bool finite, const StepParams<real>& p, cudaStream_t st) {
  const bool soa = p.layout == GEMB200_LAYOUT_SOA, mech = p.load_kind != GEMB200_LOAD_CONST_SPEED;
  if (finite && p.two_segment) {  // IL: the legs wait in their interlock state, up to three switching segments per step
    if (mech) return soa ? launch_step_t<FAM, true, real, NREF, true, true, true, true>(p, st) : launch_step_t<FAM, true, real, NREF, false, true, true, true>(p, st);
    return soa ? launch_step_t<FAM, true, real, NREF, true, true, false, true>(p, st) : launch_step_t<FAM, true, real, NREF, false, true, false, true>(p, st);
  }
#define GEMB200_PLAIN(F, M)                                                                                   \
  if (finite == F && mech == M)                                                                               \
    return soa ? launch_step_t<FAM, F, real, NREF, true, true, M>(p, st) : launch_step_t<FAM, F, real, NREF, false, true, M>(p, st);
  GEMB200_PLAIN(false, false)
  GEMB200_PLAIN(false, true)
  GEMB200_PLAIN(true, false)
  GEMB200_PLAIN(true, true)
#undef GEMB200_PLAIN
  return cudaErrorInvalidValue;
}
template <int FAM, typename real, int NREF>
static cudaError_t launch_reset_t(const StepParams<real>& p, cudaStream_t st) {
  const int grid = (p.n + 255) / 256;
  reset_kernel<FAM, real, NREF><<<grid, 256, 0, st>>>(p);
  return cudaGetLastError();
}

template <int FAM, typename real>
cudaError_t launch_step_f(bool finite, int nref, const StepParams<real>& p, cudaStream_t st) {
#define GEMB200_NREF(R)                                                                         \
  case R:                                                                                       \
    if constexpr (std::is_same<real, float>::value) {                                           \
      if (p.plain && !p.ref_feed && !p.ret_out) return launch_plain_t<FAM, real, R>(finite, p, st); \
    }                                                                                           \
    if (p.layout == GEMB200_LAYOUT_SOA) return finite ? launch_step_t<FAM, true, real, R, true>(p, st) : launch_step_t<FAM, false, real, R, true>(p, st); \
    return finite ? launch_step_t<FAM, true, real, R, false>(p, st) : launch_step_t<FAM, false, real, R, false>(p, st);
  switch (nref) {
    GEMB200_NREF(0)
    GEMB200_NREF(1)
    GEMB200_NREF(2)
    GEMB200_NREF(3)
    GEMB200_NREF(4)
  }
#undef GEMB200_NREF
  return cudaErrorInvalidValue;
}
template <int FAM, typename real>
cudaError_t launch_reset_f(int nref, const StepParams<real>& p, cudaStream_t st) {
  switch (nref) {
    case 0: return launch_reset_t<FAM, real, 0>(p, st);
    case 1: return launch_reset_t<FAM, real, 1>(p, st);
    case 2: return launch_reset_t<FAM, real, 2>(p, st);
    case 3: return launch_reset_t<FAM, real, 3>(p, st);
    case 4: return launch_reset_t<FAM, real, 4>(p, st);
  }
  return cudaErrorInvalidValue;
}


template cudaError_t launch_step_f<GEMB200_TU_FAM, GEMB200_TU_REAL>(bool, int, const StepParams<GEMB200_TU_REAL>&, cudaStream_t);
template cudaError_t launch_reset_f<GEMB200_TU_FAM, GEMB200_TU_REAL>(int, const StepParams<GEMB200_TU_REAL>&, cudaStream_t);
#endif

}  // namespace gemb200
