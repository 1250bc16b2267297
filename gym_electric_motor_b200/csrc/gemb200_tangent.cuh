// gemb200_tangent.cuh — the linearised plant along a fused rollout (gemb200_rollout_jacobians, DESIGN.md §4 "Rollout Jacobians").
//
// Per env and step the kernel writes  jac_x = d x_{k+1} / d x_k  and  jac_u = d x_{k+1} / d a_k,  x = the ODE state of get_ode_state
// ([load states | motor states], the angle last, in radians), a = the caller's action.  The primal is the unchanged env_step of
// gemb200_kernels.cuh; the tangent pass reads only the pre-step state, coefficients and action, so it runs right BEFORE env_step on the
// registers env_step is about to advance.  It is forward mode, one seed column at a time: each pass re-computes the primal stage values it
// needs, so a thread holds one primal and one tangent vector instead of an n_x x (n_x + n_u) matrix.
//
// Non-smooth points take the one-sided derivative of the branch the primal took (DESIGN.md §7): clipped duty cycles and the interlocking
// terms sgn(i) t_il / tau have derivative 0, the static-friction branch of the polynomial load is the one taken, the angle wrap has
// derivative 1.  Voltages of finite converters are piecewise constant in the state: only the angle of their rotation into the solver frame
// is differentiated, segment by segment: with an interlocking time a finite step has two or three switching segments, and the angle's
// tangent after one segment rotates the voltages of the next.
#pragma once
#include "gemb200_jac.h"
#include "gemb200_kernels.cuh"

#ifndef GEMB200_MINBLOCKS_JAC
#define GEMB200_MINBLOCKS_JAC 3  /* fp32: <= 168 registers */
#endif
#ifndef GEMB200_MINBLOCKS_JAC_F64
#define GEMB200_MINBLOCKS_JAC_F64 2  /* fp64: <= 255 registers */
#endif

namespace gemb200 {

// radians per unit of the stored angle (turns in the fp32 build, radians in fp64)
template <typename real> __device__ __forceinline__ real rad_per_ang() { return sizeof(real) == 4 ? real(6.283185307179586) : real(1); }

// d/dx of clamp01 at x: 1 on [0, 1], 0 where the primal clipped
template <typename real> __device__ __forceinline__ real clamp01_t(real x) { return (x >= real(0) && x <= real(1)) ? real(1) : real(0); }

// tangent of load_ode (mech != 0): the static-friction branch the primal takes, sgn(w) held
template <typename real>
__device__ __forceinline__ real load_ode_t(const Coef<real>& p, real eit, real w, real dw, real dtq, int mech) {
  if (mech == 2) return -(dw * eit);
  const real sign = sgn(w);
  const real da = Num<real>::abs(w) > p.omega_lim ? real(0) : p.omega_lin * dw;
  const real dtl = (real(2) * (sign * p.load_c) * w + p.load_b) * dw + da;
  return (dtq - dtl) * p.inv_j;
}

// Tangents of Model<FAM>::rhs: d = J_x(x) dx + dub (the voltage terms are linear, dub = ubias(du))
template <int FAM, typename real> struct Tan;
template <typename real> struct Tan<kDC1, real> {
  static __device__ __forceinline__ void rhs(const Coef<real>& p, real eit, const real* x, const real* dx, const real* dub, int mech, real* d) {
    const real w = x[0], i = x[1], dw = dx[0], di = dx[1];
    d[1] = p.c[0] * dw + p.c[1] * di + p.c[2] * (dw * i + w * di) + dub[0];
    d[0] = mech ? load_ode_t(p, eit, w, dw, (real(2) * p.tq[1] * i + p.tq[0]) * di, mech) : real(0);
  }
};
template <typename real> struct Tan<kDC2, real> {
  static __device__ __forceinline__ void rhs(const Coef<real>& p, real eit, const real* x, const real* dx, const real* dub, int mech, real* d) {
    const real w = x[0], ia = x[1], ie = x[2], dw = dx[0], dia = dx[1], die = dx[2];
    d[1] = p.c[0] * dia + p.c[1] * (dw * ie + w * die) + dub[0];
    d[2] = p.c[3] * die + dub[1];
    d[0] = mech ? load_ode_t(p, eit, w, dw, p.tq[0] * (dia * ie + ia * die), mech) : real(0);
  }
};
template <typename real> struct Tan<kSYNC, real> {
  static __device__ __forceinline__ void rhs(const Coef<real>& p, real eit, const real* x, const real* dx, const real* dub, int mech, real* d) {
    const real w = x[0], id = x[1], iq = x[2], dw = dx[0], did = dx[1], diq = dx[2];
    d[1] = p.c[0] * did + p.c[2] * (dw * iq + w * diq) + dub[0];
    d[2] = p.c[3] * dw + p.c[4] * diq + p.c[6] * (dw * id + w * did) + dub[1];
    d[0] = mech ? load_ode_t(p, eit, w, dw, p.tq[1] * did * iq + (p.tq[1] * id + p.tq[0]) * diq, mech) : real(0);
  }
};
template <typename real> struct Tan<kEESM, real> {
  static __device__ __forceinline__ void rhs(const Coef<real>& p, real eit, const real* x, const real* dx, const real* dub, int mech, real* d) {
    const real w = x[0], id = x[1], iq = x[2], ie = x[3], dw = dx[0], did = dx[1], diq = dx[2], die = dx[3];
    d[1] = p.c[0] * did + p.c[1] * die + p.c[4] * (dw * iq + w * diq) + dub[0];
    d[2] = p.c[5] * diq + p.c[7] * (dw * id + w * did) + p.c[8] * (dw * ie + w * die) + dub[1];
    d[3] = p.c[9] * did + p.c[10] * die + p.c[13] * (dw * iq + w * diq) + dub[2];
    d[0] = mech ? load_ode_t(p, eit, w, dw, (p.tq[0] * die + p.tq[1] * did) * iq + (p.tq[0] * ie + p.tq[1] * id) * diq, mech) : real(0);
  }
};
template <int FAM, typename real> struct TanIM {  // SCIM, and DFIM with its rotor-voltage terms
  static __device__ __forceinline__ void rhs(const Coef<real>& p, real eit, const real* x, const real* dx, const real* dub, int mech, real* d) {
    const real w = x[0], ia = x[1], ib = x[2], pa = x[3], pb = x[4];
    const real dw = dx[0], dia = dx[1], dib = dx[2], dpa = dx[3], dpb = dx[4];
    d[1] = p.c[0] * dia + p.c[1] * dpa + p.c[2] * (dw * pb + w * dpb) + dub[0];
    d[2] = p.c[0] * dib + p.c[1] * dpb - p.c[2] * (dw * pa + w * dpa) + dub[1];
    d[3] = p.c[4] * dia + p.c[5] * dpa - p.c[6] * (dw * pb + w * dpb) + (FAM == kDFIM ? dub[2] : real(0));
    d[4] = p.c[4] * dib + p.c[5] * dpb + p.c[6] * (dw * pa + w * dpa) + (FAM == kDFIM ? dub[3] : real(0));
    d[0] = mech ? load_ode_t(p, eit, w, dw, p.tq[0] * (dpa * ib + pa * dib - dpb * ia - pb * dia), mech) : real(0);
  }
};
template <typename real> struct Tan<kSCIM, real> : TanIM<kSCIM, real> {};
template <typename real> struct Tan<kDFIM, real> : TanIM<kDFIM, real> {};

// rk4_step with its tangent: x, dx advance together; dws accumulates the tangent of the omega sum with the weights 1-2-2-1
template <int FAM, typename real>
__device__ __forceinline__ void rk4_step_t(const StepParams<real>& p, const Coef<real>& kc, real* x, real* dx, const real* ub, const real* dub, real h, int mech,
                                           real& dws, const real* gt) {
  constexpr int NX = Fam<FAM>::NX;
  const real hh = real(0.5) * h, h6 = h * real(1.0 / 6.0);
  const real g0 = mech == 2 ? gt[0] : real(0), g1 = mech == 2 ? gt[1] : real(0), g2 = mech == 2 ? gt[2] : real(0);
  real k[NX], dk[NX], acc[NX], dacc[NX], xt[NX], dxt[NX];
  Model<FAM, real>::rhs(kc, p.ext_inv_tau, x, ub, mech, g0, k);
  Tan<FAM, real>::rhs(kc, p.ext_inv_tau, x, dx, dub, mech, dk);
  if (mech) dws += dx[0];
  acc[0] = real(0); dacc[0] = real(0); xt[0] = x[0]; dxt[0] = dx[0];
#pragma unroll
  for (int j = 0; j < NX; ++j) if (j > 0 || mech) { acc[j] = k[j]; dacc[j] = dk[j]; xt[j] = fm(hh, k[j], x[j]); dxt[j] = fm(hh, dk[j], dx[j]); }
  Model<FAM, real>::rhs(kc, p.ext_inv_tau, xt, ub, mech, g1, k);
  Tan<FAM, real>::rhs(kc, p.ext_inv_tau, xt, dxt, dub, mech, dk);
  if (mech) dws += real(2) * dxt[0];
#pragma unroll
  for (int j = 0; j < NX; ++j) if (j > 0 || mech) { acc[j] = fm(real(2), k[j], acc[j]); dacc[j] = fm(real(2), dk[j], dacc[j]); xt[j] = fm(hh, k[j], x[j]); dxt[j] = fm(hh, dk[j], dx[j]); }
  Model<FAM, real>::rhs(kc, p.ext_inv_tau, xt, ub, mech, g1, k);
  Tan<FAM, real>::rhs(kc, p.ext_inv_tau, xt, dxt, dub, mech, dk);
  if (mech) dws += real(2) * dxt[0];
#pragma unroll
  for (int j = 0; j < NX; ++j) if (j > 0 || mech) { acc[j] = fm(real(2), k[j], acc[j]); dacc[j] = fm(real(2), dk[j], dacc[j]); xt[j] = fm(h, k[j], x[j]); dxt[j] = fm(h, dk[j], dx[j]); }
  Model<FAM, real>::rhs(kc, p.ext_inv_tau, xt, ub, mech, g2, k);
  Tan<FAM, real>::rhs(kc, p.ext_inv_tau, xt, dxt, dub, mech, dk);
  if (mech) dws += dxt[0];
#pragma unroll
  for (int j = 0; j < NX; ++j) if (j > 0 || mech) { x[j] = fm(h6, acc[j] + k[j], x[j]); dx[j] = fm(h6, dacc[j] + dk[j], dx[j]); }
}

// integrate with its tangent over one segment; returns the tangent of the omega sum (the angle advances by kang * wsum)
template <int FAM, typename real>
__device__ __forceinline__ real integrate_t(const StepParams<real>& p, const Coef<real>& kc, real* x, real* dx, const real* ub, const real* dub, real h_seg, int mech,
                                            const real* gt) {
  constexpr int NX = Fam<FAM>::NX;
  real dws = mech ? real(0) : dx[0];  // constant speed: the sum is omega itself
  const int ns = p.nsteps;
  const real h = h_seg * p.inv_nsteps;
  if (p.solver_kind == GEMB200_SOLVER_EULER) {
#pragma unroll 1
    for (int s = 0; s < ns; ++s) {
      real d[NX], dd[NX];
      Model<FAM, real>::rhs(kc, p.ext_inv_tau, x, ub, mech, mech == 2 ? gt[ns > 1 ? 2 * ns + 2 * (s + 1) : 0] : real(0), d);  // (the nsteps quirk)
      Tan<FAM, real>::rhs(kc, p.ext_inv_tau, x, dx, dub, mech, dd);
      if (mech) dws += dx[0];
#pragma unroll
      for (int j = 0; j < NX; ++j) if (j > 0 || mech) { x[j] = fm(d[j], h, x[j]); dx[j] = fm(dd[j], h, dx[j]); }
    }
    return dws;
  }
#pragma unroll 1
  for (int s = 0; s < ns; ++s) rk4_step_t<FAM, real>(p, kc, x, dx, ub, dub, h, mech, dws, gt + 2 * s);
  return dws;
}

// Continuous 1QC/2QC/4QC slot: d cont_qc / d a on the branch the primal takes
template <typename real> __device__ __forceinline__ real cont_qc_t(int kind, real a, real i, real tot) {
  const real si = -sgn(i);
  if (kind == GEMB200_CONV_4QC) {
    const real p1 = real(0.5) * (a + real(1)), p2 = real(-0.5) * (a - real(1));
    real g1 = clamp01_t(p1), g2 = clamp01_t(p2);
    if (tot != real(0)) { g1 *= clamp01_t(fm(si, tot, clamp01(p1))); g2 *= clamp01_t(fm(si, tot, clamp01(p2))); }
    return real(0.5) * (g1 + g2);
  }
  if (kind == GEMB200_CONV_2QC) return clamp01_t(a) * clamp01_t(fm(si, tot, clamp01(a)));
  return i >= real(0) ? clamp01_t(a) : real(0);  // 1QC
}

// Currents the converter sees at the start of a segment (their signs select its branches), and sin / cos of the angle there (sn, cs: the
// synchronous motors' dq frame; sne, cse: the DFIM's rotor frame) — the same expressions as env_step
template <int FAM, typename real>
__device__ __forceinline__ void converter_currents(const StepParams<real>& p, const Coef<real>& kc, const real* x, const Ang<real>& ang, real* i_in, real* sn,
                                                   real* cs, real* sne, real* cse) {
#pragma unroll
  for (int l = 0; l < 6; ++l) i_in[l] = real(0);
  *sn = real(0); *cs = real(1); *sne = real(0); *cse = real(1);
  if constexpr (FAM == kSYNC || FAM == kEESM) {
    ang.sincos(sn, cs);
    real ab[2] = {fm(*cs, x[1], -(*sn * x[2])), fm(*sn, x[1], *cs * x[2])};
    t32(ab, i_in);
    if constexpr (FAM == kEESM) i_in[3] = x[3];
  } else if constexpr (FAM == kSCIM) {
    t32(x + 1, i_in);
  } else if constexpr (FAM == kDFIM) {
    ang.sincos(sne, cse);
    t32(x + 1, i_in);
    const real irab[2] = {fm(kc.c[8], x[3], -(kc.c[9] * x[1])), fm(kc.c[8], x[4], -(kc.c[9] * x[2]))};
    t32(irab, i_in + 3);
  } else if constexpr (FAM == kDC1) {
    i_in[0] = x[1];
  } else {
    if (p.motor_kind == GEMB200_MOTOR_SHUNT_DC) i_in[0] = x[1] + x[2]; else { i_in[0] = x[1]; i_in[1] = x[2]; }
  }
}

// The switching segments of a finite converter's step (env_step's leg and segment plan; the switching states of the previous step are read,
// env_step writes them).  Per segment s: the solver-frame voltages us[s] and their voltage terms ub[s] (constant in the state: the legs'
// states are fixed and a current-sign voltage has derivative 0), the length hs[s] and the angle factor ka[s] (d eps / d wsum, rad).  The
// primal state and angle are advanced through all but the last segment with the unchanged integrate(), so that every segment's voltages
// and rotation are those the primal step applies.  With an interlocking time a switching step has two segments, or three with two
// different times.  Returns the number of segments.
template <int FAM, typename real>
__device__ __forceinline__ int finite_segments(const StepParams<real>& p, const Coef<real>& kc, const real (&x0)[Fam<FAM>::NX], const Ang<real>& ang0,
                                               const Act<real>& act, const unsigned i, const real u_sup, const int mech, const real* gt, real (&us)[3][4],
                                               real (&ub)[3][4], real (&hs)[3], real (&ka)[3]) {
  constexpr int NX = Fam<FAM>::NX;
  const bool il = p.two_segment != 0;
  const bool il_slot[2] = {il && p.til2[0] != real(0), il && p.til2[1] != real(0)};
  const int ssw = il ? (int)p.sw[i] : 0;
  FiniteLegs legs;
#pragma unroll
  for (int l = 0; l < 6; ++l) { legs.s[l] = 0; legs.cmd[l] = 0; }
  int act1qc[2] = {0, 0};
  bool two_seg = false;
  int pend = 0, promote_mask = 0, nseg = 1;
  int seg_idx[3] = {0, 0, 0};
#pragma unroll
  for (int slot = 0; slot < 2; ++slot) {
    const int kind = p.conv_kind[slot], base = slot == 0 ? 0 : 3, av = act.ai[slot];
    const bool ils = il_slot[slot];
    if (kind == GEMB200_CONV_B6) {
#pragma unroll
      for (int l = 0; l < 3; ++l) legs.s[base + l] = f2qc_leg((ssw >> (2 * (base + l))) & 3, ((av >> (2 - l)) & 1) ? 1 : 2, ils, &two_seg, base + l, legs.cmd, &pend);
    } else if (kind == GEMB200_CONV_4QC) {
      legs.s[base] = f2qc_leg((ssw >> (2 * base)) & 3, (av & 2) ? 2 : 1, ils, &two_seg, base, legs.cmd, &pend);
      legs.s[base + 1] = f2qc_leg((ssw >> (2 * base + 2)) & 3, (av & 1) ? 2 : 1, ils, &two_seg, base + 1, legs.cmd, &pend);
    } else if (kind == GEMB200_CONV_2QC) {
      legs.s[base] = f2qc_leg((ssw >> (2 * base)) & 3, av, ils, &two_seg, base, legs.cmd, &pend);
    } else if (kind == GEMB200_CONV_1QC) {
      act1qc[slot] = av;
    }
  }
  {
    const bool w0 = (pend & 7) != 0, w1 = (pend & 56) != 0;
    if (w0 && w1 && p.til2[0] != p.til2[1]) {
      nseg = 3;
      seg_idx[0] = p.lo_slot ? 3 : 1; seg_idx[1] = 5; seg_idx[2] = p.lo_slot ? 2 : 4;
      if (p.promote) promote_mask = pend & (p.lo_slot ? 56 : 7);
    } else if (w0 || w1) {
      nseg = 2;
      const int first = w0 ? 1 : 3;
      seg_idx[0] = first; seg_idx[1] = first + 1;
    }
  }
  const real rad = rad_per_ang<real>();
  real xs[NX];
#pragma unroll
  for (int j = 0; j < NX; ++j) xs[j] = x0[j];
  Ang<real> as = ang0;
#pragma unroll 1
  for (int seg = 0; seg < nseg; ++seg) {
    const real h = two_seg ? p.seg_len[seg_idx[seg]] : p.tau;
    const int ks = two_seg ? seg_idx[seg] : 0;
    if (seg == 2 && promote_mask) {
#pragma unroll
      for (int l = 0; l < 6; ++l) if ((promote_mask >> l) & 1) legs.s[l] = legs.cmd[l];
    }
    real i_in[6], sn, cs, sne, cse, u_in[6] = {real(0), real(0), real(0), real(0), real(0), real(0)}, u[4] = {real(0), real(0), real(0), real(0)};
    converter_currents<FAM, real>(p, kc, xs, as, i_in, &sn, &cs, &sne, &cse);
    if constexpr (FAM == kSYNC || FAM == kEESM || FAM == kSCIM || FAM == kDFIM) {
#pragma unroll
      for (int l = 0; l < (FAM == kDFIM ? 6 : 3); ++l) u_in[l] = (f2qc_out<real>(legs.s[l], i_in[l]) - real(0.5)) * u_sup;
      if constexpr (FAM == kEESM) {
        const int k1 = p.conv_kind[1];
        real v;
        if (k1 == GEMB200_CONV_4QC) v = f2qc_out<real>(legs.s[3], i_in[3]) - f2qc_out<real>(legs.s[4], -i_in[3]);
        else if (k1 == GEMB200_CONV_2QC) v = f2qc_out<real>(legs.s[3], i_in[3]);
        else v = i_in[3] >= real(0) ? (real)act1qc[1] : real(1);
        u_in[3] = v * u_sup;
      }
      real ab[2];
      t23(u_in, ab);
      if constexpr (FAM == kSCIM || FAM == kDFIM) { u[0] = ab[0]; u[1] = ab[1]; }
      else { u[0] = fm(cs, ab[0], sn * ab[1]); u[1] = fm(-sn, ab[0], cs * ab[1]); }
      if constexpr (FAM == kEESM) u[2] = u_in[3];
      if constexpr (FAM == kDFIM) {
        real rab[2];
        t23(u_in + 3, rab);
        u[2] = fm(cse, rab[0], -(sne * rab[1])); u[3] = fm(sne, rab[0], cse * rab[1]);
      }
    } else {
#pragma unroll
      for (int slot = 0; slot < 2; ++slot) {
        const int kind = p.conv_kind[slot];
        if (kind == GEMB200_CONV_NONE) continue;
        const int base = slot == 0 ? 0 : 3;
        real v;
        if (kind == GEMB200_CONV_4QC) v = f2qc_out<real>(legs.s[base], i_in[slot]) - f2qc_out<real>(legs.s[base + 1], -i_in[slot]);
        else if (kind == GEMB200_CONV_2QC) v = f2qc_out<real>(legs.s[base], i_in[slot]);
        else v = i_in[slot] >= real(0) ? (real)act1qc[slot] : real(1);
        u_in[slot] = v * u_sup;
      }
      u[0] = u_in[0];
      u[1] = (FAM == kDC2 && p.motor_kind == GEMB200_MOTOR_SHUNT_DC) ? u_in[0] : u_in[1];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) us[seg][j] = u[j];
    Model<FAM, real>::ubias(kc, u, ub[seg]);
    hs[seg] = h;
    ka[seg] = Fam<FAM>::EPS ? p.kang[mech ? 1 : 0][ks][0] * rad : real(0);
    if (seg + 1 < nseg) {
      const DF<real> wsum = integrate<FAM, real>(p, kc, xs, u, h, mech, gt);
      if constexpr (Fam<FAM>::EPS) as.advance(df_mul(wsum, p.kang[mech ? 1 : 0][ks][0], p.kang[mech ? 1 : 0][ks][1]));
    }
  }
  return nseg;
}

// The tangent pass of one step of env i: writes column c of [jac_x | jac_u] for every seed c
// into this thread's staging row, jac_x row-major at jrow[r * NX1 + c], jac_u row-major at jrow[NX1 * NX1 + r * nu + c - NX1].
template <int FAM, bool FINITE, typename real>
__device__ __forceinline__ void step_tangent(const StepParams<real>& p, const Coef<real>& kc, const real (&x0)[Fam<FAM>::NX], const Ang<real>& ang, const Act<real>& act,
                                             const unsigned i, const int nu, real* jrow) {
  using F = Fam<FAM>;
  constexpr int NX = F::NX, NX1 = NX + (F::EPS ? 1 : 0);
  const int mech = p.load_kind == GEMB200_LOAD_CONST_SPEED ? 0 : (p.load_kind == GEMB200_LOAD_EXT_SPEED ? 2 : 1);
  const real rad = rad_per_ang<real>();
  const real* gt = nullptr;
  if (mech == 2) {
    const uint32_t per = 2u * (uint32_t)p.nsteps, last = (uint32_t)p.ext_len - 1u - 2u * per;
    const uint64_t j0 = (uint64_t)p.kenv[i] * per;
    gt = p.ext_tab + (j0 < last ? (uint32_t)j0 : last);
  }
  real u_sup = p.u_sup;
  if (p.supply_kind == GEMB200_SUPPLY_AC1) {  // the phase at the start of the step (env_step advances it afterwards)
    Ang<real> ph;
    ph.load(p.sup_phase, i);
    real sph, cph;
    ph.sincos(&sph, &cph);
    u_sup = p.sup_amp * sph;
  }
  // ---------------- primal, column-independent: dq rotation of the action, converter voltages and their gains ----------------
  real a[GEMB200_MAX_ACT];
#pragma unroll
  for (int j = 0; j < GEMB200_MAX_ACT; ++j) a[j] = act.a[j];
  real sa = real(0), ca = real(1), abq[2] = {real(0), real(0)};  // rotation of the dq action and the rotated (alpha-beta) action
  const bool dq = (FAM == kSYNC || FAM == kEESM || FAM == kSCIM) && !FINITE && p.action_dq == 1;
  real r2f = real(0);
  if constexpr (!FINITE && (FAM == kSYNC || FAM == kEESM || FAM == kSCIM)) {
    if (dq) {
      if constexpr (FAM == kSCIM) {
        r2f = fm(x0[3], x0[3], x0[4] * x0[4]);
        if (r2f > real(0)) { const real ir = Num<real>::rsqrt(r2f); ca = x0[3] * ir; sa = x0[4] * ir; }
      } else {
        ang.sincos_adv(p.adv_k * x0[0], &sa, &ca);
      }
      abq[0] = fm(ca, a[0], -(sa * a[1])); abq[1] = fm(sa, a[0], ca * a[1]);
      const real ue = a[2];
      t32(abq, a);
      if constexpr (FAM == kEESM) a[3] = ue;
    }
  }
  // currents seen by the converter (their signs select the branches)
  real i_in[6], sn, cs, sne, cse;
  converter_currents<FAM, real>(p, kc, x0, ang, i_in, &sn, &cs, &sne, &cse);
  // per switching segment: solver-frame voltages, their voltage terms, length and angle factor (continuous converters: one segment)
  constexpr int MS = FINITE ? 3 : 1;
  real usg[MS][4], ubg[MS][4], hsg[MS], kag[MS];
  int nseg = 1;
  real g[6] = {real(0), real(0), real(0), real(0), real(0), real(0)};  // continuous: du_in[l] = g[l] da[l]
  if constexpr (FINITE) {
    nseg = finite_segments<FAM, real>(p, kc, x0, ang, act, i, u_sup, mech, gt, usg, ubg, hsg, kag);
  } else {
    const bool interlock = p.til2[0] != real(0) || p.til2[1] != real(0);
    const real tot = p.tot2[0], tot1 = p.tot2[1];
    real u_in[6] = {real(0), real(0), real(0), real(0), real(0), real(0)};
    real* us = usg[0];
#pragma unroll
    for (int j = 0; j < 4; ++j) us[j] = real(0);
    if constexpr (FAM == kSYNC || FAM == kEESM || FAM == kSCIM || FAM == kDFIM) {
#pragma unroll
      for (int l = 0; l < (FAM == kDFIM ? 6 : 3); ++l) {
        const real pre = real(0.5) * (a[l] + real(1));
        real v = clamp01(pre);
        real gl = real(0.5) * clamp01_t(pre);
        if (interlock) { const real t = l < 3 ? tot : tot1; gl *= clamp01_t(fm(-sgn(i_in[l]), t, v)); v = c2qc(v, i_in[l], t); }
        g[l] = gl * u_sup;
        u_in[l] = (v - real(0.5)) * u_sup;
      }
      if constexpr (FAM == kEESM) {
        const int k1 = p.conv_kind[1];
        u_in[3] = cont_qc(k1, a[3], i_in[3], tot1) * u_sup;
        g[3] = cont_qc_t(k1, a[3], i_in[3], tot1) * u_sup;
      }
      real ab[2];
      t23(u_in, ab);
      if constexpr (FAM == kSCIM || FAM == kDFIM) { us[0] = ab[0]; us[1] = ab[1]; }
      else { us[0] = fm(cs, ab[0], sn * ab[1]); us[1] = fm(-sn, ab[0], cs * ab[1]); }
      if constexpr (FAM == kEESM) us[2] = u_in[3];
      if constexpr (FAM == kDFIM) {
        real rab[2];
        t23(u_in + 3, rab);
        us[2] = fm(cse, rab[0], -(sne * rab[1])); us[3] = fm(sne, rab[0], cse * rab[1]);
      }
    } else {
#pragma unroll
      for (int slot = 0; slot < 2; ++slot) {
        const int kind = p.conv_kind[slot];
        if (kind == GEMB200_CONV_NONE) continue;
        const real t = slot == 0 ? tot : tot1;
        u_in[slot] = cont_qc(kind, a[slot], i_in[slot], t) * u_sup;
        g[slot] = cont_qc_t(kind, a[slot], i_in[slot], t) * u_sup;
      }
      us[0] = u_in[0];
      us[1] = (FAM == kDC2 && p.motor_kind == GEMB200_MOTOR_SHUNT_DC) ? u_in[0] : u_in[1];
    }
    Model<FAM, real>::ubias(kc, us, ubg[0]);
    hsg[0] = p.tau;
    kag[0] = F::EPS ? p.kang[mech ? 1 : 0][0][0] * rad : real(0);  // d eps (rad) / d wsum
  }
  const real adv = p.adv_k * rad;
  // ---------------- one tangent pass per seed column ----------------
  const int ncol = NX1 + nu;
#pragma unroll 1
  for (int c = 0; c < ncol; ++c) {
    real x[NX], dx[NX];
#pragma unroll
    for (int j = 0; j < NX; ++j) { x[j] = x0[j]; dx[j] = c == j ? real(1) : real(0); }
    real de = (F::EPS && c == NX) ? real(1) : real(0);  // tangent of the angle (rad), seeded in its own column
    real da[GEMB200_MAX_ACT];
#pragma unroll
    for (int j = 0; j < GEMB200_MAX_ACT; ++j) da[j] = c - NX1 == j ? real(1) : real(0);
    if constexpr (!FINITE && (FAM == kSYNC || FAM == kEESM || FAM == kSCIM)) {
      if (dq) {  // a_abc = T32 rot(theta) a_dq: theta = eps + angle_advance tau p omega, or (SCIM) the field angle of the flux
        real dth;
        if constexpr (FAM == kSCIM) dth = r2f > real(0) ? (x0[3] * dx[4] - x0[4] * dx[3]) / r2f : real(0);
        else dth = fm(adv, dx[0], de);
        const real dab[2] = {fm(ca, da[0], -(sa * da[1])) - dth * abq[1], fm(sa, da[0], ca * da[1]) + dth * abq[0]};
        const real due = da[2];
        t32(dab, da);
        if constexpr (FAM == kEESM) da[3] = due;
      }
    }
    // continuous converters: the action part of the voltages (one segment); finite converters have none
    real dab[2] = {real(0), real(0)}, drab[2] = {real(0), real(0)}, dq3[2] = {real(0), real(0)};
    if constexpr (!FINITE) {
      real du[6];
#pragma unroll
      for (int l = 0; l < 6; ++l) du[l] = g[l] * da[l];
      if constexpr (FAM == kSYNC || FAM == kEESM || FAM == kSCIM || FAM == kDFIM) {
        t23(du, dab);
        if constexpr (FAM == kEESM) dq3[0] = du[3];
        if constexpr (FAM == kDFIM) t23(du + 3, drab);
      } else {
        dq3[0] = du[0];
        dq3[1] = (FAM == kDC2 && p.motor_kind == GEMB200_MOTOR_SHUNT_DC) ? du[0] : du[1];
      }
    }
    real dws = real(0);
#pragma unroll 1
    for (int seg = 0; seg < nseg; ++seg) {
      // segment seg rotates its voltages with the angle at its start: the angle's tangent de enters through the rotation
      const real* us = usg[seg];
      real dus[4] = {real(0), real(0), real(0), real(0)};
      if constexpr (FAM == kSCIM || FAM == kDFIM) { dus[0] = dab[0]; dus[1] = dab[1]; }
      else if constexpr (FAM == kSYNC || FAM == kEESM) { dus[0] = fm(cs, dab[0], sn * dab[1]) + de * us[1]; dus[1] = fm(-sn, dab[0], cs * dab[1]) - de * us[0]; }
      else { dus[0] = dq3[0]; dus[1] = dq3[1]; }
      if constexpr (FAM == kEESM) dus[2] = dq3[0];
      if constexpr (FAM == kDFIM) {  // rotor voltages rotated by +eps
        dus[2] = fm(cse, drab[0], -(sne * drab[1])) - de * us[3]; dus[3] = fm(sne, drab[0], cse * drab[1]) + de * us[2];
      }
      real dub[4];
      Model<FAM, real>::ubias(kc, dus, dub);
      dws = integrate_t<FAM, real>(p, kc, x, dx, ubg[seg], dub, hsg[seg], mech, gt);
      if constexpr (F::EPS) de = fm(kag[seg], dws, de);  // the wrap to (-pi, pi] has derivative 1
    }
    if (c < NX1) {
#pragma unroll
      for (int r = 0; r < NX; ++r) jrow[r * NX1 + c] = dx[r];
      if constexpr (F::EPS) jrow[NX * NX1 + c] = de;
    } else {
      real* ju = jrow + NX1 * NX1 + (c - NX1);
#pragma unroll
      for (int r = 0; r < NX; ++r) ju[r * nu] = dx[r];
      if constexpr (F::EPS) ju[NX * nu] = de;
    }
  }
}

// Coalesced copy of the warp's staged rows (width w words, stride `stride` in shared memory) to `dst` (the warp's first env's row)
template <typename real>
__device__ __forceinline__ void warp_store_jac(real* __restrict__ dst, const real* __restrict__ rows, int stride, int w, int valid, int lane) {
  const int total = valid * w;
#pragma unroll 1
  for (int k = lane; k < total; k += 32) { const int e = k / w; dst[k] = rows[e * stride + (k - e * w)]; }
}

// The K-step loop: rollout_loop with record_every = 1 plus the tangent pass and the Jacobian stores of every step
template <int FAM, bool FINITE, typename real, int NREF, bool ENVP>
__device__ __forceinline__ void jac_loop(const StepParams<real>& p, const JacOut& jo, CoefArg<real, ENVP> kc, const unsigned i, const bool active, real (&x)[Fam<FAM>::NX],
                                         Ang<real>& ang, real (&rv)[NREF > 0 ? NREF : 1], real (&rs)[NREF > 0 ? NREF : 1], uint32_t (&rend)[NREF > 0 ? NREF : 1],
                                         bool& cold_dirty, real* rows, real* row, real* jrows, real* jrow, const int jstride, const int lane, const int stride) {
  constexpr int NX1 = Fam<FAM>::NX + (Fam<FAM>::EPS ? 1 : 0);
  const int K = p.roll_steps;
  const int nu = FINITE ? 0 : jo.nu;
  const size_t n = (size_t)(unsigned)p.n;
  Out<real> out = make_out<NREF, false, real>(p, i, lane, p.n_obs);
  ClockArg<ENVP> ck = clock_of(p);
  if constexpr (ENVP) ck = id_clock(p, clock_of(p), active ? i : (unsigned)p.env_begin);
  const char* act = action_cursor<FAM, FINITE, real, false>(p, p.action, i);
  WalkCache wc{};
  Act<real> a_next{};
  if (active) a_next = load_action<FAM, FINITE, real, false>(p, act);
  constexpr bool kFeed = NREF > 0;
  const bool feed = kFeed && p.ref_feed != nullptr;
  const real* fc = nullptr;
  real f_next[NREF > 0 ? NREF : 1];
  if constexpr (kFeed) {
    if (feed) { fc = feed_cursor<NREF, false, real>(p, i); if (active) load_feed<NREF, false, real>(p, fc, f_next); }
  }
  const size_t warp_env0 = i - lane;
  real* jx = static_cast<real*>(jo.jx) + warp_env0 * (NX1 * NX1);
  real* ju = nu > 0 && jo.ju ? static_cast<real*>(jo.ju) + warp_env0 * (size_t)(NX1 * nu) : nullptr;
#pragma unroll 1
  for (int k = 0; k < K; ++k) {
    const Act<real> a_cur = a_next;
    act += p.roll_act_inc;
    if (active && k + 1 < K) a_next = load_action<FAM, FINITE, real, false>(p, act);
    if constexpr (kFeed) {
      if (feed) {
#pragma unroll
        for (int r = 0; r < NREF; ++r) rv[r] = f_next[r];
        fc += n * NREF;
        if (active && k + 1 < K) load_feed<NREF, false, real>(p, fc, f_next);
      }
    }
    if (active) step_tangent<FAM, FINITE, real>(p, kc, x, ang, a_cur, i, nu, jrow);
    __syncwarp();
    warp_store_jac(jx, jrows, jstride, NX1 * NX1, out.valid, lane);
    if (ju) warp_store_jac(ju, jrows + NX1 * NX1, jstride, NX1 * nu, out.valid, lane);
    jx += n * (NX1 * NX1);
    if (ju) ju += n * (size_t)(NX1 * nu);
    env_step<FAM, FINITE, real, NREF, false, false, false, false, ENVP>(p, kc, ck, out, true, a_cur, i, active, x, ang, rv, rs, rend, cold_dirty, wc, rows, row, lane,
                                                                        stride);
    __syncwarp();  // both staging areas are reused by the next step
    out.obs = byte_add(out.obs, p.roll_obs_inc); out.ref = byte_add(out.ref, p.roll_ref_inc);
    out.rew = byte_add(out.rew, p.roll_rew_inc); out.term = byte_add(out.term, p.roll_term_inc);
    ck.kstep += 1u;
    ck.gstep_lo += 1u;
    if (ck.gstep_lo == 0u) ck.gstep_hi += 1u;
  }
}

// The rollout-Jacobian kernel: rollout_kernel (row-per-env layout, general or ENVP coefficients, no dead time) with jac_loop.  Dynamic shared
// memory: the observation rows of the block, then its Jacobian rows (jstride words per env).
template <int FAM, bool FINITE, typename real, int NREF, bool ENVP>
__global__ void __launch_bounds__(GEMB200_BLOCK, (sizeof(real) == 4 ? GEMB200_MINBLOCKS_JAC : GEMB200_MINBLOCKS_JAC_F64))
jacobian_kernel(const __grid_constant__ StepParams<real> p, const __grid_constant__ JacOut jo, const int jstride) {
  using F = Fam<FAM>;
  constexpr int NX = F::NX, NH = hot_words(NX, NREF), NC = cold_words(NX, NREF);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  real* smem = reinterpret_cast<real*>(smem_raw);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int stride = p.row_stride;
  real* rows = smem + warp * (32 * stride);
  real* row = rows + lane * stride;
  real* jrows = smem + blockDim.x * stride + warp * (32 * jstride);
  real* jrow = jrows + lane * jstride;
  const unsigned i = (unsigned)p.env_begin + blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned n = (unsigned)p.n;
  const bool active = i < (unsigned)p.env_end;
  const int mech = p.load_kind != GEMB200_LOAD_CONST_SPEED;
  real hot[NH > 0 ? NH : 1], cold[NC];
  Ang<real> ang;
  real x[NX], rv[NREF > 0 ? NREF : 1], rs[NREF > 0 ? NREF : 1];
  uint32_t rend[NREF > 0 ? NREF : 1];
  bool cold_dirty = mech;
  if (active) {
    if constexpr (NH > 0) load_words<NH, real>(p.st, i, n, hot);
    load_words<NC, real>(p.stc, i, n, cold);
    ang.set(p.init_ang);
    if constexpr (F::EPS) ang.load(p.eps, i);
    unpack_records<NX, NREF, real>(hot, cold, x, rv, rs, rend);
  }
  if constexpr (ENVP) {
    Coef<real> kl;
    load_coef<FAM, real>(p, active ? i : (unsigned)p.env_begin, mech != 0, kl);
    jac_loop<FAM, FINITE, real, NREF, true>(p, jo, kl, i, active, x, ang, rv, rs, rend, cold_dirty, rows, row, jrows, jrow, jstride, lane, stride);
  } else {
    jac_loop<FAM, FINITE, real, NREF, false>(p, jo, p.k, i, active, x, ang, rv, rs, rend, cold_dirty, rows, row, jrows, jrow, jstride, lane, stride);
  }
  if (active) {
    pack_records<NX, NREF, real>(hot, cold, x, rv, rs, rend);
    if constexpr (NH > 0) store_words<NH, real>(p.st, i, n, hot);
    if (cold_dirty) store_words<NC, real>(p.stc, i, n, cold);
    if constexpr (F::EPS) ang.store(p.eps, i);
  }
}

}  // namespace gemb200
