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

// Parameter sensitivities: adds to d the derivative of Model<FAM>::rhs along a coefficient tangent tk at fixed (x, u), u = the solver-frame
// voltages.  The electrical rows and the voltage terms are linear in the coefficients (the DFIM's rotor voltages enter without one); the
// mechanical row inv_j (T(tq, x) - T_L(a, b, c, omega_lin)) takes the product rule, on the static-friction branch the primal takes.
template <int FAM, typename real>
__device__ __forceinline__ void coef_rhs_t(const Coef<real>& kc, const Coef<real>& tk, const real* x, const real* u, int mech, real* d) {
  constexpr int NX = Fam<FAM>::NX;
  real ub[4], e[NX];
  Model<FAM, real>::ubias(tk, u, ub);
  if constexpr (FAM == kDFIM) { ub[2] = real(0); ub[3] = real(0); }
  Model<FAM, real>::rhs(tk, real(0), x, ub, 0, real(0), e);
#pragma unroll
  for (int j = 1; j < NX; ++j) d[j] += e[j];
  if (mech == 1) {
    const real w = x[0], sign = sgn(w);
    const bool slide = Num<real>::abs(w) > kc.omega_lim;
    const real tl = fm(sign * kc.load_c * w, w, fm(kc.load_b, w, slide ? sign * kc.load_a : kc.omega_lin * w));
    const real dtl = fm(sign * tk.load_c * w, w, fm(tk.load_b, w, slide ? sign * tk.load_a : tk.omega_lin * w));
    d[0] += tk.inv_j * (Model<FAM, real>::torque(kc, x) - tl) + kc.inv_j * (Model<FAM, real>::torque(tk, x) - dtl);
  }
}

// rk4_step with its tangent: x, dx advance together; dws accumulates the tangent of the omega sum with the weights 1-2-2-1.
// PS (parameter sensitivities): the tangent also carries the coefficient tangent tk at the solver-frame voltages us
template <int FAM, typename real, bool PS = false>
__device__ __forceinline__ void rk4_step_t(const StepParams<real>& p, const Coef<real>& kc, real* x, real* dx, const real* ub, const real* dub, real h, int mech,
                                           real& dws, const real* gt, const Coef<real>* tk = nullptr, const real* us = nullptr) {
  constexpr int NX = Fam<FAM>::NX;
  const real hh = real(0.5) * h, h6 = h * real(1.0 / 6.0);
  const real g0 = mech == 2 ? gt[0] : real(0), g1 = mech == 2 ? gt[1] : real(0), g2 = mech == 2 ? gt[2] : real(0);
  real k[NX], dk[NX], acc[NX], dacc[NX], xt[NX], dxt[NX];
  Model<FAM, real>::rhs(kc, p.ext_inv_tau, x, ub, mech, g0, k);
  Tan<FAM, real>::rhs(kc, p.ext_inv_tau, x, dx, dub, mech, dk);
  if constexpr (PS) coef_rhs_t<FAM, real>(kc, *tk, x, us, mech, dk);
  if (mech) dws += dx[0];
  acc[0] = real(0); dacc[0] = real(0); xt[0] = x[0]; dxt[0] = dx[0];
#pragma unroll
  for (int j = 0; j < NX; ++j) if (j > 0 || mech) { acc[j] = k[j]; dacc[j] = dk[j]; xt[j] = fm(hh, k[j], x[j]); dxt[j] = fm(hh, dk[j], dx[j]); }
  Model<FAM, real>::rhs(kc, p.ext_inv_tau, xt, ub, mech, g1, k);
  Tan<FAM, real>::rhs(kc, p.ext_inv_tau, xt, dxt, dub, mech, dk);
  if constexpr (PS) coef_rhs_t<FAM, real>(kc, *tk, xt, us, mech, dk);
  if (mech) dws += real(2) * dxt[0];
#pragma unroll
  for (int j = 0; j < NX; ++j) if (j > 0 || mech) { acc[j] = fm(real(2), k[j], acc[j]); dacc[j] = fm(real(2), dk[j], dacc[j]); xt[j] = fm(hh, k[j], x[j]); dxt[j] = fm(hh, dk[j], dx[j]); }
  Model<FAM, real>::rhs(kc, p.ext_inv_tau, xt, ub, mech, g1, k);
  Tan<FAM, real>::rhs(kc, p.ext_inv_tau, xt, dxt, dub, mech, dk);
  if constexpr (PS) coef_rhs_t<FAM, real>(kc, *tk, xt, us, mech, dk);
  if (mech) dws += real(2) * dxt[0];
#pragma unroll
  for (int j = 0; j < NX; ++j) if (j > 0 || mech) { acc[j] = fm(real(2), k[j], acc[j]); dacc[j] = fm(real(2), dk[j], dacc[j]); xt[j] = fm(h, k[j], x[j]); dxt[j] = fm(h, dk[j], dx[j]); }
  Model<FAM, real>::rhs(kc, p.ext_inv_tau, xt, ub, mech, g2, k);
  Tan<FAM, real>::rhs(kc, p.ext_inv_tau, xt, dxt, dub, mech, dk);
  if constexpr (PS) coef_rhs_t<FAM, real>(kc, *tk, xt, us, mech, dk);
  if (mech) dws += dxt[0];
#pragma unroll
  for (int j = 0; j < NX; ++j) if (j > 0 || mech) { x[j] = fm(h6, acc[j] + k[j], x[j]); dx[j] = fm(h6, dacc[j] + dk[j], dx[j]); }
}

// integrate with its tangent over one segment; returns the tangent of the omega sum (the angle advances by kang * wsum)
template <int FAM, typename real, bool PS = false>
__device__ __forceinline__ real integrate_t(const StepParams<real>& p, const Coef<real>& kc, real* x, real* dx, const real* ub, const real* dub, real h_seg, int mech,
                                            const real* gt, const Coef<real>* tk = nullptr, const real* us = nullptr) {
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
      if constexpr (PS) coef_rhs_t<FAM, real>(kc, *tk, x, us, mech, dd);
      if (mech) dws += dx[0];
#pragma unroll
      for (int j = 0; j < NX; ++j) if (j > 0 || mech) { x[j] = fm(d[j], h, x[j]); dx[j] = fm(dd[j], h, dx[j]); }
    }
    return dws;
  }
#pragma unroll 1
  for (int s = 0; s < ns; ++s) rk4_step_t<FAM, real, PS>(p, kc, x, dx, ub, dub, h, mech, dws, gt + 2 * s, tk, us);
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

// The reward-row input of the tangent pass (return_grad_kernel): the step's supply voltage and speed-profile cursor, read before env_step
// advanced them, and this thread's coefficient row cb[b] = d(g^k r_k) / d s_b over the state-vector entries b in wmask (the weighted ones)
template <typename real> struct RwTan {
  real u_sup;
  const real* gt;
  const real* cb;
  uint32_t wmask;
};

// the supply voltage of the step that starts now (the phase env_step advances afterwards) and this env's speed-profile cursor
template <typename real> __device__ __forceinline__ real step_u_sup(const StepParams<real>& p, const unsigned i) {
  real u_sup = p.u_sup;
  if (p.supply_kind == GEMB200_SUPPLY_AC1) {
    Ang<real> ph;
    ph.load(p.sup_phase, i);
    real sph, cph;
    ph.sincos(&sph, &cph);
    u_sup = p.sup_amp * sph;
  }
  return u_sup;
}
template <typename real> __device__ __forceinline__ const real* step_gt(const StepParams<real>& p, const unsigned i) {
  if (p.load_kind != GEMB200_LOAD_EXT_SPEED) return nullptr;
  const uint32_t per = 2u * (uint32_t)p.nsteps, last = (uint32_t)p.ext_len - 1u - 2u * per;
  const uint64_t j0 = (uint64_t)p.kenv[i] * per;
  return p.ext_tab + (j0 < last ? (uint32_t)j0 : last);
}

// v -> rot(-th) v = {c v0 + s v1, -s v0 + c v1} (o: its primal) and its tangent for dv and dth
template <typename real> __device__ __forceinline__ void rotm_t(real c, real s, const real* v, const real* dv, real dth, real* d) {
  const real o0 = fm(c, v[0], s * v[1]), o1 = fm(-s, v[0], c * v[1]);
  d[0] = fm(c, dv[0], s * dv[1]) + dth * o1;
  d[1] = fm(-s, dv[0], c * dv[1]) - dth * o0;
}

// Tangent of g^k r_k for one seed column, continuous converters: sum over the weighted entries b of cb[b] * d s_b, s = env_step's state
// vector after the step (normalised).  x, dx: the state after the step and its tangent; de0, de1: the angle's tangent at the start and
// the end of the step (rad); dphi: the field angle's (SCIM / DFIM, from the state at the start); du: the converter voltages' tangent;
// dus: the solver-frame voltages'; us, rab: their primal values (rab: the DFIM's alpha-beta rotor voltages); sn, cs: the rotation of the
// synchronous motors' currents; snf, csf: the field angle; sne, cse: the DFIM's electrical angle.
template <int FAM, typename real>
__device__ __forceinline__ real reward_t(const StepParams<real>& p, const Coef<real>& kc, const RwTan<real>& rw, const real* x, const real* dx, real de0, real de1,
                                         real dphi, const real* du, const real* dus, const real* us, const real* rab, real sn, real cs, real snf, real csf,
                                         real sne, real cse) {
  const uint32_t wm = rw.wmask;
  const real* cb = rw.cb;
  real dr = real(0);
  auto add = [&](int b, real v) { if ((wm >> b) & 1u) dr = fm(cb[b], v * p.inv_lim[b], dr); };
  auto add_abc = [&](int b, const real* dab) {  // three entries b..b+2 = T32 of an alpha-beta pair
    if ((wm >> b) & 7u) { real t[3]; t32(dab, t); add(b, t[0]); add(b + 1, t[1]); add(b + 2, t[2]); }
  };
  add(0, dx[0]);
  if constexpr (FAM == kDC1) add(1, (real(2) * kc.tq[1] * x[1] + kc.tq[0]) * dx[1]);
  else if constexpr (FAM == kDC2) add(1, kc.tq[0] * (dx[1] * x[2] + x[1] * dx[2]));
  else if constexpr (FAM == kSYNC) add(1, kc.tq[1] * dx[1] * x[2] + (kc.tq[1] * x[1] + kc.tq[0]) * dx[2]);
  else if constexpr (FAM == kEESM) add(1, (kc.tq[0] * dx[3] + kc.tq[1] * dx[1]) * x[2] + (kc.tq[0] * x[3] + kc.tq[1] * x[1]) * dx[2]);
  else add(1, kc.tq[0] * (dx[3] * x[2] + x[3] * dx[2] - dx[4] * x[1] - x[4] * dx[1]));
  const real deps = de1 * (p.eps_out_scale / rad_per_ang<real>());  // the angle entry: inv_lim = 1, scaled by eps_out_scale
  if constexpr (FAM == kDC1) {
    add(2, dx[1]); add(3, du[0]);
  } else if constexpr (FAM == kDC2) {
    add(2, dx[1]); add(3, dx[2]); add(4, du[0]);
    if (p.motor_kind == GEMB200_MOTOR_SHUNT_DC) { if ((wm >> 6) & 1u) dr = fm(cb[6], fm(dx[1], p.inv_lim[2], dx[2] * p.inv_lim[3]), dr); }
    else add(5, du[1]);
  } else if constexpr (FAM == kSYNC || FAM == kEESM) {
    // i_abc = T32 q(i_dq, eps at the start of the step)
    const real ab[2] = {fm(cs, x[1], -(sn * x[2])), fm(sn, x[1], cs * x[2])};
    const real dab[2] = {fm(cs, dx[1], -(sn * dx[2])) - de0 * ab[1], fm(sn, dx[1], cs * dx[2]) + de0 * ab[0]};
    add_abc(2, dab);
    add(5, dx[1]); add(6, dx[2]);
    if constexpr (FAM == kSYNC) {
      add(7, du[0]); add(8, du[1]); add(9, du[2]); add(10, dus[0]); add(11, dus[1]);
      if ((wm >> 12) & 1u) dr = fm(cb[12], deps, dr);
    } else {
      add(7, dx[3]); add(8, du[0]); add(9, du[1]); add(10, du[2]); add(11, dus[0]); add(12, dus[1]); add(13, dus[2]);
      if ((wm >> 14) & 1u) dr = fm(cb[14], deps, dr);
    }
  } else {  // SCIM / DFIM: dq quantities in the field frame of the start of the step
    add_abc(2, dx + 1);
    real d2[2];
    rotm_t(csf, snf, x + 1, dx + 1, dphi, d2);
    add(5, d2[0]); add(6, d2[1]);
    const real uab[2] = {us[0], us[1]};  // the stator voltages in alpha-beta (the solver frame)
    real duab[2];
    t23(du, duab);
    if constexpr (FAM == kSCIM) {
      add(7, du[0]); add(8, du[1]); add(9, du[2]);
      rotm_t(csf, snf, uab, duab, dphi, d2);
      add(10, d2[0]); add(11, d2[1]);
      if ((wm >> 12) & 1u) dr = fm(cb[12], deps, dr);
    } else {
      // rotor currents (alpha-beta), in the rotor frame (rot(-eps)) and in the field frame (rot(-phi))
      const real ir[2] = {fm(kc.c[8], x[3], -(kc.c[9] * x[1])), fm(kc.c[8], x[4], -(kc.c[9] * x[2]))};
      const real dir[2] = {fm(kc.c[8], dx[3], -(kc.c[9] * dx[1])), fm(kc.c[8], dx[4], -(kc.c[9] * dx[2]))};
      if ((wm >> 7) & 7u) { rotm_t(cse, sne, ir, dir, de0, d2); add_abc(7, d2); }
      rotm_t(csf, snf, ir, dir, dphi, d2);
      add(10, d2[0]); add(11, d2[1]);
      add(12, du[0]); add(13, du[1]); add(14, du[2]);
      rotm_t(csf, snf, uab, duab, dphi, d2);
      add(15, d2[0]); add(16, d2[1]);
      add(17, du[3]); add(18, du[4]); add(19, du[5]);
      // rotor voltages rot(-(phi - eps)) of their alpha-beta pair
      const real cfe = fm(csf, cse, snf * sne), sfe = fm(snf, cse, -(csf * sne));
      real durab[2];
      t23(du + 3, durab);
      rotm_t(cfe, sfe, rab, durab, dphi - de0, d2);
      add(20, d2[0]); add(21, d2[1]);
      if ((wm >> 22) & 1u) dr = fm(cb[22], deps, dr);
    }
  }
  return dr;
}

// Parameter sensitivities: the words of the coefficient block (Coef, kCoefWords) that family FAM reads — load_coef's c and tq words and the
// six load / inertia words — kept per parameter column in the staging row; word w of that compact list is word ps_word<FAM>(w) of Coef
template <int FAM> __host__ __device__ constexpr int ps_ncw() { return FAM == kDC1 ? 4 : (FAM == kDC2 ? 5 : (FAM == kSYNC ? 7 : (FAM == kEESM ? 14 : 10))); }
template <int FAM> __host__ __device__ constexpr int ps_ntq() { return (FAM == kDC2 || FAM == kSCIM || FAM == kDFIM) ? 1 : 2; }
template <int FAM> __host__ __device__ constexpr int ps_words() { return ps_ncw<FAM>() + ps_ntq<FAM>() + 6; }
template <int FAM> __host__ __device__ constexpr int ps_word(int w) { return w < ps_ncw<FAM>() ? w : (w < ps_ncw<FAM>() + ps_ntq<FAM>() ? 20 + w - ps_ncw<FAM>() : 24 + w - ps_ncw<FAM>() - ps_ntq<FAM>()); }
template <int FAM, typename real>
__device__ __forceinline__ void ps_coef(const real* t, Coef<real>& tk) {
#pragma unroll
  for (int w = 0; w < ps_ncw<FAM>(); ++w) tk.c[w] = t[w];
#pragma unroll
  for (int w = 0; w < ps_ntq<FAM>(); ++w) tk.tq[w] = t[ps_ncw<FAM>() + w];
  const real* m = t + ps_ncw<FAM>() + ps_ntq<FAM>();
  tk.load_a = m[0]; tk.load_b = m[1]; tk.load_c = m[2]; tk.inv_j = m[3]; tk.omega_lim = m[4]; tk.omega_lin = m[5];
}

// The tangent pass of one step of env i: writes column c of [jac_x | jac_u] for every seed c
// into this thread's staging row, jac_x row-major at jrow[r * NX1 + c], jac_u row-major at jrow[NX1 * NX1 + r * nu + c - NX1].
// RW (continuous converters, return_grad_kernel): also d(g^k r_k) / d(x, a) at jrow[NX1 * (NX1 + nu) + c], from the reward-row input rw;
// the supply voltage and the speed-profile cursor then come from rw too (the pass runs after env_step, on copies of the pre-step state).
// PS (param_sens_kernel): nu = n_p parameter columns instead; jrow holds S = d x / d theta row-major [NX1][n_p], and column c's pass is seeded
// with S[:, c], no action tangent and the coefficient tangent tks[c * ps_words<FAM>() ..] (ps_coef), and overwrites S[:, c] with
// S_{k+1}[:, c] = J_x S_k[:, c] + d x_{k+1} / d theta_c.
template <int FAM, bool FINITE, typename real, bool RW = false, bool PS = false>
__device__ __forceinline__ void step_tangent(const StepParams<real>& p, const Coef<real>& kc, const real (&x0)[Fam<FAM>::NX], const Ang<real>& ang, const Act<real>& act,
                                             const unsigned i, const int nu, real* jrow, const RwTan<real>* rw = nullptr, const real* tks = nullptr) {
  static_assert(!(RW && FINITE), "return gradients: continuous converters only");
  static_assert(!(RW && PS), "return gradients and parameter sensitivities are separate kernels");
  using F = Fam<FAM>;
  constexpr int NX = F::NX, NX1 = NX + (F::EPS ? 1 : 0);
  const int mech = p.load_kind == GEMB200_LOAD_CONST_SPEED ? 0 : (p.load_kind == GEMB200_LOAD_EXT_SPEED ? 2 : 1);
  const real rad = rad_per_ang<real>();
  const real* gt = nullptr;
  real u_sup;
  if constexpr (RW) {
    gt = rw->gt;
    u_sup = rw->u_sup;
  } else {
    if (mech == 2) {
      const uint32_t per = 2u * (uint32_t)p.nsteps, last = (uint32_t)p.ext_len - 1u - 2u * per;
      const uint64_t j0 = (uint64_t)p.kenv[i] * per;
      gt = p.ext_tab + (j0 < last ? (uint32_t)j0 : last);
    }
    u_sup = p.u_sup;
    if (p.supply_kind == GEMB200_SUPPLY_AC1) {  // the phase at the start of the step (env_step advances it afterwards)
      Ang<real> ph;
      ph.load(p.sup_phase, i);
      real sph, cph;
      ph.sincos(&sph, &cph);
      u_sup = p.sup_amp * sph;
    }
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
  real rab_p[2] = {real(0), real(0)};  // RW, DFIM: the alpha-beta rotor voltages
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
        if constexpr (RW) { rab_p[0] = rab[0]; rab_p[1] = rab[1]; }
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
  real snf = real(0), csf = real(1), r2p = real(0);  // RW, SCIM / DFIM: the field angle at the start of the step
  if constexpr (RW && (FAM == kSCIM || FAM == kDFIM)) {
    r2p = fm(x0[3], x0[3], x0[4] * x0[4]);
    if (r2p > real(0)) { const real ir = Num<real>::rsqrt(r2p); csf = x0[3] * ir; snf = x0[4] * ir; }
  }
  // ---------------- one tangent pass per seed column ----------------
  const int ncol = PS ? nu : NX1 + nu;
#pragma unroll 1
  for (int c = 0; c < ncol; ++c) {
    real x[NX], dx[NX];
    real de;  // tangent of the angle (rad), seeded in its own column
    Coef<real> tk{};  // PS: the column's coefficient tangent
    if constexpr (PS) {
#pragma unroll
      for (int j = 0; j < NX; ++j) { x[j] = x0[j]; dx[j] = jrow[j * nu + c]; }
      de = F::EPS ? jrow[NX * nu + c] : real(0);
      ps_coef<FAM, real>(tks + c * ps_words<FAM>(), tk);
    } else {
#pragma unroll
      for (int j = 0; j < NX; ++j) { x[j] = x0[j]; dx[j] = c == j ? real(1) : real(0); }
      de = (F::EPS && c == NX) ? real(1) : real(0);
    }
    const real de0 = de;
    real dphi = real(0);  // RW: the field angle's tangent
    if constexpr (RW && (FAM == kSCIM || FAM == kDFIM)) dphi = r2p > real(0) ? (x0[3] * dx[4] - x0[4] * dx[3]) / r2p : real(0);
    real da[GEMB200_MAX_ACT];
#pragma unroll
    for (int j = 0; j < GEMB200_MAX_ACT; ++j) da[j] = (!PS && c - NX1 == j) ? real(1) : real(0);
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
    real dui[6], dus0[4];  // RW: the converter and solver-frame voltages' tangents
    if constexpr (!FINITE) {
      real du[6];
#pragma unroll
      for (int l = 0; l < 6; ++l) du[l] = g[l] * da[l];
      if constexpr (RW) {
#pragma unroll
        for (int l = 0; l < 6; ++l) dui[l] = du[l];
      }
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
      if constexpr (RW) {
#pragma unroll
        for (int j = 0; j < 4; ++j) dus0[j] = dus[j];
      }
      real dub[4];
      Model<FAM, real>::ubias(kc, dus, dub);
      dws = integrate_t<FAM, real, PS>(p, kc, x, dx, ubg[seg], dub, hsg[seg], mech, gt, &tk, usg[seg]);
      if constexpr (F::EPS) de = fm(kag[seg], dws, de);  // the wrap to (-pi, pi] has derivative 1
    }
    if constexpr (PS) {
#pragma unroll
      for (int r = 0; r < NX; ++r) jrow[r * nu + c] = dx[r];
      if constexpr (F::EPS) jrow[NX * nu + c] = de;
    } else if (c < NX1) {
#pragma unroll
      for (int r = 0; r < NX; ++r) jrow[r * NX1 + c] = dx[r];
      if constexpr (F::EPS) jrow[NX * NX1 + c] = de;
    } else {
      real* ju = jrow + NX1 * NX1 + (c - NX1);
#pragma unroll
      for (int r = 0; r < NX; ++r) ju[r * nu] = dx[r];
      if constexpr (F::EPS) ju[NX * nu] = de;
    }
    if constexpr (RW)
      jrow[NX1 * (NX1 + nu) + c] = reward_t<FAM, real>(p, kc, *rw, x, dx, de0, de, dphi, dui, dus0, usg[0], rab_p, sn, cs, snf, csf, sne, cse);
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

// The load counterpart of warp_store_jac: the warp's rows (width w words) from `src` (the warp's first env's row) into shared memory
template <typename real>
__device__ __forceinline__ void warp_load_jac(real* __restrict__ rows, const real* __restrict__ src, int stride, int w, int valid, int lane) {
  const int total = valid * w;
#pragma unroll 1
  for (int k = lane; k < total; k += 32) { const int e = k / w; rows[e * stride + (k - e * w)] = src[k]; }
}

// A reward term's derivative with respect to its row entry: r = bias - sum w |(row - ref) inv_len|^pw, so d r / d row =
// -w pw |e inv_len|^(pw - 1) sgn(e) inv_len with e = row - ref, taken as 0 at e = 0 (the one-sided convention of DESIGN.md §7)
template <typename real>
__device__ __forceinline__ real reward_coef(real e, real inv_len, real w, int pow1, real pw) {
  const real ae = Num<real>::abs(e) * inv_len;
  real d = sgn(e) * inv_len;
  if (!pow1) d = ae > real(0) ? d * (pw * Num<real>::pow(ae, pw - real(1))) : real(0);
  return -(w * d);
}

// The K-step loop of return_grad_kernel: rollout_loop's discounted return (same updates, same roundings), the tangent pass of every step
// up to the env's first termination with its row [J_x | J_u | d(g^k r_k)/dx | d(g^k r_k)/da] stored to the workspace, then the reverse
// sweep over those rows:  lambda = g^K value_grad (no termination) or 0;  for k = min(end, K) - 1 .. 0:  grad_a[k] = d(g^k r_k)/da +
// J_u^T lambda,  lambda = d(g^k r_k)/dx + J_x^T lambda;  grad_x0 = lambda.
template <int FAM, typename real, int NREF, bool ENVP>
__device__ __forceinline__ RetAcc<real> grad_loop(const StepParams<real>& p, const GradOut& go, CoefArg<real, ENVP> kc, const unsigned i, const bool active,
                                                  real (&x)[Fam<FAM>::NX], Ang<real>& ang, real (&rv)[NREF > 0 ? NREF : 1], real (&rs)[NREF > 0 ? NREF : 1],
                                                  uint32_t (&rend)[NREF > 0 ? NREF : 1], bool& cold_dirty, real* rows, real* row, real* jrows, real* jrow,
                                                  const int jstride, const int lane, const int stride) {
  using F = Fam<FAM>;
  constexpr int NX = F::NX, NX1 = NX + (F::EPS ? 1 : 0), NS = F::NS;
  const int K = p.roll_steps;
  const int nu = go.nu;
  const int W = NX1 * (NX1 + nu) + NX1 + nu;
  const size_t n = (size_t)(unsigned)p.n;
  Out<real> out = make_out<NREF, false, real>(p, i, lane, p.n_obs);
  ClockArg<ENVP> ck = clock_of(p);
  if constexpr (ENVP) ck = id_clock(p, clock_of(p), active ? i : (unsigned)p.env_begin);
  const char* act = action_cursor<FAM, false, real, false>(p, p.action, i);
  WalkCache wc{};
  Act<real> a_next{};
  if (active) a_next = load_action<FAM, false, real, false>(p, act);
  constexpr bool kFeed = NREF > 0;
  const bool feed = kFeed && p.ref_feed != nullptr;
  const real* fc = nullptr;
  real f_next[NREF > 0 ? NREF : 1];
  if constexpr (kFeed) {
    if (feed) { fc = feed_cursor<NREF, false, real>(p, i); if (active) load_feed<NREF, false, real>(p, fc, f_next); }
  }
  const size_t warp_env0 = i - lane;
  real* ws = static_cast<real*>(go.ws) + warp_env0 * (size_t)W;
  real* cb = jrow + W;  // the coefficient row of the reward tangent, behind the stash row
  RetAcc<real> acc{real(0), K};
  real w = real(1);
#pragma unroll 1
  for (int k = 0; k < K; ++k) {
    const Act<real> a_cur = a_next;
    act += p.roll_act_inc;
    if (active && k + 1 < K) a_next = load_action<FAM, false, real, false>(p, act);
    if constexpr (kFeed) {
      if (feed) {
#pragma unroll
        for (int r = 0; r < NREF; ++r) rv[r] = f_next[r];
        fc += n * NREF;
        if (active && k + 1 < K) load_feed<NREF, false, real>(p, fc, f_next);
      }
    }
    // what the tangent pass reads and env_step advances: the state, the angle, the references the reward compares with, the supply
    // voltage and the speed-profile cursor of this step
    const bool alive = active && acc.end == K;
    real x0[NX], rv0[NREF > 0 ? NREF : 1];
#pragma unroll
    for (int j = 0; j < NX; ++j) x0[j] = x[j];
#pragma unroll
    for (int r = 0; r < (NREF > 0 ? NREF : 1); ++r) rv0[r] = rv[r];
    const Ang<real> ang0 = ang;
    RwTan<real> rt{real(0), nullptr, cb, go.wmask};
    if (alive) { rt.u_sup = step_u_sup(p, i); rt.gt = step_gt(p, i); }
    const StepOut<real> so = env_step<FAM, false, real, NREF, false, false, false, false, ENVP>(p, kc, ck, out, k == K - 1, a_cur, i, active, x, ang, rv, rs, rend,
                                                                                               cold_dirty, wc, rows, row, lane, stride);
    if (alive) {
      acc.g = acc.g + w * so.reward;
      if (so.term) acc.end = k;
    }
    const bool lin = alive && !so.term;  // a step whose row the sweep reads
    if (lin) {  // d(w r_k) / d s_b from the row env_step left (state noise included), then the tangent pass on the pre-step copies
#pragma unroll
      for (int b = 0; b < NS; ++b) if ((go.wmask >> b) & 1u) cb[b] = real(0);
#pragma unroll
      for (int r = 0; r < NREF; ++r)
        if (p.rwr_w[r] != real(0)) cb[go.ref_base[r]] += w * reward_coef(row[p.ref_state[r]] - rv0[r], p.rwr_inv_len[r], p.rwr_w[r], p.rwr_pow1[r], p.rwr_pow[r]);
#pragma unroll 1
      for (int t = 0; t < p.n_rw; ++t)
        cb[go.rw_base[t]] += w * reward_coef(row[p.rw_state[t]], p.rw_inv_len[t], p.rw_w[t], p.rw_pow1[t], p.rw_pow[t]);
      step_tangent<FAM, false, real, true>(p, kc, x0, ang0, a_cur, i, nu, jrow, &rt);
    }
    w = w * p.discount;
    __syncwarp();
    if (__any_sync(0xffffffffu, lin)) warp_store_jac(ws, jrows, jstride, W, out.valid, lane);
    ws += n * (size_t)W;
    __syncwarp();  // both staging areas are reused by the next step
    ck.kstep += 1u;
    ck.gstep_lo += 1u;
    if (ck.gstep_lo == 0u) ck.gstep_hi += 1u;
  }
  // ---------------- reverse sweep ----------------
  real lam[NX1];
  const bool boot = active && acc.end == K && go.value_grad != nullptr;
#pragma unroll
  for (int r = 0; r < NX1; ++r) lam[r] = boot ? w * static_cast<const real*>(go.value_grad)[(size_t)i * NX1 + r] : real(0);
  real* ga_out = static_cast<real*>(go.grad_a) + (size_t)K * n * nu + warp_env0 * (size_t)nu;
#pragma unroll 1
  for (int k = K - 1; k >= 0; --k) {
    ws -= n * (size_t)W;
    ga_out -= n * (size_t)nu;
    const bool live = active && k < acc.end;
    if (__any_sync(0xffffffffu, live)) warp_load_jac(jrows, ws, jstride, W, out.valid, lane);
    __syncwarp();
    real ga[GEMB200_MAX_ACT];
    const real* jx = jrow;
    const real* ju = jrow + NX1 * NX1;
    const real* rx = jrow + NX1 * (NX1 + nu);
    const real* ru = rx + NX1;
#pragma unroll
    for (int u = 0; u < GEMB200_MAX_ACT; ++u) {
      real s = real(0);
      if (live && u < nu) {
        s = ru[u];
#pragma unroll
        for (int r = 0; r < NX1; ++r) s = fm(ju[r * nu + u], lam[r], s);
      }
      ga[u] = s;
    }
    if (live) {
      real ln[NX1];
#pragma unroll
      for (int c = 0; c < NX1; ++c) {
        real s = rx[c];
#pragma unroll
        for (int r = 0; r < NX1; ++r) s = fm(jx[r * NX1 + c], lam[r], s);
        ln[c] = s;
      }
#pragma unroll
      for (int c = 0; c < NX1; ++c) lam[c] = ln[c];
    }
    __syncwarp();
#pragma unroll
    for (int u = 0; u < GEMB200_MAX_ACT; ++u) if (u < nu) jrow[u] = ga[u];
    __syncwarp();
    warp_store_jac(ga_out, jrows, jstride, nu, out.valid, lane);
    __syncwarp();
  }
#pragma unroll
  for (int c = 0; c < NX1; ++c) jrow[c] = lam[c];
  __syncwarp();
  warp_store_jac(static_cast<real*>(go.grad_x0) + warp_env0 * NX1, jrows, jstride, NX1, out.valid, lane);
  return acc;
}

// The return-gradient kernel (continuous converters): jacobian_kernel's shape with grad_loop, and rollout_kernel's returns.  Dynamic shared
// memory: the observation rows of the block, then per env its stash row and its coefficient row (jstride words).
template <int FAM, typename real, int NREF, bool ENVP>
__global__ void __launch_bounds__(GEMB200_BLOCK, (sizeof(real) == 4 ? GEMB200_MINBLOCKS_JAC : GEMB200_MINBLOCKS_JAC_F64))
return_grad_kernel(const __grid_constant__ StepParams<real> p, const __grid_constant__ GradOut go, const int jstride) {
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
  RetAcc<real> acc;
  if constexpr (ENVP) {
    Coef<real> kl;
    load_coef<FAM, real>(p, active ? i : (unsigned)p.env_begin, mech != 0, kl);
    acc = grad_loop<FAM, real, NREF, true>(p, go, kl, i, active, x, ang, rv, rs, rend, cold_dirty, rows, row, jrows, jrow, jstride, lane, stride);
  } else {
    acc = grad_loop<FAM, real, NREF, false>(p, go, p.k, i, active, x, ang, rv, rs, rend, cold_dirty, rows, row, jrows, jrow, jstride, lane, stride);
  }
  if (active) {
    pack_records<NX, NREF, real>(hot, cold, x, rv, rs, rend);
    if constexpr (NH > 0) store_words<NH, real>(p.st, i, n, hot);
    if (cold_dirty) store_words<NC, real>(p.stc, i, n, cold);
    if constexpr (F::EPS) ang.store(p.eps, i);
    p.ret_out[i] = acc.g;
    if (p.ret_end) p.ret_end[i] = acc.end;
  }
}

// The K-step loop of param_sens_kernel: jac_loop's steps with the parameter column passes instead of the seed columns.  The thread's
// staging row holds S [NX1][n_p] (loaded from sens_io, stored back after the last step) and behind it the coefficient tangents of the n_p
// columns (ps_words<FAM>() words each).  Step k: the column passes advance S to S_{k+1} on the pre-step state, env_step advances the primal,
// S_{k+1} goes to sens_out[k], and an env that env_step has just reset (autoreset same_step) restarts from S = 0: its reset state does not
// depend on theta.
template <int FAM, bool FINITE, typename real, int NREF, bool ENVP>
__device__ __forceinline__ void psens_loop(const StepParams<real>& p, const PsOut& po, CoefArg<real, ENVP> kc, const unsigned i, const bool active, real (&x)[Fam<FAM>::NX],
                                           Ang<real>& ang, real (&rv)[NREF > 0 ? NREF : 1], real (&rs)[NREF > 0 ? NREF : 1], uint32_t (&rend)[NREF > 0 ? NREF : 1],
                                           bool& cold_dirty, real* rows, real* row, real* jrows, real* jrow, const int jstride, const int lane, const int stride) {
  constexpr int NX1 = Fam<FAM>::NX + (Fam<FAM>::EPS ? 1 : 0);
  const int K = p.roll_steps;
  const int np = po.np, ws = NX1 * np;
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
  real* sio = static_cast<real*>(po.sio) + warp_env0 * (size_t)ws;
  real* so = po.sout ? static_cast<real*>(po.sout) + warp_env0 * (size_t)ws : nullptr;
  const real* tks = jrow + ws;
  warp_load_jac(jrows, sio, jstride, ws, out.valid, lane);
  __syncwarp();
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
    if (active) step_tangent<FAM, FINITE, real, false, true>(p, kc, x, ang, a_cur, i, np, jrow, nullptr, tks);
    const StepOut<real> sto = env_step<FAM, FINITE, real, NREF, false, false, false, false, ENVP>(p, kc, ck, out, true, a_cur, i, active, x, ang, rv, rs, rend,
                                                                                                cold_dirty, wc, rows, row, lane, stride);
    __syncwarp();
    if (so) {
      warp_store_jac(so, jrows, jstride, ws, out.valid, lane);
      so += n * (size_t)ws;
      __syncwarp();
    }
    if (active && sto.term && p.autoreset == GEMB200_AUTORESET_SAME_STEP)
      for (int w = 0; w < ws; ++w) jrow[w] = real(0);
    __syncwarp();  // the observation rows are reused by the next step
    out.obs = byte_add(out.obs, p.roll_obs_inc); out.ref = byte_add(out.ref, p.roll_ref_inc);
    out.rew = byte_add(out.rew, p.roll_rew_inc); out.term = byte_add(out.term, p.roll_term_inc);
    ck.kstep += 1u;
    ck.gstep_lo += 1u;
    if (ck.gstep_lo == 0u) ck.gstep_hi += 1u;
  }
  warp_store_jac(sio, jrows, jstride, ws, out.valid, lane);
}

// The parameter-sensitivity kernel: jacobian_kernel's shape with psens_loop.  Before the loop every env derives the coefficient tangents
// of its n_p parameters once, in double precision (coef_tangent, gemb200_model.h), from its own parameter row (ENVP: praw) or the
// configuration's (po.raw), into its staging row.  Dynamic shared memory: the observation rows of the block, then per env its row of S and
// coefficient tangents (jstride words).
template <int FAM, bool FINITE, typename real, int NREF, bool ENVP>
__global__ void __launch_bounds__(GEMB200_BLOCK, (sizeof(real) == 4 ? GEMB200_MINBLOCKS_JAC : GEMB200_MINBLOCKS_JAC_F64))
param_sens_kernel(const __grid_constant__ StepParams<real> p, const __grid_constant__ PsOut po, const int jstride) {
  using F = Fam<FAM>;
  constexpr int NX = F::NX, NX1 = NX + (F::EPS ? 1 : 0), NH = hot_words(NX, NREF), NC = cold_words(NX, NREF), NW = ps_words<FAM>();
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
    double prm[kMaxDraw];
#pragma unroll 1
    for (int s = 0; s < kMaxDraw; ++s) prm[s] = ENVP ? p.praw[(size_t)s * n + i] : po.raw[s];
    real* tks = jrow + NX1 * po.np;
#pragma unroll 1
    for (int c = 0; c < po.np; ++c) {
      double t[kCoefWords];
      coef_tangent(p.motor_kind, prm, po.slot[c], t);
#pragma unroll
      for (int w = 0; w < NW; ++w) tks[c * NW + w] = (real)t[ps_word<FAM>(w)];
    }
  }
  if constexpr (ENVP) {
    Coef<real> kl;
    load_coef<FAM, real>(p, active ? i : (unsigned)p.env_begin, mech != 0, kl);
    psens_loop<FAM, FINITE, real, NREF, true>(p, po, kl, i, active, x, ang, rv, rs, rend, cold_dirty, rows, row, jrows, jrow, jstride, lane, stride);
  } else {
    psens_loop<FAM, FINITE, real, NREF, false>(p, po, p.k, i, active, x, ang, rv, rs, rend, cold_dirty, rows, row, jrows, jrow, jstride, lane, stride);
  }
  if (active) {
    pack_records<NX, NREF, real>(hot, cold, x, rv, rs, rend);
    if constexpr (NH > 0) store_words<NH, real>(p.st, i, n, hot);
    if (cold_dirty) store_words<NC, real>(p.stc, i, n, cold);
    if constexpr (F::EPS) ang.store(p.eps, i);
  }
}

}  // namespace gemb200
