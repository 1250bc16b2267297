// gemb200_model.h — the model coefficients of one env from its physical parameters (the reference's *_update_model methods).
//
// ONE derivation for the host (gemb200.cu: derive_model, gemb200_set_env_params) and the device (parameter draws at a reset,
// gemb200_kernels.cuh: redraw_env_params).  Double precision, only + - * /: the library is built with -fmad=false and the host side
// without FMA contraction, so both sides round every operation the same way and the device result equals the host result bit for bit.
#pragma once
#include "../../include/gemb200.h"
#include "gemb200_params.h"

namespace gemb200 {

template <typename T>
struct ModelCoefT {
  T c[20];  // motor model coefficients (layout per family, see Coef in gemb200_params.h)
  T tq[4];  // torque coefficients
  T inv_j, omega_lim, omega_lin;
};
using ModelCoef = ModelCoefT<double>;

// A value and its derivative along one parameter (forward mode): derive_coef_t<Dual> is the derivative of derive_coef
struct Dual {
  double v, d;
  __host__ __device__ Dual(double v_ = 0.0, double d_ = 0.0) : v(v_), d(d_) {}
};
__host__ __device__ inline Dual operator+(Dual a, Dual b) { return Dual(a.v + b.v, a.d + b.d); }
__host__ __device__ inline Dual operator-(Dual a, Dual b) { return Dual(a.v - b.v, a.d - b.d); }
__host__ __device__ inline Dual operator-(Dual a) { return Dual(-a.v, -a.d); }
__host__ __device__ inline Dual operator*(Dual a, Dual b) { return Dual(a.v * b.v, a.d * b.v + a.v * b.d); }
__host__ __device__ inline Dual operator/(Dual a, Dual b) { const double q = a.v / b.v; return Dual(q, (a.d - q * b.d) / b.v); }
__host__ __device__ inline double value_of(double x) { return x; }
__host__ __device__ inline double value_of(Dual x) { return x.v; }

// mp: motor_param[GEMB200_MAX_MOTOR_PARAM], lp: load_param[8] (slot enums of gemb200_config).  T = double: the coefficients; T = Dual: the
// coefficients with their derivative along the parameter the caller seeded (coef_tangent)
template <typename T>
__host__ __device__ inline void derive_coef_t(int motor_kind, const T* mp, const T* lp, ModelCoefT<T>* o) {
  for (int j = 0; j < 20; ++j) o->c[j] = T(0.0);
  for (int j = 0; j < 4; ++j) o->tq[j] = T(0.0);
  const T p = mp[GEMB200_MP_P], r_s = mp[GEMB200_MP_R_S], l_d = mp[GEMB200_MP_L_D], l_q = mp[GEMB200_MP_L_Q];
  T* c = o->c;
  switch (motor_kind) {
    case GEMB200_MOTOR_PERMEX_DC: {  // dc_permanently_excited_motor.py:71-75
      const T l_a = mp[GEMB200_MP_L_A];
      c[0] = -mp[GEMB200_MP_PSI_E] / l_a; c[1] = -mp[GEMB200_MP_R_A] / l_a; c[2] = T(0.0); c[3] = 1.0 / l_a;
      o->tq[0] = mp[GEMB200_MP_PSI_E]; o->tq[1] = T(0.0);
    } break;
    case GEMB200_MOTOR_SERIES_DC: {  // dc_series_motor.py:66-74
      const T l = mp[GEMB200_MP_L_A] + mp[GEMB200_MP_L_E];
      c[0] = T(0.0); c[1] = (-mp[GEMB200_MP_R_A] - mp[GEMB200_MP_R_E]) / l; c[2] = -mp[GEMB200_MP_L_E_PRIME] / l; c[3] = 1.0 / l;
      o->tq[0] = 0; o->tq[1] = mp[GEMB200_MP_L_E_PRIME];
    } break;
    case GEMB200_MOTOR_SHUNT_DC:
    case GEMB200_MOTOR_EXTEX_DC: {  // dc_motor.py:95-108
      const T l_a = mp[GEMB200_MP_L_A], l_e = mp[GEMB200_MP_L_E];
      c[0] = -mp[GEMB200_MP_R_A] / l_a; c[1] = -mp[GEMB200_MP_L_E_PRIME] / l_a; c[2] = 1.0 / l_a;
      c[3] = -mp[GEMB200_MP_R_E] / l_e; c[4] = 1.0 / l_e;
      o->tq[0] = mp[GEMB200_MP_L_E_PRIME];
    } break;
    case GEMB200_MOTOR_PMSM:
    case GEMB200_MOTOR_SYNRM: {  // permanent_magnet_synchronous_motor.py:107-139, synchronous_reluctance_motor.py:117-139
      const T psi_p = motor_kind == GEMB200_MOTOR_PMSM ? mp[GEMB200_MP_PSI_P] : T(0.0);
      c[0] = -r_s / l_d; c[1] = 1.0 / l_d; c[2] = l_q * p / l_d;
      c[3] = -psi_p * p / l_q; c[4] = -r_s / l_q; c[5] = 1.0 / l_q; c[6] = -l_d * p / l_q;
      o->tq[0] = 1.5 * p * psi_p; o->tq[1] = 1.5 * p * (l_d - l_q);
    } break;
    case GEMB200_MOTOR_EESM: {  // externally_excited_synchronous_motor.py:125-153, :200-203
      const T k = mp[GEMB200_MP_K], r_e = mp[GEMB200_MP_R_E], l_m = mp[GEMB200_MP_L_M], l_e = mp[GEMB200_MP_L_E];
      const T r_E = k * k * 1.5 * r_e, l_M = k * 1.5 * l_m, l_E = k * k * 1.5 * l_e, ik = 2.0 / 3.0 / k;
      const T sigma = 1.0 - l_M * l_M / (l_d * l_E);
      c[0] = (-r_s / sigma) / l_d; c[1] = (l_M * r_E / (sigma * l_E) * ik) / l_d; c[2] = (1.0 / sigma) / l_d;
      c[3] = (-l_M * k / (sigma * l_E)) / l_d; c[4] = (l_q * p / sigma) / l_d;
      c[5] = -r_s / l_q; c[6] = 1.0 / l_q; c[7] = -l_d * p / l_q; c[8] = -p * l_M * ik / l_q;
      const T s2 = l_E * ik;
      c[9] = (l_M * r_s / (sigma * l_d)) / s2; c[10] = (-r_E / sigma * ik) / s2; c[11] = (-l_M / (sigma * l_d)) / s2;
      c[12] = (k / sigma) / s2; c[13] = (-p * l_M * l_q / (sigma * l_d)) / s2;
      o->tq[0] = 1.5 * p * l_M * ik; o->tq[1] = 1.5 * p * (l_d - l_q);
    } break;
    case GEMB200_MOTOR_DFIM:
    case GEMB200_MOTOR_SCIM: {  // induction_motor.py:287-310, :236-249
      const T l_m = mp[GEMB200_MP_L_M], r_r = mp[GEMB200_MP_R_E];
      const T l_s = l_m + mp[GEMB200_MP_L_SIGS], l_r = l_m + mp[GEMB200_MP_L_SIGR];
      const T sigma = (l_s * l_r - l_m * l_m) / (l_s * l_r);
      const T tau_r = l_r / r_r, tau_sig = sigma * l_s / (r_s + r_r * (l_m * l_m) / (l_r * l_r));
      c[0] = -1.0 / tau_sig; c[1] = l_m * r_r / (sigma * l_s * l_r * l_r); c[2] = l_m * p / (sigma * l_r * l_s);
      c[3] = 1.0 / (sigma * l_s); c[4] = l_m / tau_r; c[5] = -1.0 / tau_r; c[6] = p;
      c[7] = -l_m / (sigma * l_r * l_s);  // rotor-voltage column of the current rows (DFIM)
      c[8] = 1.0 / l_r; c[9] = l_m / l_r;  // rotor current i_r = psi_r / l_r - l_m / l_r * i_s (physical_systems.py:946-956)
      o->tq[0] = 1.5 * p * l_m / l_r;
    } break;
  }
  // MechanicalLoad.set_j_rotor mechanical_load.py:188-193, polynomial_static_load.py:60-64
  const T j_total = lp[GEMB200_LP_J_LOAD] + mp[GEMB200_MP_J_ROTOR];
  o->inv_j = value_of(j_total) > 0 ? 1.0 / j_total : T(0.0);
  o->omega_lin = j_total / lp[GEMB200_LP_TAU_DECAY];
  o->omega_lim = value_of(j_total) > 0 ? lp[GEMB200_LP_A] / j_total * lp[GEMB200_LP_TAU_DECAY] : T(0.0);
}

__host__ __device__ inline void derive_coef(int motor_kind, const double* mp, const double* lp, ModelCoef* o) { derive_coef_t<double>(motor_kind, mp, lp, o); }

// The column of one env's coefficient block, in the word order of Coef (gemb200_params.h): put(w, value) for each of the kCoefWords words,
// from the derived coefficients o and the env's load slots lp (the load polynomial's a, b, c are block words themselves).  Every block
// column and the shared coefficients are written through it, except in redraw_env_params (gemb200_kernels.cuh), which spells its stores
// out (DESIGN §4).  `put` runs where the caller runs (host or device): no execution-space check on it.
#pragma nv_exec_check_disable
template <typename T, typename Put>
__host__ __device__ inline void coef_words(const ModelCoefT<T>& o, const T* lp, Put&& put) {
  for (int w = 0; w < kCwTq; ++w) put(w, o.c[w]);
  for (int w = 0; w < kCwLoad - kCwTq; ++w) put(kCwTq + w, o.tq[w]);
  put(kCwLoad, lp[GEMB200_LP_A]); put(kCwLoad + 1, lp[GEMB200_LP_B]); put(kCwLoad + 2, lp[GEMB200_LP_C]);
  put(kCwLoad + 3, o.inv_j); put(kCwLoad + 4, o.omega_lim); put(kCwLoad + 5, o.omega_lin);
}

// d (coefficient block) / d prm[slot] in the word order of Coef, prm = the env's physical parameters in the slot order of a parameter row
// (GEMB200_MAX_MOTOR_PARAM motor slots, then 8 load slots).  Not inlined on the device: it runs once per launch and env, and its
// double-precision body stays out of the kernels' step loop.
__host__ __device__ __noinline__ inline void coef_tangent(int motor_kind, const double* prm, int slot, double* out) {
  Dual m[GEMB200_MAX_MOTOR_PARAM], l[8];
  for (int s = 0; s < GEMB200_MAX_MOTOR_PARAM; ++s) m[s] = Dual(prm[s], s == slot ? 1.0 : 0.0);
  for (int s = 0; s < 8; ++s) l[s] = Dual(prm[GEMB200_MAX_MOTOR_PARAM + s], GEMB200_MAX_MOTOR_PARAM + s == slot ? 1.0 : 0.0);
  ModelCoefT<Dual> o;
  derive_coef_t<Dual>(motor_kind, m, l, &o);
  coef_words(o, l, [out](int w, Dual v) { out[w] = v.d; });
}

}  // namespace gemb200
