// gemb200_model.h — the model coefficients of one env from its physical parameters (the reference's *_update_model methods).
//
// ONE derivation for the host (gemb200.cu: derive_model, gemb200_set_env_params) and the device (parameter draws at a reset,
// gemb200_kernels.cuh: redraw_env_params).  Double precision, only + - * /: the library is built with -fmad=false and the host side
// without FMA contraction, so both sides round every operation the same way and the device result equals the host result bit for bit.
#pragma once
#include "../../include/gemb200.h"

namespace gemb200 {

struct ModelCoef {
  double c[20];  // motor model coefficients (layout per family, see Coef in gemb200_params.h)
  double tq[4];  // torque coefficients
  double inv_j, omega_lim, omega_lin;
};

// mp: motor_param[GEMB200_MAX_MOTOR_PARAM], lp: load_param[8] (slot enums of gemb200_config)
__host__ __device__ inline void derive_coef(int motor_kind, const double* mp, const double* lp, ModelCoef* o) {
  for (int j = 0; j < 20; ++j) o->c[j] = 0.0;
  for (int j = 0; j < 4; ++j) o->tq[j] = 0.0;
  const double p = mp[GEMB200_MP_P], r_s = mp[GEMB200_MP_R_S], l_d = mp[GEMB200_MP_L_D], l_q = mp[GEMB200_MP_L_Q];
  double* c = o->c;
  switch (motor_kind) {
    case GEMB200_MOTOR_PERMEX_DC: {  // dc_permanently_excited_motor.py:71-75
      const double l_a = mp[GEMB200_MP_L_A];
      c[0] = -mp[GEMB200_MP_PSI_E] / l_a; c[1] = -mp[GEMB200_MP_R_A] / l_a; c[2] = 0; c[3] = 1.0 / l_a;
      o->tq[0] = mp[GEMB200_MP_PSI_E]; o->tq[1] = 0;
    } break;
    case GEMB200_MOTOR_SERIES_DC: {  // dc_series_motor.py:66-74
      const double l = mp[GEMB200_MP_L_A] + mp[GEMB200_MP_L_E];
      c[0] = 0; c[1] = (-mp[GEMB200_MP_R_A] - mp[GEMB200_MP_R_E]) / l; c[2] = -mp[GEMB200_MP_L_E_PRIME] / l; c[3] = 1.0 / l;
      o->tq[0] = 0; o->tq[1] = mp[GEMB200_MP_L_E_PRIME];
    } break;
    case GEMB200_MOTOR_SHUNT_DC:
    case GEMB200_MOTOR_EXTEX_DC: {  // dc_motor.py:95-108
      const double l_a = mp[GEMB200_MP_L_A], l_e = mp[GEMB200_MP_L_E];
      c[0] = -mp[GEMB200_MP_R_A] / l_a; c[1] = -mp[GEMB200_MP_L_E_PRIME] / l_a; c[2] = 1.0 / l_a;
      c[3] = -mp[GEMB200_MP_R_E] / l_e; c[4] = 1.0 / l_e;
      o->tq[0] = mp[GEMB200_MP_L_E_PRIME];
    } break;
    case GEMB200_MOTOR_PMSM:
    case GEMB200_MOTOR_SYNRM: {  // permanent_magnet_synchronous_motor.py:107-139, synchronous_reluctance_motor.py:117-139
      const double psi_p = motor_kind == GEMB200_MOTOR_PMSM ? mp[GEMB200_MP_PSI_P] : 0.0;
      c[0] = -r_s / l_d; c[1] = 1.0 / l_d; c[2] = l_q * p / l_d;
      c[3] = -psi_p * p / l_q; c[4] = -r_s / l_q; c[5] = 1.0 / l_q; c[6] = -l_d * p / l_q;
      o->tq[0] = 1.5 * p * psi_p; o->tq[1] = 1.5 * p * (l_d - l_q);
    } break;
    case GEMB200_MOTOR_EESM: {  // externally_excited_synchronous_motor.py:125-153, :200-203
      const double k = mp[GEMB200_MP_K], r_e = mp[GEMB200_MP_R_E], l_m = mp[GEMB200_MP_L_M], l_e = mp[GEMB200_MP_L_E];
      const double r_E = k * k * 1.5 * r_e, l_M = k * 1.5 * l_m, l_E = k * k * 1.5 * l_e, ik = 2.0 / 3.0 / k;
      const double sigma = 1.0 - l_M * l_M / (l_d * l_E);
      c[0] = (-r_s / sigma) / l_d; c[1] = (l_M * r_E / (sigma * l_E) * ik) / l_d; c[2] = (1.0 / sigma) / l_d;
      c[3] = (-l_M * k / (sigma * l_E)) / l_d; c[4] = (l_q * p / sigma) / l_d;
      c[5] = -r_s / l_q; c[6] = 1.0 / l_q; c[7] = -l_d * p / l_q; c[8] = -p * l_M * ik / l_q;
      const double s2 = l_E * ik;
      c[9] = (l_M * r_s / (sigma * l_d)) / s2; c[10] = (-r_E / sigma * ik) / s2; c[11] = (-l_M / (sigma * l_d)) / s2;
      c[12] = (k / sigma) / s2; c[13] = (-p * l_M * l_q / (sigma * l_d)) / s2;
      o->tq[0] = 1.5 * p * l_M * ik; o->tq[1] = 1.5 * p * (l_d - l_q);
    } break;
    case GEMB200_MOTOR_DFIM:
    case GEMB200_MOTOR_SCIM: {  // induction_motor.py:287-310, :236-249
      const double l_m = mp[GEMB200_MP_L_M], r_r = mp[GEMB200_MP_R_E];
      const double l_s = l_m + mp[GEMB200_MP_L_SIGS], l_r = l_m + mp[GEMB200_MP_L_SIGR];
      const double sigma = (l_s * l_r - l_m * l_m) / (l_s * l_r);
      const double tau_r = l_r / r_r, tau_sig = sigma * l_s / (r_s + r_r * (l_m * l_m) / (l_r * l_r));
      c[0] = -1.0 / tau_sig; c[1] = l_m * r_r / (sigma * l_s * l_r * l_r); c[2] = l_m * p / (sigma * l_r * l_s);
      c[3] = 1.0 / (sigma * l_s); c[4] = l_m / tau_r; c[5] = -1.0 / tau_r; c[6] = p;
      c[7] = -l_m / (sigma * l_r * l_s);  // rotor-voltage column of the current rows (DFIM)
      c[8] = 1.0 / l_r; c[9] = l_m / l_r;  // rotor current i_r = psi_r / l_r - l_m / l_r * i_s (physical_systems.py:946-956)
      o->tq[0] = 1.5 * p * l_m / l_r;
    } break;
  }
  // MechanicalLoad.set_j_rotor mechanical_load.py:188-193, polynomial_static_load.py:60-64
  const double j_total = lp[GEMB200_LP_J_LOAD] + mp[GEMB200_MP_J_ROTOR];
  o->inv_j = j_total > 0 ? 1.0 / j_total : 0.0;
  o->omega_lin = j_total / lp[GEMB200_LP_TAU_DECAY];
  o->omega_lim = j_total > 0 ? lp[GEMB200_LP_A] / j_total * lp[GEMB200_LP_TAU_DECAY] : 0.0;
}

}  // namespace gemb200
