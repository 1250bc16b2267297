/*
 * gem_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * A plain-C, float64, one-env-at-a-time restatement of the reference's physical-system step
 * (upb-lea/gym-electric-motor @ 5555196, src/gym_electric_motor/...).  It exists to CHECK the CUDA path and to be
 * timed as the CPU baseline; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load it.  The product (gym_electric_motor_b200/) never links, imports or calls anything in oracle/.
 *
 * Pinning: tests/test_oracle_golden.py replays every trajectory in tests/golden/*.npz (recorded from the
 * UNMODIFIED reference by tests/golden/make_golden.py, including a regeneration of the reference's own
 * tests/integration_tests/ref_data.npz) through this file and requires agreement to <=1e-9 (Euler / RK4,
 * algorithm-identical) and <=2e-7 (dopri5, adaptive).  The known-answer vectors of the reference's own unit tests (converter
 * truth tables, PolynomialStaticLoad ODE, constraint tables, reward cases; tests/golden/make_known_answers.py) are replayed through the
 * probe entry points at the end of this file by tests/test_oracle_known_answers.py.
 *
 * Every function cites the reference lines it restates.  The structure deliberately follows the reference
 * (dense model-constant matrices, per-segment convert/integrate loop) rather than the optimised CUDA kernels.
 *
 * The POD configuration struct is the public one from include/gemb200.h (header only, no product code).
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/gemb200.h"

#define ORACLE_SOLVER_DOPRI5 100 /* oracle-only: restatement of scipy.integrate.ode('dopri5') defaults (solvers.py:139-184) */

#define MAXM 6  /* motor ODE states incl. eps */
#define MAXF 12 /* feature-vector length of the model-constant product */

typedef struct {
  /* finite 2QC (converters.py:248-310) */
  int pattern[2];
  int pattern_len;
  int switching_state; /* persists across steps AND resets (converters.py:193-197,45-54) */
  double action_start_time;
  int cur_action_i;
  /* continuous 2QC / 1QC (converters.py:130-184, 371-435) */
  double cur_action;
} sub2qc_t;

typedef struct {
  double ode[GEMB200_MAX_ODE]; /* [mechanical | motor] physical_systems.py:270 */
  double t;
  long k;
  sub2qc_t sub[6]; /* slot0: up to 3 legs (B6) or 2 (4QC) ; slot1: up to 3 (the DFIM's rotor bridge) */
  int cur_action1qc[2];
  /* reference generator slots (subepisoded_reference_generator.py) */
  double ref_value[GEMB200_MAX_REF];
  double ref_sigma[GEMB200_MAX_REF];
  int ref_left[GEMB200_MAX_REF];
  uint32_t ref_start[GEMB200_MAX_REF], ref_len[GEMB200_MAX_REF]; /* periodic generators: sub-episode start step and length */
  double fifo[GEMB200_MAX_DEAD_TIME][GEMB200_MAX_ACT]; /* DeadTimeProcessor queue (ring; slot = call counter mod steps) */
  double psi_re, psi_im; /* FluxObserver._integrated flux_observer.py:46 */
  int sw_cur[GEMB200_MAX_REF], sw_k[GEMB200_MAX_REF], sw_len[GEMB200_MAX_REF]; /* SwitchedReferenceGenerator: current entry, _k, _current_episode_length */
  double ac_phase; /* AC1PhaseSupply._phi */
  double u_rc; int rc_started; /* RCVoltageSupply: solver state and 'a previous get_voltage call exists' (voltage_supplies.py:110-123) */
  double im_prev[2]; int im_prev_set; /* induction motors: _initial_states i_salpha / i_sbeta left by the previous initialize() call */
} env_t;

typedef struct gem_oracle {
  gemb200_config cfg;
  int n_state, n_ode, n_act, n_ref, n_motor, n_cur, n_volt;
  int n_obs; /* width of the state vector after the physical_system_wrappers (n_state: the inner system's own) */
  int n_sub[2];     /* 2QC sub-converters per slot */
  int slot_off[2];  /* first sub index per slot */
  double mc[MAXM][MAXF]; /* _model_constants */
  int mc_rows, mc_cols;
  double j_total, omega_lim, omega_lin; /* polynomial_static_load.py:72-85 */
  /* derived EESM constants (externally_excited_synchronous_motor.py:129-136) */
  double l_M, i_k_rs;
  double tq0; /* SCIM torque factor */
  uint64_t gstep; /* id of the current API call (RNG counter) */
  uint64_t n_steps; /* step calls so far (dead-time ring position) */
  int exact_grid; /* 0: the reference's time grid (t accumulates, h = fl(t + tau) - t); 1: the device's (gem_oracle_set_time_grid) */
  env_t* env;
} gem_oracle;

static void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1);
static void rng4(const gem_oracle* o, int64_t env, uint32_t stream, uint32_t out[4]) {
  uint64_t g = (uint64_t)(env + o->cfg.env_index_offset);
  out[0] = (uint32_t)o->gstep; out[1] = (uint32_t)(o->gstep >> 32); out[2] = (uint32_t)g; out[3] = ((uint32_t)(g >> 32) << 8) | stream;
  philox4x32_10(out, (uint32_t)o->cfg.seed, (uint32_t)(o->cfg.seed >> 32));
}

/* ------------------------------------------------------------------------------------------------------------ */
/* Philox4x32-10 (Salmon et al., SC'11) — the published counter-based generator; the CUDA path uses the same    */
/* construction with the same (key, counter) convention so that the device reference generator can be checked   */
/* value-for-value.  The reference's numpy PCG64 streams cannot be reproduced on a device (SURVEY.md §5).        */
/* ------------------------------------------------------------------------------------------------------------ */
static void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; ++r) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c[0];
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c[2];
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k0;
    uint32_t n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k1;
    uint32_t n3 = (uint32_t)p0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}
static double u01(uint32_t x) { return ((double)x + 0.5) * (1.0 / 4294967296.0); } /* (0,1) */

/* Counter = (id of the API call lo, hi, global env index lo, (hi << 8) | stream id); key = seed.  Every reset/step
 * call of a handle gets a fresh call id, so no per-env RNG state exists.  Stream ids: */
enum { STREAM_WALK = 1, STREAM_SUBEP = 2, STREAM_INIT = 3, STREAM_SUBEP_HI = 18,
       STREAM_WALK_R = 5, STREAM_SUBEP_R = 6, STREAM_SUBEP_HI_R = 22 /* _R: draws right after a reset */,
       STREAM_SWITCH = 10, STREAM_SWITCH_R = 14 /* + slot: SwitchedReferenceGenerator super-episodes (R: at a reset) */,
       STREAM_INIT_STATE = 7, STREAM_INIT_STATE2 = 8 /* random initial ODE state */, STREAM_SUPPLY = 9 /* AC supply phase */, /* induction motors: eps_mag = word 2 of STREAM_INIT_STATE2 */ STREAM_LAPLACE = 24, STREAM_LAPLACE_R = 28 /* Laplace walk increments */,
       STREAM_WALK2 = 4 /* walk increments with <= 2 reference slots: one block per TWO call ids (counter = id >> 1, word pair = id & 1) */,
       STREAM_PERIODIC = 32 /* + 2*slot (+1): sub-episode parameters of the periodic generators, counter word 0 = start step */,
       STREAM_NOISE = 64 /* + 8*op + (state >> 2): StateNoiseProcessor */, STREAM_NOISE_R = 128 /* ... right after an auto-reset */ };

struct gem_oracle;
static void rng4(const struct gem_oracle* o, int64_t env, uint32_t stream, uint32_t out[4]);

/* ------------------------------------------------------------------------------------------------------------ */
/* dimensions — SCMLSystem._set_indices physical_systems.py:141-162, :462-485, :594-617, :737-763               */
/* ------------------------------------------------------------------------------------------------------------ */
static int slot_nsub(int kind) {
  switch (kind) {
    case GEMB200_CONV_1QC: return 1;
    case GEMB200_CONV_2QC: return 1;
    case GEMB200_CONV_4QC: return 2;
    case GEMB200_CONV_B6: return 3;
    default: return 0;
  }
}
static int slot_nvolt(int kind) { return kind == GEMB200_CONV_B6 ? 3 : (kind == GEMB200_CONV_NONE ? 0 : 1); }

static int dims(gem_oracle* o) {
  const gemb200_config* c = &o->cfg;
  switch (c->motor_kind) {
    case GEMB200_MOTOR_PERMEX_DC:
    case GEMB200_MOTOR_SERIES_DC: o->n_motor = 1; o->n_cur = 1; o->n_volt = 1; o->n_state = 5; break;
    case GEMB200_MOTOR_SHUNT_DC: o->n_motor = 2; o->n_cur = 2; o->n_volt = 1; o->n_state = 7; break; /* 6 + i_sum: every ShuntDc env
      appends CurrentSumProcessor(('i_a','i_e')) (envs/gym_dcm/shunt_dc_motor_env/*.py), restated natively */
    case GEMB200_MOTOR_EXTEX_DC: o->n_motor = 2; o->n_cur = 2; o->n_volt = 2; o->n_state = 7; break;
    case GEMB200_MOTOR_PMSM:
    case GEMB200_MOTOR_SYNRM: o->n_motor = 3; o->n_cur = 2; o->n_volt = 2; o->n_state = 14; break;
    case GEMB200_MOTOR_EESM: o->n_motor = 4; o->n_cur = 3; o->n_volt = 3; o->n_state = 16; break;
    case GEMB200_MOTOR_SCIM: o->n_motor = 5; o->n_cur = 2; o->n_volt = 2; o->n_state = 14; break;
    case GEMB200_MOTOR_DFIM: o->n_motor = 5; o->n_cur = 2; o->n_volt = 4; o->n_state = 24; break; /* physical_systems.py:891-916 */
    default: return -1;
  }
  o->n_ode = 1 + o->n_motor;
  o->n_sub[0] = slot_nsub(c->converter_kind[0]);
  o->n_sub[1] = slot_nsub(c->converter_kind[1]);
  o->slot_off[0] = 0;
  o->slot_off[1] = o->n_sub[0];
  if (c->finite) o->n_act = (c->converter_kind[0] != 0) + (c->converter_kind[1] != 0);
  else o->n_act = slot_nvolt(c->converter_kind[0]) + slot_nvolt(c->converter_kind[1]);
  if (c->action_dq) o->n_act = c->motor_kind == GEMB200_MOTOR_EESM ? 3 : (c->motor_kind == GEMB200_MOTOR_DFIM ? 4 : 2); /* dq_to_abc_action_processor.py:97-99,:110-111,:143-145 */
  o->n_ref = c->n_ref;
  /* widths after the wrappers: cos_sin_processor.py:44-58, flux_observer.py:66-75 */
  o->n_obs = o->n_state;
  for (int k = 0; k < c->n_state_ops; ++k) {
    if (c->sop_kind[k] == GEMB200_SOP_COS_SIN) o->n_obs += c->sop_idx[k][1] ? 1 : 2;
    else if (c->sop_kind[k] == GEMB200_SOP_FLUX_OBSERVER) o->n_obs += 2;
    else if (c->sop_kind[k] == GEMB200_SOP_CURRENT_SUM) o->n_obs += 1; /* current_sum_processor.py:29-31 */
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------------------------ */
/* model constants — the motors' _update_model methods                                                           */
/* ------------------------------------------------------------------------------------------------------------ */
static void update_model(gem_oracle* o) {
  const double* mp = o->cfg.motor_param;
  memset(o->mc, 0, sizeof(o->mc));
  double p = mp[GEMB200_MP_P], r_s = mp[GEMB200_MP_R_S], l_d = mp[GEMB200_MP_L_D], l_q = mp[GEMB200_MP_L_Q];
  switch (o->cfg.motor_kind) {
    case GEMB200_MOTOR_PERMEX_DC: { /* dc_permanently_excited_motor.py:71-75  features [omega, i, u] */
      double l_a = mp[GEMB200_MP_L_A];
      o->mc_rows = 1; o->mc_cols = 3;
      o->mc[0][0] = -mp[GEMB200_MP_PSI_E] / l_a; o->mc[0][1] = -mp[GEMB200_MP_R_A] / l_a; o->mc[0][2] = 1.0 / l_a;
    } break;
    case GEMB200_MOTOR_SERIES_DC: { /* dc_series_motor.py:66-70  features [i, omega*i, u] */
      double l = mp[GEMB200_MP_L_A] + mp[GEMB200_MP_L_E];
      o->mc_rows = 1; o->mc_cols = 3;
      o->mc[0][0] = (-mp[GEMB200_MP_R_A] - mp[GEMB200_MP_R_E]) / l; o->mc[0][1] = -mp[GEMB200_MP_L_E_PRIME] / l; o->mc[0][2] = 1.0 / l;
    } break;
    case GEMB200_MOTOR_SHUNT_DC:
    case GEMB200_MOTOR_EXTEX_DC: { /* dc_motor.py:95-104  features [i_a, i_e, omega*i_e, u_a, u_e] */
      double l_a = mp[GEMB200_MP_L_A], l_e = mp[GEMB200_MP_L_E];
      o->mc_rows = 2; o->mc_cols = 5;
      o->mc[0][0] = -mp[GEMB200_MP_R_A] / l_a; o->mc[0][2] = -mp[GEMB200_MP_L_E_PRIME] / l_a; o->mc[0][3] = 1.0 / l_a;
      o->mc[1][1] = -mp[GEMB200_MP_R_E] / l_e; o->mc[1][4] = 1.0 / l_e;
    } break;
    case GEMB200_MOTOR_PMSM: { /* permanent_magnet_synchronous_motor.py:107-119
                                  features [omega, i_d, i_q, u_d, u_q, omega*i_d, omega*i_q] */
      double psi_p = mp[GEMB200_MP_PSI_P];
      o->mc_rows = 3; o->mc_cols = 7;
      o->mc[0][1] = -r_s / l_d; o->mc[0][3] = 1.0 / l_d; o->mc[0][6] = l_q * p / l_d;
      o->mc[1][0] = -psi_p * p / l_q; o->mc[1][2] = -r_s / l_q; o->mc[1][4] = 1.0 / l_q; o->mc[1][5] = -l_d * p / l_q;
      o->mc[2][0] = p;
    } break;
    case GEMB200_MOTOR_SYNRM: { /* synchronous_reluctance_motor.py:117-131 */
      o->mc_rows = 3; o->mc_cols = 7;
      o->mc[0][1] = -r_s / l_d; o->mc[0][3] = 1.0 / l_d; o->mc[0][6] = l_q * p / l_d;
      o->mc[1][2] = -r_s / l_q; o->mc[1][4] = 1.0 / l_q; o->mc[1][5] = -l_d * p / l_q;
      o->mc[2][0] = p;
    } break;
    case GEMB200_MOTOR_EESM: { /* externally_excited_synchronous_motor.py:125-153
        features [omega, i_d, i_q, i_e, u_d, u_q, u_e, omega*i_d, omega*i_q, omega*i_e] */
      double k = mp[GEMB200_MP_K], r_e = mp[GEMB200_MP_R_E], l_m = mp[GEMB200_MP_L_M], l_e = mp[GEMB200_MP_L_E];
      double r_E = k * k * 3.0 / 2.0 * r_e;
      double l_M = k * 3.0 / 2.0 * l_m;
      double l_E = k * k * 3.0 / 2.0 * l_e;
      double i_k_rs = 2.0 / 3.0 / k;
      double sigma = 1.0 - l_M * l_M / (l_d * l_E);
      o->l_M = l_M; o->i_k_rs = i_k_rs;
      o->mc_rows = 4; o->mc_cols = 10;
      double (*m)[MAXF] = o->mc;
      m[0][1] = -r_s / sigma; m[0][3] = l_M * r_E / (sigma * l_E) * i_k_rs; m[0][4] = 1.0 / sigma;
      m[0][6] = -l_M * k / (sigma * l_E); m[0][8] = l_q * p / sigma;
      m[1][2] = -r_s; m[1][5] = 1.0; m[1][7] = -l_d * p; m[1][9] = -p * l_M * i_k_rs;
      m[2][1] = l_M * r_s / (sigma * l_d); m[2][3] = -r_E / sigma * i_k_rs; m[2][4] = -l_M / (sigma * l_d);
      m[2][6] = k / sigma; m[2][8] = -p * l_M * l_q / (sigma * l_d);
      m[3][0] = p;
      for (int j = 0; j < 10; ++j) { m[0][j] = m[0][j] / l_d; m[1][j] = m[1][j] / l_q; m[2][j] = m[2][j] / l_E / i_k_rs; }
    } break;
    case GEMB200_MOTOR_DFIM:
    case GEMB200_MOTOR_SCIM: { /* induction_motor.py:287-310
        features [omega, i_a, i_b, psi_a, psi_b, omega*psi_a, omega*psi_b, u_sa, u_sb, u_ra, u_rb] */
      double l_m = mp[GEMB200_MP_L_M], r_r = mp[GEMB200_MP_R_E];
      double l_s = l_m + mp[GEMB200_MP_L_SIGS], l_r = l_m + mp[GEMB200_MP_L_SIGR];
      double sigma = (l_s * l_r - l_m * l_m) / (l_s * l_r);
      double tau_r = l_r / r_r;
      double tau_sig = sigma * l_s / (r_s + r_r * (l_m * l_m) / (l_r * l_r));
      o->mc_rows = 5; o->mc_cols = 11;
      double (*m)[MAXF] = o->mc;
      m[0][1] = -1 / tau_sig; m[0][3] = l_m * r_r / (sigma * l_s * l_r * l_r); m[0][6] = l_m * p / (sigma * l_r * l_s);
      m[0][7] = 1 / (sigma * l_s); m[0][9] = -l_m / (sigma * l_r * l_s);
      m[1][2] = -1 / tau_sig; m[1][4] = l_m * r_r / (sigma * l_s * l_r * l_r); m[1][5] = -l_m * p / (sigma * l_r * l_s);
      m[1][8] = 1 / (sigma * l_s); m[1][10] = -l_m / (sigma * l_r * l_s);
      m[2][1] = l_m / tau_r; m[2][3] = -1 / tau_r; m[2][6] = -p; m[2][9] = 1;
      m[3][2] = l_m / tau_r; m[3][4] = -1 / tau_r; m[3][5] = p; m[3][10] = 1;
      m[4][0] = p;
      o->tq0 = 1.5 * p * l_m / (l_m + mp[GEMB200_MP_L_SIGR]);
    } break;
  }
  /* MechanicalLoad.set_j_rotor mechanical_load.py:188-193 ; PolynomialStaticLoad.set_j_rotor polynomial_static_load.py:60-64 */
  const double* lp = o->cfg.load_param;
  o->j_total = lp[GEMB200_LP_J_LOAD] + mp[GEMB200_MP_J_ROTOR];
  o->omega_lin = o->j_total / lp[GEMB200_LP_TAU_DECAY];
  o->omega_lim = lp[GEMB200_LP_A] / o->j_total * lp[GEMB200_LP_TAU_DECAY];
}

/* ElectricMotor.electrical_ode: np.matmul(_model_constants, features) */
static void electrical_ode(const gem_oracle* o, const double* ms, const double* u, double omega, double* d) {
  double f[MAXF];
  int n = 0;
  switch (o->cfg.motor_kind) {
    case GEMB200_MOTOR_PERMEX_DC: f[0] = omega; f[1] = ms[0]; f[2] = u[0]; n = 3; break; /* dc_permanently_excited_motor.py:81-84 */
    case GEMB200_MOTOR_SERIES_DC: f[0] = ms[0]; f[1] = omega * ms[0]; f[2] = u[0]; n = 3; break; /* dc_series_motor.py:76-81 */
    case GEMB200_MOTOR_SHUNT_DC: /* dc_shunt_motor.py:70-72: u_in -> (u, u) */
      f[0] = ms[0]; f[1] = ms[1]; f[2] = omega * ms[1]; f[3] = u[0]; f[4] = u[0]; n = 5; break;
    case GEMB200_MOTOR_EXTEX_DC: /* dc_motor.py:114-128 */
      f[0] = ms[0]; f[1] = ms[1]; f[2] = omega * ms[1]; f[3] = u[0]; f[4] = u[1]; n = 5; break;
    case GEMB200_MOTOR_PMSM:
    case GEMB200_MOTOR_SYNRM: /* synchronous_motor.py:143-168 */
      f[0] = omega; f[1] = ms[0]; f[2] = ms[1]; f[3] = u[0]; f[4] = u[1]; f[5] = omega * ms[0]; f[6] = omega * ms[1]; n = 7; break;
    case GEMB200_MOTOR_EESM: /* externally_excited_synchronous_motor.py:155-185 */
      f[0] = omega; f[1] = ms[0]; f[2] = ms[1]; f[3] = ms[2]; f[4] = u[0]; f[5] = u[1]; f[6] = u[2];
      f[7] = omega * ms[0]; f[8] = omega * ms[1]; f[9] = omega * ms[2]; n = 10; break;
    case GEMB200_MOTOR_SCIM: /* induction_motor.py:187-217 with rotor voltages 0 (squirrel_cage_induction_motor.py:121-129) */
      f[0] = omega; f[1] = ms[0]; f[2] = ms[1]; f[3] = ms[2]; f[4] = ms[3]; f[5] = omega * ms[2]; f[6] = omega * ms[3];
      f[7] = u[0]; f[8] = u[1]; f[9] = 0.0; f[10] = 0.0; n = 11; break;
    case GEMB200_MOTOR_DFIM: /* induction_motor.py:187-217, u = [u_salpha, u_sbeta, u_ralpha, u_rbeta] */
      f[0] = omega; f[1] = ms[0]; f[2] = ms[1]; f[3] = ms[2]; f[4] = ms[3]; f[5] = omega * ms[2]; f[6] = omega * ms[3];
      f[7] = u[0]; f[8] = u[1]; f[9] = u[2]; f[10] = u[3]; n = 11; break;
  }
  for (int i = 0; i < o->mc_rows; ++i) {
    double s = 0.0;
    for (int j = 0; j < n; ++j) s += o->mc[i][j] * f[j];
    d[i] = s;
  }
}

static double torque(const gem_oracle* o, const double* ms) {
  const double* mp = o->cfg.motor_param;
  switch (o->cfg.motor_kind) {
    case GEMB200_MOTOR_PERMEX_DC: return mp[GEMB200_MP_PSI_E] * ms[0];            /* dc_permanently_excited_motor.py:67-69 */
    case GEMB200_MOTOR_SERIES_DC: return mp[GEMB200_MP_L_E_PRIME] * ms[0] * ms[0]; /* dc_series_motor.py:72-74 */
    case GEMB200_MOTOR_SHUNT_DC:
    case GEMB200_MOTOR_EXTEX_DC: return mp[GEMB200_MP_L_E_PRIME] * ms[0] * ms[1];  /* dc_motor.py:106-108 */
    case GEMB200_MOTOR_PMSM: /* permanent_magnet_synchronous_motor.py:134-139 */
      return 1.5 * mp[GEMB200_MP_P] * (mp[GEMB200_MP_PSI_P] + (mp[GEMB200_MP_L_D] - mp[GEMB200_MP_L_Q]) * ms[0]) * ms[1];
    case GEMB200_MOTOR_SYNRM: /* synchronous_reluctance_motor.py:137-139 */
      return 1.5 * mp[GEMB200_MP_P] * ((mp[GEMB200_MP_L_D] - mp[GEMB200_MP_L_Q]) * ms[0]) * ms[1];
    case GEMB200_MOTOR_EESM: /* externally_excited_synchronous_motor.py:200-203 */
      return 1.5 * mp[GEMB200_MP_P] * (o->l_M * ms[2] * o->i_k_rs + (mp[GEMB200_MP_L_D] - mp[GEMB200_MP_L_Q]) * ms[0]) * ms[1];
    case GEMB200_MOTOR_DFIM:
    case GEMB200_MOTOR_SCIM: /* induction_motor.py:236-249 */
      return o->tq0 * (ms[2] * ms[1] - ms[3] * ms[0]);
  }
  return 0.0;
}

/* MechanicalLoad.mechanical_ode */
static double mechanical_ode(const gem_oracle* o, double omega, double tq, double g) {
  if (o->cfg.load_kind == GEMB200_LOAD_CONST_SPEED) return 0.0; /* constant_speed_load.py:40-42 */
  if (o->cfg.load_kind == GEMB200_LOAD_EXT_SPEED) /* external_speed_load.py:62-68; g = speed_profile(t + tau_load) at this stage's time */
    return (g - omega) / o->cfg.load_param[GEMB200_LP_TAU_LOAD];
  /* polynomial_static_load.py:87-99 */
  const double* lp = o->cfg.load_param;
  double sign = omega > 0 ? 1.0 : (omega < 0 ? -1.0 : 0.0);
  double a = fabs(omega) > o->omega_lim ? sign * lp[GEMB200_LP_A] : o->omega_lin * omega;
  double static_torque = sign * lp[GEMB200_LP_C] * omega * omega + lp[GEMB200_LP_B] * omega + a;
  return (tq - static_torque) / o->j_total;
}

/* RCVoltageSupply.system_equation voltage_supplies.py:104-113: d u_sup/dt = ((u_0 - u_sup) / R - i_sup) / C, written over the common
 * denominator; AC1PhaseSupply.get_voltage :163-166: sqrt(2) u_nominal sin(2 pi f t + phi) */
static double rc_supply_rhs(double u_sup, double u_0, double i_sup, double r, double cap) { return (u_0 - u_sup - r * i_sup) / (r * cap); }
static double ac1_voltage(double u_nominal, double f, double phi, double t) { return sqrt(2.0) * u_nominal * sin(2 * M_PI * f * t + phi); }

/* SCMLSystem._system_equation physical_systems.py:205-236 */
static void system_equation(const gem_oracle* o, const double* y, const double* u, double* dy, double g) {
  double tq = torque(o, y + 1);
  dy[0] = mechanical_ode(o, y[0], tq, g);
  electrical_ode(o, y + 1, u, y[0], dy + 1);
}

/* ------------------------------------------------------------------------------------------------------------ */
/* solvers                                                                                                       */
/* ------------------------------------------------------------------------------------------------------------ */
/* EulerSolver solvers.py:79-136 as a stepping scheme over an arbitrary right-hand side (the motor system below; the reference's
 * test system in the known-answer probe at the end of the file).  gt: external speed profile samples f(t_stage + tau_load) on the
 * grid of half sub-steps of THIS step (NULL otherwise). */
typedef void (*rhs_fn)(const void* ctx, const double* y, const double* u, double* dy, double g);
static void euler_core(rhs_fn f, const void* ctx, int n, double* y, double dt, int nsteps, const double* u, const double* gt) {
  double dy[GEMB200_MAX_ODE];
  if (nsteps <= 1) { /* solvers.py:124-136 */
    f(ctx, y, u, dy, gt ? gt[0] : 0.0);
    for (int i = 0; i < n; ++i) y[i] = y[i] + dy[i] * dt;
    return;
  }
  /* solvers.py:103-122; the time quirk (RHS evaluated one step + one sub-step late) only matters for the external speed load */
  double tau = dt / nsteps;
  for (int s = 0; s < nsteps; ++s) {
    f(ctx, y, u, dy, gt ? gt[2 * nsteps + 2 * (s + 1)] : 0.0); /* current_t = t (the END time), RHS at current_t + tau :113-118 */
    for (int i = 0; i < n; ++i) y[i] = y[i] + dy[i] * tau;
  }
}
static void motor_rhs(const void* ctx, const double* y, const double* u, double* dy, double g) { system_equation((const gem_oracle*)ctx, y, u, dy, g); }
static void integrate_euler(const gem_oracle* o, double* y, double dt, int nsteps, const double* u, const double* gt) {
  euler_core(motor_rhs, o, o->n_ode, y, dt, nsteps, u, gt);
}

static void integrate_rk4(const gem_oracle* o, double* y, double dt, int nsteps, const double* u, const double* gt) {
  /* classic RK4; mirrors the test-side RK4Solver plugin in tests/golden/make_golden.py that produced the goldens */
  int n = o->n_ode;
  if (nsteps < 1) nsteps = 1;
  double h = dt / nsteps;
  double k1[GEMB200_MAX_ODE], k2[GEMB200_MAX_ODE], k3[GEMB200_MAX_ODE], k4[GEMB200_MAX_ODE], yt[GEMB200_MAX_ODE];
  for (int s = 0; s < nsteps; ++s) {
    const double g0 = gt ? gt[2 * s] : 0.0, g1 = gt ? gt[2 * s + 1] : 0.0, g2 = gt ? gt[2 * s + 2] : 0.0; /* t, t + h/2, t + h */
    system_equation(o, y, u, k1, g0);
    for (int i = 0; i < n; ++i) yt[i] = y[i] + 0.5 * h * k1[i];
    system_equation(o, yt, u, k2, g1);
    for (int i = 0; i < n; ++i) yt[i] = y[i] + 0.5 * h * k2[i];
    system_equation(o, yt, u, k3, g1);
    for (int i = 0; i < n; ++i) yt[i] = y[i] + h * k3[i];
    system_equation(o, yt, u, k4, g2);
    for (int i = 0; i < n; ++i) y[i] = y[i] + h / 6.0 * (k1[i] + 2 * k2[i] + 2 * k3[i] + k4[i]);
  }
}

/* scipy.integrate.ode('dopri5') with the defaults the reference uses (solvers.py:155-184): rtol=1e-6, atol=1e-12,
 * nsteps=500, first_step=0 (-> Hairer's HINIT), safety=0.9, ifactor=10, dfactor=0.2, beta=0 (-> 0.04 inside the
 * integrator).  Restates the published Dormand-Prince 5(4) core (Hairer, Norsett, Wanner, "Solving ODEs I", DOPRI5);
 * scipy is a dependency of the reference, not part of /root/reference (requirements.txt:3, unpinned; 1.18.1 here). */
static double integrate_dopri5(const gem_oracle* o, double* y, double t_start, double t_end, const double* u) {
  const double dt = t_end - t_start;
  const double uround = 2.3e-16; /* dopri5.f default UROUND */
  const int n = o->n_ode;
  const double rtol = 1e-6, atol = 1e-12, safe = 0.9, fac1 = 0.2, fac2 = 10.0, beta = 0.04;
  const double expo1 = 0.2 - beta * 0.75, facc1 = 1.0 / fac1, facc2 = 1.0 / fac2;
  static const double a21 = 0.2, a31 = 3.0 / 40.0, a32 = 9.0 / 40.0, a41 = 44.0 / 45.0, a42 = -56.0 / 15.0, a43 = 32.0 / 9.0,
                      a51 = 19372.0 / 6561.0, a52 = -25360.0 / 2187.0, a53 = 64448.0 / 6561.0, a54 = -212.0 / 729.0,
                      a61 = 9017.0 / 3168.0, a62 = -355.0 / 33.0, a63 = 46732.0 / 5247.0, a64 = 49.0 / 176.0, a65 = -5103.0 / 18656.0,
                      a71 = 35.0 / 384.0, a73 = 500.0 / 1113.0, a74 = 125.0 / 192.0, a75 = -2187.0 / 6784.0, a76 = 11.0 / 84.0,
                      e1 = 71.0 / 57600.0, e3 = -71.0 / 16695.0, e4 = 71.0 / 1920.0, e5 = -17253.0 / 339200.0, e6 = 22.0 / 525.0, e7 = -1.0 / 40.0;
  double k1[GEMB200_MAX_ODE], k2[GEMB200_MAX_ODE], k3[GEMB200_MAX_ODE], k4[GEMB200_MAX_ODE], k5[GEMB200_MAX_ODE], k6[GEMB200_MAX_ODE];
  double y1[GEMB200_MAX_ODE], ysti[GEMB200_MAX_ODE];
  double x = t_start, xend = t_end, posneg = dt >= 0 ? 1.0 : -1.0, hmax = fabs(dt);
  double facold = 1e-4;
  system_equation(o, y, u, k1, 0.0);
  /* HINIT */
  double h;
  {
    double dnf = 0, dny = 0;
    for (int i = 0; i < n; ++i) { double sk = atol + rtol * fabs(y[i]); dnf += (k1[i] / sk) * (k1[i] / sk); dny += (y[i] / sk) * (y[i] / sk); }
    h = (dnf <= 1e-10 || dny <= 1e-10) ? 1e-6 : sqrt(dny / dnf) * 0.01;
    h = fmin(h, hmax) * posneg;
    for (int i = 0; i < n; ++i) y1[i] = y[i] + h * k1[i];
    system_equation(o, y1, u, k2, 0.0);
    double der2 = 0;
    for (int i = 0; i < n; ++i) { double sk = atol + rtol * fabs(y[i]); double d = (k2[i] - k1[i]) / sk; der2 += d * d; }
    der2 = sqrt(der2) / h;
    double der12 = fmax(fabs(der2), sqrt(dnf));
    double h1 = der12 <= 1e-15 ? fmax(1e-6, fabs(h) * 1e-3) : pow(0.01 / der12, 1.0 / 5.0);
    h = fmin(fmin(100 * fabs(h), h1), hmax) * posneg;
  }
  int last = 0, reject = 0;
  for (int nstep = 0; nstep <= 500; ++nstep) {
    /* IDID=-3 "step size too small": scipy only warns, ode.integrate returns the state reached so far and the
     * reference carries on with solver.t NOT advanced (physical_systems.py:514).  This really happens with the
     * default solver on Finite envs when the state is round-off-sized (|y|~1e-16, atol=1e-12), see DESIGN.md. */
    if (0.1 * fabs(h) <= fabs(x) * uround) return x;
    if ((x + 1.01 * h - xend) * posneg > 0.0) { h = xend - x; last = 1; }
    for (int i = 0; i < n; ++i) y1[i] = y[i] + h * a21 * k1[i];
    system_equation(o, y1, u, k2, 0.0);
    for (int i = 0; i < n; ++i) y1[i] = y[i] + h * (a31 * k1[i] + a32 * k2[i]);
    system_equation(o, y1, u, k3, 0.0);
    for (int i = 0; i < n; ++i) y1[i] = y[i] + h * (a41 * k1[i] + a42 * k2[i] + a43 * k3[i]);
    system_equation(o, y1, u, k4, 0.0);
    for (int i = 0; i < n; ++i) y1[i] = y[i] + h * (a51 * k1[i] + a52 * k2[i] + a53 * k3[i] + a54 * k4[i]);
    system_equation(o, y1, u, k5, 0.0);
    for (int i = 0; i < n; ++i) ysti[i] = y[i] + h * (a61 * k1[i] + a62 * k2[i] + a63 * k3[i] + a64 * k4[i] + a65 * k5[i]);
    system_equation(o, ysti, u, k6, 0.0);
    for (int i = 0; i < n; ++i) y1[i] = y[i] + h * (a71 * k1[i] + a73 * k3[i] + a74 * k4[i] + a75 * k5[i] + a76 * k6[i]);
    system_equation(o, y1, u, k2, 0.0);
    double err = 0;
    for (int i = 0; i < n; ++i) {
      k4[i] = (e1 * k1[i] + e3 * k3[i] + e4 * k4[i] + e5 * k5[i] + e6 * k6[i] + e7 * k2[i]) * h;
      double sk = atol + rtol * fmax(fabs(y[i]), fabs(y1[i]));
      err += (k4[i] / sk) * (k4[i] / sk);
    }
    err = sqrt(err / n);
    double fac11 = pow(err, expo1);
    double fac = fac11 / pow(facold, beta);
    fac = fmax(facc2, fmin(facc1, fac / safe));
    double hnew = h / fac;
    if (err <= 1.0) {
      facold = fmax(err, 1e-4);
      for (int i = 0; i < n; ++i) { k1[i] = k2[i]; y[i] = y1[i]; }
      x += h;
      if (last) return xend;
      if (fabs(hnew) > hmax) hnew = posneg * hmax;
      if (reject) hnew = posneg * fmin(fabs(hnew), fabs(h));
      reject = 0;
    } else {
      hnew = h / fmin(facc1, fac11 / safe);
      reject = 1;
      last = 0;
    }
    h = hnew;
  }
  return x; /* IDID=-2: more than nsteps=500 steps needed */
}

/* OdeSolver.integrate(t): returns the time actually reached (== t_end except for a failing dopri5) */
static double integrate(const gem_oracle* o, double* y, double t_start, double t_end, const double* u, const double* gt) {
  switch (o->cfg.solver_kind) {
    case GEMB200_SOLVER_EULER: integrate_euler(o, y, t_end - t_start, o->cfg.solver_nsteps, u, gt); return t_end;
    case GEMB200_SOLVER_RK4: integrate_rk4(o, y, t_end - t_start, o->cfg.solver_nsteps, u, gt); return t_end;
    default: return integrate_dopri5(o, y, t_start, t_end, u); /* adaptive stage times: no table for the external speed load */
  }
}

/* ------------------------------------------------------------------------------------------------------------ */
/* converters (converters.py)                                                                                    */
/* ------------------------------------------------------------------------------------------------------------ */
static double clip(double x, double lo, double hi) { return fmin(fmax(x, lo), hi); } /* min(max(.)) :146 */
static double sgn(double x) { return x > 0 ? 1.0 : (x < 0 ? -1.0 : 0.0); }         /* np.sign :184 */

/* interlocking time of the sub-converter a half bridge belongs to (slot 1 of a multi converter may have its own, converters.py:615-740) */
static double il_slot(const gem_oracle* o, int slot) {
  return (slot == 1 && o->cfg.interlocking_time1 >= 0) ? o->cfg.interlocking_time1 : o->cfg.interlocking_time;
}
/* FiniteTwoQuadrantConverter._set_switching_pattern :300-310; returns number of switching times (1 or 2) */
static int f2qc_set_action(const gem_oracle* o, sub2qc_t* s, int action, double t, double il) {
  s->action_start_time = t;
  s->cur_action_i = action;
  if (action == 0 || s->switching_state == 0 || action == s->switching_state || il == 0) {
    s->pattern[0] = action; s->pattern_len = 1;
    return 1;
  }
  s->pattern[0] = 0; s->pattern[1] = action; s->pattern_len = 2;
  return 2;
}
/* FiniteTwoQuadrantConverter.convert :270-287 */
static double f2qc_convert(const gem_oracle* o, sub2qc_t* s, double i_out, double t, double il) {
  if (t - o->cfg.tau / 1000 > s->action_start_time + il) s->switching_state = s->pattern[s->pattern_len - 1];
  else s->switching_state = s->pattern[0];
  if (s->switching_state == 0) return i_out < 0 ? 1.0 : 0.0;
  if (s->switching_state == 1) return 1.0;
  return 0.0;
}
/* FiniteTwoQuadrantConverter.i_sup :289-298 */
static double f2qc_i_sup(const sub2qc_t* s, double i_out) {
  if (s->switching_state == 0) return i_out < 0 ? i_out : 0.0;
  if (s->switching_state == 1) return i_out;
  return 0.0;
}
/* ContTwoQuadrantConverter via ContDynamicallyAveragedConverter.convert :148-158, _interlock :176-184 */
static double c2qc_convert(const gem_oracle* o, const sub2qc_t* s, double i_out, double il) {
  return clip(s->cur_action - sgn(i_out) / o->cfg.tau * il, 0.0, 1.0);
}
/* ContTwoQuadrantConverter.i_sup :429-435 */
static double c2qc_i_sup(const gem_oracle* o, const sub2qc_t* s, double i_out, double il) {
  double ic = i_out < 0 ? 1.0 : 0.0;
  return (s->cur_action + il / o->cfg.tau * (ic - s->cur_action)) * i_out;
}

static const int B6_SUBACTIONS[8][3] = {{2, 2, 2}, {2, 2, 1}, {2, 1, 2}, {2, 1, 1}, {1, 2, 2}, {1, 2, 1}, {1, 1, 2}, {1, 1, 1}}; /* :788-797 */

/* converter.set_action: returns the number of switching segments (1..3) and their END times: the sorted unique switching times of the
 * sub-converters (FiniteMultiConverter.set_action :583-595) — {t+tau}, {t+t_il, t+tau}, or with two different interlocking times
 * {t+t_lo, t+t_hi, t+tau}.  seg_off (may be NULL): the same ends as offsets from t, {tau}, {t_il, tau} or {t_lo, t_hi, tau}. */
static int conv_set_action_off(const gem_oracle* o, env_t* e, const double* act_f, const int32_t* act_i, double t, double* seg_end, double* seg_off) {
  int sw[2] = {0, 0};
  int ai = 0, af = 0;
  for (int slot = 0; slot < 2; ++slot) {
    int kind = o->cfg.converter_kind[slot];
    if (kind == GEMB200_CONV_NONE) continue;
    sub2qc_t* s = e->sub + o->slot_off[slot];
    if (o->cfg.finite) {
      int a = act_i[ai++];
      switch (kind) {
        case GEMB200_CONV_1QC: e->cur_action1qc[slot] = a; break; /* :59-61 */
        case GEMB200_CONV_2QC: if (f2qc_set_action(o, s, a, t, il_slot(o, slot)) > 1) sw[slot] = 1; break;
        case GEMB200_CONV_4QC: { /* :350-360 */
          static const int a0[4] = {1, 1, 2, 2}, a1[4] = {1, 2, 1, 2};
          if (f2qc_set_action(o, s, a0[a], t, il_slot(o, slot)) > 1) sw[slot] = 1;
          if (f2qc_set_action(o, s + 1, a1[a], t, il_slot(o, slot)) > 1) sw[slot] = 1;
        } break;
        case GEMB200_CONV_B6: /* :824-835 */
          for (int l = 0; l < 3; ++l) if (f2qc_set_action(o, s + l, B6_SUBACTIONS[a][l], t, il_slot(o, slot)) > 1) sw[slot] = 1;
          break;
      }
    } else {
      switch (kind) {
        case GEMB200_CONV_1QC: /* :371-401, clip to its action space [0,1] :144-146 */
        case GEMB200_CONV_2QC: s->cur_action = clip(act_f[af++], 0.0, 1.0); break;
        case GEMB200_CONV_4QC: { /* :484-491 */
          double a = act_f[af++];
          s[0].cur_action = clip(0.5 * (a + 1), 0.0, 1.0);
          s[1].cur_action = clip(-0.5 * (a - 1), 0.0, 1.0);
        } break;
        case GEMB200_CONV_B6: /* :897-903 */
          for (int l = 0; l < 3; ++l) s[l].cur_action = clip(0.5 * (act_f[af++] + 1), 0.0, 1.0);
          break;
      }
    }
  }
  int nseg = 0;
  const double il0 = il_slot(o, 0), il1 = il_slot(o, 1), t0 = t + il0, t1 = t + il1;
  double off[3];
  if (sw[0] && sw[1] && t0 != t1) { seg_end[nseg] = fmin(t0, t1); off[nseg++] = fmin(il0, il1); seg_end[nseg] = fmax(t0, t1); off[nseg++] = fmax(il0, il1); }
  else if (sw[0]) { seg_end[nseg] = t0; off[nseg++] = il0; }
  else if (sw[1]) { seg_end[nseg] = t1; off[nseg++] = il1; }
  seg_end[nseg] = t + o->cfg.tau; off[nseg++] = o->cfg.tau;
  if (seg_off) for (int j = 0; j < nseg; ++j) seg_off[j] = off[j];
  return nseg;
}
static int conv_set_action(const gem_oracle* o, env_t* e, const double* act_f, const int32_t* act_i, double t, double* seg_end) {
  return conv_set_action_off(o, e, act_f, act_i, t, seg_end, NULL);
}

/* converter.convert(i_out, t) -> u_in (not yet multiplied by u_sup); i_out laid out per slot */
static void conv_convert(const gem_oracle* o, env_t* e, const double* i_out, double t, double* u_out) {
  int io = 0, uo = 0;
  for (int slot = 0; slot < 2; ++slot) {
    int kind = o->cfg.converter_kind[slot];
    if (kind == GEMB200_CONV_NONE) continue;
    sub2qc_t* s = e->sub + o->slot_off[slot];
    if (o->cfg.finite) {
      switch (kind) {
        case GEMB200_CONV_1QC: u_out[uo++] = i_out[io] >= 0 ? (double)e->cur_action1qc[slot] : 1.0; io++; break; /* :236-238 */
        case GEMB200_CONV_2QC: u_out[uo++] = f2qc_convert(o, s, i_out[io], t, il_slot(o, slot)); io++; break;
        case GEMB200_CONV_4QC: u_out[uo++] = f2qc_convert(o, s, i_out[io], t, il_slot(o, slot)) - f2qc_convert(o, s + 1, -i_out[io], t, il_slot(o, slot)); io++; break; /* :346-348 */
        case GEMB200_CONV_B6: for (int l = 0; l < 3; ++l) u_out[uo++] = f2qc_convert(o, s + l, i_out[io++], t, il_slot(o, slot)) - 0.5; break; /* :814-822 */
      }
    } else {
      switch (kind) {
        case GEMB200_CONV_1QC: u_out[uo++] = clip(i_out[io] >= 0 ? s->cur_action : 1.0, 0.0, 1.0); io++; break; /* :388-394 */
        case GEMB200_CONV_2QC: u_out[uo++] = c2qc_convert(o, s, i_out[io], il_slot(o, slot)); io++; break;
        case GEMB200_CONV_4QC: u_out[uo++] = c2qc_convert(o, s, i_out[io], il_slot(o, slot)) - c2qc_convert(o, s + 1, i_out[io], il_slot(o, slot)); io++; break; /* :480-482 (same i_out for both) */
        case GEMB200_CONV_B6: for (int l = 0; l < 3; ++l) u_out[uo++] = c2qc_convert(o, s + l, i_out[io++], il_slot(o, slot)) - 0.5; break; /* :888-895 */
      }
    }
  }
}

/* converter.i_sup — computed and ignored by the ideal supply (voltage_supplies.py:70-72); kept for fidelity */
static double conv_i_sup(const gem_oracle* o, const env_t* e, const double* i_out) {
  double r = 0;
  int io = 0;
  for (int slot = 0; slot < 2; ++slot) {
    int kind = o->cfg.converter_kind[slot];
    if (kind == GEMB200_CONV_NONE) continue;
    const sub2qc_t* s = e->sub + o->slot_off[slot];
    if (o->cfg.finite) {
      switch (kind) {
        case GEMB200_CONV_1QC: r += e->cur_action1qc[slot] == 1 ? i_out[io] : 0; io++; break;
        case GEMB200_CONV_2QC: r += f2qc_i_sup(s, i_out[io]); io++; break;
        case GEMB200_CONV_4QC: r += f2qc_i_sup(s, i_out[io]) + f2qc_i_sup(s + 1, -i_out[io]); io++; break;
        case GEMB200_CONV_B6: for (int l = 0; l < 3; ++l) r += f2qc_i_sup(s + l, i_out[io++]); break;
      }
    } else {
      switch (kind) {
        case GEMB200_CONV_1QC: r += s->cur_action * i_out[io]; io++; break;
        case GEMB200_CONV_2QC: r += c2qc_i_sup(o, s, i_out[io], il_slot(o, slot)); io++; break;
        case GEMB200_CONV_4QC: r += c2qc_i_sup(o, s, i_out[io], il_slot(o, slot)) + c2qc_i_sup(o, s + 1, -i_out[io], il_slot(o, slot)); io++; break;
        case GEMB200_CONV_B6: for (int l = 0; l < 3; ++l) r += c2qc_i_sup(o, s + l, i_out[io++], il_slot(o, slot)); break;
      }
    }
  }
  return r;
}

/* converter.reset(): [0.0] per QC, [-0.5]*3 for B6 (:45-54, :805-812, :880-886); _switching_state is NOT cleared */
static void conv_reset(const gem_oracle* o, env_t* e, double* u_out) {
  int uo = 0;
  for (int slot = 0; slot < 2; ++slot) {
    int kind = o->cfg.converter_kind[slot];
    if (kind == GEMB200_CONV_NONE) continue;
    sub2qc_t* s = e->sub + o->slot_off[slot];
    for (int l = 0; l < o->n_sub[slot]; ++l) { s[l].cur_action = 0.0; s[l].cur_action_i = 0; s[l].action_start_time = 0.0; }
    e->cur_action1qc[slot] = 0;
    if (kind == GEMB200_CONV_B6) { u_out[uo++] = -0.5; u_out[uo++] = -0.5; u_out[uo++] = -0.5; }
    else u_out[uo++] = 0.0;
  }
}

/* ------------------------------------------------------------------------------------------------------------ */
/* three-phase transforms three_phase_motor.py:18-88                                                             */
/* ------------------------------------------------------------------------------------------------------------ */
/* The matrices are pre-multiplied exactly like the reference's class attributes (_t23 = 2/3 * [[...]]) and the
 * products accumulated like np.matmul does for these tiny shapes, so that even the round-off residue
 * (e.g. u_dq ~ 1e-14 V for a zero vector) is reproduced; the default dopri5's behaviour depends on it. */
static void t_23(const double* abc, double* ab) {
  const double s3 = sqrt(3.0);
  const double m00 = 2.0 / 3.0 * 1.0, m01 = 2.0 / 3.0 * -0.5, m02 = 2.0 / 3.0 * -0.5;
  const double m11 = 2.0 / 3.0 * (0.5 * s3), m12 = 2.0 / 3.0 * (-0.5 * s3);
  /* accumulation order + fused multiply-adds of the BLAS gemv numpy dispatches to here (probed: reproduces
   * np.matmul(_t23, [210,210,210]) = [-1.0325e-14, 8.88e-16] bit for bit) */
  ab[0] = fma(m02, abc[2], fma(m00, abc[0], m01 * abc[1]));
  ab[1] = fma(m12, abc[2], fma(0.0, abc[0], m11 * abc[1]));
}
static void t_32(const double* ab, double* abc) {
  const double s3 = sqrt(3.0);
  abc[0] = 1.0 * ab[0] + 0.0 * ab[1];
  abc[1] = -0.5 * ab[0] + (0.5 * s3) * ab[1];
  abc[2] = -0.5 * ab[0] + (-0.5 * s3) * ab[1];
}
static void q_rot(const double* x, double eps, double* out) {
  double c = cos(eps), s = sin(eps);
  out[0] = c * x[0] - s * x[1];
  out[1] = s * x[0] + c * x[1];
}
static void abc_to_dq(const double* abc, double eps, double* dq) { double ab[2]; t_23(abc, ab); q_rot(ab, -eps, dq); }
static void dq_to_abc(const double* dq, double eps, double* abc) { double ab[2]; q_rot(dq, eps, ab); t_32(ab, abc); }

static double wrap_eps(double eps) { /* physical_systems.py:520-522: python float % */
  double r = fmod(eps, 2 * M_PI);
  if (r < 0) r += 2 * M_PI;
  if (r > M_PI) r -= 2 * M_PI;
  return r;
}

/* standard normal CDF and its inverse (Wichura's AS 241, PPND16: relative accuracy 1e-16) for the truncated-normal initialiser */
static double norm_cdf(double x) { return 0.5 * erfc(-x * M_SQRT1_2); }
static double norm_ppf(double p) {
  static const double a[8] = {3.3871328727963666080e0, 1.3314166789178437745e+2, 1.9715909503065514427e+3, 1.3731693765509461125e+4,
                              4.5921953931549871457e+4, 6.7265770927008700853e+4, 3.3430575583588128105e+4, 2.5090809287301226727e+3};
  static const double b[8] = {1.0, 4.2313330701600911252e+1, 6.8718700749205790830e+2, 5.3941960214247511077e+3, 2.1213794301586595867e+4,
                              3.9307895800092710610e+4, 2.8729085735721942674e+4, 5.2264952788528545610e+3};
  static const double cc[8] = {1.42343711074968357734e0, 4.63033784615654529590e0, 5.76949722146069140550e0, 3.64784832476320460504e0,
                               1.27045825245236838258e0, 2.41780725177450611770e-1, 2.27238449892691845833e-2, 7.74545014278341407640e-4};
  static const double d[8] = {1.0, 2.05319162663775882187e0, 1.67638483018380384940e0, 6.89767334985100004550e-1, 1.48103976427480074590e-1,
                              1.51986665636164571966e-2, 5.47593808499534494600e-4, 1.05075007164441684324e-9};
  static const double e[8] = {6.65790464350110377720e0, 5.46378491116411436990e0, 1.78482653991729133580e0, 2.96560571828504891230e-1,
                              2.65321895265761230930e-2, 1.24266094738807843860e-3, 2.71155556874348757815e-5, 2.01033439929228813265e-7};
  static const double f[8] = {1.0, 5.99832206555887937690e-1, 1.36929880922735805310e-1, 1.48753612908506148525e-2, 7.86869131145613259100e-4,
                              1.84631831751005468180e-5, 1.42151175831644588870e-7, 2.04426310338993978564e-15};
  const double q = p - 0.5;
  double r, num = 0, den = 0;
  if (fabs(q) <= 0.425) {
    r = 0.180625 - q * q;
    for (int i = 7; i >= 0; --i) { num = num * r + a[i]; den = den * r + b[i]; }
    return q * num / den;
  }
  r = q < 0 ? p : 1 - p;
  if (r <= 0) return q < 0 ? -INFINITY : INFINITY;
  r = sqrt(-log(r));
  if (r <= 5) { r -= 1.6; for (int i = 7; i >= 0; --i) { num = num * r + cc[i]; den = den * r + d[i]; } }
  else { r -= 5; for (int i = 7; i >= 0; --i) { num = num * r + e[i]; den = den * r + f[i]; } }
  return q < 0 ? -num / den : num / den;
}

/* DoublyFedInductionMotorSystem.calculate_rotor_current physical_systems.py:946-956; y = [omega, i_sa, i_sb, psi_ra, psi_rb, eps] */
static void dfim_rotor_current(const gem_oracle* o, const double* y, double* i_r) {
  const double* mp = o->cfg.motor_param;
  const double l_r = mp[GEMB200_MP_L_M] + mp[GEMB200_MP_L_SIGR];
  i_r[0] = 1 / l_r * y[3] - mp[GEMB200_MP_L_M] / l_r * y[1];
  i_r[1] = 1 / l_r * y[4] - mp[GEMB200_MP_L_M] / l_r * y[2];
}

/* ------------------------------------------------------------------------------------------------------------ */
/* simulate                                                                                                      */
/* ------------------------------------------------------------------------------------------------------------ */
static void simulate(const gem_oracle* o, env_t* e, const double* act_f, const int32_t* act_i, double* state) {
  const gemb200_config* c = &o->cfg;
  const int mk = c->motor_kind;
  double u_sup = c->u_sup; /* IdealVoltageSupply.get_voltage voltage_supplies.py:70-72 */
  double* y = e->ode;
  double i_in[6], u_in[6], u_solver[4];
  /* exact grid: step k of the episode starts at k tau and its segments have the lengths of the offsets' differences, tau, til,
   * tau - til and |til1 - til0| (computed in double like the device's seg_len); the reference's t accumulates instead */
  double t0 = o->exact_grid ? (double)e->k * c->tau : e->t;
  double seg_end[3], seg_off[3];
  int nseg = conv_set_action_off(o, e, act_f, act_i, t0, seg_end, seg_off);
  double t_solver = t0;
  const double* gt = NULL; /* ExternalSpeedLoad: the tabulated profile restarts at every reset (e->k = steps since then) */
  if (c->load_kind == GEMB200_LOAD_EXT_SPEED) {
    const long per = 2L * c->solver_nsteps, last = (long)c->ext_speed_len - 1 - 2 * per;
    const long j0 = e->k * per;
    gt = c->ext_speed_table + (j0 < last ? j0 : last);
  }
  double eps = 0.0, eps_fs = 0.0;
  for (int seg = 0; seg < nseg; ++seg) {
    /* currents flowing into the motor at the start of the segment, in converter coordinates */
    switch (mk) {
      case GEMB200_MOTOR_PERMEX_DC:
      case GEMB200_MOTOR_SERIES_DC: i_in[0] = y[1]; break;              /* physical_systems.py:174 */
      case GEMB200_MOTOR_SHUNT_DC: i_in[0] = y[1] + y[2]; break;         /* dc_shunt_motor.py:66-68 */
      case GEMB200_MOTOR_EXTEX_DC: i_in[0] = y[1]; i_in[1] = y[2]; break; /* dc_motor.py:110-112 */
      case GEMB200_MOTOR_PMSM:
      case GEMB200_MOTOR_SYNRM: eps = y[3]; dq_to_abc(y + 1, eps, i_in); break; /* :489-493, :505 */
      case GEMB200_MOTOR_EESM: eps = y[4]; dq_to_abc(y + 1, eps, i_in); i_in[3] = y[3]; break; /* :621-624 */
      case GEMB200_MOTOR_SCIM: eps_fs = atan2(y[4], y[3]); t_32(y + 1, i_in); break; /* :775-782, :765-769 */
      case GEMB200_MOTOR_DFIM: { /* :958-963 / :975-981 */
        double i_r[2];
        eps_fs = atan2(y[4], y[3]); eps = y[5];
        t_32(y + 1, i_in);
        dfim_rotor_current(o, y, i_r);
        t_32(i_r, i_in + 3); /* alphabeta_to_abc_space(calculate_rotor_current(.)) */
      } break;
    }
    double i_sup = conv_i_sup(o, e, i_in);    /* :507 */
    if (c->supply_kind == GEMB200_SUPPLY_AC1) /* AC1PhaseSupply.get_voltage(self._t) :163-166: the step's START time for all segments */
      u_sup = ac1_voltage(c->u_sup, c->supply_param[0], e->ac_phase, t0);
    if (c->supply_kind == GEMB200_SUPPLY_RC) { /* RCVoltageSupply.get_voltage(self._t, i_sup) :115-123: one Euler step from the previous
                                                  call's time to this step's start time; a second segment sees dt = 0 */
      if (seg == 0) {
        if (e->rc_started) e->u_rc += rc_supply_rhs(e->u_rc, c->u_sup, i_sup, c->supply_param[0], c->supply_param[1]) * c->tau;
        e->rc_started = 1;
      }
      u_sup = e->u_rc;
    }
    conv_convert(o, e, i_in, t_solver, u_in); /* :509 */
    for (int j = 0; j < 6; ++j) u_in[j] *= u_sup; /* :510 */
    switch (mk) {
      case GEMB200_MOTOR_PMSM:
      case GEMB200_MOTOR_SYNRM: abc_to_dq(u_in, eps, u_solver); break;                  /* :511 */
      case GEMB200_MOTOR_EESM: abc_to_dq(u_in, eps, u_solver); u_solver[2] = u_in[3]; break; /* :642 */
      case GEMB200_MOTOR_SCIM: t_23(u_in, u_solver); break;                             /* :797-799 */
      case GEMB200_MOTOR_DFIM: { /* :969-973 */
        double u_rdq[2];
        abc_to_dq(u_in + 3, eps_fs - eps, u_rdq);
        t_23(u_in, u_solver);
        q_rot(u_rdq, eps_fs, u_solver + 2);
      } break;
      default: u_solver[0] = u_in[0]; u_solver[1] = u_in[1]; break;
    }
    if (o->exact_grid && c->solver_kind == GEMB200_SOLVER_EULER) {
      integrate_euler(o, y, seg_off[seg] - (seg ? seg_off[seg - 1] : 0.0), c->solver_nsteps, u_solver, gt);
      t_solver = t0 + seg_off[seg];
    } else if (o->exact_grid && c->solver_kind == GEMB200_SOLVER_RK4) {
      integrate_rk4(o, y, seg_off[seg] - (seg ? seg_off[seg - 1] : 0.0), c->solver_nsteps, u_solver, gt);
      t_solver = t0 + seg_off[seg];
    } else {
      t_solver = integrate(o, y, t_solver, seg_end[seg], u_solver, gt); /* :513 */
    }
  }
  e->t = t_solver;
  e->k += 1;
  /* exact grid: the angle is kept in [-pi, pi) like the device's (fmod is exact); the reference's unwrapped float64 angle rounds at the
   * ulp of its magnitude, ~5e-9 rad after 1e5 steps at p omega = 300 rad/s, more than the fp64 parity bar */
  if (o->exact_grid && mk >= GEMB200_MOTOR_PMSM) {
    double* eps_state = y + o->n_ode - 1;
    *eps_state = fmod(*eps_state, 2 * M_PI);
    if (*eps_state >= M_PI) *eps_state -= 2 * M_PI;
    else if (*eps_state < -M_PI) *eps_state += 2 * M_PI;
  }
  const double* lim = c->limits;
  double tq = torque(o, y + 1);
  int n = 0;
  state[n++] = y[0];
  state[n++] = tq;
  switch (mk) {
    case GEMB200_MOTOR_PERMEX_DC:
    case GEMB200_MOTOR_SERIES_DC: state[n++] = y[1]; state[n++] = u_in[0]; break; /* :194-201 */
    case GEMB200_MOTOR_SHUNT_DC: state[n++] = y[1]; state[n++] = y[2]; state[n++] = u_in[0]; break;
    case GEMB200_MOTOR_EXTEX_DC: state[n++] = y[1]; state[n++] = y[2]; state[n++] = u_in[0]; state[n++] = u_in[1]; break;
    case GEMB200_MOTOR_PMSM:
    case GEMB200_MOTOR_SYNRM: { /* :516-525 (eps here is the angle at the start of the LAST segment) */
      double i_abc[3];
      dq_to_abc(y + 1, eps, i_abc);
      for (int j = 0; j < 3; ++j) state[n++] = i_abc[j];
      state[n++] = y[1]; state[n++] = y[2];
      for (int j = 0; j < 3; ++j) state[n++] = u_in[j];
      state[n++] = u_solver[0]; state[n++] = u_solver[1];
      state[n++] = wrap_eps(y[3]);
    } break;
    case GEMB200_MOTOR_EESM: { /* :646-657 */
      double i_abc[3];
      dq_to_abc(y + 1, eps, i_abc);
      for (int j = 0; j < 3; ++j) state[n++] = i_abc[j];
      state[n++] = y[1]; state[n++] = y[2]; state[n++] = y[3];
      for (int j = 0; j < 3; ++j) state[n++] = u_in[j];
      state[n++] = u_solver[0]; state[n++] = u_solver[1]; state[n++] = u_solver[2];
      state[n++] = wrap_eps(y[4]);
    } break;
    case GEMB200_MOTOR_DFIM: { /* :1000-1035: eps_fs / eps are still the angles at the start of the last segment */
      double u_sdq[2], u_rdq[2], i_sdq[2], i_sabc[3], i_r[2], i_rdq[2], i_rdef[3];
      abc_to_dq(u_in, eps_fs, u_sdq);
      abc_to_dq(u_in + 3, eps_fs - eps, u_rdq);
      q_rot(y + 1, -eps_fs, i_sdq);
      dq_to_abc(i_sdq, eps_fs, i_sabc);
      dfim_rotor_current(o, y, i_r);
      q_rot(i_r, -eps_fs, i_rdq);
      dq_to_abc(i_rdq, eps_fs - eps, i_rdef);
      for (int j = 0; j < 3; ++j) state[n++] = i_sabc[j];
      state[n++] = i_sdq[0]; state[n++] = i_sdq[1];
      for (int j = 0; j < 3; ++j) state[n++] = i_rdef[j];
      state[n++] = i_rdq[0]; state[n++] = i_rdq[1];
      for (int j = 0; j < 3; ++j) state[n++] = u_in[j];
      state[n++] = u_sdq[0]; state[n++] = u_sdq[1];
      for (int j = 0; j < 3; ++j) state[n++] = u_in[3 + j];
      state[n++] = u_rdq[0]; state[n++] = u_rdq[1];
      state[n++] = wrap_eps(y[5]);
    } break;
    case GEMB200_MOTOR_SCIM: { /* :794-814: u_dq and i_dq use the field angle at the start of the last segment */
      double u_dq[2], i_dq[2], i_abc[3];
      abc_to_dq(u_in, eps_fs, u_dq);
      q_rot(y + 1, -eps_fs, i_dq);
      dq_to_abc(i_dq, eps_fs, i_abc);
      for (int j = 0; j < 3; ++j) state[n++] = i_abc[j];
      state[n++] = i_dq[0]; state[n++] = i_dq[1];
      for (int j = 0; j < 3; ++j) state[n++] = u_in[j];
      state[n++] = u_dq[0]; state[n++] = u_dq[1];
      state[n++] = wrap_eps(y[5]);
    } break;
  }
  state[n++] = u_sup;
  for (int j = 0; j < n; ++j) state[j] = state[j] / lim[j];
  /* CurrentSumProcessor.simulate physical_system_wrappers/current_sum_processor.py:52-66: sum of the NORMALISED currents */
  if (mk == GEMB200_MOTOR_SHUNT_DC) state[n] = state[2] + state[3];
}

/* SCMLSystem.reset and overrides: physical_systems.py:256-287, :527-561, :659-693, :816-847 */
static void ps_reset(const gem_oracle* o, env_t* e, double* state) {
  const gemb200_config* c = &o->cfg;
  const int mk = c->motor_kind;
  double* y = e->ode;
  for (int j = 0; j < o->n_ode; ++j) y[j] = c->init_ode[j];
  if (c->init_random) {
    /* ElectricMotor.initialize / MechanicalLoad.initialize, random_init='uniform' (electric_motor.py:236-243,
     * mechanical_load.py:131-137): value = (upper - lower) * U + lower per state; bounds derived on the host.
     * (Philox stream instead of numpy's; one uniform per ODE state in ODE order.) */
    uint32_t r0[4], r1[4];
    int64_t idx = e - o->env;
    rng4(o, idx, STREAM_INIT_STATE, r0);
    rng4(o, idx, STREAM_INIT_STATE2, r1);
    double lo[GEMB200_MAX_ODE], hi[GEMB200_MAX_ODE];
    for (int j = 0; j < o->n_ode; ++j) { lo[j] = c->init_lo[j]; hi[j] = c->init_hi[j]; }
    for (int j = 0; j < o->n_ode; ++j) {
      if (c->init_im_valid && j == 3) {
        /* InductionMotor.reset -> _update_initial_limits(omega) (squirrel_cage_induction_motor.py:146-157, doubly_fed_induction_motor.py:154-165)
         * -> _flux_limit (induction_motor.py:250-285); initialize() then takes +-|limit| (electric_motor.py:197-213).  omega = y[0] is
         * this reset's speed, the currents are the ones the PREVIOUS initialize() call left in _initial_states. */
        if (!e->im_prev_set) { e->im_prev[0] = c->init_ode[1]; e->im_prev[1] = c->init_ode[2]; e->im_prev_set = 1; }
        const double eps_mag = 2 * M_PI * u01(r1[2]) - M_PI, ce = cos(eps_mag), se = sin(eps_mag), omega = y[0];
        double psi_d_max;
        if (omega == 0) psi_d_max = c->init_im[0];
        else {
          const double i_d = ce * e->im_prev[0] + se * e->im_prev[1], i_q = -se * e->im_prev[0] + ce * e->im_prev[1]; /* q_inv */
          double psi = (c->init_im[1] * omega * i_d + c->init_im[2] * i_q + c->init_im[3]) / (-c->init_im[4] * omega);
          psi_d_max = 0.9 * fmin(fmax(psi, 0.0), fabs(c->init_im[5] * i_d));
        }
        const double lim[2] = {fabs(psi_d_max * ce), fabs(psi_d_max * se)};
        for (int q = 0; q < 2; ++q) { lo[3 + q] = fmax(-lim[q], c->init_lo[3 + q]); hi[3 + q] = fmin(lim[q], c->init_hi[3 + q]); }
      }
      const double u = u01(j < 4 ? r0[j] : r1[j - 4]);
      y[j] = lo[j] + (hi[j] - lo[j]) * u;
      if (c->init_dist[j]) { /* random_init='gaussian': scipy.stats.truncnorm(a, b, loc=mue, scale=sigma) electric_motor.py:245-258, by inversion */
        const double mu = isnan(c->init_mu[j]) ? 0.5 * (hi[j] - lo[j]) + lo[j] : c->init_mu[j], sg = c->init_sigma[j];
        const double ca = norm_cdf((lo[j] - mu) / sg), cb = norm_cdf((hi[j] - mu) / sg);
        const double g = mu + sg * norm_ppf(ca + u * (cb - ca));
        y[j] = hi[j] > lo[j] ? fmin(fmax(g, lo[j]), hi[j]) : lo[j];
      }
    }
    if (c->init_im_valid) { e->im_prev[0] = y[1]; e->im_prev[1] = y[2]; }
  }
  double u_abc[6] = {0, 0, 0, 0, 0, 0};
  conv_reset(o, e, u_abc);
  e->u_rc = c->u_sup; e->rc_started = 0; /* supply.reset() -> [u_0] */
  double u_sup0 = c->u_sup;
  if (c->supply_kind == GEMB200_SUPPLY_AC1) { /* AC1PhaseSupply.reset :157-161 */
    e->ac_phase = c->supply_param[1];
    if (c->supply_param[2] == 0.0) { uint32_t r[4]; rng4(o, e - o->env, STREAM_SUPPLY, r); e->ac_phase = u01(r[0]) * 2 * M_PI; }
    u_sup0 = ac1_voltage(c->u_sup, c->supply_param[0], e->ac_phase, 0.0);
  }
  for (int j = 0; j < 6; ++j) u_abc[j] *= u_sup0;
  e->t = 0; e->k = 0;
  memset(e->fifo, 0, sizeof(e->fifo)); /* DeadTimeProcessor.reset dead_time_processor.py:68-78: queue of zero actions */
  double tq = torque(o, y + 1);
  int n = 0;
  state[n++] = y[0];
  state[n++] = tq;
  switch (mk) {
    case GEMB200_MOTOR_PERMEX_DC:
    case GEMB200_MOTOR_SERIES_DC: state[n++] = y[1]; state[n++] = u_abc[0]; break;
    case GEMB200_MOTOR_SHUNT_DC: state[n++] = y[1]; state[n++] = y[2]; state[n++] = u_abc[0]; break;
    case GEMB200_MOTOR_EXTEX_DC: state[n++] = y[1]; state[n++] = y[2]; state[n++] = u_abc[0]; state[n++] = u_abc[1]; break;
    case GEMB200_MOTOR_PMSM:
    case GEMB200_MOTOR_SYNRM: {
      double eps = y[3], u_dq[2], i_abc[3];
      if (eps > M_PI) eps -= 2 * M_PI;
      abc_to_dq(u_abc, eps, u_dq);
      dq_to_abc(y + 1, eps, i_abc);
      for (int j = 0; j < 3; ++j) state[n++] = i_abc[j];
      state[n++] = y[1]; state[n++] = y[2];
      for (int j = 0; j < 3; ++j) state[n++] = u_abc[j];
      state[n++] = u_dq[0]; state[n++] = u_dq[1];
      state[n++] = eps;
    } break;
    case GEMB200_MOTOR_EESM: { /* :659-693 — note the reference's slot shift: u_abc has 4 entries, u_dq 2 */
      double eps = y[4], u_dq[2], i_abc[3];
      if (eps > M_PI) eps -= 2 * M_PI;
      abc_to_dq(u_abc, eps, u_dq);
      dq_to_abc(y + 1, eps, i_abc);
      for (int j = 0; j < 3; ++j) state[n++] = i_abc[j];
      state[n++] = y[1]; state[n++] = y[2]; state[n++] = y[3];
      for (int j = 0; j < 4; ++j) state[n++] = u_abc[j];
      state[n++] = u_dq[0]; state[n++] = u_dq[1];
      state[n++] = eps;
    } break;
    case GEMB200_MOTOR_DFIM: { /* :1062-1113 */
      double eps = y[5], eps_fs = atan2(y[4], y[3]), u_sdq[2], u_rdq[2], i_sdq[2], i_sabc[3], i_r[2], i_rdq[2], i_rdef[3];
      if (eps > M_PI) eps -= 2 * M_PI;
      if (eps_fs > M_PI) eps_fs -= 2 * M_PI;
      abc_to_dq(u_abc, eps_fs, u_sdq);
      abc_to_dq(u_abc + 3, eps_fs - eps, u_rdq);
      q_rot(y + 1, -eps_fs, i_sdq);
      dq_to_abc(i_sdq, eps_fs, i_sabc);
      dfim_rotor_current(o, y, i_r);
      q_rot(i_r, -(eps_fs - eps), i_rdq); /* (sic) the reset uses eps_field - eps_el here, simulate uses eps_field */
      dq_to_abc(i_rdq, eps_fs - eps, i_rdef);
      for (int j = 0; j < 3; ++j) state[n++] = i_sabc[j];
      state[n++] = i_sdq[0]; state[n++] = i_sdq[1];
      for (int j = 0; j < 3; ++j) state[n++] = i_rdef[j];
      state[n++] = i_rdq[0]; state[n++] = i_rdq[1];
      for (int j = 0; j < 3; ++j) state[n++] = u_abc[j];
      state[n++] = u_sdq[0]; state[n++] = u_sdq[1];
      for (int j = 0; j < 3; ++j) state[n++] = u_abc[3 + j];
      state[n++] = u_rdq[0]; state[n++] = u_rdq[1];
      state[n++] = eps;
    } break;
    case GEMB200_MOTOR_SCIM: {
      double eps = y[5], eps_fs = atan2(y[4], y[3]), u_dq[2], i_dq[2], i_abc[3];
      if (eps > M_PI) eps -= 2 * M_PI;
      abc_to_dq(u_abc, eps_fs, u_dq);
      q_rot(y + 1, -eps_fs, i_dq);
      dq_to_abc(i_dq, eps_fs, i_abc);
      for (int j = 0; j < 3; ++j) state[n++] = i_abc[j];
      state[n++] = i_dq[0]; state[n++] = i_dq[1];
      for (int j = 0; j < 3; ++j) state[n++] = u_abc[j];
      state[n++] = u_dq[0]; state[n++] = u_dq[1];
      state[n++] = eps;
    } break;
  }
  state[n++] = u_sup0;
  for (int j = 0; j < n; ++j) state[j] = state[j] / c->limits[j];
  if (mk == GEMB200_MOTOR_SHUNT_DC) state[n] = state[2] + state[3]; /* current_sum_processor.py:47-50 */
}

/* ------------------------------------------------------------------------------------------------------------ */
/* state-vector wrappers, applied in list order to the (normalised) vector of the inner system                  */
/* ------------------------------------------------------------------------------------------------------------ */
static void apply_state_ops(const gem_oracle* o, env_t* e, int64_t idx, double* st, int is_reset, int after_autoreset) {
  const gemb200_config* c = &o->cfg;
  int w = o->n_state;
  for (int k = 0; k < c->n_state_ops; ++k) {
    const double* q = c->sop_param[k];
    switch (c->sop_kind[k]) {
      case GEMB200_SOP_COS_SIN: { /* cos_sin_processor.py:60-89 */
        const int a = c->sop_idx[k][0];
        const double cs = cos(st[a] * M_PI), sn = sin(st[a] * M_PI);
        if (c->sop_idx[k][1]) { for (int j = a; j < w - 1; ++j) st[j] = st[j + 1]; --w; } /* np.delete(state, angle) :68 */
        st[w++] = cs; st[w++] = sn;
      } break;
      case GEMB200_SOP_FLUX_OBSERVER: { /* flux_observer.py:81-101 */
        if (is_reset) { e->psi_re = 0.0; e->psi_im = 0.0; st[w++] = 0.0; st[w++] = 0.0; break; } /* :81-83 */
        double i_s[3], ab[2];
        for (int j = 0; j < 3; ++j) i_s[j] = st[c->sop_idx[k][j]] * q[4 + j]; /* state = state_norm * limits :87-88 */
        const double omega = st[c->sop_idx[k][3]] * q[7] * q[2];              /* :89 */
        t_23(i_s, ab);
        /* delta_psi = i_ab r_r l_m / l_r - psi * complex(r_r / l_r, -omega)  :93-95 */
        const double dre = ab[0] * q[0] - (e->psi_re * q[1] + e->psi_im * omega);
        const double dim = ab[1] * q[0] - (e->psi_im * q[1] - e->psi_re * omega);
        e->psi_re += dre * c->tau; e->psi_im += dim * c->tau;                  /* :97 */
        st[w++] = sqrt(e->psi_re * e->psi_re + e->psi_im * e->psi_im) / q[3];
        st[w++] = atan2(e->psi_im, e->psi_re) / M_PI;                          /* limits [psi_limit, pi] :69,:98 */
      } break;
      case GEMB200_SOP_CURRENT_SUM: { /* current_sum_processor.py:46-66: np.sum(state[self._current_indices]) on the normalised state */
        double sum = 0.0;
        for (int j = 0; j < w; ++j) if ((c->sop_mask[k] >> j) & 1u) sum += st[j];
        st[w++] = sum;
      } break;
      case GEMB200_SOP_NOISE: { /* state_noise_processor.py:74-98; one i.i.d. draw per step (Philox instead of numpy) */
        const uint32_t mask = c->sop_mask[k];
        for (int b = 0; b * 4 < w; ++b) {
          if (((mask >> (4 * b)) & 15u) == 0) continue;
          uint32_t r[4];
          rng4(o, idx, (after_autoreset ? STREAM_NOISE_R : STREAM_NOISE) + 8 * k + b, r);
          for (int m = 0; m < 4 && 4 * b + m < w; ++m) {
            if (!((mask >> (4 * b + m)) & 1u)) continue;
            double z;
            if (c->sop_idx[k][0] == GEMB200_NOISE_UNIFORM) z = q[0] + (q[1] - q[0]) * u01(r[m]);
            else if (c->sop_idx[k][0] == GEMB200_NOISE_LAPLACE) { /* sign from bit 0, magnitude -log(V), V ~ U(0,1) from the other 31 bits */
              const double v = u01(r[m] | 1u);
              z = q[0] + q[1] * ((r[m] & 1u) ? log(v) : -log(v));
            } else { /* Box-Muller on the word pair (0,1) / (2,3); even state: cos branch, odd: sin branch */
              const double rad = sqrt(-2.0 * log(u01(r[m & 2]))), ang = 2.0 * M_PI * u01(r[(m & 2) + 1]);
              z = q[0] + q[1] * rad * ((m & 1) ? sin(ang) : cos(ang));
            }
            st[4 * b + m] += z;
          }
        }
      } break;
    }
  }
}

/* ------------------------------------------------------------------------------------------------------------ */
/* epilogue: constraints, reward, reference generators                                                           */
/* ------------------------------------------------------------------------------------------------------------ */
/* ConstraintMonitor.check_constraints core.py:834-844 with merge 'max'; constraints.py:55-58, :96-98 */
static double check_constraints(const gem_oracle* o, const double* s) {
  double v = 0.0;
  for (int ci = 0; ci < o->cfg.n_constraints; ++ci) {
    uint32_t mask = o->cfg.constraint_mask[ci];
    double vi = 0.0;
    if (o->cfg.constraint_kind[ci] == GEMB200_CONSTRAINT_LIMIT) {
      for (int j = 0; j < o->n_obs; ++j) if ((mask >> j) & 1u) if (fabs(s[j]) > 1.0) vi = 1.0;
    } else {
      double sum = 0.0;
      for (int j = 0; j < o->n_obs; ++j) if ((mask >> j) & 1u) sum += s[j] * s[j];
      vi = sum > 1.0 ? 1.0 : 0.0;
    }
    if (vi > v) v = vi;
  }
  return v;
}

/* WeightedSumOfErrors.reward weighted_sum_of_errors.py:125-129 */
static double reward(const gem_oracle* o, const double* s, const double* ref_full, double violation) {
  double sum = 0.0;
  for (int j = 0; j < o->n_obs; ++j) {
    double w = o->cfg.reward_weight[j];
    if (w == 0.0) continue; /* 0 * x = 0 for the finite x met here */
    sum += w * pow(fabs(s[j] - ref_full[j]) / o->cfg.state_length[j], o->cfg.reward_power[j]);
  }
  double wse = -sum + o->cfg.reward_bias;
  return (1.0 - violation) * wse + violation * o->cfg.violation_reward;
}

/* SubepisodedReferenceGenerator.get_reference_observation :93-100 + WienerProcess._reset_reference :30-41, one value
 * per call instead of a pre-computed sub-episode (same distribution; RNG stream differs from numpy, see header) */
static void rng4_at(const gem_oracle* o, int64_t env, uint32_t kstart, uint32_t stream, uint32_t out[4]) {
  uint64_t g = (uint64_t)(env + o->cfg.env_index_offset);
  out[0] = kstart; out[1] = 0xA5A5A5A5u; out[2] = (uint32_t)g; out[3] = ((uint32_t)(g >> 32) << 8) | stream;
  philox4x32_10(out, (uint32_t)o->cfg.seed, (uint32_t)(o->cfg.seed >> 32));
}
static double frac1(double x) { return x - floor(x); }

/* Value k steps into a sub-episode of Sinusoidal/Step/Sawtooth/TriangularReferenceGenerator._reset_reference
 * (sinusoidal_reference_generator.py:44-62, step_reference_generator.py:47-76, sawtooth_reference_generator.py:47-64,
 * triangle_reference_generator.py:51-77), parameters from the Philox block of the sub-episode instead of numpy draws. */
static double periodic_value(const gem_oracle* o, int r, int kind, const uint32_t* b, const uint32_t* cw, uint32_t k, uint32_t len) {
  const gemb200_config* c = &o->cfg;
  double A = c->ref_amp_lo[r] + (c->ref_amp_hi[r] - c->ref_amp_lo[r]) * u01(b[1]);   /* _get_current_value(amplitude_range) */
  double f = c->ref_freq_lo[r] + (c->ref_freq_hi[r] - c->ref_freq_lo[r]) * u01(b[2]);
  double lo_c = (kind == GEMB200_REF_STEP ? c->ref_margin_lo[r] : -c->ref_margin_hi[r]) + A, hi_c = c->ref_margin_hi[r] - A;
  double olo = fmin(fmax(c->ref_off_lo[r], lo_c), hi_c), ohi = fmin(fmax(c->ref_off_hi[r], lo_c), hi_c); /* np.clip(offset_range, ., .) */
  double off = olo + (ohi - olo) * u01(b[3]);
  double ph = u01(cw[0]); /* phase / 2pi */
  double wave;
  if (kind == GEMB200_REF_STEP) {
    double u = u01(cw[1]);
    double ratio = u < 0.5 ? sqrt(0.5 * u) : 1.0 - sqrt(0.5 * (1.0 - u)); /* random_generator.triangular(0, 0.5, 1) */
    uint32_t shift = (uint32_t)((1.0 / (f * c->tau)) * ph);               /* int(steps_per_period * phase) */
    uint32_t kk = (k + len - shift % len) % len;                          /* np.roll over the sub-episode */
    double x = frac1(f * c->tau * (double)kk) - ratio;                    /* f * (t % (1/f)) - high_low_ratio */
    wave = x > 0 ? 1.0 : (x < 0 ? -1.0 : 0.0);
  } else {
    double t = frac1(f * c->tau * (double)k + ph);
    if (kind == GEMB200_REF_SINUS) wave = sin(2 * M_PI * t);
    else if (kind == GEMB200_REF_SAWTOOTH) wave = 2.0 * t - 1.0;             /* scipy.signal.sawtooth(x) */
    else { double w = u01(cw[1]); wave = t < w ? 2.0 * t / w - 1.0 : (w + 1.0 - 2.0 * t) / (1.0 - w); } /* sawtooth(x, width) */
  }
  double v = A * wave + off;
  if (v > c->ref_margin_hi[r]) v = c->ref_margin_hi[r];
  if (v < c->ref_margin_lo[r]) v = c->ref_margin_lo[r];
  return v;
}

/* SwitchedReferenceGenerator._reset_reference switched_reference_generator.py:96-101: super-episode length ~ integers(lo, hi),
 * generator ~ choice(sub_generators, p) */
static void switch_generator(const gem_oracle* o, env_t* e, int64_t idx, int r, int at_reset) {
  const gemb200_config* c = &o->cfg;
  uint32_t w[4];
  rng4(o, idx, (at_reset ? STREAM_SWITCH_R : STREAM_SWITCH) + r, w);
  e->sw_len[r] = c->ref_sw_len_lo[r] + (int)(((uint64_t)w[0] * (uint64_t)(uint32_t)(c->ref_sw_len_hi[r] - c->ref_sw_len_lo[r])) >> 32);
  const double u = u01(w[1]);
  int g = c->ref_sw_first[r];
  for (int m = 1; m < c->ref_sw_count[r]; ++m) if (u >= c->ref_sw_cdf[c->ref_sw_first[r] + m - 1]) g = c->ref_sw_first[r] + m;
  e->sw_cur[r] = g;
  e->sw_k[r] = 0;
}

/* one step of the clipped random walk, wiener_process_reference_generator.py:35-40 (laplace_process_reference_generator.py:29-36 alike) */
static double walk_next(const gemb200_config* c, int g, double value, double increment) {
  double v = value + increment;
  if (v > c->ref_margin_hi[g]) v = c->ref_margin_hi[g];
  if (v < c->ref_margin_lo[g]) v = c->ref_margin_lo[g];
  return v;
}

static void ref_advance(const gem_oracle* o, env_t* e, int64_t idx, int after_reset) {
  const gemb200_config* c = &o->cfg;
  uint32_t rw[4], rs[4], rs2[4], rlap[4];
  int have_w = 0, have_s = 0, have_s2 = 0, have_lap = 0;
  uint32_t kstep = (uint32_t)o->n_steps;
  for (int r = 0; r < c->n_ref; ++r) {
    int g = r; /* parameter entry: r itself, or the sub-generator a SwitchedReferenceGenerator currently uses */
    if (c->ref_sw_count[r] > 1) { /* switched_reference_generator.py:80-94 */
      if (!after_reset && e->sw_k[r] >= e->sw_len[r]) {
        switch_generator(o, e, idx, r, 0);
        e->ref_left[r] = 0; /* sub.reset(state, self._reference): value kept (:73-76 of the subepisoded class), new sub-episode */
        if (c->ref_kind[e->sw_cur[r]] == GEMB200_REF_CONST) e->ref_value[r] = c->ref_value[e->sw_cur[r]];
      }
      g = e->sw_cur[r];
      if (!after_reset) e->sw_k[r] += 1;
    }
    int kind = c->ref_kind[g];
    if (kind >= GEMB200_REF_SINUS) {
      uint32_t b[4], cw[4];
      if (e->ref_left[r] <= 0) { /* new sub-episode (subepisoded_reference_generator.py:93-100) */
        e->ref_start[r] = kstep;
        rng4_at(o, idx, kstep, STREAM_PERIODIC + 2 * r, b);
        e->ref_len[r] = (uint32_t)((double)(c->ref_len_hi[g] - c->ref_len_lo[g]) * ((double)b[0] / 4294967296.0) + c->ref_len_lo[g]);
        e->ref_left[r] = (int)e->ref_len[r];
      } else {
        rng4_at(o, idx, e->ref_start[r], STREAM_PERIODIC + 2 * r, b);
      }
      rng4_at(o, idx, e->ref_start[r], STREAM_PERIODIC + 2 * r + 1, cw);
      e->ref_value[r] = periodic_value(o, g, kind, b, cw, kstep - e->ref_start[r], e->ref_len[r]);
      e->ref_left[r] -= 1;
      continue;
    }
    if (kind != GEMB200_REF_WIENER && kind != GEMB200_REF_LAPLACE) continue;
    if (e->ref_left[r] <= 0) {
      /* two uniforms per slot: slots 0,1 share one Philox block, slots 2,3 a second one */
      uint32_t a, b;
      if (r < 2) {
        if (!have_s) { rng4(o, idx, after_reset ? STREAM_SUBEP_R : STREAM_SUBEP, rs); have_s = 1; }
        a = rs[2 * (r & 1)]; b = rs[2 * (r & 1) + 1];
      } else {
        if (!have_s2) { rng4(o, idx, after_reset ? STREAM_SUBEP_HI_R : STREAM_SUBEP_HI, rs2); have_s2 = 1; }
        a = rs2[2 * (r & 1)]; b = rs2[2 * (r & 1) + 1];
      }
      /* int(U[0,1)*(hi-lo) + lo) subepisoded_reference_generator.py:37,:115-119 with U = a / 2^32 */
      e->ref_left[r] = (int)((double)(c->ref_len_hi[g] - c->ref_len_lo[g]) * ((double)a / 4294967296.0) + c->ref_len_lo[g]);
      double l0 = log10(c->ref_sigma_lo[g]), l1 = log10(c->ref_sigma_hi[g]);
      e->ref_sigma[r] = pow(10.0, (l1 - l0) * u01(b) + l0); /* wiener_process_reference_generator.py:31 */
    }
    double z;
    if (kind == GEMB200_REF_LAPLACE) { /* random_generator.laplace(0, sigma): inverse CDF, laplace_process_reference_generator.py:25-28 */
      if (!have_lap) { rng4(o, idx, after_reset ? STREAM_LAPLACE_R : STREAM_LAPLACE, rlap); have_lap = 1; }
      double u = u01(rlap[r]);
      z = u < 0.5 ? log(2.0 * u) : -log(2.0 * (1.0 - u));
    } else {
      if (!have_w) {
        if (o->n_ref <= 2 && !after_reset) { /* the device serves two consecutive steps from one Philox block (gemb200_kernels.cuh: WalkCache) */
          uint32_t blk[4];
          const uint64_t g = (uint64_t)(idx + c->env_index_offset), id = o->gstep >> 1;
          blk[0] = (uint32_t)id; blk[1] = (uint32_t)(id >> 32); blk[2] = (uint32_t)g; blk[3] = ((uint32_t)(g >> 32) << 8) | STREAM_WALK2;
          philox4x32_10(blk, (uint32_t)c->seed, (uint32_t)(c->seed >> 32));
          const int odd = (int)(o->gstep & 1);
          rw[0] = blk[2 * odd]; rw[1] = blk[2 * odd + 1]; rw[2] = 0; rw[3] = 0;
        } else {
          rng4(o, idx, after_reset ? STREAM_WALK_R : STREAM_WALK, rw);
        }
        have_w = 1;
      }
      /* Box-Muller: slots (0,1) from words (0,1), slots (2,3) from words (2,3) */
      double u1 = u01(rw[2 * (r >> 1)]), u2 = u01(rw[2 * (r >> 1) + 1]);
      double rad = sqrt(-2.0 * log(u1));
      z = (r & 1) ? rad * sin(2 * M_PI * u2) : rad * cos(2 * M_PI * u2);
      /* <= 2 slots: words 2, 3 of the after-reset walk block are the slots' initial values (gemb200_kernels.cuh: init_from_walk) */
      if (o->n_ref <= 2 && after_reset) e->ref_value[r] = c->ref_init_lo[g] + (c->ref_init_hi[g] - c->ref_init_lo[g]) * u01(rw[2 + r]);
    }
    e->ref_value[r] = walk_next(c, g, e->ref_value[r], e->ref_sigma[r] * z);
    e->ref_left[r] -= 1;
  }
}

/* ReferenceGenerator.reset: WienerProcessReferenceGenerator.reset :43-49 + Subepisoded.reset :71-91 */
static void ref_reset(const gem_oracle* o, env_t* e, int64_t idx) {
  const gemb200_config* c = &o->cfg;
  uint32_t ri[4];
  rng4(o, idx, STREAM_INIT, ri);
  for (int r = 0; r < c->n_ref; ++r) {
    int g = r;
    if (c->ref_sw_count[r] > 1) { switch_generator(o, e, idx, r, 1); g = e->sw_cur[r]; } /* switched_reference_generator.py:64-68 */
    if (c->ref_kind[g] == GEMB200_REF_WIENER) {
      /* with <= 2 slots the value comes from the after-reset walk block instead (set in ref_advance) */
      e->ref_value[r] = o->n_ref <= 2 ? 0.0 : c->ref_init_lo[g] + (c->ref_init_hi[g] - c->ref_init_lo[g]) * u01(ri[r]);
      e->ref_left[r] = 0; /* _current_episode_length = -1 forces a new sub-episode */
      e->ref_sigma[r] = 0;
    } else if (c->ref_kind[g] >= GEMB200_REF_LAPLACE) { /* SubepisodedReferenceGenerator.reset :71-91: value 0, new sub-episode */
      e->ref_value[r] = 0.0; e->ref_left[r] = 0; e->ref_sigma[r] = 0;
    } else {
      e->ref_value[r] = c->ref_value[g]; e->ref_left[r] = 0;
    }
  }
  ref_advance(o, e, idx, 1); /* reset() returns get_reference_observation() :82-91 via core.py:499-503 */
}

/* ------------------------------------------------------------------------------------------------------------ */
/* public API (loaded by tests/bench via ctypes)                                                                 */
/* ------------------------------------------------------------------------------------------------------------ */
void gem_oracle_reset(gem_oracle* o, const uint8_t* mask, double* obs, double* ref_next);
int gem_oracle_create(const gemb200_config* cfg, gem_oracle** out) {
  if (!cfg || cfg->struct_size != (int32_t)sizeof(gemb200_config)) return -4;
  gem_oracle* o = (gem_oracle*)calloc(1, sizeof(gem_oracle));
  o->cfg = *cfg;
  if (dims(o)) { free(o); return -1; }
  update_model(o);
  o->env = (env_t*)calloc((size_t)cfg->n_envs, sizeof(env_t));
  gem_oracle_reset(o, NULL, NULL, NULL); /* like gemb200_create: every env starts reset; API call id 1 */
  *out = o;
  return 0;
}
void gem_oracle_destroy(gem_oracle* o) { if (o) { free(o->env); free(o); } }
void gem_oracle_dims(const gem_oracle* o, int32_t* n_state, int32_t* n_ode, int32_t* n_act, int32_t* n_ref) {
  *n_state = o->n_obs; *n_ode = o->n_ode; *n_act = o->n_act; *n_ref = o->n_ref;
}

/* env.reset (core.py:300-319). mask NULL = all. obs [N][n_state], ref_next [N][n_ref] (may be NULL). */
void gem_oracle_reset(gem_oracle* o, const uint8_t* mask, double* obs, double* ref_next) {
  double st[GEMB200_MAX_STATE];
  o->gstep += 1;
  for (int64_t i = 0; i < o->cfg.n_envs; ++i) {
    if (mask && !mask[i]) continue;
    env_t* e = o->env + i;
    ps_reset(o, e, st);
    apply_state_ops(o, e, i, st, 1, 0);
    ref_reset(o, e, i);
    if (obs) memcpy(obs + i * o->n_obs, st, sizeof(double) * o->n_obs);
    if (ref_next) for (int r = 0; r < o->n_ref; ++r) ref_next[i * o->n_ref + r] = e->ref_value[r];
  }
}

/* physical-system wrappers on the ACTION side (core.py:266-267): DeadTimeProcessor and DqToAbcActionProcessor in either order.
 * In: the caller's action of env e (af or ai); out: the action the inner SCMLSystem sees (pointers redirected to abuf / ibuf). */
static void wrap_action(gem_oracle* o, env_t* e, const double** af_io, const int32_t** ai_io, double* abuf, int32_t* ibuf) {
  const double* af = *af_io;
  const int32_t* ai = *ai_io;
  for (int j = 0; j < GEMB200_MAX_ACT; ++j) abuf[j] = 0.0;
  ibuf[0] = ibuf[1] = 0;
  const gemb200_config* c = &o->cfg;
  const int slot = c->dead_time_steps > 0 ? (int)((o->n_steps - 1) % (uint64_t)c->dead_time_steps) : 0;
  if (c->finite) {
    for (int j = 0; j < o->n_act; ++j) ibuf[j] = ai[j];
    if (c->dead_time_steps > 0) /* dead_time_processor.py:80-90: apply the oldest action, store the new one */
      for (int j = 0; j < o->n_act; ++j) { int32_t old = (int32_t)e->fifo[slot][j]; e->fifo[slot][j] = ibuf[j]; ibuf[j] = old; }
    *ai_io = ibuf;
  } else {
    int na = o->n_act;
    for (int j = 0; j < na; ++j) abuf[j] = af[j];
    if (c->dead_time_steps > 0 && c->dead_time_outer)
      for (int j = 0; j < na; ++j) { double old = e->fifo[slot][j]; e->fifo[slot][j] = abuf[j]; abuf[j] = old; }
    if (c->action_dq == 3) { /* _DFIMDqToAbcActionProcessor.simulate :119-131 */
      const double adv = wrap_eps(e->ode[o->n_ode - 1]) + c->angle_advance * c->tau * e->ode[0] * c->motor_param[GEMB200_MP_P];
      const double psi_angle = atan2(e->psi_im, e->psi_re);
      double dqs[2] = {abuf[0], abuf[1]}, dqr[2] = {abuf[2], abuf[3]}, ab[2];
      q_rot(dqs, adv, ab); t_32(ab, abuf);
      q_rot(dqr, psi_angle - adv, ab); t_32(ab, abuf + 3);
      na = 6;
    } else if (c->action_dq) {
      /* _ClassicDqToAbcActionProcessor.simulate :100-106 / _EESM :147-153; angle from the last state vector:
       * wrapped epsilon + angle_advance * tau * omega * p (:89-91).  control_space='dq' = same with advance 0
       * (physical_systems.py:491-492); SCIM uses the field angle (:779-780). */
      double ang, dq[2] = {abuf[0], abuf[1]}, ab[2], ue = abuf[2];
      if (c->motor_kind == GEMB200_MOTOR_SCIM && c->action_dq == 2) /* observer angle: dq_to_abc_action_processor.py:89-91,:103-105 */
        ang = atan2(e->psi_im, e->psi_re) + c->angle_advance * c->tau * e->ode[0] * c->motor_param[GEMB200_MP_P];
      else if (c->motor_kind == GEMB200_MOTOR_SCIM) ang = atan2(e->ode[4], e->ode[3]);
      else ang = wrap_eps(e->ode[o->n_ode - 1]) + c->angle_advance * c->tau * e->ode[0] * c->motor_param[GEMB200_MP_P];
      q_rot(dq, ang, ab);
      t_32(ab, abuf);
      na = 3;
      if (c->motor_kind == GEMB200_MOTOR_EESM) { abuf[3] = ue; na = 4; }
    }
    if (c->dead_time_steps > 0 && !c->dead_time_outer)
      for (int j = 0; j < na; ++j) { double old = e->fifo[slot][j]; e->fifo[slot][j] = abuf[j]; abuf[j] = old; }
    *af_io = abuf;
  }
}

static void step_one(gem_oracle* o, int64_t i, const void* action, double* obs, double* ref_next, double* rew, uint8_t* term) {
  env_t* e = o->env + i;
  double st[GEMB200_MAX_STATE], ref_full[GEMB200_MAX_STATE];
  const double* af = o->cfg.finite ? NULL : (const double*)action + i * o->n_act;
  const int32_t* ai = o->cfg.finite ? (const int32_t*)action + i * o->n_act : NULL;
  double abuf[GEMB200_MAX_ACT];
  int32_t ibuf[2];
  wrap_action(o, e, &af, &ai, abuf, ibuf);
  simulate(o, e, af, ai, st);                                   /* core.py:344 */
  apply_state_ops(o, e, i, st, 0, 0);                           /* wrappers' simulate() */
  memset(ref_full, 0, sizeof(ref_full));
  for (int r = 0; r < o->n_ref; ++r) ref_full[o->cfg.ref_state[r]] = e->ref_value[r]; /* core.py:346 */
  double v = check_constraints(o, st);                          /* core.py:348 */
  double rw = reward(o, st, ref_full, v);                        /* core.py:349 */
  int terminated = v >= 1.0;                                    /* core.py:350 */
  ref_advance(o, e, i, 0);                                      /* core.py:351 */
  if (terminated && o->cfg.autoreset == GEMB200_AUTORESET_SAME_STEP) {
    ps_reset(o, e, st);
    apply_state_ops(o, e, i, st, 1, 1);
    ref_reset(o, e, i);
  }
  if (obs) memcpy(obs + i * o->n_obs, st, sizeof(double) * o->n_obs);
  if (ref_next) for (int r = 0; r < o->n_ref; ++r) ref_next[i * o->n_ref + r] = e->ref_value[r];
  if (rew) rew[i] = rw;
  if (term) term[i] = (uint8_t)terminated;
}

/* env.step for all envs (core.py:328-371); action: double [N][n_act] or int32 [N][n_slots].
 * nthreads > 1 splits the env range over POSIX threads (envs are independent; the reference itself is
 * single-threaded — process/thread replication is its best case, SURVEY.md §8d). */
typedef struct { gem_oracle* o; const void* action; double* obs; double* ref; double* rew; uint8_t* term; int64_t lo, hi; } job_t;
static void* step_range(void* arg) {
  job_t* j = (job_t*)arg;
  for (int64_t i = j->lo; i < j->hi; ++i) step_one(j->o, i, j->action, j->obs, j->ref, j->rew, j->term);
  return NULL;
}
void gem_oracle_step(gem_oracle* o, const void* action, double* obs, double* ref_next, double* rew, uint8_t* term, int nthreads) {
  int64_t n = o->cfg.n_envs;
  o->gstep += 1;
  o->n_steps += 1;
  if (nthreads > n) nthreads = (int)n;
  if (nthreads <= 1) {
    job_t j = {o, action, obs, ref_next, rew, term, 0, n};
    step_range(&j);
    return;
  }
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * nthreads);
  job_t* jobs = (job_t*)malloc(sizeof(job_t) * nthreads);
  for (int t = 0; t < nthreads; ++t) {
    jobs[t] = (job_t){o, action, obs, ref_next, rew, term, n * t / nthreads, n * (t + 1) / nthreads};
    pthread_create(&th[t], NULL, step_range, &jobs[t]);
  }
  for (int t = 0; t < nthreads; ++t) pthread_join(th[t], NULL);
  free(th); free(jobs);
}

/* K consecutive env.step calls with a pool of `n_sets` prepared action arrays used round-robin (set k % n_sets for step k; each set
 * is [N][n_act] doubles or [N][n_slots] int32, `set_stride_bytes` apart).  Same arithmetic and counters as K calls of gem_oracle_step;
 * the difference is purely mechanical: the worker threads live for the whole rollout and meet at two barriers per step instead of
 * being created and joined every step — what a CPU user with many cores would do, and what bench.py's CPU arm times.  Outputs hold
 * the last step's values. */
typedef struct { gem_oracle* o; const char* actions; size_t stride; int n_sets, K, tid; double* obs; double* ref; double* rew; uint8_t* term;
                 int64_t lo, hi; pthread_barrier_t* bar; } roll_t;
static void* roll_worker(void* arg) {
  roll_t* j = (roll_t*)arg;
  for (int k = 0; k < j->K; ++k) {
    if (j->tid == 0) { j->o->gstep += 1; j->o->n_steps += 1; }
    if (j->bar) pthread_barrier_wait(j->bar); /* the counters of step k are visible to every worker */
    const void* act = j->actions + (size_t)(k % j->n_sets) * j->stride;
    for (int64_t i = j->lo; i < j->hi; ++i) step_one(j->o, i, act, j->obs, j->ref, j->rew, j->term);
    if (j->bar) pthread_barrier_wait(j->bar); /* nobody is still inside step k when the counters move on */
  }
  return NULL;
}
void gem_oracle_rollout(gem_oracle* o, const void* actions, int64_t set_stride_bytes, int n_sets, int n_steps, double* obs, double* ref_next,
                        double* rew, uint8_t* term, int nthreads) {
  int64_t n = o->cfg.n_envs;
  if (nthreads > n) nthreads = (int)n;
  if (nthreads < 1) nthreads = 1;
  if (n_sets < 1 || n_steps < 1) return;
  pthread_barrier_t bar;
  if (nthreads > 1) pthread_barrier_init(&bar, NULL, (unsigned)nthreads);
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * nthreads);
  roll_t* jobs = (roll_t*)malloc(sizeof(roll_t) * nthreads);
  for (int t = 0; t < nthreads; ++t)
    jobs[t] = (roll_t){o, (const char*)actions, (size_t)set_stride_bytes, n_sets, n_steps, t, obs, ref_next, rew, term,
                       n * t / nthreads, n * (t + 1) / nthreads, nthreads > 1 ? &bar : NULL};
  for (int t = 1; t < nthreads; ++t) pthread_create(&th[t], NULL, roll_worker, &jobs[t]);
  roll_worker(&jobs[0]);
  for (int t = 1; t < nthreads; ++t) pthread_join(th[t], NULL);
  if (nthreads > 1) pthread_barrier_destroy(&bar);
  free(th); free(jobs);
}

/* Jump the handle's clock: call_id = id of the last API call (the next reset / step draws with call_id + 1), n_steps = step calls so far
 * (dead-time ring position, periodic sub-episode keys).  The device's equivalent is a checkpoint with a patched header; env state,
 * sub-episodes and dead-time queues are left as they are, so a test resets after the jump. */
void gem_oracle_set_clock(gem_oracle* o, uint64_t call_id, uint64_t n_steps) { o->gstep = call_id; o->n_steps = n_steps; }
void gem_oracle_get_clock(const gem_oracle* o, uint64_t* call_id, uint64_t* n_steps) { *call_id = o->gstep; *n_steps = o->n_steps; }
/* exact = 0: the reference's time grid (default); 1: the device's, step k of an episode over [k tau, (k + 1) tau] with its segment lengths
 * precomputed (fixed-step solvers) and the AC supply evaluated at k tau (DESIGN §2 finding 12) */
void gem_oracle_set_time_grid(gem_oracle* o, int exact) { o->exact_grid = exact != 0; }

void gem_oracle_get_ode_state(const gem_oracle* o, double* out) {
  for (int64_t i = 0; i < o->cfg.n_envs; ++i) memcpy(out + i * o->n_ode, o->env[i].ode, sizeof(double) * o->n_ode);
}
void gem_oracle_set_ode_state(gem_oracle* o, const double* in) {
  for (int64_t i = 0; i < o->cfg.n_envs; ++i) memcpy(o->env[i].ode, in + i * o->n_ode, sizeof(double) * o->n_ode);
}
void gem_oracle_get_reference(const gem_oracle* o, double* out) {
  for (int64_t i = 0; i < o->cfg.n_envs; ++i) for (int r = 0; r < o->n_ref; ++r) out[i * o->n_ref + r] = o->env[i].ref_value[r];
}
void gem_oracle_set_reference(gem_oracle* o, const double* in) {
  for (int64_t i = 0; i < o->cfg.n_envs; ++i) for (int r = 0; r < o->n_ref; ++r) o->env[i].ref_value[r] = in[i * o->n_ref + r];
}
/* sub-episode bookkeeping, exposed so that the device generator can be compared slot by slot */
void gem_oracle_get_ref_aux(const gem_oracle* o, double* sigma, int32_t* left) {
  for (int64_t i = 0; i < o->cfg.n_envs; ++i) for (int r = 0; r < o->n_ref; ++r) { sigma[i * o->n_ref + r] = o->env[i].ref_sigma[r]; left[i * o->n_ref + r] = o->env[i].ref_left[r]; }
}
/* whole sub-episode of a periodic generator from raw Philox words (pinned against numpy/scipy formulas of the reference in
 * tests/test_oracle_golden.py); params_out = [A, f, offset, phase/2pi, width-or-ratio uniform] */
void gem_oracle_periodic_block(const gem_oracle* o, int r, int kind, const uint32_t* b, const uint32_t* cw, uint32_t len, double* values, double* params_out) {
  const gemb200_config* c = &o->cfg;
  double A = c->ref_amp_lo[r] + (c->ref_amp_hi[r] - c->ref_amp_lo[r]) * u01(b[1]);
  double f = c->ref_freq_lo[r] + (c->ref_freq_hi[r] - c->ref_freq_lo[r]) * u01(b[2]);
  double lo_c = (kind == GEMB200_REF_STEP ? c->ref_margin_lo[r] : -c->ref_margin_hi[r]) + A, hi_c = c->ref_margin_hi[r] - A;
  double olo = fmin(fmax(c->ref_off_lo[r], lo_c), hi_c), ohi = fmin(fmax(c->ref_off_hi[r], lo_c), hi_c);
  params_out[0] = A; params_out[1] = f; params_out[2] = olo + (ohi - olo) * u01(b[3]); params_out[3] = u01(cw[0]); params_out[4] = u01(cw[1]);
  for (uint32_t k = 0; k < len; ++k) values[k] = periodic_value(o, r, kind, b, cw, k, len);
}
/* exposed for the known-answer tests of the reference's converter tables / solver vectors */
void gem_oracle_philox(uint32_t ctr[4], uint32_t k0, uint32_t k1) { philox4x32_10(ctr, k0, k1); }

/* ------------------------------------------------------------------------------------------------------------ */
/* probe entry points for tests/test_oracle_known_answers.py: the reference's unit tests call converters, loads,  */
/* constraints and the reward function directly, so the same granularity is exposed here (on env 0)               */
/* ------------------------------------------------------------------------------------------------------------ */
int gem_oracle_probe_set_action(gem_oracle* o, const double* act_f, const int32_t* act_i, double t) { double seg_end[3]; return conv_set_action(o, o->env, act_f, act_i, t, seg_end); }
void gem_oracle_probe_convert(gem_oracle* o, const double* i_out, double t, double* u_out) { conv_convert(o, o->env, i_out, t, u_out); }
void gem_oracle_probe_conv_reset(gem_oracle* o, double* u_out) { conv_reset(o, o->env, u_out); }
double gem_oracle_probe_i_sup(gem_oracle* o, const double* i_out) { return conv_i_sup(o, o->env, i_out); }
double gem_oracle_probe_mechanical_ode(gem_oracle* o, double omega, double tq) { return mechanical_ode(o, omega, tq, 0.0); }
/* ExternalSpeedLoad: g = speed_profile(t + tau_load), one entry of the host-tabulated profile */
double gem_oracle_probe_mechanical_ode_ext(gem_oracle* o, double omega, double tq, double g) { return mechanical_ode(o, omega, tq, g); }
double gem_oracle_probe_rc_supply_rhs(double u_sup, double u_0, double i_sup, double r, double cap) { return rc_supply_rhs(u_sup, u_0, i_sup, r, cap); }
double gem_oracle_probe_ac1_voltage(double u_nominal, double f, double phi, double t) { return ac1_voltage(u_nominal, f, phi, t); }
/* the Wiener / Laplace walk of parameter entry g from `start` with the given (already scaled) increments */
void gem_oracle_probe_walk(const gem_oracle* o, int g, double start, const double* increments, int n, double* out) {
  double v = start;
  for (int k = 0; k < n; ++k) { v = walk_next(&o->cfg, g, v, increments[k]); out[k] = v; }
}
/* the action-side wrappers of env 0 (dead-time FIFO, dq -> abc) exactly as step_one runs them, counted as one more step call; returns the
 * number of values written: the action the inner system would see */
int gem_oracle_probe_wrap_action(gem_oracle* o, const double* act_f, const int32_t* act_i, double* out_f, int32_t* out_i) {
  double abuf[GEMB200_MAX_ACT];
  int32_t ibuf[2];
  const double* af = o->cfg.finite ? NULL : act_f;
  const int32_t* ai = o->cfg.finite ? act_i : NULL;
  o->n_steps += 1;
  wrap_action(o, o->env, &af, &ai, abuf, ibuf);
  if (o->cfg.finite) { for (int j = 0; j < o->n_act; ++j) out_i[j] = ai[j]; return o->n_act; }
  const int na = o->cfg.action_dq == 3 ? 6 : (o->cfg.action_dq ? (o->cfg.motor_kind == GEMB200_MOTOR_EESM ? 4 : 3) : o->n_act);
  for (int j = 0; j < na; ++j) out_f[j] = af[j];
  return na;
}
double gem_oracle_probe_constraints(gem_oracle* o, const double* s) { return check_constraints(o, s); }
double gem_oracle_probe_reward(gem_oracle* o, const double* s, const double* ref_full, double violation) { return reward(o, s, ref_full, violation); }
/* EulerSolver known answers (tests/test_physical_systems/test_solvers.py:248-269): the stepping scheme above on the reference's test
 * system tests/conf.py:418-434 */
static void conf_system(const void* ctx, const double* st, const double* u, double* dy, double g) {
  (void)ctx; (void)g;
  const double x = st[0], y = st[1];
  dy[0] = 3 * x + 5 * y - 2 * x * y + 3 * x * x - 0.5 * y * y;
  dy[1] = 10 - 0.6 * x + 0.9 * y * y - 3 * x * x * y + u[0];
}
void gem_oracle_probe_euler(int nsteps, const double* y0, double dt, double u, double* out) {
  double y[GEMB200_MAX_ODE] = {y0[0], y0[1]};
  euler_core(conf_system, NULL, 2, y, dt, nsteps, &u, NULL);
  out[0] = y[0]; out[1] = y[1];
}

