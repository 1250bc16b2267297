/*
 * gemb200.h — C-ABI of the H100-native (sm_90a) vectorised GEM physical-system step.
 *
 * One handle = N independent motor environments of ONE (motor, converter, load, solver) combination living on
 * one CUDA device.  The library owns only the persistent per-env state (ODE state, converter switching state,
 * reference-generator state); the caller owns every I/O buffer.  All device-pointer entry points are
 * stream-ordered and asynchronous (no host synchronisation inside); the *_host entry points take plain host
 * pointers, do the H2D/D2H copies themselves and return after the results are in the host buffers.
 * Every function returns 0 on success or a negative GEMB200_E_* code and never throws; the message for the last
 * failure on the calling thread is available from gemb200_last_error().  A handle is not thread-safe; different
 * handles may be used from different threads.
 *
 * The reference (upb-lea/gym-electric-motor, pure Python) has no FFI: each entry point below replaces a Python
 * method of its plugin API and cites it (paths relative to the reference's src/gym_electric_motor/).
 * INTEGRATION.md shows the ctypes stub a reference maintainer would add.
 */
#ifndef GEMB200_H_
#define GEMB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GEMB200_ABI_VERSION 10

/* limits of the POD config */
#define GEMB200_MAX_STATE 28   /* longest state vector in scope: DFIM 24 (+ wrappers) */
#define GEMB200_MAX_ODE 8      /* SCIM: omega + 4 + eps = 6 */
#define GEMB200_MAX_ACT 6      /* DFIM: two B6 bridges; EESM: 3 (B6) + 1 (4QC) */
#define GEMB200_MAX_REF 4          /* referenced states = output slots of the reference generator */
#define GEMB200_MAX_REF_ENTRIES 12 /* generator parameter entries: the slots + the extra sub-generators of SwitchedReferenceGenerators */
#define GEMB200_MAX_DEAD_TIME 8
#define GEMB200_MAX_CONSTRAINTS 4
#define GEMB200_MAX_MOTOR_PARAM 16
#define GEMB200_MAX_STATE_OPS 4 /* state-vector wrappers stacked on one system */

/* error codes */
#define GEMB200_OK 0
#define GEMB200_E_INVALID -1    /* bad argument / unsupported combination (reference: assert / Exception) */
#define GEMB200_E_CUDA -2       /* CUDA runtime error, see gemb200_last_error() */
#define GEMB200_E_NOMEM -3
#define GEMB200_E_ABI -4        /* struct_size / abi_version mismatch */

/* motor kinds — reference physical_systems/electric_motors/<file>.py */
enum gemb200_motor_kind {
  GEMB200_MOTOR_PERMEX_DC = 0, /* dc_permanently_excited_motor.py:67-92   params: r_a l_a psi_e j_rotor */
  GEMB200_MOTOR_SERIES_DC = 1, /* dc_series_motor.py                      params: r_a r_e l_a l_e l_e_prime j_rotor */
  GEMB200_MOTOR_SHUNT_DC = 2,  /* dc_shunt_motor.py                       params: r_a r_e l_a l_e l_e_prime j_rotor */
  GEMB200_MOTOR_EXTEX_DC = 3,  /* dc_externally_excited_motor.py, dc_motor.py */
  GEMB200_MOTOR_PMSM = 4,      /* permanent_magnet_synchronous_motor.py:107-139 params: p l_d l_q r_s psi_p j_rotor */
  GEMB200_MOTOR_SYNRM = 5,     /* synchronous_reluctance_motor.py:117-139      params: p l_d l_q r_s j_rotor */
  GEMB200_MOTOR_EESM = 6,      /* externally_excited_synchronous_motor.py:125-203 params: p l_d l_q l_m l_e r_s r_e k j_rotor */
  GEMB200_MOTOR_SCIM = 7,      /* induction_motor.py:187-310, squirrel_cage_induction_motor.py:121-129
                                  params: p l_m l_sigs l_sigr r_s r_r j_rotor */
  GEMB200_MOTOR_DFIM = 8       /* doubly_fed_induction_motor.py + physical_systems.py:850-1113: the induction model with the rotor fed
                                  by a second B6 bridge (converter slot 1); same parameters as SCIM */
};

/* motor_param[] slots (physical parameters exactly as in the reference's motor_parameter dicts) */
enum gemb200_motor_param {
  GEMB200_MP_P = 0, GEMB200_MP_R_S = 1, GEMB200_MP_L_D = 2, GEMB200_MP_L_Q = 3, GEMB200_MP_PSI_P = 4,
  GEMB200_MP_J_ROTOR = 5,
  GEMB200_MP_R_A = 6, GEMB200_MP_L_A = 7, GEMB200_MP_PSI_E = 8, GEMB200_MP_R_E = 9, GEMB200_MP_L_E = 10,
  GEMB200_MP_L_E_PRIME = 11,
  GEMB200_MP_L_M = 12, GEMB200_MP_K = 13, GEMB200_MP_L_SIGS = 14, GEMB200_MP_L_SIGR = 15
  /* SCIM's r_r is passed in GEMB200_MP_R_E */
};

/* converter slots — reference physical_systems/converters.py.  A converter is 1 or 2 slots:
 * DC motors: slot0 in {1QC,2QC,4QC}; ExtEx: slot0 (armature) + slot1 (excitation);
 * PMSM/SynRM/SCIM: slot0 = B6; EESM: slot0 = B6, slot1 in {1QC,2QC,4QC}; DFIM: slot0 = B6 (stator), slot1 = B6 (rotor)
 * (Cont/FiniteMultiConverter :498-740). */
enum gemb200_converter_kind {
  GEMB200_CONV_NONE = 0,
  GEMB200_CONV_1QC = 1, /* :218-245 finite, :371-401 continuous */
  GEMB200_CONV_2QC = 2, /* :248-310 finite, :404-435 continuous */
  GEMB200_CONV_4QC = 3, /* :313-368 finite, :438-495 continuous */
  GEMB200_CONV_B6 = 4   /* :743-839 finite, :842-911 continuous */
};

enum gemb200_load_kind {
  GEMB200_LOAD_CONST_SPEED = 0, /* mechanical_loads/constant_speed_load.py:40-42 */
  GEMB200_LOAD_POLY_STATIC = 1, /* mechanical_loads/polynomial_static_load.py:87-99 */
  GEMB200_LOAD_EXT_SPEED = 2    /* mechanical_loads/external_speed_load.py:62-68: d omega/dt = (f(t + tau_load) - omega) / tau_load with the
                                   user's speed profile f TABULATED on the host: ext_speed_table[j] = f(j * tau / (2 * solver_nsteps) + tau_load),
                                   i.e. at every time a fixed-step Euler / RK4 stage can fall on; load_param[GEMB200_LP_TAU_LOAD] = tau_load;
                                   t restarts at every reset; beyond the table the last step repeats */
};
enum gemb200_load_param { GEMB200_LP_A = 0, GEMB200_LP_B = 1, GEMB200_LP_C = 2, GEMB200_LP_J_LOAD = 3, GEMB200_LP_TAU_DECAY = 4, GEMB200_LP_TAU_LOAD = 5 };

enum gemb200_supply_kind {
  GEMB200_SUPPLY_IDEAL = 0, /* voltage_supplies.py:60-72: u_sup = u_nominal */
  GEMB200_SUPPLY_RC = 1,    /* voltage_supplies.py:75-123: DC link behind an RC element, u_sup' = (u_0 - u_sup - R i_sup) / (R C), advanced once
                               per step with explicit Euler from the supply current of the converter (converters.py i_sup);
                               supply_param = {R, C} */
  GEMB200_SUPPLY_AC1 = 2    /* voltage_supplies.py:126-166: u_sup(t) = sqrt(2) u_nominal sin(2 pi f t + phi), t = time since the reset;
                               supply_param = {f [Hz], phi [rad], fixed}: fixed = 0 draws phi ~ U[0, 2 pi) per env at every reset (the
                               reference uses the unseeded global numpy RNG here, the device its Philox stream) */
};

enum gemb200_solver_kind {
  GEMB200_SOLVER_EULER = 0, /* physical_systems/solvers.py:79-136 (incl. the n-step time quirk :113-119) */
  GEMB200_SOLVER_RK4 = 1    /* classic RK4, solver_nsteps equal sub-steps per switching segment (reference has none;
                               within 1e-6 of its default dopri5, SURVEY.md §7) */
};

enum gemb200_constraint_kind {
  GEMB200_CONSTRAINT_LIMIT = 0,  /* constraints.py:55-58  any(|s_i| > 1) over the masked states */
  GEMB200_CONSTRAINT_SQUARED = 1 /* constraints.py:96-98  sum(s_i^2) > 1 over the masked states */
};

enum gemb200_ref_kind {
  GEMB200_REF_CONST = 0,   /* reference_generators/const_reference_generator.py */
  GEMB200_REF_WIENER = 1,  /* reference_generators/wiener_process_reference_generator.py:7-49 on
                              subepisoded_reference_generator.py:9-119 */
  GEMB200_REF_EXTERNAL = 2, /* value injected with gemb200_set_reference() before each step (oracle injection hook,
                               user-side generators) */
  GEMB200_REF_LAPLACE = 3,    /* reference_generators/laplace_process_reference_generator.py */
  GEMB200_REF_SINUS = 4,      /* sinusoidal_reference_generator.py */
  GEMB200_REF_STEP = 5,       /* step_reference_generator.py */
  GEMB200_REF_SAWTOOTH = 6,   /* sawtooth_reference_generator.py */
  GEMB200_REF_TRIANGULAR = 7  /* triangle_reference_generator.py */
};

/* State-vector wrappers of the reference (physical_system_wrappers/*.py) that run in the kernel after the system's own state
 * vector has been assembled, in list order (each one sees the vector produced by the previous ones).  n_state reported by
 * gemb200_query_dims, limits[], constraint masks, reward weights and ref_state[] all refer to the FINAL vector. */
enum gemb200_state_op {
  GEMB200_SOP_NONE = 0,
  GEMB200_SOP_COS_SIN = 1,       /* cos_sin_processor.py: append cos(pi*s[angle]), sin(pi*s[angle]); optionally drop the angle.
                                    sop_idx = {angle index, remove_angle} */
  GEMB200_SOP_FLUX_OBSERVER = 2, /* flux_observer.py:85-101 (induction motor): rotor-flux estimate integrated with explicit Euler,
                                    appends |psi|/psi_limit and angle(psi)/pi.  sop_idx = {i_sa, i_sb, i_sc, omega} indices,
                                    sop_param = {r_r*l_m/l_r, r_r/l_r, p, psi_limit, limit of i_sa, i_sb, i_sc, omega} */
  GEMB200_SOP_CURRENT_SUM = 4,   /* current_sum_processor.py:7-66: append i_sum = sum of the (normalised) states in sop_mask */
  GEMB200_SOP_NOISE = 3          /* state_noise_processor.py: s[j] += noise for the states in sop_mask, i.i.d. per step and env.
                                    sop_idx[0] = gemb200_noise_dist, sop_param = {loc, scale} (normal, laplace) or {low, high} */
};
enum gemb200_noise_dist { GEMB200_NOISE_NORMAL = 0, GEMB200_NOISE_UNIFORM = 1, GEMB200_NOISE_LAPLACE = 2 };

enum gemb200_dtype { GEMB200_F32 = 0 /* fp32 state; rotor angle as a double-float (two fp32, ~48 bits) in turns */, GEMB200_F64 = 1 };
enum gemb200_layout {
  GEMB200_LAYOUT_AOS = 0, /* obs[N][n_state], action[N][n_act], ref[N][n_ref]  (row per env, the gym layout) */
  GEMB200_LAYOUT_SOA = 1  /* obs[n_state][N], action[n_act][N], ref[n_ref][N]  (field-major, fully coalesced) */
};
enum gemb200_autoreset {
  GEMB200_AUTORESET_NONE = 0,     /* caller resets terminated envs with gemb200_reset(mask) (reference core.py:341) */
  GEMB200_AUTORESET_SAME_STEP = 1 /* a terminated env is reset inside the same launch; obs/ref returned are the
                                     first observation of the new episode, reward/terminated those of the old one */
};

typedef struct gemb200_config {
  int32_t struct_size; /* = sizeof(gemb200_config), set by gemb200_config_init */
  int32_t abi_version; /* = GEMB200_ABI_VERSION */
  int32_t n_envs;
  int32_t device;      /* CUDA device ordinal */
  int32_t dtype;       /* gemb200_dtype */
  int32_t layout;      /* gemb200_layout */
  int32_t autoreset;   /* gemb200_autoreset */
  int32_t finite;      /* 0: continuous converters, float actions; 1: finite converters, int32 actions [N][n_slots] */

  /* SCML components (reference physical_systems.py:54 SCMLSystem.__init__) */
  int32_t motor_kind;
  int32_t converter_kind[2];
  int32_t load_kind;
  int32_t solver_kind;
  int32_t solver_nsteps;
  double tau;                /* physical_systems.py:54; converter.tau :103 */
  double interlocking_time;  /* converters.py:37-44 */
  double u_sup;              /* IdealVoltageSupply.u_nominal voltage_supplies.py:60-72 */
  double motor_param[GEMB200_MAX_MOTOR_PARAM];
  double load_param[8];      /* a b c j_load tau_decay ; for CONST_SPEED nothing is read (omega lives in init_ode) */
  double limits[GEMB200_MAX_STATE];   /* SCMLSystem.limits physical_systems.py:105-112 (host-derived) */
  double init_ode[GEMB200_MAX_ODE];   /* constant initial ODE state [omega, motor states...] used by reset */

  /* constraint monitor (core.py:756-844) */
  int32_t n_constraints;
  int32_t constraint_kind[GEMB200_MAX_CONSTRAINTS];
  uint32_t constraint_mask[GEMB200_MAX_CONSTRAINTS]; /* bit i = state i observed */

  /* WeightedSumOfErrors (reward_functions/weighted_sum_of_errors.py:88-129), already resolved per state */
  double reward_weight[GEMB200_MAX_STATE];
  double reward_power[GEMB200_MAX_STATE];
  double state_length[GEMB200_MAX_STATE]; /* state_space.high - low */
  double reward_bias;
  double violation_reward;

  /* reference generators: one slot per referenced state (MultipleReferenceGenerator = several slots) */
  int32_t n_ref;
  int32_t ref_kind[GEMB200_MAX_REF_ENTRIES];
  int32_t ref_state[GEMB200_MAX_REF_ENTRIES];       /* index into the state vector */
  double ref_value[GEMB200_MAX_REF_ENTRIES];        /* CONST: the value; others: value after reset when no random init */
  double ref_margin_lo[GEMB200_MAX_REF_ENTRIES], ref_margin_hi[GEMB200_MAX_REF_ENTRIES];   /* clip range of the walk */
  double ref_init_lo[GEMB200_MAX_REF_ENTRIES], ref_init_hi[GEMB200_MAX_REF_ENTRIES];       /* U() range of the value at reset */
  double ref_sigma_lo[GEMB200_MAX_REF_ENTRIES], ref_sigma_hi[GEMB200_MAX_REF_ENTRIES];     /* log-uniform sigma range */
  int32_t ref_len_lo[GEMB200_MAX_REF_ENTRIES], ref_len_hi[GEMB200_MAX_REF_ENTRIES];        /* sub-episode length U(lo,hi) */

  uint64_t seed;            /* Philox key; streams are keyed by (seed, global env index) */
  int64_t env_index_offset; /* global index of env 0 of this handle (rank*N_local when sharded) */

  /* Action pre-processing of the three-phase systems (continuous converters only):
   * action_dq = 1: the action is given in dq coordinates (2 values, EESM: + u_e) and transformed in the kernel with
   *   a_abc = T32 * q(a_dq, eps + angle_advance * tau * omega * p)
   * angle_advance = 0   : SynchronousMotorSystem(control_space='dq') physical_systems.py:423-435,:491-492 (SCIM: field angle :779-780)
   * angle_advance = 0.5 (+ dead-time steps): physical_system_wrappers/dq_to_abc_action_processor.py:74-95 */
  int32_t action_dq;
  int32_t dead_time_steps;  /* DeadTimeProcessor(steps) physical_system_wrappers/dead_time_processor.py: action FIFO, 0 = off */
  int32_t dead_time_outer;  /* 1: the dead-time FIFO holds the caller's (dq) actions, 0: the transformed (abc) ones */
  int32_t init_random;      /* 0: constant initial state init_ode[]; 1: uniform in [init_lo, init_hi] per ODE state at every reset
                               (ElectricMotor.initialize / MechanicalLoad.initialize with random_init='uniform',
                               electric_motor.py:179-268, mechanical_load.py:100-167) */
  double angle_advance;
  double init_lo[GEMB200_MAX_ODE], init_hi[GEMB200_MAX_ODE]; /* ODE order [omega, motor states...]; lo == hi keeps a state constant */

  /* periodic reference generators (SINUS/STEP/SAWTOOTH/TRIANGULAR): per sub-episode amplitude ~ U(amp), frequency ~ U(freq) [Hz],
   * offset ~ U(clip(off, -margin_hi + A | margin_lo + A (STEP), margin_hi - A)); ranges already clipped to the limit margin
   * as in the generators' set_modules() */
  double ref_amp_lo[GEMB200_MAX_REF_ENTRIES], ref_amp_hi[GEMB200_MAX_REF_ENTRIES];
  double ref_freq_lo[GEMB200_MAX_REF_ENTRIES], ref_freq_hi[GEMB200_MAX_REF_ENTRIES];
  double ref_off_lo[GEMB200_MAX_REF_ENTRIES], ref_off_hi[GEMB200_MAX_REF_ENTRIES];

  /* state-vector wrappers (see gemb200_state_op).  limits[] above stays the INNER system's limits (they normalise the assembled
   * vector); the ops carry their own scaling in sop_param. */
  int32_t n_state_ops;
  int32_t sop_kind[GEMB200_MAX_STATE_OPS];
  int32_t sop_idx[GEMB200_MAX_STATE_OPS][4];
  uint32_t sop_mask[GEMB200_MAX_STATE_OPS];
  double sop_param[GEMB200_MAX_STATE_OPS][8];
  /* random_init = 'normal' / 'gaussian' (electric_motor.py:245-258, mechanical_load.py:138-150): truncated normal on [init_lo, init_hi]
   * per state; init_dist[j] = 0 uniform (lo == hi: constant), 1 truncated normal with init_mu[j], init_sigma[j]; needs init_random = 1 */
  int32_t init_dist[GEMB200_MAX_ODE];
  double init_mu[GEMB200_MAX_ODE], init_sigma[GEMB200_MAX_ODE];
  /* SwitchedReferenceGenerator (reference_generators/switched_reference_generator.py): output slot r (r < n_ref) switches between
   * ref_sw_count[r] generators (0 or 1: not switched) whose parameters occupy the entries ref_sw_first[r] .. +count-1 of the per-slot
   * arrays above; entries >= n_ref are parameter-only entries, so n_ref + extra entries <= GEMB200_MAX_REF_ENTRIES.  ref_sw_cdf[entry] is the
   * cumulative probability inside its group; the super-episode length is integers(ref_sw_len_lo[r], ref_sw_len_hi[r]). */
  int32_t ref_sw_count[GEMB200_MAX_REF], ref_sw_first[GEMB200_MAX_REF], ref_sw_len_lo[GEMB200_MAX_REF], ref_sw_len_hi[GEMB200_MAX_REF];
  double ref_sw_cdf[GEMB200_MAX_REF_ENTRIES];
  const double* ext_speed_table; /* HOST pointer, copied at gemb200_create (GEMB200_LOAD_EXT_SPEED only) */
  int32_t ext_speed_len;
  int32_t supply_kind;      /* gemb200_supply_kind; u_sup above is u_nominal (= u_0 of the RC supply) */
  double supply_param[4];
  /* Induction motors (SCIM / DFIM) with init_random: the bounds of the two rotor-flux states are re-derived per env at EVERY reset from a
   * random magnetic-field angle eps_mag ~ U(-pi, pi), the speed and the initial currents of the env's previous episode
   * (squirrel_cage_induction_motor.py:146-157, doubly_fed_induction_motor.py:154-165, induction_motor.py:250-285):
   *   omega == 0: psi_d_max = init_im[0]                                   (l_m * nominal i_sd)
   *   else      : (i_d, i_q) = q_inv(previous initial (i_salpha, i_sbeta), eps_mag),
   *               psi_d_max = 0.9 * clip((init_im[1]*omega*i_d + init_im[2]*i_q + init_im[3]) / (-init_im[4]*omega), 0, |init_im[5]*i_d|)
   *   bounds    : +-|psi_d_max * (cos, sin)(eps_mag)|, clipped to init_lo / init_hi of the flux states (the user's `interval`, else +-1e30)
   * init_im = {l_m*i_sd_nominal, p*sigma*l_s, r_s + r_r*(l_m/l_r)^2, u_sq_nominal (+ l_m/l_r * u_rq_nominal, DFIM), p*l_m/l_r, l_m, 0, 0}.
   * The reference draws eps_mag from the UNSEEDED global numpy RNG; here it comes from the env's Philox stream like every other draw.
   * A truncated-normal state (init_dist) whose init_mu is NaN takes the middle of its (per-env) interval as mue (electric_motor.py:247). */
  int32_t init_im_valid;
  double init_im[8];
  /* interlocking time of converter slot 1 when a multi converter's sub-converters differ (converters.py:615-740); < 0: same as slot 0
   * (interlocking_time above).  Finite converters with two different times integrate a switching step in up to three segments. */
  double interlocking_time1;
  /* action_dq = 3: DFIM, 4 actions (stator dq, rotor dq): stator with eps + angle_advance*tau*omega*p, rotor with the FluxObserver's
   * psi_angle minus that angle (dq_to_abc_action_processor.py:108-137); requires a GEMB200_SOP_FLUX_OBSERVER op */
  /* action_dq = 2: SCIM with a FluxObserver — the transformation angle is the observer's psi_angle (+ angle_advance*tau*omega*p),
   * dq_to_abc_action_processor.py:103-105; requires a GEMB200_SOP_FLUX_OBSERVER op */
} gemb200_config;

typedef struct gemb200_handle gemb200_handle;

/* library / error reporting */
int gemb200_version(void);
const char* gemb200_last_error(void);

/* Fill *cfg with zeros + struct_size/abi_version + neutral defaults (nsteps=1, tau_decay=1e-3, …). */
int gemb200_config_init(gemb200_config* cfg);

/* Derived sizes of a configuration (no GPU needed): n_state, n_ode, n_act (floats or ints per env), n_ref.
 * Replaces the index bookkeeping of SCMLSystem._set_indices (physical_systems.py:141-162, :462-485). */
int gemb200_query_dims(const gemb200_config* cfg, int32_t* n_state, int32_t* n_ode, int32_t* n_act, int32_t* n_ref);

/* SCMLSystem.__init__ (physical_systems.py:54-103) + ElectricMotorEnvironment.__init__ wiring (core.py:197-289):
 * validates the combination, derives the model constants from the physical parameters (the *_update_model
 * methods), allocates the per-env state on cfg->device and resets every env. */
int gemb200_create(const gemb200_config* cfg, gemb200_handle** out);
int gemb200_destroy(gemb200_handle* h);

/* ElectricMotorEnvironment.reset (core.py:300-319) -> SCMLSystem.reset (physical_systems.py:256-287, :527-561,
 * :659-693, :816-847) + ReferenceGenerator.reset.  reset_mask: device uint8[N] (non-zero = reset) or NULL for all.
 * obs_out/ref_out (device, layout per cfg, element type per cfg->dtype) may be NULL. */
int gemb200_reset(gemb200_handle* h, const uint8_t* reset_mask, void* obs_out, void* ref_out, void* stream);

/* ElectricMotorEnvironment.step (core.py:328-371): SCMLSystem.simulate (physical_systems.py:171-203, :487-525,
 * :619-657, :771-814) + get_reference + check_constraints + reward + get_reference_observation, one launch for all
 * N envs.  action: float/double [N][n_act] (continuous) or int32 [N][n_slots] (finite).  Outputs: obs [N][n_state],
 * ref_next [N][n_ref], reward [N], terminated uint8 [N]; any output pointer may be NULL. */
int gemb200_step(gemb200_handle* h, const void* action, void* obs_out, void* ref_out, void* reward_out,
                 uint8_t* terminated_out, void* stream);

/* Same call with HOST buffers (pageable or pinned): H2D of the actions, the launch, D2H of the results and a stream
 * synchronise all happen inside.  This is the drop-in for a host-side caller of env.step. */
int gemb200_step_host(gemb200_handle* h, const void* action, void* obs_out, void* ref_out, void* reward_out,
                      uint8_t* terminated_out);
int gemb200_reset_host(gemb200_handle* h, const uint8_t* reset_mask, void* obs_out, void* ref_out);

/* K consecutive env.step calls (core.py:328-371 called K times, open loop) fused into ONE launch: actions[K][N][n_act] resident on
 * the device; every env's persistent record stays in registers for all K steps (loaded once, stored once), the clock, the RNG call
 * ids and the dead-time ring advance exactly as K separate gemb200_step calls would, so results are bit-identical to them.
 * gemb200_rollout returns the outputs of the LAST step ([N][..] tensors).  gemb200_rollout_record additionally streams the outputs
 * of steps m, 2m, ... (m = record_every >= 1) into [K / m][N][..] tensors (m = 1: the full trajectory); record_every = 0 is
 * gemb200_rollout.  Any output pointer may be NULL. */
int gemb200_rollout(gemb200_handle* h, const void* actions, int32_t n_steps, void* obs_out, void* ref_out,
                    void* reward_out, uint8_t* terminated_out, void* stream);
int gemb200_rollout_record(gemb200_handle* h, const void* actions, int32_t n_steps, int32_t record_every, void* obs_out, void* ref_out,
                           void* reward_out, uint8_t* terminated_out, void* stream);

/* gemb200_rollout_record with a per-step reference feed: references[K][N][n_ref] (cfg->layout SoA: [K][n_ref][N]) in the handle's dtype,
 * resident on the device.  Before step k, row k overwrites the stored value of EVERY reference slot, not only the External ones: the call
 * gives exactly the outputs, final state and clock of K iterations of gemb200_set_reference(row k) + gemb200_step.  So the ref output of
 * step k is what that sequence gives: for an External slot the value step k was scored against (the reset value on an env that was
 * auto-reset in step k).  Stream-ordered, no host synchronisation; capturable in a CUDA graph under the device clock.  references ==
 * NULL: exactly gemb200_rollout_record.  A feed into a configuration without reference slots (n_ref == 0) is GEMB200_E_INVALID. */
int gemb200_rollout_record_ref(gemb200_handle* h, const void* actions, const void* references, int32_t n_steps, int32_t record_every,
                               void* obs_out, void* ref_out, void* reward_out, uint8_t* terminated_out, void* stream);

/* Discounted returns of a fused rollout: n_steps >= 1 steps in ONE launch, scored in registers.  Per env i, with gamma = discount rounded
 * to the handle's dtype:
 *   end_step_out[i] (int32, [N]) = the 0-based index of the env's first step with terminated = 1, or n_steps if there is none;
 *   return_out[i] ([N], the handle's dtype) = sum of gamma^k * reward_k over k = 0 .. min(end_step, n_steps - 1): the terminating step's
 *   reward counts, nothing after it does, whatever the auto-reset mode does to the env afterwards.  Computed as w = 1, G = 0; per step
 *   G = G + (w * r_k) while not yet terminated, then w = w * gamma; two roundings per update, no FMA.
 * obs_out / ref_out take the LAST step's outputs as gemb200_rollout_record(record_every = 0) writes them.  The final state, clock and
 * RNG position are exactly those of gemb200_rollout_record_ref with the same arguments.  references: the reference feed of
 * gemb200_rollout_record_ref, or NULL.  end_step_out, obs_out, ref_out may be NULL; return_out may not.  The returns and end steps go to the
 * caller's buffers only: bound peers (gemb200_bind_peers) do not gather them.  Stream-ordered, capturable in a
 * CUDA graph under the device clock.  GEMB200_E_INVALID: NULL handle or return_out, n_steps out of [1, 2^24], a discount that is not a
 * finite number in [0, 1], a feed into a configuration with n_ref == 0. */
int gemb200_rollout_returns(gemb200_handle* h, const void* actions, const void* references, int32_t n_steps, double discount,
                            void* return_out, int32_t* end_step_out, void* obs_out, void* ref_out, void* stream);

/* The linearised plant along a fused rollout (SCMLSystem._system_jacobian, physical_systems.py:238, integrated over each step).
 * gemb200_query_jacobian_dims: n_x = n_ode (the state of gemb200_get_ode_state: [load states | motor states], the angle last, in radians)
 * and n_u = n_act (0 for finite converters: their actions are integers).  Needs no GPU.  GEMB200_E_INVALID for every configuration the
 * launch refuses (DESIGN.md §7): a dead time, the RC supply, dq actions on the FluxObserver angle (action_dq = 2, 3), the SoA layout.
 * gemb200_rollout_jacobians: n_steps >= 1 open-loop steps in ONE launch.  Per step k and env i
 *   jac_x_out[k][i] = d x_{k+1} / d x_k  ([n_x][n_x], row-major),   jac_u_out[k][i] = d x_{k+1} / d a_k  ([n_x][n_u]),
 * a = the caller's action as passed to gemb200_step; both in the handle's dtype, [K][N][n_x][..].  At non-smooth points the derivative is
 * the one-sided one of the branch the step took (clipped duty cycle: 0; interlocking and current-sign voltages: 0; angle wrap: 1).  A
 * terminating step reports the Jacobian of the physical step it took; terminated_out tells which rows precede an auto-reset.
 * obs_out / ref_out / reward_out / terminated_out receive exactly what gemb200_rollout_record_ref(record_every = 1) writes, and the final
 * state, clock and RNG position are those of that call.  references: its reference feed, or NULL.  Any output may be NULL except
 * jac_x_out; jac_u_out is ignored when n_u == 0.  The Jacobians go to the caller's buffers only: bound peers do not gather them.
 * Stream-ordered, capturable in a CUDA graph under the device clock. */
int gemb200_query_jacobian_dims(const gemb200_config* cfg, int32_t* n_x, int32_t* n_u);
int gemb200_rollout_jacobians(gemb200_handle* h, const void* actions, const void* references, int32_t n_steps, void* jac_x_out, void* jac_u_out,
                              void* obs_out, void* ref_out, void* reward_out, uint8_t* terminated_out, void* stream);

/* Gradients of rollout returns (continuous converters).  gemb200_query_return_grad_dims (needs no GPU): n_x = n_ode and n_u = n_act as for
 * the Jacobians, ws_words = n_x (n_x + n_u) + n_x + n_u; refuses everything gemb200_query_jacobian_dims refuses, finite converters, and a
 * reward that weights an entry a state wrapper appends (GEMB200_E_INVALID, DESIGN.md §7).
 * gemb200_rollout_return_grads: n_steps = K open-loop steps in ONE launch.  return_out [N], end_step_out [N] (may be NULL), obs_out and
 * ref_out (may be NULL) are exactly what gemb200_rollout_returns(actions, references, K, discount) writes, and the final state, clock and
 * RNG position are those of that call.  Per env i with e = end_step[i]:
 *   grad_a_out [K][N][n_u] = d return[i] / d a_k[i] (the caller's action, dq under action_dq = 1), 0 for k >= e;
 *   grad_x0_out [N][n_x]   = d return[i] / d x_0[i] (x as gemb200_get_ode_state: the angle last, in radians), 0 when e == 0.
 * value_grad [N][n_x] (or NULL) adds gamma^K value_grad[i] to the adjoint of every env with e == K (return_out is unchanged).  Non-smooth
 * points take the one-sided derivative of the branch the step took, and termination has derivative 0.  workspace: the caller's work buffer of at
 * least K * N * ws_words * sizeof(real) bytes (one linearised step per env and step); the call allocates nothing.  All buffers are device
 * memory in the handle's dtype, row-per-env.  Stream-ordered, capturable in a CUDA graph under the device clock. */
int gemb200_query_return_grad_dims(const gemb200_config* cfg, int32_t* n_x, int32_t* n_u, int32_t* ws_words);
int gemb200_rollout_return_grads(gemb200_handle* h, const void* actions, const void* references, int32_t n_steps, double discount, const void* value_grad,
                                 void* workspace, uint64_t workspace_bytes, void* return_out, int32_t* end_step_out, void* grad_a_out, void* grad_x0_out,
                                 void* obs_out, void* ref_out, void* stream);

/* Parameter sensitivities along a fused rollout: d x_k / d theta of the physical parameters theta, forward mode.  slots[0 .. n_p - 1]: the
 * parameters, in the slot numbers of a parameter row (GEMB200_MP_* for the motor, GEMB200_MAX_MOTOR_PARAM + GEMB200_LP_* for the load).
 * Accepted: every motor slot but GEMB200_MP_P (the angle increments are per handle) and GEMB200_MP_K (the EESM's coefficients are invariant
 * in it), and the load slots A, B, C, J_LOAD; 1 <= n_p <= 12, no slot twice.  A slot that does not enter the configuration's model has
 * sensitivity 0.  Limits, the normalisation and the FluxObserver constants are held fixed.
 * gemb200_query_param_sens_dims (needs no GPU): n_x = n_ode as for the Jacobians; GEMB200_E_INVALID for everything
 * gemb200_query_jacobian_dims refuses and for a refused slot list (DESIGN.md §7).
 * gemb200_coef_tangents (needs no GPU): out[a][30] = d (coefficient block) / d theta_a at the parameter row (motor_param[16], load_param[8];
 * NULL: the configuration's), in the word order of the per-env coefficient block: c[20], tq[4], load a, b, c, inv_j, omega_lim, omega_lin
 * — the derivation the launch runs on the device.
 * gemb200_rollout_param_sens: n_steps = K open-loop steps in ONE launch; each env is differentiated with respect to its own parameters (its
 * per-env block, or the configuration's).  sens_io [N][n_x][n_p]: S_0 on entry (zeros: the trajectory from the current state), S_K on
 * return, so that launches chain.  sens_out [K][N][n_x][n_p] (or NULL): S_{k+1} = d x_{k+1} / d theta after every step k.  x as
 * gemb200_get_ode_state (the angle last, in radians).  Non-smooth points as for the Jacobians.  A terminating step reports the sensitivity
 * of the physical step it took; under autoreset same_step the carried S of a reset env then restarts from 0.  obs_out / ref_out / reward_out
 * / terminated_out, the final state, clock and RNG position are exactly those of gemb200_rollout_record_ref(record_every = 1).  Refused
 * while parameter draws at resets are on.  All buffers are device memory in the handle's dtype; the call allocates nothing.
 * Stream-ordered, capturable in a CUDA graph under the device clock. */
int gemb200_query_param_sens_dims(const gemb200_config* cfg, int32_t n_p, const int32_t* slots, int32_t* n_x);
int gemb200_coef_tangents(const gemb200_config* cfg, const double* motor_param, const double* load_param, int32_t n_p, const int32_t* slots, double* out);
int gemb200_rollout_param_sens(gemb200_handle* h, const void* actions, const void* references, int32_t n_steps, int32_t n_p, const int32_t* slots,
                               void* sens_io, void* sens_out, void* obs_out, void* ref_out, void* reward_out, uint8_t* terminated_out, void* stream);

/* OdeSolver.y / set_initial_value (physical_systems/solvers.py:4-76): ODE state as double [N][n_ode]
 * (AoS, device), angle unwrapped to (-pi, pi].  Used for checkpointing and oracle injection. */
int gemb200_get_ode_state(gemb200_handle* h, double* ode_out, void* stream);
int gemb200_set_ode_state(gemb200_handle* h, const double* ode_in, void* stream);

/* Reference-generator value that the NEXT step's reward is computed against (ReferenceGenerator.get_reference,
 * core.py:439-452): double [N][n_ref] (device). */
int gemb200_get_reference(gemb200_handle* h, double* ref_out, void* stream);
int gemb200_set_reference(gemb200_handle* h, const double* ref_in, void* stream);

/* ElectricMotorEnvironment.reset(seed=...) -> _seed(seed) (core.py:300-319): re-key the handle's RNG streams with `seed` and start every
 * counter and persistent array over, then reset all envs — afterwards the handle is indistinguishable from a freshly created one with
 * cfg.seed = seed, so equal seeds give identical episodes.  Stream-ordered. */
int gemb200_reseed(gemb200_handle* h, uint64_t seed, void* stream);

/* Device-resident clock — CUDA-graph support for the closed loop (core.py:328-371 called once per control step with a policy in between;
 * SURVEY.md §8f row 4).  By default every launch carries its clock (RNG call id, step count = sub-episode clock, dead-time ring position)
 * in the kernel parameters, taken from the handle's host counters, so no two launches are alike and a captured launch cannot be replayed.
 * While the device clock is enabled, gemb200_step / gemb200_rollout(_record) / gemb200_reset read the clock from device memory instead and
 * enqueue a one-thread kernel behind the launch that advances it: a launch then depends on nothing the host changes between calls, and
 * { policy, gemb200_step } x K can be captured ONCE (cudaStreamBeginCapture / torch.cuda.graph) and replayed any number of times — the
 * results are bit-identical to the same sequence of ordinary calls.  The host counters are stale while it is on; gemb200_get_clock,
 * gemb200_checkpoint_save and switching it off read the clock back (synchronising `stream`).  gemb200_step_host's chunked pipeline is not
 * available in this mode.  enable: 1 = on (uploads the current clock, stream-ordered), 0 = off. */
int gemb200_set_device_clock(gemb200_handle* h, int32_t enable, void* stream);
/* Number of API calls that drew random numbers (RNG call id) and of env steps so far; synchronises `stream` when the device clock is on. */
int gemb200_get_clock(gemb200_handle* h, uint64_t* call_id, uint64_t* n_steps, void* stream);

/* Per-env parameter blocks (domain randomisation; SURVEY.md §8f row 4 — the batched counterpart of constructing N reference envs with N
 * different motor_parameter / load_parameter dicts): env i takes its motor constants from motor_param[i][GEMB200_MAX_MOTOR_PARAM] and its load
 * polynomial / inertia from load_param[i][8] (HOST arrays, same slot enums as gemb200_config; either may be NULL = keep the configuration's
 * values).  The model coefficients are derived per env on the host exactly like the shared ones and live in a [30][N] device table that
 * every thread reads instead of the constant bank (36 B per PMSM env and launch; a fused rollout reads them once per K steps).  Limits,
 * nominal values, reward, constraints and references stay those of the configuration.  Both NULL: back to shared coefficients.
 * Every motor row must keep the configuration's pole pairs (GEMB200_MP_P), else GEMB200_E_INVALID: the angle increments and the dq advance
 * are prepared on the host per handle.  The flux limits of an induction motor with random initial states (init_im) and the FluxObserver
 * constants (sop_param) stay the handle's as well.
 * Takes effect from the next reset / step; synchronises the device. */
int gemb200_set_env_params(gemb200_handle* h, const double* motor_param, const double* load_param);

/* Per-episode domain randomisation: from this call on, EVERY reset of an env (gemb200_reset, the in-kernel auto-reset of step and rollout,
 * and therefore captured graphs) draws new values for n parameters from the env's own Philox stream, keyed by (seed, global env index,
 * call id, stream), so equal seeds give equal parameter sequences independent of sharding.  slot[j]: GEMB200_MP_* for the motor,
 * GEMB200_MAX_MOTOR_PARAM + GEMB200_LP_* for the load; kind[j]: GEMB200_DIST_*; bounds lo[j] <= hi[j], finite, lo > 0 for log-uniform.
 * A drawn value is rounded to the handle's dtype and stored; the env's coefficients are derived on the device from the stored values by
 * the same code gemb200_set_env_params runs on the host, and the new episode (its reset observation included) uses them.  Parameters that
 * are not drawn keep their per-env or shared value.  The call draws nothing itself: each env keeps its dynamics until its next reset.
 * Without per-env blocks the call first fills them from the shared parameters, on the device.  n = 0: no more draws (the envs keep their
 * last values); gemb200_set_env_params(h, NULL, NULL) returns to the shared coefficients and also ends the draws.
 * Refused (GEMB200_E_INVALID): pole pairs (host-prepared angle increments), the flux-limit parameters l_m, l_sigs, l_sigr, r_s, r_r of an
 * induction motor with random initial states (host-prepared init_im), the field-major (SoA) I/O layout, repeated or unknown slots and bad
 * bounds.  While draws are on, gemb200_checkpoint_save / _load and gemb200_pack_envs / _unpack_envs return GEMB200_E_INVALID: the drawn
 * parameters are per-episode state that neither format carries (gemb200_pack_envs_params / _unpack_envs_params below carry them with the
 * state rows).  Synchronises the device. */
enum gemb200_dist_kind { GEMB200_DIST_UNIFORM = 0, GEMB200_DIST_LOG_UNIFORM = 1 };
int gemb200_set_param_randomization(gemb200_handle* h, int32_t n, const int32_t* slot, const int32_t* kind, const double* lo, const double* hi);
/* Stream-ordered copy of the stored values of the drawn parameters into the device buffer out[n][n_envs] (handle dtype; order of the slots
 * given to gemb200_set_param_randomization).  GEMB200_E_INVALID while no parameters are drawn. */
int gemb200_get_env_params(gemb200_handle* h, void* out, void* stream);

/* Fused aggregated return of the sharded layout (one process per GPU, SURVEY.md §8e: the ONE collective of the north star, done by the
 * step kernel itself instead of a separate NCCL all-gather).  Every rank owns a gather buffer (gemb200_peer_buffer_alloc: cudaMalloc +
 * IPC handle) of world sections; the ranks exchange the 64-byte handles out of band and map each other's buffers
 * (gemb200_peer_buffer_open: cudaIpcOpenMemHandle with the consumer's device current, peer access enabled lazily).  After
 * gemb200_bind_peers(h, world, delta) every step launch stores obs / ref / reward / terminated not only into the caller's tensors (which
 * must be this rank's section of its OWN buffer) but also at the same byte offset + delta[d] — i.e. into this rank's section of every
 * destination d — over NVLink, and fences the stores at system scope.  gemb200_peer_signal (flag store after the step, stream-ordered)
 * and gemb200_peer_wait (polls local flags; gives up after ~2 s and reports through *err_dev instead of hanging) are the flag protocol
 * that replaces the collective's synchronisation.  n_dst = 0 unbinds.  Row-per-env (AoS) layout only. */
int gemb200_peer_buffer_alloc(int32_t device, int64_t bytes, void** dev_ptr, void* ipc_handle64);
int gemb200_peer_buffer_open(int32_t device, const void* ipc_handle64, void** dev_ptr);
int gemb200_peer_buffer_close(int32_t device, void* dev_ptr);
int gemb200_peer_buffer_free(int32_t device, void* dev_ptr);
int gemb200_bind_peers(gemb200_handle* h, int32_t n_dst, const int64_t* dst_delta);
int gemb200_peer_signal(gemb200_handle* h, int32_t n_dst, uint32_t* const* flag_ptrs_dev, uint32_t value, void* stream);
int gemb200_peer_wait(gemb200_handle* h, int32_t n_src, const uint32_t* flags_dev, uint32_t value, int32_t* err_dev, void* stream);

/* Opaque checkpoint of everything a handle owns (ODE state, switching state, reference state, step counter):
 * size query, export to / import from a HOST blob.  The blob starts with a header (magic, ABI version, dtype, n_envs, record layout,
 * fingerprint of the configuration); gemb200_checkpoint_load refuses a blob written by a handle of another configuration
 * (GEMB200_E_INVALID) or ABI (GEMB200_E_ABI) instead of reinterpreting it. */
int64_t gemb200_checkpoint_size(gemb200_handle* h);
int gemb200_checkpoint_save(gemb200_handle* h, void* host_blob);
int gemb200_checkpoint_load(gemb200_handle* h, const void* host_blob);

/* Per-env state snapshots on the device (the batched counterpart of copy.deepcopy(env) in the reference): branch, archive and fan out
 * environments without a host round trip.  gemb200_pack_envs copies the complete persistent state of chosen envs into packed rows,
 * gemb200_unpack_envs puts rows into chosen envs of any handle of the same record layout (a plant handle of N envs can seed a model handle
 * of N*C envs; n_envs, seed, env_index_offset, tau, solver, parameters, limits, reward, constraints and I/O layout may all differ).
 * All pointers are device pointers; both calls are stream-ordered, never synchronise the host and can be captured in a CUDA graph (with
 * the device clock on they read the step count and the dead-time ring position from device memory).  Entries of env_idx / row_idx that
 * are out of range are skipped (pack leaves that row untouched).  Two entries of env_idx naming the same env in one unpack race.
 *
 * Row format: `words` 32-bit words per env, the persistent per-env arrays of the handle in the checkpoint's section order, each copied as
 * raw words (fp64 values as two words, low word first; a uint16 switching state zero-extended to one word):
 *   hot record [hot_words]   x_1..x_{nx-1}, reference value per slot                              (real)
 *   cold record [cold_words] omega, sigma or periodic start step per slot, sub-episode end per slot (real)
 *   angle                    double (DC motors: absent)
 *   finite switching state   uint16 -> 1 word (finite converters with interlocking time or an RC supply)
 *   dead-time queue          [dead_time_steps][fifo_dim] real, OLDEST entry first
 *   FluxObserver integrator  [4] real
 *   RC supply                [2] real
 *   AC supply phase          double
 *   switched generators      [n_ref][2] uint32: parameter entry, super-episode end
 *   external-profile clock   uint32 steps since the reset
 *   im_prev                  [2] real (induction motors with random initial states)
 * Fields kept against the handle's step count are stored RELATIVE to it (u32 difference, the same u32 encoding the record uses: the float
 * bit pattern in fp32, the integral double value in fp64): the sub-episode ends, the start step of a slot whose current generator is
 * periodic (sinus / step / sawtooth / triangular), and the super-episode ends.  Unpack re-bases them on the destination's step count.
 * Not in the row: the per-env parameter table (configuration, like in the checkpoint) and the RNG identity — a restored env draws the
 * random numbers of ITS OWN (seed, global index) from then on, unless it adopts its source's (gemb200_adopt_rng_ids below); and keeps
 * its own physical parameters, unless it takes its source's (gemb200_unpack_envs_params below).
 * layout_id: FNV-1a over what decides the row format (dtype, motor, n_ode, n_ref, generator kinds and switched grouping, switching-state
 * array, dead time and its order and queue width, state-op kinds, supply, external speed load, induction motor with random initial
 * states); not over n_envs, seed, offsets, device, tau, solver, parameters, limits, reward, constraints, autoreset or layout. */
/* words per env of a packed record and the id of its layout; no GPU needed (like gemb200_query_dims) */
int gemb200_query_env_record(const gemb200_config* cfg, int32_t* words, uint64_t* layout_id);
/* rows[j][0..words) = packed state of env env_idx[j] (env_idx NULL: env j), j < m */
int gemb200_pack_envs(gemb200_handle* h, const int32_t* env_idx, int32_t m, uint32_t* rows, void* stream);
/* env env_idx[j] (NULL: j) takes the state in rows[row_idx[j]] (NULL: row j), j < m; row_idx entries index [0, n_rows); refuses rows
 * of another layout_id with GEMB200_E_INVALID */
int gemb200_unpack_envs(gemb200_handle* h, const uint32_t* rows, int32_t n_rows, uint64_t layout_id, const int32_t* row_idx,
                        const int32_t* env_idx, int32_t m, void* stream);

/* RNG identities: copy.deepcopy(env) semantics for restored envs (opt-in; DESIGN §7).  Every random draw of an env is keyed by its
 * identity: a Philox key, a global env index, an RNG call-id offset and a step offset — by default the handle's seed, env_index_offset + i,
 * 0 and 0.  gemb200_pack_rng_ids exports the EFFECTIVE identity of chosen envs as rows of GEMB200_RNG_ID_WORDS uint32:
 *   [0] key lo  [1] key hi  [2] global env index lo  [3] hi  [4] call id of the env's next call lo  [5] hi  [6] its step count  [7] 0
 * (taken from the handle's clock; with the device clock on, from device memory).  gemb200_adopt_rng_ids gives env env_idx[j] (NULL: j)
 * identity row row_idx[j] (NULL: j): it stores the row's key and index and the differences between the row's call id / step count and
 * this handle's at the time of the call.  From then on every draw of that env — step, rollout, reset (masked or not), in-kernel auto-reset
 * and captured graphs; reference walks, sub-episodes, periodic and switched generators, initial values, random initial states, supply
 * phase, state noise, parameter draws — uses that identity.  Replay property: pack env s of handle A with gemb200_pack_envs and
 * gemb200_pack_rng_ids, unpack and adopt both into env d of handle B (other n_envs, seed or env_index_offset allowed, the same handle
 * too); the same sequence of calls on A and B with the same actions for s and d then gives env d bit for bit the outputs of env s.
 * Packing an env that holds an adopted identity exports it advanced to now, so a branch of a branch replays the original.
 * gemb200_unpack_envs gives the destination envs their own identity back; gemb200_reseed and gemb200_clear_rng_ids give it back to every
 * env and return a handle whose per-env parameter blocks only the adoption made to its shared-coefficient kernels.  Adoption needs the row-per-env I/O layout and is refused while parameters are drawn per reset (GEMB200_E_INVALID); while an
 * identity is adopted (until gemb200_clear_rng_ids or gemb200_reseed) gemb200_checkpoint_save / _load return GEMB200_E_INVALID: the blob
 * carries no identities.  The first adoption on a handle without per-env parameter blocks fills them from the shared parameters
 * (synchronises the device, not capturable); from then on the handle runs its per-env parameter kernels.  All calls are stream-ordered,
 * take device pointers and skip out-of-range entries; apart from that first adoption they never synchronise and can be captured.
 * A CUDA graph keeps the launch parameters it was captured with: capture step / rollout / reset launches AFTER the first adoption (and
 * again after gemb200_clear_rng_ids or gemb200_reseed) for them to read the identities; adoptions into a handle whose identities are in use
 * are seen by graphs captured since then. */
#define GEMB200_RNG_ID_WORDS 8
/* ids[j][0..GEMB200_RNG_ID_WORDS) = effective identity of env env_idx[j] (env_idx NULL: env j), j < m */
int gemb200_pack_rng_ids(gemb200_handle* h, const int32_t* env_idx, int32_t m, uint32_t* ids, void* stream);
/* env env_idx[j] (NULL: j) adopts identity row ids[row_idx[j]] (NULL: row j), j < m; row_idx entries index [0, n_ids) */
int gemb200_adopt_rng_ids(gemb200_handle* h, const uint32_t* ids, int32_t n_ids, const int32_t* row_idx, const int32_t* env_idx, int32_t m, void* stream);
/* every env draws with its own identity again */
int gemb200_clear_rng_ids(gemb200_handle* h, void* stream);

/* Per-env physical parameters in snapshots (opt-in; DESIGN §7): branch and deep-copy envs whose parameters are their own — set from the
 * host (gemb200_set_env_params) or drawn at every reset (gemb200_set_param_randomization).  A parameter row is GEMB200_ENV_PARAM_SLOTS
 * doubles in the slot order of gemb200_config: motor_param[GEMB200_MP_*], then load_param[GEMB200_LP_*] (the slot numbers of
 * gemb200_set_param_randomization).
 * gemb200_pack_envs_params is gemb200_pack_envs plus the parameter rows params[j][..] of env env_idx[j]: an env's per-env values, copied
 * exactly (drawn values are stored rounded to the handle's dtype), or the configuration's on a handle without per-env blocks.
 * gemb200_unpack_envs_params is gemb200_unpack_envs plus parameter adoption, plus identity adoption when ids is non-NULL (the
 * gemb200_adopt_rng_ids semantics, ids[row_idx[j]] with the same n_rows): env env_idx[j] stores every slot of row row_idx[j] except the
 * pole pairs, which are per handle (the angle increments are prepared on the host; the caller checks that source and destination agree),
 * and its per-env coefficients are derived from them on the device by the code that derives drawn parameters.  The restored env then runs
 * its current episode on its source's plant; with draws on, its next reset draws new values as usual (with an adopted identity: its
 * source's draws).  Rows are used as given, like gemb200_set_env_params rows, but not checked: a zero inductance gives non-finite
 * coefficients.  For an induction motor with random initial states the flux limits (init_im) stay the handle's, derived on the host from
 * the configuration: a row with other l_m, l_sigs, l_sigr, r_s or r_r behaves like a gemb200_set_env_params row with those values.
 * After an unpack with params the handle's per-env blocks are the caller's: its other envs keep their values (the shared parameters on a
 * handle without blocks), but derive a constant initial state's reset observation on the device (DESIGN §4: last bits of the induction
 * motors).  Both calls are accepted while parameters are drawn per reset, need the row-per-env I/O layout and non-NULL rows and params
 * (GEMB200_E_INVALID otherwise), are stream-ordered and can be captured in a CUDA graph — except the first unpack on a handle without
 * per-env blocks, which fills them from the shared parameters and synchronises the device.  gemb200_pack_envs / _unpack_envs, their row
 * format and layout_id are unchanged, and still refused while draws are on. */
#define GEMB200_ENV_PARAM_SLOTS 24 /* GEMB200_MAX_MOTOR_PARAM motor slots, then 8 load slots */
int gemb200_pack_envs_params(gemb200_handle* h, const int32_t* env_idx, int32_t m, uint32_t* rows, double* params, void* stream);
int gemb200_unpack_envs_params(gemb200_handle* h, const uint32_t* rows, const double* params, const uint32_t* ids, int32_t n_rows,
                               uint64_t layout_id, const int32_t* row_idx, const int32_t* env_idx, int32_t m, void* stream);

/* Introspection used by bench.py: number of kernel launches issued through this handle so far, and the
 * CUDA-event time in ms of the step launches since the last call (see DESIGN.md "Measurement"). */
int64_t gemb200_launch_count(gemb200_handle* h);
int gemb200_kernel_time_begin(gemb200_handle* h, void* stream);
int gemb200_kernel_time_end(gemb200_handle* h, void* stream, float* ms_out);

#ifdef __cplusplus
}
#endif
#endif /* GEMB200_H_ */
