// gemb200.cu — C-ABI implementation (include/gemb200.h): handle management, host-side derivation of the model
// constants from the physical parameters (the reference's *_update_model methods), kernel dispatch.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <limits>
#include <string>
#include <type_traits>
#include <vector>

#include "gemb200_jac.h"
#include "gemb200_launch.cuh"

using namespace gemb200;

// ----------------------------------------------------------------------------------------------------------------
// error reporting
// ----------------------------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;
static int fail(int code, const std::string& msg) { g_last_error = msg; return code; }
#define CUDA_TRY(expr)                                                                                 \
  do {                                                                                                 \
    cudaError_t e_ = (expr);                                                                           \
    if (e_ != cudaSuccess) return fail(GEMB200_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_)); \
  } while (0)

// ----------------------------------------------------------------------------------------------------------------
// handle
// ----------------------------------------------------------------------------------------------------------------
enum BlockSource {   // per-env parameter blocks of a handle
  kBlocksNone = 0,   // none: every env uses the shared coefficients
  kBlocksShared = 1, // the shared parameters, filled by an adoption of RNG identities (which only the ENVP instantiations read)
  kBlocksCaller = 2  // the caller's: rows of gemb200_set_env_params, or parameter draws
};
struct gemb200_handle {
  gemb200_config cfg;
  int fam = 0, n_state = 0, n_ode = 0, n_act = 0, n_ref = 0, nx = 0;
  bool has_eps = false, any_wiener = false, two_segment = false;
  size_t rsz = 4;  // sizeof(real)
  // persistent per-env device state: allocated, freed, saved, reseeded and packed by walking sections()
  int NH = 0, NC = 0;  // words per env in the hot / cold record
  void* d_st = nullptr;
  void* d_stc = nullptr;
  double* d_eps = nullptr;
  uint16_t* d_sw = nullptr;
  void* d_fifo = nullptr;
  int fifo_dim = 0;
  void* d_sup = nullptr;   // RC supply state [2][n]
  double* d_supph = nullptr;  // AC supply phase [n]
  uint32_t* d_kenv = nullptr;  // steps since the reset per env (external speed profile)
  uint32_t* d_swst = nullptr;  // switched reference generators [n_ref][2][n]
  void* d_obsv = nullptr;  // FluxObserver integrator [4][n]: re, im, compensation of re, of im
  void* d_imprev = nullptr;  // induction motors with random initial states [2][n]: initial currents of the env's previous episode
  // other device buffers
  void* d_ext = nullptr;       // external speed profile table (real)
  void* d_envp = nullptr;    // per-env model coefficients [kCoefWords][n] (gemb200_set_env_params), allocated at the first use
  double* d_praw = nullptr;  // physical parameters per env [kMaxDraw][n] (double), valid whenever d_envp is in use
  ParamDraw* d_draw = nullptr;  // distributions of the parameters drawn at every reset (gemb200_set_param_randomization)
  uint32_t* d_rngid = nullptr;  // RNG identities [kRngIdWords][n] (gemb200_adopt_rng_ids), allocated at the first adoption
  // launch mode: which instantiation a launch takes (PLAIN, general or ENVP, DESIGN §4).  apply_mode() derives the mode fields of the
  // live StepParams from these; every entry point that changes one of them calls it.
  BlockSource blocks = kBlocksNone;  // where the per-env parameter blocks in d_envp / d_praw come from
  int n_draw = 0;            // parameters drawn per reset (0: none)
  bool ids_in_use = false;   // adopted RNG identities in d_rngid, since the last reseed / gemb200_clear_rng_ids
  int n_dst = 0;             // peer destinations of the output stores (gemb200_bind_peers)
  int64_t dst_delta[8] = {};
  bool plain_shape = false;  // the configuration has the PLAIN shape (fill_params), which per-env blocks and peer stores switch off
  int n_obs = 0, row_stride = 0;
  StepParams<float> pf;      // the parameter block of the handle's dtype is the live one; only with_params() names them
  StepParams<double> pd;
  uint64_t gstep = 0;
  uint64_t n_steps = 0;  // step calls so far (dead-time ring position)
  uint64_t ext_hash = 0; // FNV-1a of the external speed profile table (part of the checkpoint fingerprint)
  uint32_t* d_clock = nullptr;  // device-resident clock (gemb200_set_device_clock): {call id lo, hi, step count lo, ring position, step count hi, -, -, -}
  bool dev_clock = false;       // launches read d_clock instead of gstep / n_steps (which are then stale until the clock is pulled back)
  int64_t launches = 0;
  // host-buffer path
  cudaStream_t hstream = nullptr;
  cudaStream_t hpipe[3] = {nullptr, nullptr, nullptr};
  void *d_act = nullptr, *d_obs = nullptr, *d_ref = nullptr, *d_rew = nullptr;
  uint8_t *d_term = nullptr, *d_mask = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

// The one dispatch on the handle's dtype: f(the live StepParams<real>).  Inside f, decltype(p.tau) is `real`.
template <typename F>
static auto with_params(gemb200_handle* h, F&& f) {
  if (h->cfg.dtype == GEMB200_F32) return f(h->pf);
  return f(h->pd);
}
// the mode fields of the live StepParams, derived from the handle's launch mode
static void apply_mode(gemb200_handle* h) {
  with_params(h, [h](auto& p) {
    using real = decltype(p.tau);
    p.envp = h->blocks != kBlocksNone ? static_cast<const real*>(h->d_envp) : nullptr;
    p.praw = h->d_praw;
    p.coef_shared = h->blocks == kBlocksShared;
    p.n_draw = h->n_draw;
    p.draw = h->d_draw;
    p.rngid = h->ids_in_use ? h->d_rngid : nullptr;
    p.n_dst = h->n_dst;
    std::memcpy(p.dst_delta, h->dst_delta, sizeof(p.dst_delta));
    // the PLAIN instantiations read the shared constant-bank coefficients and store to the caller's tensors only
    p.plain = h->plain_shape && h->blocks == kBlocksNone && h->n_dst == 0;
  });
}
// neither checkpoints nor packed rows carry the parameters drawn per reset (DESIGN §7)
static bool draws_on(const gemb200_handle* h) { return h->n_draw > 0; }

// ----------------------------------------------------------------------------------------------------------------
// dimensions / validation (SCMLSystem._set_indices physical_systems.py:141-162, :462-485, :594-617, :737-763)
// ----------------------------------------------------------------------------------------------------------------
static bool is_qc(int k) { return k == GEMB200_CONV_1QC || k == GEMB200_CONV_2QC || k == GEMB200_CONV_4QC; }

struct Dims { int fam, n_state, n_ode, n_act, nx; bool has_eps; int n_obs = 0; bool has_observer = false; };  // n_state: the system's own vector, n_obs: after the wrappers

static int derive_dims(const gemb200_config* c, Dims* d) {
  const int k0 = c->converter_kind[0], k1 = c->converter_kind[1];
  switch (c->motor_kind) {
    case GEMB200_MOTOR_PERMEX_DC:
    case GEMB200_MOTOR_SERIES_DC: *d = {kDC1, 5, 2, 1, 2, false}; break;
    case GEMB200_MOTOR_SHUNT_DC: *d = {kDC2, 7, 3, 1, 3, false}; break;
    case GEMB200_MOTOR_EXTEX_DC: *d = {kDC2, 7, 3, 2, 3, false}; break;
    case GEMB200_MOTOR_PMSM:
    case GEMB200_MOTOR_SYNRM: *d = {kSYNC, 14, 4, c->finite ? 1 : 3, 3, true}; break;
    case GEMB200_MOTOR_EESM: *d = {kEESM, 16, 5, c->finite ? 2 : 4, 4, true}; break;
    case GEMB200_MOTOR_SCIM: *d = {kSCIM, 14, 6, c->finite ? 1 : 3, 5, true}; break;
    case GEMB200_MOTOR_DFIM: *d = {kDFIM, 24, 6, c->finite ? 2 : 6, 5, true}; break;
    default: return fail(GEMB200_E_INVALID, "unknown motor_kind");
  }
  const bool three_phase = d->fam >= kSYNC;
  if (c->action_dq) {
    if (!three_phase || c->finite) return fail(GEMB200_E_INVALID, "dq actions need a three-phase motor with a continuous converter");
    d->n_act = c->motor_kind == GEMB200_MOTOR_EESM ? 3 : (c->motor_kind == GEMB200_MOTOR_DFIM ? 4 : 2);
  }
  // state-vector wrappers (gemb200_state_op): width bookkeeping as in the wrappers' set_physical_system
  d->n_obs = d->n_state;
  if (c->n_state_ops < 0 || c->n_state_ops > GEMB200_MAX_STATE_OPS) return fail(GEMB200_E_INVALID, "n_state_ops out of range");
  for (int k = 0; k < c->n_state_ops; ++k) {
    switch (c->sop_kind[k]) {
      case GEMB200_SOP_COS_SIN:
        if (c->sop_idx[k][0] < 0 || c->sop_idx[k][0] >= d->n_obs) return fail(GEMB200_E_INVALID, "CosSinProcessor: angle index out of range");
        d->n_obs += c->sop_idx[k][1] ? 1 : 2;
        break;
      case GEMB200_SOP_FLUX_OBSERVER:
        if (c->motor_kind != GEMB200_MOTOR_SCIM && c->motor_kind != GEMB200_MOTOR_DFIM) return fail(GEMB200_E_INVALID, "FluxObserver needs an induction motor (flux_observer.py:57-60)");
        if (d->has_observer) return fail(GEMB200_E_INVALID, "only one FluxObserver per system");
        for (int q = 0; q < 4; ++q)
          if (c->sop_idx[k][q] < 0 || c->sop_idx[k][q] >= d->n_obs) return fail(GEMB200_E_INVALID, "FluxObserver: state index out of range");
        if (!(c->sop_param[k][3] > 0)) return fail(GEMB200_E_INVALID, "FluxObserver: psi_limit must be positive");
        d->has_observer = true;
        d->n_obs += 2;
        break;
      case GEMB200_SOP_CURRENT_SUM:
        if (c->sop_mask[k] == 0 || (d->n_obs < 32 && (c->sop_mask[k] >> d->n_obs) != 0)) return fail(GEMB200_E_INVALID, "CurrentSumProcessor: state indices out of range");
        d->n_obs += 1;
        break;
      case GEMB200_SOP_NOISE:
        if (c->sop_idx[k][0] < GEMB200_NOISE_NORMAL || c->sop_idx[k][0] > GEMB200_NOISE_LAPLACE) return fail(GEMB200_E_INVALID, "StateNoiseProcessor: unknown distribution");
        if (d->n_obs < 32 && (c->sop_mask[k] >> d->n_obs) != 0) return fail(GEMB200_E_INVALID, "StateNoiseProcessor: state index out of range");
        break;
      default: return fail(GEMB200_E_INVALID, "unknown state op");
    }
    if (d->n_obs > GEMB200_MAX_STATE) return fail(GEMB200_E_INVALID, "state vector too long");
  }
  if (c->action_dq == 2 && !(c->motor_kind == GEMB200_MOTOR_SCIM && d->has_observer))
    return fail(GEMB200_E_INVALID, "action_dq = 2 (observer angle) needs a SCIM with a FluxObserver");
  if (c->motor_kind == GEMB200_MOTOR_DFIM && c->action_dq && !(c->action_dq == 3 && d->has_observer))
    return fail(GEMB200_E_INVALID, "DFIM dq actions are action_dq = 3 and need a FluxObserver (dq_to_abc_action_processor.py:108-137)");
  if (c->action_dq == 3 && c->motor_kind != GEMB200_MOTOR_DFIM) return fail(GEMB200_E_INVALID, "action_dq = 3 is the DFIM processor");
  if (three_phase) {
    if (k0 != GEMB200_CONV_B6) return fail(GEMB200_E_INVALID, "three-phase motors need a B6 bridge in converter slot 0");
    if (c->motor_kind == GEMB200_MOTOR_EESM) {
      if (!is_qc(k1)) return fail(GEMB200_E_INVALID, "EESM needs a 1QC/2QC/4QC excitation converter in slot 1");
    } else if (c->motor_kind == GEMB200_MOTOR_DFIM) {
      if (k1 != GEMB200_CONV_B6) return fail(GEMB200_E_INVALID, "DFIM needs a second B6 bridge (rotor) in converter slot 1");
    } else if (k1 != GEMB200_CONV_NONE) return fail(GEMB200_E_INVALID, "converter slot 1 must be NONE for this motor");
  } else {
    if (!is_qc(k0)) return fail(GEMB200_E_INVALID, "DC motors need a 1QC/2QC/4QC converter in slot 0");
    if (c->motor_kind == GEMB200_MOTOR_EXTEX_DC) {
      if (!is_qc(k1)) return fail(GEMB200_E_INVALID, "ExtEx DC motor needs an excitation converter in slot 1");
    } else if (k1 != GEMB200_CONV_NONE) return fail(GEMB200_E_INVALID, "converter slot 1 must be NONE for this motor");
  }
  return GEMB200_OK;
}

static int validate(const gemb200_config* c) {
  if (!c) return fail(GEMB200_E_INVALID, "config is NULL");
  if (c->struct_size != (int32_t)sizeof(gemb200_config) || c->abi_version != GEMB200_ABI_VERSION)
    return fail(GEMB200_E_ABI, "gemb200_config struct_size/abi_version mismatch (use gemb200_config_init)");
  if (c->n_envs < 1) return fail(GEMB200_E_INVALID, "n_envs must be >= 1");
  if (c->dtype != GEMB200_F32 && c->dtype != GEMB200_F64) return fail(GEMB200_E_INVALID, "bad dtype");
  if (c->layout != GEMB200_LAYOUT_AOS && c->layout != GEMB200_LAYOUT_SOA) return fail(GEMB200_E_INVALID, "bad layout");
  if (c->solver_kind != GEMB200_SOLVER_EULER && c->solver_kind != GEMB200_SOLVER_RK4)
    return fail(GEMB200_E_INVALID, "solver_kind must be EULER or RK4 (the scipy solvers of the reference map to RK4 sub-stepping, see DESIGN.md)");
  if (c->solver_nsteps < 1 || c->solver_nsteps > 1024) return fail(GEMB200_E_INVALID, "solver_nsteps out of range");
  if (!(c->tau > 0)) return fail(GEMB200_E_INVALID, "tau must be positive");
  if (c->interlocking_time < 0 || c->interlocking_time >= c->tau) return fail(GEMB200_E_INVALID, "interlocking_time must be in [0, tau)");
  if (c->interlocking_time1 >= c->tau) return fail(GEMB200_E_INVALID, "interlocking_time1 must be < tau (negative: same as interlocking_time)");
  if (c->load_kind < GEMB200_LOAD_CONST_SPEED || c->load_kind > GEMB200_LOAD_EXT_SPEED) return fail(GEMB200_E_INVALID, "bad load_kind");
  if (c->load_kind == GEMB200_LOAD_EXT_SPEED) {
    if (!c->ext_speed_table || c->ext_speed_len < 4 * c->solver_nsteps + 2) return fail(GEMB200_E_INVALID, "external speed load: table missing or shorter than two steps");
    if (!(c->load_param[GEMB200_LP_TAU_LOAD] > 0)) return fail(GEMB200_E_INVALID, "external speed load: tau_load must be positive");
    if (c->finite && (c->interlocking_time > 0 || c->interlocking_time1 > 0)) return fail(GEMB200_E_INVALID, "external speed load with two-segment steps (finite converter + interlocking time) is not supported: the segment times are off the table grid");
  }
  if (c->n_ref < 0 || c->n_ref > GEMB200_MAX_REF) return fail(GEMB200_E_INVALID, "n_ref out of range");
  if (c->dead_time_steps < 0 || c->dead_time_steps > GEMB200_MAX_DEAD_TIME) return fail(GEMB200_E_INVALID, "dead_time_steps out of range");
  const bool induction = c->motor_kind == GEMB200_MOTOR_SCIM || c->motor_kind == GEMB200_MOTOR_DFIM;
  if (c->init_random && induction && !c->init_im_valid)
    return fail(GEMB200_E_INVALID, "random initial states of an induction motor need init_im (flux-limit constants, see gemb200.h)");
  if (c->init_im_valid && !(induction && c->init_random)) return fail(GEMB200_E_INVALID, "init_im is for induction motors with init_random");
  if (c->init_im_valid && !(c->init_im[4] != 0.0)) return fail(GEMB200_E_INVALID, "init_im[4] (p * l_m / l_r) must be non-zero");
  for (int j = 0; j < GEMB200_MAX_ODE; ++j)
    if (c->init_random && c->init_dist[j] && !(c->init_sigma[j] > 0 && (c->init_hi[j] > c->init_lo[j])))
      return fail(GEMB200_E_INVALID, "truncated-normal initial state needs sigma > 0 and a non-empty interval");
  if (c->supply_kind < GEMB200_SUPPLY_IDEAL || c->supply_kind > GEMB200_SUPPLY_AC1) return fail(GEMB200_E_INVALID, "bad supply_kind");
  if (c->supply_kind == GEMB200_SUPPLY_AC1 && !(c->supply_param[0] > 0)) return fail(GEMB200_E_INVALID, "AC supply needs a positive frequency");
  if (c->supply_kind == GEMB200_SUPPLY_RC && !(c->supply_param[0] > 0 && c->supply_param[1] > 0)) return fail(GEMB200_E_INVALID, "RC supply needs R > 0 and C > 0");
  if (c->n_constraints < 0 || c->n_constraints > GEMB200_MAX_CONSTRAINTS) return fail(GEMB200_E_INVALID, "n_constraints out of range");
  for (int i = 0; i < c->n_constraints; ++i)
    if (c->constraint_kind[i] != GEMB200_CONSTRAINT_LIMIT && c->constraint_kind[i] != GEMB200_CONSTRAINT_SQUARED) return fail(GEMB200_E_INVALID, "bad constraint_kind");
  if (c->autoreset != GEMB200_AUTORESET_NONE && c->autoreset != GEMB200_AUTORESET_SAME_STEP) return fail(GEMB200_E_INVALID, "bad autoreset mode");
  Dims d;
  int rc = derive_dims(c, &d);
  if (rc) return rc;
  if (c->finite && (c->interlocking_time > 0 || c->interlocking_time1 > 0) && c->motor_kind == GEMB200_MOTOR_EESM)
    return fail(GEMB200_E_INVALID, "finite EESM with interlocking time: the reference raises in this configuration "
                                   "(physical_systems.py:632 slices u_in[:2]); not supported");
  int n_entries = c->n_ref;  // parameter entries in use: the output slots plus the extra sub-generators of switched slots
  for (int r = 0; r < c->n_ref; ++r) {
    if (c->ref_sw_count[r] <= 1) continue;
    const int first = c->ref_sw_first[r], cnt = c->ref_sw_count[r];
    if (first < 0 || first + cnt > GEMB200_MAX_REF_ENTRIES) return fail(GEMB200_E_INVALID, "switched reference generator: parameter entries out of range");
    if (first + cnt > n_entries) n_entries = first + cnt;
    if (c->ref_sw_len_lo[r] < 1 || c->ref_sw_len_hi[r] <= c->ref_sw_len_lo[r]) return fail(GEMB200_E_INVALID, "switched reference generator: bad super-episode length range");
    for (int m = 0; m < cnt; ++m) {
      const int k = c->ref_kind[first + m];
      if (k == GEMB200_REF_EXTERNAL) return fail(GEMB200_E_INVALID, "switched reference generator: external sub-generators are not supported");
      if (!(c->ref_sw_cdf[first + m] > 0 && c->ref_sw_cdf[first + m] <= 1.0 + 1e-12)) return fail(GEMB200_E_INVALID, "switched reference generator: bad probabilities");
    }
  }
  for (int r = 0; r < c->n_ref; ++r)
    if (c->ref_state[r] < 0 || c->ref_state[r] >= d.n_obs) return fail(GEMB200_E_INVALID, "ref_state out of range");
  for (int r = 0; r < n_entries; ++r) {
    if (c->ref_kind[r] < GEMB200_REF_CONST || c->ref_kind[r] > GEMB200_REF_TRIANGULAR) return fail(GEMB200_E_INVALID, "bad ref_kind");
    const bool subep = c->ref_kind[r] == GEMB200_REF_WIENER || c->ref_kind[r] >= GEMB200_REF_LAPLACE;
    const bool walk = c->ref_kind[r] == GEMB200_REF_WIENER || c->ref_kind[r] == GEMB200_REF_LAPLACE;
    if (subep && (c->ref_len_lo[r] < 1 || c->ref_len_hi[r] < c->ref_len_lo[r] || c->ref_len_hi[r] > (1 << 24)))
      return fail(GEMB200_E_INVALID, "bad sub-episode length range");
    if (walk && !(c->ref_sigma_lo[r] > 0 && c->ref_sigma_hi[r] >= c->ref_sigma_lo[r])) return fail(GEMB200_E_INVALID, "bad sigma range");
    if (c->ref_kind[r] >= GEMB200_REF_SINUS && !(c->ref_freq_lo[r] > 0 && c->ref_freq_hi[r] >= c->ref_freq_lo[r] && c->ref_amp_lo[r] >= 0))
      return fail(GEMB200_E_INVALID, "bad amplitude / frequency range of a periodic reference generator");
  }
  for (int j = 0; j < d.n_obs; ++j)
    if (c->reward_weight[j] != 0.0 && !(c->state_length[j] > 0)) return fail(GEMB200_E_INVALID, "state_length must be positive for every weighted state");
  for (int j = 0; j < d.n_state; ++j)
    if (!(c->limits[j] != 0.0) && !(c->motor_kind == GEMB200_MOTOR_SHUNT_DC && j == 6)) return fail(GEMB200_E_INVALID, "limits must be non-zero");
  const double j_total = c->load_param[GEMB200_LP_J_LOAD] + c->motor_param[GEMB200_MP_J_ROTOR];
  if (c->load_kind == GEMB200_LOAD_POLY_STATIC && !(j_total > 0)) return fail(GEMB200_E_INVALID, "total inertia must be positive");
  if ((int64_t)c->n_envs * (int64_t)(hot_words(d.nx, c->n_ref) + cold_words(d.nx, c->n_ref) > d.n_obs ? hot_words(d.nx, c->n_ref) + cold_words(d.nx, c->n_ref) : d.n_obs) >= (int64_t)1 << 31)
    return fail(GEMB200_E_INVALID, "n_envs too large for 32-bit element indexing in one handle; shard the batch");
  return GEMB200_OK;
}

// which optional per-env arrays a configuration has (gemb200_create allocates them, sections() lists them)
static int fifo_dim_of(const gemb200_config* c, const Dims& d) {
  if (c->dead_time_steps <= 0) return 0;
  // queue width: caller-side actions when the dead time wraps the dq transformation (or there is none), else abc(+e)
  const int inner = c->finite ? d.n_act : (d.fam == kDFIM ? 6 : (d.fam == kEESM ? 4 : (d.fam >= kSYNC ? 3 : d.n_act)));
  return (c->action_dq && !c->dead_time_outer) ? inner : d.n_act;
}
static bool has_sw_state(const gemb200_config* c) {  // finite switching states: two-segment steps (interlocking time) or an RC supply
  return c->finite && (c->interlocking_time > 0 || c->interlocking_time1 > 0 || c->supply_kind == GEMB200_SUPPLY_RC);
}
static bool any_switched_slot(const gemb200_config* c) {
  for (int r = 0; r < c->n_ref; ++r) if (c->ref_sw_count[r] > 1) return true;
  return false;
}
constexpr int kMaxSections = 16;
// The persistent per-env arrays of a configuration, in checkpoint order.  One table serves the allocation at create and the release at
// destroy (slot: where the handle keeps the array's device pointer, bytes), the checkpoint blob, the reseed and the packed env records of
// gemb200_pack_envs / gemb200_unpack_envs (element size, elements per env, placement, clock-relative fields), so an array cannot be in
// one and missing from another.  h == nullptr: shapes only (slot = nullptr).
// checkpoint blob: [header][hot records][cold records][eps][sw][dead-time queue]...  The header pins the blob to the configuration that
// wrote it: a blob of equal size from another motor / seed / tau / generator set is refused instead of being reinterpreted.
enum SecPlace { kPlanar = 0, kRecord = 1 };  // planar: element e of env i at [e * n + i]; record: 16-byte chunked record (word_offset)
enum SecClock {
  kClkNone = 0,
  kClkCold = 1,  // cold record: sub-episode ends, and the start step of a slot whose current generator is periodic
  kClkSwst = 2,  // switched generators [n_ref][2]: the super-episode end (odd elements)
  kClkRing = 3   // dead-time ring [dead_time_steps][fifo_dim], stored oldest entry first in a row
};
struct Section { void** slot; size_t bytes; int esz, per_env, place, clk; };  // esz: bytes per element
static int config_sections(const gemb200_config* c, gemb200_handle* h, Section* s) {
  Dims d;
  derive_dims(c, &d);
  const size_t n = (size_t)c->n_envs;
  const int rsz = c->dtype == GEMB200_F32 ? 4 : 8;
  int k = 0;
  auto add = [&](void* p, int esz, int per_env, int place, int clk) { s[k++] = {static_cast<void**>(p), n * (size_t)per_env * esz, esz, per_env, place, clk}; };
  add(h ? &h->d_st : nullptr, rsz, hot_words(d.nx, c->n_ref), kRecord, kClkNone);
  add(h ? &h->d_stc : nullptr, rsz, cold_words(d.nx, c->n_ref), kRecord, kClkCold);
  if (d.has_eps) add(h ? &h->d_eps : nullptr, 8, 1, kPlanar, kClkNone);
  if (has_sw_state(c)) add(h ? &h->d_sw : nullptr, 2, 1, kPlanar, kClkNone);
  if (c->dead_time_steps > 0) add(h ? &h->d_fifo : nullptr, rsz, c->dead_time_steps * fifo_dim_of(c, d), kPlanar, kClkRing);
  if (d.has_observer) add(h ? &h->d_obsv : nullptr, rsz, 4, kPlanar, kClkNone);
  if (c->supply_kind == GEMB200_SUPPLY_RC) add(h ? &h->d_sup : nullptr, rsz, 2, kPlanar, kClkNone);
  if (c->supply_kind == GEMB200_SUPPLY_AC1) add(h ? &h->d_supph : nullptr, 8, 1, kPlanar, kClkNone);
  if (any_switched_slot(c)) add(h ? &h->d_swst : nullptr, 4, 2 * c->n_ref, kPlanar, kClkSwst);
  if (c->load_kind == GEMB200_LOAD_EXT_SPEED) add(h ? &h->d_kenv : nullptr, 4, 1, kPlanar, kClkNone);
  if (c->init_im_valid) add(h ? &h->d_imprev : nullptr, rsz, 2, kPlanar, kClkNone);
  return k;  // (the per-env parameter table is configuration, not state: re-apply gemb200_set_env_params after a load; parameter draws
             //  per reset make it state, so checkpoints and snapshots are refused while they are on)
}
static int sections(gemb200_handle* h, Section* s) { return config_sections(&h->cfg, h, s); }
static int row_words(const Section& s) { return s.per_env * (s.esz == 8 ? 2 : 1); }

// ----------------------------------------------------------------------------------------------------------------
// model constants (double) -> StepParams<real>
// ----------------------------------------------------------------------------------------------------------------
struct Derived {
  double c[20] = {0};
  double tq[4] = {0};
  double reset_obs[GEMB200_MAX_STATE] = {0};
  double reset_obs_du[GEMB200_MAX_STATE] = {0};  // d reset_obs / d u_sup (the voltage entries are linear in u_sup)
  double inv_j = 0, omega_lim = 0, omega_lin = 0;
};

static void derive_model(const gemb200_config* cfg, const Dims& dm, Derived* o) {
  ModelCoef mc;
  derive_coef(cfg->motor_kind, cfg->motor_param, cfg->load_param, &mc);  // gemb200_model.h: shared with the parameter draws on the device
  for (int j = 0; j < 20; ++j) o->c[j] = mc.c[j];
  for (int j = 0; j < 4; ++j) o->tq[j] = mc.tq[j];
  o->inv_j = mc.inv_j; o->omega_lim = mc.omega_lim; o->omega_lin = mc.omega_lin;

  // observation right after reset (SCMLSystem.reset physical_systems.py:256-287, :527-561, :659-693, :816-847) for the
  // constant initial state; converter.reset() gives 0 per QC and -0.5 per B6 leg (converters.py:45-54, :880-886)
  const double* y = cfg->init_ode;
  const double U = cfg->u_sup;
  double* s = o->reset_obs;
  int n = 0;
  s[n++] = y[0];
  switch (dm.fam) {
    case kDC1: s[n++] = (o->tq[0] + o->tq[1] * y[1]) * y[1]; s[n++] = y[1]; s[n++] = 0.0; break;
    case kDC2:
      s[n++] = o->tq[0] * y[1] * y[2]; s[n++] = y[1]; s[n++] = y[2]; s[n++] = 0.0;
      if (cfg->motor_kind == GEMB200_MOTOR_EXTEX_DC) s[n++] = 0.0;
      break;
    default: {
      double eps = y[dm.nx];
      if (eps > M_PI) eps -= 2 * M_PI;
      const double ua = -0.5 * U;
      // abc -> alpha/beta of (ua,ua,ua) is mathematically 0 (the reference shows ~1e-17 round-off here)
      const double ualpha = 2.0 / 3.0 * (ua - 0.5 * ua - 0.5 * ua), ubeta = 2.0 / 3.0 * (0.5 * std::sqrt(3.0) * ua - 0.5 * std::sqrt(3.0) * ua);
      double cs, sn, tqv, ia, ib;
      if (dm.fam == kSCIM || dm.fam == kDFIM) {
        const double ef = std::atan2(y[4], y[3]);
        cs = std::cos(ef); sn = std::sin(ef);
        tqv = o->tq[0] * (y[3] * y[2] - y[4] * y[1]);
        ia = y[1]; ib = y[2];
      } else {
        cs = std::cos(eps); sn = std::sin(eps);
        tqv = dm.fam == kSYNC ? (o->tq[0] + o->tq[1] * y[1]) * y[2] : (o->tq[0] * y[3] + o->tq[1] * y[1]) * y[2];
        ia = cs * y[1] - sn * y[2]; ib = sn * y[1] + cs * y[2];
      }
      const double ud = cs * ualpha + sn * ubeta, uq = -sn * ualpha + cs * ubeta;
      s[n++] = tqv;
      s[n++] = ia; s[n++] = -0.5 * ia + 0.5 * std::sqrt(3.0) * ib; s[n++] = -0.5 * ia - 0.5 * std::sqrt(3.0) * ib;
      if (dm.fam == kDFIM) {
        // physical_systems.py:1062-1113: i_sdq in the field frame; i_rdq (sic) with the angle eps_field - eps_el, i_rdef = its inverse;
        // all six bridge legs at -0.5 u_sup, whose alpha-beta image is 0
        const double ira = o->c[8] * y[3] - o->c[9] * y[1], irb = o->c[8] * y[4] - o->c[9] * y[2];
        const double cfe = std::cos(std::atan2(y[4], y[3]) - eps), sfe = std::sin(std::atan2(y[4], y[3]) - eps);
        s[n++] = cs * y[1] + sn * y[2]; s[n++] = -sn * y[1] + cs * y[2];
        s[n++] = ira; s[n++] = -0.5 * ira + 0.5 * std::sqrt(3.0) * irb; s[n++] = -0.5 * ira - 0.5 * std::sqrt(3.0) * irb;
        s[n++] = cfe * ira + sfe * irb; s[n++] = -sfe * ira + cfe * irb;
        s[n++] = ua; s[n++] = ua; s[n++] = ua; s[n++] = ud; s[n++] = uq;
        s[n++] = ua; s[n++] = ua; s[n++] = ua; s[n++] = cfe * ualpha + sfe * ubeta; s[n++] = -sfe * ualpha + cfe * ubeta;
        s[n++] = eps;
        break;
      }
      if (dm.fam == kSCIM) { s[n++] = cs * y[1] + sn * y[2]; s[n++] = -sn * y[1] + cs * y[2]; }
      else { s[n++] = y[1]; s[n++] = y[2]; }
      if (dm.fam == kEESM) {
        // reference quirk (:659-693): u_abc has 4 entries [ua,ub,uc,u_e=0], then u_dq -> the slots named
        // u_sd,u_sq,u_e receive (0, u_d, u_q)
        s[n++] = y[3];
        s[n++] = ua; s[n++] = ua; s[n++] = ua; s[n++] = 0.0; s[n++] = ud; s[n++] = uq;
      } else {
        s[n++] = ua; s[n++] = ua; s[n++] = ua; s[n++] = ud; s[n++] = uq;
      }
      s[n++] = eps;
    } break;
  }
  s[n++] = U;
  for (int j = 0; j < n; ++j) s[j] /= cfg->limits[j];
  if (cfg->motor_kind == GEMB200_MOTOR_SHUNT_DC) s[n] = s[2] + s[3];
}

template <typename real>
static void set_seed(StepParams<real>* p, uint64_t seed) {
  p->seed_lo = (uint32_t)seed; p->seed_hi = (uint32_t)(seed >> 32);
  for (int r = 0; r < 10; ++r) { p->rk[r][0] = p->seed_lo + (uint32_t)r * 0x9E3779B9u; p->rk[r][1] = p->seed_hi + (uint32_t)r * 0xBB67AE85u; }
}

// fills the parameter block of a fresh handle (launch mode off: apply_mode() sets those fields); returns whether the configuration has the
// PLAIN shape
template <typename real>
static bool fill_params(const gemb200_handle* h, const Dims& dm, const Derived& dv, StepParams<real>* p) {
  const gemb200_config& c = h->cfg;
  std::memset(p, 0, sizeof(*p));
  p->n = c.n_envs;
  p->env_begin = 0; p->env_end = c.n_envs;
  p->env_offset = c.env_index_offset;
  set_seed(p, c.seed);
  p->st = static_cast<real*>(h->d_st);
  p->stc = static_cast<real*>(h->d_stc);
  p->kstep = 0;
  p->eps = h->d_eps;
  p->sw = h->d_sw;
  p->layout = c.layout;
  p->n_act = dm.n_act;
  p->fifo = static_cast<real*>(h->d_fifo);
  p->action_dq = c.action_dq;
  p->dead_steps = c.dead_time_steps; p->dead_outer = c.dead_time_outer; p->fifo_dim = h->fifo_dim; p->fifo_slot = 0;
  p->adv_k = (real)(c.angle_advance * c.tau * c.motor_param[GEMB200_MP_P] * (sizeof(real) == 4 ? 1.0 / (2 * M_PI) : 1.0));
  p->inv_nsteps = (real)(1.0 / c.solver_nsteps);
  p->motor_kind = c.motor_kind;
  p->conv_kind[0] = c.converter_kind[0]; p->conv_kind[1] = c.converter_kind[1];
  p->load_kind = c.load_kind; p->solver_kind = c.solver_kind; p->nsteps = c.solver_nsteps;
  p->autoreset = c.autoreset;
  p->two_segment = h->two_segment;
  const double til0 = c.interlocking_time, til1 = c.interlocking_time1 < 0 ? c.interlocking_time : c.interlocking_time1;
  p->tau = (real)c.tau;
  p->til2[0] = (real)til0; p->til2[1] = (real)til1;
  p->tot2[0] = (real)(til0 / c.tau); p->tot2[1] = (real)(til1 / c.tau);
  p->lo_slot = til1 < til0 ? 1 : 0;
  p->promote = std::fabs(til1 - til0) - c.tau / 1000 > 0;  // t_hi - tau/1000 > t_start + t_lo (converters.py:273)
  const double hs[6] = {c.tau, til0, c.tau - til0, til1, c.tau - til1, std::fabs(til1 - til0)};
  for (int q = 0; q < 6; ++q) p->seg_len[q] = (real)hs[q];
  p->u_sup = (real)c.u_sup;
  {  // angle increment factors (see StepParams::kang) for every segment length of seg_len
    const double pp = c.motor_param[GEMB200_MP_P];
    const double unit = sizeof(real) == 4 ? 1.0 / (2 * M_PI) : 1.0;  // fp32 build keeps the angle in turns
    for (int sidx = 0; sidx < 6; ++sidx) {
      const double k_tot = pp * hs[sidx] * unit;
      const double k_sub = pp * (hs[sidx] / c.solver_nsteps) * (c.solver_kind == GEMB200_SOLVER_RK4 ? 1.0 / 6.0 : 1.0) * unit;
      const double ks[2] = {k_tot, k_sub};
      for (int m = 0; m < 2; ++m) {
        p->kang[m][sidx][0] = (real)ks[m];
        p->kang[m][sidx][1] = (real)(ks[m] - (double)p->kang[m][sidx][0]);
      }
    }
  }
  for (int j = 0; j < 20; ++j) p->k.c[j] = (real)dv.c[j];
  for (int j = 0; j < 4; ++j) p->k.tq[j] = (real)dv.tq[j];
  p->k.load_a = (real)c.load_param[GEMB200_LP_A]; p->k.load_b = (real)c.load_param[GEMB200_LP_B]; p->k.load_c = (real)c.load_param[GEMB200_LP_C];
  p->k.inv_j = (real)dv.inv_j; p->k.omega_lim = (real)dv.omega_lim; p->k.omega_lin = (real)dv.omega_lin;
  for (int j = 0; j < dm.n_state; ++j) {
    p->inv_lim[j] = c.limits[j] != 0.0 ? (real)(1.0 / c.limits[j]) : real(0);
    p->reset_obs[j] = (real)dv.reset_obs[j];
  }
  for (int j = 0; j < dm.nx; ++j) p->init_x[j] = (real)c.init_ode[j];
  if (dm.has_eps) {
    double e = c.init_ode[dm.nx];
    e = e - 2 * M_PI * std::rint(e / (2 * M_PI));
    if (e <= -M_PI) e += 2 * M_PI;
    const int eps_idx = dm.n_state - 2;  // [..., epsilon, u_sup]
    if (sizeof(real) == 4) {
      const double t = e / (2 * M_PI);
      p->init_ang[0] = (real)t; p->init_ang[1] = (real)(t - (double)p->init_ang[0]);
      p->eps_out_scale = (real)(2 * M_PI / c.limits[eps_idx]);
    } else {
      p->init_ang[0] = (real)e; p->init_ang[1] = real(0);
      p->eps_out_scale = (real)(1.0 / c.limits[eps_idx]);
    }
    p->inv_lim[eps_idx] = real(1);  // the angle entry is already normalised by eps_out_scale
  }
  p->init_random = c.init_random;
  p->init_im_valid = c.init_im_valid;
  for (int j = 0; j < 8; ++j) p->init_im[j] = (real)c.init_im[j];
  p->im_prev = static_cast<real*>(h->d_imprev);
  {  // truncated-normal states: CDF bounds prepared in double; the angle entry is converted to the stored unit like init_lo
    const int nst = dm.nx + (dm.has_eps ? 1 : 0);
    for (int j = 0; j < nst; ++j) {
      if (!c.init_random || !c.init_dist[j]) continue;
      const double unit = (j == dm.nx && sizeof(real) == 4) ? 1.0 / (2 * M_PI) : 1.0;
      p->init_mid[j] = std::isnan(c.init_mu[j]);  // mue = middle of the (possibly per-env) interval
      const double mu = p->init_mid[j] ? 0.5 * (c.init_hi[j] - c.init_lo[j]) + c.init_lo[j] : c.init_mu[j], sg = c.init_sigma[j];
      const double ca = 0.5 * std::erfc(-(c.init_lo[j] - mu) / sg * M_SQRT1_2), cb = 0.5 * std::erfc(-(c.init_hi[j] - mu) / sg * M_SQRT1_2);
      p->init_gauss = 1; p->init_dist[j] = 1;
      p->init_mu[j] = (real)(mu * unit); p->init_sigma[j] = (real)(sg * unit);
      p->init_ca[j] = (real)ca; p->init_cspan[j] = (real)(cb - ca);
    }
  }
  for (int j = 0; j < dm.nx; ++j) { p->init_lo[j] = (real)c.init_lo[j]; p->init_span[j] = (real)(c.init_hi[j] - c.init_lo[j]); }
  if (dm.has_eps) {
    const double unit = sizeof(real) == 4 ? 1.0 / (2 * M_PI) : 1.0;
    p->init_lo[dm.nx] = (real)(c.init_lo[dm.nx] * unit); p->init_span[dm.nx] = (real)((c.init_hi[dm.nx] - c.init_lo[dm.nx]) * unit);
  }
  for (int i = 0; i < c.n_constraints; ++i) {
    if (c.constraint_kind[i] == GEMB200_CONSTRAINT_SQUARED) {
      int cnt = 0;
      for (int j = 0; j < dm.n_obs; ++j) if ((c.constraint_mask[i] >> j) & 1u) p->sq_idx[p->n_sq][cnt++] = j;
      p->sq_cnt[p->n_sq++] = cnt;
    } else {
      for (int j = 0; j < dm.n_obs; ++j) {
        if (!((c.constraint_mask[i] >> j) & 1u)) continue;
        bool seen = false;
        for (int q = 0; q < p->n_lim; ++q) seen = seen || p->lim_idx[q] == j;
        if (!seen) p->lim_idx[p->n_lim++] = j;
      }
    }
  }
  // WeightedSumOfErrors: only non-zero weights become terms (weighted_sum_of_errors.py:128-129)
  int t = 0;
  for (int j = 0; j < dm.n_obs; ++j) {
    if (c.reward_weight[j] == 0.0) continue;
    int slot = -1;
    for (int r = 0; r < c.n_ref; ++r) if (c.ref_state[r] == j) slot = r;  // the last generator of a state wins (multiple_reference_generator.py:70-78)
    if (slot >= 0) {
      p->rwr_w[slot] = (real)c.reward_weight[j];
      p->rwr_inv_len[slot] = (real)(1.0 / c.state_length[j]);
      p->rwr_pow[slot] = (real)c.reward_power[j];
      p->rwr_pow1[slot] = c.reward_power[j] == 1.0;
      continue;
    }
    p->rw_state[t] = j;
    p->rw_w[t] = (real)c.reward_weight[j];
    p->rw_inv_len[t] = (real)(1.0 / c.state_length[j]);
    p->rw_pow[t] = (real)c.reward_power[j];
    p->rw_pow1[t] = c.reward_power[j] == 1.0;
    ++t;
  }
  p->n_rw = t;
  for (int r = 0; r < kMaxRef; ++r) if (p->rwr_w[r] == real(0)) p->rwr_pow1[r] = 1;  // unused slots: no pow()
  p->bias = (real)c.reward_bias; p->viol_reward = (real)c.violation_reward;
  // PLAIN shape (step_kernel): decided here once; GEMB200_NO_PLAIN=1 in the environment forces the general instantiation (A/B runs)
  bool plain_shape;
  {
    bool plain =
                 c.load_kind != GEMB200_LOAD_EXT_SPEED && c.supply_kind == GEMB200_SUPPLY_IDEAL && (c.finite || (c.interlocking_time == 0.0 && !(c.interlocking_time1 > 0.0))) && c.dead_time_steps == 0 && !c.action_dq && c.n_state_ops == 0 &&
                 c.converter_kind[0] != GEMB200_CONV_1QC && c.converter_kind[1] != GEMB200_CONV_1QC &&
                 p->n_rw == 0 && p->n_lim <= 2 && p->n_sq <= 1 && (p->n_sq == 0 || p->sq_cnt[0] == 2);
    for (int r = 0; r < c.n_ref; ++r) plain = plain && c.ref_kind[r] == GEMB200_REF_WIENER && p->rwr_pow1[r] && c.ref_sw_count[r] <= 1;
    // PLAIN monitor, branch-free: word offsets of the (at most) two limit-checked states and the two states of the squared constraint in the
    // staged row; an unused check compares entry 0 with +inf
    const real inf = std::numeric_limits<real>::infinity();
    for (int q = 0; q < 2; ++q) { p->mon_off[q] = p->n_lim > q ? p->lim_idx[q] * (int)sizeof(real) : 0; p->mon_thr[q] = p->n_lim > q ? real(1) : inf; }
    for (int q = 0; q < 2; ++q) p->mon_off[2 + q] = (p->n_sq > 0 && p->sq_cnt[0] == 2) ? p->sq_idx[0][q] * (int)sizeof(real) : 0;
    p->mon_thr[2] = p->n_sq > 0 ? real(1) : inf;
    const char* off = std::getenv("GEMB200_NO_PLAIN");
    plain_shape = plain && !(off && off[0] == '1');
  }
  {  // L2 prefetch distance: one wave of resident threads (SMs x blocks/SM x block size); GEMB200_PF_DIST overrides (0 = off)
    int sms = 132;  // H100 SXM; the attribute query below gives the real count
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c.device);
    p->pf_dist = sms * 4 * GEMB200_BLOCK;  // one wave of 4 blocks per SM
    if (const char* e = std::getenv("GEMB200_PF_DIST")) p->pf_dist = std::atoi(e);
  }
  p->ext_tab = static_cast<const real*>(h->d_ext);
  p->ext_len = c.ext_speed_len;
  p->ext_inv_tau = c.load_kind == GEMB200_LOAD_EXT_SPEED ? (real)(1.0 / c.load_param[GEMB200_LP_TAU_LOAD]) : real(0);
  p->kenv = h->d_kenv;
  p->supply_kind = c.supply_kind;
  p->sup = static_cast<real*>(h->d_sup);
  p->sup_k1 = c.supply_kind == GEMB200_SUPPLY_RC ? (real)(c.tau / (c.supply_param[0] * c.supply_param[1])) : real(0);
  p->sup_k2 = (real)c.supply_param[0];
  p->sup_phase = h->d_supph;
  if (c.supply_kind == GEMB200_SUPPLY_AC1) {
    const double unit = sizeof(real) == 4 ? 1.0 / (2 * M_PI) : 1.0;  // fp32 build: turns as double-float
    const double kph = 2 * M_PI * c.supply_param[0] * c.tau * unit;
    double ph0 = c.supply_param[1];
    ph0 = ph0 - 2 * M_PI * std::rint(ph0 / (2 * M_PI));
    ph0 *= unit;
    p->sup_amp = (real)(std::sqrt(2.0) * c.u_sup);
    p->sup_kph[0] = (real)kph; p->sup_kph[1] = sizeof(real) == 4 ? (real)(kph - (double)p->sup_kph[0]) : real(0);
    p->sup_ph0[0] = (real)ph0; p->sup_ph0[1] = sizeof(real) == 4 ? (real)(ph0 - (double)p->sup_ph0[0]) : real(0);
    p->sup_fixed = c.supply_param[2] != 0.0;
  }
  for (int j = 0; j < dm.n_state; ++j) p->reset_obs_du[j] = (real)dv.reset_obs_du[j];
  p->n_sops = c.n_state_ops;
  p->n_obs = dm.n_obs;
  p->row_stride = h->row_stride;
  p->obsv = static_cast<real*>(h->d_obsv);
  for (int k = 0; k < c.n_state_ops; ++k) {
    p->sop_kind[k] = c.sop_kind[k];
    p->sop_mask[k] = c.sop_mask[k];
    for (int q = 0; q < 4; ++q) p->sop_idx[k][q] = c.sop_idx[k][q];
    for (int q = 0; q < 8; ++q) p->sop_param[k][q] = (real)c.sop_param[k][q];
  }
  p->n_ref = c.n_ref;
  p->swst = h->d_swst;
  for (int r = 0; r < c.n_ref; ++r) {
    p->sw_count[r] = c.ref_sw_count[r] > 1 ? c.ref_sw_count[r] : 0;
    p->sw_first[r] = c.ref_sw_first[r];
    p->sw_len_lo[r] = c.ref_sw_len_lo[r]; p->sw_len_span[r] = c.ref_sw_len_hi[r] - c.ref_sw_len_lo[r];
  }
  for (int r = 0; r < GEMB200_MAX_REF_ENTRIES; ++r) p->sw_cdf[r] = (real)c.ref_sw_cdf[r];
  p->any_wiener = h->any_wiener;
  p->ref_tau = (real)c.tau;
  p->ref_tau_d = c.tau;
  for (int r = 0; r < GEMB200_MAX_REF_ENTRIES; ++r) {  // all parameter entries (switched sub-generators live beyond n_ref)
    p->ref_kind[r] = c.ref_kind[r]; p->ref_state[r] = c.ref_state[r];
    p->ref_const[r] = (real)c.ref_value[r];
    p->ref_lo[r] = (real)c.ref_margin_lo[r]; p->ref_hi[r] = (real)c.ref_margin_hi[r];
    p->ref_init_lo[r] = (real)c.ref_init_lo[r]; p->ref_init_span[r] = (real)(c.ref_init_hi[r] - c.ref_init_lo[r]);
    p->ref_amp_lo[r] = (real)c.ref_amp_lo[r]; p->ref_amp_span[r] = (real)(c.ref_amp_hi[r] - c.ref_amp_lo[r]);
    p->ref_freq_lo[r] = (real)c.ref_freq_lo[r]; p->ref_freq_span[r] = (real)(c.ref_freq_hi[r] - c.ref_freq_lo[r]);
    p->ref_freq_lo_d[r] = c.ref_freq_lo[r]; p->ref_freq_span_d[r] = c.ref_freq_hi[r] - c.ref_freq_lo[r];
    p->ref_off_lo[r] = (real)c.ref_off_lo[r]; p->ref_off_hi[r] = (real)c.ref_off_hi[r];
    if (c.ref_kind[r] == GEMB200_REF_WIENER || c.ref_kind[r] == GEMB200_REF_LAPLACE) {
      p->ref_lsig_lo[r] = (real)std::log10(c.ref_sigma_lo[r]);
      p->ref_lsig_span[r] = (real)(std::log10(c.ref_sigma_hi[r]) - std::log10(c.ref_sigma_lo[r]));
    }
    p->ref_len_lo[r] = c.ref_len_lo[r]; p->ref_len_span[r] = c.ref_len_hi[r] - c.ref_len_lo[r];
  }
  return plain_shape;
}

// ----------------------------------------------------------------------------------------------------------------
// kernel dispatch (the instantiations live in gemb200_step_tu.cu and gemb200_tangent_tu.cu, one TU per family x real and kind)
// ----------------------------------------------------------------------------------------------------------------
// launch(std::integral_constant<int, FAM>{}) for motor family fam.  GEMB200_ONLY_FAM=<family>: experiment builds (tools/build_variants.py
// --only) that carry the fp32 step and reset kernels of ONE motor family and no tangent kernels (TANGENT: a tangent-rollout launch); every
// other launch fails with cudaErrorInvalidValue instead of leaving unresolved symbols.  Never defined in the product build.
template <bool TANGENT, typename real, typename L>
static cudaError_t for_family(int fam, L&& launch) {
#ifdef GEMB200_ONLY_FAM
  if constexpr (!TANGENT && std::is_same<real, float>::value) { if (fam == GEMB200_ONLY_FAM) return launch(std::integral_constant<int, GEMB200_ONLY_FAM>{}); }
  return cudaErrorInvalidValue;
#else
  switch (fam) {
    case kDC1: return launch(std::integral_constant<int, kDC1>{});
    case kDC2: return launch(std::integral_constant<int, kDC2>{});
    case kSYNC: return launch(std::integral_constant<int, kSYNC>{});
    case kEESM: return launch(std::integral_constant<int, kEESM>{});
    case kSCIM: return launch(std::integral_constant<int, kSCIM>{});
    case kDFIM: return launch(std::integral_constant<int, kDFIM>{});
  }
  return cudaErrorInvalidValue;
#endif
}

template <typename real>
static void set_roll_strides(const gemb200_handle* h, StepParams<real>& p) {
  const int64_t n = h->cfg.n_envs;
  p.out_has = (p.obs ? 1 : 0) | ((p.ref_out && h->n_ref > 0) ? 2 : 0) | (p.reward ? 4 : 0) | (p.term ? 8 : 0);
  p.roll_act_inc = n * h->n_act * (int64_t)(h->cfg.finite ? sizeof(int32_t) : sizeof(real));
  p.roll_obs_inc = p.obs ? n * h->n_obs * (int64_t)sizeof(real) : 0;
  p.roll_ref_inc = p.ref_out ? n * h->n_ref * (int64_t)sizeof(real) : 0;
  p.roll_rew_inc = p.reward ? n * (int64_t)sizeof(real) : 0;
  p.roll_term_inc = p.term ? n : 0;
}

// ---- device-resident clock: the call id of the NEXT call, the step count and the dead-time ring position live in device memory and are
// advanced by a one-thread kernel behind every launch, so that a launch depends on nothing the host changes between calls (CUDA graphs)
__global__ void clock_tick_kernel(uint32_t* c, uint32_t d_call, uint32_t d_step, uint32_t dead_steps) {
  const uint64_t g = (((uint64_t)c[1] << 32) | c[0]) + d_call, s = (((uint64_t)c[4] << 32) | c[2]) + d_step;
  c[0] = (uint32_t)g; c[1] = (uint32_t)(g >> 32); c[2] = (uint32_t)s; c[4] = (uint32_t)(s >> 32);
  c[3] = dead_steps ? (uint32_t)(s % dead_steps) : 0u;
}
static int push_clock(gemb200_handle* h, cudaStream_t st) {  // host counters -> device (stream-ordered; the source is a by-value kernel argument)
  const uint64_t g1 = h->gstep + 1, s = h->n_steps;
  const uint32_t dead = (uint32_t)h->cfg.dead_time_steps;
  const uint32_t v[8] = {(uint32_t)g1, (uint32_t)(g1 >> 32), (uint32_t)s, dead ? (uint32_t)(s % dead) : 0u, (uint32_t)(s >> 32), 0u, 0u, 0u};
  CUDA_TRY(cudaMemcpyAsync(h->d_clock, v, sizeof(v), cudaMemcpyHostToDevice, st));  // pageable source: staged before the call returns
  return GEMB200_OK;
}
static int pull_clock(gemb200_handle* h, cudaStream_t st) {  // device -> host counters (synchronises the stream)
  uint32_t v[8];
  CUDA_TRY(cudaMemcpyAsync(v, h->d_clock, sizeof(v), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  h->gstep = ((((uint64_t)v[1]) << 32) | v[0]) - 1;
  h->n_steps = (((uint64_t)v[4]) << 32) | v[2];
  return GEMB200_OK;
}
static int tick_clock(gemb200_handle* h, uint32_t d_call, uint32_t d_step, cudaStream_t st) {
  clock_tick_kernel<<<1, 1, 0, st>>>(h->d_clock, d_call, d_step, (uint32_t)h->cfg.dead_time_steps);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return GEMB200_OK;
}

// One launch over envs [begin, end) (end < 0: all).  new_call: this launch starts a new API call (fresh RNG call ids);
// the chunks of one pipelined host step share them.  roll > 0: `roll` fused steps (rollout_kernel) whose call ids, step clock and
// dead-time ring positions are exactly those of `roll` consecutive single-step calls; outputs every `every` steps (0: last only).
// feed: the reference values of every step (StepParams::ref_feed), or NULL.  ret / ret_end / discount: the discounted returns of a
// rollout (StepParams::ret_out), or NULL.  tan: the outputs of a tangent rollout (JacOut: gemb200_rollout_jacobians, GradOut:
// gemb200_rollout_return_grads, PsOut: gemb200_rollout_param_sens), or NULL; with them the launch takes that kind's kernel
// (gemb200_tangent.cuh) instead of the step / rollout kernels.
template <typename TanOut = void>
static int do_step(gemb200_handle* h, const void* action, void* obs, void* ref, void* rew, uint8_t* term, cudaStream_t st,
                   int begin = 0, int end = -1, bool new_call = true, int roll = 0, int every = 0, const void* feed = nullptr,
                   void* ret = nullptr, int32_t* ret_end = nullptr, double discount = 1.0, const TanOut* tan = nullptr) {
  if (!action) return fail(GEMB200_E_INVALID, "action is NULL");
  const uint64_t ksteps = roll > 0 ? (uint64_t)roll : 1;
  const bool dev_clock = h->dev_clock;
  if (dev_clock && (!new_call || begin != 0 || (end >= 0 && end != h->cfg.n_envs)))
    return fail(GEMB200_E_INVALID, "the host-buffer step is not available while the device-resident clock is enabled");
  if (new_call && !dev_clock) { h->gstep += ksteps; h->n_steps += ksteps; }
  const uint64_t g0 = h->gstep - (ksteps - 1), n0 = h->n_steps - (ksteps - 1);  // call id / step count of the FIRST step of this launch
  if (end < 0) end = h->cfg.n_envs;
  const int fifo_slot = h->cfg.dead_time_steps > 0 ? (int)((n0 - 1) % (uint64_t)h->cfg.dead_time_steps) : 0;
  const cudaError_t e = with_params(h, [&](auto& p) {
    using real = decltype(p.tau);
    p.env_begin = begin; p.env_end = end; p.fifo_slot = fifo_slot; p.kstep = dev_clock ? 1u : (uint32_t)n0;
    p.gstep_lo = (uint32_t)g0; p.gstep_hi = (uint32_t)(g0 >> 32); p.clock_dev = dev_clock ? h->d_clock : nullptr;
    p.roll_steps = roll; p.record_every = every;
    p.action = action; p.obs = (real*)obs; p.ref_out = (real*)ref; p.reward = (real*)rew; p.term = term;
    p.ref_feed = static_cast<const real*>(feed);
    p.ret_out = static_cast<real*>(ret); p.ret_end = ret_end; p.discount = (real)discount;
    set_roll_strides(h, p);
    const bool finite = h->cfg.finite != 0;
    if constexpr (!std::is_void<TanOut>::value) {
      if (tan) return for_family<true, real>(h->fam, [&](auto f) { return launch_tangent_f<decltype(f)::value, real>(finite, h->n_ref, p, *tan, st); });
    }
    return for_family<false, real>(h->fam, [&](auto f) { return launch_step_f<decltype(f)::value, real>(finite, h->n_ref, p, st); });
  });
  if (e != cudaSuccess) return fail(GEMB200_E_CUDA, std::string(roll > 0 ? "rollout launch: " : "step launch: ") + cudaGetErrorString(e));
  h->launches += 1;
  // (the alternative is to advance the clock from the step kernel itself — its last block to finish, one atomic per block; at N = 65 536 the
  // grid has 2048 small blocks that would each pay that atomic, so the tick is a separate one-thread node)
  if (dev_clock) return tick_clock(h, (uint32_t)ksteps, (uint32_t)ksteps, st);
  return GEMB200_OK;
}

static int do_reset(gemb200_handle* h, const uint8_t* mask, void* obs, void* ref, cudaStream_t st) {
  const bool dev_clock = h->dev_clock;
  if (!dev_clock) h->gstep += 1;
  const cudaError_t e = with_params(h, [&](auto& p) {
    using real = decltype(p.tau);
    p.clock_dev = dev_clock ? h->d_clock : nullptr;
    p.gstep_lo = (uint32_t)h->gstep; p.gstep_hi = (uint32_t)(h->gstep >> 32);
    p.reset_mask = mask; p.obs = (real*)obs; p.ref_out = (real*)ref; p.kstep = dev_clock ? 0u : (uint32_t)h->n_steps;
    const cudaError_t le = for_family<false, real>(h->fam, [&](auto f) { return launch_reset_f<decltype(f)::value, real>(h->n_ref, p, st); });
    p.reset_mask = nullptr;
    return le;
  });
  if (e != cudaSuccess) return fail(GEMB200_E_CUDA, std::string("reset launch: ") + cudaGetErrorString(e));
  h->launches += 1;
  if (dev_clock) return tick_clock(h, 1u, 0u, st);
  return GEMB200_OK;
}

// induction motors: before the first reset the "previous" initial currents are the constant ones (_initial_states of a fresh motor)
static int fill_imprev(gemb200_handle* h, cudaStream_t st) {
  if (!h->d_imprev) return GEMB200_OK;
  const size_t n = (size_t)h->cfg.n_envs;
  return with_params(h, [&](auto& p) {
    using real = decltype(p.tau);
    std::vector<real> v(2 * n);
    for (size_t q = 0; q < n; ++q) { v[q] = (real)h->cfg.init_ode[1]; v[n + q] = (real)h->cfg.init_ode[2]; }
    CUDA_TRY(cudaMemcpyAsync(h->d_imprev, v.data(), v.size() * sizeof(real), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return GEMB200_OK;
  });
}

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// one launch of an ODE-state / reference accessor kernel over every env: launch(live StepParams, n, grid, stream)
template <typename F>
static int launch_accessor(gemb200_handle* h, void* stream, F&& launch) {
  DeviceGuard guard(h->cfg.device);
  const int n = h->cfg.n_envs, grid = (n + 255) / 256;
  with_params(h, [&](auto& p) { launch(p, n, grid, (cudaStream_t)stream); });
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return GEMB200_OK;
}

// ----------------------------------------------------------------------------------------------------------------
// C-ABI
// ----------------------------------------------------------------------------------------------------------------
// The checks the rollout entry points share, behind the handle check and each entry's own checks, in the order they fail: n_steps, then
// the entry's check that must fail right after it (`after_n_steps`: its message when it fails, else NULL; record_every reads n_steps), then
// the reference feed
static int check_rollout(const gemb200_handle* h, int32_t n_steps, const void* references, const char* after_n_steps = nullptr) {
  if (n_steps < 1 || n_steps > (1 << 24)) return fail(GEMB200_E_INVALID, "n_steps must be in [1, 2^24]");
  if (after_n_steps) return fail(GEMB200_E_INVALID, after_n_steps);
  if (references && h->n_ref == 0) return fail(GEMB200_E_INVALID, "a reference feed needs a configuration with reference slots (n_ref > 0)");
  return GEMB200_OK;
}
static const char* check_discount(double discount) { return discount >= 0.0 && discount <= 1.0 ? nullptr : "discount must be finite and in [0, 1]"; }

extern "C" {

int gemb200_version(void) { return GEMB200_ABI_VERSION; }
const char* gemb200_last_error(void) { return g_last_error.c_str(); }

int gemb200_config_init(gemb200_config* cfg) {
  if (!cfg) return fail(GEMB200_E_INVALID, "config is NULL");
  std::memset(cfg, 0, sizeof(*cfg));
  cfg->struct_size = (int32_t)sizeof(gemb200_config);
  cfg->abi_version = GEMB200_ABI_VERSION;
  cfg->n_envs = 1;
  cfg->solver_kind = GEMB200_SOLVER_RK4;
  cfg->solver_nsteps = 1;
  cfg->tau = 1e-4;
  cfg->load_param[GEMB200_LP_TAU_DECAY] = 1e-3;
  cfg->interlocking_time1 = -1.0;
  for (int i = 0; i < GEMB200_MAX_STATE; ++i) { cfg->limits[i] = 1.0; cfg->state_length[i] = 2.0; cfg->reward_power[i] = 1.0; }
  for (int r = 0; r < GEMB200_MAX_REF_ENTRIES; ++r) {
    cfg->ref_len_lo[r] = 500; cfg->ref_len_hi[r] = 2000;
    cfg->ref_sigma_lo[r] = 1e-3; cfg->ref_sigma_hi[r] = 1e-1;
    cfg->ref_margin_lo[r] = -1; cfg->ref_margin_hi[r] = 1; cfg->ref_init_lo[r] = -1; cfg->ref_init_hi[r] = 1;
  }
  return GEMB200_OK;
}

int gemb200_query_dims(const gemb200_config* cfg, int32_t* n_state, int32_t* n_ode, int32_t* n_act, int32_t* n_ref) {
  if (!cfg) return fail(GEMB200_E_INVALID, "config is NULL");
  Dims d;
  int rc = derive_dims(cfg, &d);
  if (rc) return rc;
  if (n_state) *n_state = d.n_obs;
  if (n_ode) *n_ode = d.n_ode;
  if (n_act) *n_act = d.n_act;
  if (n_ref) *n_ref = cfg->n_ref;
  return GEMB200_OK;
}

// Configurations whose rollout Jacobians the library does not compute (DESIGN.md §7, "Rollout Jacobians"): the reason, or nullptr
static const char* jacobian_refusal(const gemb200_config* c) {
  if (c->dead_time_steps > 0) return "rollout Jacobians: a dead time is refused, the action enters through the queue, which is not part of the ODE state (DESIGN.md §7)";
  if (c->supply_kind == GEMB200_SUPPLY_RC) return "rollout Jacobians: the RC supply is refused, its state couples through i_sup and is not part of the ODE state (DESIGN.md §7)";
  if (c->action_dq == 2 || c->action_dq == 3)
    return "rollout Jacobians: dq actions on the FluxObserver angle are refused, the control path reads an observer state that is not part of the ODE state (DESIGN.md §7)";
  if (c->layout == GEMB200_LAYOUT_SOA) return "rollout Jacobians: the SoA layout is refused, the launch writes row-per-env outputs only (DESIGN.md §7)";
  return nullptr;
}

int gemb200_query_jacobian_dims(const gemb200_config* cfg, int32_t* n_x, int32_t* n_u) {
  if (!cfg) return fail(GEMB200_E_INVALID, "config is NULL");
  Dims d;
  int rc = derive_dims(cfg, &d);
  if (rc) return rc;
  if (const char* why = jacobian_refusal(cfg)) return fail(GEMB200_E_INVALID, why);
  if (n_x) *n_x = d.n_ode;
  if (n_u) *n_u = cfg->finite ? 0 : d.n_act;
  return GEMB200_OK;
}

// The entry of the family's state vector (before the wrappers) behind each entry of the observation row, or -1 for an entry a wrapper
// appends (CosSin, FluxObserver, CurrentSum); returns the row width
static int row_bases(const gemb200_config* c, int n_state, int8_t (&base)[GEMB200_MAX_STATE]) {
  int w = n_state;
  for (int j = 0; j < GEMB200_MAX_STATE; ++j) base[j] = j < n_state ? (int8_t)j : (int8_t)-1;
  for (int k = 0; k < c->n_state_ops; ++k) {
    switch (c->sop_kind[k]) {
      case GEMB200_SOP_COS_SIN:
        if (c->sop_idx[k][1]) { for (int j = c->sop_idx[k][0]; j < w - 1; ++j) base[j] = base[j + 1]; --w; }  // remove_angle
        base[w] = base[w + 1] = -1;
        w += 2;
        break;
      case GEMB200_SOP_FLUX_OBSERVER: base[w] = base[w + 1] = -1; w += 2; break;
      case GEMB200_SOP_CURRENT_SUM: base[w] = -1; w += 1; break;
      default: break;  // state noise: additive, the entry keeps its base
    }
  }
  return w;
}

// Configurations whose return gradients the library does not compute (DESIGN.md §7, "Return gradients"): the reason, or nullptr.
// Call after derive_dims succeeded.
static const char* return_grad_refusal(const gemb200_config* c, const Dims& d) {
  if (const char* why = jacobian_refusal(c)) return why;
  if (c->finite) return "return gradients: finite converters are refused, their actions are integers without a derivative (DESIGN.md §7)";
  int8_t base[GEMB200_MAX_STATE];
  const int w = row_bases(c, d.n_state, base);
  for (int j = 0; j < w; ++j)
    if (c->reward_weight[j] != 0.0 && base[j] < 0)
      return "return gradients: the reward weights an entry a state wrapper appends (CosSin, FluxObserver, CurrentSum), which is not a function of the ODE state in the tangent pass (DESIGN.md §7)";
  return nullptr;
}

int gemb200_query_return_grad_dims(const gemb200_config* cfg, int32_t* n_x, int32_t* n_u, int32_t* ws_words) {
  if (!cfg) return fail(GEMB200_E_INVALID, "config is NULL");
  Dims d;
  int rc = derive_dims(cfg, &d);
  if (rc) return rc;
  if (const char* why = return_grad_refusal(cfg, d)) return fail(GEMB200_E_INVALID, why);
  if (n_x) *n_x = d.n_ode;
  if (n_u) *n_u = d.n_act;
  if (ws_words) *ws_words = d.n_ode * (d.n_ode + d.n_act) + d.n_ode + d.n_act;
  return GEMB200_OK;
}

// Parameter sensitivities (DESIGN.md §7, "Parameter sensitivities"): the reason a configuration or a list of parameter slots is refused,
// or nullptr.  Accepted: every motor slot but the pole pairs and the EESM's k, and the load slots a, b, c, j_load.
static const char* param_sens_refusal(const gemb200_config* c, int32_t n_p, const int32_t* slots) {
  if (const char* why = jacobian_refusal(c)) return why;
  if (n_p < 1 || n_p > kMaxSensParams) return "parameter sensitivities: n_p must be in [1, 12] (DESIGN.md §7)";
  if (!slots) return "parameter sensitivities: slots is NULL";
  for (int a = 0; a < n_p; ++a) {
    const int s = slots[a];
    const bool motor = s >= 0 && s < GEMB200_MAX_MOTOR_PARAM;
    const int l = s - GEMB200_MAX_MOTOR_PARAM;
    if (!motor && !(l == GEMB200_LP_A || l == GEMB200_LP_B || l == GEMB200_LP_C || l == GEMB200_LP_J_LOAD))
      return "parameter sensitivities: a slot is neither a motor slot nor one of the load slots a, b, c, j_load (DESIGN.md §7)";
    if (s == GEMB200_MP_P) return "parameter sensitivities: the pole pairs are refused, the angle increments are prepared per handle (DESIGN.md §7)";
    if (s == GEMB200_MP_K) return "parameter sensitivities: the EESM's k is refused, the model coefficients are invariant in it (DESIGN.md §7)";
    for (int b = 0; b < a; ++b)
      if (slots[b] == s) return "parameter sensitivities: duplicate slot (DESIGN.md §7)";
  }
  return nullptr;
}

int gemb200_query_param_sens_dims(const gemb200_config* cfg, int32_t n_p, const int32_t* slots, int32_t* n_x) {
  if (!cfg) return fail(GEMB200_E_INVALID, "config is NULL");
  Dims d;
  int rc = derive_dims(cfg, &d);
  if (rc) return rc;
  if (const char* why = param_sens_refusal(cfg, n_p, slots)) return fail(GEMB200_E_INVALID, why);
  if (n_x) *n_x = d.n_ode;
  return GEMB200_OK;
}

int gemb200_coef_tangents(const gemb200_config* cfg, const double* motor_param, const double* load_param, int32_t n_p, const int32_t* slots, double* out) {
  if (!cfg) return fail(GEMB200_E_INVALID, "config is NULL");
  if (!out) return fail(GEMB200_E_INVALID, "out is NULL");
  Dims d;
  int rc = derive_dims(cfg, &d);
  if (rc) return rc;
  if (const char* why = param_sens_refusal(cfg, n_p, slots)) return fail(GEMB200_E_INVALID, why);
  double prm[kMaxDraw];
  for (int s = 0; s < GEMB200_MAX_MOTOR_PARAM; ++s) prm[s] = motor_param ? motor_param[s] : cfg->motor_param[s];
  for (int s = 0; s < 8; ++s) prm[GEMB200_MAX_MOTOR_PARAM + s] = load_param ? load_param[s] : cfg->load_param[s];
  for (int a = 0; a < n_p; ++a) coef_tangent(cfg->motor_kind, prm, slots[a], out + (size_t)a * kCoefWords);
  return GEMB200_OK;
}

int gemb200_create(const gemb200_config* cfg, gemb200_handle** out) {
  if (!out) return fail(GEMB200_E_INVALID, "out is NULL");
  *out = nullptr;
  int rc = validate(cfg);
  if (rc) return rc;
  int ndev = 0;
  CUDA_TRY(cudaGetDeviceCount(&ndev));
  if (cfg->device < 0 || cfg->device >= ndev) return fail(GEMB200_E_INVALID, "device ordinal out of range");
  DeviceGuard guard(cfg->device);
  gemb200_handle* h = new (std::nothrow) gemb200_handle();
  if (!h) return fail(GEMB200_E_NOMEM, "out of host memory");
  h->cfg = *cfg;
  Dims d;
  derive_dims(cfg, &d);
  h->fam = d.fam; h->n_state = d.n_state; h->n_ode = d.n_ode; h->n_act = d.n_act; h->nx = d.nx; h->has_eps = d.has_eps;
  h->n_obs = d.n_obs;
  h->row_stride = cfg->n_state_ops > 0 ? (d.n_obs | 1) : (d.fam == kEESM ? 17 : (d.fam == kDFIM ? 25 : d.n_state));  // Fam<>::PAD without wrappers
  h->n_ref = cfg->n_ref;
  h->rsz = cfg->dtype == GEMB200_F32 ? 4 : 8;
  h->two_segment = cfg->finite && (cfg->interlocking_time > 0 || cfg->interlocking_time1 > 0);
  for (int r = 0; r < GEMB200_MAX_REF_ENTRIES; ++r) {  // any generator that advances by itself (Wiener, Laplace, periodic), incl. switched subs
    bool used = r < cfg->n_ref;
    for (int q = 0; q < cfg->n_ref; ++q) used = used || (cfg->ref_sw_count[q] > 1 && r >= cfg->ref_sw_first[q] && r < cfg->ref_sw_first[q] + cfg->ref_sw_count[q]);
    if (used) h->any_wiener = h->any_wiener || cfg->ref_kind[r] == GEMB200_REF_WIENER || cfg->ref_kind[r] >= GEMB200_REF_LAPLACE;
  }
  h->NH = hot_words(d.nx, cfg->n_ref); h->NC = cold_words(d.nx, cfg->n_ref);
  h->fifo_dim = fifo_dim_of(cfg, d);
  {  // every per-env array, zero-filled, then the speed-profile table
    Section s[kMaxSections];
    const int k = sections(h, s);
    cudaError_t e = cudaSuccess;
    for (int q = 0; q < k && e == cudaSuccess; ++q)
      if ((e = cudaMalloc(s[q].slot, s[q].bytes)) == cudaSuccess) cudaMemset(*s[q].slot, 0, s[q].bytes);
    if (e == cudaSuccess && cfg->load_kind == GEMB200_LOAD_EXT_SPEED) e = cudaMalloc(&h->d_ext, (size_t)cfg->ext_speed_len * h->rsz);
    if (e != cudaSuccess) { gemb200_destroy(h); return fail(e == cudaErrorMemoryAllocation ? GEMB200_E_NOMEM : GEMB200_E_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e)); }
  }
  if (cfg->load_kind == GEMB200_LOAD_EXT_SPEED) {
    with_params(h, [&](auto& p) {
      using real = decltype(p.tau);
      std::vector<real> tmp(cfg->ext_speed_table, cfg->ext_speed_table + cfg->ext_speed_len);
      cudaMemcpy(h->d_ext, tmp.data(), tmp.size() * sizeof(real), cudaMemcpyHostToDevice);
    });
    {
      uint64_t x = 1469598103934665603ull;
      const unsigned char* tb = reinterpret_cast<const unsigned char*>(cfg->ext_speed_table);
      for (size_t q = 0; q < (size_t)cfg->ext_speed_len * sizeof(double); ++q) { x ^= tb[q]; x *= 1099511628211ull; }
      h->ext_hash = x;
    }
    h->cfg.ext_speed_table = nullptr;  // the caller's buffer is not referenced after create
  }
  Derived dv;
  derive_model(cfg, d, &dv);
  {  // same derivation one volt higher: the difference is the u_sup-proportional part of the reset observation
    gemb200_config c1 = *cfg;
    c1.u_sup += 1.0;
    Derived dv1;
    derive_model(&c1, d, &dv1);
    for (int j = 0; j < d.n_state; ++j) dv.reset_obs_du[j] = dv1.reset_obs[j] - dv.reset_obs[j];
  }
  h->plain_shape = with_params(h, [&](auto& p) { return fill_params(h, d, dv, &p); });
  apply_mode(h);
  cudaEventCreate(&h->ev0);
  cudaEventCreate(&h->ev1);
  rc = fill_imprev(h, nullptr);
  if (rc) { gemb200_destroy(h); return rc; }
  rc = do_reset(h, nullptr, nullptr, nullptr, nullptr);
  if (rc) { gemb200_destroy(h); return rc; }
  cudaError_t e = cudaStreamSynchronize(nullptr);
  if (e != cudaSuccess) { gemb200_destroy(h); return fail(GEMB200_E_CUDA, std::string("initial reset: ") + cudaGetErrorString(e)); }
  *out = h;
  return GEMB200_OK;
}

int gemb200_destroy(gemb200_handle* h) {
  if (!h) return GEMB200_OK;
  DeviceGuard guard(h->cfg.device);
  Section s[kMaxSections];
  for (int q = 0, ns = sections(h, s); q < ns; ++q) cudaFree(*s[q].slot);
  cudaFree(h->d_ext); cudaFree(h->d_envp); cudaFree(h->d_clock); cudaFree(h->d_praw); cudaFree(h->d_draw); cudaFree(h->d_rngid);
  cudaFree(h->d_act); cudaFree(h->d_obs); cudaFree(h->d_ref); cudaFree(h->d_rew); cudaFree(h->d_term); cudaFree(h->d_mask);
  if (h->hstream) cudaStreamDestroy(h->hstream);
  for (int k = 0; k < 3; ++k) if (h->hpipe[k]) cudaStreamDestroy(h->hpipe[k]);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  delete h;
  return GEMB200_OK;
}

int gemb200_reset(gemb200_handle* h, const uint8_t* reset_mask, void* obs_out, void* ref_out, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  DeviceGuard guard(h->cfg.device);
  return do_reset(h, reset_mask, obs_out, ref_out, (cudaStream_t)stream);
}

int gemb200_step(gemb200_handle* h, const void* action, void* obs_out, void* ref_out, void* reward_out, uint8_t* terminated_out, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  DeviceGuard guard(h->cfg.device);
  return do_step(h, action, obs_out, ref_out, reward_out, terminated_out, (cudaStream_t)stream);
}

int gemb200_rollout_record(gemb200_handle* h, const void* actions, int32_t n_steps, int32_t record_every, void* obs_out, void* ref_out,
                           void* reward_out, uint8_t* terminated_out, void* stream) {
  return gemb200_rollout_record_ref(h, actions, nullptr, n_steps, record_every, obs_out, ref_out, reward_out, terminated_out, stream);
}

int gemb200_rollout_record_ref(gemb200_handle* h, const void* actions, const void* references, int32_t n_steps, int32_t record_every,
                               void* obs_out, void* ref_out, void* reward_out, uint8_t* terminated_out, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  const char* every = record_every < 0 || record_every > n_steps ? "record_every must be in [0, n_steps]" : nullptr;
  if (int rc = check_rollout(h, n_steps, references, every)) return rc;
  DeviceGuard guard(h->cfg.device);
  return do_step(h, actions, obs_out, ref_out, reward_out, terminated_out, (cudaStream_t)stream, 0, -1, true, n_steps, record_every, references);
}

int gemb200_rollout_returns(gemb200_handle* h, const void* actions, const void* references, int32_t n_steps, double discount,
                            void* return_out, int32_t* end_step_out, void* obs_out, void* ref_out, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (!return_out) return fail(GEMB200_E_INVALID, "return_out is NULL");
  if (int rc = check_rollout(h, n_steps, references, check_discount(discount))) return rc;
  DeviceGuard guard(h->cfg.device);
  return do_step(h, actions, obs_out, ref_out, nullptr, nullptr, (cudaStream_t)stream, 0, -1, true, n_steps, 0, references, return_out,
                 end_step_out, discount);
}

int gemb200_rollout_jacobians(gemb200_handle* h, const void* actions, const void* references, int32_t n_steps, void* jac_x_out, void* jac_u_out,
                              void* obs_out, void* ref_out, void* reward_out, uint8_t* terminated_out, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (const char* why = jacobian_refusal(&h->cfg)) return fail(GEMB200_E_INVALID, why);
  if (!jac_x_out) return fail(GEMB200_E_INVALID, "jac_x_out is NULL");
  if (int rc = check_rollout(h, n_steps, references)) return rc;
  const JacOut jo{jac_x_out, h->cfg.finite ? nullptr : jac_u_out, h->cfg.finite ? 0 : h->n_act};
  DeviceGuard guard(h->cfg.device);
  return do_step(h, actions, obs_out, ref_out, reward_out, terminated_out, (cudaStream_t)stream, 0, -1, true, n_steps, 1, references, nullptr, nullptr,
                 1.0, &jo);
}

int gemb200_rollout_return_grads(gemb200_handle* h, const void* actions, const void* references, int32_t n_steps, double discount, const void* value_grad,
                                 void* workspace, uint64_t workspace_bytes, void* return_out, int32_t* end_step_out, void* grad_a_out, void* grad_x0_out,
                                 void* obs_out, void* ref_out, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  Dims d;
  derive_dims(&h->cfg, &d);
  if (const char* why = return_grad_refusal(&h->cfg, d)) return fail(GEMB200_E_INVALID, why);
  if (!return_out) return fail(GEMB200_E_INVALID, "return_out is NULL");
  if (!grad_a_out) return fail(GEMB200_E_INVALID, "grad_a_out is NULL");
  if (!grad_x0_out) return fail(GEMB200_E_INVALID, "grad_x0_out is NULL");
  if (!workspace) return fail(GEMB200_E_INVALID, "workspace is NULL");
  if (int rc = check_rollout(h, n_steps, references, check_discount(discount))) return rc;
  const uint64_t words = (uint64_t)(d.n_ode * (d.n_ode + d.n_act) + d.n_ode + d.n_act);
  const uint64_t need = (uint64_t)n_steps * (uint64_t)h->cfg.n_envs * words * (uint64_t)h->rsz;
  if (workspace_bytes < need) return fail(GEMB200_E_INVALID, "workspace too small: it needs n_steps * n_envs * ws_words * sizeof(real) bytes (gemb200_query_return_grad_dims)");
  GradOut go{};
  go.ws = workspace; go.grad_a = grad_a_out; go.grad_x0 = grad_x0_out; go.value_grad = value_grad; go.nu = h->n_act;
  {  // the state-vector entry behind every reward term, in fill_params' order of the terms
    int8_t base[GEMB200_MAX_STATE];
    const int w = row_bases(&h->cfg, d.n_state, base);
    int t = 0;
    for (int j = 0; j < w; ++j) {
      if (h->cfg.reward_weight[j] == 0.0) continue;
      int slot = -1;
      for (int r = 0; r < h->cfg.n_ref; ++r) if (h->cfg.ref_state[r] == j) slot = r;
      if (slot >= 0) go.ref_base[slot] = base[j]; else go.rw_base[t++] = base[j];
      go.wmask |= 1u << base[j];
    }
  }
  DeviceGuard guard(h->cfg.device);
  return do_step(h, actions, obs_out, ref_out, nullptr, nullptr, (cudaStream_t)stream, 0, -1, true, n_steps, 0, references, return_out, end_step_out,
                 discount, &go);
}

int gemb200_rollout_param_sens(gemb200_handle* h, const void* actions, const void* references, int32_t n_steps, int32_t n_p, const int32_t* slots,
                               void* sens_io, void* sens_out, void* obs_out, void* ref_out, void* reward_out, uint8_t* terminated_out, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (const char* why = param_sens_refusal(&h->cfg, n_p, slots)) return fail(GEMB200_E_INVALID, why);
  if (draws_on(h))
    return fail(GEMB200_E_INVALID, "parameter sensitivities: parameter draws at resets are on, the parameters would change inside the launch (DESIGN.md §7)");
  if (!sens_io) return fail(GEMB200_E_INVALID, "sens_io is NULL");
  if (int rc = check_rollout(h, n_steps, references)) return rc;
  PsOut po{};
  po.sio = sens_io; po.sout = sens_out; po.np = n_p;
  for (int a = 0; a < n_p; ++a) po.slot[a] = slots[a];
  for (int s = 0; s < GEMB200_MAX_MOTOR_PARAM; ++s) po.raw[s] = h->cfg.motor_param[s];
  for (int s = 0; s < 8; ++s) po.raw[GEMB200_MAX_MOTOR_PARAM + s] = h->cfg.load_param[s];
  DeviceGuard guard(h->cfg.device);
  return do_step(h, actions, obs_out, ref_out, reward_out, terminated_out, (cudaStream_t)stream, 0, -1, true, n_steps, 1, references, nullptr, nullptr,
                 1.0, &po);
}

int gemb200_rollout(gemb200_handle* h, const void* actions, int32_t n_steps, void* obs_out, void* ref_out, void* reward_out,
                    uint8_t* terminated_out, void* stream) {
  return gemb200_rollout_record(h, actions, n_steps, 0, obs_out, ref_out, reward_out, terminated_out, stream);
}

// Domain randomisation (SURVEY.md §8f row 4; the batched counterpart of constructing N reference envs with N motor_parameter / load_parameter
// dicts): every env gets its own model coefficients, derived here exactly like the shared ones (the *_update_model methods,
// mechanical_load.py:188-193) from ITS physical parameters.  Limits, nominal values, reward and reference settings stay those of the
// handle's configuration.  NULL motor_param: back to the shared coefficients.
static int fill_shared_blocks(gemb200_handle* h);
int gemb200_set_env_params(gemb200_handle* h, const double* motor_param, const double* load_param) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  DeviceGuard guard(h->cfg.device);
  CUDA_TRY(cudaDeviceSynchronize());
  if (h->cfg.layout != GEMB200_LAYOUT_AOS && (motor_param || load_param))
    return fail(GEMB200_E_INVALID, "per-env parameter blocks need the row-per-env (AoS) I/O layout");
  if (!motor_param && !load_param) {
    h->n_draw = 0;  // shared coefficients again: no parameter draws either
    int rc = GEMB200_OK;
    if (h->ids_in_use) {  // adopted RNG identities are read by the ENVP instantiations only: the blocks take the shared parameters instead
      rc = fill_shared_blocks(h);
      if (!rc) h->blocks = kBlocksShared;
    } else {
      h->blocks = kBlocksNone;
    }
    apply_mode(h);
    return rc;
  }
  const size_t n = (size_t)h->cfg.n_envs;
  Dims d;
  derive_dims(&h->cfg, &d);
  std::vector<double> tab((size_t)kCoefWords * n);
  std::vector<double> raw((size_t)kMaxDraw * n);  // the physical parameters themselves: what parameter draws at a reset start from
  gemb200_config c = h->cfg;
  for (size_t i = 0; i < n; ++i) {
    if (motor_param) std::memcpy(c.motor_param, motor_param + i * GEMB200_MAX_MOTOR_PARAM, sizeof(c.motor_param));
    if (load_param) std::memcpy(c.load_param, load_param + i * 8, sizeof(c.load_param));
    if (c.motor_param[GEMB200_MP_P] != h->cfg.motor_param[GEMB200_MP_P])
      return fail(GEMB200_E_INVALID, "pole pairs cannot differ per env: the angle increments are prepared on the host per handle");
    for (int s = 0; s < GEMB200_MAX_MOTOR_PARAM; ++s) raw[(size_t)s * n + i] = c.motor_param[s];
    for (int s = 0; s < 8; ++s) raw[(size_t)(GEMB200_MAX_MOTOR_PARAM + s) * n + i] = c.load_param[s];
    if (c.load_kind == GEMB200_LOAD_POLY_STATIC && !(c.load_param[GEMB200_LP_J_LOAD] + c.motor_param[GEMB200_MP_J_ROTOR] > 0))
      return fail(GEMB200_E_INVALID, "per-env parameters: total inertia must be positive for every env");
    Derived dv;
    derive_model(&c, d, &dv);
    for (int w = 0; w < 20; ++w) tab[(size_t)w * n + i] = dv.c[w];
    for (int w = 0; w < 4; ++w) tab[(size_t)(20 + w) * n + i] = dv.tq[w];
    tab[(size_t)24 * n + i] = c.load_param[GEMB200_LP_A]; tab[(size_t)25 * n + i] = c.load_param[GEMB200_LP_B]; tab[(size_t)26 * n + i] = c.load_param[GEMB200_LP_C];
    tab[(size_t)27 * n + i] = dv.inv_j; tab[(size_t)28 * n + i] = dv.omega_lim; tab[(size_t)29 * n + i] = dv.omega_lin;
  }
  for (double v : tab) if (!std::isfinite(v)) return fail(GEMB200_E_INVALID, "per-env parameters: a derived model coefficient is not finite (zero inductance?)");
  if (!h->d_envp) CUDA_TRY(cudaMalloc(&h->d_envp, tab.size() * h->rsz));
  if (!h->d_praw) CUDA_TRY(cudaMalloc(&h->d_praw, raw.size() * sizeof(double)));
  CUDA_TRY(cudaMemcpy(h->d_praw, raw.data(), raw.size() * sizeof(double), cudaMemcpyHostToDevice));
  const int rc = with_params(h, [&](auto& p) {
    using real = decltype(p.tau);
    const std::vector<real> t(tab.begin(), tab.end());
    CUDA_TRY(cudaMemcpy(h->d_envp, t.data(), t.size() * sizeof(real), cudaMemcpyHostToDevice));
    return GEMB200_OK;
  });
  if (rc) return rc;
  h->blocks = kBlocksCaller;
  apply_mode(h);
  return GEMB200_OK;
}

}  // extern "C"

// Per-env parameter blocks filled on the device from the shared configuration: every env gets the shared coefficients (the values
// gemb200_set_env_params derives from rows equal to the configuration's) and the configuration's physical parameters.
struct RawParams { double v[kMaxDraw]; };
template <typename real>
__global__ void fill_env_params_kernel(real* envp, double* praw, const Coef<real> k, const RawParams raw, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t nn = (size_t)n;
  for (int w = 0; w < 20; ++w) envp[w * nn + i] = k.c[w];
  for (int w = 0; w < 4; ++w) envp[(20 + w) * nn + i] = k.tq[w];
  envp[24 * nn + i] = k.load_a; envp[25 * nn + i] = k.load_b; envp[26 * nn + i] = k.load_c;
  envp[27 * nn + i] = k.inv_j; envp[28 * nn + i] = k.omega_lim; envp[29 * nn + i] = k.omega_lin;
  for (int s = 0; s < kMaxDraw; ++s) praw[s * nn + i] = raw.v[s];
}
// the configuration's physical parameters in the slot order of praw
static RawParams config_params(const gemb200_handle* h) {
  RawParams raw;
  for (int s = 0; s < GEMB200_MAX_MOTOR_PARAM; ++s) raw.v[s] = h->cfg.motor_param[s];
  for (int s = 0; s < 8; ++s) raw.v[GEMB200_MAX_MOTOR_PARAM + s] = h->cfg.load_param[s];
  return raw;
}
// no adopted identities any more: launches key every env by its own identity again, and blocks that only an adoption made go, so that the
// handle runs its shared-coefficient kernels like a fresh one (the identity array stays allocated for the next adoption)
static void drop_rng_ids(gemb200_handle* h) {
  h->ids_in_use = false;
  if (h->blocks == kBlocksShared) h->blocks = kBlocksNone;
  apply_mode(h);
}
// every env's block := the shared parameters (synchronises); the caller sets the handle's blocks and applies the mode
static int fill_shared_blocks(gemb200_handle* h) {
  const size_t nn = (size_t)h->cfg.n_envs;
  if (!h->d_envp) CUDA_TRY(cudaMalloc(&h->d_envp, (size_t)kCoefWords * nn * h->rsz));
  if (!h->d_praw) CUDA_TRY(cudaMalloc(&h->d_praw, (size_t)kMaxDraw * nn * sizeof(double)));
  const RawParams raw = config_params(h);
  const int grid = (int)((nn + 255) / 256);
  with_params(h, [&](auto& p) {
    using real = decltype(p.tau);
    fill_env_params_kernel<real><<<grid, 256>>>(static_cast<real*>(h->d_envp), h->d_praw, p.k, raw, (int)nn);
  });
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaDeviceSynchronize());
  return GEMB200_OK;
}
// out[j][i] = stored value of drawn parameter j of env i, in the handle's dtype
template <typename real>
__global__ void get_env_params_kernel(const double* praw, const ParamDraw* d, int n_draw, real* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int j = 0; j < n_draw; ++j) out[(size_t)j * n + i] = (real)praw[(size_t)d->slot[j] * n + i];
}

extern "C" {

int gemb200_set_param_randomization(gemb200_handle* h, int32_t n, const int32_t* slot, const int32_t* kind, const double* lo, const double* hi) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (n < 0 || n > kMaxDraw) return fail(GEMB200_E_INVALID, "number of drawn parameters out of range");
  if (n > 0 && (!slot || !kind || !lo || !hi)) return fail(GEMB200_E_INVALID, "NULL argument");
  DeviceGuard guard(h->cfg.device);
  CUDA_TRY(cudaDeviceSynchronize());
  if (n == 0) {  // no more draws; the envs keep their last values
    h->n_draw = 0;
    apply_mode(h);
    return GEMB200_OK;
  }
  if (h->cfg.layout != GEMB200_LAYOUT_AOS) return fail(GEMB200_E_INVALID, "parameter draws need the row-per-env (AoS) I/O layout (per-env parameter blocks)");
  const bool flux_limits = h->cfg.init_im_valid != 0;  // induction motor with random initial states: init_im is derived on the host
  ParamDraw pd;
  std::memset(&pd, 0, sizeof(pd));
  bool seen[kMaxDraw] = {};
  for (int j = 0; j < n; ++j) {
    const int s = slot[j];
    const bool motor = s >= 0 && s < GEMB200_MAX_MOTOR_PARAM, load = s >= GEMB200_MAX_MOTOR_PARAM && s <= GEMB200_MAX_MOTOR_PARAM + GEMB200_LP_J_LOAD;
    if (!motor && !load) return fail(GEMB200_E_INVALID, "unknown parameter slot (motor: GEMB200_MP_*, load: GEMB200_MAX_MOTOR_PARAM + GEMB200_LP_A.._J_LOAD)");
    if (s == GEMB200_MP_P) return fail(GEMB200_E_INVALID, "pole pairs cannot be drawn per env: the angle increments are prepared on the host per handle");
    if (flux_limits && (s == GEMB200_MP_L_M || s == GEMB200_MP_L_SIGS || s == GEMB200_MP_L_SIGR || s == GEMB200_MP_R_S || s == GEMB200_MP_R_E))
      return fail(GEMB200_E_INVALID, "l_m, l_sigs, l_sigr, r_s and r_r of an induction motor with random initial states enter the host-derived flux limits (init_im); not supported");
    if (seen[s]) return fail(GEMB200_E_INVALID, "parameter slot given twice");
    seen[s] = true;
    if (kind[j] != GEMB200_DIST_UNIFORM && kind[j] != GEMB200_DIST_LOG_UNIFORM) return fail(GEMB200_E_INVALID, "unknown distribution kind");
    if (!std::isfinite(lo[j]) || !std::isfinite(hi[j]) || lo[j] > hi[j]) return fail(GEMB200_E_INVALID, "distribution bounds must be finite with lo <= hi");
    if (kind[j] == GEMB200_DIST_LOG_UNIFORM && !(lo[j] > 0)) return fail(GEMB200_E_INVALID, "log-uniform bounds must be positive");
    pd.slot[j] = s; pd.kind[j] = kind[j]; pd.lo[j] = lo[j]; pd.hi[j] = hi[j];
    if (kind[j] == GEMB200_DIST_LOG_UNIFORM) { pd.a[j] = std::log(lo[j]); pd.b[j] = std::log(hi[j]) - std::log(lo[j]); }
    else { pd.a[j] = lo[j]; pd.b[j] = hi[j] - lo[j]; }
  }
  if (!h->d_draw) CUDA_TRY(cudaMalloc(&h->d_draw, sizeof(ParamDraw)));
  CUDA_TRY(cudaMemcpy(h->d_draw, &pd, sizeof(pd), cudaMemcpyHostToDevice));
  if (h->blocks == kBlocksNone) {  // no per-env blocks yet: every env starts from the shared parameters
    const int rc = fill_shared_blocks(h);
    if (rc) return rc;
  }
  h->blocks = kBlocksCaller;  // the draws change the blocks: they are the caller's from now on
  h->n_draw = n;
  apply_mode(h);
  return GEMB200_OK;
}

int gemb200_get_env_params(gemb200_handle* h, void* out, void* stream) {
  if (!h || !out) return fail(GEMB200_E_INVALID, "NULL argument");
  if (!draws_on(h)) return fail(GEMB200_E_INVALID, "no parameters are drawn (gemb200_set_param_randomization)");
  DeviceGuard guard(h->cfg.device);
  const int n = h->cfg.n_envs, grid = (n + 255) / 256;
  with_params(h, [&](auto& p) {
    using real = decltype(p.tau);
    get_env_params_kernel<real><<<grid, 256, 0, (cudaStream_t)stream>>>(h->d_praw, h->d_draw, h->n_draw, static_cast<real*>(out), n);
  });
  CUDA_TRY(cudaGetLastError());
  return GEMB200_OK;
}

// ----------------------------------------------------------------------------------------------------------------
// Fused aggregated return over NVLink (SURVEY.md §8e: the sharded layout's ONE collective, done by the step kernel itself)
// ----------------------------------------------------------------------------------------------------------------
// Flags: one uint32 per (slot, source rank), written by the source with a system-scope store after its step kernel has finished (every
// thread of the step kernel fences its peer stores at system scope before it exits), polled by the owner.
__global__ void peer_signal_kernel(uint32_t* const* flags, int n, uint32_t value) {
  const int d = threadIdx.x;
  if (d < n) {
    __threadfence_system();
    *reinterpret_cast<volatile uint32_t*>(flags[d]) = value;
    __threadfence_system();
  }
}
// spins until all n flags are >= value (wrap-safe signed distance); gives up after ~4e9 cycles and raises *err so that a lost peer cannot hang the GPU
__global__ void peer_wait_kernel(const uint32_t* flags, int n, uint32_t value, int* err) {
  const int s = threadIdx.x;
  if (s < n) {
    const long long t0 = clock64();
    while ((int32_t)(*reinterpret_cast<const volatile uint32_t*>(flags + s) - value) < 0) {
      if (clock64() - t0 > 4000000000LL) { atomicExch(err, 1 + s); break; }
      __nanosleep(200);
    }
    __threadfence_system();
  }
}

int gemb200_peer_buffer_alloc(int32_t device, int64_t bytes, void** dev_ptr, void* ipc_handle64) {
  if (!dev_ptr || !ipc_handle64 || bytes <= 0) return fail(GEMB200_E_INVALID, "bad argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  DeviceGuard guard(device);
  CUDA_TRY(cudaMalloc(dev_ptr, (size_t)bytes));
  CUDA_TRY(cudaMemset(*dev_ptr, 0, (size_t)bytes));
  cudaIpcMemHandle_t hd;
  CUDA_TRY(cudaIpcGetMemHandle(&hd, *dev_ptr));
  std::memcpy(ipc_handle64, &hd, sizeof(hd));
  CUDA_TRY(cudaDeviceSynchronize());
  return GEMB200_OK;
}
int gemb200_peer_buffer_open(int32_t device, const void* ipc_handle64, void** dev_ptr) {
  if (!dev_ptr || !ipc_handle64) return fail(GEMB200_E_INVALID, "bad argument");
  DeviceGuard guard(device);  // the CONSUMER's device is current: the mapping lives in this context and peer access is enabled lazily
  cudaIpcMemHandle_t hd;
  std::memcpy(&hd, ipc_handle64, sizeof(hd));
  CUDA_TRY(cudaIpcOpenMemHandle(dev_ptr, hd, cudaIpcMemLazyEnablePeerAccess));
  return GEMB200_OK;
}
int gemb200_peer_buffer_close(int32_t device, void* dev_ptr) {
  DeviceGuard guard(device);
  CUDA_TRY(cudaIpcCloseMemHandle(dev_ptr));
  return GEMB200_OK;
}
int gemb200_peer_buffer_free(int32_t device, void* dev_ptr) {
  DeviceGuard guard(device);
  CUDA_TRY(cudaFree(dev_ptr));
  return GEMB200_OK;
}
int gemb200_bind_peers(gemb200_handle* h, int32_t n_dst, const int64_t* dst_delta) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (n_dst < 0 || n_dst > 8 || (n_dst > 0 && !dst_delta)) return fail(GEMB200_E_INVALID, "n_dst must be in [0, 8]");
  if (n_dst > 0 && h->cfg.layout != GEMB200_LAYOUT_AOS) return fail(GEMB200_E_INVALID, "peer destinations need the row-per-env (AoS) layout");
  h->n_dst = n_dst;
  for (int d = 0; d < n_dst; ++d) h->dst_delta[d] = dst_delta[d];
  apply_mode(h);
  return GEMB200_OK;
}
int gemb200_peer_signal(gemb200_handle* h, int32_t n_dst, uint32_t* const* flag_ptrs_dev, uint32_t value, void* stream) {
  if (!h || n_dst < 1 || n_dst > 32 || !flag_ptrs_dev) return fail(GEMB200_E_INVALID, "bad argument");
  DeviceGuard guard(h->cfg.device);
  peer_signal_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(flag_ptrs_dev, n_dst, value);
  CUDA_TRY(cudaGetLastError());
  return GEMB200_OK;
}
int gemb200_peer_wait(gemb200_handle* h, int32_t n_src, const uint32_t* flags_dev, uint32_t value, int32_t* err_dev, void* stream) {
  if (!h || n_src < 1 || n_src > 32 || !flags_dev || !err_dev) return fail(GEMB200_E_INVALID, "bad argument");
  DeviceGuard guard(h->cfg.device);
  peer_wait_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(flags_dev, n_src, value, err_dev);
  CUDA_TRY(cudaGetLastError());
  return GEMB200_OK;
}

static int ensure_host_buffers(gemb200_handle* h) {
  if (h->hstream) return GEMB200_OK;
  const size_t n = (size_t)h->cfg.n_envs;
  CUDA_TRY(cudaStreamCreateWithFlags(&h->hstream, cudaStreamNonBlocking));
  for (int k = 0; k < 3; ++k) CUDA_TRY(cudaStreamCreateWithFlags(&h->hpipe[k], cudaStreamNonBlocking));
  CUDA_TRY(cudaMalloc(&h->d_act, n * h->n_act * (h->cfg.finite ? sizeof(int32_t) : h->rsz)));
  CUDA_TRY(cudaMalloc(&h->d_obs, n * h->n_obs * h->rsz));
  CUDA_TRY(cudaMalloc(&h->d_ref, n * (h->n_ref > 0 ? h->n_ref : 1) * h->rsz));
  CUDA_TRY(cudaMalloc(&h->d_rew, n * h->rsz));
  CUDA_TRY(cudaMalloc((void**)&h->d_term, n));
  CUDA_TRY(cudaMalloc((void**)&h->d_mask, n));
  return GEMB200_OK;
}

int gemb200_step_host(gemb200_handle* h, const void* action, void* obs_out, void* ref_out, void* reward_out, uint8_t* terminated_out) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (!action) return fail(GEMB200_E_INVALID, "action is NULL");
  DeviceGuard guard(h->cfg.device);
  int rc = ensure_host_buffers(h);
  if (rc) return rc;
  const size_t n = (size_t)h->cfg.n_envs;
  const size_t asz = (size_t)h->n_act * (h->cfg.finite ? sizeof(int32_t) : h->rsz);  // action bytes per env
  // Row-per-env buffers are contiguous per env range, so a large batch is cut into chunks that flow through three
  // streams: the D2H of chunk c overlaps the H2D + launch of chunk c+1 (PCIe is full duplex).  One API call = one RNG id.
  const bool pipelined = h->cfg.layout == GEMB200_LAYOUT_AOS && n >= (size_t)1 << 16;
  static const int chunks_env = [] { const char* e = std::getenv("GEMB200_HOST_CHUNKS"); return e ? std::atoi(e) : 0; }();  // experiment knob
  const int nchunk = pipelined ? (chunks_env > 0 ? chunks_env : 4) : 1;  // PCIe D2H bound; 4 keeps the copy count low
  const size_t per = pipelined ? ((n / nchunk + 255) / 256) * 256 : n;
  bool first = true;
  for (int c = 0; c < nchunk; ++c) {
    const size_t b = (size_t)c * per, e = (b + per < n) ? b + per : n;
    if (b >= e) break;
    cudaStream_t st = pipelined ? h->hpipe[c % 3] : h->hstream;
    CUDA_TRY(cudaMemcpyAsync((char*)h->d_act + b * asz, (const char*)action + b * asz, (e - b) * asz, cudaMemcpyHostToDevice, st));
    rc = do_step(h, h->d_act, obs_out ? h->d_obs : nullptr, (ref_out && h->n_ref) ? h->d_ref : nullptr, reward_out ? h->d_rew : nullptr,
                 terminated_out ? h->d_term : nullptr, st, (int)b, (int)e, first);
    first = false;
    if (rc) return rc;
    if (pipelined) {
      const size_t os = (size_t)h->n_obs * h->rsz, rs = (size_t)h->n_ref * h->rsz;
      if (obs_out) CUDA_TRY(cudaMemcpyAsync((char*)obs_out + b * os, (char*)h->d_obs + b * os, (e - b) * os, cudaMemcpyDeviceToHost, st));
      if (ref_out && h->n_ref) CUDA_TRY(cudaMemcpyAsync((char*)ref_out + b * rs, (char*)h->d_ref + b * rs, (e - b) * rs, cudaMemcpyDeviceToHost, st));
      if (reward_out) CUDA_TRY(cudaMemcpyAsync((char*)reward_out + b * h->rsz, (char*)h->d_rew + b * h->rsz, (e - b) * h->rsz, cudaMemcpyDeviceToHost, st));
      if (terminated_out) CUDA_TRY(cudaMemcpyAsync(terminated_out + b, h->d_term + b, e - b, cudaMemcpyDeviceToHost, st));
    }
  }
  if (pipelined) {
    for (int k = 0; k < 3; ++k) CUDA_TRY(cudaStreamSynchronize(h->hpipe[k]));
    return GEMB200_OK;
  }
  cudaStream_t st = h->hstream;
  if (obs_out) CUDA_TRY(cudaMemcpyAsync(obs_out, h->d_obs, n * h->n_obs * h->rsz, cudaMemcpyDeviceToHost, st));
  if (ref_out && h->n_ref) CUDA_TRY(cudaMemcpyAsync(ref_out, h->d_ref, n * h->n_ref * h->rsz, cudaMemcpyDeviceToHost, st));
  if (reward_out) CUDA_TRY(cudaMemcpyAsync(reward_out, h->d_rew, n * h->rsz, cudaMemcpyDeviceToHost, st));
  if (terminated_out) CUDA_TRY(cudaMemcpyAsync(terminated_out, h->d_term, n, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return GEMB200_OK;
}

int gemb200_reset_host(gemb200_handle* h, const uint8_t* reset_mask, void* obs_out, void* ref_out) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  DeviceGuard guard(h->cfg.device);
  int rc = ensure_host_buffers(h);
  if (rc) return rc;
  const size_t n = (size_t)h->cfg.n_envs;
  cudaStream_t st = h->hstream;
  if (reset_mask) CUDA_TRY(cudaMemcpyAsync(h->d_mask, reset_mask, n, cudaMemcpyHostToDevice, st));
  if (reset_mask && (obs_out || ref_out)) {
    // unmasked envs keep the caller's previous values: pre-load the device staging buffers with them
    if (obs_out) CUDA_TRY(cudaMemcpyAsync(h->d_obs, obs_out, n * h->n_obs * h->rsz, cudaMemcpyHostToDevice, st));
    if (ref_out && h->n_ref) CUDA_TRY(cudaMemcpyAsync(h->d_ref, ref_out, n * h->n_ref * h->rsz, cudaMemcpyHostToDevice, st));
  }
  rc = do_reset(h, reset_mask ? h->d_mask : nullptr, obs_out ? h->d_obs : nullptr, (ref_out && h->n_ref) ? h->d_ref : nullptr, st);
  if (rc) return rc;
  if (obs_out) CUDA_TRY(cudaMemcpyAsync(obs_out, h->d_obs, n * h->n_obs * h->rsz, cudaMemcpyDeviceToHost, st));
  if (ref_out && h->n_ref) CUDA_TRY(cudaMemcpyAsync(ref_out, h->d_ref, n * h->n_ref * h->rsz, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return GEMB200_OK;
}

int gemb200_get_ode_state(gemb200_handle* h, double* ode_out, void* stream) {
  if (!h || !ode_out) return fail(GEMB200_E_INVALID, "NULL argument");
  return launch_accessor(h, stream, [&](auto& p, int n, int grid, cudaStream_t st) {
    using real = decltype(p.tau);
    get_ode_kernel<real><<<grid, 256, 0, st>>>((const real*)h->d_st, (const real*)h->d_stc, h->d_eps, ode_out, n, h->nx, h->n_ref, h->has_eps);
  });
}
int gemb200_set_ode_state(gemb200_handle* h, const double* ode_in, void* stream) {
  if (!h || !ode_in) return fail(GEMB200_E_INVALID, "NULL argument");
  return launch_accessor(h, stream, [&](auto& p, int n, int grid, cudaStream_t st) {
    using real = decltype(p.tau);
    set_ode_kernel<real><<<grid, 256, 0, st>>>((real*)h->d_st, (real*)h->d_stc, h->d_eps, ode_in, n, h->nx, h->n_ref, h->has_eps);
  });
}
int gemb200_get_reference(gemb200_handle* h, double* ref_out, void* stream) {
  if (!h || !ref_out) return fail(GEMB200_E_INVALID, "NULL argument");
  if (h->n_ref == 0) return GEMB200_OK;
  return launch_accessor(h, stream, [&](auto& p, int n, int grid, cudaStream_t st) {
    using real = decltype(p.tau);
    get_ref_kernel<real><<<grid, 256, 0, st>>>((const real*)h->d_st, ref_out, n, h->nx, h->n_ref);
  });
}
int gemb200_set_reference(gemb200_handle* h, const double* ref_in, void* stream) {
  if (!h || !ref_in) return fail(GEMB200_E_INVALID, "NULL argument");
  if (h->n_ref == 0) return GEMB200_OK;
  return launch_accessor(h, stream, [&](auto& p, int n, int grid, cudaStream_t st) {
    using real = decltype(p.tau);
    set_ref_kernel<real><<<grid, 256, 0, st>>>((real*)h->d_st, ref_in, n, h->nx, h->n_ref);
  });
}

struct CheckpointHeader {
  char magic[8];          // "GEMB200C"
  int32_t abi, dtype, n_envs, n_sections, nh, nc, reserved[2];
  uint64_t config_hash, payload_bytes, gstep, n_steps;
};
// FNV-1a over the configuration, leaving out what may legitimately differ between writer and reader: the device ordinal and the
// host pointer of the speed-profile table (whose CONTENT is hashed at create)
static uint64_t config_hash(const gemb200_handle* h) {
  gemb200_config c = h->cfg;
  c.device = 0;
  c.ext_speed_table = nullptr;
  uint64_t x = 1469598103934665603ull;
  const unsigned char* b = reinterpret_cast<const unsigned char*>(&c);
  for (size_t i = 0; i < sizeof(c); ++i) { x ^= b[i]; x *= 1099511628211ull; }
  x ^= h->ext_hash; x *= 1099511628211ull;
  return x;
}
static void make_header(gemb200_handle* h, CheckpointHeader* hd) {
  std::memset(hd, 0, sizeof(*hd));
  std::memcpy(hd->magic, "GEMB200C", 8);
  hd->abi = GEMB200_ABI_VERSION; hd->dtype = h->cfg.dtype; hd->n_envs = h->cfg.n_envs; hd->nh = h->NH; hd->nc = h->NC;
  Section s[kMaxSections];
  hd->n_sections = sections(h, s);
  for (int i = 0; i < hd->n_sections; ++i) hd->payload_bytes += s[i].bytes;
  hd->config_hash = config_hash(h);
  hd->gstep = h->gstep; hd->n_steps = h->n_steps;
}
int64_t gemb200_checkpoint_size(gemb200_handle* h) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  CheckpointHeader hd;
  make_header(h, &hd);
  return (int64_t)sizeof(hd) + (int64_t)hd.payload_bytes;
}
int gemb200_checkpoint_save(gemb200_handle* h, void* host_blob) {
  if (!h || !host_blob) return fail(GEMB200_E_INVALID, "NULL argument");
  if (draws_on(h)) return fail(GEMB200_E_INVALID, "checkpoints do not carry the parameters drawn per reset; switch the draws off first (DESIGN §7)");
  if (h->ids_in_use) return fail(GEMB200_E_INVALID, "checkpoints do not carry adopted RNG identities; clear them first (gemb200_clear_rng_ids, DESIGN §7)");
  DeviceGuard guard(h->cfg.device);
  CUDA_TRY(cudaDeviceSynchronize());
  if (h->dev_clock) { int rc = pull_clock(h, nullptr); if (rc) return rc; }  // the header carries the clock
  char* b = (char*)host_blob;
  CheckpointHeader hd;
  make_header(h, &hd);
  std::memcpy(b, &hd, sizeof(hd)); b += sizeof(hd);
  Section s[kMaxSections];
  const int k = sections(h, s);
  for (int i = 0; i < k; ++i) { CUDA_TRY(cudaMemcpy(b, *s[i].slot, s[i].bytes, cudaMemcpyDeviceToHost)); b += s[i].bytes; }
  return GEMB200_OK;
}
int gemb200_checkpoint_load(gemb200_handle* h, const void* host_blob) {
  if (!h || !host_blob) return fail(GEMB200_E_INVALID, "NULL argument");
  if (draws_on(h)) return fail(GEMB200_E_INVALID, "checkpoints do not carry the parameters drawn per reset; switch the draws off first (DESIGN §7)");
  if (h->ids_in_use) return fail(GEMB200_E_INVALID, "checkpoints do not carry adopted RNG identities; clear them first (gemb200_clear_rng_ids, DESIGN §7)");
  DeviceGuard guard(h->cfg.device);
  CheckpointHeader want, got;
  make_header(h, &want);
  std::memcpy(&got, host_blob, sizeof(got));
  if (std::memcmp(got.magic, want.magic, 8) != 0) return fail(GEMB200_E_INVALID, "checkpoint: not a gemb200 checkpoint blob (bad magic)");
  if (got.abi != want.abi) return fail(GEMB200_E_ABI, "checkpoint: written by another ABI version");
  if (got.dtype != want.dtype || got.n_envs != want.n_envs || got.n_sections != want.n_sections || got.nh != want.nh || got.nc != want.nc ||
      got.payload_bytes != want.payload_bytes)
    return fail(GEMB200_E_INVALID, "checkpoint: dtype / n_envs / record layout differ from this handle");
  if (got.config_hash != want.config_hash)
    return fail(GEMB200_E_INVALID, "checkpoint: written by a handle with a different configuration (motor, parameters, seed, tau, generators, ...)");
  CUDA_TRY(cudaDeviceSynchronize());
  const char* b = (const char*)host_blob + sizeof(got);
  h->gstep = got.gstep; h->n_steps = got.n_steps;
  Section s[kMaxSections];
  const int k = sections(h, s);
  for (int i = 0; i < k; ++i) { CUDA_TRY(cudaMemcpy(*s[i].slot, b, s[i].bytes, cudaMemcpyHostToDevice)); b += s[i].bytes; }
  if (h->dev_clock) { int rc = push_clock(h, nullptr); if (rc) return rc; CUDA_TRY(cudaDeviceSynchronize()); }
  return GEMB200_OK;
}

// ElectricMotorEnvironment.reset(seed) -> _seed(seed) re-seeds every component (core.py:300-319, utils / RandomComponent.seed): a handle
// re-keyed with `seed` behaves exactly like a freshly created one with that seed — call ids, step clock, dead-time ring, switching
// states and every other persistent array start over — so equal seeds give identical episodes.
int gemb200_reseed(gemb200_handle* h, uint64_t seed, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  DeviceGuard guard(h->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  h->cfg.seed = seed;
  h->gstep = 0; h->n_steps = 0;
  if (h->dev_clock) { int rc = push_clock(h, st); if (rc) return rc; }
  with_params(h, [&](auto& p) { set_seed(&p, seed); });
  drop_rng_ids(h);  // every env draws with its own identity again
  Section s[kMaxSections];
  const int k = sections(h, s);
  for (int i = 0; i < k; ++i) {
    CUDA_TRY(cudaMemsetAsync(*s[i].slot, 0, s[i].bytes, st));
  }
  int rc = fill_imprev(h, st);
  if (rc) return rc;
  return do_reset(h, nullptr, nullptr, nullptr, st);
}

// Device-resident clock on / off (include/gemb200.h).  On: the host counters are uploaded; off: they are read back (synchronises `stream`).
int gemb200_set_device_clock(gemb200_handle* h, int32_t enable, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  DeviceGuard guard(h->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  if (enable && !h->dev_clock) {
    if (!h->d_clock) CUDA_TRY(cudaMalloc(&h->d_clock, 8 * sizeof(uint32_t)));
    int rc = push_clock(h, st);
    if (rc) return rc;
    h->dev_clock = true;
  } else if (!enable && h->dev_clock) {
    int rc = pull_clock(h, st);
    if (rc) return rc;
    h->dev_clock = false;
  }
  return GEMB200_OK;
}
int gemb200_get_clock(gemb200_handle* h, uint64_t* call_id, uint64_t* n_steps, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  DeviceGuard guard(h->cfg.device);
  if (h->dev_clock) { int rc = pull_clock(h, (cudaStream_t)stream); if (rc) return rc; }
  if (call_id) *call_id = h->gstep;
  if (n_steps) *n_steps = h->n_steps;
  return GEMB200_OK;
}

int64_t gemb200_launch_count(gemb200_handle* h) { return h ? h->launches : 0; }
int gemb200_kernel_time_begin(gemb200_handle* h, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  DeviceGuard guard(h->cfg.device);
  CUDA_TRY(cudaEventRecord(h->ev0, (cudaStream_t)stream));
  return GEMB200_OK;
}
int gemb200_kernel_time_end(gemb200_handle* h, void* stream, float* ms_out) {
  if (!h || !ms_out) return fail(GEMB200_E_INVALID, "NULL argument");
  DeviceGuard guard(h->cfg.device);
  CUDA_TRY(cudaEventRecord(h->ev1, (cudaStream_t)stream));
  CUDA_TRY(cudaEventSynchronize(h->ev1));
  CUDA_TRY(cudaEventElapsedTime(ms_out, h->ev0, h->ev1));
  return GEMB200_OK;
}

}  // extern "C"

// ----------------------------------------------------------------------------------------------------------------
// Per-env state snapshots (gemb200_pack_envs / gemb200_unpack_envs): packed rows of 32-bit words, format in include/gemb200.h
// ----------------------------------------------------------------------------------------------------------------
// The two kernels know nothing about motor families: the section table drives them.  A block of B threads owns B rows.  Each thread moves
// the arrays of its env to / from its row in shared memory — consecutive threads touch consecutive envs, so the SoA arrays are read and
// written coalesced, the chunked records with the step kernel's 16-byte accesses — and the block moves its rows to / from global memory
// word by word, so the [m][words] rows are read and written contiguously as well (the obs row store of the step kernel does the same).
struct RecSec { char* ptr; int esz, per_env, place, clk, row_off; };
struct RecArgs {
  RecSec sec[kMaxSections];
  int n_sec, n, words, stride;  // sections, envs of the handle, words per row, shared-memory words per row (odd: no bank conflicts)
  uint32_t div_magic;           // ceil(2^32 / words): row of a block-local word index with one multiply-high
  int rsz, n_ref, dead, fifo_dim, swst_off;  // swst_off: row word of the switched-generator section, -1 without one
  int sw_count[kMaxRef], ref_kind[kMaxRefEntries];
  uint32_t kstep;                // step count (sub-episode clock) and dead-time ring position of the host clock ...
  int32_t ring;
  const uint32_t* clock_dev;     // ... or of the device-resident clock (gemb200_set_device_clock), read like clock_of() does
  uint32_t* rngid;               // RNG identities [kRngIdWords][n] (nullptr: none adopted yet); unpack gives the envs their own back
  uint32_t seed_lo, seed_hi;
  int64_t env_offset;
};
constexpr int kRecBlockMax = 128;

// env i's own RNG identity: the handle's seed, its global index, no offsets (the keying of an env that adopted none)
__device__ __forceinline__ void set_own_rng_id(uint32_t* ids, size_t n, unsigned i, uint32_t seed_lo, uint32_t seed_hi, int64_t env_offset) {
  const uint64_t g = (uint64_t)(env_offset + i);
  ids[i] = seed_lo; ids[n + i] = seed_hi; ids[2 * n + i] = (uint32_t)g; ids[3 * n + i] = (uint32_t)(g >> 32);
  ids[4 * n + i] = 0u; ids[5 * n + i] = 0u; ids[6 * n + i] = 0u; ids[7 * n + i] = 0u;
}
__device__ __forceinline__ void rec_clock(const RecArgs& a, uint32_t* kstep, int* ring) {
  if (a.clock_dev) { *kstep = a.clock_dev[2]; *ring = (int)a.clock_dev[3]; }
  else { *kstep = a.kstep; *ring = a.ring; }
}
// element idx of an array of esz-byte elements <-> its row words (two for a double, low word first; a uint16 zero-extended to one)
template <bool TO_ROW>
__device__ __forceinline__ void move_elem(char* p, int esz, size_t idx, uint32_t* w) {
  if (esz == 8) {
    uint2* q = reinterpret_cast<uint2*>(p) + idx;
    if (TO_ROW) { const uint2 v = *q; w[0] = v.x; w[1] = v.y; } else *q = make_uint2(w[0], w[1]);
  } else if (esz == 4) {
    uint32_t* q = reinterpret_cast<uint32_t*>(p) + idx;
    if (TO_ROW) w[0] = *q; else *q = w[0];
  } else {
    uint16_t* q = reinterpret_cast<uint16_t*>(p) + idx;
    if (TO_ROW) w[0] = *q; else *q = (uint16_t)w[0];
  }
}
// every section of env i <-> the row; the dead-time ring is rotated so that the row holds it oldest entry first
template <bool TO_ROW>
__device__ __forceinline__ void move_env(const RecArgs& a, unsigned i, int ring, uint32_t* row) {
  const size_t n = (size_t)a.n;
  for (int s = 0; s < a.n_sec; ++s) {
    const RecSec& S = a.sec[s];
    uint32_t* w = row + S.row_off;
    if (S.place == kRecord) {  // 16-byte chunks, then (fp32) one 8-byte chunk, then one element: gemb200_params.h word_offset()
      const int vw = 16 / S.esz, nfull = S.per_env / vw, wpe = S.esz / 4;
      for (int c = 0; c < nfull; ++c) {
        uint4* q = reinterpret_cast<uint4*>(S.ptr + (size_t)c * 16 * n) + i;
        uint32_t* d = w + 4 * c;
        if (TO_ROW) { const uint4 v = *q; d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w; }
        else *q = make_uint4(d[0], d[1], d[2], d[3]);
      }
      int e = nfull * vw;
      if (vw == 4 && S.per_env - e >= 2) {
        uint2* q = reinterpret_cast<uint2*>(S.ptr + (size_t)e * 4 * n) + i;
        uint32_t* d = w + e;
        if (TO_ROW) { const uint2 v = *q; d[0] = v.x; d[1] = v.y; } else *q = make_uint2(d[0], d[1]);
        e += 2;
      }
      if (e < S.per_env) move_elem<TO_ROW>(S.ptr + (size_t)e * S.esz * n, S.esz, i, w + e * wpe);
    } else {
      const int wpe = S.esz == 8 ? 2 : 1;
      for (int q = 0; q < S.per_env; ++q) {
        int ae = q;
        if (S.clk == kClkRing) {  // row entry `slot` (0 = oldest) lives in ring slot (ring + slot) mod dead
          const int slot = q / a.fifo_dim, j = q - slot * a.fifo_dim;
          int rs = slot + ring;
          if (rs >= a.dead) rs -= a.dead;
          ae = rs * a.fifo_dim + j;
        }
        move_elem<TO_ROW>(S.ptr, S.esz, (size_t)ae * n + i, w + q * wpe);
      }
    }
  }
}
// a step index kept in a `real` record element (gemb200_kernels.cuh word_to_u32 / u32_to_word): the float's bit pattern, the double's value
__device__ __forceinline__ uint32_t elem_u32(const uint32_t* w, int rsz) { return rsz == 4 ? w[0] : (uint32_t)__hiloint2double((int)w[1], (int)w[0]); }
__device__ __forceinline__ void set_elem_u32(uint32_t* w, int rsz, uint32_t u) {
  if (rsz == 4) { w[0] = u; return; }
  const double d = (double)u;
  w[0] = (uint32_t)__double2loint(d); w[1] = (uint32_t)__double2hiint(d);
}
// adds `delta` to every clock-relative field of a row: -clock makes them relative (pack), +clock re-bases them (unpack)
__device__ __forceinline__ void rebase_row(const RecArgs& a, uint32_t* row, uint32_t delta) {
  for (int s = 0; s < a.n_sec; ++s) {
    const RecSec& S = a.sec[s];
    uint32_t* w = row + S.row_off;
    if (S.clk == kClkCold) {  // cold record [omega | sigma or periodic start per slot | sub-episode end per slot]
      const int wpe = a.rsz / 4;
      for (int r = 0; r < a.n_ref; ++r) {
        uint32_t* end = w + (1 + a.n_ref + r) * wpe;
        set_elem_u32(end, a.rsz, elem_u32(end, a.rsz) + delta);
        const unsigned g = (a.sw_count[r] > 1 && a.swst_off >= 0) ? row[a.swst_off + 2 * r] : (unsigned)r;  // the slot's current generator
        if (g < (unsigned)kMaxRefEntries && a.ref_kind[g] >= GEMB200_REF_SINUS) {
          uint32_t* start = w + (1 + r) * wpe;
          set_elem_u32(start, a.rsz, elem_u32(start, a.rsz) + delta);
        }
      }
    } else if (S.clk == kClkSwst) {  // [n_ref][2]: parameter entry, super-episode end
      for (int r = 0; r < a.n_ref; ++r) w[2 * r + 1] += delta;
    }
  }
}

__global__ void __launch_bounds__(kRecBlockMax) pack_envs_kernel(const RecArgs a, const int32_t* __restrict__ env_idx, int m, uint32_t* __restrict__ rows) {
  extern __shared__ uint32_t srow[];
  __shared__ int ok[kRecBlockMax];
  const int t = threadIdx.x, j0 = blockIdx.x * blockDim.x, j = j0 + t;
  bool valid = false;
  if (j < m) {
    const int i = env_idx ? env_idx[j] : j;
    valid = i >= 0 && i < a.n;
    if (valid) {
      uint32_t kstep;
      int ring;
      rec_clock(a, &kstep, &ring);
      uint32_t* row = srow + t * a.stride;
      move_env<true>(a, (unsigned)i, ring, row);
      rebase_row(a, row, 0u - kstep);
    }
  }
  ok[t] = valid;
  __syncthreads();
  const unsigned total = (unsigned)min((int)blockDim.x, m - j0) * (unsigned)a.words;
  uint32_t* dst = rows + (size_t)j0 * a.words;
  for (unsigned k = t; k < total; k += blockDim.x) {
    const unsigned e = __umulhi(k, a.div_magic), w = k - e * a.words;
    if (ok[e]) dst[k] = srow[e * a.stride + w];
  }
}

__global__ void __launch_bounds__(kRecBlockMax) unpack_envs_kernel(const RecArgs a, const uint32_t* __restrict__ rows, int n_rows, const int32_t* __restrict__ row_idx,
                                                                  const int32_t* __restrict__ env_idx, int m) {
  extern __shared__ uint32_t srow[];
  __shared__ int src[kRecBlockMax];
  const int t = threadIdx.x, j0 = blockIdx.x * blockDim.x, j = j0 + t;
  int i = -1, r = -1;
  if (j < m) {
    r = row_idx ? row_idx[j] : j;
    i = env_idx ? env_idx[j] : j;
    if (r < 0 || r >= n_rows || i < 0 || i >= a.n) r = -1;
  }
  src[t] = r;
  __syncthreads();
  const unsigned total = (unsigned)min((int)blockDim.x, m - j0) * (unsigned)a.words;
  for (unsigned k = t; k < total; k += blockDim.x) {
    const unsigned e = __umulhi(k, a.div_magic), w = k - e * a.words;
    const int rr = src[e];
    if (rr >= 0) srow[e * a.stride + w] = __ldg(rows + (size_t)rr * a.words + w);
  }
  __syncthreads();
  if (r >= 0) {
    uint32_t kstep;
    int ring;
    rec_clock(a, &kstep, &ring);
    uint32_t* row = srow + t * a.stride;
    rebase_row(a, row, kstep);
    move_env<false>(a, (unsigned)i, ring, row);
    if (a.rngid) set_own_rng_id(a.rngid, (size_t)a.n, (unsigned)i, a.seed_lo, a.seed_hi, a.env_offset);
  }
}

// FNV-1a over what decides the row format (include/gemb200.h); n_envs, seed, offsets, tau, parameters, reward, ... stay out, so rows move
// between handles of one env that differ in size or seed
static uint64_t record_layout_id(const gemb200_config* c, int words) {
  Dims d;
  derive_dims(c, &d);
  uint64_t x = 1469598103934665603ull;
  auto mix = [&](int64_t v) { for (int b = 0; b < 8; ++b) { x ^= (uint64_t)(v >> (8 * b)) & 0xffu; x *= 1099511628211ull; } };
  mix(0x47454D5245434F52ll);  // format tag
  mix(words);
  mix(c->dtype); mix(c->motor_kind); mix(d.n_ode); mix(c->n_ref);
  int n_entries = c->n_ref;
  for (int r = 0; r < c->n_ref; ++r) {
    const bool sw = c->ref_sw_count[r] > 1;
    mix(sw ? c->ref_sw_count[r] : 0); mix(sw ? c->ref_sw_first[r] : 0);
    if (sw && c->ref_sw_first[r] + c->ref_sw_count[r] > n_entries) n_entries = c->ref_sw_first[r] + c->ref_sw_count[r];
  }
  for (int e = 0; e < n_entries; ++e) mix(c->ref_kind[e]);
  mix(has_sw_state(c));
  mix(c->dead_time_steps); mix(c->dead_time_steps > 0 ? c->dead_time_outer : 0); mix(fifo_dim_of(c, d));
  mix(c->n_state_ops);
  for (int k = 0; k < c->n_state_ops; ++k) mix(c->sop_kind[k]);
  mix(c->supply_kind);
  mix(c->load_kind == GEMB200_LOAD_EXT_SPEED);
  mix(c->init_im_valid);
  return x;
}
static int record_words(const gemb200_config* c) {
  Section s[kMaxSections];
  const int k = config_sections(c, nullptr, s);
  int w = 0;
  for (int q = 0; q < k; ++q) w += row_words(s[q]);
  return w;
}
static void record_args(gemb200_handle* h, RecArgs* a) {
  std::memset(a, 0, sizeof(*a));
  Section s[kMaxSections];
  const int k = sections(h, s);
  int off = 0;
  a->swst_off = -1;
  for (int q = 0; q < k; ++q) {
    a->sec[q] = {static_cast<char*>(*s[q].slot), s[q].esz, s[q].per_env, s[q].place, s[q].clk, off};
    if (s[q].clk == kClkSwst) a->swst_off = off;
    off += row_words(s[q]);
  }
  a->n_sec = k; a->n = h->cfg.n_envs; a->words = off; a->stride = off | 1;
  a->div_magic = (uint32_t)((((uint64_t)1 << 32) + (uint64_t)off - 1) / (uint64_t)off);  // words >= 2: hot and cold record
  a->rsz = (int)h->rsz; a->n_ref = h->n_ref; a->dead = h->cfg.dead_time_steps; a->fifo_dim = h->fifo_dim;
  for (int r = 0; r < kMaxRef; ++r) a->sw_count[r] = (r < h->n_ref && h->cfg.ref_sw_count[r] > 1) ? h->cfg.ref_sw_count[r] : 0;
  for (int e = 0; e < kMaxRefEntries; ++e) a->ref_kind[e] = h->cfg.ref_kind[e];
  a->kstep = (uint32_t)h->n_steps;
  a->ring = a->dead > 0 ? (int)(h->n_steps % (uint64_t)a->dead) : 0;
  a->clock_dev = h->dev_clock ? h->d_clock : nullptr;
  a->rngid = h->ids_in_use ? h->d_rngid : nullptr;
  a->seed_lo = (uint32_t)h->cfg.seed; a->seed_hi = (uint32_t)(h->cfg.seed >> 32);
  a->env_offset = h->cfg.env_index_offset;
}
static int record_block(int stride) {  // largest block whose rows fit the default 48 KB of shared memory
  for (int b = kRecBlockMax; b >= 32; b >>= 1)
    if ((size_t)b * (size_t)stride * sizeof(uint32_t) <= 48 * 1024) return b;
  return 0;
}

// the state rows of gemb200_pack_envs / gemb200_unpack_envs, without their refusal under parameter draws
static int pack_env_rows(gemb200_handle* h, const int32_t* env_idx, int32_t m, uint32_t* rows, void* stream) {
  if (m < 0) return fail(GEMB200_E_INVALID, "m must be >= 0");
  if (m == 0) return GEMB200_OK;
  if (!rows) return fail(GEMB200_E_INVALID, "rows is NULL");
  DeviceGuard guard(h->cfg.device);
  RecArgs a;
  record_args(h, &a);
  const int block = record_block(a.stride);
  if (!block) return fail(GEMB200_E_INVALID, "packed env record too long for the shared-memory staging");
  const int grid = (int)(((int64_t)m + block - 1) / block);
  pack_envs_kernel<<<grid, block, (size_t)block * a.stride * sizeof(uint32_t), (cudaStream_t)stream>>>(a, env_idx, m, rows);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return GEMB200_OK;
}
// refuses rows of another record layout before anything else
static int check_row_layout(gemb200_handle* h, uint64_t layout_id) {
  if (layout_id != record_layout_id(&h->cfg, record_words(&h->cfg)))
    return fail(GEMB200_E_INVALID, "unpack: the rows were packed from a handle with another record layout (motor, dtype, generators, dead time, ...)");
  return GEMB200_OK;
}
static int unpack_env_rows(gemb200_handle* h, const uint32_t* rows, int32_t n_rows, uint64_t layout_id, const int32_t* row_idx,
                           const int32_t* env_idx, int32_t m, void* stream) {
  if (m < 0 || n_rows < 0) return fail(GEMB200_E_INVALID, "m and n_rows must be >= 0");
  RecArgs a;
  record_args(h, &a);
  if (layout_id != record_layout_id(&h->cfg, a.words))
    return fail(GEMB200_E_INVALID, "unpack: the rows were packed from a handle with another record layout (motor, dtype, generators, dead time, ...)");
  if (m == 0 || n_rows == 0) return GEMB200_OK;
  if (!rows) return fail(GEMB200_E_INVALID, "rows is NULL");
  DeviceGuard guard(h->cfg.device);
  const int block = record_block(a.stride);
  if (!block) return fail(GEMB200_E_INVALID, "packed env record too long for the shared-memory staging");
  const int grid = (int)(((int64_t)m + block - 1) / block);
  unpack_envs_kernel<<<grid, block, (size_t)block * a.stride * sizeof(uint32_t), (cudaStream_t)stream>>>(a, rows, n_rows, row_idx, env_idx, m);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return GEMB200_OK;
}

extern "C" {

int gemb200_query_env_record(const gemb200_config* cfg, int32_t* words, uint64_t* layout_id) {
  int rc = validate(cfg);
  if (rc) return rc;
  const int w = record_words(cfg);
  if (words) *words = w;
  if (layout_id) *layout_id = record_layout_id(cfg, w);
  return GEMB200_OK;
}

int gemb200_pack_envs(gemb200_handle* h, const int32_t* env_idx, int32_t m, uint32_t* rows, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (draws_on(h)) return fail(GEMB200_E_INVALID, "snapshot rows do not carry the parameters drawn per reset; switch the draws off first (DESIGN §7)");
  return pack_env_rows(h, env_idx, m, rows, stream);
}

int gemb200_unpack_envs(gemb200_handle* h, const uint32_t* rows, int32_t n_rows, uint64_t layout_id, const int32_t* row_idx,
                        const int32_t* env_idx, int32_t m, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (draws_on(h)) return fail(GEMB200_E_INVALID, "snapshot rows do not carry the parameters drawn per reset; switch the draws off first (DESIGN §7)");
  return unpack_env_rows(h, rows, n_rows, layout_id, row_idx, env_idx, m, stream);
}

}  // extern "C"

// ----------------------------------------------------------------------------------------------------------------
// RNG identities (gemb200_pack_rng_ids / gemb200_adopt_rng_ids / gemb200_clear_rng_ids; row format in include/gemb200.h)
// ----------------------------------------------------------------------------------------------------------------
static_assert(kRngIdWords == GEMB200_RNG_ID_WORDS, "RNG identity row width");
// the handle's clock as the identities see it: the call id of the NEXT call and the step count, from the host counters or d_clock
struct IdClockArgs { uint64_t call; uint32_t steps; const uint32_t* dev; };
__device__ __forceinline__ void id_clock_now(const IdClockArgs& c, uint64_t* call, uint32_t* steps) {
  if (c.dev) { *call = ((uint64_t)c.dev[1] << 32) | c.dev[0]; *steps = c.dev[2]; }
  else { *call = c.call; *steps = c.steps; }
}
static IdClockArgs id_clock_args(const gemb200_handle* h) { return IdClockArgs{h->gstep + 1, (uint32_t)h->n_steps, h->dev_clock ? h->d_clock : nullptr}; }

__global__ void own_rng_ids_kernel(uint32_t* ids, int n, uint32_t seed_lo, uint32_t seed_hi, int64_t env_offset) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) set_own_rng_id(ids, (size_t)n, (unsigned)i, seed_lo, seed_hi, env_offset);
}
// one thread per output word: row j of env env_idx[j] = its effective identity (ids NULL: every env has its own), the rows written contiguously
__global__ void pack_rng_ids_kernel(const uint32_t* __restrict__ ids, int n, uint32_t seed_lo, uint32_t seed_hi, int64_t env_offset, const IdClockArgs c,
                                    const int32_t* __restrict__ env_idx, int m, uint32_t* __restrict__ out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= (int64_t)m * kRngIdWords) return;
  const int j = (int)(k / kRngIdWords), w = (int)(k % kRngIdWords);
  const int i = env_idx ? env_idx[j] : j;
  if (i < 0 || i >= n) return;
  const size_t nn = (size_t)n;
  const uint64_t g = (uint64_t)(env_offset + i);
  uint64_t call;
  uint32_t steps, v = 0u;
  id_clock_now(c, &call, &steps);
  if (w < 4) v = ids ? ids[w * nn + i] : (w == 0 ? seed_lo : (w == 1 ? seed_hi : (w == 2 ? (uint32_t)g : (uint32_t)(g >> 32))));
  else if (w < 6) {
    const uint64_t e = call + (ids ? (((uint64_t)ids[5 * nn + i] << 32) | ids[4 * nn + i]) : 0u);
    v = w == 4 ? (uint32_t)e : (uint32_t)(e >> 32);
  } else if (w == 6) v = steps + (ids ? ids[6 * nn + i] : 0u);
  out[k] = v;
}
// env env_idx[j] takes identity row row_idx[j]: its key and global index, and offsets that map this handle's clock onto the source's
__global__ void adopt_rng_ids_kernel(uint32_t* __restrict__ ids, int n, const IdClockArgs c, const uint32_t* __restrict__ rows, int n_rows,
                                     const int32_t* __restrict__ row_idx, const int32_t* __restrict__ env_idx, int m) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const int r = row_idx ? row_idx[j] : j, i = env_idx ? env_idx[j] : j;
  if (r < 0 || r >= n_rows || i < 0 || i >= n) return;
  uint32_t w[kRngIdWords];
#pragma unroll
  for (int q = 0; q < kRngIdWords; ++q) w[q] = __ldg(rows + (size_t)r * kRngIdWords + q);
  uint64_t call;
  uint32_t steps;
  id_clock_now(c, &call, &steps);
  const uint64_t dcall = (((uint64_t)w[5] << 32) | w[4]) - call;
  const size_t nn = (size_t)n;
  ids[i] = w[0]; ids[nn + i] = w[1]; ids[2 * nn + i] = w[2]; ids[3 * nn + i] = w[3];
  ids[4 * nn + i] = (uint32_t)dcall; ids[5 * nn + i] = (uint32_t)(dcall >> 32); ids[6 * nn + i] = w[6] - steps; ids[7 * nn + i] = 0u;
}

static int launch_own_rng_ids(gemb200_handle* h, cudaStream_t st) {
  const int n = h->cfg.n_envs;
  own_rng_ids_kernel<<<(n + 255) / 256, 256, 0, st>>>(h->d_rngid, n, (uint32_t)h->cfg.seed, (uint32_t)(h->cfg.seed >> 32), h->cfg.env_index_offset);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return GEMB200_OK;
}

// gemb200_adopt_rng_ids without its refusals (layout, parameter draws)
static int adopt_rng_id_rows(gemb200_handle* h, const uint32_t* ids, int32_t n_ids, const int32_t* row_idx, const int32_t* env_idx, int32_t m,
                             cudaStream_t st) {
  if (m < 0 || n_ids < 0) return fail(GEMB200_E_INVALID, "m and n_ids must be >= 0");
  if (m == 0 || n_ids == 0) return GEMB200_OK;
  if (!ids) return fail(GEMB200_E_INVALID, "ids is NULL");
  DeviceGuard guard(h->cfg.device);
  if (h->blocks == kBlocksNone) {  // first adoption: the shared parameters into per-env blocks, so that the handle runs the ENVP instantiations (synchronises)
    const int rc = fill_shared_blocks(h);
    if (rc) return rc;
    h->blocks = kBlocksShared;
  }
  if (!h->d_rngid) CUDA_TRY(cudaMalloc(&h->d_rngid, (size_t)kRngIdWords * (size_t)h->cfg.n_envs * sizeof(uint32_t)));
  if (!h->ids_in_use) {  // every other env keeps its own identity
    const int rc = launch_own_rng_ids(h, st);
    if (rc) return rc;
    h->ids_in_use = true;
  }
  apply_mode(h);
  adopt_rng_ids_kernel<<<(m + 255) / 256, 256, 0, st>>>(h->d_rngid, h->cfg.n_envs, id_clock_args(h), ids, n_ids, row_idx, env_idx, m);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return GEMB200_OK;
}

extern "C" {

int gemb200_pack_rng_ids(gemb200_handle* h, const int32_t* env_idx, int32_t m, uint32_t* ids, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (m < 0) return fail(GEMB200_E_INVALID, "m must be >= 0");
  if (m == 0) return GEMB200_OK;
  if (!ids) return fail(GEMB200_E_INVALID, "ids is NULL");
  DeviceGuard guard(h->cfg.device);
  const int64_t words = (int64_t)m * kRngIdWords;
  pack_rng_ids_kernel<<<(unsigned)((words + 255) / 256), 256, 0, (cudaStream_t)stream>>>(h->ids_in_use ? h->d_rngid : nullptr, h->cfg.n_envs, (uint32_t)h->cfg.seed,
                                                                                        (uint32_t)(h->cfg.seed >> 32), h->cfg.env_index_offset, id_clock_args(h), env_idx, m, ids);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return GEMB200_OK;
}

int gemb200_adopt_rng_ids(gemb200_handle* h, const uint32_t* ids, int32_t n_ids, const int32_t* row_idx, const int32_t* env_idx, int32_t m, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (h->cfg.layout != GEMB200_LAYOUT_AOS)
    return fail(GEMB200_E_INVALID, "adopted RNG identities are read by the per-env parameter instantiations, which need the row-per-env (AoS) I/O layout (DESIGN §7)");
  if (draws_on(h)) return fail(GEMB200_E_INVALID, "RNG identities cannot be adopted while parameters are drawn per reset: snapshots are refused then (DESIGN §7)");
  return adopt_rng_id_rows(h, ids, n_ids, row_idx, env_idx, m, (cudaStream_t)stream);
}

int gemb200_clear_rng_ids(gemb200_handle* h, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  (void)stream;  // launches enqueued before the call keep the identities they were launched with
  drop_rng_ids(h);
  return GEMB200_OK;
}

}  // extern "C"

// ----------------------------------------------------------------------------------------------------------------
// Per-env physical parameters in snapshots (gemb200_pack_envs_params / gemb200_unpack_envs_params; row format in include/gemb200.h)
// ----------------------------------------------------------------------------------------------------------------
// A parameter row is the env's praw column: kMaxDraw doubles.  Both kernels stage a block's rows in shared memory like pack_envs_kernel /
// unpack_envs_kernel: the planar praw[kMaxDraw][n] is read and written with consecutive threads on consecutive envs, the [m][kMaxDraw]
// rows word-contiguously by the whole block.
static_assert(kMaxDraw == GEMB200_ENV_PARAM_SLOTS, "parameter row width");
constexpr int kParBlock = 128;
constexpr int kParStride = kMaxDraw + 1;  // odd stride in doubles: a half-warp's 8-byte shared accesses to its rows hit distinct banks

// rows[j] = parameters of env env_idx[j] (NULL: j); praw NULL (a handle without per-env blocks): the configuration's, from `cfg`
__global__ void __launch_bounds__(kParBlock) pack_env_params_kernel(const double* __restrict__ praw, const RawParams cfg, int n,
                                                                    const int32_t* __restrict__ env_idx, int m, double* __restrict__ rows) {
  __shared__ double srow[kParBlock * kParStride];
  __shared__ int ok[kParBlock];
  const int t = threadIdx.x, j0 = blockIdx.x * kParBlock, j = j0 + t;
  bool valid = false;
  if (j < m) {
    const int i = env_idx ? env_idx[j] : j;
    valid = i >= 0 && i < n;
    if (valid) {
      double* row = srow + t * kParStride;
      if (praw) {
        for (int s = 0; s < kMaxDraw; ++s) row[s] = praw[(size_t)s * n + i];
      } else {
        for (int s = 0; s < kMaxDraw; ++s) row[s] = cfg.v[s];
      }
    }
  }
  ok[t] = valid;
  __syncthreads();
  const int total = min(kParBlock, m - j0) * kMaxDraw;
  double* dst = rows + (size_t)j0 * kMaxDraw;
  for (int k = t; k < total; k += kParBlock) {
    const int e = k / kMaxDraw, w = k - e * kMaxDraw;
    if (ok[e]) dst[k] = srow[e * kParStride + w];
  }
}

// Env i's column of the per-env parameter block envp [kCoefWords][n], derived from its physical parameters prm[kMaxDraw] by derive_coef
// (gemb200_model.h), the derivation of the parameter draws and of gemb200_set_env_params.  The same stores end redraw_env_params
// (gemb200_kernels.cuh); calling this function from there changes the register allocation of every reset kernel and ENVP step / rollout
// kernel of the step translation units (DESIGN §4), so the eight lines are kept in both places.
template <typename real>
__device__ __forceinline__ void write_env_coef(int motor_kind, const double* prm, real* envp, unsigned i, size_t n) {
  ModelCoef mc;
  derive_coef(motor_kind, prm, prm + GEMB200_MAX_MOTOR_PARAM, &mc);
  real* e = envp + i;
  for (int w = 0; w < 20; ++w) e[(size_t)w * n] = (real)mc.c[w];
  for (int w = 0; w < 4; ++w) e[(size_t)(20 + w) * n] = (real)mc.tq[w];
  e[(size_t)24 * n] = (real)prm[GEMB200_MAX_MOTOR_PARAM + GEMB200_LP_A];
  e[(size_t)25 * n] = (real)prm[GEMB200_MAX_MOTOR_PARAM + GEMB200_LP_B];
  e[(size_t)26 * n] = (real)prm[GEMB200_MAX_MOTOR_PARAM + GEMB200_LP_C];
  e[(size_t)27 * n] = (real)mc.inv_j; e[(size_t)28 * n] = (real)mc.omega_lim; e[(size_t)29 * n] = (real)mc.omega_lin;
}

// env env_idx[j] (NULL: j) takes parameter row row_idx[j] (NULL: j): every slot but the pole pairs (per handle: the angle increments are
// prepared on the host) into praw, and the coefficients derived from them into its envp column (write_env_coef, as a parameter draw does)
template <typename real>
__global__ void __launch_bounds__(kParBlock) adopt_env_params_kernel(double* __restrict__ praw, real* __restrict__ envp, int n, int motor_kind,
                                                                     const double* __restrict__ rows, int n_rows, const int32_t* __restrict__ row_idx,
                                                                     const int32_t* __restrict__ env_idx, int m) {
  __shared__ double srow[kParBlock * kParStride];
  __shared__ int src[kParBlock];
  const int t = threadIdx.x, j0 = blockIdx.x * kParBlock, j = j0 + t;
  int i = -1, r = -1;
  if (j < m) {
    r = row_idx ? row_idx[j] : j;
    i = env_idx ? env_idx[j] : j;
    if (r < 0 || r >= n_rows || i < 0 || i >= n) r = -1;
  }
  src[t] = r;
  __syncthreads();
  const int total = min(kParBlock, m - j0) * kMaxDraw;
  for (int k = t; k < total; k += kParBlock) {
    const int e = k / kMaxDraw, w = k - e * kMaxDraw;
    const int rr = src[e];
    if (rr >= 0) srow[e * kParStride + w] = __ldg(rows + (size_t)rr * kMaxDraw + w);
  }
  __syncthreads();
  if (r < 0) return;
  const size_t nn = (size_t)n;
  const double* row = srow + t * kParStride;
  double prm[kMaxDraw];
#pragma unroll
  for (int s = 0; s < kMaxDraw; ++s) prm[s] = row[s];
  prm[GEMB200_MP_P] = praw[(size_t)GEMB200_MP_P * nn + i];
#pragma unroll
  for (int s = 0; s < kMaxDraw; ++s)
    if (s != GEMB200_MP_P) praw[(size_t)s * nn + i] = prm[s];
  write_env_coef<real>(motor_kind, prm, envp, (unsigned)i, nn);
}

extern "C" {

int gemb200_pack_envs_params(gemb200_handle* h, const int32_t* env_idx, int32_t m, uint32_t* rows, double* params, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (h->cfg.layout != GEMB200_LAYOUT_AOS) return fail(GEMB200_E_INVALID, "parameter rows need the row-per-env (AoS) I/O layout (per-env parameter blocks)");
  if (!rows || !params) return fail(GEMB200_E_INVALID, "rows and params are required");
  const int rc = pack_env_rows(h, env_idx, m, rows, stream);
  if (rc || m == 0) return rc;
  DeviceGuard guard(h->cfg.device);
  pack_env_params_kernel<<<(m + kParBlock - 1) / kParBlock, kParBlock, 0, (cudaStream_t)stream>>>(
      h->blocks != kBlocksNone ? h->d_praw : nullptr, config_params(h), h->cfg.n_envs, env_idx, m, params);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return GEMB200_OK;
}

int gemb200_unpack_envs_params(gemb200_handle* h, const uint32_t* rows, const double* params, const uint32_t* ids, int32_t n_rows,
                               uint64_t layout_id, const int32_t* row_idx, const int32_t* env_idx, int32_t m, void* stream) {
  if (!h) return fail(GEMB200_E_INVALID, "handle is NULL");
  if (h->cfg.layout != GEMB200_LAYOUT_AOS) return fail(GEMB200_E_INVALID, "parameter rows need the row-per-env (AoS) I/O layout (per-env parameter blocks)");
  if (!rows || !params) return fail(GEMB200_E_INVALID, "rows and params are required");
  if (m < 0 || n_rows < 0) return fail(GEMB200_E_INVALID, "m and n_rows must be >= 0");
  int rc = check_row_layout(h, layout_id);
  if (rc || m == 0 || n_rows == 0) return rc;
  DeviceGuard guard(h->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  if (h->blocks == kBlocksNone) {  // no per-env blocks yet: every other env keeps the shared parameters (synchronises)
    rc = fill_shared_blocks(h);
    if (rc) return rc;
  }
  h->blocks = kBlocksCaller;  // the blocks hold rows of the caller's now
  apply_mode(h);
  rc = unpack_env_rows(h, rows, n_rows, layout_id, row_idx, env_idx, m, stream);
  if (rc) return rc;
  with_params(h, [&](auto& p) {
    using real = decltype(p.tau);
    adopt_env_params_kernel<real><<<(m + kParBlock - 1) / kParBlock, kParBlock, 0, st>>>(h->d_praw, static_cast<real*>(h->d_envp), h->cfg.n_envs,
                                                                                          h->cfg.motor_kind, params, n_rows, row_idx, env_idx, m);
  });
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  return ids ? adopt_rng_id_rows(h, ids, n_rows, row_idx, env_idx, m, st) : GEMB200_OK;
}

}  // extern "C"
