// gemb200_params.h — kernel parameter block (passed by value in the kernel-parameter constant bank).
//
// Everything a thread needs besides its own env's state is here, so a launch reads no global-memory parameter
// table: uniform operands come straight from the constant bank (c[0x0][...]) at no issue cost.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace gemb200 {

constexpr int kMaxState = 28;
constexpr int kMaxRef = 4;          // referenced states = output slots
constexpr int kMaxRefEntries = 12;  // generator parameter entries (slots + switched sub-generators)
constexpr int kMaxConstraints = 4;
constexpr int kMaxStateOps = 4;
constexpr int kMaxX = 6;  // real-typed ODE states per env (omega + motor states without the angle): SCIM 5

// words of persistent state per env and their placement (shared by host and device code)
// Two records per env: HOT (read and written every step): currents/fluxes x_1.. and the reference values;
// COLD (read every step, written only when it changes): omega (constant-speed load), the Wiener sigmas and the absolute step
// index at which each sub-episode ends.  Skipping the unchanged words saves 16 B of the 109 B written per PMSM env-step.
__host__ __device__ constexpr int hot_words(int nx, int nref) { return nx - 1 + nref; }
__host__ __device__ constexpr int cold_words(int nx, int nref) { (void)nx; return 1 + 2 * nref; }
// element offset (in units of `real`) of word w of env i; vw = 16 / sizeof(real) words per 16-byte chunk
__host__ __device__ inline size_t word_offset(int w, size_t i, size_t n, int W, int vw) {
  const int nfull = (W / vw) * vw;
  if (w < nfull) return (size_t)(w / vw) * vw * n + i * vw + (w % vw);
  int rem = W - nfull, base = nfull;  // remaining words: for vw == 4 an optional 2-word chunk, then an optional 1-word chunk
  if (vw == 4 && rem >= 2) {
    if (w < base + 2) return (size_t)base * n + i * 2 + (w - base);
    base += 2;
  }
  return (size_t)base * n + i + (w - base);
}

// Motor families = template specialisations of the step kernel.
enum MotorFamily : int {
  kDC1 = 0,   // one armature current: PermEx, Series       state [omega, torque, i, u, u_sup]
  kDC2 = 1,   // two currents: Shunt (+i_sum), ExtEx         state [omega, torque, i_a, i_e, u(_a), (u_e,) u_sup(, i_sum)]
  kSYNC = 2,  // PMSM, SynRM                                 14 states
  kEESM = 3,  // 16 states
  kSCIM = 4,  // 14 states
  kDFIM = 5   // 24 states: SCIM model + rotor voltages from a second B6 bridge
};

// RNG stream ids (word 3 of the Philox counter); shared convention with the test oracle.
enum : uint32_t {
  kStreamWalk = 1, kStreamSubep = 2, kStreamInit = 3, kStreamSubepHi = 18,
  kStreamWalkR = 5, kStreamSubepR = 6, kStreamSubepHiR = 22,  // "R": draws made right after an in-kernel auto-reset
  kStreamInitState = 7, kStreamInitState2 = 8,                // random initial ODE state
  kStreamSwitch = 10, kStreamSwitchR = 14,                    // + slot: SwitchedReferenceGenerator super-episode (R: at a reset)
  kStreamSupply = 9,                                          // AC supply phase at reset
  kStreamWalk2 = 4,                                           // walk increments of envs with <= 2 reference slots: ONE block serves two
                                                              //   consecutive call ids (counter words 0,1 = id >> 1, word pair = id & 1)
  kStreamLaplace = 24, kStreamLaplaceR = 28,                  // Laplace walk increments (R: right after an in-kernel auto-reset)
  kStreamPeriodic = 32,                                       // + 2*slot (+1): sub-episode parameters of the periodic generators,
                                                              //   counter word 0 = step index of the sub-episode start
  kStreamParam = 40, kStreamParamR = 48,                      // + j/4: parameter draws at a reset (reset_kernel; R: in-kernel auto-reset),
                                                              //   one block of four uniforms per four drawn parameters
  kStreamNoise = 64,                                          // + 8*op + (state index >> 2): StateNoiseProcessor draws
  kStreamNoiseR = 128                                         //   ... right after an in-kernel auto-reset
};

// physical parameter slots of one env: GEMB200_MAX_MOTOR_PARAM motor slots, then 8 load slots (gemb200_set_param_randomization)
constexpr int kMaxDraw = 16 + 8;

// every stream id (base + its offsets) is used by exactly one consumer: ranges [base, base + width)
constexpr bool streams_disjoint() {
  constexpr uint32_t r[][2] = {{kStreamWalk, 1}, {kStreamSubep, 1}, {kStreamInit, 1}, {kStreamWalkR, 1}, {kStreamSubepR, 1}, {kStreamInitState, 1}, {kStreamInitState2, 1},
                               {kStreamSupply, 1}, {kStreamSwitch, kMaxRef}, {kStreamSwitchR, kMaxRef}, {kStreamSubepHi, 1}, {kStreamSubepHiR, 1}, {kStreamLaplace, 1},
                               {kStreamLaplaceR, 1}, {kStreamWalk2, 1}, {kStreamPeriodic, 2 * kMaxRef}, {kStreamNoise, 8 * kMaxStateOps}, {kStreamNoiseR, 8 * kMaxStateOps},
                               {kStreamParam, (kMaxDraw + 3) / 4}, {kStreamParamR, (kMaxDraw + 3) / 4}};
  constexpr int n = sizeof(r) / sizeof(r[0]);
  for (int a = 0; a < n; ++a)
    for (int b = a + 1; b < n; ++b)
      if (r[a][0] < r[b][0] + r[b][1] && r[b][0] < r[a][0] + r[a][1]) return false;
  for (int a = 0; a < n; ++a)
    if (r[a][0] + r[a][1] > 256) return false;  // the id shares counter word 3 with the high bits of the env index: 8 bits
  return true;
}
static_assert(streams_disjoint(), "RNG stream id ranges overlap");

// Model coefficients of ONE env: the motor's sparse constant matrix (layout per family, gemb200_model.h: derive_coef), torque coefficients,
// load polynomial and inertia.  Shared by the whole batch in the constant bank (StepParams::k) — or, with per-env parameter blocks
// (gemb200_set_env_params: domain randomisation), loaded per thread from StepParams::envp.
// The same 30 words are a per-env block's column: word w of Coef is word w of the block (c at 0, tq at kCwTq, then the six load words a, b, c,
// inv_j, omega_lim, omega_lin at kCwLoad ..  kCwLoad + 5).
constexpr int kCoefWords = 30, kCwTq = 20, kCwLoad = 24;
template <typename real>
struct Coef {
  real c[20];  // motor model coefficients
  real tq[4];  // torque coefficients
  real load_a, load_b, load_c, inv_j, omega_lim, omega_lin;
};
template <typename real>
constexpr bool coef_layout() {
  return offsetof(Coef<real>, tq) == kCwTq * sizeof(real) && offsetof(Coef<real>, load_a) == kCwLoad * sizeof(real) &&
         offsetof(Coef<real>, omega_lin) == (kCwLoad + 5) * sizeof(real) && sizeof(Coef<real>) == kCoefWords * sizeof(real);
}
static_assert(coef_layout<float>() && coef_layout<double>(), "Coef is the word order of a per-env block");
// the words of c and of tq that family fam reads (derive_coef leaves the others 0)
__host__ __device__ constexpr int coef_nc(int fam) { return fam == kDC1 ? 4 : (fam == kDC2 ? 5 : (fam == kSYNC ? 7 : (fam == kEESM ? 14 : 10))); }
__host__ __device__ constexpr int coef_ntq(int fam) { return (fam == kDC2 || fam == kSCIM || fam == kDFIM) ? 1 : 2; }

// Distributions of the parameters drawn at every reset (gemb200_set_param_randomization), in device memory behind StepParams::draw.
// Draw j: v = a + b * U (uniform: a = lo, b = hi - lo; log-uniform: exp of it, a = log lo, b = log hi - log lo), clamped to [lo, hi].
struct ParamDraw {
  int32_t slot[kMaxDraw];  // parameter slot: GEMB200_MP_* or GEMB200_MAX_MOTOR_PARAM + GEMB200_LP_*
  int32_t kind[kMaxDraw];  // GEMB200_DIST_*
  double a[kMaxDraw], b[kMaxDraw], lo[kMaxDraw], hi[kMaxDraw];
};

template <typename real>
struct StepParams {
  // ---- batch ----
  int32_t n;              // envs in this handle
  int32_t env_begin, env_end;  // sub-range of envs processed by this launch (chunked host-buffer pipeline); default [0, n)
  int64_t env_offset;     // global index of env 0 (sharding)
  uint32_t seed_lo, seed_hi;
  uint32_t rk[10][2];     // Philox4x32-10 round keys: seed + r * (0x9E3779B9, 0xBB67AE85)
  uint32_t gstep_lo, gstep_hi;  // unique id of this API call (reset or step): RNG counter words 0,1
  // ---- persistent per-env state (owned by the handle) ----
  // `st`  (hot):  [x_1..x_{NX-1} | ref value per slot]            hot_words() words per env
  // `stc` (cold): [omega | sigma per slot | sub-episode end per slot]  cold_words() words per env (ends are uint32 bit patterns)
  // Each record is stored as SoA of VECTOR CHUNKS (16-byte chunks first, then an 8-byte, then a 4-byte chunk) so that a thread
  // moves it with fully coalesced 128-bit accesses (see word_offset()).
  real* st;
  real* stc;
  uint32_t kstep;         // number of step calls so far: the clock of the sub-episode ends
  // Device-resident clock (gemb200_set_device_clock: launches that a CUDA graph can replay): {call id lo, hi, step count, dead-time ring
  // position} of the NEXT call, advanced by a one-thread kernel behind every launch; kstep then holds the bias (1: step, 0: reset) and the
  // gstep_* / fifo_slot fields are ignored.  nullptr: the clock comes from the host with every launch.
  const uint32_t* clock_dev;
  double* eps;            // [n]       electrical angle, wrapped to (-pi, pi]; nullptr for DC
  uint16_t* sw;           // [n] finite 2QC switching states, 2 bits per leg; nullptr unless finite && interlock
  real* fifo;             // [dead_steps][fifo_dim][n] DeadTimeProcessor action queue (ring, slot fifo_slot is oldest = next to overwrite)
  // ---- I/O of this call (caller-owned) ----
  const void* action;
  real* obs;
  real* ref_out;
  real* reward;
  uint8_t* term;
  const uint8_t* reset_mask;  // reset kernel only
  int32_t out_has;            // which of obs / ref_out / reward / term are requested (bits 0..3; set by the host with the pointers)
  // ---- system ----
  int32_t motor_kind;     // gemb200_motor_kind (runtime variant inside a family)
  int32_t conv_kind[2];
  int32_t load_kind;
  int32_t solver_kind;
  int32_t nsteps;
  int32_t autoreset;
  int32_t layout;         // gemb200_layout of the I/O tensors
  int32_t n_act;
  int32_t two_segment;    // finite && interlocking_time > 0
  int32_t action_dq;      // action given in dq coordinates (see gemb200_config::action_dq)
  int32_t dead_steps, dead_outer, fifo_dim, fifo_slot;
  real adv_k;             // angle advance per (rad/s) of omega, in the stored angle unit: angle_advance * tau * p (/2pi in turns)
  real inv_nsteps;
  real tau;               // step
  // interlocking time per converter slot (multi converters may give their sub-converters different ones, converters.py:615-740);
  // seg_len = lengths a switching segment can have: {tau, til0, tau - til0, til1, tau - til1, |til1 - til0|}; lo_slot = the slot with the
  // smaller time; promote = the legs of lo_slot reach their commanded state in a THIRD segment (|til1 - til0| > tau / 1000, converters.py:273)
  real til2[2];
  real tot2[2];           // til / tau per slot
  real seg_len[6];
  int32_t lo_slot, promote;
  real u_sup;
  // Electrical angle: d eps/dt = p * omega.  fp64 build: radians in a double.  fp32 build: TURNS as an unevaluated sum of two
  // floats (hi, lo) — "double-float", ~48 bits — so that neither fp64 arithmetic nor fp64<->fp32 conversions (slow XU-pipe
  // instructions) are needed.  kang[m][s] = factor that turns the integrator's omega sum of segment s
  // (index into seg_len) into the angle increment; m = 0: constant speed (sum = omega, factor = p*h_seg),
  // m = 1: sum over sub-steps (factor = p*h or p*h/6 for RK4); units: turns (fp32 build) or radians (fp64 build); [..][2] = hi, lo.
  real kang[2][6][2];
  real eps_out_scale;     // normalised angle output = (hi + lo) * eps_out_scale  (2*pi/limit in turns, 1/limit in radians)
  real init_ang[2];       // initial angle in the stored representation
  Coef<real> k;           // shared model coefficients
  const real* envp;       // [kCoefWords][n] per-env coefficients (word w of env i at envp[w * n + i]); nullptr: every env uses `k`
  real inv_lim[kMaxState];
  real init_x[kMaxX];
  real reset_obs[kMaxState];  // observation right after a reset (constant initial state)
  int32_t init_random;        // 1: uniform initial state per reset (init_lo + init_span * U); the angle entry [NX] is in the stored unit
  real init_lo[kMaxX + 1], init_span[kMaxX + 1];
  // truncated-normal initial states: x = mu + sigma * Phi^-1(ca + U * cspan), ca = Phi((lo - mu) / sigma); init_gauss = any such state
  // induction motors: flux bounds re-derived per env and reset (gemb200.h: init_im); im_prev = [2][n] initial currents of the env's previous
  // episode (what the reference keeps in _initial_states between initialize() calls); init_mid[j]: truncated normal around the interval's middle
  int32_t init_im_valid;
  real init_im[8];
  real* im_prev;
  int32_t init_mid[kMaxX + 1];
  int32_t init_gauss, init_dist[kMaxX + 1];
  real init_mu[kMaxX + 1], init_sigma[kMaxX + 1], init_ca[kMaxX + 1], init_cspan[kMaxX + 1];
  // ---- constraint monitor: merge = max, so all LimitConstraints collapse into ONE list of observed states; every
  //      SquaredConstraint keeps its own list ----
  int32_t n_lim;
  int32_t lim_idx[kMaxState];
  int32_t n_sq;
  int32_t sq_cnt[kMaxConstraints];
  int32_t sq_idx[kMaxConstraints][kMaxState];
  int32_t mon_off[4];     // PLAIN shape: BYTE offsets in the staged row of the <= 2 limit-checked states and of the squared constraint's two states (0 when unused)
  real mon_thr[3];        //              their thresholds: 1, or +inf for an unused check
  // ---- reward: sum of  w * (|s[idx] - ref| * inv_len)^pow.  Terms of referenced states are indexed by reference slot (the
  //      reference value is then a register); rw_* are the weighted states WITHOUT a reference (compared with 0) ----
  real rwr_w[kMaxRef], rwr_inv_len[kMaxRef], rwr_pow[kMaxRef];
  int32_t rwr_pow1[kMaxRef];
  int32_t n_rw;
  int32_t rw_state[kMaxState];
  int32_t rw_pow1[kMaxState];  // 1 if power == 1
  real rw_w[kMaxState];
  real rw_inv_len[kMaxState];
  real rw_pow[kMaxState];
  real bias, viol_reward;
  // ---- reference generators ----
  int32_t n_ref;
  int32_t any_wiener;
  int32_t ref_kind[kMaxRefEntries];
  int32_t ref_state[kMaxRefEntries];
  real ref_const[kMaxRefEntries];
  real ref_lo[kMaxRefEntries], ref_hi[kMaxRefEntries];
  real ref_init_lo[kMaxRefEntries], ref_init_span[kMaxRefEntries];
  real ref_lsig_lo[kMaxRefEntries], ref_lsig_span[kMaxRefEntries];  // log10 sigma range
  int32_t ref_len_lo[kMaxRefEntries], ref_len_span[kMaxRefEntries];
  // periodic generators (sinus / step / sawtooth / triangular): parameter ranges per slot, tau for the phase increment
  real ref_amp_lo[kMaxRefEntries], ref_amp_span[kMaxRefEntries], ref_freq_lo[kMaxRefEntries], ref_freq_span[kMaxRefEntries], ref_off_lo[kMaxRefEntries], ref_off_hi[kMaxRefEntries];
  real ref_tau;
  // SwitchedReferenceGenerator: output slot r switches between the parameter entries sw_first[r] .. +sw_count[r]-1 of the arrays above
  int32_t sw_count[kMaxRef], sw_first[kMaxRef], sw_len_lo[kMaxRef], sw_len_span[kMaxRef];
  real sw_cdf[kMaxRefEntries];
  uint32_t* swst;          // [n_ref][2][n]: current parameter entry, step at which the super-episode ends; nullptr unless switched
  // ---- state-vector wrappers (gemb200.h: gemb200_state_op), applied in order after the system's own vector is assembled ----
  int32_t n_sops;
  int32_t row_stride;      // shared-memory words per staged row: Fam::PAD without wrappers, else (final width | 1)
  int32_t n_obs;           // final width of the observation
  int32_t sop_kind[kMaxStateOps];
  int32_t sop_idx[kMaxStateOps][4];
  uint32_t sop_mask[kMaxStateOps];
  real sop_param[kMaxStateOps][8];
  // external speed profile (GEMB200_LOAD_EXT_SPEED): table of f(j * tau / (2 nsteps) + tau_load), per-env steps since the reset
  const real* ext_tab;
  int32_t ext_len;
  real ext_inv_tau;
  uint32_t* kenv;
  int32_t supply_kind;     // gemb200_supply_kind
  real sup_k1, sup_k2;     // RC supply: tau / (R C), R
  // AC supply: phase kept like the electrical angle (Ang<real>: turns as double-float in fp32, radians in a double), advanced by
  // f * tau per step; amplitude sqrt(2) * u_nominal; sup_ph0 = fixed phase in the stored unit, sup_fixed = 0: random per reset
  real sup_amp, sup_kph[2], sup_ph0[2];
  int32_t sup_fixed;
  double* sup_phase;       // [n]; nullptr unless AC supply
  real reset_obs_du[kMaxState];  // d reset_obs / d u_sup (supplies whose voltage at reset differs per env)
  real* sup;               // [2][n] RC supply: u_sup, 'has a previous call' flag (0 right after a reset); nullptr for the ideal supply
  real* obsv;              // [4][n] FluxObserver integrator (re, im, compensation terms); nullptr without one
  int32_t pf_dist;         // envs between a thread's env and the one it prefetches into L2 (0: off); ~ one wave of resident threads
  int32_t plain;           // 1: this configuration has the PLAIN shape (see step_kernel) -> specialised instantiation
  int32_t any_random_ref;  // any slot that draws random numbers per step (Wiener / Laplace / periodic)
  // ---- fused rollout (rollout_kernel): number of steps of this launch; outputs recorded every `record_every` steps (0: last step only) ----
  int32_t roll_steps, record_every;
  // per-step strides of the rollout's cursors, prepared on the host, all in BYTES (0 for an output that is not requested): action tensor
  // per step, obs / ref / reward / terminated slices per recorded step
  int64_t roll_act_inc, roll_obs_inc, roll_ref_inc, roll_rew_inc, roll_term_inc;
  // ---- fused aggregated return over NVLink (gemb200_bind_peers): destinations of the output stores as byte distances from the caller's
  //      tensors; 0 destinations = the caller's tensors only ----
  int32_t n_dst;
  int64_t dst_delta[8];
  // ---- parameter draws at every reset (gemb200_set_param_randomization; read by the ENVP instantiations and reset_kernel only).  Kept
  //      at the end of the block so that the constant-bank offsets of every other field stay where they were ----
  int32_t n_draw;          // parameters drawn per reset (0: none)
  const ParamDraw* draw;   // their distributions
  double* praw;            // [kMaxDraw][n] physical parameters of every env; drawn values are stored rounded to real
  // ---- adopted RNG identities (gemb200_adopt_rng_ids; read by the ENVP instantiations and reset_kernel only, once per launch):
  //      [kRngIdWords][n] u32 = Philox key lo, hi | global env index lo, hi | call-id offset lo, hi | step offset | spare.
  //      nullptr: every env draws with its own identity (seed, env_offset + i, 0, 0) ----
  const uint32_t* rngid;
  int32_t coef_shared;     // 1: the per-env blocks hold the shared parameters (made by the first adoption): reset observations from reset_obs
  // ---- reference feed (gemb200_rollout_record_ref; read by the general and ENVP instantiations only, never PLAIN): the caller's reference
  //      values of every step of this launch, [K][N][n_ref] (row-per-env) or [K][n_ref][N] (field-major).  Step k first overwrites the
  //      stored value of EVERY slot with row k, as gemb200_set_reference would.  nullptr: no feed ----
  const real* ref_feed;
  // ---- discounted returns (gemb200_rollout_returns; rollout kernel, general and ENVP instantiations only, never PLAIN): per env
  //      ret_out[i] = sum of discount^k * reward_k over the steps up to and including its first terminated one, ret_end[i] = the index
  //      of that step (roll_steps if none; ret_end may be nullptr).  ret_out == nullptr: no returns ----
  real* ret_out;
  int32_t* ret_end;
  real discount;
  // ---- periodic generators in the fp32 build (periodic_value; general instantiations only, never PLAIN): the frequency range and tau in
  //      double, so that the phase f tau k + phase of a long sub-episode is formed and reduced in double (DESIGN §2 finding 13) ----
  double ref_freq_lo_d[kMaxRefEntries], ref_freq_span_d[kMaxRefEntries];
  double ref_tau_d;
};
constexpr int kRngIdWords = 8;

}  // namespace gemb200
