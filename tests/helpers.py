"""Shared test helpers: golden-fixture loading and golden-meta -> gemb200_config translation, the golden-based device configurations and
random actions of the parity and rollout tests, the per-env parameter cases, and a handle stand-in for argument checks without a GPU.

The translation here is deliberately independent of the product's own spec compiler
(gym_electric_motor_b200/spec.py): it takes limits / weights verbatim from the values the REFERENCE reported
when the golden was recorded, so oracle-vs-golden tests do not depend on the product's host logic.
"""
import ctypes as C
import glob
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from gym_electric_motor_b200 import _cabi as K  # noqa: E402
from gym_electric_motor_b200.vector_sim import VectorSim  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")

MOTOR_KIND = {
    "DcPermanentlyExcitedMotor": K.MOTOR_PERMEX_DC,
    "DcSeriesMotor": K.MOTOR_SERIES_DC,
    "DcShuntMotor": K.MOTOR_SHUNT_DC,
    "DcExternallyExcitedMotor": K.MOTOR_EXTEX_DC,
    "PermanentMagnetSynchronousMotor": K.MOTOR_PMSM,
    "SynchronousReluctanceMotor": K.MOTOR_SYNRM,
    "ExternallyExcitedSynchronousMotor": K.MOTOR_EESM,
    "SquirrelCageInductionMotor": K.MOTOR_SCIM,
    "DoublyFedInductionMotor": K.MOTOR_DFIM,
}
MP_SLOT = dict(
    p=K.MP_P, r_s=K.MP_R_S, l_d=K.MP_L_D, l_q=K.MP_L_Q, psi_p=K.MP_PSI_P, j_rotor=K.MP_J_ROTOR, r_a=K.MP_R_A,
    l_a=K.MP_L_A, psi_e=K.MP_PSI_E, r_e=K.MP_R_E, l_e=K.MP_L_E, l_e_prime=K.MP_L_E_PRIME, l_m=K.MP_L_M, k=K.MP_K,
    l_sigs=K.MP_L_SIGS, l_sigr=K.MP_L_SIGR, r_r=K.MP_R_E,
)
CONV = {
    "ContOneQuadrantConverter": (0, [K.CONV_1QC]),
    "ContTwoQuadrantConverter": (0, [K.CONV_2QC]),
    "ContFourQuadrantConverter": (0, [K.CONV_4QC]),
    "ContB6BridgeConverter": (0, [K.CONV_B6]),
    "FiniteOneQuadrantConverter": (1, [K.CONV_1QC]),
    "FiniteTwoQuadrantConverter": (1, [K.CONV_2QC]),
    "FiniteFourQuadrantConverter": (1, [K.CONV_4QC]),
    "FiniteB6BridgeConverter": (1, [K.CONV_B6]),
}
N_MOTOR_ODE = {K.MOTOR_PERMEX_DC: 1, K.MOTOR_SERIES_DC: 1, K.MOTOR_SHUNT_DC: 2, K.MOTOR_EXTEX_DC: 2, K.MOTOR_PMSM: 3,
               K.MOTOR_SYNRM: 3, K.MOTOR_EESM: 4, K.MOTOR_SCIM: 5, K.MOTOR_DFIM: 5}


def golden_names():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "*.npz")) if "ref_data" not in p)


def load_golden(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False)
    d = {k: z[k] for k in z.files if k != "meta"}
    d["meta"] = json.loads(str(z["meta"]))
    return d


def solver_from_name(name):
    """'euler', 'euler3', 'rk4', 'rk4x2', 'dopri5' -> (kind, nsteps); dopri5 is oracle-only (kind 100)."""
    if name == "dopri5":
        return 100, 1
    if name.startswith("euler"):
        return K.SOLVER_EULER, int(name[5:] or 1)
    if name.startswith("rk4x"):
        return K.SOLVER_RK4, int(name[4:])
    if name == "rk4":
        return K.SOLVER_RK4, 1
    raise ValueError(name)


def len_steps_hint(meta):
    return int(meta["case"].get("steps", 2000))


def config_from_meta(meta, n_envs=1, solver=None, ref_kind=K.REF_EXTERNAL, dtype=K.F64, layout=K.LAYOUT_AOS,
                     autoreset=K.AUTORESET_NONE, seed=0, reset_ode=None):
    cfg = K.new_config()
    cfg.n_envs = n_envs
    cfg.dtype, cfg.layout, cfg.autoreset = dtype, layout, autoreset
    mk = MOTOR_KIND[meta["motor_class"]]
    cfg.motor_kind = mk
    cc = meta["converter_class"]
    if cc in CONV:
        cfg.finite, kinds = CONV[cc]
    elif cc in ("ContMultiConverter", "FiniteMultiConverter"):
        cfg.finite = int(cc.startswith("Finite"))
        sub = {"ContFourQuadrantConverter": K.CONV_4QC, "ContTwoQuadrantConverter": K.CONV_2QC, "ContOneQuadrantConverter": K.CONV_1QC,
               "FiniteFourQuadrantConverter": K.CONV_4QC, "FiniteTwoQuadrantConverter": K.CONV_2QC, "FiniteOneQuadrantConverter": K.CONV_1QC,
               "ContB6BridgeConverter": K.CONV_B6, "FiniteB6BridgeConverter": K.CONV_B6}
        multi = meta["case"].get("multi")
        if multi:
            kinds = [sub[name] for name, _ in multi]
        else:
            kinds = [K.CONV_B6, K.CONV_4QC] if mk == K.MOTOR_EESM else ([K.CONV_B6, K.CONV_B6] if mk == K.MOTOR_DFIM else [K.CONV_4QC, K.CONV_4QC])
    else:
        raise ValueError(cc)
    for i, kd in enumerate(kinds):
        cfg.converter_kind[i] = kd
    cfg.load_kind = {"ConstantSpeedLoad": K.LOAD_CONST_SPEED, "ExternalSpeedLoad": K.LOAD_EXT_SPEED}.get(meta["load_class"], K.LOAD_POLY_STATIC)
    kind, nsteps = solver_from_name(solver or meta["case"]["solver"])
    cfg.solver_kind, cfg.solver_nsteps = kind, nsteps
    cfg.tau = meta["tau"]
    if cfg.load_kind == K.LOAD_EXT_SPEED:  # tabulated speed profile: f(j tau / (2 nsteps) + tau_load), make_golden.py:sin_profile
        es = meta["ext_speed"]
        per = 2 * nsteps
        j = np.arange(per * (len_steps_hint(meta) + 8) + 2 * per + 1)
        t = j * (meta["tau"] / per) + es["tau"]
        tab = np.ascontiguousarray(es["o"] + es["a"] * np.sin(2 * np.pi * es["f"] * t))
        cfg.load_param[K.LP_TAU_LOAD] = es["tau"]
        cfg.ext_speed_table, cfg.ext_speed_len = tab.ctypes.data, len(tab)
        cfg._keepalive = tab
    cfg.interlocking_time = meta["interlocking_time"]
    ils = meta.get("interlocking_times") or []
    if len(ils) == 2 and ils[0] != ils[1]:  # multi converter whose sub-converters differ: one time per converter slot
        cfg.interlocking_time, cfg.interlocking_time1 = ils[0], ils[1]
    cfg.u_sup = meta["u_sup"]
    if meta.get("supply_class") == "AC1PhaseSupply":
        cfg.supply_kind = K.SUPPLY_AC1
        cfg.supply_param[0], cfg.supply_param[1], cfg.supply_param[2] = meta["supply_parameter"]["f"], meta["supply_parameter"]["phase"], 1.0
    if meta.get("supply_class") == "RCVoltageSupply":
        cfg.supply_kind = K.SUPPLY_RC
        cfg.supply_param[0], cfg.supply_param[1] = meta["supply_parameter"]["R"], meta["supply_parameter"]["C"]
    for k, v in meta["motor_parameter"].items():
        if k in MP_SLOT:
            cfg.motor_param[MP_SLOT[k]] = v
    lp = meta.get("load_parameter") or {}
    cfg.load_param[K.LP_A] = lp.get("a", 0.0)
    cfg.load_param[K.LP_B] = lp.get("b", 0.0)
    cfg.load_param[K.LP_C] = lp.get("c", 0.0)
    # j_total = j_load + j_rotor (mechanical_load.py:188-193); golden meta stores j_total
    cfg.load_param[K.LP_J_LOAD] = meta["j_total"] - meta["motor_parameter"]["j_rotor"]
    cfg.load_param[K.LP_TAU_DECAY] = 1e-3
    n_state = len(meta["state_names"])
    # cfg.limits normalises the inner system's own vector; weights / lengths refer to the final (wrapped) vector
    for i, v in enumerate(meta.get("base_limits", meta["limits"])):
        cfg.limits[i] = v
    for i in range(n_state):
        cfg.reward_weight[i] = meta["reward_weights"][i]
        cfg.reward_power[i] = meta["reward_power"][i]
        cfg.state_length[i] = meta["state_length"][i]
    cfg.reward_bias = meta["reward_bias"]
    cfg.violation_reward = meta["violation_reward"]
    n_ode = 1 + N_MOTOR_ODE[mk]
    if reset_ode is not None:
        for i in range(n_ode):
            cfg.init_ode[i] = float(reset_ode[i])
    names = meta["state_names"]
    cfg.n_constraints = len(meta["constraints"])
    for ci, con in enumerate(meta["constraints"]):
        cfg.constraint_kind[ci] = K.CONSTRAINT_SQUARED if con["kind"] == "SquaredConstraint" else K.CONSTRAINT_LIMIT
        m = 0
        for s in con["states"]:
            m |= 1 << names.index(s)
        cfg.constraint_mask[ci] = m
    ref_names = meta["reference_names"]
    cfg.n_ref = len(ref_names)
    for r, rn in enumerate(ref_names):
        cfg.ref_kind[r] = ref_kind
        cfg.ref_state[r] = names.index(rn)
    cfg.seed = seed
    # physical-system wrappers recorded with the golden (list order = reference order: later entries wrap earlier ones)
    dq, dead, outer, adv = 0, 0, 0, 0.0
    cur_names = list(meta.get("base_state_names", names))  # state vector as seen by the next wrapper
    cur_limits = list(meta.get("base_limits", meta["limits"]))
    nops = 0
    for kind, arg in meta["case"].get("wrappers", []) or []:
        if kind == "DeadTime":
            dead, outer = int(arg), (1 if dq else 0)
        elif kind == "CosSin":  # cos_sin_processor.py:39-58
            idx, rm = cur_names.index(arg[0]), int(arg[1])
            cfg.sop_kind[nops] = K.SOP_COS_SIN
            cfg.sop_idx[nops][0], cfg.sop_idx[nops][1] = idx, rm
            if rm:
                del cur_names[idx], cur_limits[idx]
            cur_names += [f"cos({arg[0]})", f"sin({arg[0]})"]
            cur_limits += [1.0, 1.0]
            nops += 1
        elif kind == "FluxObserver":  # flux_observer.py:56-79
            mp = meta["motor_parameter"]
            l_r = mp["l_m"] + mp["l_sigr"]
            psi_limit = mp["l_m"] * cur_limits[cur_names.index("i_sd")]
            idx = [cur_names.index(n) for n in ("i_sa", "i_sb", "i_sc", "omega")]
            cfg.sop_kind[nops] = K.SOP_FLUX_OBSERVER
            for q, v in enumerate(idx):
                cfg.sop_idx[nops][q] = v
            for q, v in enumerate([mp["r_r"] * mp["l_m"] / l_r, mp["r_r"] / l_r, mp["p"], psi_limit] + [cur_limits[j] for j in idx]):
                cfg.sop_param[nops][q] = v
            cur_names += ["psi_abs", "psi_angle"]
            cur_limits += [psi_limit, np.pi]
            nops += 1
        else:
            dq, adv = (3 if arg == "DFIM" else (2 if arg == "SCIM" else 1)), 0.5 + dead
    cfg.n_state_ops = nops
    assert cur_names == names or not nops, (cur_names, names)
    cfg.action_dq, cfg.dead_time_steps, cfg.dead_time_outer, cfg.angle_advance = dq, dead, outer, adv
    return cfg


def replay_golden(sim, g, inject_refs=True):
    """Drive `sim` (Oracle or device env with the same reset/step/set_reference API, N=1) through a golden
    trajectory: same actions, reference injected before every step, reset on termination exactly where the
    reference harness did (tests/golden/make_golden.py:record).  Returns dict of arrays shaped like the golden."""
    K_ = len(g["actions"])
    ref_idx = [g["meta"]["state_names"].index(n) for n in g["meta"]["reference_names"]]
    obs0, _ = sim.reset()
    out = dict(states=np.zeros_like(g["states"]), rewards=np.zeros(K_), terminated=np.zeros(K_, dtype=np.uint8),
               reset_state=np.asarray(obs0, dtype=np.float64)[0])
    for k in range(K_):
        if inject_refs and ref_idx:
            sim.set_reference(g["refs_used"][k][ref_idx][None, :])
        obs, ref, rew, term = sim.step(g["actions"][k][None, ...] if g["actions"].ndim > 1 else g["actions"][k : k + 1])
        out["states"][k] = np.asarray(obs, dtype=np.float64)[0]
        out["rewards"][k] = float(np.asarray(rew)[0])
        out["terminated"][k] = int(np.asarray(term)[0])
        if g["terminated"][k]:
            sim.reset()
    return out


def switched_config(n, kinds_cfg, p, length, name="permex_sc_euler3", seed=3, dtype=K.F64):
    """config with ONE switched reference slot on the golden's referenced state; kinds_cfg = list of dicts written into the extra
    parameter entries 1.. (entry 0 is the output slot itself)."""
    g = load_golden(name)
    cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=g["reset_ode"], solver="rk4", ref_kind=K.REF_WIENER, seed=seed, dtype=dtype,
                           autoreset=K.AUTORESET_SAME_STEP)
    assert cfg.n_ref == 1
    cfg.n_constraints = 0
    cfg.ref_sw_count[0], cfg.ref_sw_first[0] = len(kinds_cfg), 1
    cfg.ref_sw_len_lo[0], cfg.ref_sw_len_hi[0] = length
    acc = 0.0
    for j, kc in enumerate(kinds_cfg):
        e = 1 + j
        cfg.ref_state[e] = cfg.ref_state[0]
        cfg.ref_kind[e] = kc["kind"]
        cfg.ref_value[e] = kc.get("value", 0.0)
        cfg.ref_margin_lo[e], cfg.ref_margin_hi[e] = kc.get("margin", (-0.8, 0.8))
        cfg.ref_init_lo[e], cfg.ref_init_hi[e] = kc.get("margin", (-0.8, 0.8))
        cfg.ref_sigma_lo[e], cfg.ref_sigma_hi[e] = kc.get("sigma", (1e-3, 1e-2))
        cfg.ref_len_lo[e], cfg.ref_len_hi[e] = kc.get("length", (8, 30))
        cfg.ref_amp_lo[e], cfg.ref_amp_hi[e] = kc.get("amp", (0.1, 0.4))
        cfg.ref_freq_lo[e], cfg.ref_freq_hi[e] = kc.get("freq", (50.0, 400.0))
        cfg.ref_off_lo[e], cfg.ref_off_hi[e] = kc.get("off", (-0.3, 0.3))
        acc += p[j]
        cfg.ref_sw_cdf[e] = acc if j < len(kinds_cfg) - 1 else 1.0
    return cfg


def golden_reset_state(g):
    """Reset observation of a golden.  Reference quirk: CosSinProcessor(remove_angle=True).reset() returns the vector WITH the
    angle it removes in simulate() (cos_sin_processor.py:60-63 vs :65-70); a batched tensor has one width, so the device path
    and the oracle remove it at reset too — compare against the golden with that column deleted."""
    rs = np.asarray(g["reset_state"], dtype=np.float64)
    names = list(g["meta"].get("base_state_names", g["meta"]["state_names"]))
    for kind, arg in g["meta"]["case"].get("wrappers", []) or []:
        if kind == "CosSin":
            if int(arg[1]):  # env.reset() then cuts the un-shortened vector with its state filter: [..., angle, ..., cos] — sin is lost
                a = names.index(arg[0])
                rs = np.delete(np.concatenate((rs, [np.sin(np.pi * rs[a])])), a)
            if int(arg[1]):
                names.remove(arg[0])
            names += [f"cos({arg[0]})", f"sin({arg[0]})"]
        elif kind == "FluxObserver":
            names += ["psi_abs", "psi_angle"]
    return rs


def col_rel_err(a, b):
    """max over columns of max|a-b| / max(|b|) — the 'column-relative' error of SURVEY.md §7."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    scale = np.maximum(np.abs(b).max(axis=0), 1e-12)
    return float((np.abs(a - b).max(axis=0) / scale).max())


# ------------------------------------------------------------------------------------------------- device configurations of the goldens
TOL = {K.F64: 1e-9, K.F32: 1e-5}
# dopri5 goldens are compared against RK4 with 2 sub-steps: accuracy of the substitute solver, not identity
TOL_DOPRI = {K.F64: 2e-6, K.F32: 1e-5}
# SCIM with dq actions transformed by the FluxObserver's angle: psi_obs is a running sum of current samples with heavy cancellation
# under random actions, so rounding-level differences of the currents (1e-7 relative in fp32, 1e-16 in fp64) come back amplified
# ~100x through angle(psi_obs) into the applied voltages.  Conditioning of the configuration, not of the kernel: the same
# trajectories without that feedback (scim_cc_flux_rk4) hold the plain tolerance.
TOL_OBSERVER_FEEDBACK = {K.F64: 1e-8, K.F32: 1e-3}


# Induction motors: the state columns expressed in the rotor-flux (field) frame, in (d, q) pairs.  That frame's angle is decided by round-off
# while the rotor flux is still (numerically) zero after a reset, in the reference itself (DESIGN.md finding 3), so oracle comparisons
# take the magnitude of each pair for envs whose flux is below 1e-3 (fold_weak_dq)
WEAK_DQ_PAIRS = {K.MOTOR_SCIM: ((5, 6), (10, 11)), K.MOTOR_DFIM: ((5, 6), (10, 11), (15, 16), (20, 21))}


def fold_weak_dq(pairs, weak, *arrs):
    """in place, for the rows `weak` of each [N, n_state] array: (d, q) -> (hypot(d, q), 0) for every pair the array has"""
    for arr in arrs:
        for p_, q_ in pairs:
            if q_ < arr.shape[1]:
                arr[weak, p_] = np.hypot(arr[weak, p_], arr[weak, q_])
                arr[weak, q_] = 0.0


def _tol(name, dtype, is_dopri=False, batch=False):
    if "flux_dq" in name or "flux_cossin_dead1" in name:
        return TOL_OBSERVER_FEEDBACK[dtype]
    if name.startswith("dfim_fin") and dtype == K.F32:
        # tau = 1e-5: the rotor flux stays at ~1 % of nominal for the whole run, so the field-frame (dq) columns carry the fp32
        # flux noise divided by that small magnitude; the frame-independent columns hold 2e-6
        return 3e-5
    return (TOL_DOPRI if is_dopri else TOL)[dtype]


class DeviceAdapter:
    """Gives VectorSim the numpy reset/step/set_reference API that helpers.replay_golden drives."""

    def __init__(self, cfg):
        from gym_electric_motor_b200.vector_sim import VectorSim

        self.sim = VectorSim(cfg)

    def reset(self, mask=None):
        obs, ref = self.sim.reset(mask)
        return obs.double().cpu().numpy(), ref.double().cpu().numpy()

    def step(self, action):
        obs, ref, rew, term = self.sim.step(np.asarray(action))
        return obs.double().cpu().numpy(), ref.double().cpu().numpy(), rew.double().cpu().numpy(), term.cpu().numpy()

    def set_reference(self, r):
        self.sim.set_reference(r)


def _random_actions(rng, g, n, steps):
    a = g["actions"]
    if a.ndim == 1:
        hi = int(a.max()) + 1
        return rng.integers(0, max(hi, 2), size=(steps, n, 1)).astype(np.int32)
    if a.dtype.kind == "i":
        hi = a.max(axis=0) + 1
        return (rng.random((steps, n, a.shape[1])) * hi).astype(np.int32)
    # smooth-ish random actions so that currents build up and constraints trigger
    base = rng.uniform(-1, 1, size=(steps, n, a.shape[1]))
    hold = rng.uniform(-1, 1, size=(1, n, a.shape[1]))
    lo, hi = a.min(), a.max()
    out = 0.5 * base + 0.5 * hold
    if lo >= 0:
        out = np.abs(out)
    return out


# plain / general instantiations, every motor family, the side state that lives outside the registers (switching states, dead-time
# ring, RC / AC supply, flux observer, external speed profile position, switched generators)
ROLLOUT_CASES = ["pmsm_cc_rk4", "pmsm_sc_polyload_rk4", "pmsm_fin_sc_rk4", "pmsm_fin_sc_rk4_interlock", "pmsm_cc_euler3", "synrm_cc_rk4",
                 "eesm_cc_rk4", "eesm_fin_cc_rk4", "scim_cc_rk4", "scim_fin_cc_interlock_rk4", "dfim_cc_rk4", "permex_cc_rk4", "series_cc_rk4",
                 "shunt_cc_rk4", "extex_cc_rk4", "permex_fin_sc_rc_interlock_rk4", "pmsm_cc_ac_rk4", "pmsm_cc_extspeed_rk4",
                 "scim_sc_flux_cossin_dead1_rk4", "eesm_cc_rc_dq_dead1_rk4", "pmsm_cc_cossin_rk4", "dfim_cc_flux_dq_rk4",
                 "extex_fin_cc_interlock2_rk4", "dfim_fin_sc_interlock2_rk4"]


def _mk(name, n, dtype, layout, ref_kind=K.REF_WIENER):
    g = load_golden(name)
    init = np.array(g["reset_ode"], dtype=float)
    n_ode = len(init)
    init[1:] = [0.7, -0.4, 0.02, 0.03, 0.3][: n_ode - 1] if g["meta"]["motor_class"] in ("SquirrelCageInductionMotor", "DoublyFedInductionMotor") else \
        [0.9, -0.6, 0.5, 0.3][: n_ode - 1]
    cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=init, dtype=dtype, solver=None, ref_kind=ref_kind, autoreset=K.AUTORESET_SAME_STEP, seed=77,
                           layout=layout)
    for r in range(cfg.n_ref):
        cfg.ref_margin_lo[r], cfg.ref_margin_hi[r] = -0.7, 0.7
        cfg.ref_init_lo[r], cfg.ref_init_hi[r] = -0.7, 0.7
        cfg.ref_len_lo[r], cfg.ref_len_hi[r] = 3, 9  # several sub-episode changes inside one rollout
    cfg.env_index_offset = 12345
    if cfg.supply_kind == K.SUPPLY_AC1:
        cfg.supply_param[2] = 0.0
    return g, cfg


# -------------------------------------------------------------------------------------------------------------- per-env parameter cases
LP_SLOT = dict(a=K.LP_A, b=K.LP_B, c=K.LP_C, j_load=K.LP_J_LOAD)
# j_rotor enters only the load words (inv_j, omega_lim, omega_lin): it is a slot of the configurations whose load integrates omega, and
# cannot matter under a constant-speed load (CC configurations), where it is left out
_DC_SEP = ("r_a", "r_e", "l_a", "l_e", "l_e_prime")
_IM = ("r_s", "r_r", "l_m", "l_sigs", "l_sigr")
MOTOR_SLOTS = dict(PermExDc=("r_a", "l_a", "psi_e"), SeriesDc=_DC_SEP, ShuntDc=_DC_SEP, ExtExDc=_DC_SEP, PMSM=("r_s", "l_d", "l_q", "psi_p"),
                   SynRM=("r_s", "l_d", "l_q"), EESM=("r_s", "l_d", "l_q", "l_m", "r_e", "l_e"), SCIM=_IM, DFIM=_IM)
# EESM's k is left out: it only refers the excitation circuit to the stator side and back, so every coefficient of the model
# (derive_coef: r_E, l_M, l_E and 2 / (3 k) enter as k-free ratios) and therefore every output is the same for any k
# integrating loads with every polynomial term non-zero (the defaults have c = 0, some a = b = 0), so that a, b and c each matter
LOADS = dict(PermExDc=dict(a=6.0, b=0.05, c=5e-4, j_load=0.02), SeriesDc=dict(a=0.3, b=0.05, c=2e-4, j_load=1e-4),
             ShuntDc=dict(a=0.6, b=0.02, c=2e-4, j_load=2e-3), ExtExDc=dict(a=0.6, b=0.02, c=2e-4, j_load=2e-3),
             PMSM=dict(a=2.0, b=0.05, c=5e-3, j_load=1e-3), SynRM=dict(a=0.3, b=0.01, c=1e-5, j_load=1e-4),
             EESM=dict(a=100.0, b=1.0, c=5e-3, j_load=0.3), SCIM=dict(a=0.3, b=0.01, c=3e-4, j_load=1e-4),
             DFIM=dict(a=1.0, b=0.02, c=2e-4, j_load=1e-3))
# the finite PMSM runs at tau = 1e-5, a tenth of the continuous envs' time: stronger load terms and a load inertia comparable to the rotor's
FINITE_PMSM_LOAD = dict(a=20.0, b=0.5, c=5e-3, j_load=0.04)


def _wrappers(*spec):
    from gym_electric_motor_b200 import physical_system_wrappers as psw

    out = []
    for kind, arg in spec:
        out.append(psw.DeadTimeProcessor(steps=arg) if kind == "DeadTime" else psw.FluxObserver() if kind == "FluxObserver"
                   else psw.DqToAbcActionProcessor.make(arg))
    return out


def _sc(motor_name, **kw):
    load = dict(load_parameter=dict(LOADS[motor_name]))
    load.update(kw.pop("load", {}))
    return dict(load=load, **kw)


# id -> (env id, gem.make kwargs); a function so that every make gets fresh wrapper / initializer objects
ENV_PARAM_CASES = {
    "sc-permex": lambda: ("Cont-SC-PermExDc-v0", _sc("PermExDc")),
    "sc-series": lambda: ("Cont-SC-SeriesDc-v0", _sc("SeriesDc")),
    "sc-shunt": lambda: ("Cont-SC-ShuntDc-v0", _sc("ShuntDc")),
    "sc-extex": lambda: ("Cont-SC-ExtExDc-v0", _sc("ExtExDc")),
    "sc-pmsm": lambda: ("Cont-SC-PMSM-v0", _sc("PMSM")),
    "sc-synrm": lambda: ("Cont-SC-SynRM-v0", _sc("SynRM")),
    "sc-eesm": lambda: ("Cont-SC-EESM-v0", _sc("EESM")),
    "sc-scim": lambda: ("Cont-SC-SCIM-v0", _sc("SCIM")),
    "sc-dfim": lambda: ("Cont-SC-DFIM-v0", _sc("DFIM")),
    "cc-dfim": lambda: ("Cont-CC-DFIM-v0", {}),
    # finite converters: a B6 bridge with interlocking time, and a multi converter (two 4QC) on a two-circuit DC motor
    "fin-sc-pmsm-interlock": lambda: ("Finite-SC-PMSM-v0", _sc("PMSM", converter=dict(interlocking_time=1e-6),
                                                                               load=dict(load_parameter=dict(FINITE_PMSM_LOAD)))),
    "fin-cc-extex": lambda: ("Finite-CC-ExtExDc-v0", {}),
    # dq actions with the angle advance of a dead time in front (the dq advance adv_k)
    "cc-pmsm-dq-dead": lambda: ("Cont-CC-PMSM-v0", dict(physical_system_wrappers=_wrappers(("DeadTime", 1), ("DqToAbc", "PMSM")))),
    # dq actions transformed with the FluxObserver's angle
    "cc-scim-observer-dq": lambda: ("Cont-CC-SCIM-v0", dict(physical_system_wrappers=_wrappers(("FluxObserver", None), ("DqToAbc", "SCIM")))),
    # random initial states: the reset observation is derived on the device from the env's own coefficients
    "sc-pmsm-gaussian-init": lambda: ("Cont-SC-PMSM-v0", _sc("PMSM", motor=dict(motor_initializer=dict(random_init="gaussian", random_params=(None, 0.3))),
                                                             load=dict(load_initializer=dict(random_init="uniform", interval=[[-50.0, 120.0]])))),
    "sc-scim-uniform-init": lambda: ("Cont-SC-SCIM-v0", _sc("SCIM", motor=dict(motor_initializer=dict(random_init="uniform")))),
}


def motor_of(env_id):
    return env_id.split("-")[2]


# -------------------------------------------------------------------------------------------------------- argument checks without a GPU
class _NoLaunch:
    def __getattr__(self, name):
        raise AssertionError(f"{name} was called: a bad reference feed must be refused before any launch")


class NoLaunchSim(VectorSim):
    """VectorSim on the CPU device whose library calls fail: every check of a feed runs, no launch does"""

    def __init__(self, cfg, reuse_outputs=True):
        d = [C.c_int32() for _ in range(4)]
        K.check(K.load_library().gemb200_query_dims(C.byref(cfg), *[C.byref(x) for x in d]), "gemb200_query_dims")
        self.n_state, self.n_ode, self.n_act, self.n_ref = [x.value for x in d]
        self.cfg, self.n, self.finite = cfg, int(cfg.n_envs), bool(cfg.finite)
        self.soa = cfg.layout == K.LAYOUT_SOA
        self.dtype = torch.float32 if cfg.dtype == K.F32 else torch.float64
        self.act_dtype = torch.int32 if self.finite else self.dtype
        self.device = torch.device("cpu")
        self._lib, self._h, self._reuse, self._out = _NoLaunch(), None, reuse_outputs, None


@pytest.fixture
def no_launch(monkeypatch):
    import gym_electric_motor_b200.vector_sim as vs

    monkeypatch.setattr(vs, "VectorSim", NoLaunchSim)


def _env(**kw):
    """six PMSM envs with both references fed by the caller (the N = 6 of the argument-check tests)"""
    import gym_electric_motor_b200 as gem

    rg = gem.reference_generators.MultipleReferenceGenerator([gem.reference_generators.ExternalReferenceGenerator("i_sd"),
                                                              gem.reference_generators.ExternalReferenceGenerator("i_sq")])
    return gem.make("Cont-CC-PMSM-v0", num_envs=6, reference_generator=rg, dtype="float32", **kw)
