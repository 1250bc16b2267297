"""Per-env parameter blocks (the ENVP instantiations: every env loads its model coefficients from its own column of the per-env table,
`load_coef` in gemb200_kernels.cuh) against the float64 oracle, slot by slot, in every motor family and through the wrappers.

For each configuration ONE handle holds
  * a control group with the configuration's parameters,
  * one group per parameter slot the configuration uses, with only that slot scaled,
  * a mixed group in which every slot is drawn independently for every env (coefficients derived from several parameters: EESM's
    sigma, the induction motors' tau_sigma),
and every group (every env of the mixed group) is compared with an oracle configured with the group's row through the ordinary
shared-parameter path, at the group's global env indices (same Philox streams: Wiener references, random initial states and auto-resets
line up).  Half of the steps run through the fused rollout, half through single steps.  A second oracle per slot group, run with the
configuration's row on the same env indices, shows that the scaled slot moves the outputs: a family that took that coefficient from the
shared bank would fail here.

What stays per handle (DESIGN.md §7), and is therefore kept as the handle's in every group oracle: pole pairs (refused per env, last
test), the flux limits `init_im` of induction-motor random initial states, and the FluxObserver constants (the observer models the
nominal motor).
"""
import ctypes as C

import numpy as np
import pytest

from gpu_helpers import torch_cuda  # noqa: F401
from helpers import ENV_PARAM_CASES, LP_SLOT, MOTOR_SLOTS, MP_SLOT, motor_of
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

TOL = {K.F64: 1e-9, K.F32: 1e-5}
# observer-angle dq actions: rounding comes back amplified through angle(psi_obs) in the tail of the batch (DESIGN.md finding 11)
TOL_OBSERVER_FEEDBACK = {K.F64: 1e-8, K.F32: 1e-3}
MOVES = 1e-3  # a scaled slot must move some output column by this much (column-relative): 100x the fp32 bar
GROUP, MIXED, STEPS, OFFSET = 37, 16, 64, 3000  # group sizes deliberately not multiples of 32
# factor of the slot groups: large, but RK4 at the env's tau stays stable (resistances down, everything else up)
FACTOR = dict(r_a=0.6, r_e=0.6, r_s=0.6, r_r=0.6)
DEFAULT_FACTOR = 1.7

# initial speed of the integrating loads with a constant initial state, as a fraction of the speed limit: running envs, where the speed
# dependent load terms b * omega and c * omega^2 matter within the test's few milliseconds; Cont-SC-PMSM starts from standstill instead,
# in the static-friction band |omega| <= omega_lim where the load torque is omega_lin * omega
OMEGA0 = {"sc-pmsm": 0.0}


def slots_of(env_id, cfg):
    """(name, slot index in the 24-wide row, is_load) of every slot the configuration uses"""
    names = [(nm, MP_SLOT[nm], False) for nm in MOTOR_SLOTS[motor_of(env_id)]]
    if cfg.load_kind == K.LOAD_POLY_STATIC:
        names.append(("j_rotor", K.MP_J_ROTOR, False))
        names += [(nm, LP_SLOT[nm], True) for nm in ("a", "b", "c", "j_load")]
    return names


def make_config(case, n, dtype):
    """the device configuration of a case: RK4, auto-reset, Wiener references; non-zero initial currents / fluxes where the initial state
    is constant (with zero currents the torque and rotor-current terms of the reset observation would be zero)"""
    import gym_electric_motor_b200 as gem

    env_id, kw = ENV_PARAM_CASES[case]()
    env = gem.make(env_id, num_envs=n, ode_solver=gem.physical_systems.RK4Solver(), autoreset="same_step", seed=17,
                   dtype="float64" if dtype == K.F64 else "float32", env_index_offset=OFFSET, **kw)
    cfg = env.build_config()
    cfg.dtype = dtype
    assert cfg.env_index_offset == OFFSET and cfg.layout == K.LAYOUT_AOS
    if not cfg.init_random:
        induction = cfg.motor_kind in (K.MOTOR_SCIM, K.MOTOR_DFIM)
        vals = [0.7, -0.4, 0.02, 0.03, 0.3] if induction else [0.9, -0.6, 0.5, 0.3]
        n_motor = {K.MOTOR_PERMEX_DC: 1, K.MOTOR_SERIES_DC: 1, K.MOTOR_SHUNT_DC: 2, K.MOTOR_EXTEX_DC: 2, K.MOTOR_PMSM: 3, K.MOTOR_SYNRM: 3,
                   K.MOTOR_EESM: 4, K.MOTOR_SCIM: 5, K.MOTOR_DFIM: 5}[cfg.motor_kind]
        for j in range(n_motor):
            cfg.init_ode[1 + j] = vals[j]
        if cfg.load_kind == K.LOAD_POLY_STATIC:
            cfg.init_ode[0] = OMEGA0.get(case, 0.2) * cfg.limits[0]
    return env_id, env, cfg


def _eesm_sigma(mp):
    k, l_m, l_e, l_d = mp[K.MP_K], mp[K.MP_L_M], mp[K.MP_L_E], mp[K.MP_L_D]
    l_M, l_E = k * 1.5 * l_m, k * k * 1.5 * l_e
    return 1.0 - l_M * l_M / (l_d * l_E)


def build_groups(env_id, cfg, rng):
    """[(name, motor row [16], load row [8], count)]: control, one group per slot, MIXED single-env groups"""
    mp0, lp0 = np.array(list(cfg.motor_param)), np.array(list(cfg.load_param))
    slots = slots_of(env_id, cfg)
    groups = [("control", mp0, lp0, GROUP)]
    for name, s, is_load in slots:
        mp, lp = mp0.copy(), lp0.copy()
        (lp if is_load else mp)[s] *= FACTOR.get(name, DEFAULT_FACTOR)
        groups.append((name, mp, lp, GROUP))
    for j in range(MIXED):
        while True:
            mp, lp = mp0.copy(), lp0.copy()
            for name, s, is_load in slots:
                (lp if is_load else mp)[s] *= rng.uniform(0.6, 1.4)
            # EESM: the draws must keep sigma = 1 - l_M^2 / (l_d l_E) away from 0, where the model is singular (a property of the
            # motor, not of the kernel: the configuration's sigma is -0.31)
            if cfg.motor_kind != K.MOTOR_EESM or abs(_eesm_sigma(mp)) > 0.1:
                break
        groups.append((f"mixed{j}", mp, lp, 1))
    return groups


def group_oracle(oracle_lib, cfg, mp, lp, count, start):
    """N = count float64 oracle with the group's physical parameters at global env indices OFFSET + start ..; everything else (limits,
    init_im, observer constants) is the handle's"""
    c = type(cfg).from_buffer_copy(cfg)
    c.n_envs, c.dtype, c.env_index_offset = count, K.F64, OFFSET + start
    for j in range(K.MAX_MOTOR_PARAM):
        c.motor_param[j] = mp[j]
    for j in range(8):
        c.load_param[j] = lp[j]
    return oracle_lib.Oracle(c, nthreads=4)


def random_actions(env, n, steps, rng):
    sp = env.action_space
    if hasattr(sp, "nvec"):
        return np.stack([np.stack([rng.integers(0, int(m), size=n) for m in sp.nvec], axis=1) for _ in range(steps)]).astype(np.int32)
    if hasattr(sp, "n"):
        return rng.integers(0, int(sp.n), size=(steps, n, 1)).astype(np.int32)
    lo, hi = np.asarray(sp.low, dtype=np.float64), np.asarray(sp.high, dtype=np.float64)
    return lo + (hi - lo) * rng.random((steps, n, len(lo)))


def run_oracles(oras, slices, actions, induction):
    """the oracles' reset and trajectories, assembled in the handle's env order; psi = rotor flux before each step (induction motors)"""
    r0 = [o.reset() for o in oras]
    out = dict(obs0=np.concatenate([r[0] for r in r0]), ref0=np.concatenate([r[1] for r in r0]))
    out["psi0"] = np.concatenate([o.get_ode_state()[:, 3:5] for o in oras]) if induction else None
    obs, ref, rew, term, psi = [], [], [], [], []
    for a in actions:
        if induction:
            psi.append(np.concatenate([o.get_ode_state()[:, 3:5] for o in oras]))
        res = [o.step(a[sl]) for o, sl in zip(oras, slices)]
        obs.append(np.concatenate([r[0] for r in res]))
        ref.append(np.concatenate([r[1] for r in res]))
        rew.append(np.concatenate([r[2] for r in res]))
        term.append(np.concatenate([r[3] for r in res]).astype(np.uint8))
    out.update(obs=np.array(obs), ref=np.array(ref), rew=np.array(rew), term=np.array(term), psi=np.array(psi) if induction else None)
    return out


def run_device(torch, sim, actions):
    """reset, the first half of the steps through ONE fused rollout (every step recorded), the second half through single steps"""
    host = lambda x: x.double().cpu().numpy()  # noqa: E731
    obs0, ref0 = sim.reset()
    out = dict(obs0=host(obs0), ref0=host(ref0))
    half = len(actions) // 2
    dev = torch.as_tensor(actions[:half], device="cuda").to(sim.act_dtype).contiguous()
    o, r, w, t = sim.rollout(dev, record_every=1)
    obs, ref, rew, term = [host(o)], [host(r)], [host(w)], [t.cpu().numpy().astype(np.uint8)]
    for a in actions[half:]:
        o, r, w, t = sim.step(a)
        obs.append(host(o)[None])
        ref.append(host(r)[None])
        rew.append(host(w)[None])
        term.append(t.cpu().numpy().astype(np.uint8)[None])
    out.update(obs=np.concatenate(obs), ref=np.concatenate(ref), rew=np.concatenate(rew), term=np.concatenate(term))
    return out


def dq_pairs(motor_kind):
    if motor_kind == K.MOTOR_SCIM:
        return ((5, 6), (10, 11))
    if motor_kind == K.MOTOR_DFIM:
        return ((5, 6), (10, 11), (15, 16), (20, 21))
    return ()


def weak_frame(d, o, psi, pairs):
    """SCIM / DFIM: while |psi_r| < 1e-3 the field frame is undefined (DESIGN.md finding 3): dq columns compared through their magnitude"""
    if not pairs:
        return d, o
    d, o = d.copy(), o.copy()
    weak = np.hypot(psi[:, 0], psi[:, 1]) < 1e-3
    for arr in (d, o):
        for a_, b_ in pairs:
            arr[weak, a_] = np.hypot(arr[weak, a_], arr[weak, b_])
            arr[weak, b_] = 0.0
    return d, o


def compare(dev, ora, state_names, motor_kind, dtype, observer, sign_events):
    """device vs oracle with the rules of tests/test_gpu_parity.py: (description of the first failure or None, envs still compared at the
    end, envs that held the plain tolerance); the caller bounds the fraction of dropped envs over the whole handle"""
    n = dev["obs0"].shape[0]
    tol = (TOL_OBSERVER_FEEDBACK if observer else TOL)[dtype]
    pairs = dq_pairs(motor_kind)
    ang = [j for j, nm in enumerate(state_names) if nm in ("epsilon", "psi_angle")]

    def diff_of(d, o):
        diff = np.abs(d - o)
        for j in ang:  # normalised angles live on a circle of circumference 2
            diff[:, j] = np.abs((d[:, j] - o[:, j] + 1.0) % 2.0 - 1.0)
        return diff

    d0, o0 = weak_frame(dev["obs0"], ora["obs0"], ora["psi0"], pairs) if pairs else (dev["obs0"], ora["obs0"])
    scale = np.maximum(np.abs(o0).max(axis=0), 1e-3)
    err = (diff_of(d0, o0) / scale).max()
    if not err < TOL[dtype]:
        return f"reset observation: column-relative error {err:.3e}", None, None
    if dev["ref0"].size and not np.abs(dev["ref0"] - ora["ref0"]).max() < 20 * TOL[dtype]:
        return "reset reference", None, None
    alive = np.ones(n, dtype=bool)
    within_plain = np.ones(n, dtype=bool)
    for k in range(len(ora["obs"])):
        o_term, d_term = ora["term"][k], dev["term"][k]
        alive &= ~(o_term != d_term)  # a constraint within rounding of its threshold: the episodes diverge from here on
        o_obs = ora["obs"][k]
        scale = np.maximum(scale, np.abs(o_obs[alive]).max(axis=0, initial=0.0))
        d, o = dev["obs"][k], o_obs
        if pairs:  # after an auto-reset the returned vector is the reset one: compared through magnitudes as well
            d, o = weak_frame(d, o, np.where(o_term[:, None] > 0, 0.0, ora["psi"][k]), pairs)
        rel = (diff_of(d, o) / scale).max(axis=1)
        if observer:
            within_plain &= ~(alive & (rel >= TOL[dtype]))
            alive &= ~(rel >= tol)  # tail allowance: such envs count as diverged, at most 1 % may
        if sign_events and dtype == K.F32:
            # finite legs waiting in their interlock state output by the SIGN of their current (converters.py:277-287), decided within fp32
            # rounding for a few envs per 10^5 leg-steps: a discrete event after which the episode is another one; such envs leave the
            # comparison (at most 1 % may, asserted below), as in test_gpu_parity.py
            alive &= ~(rel >= tol)
        err = rel[alive].max(initial=0.0)
        if not err < tol:
            worst = int(np.flatnonzero(alive)[np.argmax(rel[alive])])
            return f"step {k}: column-relative state error {err:.3e} (env {worst})", None, None
        if dev["ref"].size and not np.abs(dev["ref"][k] - ora["ref"][k])[alive].max(initial=0.0) < 20 * tol:
            return f"step {k}: reference", None, None
        if not np.abs(dev["rew"][k] - ora["rew"][k])[alive].max(initial=0.0) < 20 * tol:
            return f"step {k}: reward", None, None
    return None, alive, within_plain


def moved(scaled, base):
    """max column-relative distance between two oracle runs of the same envs (reset observation, every step's observation and reward)"""
    a = np.concatenate([scaled["obs0"][None], scaled["obs"]]).reshape(-1, scaled["obs"].shape[-1])
    b = np.concatenate([base["obs0"][None], base["obs"]]).reshape(-1, base["obs"].shape[-1])
    a = np.concatenate([a, np.concatenate([np.zeros_like(scaled["rew"][:1]), scaled["rew"]]).reshape(-1, 1)], axis=1)
    b = np.concatenate([b, np.concatenate([np.zeros_like(base["rew"][:1]), base["rew"]]).reshape(-1, 1)], axis=1)
    return float((np.abs(a - b).max(axis=0) / np.maximum(np.abs(b).max(axis=0), 1e-3)).max())


def oracle_matrix(oracle_lib, case, dtype, n=None):
    """everything of one case that needs no GPU: configuration, groups, actions, oracle trajectories (assembled), and the
    non-vacuity distance of every slot group"""
    rng = np.random.default_rng(sum(map(ord, case)))
    env_id, env, cfg = make_config(case, 1, dtype)
    groups = build_groups(env_id, cfg, rng)
    counts = [g[3] for g in groups]
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(int)
    n = int(sum(counts))
    env_id, env, cfg = make_config(case, n, dtype)
    slices = [slice(s, s + c) for s, c in zip(starts, counts)]
    actions = random_actions(env, n, STEPS, rng)
    induction = cfg.motor_kind in (K.MOTOR_SCIM, K.MOTOR_DFIM)
    oras = [group_oracle(oracle_lib, cfg, mp, lp, c, s) for (_, mp, lp, c), s in zip(groups, starts)]
    ora = run_oracles(oras, slices, actions, induction)
    mp0, lp0 = groups[0][1], groups[0][2]
    movement = {}
    for (name, mp, lp, c), s, sl in zip(groups, starts, slices):
        if name == "control" or name.startswith("mixed"):
            continue
        base = run_oracles([group_oracle(oracle_lib, cfg, mp0, lp0, c, s)], [slice(None)], actions[:, sl], induction)
        scaled = dict(obs0=ora["obs0"][sl], obs=ora["obs"][:, sl], rew=ora["rew"][:, sl])
        movement[name] = moved(scaled, base)
    mp_rows = np.concatenate([np.tile(g[1], (g[3], 1)) for g in groups])
    lp_rows = np.concatenate([np.tile(g[2], (g[3], 1)) for g in groups])
    return dict(env_id=env_id, env=env, cfg=cfg, groups=groups, slices=slices, actions=actions, ora=ora, movement=movement,
                mp_rows=mp_rows, lp_rows=lp_rows)


@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("case", list(ENV_PARAM_CASES))
def test_per_env_slot_groups_match_per_group_oracles(torch_cuda, oracle_lib, case, dtype):
    from gym_electric_motor_b200.vector_sim import VectorSim

    m = oracle_matrix(oracle_lib, case, dtype)
    # (b) not vacuous: every scaled slot moves some output of its group's oracle
    flat = {name: d for name, d in m["movement"].items() if not d >= MOVES}
    assert not flat, f"{case}: slots that do not move the outputs: {flat}"
    # (a) the device with per-env blocks against the per-group oracles
    sim = VectorSim(m["cfg"])
    try:
        sim.set_env_params(m["mp_rows"], m["lp_rows"])
        dev = run_device(torch_cuda, sim, m["actions"])
    finally:
        sim.close()
    observer, sign_events = "observer" in case, "interlock" in case
    names = list(m["env"].physical_system.state_names)
    mixed = slice(m["slices"][-MIXED].start, m["slices"][-1].stop)
    parts = [(name, sl) for (name, _, _, _), sl in zip(m["groups"], m["slices"]) if not name.startswith("mixed")] + [("mixed", mixed)]
    alive, within_plain = [], []
    for name, sl in parts:
        sub = lambda x: {k: (None if v is None else (v[sl] if k in ("obs0", "ref0", "psi0") else v[:, sl])) for k, v in x.items()}  # noqa: E731
        msg, a, w = compare(sub(dev), sub(m["ora"]), names, m["cfg"].motor_kind, dtype, observer, sign_events)
        assert msg is None, f"{case}, group {name}: {msg}"
        alive.append(a)
        within_plain.append(w)
    alive, within_plain = np.concatenate(alive), np.concatenate(within_plain)
    assert alive.mean() >= 0.99, f"{case}: {int((~alive).sum())} of {alive.size} envs split from their oracle"
    if observer and dtype == K.F32:
        assert within_plain.mean() > 0.9, f"{case}: only {within_plain.mean():.3f} of the envs within {TOL[dtype]:g}"


def test_set_env_params_refuses_per_env_pole_pairs(torch_cuda):
    """the C-ABI refuses a row whose pole pairs differ from the configuration's (the angle increments kang and the dq advance adv_k are
    per handle); rows with the configuration's pole pairs are accepted, and a refused call leaves the handle as it was"""
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.vector_sim import VectorSim

    n = 45
    cfg = gem.make("Cont-CC-PMSM-v0", num_envs=n, ode_solver=gem.physical_systems.RK4Solver(), seed=2).build_config()
    a, b = VectorSim(cfg), VectorSim(cfg)
    try:
        mp = np.tile(np.array(list(cfg.motor_param)), (n, 1))
        mp[:, K.MP_R_S] *= np.linspace(0.8, 1.2, n)
        vp = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
        bad = mp.copy()
        bad[33, K.MP_P] += 1
        assert a._lib.gemb200_set_env_params(a._h, vp(bad), None) == K.E_INVALID
        assert b"pole pairs" in a._lib.gemb200_last_error()
        with pytest.raises(ValueError, match="pole pairs"):
            a.set_env_params(bad)
        assert a._lib.gemb200_set_env_params(a._h, vp(mp), None) == 0
        b.set_env_params(mp)
        oa, _ = a.reset()
        ob, _ = b.reset()
        assert torch_cuda.equal(oa, ob)
        act = torch_cuda.rand((n, 3), device="cuda", generator=torch_cuda.Generator(device="cuda").manual_seed(1)) * 2 - 1
        assert torch_cuda.equal(a.step(act)[0], b.step(act)[0])
    finally:
        a.close()
        b.close()
