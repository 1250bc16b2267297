"""Rollout Jacobians on the device: `rollout_jacobians(actions)` runs K steps in one launch and also returns jac_x = d x_{k+1} / d x_k and
jac_u = d x_{k+1} / d a_k per env and step.

- Primal identity: twin handles with equal seeds, A runs `rollout(actions, record_every=1)`, B runs `rollout_jacobians`; outputs, clock and
  the persistent state (checkpoint blob, or snapshot rows and the next steps where checkpoints are refused) must be the same.
- Fusion identity: a K-step launch gives the Jacobians of K one-step launches bit for bit.
- Known answer: PMSM and SynRM at constant speed with an unclipped continuous B6 bridge have linear current dynamics; the RK4 current block
  and its action block have closed forms.
- Finite differences: central differences of the float64 step itself (perturbed copies as envs of one handle, one launch), at every
  family, load mode, solver, converter kind, dq actions and the AC supply."""
import math

import numpy as np
import pytest

from test_gpu_parity import torch_cuda  # noqa: F401
from test_gpu_rollout_returns import ENV_IDS, _actions, _blob, _bits, _eq, _make, _next_steps, _same
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

N = 300
HORIZONS = (64, 7, 1)


def _pair(torch, a_env, b_env, acts, refs=None, what="", bitwise=False):
    k = int(acts.shape[0])
    (obs, ref), rew, term = a_env.rollout(acts, record_every=1, references=refs)
    (jx, ju), ((o_b, r_b), w_b, t_b) = b_env.rollout_jacobians(acts, references=refs)
    nx, nu = b_env.sim.jacobian_dims()
    assert jx.shape == (k, b_env.sim.n, nx, nx) and jx.dtype == b_env.sim.dtype, what
    assert (ju is None) == (nu == 0), what
    if ju is not None:
        assert ju.shape == (k, b_env.sim.n, nx, nu)
    assert bool(torch.isfinite(jx).all()), what
    for name, x, y in (("obs", obs, o_b), ("ref", ref, r_b), ("reward", rew, w_b), ("terminated", term, t_b)):
        # bit for bit where the twin's rollout runs the general kernel; against its PLAIN kernel equal values (the sign of a zero may differ)
        (_eq if bitwise else _same)(torch, y, x, (what, name))
    assert a_env.sim.clock() == b_env.sim.clock(), what
    return jx, ju, term


@pytest.mark.parametrize("autoreset", ["same_step", "none"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("family", list(ENV_IDS))
def test_primal_equals_recorded_rollout(torch_cuda, family, dtype, autoreset):
    torch = torch_cuda
    a_env, b_env = _make(family, dtype, "aos", autoreset), _make(family, dtype, "aos", autoreset)
    terminated = 0
    for seed, k in enumerate(HORIZONS):
        if autoreset == "none":
            a_env.reset()
            b_env.reset()
        _, _, term = _pair(torch, a_env, b_env, _actions(torch, a_env, k, seed=seed), what=(family, dtype, autoreset, k))
        terminated += int(term.sum())
    assert terminated > 0
    assert np.array_equal(_blob(a_env), _blob(b_env))
    _next_steps(torch, a_env, b_env)


def test_reference_feed(torch_cuda):
    from test_gpu_rollout_returns import _ext_env

    torch = torch_cuda
    a_env, b_env = _ext_env(), _ext_env()
    sim = a_env.sim
    for k in (64, 7):
        refs = torch.as_tensor(np.random.default_rng(k).uniform(-0.9, 0.9, size=(k,) + sim._shape(sim.n_ref)), dtype=sim.dtype, device="cuda")
        _pair(torch, a_env, b_env, _actions(torch, a_env, k, seed=k), refs=refs.contiguous(), what=("feed", k), bitwise=True)
    assert np.array_equal(_blob(a_env), _blob(b_env))


def test_per_env_blocks_draws_and_identities(torch_cuda):
    torch = torch_cuda
    for mode in ("blocks", "draws", "identities"):
        a_env, b_env = _make("pmsm"), _make("pmsm")
        r_s = float(a_env.sim.cfg.motor_param[K.MP_R_S])
        for env in (a_env, b_env):
            if mode == "blocks":
                env.set_env_parameters(motor_parameter={"r_s": r_s * np.linspace(0.8, 1.2, N)})
            elif mode == "draws":
                env.randomize_env_parameters(motor_parameter={"r_s": (0.8 * r_s, 1.2 * r_s)})
                env.reset()
            else:
                env.step(_actions(torch, env, 1, seed=3)[0])
                env.restore_envs(env.snapshot_envs(list(range(8)), rng=True), idx=list(range(100, 164)), rows=np.repeat(np.arange(8), 8), rng="source")
        for k in (64, 7):
            _pair(torch, a_env, b_env, _actions(torch, a_env, k, seed=k), what=(mode, k), bitwise=True)  # both run ENVP
        _next_steps(torch, a_env, b_env)


_POLY = dict(a=0.01, b=0.02, c=1e-4, j_load=1e-3)
PER_ENV_CASES = {  # env id, polynomial load?, which parameter dict, slot
    "pmsm-r_s": ("Cont-CC-PMSM-v0", False, "motor", "r_s"),
    "pmsm-poly-c": ("Cont-CC-PMSM-v0", True, "load", "c"),
    "pmsm-poly-j_load": ("Cont-CC-PMSM-v0", True, "load", "j_load"),
    "scim-poly-r_r": ("Cont-CC-SCIM-v0", True, "motor", "r_r"),
    "dfim-l_m": ("Cont-CC-DFIM-v0", False, "motor", "l_m"),
}


@pytest.mark.parametrize("case", list(PER_ENV_CASES))
def test_per_env_parameters_give_the_single_parameter_jacobians(torch_cuda, case):
    """env i of a handle with a per-env parameter has the Jacobians of a handle whose shared parameter is env i's, over three steps"""
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200 import physical_systems as ps

    torch = torch_cuda
    env_id, poly, kind, slot = PER_ENV_CASES[case]
    m = 64
    scale = np.linspace(0.7, 1.3, m)

    def make(extra=None):
        load_p = dict(_POLY, **(extra or {})) if kind == "load" else dict(_POLY)
        kw = dict(load=ps.PolynomialStaticLoad(load_parameter=load_p)) if poly else {}
        if kind == "motor" and extra:
            kw["motor"] = dict(motor_parameter=extra)
        env = gem.make(env_id, num_envs=m, device="cuda", dtype="float64", autoreset="none", seed=3, **kw)
        env.reset()
        return env

    env = make()
    ps_ = env.physical_system
    base = float(ps_.mechanical_load.load_parameter[slot] if kind == "load" else ps_.electrical_motor.motor_parameter[slot])
    if kind == "load":
        env.set_env_parameters(load_parameter={slot: base * scale})
    else:
        env.set_env_parameters(motor_parameter={slot: base * scale})
    x0 = env.sim.get_ode_state()
    x0[:, 0] = 150.0  # outside the static-friction band: the speed-dependent load terms are live
    env.sim.set_ode_state(x0)
    acts = _actions(torch, env, 3, seed=4)
    (jx, ju), _ = env.sim.rollout_jacobians(acts)
    for i in (0, 21, 63):
        one = make({slot: base * scale[i]})
        one.sim.set_ode_state(x0)
        (jx1, ju1), _ = one.sim.rollout_jacobians(acts)
        for k in range(3):
            assert torch.allclose(jx[k, i], jx1[k, i], rtol=1e-12, atol=1e-12), (case, i, k)
            assert torch.allclose(ju[k, i], ju1[k, i], rtol=1e-12, atol=1e-12), (case, i, k)
    assert not torch.allclose(jx[:, 0], jx[:, 63], rtol=1e-9, atol=0)  # the slot moves the Jacobians


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("family", list(ENV_IDS))
def test_fusion_identity(torch_cuda, family, dtype):
    torch = torch_cuda
    a_env, b_env = _make(family, dtype), _make(family, dtype)
    k = 7
    acts = _actions(torch, a_env, k, seed=1)
    (jx, ju), _ = a_env.sim.rollout_jacobians(acts)
    for j in range(k):
        (jx1, ju1), _ = b_env.sim.rollout_jacobians(acts[j:j + 1].contiguous())
        assert torch.equal(_bits(torch, jx[j]), _bits(torch, jx1[0])), (family, dtype, j)
        if ju is not None:
            assert torch.equal(_bits(torch, ju[j]), _bits(torch, ju1[0])), (family, dtype, j)
    assert np.array_equal(_blob(a_env), _blob(b_env))


INTERLOCK_CASES = {  # finite converters with interlocking time: two segments, or three with two different times
    "pmsm": ("Finite-CC-PMSM-v0", 2e-6, -1.0),
    "dfim-two-times": ("Finite-CC-DFIM-v0", 2e-6, 5e-6),
    "extex-two-times": ("Finite-CC-ExtExDc-v0", 5e-6, 2e-6),
    "permex": ("Finite-CC-PermExDc-v0", 3e-6, -1.0),
}


@pytest.mark.parametrize("autoreset", ["same_step", "none"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("case", list(INTERLOCK_CASES))
def test_interlocked_finite_primal_and_fusion(torch_cuda, case, dtype, autoreset):
    """twins driven through the same steps (the switching state persists): A records a rollout, B runs rollout_jacobians — same outputs,
    clock and checkpoint; then a K-step launch against K one-step launches on a third twin, bit for bit"""
    from gym_electric_motor_b200.vector_sim import VectorSim

    torch = torch_cuda
    env_id, til, til1 = INTERLOCK_CASES[case]
    cfg = _cfg(env_id, N, dtype, til=til, til1=til1, autoreset=autoreset)
    sims = [VectorSim(cfg) for _ in range(3)]
    for s_ in sims:
        s_.reset()
    n_switch = {K.CONV_B6: 8, K.CONV_4QC: 4, K.CONV_2QC: 3, K.CONV_1QC: 2}
    hi = np.array([n_switch[cfg.converter_kind[j]] for j in range(sims[0].n_act)])
    rng = np.random.default_rng(1)
    a_sim, b_sim, c_sim = sims
    for k in HORIZONS:
        if autoreset == "none":
            for s_ in sims:
                s_.reset()
        acts = torch.as_tensor(rng.integers(0, hi, (k, N, sims[0].n_act)), dtype=torch.int32, device="cuda").contiguous()
        obs, ref, rew, term = a_sim.rollout(acts, record_every=1)
        (jx, ju), (o_b, r_b, w_b, t_b) = b_sim.rollout_jacobians(acts)
        assert ju is None and bool(torch.isfinite(jx).all())
        for name, x, y in (("obs", obs, o_b), ("ref", ref, r_b), ("reward", rew, w_b), ("terminated", term, t_b)):
            _same(torch, y, x, (case, dtype, autoreset, k, name))
        assert a_sim.clock() == b_sim.clock()
        for j in range(k):
            (jx1, _), _ = c_sim.rollout_jacobians(acts[j:j + 1].contiguous())
            assert torch.equal(_bits(torch, jx[j]), _bits(torch, jx1[0])), (case, dtype, autoreset, k, j)
    assert np.array_equal(a_sim.state_dict()["blob"], b_sim.state_dict()["blob"])
    assert np.array_equal(b_sim.state_dict()["blob"], c_sim.state_dict()["blob"])


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_cuda_graph_capture(torch_cuda, dtype):
    torch = torch_cuda
    k = 12
    eager, cap, rec = _make("pmsm", dtype), _make("pmsm", dtype), _make("pmsm", dtype)
    nx, nu = cap.sim.jacobian_dims()
    static = _actions(torch, cap, k, seed=0).clone()
    dt = cap.sim.dtype
    jx = torch.empty((k, N, nx, nx), dtype=dt, device="cuda")
    ju = torch.empty((k, N, nx, nu), dtype=dt, device="cuda")
    obs = torch.empty((k, N, cap.sim.n_state), dtype=dt, device="cuda")
    rew = torch.empty((k, N), dtype=dt, device="cuda")
    term = torch.empty((k, N), dtype=torch.uint8, device="cuda")
    for env in (eager, cap, rec):
        env.sim.set_device_clock(True)
    sim = cap.sim
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sim.rollout_jacobians_into(static, k, jx, ju, obs, None, rew, term)
    for rnd in range(3):
        acts = _actions(torch, eager, k, seed=10 + rnd)
        static.copy_(acts)
        graph.replay()
        (ex, eu), (eo, _, _, _) = eager.sim.rollout_jacobians(acts)
        assert torch.equal(_bits(torch, jx), _bits(torch, ex)), rnd
        assert torch.equal(_bits(torch, ju), _bits(torch, eu)), rnd
        assert torch.equal(_bits(torch, obs), _bits(torch, eo)), rnd
        ro, _, rw, rt = rec.sim.rollout(acts, record_every=1)  # the recorded rollout the captured launch replaces (PLAIN kernel)
        _same(torch, obs, ro, (rnd, "obs vs rollout"))
        _same(torch, rew, rw, (rnd, "reward vs rollout"))
        assert torch.equal(term, rt), rnd
    assert eager.sim.clock() == cap.sim.clock() == rec.sim.clock()
    assert np.array_equal(_blob(eager), _blob(cap)) and np.array_equal(_blob(cap), _blob(rec))


# ---------------------------------------------------------------------------------------------------------------- known answer
@pytest.mark.parametrize("env_id", ["Cont-CC-PMSM-v0", "Cont-CC-SynRM-v0"])
def test_known_answer_linear_current_dynamics(torch_cuda, env_id):
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.vector_sim import VectorSim

    torch = torch_cuda
    m, ns = 40, 3
    cfg = gem.make(env_id, num_envs=m, dtype="float64", autoreset="none", seed=3).build_config()
    cfg.load_kind, cfg.solver_kind, cfg.solver_nsteps = K.LOAD_CONST_SPEED, K.SOLVER_RK4, ns
    sim = VectorSim(cfg)
    sim.reset()
    rng = np.random.default_rng(0)
    x0 = sim.get_ode_state().cpu().numpy()
    x0[:, 0] = rng.uniform(-300, 300, m)
    x0[:, 3] = rng.uniform(-3, 3, m)
    sim.set_ode_state(x0)
    acts = torch.as_tensor(rng.uniform(-0.6, 0.6, (1, m, 3)), dtype=torch.float64, device="cuda")
    (jx, ju), _ = sim.rollout_jacobians(acts)
    jx, ju = jx[0].cpu().numpy(), ju[0].cpu().numpy()
    mp = cfg.motor_param
    p, r, ld, lq = mp[K.MP_P], mp[K.MP_R_S], mp[K.MP_L_D], mp[K.MP_L_Q]
    h = cfg.tau / ns
    t23 = np.array([[2 / 3, -1 / 3, -1 / 3], [0.0, 1 / np.sqrt(3), -1 / np.sqrt(3)]])
    worst_x = worst_u = 0.0
    for i in range(m):
        w, eps = x0[i, 0], x0[i, 3]
        mm = np.array([[-r / ld, p * w * lq / ld], [-p * w * ld / lq, -r / lq]])
        hm = h * mm
        phi = sum(np.linalg.matrix_power(hm, j) / math.factorial(j) for j in range(5))
        gam = sum(h ** j * np.linalg.matrix_power(mm, j - 1) / math.factorial(j) for j in range(1, 5))
        phi_n = np.linalg.matrix_power(phi, ns)
        gam_n = sum(np.linalg.matrix_power(phi, s) @ gam for s in range(ns))
        c, s = np.cos(eps), np.sin(eps)
        b = np.diag([1 / ld, 1 / lq]) @ np.array([[c, s], [-s, c]]) @ t23 * (0.5 * cfg.u_sup)
        jxb, jub = jx[i, 1:3, 1:3], ju[i, 1:3, :]
        worst_x = max(worst_x, (np.abs(jxb - phi_n).max(0) / np.abs(phi_n).max(0)).max())
        ref_u = gam_n @ b
        worst_u = max(worst_u, (np.abs(jub - ref_u).max(0) / np.abs(ref_u).max(0)).max())
        assert np.array_equal(jx[i, 0], np.eye(4)[0])  # constant speed: omega's row is e_omega
        assert np.all(ju[i, 0] == 0)
    assert worst_x <= 1e-13 and worst_u <= 1e-13, (worst_x, worst_u)


# ---------------------------------------------------------------------------------------------------------------- finite differences
_KEEP = []


def _profile(t, amplitude, frequency):
    return amplitude * np.sin(2 * np.pi * frequency * t)


def _cfg(env_id, n, dtype, solver=K.SOLVER_RK4, nsteps=1, load=None, supply=None, action_dq=0, til=None, til1=None, autoreset="none"):
    import gym_electric_motor_b200 as gem

    kw = {}
    if load == "ext":  # a speed profile the load follows with its time constant (ExternalSpeedLoad)
        kw["load"] = gem.physical_systems.ExternalSpeedLoad(speed_profile=_profile, speed_profile_kwargs=dict(amplitude=120.0, frequency=7.0),
                                                          tau=1e-4, horizon_steps=2000)
    env = gem.make(env_id, num_envs=n, dtype=dtype, autoreset=autoreset, seed=11, **kw)
    _KEEP.append(env)  # the config points into the load's speed table, which the env owns
    cfg = env.build_config()
    cfg.solver_kind, cfg.solver_nsteps = solver, nsteps
    if load == "const":
        cfg.load_kind = K.LOAD_CONST_SPEED
    elif load == "poly":
        cfg.load_kind = K.LOAD_POLY_STATIC
        cfg.load_param[K.LP_A], cfg.load_param[K.LP_B], cfg.load_param[K.LP_C] = 0.01, 0.02, 1e-4
        cfg.load_param[K.LP_J_LOAD] = 1e-3
    if supply == "ac1":
        cfg.supply_kind, cfg.supply_param[0], cfg.supply_param[1], cfg.supply_param[2] = K.SUPPLY_AC1, 50.0, 0.3, 1.0
    if action_dq:
        cfg.action_dq = action_dq
    if til is not None:
        cfg.interlocking_time = til
    if til1 is not None:
        cfg.interlocking_time1 = til1
    return cfg


FD_CASES = {
    "permex-poly-rk4": ("Cont-CC-PermExDc-v0", dict(load="poly")),
    "series-poly-euler3": ("Cont-CC-SeriesDc-v0", dict(load="poly", solver=K.SOLVER_EULER, nsteps=3)),
    "shunt-const-rk4-3": ("Cont-CC-ShuntDc-v0", dict(load="const", nsteps=3)),
    "extex-poly-rk4-interlock": ("Cont-CC-ExtExDc-v0", dict(load="poly", til=2e-6)),
    "pmsm-poly-euler1": ("Cont-CC-PMSM-v0", dict(load="poly", solver=K.SOLVER_EULER)),
    "pmsm-const-rk4-dq": ("Cont-CC-PMSM-v0", dict(load="const", action_dq=1)),
    "synrm-poly-rk4-3-ac1": ("Cont-CC-SynRM-v0", dict(load="poly", nsteps=3, supply="ac1")),
    "pmsm-ext-rk4-3": ("Cont-CC-PMSM-v0", dict(load="ext", nsteps=3)),
    "extex-ext-euler3": ("Cont-CC-ExtExDc-v0", dict(load="ext", solver=K.SOLVER_EULER, nsteps=3)),
    "eesm-poly-rk4": ("Cont-CC-EESM-v0", dict(load="poly")),
    "eesm-const-euler3-dq": ("Cont-CC-EESM-v0", dict(load="const", solver=K.SOLVER_EULER, nsteps=3, action_dq=1)),
    "scim-poly-rk4": ("Cont-CC-SCIM-v0", dict(load="poly")),
    "scim-const-rk4-dq": ("Cont-CC-SCIM-v0", dict(load="const", action_dq=1)),
    "dfim-poly-rk4-3": ("Cont-CC-DFIM-v0", dict(load="poly", nsteps=3)),
    "dfim-const-euler1": ("Cont-CC-DFIM-v0", dict(load="const", solver=K.SOLVER_EULER)),
    "pmsm-finite-poly-rk4": ("Finite-CC-PMSM-v0", dict(load="poly", til=0.0)),
    "scim-finite-const-rk4": ("Finite-CC-SCIM-v0", dict(load="const", til=0.0)),
    "permex-finite-poly-euler3": ("Finite-CC-PermExDc-v0", dict(load="poly", solver=K.SOLVER_EULER, nsteps=3, til=0.0)),
    # interlocking time: two switching segments per switching step, three with two different times (the DFIM's two bridges)
    "pmsm-finite-interlock-poly-rk4": ("Finite-CC-PMSM-v0", dict(load="poly", til=2e-6)),
    "scim-finite-interlock-const-euler3": ("Finite-CC-SCIM-v0", dict(load="const", solver=K.SOLVER_EULER, nsteps=3, til=3e-6)),
    "dfim-finite-interlock2-poly-rk4": ("Finite-CC-DFIM-v0", dict(load="poly", til=2e-6, til1=5e-6)),
    "dfim-finite-interlock2b-const-rk4-3": ("Finite-CC-DFIM-v0", dict(load="const", nsteps=3, til=4e-6, til1=1e-6)),
    "permex-finite-interlock-poly-rk4": ("Finite-CC-PermExDc-v0", dict(load="poly", til=2e-6)),
    "extex-finite-interlock2-poly-rk4": ("Finite-CC-ExtExDc-v0", dict(load="poly", til=2e-6, til1=5e-6)),
}


@pytest.mark.parametrize("case", list(FD_CASES))
def test_against_central_differences(torch_cuda, case):
    from gym_electric_motor_b200.vector_sim import VectorSim

    torch = torch_cuda
    env_id, kw = FD_CASES[case]
    m = 32
    # base points: the state after a few random steps (angle kept away from the wrap)
    c0 = _cfg(env_id, m, "float64", **kw)
    s0 = VectorSim(c0)
    s0.reset()
    nx, nu = s0.jacobian_dims()
    rng = np.random.default_rng(5)

    n_switch = {K.CONV_B6: 8, K.CONV_4QC: 4, K.CONV_2QC: 3, K.CONV_1QC: 2, K.CONV_NONE: 1}

    def draw_actions(k, n):
        if s0.finite:  # a switching state per converter slot, within the slot's range
            hi = np.array([n_switch[c0.converter_kind[j]] for j in range(s0.n_act)])
            return torch.as_tensor(rng.integers(0, hi, (k, n, s0.n_act)), dtype=torch.int32, device="cuda").contiguous()
        # beyond +-1 on purpose: about a quarter of the legs clip, where the action derivative is 0
        return torch.as_tensor(rng.uniform(-1.3, 1.3, (k, n, s0.n_act)), dtype=torch.float64, device="cuda").contiguous()

    s0.rollout(draw_actions(3, m), record_every=1)
    x0 = s0.get_ode_state().cpu().numpy()
    has_eps = c0.motor_kind >= K.MOTOR_PMSM
    if has_eps:
        x0[:, -1] = np.clip(x0[:, -1], -2.5, 2.5)
    if s0.finite:  # no current exactly at 0: there a leg waiting in its interlock state switches its voltage with the current's sign
        cur = slice(1, c0.motor_kind >= K.MOTOR_PMSM and 3 or x0.shape[1])
        x0[:, cur] += rng.choice([-1.0, 1.0], x0[:, cur].shape) * rng.uniform(0.5, 2.0, x0[:, cur].shape)
    if c0.motor_kind in (K.MOTOR_SCIM, K.MOTOR_DFIM):  # a built-up rotor flux: near zero the field angle turns with any perturbation
        mag, ang = rng.uniform(0.2, 0.8, m), rng.uniform(-np.pi, np.pi, m)
        x0[:, 3], x0[:, 4] = mag * np.cos(ang), mag * np.sin(ang)
    a0 = draw_actions(1, m)[0].cpu().numpy()
    # finite converters: one step with other switching states first, the same on every copy of a base env (the switching state persists
    # across steps and decides, with an interlocking time, how many segments the linearised step has)
    a_prev = draw_actions(1, m)[0].cpu().numpy() if s0.finite else None
    ncol = nx + nu
    reps = 2 * ncol + 1
    n = m * reps
    cfd = _cfg(env_id, n, "float64", **kw)
    sim = VectorSim(cfd)
    sim.reset()
    xs = np.repeat(x0, reps, axis=0)
    acts = np.repeat(a0, reps, axis=0).astype(np.float64 if nu else np.int32)
    steps = np.zeros(ncol)
    for c in range(ncol):
        if c < nx:
            hc = 1e-6 * max(1.0, float(np.abs(x0[:, c]).max()))
            xs[2 * c + 1::reps, c] += hc
            xs[2 * c + 2::reps, c] -= hc
        else:
            hc = 1e-6
            acts[2 * c + 1::reps, c - nx] += hc
            acts[2 * c + 2::reps, c - nx] -= hc
        steps[c] = hc
    if s0.finite:
        sim.step(torch.as_tensor(np.repeat(a_prev, reps, axis=0), device="cuda").contiguous())
    sim.set_ode_state(xs)
    a_t = torch.as_tensor(acts[None], device="cuda").contiguous()
    (jx, ju), _ = sim.rollout_jacobians(a_t)
    x1 = sim.get_ode_state().cpu().numpy().reshape(m, reps, nx)
    jac = jx[0].cpu().numpy()[::reps]
    if nu:
        jac = np.concatenate([jac, ju[0].cpu().numpy()[::reps]], axis=2)
    # the same base points in fp32
    c32 = _cfg(env_id, m, "float32", **kw)
    s32 = VectorSim(c32)
    s32.reset()
    if s0.finite:
        s32.step(torch.as_tensor(a_prev, device="cuda").contiguous())
    s32.set_ode_state(x0)
    a32 = torch.as_tensor(a0[None], device="cuda").to(torch.int32 if nu == 0 else torch.float32).contiguous()
    (jx32, ju32), _ = s32.rollout_jacobians(a32)
    jac32 = jx32[0].double().cpu().numpy()
    if nu:
        jac32 = np.concatenate([jac32, ju32[0].double().cpu().numpy()], axis=2)

    def wrap(d):
        if has_eps:
            d = d.copy()
            d[..., -1] = (d[..., -1] + np.pi) % (2 * np.pi) - np.pi
        return d

    skipped = total = 0
    worst64 = worst32 = 0.0
    for b in range(m):
        for c in range(ncol):
            hc = steps[c]
            plus, minus, mid = x1[b, 2 * c + 1], x1[b, 2 * c + 2], x1[b, 0]
            fd = wrap(plus - minus) / (2 * hc)
            right, left = wrap(plus - mid) / hc, wrap(mid - minus) / hc
            scale = max(np.abs(fd).max(), 1e-300)
            total += 1
            if np.abs(right - left).max() / scale > 1e-4:  # the stencil straddles a kink (clipping, current sign, friction branch)
                skipped += 1
                continue
            worst64 = max(worst64, np.abs(jac[b, :, c] - fd).max() / scale)
            worst32 = max(worst32, np.abs(jac32[b, :, c] - fd).max() / scale)
    assert skipped <= total // 100, (case, skipped, total)
    assert worst64 <= 1e-7, (case, worst64)
    assert worst32 <= 2e-4, (case, worst32)


# ---------------------------------------------------------------------------------------------------------------- the reference's Jacobian
@pytest.mark.parametrize("dtype,tol", [("float64", 1e-12), ("float32", 1e-5)])
def test_euler_step_equals_reference_system_jacobian(torch_cuda, dtype, tol):
    """with Euler and one sub-step x_{k+1} = x_k + tau f(x_k, u): every column of jac_x but the angle's (where the rotation of the converter
    voltages enters) is I + tau J_ref, J_ref = the reference's SCMLSystem._system_jacobian at the fixture's points (set with set_ode_state;
    continuous converters without interlocking and without dq actions, so the applied voltages do not depend on the other states)"""
    import os

    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200 import physical_systems as ps

    torch = torch_cuda
    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jacobians", "system_jacobians.npz"))
    for c in sorted({k.split("/")[0] for k in d.files}):
        motor, load = c.split("_")
        x, jref, tau = d[c + "/x"], d[c + "/jac"], float(d[c + "/tau"])
        m, nx = x.shape
        ld = ps.ConstantSpeedLoad(omega_fixed=80.0) if load == "const" else ps.PolynomialStaticLoad(load_parameter=dict(a=0.01, b=0.02, c=1e-4, j_load=1e-3))
        env = gem.make(f"Cont-CC-{motor}-v0", num_envs=m, device="cuda", dtype=dtype, load=ld, ode_solver=ps.EulerSolver(), autoreset="none", seed=1)
        env.reset()
        sim = env.sim
        assert sim.cfg.solver_kind == K.SOLVER_EULER and sim.cfg.solver_nsteps == 1 and abs(sim.cfg.tau - tau) < 1e-15
        sim.set_ode_state(x)
        acts = torch.as_tensor(np.random.default_rng(0).uniform(-0.5, 0.5, (1, m, sim.n_act)), dtype=sim.dtype, device="cuda")
        (jx, _), _ = sim.rollout_jacobians(acts)
        jx = jx[0].double().cpu().numpy()
        expect = np.eye(nx)[None] + tau * jref
        cols = range(nx - 1) if motor in ("PMSM", "SynRM", "EESM", "SCIM", "DFIM") else range(nx)
        for j in cols:
            err = np.abs(jx[:, :, j] - expect[:, :, j]).max(1) / np.abs(expect[:, :, j]).max(1)
            assert err.max() <= tol, (c, dtype, j, err.max())
