"""Parameter sensitivities on the device: `rollout_param_sensitivities(actions, params)` runs K steps in one launch and carries
S = d x / d theta of every env's own physical parameters.

- Primal identity: twin handles with equal seeds, A runs `rollout(actions, record_every=1)`, B runs `rollout_param_sensitivities`; outputs,
  clock and the persistent state (checkpoint blob) must be the same, with shared coefficients and with per-env blocks.
- Chaining: K1 + K2 launches carrying `sens_last` equal one K launch bit for bit.
- Carry: the fused S against the recursion S_{k+1} = J_x[k] S_k + P_k with J_x from `rollout_jacobians` and P_k from one-step launches.
- Central differences of the device's float64 step: perturbed copies theta_j (1 +- h) are envs of one handle with per-env blocks.
- Per-env blocks that hold the shared parameters give the shared handle's bits.
- System identification: Gauss-Newton on S recovers perturbed motor and load parameters from recorded trajectories."""
import numpy as np
import pytest

from fd_helpers import SLOT, _cfg, _wrap, build_up_flux, currents_off_zero, sens_check, switching_states
from gpu_helpers import ENV_IDS, _actions, _blob, _eq, _make, _next_steps, _same, torch_cuda  # noqa: F401
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

N = 300
PARAMS = {"permex": ["r_a", "l_a", "psi_e", "j_rotor"], "extex": ["r_a", "l_a", "l_e", "r_e", "l_e_prime"], "pmsm": ["r_s", "l_d", "l_q", "psi_p"],
          "eesm": ["r_s", "l_d", "l_q", "r_e", "l_m", "l_e"], "scim": ["r_s", "r_r", "l_m", "l_sigs", "l_sigr"],
          "dfim": ["r_s", "r_r", "l_m", "l_sigs", "l_sigr"]}
PARAMS.update({f + "_finite": PARAMS[f] for f in list(PARAMS)})
# every family with a continuous and with a finite converter
PRIMAL_IDS = dict(ENV_IDS, permex_finite="Finite-CC-PermExDc-v0", extex_finite="Finite-CC-ExtExDc-v0", eesm_finite="Finite-CC-EESM-v0",
                  scim_finite="Finite-CC-SCIM-v0", dfim_finite="Finite-CC-DFIM-v0")


def _pair(torch, a_env, b_env, acts, names, sens0=None, what=""):
    k = int(acts.shape[0])
    (obs, ref), rew, term = a_env.rollout(acts, record_every=1)
    (so, sl), ((o_b, r_b), w_b, t_b) = b_env.rollout_param_sensitivities(acts, names, sens0=sens0)
    nx = b_env.sim.n_ode
    assert so.shape == (k, b_env.sim.n, nx, len(names)) and so.dtype == b_env.sim.dtype and sl.shape == (b_env.sim.n, nx, len(names)), what
    assert bool(torch.isfinite(so).all()), what
    for name, x, y in (("obs", obs, o_b), ("ref", ref, r_b), ("reward", rew, w_b), ("terminated", term, t_b)):
        _same(torch, y, x, (what, name))
    assert a_env.sim.clock() == b_env.sim.clock(), what
    return so, sl, t_b


@pytest.mark.parametrize("blocks", ["shared", "envp"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("family", list(PRIMAL_IDS))
def test_primal_identity_and_chaining(torch_cuda, family, dtype, blocks):
    import gym_electric_motor_b200 as gem

    torch = torch_cuda

    def make():
        env = gem.make(PRIMAL_IDS[family], num_envs=N, device="cuda", dtype=dtype, layout="aos", autoreset="same_step", seed=7)
        env.reset()
        return env

    a_env, b_env, c_env = make(), make(), make()
    x0 = a_env.sim.get_ode_state()
    x0[:N // 4, 1] = 1e3  # a first current far beyond its limit: these envs terminate in the first step and are reset in it
    for env in (a_env, b_env, c_env):
        env.sim.set_ode_state(x0)
    names = PARAMS[family]
    if blocks == "envp":
        for env in (a_env, b_env, c_env):
            base = env.sim.cfg.motor_param[env.param_slots([names[0]])[0]]
            env.set_env_parameters(motor_parameter={names[0]: base * np.linspace(0.8, 1.2, N)})
    terminated = 0
    for seed, k in enumerate((64, 7, 1)):
        acts = _actions(torch, a_env, k, seed=seed)
        so, sl, term = _pair(torch, a_env, b_env, acts, names, what=(family, dtype, blocks, k))
        terminated += int(term.sum())
        # the same steps as two chained launches on the third twin
        k1 = k // 2
        if k1:
            (s1, l1), _ = c_env.rollout_param_sensitivities(acts[:k1], names)
            (s2, l2), _ = c_env.rollout_param_sensitivities(acts[k1:], names, sens0=l1)
            _eq(torch, torch.cat([s1, s2]), so, (family, dtype, blocks, k, "chained sens_out"))
            _eq(torch, l2, sl, (family, dtype, blocks, k, "chained sens_last"))
        else:
            c_env.rollout_param_sensitivities(acts, names)
        alive = ~term[-1].bool()
        _eq(torch, so[-1][alive], sl[alive], "sens_out[K-1] is sens_last where the last step did not reset")
        assert bool((sl[~alive] == 0).all()), "an env reset in the last step carries S = 0"
    assert terminated > 0
    assert np.array_equal(_blob(a_env), _blob(b_env)) and np.array_equal(_blob(a_env), _blob(c_env))
    _next_steps(torch, a_env, b_env)


def _poly_load(**over):
    import gym_electric_motor_b200 as gem

    p = dict(a=0.01, b=0.02, c=1e-4, j_load=1e-3)
    p.update(over)
    return gem.physical_systems.PolynomialStaticLoad(load_parameter=p)


def _env(env_id, n, dtype="float64", seed=3, **kw):
    import gym_electric_motor_b200 as gem

    env = gem.make(env_id, num_envs=n, device="cuda", dtype=dtype, autoreset="none", seed=seed, **kw)
    env.reset()
    return env


@pytest.mark.parametrize("family", ["pmsm", "scim", "pmsm_finite", "eesm"])
def test_carry_against_the_jacobian_recursion(torch_cuda, family):
    torch = torch_cuda
    k = 16
    kw = dict(load=_poly_load()) if family != "pmsm_finite" else {}
    envs = [_env(ENV_IDS[family], N, **kw) for _ in range(3)]
    names = PARAMS[family] + (["j_rotor", "b"] if kw else [])
    x0 = envs[0].sim.get_ode_state()
    if kw:
        x0[:, 0] = torch.linspace(-200, 200, N, dtype=torch.float64, device="cuda")
    for env in envs:
        env.sim.set_ode_state(x0)
    acts = _actions(torch, envs[0], k, seed=5)
    s0 = torch.as_tensor(np.random.default_rng(1).normal(size=(N, envs[0].sim.n_ode, len(names))), device="cuda")
    (so, _), _ = envs[0].rollout_param_sensitivities(acts, names, sens0=s0)
    (jx, _), _ = envs[1].rollout_jacobians(acts)
    s = s0
    for j in range(k):
        (p1, _), _ = envs[2].rollout_param_sensitivities(acts[j:j + 1], names)
        s = torch.matmul(jx[j], s) + p1[0]
        scale = s.abs().amax(dim=(1, 2), keepdim=True).clamp_min(1e-300)
        err = ((so[j] - s).abs() / scale).max().item()
        assert err <= 1e-12, (family, j, err)


def _fd_case(torch, env_id, names, k, m=16, dtype="float64", rel_h=1e-4, tol=1e-7, omega=None, expect_zero=(), tweak=None, **cfg_kw):
    """central differences of the float64 step against S of a `dtype` handle: the perturbed copies theta_j (1 +- h) are envs of ONE float64
    handle with per-env blocks, driven one step per launch so that every step's state can be read.  Every entry must be within tol of its
    column's scale plus the reference's own error: its row's rounding floor 64 eps (|x_r| + 1) / h and twice the distance between the
    central differences with steps h and 2h.  Stencils whose forward and backward differences disagree (a
    kink or a termination crossed between the copies) are counted and must be at most 1 % of all."""
    from gym_electric_motor_b200.vector_sim import VectorSim

    n_p = len(names)
    copies = 1 + 4 * n_p  # per parameter: +h, -h, +2h, -2h
    slots = [SLOT[nm] for nm in names]
    c_fd, c_s = _cfg(env_id, m * copies, "float64", **cfg_kw), _cfg(env_id, m, dtype, **cfg_kw)
    for c in (c_fd, c_s):
        if tweak:
            tweak(c)
    fd, ss = VectorSim(c_fd), VectorSim(c_s)
    fd.reset()
    ss.reset()
    row = np.array(list(c_fd.motor_param) + list(c_fd.load_param))
    theta = row[slots]
    h = rel_h * np.where(theta != 0, np.abs(theta), 1.0)
    prm = np.tile(row, (m * copies, 1))
    for j, slot in enumerate(slots):
        for q, dq in enumerate((h[j], -h[j], 2 * h[j], -2 * h[j])):
            prm[(1 + 4 * j + q) * m:(2 + 4 * j + q) * m, slot] += dq
    fd.set_env_params(np.ascontiguousarray(prm[:, :K.MAX_MOTOR_PARAM]), np.ascontiguousarray(prm[:, K.MAX_MOTOR_PARAM:]))
    rng = np.random.default_rng(5)
    x0 = ss.get_ode_state().cpu().numpy()
    if omega is not None:
        x0[:, 0] = omega
    has_eps = c_s.motor_kind >= K.MOTOR_PMSM
    build_up_flux(rng, c_s, x0)
    currents_off_zero(rng, c_s, x0)
    ss.set_ode_state(x0)
    fd.set_ode_state(np.tile(x0, (copies, 1)))
    if ss.finite:
        a = switching_states(rng, c_s, (k, m, ss.n_act))
        acts = torch.as_tensor(a, dtype=torch.int32, device="cuda").contiguous()
    else:
        a = rng.uniform(-0.9, 0.9, (k, m, ss.n_act))
        acts = torch.as_tensor(a, dtype=ss.dtype, device="cuda").contiguous()
    acts_fd = torch.as_tensor(np.tile(a, (1, copies, 1)), dtype=fd.act_dtype, device="cuda").contiguous()
    nx = fd.n_ode
    sl = None
    kinks = total = 0
    for step in range(k):
        (so, sl), _ = ss.rollout_param_sens(acts[step:step + 1], slots, sens0=sl)
        fd.rollout(acts_fd[step:step + 1], 1)
        x = fd.get_ode_state().cpu().numpy().reshape(copies, m, nx)
        s = so[0].double().cpu().numpy()
        for j in range(n_p):
            mid = x[0]
            dup, ddn, dup2, ddn2 = x[1 + 4 * j] - mid, mid - x[2 + 4 * j], x[3 + 4 * j] - mid, mid - x[4 + 4 * j]
            if has_eps:
                for v in (dup, ddn, dup2, ddn2):
                    v[:, -1] = _wrap(v[:, -1])
            # the reference's own error: each row's rounding floor, and twice the distance to the 2h difference (that distance is 3/4 of
            # the 2h difference's truncation error, i.e. 3x the h difference's, plus rounding that reaches the row from the other states)
            d, scale, err, kink, bad = sens_check(s[:, :, j], dup, ddn, mid, h[j], tol, d2h=(dup2 + ddn2) / (4 * h[j]))
            if names[j] in expect_zero:
                assert np.all(s[:, :, j] == 0) and np.all(d == 0), (env_id, names[j], "a parameter that does not enter: exact 0")
                continue
            kinks += int(kink.sum())
            total += m
            assert not bad.any(), (env_id, dtype, names[j], step, (err / np.maximum(scale, 1e-300)).max(axis=1)[bad].max())
    assert kinks <= 0.01 * max(total, 1), (env_id, names, kinks, total)


MOTORS = {"permex": ("Cont-CC-PermExDc-v0", ["r_a", "l_a", "psi_e", "j_rotor", "a", "b", "c", "j_load"]),
          "series": ("Cont-CC-SeriesDc-v0", ["r_a", "l_a", "r_e", "l_e", "l_e_prime", "j_rotor", "b", "c"]),
          "shunt": ("Cont-CC-ShuntDc-v0", ["r_a", "l_a", "r_e", "l_e", "l_e_prime", "j_rotor", "b", "c"]),
          "extex": ("Cont-CC-ExtExDc-v0", ["r_a", "l_a", "r_e", "l_e", "l_e_prime", "j_rotor", "a", "b", "c", "j_load"]),
          "pmsm": ("Cont-CC-PMSM-v0", ["r_s", "l_d", "l_q", "psi_p", "j_rotor", "a", "b", "c", "j_load"]),
          "synrm": ("Cont-CC-SynRM-v0", ["r_s", "l_d", "l_q", "j_rotor", "b", "c"]),
          "eesm": ("Cont-CC-EESM-v0", ["r_s", "l_d", "l_q", "r_e", "l_m", "l_e", "j_rotor", "a", "b", "c", "j_load"]),
          "scim": ("Cont-CC-SCIM-v0", ["r_s", "r_r", "l_m", "l_sigs", "l_sigr", "j_rotor", "b", "c", "j_load"]),
          "dfim": ("Cont-CC-DFIM-v0", ["r_s", "r_r", "l_m", "l_sigs", "l_sigr", "j_rotor", "b", "c", "j_load"])}
SPEEDS = np.linspace(-150, 150, 16)  # running speeds of both signs, outside the static-friction band
MECH = ("j_rotor", "a", "b", "c", "j_load")


@pytest.mark.parametrize("k", [1, 8, 64])
@pytest.mark.parametrize("motor", list(MOTORS))
def test_central_differences_polynomial_load(torch_cuda, motor, k):
    env_id, names = MOTORS[motor]
    _fd_case(torch_cuda, env_id, names, k, omega=SPEEDS, load="poly")


def test_central_differences_friction_band(torch_cuda):
    """speeds inside the static-friction band |omega| <= omega_lim: the linear branch of the load"""
    def band(c):
        c.load_param[K.LP_A] = 2.0

    env_id, names = MOTORS["pmsm"]
    _fd_case(torch_cuda, env_id, names, 8, omega=np.linspace(-0.02, 0.02, 16), load="poly", tweak=band)


@pytest.mark.parametrize("motor", ["pmsm", "scim", "extex"])
@pytest.mark.parametrize("load", ["const", "ext"])
def test_central_differences_constant_and_external_speed(torch_cuda, motor, load):
    """the mechanical parameters do not enter under a load that holds or prescribes omega: exact 0 columns"""
    env_id, names = MOTORS[motor]
    _fd_case(torch_cuda, env_id, names, 8, omega=SPEEDS if load == "const" else None, expect_zero=MECH, load=load, nsteps=2)


@pytest.mark.parametrize("case", ["euler1", "euler3", "rk4_3"])
@pytest.mark.parametrize("motor", ["pmsm", "scim", "series"])
def test_central_differences_solvers(torch_cuda, motor, case):
    solver = K.SOLVER_EULER if case.startswith("euler") else K.SOLVER_RK4
    env_id, names = MOTORS[motor]
    _fd_case(torch_cuda, env_id, names, 8, omega=SPEEDS, load="poly", solver=solver, nsteps=int(case[-1]))


FINITE_CASES = {
    "pmsm": ("Finite-CC-PMSM-v0", dict(til=0.0)),
    "pmsm-interlock": ("Finite-CC-PMSM-v0", dict(til=2e-6)),
    "scim-interlock-euler3": ("Finite-CC-SCIM-v0", dict(til=3e-6, solver=K.SOLVER_EULER, nsteps=3)),
    "dfim-interlock2": ("Finite-CC-DFIM-v0", dict(til=2e-6, til1=5e-6)),
    "extex-interlock2": ("Finite-CC-ExtExDc-v0", dict(til=2e-6, til1=5e-6)),
}


@pytest.mark.parametrize("case", list(FINITE_CASES))
def test_central_differences_finite(torch_cuda, case):
    env_id, kw = FINITE_CASES[case]
    motor = {"PMSM": "pmsm", "SCIM": "scim", "DFIM": "dfim", "ExtExDc": "extex"}[env_id.split("-")[2]]
    _fd_case(torch_cuda, env_id, MOTORS[motor][1], 8, omega=SPEEDS, load="poly", **kw)


@pytest.mark.parametrize("case", ["pmsm-dq", "eesm-dq", "scim-dq", "synrm-ac1"])
def test_central_differences_dq_actions_and_ac_supply(torch_cuda, case):
    motor, what = case.split("-")
    env_id, names = MOTORS[motor]
    kw = dict(action_dq=1) if what == "dq" else dict(supply="ac1")
    _fd_case(torch_cuda, env_id, names, 8, omega=SPEEDS, load="poly", **kw)


@pytest.mark.parametrize("motor", ["pmsm", "scim", "dfim", "extex"])
def test_central_differences_float32(torch_cuda, motor):
    """the fp32 sensitivities against the float64 step's differences"""
    env_id, names = MOTORS[motor]
    _fd_case(torch_cuda, env_id, names, 8, dtype="float32", tol=2e-4, omega=SPEEDS, load="poly")


def test_blocks_of_the_shared_parameters_give_the_shared_bits(torch_cuda):
    """adopted RNG identities make per-env blocks that hold the shared parameters: the ENVP kernel derives the coefficient tangents from
    praw and must give the bits of the shared handle"""
    torch = torch_cuda
    a_env, b_env = _make("pmsm", "float64"), _make("pmsm", "float64")
    b_env.restore_envs(b_env.snapshot_envs(list(range(N)), rng=True), rng="source")
    acts = _actions(torch, a_env, 8, seed=2)
    names = PARAMS["pmsm"]
    (sa, la), _ = a_env.rollout_param_sensitivities(acts, names)
    (sb, lb), _ = b_env.rollout_param_sensitivities(acts, names)
    _eq(torch, sb, sa, "sens_out")
    _eq(torch, lb, la, "sens_last")


def test_per_env_parameters_match_their_own_handles(torch_cuda):
    """env i of a handle with drawn per-env parameters has the sensitivities of a handle whose shared parameters are env i's"""
    torch = torch_cuda
    names = ["r_s", "l_d", "l_q", "psi_p", "j_rotor", "b"]
    m = 32
    rng = np.random.default_rng(4)
    env = _env("Cont-CC-PMSM-v0", m, load=_poly_load())
    cfg = env.sim.cfg
    slots = env.param_slots(names)
    vals = {nm: cfg.motor_param[s] * rng.uniform(0.7, 1.3, m) for nm, s in zip(names, slots) if s < K.MAX_MOTOR_PARAM}
    lvals = {"b": cfg.load_param[K.LP_B] * rng.uniform(0.7, 1.3, m)}
    env.set_env_parameters(motor_parameter=vals, load_parameter=lvals)
    x0 = env.sim.get_ode_state()
    x0[:, 0] = 120.0
    env.sim.set_ode_state(x0)
    acts = _actions(torch, env, 6, seed=9)
    (so, _), _ = env.rollout_param_sensitivities(acts, names)
    for i in (0, 13, 31):
        one = _env("Cont-CC-PMSM-v0", m, load=_poly_load(b=float(lvals["b"][i])), motor=dict(motor_parameter={nm: float(v[i]) for nm, v in vals.items()}))
        one.sim.set_ode_state(x0)
        (s1, _), _ = one.rollout_param_sensitivities(acts, names)
        assert torch.allclose(so[:, i], s1[:, i], rtol=1e-12, atol=1e-300), i
    assert not torch.allclose(so[:, 0], so[:, 31], rtol=1e-6)


def _gauss_newton(torch, env_id, names, n, k, load_kw=None, omega=None, iters=8, seed=0):
    """record k steps of U(-1, 1) actions on a handle with the true parameters (+-30 % of nominal), then fit a handle that starts from the
    nominal ones: every iteration restores the same start, runs one k-step launch that records the states and S, and takes a Gauss-Newton
    step per env"""
    kw = dict(load=_poly_load(**(load_kw or {})))
    true_env, model = _env(env_id, n, **kw), _env(env_id, n, **kw)
    cfg = true_env.sim.cfg
    slots = true_env.param_slots(names)
    row = np.array(list(cfg.motor_param) + list(cfg.load_param))
    nominal = row[slots]
    rng = np.random.default_rng(seed)
    truth = nominal * rng.choice([0.7, 1.3], size=(n, len(names))) * rng.uniform(0.95, 1.05, size=(n, len(names)))

    def apply(env, theta):
        mp = {nm: theta[:, j] for j, (nm, s) in enumerate(zip(names, slots)) if s < K.MAX_MOTOR_PARAM}
        lp = {nm: theta[:, j] for j, (nm, s) in enumerate(zip(names, slots)) if s >= K.MAX_MOTOR_PARAM}
        env.set_env_parameters(motor_parameter=mp or None, load_parameter=lp or None)

    apply(true_env, truth)
    x0 = true_env.sim.get_ode_state()
    if omega is not None:
        x0[:, 0] = omega
    sim = true_env.sim
    acts = torch.as_tensor(rng.uniform(-1, 1, size=(k,) + sim._shape(sim.n_act)), dtype=sim.dtype, device="cuda").contiguous()
    nx = sim.n_ode
    rows = list(range(nx - 1)) if cfg.motor_kind >= K.MOTOR_PMSM else list(range(nx))  # the angle is a sum of omega: left out
    if cfg.load_kind == K.LOAD_CONST_SPEED:
        rows = rows[1:]

    # the recorded states of those rows: observation entries (x / limit) scaled back
    ode_names = {K.MOTOR_PMSM: ["omega", "i_sd", "i_sq"], K.MOTOR_SYNRM: ["omega", "i_sd", "i_sq"]}[cfg.motor_kind]
    state_names = list(true_env.state_names)
    obs_idx = [state_names.index(ode_names[r]) for r in rows]
    lim = torch.as_tensor([cfg.limits[q] for q in obs_idx], dtype=torch.float64, device="cuda")

    def traj(env):
        """one K-step launch from x0: the recorded states and S of every step"""
        env.sim.set_ode_state(x0)
        (so, _), (obs, _, _, _) = env.sim.rollout_param_sens(acts, slots)
        return obs[:, :, obs_idx] * lim, so[:, :, rows]

    x_true, _ = traj(true_env)
    w = 1.0 / x_true.abs().amax(dim=(0, 1)).clamp_min(1e-12)  # each state row in its own unit
    theta = np.tile(nominal, (n, 1))
    for _ in range(iters):
        apply(model, theta)
        x, s = traj(model)
        r = ((x_true - x) * w).permute(1, 0, 2).reshape(n, -1)  # [n, k * rows]
        jac = (s * w[None, None, :, None]).permute(1, 0, 2, 3).reshape(n, -1, len(names))
        sc = torch.as_tensor(theta, device="cuda")  # columns in relative units
        step = torch.linalg.lstsq(jac * sc[:, None, :], r[..., None]).solution[..., 0] * sc
        theta = theta + step.cpu().numpy()
    rel = np.abs(theta / truth - 1).max(axis=1)
    return rel


def test_system_identification_pmsm(torch_cuda):
    rel = _gauss_newton(torch_cuda, "Cont-CC-PMSM-v0", ["r_s", "l_d", "l_q", "psi_p"], 1024, 64, omega=100.0)
    assert np.mean(rel <= 1e-6) >= 0.99, (np.mean(rel <= 1e-6), np.median(rel), rel.max())


def test_system_identification_load(torch_cuda):
    rel = _gauss_newton(torch_cuda, "Cont-CC-PMSM-v0", ["j_rotor", "b", "c"], 1024, 64, load_kw=dict(a=0.0, b=0.02, c=1e-4, j_load=1e-3), omega=100.0)
    assert np.mean(rel <= 1e-6) >= 0.99, (np.mean(rel <= 1e-6), np.median(rel), rel.max())
