"""Return gradients on the device (`rollout_return_grads`, `differentiable_returns`) against central differences of the float64 oracle.

Every perturbed copy of a case is its own oracle instance with the device's configuration, seed and env_index_offset: all copies sit at the
same global env indices, so they draw exactly the device's reference walk and state noise (Philox streams keyed by env index and step).
That lets the device run without a reference feed, under its own generators, state wrappers and noise, and still be differentiated by
central differences.  Per case:
  * device and oracle reset and run the same warm-up steps; then both get the same x0 (`set_ode_state`) and the device's references
    (`set_reference`);
  * the device's returns and end steps must be the oracle's (the primal check);
  * d return / d (x0, a_0 .. a_K-1) must match central differences of the oracle's float64 returns, relative to each env's gradient scale;
  * a non-vacuity check: the weighted entry / wrapper a case is about must move the gradient (u_sup, a function of time only, must not).
A CPU test (test_return_grads_oracle_harness.py) checks the harness itself against a closed form."""
import numpy as np
import pytest

from fd_helpers import build_up_flux, clip_angle, compare_fd, oracle_fd
from gpu_helpers import torch_cuda  # noqa: F401
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

OFFSET = 7000  # global index of env 0: device and every oracle copy draw the streams of envs OFFSET ..
TOL64 = 1e-5
# fp32 device gradients against the float64 oracle, on smooth rewards (exponent 2, actions inside the clip range, K = 8): the tangent
# integrations and the sweep carry fp32 rounding (~6e-8 relative per operation) through 8 steps whose maps are well conditioned (the current
# dynamics' eigenvalues times tau are O(1)), and x0 itself is rounded to fp32.  Measured on an H100 over the 0 .. 4 reference-slot cases
# (PMSM, TC-PMSM, EESM): worst 2.6e-7 .. 6.4e-7 of the gradient scale.  1e-5 leaves a factor ~15 for other seeds and states; a wrong
# coefficient or a wrong sweep term is >= 1e-3 (MOVES).
TOL32 = 1e-5
MOVES = 1e-3  # a weighted entry / wrapper must move the gradient by this much of its scale
_KEEP = []


# ------------------------------------------------------------------------------------------------------------------ the oracle side
def ode_has_angle(cfg):
    return cfg.motor_kind >= K.MOTOR_PMSM


def flat_grad(ga, gx):
    """[m, n_x + K n_u]: grad_x0, then grad_a step by step"""
    k_steps, m, nu = ga.shape
    return np.concatenate([gx, ga.transpose(1, 0, 2).reshape(m, k_steps * nu)], axis=1)


# ------------------------------------------------------------------------------------------------------------------ the cases
def _psw():
    from gym_electric_motor_b200 import physical_system_wrappers as psw

    return psw


def _make_cfg(env_id, m, autoreset="none", seed=13, **kw):
    import gym_electric_motor_b200 as gem

    env = gem.make(env_id, num_envs=m, dtype="float64", autoreset=autoreset, seed=seed, env_index_offset=OFFSET, **kw)
    _KEEP.append(env)
    cfg = env.build_config()
    cfg.dtype = K.F64
    return cfg, list(env.state_names)


def _poly(cfg):
    cfg.load_kind = K.LOAD_POLY_STATIC
    cfg.load_param[K.LP_A], cfg.load_param[K.LP_B], cfg.load_param[K.LP_C] = 0.01, 0.02, 1e-4
    cfg.load_param[K.LP_J_LOAD] = 1e-3


def _power(cfg, p):
    for j in range(K.MAX_STATE):
        cfg.reward_power[j] = p


def _ac1(cfg):
    cfg.supply_kind, cfg.supply_param[0], cfg.supply_param[1], cfg.supply_param[2] = K.SUPPLY_AC1, 50.0, 0.3, 1.0


def _copy_slot(cfg, src, dst, state):
    for f in ("ref_kind", "ref_value", "ref_margin_lo", "ref_margin_hi", "ref_init_lo", "ref_init_hi", "ref_sigma_lo", "ref_sigma_hi", "ref_len_lo",
              "ref_len_hi", "ref_amp_lo", "ref_amp_hi", "ref_freq_lo", "ref_freq_hi", "ref_off_lo", "ref_off_hi"):
        getattr(cfg, f)[dst] = getattr(cfg, f)[src]
    cfg.ref_state[dst] = state


class Case:
    """env id / config builder and the set-up of one comparison.  build(m) -> (cfg, state names); zero: row entries whose weight, set to
    0, must move the gradient (same_zero: must leave it unchanged); noise_moves: setting the noise scale to 0 must move the gradient;
    omega0: the initial speed (the induction motors' long horizons start at standstill: no back-EMF drives the currents past their
    limits); i0: initial dq currents drawn in +-i0 of their limits (the same-step case: some envs trip inside the horizon)."""

    def __init__(self, build, k=3, gamma=0.9, m=12, amp=1.2, warm=3, zero=(), same_zero=(), noise_moves=False, term=None, vg=False, envp=False,
                 omega0=None, i0=None):
        self.build, self.k, self.gamma, self.m, self.amp, self.warm, self.omega0, self.i0 = build, k, gamma, m, amp, warm, omega0, i0
        self.zero, self.same_zero, self.noise_moves, self.term, self.vg, self.envp = zero, same_zero, noise_moves, term, vg, envp


def _default(env_id, power=None, poly=False):
    def build(m):
        cfg, names = _make_cfg(env_id, m)
        if power is not None:
            _power(cfg, power)
        if poly:
            _poly(cfg)
        return cfg, names
    return build


def _switched(m):
    from helpers import switched_config

    kinds = [dict(kind=K.REF_CONST, value=0.25), dict(kind=K.REF_WIENER, margin=(-0.5, 0.5)), dict(kind=K.REF_SINUS)]
    cfg = switched_config(m, kinds, [0.3, 0.4, 0.3], (2, 4), seed=21)  # super-episodes of 2 .. 4 steps: switches inside the horizon
    cfg.env_index_offset = OFFSET
    cfg.autoreset = K.AUTORESET_NONE
    _power(cfg, 2.0)  # the coefficient follows row - ref itself (exponent 1: only its sign), so it sees which reference the step compares with
    return cfg, None


def _laplace_sawtooth(m):
    cfg, names = _make_cfg("Cont-CC-PMSM-v0", m)
    for r, kind in enumerate((K.REF_LAPLACE, K.REF_SAWTOOTH)):
        cfg.ref_kind[r] = kind
        cfg.ref_margin_lo[r], cfg.ref_margin_hi[r] = -0.6, 0.6
        cfg.ref_init_lo[r], cfg.ref_init_hi[r] = -0.6, 0.6
        cfg.ref_amp_lo[r], cfg.ref_amp_hi[r] = 0.05, 0.6
        cfg.ref_freq_lo[r], cfg.ref_freq_hi[r] = 200.0, 900.0
        cfg.ref_off_lo[r], cfg.ref_off_hi[r] = -0.6, 0.6
        cfg.ref_len_lo[r], cfg.ref_len_hi[r] = 2, 5
    _power(cfg, 2.0)
    return cfg, names


def _pmsm_noise_cossin_ac1(m):
    psw = _psw()
    cfg, names = _make_cfg("Cont-CC-PMSM-v0", m, physical_system_wrappers=[
        psw.StateNoiseProcessor(["i_sd", "i_sq", "u_sup"], "normal", dict(loc=0.0, scale=0.02)), psw.CosSinProcessor("epsilon", remove_angle=True)])
    _ac1(cfg)
    _power(cfg, 2.0)
    cfg.reward_weight[names.index("u_sup")] = 0.3  # row entry 12 = state entry 13 (the angle is removed): a function of time only
    return cfg, names


def _scim_observer_noise(m):
    psw = _psw()
    cfg, names = _make_cfg("Cont-CC-SCIM-v0", m, physical_system_wrappers=[
        psw.FluxObserver(), psw.StateNoiseProcessor(["i_sd", "i_sq", "torque"], "normal", dict(loc=0.0, scale=0.02))])
    _power(cfg, 2.0)
    cfg.reward_weight[names.index("torque")] = 0.2
    assert K.SOP_FLUX_OBSERVER in list(cfg.sop_kind[:cfg.n_state_ops])
    return cfg, names


def _shunt_isum(m):
    """the shunt motor's own i_sum entry (its system carries the current sum; no state op)"""
    cfg, names = _make_cfg("Cont-CC-ShuntDc-v0", m, physical_system_wrappers=[_psw().CurrentSumProcessor(("i_a", "i_e"))])
    _power(cfg, 2.0)
    cfg.reward_weight[names.index("i_sum")] = 0.3
    return cfg, names


def _extex_current_sum_op(m):
    cfg, names = _make_cfg("Cont-CC-ExtExDc-v0", m, physical_system_wrappers=[_psw().CurrentSumProcessor(("i_a", "i_e"))])
    assert K.SOP_CURRENT_SUM in list(cfg.sop_kind[:cfg.n_state_ops]) and names[-1] == "i_sum"  # appended by the state op, unweighted
    _poly(cfg)
    _power(cfg, 2.0)
    cfg.reward_weight[names.index("i_e")] = 0.3
    return cfg, names


def _pmsm_cossin_eps(m):
    cfg, names = _make_cfg("Cont-CC-PMSM-v0", m, physical_system_wrappers=[_psw().CosSinProcessor("epsilon")])
    _power(cfg, 2.0)
    cfg.reward_weight[names.index("epsilon")] = 0.2
    return cfg, names


def _pmsm_shapes(m):
    cfg, names = _make_cfg("Cont-CC-PMSM-v0", m)
    _poly(cfg)
    for nm, w, p in (("i_sd", 0.5, 1.5), ("i_sq", 0.5, 3.0), ("omega", 0.1, 2.0), ("torque", 0.15, 0.5), ("u_sd", 0.1, 1.0), ("i_a", 0.1, 2.0)):
        cfg.reward_weight[names.index(nm)], cfg.reward_power[names.index(nm)] = w, p
    cfg.reward_bias, cfg.violation_reward = 1.5, -4.0
    return cfg, names


def _same_step(m):
    cfg, names = _make_cfg("Cont-CC-PMSM-v0", m, autoreset="same_step")
    _power(cfg, 2.0)
    return cfg, names


def _nref(n_ref, env_id="Cont-CC-PMSM-v0"):
    """exponent 2 everywhere (smooth: the fp32 cases); 0 slots: weights on unreferenced entries only; 4: PMSM with i_sd, i_sq, u_sd, u_sq
    referenced, slots 2 and 3 copies of the Wiener slot 0"""
    def build(m):
        cfg, names = _make_cfg(env_id, m)
        _power(cfg, 2.0)
        if n_ref == 0:
            cfg.n_ref = 0
            cfg.reward_weight[names.index("i_sd")], cfg.reward_weight[names.index("i_sq")] = 0.4, 0.6
            cfg.reward_weight[names.index("u_sq")] = 0.2
        elif n_ref == 4:
            cfg.n_ref = 4
            for dst, nm in ((2, "u_sd"), (3, "u_sq")):
                _copy_slot(cfg, 0, dst, names.index(nm))
                cfg.reward_weight[names.index(nm)] = 0.2
            for nm, w in (("i_sd", 0.2), ("i_sq", 0.4)):
                cfg.reward_weight[names.index(nm)] = w
            # a distinct exponent per slot: the coefficient of slot r must use slot r's exponent
            cfg.reward_power[names.index("u_sq")] = 3.0
        assert cfg.n_ref == n_ref
        return cfg, names
    return build


OWN = {  # own generators (no feed), fp64, autoreset none
    "pmsm-cc-wiener": Case(_default("Cont-CC-PMSM-v0")),
    "permex-sc-wiener": Case(_default("Cont-SC-PermExDc-v0"), amp=0.3),
    "pmsm-tc-wiener": Case(_default("Cont-TC-PMSM-v0")),
    "eesm-cc-wiener-3slots": Case(_default("Cont-CC-EESM-v0"), amp=0.8),
    "scim-cc-wiener": Case(_default("Cont-CC-SCIM-v0"), k=8, gamma=0.0, amp=0.6, omega0=0.0),
    "dfim-cc-wiener": Case(_default("Cont-CC-DFIM-v0")),
    "permex-switched-const-wiener-sinus": Case(_switched, k=8),
    "pmsm-laplace-sawtooth": Case(_laplace_sawtooth, k=8),
}
WRAPPERS = {
    "pmsm-noise-cossin-remove-angle-ac1": Case(_pmsm_noise_cossin_ac1, same_zero=("u_sup",), noise_moves=True),
    "scim-observer-noise": Case(_scim_observer_noise, zero=("torque",), noise_moves=True),
    "shunt-i_sum": Case(_shunt_isum, amp=0.3, zero=("i_sum",)),
    "extex-current-sum-op": Case(_extex_current_sum_op, amp=0.3, zero=("i_e",)),
    "pmsm-cossin-weighted-eps": Case(_pmsm_cossin_eps, zero=("epsilon",)),
}
SHAPES = {
    "pmsm-mixed-exponents-bias-violation-unreferenced": Case(_pmsm_shapes, k=8, gamma=1.0, zero=("omega", "torque", "u_sd", "i_a")),
}
HORIZONS = {
    "pmsm-k1": Case(_default("Cont-CC-PMSM-v0", poly=True), k=1, gamma=1.0),
    "pmsm-k32": Case(_default("Cont-CC-PMSM-v0", power=2.0, poly=True), k=32, gamma=0.99, m=8, amp=0.5),
    "scim-k1": Case(_default("Cont-CC-SCIM-v0", poly=True), k=1),
    "scim-k32": Case(_default("Cont-CC-SCIM-v0", power=2.0), k=32, gamma=0.99, m=8, amp=0.3, omega0=0.0),
}
SAME_STEP = {  # saturating actions: some envs trip their current limits inside the horizon, the others run through
    "pmsm-same-step-terminations": Case(_same_step, k=16, m=20, amp=None, term=(0.3, 0.7), i0=0.98),
}
VALUE_GRAD = {
    "pmsm-value-grad": Case(_default("Cont-CC-PMSM-v0", power=2.0, poly=True), k=8, amp=0.8, vg=True),
    "scim-value-grad": Case(_default("Cont-CC-SCIM-v0", power=2.0, poly=True), k=8, amp=0.5, vg=True, omega0=0.0),
}
ENVP = {
    "pmsm-poly-per-env-r_s-j_load": Case(_default("Cont-CC-PMSM-v0", power=2.0, poly=True), k=6, m=8, amp=0.8, envp=True),
}
NREF = {  # K = 8, exponent 2, actions inside the clip range: smooth, so the fp32 build runs them too
    0: Case(_nref(0), k=8, amp=0.8, zero=("u_sq",)),
    1: Case(_nref(1, "Cont-TC-PMSM-v0"), k=8, amp=0.8),
    2: Case(_nref(2), k=8, amp=0.8),
    3: Case(_nref(3, "Cont-CC-EESM-v0"), k=8, amp=0.6),
    4: Case(_nref(4), k=8, amp=0.8, zero=("u_sq",)),
}


# ------------------------------------------------------------------------------------------------------------------ the harness
def _saturating(rng, k, m, nu):
    """per-env magnitude, sign constant over stretches of 4 steps: currents trip their limits after an env-dependent number of steps"""
    mag = rng.uniform(0.2, 1.0, (1, m, 1))
    return np.repeat(rng.choice([-1.0, 1.0], size=((k + 3) // 4, m, nu)), 4, axis=0)[:k] * mag


class Setup:
    """one case prepared on the device: warm-up actions, x0, references, actions, the config (fp64) and its per-env parameters"""

    def __init__(self, case, seed=5):
        from gym_electric_motor_b200.vector_sim import VectorSim

        self.case = case
        self.cfg, self.names = case.build(case.m)
        m = case.m
        rng = np.random.default_rng(seed)
        sim = VectorSim(self.cfg)
        nx, nu, _ = sim.return_grad_dims()
        self.nx, self.nu = nx, nu
        self.mp = self.lp = None
        if case.envp:
            self.mp = np.tile(np.array(list(self.cfg.motor_param)), (m, 1))
            self.lp = np.tile(np.array(list(self.cfg.load_param)), (m, 1))
            self.mp[:, K.MP_R_S] *= np.linspace(0.7, 1.3, m)
            self.lp[:, K.LP_J_LOAD] *= np.linspace(1.4, 0.6, m)
        self.warm = rng.uniform(-0.3, 0.3, (case.warm, m, nu))
        self._prepare(sim)
        x0 = sim.get_ode_state().cpu().numpy()
        clip_angle(self.cfg, x0)
        build_up_flux(rng, self.cfg, x0)  # the field frame is defined (DESIGN.md finding 3)
        if case.envp:
            x0[:, 0] = 150.0  # outside the static-friction band: the speed-dependent load terms are live
        if case.omega0 is not None:
            x0[:, 0] = case.omega0
        if case.i0 is not None:
            for j, nm in ((1, "i_sd"), (2, "i_sq")):
                x0[:, j] = rng.uniform(-case.i0, case.i0, m) * self.cfg.limits[self.names.index(nm)]
        self.x0 = x0
        self.ref0 = sim.get_reference().cpu().numpy()
        self.acts = _saturating(rng, case.k, m, nu) if case.amp is None else rng.uniform(-case.amp, case.amp, (case.k, m, nu))
        self.vg = rng.normal(size=(m, nx)) / np.maximum(1.0, np.abs(x0).max(0)) if case.vg else None

    def _prepare(self, sim):
        if self.mp is not None:
            sim.set_env_params(self.mp, self.lp)
        sim.reset()
        for a in self.warm:
            sim.step(a)

    def device(self, torch, dtype=K.F64, edit=None):
        """returns, end steps and [m, n_col] gradients of the device, from x0 and the references, without a feed; edit(cfg) changes the
        configuration (a weight, the noise) of this run only"""
        from gym_electric_motor_b200.vector_sim import VectorSim

        cfg = type(self.cfg).from_buffer_copy(self.cfg)
        cfg.dtype = dtype
        if edit is not None:
            edit(cfg)
        sim = VectorSim(cfg)
        self._prepare(sim)
        sim.set_ode_state(self.x0)
        sim.set_reference(self.ref0)
        dt = torch.float64 if dtype == K.F64 else torch.float32
        vg = None if self.vg is None else torch.as_tensor(self.vg, dtype=dt, device="cuda").contiguous()
        ret, end, _, ga, gx = sim.rollout_return_grads(torch.as_tensor(self.acts, dtype=dt, device="cuda").contiguous(), self.case.gamma, value_grad=vg)
        ga = ga.double().cpu().numpy()
        return ret.double().cpu().numpy(), end.cpu().numpy(), ga, flat_grad(ga, gx.double().cpu().numpy())

    def oracles(self, oracle_lib):
        cfg = type(self.cfg).from_buffer_copy(self.cfg)
        cfg.dtype = K.F64
        if self.mp is None:
            return lambda: [(oracle_lib.Oracle(cfg), slice(None))]

        def per_env():  # N = 1 oracles at the env's global index with the env's parameters (DESIGN.md §7: per-env blocks)
            out = []
            for i in range(self.case.m):
                c = type(cfg).from_buffer_copy(cfg)
                c.n_envs, c.env_index_offset = 1, OFFSET + i
                for j in range(K.MAX_MOTOR_PARAM):
                    c.motor_param[j] = self.mp[i, j]
                for j in range(8):
                    c.load_param[j] = self.lp[i, j]
                out.append((oracle_lib.Oracle(c), slice(i, i + 1)))
            return out
        return per_env

    def fd(self, oracle_lib):
        return oracle_fd(self.oracles(oracle_lib), self.warm, self.x0, self.acts, self.case.gamma, ref0=self.ref0, value_grad=self.vg,
                         angle=ode_has_angle(self.cfg))


def check_case(torch, oracle_lib, name, case, dtype=K.F64):
    st = Setup(case)
    k, m = case.k, case.m
    ret, end, ga, grad = st.device(torch, dtype)
    fd = st.fd(oracle_lib)
    # the primal: the device's returns and end steps are the oracle's
    assert np.array_equal(end, fd["end"]), (name, end, fd["end"])
    primal_tol = (1e-9 if dtype == K.F64 else 1e-4) * k
    assert np.all(np.abs(ret - fd["ret"]) <= primal_tol * np.maximum(1.0, np.abs(fd["ret"]))), (name, np.abs(ret - fd["ret"]).max())
    kk = np.arange(k)[:, None]
    assert np.all(ga[kk >= end[None, :]] == 0.0), "grad_a after the first termination"
    worst, excluded, total = compare_fd(f"{name} [{'f64' if dtype == K.F64 else 'f32'}]", grad, fd, TOL64 if dtype == K.F64 else TOL32)
    assert excluded <= total // 5, (name, excluded, total)
    assert worst < (TOL64 if dtype == K.F64 else TOL32), (name, worst)
    alive = int((end == k).sum())
    if case.term is None:
        assert alive >= m / 2, (name, alive, m)
    else:  # same-step resets: a share of the envs terminates inside the horizon; their gradients up to the end step were compared too
        lo, hi = case.term
        assert lo * m <= m - alive <= hi * m, (name, alive, m)
        assert np.any((end > 0) & (end < k))
    scale = np.maximum(np.abs(grad).max(1, keepdims=True), 1e-300)  # envs ending at step 0 have zero gradients
    for nm in case.zero:
        j = st.names.index(nm)
        _, _, _, g0 = st.device(torch, dtype, edit=lambda c, j=j: c.reward_weight.__setitem__(j, 0.0))
        moved = (np.abs(grad - g0) / scale).max()
        assert moved >= MOVES, (name, nm, moved)
    for nm in case.same_zero:
        j = st.names.index(nm)
        _, _, _, g0 = st.device(torch, dtype, edit=lambda c, j=j: c.reward_weight.__setitem__(j, 0.0))
        assert (np.abs(grad - g0) / scale).max() <= 1e-12, (name, nm)
    if case.noise_moves:
        def quiet(c):
            for s in range(c.n_state_ops):
                if c.sop_kind[s] == K.SOP_NOISE:
                    c.sop_param[s][1] = 0.0
        _, _, _, g0 = st.device(torch, dtype, edit=quiet)
        moved = (np.abs(grad - g0) / scale).max()
        assert moved >= MOVES, (name, "noise", moved)
    return st, grad, fd


ALL = dict(**OWN, **WRAPPERS, **SHAPES, **HORIZONS, **SAME_STEP, **VALUE_GRAD, **ENVP)


@pytest.mark.parametrize("case", list(ALL))
def test_return_grads_against_oracle_central_differences(torch_cuda, oracle_lib, case):
    check_case(torch_cuda, oracle_lib, case, ALL[case])


@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("n_ref", list(NREF))
def test_every_reference_count_against_oracle(torch_cuda, oracle_lib, n_ref, dtype):
    """the 0 .. 4 reference-slot instantiations of the return-gradient kernel, fp64 and fp32, against the fp64 oracle"""
    check_case(torch_cuda, oracle_lib, f"nref{n_ref}", NREF[n_ref], dtype)


def test_value_grad_case_is_not_vacuous(torch_cuda, oracle_lib):
    """the value_grad case is not vacuous: without value_grad the same set-up gives other gradients for the envs that run the horizon"""
    torch = torch_cuda
    st = Setup(VALUE_GRAD["pmsm-value-grad"])
    _, end, _, grad = st.device(torch)
    st.vg = None
    _, _, _, g0 = st.device(torch)
    full = end == st.case.k
    assert full.sum() >= st.case.m / 2
    scale = np.maximum(np.abs(grad).max(1), 1e-300)
    assert ((np.abs(grad - g0).max(1) / scale)[full] >= MOVES).all()


# ------------------------------------------------------------------------------------------------------------------ autograd
def test_differentiable_returns_under_gradcheck(torch_cuda):
    """`differentiable_returns` as a function of the action sequence: every evaluation first restores the envs from one snapshot with the
    source's random stream, so the function is deterministic, and torch.autograd.gradcheck compares the full N x (K N n_u) Jacobian
    (every grad_output, the zero cross-env blocks) with its own finite differences"""
    import gym_electric_motor_b200 as gem

    torch = torch_cuda
    n, k = 6, 3
    env = gem.make("Cont-CC-PMSM-v0", num_envs=n, device="cuda", dtype="float64", autoreset="none", seed=9)
    env.reset()
    env.step(torch.as_tensor(np.random.default_rng(1).uniform(-0.3, 0.3, (n, 3)), device="cuda"))
    idx = torch.arange(n, device="cuda")
    snap = env.snapshot_envs(idx, rng=True, params=True)

    def returns(a):
        env.restore_envs(snap, idx=idx, rng="source", params="source")
        return env.differentiable_returns(a, 0.9)

    a = torch.as_tensor(np.random.default_rng(2).uniform(-0.8, 0.8, (k, n, 3)), device="cuda").requires_grad_(True)
    r1, r2 = returns(a).detach(), returns(a).detach()
    assert torch.equal(r1, r2)
    assert torch.autograd.gradcheck(returns, (a,), eps=1e-6, atol=1e-7, rtol=1e-4)
