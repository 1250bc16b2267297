"""Gradients of rollout returns on the device (`rollout_return_grads`, `differentiable_returns`).
- primal: returns, end steps, last outputs and the persistent state are bit for bit those of `rollout_returns` on a twin handle;
- sweep: the part value_grad adds equals a float64 host reverse sweep over a twin's `rollout_jacobians` (stash and sweep alone);
- central differences of the returns over perturbed copies of base envs (one handle, references fed, so every copy sees the same walk);
- truncation at the first termination and the bootstrap value gradient;
- the autograd wrapper under a torch policy."""
import numpy as np
import pytest

from fd_helpers import _cfg, build_up_flux, clip_angle, compare_fd, stencil
from gpu_helpers import ENV_IDS, _actions, _blob, _eq, _make, _next_steps, torch_cuda  # noqa: F401
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

N = 300
FAMILIES = ("permex", "extex", "pmsm", "eesm", "scim", "dfim")


@pytest.mark.parametrize("k", (64, 7, 1))
@pytest.mark.parametrize("autoreset", ["same_step", "none"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("family", FAMILIES)
def test_primal_equals_rollout_returns(torch_cuda, family, dtype, autoreset, k):
    torch = torch_cuda
    a_env, b_env = _make(family, dtype, autoreset=autoreset), _make(family, dtype, autoreset=autoreset)
    acts = _actions(torch, a_env, k)
    ret, end, (obs, ref) = a_env.rollout_returns(acts, 0.9)
    ret2, end2, (obs2, ref2), ga, gx = b_env.rollout_return_grads(acts, 0.9)
    _eq(torch, ret2, ret, "returns")
    _eq(torch, end2, end, "end_step")
    _eq(torch, obs2, obs, "obs")
    _eq(torch, ref2, ref, "ref")
    assert a_env.sim.clock() == b_env.sim.clock()
    assert np.array_equal(_blob(a_env), _blob(b_env))
    _next_steps(torch, a_env, b_env)
    assert torch.isfinite(ga).all() and torch.isfinite(gx).all()
    kk = torch.arange(k, device="cuda")[:, None]
    assert bool((ga[kk >= end[None, :].long()] == 0).all()), "grad_a after the first termination"
    assert bool((gx[end == 0] == 0).all()), "grad_x0 of envs terminating at step 0"


SWEEP_FAMILIES = ("permex", "extex", "pmsm", "eesm", "scim", "dfim")


@pytest.mark.parametrize("family", SWEEP_FAMILIES)
def test_sweep_equals_host_sweep_over_jacobians(torch_cuda, family):
    """the part of the gradients that value_grad adds is linear in it and does not involve the reward: grad(vg) - grad(0) =
    lambda-propagation of gamma^K vg through the Jacobians alone.  A float64 host sweep over a twin's `rollout_jacobians` must give it to
    1e-12: this pins the stash and the reverse sweep separately from the reward tangent (which the central differences below check)."""
    torch = torch_cuda
    k, gamma = 12, 0.95
    a_env, b_env, c_env = (_make(family, "float64", autoreset="none") for _ in range(3))
    acts = (_actions(torch, a_env, k) * 0.2).contiguous()  # mild: most envs run the whole horizon
    n = acts.shape[1]
    _, _, _, ga0, gx0 = a_env.rollout_return_grads(acts, gamma)
    nx = gx0.shape[1]
    vg = torch.as_tensor(np.random.default_rng(2).normal(size=(n, nx)), device="cuda").contiguous()
    _, end, _, ga1, gx1 = b_env.rollout_return_grads(acts, gamma, value_grad=vg)
    (jx, ju), _ = c_env.rollout_jacobians(acts)
    jx, ju = jx.cpu().numpy(), ju.cpu().numpy()
    endn = end.cpu().numpy()
    g = 1.0
    for _ in range(k):
        g *= gamma
    lam = np.where((endn == k)[:, None], g * vg.cpu().numpy(), 0.0)
    ga_h = np.zeros(ju.shape[:3][:2] + (ju.shape[3],))
    for j in range(k - 1, -1, -1):
        ga_h[j] = np.einsum("nru,nr->nu", ju[j], lam)
        lam = np.einsum("nrc,nr->nc", jx[j], lam)
    dga, dgx = (ga1 - ga0).cpu().numpy(), (gx1 - gx0).cpu().numpy()
    assert (endn == k).sum() > 0
    scale = max(np.abs(lam).max(), np.abs(ga_h).max(), 1e-300)
    # (grad(vg) - grad(0)) cancels the reward part up to its own rounding: relative to the full gradients' size
    full = max(gx1.abs().max().item(), ga1.abs().max().item(), scale)
    assert np.abs(dga - ga_h).max() / full < 1e-12, family
    assert np.abs(dgx - lam).max() / full < 1e-12, family


FD_CASES = {
    "permex-poly-rk4": ("Cont-CC-PermExDc-v0", dict(load="poly"), None),
    "series-poly-euler3-p2": ("Cont-CC-SeriesDc-v0", dict(load="poly", solver=K.SOLVER_EULER, nsteps=3), 2.0),
    "shunt-const-rk4-3": ("Cont-CC-ShuntDc-v0", dict(load="const", nsteps=3), None),
    "extex-poly-rk4-interlock": ("Cont-CC-ExtExDc-v0", dict(load="poly", til=2e-6), 1.5),
    "pmsm-poly-euler1-p2": ("Cont-CC-PMSM-v0", dict(load="poly", solver=K.SOLVER_EULER), 2.0),
    "pmsm-const-rk4-dq": ("Cont-CC-PMSM-v0", dict(load="const", action_dq=1), None),
    "synrm-poly-rk4-3-ac1": ("Cont-CC-SynRM-v0", dict(load="poly", nsteps=3, supply="ac1"), None),
    "pmsm-ext-rk4-3": ("Cont-CC-PMSM-v0", dict(load="ext", nsteps=3), 2.0),
    "pmsm-tc-poly": ("Cont-TC-PMSM-v0", dict(load="poly"), None),
    "pmsm-sc-poly": ("Cont-SC-PMSM-v0", dict(load="poly"), 2.0),
    "eesm-poly-rk4": ("Cont-CC-EESM-v0", dict(load="poly"), None),
    "eesm-const-euler3-dq": ("Cont-CC-EESM-v0", dict(load="const", solver=K.SOLVER_EULER, nsteps=3, action_dq=1), 2.0),
    "scim-poly-rk4": ("Cont-CC-SCIM-v0", dict(load="poly"), None),
    "scim-const-rk4-dq-p2": ("Cont-CC-SCIM-v0", dict(load="const", action_dq=1), 2.0),
    "scim-tc-poly": ("Cont-TC-SCIM-v0", dict(load="poly"), None),
    "dfim-poly-rk4-3": ("Cont-CC-DFIM-v0", dict(load="poly", nsteps=3), None),
    "dfim-const-euler1-p2": ("Cont-CC-DFIM-v0", dict(load="const", solver=K.SOLVER_EULER), 2.0),
}


def _weight_every_entry(cfg, n_state, rng):
    """weights on every entry of the state vector (so the reward tangent of each is exercised), the referenced ones kept"""
    for j in range(n_state):
        if cfg.reward_weight[j] == 0.0:
            cfg.reward_weight[j] = float(rng.uniform(0.05, 0.3))


@pytest.mark.parametrize("case", list(FD_CASES))
def test_against_central_differences(torch_cuda, case):
    from gym_electric_motor_b200.vector_sim import VectorSim

    torch = torch_cuda
    env_id, kw, power = FD_CASES[case]
    m, k, gamma = 12, 3, 0.9
    rng = np.random.default_rng(5)

    def cfg(n):
        c = _cfg(env_id, n, "float64", **kw)
        r = np.random.default_rng(1)
        _weight_every_entry(c, _n_state(c), r)
        if power is not None:
            for j in range(K.MAX_STATE):
                c.reward_power[j] = power
        c.violation_reward = -3.0
        return c

    s0 = VectorSim(cfg(m))
    s0.reset()
    nx, nu, _ = s0.return_grad_dims()
    s0.rollout(torch.as_tensor(rng.uniform(-1.0, 1.0, (3, m, nu)), device="cuda").contiguous(), record_every=1)
    x0 = s0.get_ode_state().cpu().numpy()
    clip_angle(s0.cfg, x0)
    build_up_flux(rng, s0.cfg, x0)
    a0 = rng.uniform(-1.3, 1.3, (k, m, nu))
    nref = s0.n_ref
    r0 = rng.uniform(-0.5, 0.5, (k, m, nref))
    xs, acts, steps, reps = stencil(x0, a0, nu)
    sim = VectorSim(cfg(m * reps))
    sim.reset()
    sim.set_ode_state(xs)
    refs = torch.as_tensor(np.repeat(r0, reps, axis=1), device="cuda").contiguous() if nref else None
    ret, end, _, ga, gx = sim.rollout_return_grads(torch.as_tensor(acts, device="cuda").contiguous(), gamma, references=refs)
    ret, end = ret.cpu().numpy().reshape(m, reps), end.cpu().numpy().reshape(m, reps)
    grad = np.concatenate([gx.cpu().numpy()[::reps], ga.cpu().numpy()[:, ::reps].transpose(1, 0, 2).reshape(m, -1)], axis=1)
    fd = dict(target=ret[:, 0], end=end[:, 0], plus=ret[:, 1::2], minus=ret[:, 2::2], end_p=end[:, 1::2], end_m=end[:, 2::2], h=steps)
    worst, skipped, total = compare_fd(case, grad, fd, 1e-5)
    assert skipped <= total // 5, (case, skipped, total)
    assert worst < 1e-5, (case, worst)


def _n_state(c):
    from gym_electric_motor_b200 import _cabi as KK
    import ctypes as C

    lib = KK.load_library()
    d = [C.c_int32() for _ in range(4)]
    KK.check(lib.gemb200_query_dims(C.byref(c), *[C.byref(x) for x in d]), "gemb200_query_dims")
    return d[0].value


def test_truncation_and_value_grad(torch_cuda):
    """envs that terminate have grad_a == 0 from their end step on; value_grad leaves returns and every env with end_step < K unchanged,
    and adds gamma^K (J_K-1 ... J_0)^T value_grad to grad_x0 of the others, with the Jacobians of a twin's `rollout_jacobians`"""
    torch = torch_cuda
    k, gamma = 64, 0.99
    a_env, b_env, c_env = (_make("pmsm", "float64", autoreset="none") for _ in range(3))
    acts = _actions(torch, a_env, k)
    n = acts.shape[1]
    nx = 4
    vg = torch.as_tensor(np.random.default_rng(2).normal(size=(n, nx)), device="cuda").contiguous()
    ret, end, _, ga, gx = a_env.rollout_return_grads(acts, gamma)
    ret2, end2, _, ga2, gx2 = b_env.rollout_return_grads(acts, gamma, value_grad=vg)
    _eq(torch, ret2, ret, "returns unchanged by value_grad")
    alive = end == k
    assert 0 < int(alive.sum()) < n
    assert torch.equal(ga2[:, ~alive], ga[:, ~alive]) and torch.equal(gx2[~alive], gx[~alive])
    assert not torch.equal(gx2[alive], gx[alive])
    # the bootstrap part is linear in value_grad: it equals gamma^K J_total^T vg, J_total from the Jacobians of a twin
    (jx, ju), _ = c_env.rollout_jacobians(acts)
    lam = (gamma ** k) * vg[alive]
    for j in range(k - 1, -1, -1):
        lam = torch.einsum("nrc,nr->nc", jx[j][alive], lam)
    diff = gx2[alive] - gx[alive]
    assert (diff - lam).abs().max().item() <= 1e-9 * max(lam.abs().max().item(), 1.0)


def test_autograd_under_a_linear_policy(torch_cuda):
    torch = torch_cuda
    import gym_electric_motor_b200 as gem

    n, k = 256, 5
    env = gem.make("Cont-CC-PMSM-v0", num_envs=n, device="cuda", dtype="float64", seed=3)
    twin = gem.make("Cont-CC-PMSM-v0", num_envs=n, device="cuda", dtype="float64", seed=3)
    env.reset(), twin.reset()
    torch.manual_seed(0)
    policy = torch.nn.Linear(4, 3, dtype=torch.float64, device="cuda")
    feats = torch.randn(k, n, 4, dtype=torch.float64, device="cuda")
    acts = torch.tanh(policy(feats))
    J = env.differentiable_returns(acts, 0.95)
    (-J.sum()).backward()
    ret, _, _, ga, _ = twin.rollout_return_grads(acts.detach().contiguous(), 0.95)
    _eq(torch, J.detach(), ret, "returns")
    # by hand: d(-sum J)/d a = -ga; through tanh and the linear layer
    ga_pre = -ga * (1 - acts.detach() ** 2)
    w_grad = torch.einsum("knu,kni->ui", ga_pre, feats)
    b_grad = ga_pre.sum((0, 1))
    assert torch.allclose(policy.weight.grad, w_grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(policy.bias.grad, b_grad, rtol=1e-12, atol=1e-12)


_POLY = dict(a=0.01, b=0.02, c=1e-4, j_load=1e-3)
PER_ENV_CASES = {  # env id, polynomial load?, which parameter dict, slot
    "pmsm-r_s": ("Cont-CC-PMSM-v0", False, "motor", "r_s"),
    "pmsm-poly-j_load": ("Cont-CC-PMSM-v0", True, "load", "j_load"),
    "scim-poly-r_r": ("Cont-CC-SCIM-v0", True, "motor", "r_r"),
    "dfim-l_m": ("Cont-CC-DFIM-v0", False, "motor", "l_m"),
}


@pytest.mark.parametrize("rng_ids", [False, True])
@pytest.mark.parametrize("case", list(PER_ENV_CASES))
def test_per_env_parameters_give_the_single_parameter_gradients(torch_cuda, case, rng_ids):
    """env i of a handle with a per-env parameter (ENVP kernel; with rng_ids also adopted RNG identities) has the returns and gradients of
    a handle whose shared parameter is env i's, from the same state and under the same fed references"""
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200 import physical_systems as ps

    torch = torch_cuda
    env_id, poly, kind, slot = PER_ENV_CASES[case]
    m, k, gamma = 64, 6, 0.9
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
    if rng_ids:  # every env adopts its own RNG identity (a restore from itself with the source's stream)
        idx = torch.arange(m, device="cuda")
        env.restore_envs(env.snapshot_envs(idx, rng=True, params=True), idx=idx, rng="source", params="source")
    x0 = env.sim.get_ode_state()
    x0[:, 0] = 150.0  # outside the static-friction band: the speed-dependent load terms are live
    env.sim.set_ode_state(x0)
    acts = (_actions(torch, env, k, seed=4) * 0.5).contiguous()
    n_ref = env.sim.n_ref
    refs = torch.as_tensor(np.random.default_rng(6).uniform(-0.5, 0.5, (k, m, n_ref)), device="cuda").contiguous()
    ret, end, _, ga, gx = env.sim.rollout_return_grads(acts, gamma, references=refs)
    for i in (0, 21, 63):
        one = make({slot: base * scale[i]})
        one.sim.set_ode_state(x0)
        ret1, end1, _, ga1, gx1 = one.sim.rollout_return_grads(acts, gamma, references=refs)
        assert end[i].item() == end1[i].item(), (case, i)
        sc = max(gx1[i].abs().max().item(), ga1[:, i].abs().max().item())
        assert abs(ret[i].item() - ret1[i].item()) <= 1e-12 * max(abs(ret1[i].item()), 1.0), (case, i)
        assert (ga[:, i] - ga1[:, i]).abs().max().item() <= 1e-12 * sc, (case, i)
        assert (gx[i] - gx1[i]).abs().max().item() <= 1e-12 * sc, (case, i)
    assert not torch.allclose(gx[0], gx[63], rtol=1e-9, atol=0)  # the slot moves the gradients


@pytest.mark.parametrize("family", FAMILIES)
def test_float32_against_float64(torch_cuda, family):
    """the fp32 build of the same configuration, state and actions: its gradients carry fp32 rounding through K tangent integrations and
    the sweep.  The rewards are smooth here (exponent 2, actions inside the clip range), so no branch differs between the dtypes, and the
    error grows like K times the single-step one: 8 steps of relative rounding ~1e-7 amplified by the condition of the step maps (the
    current dynamics' eigenvalues times tau are O(1)) stay well below 1e-3 of the gradient's scale."""
    from gym_electric_motor_b200.vector_sim import VectorSim

    torch = torch_cuda
    env_id = ENV_IDS[family]
    n, k, gamma = 256, 8, 0.95

    def cfg(dtype):
        c = _cfg(env_id, n, dtype, load="poly")
        for j in range(K.MAX_STATE):
            c.reward_power[j] = 2.0
        return c

    s64, s32 = VectorSim(cfg("float64")), VectorSim(cfg("float32"))
    s64.reset(), s32.reset()
    nx, nu, _ = s64.return_grad_dims()
    x0 = s64.get_ode_state()
    if family in ("permex", "extex"):  # from standstill: no back-EMF drives the currents past their limits
        x0[:, 0] = 0.0
        s64.set_ode_state(x0)
    s32.set_ode_state(x0)
    rng = np.random.default_rng(8)
    amp = 0.1 if family in ("permex", "extex") else 0.6  # the DC machines' currents pass their limits within K steps at larger duty
    a = rng.uniform(-amp, amp, (k, n, nu))
    refs = rng.uniform(-0.5, 0.5, (k, n, s64.n_ref))
    out = {}
    for s, dt in ((s64, torch.float64), (s32, torch.float32)):
        r = torch.as_tensor(refs, dtype=dt, device="cuda").contiguous() if s.n_ref else None
        out[dt] = s.rollout_return_grads(torch.as_tensor(a, dtype=dt, device="cuda").contiguous(), gamma, references=r)
    _, end64, _, ga64, gx64 = out[torch.float64]
    _, end32, _, ga32, gx32 = out[torch.float32]
    same = (end64 == end32) & (end64 >= 1)  # the same steps differentiated in both dtypes, at least one
    assert int(same.sum()) >= n // 4
    g64 = torch.cat([gx64, ga64.transpose(0, 1).reshape(n, -1)], 1)[same]
    g32 = torch.cat([gx32, ga32.transpose(0, 1).reshape(n, -1)], 1)[same].double()
    rel = ((g32 - g64).abs().amax(1) / g64.abs().amax(1).clamp_min(1e-30))
    print(f"{family}: fp32 vs fp64 worst {rel.max().item():.2e}, median {rel.median().item():.2e}")
    assert rel.max().item() < 1e-3, family
