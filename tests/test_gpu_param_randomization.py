"""Per-episode domain randomisation on the device (gemb200_set_param_randomization): parameter draws at every reset, the device
derivation against the host one, auto-resets inside fused rollouts and graphs, determinism, off switches and refusals."""
import ctypes as C

import numpy as np
import pytest

from gym_electric_motor_b200 import _cabi as K
from gpu_helpers import torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

DTYPES = pytest.mark.parametrize("dtype", ["float32", "float64"])
FAMILY_ENVS = ["Cont-CC-PMSM-v0", "Cont-CC-SynRM-v0", "Cont-CC-EESM-v0", "Cont-CC-SCIM-v0", "Cont-CC-DFIM-v0", "Cont-CC-PermExDc-v0",
               "Cont-CC-SeriesDc-v0", "Cont-CC-ShuntDc-v0", "Cont-CC-ExtExDc-v0", "Finite-CC-PMSM-v0"]


def _make(env_id, n, dtype, seed=7, offset=0, **kw):
    import gym_electric_motor_b200 as gem

    return gem.make(env_id, num_envs=n, autoreset="same_step", seed=seed, dtype=dtype, env_index_offset=offset, **kw)


def _spec(env):
    """every non-zero motor parameter of the env except the pole pairs, +-20 %, alternately uniform and log-uniform; plus j_load"""
    cfg = env.build_config()
    spec, used = {}, set()
    for name, slot in env._MP_SLOT.items():
        v = cfg.motor_param[slot]
        if slot == K.MP_P or slot in used or v == 0:
            continue
        used.add(slot)
        lo, hi = sorted((0.8 * v, 1.25 * v))
        spec[name] = ("log_uniform", lo, hi) if (len(spec) % 2 and lo > 0) else (lo, hi)
    return spec, {"j_load": (0.0, 1e-3)}


def _actions(env, k, rng, scale=1.0):
    sp = env.action_space
    if hasattr(sp, "low"):
        return rng.uniform(-scale, scale, size=(k, env.num_envs, len(sp.low)))
    nvec = list(sp.nvec) if hasattr(sp, "nvec") else [sp.n]  # MultiDiscrete or Discrete
    return np.stack([np.stack([rng.integers(0, int(m), size=env.num_envs) for m in nvec], axis=1) for _ in range(k)]).astype(np.int32)


def _host_rows(env, theta):
    """motor / load parameter rows of the env's configuration with the drawn values theta {name: tensor[N]} put in"""
    cfg, n = env.build_config(), env.num_envs
    mp = np.tile(np.array(list(cfg.motor_param)), (n, 1))
    lp = np.tile(np.array(list(cfg.load_param)), (n, 1))
    for name, vals in theta.items():
        v = vals.double().cpu().numpy()
        if name in env._MP_SLOT:
            mp[:, env._MP_SLOT[name]] = v
        else:
            lp[:, env._LP_SLOT[name]] = v
    return mp, lp


@DTYPES
def test_draws_lie_in_bounds_follow_their_distribution_and_leave_other_slots(torch_cuda, dtype):
    torch = torch_cuda
    from scipy import stats

    n = 1 << 16
    env = _make("Cont-CC-PMSM-v0", n, dtype)
    cfg = env.build_config()
    env.randomize_env_parameters(motor_parameter={"r_s": (0.01, 0.03), "l_d": ("log_uniform", 1e-4, 1e-3)})
    th0 = env.env_parameters()
    assert torch.equal(th0["r_s"], torch.full((n,), cfg.motor_param[K.MP_R_S], dtype=th0["r_s"].dtype, device="cuda"))  # no draw yet
    env.reset()
    th = env.env_parameters()
    rd = np.float32 if dtype == "float32" else np.float64
    rs, ld = th["r_s"].double().cpu().numpy(), th["l_d"].double().cpu().numpy()
    assert rs.min() >= rd(0.01) and rs.max() <= rd(0.03) and ld.min() >= rd(1e-4) and ld.max() <= rd(1e-3)
    assert stats.kstest(rs, "uniform", args=(0.01, 0.02)).pvalue > 1e-3
    assert stats.kstest(np.log(ld), "uniform", args=(np.log(1e-4), np.log(1e-3) - np.log(1e-4))).pvalue > 1e-3
    # a slot that has not been drawn yet holds the configuration's value in every env; the drawn slots keep their values without a reset
    env.randomize_env_parameters(motor_parameter={"r_s": (0.01, 0.03), "l_q": (1e-4, 1e-3)})
    th2 = env.env_parameters()
    assert torch.equal(th2["r_s"], th["r_s"])
    assert torch.equal(th2["l_q"], torch.full((n,), cfg.motor_param[K.MP_L_Q], dtype=th2["l_q"].dtype, device="cuda"))


@DTYPES
@pytest.mark.parametrize("env_id", FAMILY_ENVS)
def test_device_derivation_equals_host_derivation(torch_cuda, env_id, dtype):
    """Handle A draws at its reset; handle B gets A's stored values through the host path (gemb200_set_env_params).  Same seed, same
    actions: every output equals bit for bit until the env's first termination.  At that step reward, terminated flag and reference still
    agree; A's observation there is its new episode's reset observation on freshly drawn parameters, B's on the old ones."""
    torch = torch_cuda
    n, steps = 2048, 24
    a_env, b_env = _make(env_id, n, dtype), _make(env_id, n, dtype)
    mspec, lspec = _spec(a_env)
    a_env.randomize_env_parameters(mspec, lspec)
    (sa, ra), _ = a_env.reset()
    theta = {k: v.clone() for k, v in a_env.env_parameters().items()}
    mp, lp = _host_rows(b_env, theta)
    b_env.sim.set_env_params(mp, lp)
    (sb, rb), _ = b_env.reset()
    assert torch.equal(sa, sb) and torch.equal(ra, rb)
    acts = torch.as_tensor(_actions(a_env, steps, np.random.default_rng(3)), device="cuda")
    alive = torch.ones(n, dtype=torch.bool, device="cuda")
    for k in range(steps):
        (sa, ra), wa, ta, _, _ = a_env.step(acts[k])
        (sb, rb), wb, tb, _, _ = b_env.step(acts[k])
        assert torch.equal(wa[alive], wb[alive]) and torch.equal(ta[alive], tb[alive]) and torch.equal(ra[alive], rb[alive]), k
        before = alive & ~ta
        assert torch.equal(sa[before], sb[before]), k
        alive = before


@DTYPES
@pytest.mark.parametrize("env_id", ["Cont-CC-SCIM-v0", "Cont-CC-PMSM-v0", "Finite-CC-PMSM-v0"])
def test_rollout_under_randomisation_equals_single_steps(torch_cuda, env_id, dtype):
    torch = torch_cuda
    n, steps = 4096, 32
    envs = [_make(env_id, n, dtype) for _ in range(2)]
    for e in envs:
        e.randomize_env_parameters(*_spec(e))
        e.reset()
    th0 = {k: v.clone() for k, v in envs[0].env_parameters().items()}
    acts = torch.as_tensor(_actions(envs[0], steps, np.random.default_rng(5)), device="cuda")
    (so, ro), wo, to = envs[0].rollout(acts, record_every=1)
    ever = torch.zeros(n, dtype=torch.bool, device="cuda")
    for k in range(steps):
        (s, r), w, t, _, _ = envs[1].step(acts[k])
        assert torch.equal(so[k], s) and torch.equal(ro[k], r) and torch.equal(wo[k], w) and torch.equal(to[k], t), k
        ever |= t
    th_r, th_s = envs[0].env_parameters(), envs[1].env_parameters()
    if "SCIM" in env_id:
        assert ever.any()
    for name in th0:
        assert torch.equal(th_r[name], th_s[name])
        assert torch.equal(th_r[name][~ever], th0[name][~ever])  # never reset: old values, bit for bit
        assert bool((th_r[name][ever] != th0[name][ever]).all())  # reset at least once: a new draw in every slot


@DTYPES
@pytest.mark.parametrize("env_id", ["Cont-CC-PMSM-v0", "Cont-CC-EESM-v0", "Cont-CC-PermExDc-v0"])
def test_physics_after_an_in_kernel_reset_matches_single_env_oracles(torch_cuda, oracle_lib, env_id, dtype):
    torch = torch_cuda
    n, m, tol = 4096, 64, (1e-5 if dtype == "float32" else 1e-9)
    env = _make(env_id, n, dtype)
    env.randomize_env_parameters(*_spec(env))
    env.reset()
    sp = env.action_space
    push = -torch.ones((16, n, len(sp.low)), dtype=env.sim.dtype, device="cuda")  # drives the currents into their limits: auto-resets
    push[..., 0] = 1.0  # (equal phase voltages of a B6 bridge would cancel)
    _, _, term = env.rollout(push, record_every=1)
    reset_envs = torch.nonzero(term.any(0)).flatten()[:m].cpu().numpy()
    assert len(reset_envs) == m
    y = env.sim.get_ode_state().cpu().numpy()
    theta = env.env_parameters()
    mp, lp = _host_rows(env, theta)
    oras = []
    for i in reset_envs:
        cfg = env.build_config()
        cfg.n_envs, cfg.dtype, cfg.env_index_offset = 1, K.F64, int(i)
        for j in range(K.MAX_MOTOR_PARAM):
            cfg.motor_param[j] = mp[i, j]
        for j in range(8):
            cfg.load_param[j] = lp[i, j]
        ora = oracle_lib.Oracle(cfg)
        ora.reset()
        ora.set_ode_state(y[i:i + 1])
        oras.append(ora)
    acts = _actions(env, 20, np.random.default_rng(9), scale=0.1)
    live = np.ones(m, dtype=bool)
    for k in range(20):
        (s, _), _, t, _, _ = env.step(torch.as_tensor(acts[k], device="cuda"))
        s, t = s.double().cpu().numpy()[reset_envs], t.cpu().numpy()[reset_envs]
        for q, (i, ora) in enumerate(zip(reset_envs, oras)):
            o_s, _, _, o_t = ora.step(acts[k][i:i + 1])
            live[q] &= not t[q]
            if live[q]:
                assert np.abs(s[q] - o_s[0]).max() < tol, (k, i)


@DTYPES
def test_draws_are_reproducible_and_independent_of_sharding(torch_cuda, dtype):
    torch = torch_cuda
    n, steps, env_id = 4096, 32, "Cont-CC-SCIM-v0"
    acts = None
    runs = []
    for _ in range(2):
        e = _make(env_id, n, dtype, seed=11)
        e.randomize_env_parameters(*_spec(e))
        e.reset()
        acts = torch.as_tensor(_actions(e, steps, np.random.default_rng(1)), device="cuda") if acts is None else acts
        e.rollout(acts, record_every=0)
        runs.append(e.env_parameters())
    for name in runs[0]:
        assert torch.equal(runs[0][name], runs[1][name])
    # reset(seed=s) reproduces the draws
    e = _make(env_id, n, dtype, seed=11)
    e.randomize_env_parameters(*_spec(e))
    e.reset(seed=99)
    first = {k: v.clone() for k, v in e.env_parameters().items()}
    e.rollout(acts, record_every=0)
    e.reset(seed=99)
    for name, v in e.env_parameters().items():
        assert torch.equal(v, first[name])
    # one handle of N envs == two handles of N/2 with env_index_offset
    halves = []
    for off in (0, n // 2):
        h = _make(env_id, n // 2, dtype, seed=11, offset=off)
        h.randomize_env_parameters(*_spec(h))
        h.reset()
        h.rollout(acts[:, off:off + n // 2].contiguous(), record_every=0)
        halves.append(h.env_parameters())
    for name in runs[0]:
        assert torch.equal(runs[0][name], torch.cat([halves[0][name], halves[1][name]]))


@DTYPES
def test_captured_graph_under_randomisation_equals_eager_loop(torch_cuda, dtype):
    torch = torch_cuda
    n, steps, env_id = 4096, 16, "Cont-CC-SCIM-v0"
    envs = [_make(env_id, n, dtype, seed=5) for _ in range(2)]
    for e in envs:
        e.randomize_env_parameters(*_spec(e))
        e.reset()
    a = torch.as_tensor(_actions(envs[0], 1, np.random.default_rng(2))[0], device="cuda")
    policy = lambda s, r: a  # noqa: E731
    cap = envs[0].capture_steps(policy, steps, record=True, warmup=0)
    cap.replay()
    for k in range(steps):
        (s, r), w, t, _, _ = envs[1].step(a)
        assert torch.equal(cap.states[k], s) and torch.equal(cap.rewards[k], w) and torch.equal(cap.terminateds[k], t.view(torch.uint8)), k
    cap.release()
    for name, v in envs[0].env_parameters().items():
        assert torch.equal(v, envs[1].env_parameters()[name])


@DTYPES
def test_off_switches(torch_cuda, dtype):
    torch = torch_cuda
    n, steps, env_id = 4096, 24, "Cont-CC-SCIM-v0"
    # randomize_env_parameters(): no more draws; the last values stay through resets (B runs them through the host path)
    a_env, b_env = _make(env_id, n, dtype), _make(env_id, n, dtype)
    a_env.randomize_env_parameters(*_spec(a_env))
    a_env.reset()
    theta = {k: v.clone() for k, v in a_env.env_parameters().items()}
    a_env.randomize_env_parameters()
    assert a_env.env_parameters() == {}
    b_env.sim.set_env_params(*_host_rows(b_env, theta))
    acts = torch.as_tensor(_actions(a_env, steps, np.random.default_rng(4)), device="cuda")
    ta_ = torch.zeros(n, dtype=torch.bool, device="cuda")
    for e in (a_env, b_env):
        e.reset(seed=3)
    for k in range(steps):
        (sa, _), wa, ta, _, _ = a_env.step(acts[k])
        (sb, _), wb, tb, _, _ = b_env.step(acts[k])
        assert torch.equal(sa, sb) and torch.equal(wa, wb) and torch.equal(ta, tb), k
        ta_ |= ta
    assert ta_.any()  # resets happened, and drew nothing
    # set_env_parameters(): back to the shared coefficients, bit-identical to a fresh env
    a_env.randomize_env_parameters(*_spec(a_env))
    a_env.rollout(acts, record_every=0)
    a_env.set_env_parameters()
    fresh = _make(env_id, n, dtype)
    (s1, _), _ = a_env.reset(seed=8)
    (s2, _), _ = fresh.reset(seed=8)
    assert torch.equal(s1, s2)
    o1, o2 = a_env.rollout(acts, record_every=1), fresh.rollout(acts, record_every=1)
    for x, y in zip((o1[0][0], o1[1], o1[2]), (o2[0][0], o2[1], o2[2])):
        assert torch.equal(x, y)


def test_refusals_on_the_device_path(torch_cuda):
    torch = torch_cuda
    env = _make("Cont-CC-PMSM-v0", 256, "float32")
    env.randomize_env_parameters(motor_parameter={"r_s": (0.01, 0.03)})
    env.reset()
    with pytest.raises(NotImplementedError, match="DESIGN"):
        env.state_dict()
    with pytest.raises(NotImplementedError, match="DESIGN"):
        env.snapshot_envs()
    with pytest.raises(NotImplementedError, match="DESIGN"):
        env.sim.load_state_dict({"blob": np.zeros(1, np.uint8)})
    lib, h = K.load_library(), env.sim._h
    # the C-ABI refuses the same calls, and pole pairs, unknown slots and bad bounds
    size = lib.gemb200_checkpoint_size(h)
    buf = np.empty(size, dtype=np.uint8)
    assert lib.gemb200_checkpoint_save(h, buf.ctypes.data_as(C.c_void_p)) == K.E_INVALID
    rows = torch.empty((256, env.sim.record_layout()[0]), dtype=torch.int32, device="cuda")
    assert lib.gemb200_pack_envs(h, None, 256, C.c_void_p(rows.data_ptr()), None) == K.E_INVALID

    def call(slot, kind, lo, hi):
        return lib.gemb200_set_param_randomization(h, 1, (C.c_int32 * 1)(slot), (C.c_int32 * 1)(kind), (C.c_double * 1)(lo), (C.c_double * 1)(hi))

    assert call(K.MP_P, K.DIST_UNIFORM, 2, 4) == K.E_INVALID
    assert call(K.MAX_DRAW, K.DIST_UNIFORM, 0, 1) == K.E_INVALID
    assert call(K.MP_R_S, K.DIST_UNIFORM, 1, 0) == K.E_INVALID
    assert call(K.MP_R_S, K.DIST_LOG_UNIFORM, 0, 1) == K.E_INVALID
    assert call(K.MP_R_S, K.DIST_UNIFORM, 0, float("inf")) == K.E_INVALID
    env.randomize_env_parameters()  # off: checkpoints work again
    assert lib.gemb200_checkpoint_save(h, buf.ctypes.data_as(C.c_void_p)) == 0
    out = torch.empty(256, device="cuda")
    assert lib.gemb200_get_env_params(h, C.c_void_p(out.data_ptr()), None) == K.E_INVALID
    soa = _make("Cont-CC-PMSM-v0", 256, "float32", layout="soa")
    with pytest.raises(ValueError):
        soa.randomize_env_parameters(motor_parameter={"r_s": (0.01, 0.03)})
    lib_soa = soa.sim
    assert lib.gemb200_set_param_randomization(lib_soa._h, 1, (C.c_int32 * 1)(K.MP_R_S), (C.c_int32 * 1)(0), (C.c_double * 1)(0.01),
                                               (C.c_double * 1)(0.03)) == K.E_INVALID
