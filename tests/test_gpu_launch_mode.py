"""Which kernel and instantiation a handle launches: the step / rollout instantiation as its per-env parameters, draws, RNG identities and
peer destinations come and go, and the kernels of a reference feed, of Jacobians, of parameter sensitivities, of return gradients and of
discounted returns; and the block size of step and rollout launches at the batch sizes of the launch-shape tests.

The PLAIN, general and ENVP instantiations give bit-identical results (DESIGN.md §2), so no output test notices a handle that takes the
wrong one; only its speed does (DESIGN.md §4: shared coefficients against per-env blocks).  These tests read the kernel and its
instantiation from the kernel names that torch.profiler records (gpu_helpers._kernels).  The module runs before the suite's long GPU
modules: later in a full `-m gpu` session the profiler records no kernels at all."""
import ctypes as C

import numpy as np
import pytest

from gpu_helpers import N as N_SMALL, _kernels, _launches, launch_block, launch_sizes, torch_cuda  # noqa: F401
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

N = 4096
NAMES = ["r_s", "l_d", "l_q", "psi_p"]


def test_launch_mode_transitions(torch_cuda):
    torch = torch_cuda
    import gym_electric_motor_b200 as gem

    # bench.py's pmsm workload at a small size: fp32, AoS, RK4 (the PLAIN shape)
    env = gem.make("Cont-CC-PMSM-v0", num_envs=N, device="cuda", dtype="float32", ode_solver=gem.physical_systems.RK4Solver(),
                   autoreset="same_step", seed=0)
    env.reset()
    sim = env.sim
    rng = np.random.default_rng(0)
    r_s = float(sim.cfg.motor_param[K.MP_R_S])
    per_env = {"r_s": r_s * np.linspace(0.9, 1.1, N)}

    def act(*lead):
        return torch.as_tensor(rng.uniform(-1, 1, size=lead + (N, 3)), dtype=torch.float32, device="cuda")

    def adopt():
        env.restore_envs(env.snapshot_envs([0], rng=True), idx=[5], rng="source")

    def bind_peers(n_dst):
        delta = (C.c_int64 * 1)(0)  # delta 0: the peer stores land on the caller's own tensors
        K.check(sim._lib.gemb200_bind_peers(sim._h, n_dst, C.cast(delta, C.c_void_p) if n_dst else None), "gemb200_bind_peers")

    transitions = [
        ("fresh env", lambda: None, "PLAIN"),
        ("per-env r_s", lambda: env.set_env_parameters(motor_parameter=per_env), "ENVP"),
        ("shared parameters", lambda: env.set_env_parameters(), "PLAIN"),
        ("adopt", adopt, "ENVP"),
        ("clear identities", env.clear_rng_identities, "PLAIN"),
        ("adopt, per-env r_s, clear identities",
         lambda: (adopt(), env.set_env_parameters(motor_parameter=per_env), env.clear_rng_identities()), "ENVP"),
        ("shared parameters", lambda: env.set_env_parameters(), "PLAIN"),
        ("adopt, shared parameters", lambda: (adopt(), env.set_env_parameters()), "ENVP"),
        ("clear identities", env.clear_rng_identities, "PLAIN"),
        ("draw r_s", lambda: env.randomize_env_parameters(motor_parameter={"r_s": (0.9 * r_s, 1.1 * r_s)}), "ENVP"),
        ("stop draws", lambda: env.randomize_env_parameters(), "ENVP"),
        ("shared parameters", lambda: env.set_env_parameters(), "PLAIN"),
        ("adopt, reseed", lambda: (adopt(), env.reset(seed=3)), "PLAIN"),
        ("per-env r_s, reseed", lambda: (env.set_env_parameters(motor_parameter=per_env), env.reset(seed=4)), "ENVP"),
        ("shared parameters, one peer destination", lambda: (env.set_env_parameters(), bind_peers(1)), "general"),
        ("no peer destinations", lambda: bind_peers(0), "PLAIN"),
    ]
    _kernels(torch, lambda: env.step(act()))  # the profiler's first session pays its set-up
    seen, want = [], []
    for k, (what, change, expected) in enumerate(transitions):
        change()
        got = _kernels(torch, lambda: env.step(act())) + _kernels(torch, lambda: env.rollout(act(2), record_every=1))
        assert [kernel for kernel, _ in got] == ["step_kernel", "rollout_kernel"], (k, what, got)
        seen.append((k, what, [mode for _, mode in got]))
        want.append((k, what, [expected, expected]))
    assert seen == want


def _make(n, dtype="float32", seed=0):
    """bench.py's pmsm workload: fp32, AoS, RK4 (the PLAIN shape)"""
    import gym_electric_motor_b200 as gem

    env = gem.make("Cont-CC-PMSM-v0", num_envs=n, device="cuda", dtype=dtype, ode_solver=gem.physical_systems.RK4Solver(), autoreset="same_step",
                   seed=seed)
    env.reset()
    return env


def test_feed_launch_modes(torch_cuda):
    """a step and a rollout with a reference feed: never PLAIN (the PLAIN kernels have no feed), general with shared coefficients, ENVP with
    per-env parameter blocks; without a feed the PLAIN shape keeps its PLAIN kernels"""
    torch = torch_cuda
    env = _make(N)
    acts = torch.zeros(2, N, 3, device="cuda")
    refs = torch.zeros(2, N, 2, device="cuda")

    def modes(feed):  # a step and a rollout in one profiler session
        if feed:
            return sorted(_kernels(torch, lambda: (env.step(acts[0], reference=refs[0]), env.rollout(acts, record_every=1, references=refs))))
        return sorted(_kernels(torch, lambda: (env.step(acts[0]), env.rollout(acts, record_every=1))))

    modes(False)  # the profiler's first session pays its set-up
    assert modes(False) == [("rollout_kernel", "PLAIN"), ("step_kernel", "PLAIN")]
    assert modes(True) == [("rollout_kernel", "general")] * 2  # step(action, reference=r) is the K = 1 rollout
    r_s = float(env.sim.cfg.motor_param[K.MP_R_S])
    env.set_env_parameters(motor_parameter={"r_s": r_s * np.linspace(0.9, 1.1, N)})
    assert modes(True) == [("rollout_kernel", "ENVP")] * 2
    env.set_env_parameters()
    assert modes(False) == [("rollout_kernel", "PLAIN"), ("step_kernel", "PLAIN")]


def _tangent_launch_modes(torch, tangent, kernel, identities=True):
    """a recorded rollout and tangent(env, acts): the tangent kernel, with shared coefficients or (per-env blocks, adopted RNG identities) its
    ENVP variant, and never a step or rollout kernel; the rollout keeps its PLAIN kernel without per-env state"""
    env = _make(N)
    acts = torch.zeros(2, N, 3, device="cuda")
    both = lambda: (env.rollout(acts, record_every=1), tangent(env, acts))  # noqa: E731
    _kernels(torch, both)  # the profiler's first session pays its set-up
    assert sorted(_kernels(torch, both)) == [(kernel, "shared"), ("rollout_kernel", "PLAIN")]
    r_s = float(env.sim.cfg.motor_param[K.MP_R_S])
    env.set_env_parameters(motor_parameter={"r_s": r_s * np.linspace(0.9, 1.1, N)})
    assert sorted(_kernels(torch, both)) == [(kernel, "ENVP"), ("rollout_kernel", "ENVP")]
    env.set_env_parameters()
    if identities:
        env.restore_envs(env.snapshot_envs([0], rng=True), idx=[5], rng="source")
        assert sorted(_kernels(torch, both)) == [(kernel, "ENVP"), ("rollout_kernel", "ENVP")]


def test_jacobian_launch_modes(torch_cuda):
    _tangent_launch_modes(torch_cuda, lambda env, acts: env.rollout_jacobians(acts), "jacobian_kernel")


def test_param_sens_launch_modes(torch_cuda):
    _tangent_launch_modes(torch_cuda, lambda env, acts: env.rollout_param_sensitivities(acts, NAMES), "param_sens_kernel")


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_device_clock_and_cuda_graph(torch_cuda, dtype):
    """under the device clock rollout_param_sens_into is stream-ordered and capturable: an eager launch and replays of a captured one give,
    round after round, the bits of host-clock launches on a twin (sens_io refilled with zeros in place before each replay)"""
    torch = torch_cuda
    n, k = 1000, 12
    host, dev, cap = _make(n, dtype), _make(n, dtype), _make(n, dtype)
    dev.sim.set_device_clock(True)
    cap.sim.set_device_clock(True)
    sim = cap.sim
    slots = cap.param_slots(NAMES)
    nx = sim.n_ode
    rng = np.random.default_rng(0)
    static = torch.zeros(k, n, 3, dtype=sim.dtype, device="cuda")
    sio = torch.zeros(n, nx, len(NAMES), dtype=sim.dtype, device="cuda")
    so = torch.empty(k, n, nx, len(NAMES), dtype=sim.dtype, device="cuda")
    obs = torch.empty((k,) + sim._shape(sim.n_state), dtype=sim.dtype, device="cuda")
    ref = torch.empty((k,) + sim._shape(sim.n_ref), dtype=sim.dtype, device="cuda")
    rew = torch.empty(k, n, dtype=sim.dtype, device="cuda")
    term = torch.empty(k, n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sim.rollout_param_sens_into(static, k, slots, sio, so, obs, ref, rew, term)
    terminated = 0
    for rnd in range(3):
        acts = torch.as_tensor(rng.uniform(-1, 1, size=(k, n, 3)), dtype=sim.dtype, device="cuda").contiguous()
        static.copy_(acts)
        sio.zero_()
        graph.replay()
        (s_h, l_h), ((o_h, r_h), w_h, t_h) = host.rollout_param_sensitivities(acts, NAMES)
        (s_d, l_d), ((o_d, r_d), w_d, t_d) = dev.rollout_param_sensitivities(acts, NAMES)
        for name, a, b, c in (("sens", s_h, s_d, so), ("sens_last", l_h, l_d, sio), ("obs", o_h, o_d, obs), ("reward", w_h, w_d, rew)):
            assert torch.equal(a, b) and torch.equal(a, c), (rnd, name)
        assert torch.equal(t_h.to(torch.uint8), term)
        terminated += int(t_h.sum())
    assert terminated > 0
    assert host.sim.clock() == dev.sim.clock() == cap.sim.clock()


def test_launch_blocks(torch_cuda, tmp_path):
    """the block size of the step and rollout launches (pick_block): 32, 64 and 128 threads at N = 300, N64 and N128 (gpu_helpers.launch_sizes)
    for the PLAIN shape, a general instantiation (state wrappers widen its rows) and per-env blocks (ENVP); and the pipelined host step at
    NHOST: four chunks of 64-thread blocks, while the twin's full-batch device step launches 128.  test_gpu_launch_shape relies on these
    shapes: if pick_block changes, this test fails instead of letting those tests quietly run one-warp blocks."""
    torch = torch_cuda
    import gym_electric_motor_b200 as gem
    from helpers import ENV_PARAM_CASES

    sz = launch_sizes()
    s = sz["S"]

    def general(n):
        env_id, kw = ENV_PARAM_CASES["cc-scim-observer-dq"]()
        env = gem.make(env_id, num_envs=n, device="cuda", dtype="float32", autoreset="same_step", seed=0, **kw)
        env.reset()
        return env

    def envp(n):
        env = _make(n)
        r_s = float(env.sim.cfg.motor_param[K.MP_R_S])
        env.set_env_parameters(motor_parameter={"r_s": r_s * np.linspace(0.9, 1.1, n)})
        return env

    _launches(torch, lambda: None, tmp_path)  # the profiler's first session pays its set-up
    seen, want = [], []
    for mode, mk in (("PLAIN", _make), ("general", general), ("ENVP", envp)):
        for n in (N_SMALL, sz["N64"], sz["N128"]):
            env = mk(n)
            n_act = env.sim.n_act
            acts = torch.zeros(2, n, n_act, device="cuda")
            got = _launches(torch, lambda: (env.step(acts[0]), env.rollout(acts, record_every=1)), tmp_path)
            block = launch_block(n, s)
            seen.append((mode, n, got))
            want.append((mode, n, [(k, mode, block, (n + block - 1) // block) for k in ("step_kernel", "rollout_kernel")]))
            env.close()
    assert [launch_block(n, s) for n in (N_SMALL, sz["N64"], sz["N128"])] == [32, 64, 128]
    assert seen == want
    # the pipelined host step: four chunks of whole 256-env blocks, one launch each, against the twin's one launch over all envs
    n = sz["NHOST"]
    host, twin = _make(n), _make(n)
    a = np.zeros((n, 3), dtype=np.float32)
    per = ((n + 3) // 4 + 255) // 256 * 256
    chunks = [min(per, n - b) for b in range(0, n, per)]
    got = _launches(torch, lambda: (host.sim.step_host(a), twin.sim.step(torch.zeros(n, 3, device="cuda"))), tmp_path)
    assert [launch_block(c, s) for c in chunks] == [64] * 4
    assert got == [("step_kernel", "PLAIN", 64, (c + 63) // 64) for c in chunks] + [("step_kernel", "PLAIN", 128, (n + 127) // 128)]


def test_return_grad_launch_modes(torch_cuda):
    _tangent_launch_modes(torch_cuda, lambda env, acts: env.rollout_return_grads(acts, 0.9), "return_grad_kernel", identities=False)


def test_returns_launch_modes(torch_cuda):
    """a rollout with discounted returns: never PLAIN (the PLAIN kernels have no returns), general with shared coefficients, ENVP with
    per-env blocks or adopted RNG identities; launches without returns keep their PLAIN kernels"""
    torch = torch_cuda
    env = _make(N)
    acts = torch.zeros(2, N, 3, device="cuda")

    def modes(returns):  # a step, a rollout and (with returns) a scored rollout in one profiler session
        if returns:
            return sorted(_kernels(torch, lambda: (env.step(acts[0]), env.rollout(acts, record_every=0), env.rollout_returns(acts, 0.9))))
        return sorted(_kernels(torch, lambda: (env.step(acts[0]), env.rollout(acts, record_every=0))))

    modes(False)  # the profiler's first session pays its set-up
    plain = [("rollout_kernel", "PLAIN"), ("step_kernel", "PLAIN")]
    assert modes(False) == plain
    assert modes(True) == [("rollout_kernel", "PLAIN"), ("rollout_kernel", "general"), ("step_kernel", "PLAIN")]
    r_s = float(env.sim.cfg.motor_param[K.MP_R_S])
    env.set_env_parameters(motor_parameter={"r_s": r_s * np.linspace(0.9, 1.1, N)})
    assert modes(True) == [("rollout_kernel", "ENVP")] * 2 + [("step_kernel", "ENVP")]
    env.set_env_parameters()
    assert modes(False) == plain
    env.restore_envs(env.snapshot_envs([0], rng=True), idx=[5], rng="source")  # adopted identities: the ENVP kernels read them
    assert modes(True) == [("rollout_kernel", "ENVP")] * 2 + [("step_kernel", "ENVP")]
