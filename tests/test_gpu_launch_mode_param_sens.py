"""Which kernel a parameter-sensitivity launch takes: its own `param_sens_kernel`, with shared coefficients or (per-env blocks, adopted RNG
identities) the ENVP variant, and never a step or rollout kernel; and the launch under the device clock, eager and captured in a CUDA graph,
gives the bits of the host-clock launch.  Same profiler method as tests/test_gpu_launch_mode.py."""
import re

import numpy as np
import pytest

from test_gpu_parity import torch_cuda  # noqa: F401
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

NAMES = ["r_s", "l_d", "l_q", "psi_p"]


def _kernels(torch, fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = []
    for e in prof.events():
        m = re.search(r"(param_sens_kernel|step_kernel|rollout_kernel)<([^>]*)>", e.name)
        if not m:
            continue
        args = [a.strip() for a in m.group(2).split(",")]
        on = [a in ("true", "(bool)1", "1") for a in args]
        if m.group(1) == "param_sens_kernel":
            out.append((m.group(1), "ENVP" if on[4] else "shared"))
        else:
            out.append((m.group(1), "PLAIN" if on[5] else ("ENVP" if on[7] else "general")))
    return sorted(out)


def _make(n, dtype="float32", seed=0):
    import gym_electric_motor_b200 as gem

    env = gem.make("Cont-CC-PMSM-v0", num_envs=n, device="cuda", dtype=dtype, ode_solver=gem.physical_systems.RK4Solver(), autoreset="same_step",
                   seed=seed)
    env.reset()
    return env


def test_launch_modes(torch_cuda):
    torch = torch_cuda
    n = 4096
    env = _make(n)
    acts = torch.zeros(2, n, 3, device="cuda")
    both = lambda: (env.rollout(acts, record_every=1), env.rollout_param_sensitivities(acts, NAMES))  # noqa: E731
    _kernels(torch, both)  # the profiler's first session pays its set-up
    assert _kernels(torch, both) == [("param_sens_kernel", "shared"), ("rollout_kernel", "PLAIN")]
    r_s = float(env.sim.cfg.motor_param[K.MP_R_S])
    env.set_env_parameters(motor_parameter={"r_s": r_s * np.linspace(0.9, 1.1, n)})
    assert _kernels(torch, both) == [("param_sens_kernel", "ENVP"), ("rollout_kernel", "ENVP")]
    env.set_env_parameters()
    env.restore_envs(env.snapshot_envs([0], rng=True), idx=[5], rng="source")
    assert _kernels(torch, both) == [("param_sens_kernel", "ENVP"), ("rollout_kernel", "ENVP")]


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
