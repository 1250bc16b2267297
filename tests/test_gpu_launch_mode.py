"""Which step / rollout instantiation a handle launches as its per-env parameters, draws, RNG identities and peer destinations come and go.

The PLAIN, general and ENVP instantiations give bit-identical results (DESIGN.md §2), so no output test notices a handle that takes the
wrong one; only its speed does (DESIGN.md §4: shared coefficients against per-env blocks).  This test reads the instantiation from the
kernel name that torch.profiler records: PLAIN is the 6th and ENVP the 8th template argument of step_kernel / rollout_kernel."""
import ctypes as C
import re

import numpy as np
import pytest

from test_gpu_parity import torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

N = 4096


def _modes(torch, fn):
    """instantiations ("PLAIN", "ENVP" or "general") of the step and rollout kernels that fn() launches"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    modes = []
    for e in prof.events():
        m = re.search(r"(step_kernel|rollout_kernel)<([^>]*)>", e.name)
        if not m:
            continue
        args = [a.strip() for a in m.group(2).split(",")]
        on = [a in ("true", "(bool)1", "1") for a in args]
        modes.append((m.group(1), "PLAIN" if on[5] else ("ENVP" if on[7] else "general")))
    return modes


def test_launch_mode_transitions(torch_cuda):
    torch = torch_cuda
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200 import _cabi as K

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
    _modes(torch, lambda: env.step(act()))  # the profiler's first session pays its set-up
    seen, want = [], []
    for k, (what, change, expected) in enumerate(transitions):
        change()
        got = _modes(torch, lambda: env.step(act())) + _modes(torch, lambda: env.rollout(act(2), record_every=1))
        assert [kernel for kernel, _ in got] == ["step_kernel", "rollout_kernel"], (k, what, got)
        seen.append((k, what, [mode for _, mode in got]))
        want.append((k, what, [expected, expected]))
    assert seen == want
