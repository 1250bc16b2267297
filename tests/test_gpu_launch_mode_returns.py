"""Which rollout instantiation a launch with discounted returns takes: never PLAIN (the PLAIN kernels have no returns), general with shared
coefficients, ENVP with per-env blocks or adopted RNG identities; launches without returns keep their PLAIN kernels.  Same profiler method
as tests/test_gpu_launch_mode.py, and like tests/test_gpu_launch_mode_feed.py this module runs before the suite's long GPU modules: later
in a full `-m gpu` session the profiler records no kernels at all."""
import numpy as np
import pytest

from test_gpu_launch_mode import _modes
from test_gpu_parity import torch_cuda  # noqa: F401
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu


def test_launch_modes(torch_cuda):
    torch = torch_cuda
    import gym_electric_motor_b200 as gem

    n = 4096
    env = gem.make("Cont-CC-PMSM-v0", num_envs=n, device="cuda", dtype="float32", ode_solver=gem.physical_systems.RK4Solver(),
                   autoreset="same_step", seed=0)
    env.reset()
    acts = torch.zeros(2, n, 3, device="cuda")

    def modes(returns):  # a step, a rollout and (with returns) a scored rollout in one profiler session
        if returns:
            return sorted(_modes(torch, lambda: (env.step(acts[0]), env.rollout(acts, record_every=0), env.rollout_returns(acts, 0.9))))
        return sorted(_modes(torch, lambda: (env.step(acts[0]), env.rollout(acts, record_every=0))))

    modes(False)  # the profiler's first session pays its set-up
    plain = [("rollout_kernel", "PLAIN"), ("step_kernel", "PLAIN")]
    assert modes(False) == plain
    assert modes(True) == [("rollout_kernel", "PLAIN"), ("rollout_kernel", "general"), ("step_kernel", "PLAIN")]
    r_s = float(env.sim.cfg.motor_param[K.MP_R_S])
    env.set_env_parameters(motor_parameter={"r_s": r_s * np.linspace(0.9, 1.1, n)})
    assert modes(True) == [("rollout_kernel", "ENVP")] * 2 + [("step_kernel", "ENVP")]
    env.set_env_parameters()
    assert modes(False) == plain
    env.restore_envs(env.snapshot_envs([0], rng=True), idx=[5], rng="source")  # adopted identities: the ENVP kernels read them
    assert modes(True) == [("rollout_kernel", "ENVP")] * 2 + [("step_kernel", "ENVP")]
