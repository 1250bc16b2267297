"""Which instantiation a step and a rollout with a reference feed launch: never PLAIN (the PLAIN kernels have no feed), general with shared
coefficients, ENVP with per-env parameter blocks; without a feed the PLAIN shape keeps its PLAIN kernels.  Same profiler method as
tests/test_gpu_launch_mode.py, and like it this module runs before the suite's long GPU modules: later in a full `-m gpu` session the
profiler records no kernels at all."""
import numpy as np
import pytest

from test_gpu_launch_mode import _modes
from test_gpu_parity import torch_cuda  # noqa: F401
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu


def test_launch_modes(torch_cuda):
    torch = torch_cuda
    import gym_electric_motor_b200 as gem

    env = gem.make("Cont-CC-PMSM-v0", num_envs=4096, device="cuda", dtype="float32", ode_solver=gem.physical_systems.RK4Solver(),
                   autoreset="same_step", seed=0)
    env.reset()
    acts = torch.zeros(2, 4096, 3, device="cuda")
    refs = torch.zeros(2, 4096, 2, device="cuda")

    def modes(feed):  # a step and a rollout in one profiler session
        if feed:
            return sorted(_modes(torch, lambda: (env.step(acts[0], reference=refs[0]), env.rollout(acts, record_every=1, references=refs))))
        return sorted(_modes(torch, lambda: (env.step(acts[0]), env.rollout(acts, record_every=1))))

    modes(False)  # the profiler's first session pays its set-up
    assert modes(False) == [("rollout_kernel", "PLAIN"), ("step_kernel", "PLAIN")]
    assert modes(True) == [("rollout_kernel", "general")] * 2  # step(action, reference=r) is the K = 1 rollout
    r_s = float(env.sim.cfg.motor_param[K.MP_R_S])
    env.set_env_parameters(motor_parameter={"r_s": r_s * np.linspace(0.9, 1.1, 4096)})
    assert modes(True) == [("rollout_kernel", "ENVP")] * 2
    env.set_env_parameters()
    assert modes(False) == [("rollout_kernel", "PLAIN"), ("step_kernel", "PLAIN")]
