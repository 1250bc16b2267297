"""Which kernel a return-gradient launch takes: its own `return_grad_kernel`, with shared coefficients or (per-env blocks) the ENVP
variant, and never a step, rollout or Jacobian kernel; launches without gradients keep their PLAIN kernels.  Same profiler method as
tests/test_gpu_launch_mode_jacobians.py."""
import re

import numpy as np
import pytest

from test_gpu_parity import torch_cuda  # noqa: F401
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu


def _kernels(torch, fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = []
    for e in prof.events():
        m = re.search(r"(return_grad_kernel|jacobian_kernel|step_kernel|rollout_kernel)<([^>]*)>", e.name)
        if not m:
            continue
        args = [a.strip() for a in m.group(2).split(",")]
        on = [a in ("true", "(bool)1", "1") for a in args]
        if m.group(1) == "return_grad_kernel":
            out.append((m.group(1), "ENVP" if on[3] else "shared"))
        elif m.group(1) == "jacobian_kernel":
            out.append((m.group(1), "ENVP" if on[4] else "shared"))
        else:
            out.append((m.group(1), "PLAIN" if on[5] else ("ENVP" if on[7] else "general")))
    return sorted(out)


def test_launch_modes(torch_cuda):
    torch = torch_cuda
    import gym_electric_motor_b200 as gem

    n = 4096
    env = gem.make("Cont-CC-PMSM-v0", num_envs=n, device="cuda", dtype="float32", ode_solver=gem.physical_systems.RK4Solver(),
                   autoreset="same_step", seed=0)
    env.reset()
    acts = torch.zeros(2, n, 3, device="cuda")
    both = lambda: (env.rollout(acts, record_every=1), env.rollout_return_grads(acts, 0.9))  # noqa: E731
    _kernels(torch, both)  # the profiler's first session pays its set-up
    assert _kernels(torch, both) == [("return_grad_kernel", "shared"), ("rollout_kernel", "PLAIN")]
    r_s = float(env.sim.cfg.motor_param[K.MP_R_S])
    env.set_env_parameters(motor_parameter={"r_s": r_s * np.linspace(0.9, 1.1, n)})
    assert _kernels(torch, both) == [("return_grad_kernel", "ENVP"), ("rollout_kernel", "ENVP")]
    env.set_env_parameters()
