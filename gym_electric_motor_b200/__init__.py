"""gym_electric_motor_b200 — H100-native vectorised physical-system step for gym-electric-motor (GEM).

    import gym_electric_motor_b200 as gem
    env = gem.make("Cont-CC-PMSM-v0", num_envs=1 << 20, ode_solver=gem.physical_systems.RK4Solver())
    (state, ref), _ = env.reset(seed=0)
    (state, ref), reward, terminated, truncated, _ = env.step(actions)      # torch tensors on the GPU, one launch

The package mirrors the reference's surface for the hot path only (SURVEY.md §8): `make`, the batched
`ElectricMotorEnvironment`, the SCML component classes, reference generators, reward function and constraints.
All compute runs in libgemb200.so (hand-written sm_90a CUDA, C-ABI in include/gemb200.h); importing this package
does not need a GPU, creating an environment does.
"""
from . import envs, physical_system_wrappers, physical_systems, reference_generators, reward_functions, vector, visualization  # noqa: F401
from .constraints import Constraint, ConstraintMonitor, LimitConstraint, SquaredConstraint  # noqa: F401
from .core import Callback, ElectricMotorEnvironment, ElectricMotorVisualization  # noqa: F401
from .envs import env_ids, make  # noqa: F401
from .physical_systems import PhysicalSystem  # noqa: F401
from .reference_generators import ReferenceGenerator  # noqa: F401
from .reward_functions import RewardFunction, WeightedSumOfErrors  # noqa: F401
from .snapshot import EnvSnapshot  # noqa: F401

__version__ = "0.1.0"

_ALIASED_SUBMODULES = ("physical_systems", "physical_systems.solvers", "physical_systems.mechanical_loads", "physical_systems.converters",
                       "physical_systems.electric_motors", "physical_systems.voltage_supplies", "physical_systems.physical_systems",
                       "reference_generators", "physical_system_wrappers", "reward_functions", "constraints", "core", "utils", "envs", "envs.motors",
                       "visualization")


def install_as_gym_electric_motor():
    """Make `import gym_electric_motor as gem` (and `from gym_electric_motor.<submodule> import ...`) in EXISTING agent code resolve to
    this package: registers it and its submodules under the reference's module names in `sys.modules`.  Call it once before the
    agent's imports.  Refuses when the real gym_electric_motor has already been imported (the two cannot be mixed in one process)."""
    import importlib
    import sys

    me = sys.modules[__name__]
    other = sys.modules.get("gym_electric_motor")
    if other is not None and other is not me:
        raise RuntimeError("gym_electric_motor is already imported in this process; install the alias before importing agent code")
    sys.modules["gym_electric_motor"] = me
    for sub in _ALIASED_SUBMODULES:
        sys.modules["gym_electric_motor." + sub] = importlib.import_module(__name__ + "." + sub)
    sys.modules["gym_electric_motor.visualization.motor_dashboard"] = sys.modules["gym_electric_motor.visualization"]  # one flat module here
    me.gym_electric_motor = me  # `from gym_electric_motor import gym_electric_motor as gem` (seen in the reference's notebooks)
    return me
