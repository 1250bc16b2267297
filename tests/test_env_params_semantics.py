"""Per-env physical parameters without a GPU: the pole-pair refusal of `set_env_parameters` / `VectorSim.set_env_params` around a scripted
handle, and an audit of what the host derives from the physical parameters.

Per-env rows replace the model coefficients only; everything else a configuration carries stays the handle's.  The audit makes every
configuration of tests/test_gpu_env_params_oracle.py with each slot doubled and compares the config field by field: the only fields that
may move are the parameters themselves, the limit / normalisation fields, and the two documented per-handle constants (DESIGN.md §7):
the induction motors' flux limits `init_im` and the FluxObserver constants `sop_param`.  A new host-side constant derived from a physical
parameter fails here and has to be decided on (per env, or documented as per handle).
"""
import ctypes as C

import numpy as np
import pytest

import gym_electric_motor_b200 as gem
from gym_electric_motor_b200 import _cabi as K
from helpers import ENV_PARAM_CASES, LP_SLOT, MOTOR_SLOTS, motor_of

PARAM_FIELDS = {"motor_param", "load_param"}
# limits and nominal values derive from the motor parameters (e.g. the torque limit of a synchronous motor); the random initial state
# box / gaussian mean and the reward's state lengths (the FluxObserver's psi_abs limit is l_m * i_sd,limit) from the limits
LIMIT_FIELDS = {"limits", "state_length", "init_lo", "init_hi", "init_mu", "init_sigma"}
PER_HANDLE_FIELDS = {"init_im", "sop_param"}
IGNORED = {"ext_speed_table"}  # a host pointer


def _value(cfg, name):
    v = getattr(cfg, name)
    if isinstance(v, C.Array):
        return [list(x) if isinstance(x, C.Array) else x for x in v]
    return v


def _make(case, motor_parameter=None, load_parameter=None):
    env_id, kw = ENV_PARAM_CASES[case]()
    if motor_parameter:
        kw["motor"] = dict(kw.get("motor", {}), motor_parameter=motor_parameter)
    if load_parameter:
        load = dict(kw.get("load", {}))
        load["load_parameter"] = dict(load.get("load_parameter", {}), **load_parameter)
        kw["load"] = load
    return gem.make(env_id, ode_solver=gem.physical_systems.RK4Solver(), seed=17, **kw)


@pytest.mark.parametrize("case", list(ENV_PARAM_CASES))
def test_only_parameters_limits_and_documented_constants_follow_the_physical_parameters(case):
    env = _make(case)
    base = env.build_config()
    motor = env.physical_system.electrical_motor
    names = [(n, False) for n in MOTOR_SLOTS[motor_of(env.env_id)]]
    if motor_of(env.env_id) == "EESM":
        names.append(("k", False))  # no output depends on it, but the host must not derive anything else from it either
    if base.load_kind == K.LOAD_POLY_STATIC:
        names += [("j_rotor", False)] + [(n, True) for n in LP_SLOT]
    fields = [f for f, _ in type(base)._fields_ if f not in IGNORED]
    for name, is_load in names:
        if is_load:
            scaled = _make(case, load_parameter={name: 2.0 * base.load_param[LP_SLOT[name]]})
        else:
            scaled = _make(case, motor_parameter={name: 2.0 * motor.motor_parameter[name]})
        cfg = scaled.build_config()
        moved = {f for f in fields if _value(cfg, f) != _value(base, f)}
        assert moved & PARAM_FIELDS, (case, name)  # the parameter itself arrived
        extra = moved - PARAM_FIELDS - LIMIT_FIELDS - PER_HANDLE_FIELDS
        assert not extra, f"{case}: {name} x2 moves host-derived fields {sorted(extra)}"


# ---------------------------------------------------------------------------------------------------- pole-pair refusal (no GPU)
class EnvParamHandle:
    """the VectorSim surface `set_env_parameters` uses; records the rows it is given instead of uploading them"""

    def __init__(self, cfg, reuse_outputs=True):
        self.cfg, self.n, self.soa = cfg, cfg.n_envs, cfg.layout == K.LAYOUT_SOA
        self.calls = []
        EnvParamHandle.last = self

    def set_env_params(self, motor_param=None, load_param=None):
        self.calls.append((motor_param, load_param))

    def close(self):
        pass


@pytest.fixture
def handle(monkeypatch):
    import gym_electric_motor_b200.vector_sim as vs

    monkeypatch.setattr(vs, "VectorSim", EnvParamHandle)
    return EnvParamHandle


def test_set_env_parameters_refuses_per_env_pole_pairs(handle):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=5)
    p = env.build_config().motor_param[K.MP_P]
    with pytest.raises(ValueError, match="pole pairs"):
        env.set_env_parameters(motor_parameter={"p": [p, p, p + 1, p, p]})
    with pytest.raises(ValueError, match="pole pairs"):
        env.set_env_parameters(motor_parameter={"p": 2 * p, "r_s": 0.02})
    assert not handle.last.calls  # refused before the handle is called
    # the tile-and-edit pattern: pole pairs equal to the env's are accepted
    env.set_env_parameters(motor_parameter={"p": p, "r_s": np.linspace(0.01, 0.03, 5)})
    env.set_env_parameters(motor_parameter={"p": [p] * 5})
    env.set_env_parameters(load_parameter={"j_load": 1e-3})
    assert len(handle.last.calls) == 3
    mp, _ = handle.last.calls[0]
    assert np.all(mp[:, K.MP_P] == p) and np.allclose(mp[:, K.MP_R_S], np.linspace(0.01, 0.03, 5))


def test_vector_sim_set_env_params_refuses_per_env_pole_pairs():
    from gym_electric_motor_b200.vector_sim import VectorSim

    cfg = gem.make("Cont-SC-SCIM-v0", num_envs=4).build_config()
    sim = VectorSim.__new__(VectorSim)  # no device: only the host check before the C-ABI call runs

    class Lib:
        calls = []

        def gemb200_set_env_params(self, h, mp, lp):
            Lib.calls.append((mp, lp))
            return 0

    sim.cfg, sim.n, sim._h, sim._lib = cfg, 4, None, Lib()
    mp = np.tile(np.array(list(cfg.motor_param)), (4, 1))
    bad = mp.copy()
    bad[3, K.MP_P] = 3.0
    with pytest.raises(ValueError, match="pole pairs"):
        sim.set_env_params(bad, None)
    bad[3, K.MP_P] = np.nan
    with pytest.raises(ValueError, match="pole pairs"):
        sim.set_env_params(bad, None)
    assert not Lib.calls
    sim.set_env_params(mp, None)
    sim.set_env_params(None, np.tile(np.array(list(cfg.load_param)), (4, 1)))  # load rows only: the configuration's pole pairs
    assert len(Lib.calls) == 2
