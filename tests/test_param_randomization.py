"""Per-episode domain randomisation without a GPU: the encoding of the distributions into slots, kinds and bounds, the argument checks and
refusals of ElectricMotorEnvironment.randomize_env_parameters that fire before any device call, and the new C-ABI symbols."""
import ctypes as C
import os

import pytest

import gym_electric_motor_b200 as gem
from gym_electric_motor_b200 import _cabi as K
from gym_electric_motor_b200.core import ElectricMotorEnvironment as Env
from gym_electric_motor_b200.randomization import encode_distributions, parse_distribution

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "gemb200.h")


def test_encoding_of_motor_and_load_distributions():
    names, slots, kinds, lo, hi = encode_distributions({"r_s": (0.1, 0.2), "l_d": ("log_uniform", 1e-4, 1e-3)}, {"j_load": ("uniform", 0, 1)},
                                                       Env._MP_SLOT, Env._LP_SLOT)
    assert names == ["r_s", "l_d", "j_load"]
    assert slots == [K.MP_R_S, K.MP_L_D, K.MAX_MOTOR_PARAM + K.LP_J_LOAD]
    assert kinds == [K.DIST_UNIFORM, K.DIST_LOG_UNIFORM, K.DIST_UNIFORM]
    assert lo == [0.1, 1e-4, 0.0] and hi == [0.2, 1e-3, 1.0]
    assert all(0 <= s < K.MAX_DRAW for s in slots)


def test_empty_spec_encodes_to_nothing():
    assert encode_distributions(None, None, Env._MP_SLOT, Env._LP_SLOT) == ([], [], [], [], [])


@pytest.mark.parametrize("spec", [(2.0, 1.0), ("log_uniform", 0.0, 1.0), ("log_uniform", -1.0, 1.0), (0.0, float("inf")), (float("nan"), 1.0),
                                  ("normal", 0.0, 1.0), (1.0,), 0.5, ("a", "b")])
def test_bad_distributions_raise_value_error(spec):
    with pytest.raises(ValueError):
        parse_distribution("r_s", spec)


def test_degenerate_interval_is_allowed():
    assert parse_distribution("r_s", (0.5, 0.5)) == (K.DIST_UNIFORM, 0.5, 0.5)


def test_unknown_names_raise_key_error():
    with pytest.raises(KeyError):
        encode_distributions({"r_x": (0, 1)}, None, Env._MP_SLOT, Env._LP_SLOT)
    with pytest.raises(KeyError):
        encode_distributions(None, {"tau_decay": (0, 1)}, Env._MP_SLOT, Env._LP_SLOT)


def test_pole_pairs_and_repeated_slots_are_refused():
    with pytest.raises(ValueError, match="pole pairs"):
        encode_distributions({"p": (2, 4)}, None, Env._MP_SLOT, Env._LP_SLOT)
    with pytest.raises(ValueError):  # r_r is the rotor resistance slot r_e
        encode_distributions({"r_e": (1, 2), "r_r": (1, 2)}, None, Env._MP_SLOT, Env._LP_SLOT)


@pytest.mark.parametrize("name", ["l_m", "l_sigs", "l_sigr", "r_s", "r_r"])
def test_flux_limit_parameters_of_random_induction_initial_states_are_refused(name):
    with pytest.raises(NotImplementedError, match="DESIGN"):
        encode_distributions({name: (0.1, 0.2)}, None, Env._MP_SLOT, Env._LP_SLOT, flux_limits=True)
    encode_distributions({"j_rotor": (0.1, 0.2)}, None, Env._MP_SLOT, Env._LP_SLOT, flux_limits=True)


def test_env_refusals_before_any_device_call():
    with pytest.raises(TypeError):
        gem.make("Cont-CC-PMSM-v0").randomize_env_parameters(motor_parameter={"r_s": (0.1, 0.2)})
    with pytest.raises(ValueError):
        gem.make("Cont-CC-PMSM-v0", num_envs=4, layout="soa").randomize_env_parameters(motor_parameter={"r_s": (0.1, 0.2)})
    env = gem.make("Cont-CC-PMSM-v0", num_envs=4)
    with pytest.raises(KeyError):
        env.randomize_env_parameters(motor_parameter={"nope": (0.1, 0.2)})
    with pytest.raises(ValueError):
        env.randomize_env_parameters(motor_parameter={"p": (2, 4)})
    with pytest.raises(ValueError):
        env.randomize_env_parameters(load_parameter={"j_load": (1.0, 0.0)})
    assert env._sim is None  # nothing reached the device


def test_cabi_symbols_and_prototypes():
    assert "gemb200_set_param_randomization" in K.SYMBOLS and "gemb200_get_env_params" in K.SYMBOLS
    text = open(HEADER).read()
    assert "int gemb200_set_param_randomization(gemb200_handle* h, int32_t n, const int32_t* slot, const int32_t* kind, const double* lo, const double* hi);" in text
    assert "int gemb200_get_env_params(gemb200_handle* h, void* out, void* stream);" in text
    assert "GEMB200_DIST_UNIFORM = 0, GEMB200_DIST_LOG_UNIFORM = 1" in text
    lib = K.load_library()
    assert lib.gemb200_set_param_randomization.argtypes == [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    assert lib.gemb200_get_env_params.argtypes == [C.c_void_p, C.c_void_p, C.c_void_p]
    assert lib.gemb200_set_param_randomization(None, 0, None, None, None, None) == K.E_INVALID
