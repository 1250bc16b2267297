"""Discounted returns of a fused rollout (env.rollout_returns, VectorSim.rollout_returns_into, gemb200_rollout_returns) without a GPU:
argument checks, which must refuse bad actions, a bad discount or a bad feed before anything is launched, the scalar refusal, the C-ABI
symbol and its refusals.  The handle class is the launch-refusing stand-in of tests/test_reference_feed.py; the results are covered by
tests/test_gpu_rollout_returns.py."""
import ctypes as C

import numpy as np
import pytest
import torch

import gym_electric_motor_b200 as gem
from gym_electric_motor_b200 import _cabi as K
from helpers import _env, no_launch  # noqa: F401

N = 6


def test_action_checks(no_launch):
    env = _env()
    bad = {
        "shape": torch.zeros(4, N, 2),
        "layout": torch.zeros(4, 3, N),          # the SoA shape on an AoS env
        "2-D": torch.zeros(N, 3),
        "dtype": torch.zeros(4, N, 3, dtype=torch.float64),
        "device": torch.zeros(4, N, 3, device="meta"),
        "contiguity": torch.zeros(4, 3, N).transpose(1, 2),
        "numpy": np.zeros((4, N, 3), dtype=np.float32),
        "K = 0": torch.zeros(0, N, 3),
    }
    for what, acts in bad.items():
        with pytest.raises(ValueError):
            env.rollout_returns(acts)
    with pytest.raises(AssertionError, match="was called"):  # good actions get as far as the launch
        env.rollout_returns(torch.zeros(4, N, 3))


def test_soa_action_shape(no_launch):
    env = _env(layout="soa")
    with pytest.raises(ValueError):
        env.rollout_returns(torch.zeros(3, N, 3))
    with pytest.raises(AssertionError, match="was called"):
        env.rollout_returns(torch.zeros(3, 3, N))


def test_finite_actions_are_int32(no_launch):
    env = gem.make("Finite-CC-PMSM-v0", num_envs=N, dtype="float32")
    with pytest.raises(ValueError):
        env.rollout_returns(torch.zeros(2, N, 1))  # float switching states
    with pytest.raises(AssertionError, match="was called"):
        env.rollout_returns(torch.zeros(2, N, 1, dtype=torch.int32))


@pytest.mark.parametrize("discount", [float("nan"), -0.1, 1.5, float("inf"), -float("inf")])
def test_discount_checks(no_launch, discount):
    env = _env()
    acts = torch.zeros(4, N, 3)
    with pytest.raises(ValueError, match="discount"):
        env.rollout_returns(acts, discount=discount)
    with pytest.raises(ValueError, match="discount"):
        env.sim.rollout_returns_into(acts, 4, discount, torch.zeros(N))


@pytest.mark.parametrize("discount", [0.0, 0.9, 1.0, 1])
def test_good_discounts_reach_the_launch(no_launch, discount):
    env = _env()
    with pytest.raises(AssertionError, match="was called"):
        env.rollout_returns(torch.zeros(4, N, 3), discount=discount)


def test_feed_checks(no_launch):
    env = _env()
    acts = torch.zeros(4, N, 3)
    for refs in (torch.zeros(4, N, 3), torch.zeros(4, 2, N), torch.zeros(5, N, 2), torch.zeros(4, N, 2, dtype=torch.float64),
                 torch.zeros(4, N, 2, device="meta"), torch.zeros(4, 2, N).transpose(1, 2), np.zeros((4, N, 2), dtype=np.float32)):
        with pytest.raises(ValueError):
            env.rollout_returns(acts, references=refs)
        with pytest.raises(ValueError):
            env.sim.rollout_returns_into(acts, 4, 1.0, torch.zeros(N), references=refs)
    with pytest.raises(AssertionError, match="was called"):
        env.rollout_returns(acts, discount=0.5, references=torch.zeros(4, N, 2))


def test_feed_needs_reference_slots(no_launch):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=N, reference_generator=gem.reference_generators.ZeroReferenceGenerator(), dtype="float32")
    with pytest.raises(ValueError, match="n_ref == 0"):
        env.rollout_returns(torch.zeros(2, N, 3), references=torch.zeros(2, N, 0))


def test_scalar_env_refuses(no_launch):
    env = gem.make("Cont-CC-PMSM-v0")
    with pytest.raises(TypeError):
        env.rollout_returns(torch.zeros(2, 1, 3))


def test_cabi_symbol_and_refusals():
    assert "gemb200_rollout_returns" in K.SYMBOLS
    lib = K.load_library()
    assert lib.gemb200_rollout_returns.argtypes is not None
    assert lib.gemb200_version() == K.ABI_VERSION == 10  # a new entry point, no new ABI version
    buf = (C.c_float * 8)()
    p = C.cast(buf, C.c_void_p)
    i32 = (C.c_int32 * 8)()
    rc = lib.gemb200_rollout_returns(None, p, None, 1, 1.0, p, C.cast(i32, C.c_void_p), None, None, None)
    assert rc == K.E_INVALID and b"handle is NULL" in lib.gemb200_last_error()
    # the arguments below are refused before the handle is read, so a stand-in pointer is enough
    fake = C.cast((C.c_uint8 * 64)(), C.c_void_p)
    rc = lib.gemb200_rollout_returns(fake, p, None, 1, 1.0, None, None, None, None, None)
    assert rc == K.E_INVALID and b"return_out is NULL" in lib.gemb200_last_error()
    for g in (float("nan"), -0.5, 2.0, float("inf")):
        rc = lib.gemb200_rollout_returns(fake, p, None, 1, g, p, None, None, None, None)
        assert rc == K.E_INVALID and b"discount" in lib.gemb200_last_error()
    rc = lib.gemb200_rollout_returns(fake, p, None, 0, 1.0, p, None, None, None, None)
    assert rc == K.E_INVALID and b"n_steps" in lib.gemb200_last_error()
