"""Reference feed (env.step(action, reference=...), env.rollout(..., references=...), capture_steps(..., references=...)) without a GPU:
argument checks, which must refuse a bad feed before anything is launched, the C-ABI symbol and its NULL-handle refusal.  The handle
class is replaced by a stand-in that computes dimensions with the real library but fails on any launch; the results of a feed are
covered by tests/test_gpu_reference_feed.py."""
import ctypes as C

import numpy as np
import pytest
import torch

import gym_electric_motor_b200 as gem
from gym_electric_motor_b200 import _cabi as K
from helpers import _env, no_launch  # noqa: F401

N = 6  # the envs of helpers._env


def test_rollout_feed_argument_checks(no_launch):
    env = _env()
    acts = torch.zeros(4, N, 3)
    good = torch.zeros(4, N, 2)
    bad = {
        "shape": torch.zeros(4, N, 3),
        "layout": torch.zeros(4, 2, N),          # the SoA shape on an AoS env
        "K": torch.zeros(5, N, 2),
        "dtype": torch.zeros(4, N, 2, dtype=torch.float64),
        "device": torch.zeros(4, N, 2, device="meta"),
        "contiguity": torch.zeros(4, 2, N).transpose(1, 2),
        "numpy": np.zeros((4, N, 2), dtype=np.float32),
    }
    for what, refs in bad.items():
        with pytest.raises(ValueError):
            env.rollout(acts, references=refs)
        with pytest.raises(ValueError):
            env.sim.rollout_into(acts, 4, 1, None, None, None, None, references=refs)
    with pytest.raises(AssertionError, match="was called"):  # a good feed gets as far as the launch
        env.rollout(acts, references=good)


def test_step_feed_argument_checks(no_launch):
    env = _env()
    a = torch.zeros(N, 3)
    for refs in (torch.zeros(N, 3), torch.zeros(2, N), torch.zeros(N, 2, dtype=torch.float64), torch.zeros(1, N, 2), [[0.0, 0.0]] * N):
        with pytest.raises(ValueError):
            env.step(a, reference=refs)
    with pytest.raises(AssertionError, match="was called"):
        env.step(a, reference=torch.zeros(N, 2))


def test_soa_feed_shape(no_launch):
    env = _env(layout="soa")
    with pytest.raises(ValueError):
        env.rollout(torch.zeros(3, 3, N), references=torch.zeros(3, N, 2))
    with pytest.raises(AssertionError, match="was called"):
        env.rollout(torch.zeros(3, 3, N), references=torch.zeros(3, 2, N))


def test_capture_feed_argument_checks(no_launch):
    env = _env()
    policy = lambda s, r: torch.zeros(N, 3)  # noqa: E731
    for refs in (torch.zeros(4, N, 2), torch.zeros(3, N, 2, dtype=torch.float64), torch.zeros(3, 2, N)):
        with pytest.raises(ValueError):  # before the warm-up step, which would launch
            env.capture_steps(policy, 3, references=refs)


def test_feed_needs_reference_slots(no_launch):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=N, reference_generator=gem.reference_generators.ZeroReferenceGenerator(), dtype="float32")
    assert env.sim.n_ref == 0
    with pytest.raises(ValueError, match="n_ref == 0"):
        env.rollout(torch.zeros(2, N, 3), references=torch.zeros(2, N, 0))
    with pytest.raises(ValueError, match="n_ref == 0"):
        env.step(torch.zeros(N, 3), reference=torch.zeros(N, 0))


def test_scalar_env_refuses_a_feed(no_launch):
    env = gem.make("Cont-CC-PMSM-v0")
    with pytest.raises(TypeError):
        env.step(np.zeros(3), reference=torch.zeros(1, 2))
    with pytest.raises(TypeError):
        env.rollout(torch.zeros(2, 1, 3), references=torch.zeros(2, 1, 2))


def test_vector_facade_passes_the_feed(monkeypatch):
    venv = gem.vector.make_vec("Cont-CC-PMSM-v0", num_envs=N)
    seen = []
    monkeypatch.setattr(venv.env, "step", lambda *a: seen.append(a) or ((torch.zeros(N, 14), torch.zeros(N, 2)), torch.zeros(N),
                                                                        torch.zeros(N, dtype=torch.bool), False, {}))
    r = torch.zeros(N, 2)
    venv.step(torch.zeros(N, 3), reference=r)
    venv.step(torch.zeros(N, 3))
    assert seen[0][1] is r and len(seen[1]) == 1  # no feed: the env's step is called exactly as before


def test_cabi_symbol_and_null_handle():
    assert "gemb200_rollout_record_ref" in K.SYMBOLS
    lib = K.load_library()
    assert lib.gemb200_rollout_record_ref.argtypes is not None
    buf = (C.c_float * 8)()
    rc = lib.gemb200_rollout_record_ref(None, C.cast(buf, C.c_void_p), C.cast(buf, C.c_void_p), 1, 0, None, None, None, None, None)
    assert rc == K.E_INVALID
    assert b"NULL" in lib.gemb200_last_error()
