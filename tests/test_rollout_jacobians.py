"""Rollout Jacobians (env.rollout_jacobians, VectorSim.rollout_jacobians_into, gemb200_query_jacobian_dims, gemb200_rollout_jacobians)
without a GPU: the dimensions and the refusal set over every registered env id and the refused configuration fields, the Python argument
checks, which must refuse bad actions or a bad feed before anything is launched, the scalar refusal and the C-ABI refusals.  The results
are covered by tests/test_gpu_rollout_jacobians.py."""
import ctypes as C

import numpy as np
import pytest
import torch

import gym_electric_motor_b200 as gem
from gym_electric_motor_b200 import _cabi as K
from test_reference_feed import _env, no_launch  # noqa: F401

N = 6


def _registered_ids():
    return sorted(gem.env_ids())


def _dims(cfg):
    lib = K.load_library()
    d = [C.c_int32() for _ in range(4)]
    K.check(lib.gemb200_query_dims(C.byref(cfg), *[C.byref(x) for x in d]), "gemb200_query_dims")
    nx, nu = C.c_int32(-1), C.c_int32(-1)
    rc = lib.gemb200_query_jacobian_dims(C.byref(cfg), C.byref(nx), C.byref(nu))
    return rc, (nx.value, nu.value), (d[1].value, d[2].value), lib.gemb200_last_error()


def _expected_refusal(cfg):
    """the refusal list of the feature, written out here so that the supported scope cannot drift: a dead time, the RC supply, dq actions on
    the FluxObserver angle, the SoA layout (DESIGN.md §7).  Everything else is supported, finite converters with interlocking time included."""
    return cfg.dead_time_steps > 0 or cfg.supply_kind == K.SUPPLY_RC or cfg.action_dq in (2, 3) or cfg.layout == K.LAYOUT_SOA


def test_dims_and_refusals_of_every_env_id():
    ids = _registered_ids()
    assert len(ids) == 54
    refused = supported = 0
    for env_id in ids:
        cfg = gem.make(env_id, num_envs=4, dtype="float32").build_config()
        for variant in ("default", "dead_time", "rc", "soa", "dq"):
            c = type(cfg).from_buffer_copy(cfg)
            if variant == "dead_time":
                c.dead_time_steps = 1
            elif variant == "rc":
                c.supply_kind, c.supply_param[0], c.supply_param[1] = K.SUPPLY_RC, 1.0, 1e-3
            elif variant == "soa":
                c.layout = K.LAYOUT_SOA
            elif variant == "dq":
                if c.finite or c.motor_kind not in (K.MOTOR_PMSM, K.MOTOR_SYNRM, K.MOTOR_EESM, K.MOTOR_SCIM):
                    continue
                c.action_dq = 1
            rc, (nx, nu), (n_ode, n_act), msg = _dims(c)
            if _expected_refusal(c):
                assert rc == K.E_INVALID and b"DESIGN.md \xc2\xa77" in msg, (env_id, variant, rc, msg)
                refused += 1
            else:
                assert rc == 0, (env_id, variant, msg)
                assert (nx, nu) == (n_ode, 0 if c.finite else n_act), (env_id, variant)
                supported += 1
    assert refused == 3 * 54 and supported >= 54


def test_finite_converters_with_interlocking_time_are_supported():
    """one or two interlocking times (two- and three-segment steps), in every finite family"""
    for env_id in ("Finite-CC-PMSM-v0", "Finite-CC-DFIM-v0", "Finite-CC-SCIM-v0", "Finite-CC-PermExDc-v0", "Finite-CC-ExtExDc-v0"):
        cfg = gem.make(env_id, num_envs=4, dtype="float32").build_config()
        for til, til1 in ((0.0, -1.0), (1e-6, -1.0), (1e-6, 3e-6)):
            c = type(cfg).from_buffer_copy(cfg)
            c.interlocking_time, c.interlocking_time1 = til, til1
            rc, (nx, nu), (n_ode, _), msg = _dims(c)
            assert rc == 0, (env_id, til, til1, msg)
            assert (nx, nu) == (n_ode, 0)


def test_observer_dq_actions_are_refused():
    """SCIM with a FluxObserver: abc and field-angle dq actions are supported, dq actions on the observer's angle are refused"""
    cfg = gem.make("Cont-CC-SCIM-v0", num_envs=4, dtype="float32").build_config()
    cfg.n_state_ops, cfg.sop_kind[0] = 1, K.SOP_FLUX_OBSERVER
    for q in range(4):
        cfg.sop_idx[0][q] = q + 2
    cfg.sop_param[0][3] = 1.0
    for dq, ok in ((0, True), (1, True), (2, False)):
        c = type(cfg).from_buffer_copy(cfg)
        c.action_dq = dq
        rc, (nx, nu), _, msg = _dims(c)
        assert (rc == 0) == ok, (dq, msg)
        if ok:
            assert (nx, nu) == (6, 3 if dq == 0 else 2)
        else:
            assert b"observer" in msg


def test_action_and_feed_checks(no_launch):
    env = _env()
    for acts in (torch.zeros(4, N, 2), torch.zeros(N, 3), torch.zeros(4, N, 3, dtype=torch.float64), torch.zeros(0, N, 3),
                 np.zeros((4, N, 3), dtype=np.float32), torch.zeros(4, 3, N).transpose(1, 2)):
        with pytest.raises(ValueError):
            env.rollout_jacobians(acts)
    acts = torch.zeros(4, N, 3)
    for refs in (torch.zeros(4, N, 3), torch.zeros(5, N, 2), torch.zeros(4, N, 2, dtype=torch.float64), np.zeros((4, N, 2), dtype=np.float32)):
        with pytest.raises(ValueError):
            env.rollout_jacobians(acts, references=refs)
        with pytest.raises(ValueError):
            env.sim.rollout_jacobians_into(acts, 4, torch.zeros(4, N, 4, 4), references=refs)
    with pytest.raises(AssertionError, match="was called"):  # good arguments get as far as the launch
        env.rollout_jacobians(acts, references=torch.zeros(4, N, 2))


def test_refused_configuration_raises_not_implemented(no_launch):
    env = _env(layout="soa")
    with pytest.raises(NotImplementedError, match="DESIGN.md"):
        env.rollout_jacobians(torch.zeros(3, 3, N))


def test_scalar_env_refuses(no_launch):
    env = gem.make("Cont-CC-PMSM-v0")
    with pytest.raises(TypeError):
        env.rollout_jacobians(torch.zeros(2, 1, 3))


def test_calc_jacobian_is_accepted_and_ignored():
    a = gem.make("Cont-CC-PMSM-v0", num_envs=4, dtype="float32", calc_jacobian=False).build_config()
    b = gem.make("Cont-CC-PMSM-v0", num_envs=4, dtype="float32", calc_jacobian=True).build_config()
    assert bytes(a) == bytes(b)


def test_cabi_symbol_and_refusals():
    assert {"gemb200_query_jacobian_dims", "gemb200_rollout_jacobians"} <= set(K.SYMBOLS)
    lib = K.load_library()
    assert lib.gemb200_version() == K.ABI_VERSION == 10  # new entry points, no new ABI version
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    rc = lib.gemb200_rollout_jacobians(None, p, None, 1, p, None, None, None, None, None, None)
    assert rc == K.E_INVALID and b"handle is NULL" in lib.gemb200_last_error()
    assert lib.gemb200_query_jacobian_dims(None, None, None) == K.E_INVALID


def test_reference_jacobian_fixture_agrees_with_its_own_system_equation():
    """tests/golden/jacobians/system_jacobians.npz (tests/golden/make_system_jacobians.py, recorded from the unmodified reference): for every motor under a
    constant-speed and a polynomial static load, SCMLSystem._system_jacobian equals central differences of SCMLSystem._system_equation at
    the recorded points (column-relative, the differences' own accuracy).  The device Jacobians are checked against these matrices on the
    GPU (tests/test_gpu_rollout_jacobians.py)."""
    import os

    d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jacobians", "system_jacobians.npz"))
    cases = sorted({k.split("/")[0] for k in d.files})
    assert len(cases) == 18
    for c in cases:
        jac, fd, x = d[c + "/jac"], d[c + "/fd"], d[c + "/x"]
        assert jac.shape == fd.shape == (x.shape[0], x.shape[1], x.shape[1]) and x.shape[0] >= 6
        scale = np.maximum(np.abs(fd).max(axis=1, keepdims=True), 1e-12)
        assert (np.abs(jac - fd) / scale).max() < 1e-4, c
