"""Gradients of rollout returns (env.rollout_return_grads, env.differentiable_returns, gemb200_query_return_grad_dims,
gemb200_rollout_return_grads) without a GPU: the dimensions and the refusal set over every registered env id and the refused configuration
fields, the Python argument checks, which must refuse bad arguments before anything is launched, the scalar refusal and the C-ABI
refusals.  The results are covered by tests/test_gpu_rollout_return_grads.py."""
import ctypes as C

import numpy as np
import pytest
import torch

import gym_electric_motor_b200 as gem
from gym_electric_motor_b200 import _cabi as K
from helpers import _env, no_launch  # noqa: F401

N = 6


def _dims(cfg):
    lib = K.load_library()
    d = [C.c_int32() for _ in range(4)]
    K.check(lib.gemb200_query_dims(C.byref(cfg), *[C.byref(x) for x in d]), "gemb200_query_dims")
    nx, nu, ww = C.c_int32(-1), C.c_int32(-1), C.c_int32(-1)
    rc = lib.gemb200_query_return_grad_dims(C.byref(cfg), C.byref(nx), C.byref(nu), C.byref(ww))
    return rc, (nx.value, nu.value, ww.value), (d[1].value, d[2].value), lib.gemb200_last_error()


def _expected_refusal(cfg):
    """the refusal list of the feature, written out here so that the supported scope cannot drift: everything the rollout Jacobians refuse
    (a dead time, the RC supply, dq actions on the FluxObserver angle, the SoA layout), finite converters, and a reward weight on an entry
    a state wrapper appends (DESIGN.md §7)."""
    return (cfg.dead_time_steps > 0 or cfg.supply_kind == K.SUPPLY_RC or cfg.action_dq in (2, 3) or cfg.layout == K.LAYOUT_SOA
            or cfg.finite)


def test_dims_and_refusals_of_every_env_id():
    ids = sorted(gem.env_ids())
    assert len(ids) == 54
    refused = supported = 0
    for env_id in ids:
        cfg = gem.make(env_id, num_envs=4, dtype="float32").build_config()
        for variant in ("default", "dead_time", "rc", "soa", "dq1", "dq2", "dq3"):
            c = type(cfg).from_buffer_copy(cfg)
            if variant == "dead_time":
                c.dead_time_steps = 1
            elif variant == "rc":
                c.supply_kind, c.supply_param[0], c.supply_param[1] = K.SUPPLY_RC, 1.0, 1e-3
            elif variant == "soa":
                c.layout = K.LAYOUT_SOA
            elif variant.startswith("dq"):
                dq = int(variant[2])
                motors = {1: (K.MOTOR_PMSM, K.MOTOR_SYNRM, K.MOTOR_EESM, K.MOTOR_SCIM), 2: (K.MOTOR_SCIM,), 3: (K.MOTOR_DFIM,)}[dq]
                if c.finite or c.motor_kind not in motors:
                    continue
                if dq > 1:  # dq actions on the observer angle: an induction motor with a FluxObserver
                    c.n_state_ops, c.sop_kind[0] = 1, K.SOP_FLUX_OBSERVER
                    for q in range(4):
                        c.sop_idx[0][q] = q + 2
                    c.sop_param[0][3] = 1.0
                c.action_dq = dq
            rc, (nx, nu, ww), (n_ode, n_act), msg = _dims(c)
            if _expected_refusal(c):
                assert rc == K.E_INVALID and b"DESIGN.md \xc2\xa77" in msg, (env_id, variant, rc, msg)
                refused += 1
            else:
                assert rc == 0, (env_id, variant, msg)
                assert (nx, nu) == (n_ode, n_act), (env_id, variant)
                assert ww == nx * (nx + nu) + nx + nu
                supported += 1
    assert supported >= 27 and refused >= 54 * 3


def test_workspace_words():
    for env_id, nx, nu in (("Cont-CC-PMSM-v0", 4, 3), ("Cont-CC-DFIM-v0", 6, 6), ("Cont-CC-PermExDc-v0", 2, 1)):
        rc, (x, u, ww), _, msg = _dims(gem.make(env_id, num_envs=4, dtype="float32").build_config())
        assert rc == 0, msg
        assert (x, u) == (nx, nu) and ww == nx * (nx + nu) + nx + nu
    assert _dims(gem.make("Cont-CC-PMSM-v0", num_envs=4, dtype="float32").build_config())[1][2] == 35  # 140 B per env-step in fp32
    assert _dims(gem.make("Cont-CC-DFIM-v0", num_envs=4, dtype="float32").build_config())[1][2] == 84


def test_reward_on_an_appended_entry_is_refused():
    """CosSin (with and without remove_angle) and FluxObserver entries: refused only when the reward weights them; a CosSin that removes
    the angle shifts the weighted base entries behind it, which stay supported"""
    cfg = gem.make("Cont-CC-SCIM-v0", num_envs=4, dtype="float32").build_config()
    n_state = 14
    for sop, width, remove in ((K.SOP_COS_SIN, 2, 0), (K.SOP_COS_SIN, 1, 1), (K.SOP_FLUX_OBSERVER, 2, 0)):
        c = type(cfg).from_buffer_copy(cfg)
        c.n_state_ops, c.sop_kind[0] = 1, sop
        if sop == K.SOP_COS_SIN:
            c.sop_idx[0][0], c.sop_idx[0][1] = 12, remove
        else:
            for q in range(4):
                c.sop_idx[0][q] = q + 2
            c.sop_param[0][3] = 1.0
        rc, _, _, msg = _dims(c)
        assert rc == 0, msg
        for j in range(n_state + width):
            d = type(c).from_buffer_copy(c)
            for q in range(n_state + width):
                d.reward_weight[q] = 0.0
            d.n_ref = 0
            d.reward_weight[j] = 1.0
            rc, _, _, msg = _dims(d)
            appended = j >= n_state + width - (2 if sop == K.SOP_COS_SIN else 2)
            assert (rc == K.E_INVALID) == appended, (sop, remove, j, msg)
            if appended:
                assert b"appends" in msg


def test_action_discount_feed_and_value_grad_checks(no_launch):
    env = _env()
    for acts in (torch.zeros(4, N, 2), torch.zeros(N, 3), torch.zeros(4, N, 3, dtype=torch.float64), torch.zeros(0, N, 3),
                 np.zeros((4, N, 3), dtype=np.float32), torch.zeros(4, 3, N).transpose(1, 2)):
        with pytest.raises(ValueError):
            env.rollout_return_grads(acts)
        with pytest.raises(ValueError):
            env.differentiable_returns(acts)
    acts = torch.zeros(4, N, 3)
    for g in (-0.1, 1.5, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            env.rollout_return_grads(acts, g)
    for refs in (torch.zeros(4, N, 3), torch.zeros(5, N, 2), torch.zeros(4, N, 2, dtype=torch.float64), np.zeros((4, N, 2), dtype=np.float32)):
        with pytest.raises(ValueError):
            env.rollout_return_grads(acts, references=refs)
    for vg in (torch.zeros(N, 3), torch.zeros(N, 4, dtype=torch.float64), torch.zeros(N + 1, 4), np.zeros((N, 4), dtype=np.float32),
               torch.zeros(4, N).t()):
        with pytest.raises(ValueError):
            env.rollout_return_grads(acts, value_grad=vg)
    with pytest.raises(AssertionError, match="was called"):  # good arguments get as far as the launch
        env.rollout_return_grads(acts, 0.9, references=torch.zeros(4, N, 2), value_grad=torch.zeros(N, 4))


def test_refused_configuration_raises_not_implemented(no_launch):
    with pytest.raises(NotImplementedError, match="DESIGN.md"):
        _env(layout="soa").rollout_return_grads(torch.zeros(3, 3, N))
    env = gem.make("Finite-CC-PMSM-v0", num_envs=N, dtype="float32")
    with pytest.raises(NotImplementedError, match="finite"):
        env.rollout_return_grads(torch.zeros(3, N, 1, dtype=torch.int32))


def test_scalar_env_refuses(no_launch):
    env = gem.make("Cont-CC-PMSM-v0")
    with pytest.raises(TypeError):
        env.rollout_return_grads(torch.zeros(2, 1, 3))
    with pytest.raises(TypeError):
        env.differentiable_returns(torch.zeros(2, 1, 3))


def test_cabi_symbol_and_refusals():
    assert {"gemb200_query_return_grad_dims", "gemb200_rollout_return_grads"} <= set(K.SYMBOLS)
    lib = K.load_library()
    assert lib.gemb200_version() == K.ABI_VERSION == 10  # new entry points, no new ABI version
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    rc = lib.gemb200_rollout_return_grads(None, p, None, 1, 1.0, None, p, 256, p, None, p, p, None, None, None)
    assert rc == K.E_INVALID and b"handle is NULL" in lib.gemb200_last_error()
    assert lib.gemb200_query_return_grad_dims(None, None, None, None) == K.E_INVALID
    c = gem.make("Cont-CC-PMSM-v0", num_envs=4, dtype="float32", layout="soa").build_config()
    assert lib.gemb200_query_return_grad_dims(C.byref(c), None, None, None) == K.E_INVALID
    assert b"SoA" in lib.gemb200_last_error()
