"""Kernel vs oracle for every configuration of the user-kwargs matrix (tests/agent_surface/kwargs_matrix_harness.py: 95 kwarg combinations +
the 54 default ids), built through the HOST API (`gem.make(**kwargs)` -> `env.build_config()`), float64 build, 6 envs, 12 steps with fixed
actions: states, rewards, terminations, next references."""
import numpy as np
import pytest

from gym_electric_motor_b200 import _cabi as K
from helpers import WEAK_DQ_PAIRS, fold_weak_dq

pytestmark = pytest.mark.gpu


def _cases():
    import os
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "agent_surface"))
    import kwargs_matrix_harness as h

    return h.CASES, h.PRELUDE


def sim_n_ode(cfg):
    d = [K.C.c_int32() for _ in range(4)]
    K.check(K.load_library().gemb200_query_dims(K.C.byref(cfg), *[K.C.byref(x) for x in d]), "query_dims")
    return d[1].value


CASES, PRELUDE = _cases()
REFUSED = ("synrm_dq",)  # refused on the host, as by the reference (DqToAbcActionProcessor has no SynRM entry)


@pytest.mark.parametrize("case", sorted(c for c in CASES if c not in REFUSED and not c.startswith("err_")))
def test_device_matches_oracle_for_host_built_config(oracle_lib, case):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.vector_sim import VectorSim

    ns = {"gem": gem}
    exec(PRELUDE, ns)
    env = eval(CASES[case], ns)
    cfg = env.build_config()
    n = 6
    cfg.n_envs, cfg.dtype, cfg.seed, cfg.autoreset = n, K.F64, 5, K.AUTORESET_SAME_STEP
    if cfg.finite and cfg.interlocking_time > 0 and not cfg.init_random:
        # a leg in its interlock (freewheeling) state outputs by the SIGN of its current; from the exactly-zero initial state that sign is
        # round-off noise — in the reference as well (tests/test_gpu_parity.py: BATCH_CASES note) — so start from non-zero currents
        for j, v in enumerate([0.9, -0.6, 0.02, 0.03][: max(0, sim_n_ode(cfg) - 2)]):
            cfg.init_ode[1 + j] = v
    ora, sim = oracle_lib.Oracle(cfg), VectorSim(cfg)
    o_obs, o_ref = ora.reset()
    d_obs, d_ref = sim.reset()
    assert np.abs(d_obs.double().cpu().numpy() - o_obs).max() < 1e-9 and np.abs(d_ref.double().cpu().numpy() - o_ref).max() < 1e-9
    rng = np.random.default_rng(3)
    sp = env.action_space
    # Induction motors: the dq columns are expressed in the rotor-flux frame, whose angle is decided by round-off while the flux is
    # still (numerically) zero after the reset — in the reference itself (DESIGN.md finding 3; same treatment as
    # test_gpu_parity.test_device_reproduces_reference_trajectory): there the dq pairs are compared through their magnitude and the
    # reward (which sees i_sd / i_sq in current-control envs) is not compared.
    dq_pairs = WEAK_DQ_PAIRS.get(cfg.motor_kind, ())
    for k in range(12):
        if hasattr(sp, "low"):
            a = rng.uniform(sp.low, sp.high, size=(n, len(sp.low)))
        elif hasattr(sp, "nvec"):
            a = np.stack([rng.integers(0, int(m), size=n) for m in sp.nvec], axis=1).astype(np.int32)
        else:
            a = rng.integers(0, sp.n, size=(n, 1)).astype(np.int32)
        psi = ora.get_ode_state()[:, 3:5] if dq_pairs else None
        o = ora.step(a)
        d = sim.step(a)
        tol = 1e-8
        d_obs, o_obs = d[0].double().cpu().numpy().copy(), o[0].copy()
        weak = np.zeros(n, dtype=bool)
        if dq_pairs:
            weak = np.hypot(psi[:, 0], psi[:, 1]) < 1e-3
            fold_weak_dq(dq_pairs, weak, d_obs, o_obs)
        assert np.abs(d_obs - o_obs).max() < tol, (case, k)
        assert np.abs(d[1].double().cpu().numpy() - o[1]).max() < tol, (case, k)
        assert np.abs(d[2].double().cpu().numpy() - o[2])[~weak].max(initial=0.0) < 10 * tol, (case, k)
        assert np.array_equal(d[3].cpu().numpy().astype(np.uint8)[~weak], o[3][~weak]), (case, k)
    sim.close()
