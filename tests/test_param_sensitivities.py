"""Parameter sensitivities (env.rollout_param_sensitivities, VectorSim.rollout_param_sens, gemb200_query_param_sens_dims,
gemb200_coef_tangents, gemb200_rollout_param_sens) without a GPU: the dimensions and refusals of the query, the coefficient tangents of
every motor kind and accepted slot against central differences of the model derivation (written out here from the reference's
*_update_model methods) and against closed forms, the name-to-slot mapping and the Python argument checks, which must refuse bad input
before anything is launched.  The launch itself is covered by tests/test_gpu_param_sensitivities.py."""
import ctypes as C

import numpy as np
import pytest
import torch

import gym_electric_motor_b200 as gem
from gym_electric_motor_b200 import _cabi as K
from helpers import NoLaunchSim, no_launch  # noqa: F401

N = 6
MOTOR_IDS = {K.MOTOR_PERMEX_DC: "Cont-CC-PermExDc-v0", K.MOTOR_SERIES_DC: "Cont-CC-SeriesDc-v0", K.MOTOR_SHUNT_DC: "Cont-CC-ShuntDc-v0",
             K.MOTOR_EXTEX_DC: "Cont-CC-ExtExDc-v0", K.MOTOR_PMSM: "Cont-CC-PMSM-v0", K.MOTOR_SYNRM: "Cont-CC-SynRM-v0",
             K.MOTOR_EESM: "Cont-CC-EESM-v0", K.MOTOR_SCIM: "Cont-CC-SCIM-v0", K.MOTOR_DFIM: "Cont-CC-DFIM-v0"}
LOAD_SLOTS = [K.MAX_MOTOR_PARAM + s for s in (K.LP_A, K.LP_B, K.LP_C, K.LP_J_LOAD)]
ACCEPTED = [s for s in range(K.MAX_MOTOR_PARAM) if s not in (K.MP_P, K.MP_K)] + LOAD_SLOTS


def _cfg(motor_kind, poly=True):
    kw = {}
    if poly:
        kw["load"] = gem.physical_systems.PolynomialStaticLoad(load_parameter=dict(a=0.01, b=0.02, c=1e-4, j_load=1e-3))
    return gem.make(MOTOR_IDS[motor_kind], num_envs=N, dtype="float64", **kw).build_config()


def _query(cfg, slots):
    lib = K.load_library()
    arr = (C.c_int32 * max(len(slots), 1))(*slots)
    nx = C.c_int32(-1)
    rc = lib.gemb200_query_param_sens_dims(C.byref(cfg), len(slots), arr, C.byref(nx))
    return rc, nx.value, lib.gemb200_last_error()


def _tangents(cfg, slots, prm=None):
    lib = K.load_library()
    arr = (C.c_int32 * len(slots))(*slots)
    out = np.full((len(slots), 30), np.nan)
    mp = lp = None
    if prm is not None:
        mp = np.ascontiguousarray(prm[:K.MAX_MOTOR_PARAM])
        lp = np.ascontiguousarray(prm[K.MAX_MOTOR_PARAM:])
    K.check(lib.gemb200_coef_tangents(C.byref(cfg), None if mp is None else mp.ctypes.data, None if lp is None else lp.ctypes.data, len(slots), arr,
                                      out.ctypes.data), "gemb200_coef_tangents")
    return out


def _derive(kind, prm):
    """the coefficient block [30] of a parameter row: the reference's *_update_model constants in the library's layout (gemb200_params.h,
    Coef), written out independently of gemb200_model.h"""
    mp, lp = prm[:K.MAX_MOTOR_PARAM], prm[K.MAX_MOTOR_PARAM:]
    c, tq = np.zeros(20), np.zeros(4)
    p, r_s, l_d, l_q = mp[K.MP_P], mp[K.MP_R_S], mp[K.MP_L_D], mp[K.MP_L_Q]
    if kind == K.MOTOR_PERMEX_DC:
        l_a = mp[K.MP_L_A]
        c[:4] = [-mp[K.MP_PSI_E] / l_a, -mp[K.MP_R_A] / l_a, 0, 1 / l_a]
        tq[0] = mp[K.MP_PSI_E]
    elif kind == K.MOTOR_SERIES_DC:
        l = mp[K.MP_L_A] + mp[K.MP_L_E]
        c[:4] = [0, -(mp[K.MP_R_A] + mp[K.MP_R_E]) / l, -mp[K.MP_L_E_PRIME] / l, 1 / l]
        tq[1] = mp[K.MP_L_E_PRIME]
    elif kind in (K.MOTOR_SHUNT_DC, K.MOTOR_EXTEX_DC):
        l_a, l_e = mp[K.MP_L_A], mp[K.MP_L_E]
        c[:5] = [-mp[K.MP_R_A] / l_a, -mp[K.MP_L_E_PRIME] / l_a, 1 / l_a, -mp[K.MP_R_E] / l_e, 1 / l_e]
        tq[0] = mp[K.MP_L_E_PRIME]
    elif kind in (K.MOTOR_PMSM, K.MOTOR_SYNRM):
        psi = mp[K.MP_PSI_P] if kind == K.MOTOR_PMSM else 0.0
        c[:7] = [-r_s / l_d, 1 / l_d, l_q * p / l_d, -psi * p / l_q, -r_s / l_q, 1 / l_q, -l_d * p / l_q]
        tq[:2] = [1.5 * p * psi, 1.5 * p * (l_d - l_q)]
    elif kind == K.MOTOR_EESM:
        k = mp[K.MP_K]
        r_E, l_M, l_E = k * k * 1.5 * mp[K.MP_R_E], k * 1.5 * mp[K.MP_L_M], k * k * 1.5 * mp[K.MP_L_E]
        ik = 2 / 3 / k
        sg = 1 - l_M * l_M / (l_d * l_E)
        s2 = l_E * ik
        c[:14] = [-r_s / sg / l_d, l_M * r_E / (sg * l_E) * ik / l_d, 1 / sg / l_d, -l_M * k / (sg * l_E) / l_d, l_q * p / sg / l_d,
                  -r_s / l_q, 1 / l_q, -l_d * p / l_q, -p * l_M * ik / l_q,
                  l_M * r_s / (sg * l_d) / s2, -r_E / sg * ik / s2, -l_M / (sg * l_d) / s2, k / sg / s2, -p * l_M * l_q / (sg * l_d) / s2]
        tq[:2] = [1.5 * p * l_M * ik, 1.5 * p * (l_d - l_q)]
    else:
        l_m, r_r = mp[K.MP_L_M], mp[K.MP_R_E]
        l_s, l_r = l_m + mp[K.MP_L_SIGS], l_m + mp[K.MP_L_SIGR]
        sg = (l_s * l_r - l_m ** 2) / (l_s * l_r)
        tau_r, tau_sig = l_r / r_r, sg * l_s / (r_s + r_r * l_m ** 2 / l_r ** 2)
        c[:10] = [-1 / tau_sig, l_m * r_r / (sg * l_s * l_r ** 2), l_m * p / (sg * l_r * l_s), 1 / (sg * l_s), l_m / tau_r, -1 / tau_r, p,
                  -l_m / (sg * l_r * l_s), 1 / l_r, l_m / l_r]
        tq[0] = 1.5 * p * l_m / l_r
    j = lp[K.LP_J_LOAD] + mp[K.MP_J_ROTOR]
    mech = [lp[K.LP_A], lp[K.LP_B], lp[K.LP_C], 1 / j, lp[K.LP_A] / j * lp[K.LP_TAU_DECAY], j / lp[K.LP_TAU_DECAY]]
    return np.concatenate([c, tq, mech])


def _row(cfg):
    return np.array(list(cfg.motor_param) + list(cfg.load_param), dtype=np.float64)


def test_dims_and_refusals():
    for kind in MOTOR_IDS:
        cfg = _cfg(kind)
        rc, nx, msg = _query(cfg, [K.MP_R_S])
        assert rc == 0, (kind, msg)
        d = [C.c_int32() for _ in range(4)]
        K.check(K.load_library().gemb200_query_dims(C.byref(cfg), *[C.byref(x) for x in d]), "gemb200_query_dims")
        assert nx == d[1].value, kind
        assert _query(cfg, ACCEPTED[:12])[0] == 0 and _query(cfg, ACCEPTED[-12:])[0] == 0
        for slots in ([], ACCEPTED[:13], [K.MP_P], [K.MP_K], [K.MP_R_S, K.MP_R_S], [K.MAX_MOTOR_PARAM + K.LP_TAU_DECAY],
                      [K.MAX_MOTOR_PARAM + K.LP_TAU_LOAD], [-1], [K.MAX_MOTOR_PARAM + 8]):
            rc, _, msg = _query(cfg, slots)
            assert rc == K.E_INVALID and b"DESIGN.md \xc2\xa77" in msg, (kind, slots, msg)
    cfg = _cfg(K.MOTOR_PMSM)
    for field, value in (("dead_time_steps", 1), ("layout", K.LAYOUT_SOA)):  # dq actions on the observer angle: jacobian_refusal, shared
        c = type(cfg).from_buffer_copy(cfg)
        setattr(c, field, value)
        rc, _, msg = _query(c, [K.MP_R_S])
        assert rc == K.E_INVALID and b"DESIGN.md \xc2\xa77" in msg, (field, msg)
    c = type(cfg).from_buffer_copy(cfg)
    c.supply_kind, c.supply_param[0], c.supply_param[1] = K.SUPPLY_RC, 1.0, 1e-3
    assert _query(c, [K.MP_R_S])[0] == K.E_INVALID
    finite = gem.make("Finite-CC-PMSM-v0", num_envs=N, dtype="float64").build_config()
    assert _query(finite, [K.MP_R_S])[:2] == (0, 4)  # finite converters are supported


@pytest.mark.parametrize("kind", list(MOTOR_IDS))
def test_coef_tangents_against_central_differences(kind):
    cfg = _cfg(kind)
    prm = _row(cfg)
    t = np.concatenate([_tangents(cfg, ACCEPTED[:12]), _tangents(cfg, ACCEPTED[12:])])
    assert np.array_equal(t[:12], _tangents(cfg, ACCEPTED[:12], prm))  # NULL rows: the configuration's
    assert np.array_equal(t[3], _tangents(cfg, [ACCEPTED[3]])[0])  # a column does not depend on the others
    for a, slot in enumerate(ACCEPTED):
        h = 1e-6 * (abs(prm[slot]) if prm[slot] != 0 else 1.0)
        up, dn = prm.copy(), prm.copy()
        up[slot] += h
        dn[slot] -= h
        fd = (_derive(kind, up) - _derive(kind, dn)) / (2 * h)
        scale = max(np.abs(fd).max(), np.abs(t[a]).max(), 1e-300)
        assert np.abs(t[a] - fd).max() <= 1e-7 * scale, (kind, slot, np.abs(t[a] - fd).max() / scale)
        used = _derive(kind, up) != _derive(kind, dn)
        assert np.all(t[a][~used] == 0), (kind, slot, "exact zeros where the slot does not enter", np.nonzero(t[a][~used]))


def test_coef_tangents_closed_forms_pmsm():
    cfg = _cfg(K.MOTOR_PMSM)
    mp = np.array(list(cfg.motor_param))
    lp = np.array(list(cfg.load_param))
    p, r_s, l_d, l_q, psi = mp[K.MP_P], mp[K.MP_R_S], mp[K.MP_L_D], mp[K.MP_L_Q], mp[K.MP_PSI_P]
    slots = [K.MP_R_S, K.MP_L_D, K.MP_L_Q, K.MP_PSI_P, K.MP_J_ROTOR, K.MAX_MOTOR_PARAM + K.LP_A, K.MAX_MOTOR_PARAM + K.LP_J_LOAD]
    t = _tangents(cfg, slots)
    rs, ld, lq, ps, jr, la, jl = t
    assert rs[0] == pytest.approx(-1 / l_d, rel=1e-15) and rs[4] == pytest.approx(-1 / l_q, rel=1e-15)
    assert np.count_nonzero(rs) == 2
    assert ld[0] == pytest.approx(r_s / l_d ** 2, rel=1e-14) and ld[1] == pytest.approx(-1 / l_d ** 2, rel=1e-14)
    assert ld[2] == pytest.approx(-l_q * p / l_d ** 2, rel=1e-14) and ld[6] == pytest.approx(-p / l_q, rel=1e-14)
    assert ld[21] == pytest.approx(1.5 * p, rel=1e-15)
    assert lq[21] == pytest.approx(-1.5 * p, rel=1e-15)
    assert lq[2] == pytest.approx(p / l_d, rel=1e-14) and lq[3] == pytest.approx(psi * p / l_q ** 2, rel=1e-14)
    assert ps[3] == pytest.approx(-p / l_q, rel=1e-15) and ps[20] == pytest.approx(1.5 * p, rel=1e-15) and np.count_nonzero(ps) == 2
    j = lp[K.LP_J_LOAD] + mp[K.MP_J_ROTOR]
    for col in (jr, jl):
        assert col[27] == pytest.approx(-1 / j ** 2, rel=1e-14)
        assert col[28] == pytest.approx(-lp[K.LP_A] * lp[K.LP_TAU_DECAY] / j ** 2, rel=1e-14)
        assert col[29] == pytest.approx(1 / lp[K.LP_TAU_DECAY], rel=1e-15)
        assert np.count_nonzero(col[:27]) == 0
    assert la[24] == 1 and la[28] == pytest.approx(lp[K.LP_TAU_DECAY] / j, rel=1e-15) and np.count_nonzero(la) == 2


def test_coef_tangents_at_a_given_row():
    cfg = _cfg(K.MOTOR_SCIM)
    prm = _row(cfg)
    prm2 = prm.copy()
    prm2[K.MP_R_S] *= 1.3
    prm2[K.MP_L_M] *= 0.8
    a, b = _tangents(cfg, ACCEPTED[:12], prm2), _tangents(cfg, ACCEPTED[:12])
    assert not np.array_equal(a, b)
    cfg2 = type(cfg).from_buffer_copy(cfg)
    for s in range(K.MAX_MOTOR_PARAM):
        cfg2.motor_param[s] = prm2[s]
    assert np.array_equal(a, _tangents(cfg2, ACCEPTED[:12]))


def test_param_names(no_launch):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=N, dtype="float64")
    assert env.param_slots(["r_s", "l_d", "l_q", "psi_p"]) == [K.MP_R_S, K.MP_L_D, K.MP_L_Q, K.MP_PSI_P]
    assert env.param_slots(["j_rotor", "a", "b", "c", "j_load"]) == [K.MP_J_ROTOR] + LOAD_SLOTS[:3] + [LOAD_SLOTS[3]]
    assert env.param_slots("r_r") == [K.MP_R_E]
    with pytest.raises(KeyError):
        env.param_slots(["r_s", "nope"])
    with pytest.raises(KeyError):
        env.param_slots(["tau_decay"])
    for bad in (["p"], ["k"], ["r_s", "r_s"], ["r_e", "r_r"], []):
        with pytest.raises(ValueError):
            env.param_slots(bad)
    with pytest.raises(ValueError):
        env.param_slots(["r_s", "l_d", "l_q", "psi_p", "j_rotor", "r_a", "l_a", "psi_e", "r_e", "l_e", "l_e_prime", "l_m", "a"])
    acts = torch.zeros(4, N, 3, dtype=torch.float64)
    for bad in (torch.zeros(4, N, 2, dtype=torch.float64), torch.zeros(4, N, 3), torch.zeros(0, N, 3, dtype=torch.float64), "x"):
        with pytest.raises(ValueError):
            env.rollout_param_sensitivities(bad, ["r_s"])
    for bad in (torch.zeros(N, 4, 2, dtype=torch.float64), torch.zeros(N, 4, 1), torch.zeros(N, 3, 1, dtype=torch.float64), np.zeros((N, 4, 1))):
        with pytest.raises(ValueError):
            env.rollout_param_sensitivities(acts, ["r_s"], sens0=bad)
    with pytest.raises(ValueError):
        env.rollout_param_sensitivities(acts, ["r_s"], references=torch.zeros(3, N, 2, dtype=torch.float64))
    with pytest.raises(ValueError):
        env.rollout_param_sensitivities(acts, ["p"])
    with pytest.raises(KeyError):
        env.rollout_param_sensitivities(acts, ["q"])

    cfg = env.build_config()
    cfg.dead_time_steps = 1
    with pytest.raises(NotImplementedError):
        NoLaunchSim(cfg).param_sens_dims([K.MP_R_S])


def test_scalar_env_and_null_handle():
    env = gem.make("Cont-CC-PMSM-v0")
    with pytest.raises(TypeError):
        env.rollout_param_sensitivities(torch.zeros(1, 1, 3), ["r_s"])
    lib = K.load_library()
    arr = (C.c_int32 * 1)(K.MP_R_S)
    assert lib.gemb200_rollout_param_sens(None, None, None, 1, 1, arr, None, None, None, None, None, None, None) == K.E_INVALID
    assert lib.gemb200_query_param_sens_dims(None, 1, arr, None) == K.E_INVALID
    assert lib.gemb200_coef_tangents(None, None, None, 1, arr, None) == K.E_INVALID
