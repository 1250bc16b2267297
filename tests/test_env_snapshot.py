"""Per-env state snapshots without a GPU: the packed record size and layout id of gemb200_query_env_record against the row format of
include/gemb200.h, and the argument checks of ElectricMotorEnvironment.snapshot_envs / restore_envs around a scripted handle."""
import ctypes as C

import numpy as np
import pytest
import torch

import gym_electric_motor_b200 as gem
from gym_electric_motor_b200 import _cabi as K
from gym_electric_motor_b200.snapshot import EnvSnapshot
from helpers import config_from_meta, load_golden


def _record(cfg):
    w, lid = C.c_int32(), C.c_uint64()
    K.check(K.load_library().gemb200_query_env_record(C.byref(cfg), C.byref(w), C.byref(lid)), "gemb200_query_env_record")
    return w.value, lid.value


def _dims(cfg):
    d = [C.c_int32() for _ in range(4)]
    K.check(K.load_library().gemb200_query_dims(C.byref(cfg), *[C.byref(x) for x in d]), "gemb200_query_dims")
    return [x.value for x in d]


def _golden_cfg(name, dtype=K.F64, n=3, **kw):
    g = load_golden(name)
    return config_from_meta(g["meta"], n_envs=n, reset_ode=g["reset_ode"], dtype=dtype, ref_kind=kw.pop("ref_kind", K.REF_WIENER), **kw)


def _words_from_format(cfg):
    """the row format of include/gemb200.h, restated independently of the library"""
    n_state, n_ode, n_act, n_ref = _dims(cfg)
    three_phase = cfg.motor_kind >= K.MOTOR_PMSM
    nx = n_ode - (1 if three_phase else 0)
    wr = 1 if cfg.dtype == K.F32 else 2  # words per real
    words = (nx - 1 + n_ref) * wr + (1 + 2 * n_ref) * wr   # hot + cold record
    words += 2 if three_phase else 0                      # angle (double)
    if cfg.finite and (cfg.interlocking_time > 0 or cfg.interlocking_time1 > 0 or cfg.supply_kind == K.SUPPLY_RC):
        words += 1                                        # switching state
    if cfg.dead_time_steps:
        fam_inner = {K.MOTOR_DFIM: 6, K.MOTOR_EESM: 4}.get(cfg.motor_kind, 3 if three_phase else n_act)
        fifo_dim = (n_act if cfg.finite else fam_inner) if (cfg.action_dq and not cfg.dead_time_outer) else n_act
        words += cfg.dead_time_steps * fifo_dim * wr
    if any(cfg.sop_kind[k] == K.SOP_FLUX_OBSERVER for k in range(cfg.n_state_ops)):
        words += 4 * wr
    words += {K.SUPPLY_RC: 2 * wr, K.SUPPLY_AC1: 2}.get(cfg.supply_kind, 0)
    if any(cfg.ref_sw_count[r] > 1 for r in range(n_ref)):
        words += 2 * n_ref
    words += 1 if cfg.load_kind == K.LOAD_EXT_SPEED else 0
    words += 2 * wr if cfg.init_im_valid else 0
    return words


def test_pmsm_cc_f32_record_is_11_words():
    cfg = gem.make("Cont-CC-PMSM-v0", num_envs=4).build_config()
    assert cfg.dtype == K.F32 and _record(cfg)[0] == 11 == _words_from_format(cfg)


@pytest.mark.parametrize("name", ["pmsm_cc_rk4", "dfim_cc_rk4", "dfim_cc_flux_dq_rk4", "scim_sc_flux_cossin_dead1_rk4", "eesm_cc_rc_dq_dead1_rk4",
                                  "pmsm_cc_ac_rk4", "pmsm_cc_extspeed_rk4", "permex_fin_sc_rc_interlock_rk4", "pmsm_fin_sc_rk4_interlock"])
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
def test_words_follow_the_row_format(name, dtype):
    cfg = _golden_cfg(name, dtype)
    assert _record(cfg)[0] == _words_from_format(cfg), name


def test_dead_time_ring_and_switched_generators_in_the_row():
    cfg = _golden_cfg("pmsm_cc_rk4")
    cfg.dead_time_steps = 3
    assert _record(cfg)[0] == _words_from_format(cfg) == 20 + 2 * 3 * 3
    from helpers import switched_config

    sw = switched_config(5, [dict(kind=K.REF_WIENER), dict(kind=K.REF_SINUS)], [0.5, 0.5], (5, 12))
    assert _record(sw)[0] == _words_from_format(sw)


def test_layout_id_ignores_size_seed_and_parameters():
    base = _golden_cfg("pmsm_cc_rk4", K.F32, n=7)
    _, lid = _record(base)
    variants = []
    for change in (lambda c: setattr(c, "n_envs", 1 << 20), lambda c: setattr(c, "seed", 999), lambda c: setattr(c, "tau", 5e-5),
                   lambda c: setattr(c, "env_index_offset", 4096), lambda c: c.motor_param.__setitem__(K.MP_R_S, 2.5 * c.motor_param[K.MP_R_S]),
                   lambda c: setattr(c, "reward_bias", 0.5), lambda c: setattr(c, "layout", K.LAYOUT_SOA), lambda c: setattr(c, "solver_kind", K.SOLVER_EULER)):
        c = _golden_cfg("pmsm_cc_rk4", K.F32, n=7)
        change(c)
        variants.append(_record(c)[1])
    assert all(v == lid for v in variants)


def test_layout_id_differs_across_what_shapes_the_row():
    _, lid = _record(_golden_cfg("pmsm_cc_rk4", K.F32))
    other = {
        "dtype": _golden_cfg("pmsm_cc_rk4", K.F64),
        "motor": _golden_cfg("synrm_cc_rk4", K.F32),
        "generator kind": _golden_cfg("pmsm_cc_rk4", K.F32, ref_kind=K.REF_CONST),
        "observer": _golden_cfg("dfim_cc_flux_dq_rk4", K.F32),
        "supply": _golden_cfg("pmsm_cc_ac_rk4", K.F32),
    }
    dead = _golden_cfg("pmsm_cc_rk4", K.F32)
    dead.dead_time_steps = 2
    other["dead time"] = dead
    one_ref = _golden_cfg("pmsm_cc_rk4", K.F32)
    one_ref.n_ref = 1
    other["n_ref"] = one_ref
    ids = {k: _record(c)[1] for k, c in other.items()}
    assert all(v != lid for v in ids.values()), ids
    assert len(set(ids.values())) == len(ids)
    # DFIM without / with the observer: same motor, one array more
    assert _record(_golden_cfg("dfim_cc_rk4", K.F32))[1] != ids["observer"]


# ---------------------------------------------------------------------------------------------------- argument checks (no GPU)
class SnapshotHandle:
    """the VectorSim surface snapshot_envs / restore_envs use; records the calls instead of launching kernels"""

    def __init__(self, cfg, reuse_outputs=True):
        self.cfg, self.n, self.soa = cfg, cfg.n_envs, False
        self.calls = []
        SnapshotHandle.last = self

    def record_layout(self):
        return _record(self.cfg)

    def snapshot(self, idx=None):
        self.calls.append(("snapshot", idx))
        words, lid = self.record_layout()
        m = self.n if idx is None else len(idx)
        return EnvSnapshot(torch.zeros((m, words), dtype=torch.int32), lid, torch.float32)

    def restore(self, snap, idx=None, rows=None):
        self.calls.append(("restore", idx, rows))

    def close(self):
        pass


@pytest.fixture
def handle(monkeypatch):
    import gym_electric_motor_b200.vector_sim as vs

    monkeypatch.setattr(vs, "VectorSim", SnapshotHandle)
    return SnapshotHandle


def test_scalar_env_refuses_snapshots(handle):
    env = gem.make("Cont-CC-PMSM-v0")
    with pytest.raises(TypeError):
        env.snapshot_envs()
    with pytest.raises(TypeError):
        env.restore_envs(None)


def test_host_indices_are_range_checked(handle):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=6)
    snap = env.snapshot_envs([0, 5, 2])
    assert len(snap) == 3 and snap.words == 11 and len(snap[1:]) == 2 and len(snap[[2, 0, 0, 1]]) == 4
    for bad in ([0, 6], np.array([-1]), torch.tensor([7])):
        with pytest.raises(IndexError):
            env.snapshot_envs(bad)
        with pytest.raises(IndexError):
            env.restore_envs(snap, idx=bad)
    with pytest.raises(IndexError):
        env.restore_envs(snap, idx=[0, 1], rows=[0, 3])   # the snapshot has 3 rows
    env.restore_envs(snap, idx=np.array([4, 1, 3]), rows=[2, 2, 0])
    assert handle.last.calls[-1][0] == "restore" and list(handle.last.calls[-1][1]) == [4, 1, 3]


def test_wrong_layout_or_width_is_refused(handle):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=4)
    words, lid = _record(env.build_config())
    other = gem.make("Cont-CC-SynRM-v0", num_envs=4)
    w2, lid2 = _record(other.build_config())
    with pytest.raises(ValueError, match="layout"):
        env.restore_envs(EnvSnapshot(torch.zeros((2, w2), dtype=torch.int32), lid2, torch.float32))
    with pytest.raises(ValueError, match="words"):
        env.restore_envs(EnvSnapshot(torch.zeros((2, words + 1), dtype=torch.int32), lid, torch.float32))
    with pytest.raises(ValueError):
        env.restore_envs(torch.zeros((2, words), dtype=torch.int32))
    assert not [c for c in handle.last.calls if c[0] == "restore"]
