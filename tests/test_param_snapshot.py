"""Per-env physical parameters in snapshots without a GPU: the new C-ABI symbols and row width, EnvSnapshot params validation, slicing and
repr, and the argument checks of snapshot_envs(params=...) / restore_envs(params=...) around a scripted handle."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest
import torch

import gym_electric_motor_b200 as gem
from gym_electric_motor_b200 import _cabi as K
from gym_electric_motor_b200.snapshot import EnvSnapshot

HEADER = Path(__file__).resolve().parents[1] / "include" / "gemb200.h"


def test_symbols_and_row_width():
    lib = K.load_library()
    for name in ("gemb200_pack_envs_params", "gemb200_unpack_envs_params"):
        assert name in K.SYMBOLS and hasattr(lib, name)
    text = HEADER.read_text()
    assert int(re.search(r"#define GEMB200_ENV_PARAM_SLOTS (\d+)", text).group(1)) == K.ENV_PARAM_SLOTS == K.MAX_MOTOR_PARAM + 8 == 24
    assert int(re.search(r"#define GEMB200_ABI_VERSION (\d+)", text).group(1)) == K.ABI_VERSION  # unchanged ABI


def test_null_handle_is_refused():
    lib = K.load_library()
    assert lib.gemb200_pack_envs_params(None, None, 1, None, None, None) == K.E_INVALID
    assert lib.gemb200_unpack_envs_params(None, None, None, None, 1, 0, None, None, 1, None) == K.E_INVALID


def _snap(m=5, words=11, rng=True, params=True, p=3.0):
    rows = torch.arange(m * words, dtype=torch.int32).reshape(m, words)
    ids = torch.arange(1000, 1000 + m * K.RNG_ID_WORDS, dtype=torch.int32).reshape(m, K.RNG_ID_WORDS) if rng else None
    prm = torch.arange(m * K.ENV_PARAM_SLOTS, dtype=torch.float64).reshape(m, K.ENV_PARAM_SLOTS) if params else None
    return EnvSnapshot(rows, 0x1234, torch.float32, ids, prm, p if params else None)


@pytest.mark.parametrize("rng", [True, False], ids=["with_ids", "without_ids"])
def test_slicing_keeps_rows_identities_and_params_together(rng):
    s = _snap(rng=rng)
    for sel, want in ((2, [2]), (-1, [4]), (slice(1, 4), [1, 2, 3]), ([3, 0, 0], [3, 0, 0]), (np.array([4, 1]), [4, 1]), (torch.tensor([2, 2]), [2, 2])):
        sub = s[sel]
        assert torch.equal(sub.rows, s.rows[want])
        assert torch.equal(sub.params, s.params[want]) and sub.params.is_contiguous() and sub.params.dtype == torch.float64
        assert sub.pole_pairs == 3.0
        if rng:
            assert torch.equal(sub.rng, s.rng[want])
        else:
            assert sub.rng is None
    assert "params=yes" in repr(s)
    assert "params=no" in repr(_snap(params=False)) and _snap(params=False)[1:3].params is None


def test_params_shape_and_dtype_are_checked():
    rows = torch.zeros((3, 11), dtype=torch.int32)
    EnvSnapshot(rows, 1, torch.float32)  # the old constructors still work
    EnvSnapshot(rows, 1, torch.float32, None)
    EnvSnapshot(rows, 1, torch.float32, None, torch.zeros((3, K.ENV_PARAM_SLOTS), dtype=torch.float64), 4)
    for bad in (torch.zeros((2, K.ENV_PARAM_SLOTS), dtype=torch.float64), torch.zeros((3, 16), dtype=torch.float64),
                torch.zeros((3, K.ENV_PARAM_SLOTS), dtype=torch.float32), np.zeros((3, K.ENV_PARAM_SLOTS))):
        with pytest.raises(ValueError, match="params"):
            EnvSnapshot(rows, 1, torch.float32, None, bad, 4)
    with pytest.raises(ValueError, match="pole_pairs"):
        EnvSnapshot(rows, 1, torch.float32, None, torch.zeros((3, K.ENV_PARAM_SLOTS), dtype=torch.float64))


# ---------------------------------------------------------------------------------------------------- argument checks (no GPU)
def _record(cfg):
    w, lid = C.c_int32(), C.c_uint64()
    K.check(K.load_library().gemb200_query_env_record(C.byref(cfg), C.byref(w), C.byref(lid)), "gemb200_query_env_record")
    return w.value, lid.value


class ParamHandle:
    """the VectorSim surface the env methods use; records the calls (with their exact shapes) instead of launching kernels"""

    def __init__(self, cfg, reuse_outputs=True):
        self.cfg, self.n, self.soa = cfg, cfg.n_envs, cfg.layout == K.LAYOUT_SOA
        self.calls = []
        ParamHandle.last = self

    def record_layout(self):
        return _record(self.cfg)

    def snapshot(self, idx=None, **kw):
        self.calls.append(("snapshot", idx, kw))
        words, lid = self.record_layout()
        m = self.n if idx is None else len(idx)
        ids = torch.zeros((m, K.RNG_ID_WORDS), dtype=torch.int32) if kw.get("rng") else None
        prm = torch.zeros((m, K.ENV_PARAM_SLOTS), dtype=torch.float64) if kw.get("params") else None
        return EnvSnapshot(torch.zeros((m, words), dtype=torch.int32), lid, torch.float32, ids, prm,
                           float(self.cfg.motor_param[K.MP_P]) if prm is not None else None)

    def restore(self, snap, idx=None, rows=None, **kw):
        self.calls.append(("restore", idx, rows, kw))

    def close(self):
        pass


@pytest.fixture
def handle(monkeypatch):
    import gym_electric_motor_b200.vector_sim as vs

    monkeypatch.setattr(vs, "VectorSim", ParamHandle)
    return ParamHandle


def _restores(h):
    return [c for c in h.last.calls if c[0] == "restore"]


def test_scalar_env_refuses_params(handle):
    env = gem.make("Cont-CC-PMSM-v0")
    with pytest.raises(TypeError):
        env.snapshot_envs(params=True)
    with pytest.raises(TypeError):
        env.restore_envs(None, params="source")


def test_default_call_shapes_are_unchanged(handle):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=6)
    snap = env.snapshot_envs([1, 4])
    assert handle.last.calls[-1][2] == {}
    env.snapshot_envs([1], rng=True)
    assert handle.last.calls[-1][2] == {"rng": True}
    env.restore_envs(snap, idx=[0, 2])
    assert handle.last.calls[-1][3] == {}
    env.restore_envs(env.snapshot_envs([0], rng=True), idx=[3], rng="source")
    assert handle.last.calls[-1][3] == {"rng": "source"}


def test_params_are_packed_and_adopted_on_request(handle):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=6)
    snap = env.snapshot_envs([1, 4], params=True)
    assert handle.last.calls[-1][2] == {"rng": False, "params": True}
    assert snap.params.shape == (2, K.ENV_PARAM_SLOTS) and snap.rng is None
    env.restore_envs(snap, idx=[0, 2, 3], rows=[1, 1, 0], params="source")
    assert handle.last.calls[-1][3] == {"rng": "own", "params": "source"}
    snap = env.snapshot_envs([2], rng=True, params=True)
    assert handle.last.calls[-1][2] == {"rng": True, "params": True}
    env.restore_envs(snap, idx=[5], rng="source", params="source")
    assert handle.last.calls[-1][3] == {"rng": "source", "params": "source"}
    env.restore_envs(snap, idx=[5])  # a snapshot with params restores without them as well
    assert handle.last.calls[-1][3] == {}


def test_source_without_params_is_refused(handle):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=4)
    snap = env.snapshot_envs([0, 1], rng=True)
    with pytest.raises(ValueError, match="params=True"):
        env.restore_envs(snap, idx=[2, 3], params="source")
    assert not _restores(handle)


@pytest.mark.parametrize("bad", ["deepcopy", True, None, "Source", 1])
def test_bad_params_value_is_refused(handle, bad):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=4)
    snap = env.snapshot_envs([0], params=True)
    with pytest.raises(ValueError, match="params"):
        env.restore_envs(snap, idx=[1], params=bad)
    assert not _restores(handle)


def test_pole_pair_mismatch_is_refused(handle):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=4)
    snap = env.snapshot_envs([0, 1], params=True)
    other = EnvSnapshot(snap.rows, snap.layout_id, snap.dtype, None, snap.params, snap.pole_pairs + 1)
    with pytest.raises(ValueError, match="pole pairs"):
        env.restore_envs(other, idx=[2, 3], params="source")
    env.restore_envs(other, idx=[2, 3])  # without params the pole pairs do not matter
    assert [c[3] for c in _restores(handle)] == [{}]


def test_soa_layout_refuses_params(handle):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=4, layout="soa")
    with pytest.raises(ValueError, match="row-per-env"):
        env.snapshot_envs([0], params=True)
    assert not [c for c in handle.last.calls if c[0] == "snapshot"]
    words, lid = handle.last.record_layout()
    snap = EnvSnapshot(torch.zeros((1, words), dtype=torch.int32), lid, torch.float32, None,
                       torch.zeros((1, K.ENV_PARAM_SLOTS), dtype=torch.float64), float(handle.last.cfg.motor_param[K.MP_P]))
    with pytest.raises(ValueError, match="row-per-env"):
        env.restore_envs(snap, idx=[1], params="source")
    env.restore_envs(snap, idx=[1])  # the default restore is not affected
    assert [c[3] for c in _restores(handle)] == [{}]
