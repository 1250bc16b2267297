"""RNG identities without a GPU: the new C-ABI symbols and row width, EnvSnapshot slicing with and without identities, and the argument
checks of snapshot_envs(rng=...) / restore_envs(rng=...) / clear_rng_identities around a scripted handle."""
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
    for name in ("gemb200_pack_rng_ids", "gemb200_adopt_rng_ids", "gemb200_clear_rng_ids"):
        assert name in K.SYMBOLS and hasattr(lib, name)
    text = HEADER.read_text()
    assert int(re.search(r"#define GEMB200_RNG_ID_WORDS (\d+)", text).group(1)) == K.RNG_ID_WORDS == 8
    assert int(re.search(r"#define GEMB200_ABI_VERSION (\d+)", text).group(1)) == K.ABI_VERSION  # unchanged ABI
    assert lib.gemb200_pack_rng_ids(None, None, 1, None, None) == K.E_INVALID  # NULL handle: refused without a GPU
    assert lib.gemb200_adopt_rng_ids(None, None, 1, None, None, 1, None) == K.E_INVALID
    assert lib.gemb200_clear_rng_ids(None, None) == K.E_INVALID


def _snap(m=5, words=11, rng=True):
    rows = torch.arange(m * words, dtype=torch.int32).reshape(m, words)
    ids = torch.arange(1000, 1000 + m * K.RNG_ID_WORDS, dtype=torch.int32).reshape(m, K.RNG_ID_WORDS) if rng else None
    return EnvSnapshot(rows, 0x1234, torch.float32, ids)


@pytest.mark.parametrize("rng", [True, False], ids=["with_ids", "without_ids"])
def test_snapshot_slicing_keeps_rows_and_identities_together(rng):
    s = _snap(rng=rng)
    for sel, want in ((2, [2]), (-1, [4]), (slice(1, 4), [1, 2, 3]), ([3, 0, 0], [3, 0, 0]), (np.array([4, 1]), [4, 1]), (torch.tensor([2, 2]), [2, 2])):
        sub = s[sel]
        assert torch.equal(sub.rows, s.rows[want])
        if rng:
            assert torch.equal(sub.rng, s.rng[want]) and sub.rng.is_contiguous()
        else:
            assert sub.rng is None
    assert "rng=yes" in repr(s) if rng else "rng=no" in repr(s)


def test_snapshot_identity_shape_is_checked():
    rows = torch.zeros((3, 11), dtype=torch.int32)
    EnvSnapshot(rows, 1, torch.float32)  # the old constructor still works
    for bad in (torch.zeros((2, K.RNG_ID_WORDS), dtype=torch.int32), torch.zeros((3, 7), dtype=torch.int32), torch.zeros((3, K.RNG_ID_WORDS), dtype=torch.int64)):
        with pytest.raises(ValueError):
            EnvSnapshot(rows, 1, torch.float32, bad)


# ---------------------------------------------------------------------------------------------------- argument checks (no GPU)
def _record(cfg):
    w, lid = C.c_int32(), C.c_uint64()
    K.check(K.load_library().gemb200_query_env_record(C.byref(cfg), C.byref(w), C.byref(lid)), "gemb200_query_env_record")
    return w.value, lid.value


class IdHandle:
    """the VectorSim surface the env methods use; records the calls instead of launching kernels"""

    def __init__(self, cfg, reuse_outputs=True):
        self.cfg, self.n, self.soa = cfg, cfg.n_envs, cfg.layout == K.LAYOUT_SOA
        self.calls = []
        IdHandle.last = self

    def record_layout(self):
        return _record(self.cfg)

    def snapshot(self, idx=None, rng=False):
        self.calls.append(("snapshot", idx, rng))
        words, lid = self.record_layout()
        m = self.n if idx is None else len(idx)
        ids = torch.zeros((m, K.RNG_ID_WORDS), dtype=torch.int32) if rng else None
        return EnvSnapshot(torch.zeros((m, words), dtype=torch.int32), lid, torch.float32, ids)

    def restore(self, snap, idx=None, rows=None, rng="own"):
        self.calls.append(("restore", idx, rows, rng))

    def clear_rng_ids(self):
        self.calls.append(("clear",))

    def close(self):
        pass


@pytest.fixture
def handle(monkeypatch):
    import gym_electric_motor_b200.vector_sim as vs

    monkeypatch.setattr(vs, "VectorSim", IdHandle)
    return IdHandle


def test_scalar_env_refuses_identities(handle):
    env = gem.make("Cont-CC-PMSM-v0")
    with pytest.raises(TypeError):
        env.snapshot_envs(rng=True)
    with pytest.raises(TypeError):
        env.restore_envs(None, rng="source")
    with pytest.raises(TypeError):
        env.clear_rng_identities()


def test_identities_are_packed_and_adopted_on_request(handle):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=6)
    snap = env.snapshot_envs([1, 4], rng=True)
    assert snap.rng is not None and snap.rng.shape == (2, K.RNG_ID_WORDS)
    assert handle.last.calls[-1][2] is True
    env.restore_envs(snap, idx=[0, 2, 3], rows=[1, 1, 0], rng="source")
    assert handle.last.calls[-1][0] == "restore" and handle.last.calls[-1][3] == "source"
    env.restore_envs(snap, idx=[5])
    assert handle.last.calls[-1][3] == "own"
    env.clear_rng_identities()
    assert handle.last.calls[-1] == ("clear",)
    assert env.snapshot_envs([0]).rng is None


def test_source_without_identities_is_refused(handle):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=4)
    snap = env.snapshot_envs([0, 1])
    with pytest.raises(ValueError, match="rng=True"):
        env.restore_envs(snap, idx=[2, 3], rng="source")
    assert not [c for c in handle.last.calls if c[0] == "restore"]


@pytest.mark.parametrize("bad", ["deepcopy", True, None, "Source"])
def test_bad_rng_value_is_refused(handle, bad):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=4)
    snap = env.snapshot_envs([0], rng=True)
    with pytest.raises(ValueError, match="rng"):
        env.restore_envs(snap, idx=[1], rng=bad)
    assert not [c for c in handle.last.calls if c[0] == "restore"]


def test_soa_layout_refuses_adoption(handle):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=4, layout="soa")
    snap = env.snapshot_envs([0], rng=True)
    with pytest.raises(ValueError, match="row-per-env"):
        env.restore_envs(snap, idx=[1], rng="source")
    env.restore_envs(snap, idx=[1])  # the default restore is not affected
    assert [c[3] for c in handle.last.calls if c[0] == "restore"] == ["own"]
