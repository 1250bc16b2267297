"""Per-env state snapshots on the device: the batched counterpart of branching a reference env with `copy.deepcopy(env)`.

An `EnvSnapshot` holds the complete persistent state of m envs as packed rows (gemb200_pack_envs; row format in include/gemb200.h): a
plain device `torch.int32` tensor [m, words] that the caller may keep, concatenate, index or send to another rank, and that
`VectorSim.restore` / `ElectricMotorEnvironment.restore_envs` put into any envs of a handle with the same record layout — the same env in
another batch size, seed or index offset, or with other per-env parameters.  A restored env continues exactly like its source, except
that it draws the random numbers of its own (seed, global env index) from then on — unless the snapshot was taken with `rng=True` and is
restored with `rng="source"`: the env then adopts its source's RNG identity and repeats the source's draws (copy.deepcopy semantics).
A snapshot taken with `params=True` also holds the envs' physical parameters; restored with `params="source"`, every env takes its source's
(its own per-env values, drawn or set from the host) and runs its current episode on the source's plant.
"""
import numpy as np
import torch

from ._cabi import ENV_PARAM_SLOTS, MP_P, RNG_ID_WORDS


class EnvSnapshot:
    """Packed state of m envs: `rows` [m, words] int32 on the device, `layout_id` of the record layout, `dtype` of the handle's state,
    `rng` [m, RNG_ID_WORDS] int32 = the envs' RNG identities (gemb200_pack_rng_ids) or None,
    `params` [m, ENV_PARAM_SLOTS] float64 = the envs' physical parameters (gemb200_pack_envs_params; slots `_cabi.MP_*`, then
    `_cabi.MAX_MOTOR_PARAM + _cabi.LP_*`) or None, and `pole_pairs`, the source handle's pole pairs (host float) when `params` is set.
    `params` is a plain tensor: editing it before a restore gives the restored envs the edited values (an ensemble of plants).
    `len(snap)` is m; `snap[k]`, `snap[a:b]`, `snap[index list / tensor]` are sub-snapshots of the selected rows."""

    __slots__ = ("rows", "layout_id", "dtype", "rng", "params", "pole_pairs")

    def __init__(self, rows, layout_id, dtype, rng=None, params=None, pole_pairs=None):
        if not isinstance(rows, torch.Tensor) or rows.dtype != torch.int32 or rows.dim() != 2:
            raise ValueError("EnvSnapshot rows must be a 2-D torch.int32 tensor [m, words]")
        if rng is not None and (not isinstance(rng, torch.Tensor) or rng.dtype != torch.int32 or tuple(rng.shape) != (rows.shape[0], RNG_ID_WORDS)):
            raise ValueError(f"EnvSnapshot rng must be a torch.int32 tensor [m, {RNG_ID_WORDS}] with one row per snapshot row")
        if params is not None:
            if not isinstance(params, torch.Tensor) or params.dtype != torch.float64 or tuple(params.shape) != (rows.shape[0], ENV_PARAM_SLOTS):
                raise ValueError(f"EnvSnapshot params must be a torch.float64 tensor [m, {ENV_PARAM_SLOTS}] with one row per snapshot row")
            if pole_pairs is None:
                raise ValueError("EnvSnapshot params need the source's pole_pairs")
        self.rows = rows
        self.layout_id = int(layout_id)
        self.dtype = dtype
        self.rng = rng
        self.params = params
        self.pole_pairs = None if params is None else float(pole_pairs)

    def __len__(self):
        return int(self.rows.shape[0])

    @property
    def words(self):
        return int(self.rows.shape[1])

    def __getitem__(self, idx):
        if isinstance(idx, (int, np.integer)):
            k = int(idx) + (len(self) if int(idx) < 0 else 0)
            if not 0 <= k < len(self):
                raise IndexError(f"snapshot index {idx} out of range for {len(self)} rows")
            sel = slice(k, k + 1)
        elif isinstance(idx, slice):
            sel = idx
        else:
            sel = torch.as_tensor(np.asarray(idx) if not isinstance(idx, torch.Tensor) else idx, device=self.rows.device).long()

        def pick(t):
            return None if t is None else t[sel if isinstance(sel, slice) else sel.to(t.device)].contiguous()

        return EnvSnapshot(self.rows[sel].contiguous(), self.layout_id, self.dtype, pick(self.rng), pick(self.params), self.pole_pairs)

    def __repr__(self):
        return (f"EnvSnapshot(m={len(self)}, words={self.words}, layout_id={self.layout_id:#018x}, dtype={self.dtype}, "
                f"rng={'yes' if self.rng is not None else 'no'}, params={'yes' if self.params is not None else 'no'})")


def check_host_index(idx, bound, what):
    """Range check of a host-side index argument (list, numpy array, CPU tensor): IndexError unless every entry is in [0, bound).
    None and device tensors pass unchanged (the kernels skip out-of-range entries of a device index)."""
    if idx is None or (isinstance(idx, torch.Tensor) and idx.is_cuda):
        return idx
    a = np.asarray(idx.cpu() if isinstance(idx, torch.Tensor) else idx).reshape(-1)
    if a.size and not np.issubdtype(a.dtype, np.integer):
        raise IndexError(f"{what} must hold integers, got {a.dtype}")
    if a.size and (a.min() < 0 or a.max() >= bound):
        raise IndexError(f"{what} out of range: entries must be in [0, {bound})")
    return a


def check_rng_mode(snap, rng, soa):
    """the `rng` argument of a restore: "own" (the envs keep drawing their own numbers) or "source" (they adopt the snapshot's RNG
    identities, which need a snapshot taken with rng=True and the row-per-env layout); ValueError otherwise"""
    if rng not in ("own", "source"):
        raise ValueError(f"rng must be 'own' or 'source', got {rng!r}")
    if rng == "source":
        if snap.rng is None:
            raise ValueError("rng='source' needs a snapshot taken with rng=True (it carries no RNG identities)")
        if soa:
            raise ValueError("adopted RNG identities need the row-per-env layout (layout='aos'), like per-env parameter blocks (DESIGN.md §7)")
    return rng == "source"


def check_params_layout(soa):
    """ValueError on the field-major layout: parameter rows belong to per-env parameter blocks, which need the row-per-env layout"""
    if soa:
        raise ValueError("parameter rows need the row-per-env layout (layout='aos'), like every per-env parameter block (DESIGN.md §7)")


def check_params_mode(snap, params, soa, pole_pairs):
    """the `params` argument of a restore: "own" (the envs keep their physical parameters) or "source" (they take the snapshot's, which
    needs a snapshot taken with params=True, the row-per-env layout and the source's pole pairs, which are per handle); ValueError
    otherwise"""
    if params not in ("own", "source"):
        raise ValueError(f"params must be 'own' or 'source', got {params!r}")
    if params == "source":
        if snap.params is None:
            raise ValueError("params='source' needs a snapshot taken with params=True (it carries no physical parameters)")
        check_params_layout(soa)
        if float(snap.pole_pairs) != float(pole_pairs):
            raise ValueError(f"params='source': the snapshot's pole pairs ({snap.pole_pairs:g}) differ from this env's ({float(pole_pairs):g}); "
                             "pole pairs are per env kind, not per env")
    return params == "source"


def check_layout(snap, words, layout_id):
    """ValueError unless `snap` was packed from a handle with this record layout"""
    if not isinstance(snap, EnvSnapshot):
        raise ValueError(f"expected an EnvSnapshot, got {type(snap).__name__}")
    if snap.layout_id != int(layout_id):
        raise ValueError(f"snapshot of another record layout (layout_id {snap.layout_id:#018x}, this env has {int(layout_id):#018x}): "
                         "motor, dtype, generators, dead time, wrappers or supply differ")
    if snap.words != int(words):
        raise ValueError(f"snapshot rows have {snap.words} words, this env's record has {int(words)}")
