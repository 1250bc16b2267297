"""Per-episode domain randomisation: the user's parameter distributions as the slot / kind / bound arrays of
gemb200_set_param_randomization (include/gemb200.h).

A distribution is `(lo, hi)` (uniform) or `(kind, lo, hi)` with kind "uniform" or "log_uniform".  All checks here run on the host,
before any device call.
"""
import math

import numpy as np

from . import _cabi as K

DIST_KINDS = {"uniform": K.DIST_UNIFORM, "log_uniform": K.DIST_LOG_UNIFORM}
# parameters of an induction motor that enter the host-derived flux-limit constants of random initial states (gemb200.h: init_im)
FLUX_LIMIT_SLOTS = frozenset((K.MP_L_M, K.MP_L_SIGS, K.MP_L_SIGR, K.MP_R_S, K.MP_R_E))


def parse_distribution(name, spec):
    """(kind enum, lo, hi) of one parameter's distribution; ValueError for anything else"""
    if isinstance(spec, (tuple, list)) and len(spec) == 3 and isinstance(spec[0], str):
        kind, lo, hi = spec
    elif isinstance(spec, (tuple, list)) and len(spec) == 2:
        kind, (lo, hi) = "uniform", spec
    else:
        raise ValueError(f"{name}: a distribution is (lo, hi) or ('uniform' | 'log_uniform', lo, hi), got {spec!r}")
    if kind not in DIST_KINDS:
        raise ValueError(f"{name}: unknown distribution {kind!r} (use 'uniform' or 'log_uniform')")
    try:
        lo, hi = float(lo), float(hi)
    except (TypeError, ValueError):
        raise ValueError(f"{name}: bounds must be numbers, got {spec!r}") from None
    if not (math.isfinite(lo) and math.isfinite(hi)):
        raise ValueError(f"{name}: bounds must be finite")
    if lo > hi:
        raise ValueError(f"{name}: lo ({lo}) > hi ({hi})")
    if kind == "log_uniform" and lo <= 0:
        raise ValueError(f"{name}: log_uniform needs lo > 0")
    return DIST_KINDS[kind], lo, hi


def check_pole_pairs(rows_p, pole_pairs):
    """per-env rows (`set_env_parameters`, `VectorSim.set_env_params`) keep the handle's pole pairs: ValueError otherwise"""
    rows_p = np.asarray(rows_p, dtype=np.float64)
    bad = np.flatnonzero(rows_p != float(pole_pairs))
    if bad.size:
        raise ValueError(f"pole pairs 'p' cannot differ per env (env {int(bad[0])}: {rows_p[bad[0]]:g}, this env kind: {float(pole_pairs):g}): "
                         "the angle increments are prepared per handle on the host")


def encode_distributions(motor_parameter, load_parameter, mp_slot, lp_slot, flux_limits=False):
    """names -> (names, slots, kinds, lo, hi) in argument order.  mp_slot / lp_slot map the reference's parameter names to GEMB200_MP_* /
    GEMB200_LP_*; load slots are offset by MAX_MOTOR_PARAM.  flux_limits: the env is an induction motor with random initial states."""
    names, slots, kinds, los, his = [], [], [], [], []
    for table, params, base, what in ((mp_slot, motor_parameter, 0, "motor"), (lp_slot, load_parameter, K.MAX_MOTOR_PARAM, "load")):
        for name, spec in (params or {}).items():
            if name not in table:
                raise KeyError(f"unknown {what} parameter {name!r}")
            slot = base + table[name]
            if base == 0 and slot == K.MP_P:
                raise ValueError("pole pairs 'p' cannot be drawn per env: the angle increments are prepared per handle on the host")
            if base == 0 and flux_limits and slot in FLUX_LIMIT_SLOTS:
                raise NotImplementedError(f"{name!r} of an induction motor with random initial states enters the host-derived flux limits "
                                          "of the initial states and cannot be drawn per env (DESIGN.md §7)")
            if slot in slots:
                raise ValueError(f"{name!r} names a parameter that is already drawn")
            kind, lo, hi = parse_distribution(name, spec)
            names.append(name)
            slots.append(slot)
            kinds.append(kind)
            los.append(lo)
            his.append(hi)
    return names, slots, kinds, los, his
