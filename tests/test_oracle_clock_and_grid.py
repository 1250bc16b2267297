"""The oracle's clock jump and time-grid hooks (CPU only).

`Oracle.set_clock` puts a handle at any (call id, step count) so that long-horizon GPU tests can compare both sides right at the 32-bit
wrap-arounds without stepping there.  `Oracle.set_time_grid(True)` switches from the reference's time grid (t accumulated with
t += tau, each step integrated over fl(t + tau) - t) to the device's (step k of an episode over [k tau, (k + 1) tau], segment lengths
precomputed, angle kept reduced): the grid the device is compared on over long episodes (DESIGN §2 finding 12).
"""
from fractions import Fraction
import math

import numpy as np
import pytest

from helpers import load_golden, config_from_meta
from gym_electric_motor_b200 import _cabi as K

TAU = 1e-4


def _pmsm_cfg(n, ref_kind=K.REF_WIENER, speed=100.0, supply=None, seed=11):
    g = load_golden("pmsm_cc_rk4")
    cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=[speed, 0.5, -0.25, 0.75], dtype=K.F64, solver="rk4", ref_kind=ref_kind,
                           autoreset=K.AUTORESET_SAME_STEP, seed=seed)
    cfg.n_constraints = 0
    cfg.env_index_offset = 3 * n
    if supply == "ac":
        cfg.supply_kind = K.SUPPLY_AC1
        cfg.supply_param[0], cfg.supply_param[1], cfg.supply_param[2] = 50.0, 0.0, 0.0  # 50 Hz, random phase per env and reset
    return cfg


def _periodic(cfg):
    """slot 0 sinusoidal, slot 1 sawtooth with short sub-episodes: their Philox blocks are keyed by the step count"""
    for r, kind in enumerate((K.REF_SINUS, K.REF_SAWTOOTH)):
        cfg.ref_kind[r] = kind
        cfg.ref_amp_lo[r], cfg.ref_amp_hi[r] = 0.05, 0.6
        cfg.ref_freq_lo[r], cfg.ref_freq_hi[r] = 20.0, 400.0
        cfg.ref_off_lo[r], cfg.ref_off_hi[r] = -0.6, 0.6
        cfg.ref_len_lo[r], cfg.ref_len_hi[r] = 3, 17
    return cfg


def _actions(rng, steps, n):
    return 0.3 * rng.uniform(-1, 1, size=(steps, n, 3))


@pytest.mark.parametrize("kind", ["wiener", "periodic", "ac"])
def test_jumped_clock_equals_natural_clock(oracle_lib, kind):
    """Oracle stepped to (c, n) and oracle jumped there give identical trajectories after a full reset."""
    n, steps = 9, 60
    mk = (lambda: _periodic(_pmsm_cfg(n))) if kind == "periodic" else (lambda: _pmsm_cfg(n, supply="ac" if kind == "ac" else None))
    rng = np.random.default_rng(5)
    natural = oracle_lib.Oracle(mk())
    for a in _actions(rng, 37, n):
        natural.step(a)
    natural.reset()
    natural.step(_actions(rng, 1, n)[0])
    clock = natural.clock()
    assert clock == (40, 38)  # create + 37 steps + reset + 1 step; the handle's first call (create's reset) has id 1
    jumped = oracle_lib.Oracle(mk())
    jumped.set_clock(*clock)
    assert jumped.clock() == clock
    o1, r1 = natural.reset()
    o2, r2 = jumped.reset()
    assert np.array_equal(o1, o2) and np.array_equal(r1, r2)
    for a in _actions(rng, steps, n):
        out1, out2 = natural.step(a), jumped.step(a)
        for x, y in zip(out1, out2):
            assert np.array_equal(x, y)
    assert natural.clock() == jumped.clock()


def test_jumped_clock_moves_the_random_streams(oracle_lib):
    """The jump is not a no-op: another clock draws other references (the comparison above is not vacuous)."""
    n = 9
    a, b = oracle_lib.Oracle(_periodic(_pmsm_cfg(n))), oracle_lib.Oracle(_periodic(_pmsm_cfg(n)))
    b.set_clock(2**32 - 3, 2**32 - 2)
    _, ra = a.reset()
    _, rb = b.reset()
    assert not np.array_equal(ra, rb)


@pytest.mark.parametrize("name,solver", [("pmsm_cc_rk4", "rk4"), ("pmsm_fin_sc_rk4_interlock", "rk4"), ("extex_fin_cc_interlock2_rk4", "rk4"),
                                         ("permex_cc_euler_10k", "euler"), ("scim_cc_rk4", "euler3"), ("pmsm_cc_ac_rk4", "rk4")])
def test_exact_and_faithful_grids_agree_over_a_short_run(oracle_lib, name, solver):
    """Over 1000 steps the two grids differ by rounding only (<= 1e-12 of each column's scale), in every segment layout."""
    g = load_golden(name)
    n, steps = 16, 1000
    init = np.array(g["reset_ode"], dtype=float)
    init[1:] = [0.9, -0.6, 0.5, 0.3][: len(init) - 1] if g["meta"]["motor_class"] not in ("SquirrelCageInductionMotor",) else [0.7, -0.4, 0.02, 0.03, 0.3]

    def mk():
        cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=init, dtype=K.F64, solver=solver, ref_kind=K.REF_WIENER, seed=3)
        cfg.n_constraints = 0
        return cfg

    faithful, exact = oracle_lib.Oracle(mk()), oracle_lib.Oracle(mk())
    exact.set_time_grid(True)
    o1, _ = faithful.reset()
    o2, _ = exact.reset()
    rng = np.random.default_rng(8)
    if faithful.finite:
        acts = rng.integers(0, 4 if name.startswith("extex") else 8, size=(steps, n, faithful.n_act)).astype(np.int32)
    else:
        acts = _actions(rng, steps, n)[..., : faithful.n_act]
    ang = [j for j, nm in enumerate(g["meta"]["state_names"]) if nm == "epsilon"]
    scale = np.maximum(np.abs(o1).max(axis=0), 1e-3)
    worst = 0.0
    for a in acts:
        o1, *_ = faithful.step(a)
        o2, *_ = exact.step(a)
        scale = np.maximum(scale, np.abs(o1).max(axis=0))
        d = np.abs(o1 - o2)
        for j in ang:
            d[:, j] = np.abs((o1[:, j] - o2[:, j] + 1.0) % 2.0 - 1.0)
        worst = max(worst, (d / scale).max())
    assert worst <= 1e-12, worst


def _replayed_time(steps):
    t = 0.0
    for _ in range(steps):
        t += TAU
    return t


def test_exact_grid_angle_is_accurate_and_the_faithful_one_follows_the_reference(oracle_lib):
    """PMSM at a constant 100 rad/s (p = 3), 10^5 steps.  The exact grid's angle is p omega K tau mod 2 pi to 1e-11 rad.  The faithful
    angle is the reference's recurrence eps += h / 6 (6 p omega) with h = fl(t + tau) - t, replayed here bit for bit: it differs from
    the exact one by p omega (t_K - K tau) = -3.0e-9 rad plus the rounding of the unwrapped float64 sum (-5.1e-9 rad here), so the closed
    form alone does not predict the difference of the angles."""
    n, steps, speed = 2, 10**5, 100.0
    faithful, exact = oracle_lib.Oracle(_pmsm_cfg(n, speed=speed)), oracle_lib.Oracle(_pmsm_cfg(n, speed=speed))
    exact.set_time_grid(True)
    pool = np.zeros((1, n, 3))
    for o in (faithful, exact):
        o.reset()
        o.rollout(pool, steps)
    p = _pmsm_cfg(1).motor_param[K.MP_P]
    y0 = _pmsm_cfg(1).init_ode[3]
    e_f, e_x = faithful.get_ode_state()[:, 3], exact.get_ode_state()[:, 3]
    # the exact grid against the true angle, reduced into [-pi, pi) with exact rational arithmetic
    two_pi = Fraction(2 * math.pi)
    true = Fraction(y0) + Fraction(p * speed) * steps * Fraction(TAU)
    true_red = float(true - two_pi * math.floor(true / two_pi))
    true_red = true_red - 2 * math.pi if true_red >= math.pi else true_red
    assert np.abs(e_x - true_red).max() < 1e-11, (e_x, true_red)
    # the faithful grid: the reference's own recurrence, replayed
    eps, t = y0, 0.0
    for _ in range(steps):
        tn = t + TAU
        h, t = tn - t, tn
        eps = eps + h / 6.0 * (6.0 * p * speed)
    assert np.all(e_f == eps)
    closed = float(p * speed * (Fraction(t) - steps * Fraction(TAU)))
    assert t == _replayed_time(steps) and abs(closed + 2.99e-9) < 1e-11
    recurrence_rounding = float(Fraction(eps) - true) - closed
    assert abs(recurrence_rounding) > abs(closed)  # why the angle itself cannot carry the closed form to 1e-3


def test_faithful_minus_exact_supply_voltage_follows_the_closed_form(oracle_lib):
    """The AC supply (50 Hz, U_N = 400 V) is evaluated at each step's start time.  After K = 10^5 steps the faithful-minus-exact u_sup
    is sqrt(2) U_N 2 pi f (t_{K-1} - (K-1) tau) cos(2 pi f (K-1) tau + phi), t replayed in Python: checked to 1e-3 relative."""
    n, steps = 4, 10**5

    def mk():
        cfg = _pmsm_cfg(n, supply="ac")
        cfg.supply_param[1], cfg.supply_param[2] = 0.25, 1.0  # fixed phase
        return cfg

    faithful, exact = oracle_lib.Oracle(mk()), oracle_lib.Oracle(mk())
    exact.set_time_grid(True)
    pool = np.zeros((1, n, 3))
    outs = []
    for o in (faithful, exact):
        o.reset()
        outs.append(o.rollout(pool, steps)[0])
    cfg = mk()
    lim, u_n, f, phi = cfg.limits[13], cfg.u_sup, cfg.supply_param[0], cfg.supply_param[1]
    t_start = _replayed_time(steps - 1)
    k_tau = (steps - 1) * Fraction(TAU)
    dt = float(Fraction(t_start) - k_tau)
    phase = 2 * math.pi * f * float(k_tau) + phi
    expected = math.sqrt(2) * u_n * 2 * math.pi * f * dt * math.cos(phase) / lim
    got = outs[0][:, 13] - outs[1][:, 13]
    assert abs(expected) > 1e-10
    assert np.abs(got / expected - 1).max() < 1e-3, (got, expected)
