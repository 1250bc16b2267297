"""Long episodes and 32-bit counter wrap-arounds of the primal step against the float64 oracle (run on the H100 with `-m gpu`).

RL training on a constant-speed load runs one episode for 10^5-10^6 steps and one handle for up to 2^32 steps.  These tests run the
device that long and jump both sides' clocks to the edges where the uint32 step count, the 64-bit Philox call id split into two words
and the fp32 record words of sub-episode bounds change behaviour.

- Long episodes are compared with the oracle on the device's time grid (`Oracle.set_time_grid(True)`, DESIGN §2 finding 12); the
  reference's own grid drifts away from it by more than the fp64 bar (test_reference_time_grid_drift).
- Parameters, speeds and initial states are fp32-exact, so the fp32 comparison measures the kernel's accumulation, not input rounding.
- Clock jumps: the device loads a checkpoint whose header carries the target clock, the oracle uses `Oracle.set_clock`; both reset.
"""
import math
import zlib
from fractions import Fraction

import numpy as np
import pytest

from helpers import load_golden, config_from_meta, switched_config
from gym_electric_motor_b200 import _cabi as K
from gpu_helpers import torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

TOL = {K.F64: 1e-9, K.F32: 1e-5}
N = 200  # not a multiple of the block size
DT_IDS = {K.F64: "f64", K.F32: "f32"}


def _f32(x):
    return float(np.float32(x))


def _fp32_exact(cfg):
    """round every physical input to the nearest float32, on both sides"""
    for arr, n in ((cfg.motor_param, K.MAX_MOTOR_PARAM), (cfg.load_param, 8), (cfg.init_ode, len(cfg.init_ode)), (cfg.supply_param, len(cfg.supply_param))):
        for j in range(n):
            arr[j] = _f32(arr[j])
    cfg.u_sup = _f32(cfg.u_sup)
    return cfg


def _sim(cfg):
    from gym_electric_motor_b200.vector_sim import VectorSim

    return VectorSim(cfg)


def _np(t):
    return t.double().cpu().numpy()


# ------------------------------------------------------------------------------------------------ A. long episodes, exact-grid oracle
def _case_cfg(case, dtype, n=N):
    """(config, action pool [P, n, n_act], angle columns) of one long-episode case; the same config builds the oracle (with K.F64)"""
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    ode_sm = [0.0, 0.5, -0.25, 0.75]
    solver = "rk4"
    if case in ("pmsm_const_pos", "pmsm_const_neg", "pmsm_ac", "pmsm_dead3_dq", "pmsm_extspeed"):
        name = {"pmsm_ac": "pmsm_cc_ac_rk4", "pmsm_extspeed": "pmsm_cc_extspeed_rk4"}.get(case, "pmsm_cc_rk4")
        speed = -125.0 if case == "pmsm_const_neg" else 100.0
        init = [speed] + ode_sm[1:]
    elif case == "synrm_poly":
        name, init = "synrm_cc_rk4", [0.0, 0.5, -0.25, 0.75]
    elif case == "eesm_poly":
        name, init = "eesm_cc_rk4", [0.0, 0.5, -0.25, 2.0, 0.75]
    elif case == "scim_flux":
        name, init = "scim_cc_flux_rk4", [50.0, 0.5, -0.25, 0.0625, 0.03125, 0.75]
    elif case == "permex_rc":
        name, init = "permex_sc_rc_rk4", [10.0, 0.5]
    elif case == "pmsm_fin_interlock":
        name, init = "pmsm_fin_sc_rk4_interlock", [100.0] + ode_sm[1:]
    else:
        raise ValueError(case)
    g = load_golden(name)
    cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=init[: len(g["reset_ode"])], dtype=dtype, solver=solver, ref_kind=K.REF_WIENER,
                           autoreset=K.AUTORESET_SAME_STEP, seed=2026)
    cfg.env_index_offset = 5 * n + 3
    cfg.n_constraints = 0  # limits out of reach: the episode must last the whole run (asserted on both sides)
    if cfg.load_kind == K.LOAD_EXT_SPEED:
        _ext_speed_horizon(cfg, g["meta"], 2000)
    if case == "pmsm_ac":
        cfg.supply_param[2] = 0.0  # random phase per env
    if case in ("synrm_poly", "eesm_poly"):
        # the speed is a state: a viscous polynomial load, and dq actions so that the voltages turn with the rotor and drive it to a
        # steady speed per env (SynRM 5-28 rad/s, EESM 1.5-9 rad/s)
        cfg.load_kind, cfg.action_dq = K.LOAD_POLY_STATIC, 1
        cfg.load_param[K.LP_A], cfg.load_param[K.LP_B], cfg.load_param[K.LP_C], cfg.load_param[K.LP_J_LOAD] = 0.0, 0.05, 0.0, 0.01
    if case == "eesm_poly":
        # with the registered env's L_m = 1.589 mH the reference's EESM model is open-loop unstable: at a constant 20 rad/s and zero
        # voltage its currents grow e-fold every ~0.04 s (the oracle reaches NaN within 2500 steps), so no open-loop episode is long
        cfg.motor_param[K.MP_L_M] = 0.0008
    if case == "pmsm_dead3_dq":
        cfg.dead_time_steps, cfg.action_dq = 3, 1
    if case == "pmsm_fin_interlock":
        assert cfg.finite and cfg.tau == 1e-5 and cfg.interlocking_time > 0
    _fp32_exact(cfg)
    names = g["meta"]["state_names"]
    ang = [j for j, nm in enumerate(names) if nm in ("epsilon",)]
    if cfg.finite:
        n_act = 1
        pool = rng.integers(0, 8, size=(4, n, n_act)).astype(np.int32)
    else:
        from oracle.gem_oracle import Oracle

        n_act = Oracle(cfg).n_act
        hold = rng.uniform(-0.25, 0.25, size=(1, n, n_act))
        pool = (hold + rng.uniform(-0.05, 0.05, size=(4, n, n_act))).astype(np.float32).astype(np.float64)
        if case == "permex_rc":
            pool = np.abs(pool) * 0.5
        if case in ("synrm_poly", "eesm_poly"):  # d, q (and excitation) voltages of one sign: the rotor settles at a speed of one sign
            pool = (0.02 + 0.5 * np.abs(pool) * 0.25).astype(np.float32).astype(np.float64)
            if case == "eesm_poly":
                pool[..., 2] = (0.01 * pool[..., 2]).astype(np.float32)
    return cfg, pool, ang


def _ext_speed_horizon(cfg, meta, steps):
    """ExternalSpeedLoad: a tabulated profile of `steps` steps (fp32-exact samples), so that a longer run goes past its horizon and then
    repeats the profile's last step"""
    es, per = meta["ext_speed"], 2 * cfg.solver_nsteps
    j = np.arange(per * steps + 2 * per + 1)
    t = j * (cfg.tau / per) + es["tau"]
    tab = np.ascontiguousarray((es["o"] + es["a"] * np.sin(2 * np.pi * es["f"] * t)).astype(np.float32).astype(np.float64))
    cfg.ext_speed_table, cfg.ext_speed_len = tab.ctypes.data, len(tab)
    cfg._keepalive = tab
    return cfg


def _run_long(torch, case, dtypes, steps, chunk, every, n=N):
    """Devices of the given dtypes and the exact-grid oracle over `steps` steps (device: fused chunks of `chunk` steps, every step recorded and
    checked for terminations; oracle: `rollout` between samples).  Returns ({dtype: [worst error of the obs samples and the ODE state, per chunk]}, devices, oracle,
    {dtype: largest |omega_device - omega_oracle| at the chunk ends})."""
    from oracle.gem_oracle import Oracle

    ocfg, pool, ang = _case_cfg(case, K.F64, n)
    ora = Oracle(ocfg)
    ora.set_time_grid(True)
    devs = {dt: _sim(_case_cfg(case, dt, n)[0]) for dt in dtypes}
    o_obs, _ = ora.reset()
    for dev in devs.values():
        dev.reset()
    P = pool.shape[0]
    acts = {dt: torch.as_tensor(pool, device="cuda").to(dev.act_dtype) for dt, dev in devs.items()}
    scale = np.maximum(np.abs(o_obs).max(axis=0), 1e-3)
    worst = {dt: [] for dt in dtypes}
    dspeed = {dt: 0.0 for dt in dtypes}
    s0 = 0
    while s0 < steps:
        kc = min(chunk, steps - s0)
        idx = torch.arange(s0, s0 + kc, device="cuda") % P
        outs = {}
        for dt, dev in devs.items():
            obs, _, _, term = dev.rollout(acts[dt][idx].contiguous(), record_every=1)
            assert int(term.sum()) == 0, f"{case}: an env terminated in steps [{s0}, {s0 + kc})"
            outs[dt] = obs[every - 1::every].double().cpu().numpy()
        pos = s0
        for dt in dtypes:
            worst[dt].append(0.0)
        for q, j in enumerate(range(every - 1, kc, every)):
            o_obs, _, _, o_term = ora.rollout(np.roll(pool, -(pos % P), axis=0), s0 + j + 1 - pos)
            pos = s0 + j + 1
            assert not o_term.any()
            scale = np.maximum(scale, np.abs(o_obs).max(axis=0))
            for dt in dtypes:
                d = outs[dt][q]
                diff = np.abs(d - o_obs)
                for c in ang:  # normalised angles live on a circle of circumference 2
                    diff[:, c] = np.abs((d[:, c] - o_obs[:, c] + 1.0) % 2.0 - 1.0)
                worst[dt][-1] = max(worst[dt][-1], (diff / scale).max())
        if pos < s0 + kc:
            ora.rollout(np.roll(pool, -(pos % P), axis=0), s0 + kc - pos)
        s0 += kc
        y_o = ora.get_ode_state()
        for dt, dev in devs.items():
            y_d = _np(dev.get_ode_state())
            dy = np.abs(y_d - y_o)
            dspeed[dt] = max(dspeed[dt], dy[:, 0].max())
            if ocfg.motor_kind >= K.MOTOR_PMSM:  # the angle, in radians
                dy[:, -1] = np.abs((y_d[:, -1] - y_o[:, -1] + math.pi) % (2 * math.pi) - math.pi)
            worst[dt][-1] = max(worst[dt][-1], (dy / np.maximum(np.abs(y_o).max(axis=0), 1e-3)).max())
    for dev in devs.values():
        assert dev.clock()[1] == steps
    return worst, devs, ora, dspeed


LONG_CASES = ["pmsm_const_pos", "pmsm_const_neg", "synrm_poly", "eesm_poly", "pmsm_ac", "pmsm_dead3_dq", "pmsm_extspeed", "permex_rc", "scim_flux",
              "pmsm_fin_interlock"]


@pytest.mark.parametrize("case", LONG_CASES)
def test_long_episode_matches_exact_grid_oracle(torch_cuda, case):
    """One episode of 10^5 steps in fused chunks, fp64 and fp32 devices: every 2500th step and every chunk end's ODE state against the
    exact-grid oracle, angles on the circle; no env may terminate.  fp64 holds 1e-9 column-relative everywhere (worst measured 5e-12).
    fp32 holds 1e-5 where the speed is fixed (worst measured 1.4e-6 after 10^5 steps); where it is not, DESIGN §2 finding 12 has the
    measured reasons for the other fp32 bars:
    - pmsm_extspeed, synrm_poly, eesm_poly: the speed is an fp32 state, so the angle drifts by up to p |omega| 2^-24 t (7e-5 of pi
      after 10 s at 122 rad/s);
    - permex_rc / scim_flux: small columns (the armature current at 3 % of its limit; the field-frame d current and voltage) carry a
      steady fp32 offset of up to 3.8e-4 / 5.7e-5 of their scale: the bar is that it does not grow over the second half of the run;
    - pmsm_fin_interlock: legs waiting in their interlock state switch by the sign of their current, and in fp32 that sign flips
      for most envs within 10^5 steps at tau = 1e-5 (187 of 200): fp64 only."""
    chunk = 997 * 5 if case == "pmsm_dead3_dq" else 10**4  # 997: dead-time ring positions cross launch boundaries
    steps = 10**5
    worst, _, ora, dspeed = _run_long(torch_cuda, case, (K.F64, K.F32) if case != "pmsm_fin_interlock" else (K.F64,), steps, chunk, 2500)
    w64 = np.array(worst[K.F64])
    print(f"{case}: worst error f64 {w64.max():.3e}" + (f", f32 {max(worst[K.F32]):.3e}" if K.F32 in worst else ""))
    assert w64.max() < TOL[K.F64], w64
    if K.F32 not in worst:
        return
    w32 = np.array(worst[K.F32])
    cfg = ora.cfg
    if case == "pmsm_extspeed":
        omega = np.abs(ora.get_ode_state()[:, 0]).max()
        assert w32.max() < TOL[K.F32] + cfg.motor_param[K.MP_P] * omega * 2.0**-24 * steps * cfg.tau / math.pi, w32
    elif case in ("synrm_poly", "eesm_poly"):
        # near its load equilibrium the fp32 speed state stalls where an RK4 increment falls below half an ulp of omega (DESIGN §2
        # finding 12): the speed itself must stay within 2e-4 of the oracle's, and every other fp32 error must be what that offset
        # explains, the angle integrating p d_omega over the run (and the abc / dq columns following the angle)
        omega = np.abs(ora.get_ode_state()[:, 0]).max()
        print(f"{case}: fp32 speed offset {dspeed[K.F32]:.3e} rad/s of {omega:.3g}")
        assert dspeed[K.F32] < 2e-4 * omega, dspeed
        assert w32.max() < TOL[K.F32] + cfg.motor_param[K.MP_P] * dspeed[K.F32] * steps * cfg.tau, w32
    elif case in ("permex_rc", "scim_flux"):
        half = len(w32) // 2
        assert w32.max() < 1e-3 and w32[half:].max() <= 1.1 * w32[:half].max(), w32
    else:
        assert w32.max() < TOL[K.F32], w32


# ------------------------------------------------------------------------------------------------ B. the reference's time grid
MILLION_ENVS = 32  # 10^6 oracle steps of 32 envs take ~16 s of one CPU core


def test_reference_time_grid_drift(torch_cuda):
    """Finding 12 (DESIGN §2): PMSM at a constant 100 rad/s (p = 3) for 10^6 steps.  The device integrates every step over exactly tau and
    matches the exact-grid oracle, fp64 to 1e-9 and fp32 (the double-float angle) to 1e-5; the reference's grid integrates over
    fl(t + tau) - t with t accumulated, and its unwrapped float64 angle rounds at the ulp of ~3e4 rad.  Both put the faithful oracle's
    angle off the true p omega K tau, by more than the fp64 bar: the fp64 device's distance from the faithful oracle is exactly that error."""
    steps, n = 10**6, MILLION_ENVS
    worst, devs, _, _ = _run_long(torch_cuda, "pmsm_const_pos", (K.F64, K.F32), steps, 10**5, 50000, n)
    print(f"10^6 steps, constant speed: worst error f64 {max(worst[K.F64]):.3e}, f32 {max(worst[K.F32]):.3e}")
    assert max(worst[K.F64]) < TOL[K.F64] and max(worst[K.F32]) < TOL[K.F32], worst
    dev = devs[K.F64]
    from oracle.gem_oracle import Oracle

    cfg, pool, _ = _case_cfg("pmsm_const_pos", K.F64, n)
    faithful = Oracle(cfg)
    faithful.reset()
    faithful.rollout(pool, steps)
    e_dev, e_f = _np(dev.get_ode_state())[:, 3], faithful.get_ode_state()[:, 3]
    p, w, y0 = cfg.motor_param[K.MP_P], cfg.init_ode[0], cfg.init_ode[3]
    true = Fraction(y0) + Fraction(p * w) * steps * Fraction(1e-4)
    t = 0.0
    for _ in range(steps):
        t += 1e-4
    closed = float(Fraction(p * w) * (Fraction(t) - steps * Fraction(1e-4)))
    faithful_err = float(Fraction(float(e_f[0])) - true)
    got = (e_dev - e_f + math.pi) % (2 * math.pi) - math.pi
    print(f"time grid: device vs exact-grid oracle {max(worst[K.F64]):.3e}; t_K - K tau = {t - steps * 1e-4:.3e} s, p omega (t_K - K tau) = {closed:.3e} rad, faithful angle - true = {faithful_err:.3e} rad, "
          f"device - faithful = {got.min():.3e} .. {got.max():.3e} rad")
    assert np.all(e_f == e_f[0])
    assert np.abs(got + faithful_err).max() < 1e-9 * math.pi
    assert np.abs(got).min() > 1e-9 * math.pi and abs(closed) > 1e-9 * math.pi


def test_million_step_ac_supply_episode(torch_cuda):
    """PMSM behind the single-phase AC supply, a random phase per env, for 10^6 steps: the supply phase is a double-float accumulator in
    fp32 (`sup_phase` advanced by `sup_kph` every step); fp64 1e-9, fp32 1e-5 against the exact-grid oracle."""
    worst, _, _, _ = _run_long(torch_cuda, "pmsm_ac", (K.F64, K.F32), 10**6, 10**5, 50000, MILLION_ENVS)
    print(f"10^6 steps, AC supply: worst error f64 {max(worst[K.F64]):.3e}, f32 {max(worst[K.F32]):.3e}")
    assert max(worst[K.F64]) < TOL[K.F64] and max(worst[K.F32]) < TOL[K.F32], worst


# ------------------------------------------------------------------------------------------------ C. long periodic sub-episodes
PERIODIC = [K.REF_SINUS, K.REF_SAWTOOTH, K.REF_TRIANGULAR, K.REF_STEP]


def _periodic_cfg(dtype, kinds, freq, n=N):
    g = load_golden("pmsm_cc_rk4")
    cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=[100.0, 0.5, -0.25, 0.75], dtype=dtype, solver="rk4", ref_kind=K.REF_WIENER,
                           autoreset=K.AUTORESET_SAME_STEP, seed=777)
    cfg.env_index_offset = 11
    cfg.n_constraints = 0
    for r in range(2):
        cfg.ref_kind[r] = kinds[r]
        cfg.ref_margin_lo[r], cfg.ref_margin_hi[r] = -1.0, 1.0
        cfg.ref_amp_lo[r], cfg.ref_amp_hi[r] = 0.25, 0.5
        cfg.ref_freq_lo[r], cfg.ref_freq_hi[r] = freq
        cfg.ref_off_lo[r], cfg.ref_off_hi[r] = -0.25, 0.25
        cfg.ref_len_lo[r], cfg.ref_len_hi[r] = 2 * 10**4, 10**5
    return _fp32_exact(cfg)


@pytest.mark.parametrize("freq", [(1.0, 10.0), (20.0, 400.0)], ids=["1-10Hz", "20-400Hz"])
@pytest.mark.parametrize("kinds", [(K.REF_SINUS, K.REF_TRIANGULAR), (K.REF_SAWTOOTH, K.REF_STEP)], ids=["sin_tri", "saw_step"])
def test_long_periodic_sub_episodes_match_oracle(torch_cuda, kinds, freq):
    """Sub-episodes of 2e4..1e5 steps over a 1.2e5-step run, fp64 and fp32 devices: every 1000th reference value against the oracle."""
    from oracle.gem_oracle import Oracle

    steps, every = 12 * 10**4, 1000
    devs = {dt: _sim(_periodic_cfg(dt, kinds, freq)) for dt in (K.F64, K.F32)}
    ora = Oracle(_periodic_cfg(K.F64, kinds, freq))
    ora.set_time_grid(True)
    ora.reset()
    pool = np.zeros((1, N, 3))
    errs = {dt: [] for dt in devs}
    for dev in devs.values():
        dev.reset()
    for _ in range(steps // every):
        _, o_ref, _, _ = ora.rollout(pool, every)
        for dt, dev in devs.items():
            _, d_ref, _, _ = dev.rollout(torch_cuda.zeros((every, N, 3), device="cuda", dtype=dev.act_dtype))
            errs[dt].append(np.abs(_np(d_ref) - o_ref))
    for dtype in (K.F64, K.F32):
        err = np.stack(errs[dtype])  # [samples, N, slot]
        print(f"periodic {kinds} {freq} {DT_IDS[dtype]}: worst per slot {err.max(axis=(0, 1))}, > bar: {(err > TOL[dtype]).sum(axis=(0, 1))} of {err.shape[0] * N}")
        for r, kind in enumerate(kinds):
            e = err[:, :, r]
            # no exemption at the discontinuities of the sawtooth and the step: the phase and the step's edge test are the oracle's double
            # arithmetic in both dtypes, so a sample cannot land on the other side of an edge
            assert e.max() < TOL[dtype], (DT_IDS[dtype], kind, e.max())


# ------------------------------------------------------------------------------------------------ D. clock edges
def _switched_edge_cfg(dtype, n=N):
    """PermExDc whose one reference slot switches between a Wiener, a sinusoidal and a step generator every 7..25 steps, dead time 3"""
    kinds = [dict(kind=K.REF_WIENER, margin=(-0.5, 0.5), length=(2, 9)), dict(kind=K.REF_SINUS, length=(3, 17)),
             dict(kind=K.REF_STEP, amp=(0.05, 0.2), length=(3, 17))]
    cfg = switched_config(n, kinds, [0.3, 0.4, 0.3], (7, 25), seed=21, dtype=dtype)
    cfg.env_index_offset = 1 << 33
    cfg.dead_time_steps = 3
    return _fp32_exact(cfg)


def _edge_cfg(dtype, n=N, gen="periodic"):
    """PMSM with a Wiener slot and a sinusoidal slot of short sub-episodes (starts and ends land on the edges), dead time 3 (2^32 mod 3 != 0);
    gen="switched": _switched_edge_cfg"""
    if gen == "switched":
        return _switched_edge_cfg(dtype, n)
    g = load_golden("pmsm_cc_rk4")
    cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=[100.0, 0.5, -0.25, 0.75], dtype=dtype, solver="rk4", ref_kind=K.REF_WIENER,
                           autoreset=K.AUTORESET_SAME_STEP, seed=99)
    cfg.env_index_offset = 1 << 33  # the env index's high word feeds the Philox counter too
    cfg.n_constraints = 0
    cfg.dead_time_steps = 3
    cfg.ref_len_lo[0], cfg.ref_len_hi[0] = 2, 9
    cfg.ref_kind[1] = K.REF_SINUS
    cfg.ref_amp_lo[1], cfg.ref_amp_hi[1] = 0.05, 0.5
    cfg.ref_freq_lo[1], cfg.ref_freq_hi[1] = 20.0, 400.0
    cfg.ref_off_lo[1], cfg.ref_off_hi[1] = -0.4, 0.4
    cfg.ref_len_lo[1], cfg.ref_len_hi[1] = 3, 17
    return _fp32_exact(cfg)


def _clock_offsets(sim):
    """byte offsets of the call id and the step count in the checkpoint header, found by their values after a known run"""
    c, s = sim.clock()
    assert c != s
    head = np.frombuffer(sim.state_dict()["blob"][:128].tobytes(), dtype=np.uint64)
    oc, os_ = np.nonzero(head == c)[0], np.nonzero(head == s)[0]
    assert len(oc) == 1 and len(os_) == 1, (head, c, s)
    return 8 * int(oc[0]), 8 * int(os_[0])


def _jump(sim, offsets, call_id, n_steps):
    """put a device handle at (call id, step count) through its checkpoint header; the caller resets it afterwards"""
    blob = sim.state_dict()["blob"].copy()
    blob[offsets[0]:offsets[0] + 8] = np.frombuffer(np.uint64(call_id).tobytes(), dtype=np.uint8)
    blob[offsets[1]:offsets[1] + 8] = np.frombuffer(np.uint64(n_steps).tobytes(), dtype=np.uint8)
    sim.load_state_dict({"blob": blob})
    assert sim.clock() == (call_id, n_steps)


def _offsets_for(dtype):
    probe = _sim(_edge_cfg(dtype, 8))
    probe.step(np.zeros((8, 3)))
    probe.step(np.zeros((8, 3)))
    return _clock_offsets(probe)


@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
def test_jumped_device_handle_equals_naturally_stepped_one(torch_cuda, dtype):
    """Harness check: a handle stepped to a clock and a handle jumped there by its checkpoint header run identically after a reset."""
    n = 64
    rng = np.random.default_rng(4)
    natural, jumped = _sim(_edge_cfg(dtype, n)), _sim(_edge_cfg(dtype, n))
    for _ in range(23):
        natural.step(0.2 * rng.uniform(-1, 1, size=(n, 3)))
    natural.reset()
    natural.step(np.zeros((n, 3)))
    clock = natural.clock()
    assert clock == (26, 24)  # create's reset is call 1, 23 steps, a reset, a step
    _jump(jumped, _offsets_for(dtype), *clock)
    for a, b in zip(natural.reset(), jumped.reset()):
        assert torch_cuda.equal(a, b)
    acts = torch_cuda.as_tensor(0.2 * rng.uniform(-1, 1, size=(40, n, 3)), device="cuda").to(natural.act_dtype)
    for x, y in zip(natural.rollout(acts, record_every=1), jumped.rollout(acts, record_every=1)):
        assert torch_cuda.equal(x, y)
    assert natural.clock() == jumped.clock()


EDGES = [(2**31 - 2**23 - 50 + 7, 2**31 - 2**23 - 50), (2**31 - 50 + 7, 2**31 - 50), (2**32 - 50 + 7, 2**32 - 50),
         (2**32 - 52, 1000), (3 * 2**32 - 51, 1000)]
EDGE_IDS = ["steps_2^31-2^23", "steps_2^31", "steps_2^32", "call_2^32_even", "call_3x2^32_odd"]


def _cmp(d, o, scale, tol, what):
    d = d.double().cpu().numpy()
    if d.ndim == 1:
        d, o = d[:, None], o[:, None]
    err = (np.abs(d - o) / scale).max()
    assert err < tol, (what, err)


@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("clock", EDGES, ids=EDGE_IDS)
@pytest.mark.parametrize("gen", ["periodic", "switched"])
def test_clock_edges_match_oracle(torch_cuda, gen, clock, dtype):
    """300 steps across an edge of the step count or the call id (the edge falls on step 50): three handles jumped to the same clock.
    - `twin`: single steps with the host clock, against the oracle at the parity bars;
    - `fused`: single steps and fused rollouts, one of them straddling the edge;
    - `graph`: the device clock, eager steps, then a CUDA graph of 10 steps replayed across the edge, then a rollout.
    `fused` and `graph` must equal `twin` bit for bit, and all clocks must agree at the end."""
    from oracle.gem_oracle import Oracle

    torch = torch_cuda
    n, tol, total = N, TOL[dtype], 300
    offs = _offsets_for(dtype)
    twin, fused, graph = (_sim(_edge_cfg(dtype, n, gen)) for _ in range(3))
    ora = Oracle(_edge_cfg(K.F64, n, gen))
    for s in (twin, fused, graph):
        _jump(s, offs, *clock)
    ora.set_clock(*clock)
    o_obs, o_ref = ora.reset()
    resets = [tuple(x.clone() for x in s.reset()) for s in (twin, fused, graph)]
    for r in resets[1:]:
        assert all(torch.equal(x, y) for x, y in zip(r, resets[0]))
    scale = np.maximum(np.abs(o_obs).max(axis=0), 1e-3)
    _cmp(resets[0][0], o_obs, scale, tol, "reset obs")
    _cmp(resets[0][1], o_ref, 1.0, 20 * tol, "reset ref")
    rng = np.random.default_rng(clock[1] % 1000)
    acts = (0.2 * rng.uniform(-1, 1, size=(total, n, ora.n_act))).astype(np.float32).astype(np.float64)
    ta = torch.as_tensor(acts, device="cuda").to(twin.act_dtype)

    ref_out = [tuple(x.clone() for x in twin.step(ta[k])) for k in range(total)]
    for k in range(total):
        o_obs, o_ref, o_rew, o_term = ora.step(acts[k])
        d = ref_out[k]
        scale = np.maximum(scale, np.abs(o_obs).max(axis=0))
        _cmp(d[0], o_obs, scale, tol, ("obs", k))
        _cmp(d[1], o_ref, 1.0, 20 * tol, ("ref", k))
        _cmp(d[2], o_rew, 1.0, 20 * tol, ("rew", k))
        assert not o_term.any() and not d[3].any()

    mismatches = []  # (phase, first differing step) of every phase: one phase's failure does not hide another's

    def check(outs, k0, what):
        for j, o in enumerate(outs):
            if not all(torch.equal(x, y) for x, y in zip(o, ref_out[k0 + j])):
                mismatches.append((what, k0 + j))
                return

    # fused: 20 single steps, a rollout over steps 20..89 (the edge at 50), 30 single steps, a rollout to the end
    k = 0
    for kind, m in (("step", 20), ("roll", 70), ("step", 30), ("roll", total - 120)):
        if kind == "step":
            outs = [tuple(x.clone() for x in fused.step(ta[k + j])) for j in range(m)]
        else:
            rec = fused.rollout(ta[k:k + m].contiguous(), record_every=1)
            outs = [tuple(x[j] for x in rec) for j in range(m)]
        check(outs, k, ("fused", kind))
        k += m
    # graph: device clock, 30 eager steps, a graph of 10 steps replayed 3 times over steps 30..59, a rollout to the end
    graph.set_device_clock(True)
    check([tuple(x.clone() for x in graph.step(ta[j])) for j in range(30)], 0, "device clock")
    abuf = ta[30:40].clone()
    g, rec = torch.cuda.CUDAGraph(), []
    with torch.cuda.graph(g):
        for j in range(10):
            rec.append(tuple(x.clone() for x in graph.step(abuf[j])))
    for r in range(3):
        abuf.copy_(ta[30 + 10 * r:40 + 10 * r])
        g.replay()
        torch.cuda.synchronize()
        check([tuple(x.clone() for x in o) for o in rec], 30 + 10 * r, "graph replay")
    rec = graph.rollout(ta[60:].contiguous(), record_every=1)
    check([tuple(x[j] for x in rec) for j in range(total - 60)], 60, "device-clock rollout")
    want = (clock[0] + 1 + total, clock[1] + total)
    clocks = {"twin": twin.clock(), "fused": fused.clock(), "graph": graph.clock(), "oracle": ora.clock()}
    assert not mismatches and all(c == want for c in clocks.values()), (mismatches, clocks, want)


# ------------------------------------------------------------------------------------------------ E. tangent launches at the edges
@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("clock", [EDGES[2], EDGES[4]], ids=[EDGE_IDS[2], EDGE_IDS[4]])
@pytest.mark.parametrize("launch", ["returns", "jacobians", "param_sens", "return_grads"])
def test_tangent_launch_across_edge_equals_rollout(torch_cuda, launch, clock, dtype):
    """Each tangent loop carries the call id and the step count itself: across an edge its primal outputs, clock and checkpoint equal
    those of rollout(record_every=1) on a twin."""
    n, kk = 96, 120
    offs = _offsets_for(dtype)
    cfg = _edge_cfg(dtype, n)
    cfg.dead_time_steps = 0  # the tangent rollouts refuse a dead time
    sims = [_sim(cfg) for _ in range(2)]
    for s in sims:
        _jump(s, offs, *clock)
        s.reset()
    tan, ref_sim = sims
    rng = np.random.default_rng(12)
    ta = torch_cuda.as_tensor(0.2 * rng.uniform(-1, 1, size=(kk, n, 3)), device="cuda").to(tan.act_dtype).contiguous()
    obs, ref, rew, term = ref_sim.rollout(ta, record_every=1)
    if launch == "returns":
        _, end, (o_last, r_last) = tan.rollout_returns(ta, 0.9)
        got = [(o_last, obs[-1]), (r_last, ref[-1])]
        assert int((end != kk).sum()) == 0
    elif launch == "return_grads":
        _, end, (o_last, r_last), _, _ = tan.rollout_return_grads(ta, 0.9)
        got = [(o_last, obs[-1]), (r_last, ref[-1])]
    elif launch == "jacobians":
        _, outs = tan.rollout_jacobians(ta)
        got = list(zip(outs, (obs, ref, rew, term)))
    else:
        _, outs = tan.rollout_param_sens(ta, [K.MP_R_S])
        got = list(zip(outs, (obs, ref, rew, term)))
    for a, b in got:
        assert torch_cuda.equal(a, b)
    assert tan.clock() == ref_sim.clock() == (clock[0] + 1 + kk, clock[1] + kk)
    assert np.array_equal(tan.state_dict()["blob"], ref_sim.state_dict()["blob"])


# ------------------------------------------------------------------------------------------------ F. snapshots across the wrap
@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("gen", ["periodic", "switched"])
def test_snapshots_across_the_wrap_continue_their_source(torch_cuda, gen, dtype):
    """Envs packed with open sub-episodes 20 steps before the step count wraps at 2^32 and restored with rng="source" into a handle at a
    small clock continue their source's trajectory bit for bit across the wrap; and the reverse: envs packed at the small clock and
    restored into the handle 20 steps before the wrap, which they then cross.  Both snapshots are taken before either handle moves on."""
    torch = torch_cuda
    n, m, steps = 64, 24, 60

    def cfg():
        c = _edge_cfg(dtype, n, gen)
        c.dead_time_steps = 0
        return c

    offs = _offsets_for(dtype)
    high, low = _sim(cfg()), _sim(cfg())
    _jump(high, offs, 2**32 + 5, 2**32 - 30)
    high.reset()
    low.reset()
    rng = np.random.default_rng(31)
    n_act = high.n_act
    warm = torch.as_tensor(0.2 * rng.uniform(-1, 1, size=(10, n, n_act)), device="cuda").to(high.act_dtype)
    high.rollout(warm, record_every=1)
    low.rollout(warm[:7].contiguous(), record_every=1)
    assert high.clock()[1] == 2**32 - 20 and low.clock()[1] == 7
    src_rows, dst_rows = np.arange(m), np.arange(n - m, n)
    snap_high, snap_low = high.snapshot(src_rows, rng=True), low.snapshot(src_rows, rng=True)
    low.restore(snap_high, idx=dst_rows, rng="source")
    high.restore(snap_low, idx=dst_rows, rng="source")
    acts = torch.as_tensor(0.2 * rng.uniform(-1, 1, size=(steps, n, n_act)), device="cuda").to(high.act_dtype)
    acts[:, dst_rows] = acts[:, src_rows]
    a = high.rollout(acts, record_every=1)
    b = low.rollout(acts, record_every=1)
    for x, y in zip(a, b):
        assert torch.equal(x[:, src_rows], y[:, dst_rows]), "high -> low"
        assert torch.equal(y[:, src_rows], x[:, dst_rows]), "low -> high"
    assert high.clock()[1] == 2**32 + steps - 20
