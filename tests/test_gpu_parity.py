"""GPU parity tests (run on the H100 with `-m gpu`): the CUDA path, called through the C-ABI, against
 (1) the golden trajectories recorded from the unmodified reference, and
 (2) the float64 CPU oracle on many envs with random actions, auto-reset and the Wiener reference generator.

Tolerances: float64 build 1e-9 column-relative (algorithm-identical to the oracle); float32 build 1e-5
column-relative — the bar BASELINE.json's north_star sets for state trajectories.
"""
import numpy as np
import pytest

from helpers import golden_reset_state, switched_config, col_rel_err, config_from_meta, golden_names, load_golden, replay_golden
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

TOL = {K.F64: 1e-9, K.F32: 1e-5}
# dopri5 goldens are compared against RK4 with 2 sub-steps: accuracy of the substitute solver, not identity
TOL_DOPRI = {K.F64: 2e-6, K.F32: 1e-5}
# SCIM with dq actions transformed by the FluxObserver's angle: psi_obs is a running sum of current samples with heavy cancellation
# under random actions, so rounding-level differences of the currents (1e-7 relative in fp32, 1e-16 in fp64) come back amplified
# ~100x through angle(psi_obs) into the applied voltages.  Conditioning of the configuration, not of the kernel: the same
# trajectories without that feedback (scim_cc_flux_rk4) hold the plain tolerance.
TOL_OBSERVER_FEEDBACK = {K.F64: 1e-8, K.F32: 1e-3}


def _tol(name, dtype, is_dopri=False, batch=False):
    if "flux_dq" in name or "flux_cossin_dead1" in name:
        return TOL_OBSERVER_FEEDBACK[dtype]
    if name.startswith("dfim_fin") and dtype == K.F32:
        # tau = 1e-5: the rotor flux stays at ~1 % of nominal for the whole run, so the field-frame (dq) columns carry the fp32
        # flux noise divided by that small magnitude; the frame-independent columns hold 2e-6
        return 3e-5
    return (TOL_DOPRI if is_dopri else TOL)[dtype]


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


class DeviceAdapter:
    """Gives VectorSim the numpy reset/step/set_reference API that helpers.replay_golden drives."""

    def __init__(self, cfg):
        from gym_electric_motor_b200.vector_sim import VectorSim

        self.sim = VectorSim(cfg)

    def reset(self, mask=None):
        obs, ref = self.sim.reset(mask)
        return obs.double().cpu().numpy(), ref.double().cpu().numpy()

    def step(self, action):
        obs, ref, rew, term = self.sim.step(np.asarray(action))
        return obs.double().cpu().numpy(), ref.double().cpu().numpy(), rew.double().cpu().numpy(), term.cpu().numpy()

    def set_reference(self, r):
        self.sim.set_reference(r)


def _golden_cases():
    out = []
    for name in golden_names():
        for dt in (K.F64, K.F32):
            out.append(pytest.param(name, dt, id=f"{name}-{'f64' if dt == K.F64 else 'f32'}"))
    return out


@pytest.mark.parametrize("name,dtype", _golden_cases())
def test_device_reproduces_reference_trajectory(torch_cuda, name, dtype):
    g = load_golden(name)
    solver = g["meta"]["case"]["solver"]
    is_dopri = solver == "dopri5"
    if is_dopri and name == "pmsm_fin_sc_dopri5":
        pytest.skip("the reference's default dopri5 silently drops steps here (scipy 'step size too small'); "
                    "only the oracle restates that pathology, see DESIGN.md")
    cfg = config_from_meta(g["meta"], reset_ode=g["reset_ode"], dtype=dtype, solver="rk4x2" if is_dopri else solver)
    sim = DeviceAdapter(cfg)
    out = replay_golden(sim, g)
    tol = _tol(name, dtype, is_dopri)
    assert np.abs(out["reset_state"] - golden_reset_state(g)).max() < 1e-6
    if g["meta"]["motor_class"] in ("SquirrelCageInductionMotor", "DoublyFedInductionMotor"):
        # i_sd/i_sq/u_sd/u_sq are expressed in the rotor-flux frame, angle = atan2(psi_b, psi_a)
        # (physical_systems.py:765-769).  While the flux is still (numerically) zero after a reset that angle is
        # ill-conditioned — decided by round-off noise in the reference itself (|psi| ~ 1e-28 at step 1) and by fp32
        # ripple noise (~1e-9 Wb) on the device.  Below 1e-3 Wb (0.2 % of nominal flux) the dq columns are therefore
        # compared through their frame-invariant magnitude; all other columns are always compared as they are.
        psi = np.vstack([g["reset_ode"][None, :], g["ode_states"][:-1]])[:, 3:5]
        weak = np.hypot(psi[:, 0], psi[:, 1]) < 1e-3
        for arr in (out["states"], g["states"]):
            for a, b in (((5, 6), (10, 11)) if g["meta"]["motor_class"] == "SquirrelCageInductionMotor" else ((5, 6), (10, 11), (15, 16), (20, 21))):  # dq pairs
                arr[weak, a] = np.hypot(arr[weak, a], arr[weak, b])
                arr[weak, b] = 0.0
    err = col_rel_err(out["states"], g["states"])
    cols = np.abs(out["states"] - g["states"]).max(axis=0) / np.maximum(np.abs(g["states"]).max(axis=0), 1e-12)
    assert err < tol, f"{name}: column-relative state error {err:.3e}; per column {np.array2string(cols, precision=1)}"
    # terminations / rewards: identical unless a constraint sits within rounding of its threshold
    mism = np.nonzero(out["terminated"] != g["terminated"])[0]
    assert len(mism) == 0, f"termination mismatch at steps {mism[:5]}"
    assert np.abs(out["rewards"] - g["rewards"]).max() < 10 * tol


BATCH_CASES = [
    ("pmsm_cc_rk4", "rk4"), ("pmsm_cc_euler3", "euler3"), ("pmsm_sc_polyload_rk4", "rk4"), ("pmsm_fin_sc_rk4_interlock", "rk4"),
    ("synrm_cc_rk4", "rk4x2"), ("eesm_cc_rk4", "rk4"), ("eesm_fin_cc_rk4", "rk4"), ("scim_cc_rk4", "rk4"),
    ("scim_fin_cc_interlock_rk4", "rk4"), ("permex_cc_euler_10k", "euler"), ("permex_fin4qc_interlock_rk4", "rk4"),
    ("series_cc_rk4", "rk4"), ("shunt_cc_rk4", "rk4"), ("extex_cc_rk4", "rk4"),
    # RC voltage supply behind continuous / finite, single / multi converters
    ("permex_sc_rc_rk4", "rk4"), ("permex_fin_sc_rc_interlock_rk4", "rk4"), ("pmsm_fin_cc_rc_rk4", "rk4"), ("eesm_fin_cc_rc_rk4", "rk4"),
    ("pmsm_cc_rc_interlock_euler3", "euler3"), ("dfim_cc_rc_rk4", "rk4"),
    # ExternalSpeedLoad: tabulated speed profile, incl. the Euler-n look-ahead quirk and RK4 sub-steps
    ("pmsm_cc_extspeed_rk4", "rk4"), ("permex_cc_extspeed_euler3", "euler3"), ("scim_cc_extspeed_rk4x2", "rk4x2"), ("pmsm_fin_cc_extspeed_euler", "euler"),
    # single-phase AC supply; the batch test draws a random phase per env and reset (goldens: fixed phase)
    ("permex_sc_ac_rk4", "rk4"), ("series_fin_cc_ac_interlock_rk4", "rk4"), ("pmsm_cc_ac_rk4", "rk4"),
    ("dfim_cc_flux_dq_rk4", "rk4"), ("dfim_cc_rk4", "rk4"), ("dfim_sc_rk4", "rk4x2"), ("dfim_fin_sc_interlock_rk4", "rk4"), ("dfim_cc_interlock_rk4", "euler3"),
    # multi converters whose sub-converters have different interlocking times (per-slot dead time; three switching segments when finite)
    ("extex_cc_interlock2_rk4", "rk4"), ("eesm_cc_interlock2_rk4", "rk4"), ("extex_fin_cc_interlock2_rk4", "rk4"), ("extex_fin_cc_interlock2b_rk4", "euler3"),
    ("dfim_fin_sc_interlock2_rk4", "rk4"),
    # state-vector wrappers (CosSinProcessor, FluxObserver, FluxObserver angle for dq actions, dead time in front)
    ("pmsm_cc_cossin_rk4", "rk4"), ("pmsm_sc_cossin_rm_rk4", "rk4"), ("scim_cc_flux_dq_rk4", "rk4"), ("scim_sc_flux_cossin_dead1_rk4", "rk4"),
]


def _random_actions(rng, g, n, steps):
    a = g["actions"]
    if a.ndim == 1:
        hi = int(a.max()) + 1
        return rng.integers(0, max(hi, 2), size=(steps, n, 1)).astype(np.int32)
    if a.dtype.kind == "i":
        hi = a.max(axis=0) + 1
        return (rng.random((steps, n, a.shape[1])) * hi).astype(np.int32)
    # smooth-ish random actions so that currents build up and constraints trigger
    base = rng.uniform(-1, 1, size=(steps, n, a.shape[1]))
    hold = rng.uniform(-1, 1, size=(1, n, a.shape[1]))
    lo, hi = a.min(), a.max()
    out = 0.5 * base + 0.5 * hold
    if lo >= 0:
        out = np.abs(out)
    return out


@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name,solver", BATCH_CASES)
def test_device_matches_oracle_on_batch(torch_cuda, oracle_lib, name, solver, dtype):
    """N envs, random actions, Wiener references (same Philox streams on both sides), in-kernel auto-reset."""
    g = load_golden(name)
    n, steps = 1000, 150  # n deliberately not a multiple of the warp / block size
    rng = np.random.default_rng(42)
    actions = _random_actions(rng, g, n, steps)

    # Non-zero initial currents / flux / angle: with exactly-zero currents the freewheeling voltage of a finite converter
    # leg in its interlock state is decided by the sign of round-off noise (in the reference, too).
    init = np.array(g["reset_ode"], dtype=float)
    n_ode = len(init)
    init[1:] = [0.7, -0.4, 0.02, 0.03, 0.3][: n_ode - 1] if g["meta"]["motor_class"] in ("SquirrelCageInductionMotor", "DoublyFedInductionMotor") else \
        [0.9, -0.6, 0.5, 0.3][: n_ode - 1]

    def mk(dt):
        cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=init, dtype=dt, solver=solver, ref_kind=K.REF_WIENER,
                               autoreset=K.AUTORESET_SAME_STEP, seed=1234)
        for r in range(cfg.n_ref):
            cfg.ref_margin_lo[r], cfg.ref_margin_hi[r] = -0.7, 0.7
            cfg.ref_init_lo[r], cfg.ref_init_hi[r] = -0.7, 0.7
            cfg.ref_len_lo[r], cfg.ref_len_hi[r] = 5, 40  # many sub-episode changes inside the test
        cfg.env_index_offset = 7 * n
        if cfg.supply_kind == K.SUPPLY_AC1:
            cfg.supply_param[2] = 0.0  # phase ~ U[0, 2 pi) per env at every reset (Philox stream 9 on both sides)
        return cfg

    dev = DeviceAdapter(mk(dtype))
    ora = oracle_lib.Oracle(mk(K.F64), nthreads=8)
    o_obs, o_ref = ora.reset()
    d_obs, d_ref = dev.reset()
    tol = _tol(name, dtype, batch=True)
    assert np.abs(d_obs - o_obs).max() < 1e-6
    assert np.abs(d_ref - o_ref).max() < max(tol, 1e-12) * 10
    alive = np.ones(n, dtype=bool)  # envs whose device/oracle episodes are still aligned
    scale = np.maximum(np.abs(o_obs).max(axis=0), 1e-3)
    ang_cols = [j for j, nm in enumerate(g["meta"]["state_names"]) if nm in ("epsilon", "psi_angle")]
    feedback = "flux_dq" in name or "flux_cossin_dead1" in name
    sign_events = name == "dfim_fin_sc_interlock2_rk4"
    within_plain = np.ones(n, dtype=bool)  # feedback configurations: envs that never left the PLAIN tolerance
    n_term = 0
    for k in range(steps):
        o_obs, o_ref, o_rew, o_term = ora.step(actions[k])
        d_obs, d_ref, d_rew, d_term = dev.step(actions[k])
        split = alive & (o_term != d_term)
        alive &= ~split  # a constraint within rounding of its threshold: episodes diverge from here on
        scale = np.maximum(scale, np.abs(o_obs[alive]).max(axis=0))
        diff = np.abs(d_obs - o_obs)
        for j in ang_cols:  # normalised angles live on a circle of circumference 2: +1 and -1 are the same point
            diff[:, j] = np.abs((d_obs[:, j] - o_obs[:, j] + 1.0) % 2.0 - 1.0)
        if feedback and dtype == K.F32:
            # closed loop through angle(psi_obs): an env whose observer flux passes near zero amplifies rounding-level differences
            # without bound (see TOL_OBSERVER_FEEDBACK); such envs are counted as diverged — at most 1 % may — instead of failing the run
            within_plain &= ~(alive & ((diff / scale).max(axis=1) >= TOL[dtype]))
            alive &= ~((diff / scale).max(axis=1) >= tol)
        if sign_events and dtype == K.F32:
            # finite legs waiting in their interlock state output by the SIGN of their current (converters.py:277-287); with three
            # segments per step and the rotor bridge fed with alpha-beta rotor currents (a difference of two large terms) that sign is decided
            # within fp32 rounding for a few envs per 10^5 leg-steps: a discrete event, after which the episode is a different one.
            # Such envs leave the comparison (at most 1 % may, asserted below; 7 of 1000 observed); fp64 holds every env.
            alive &= ~((diff / scale).max(axis=1) >= tol)
        err = (diff[alive] / scale).max()
        assert err < tol, f"step {k}: state error {err:.3e}"
        assert np.abs(d_ref - o_ref)[alive].max() < 20 * tol if d_ref.size else True
        assert np.abs(d_rew - o_rew)[alive].max() < 20 * tol
        n_term += int(o_term[alive].sum())
    assert alive.mean() > (0.99 if (feedback or sign_events) else 0.995), f"too many diverged envs: {n - alive.sum()}"  # sign_events fp32: 7 of 1000 seen
    if feedback and dtype == K.F32:
        # the loose tolerance is a TAIL allowance (tests/test_oracle_golden.py::test_observer_feedback_configuration_amplifies_rounding: fewer
        # than 5 % of the envs amplify rounding by > 100x): the bulk of the batch has to hold the plain fp32 bar
        assert within_plain.mean() > 0.9, f"only {within_plain.mean():.3f} of the envs within {TOL[dtype]:g}"
    if name not in ("series_cc_rk4",) and "_fin" not in name:  # finite envs: tau = 1e-5, 150 steps are too short to trip
        assert n_term > 0, "test is meant to exercise termination + auto-reset"


@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("dist,params", [(K.NOISE_NORMAL, (0.01, 0.05)), (K.NOISE_UNIFORM, (-0.02, 0.04)), (K.NOISE_LAPLACE, (0.0, 0.03))])
def test_state_noise_processor_matches_oracle_and_distribution(torch_cuda, oracle_lib, dist, params, dtype):
    """StateNoiseProcessor (state_noise_processor.py:74-98) as a state op: device == oracle value for value (same Philox
    convention), and the noise itself has the requested distribution (moments checked against numpy's definitions)."""
    g = load_golden("pmsm_cc_rk4")
    n, steps = 2048, 12
    names = g["meta"]["state_names"]
    noisy = [names.index(s) for s in ("omega", "i_sd", "i_sq", "u_sup")]

    def mk(dt, with_noise=True):
        cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=g["reset_ode"], dtype=dt, solver="rk4", ref_kind=K.REF_WIENER,
                               autoreset=K.AUTORESET_SAME_STEP, seed=99)
        cfg.n_constraints = 0  # keep episodes running: the clean twin must stay aligned
        if with_noise:
            cfg.n_state_ops = 1
            cfg.sop_kind[0] = K.SOP_NOISE
            cfg.sop_idx[0][0] = dist
            cfg.sop_mask[0] = sum(1 << j for j in noisy)
            cfg.sop_param[0][0], cfg.sop_param[0][1] = params
        return cfg

    dev, ora, clean = DeviceAdapter(mk(dtype)), oracle_lib.Oracle(mk(K.F64), nthreads=8), oracle_lib.Oracle(mk(K.F64, False), nthreads=8)
    rng = np.random.default_rng(3)
    d0, _ = dev.reset()
    o0, _ = ora.reset()
    c0, _ = clean.reset()
    tol = 1e-9 if dtype == K.F64 else 2e-6
    assert np.abs(d0 - o0).max() < tol  # the noise is added at reset as well (:74-78)
    samples = [(o0 - c0)[:, noisy]]
    for k in range(steps):
        a = rng.uniform(-0.3, 0.3, size=(n, 3))
        d_obs, _, d_rew, _ = dev.step(a)
        o_obs, _, o_rew, _ = ora.step(a)
        c_obs, _, _, _ = clean.step(a)
        assert np.abs(d_obs - o_obs).max() < tol, k
        assert np.abs(d_rew - o_rew).max() < 10 * tol  # the reward sees the noisy state (it is computed on the wrapped system)
        others = [j for j in range(len(names)) if j not in noisy]
        assert np.abs(o_obs[:, others] - c_obs[:, others]).max() == 0.0
        samples.append((o_obs - c_obs)[:, noisy])
    z = np.concatenate(samples).ravel()
    a0, a1 = params
    if dist == K.NOISE_NORMAL:
        mean, std, kurt = a0, a1, 3.0
    elif dist == K.NOISE_UNIFORM:
        mean, std, kurt = 0.5 * (a0 + a1), (a1 - a0) / np.sqrt(12.0), 1.8
    else:
        mean, std, kurt = a0, a1 * np.sqrt(2.0), 6.0
    m = len(z)
    assert abs(z.mean() - mean) < 5 * std / np.sqrt(m)
    assert abs(z.std() / std - 1) < 0.02
    assert abs(((z - z.mean()) ** 4).mean() / z.var() ** 2 / kurt - 1) < 0.1
    if dist == K.NOISE_UNIFORM:
        assert z.min() >= a0 and z.max() <= a1


@pytest.mark.parametrize("dev_solver,ora_solver,dtype,n,tol", [
    ("rk4", "rk4", K.F32, 1024, 1e-5), ("rk4", "rk4", K.F64, 1024, 1e-9), ("rk4x2", "rk4x2", K.F32, 1024, 1e-5),
    ("rk4x2", "dopri5", K.F64, 256, 2e-6), ("rk4x2", "dopri5", K.F32, 256, 1e-5)])
def test_headline_config_long_horizon(torch_cuda, oracle_lib, dev_solver, ora_solver, dtype, n, tol):
    """SURVEY.md §8(d) item 2: Cont-CC-PMSM-v0, zero-initialised, omega = 100 rad/s, U(-1,1)^3 actions, 1000 steps; the CUDA path
    (RK4 x1 / x2) against the oracle driven by the algorithm-identical RK4 and by the reference's default dopri5, auto-reset on.
    State, reward and termination are compared for every env and step; an env whose termination differs (a constraint within
    rounding of its threshold) is dropped from then on — at most 0.5 % may."""
    g = load_golden("pmsm_cc_rk4")
    steps = 1000
    rng = np.random.default_rng(2024)

    def mk(dt, solver):
        return config_from_meta(g["meta"], n_envs=n, reset_ode=g["reset_ode"], dtype=dt, solver=solver, ref_kind=K.REF_WIENER,
                                autoreset=K.AUTORESET_SAME_STEP, seed=7)

    dev, ora = DeviceAdapter(mk(dtype, dev_solver)), oracle_lib.Oracle(mk(K.F64, ora_solver), nthreads=16)
    d_obs, d_ref = dev.reset()
    o_obs, o_ref = ora.reset()
    assert np.abs(d_obs - o_obs).max() < 1e-6 and np.abs(d_ref - o_ref).max() < 1e-5
    alive = np.ones(n, dtype=bool)
    scale = np.maximum(np.abs(o_obs).max(axis=0), 1e-3)
    worst, n_term = 0.0, 0
    for k in range(steps):
        a = rng.uniform(-1, 1, size=(n, 3))
        d_obs, d_ref, d_rew, d_term = dev.step(a)
        o_obs, o_ref, o_rew, o_term = ora.step(a)
        alive &= ~(o_term != d_term)
        scale = np.maximum(scale, np.abs(o_obs[alive]).max(axis=0))
        diff = np.abs(d_obs - o_obs)
        diff[:, 12] = np.abs((d_obs[:, 12] - o_obs[:, 12] + 1.0) % 2.0 - 1.0)  # epsilon lives on a circle
        err = (diff[alive] / scale).max()
        worst = max(worst, err)
        assert err < tol, f"step {k}: state error {err:.3e}"
        assert np.abs(d_rew - o_rew)[alive].max() < 20 * tol and np.abs(d_ref - o_ref)[alive].max() < 20 * max(tol, 1e-7)
        n_term += int(o_term[alive].sum())
    assert alive.mean() > 0.995 and n_term > n // 4, (alive.mean(), n_term)  # random actions do trip the current limit


@pytest.mark.parametrize("name,solver", [("pmsm_cc_rk4", "rk4"), ("pmsm_fin_sc_rk4", "rk4"), ("eesm_cc_rk4", "rk4x2"), ("scim_sc_rk4", "euler"),
                                         ("dfim_cc_rk4", "rk4"), ("extex_cc_rk4", "rk4"), ("permex_cc_rk4", "euler3"),
                                         # finite converters with an interlocking time: the PLAIN instantiations' IL variant (two / three switching segments)
                                         ("pmsm_fin_sc_rk4_interlock", "rk4"), ("scim_fin_cc_interlock_rk4", "rk4"), ("permex_fin4qc_interlock_rk4", "rk4"),
                                         ("extex_fin_cc_interlock2_rk4", "rk4"), ("dfim_fin_sc_interlock2_rk4", "rk4")])
def test_plain_and_general_instantiations_agree(torch_cuda, monkeypatch, name, solver):
    """The PLAIN instantiation (compile-time folded switches, the headline path) and the general one (GEMB200_NO_PLAIN=1) are the same
    source: same envs, same Philox streams, same actions -> same trajectories up to fp32 contraction differences, identical
    terminations; the launch-count shows that both really ran their own kernel."""
    g = load_golden(name)
    n, steps = 3000, 120
    rng = np.random.default_rng(1)
    actions = _random_actions(rng, g, n, steps)

    def mk():
        return config_from_meta(g["meta"], n_envs=n, reset_ode=g["reset_ode"], dtype=K.F32, solver=solver, ref_kind=K.REF_WIENER,
                                autoreset=K.AUTORESET_SAME_STEP, seed=5)

    plain = DeviceAdapter(mk())
    monkeypatch.setenv("GEMB200_NO_PLAIN", "1")
    general = DeviceAdapter(mk())
    monkeypatch.delenv("GEMB200_NO_PLAIN")
    a0, b0 = plain.reset(), general.reset()
    assert np.array_equal(a0[0], b0[0]) and np.array_equal(a0[1], b0[1])
    alive = np.ones(n, dtype=bool)
    for k in range(steps):
        pa, pb = plain.step(actions[k]), general.step(actions[k])
        alive &= ~(pa[3] != pb[3])
        scale = np.maximum(np.abs(pb[0][alive]).max(axis=0), 1e-3)
        assert (np.abs(pa[0] - pb[0])[alive] / scale).max() < 2e-5, k
        assert np.abs(pa[1] - pb[1])[alive].max() < 1e-5 and np.abs(pa[2] - pb[2])[alive].max() < 1e-4
    assert alive.mean() > 0.995


def _cfg(name, n, dtype=K.F32, **kw):
    g = load_golden(name)
    return g, config_from_meta(g["meta"], n_envs=n, reset_ode=g["reset_ode"], dtype=dtype, solver="rk4", ref_kind=K.REF_WIENER,
                               autoreset=K.AUTORESET_SAME_STEP, seed=3, **kw)


@pytest.mark.parametrize("name", ["pmsm_cc_rk4", "eesm_cc_rk4", "permex_cc_rk4", "extex_cc_rk4", "scim_fin_sc_rk4", "dfim_cc_rk4",
                                  "scim_sc_flux_cossin_dead1_rk4", "pmsm_sc_cossin_rm_rk4", "permex_sc_rc_rk4"])
@pytest.mark.parametrize("n", [1, 31, 33, 257, 4096 + 5])
def test_layouts_and_host_path_agree_bitwise(torch_cuda, name, n):
    """row-per-env (AoS, smem transpose + vector stores) vs the host-buffer entry point: bit-for-bit (same kernel).
    Field-major (SoA) is a separate template instantiation of the same source, so the compiler may contract FMAs differently:
    it has to agree to a few ulp (and terminations exactly)."""

    def close(x, y):
        return torch.allclose(x, y, rtol=2e-6, atol=2e-7)

    import torch
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, cfg_a = _cfg(name, n, layout=K.LAYOUT_AOS)
    _, cfg_s = _cfg(name, n, layout=K.LAYOUT_SOA)
    _, cfg_h = _cfg(name, n, layout=K.LAYOUT_AOS)
    sa, ss, sh = VectorSim(cfg_a), VectorSim(cfg_s), VectorSim(cfg_h)
    rng = np.random.default_rng(0)
    steps = 20
    acts = _random_actions(rng, g, n, steps)
    ra, rs, rh = sa.reset(), ss.reset(), sh.reset_host()
    assert close(ra[0], rs[0].T) and close(ra[1], rs[1].T)
    assert np.array_equal(ra[0].cpu().numpy(), rh[0])
    for k in range(steps):
        a = acts[k]
        oa = sa.step(a)
        os_ = ss.step(np.ascontiguousarray(a.T) if not sa.finite else np.ascontiguousarray(a.reshape(n, -1).T))
        oh = sh.step_host(a)
        assert close(oa[0], os_[0].T) and close(oa[1], os_[1].T)
        assert close(oa[2], os_[2]) and torch.equal(oa[3], os_[3])
        for x, y in zip(oa, oh):
            assert np.array_equal(x.cpu().numpy(), y)


@pytest.mark.parametrize("name", ["pmsm_fin_sc_rk4_interlock", "scim_sc_flux_cossin_dead1_rk4", "permex_fin_sc_rc_interlock_rk4", "pmsm_cc_ac_rk4",
                                  "pmsm_cc_extspeed_rk4"])
def test_checkpoint_roundtrip(torch_cuda, name):
    """state_dict covers every persistent array: records, angle, switching states, dead-time queue, observer, supply, profile clock"""
    import torch
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, cfg = _cfg(name, 513)
    sim = VectorSim(cfg, reuse_outputs=False)
    rng = np.random.default_rng(1)
    acts = _random_actions(rng, g, 513, 30)
    sim.reset()
    for k in range(10):
        sim.step(acts[k])
    sd = sim.state_dict()
    a = [sim.step(acts[k]) for k in range(10, 30)]
    sim.load_state_dict(sd)
    b = [sim.step(acts[k]) for k in range(10, 30)]
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert torch.equal(u, v)


def test_masked_reset_and_get_set_state(torch_cuda):
    import torch
    from gym_electric_motor_b200.vector_sim import VectorSim

    g = load_golden("pmsm_cc_rk4")
    n = 300
    cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=g["reset_ode"], dtype=K.F32, solver="rk4", ref_kind=K.REF_CONST)
    sim = VectorSim(cfg, reuse_outputs=False)
    rng = np.random.default_rng(2)
    for _ in range(5):
        sim.step(rng.uniform(-1, 1, size=(n, 3)))
    y = sim.get_ode_state()
    assert (y[:, 1:3].abs().sum(dim=1) > 0).all()
    mask = torch.zeros(n, dtype=torch.uint8)
    mask[::3] = 1
    sim.reset(mask)
    y2 = sim.get_ode_state()
    m = mask.bool().cuda()
    assert torch.equal(y2[~m], y[~m])
    assert (y2[m][:, 1:] == 0).all() and torch.allclose(y2[m][:, 0], torch.full_like(y2[m][:, 0], float(g["reset_ode"][0])))
    y3 = y.clone()
    y3[:, 3] = y3[:, 3] + 4 * np.pi  # angle is stored wrapped
    sim.set_ode_state(y3)
    assert torch.allclose(sim.get_ode_state(), y, atol=1e-6)


def test_full_size_replication_property(torch_cuda, oracle_lib):
    """BASELINE size (N = 2^20, Cont-CC-PMSM-v0, RK4): 1024 distinct action streams, each replicated 1024 times across the
    grid.  Size-independent properties: every replica is bit-identical to its prototype (no indexing/tail/layout
    error anywhere in the 4096-block grid) and the prototypes match the CPU oracle."""
    import torch
    from gym_electric_motor_b200.vector_sim import VectorSim

    g = load_golden("pmsm_cc_rk4")
    n, proto, steps = 1 << 20, 1024, 25
    cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=g["reset_ode"], dtype=K.F32, solver="rk4", ref_kind=K.REF_CONST)
    cfg_o = config_from_meta(g["meta"], n_envs=proto, reset_ode=g["reset_ode"], dtype=K.F64, solver="rk4", ref_kind=K.REF_CONST)
    for c in (cfg, cfg_o):
        for r in range(c.n_ref):
            c.ref_value[r] = 0.1 * (r + 1)
    sim = VectorSim(cfg)
    ora = oracle_lib.Oracle(cfg_o, nthreads=8)
    sim.reset()
    ora.reset()
    rng = np.random.default_rng(9)
    for k in range(steps):
        a = rng.uniform(-1, 1, size=(proto, 3))
        a_dev = torch.as_tensor(a, dtype=torch.float32, device="cuda").repeat(n // proto, 1)
        obs, ref, rew, term = sim.step(a_dev)
        o_obs, _, o_rew, o_term = ora.step(a)
        v = obs.view(n // proto, proto, -1)
        assert torch.equal(v, v[0:1].expand_as(v))
        assert torch.equal(rew.view(-1, proto), rew[:proto].expand(n // proto, proto))
        d = obs[:proto].double().cpu().numpy()
        assert col_rel_err(d, o_obs) < 1e-5 or np.abs(d - o_obs).max() < 1e-6
        assert np.abs(rew[:proto].double().cpu().numpy() - o_rew).max() < 1e-4


@pytest.mark.parametrize("name,solver", [("pmsm_fin_sc_rk4", "rk4"), ("scim_cc_rk4", "rk4")])
def test_full_size_replication_property_other_configs(torch_cuda, oracle_lib, name, solver):
    """BASELINE configs[2] (Finite-SC-PMSM, N = 2^20) and configs[3] (Cont-CC-SCIM, N = 2^20): 1024 action streams replicated 1024 times
    across the grid; every replica bit-identical to its prototype after single-step launches AND after a fused rollout, the prototypes
    equal to the oracle."""
    import torch
    from gym_electric_motor_b200.vector_sim import VectorSim

    g = load_golden(name)
    n, proto, steps = 1 << 20, 1024, 20
    init = np.array(g["reset_ode"], dtype=float)
    if name.startswith("scim"):
        init[1:] = [0.7, -0.4, 0.02, 0.03, 0.3]  # a defined field frame from step 0 on (DESIGN.md finding 3)
    mk = lambda nn, dt: config_from_meta(g["meta"], n_envs=nn, reset_ode=init, dtype=dt, solver=solver, ref_kind=K.REF_CONST)  # noqa: E731
    cfg, cfg_o = mk(n, K.F32), mk(proto, K.F64)
    for c in (cfg, cfg_o):
        for r in range(c.n_ref):
            c.ref_value[r] = 0.1 * (r + 1)
    sim, sim2, ora = VectorSim(cfg), VectorSim(cfg), oracle_lib.Oracle(cfg_o, nthreads=8)
    sim.reset()
    sim2.reset()
    ora.reset()
    rng = np.random.default_rng(9)
    acts = _random_actions(rng, g, proto, steps)
    adt = torch.int32 if sim.finite else torch.float32
    dev = torch.as_tensor(acts.reshape(steps, proto, sim.n_act), device="cuda").to(adt).repeat(1, n // proto, 1).contiguous()
    for k in range(steps):
        obs, ref, rew, term = sim.step(dev[k])
        o_obs, _, o_rew, o_term = ora.step(acts[k])
        v = obs.view(n // proto, proto, -1)
        assert torch.equal(v, v[0:1].expand_as(v)) and torch.equal(rew.view(-1, proto), rew[:proto].expand(n // proto, proto))
        d = obs[:proto].double().cpu().numpy()
        assert col_rel_err(d, o_obs) < 1e-5 or np.abs(d - o_obs).max() < 1e-6, k
        assert np.array_equal(term[:proto].cpu().numpy(), o_term)
    last = sim2.rollout(dev, record_every=0)
    assert torch.equal(last[0], obs) and torch.equal(last[2], rew) and torch.equal(last[3], term)


def test_public_api_scalar_and_batched(torch_cuda):
    """gem.make surface: scalar (num_envs=None) contract of the reference and the batched contract agree with each other and
    with the recorded reference trajectory (Cont-CC-PMSM-v0, RK4 plugin golden)."""
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.reference_generators import ExternalReferenceGenerator, MultipleReferenceGenerator

    g = load_golden("pmsm_cc_rk4")

    def mk(**kw):
        rg = MultipleReferenceGenerator([ExternalReferenceGenerator("i_sd"), ExternalReferenceGenerator("i_sq")])
        return gem.make("Cont-CC-PMSM-v0", ode_solver=gem.physical_systems.RK4Solver(), reference_generator=rg, dtype="float64", **kw)

    env1, envn = mk(), mk(num_envs=5)
    (s, r), info = env1.reset(seed=3)
    assert s.shape == (14,) and r.shape == (2,) and info == {}
    np.testing.assert_allclose(s, golden_reset_state(g), atol=1e-12)
    (sb, rb), _ = envn.reset(seed=3)
    assert tuple(sb.shape) == (5, 14) and tuple(rb.shape) == (5, 2)
    ref_idx = [g["meta"]["state_names"].index(nm) for nm in g["meta"]["reference_names"]]
    for k in range(40):
        refs = g["refs_used"][k][ref_idx]
        env1.set_reference(refs[None, :])
        envn.set_reference(np.tile(refs, (5, 1)))
        (s, r), rew, term, trunc, _ = env1.step(g["actions"][k])
        (sb, rb), rewb, termb, truncb, _ = envn.step(np.tile(g["actions"][k], (5, 1)))
        assert isinstance(rew, float) and isinstance(term, bool) and trunc is False
        np.testing.assert_allclose(s, g["states"][k], rtol=0, atol=1e-9)
        assert rew == pytest.approx(g["rewards"][k], abs=1e-9) and term == bool(g["terminated"][k])
        np.testing.assert_allclose(sb.cpu().numpy(), np.tile(s, (5, 1)), atol=1e-12)
        assert termb.dtype == torch_cuda.bool and bool(termb[0]) == term
        if term:
            with pytest.raises(AssertionError):
                env1.step(g["actions"][k])  # core.py:341
            env1.reset()
            envn.reset()
    env1.close()
    envn.close()


def test_mixed_motor_batch(torch_cuda, oracle_lib):
    """configs[4]: PMSM + SynRM + EESM segmented per type, one launch per type on its own stream; each segment must equal
    the same env stepped alone."""
    import torch
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.mixed import MixedEnvBatch

    RK4 = gem.physical_systems.RK4Solver
    ids = [("Cont-CC-PMSM-v0", dict(ode_solver=RK4())), ("Cont-CC-SynRM-v0", dict(ode_solver=RK4())), ("Cont-CC-EESM-v0", dict(ode_solver=RK4()))]
    n = 3 * 700
    mixed = MixedEnvBatch(ids, n, autoreset="same_step", seed=5)
    solo = [gem.make(e, num_envs=700, autoreset="same_step", seed=5, env_index_offset=t * 700, **kw) for t, (e, kw) in enumerate(ids)]
    mixed.reset()
    for e in solo:
        e.reset()
    gen = torch.Generator(device="cuda").manual_seed(0)
    for k in range(25):
        acts = [torch.rand((700, 4 if t == 2 else 3), generator=gen, device="cuda") * 2 - 1 for t in range(3)]
        res = mixed.step(acts)
        torch.cuda.synchronize()
        for t in range(3):
            (s, r), rew, term, _, _ = solo[t].step(acts[t])
            (sm, rm), rewm, termm, _, _ = res[t]
            assert torch.equal(s, sm) and torch.equal(r, rm) and torch.equal(rew, rewm) and torch.equal(term, termm)
    glob = torch.arange(n, device="cuda")
    parts = mixed.split_interleaved(glob)
    assert [int(p[1]) for p in parts] == [3, 4, 5]


def test_mixed_motor_batch_matches_oracle(torch_cuda, oracle_lib):
    """configs[4] against the ORACLE (not against the kernel itself): every type segment of a mixed PMSM + SynRM + EESM batch, stepped
    through MixedEnvBatch (one launch per type, own stream) and through the fused rollout, equals the float64 oracle of that segment's
    configuration (same global env indices -> same Philox streams) within the fp32 bar."""
    import torch
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.mixed import MixedEnvBatch

    RK4 = gem.physical_systems.RK4Solver
    ids = [("Cont-CC-PMSM-v0", dict(ode_solver=RK4())), ("Cont-CC-SynRM-v0", dict(ode_solver=RK4())), ("Cont-CC-EESM-v0", dict(ode_solver=RK4()))]
    per, steps = 512, 60
    mixed = MixedEnvBatch(ids, 3 * per, autoreset="same_step", seed=9, env_index_offset=3000)
    oras = []
    for env in mixed.envs:
        cfg = env.build_config()
        cfg.dtype = K.F64
        oras.append(oracle_lib.Oracle(cfg, nthreads=8))
    res = mixed.reset()
    for t, ora in enumerate(oras):
        o_obs, o_ref = ora.reset()
        assert np.abs(res[t][0][0].double().cpu().numpy() - o_obs).max() < 1e-6
    rng = np.random.default_rng(2)
    alive = [np.ones(per, dtype=bool) for _ in ids]
    n_term = 0
    for k in range(steps):
        acts = [rng.uniform(-1, 1, size=(per, 4 if t == 2 else 3)) for t in range(3)]
        res = mixed.step([torch.as_tensor(a, dtype=torch.float32, device="cuda") for a in acts])
        torch.cuda.synchronize()
        for t, ora in enumerate(oras):
            o_obs, o_ref, o_rew, o_term = ora.step(acts[t])
            (s, r), rew, term, _, _ = res[t]
            alive[t] &= ~(o_term != term.cpu().numpy().astype(np.uint8))
            d = np.abs(s.double().cpu().numpy() - o_obs)
            eps_col = mixed.envs[t].physical_system.state_names.index("epsilon")
            d[:, eps_col] = np.abs((s.double().cpu().numpy()[:, eps_col] - o_obs[:, eps_col] + 1.0) % 2.0 - 1.0)
            assert d[alive[t]].max() < 2e-5, (t, k)
            assert np.abs(r.double().cpu().numpy() - o_ref)[alive[t]].max() < 2e-4 and np.abs(rew.double().cpu().numpy() - o_rew)[alive[t]].max() < 2e-4
            n_term += int(o_term[alive[t]].sum())
    assert all(a.mean() > 0.99 for a in alive) and n_term > 0


@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("dist", ["uniform", "gaussian"])
@pytest.mark.parametrize("name", ["pmsm_sc_rk4", "eesm_cc_rk4", "extex_cc_rk4", "permex_cc_rk4"])
def test_random_initial_states_match_oracle(torch_cuda, oracle_lib, name, dist, dtype):
    """random_init='uniform' / 'gaussian' (truncated normal) on the device: same Philox draws as the oracle at reset and at every
    in-kernel auto-reset; the reset observation is computed from the sampled state."""
    g = load_golden(name)
    n, steps = 777, 60
    init = np.array(g["reset_ode"], dtype=float)
    n_ode = len(init)
    lim = np.array(g["meta"]["limits"])
    names = g["meta"]["state_names"]
    span = np.array([0.3 * lim[0]] + [0.6 * lim[names.index("i_sd" if "i_sd" in names else ("i_a" if "i_a" in names else "i"))]] * (n_ode - 1))
    if "epsilon" in names:
        span[-1] = np.pi

    def mk(dt):
        cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=init, dtype=dt, solver="rk4", ref_kind=K.REF_WIENER, autoreset=K.AUTORESET_SAME_STEP, seed=77)
        cfg.init_random = 1
        for j in range(n_ode):
            cfg.init_lo[j], cfg.init_hi[j] = -span[j], span[j]
            if dist == "gaussian":  # off-centre mean, sigma comparable to the interval: both truncation tails matter
                cfg.init_dist[j], cfg.init_mu[j], cfg.init_sigma[j] = 1, 0.3 * span[j], 0.8 * span[j]
        return cfg

    dev = DeviceAdapter(mk(dtype))
    ora = oracle_lib.Oracle(mk(K.F64), nthreads=8)
    o_obs, o_ref = ora.reset()
    d_obs, d_ref = dev.reset()
    tol = TOL[dtype]
    assert np.abs(d_obs - o_obs).max() < 20 * tol
    y = dev.sim.get_ode_state().cpu().numpy()
    assert np.abs(y - ora.get_ode_state()).max() / np.abs(span).max() < 20 * tol
    assert np.unique(np.round(y[:, 1], 6)).size > n // 2  # really random per env
    rng = np.random.default_rng(5)
    acts = _random_actions(rng, g, n, steps)
    alive = np.ones(n, dtype=bool)
    n_term = 0
    for k in range(steps):
        o_obs, o_ref, o_rew, o_term = ora.step(acts[k])
        d_obs, d_ref, d_rew, d_term = dev.step(acts[k])
        alive &= ~(o_term != d_term)
        assert np.abs(d_obs - o_obs)[alive].max() < 50 * tol, k
        n_term += int(o_term[alive].sum())
    assert alive.mean() > 0.99 and n_term > 0


@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("case", ["wiener_sinus_step", "const_laplace_triangular", "two_const"])
def test_switched_reference_generator_matches_oracle(torch_cuda, oracle_lib, case, dtype):
    """SwitchedReferenceGenerator in the fused epilogue vs the oracle (same Philox convention): every reference value, reward and
    the reset references of auto-reset envs, with super-episodes short enough for dozens of switches per env."""
    kinds = dict(
        wiener_sinus_step=[dict(kind=K.REF_WIENER, margin=(-0.5, 0.5)), dict(kind=K.REF_SINUS), dict(kind=K.REF_STEP, amp=(0.05, 0.2))],
        const_laplace_triangular=[dict(kind=K.REF_CONST, value=0.25), dict(kind=K.REF_LAPLACE, sigma=(1e-3, 5e-3)), dict(kind=K.REF_TRIANGULAR)],
        two_const=[dict(kind=K.REF_CONST, value=-0.4), dict(kind=K.REF_CONST, value=0.7)])[case]
    n, steps = 700, 300
    p = [1.0 / len(kinds)] * len(kinds)

    def mk(dt):
        cfg = switched_config(n, kinds, p, (7, 25), seed=21, dtype=dt)
        cfg.n_constraints = 1  # terminations + in-kernel auto-reset: the generator is re-chosen at the reset
        return cfg

    dev, ora = DeviceAdapter(mk(dtype)), oracle_lib.Oracle(mk(K.F64), nthreads=8)
    d_obs, d_ref = dev.reset()
    o_obs, o_ref = ora.reset()
    tol = 1e-9 if dtype == K.F64 else 2e-5
    assert np.abs(d_ref - o_ref).max() < tol
    rng = np.random.default_rng(8)
    alive = np.ones(n, dtype=bool)
    distinct = set()
    for k in range(steps):
        a = rng.uniform(-1, 1, size=(n, 1))
        d_obs, d_ref, d_rew, d_term = dev.step(a)
        o_obs, o_ref, o_rew, o_term = ora.step(a)
        alive &= ~(o_term != d_term)
        assert np.abs(d_ref - o_ref)[alive].max() < tol, k
        assert np.abs(d_rew - o_rew)[alive].max() < 20 * tol, k
        distinct.update(np.round(o_ref[:5, 0], 3).tolist())
    assert alive.mean() > 0.99 and len(distinct) > (1 if case == "two_const" else 20)


@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("kinds", [(K.REF_LAPLACE, K.REF_WIENER), (K.REF_SINUS, K.REF_STEP), (K.REF_SAWTOOTH, K.REF_TRIANGULAR)])
def test_more_reference_generators_match_oracle(torch_cuda, oracle_lib, kinds, dtype):
    """Laplace / sinusoidal / step / sawtooth / triangular generators in the fused epilogue vs the oracle (same Philox blocks)."""
    g = load_golden("pmsm_cc_rk4")
    n, steps = 600, 160

    def mk(dt):
        cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=g["reset_ode"], dtype=dt, solver="rk4", ref_kind=K.REF_WIENER,
                               autoreset=K.AUTORESET_SAME_STEP, seed=4242)
        for r in range(2):
            cfg.ref_kind[r] = kinds[r]
            cfg.ref_margin_lo[r], cfg.ref_margin_hi[r] = -0.6, 0.6
            cfg.ref_init_lo[r], cfg.ref_init_hi[r] = -0.6, 0.6
            cfg.ref_amp_lo[r], cfg.ref_amp_hi[r] = 0.05, 0.6
            cfg.ref_freq_lo[r], cfg.ref_freq_hi[r] = 20.0, 400.0
            cfg.ref_off_lo[r], cfg.ref_off_hi[r] = -0.6, 0.6
            cfg.ref_len_lo[r], cfg.ref_len_hi[r] = 7, 45
        return cfg

    dev = DeviceAdapter(mk(dtype))
    ora = oracle_lib.Oracle(mk(K.F64), nthreads=8)
    _, o_ref = ora.reset()
    _, d_ref = dev.reset()
    tol = 1e-9 if dtype == K.F64 else 1e-5  # fp32: the phase is formed in double (DESIGN §2 finding 13)
    bad = int((np.abs(d_ref - o_ref) > tol).sum())
    total = d_ref.size
    rng = np.random.default_rng(1)
    alive = np.ones(n, dtype=bool)
    for k in range(steps):
        a = rng.uniform(-0.3, 0.3, size=(n, 3))
        _, o_ref, o_rew, o_term = ora.step(a)
        _, d_ref, d_rew, d_term = dev.step(a)
        alive &= ~(o_term != d_term)  # terminations (and the generator restarts they trigger) must coincide; borderline envs drop out
        bad += int((np.abs(d_ref - o_ref)[alive] > tol).sum())
        total += int(alive.sum()) * d_ref.shape[1]
    assert alive.mean() > 0.99
    # discontinuous waves may differ exactly at an edge in fp32 (phase rounding); everything else has to agree
    assert bad <= (0 if dtype == K.F64 else 0.004 * total), (bad, total)


@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("dist", ["uniform", "gaussian"])
@pytest.mark.parametrize("env_id,load_iv", [("Cont-SC-SCIM-v0", None), ("Cont-CC-SCIM-v0", None), ("Cont-SC-DFIM-v0", None), ("Cont-SC-SCIM-v0", [[-50.0, 120.0]]),
                                            ("Finite-CC-DFIM-v0", [[20.0, 90.0]])])
def test_induction_motor_random_initial_states_match_oracle(torch_cuda, oracle_lib, env_id, load_iv, dist, dtype):
    """SCIM / DFIM random initial states (per-reset flux bounds from a random field angle, the speed and the previous reset's initial
    currents; squirrel_cage_induction_motor.py:146-157, induction_motor.py:250-285) built through gem.make: reset observations, ODE
    states and 40 steps with in-kernel auto-resets, value for value against the oracle (same Philox streams).  The oracle's
    distribution is pinned to the reference in tests/test_oracle_golden.py."""
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.vector_sim import VectorSim

    n = 600
    load = dict(load_initializer=dict(random_init="uniform", interval=load_iv)) if load_iv else None
    env = gem.make(env_id, num_envs=n, motor=dict(motor_initializer=dict(random_init=dist, random_params=(None, 0.3) if dist == "gaussian" else (None, None))),
                   load=load, ode_solver=gem.physical_systems.RK4Solver(), autoreset="same_step", seed=4)
    cfg_d, cfg_o = env.build_config(), env.build_config()
    cfg_d.dtype, cfg_o.dtype = dtype, K.F64
    cfg_d.env_index_offset = cfg_o.env_index_offset = 999
    sim, ora = VectorSim(cfg_d), oracle_lib.Oracle(cfg_o, nthreads=8)
    tol = 1e-9 if dtype == K.F64 else 2e-5
    dq = ((5, 6), (10, 11)) if "SCIM" in env_id else ((5, 6), (10, 11), (15, 16), (20, 21))

    def cmp_obs(d, o, psi):
        d, o = d.copy(), o.copy()
        weak = np.hypot(psi[:, 0], psi[:, 1]) < 1e-3  # field frame undefined while the flux is ~0 (DESIGN.md finding 3): compare magnitudes
        for arr in (d, o):
            for a_, b_ in dq:
                arr[weak, a_] = np.hypot(arr[weak, a_], arr[weak, b_])
                arr[weak, b_] = 0.0
        return d, o, weak

    for rep in range(3):  # the 2nd and 3rd reset see the previous reset's initial currents
        d_obs, _ = sim.reset()
        o_obs, _ = ora.reset()
        y_d, y_o = sim.get_ode_state().cpu().numpy(), ora.get_ode_state()
        assert np.abs(y_d - y_o).max() < (1e-12 if dtype == K.F64 else 5e-4), rep  # fp32: the angle entry carries ~1e-7 * 2 pi, currents 1e-6 relative
        d, o, _ = cmp_obs(d_obs.double().cpu().numpy(), o_obs, y_o[:, 3:5])
        assert np.abs(d - o).max() < 20 * tol, rep
    assert np.abs(y_o[:, 3:5]).max() > 0 or "CC" in env_id
    rng = np.random.default_rng(3)
    sp = env.action_space
    alive = np.ones(n, dtype=bool)
    n_term = 0
    for k in range(40):
        a = rng.uniform(-1, 1, size=(n, len(sp.low))) if hasattr(sp, "low") else np.stack([rng.integers(0, int(m), size=n) for m in sp.nvec], axis=1).astype(np.int32)
        psi = ora.get_ode_state()[:, 3:5]
        o = ora.step(a)
        dv = sim.step(a)
        alive &= ~(o[3] != dv[3].cpu().numpy())
        d, oo, weak = cmp_obs(dv[0].double().cpu().numpy(), o[0], np.where(o[3][:, None] > 0, 0.0, psi))  # after an auto-reset the returned vector is the reset one
        m = alive & ~(o[3] > 0)
        assert np.abs(d - oo)[m].max() < 50 * tol, k
        n_term += int(o[3][alive].sum())
    assert alive.mean() > 0.98
    sim.close()


@pytest.mark.parametrize("env_id", ["Cont-CC-PMSM-v0", "Finite-SC-PMSM-v0", "Cont-SC-PermExDc-v0"])
def test_repeated_seeded_reset_gives_identical_episodes(torch_cuda, env_id):
    """reference: reset(seed) -> _seed(seed) re-seeds every component on EVERY seeded reset (core.py:300-304), so equal seeds give
    identical episodes — also the seed the env already has, also seed 0 on a fresh env, also after steps (ADVICE r1)."""
    import torch
    import gym_electric_motor_b200 as gem

    n = 512
    env = gem.make(env_id, num_envs=n, autoreset="same_step", ode_solver=gem.physical_systems.RK4Solver())
    fresh = gem.make(env_id, num_envs=n, autoreset="same_step", ode_solver=gem.physical_systems.RK4Solver(), seed=42)
    g = torch.Generator(device="cuda").manual_seed(0)
    if hasattr(env.action_space, "low"):
        acts = [torch.rand((n, len(env.action_space.low)), generator=g, device="cuda") * 2 - 1 for _ in range(30)]
    else:
        acts = [torch.randint(0, env.action_space.n, (n, 1), generator=g, device="cuda", dtype=torch.int32) for _ in range(30)]

    def episode(e, seed):
        (s, r), _ = e.reset(seed=seed)
        out = [(s.clone(), r.clone())]
        for a in acts:
            (s, r), w, t, _, _ = e.step(a)
            out.append((s.clone(), r.clone(), w.clone(), t.clone()))
        return out

    def same(x, y):
        return all(all(torch.equal(p, q) for p, q in zip(a, b)) for a, b in zip(x, y))

    e0a, e0b = episode(env, 0), episode(env, 0)      # seed 0 on a fresh env (whose stored default is 0), then again
    assert same(e0a, e0b)
    e42a, e42b = episode(env, 42), episode(env, 42)  # repeated seed after other episodes
    assert same(e42a, e42b) and not same(e0a, e42a)
    assert same(e42a, episode(fresh, 42))            # and equal to a freshly made env with that seed
    (s1, r1), _ = env.reset()                        # an unseeded reset continues the streams: new references
    assert not torch.equal(r1, e42a[0][1])


def test_checkpoint_of_another_configuration_is_refused(torch_cuda):
    """a blob of EQUAL size from another configuration (ADVICE r1: PMSM vs SynRM, another seed, another tau) must not load"""
    import gym_electric_motor_b200 as gem

    n = 64
    a = gem.make("Cont-CC-PMSM-v0", num_envs=n, seed=1)
    others = [gem.make("Cont-CC-SynRM-v0", num_envs=n, seed=1), gem.make("Cont-CC-PMSM-v0", num_envs=n, seed=2), gem.make("Cont-CC-PMSM-v0", num_envs=n, seed=1, tau=5e-5)]
    for e in [a] + others:
        e.reset()
    blob = a.state_dict()
    twin = gem.make("Cont-CC-PMSM-v0", num_envs=n, seed=1)
    twin.reset()
    twin.load_state_dict(blob)  # same configuration: accepted
    for e in others:
        assert e.state_dict()["blob"].size == blob["blob"].size
        with pytest.raises(K.GemB200Error, match="different configuration"):
            e.load_state_dict(blob)
    bad = {"blob": blob["blob"].copy()}
    bad["blob"][0] ^= 0xFF
    with pytest.raises(K.GemB200Error, match="bad magic"):
        twin.load_state_dict(bad)


def test_vector_facade_steps(torch_cuda):
    import gym_electric_motor_b200 as gem

    venv = gem.vector.make_vec("Cont-CC-PMSM-v0", num_envs=64, flatten_obs=True, ode_solver=gem.physical_systems.RK4Solver())
    obs, info = venv.reset(seed=1)
    assert tuple(obs.shape) == (64, 16)
    for _ in range(5):
        obs, rew, term, trunc, info = venv.step(torch_cuda.zeros((64, 3), device="cuda"))
    assert tuple(rew.shape) == (64,) and term.dtype == torch_cuda.bool and not trunc.any()
    venv.close()
