"""Fused K-step rollout (gemb200_rollout / gemb200_rollout_record = rollout_kernel) against K single-step launches (gemb200_step =
step_kernel) of the SAME configuration: the reference semantics are `env.step` called K times (core.py:328-371), so the bar is
bit-for-bit equality of every recorded output, of the persistent state afterwards (checkpoint blob) and of the steps that follow.
Oracle parity of the rollout path itself: test_rollout_matches_oracle."""
import numpy as np
import pytest

from gpu_helpers import _dev_actions, launch_sizes, torch_cuda  # noqa: F401
from helpers import ROLLOUT_CASES, WEAK_DQ_PAIRS, _mk, _random_actions, _tol, config_from_meta, fold_weak_dq, load_golden, switched_config
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

@pytest.mark.parametrize("layout", [K.LAYOUT_AOS, K.LAYOUT_SOA], ids=["aos", "soa"])
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ROLLOUT_CASES)
def test_rollout_is_bit_identical_to_repeated_steps(torch_cuda, name, dtype, layout):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    n, k_total = 777, 24  # not a multiple of the warp / block size; long enough for terminations + auto-resets + new sub-episodes
    g, cfg = _mk(name, n, dtype, layout)
    a, b, c = VectorSim(cfg), VectorSim(cfg), VectorSim(cfg)
    rng = np.random.default_rng(5)
    acts = _random_actions(rng, g, n, k_total + 3)
    dev = _dev_actions(torch, a, acts)
    for s in (a, b, c):
        s.reset()
    # a: K single-step launches, keeping every output
    per_step = []
    for k in range(k_total):
        per_step.append(tuple(t.clone() for t in a.step(dev[k])))
    # b: ONE launch, full trajectory
    obs, ref, rew, term = b.rollout(dev[:k_total], record_every=1)
    for k in range(k_total):
        assert torch.equal(obs[k], per_step[k][0]), (name, "obs", k)
        assert torch.equal(ref[k], per_step[k][1]), (name, "ref", k)
        assert torch.equal(rew[k], per_step[k][2]), (name, "reward", k)
        assert torch.equal(term[k], per_step[k][3]), (name, "terminated", k)
    # c: 5 fused steps (last only) + 7 (every step) + 12 (every 4th): the clock carries over between launches
    last = c.rollout(dev[:5], record_every=0)
    for x, y in zip(last, per_step[4]):
        assert torch.equal(x, y), (name, "last-only")
    o7 = c.rollout(dev[5:12], record_every=1)
    for j in range(7):
        assert torch.equal(o7[0][j], per_step[5 + j][0]) and torch.equal(o7[3][j], per_step[5 + j][3])
    o12 = c.rollout(dev[12:24], record_every=4)
    assert o12[0].shape[0] == 3
    for j in range(3):
        for q in range(4):
            assert torch.equal(o12[q][j], per_step[12 + 4 * j + 3][q]), (name, "every 4th", j, q)
    # persistent state afterwards: everything a handle owns, byte for byte
    blobs = [s.state_dict()["blob"] for s in (a, b, c)]
    assert np.array_equal(blobs[0], blobs[1]) and np.array_equal(blobs[0], blobs[2])
    # and the steps that follow agree as well
    for k in range(k_total, k_total + 3):
        outs = [tuple(t.clone() for t in s.step(dev[k])) for s in (a, b, c)]
        for q in range(4):
            assert torch.equal(outs[0][q], outs[1][q]) and torch.equal(outs[0][q], outs[2][q])
    n_term = sum(int(p[3].sum().item()) for p in per_step)
    if name in ("pmsm_cc_rk4", "eesm_cc_rk4", "permex_cc_rk4"):
        assert n_term > 0, "the case is meant to cross terminations + in-kernel resets inside the rollout"
    for s in (a, b, c):
        s.close()


@pytest.mark.parametrize("case", ["wiener_sinus_step", "const_laplace_triangular"])
def test_rollout_with_switched_and_periodic_generators(torch_cuda, case):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    kinds = dict(
        wiener_sinus_step=[dict(kind=K.REF_WIENER, margin=(-0.5, 0.5)), dict(kind=K.REF_SINUS), dict(kind=K.REF_STEP, amp=(0.05, 0.2))],
        const_laplace_triangular=[dict(kind=K.REF_CONST, value=0.25), dict(kind=K.REF_LAPLACE, sigma=(1e-3, 5e-3)), dict(kind=K.REF_TRIANGULAR)])[case]
    n, k_total = 300, 60
    cfg = switched_config(n, kinds, [1.0 / 3] * 3, (5, 12), seed=21, dtype=K.F32)
    cfg.n_constraints = 1
    a, b = VectorSim(cfg), VectorSim(cfg)
    rng = np.random.default_rng(1)
    acts = rng.uniform(-1, 1, size=(k_total, n, a.n_act))
    dev = _dev_actions(torch, a, acts)
    a.reset()
    b.reset()
    per_step = [tuple(t.clone() for t in a.step(dev[k])) for k in range(k_total)]
    out = b.rollout(dev, record_every=1)
    for k in range(k_total):
        for q in range(4):
            assert torch.equal(out[q][k], per_step[k][q]), (case, k, q)
    assert np.array_equal(a.state_dict()["blob"], b.state_dict()["blob"])


ORACLE_NAMES = ["pmsm_cc_rk4", "pmsm_fin_sc_rk4", "scim_cc_rk4", "eesm_cc_rk4", "permex_cc_rk4"]
# at the launch shapes of large batches (gpu_helpers.launch_sizes: 64- and 128-thread blocks) also a wrapper, a dead-time + RC + dq, an AC
# supply, an external speed profile and a DFIM configuration
ORACLE_CASES = [pytest.param(name, 1000, id=name) for name in ORACLE_NAMES] + [
    pytest.param(name, size, id=f"{name}-{size}") for size in ("N64", "N128")
    for name in ORACLE_NAMES + ["pmsm_cc_cossin_rk4", "eesm_cc_rc_dq_dead1_rk4", "pmsm_cc_ac_rk4", "pmsm_cc_extspeed_rk4", "dfim_cc_rk4"]]


@pytest.mark.parametrize("dtype", [K.F64, K.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("name,n", ORACLE_CASES)
def test_rollout_matches_oracle(torch_cuda, oracle_lib, name, n, dtype):
    """the rollout path against the CPU oracle directly (not only through the step kernel): full trajectory of every env, 1000 envs x 60
    steps, and whole batches of N64 / N128 envs (one-warp blocks no longer) x 12 steps"""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    n, k_total = (n, 60) if n == 1000 else (launch_sizes()[n], 12)
    tol = _tol(name, dtype)
    g, cfg = _mk(name, n, dtype, K.LAYOUT_AOS)
    _, cfg_o = _mk(name, n, K.F64, K.LAYOUT_AOS)
    sim, ora = VectorSim(cfg), oracle_lib.Oracle(cfg_o, nthreads=8)
    rng = np.random.default_rng(11)
    acts = _random_actions(rng, g, n, k_total)
    sim.reset()
    ora.reset()
    obs, ref, rew, term = [t.cpu().numpy() for t in sim.rollout(_dev_actions(torch, sim, acts), record_every=1)]
    alive = np.ones(n, dtype=bool)
    scale = np.full(obs.shape[2], 1e-3)
    weak_dq = WEAK_DQ_PAIRS.get(cfg.motor_kind, ())
    for k in range(k_total):
        psi = ora.get_ode_state()[:, 3:5] if weak_dq else None
        o_obs, o_ref, o_rew, o_term = ora.step(acts[k])
        d_obs = obs[k].astype(np.float64)
        if weak_dq:  # field-frame columns while the rotor flux is ~0 (DESIGN.md finding 3): compare the magnitude
            fold_weak_dq(weak_dq, np.hypot(psi[:, 0], psi[:, 1]) < 1e-3, d_obs, o_obs)
        alive &= ~(alive & (o_term != term[k]))  # a constraint within rounding of its threshold: the episodes diverge from here
        scale = np.maximum(scale, np.abs(o_obs[alive]).max(axis=0))
        diff = np.abs(d_obs - o_obs)
        for j, nm in enumerate(g["meta"]["state_names"]):
            if nm == "epsilon":
                diff[:, j] = np.abs((d_obs[:, j] - o_obs[:, j] + 1.0) % 2.0 - 1.0)
        assert (diff[alive] / scale).max() < tol, (name, k)
        assert np.abs(rew[k] - o_rew)[alive].max() < 20 * tol
        if ref.shape[-1]:
            assert np.abs(ref[k] - o_ref)[alive].max() < 20 * tol
    assert alive.mean() > 0.995


@pytest.mark.parametrize("layout", [K.LAYOUT_AOS, K.LAYOUT_SOA], ids=["aos", "soa"])
@pytest.mark.parametrize("name", ["pmsm_cc_rk4", "eesm_cc_rc_dq_dead1_rk4"])  # PLAIN and general instantiation
def test_any_subset_of_outputs_may_be_requested(torch_cuda, name, layout):
    """Every output of gemb200_step / gemb200_rollout_record is optional (NULL): the requested ones carry the same bits as in the all-outputs
    call (the kernels have a fast path for "all four" and a per-output path), the others are not written, the persistent state does not
    depend on what was asked for."""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim, _ptr

    n, k_total, every = 333, 6, 2
    g, cfg = _mk(name, n, K.F32, layout)
    rng = np.random.default_rng(11)
    acts = _random_actions(rng, g, n, k_total + 1)
    full = VectorSim(cfg)
    dev = _dev_actions(torch, full, acts)
    full.reset()
    want = full.rollout(dev[:k_total], record_every=every)
    want_step = tuple(t.clone() for t in full.step(dev[k_total]))
    blob = full.state_dict()["blob"]
    for mask in (0b0001, 0b0110, 0b1000, 0b1011, 0b0000):
        sim = VectorSim(cfg)
        sim.reset()
        outs = [torch.full_like(w, 7) for w in want]
        sel = [o if (mask >> q) & 1 else None for q, o in enumerate(outs)]
        sim.rollout_into(dev[:k_total], k_total, every, *sel)
        single = [torch.full_like(w, 7) for w in want_step]
        ssel = [o if (mask >> q) & 1 else None for q, o in enumerate(single)]
        K.check(sim._lib.gemb200_step(sim._h, _ptr(dev[k_total]), _ptr(ssel[0]), _ptr(ssel[1]) if sim.n_ref else None, _ptr(ssel[2]), _ptr(ssel[3]),
                                      sim._stream()), "gemb200_step")
        torch.cuda.synchronize()
        for q in range(4):
            if (mask >> q) & 1:
                assert torch.equal(outs[q], want[q]) and torch.equal(single[q], want_step[q]), (name, mask, q)
            else:
                assert bool((outs[q] == 7).all()) and bool((single[q] == 7).all()), (name, mask, q, "written although not requested")
        assert np.array_equal(sim.state_dict()["blob"], blob), (name, mask)
        sim.close()
    full.close()


@pytest.mark.parametrize("name", ["pmsm_cc_rk4", "eesm_cc_rc_dq_dead1_rk4", "pmsm_fin_sc_rk4_interlock"])
def test_device_clock_gives_the_same_bits_as_the_host_clock(torch_cuda, name):
    """gemb200_set_device_clock: step / rollout / reset launches that read the RNG call id, the step count and the dead-time ring position
    from device memory (and tick them with a one-thread kernel) must reproduce the host-clocked launches exactly — outputs, persistent
    state and the clock itself — also across switching the mode on and off and a checkpoint taken while it is on."""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    n = 500
    g, cfg = _mk(name, n, K.F32, K.LAYOUT_AOS)
    if cfg.dead_time_steps:
        cfg.dead_time_steps = 3  # a ring longer than one slot: the position is (step count) mod 3
    rng = np.random.default_rng(3)
    acts = _random_actions(rng, g, n, 40)
    a, b = VectorSim(cfg), VectorSim(cfg)
    dev = _dev_actions(torch, a, acts)
    for s in (a, b):
        s.reset()
    b.set_device_clock(True)
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mask[::7] = 1

    def both(fn):
        ra, rb = fn(a), fn(b)
        for x, y in zip(ra, rb):
            assert torch.equal(x, y)

    for k in range(5):
        both(lambda s: tuple(t.clone() for t in s.step(dev[k])))
    both(lambda s: s.rollout(dev[5:16], record_every=1))
    both(lambda s: tuple(t.clone() for t in s.reset(mask)))
    both(lambda s: s.rollout(dev[16:23], record_every=0))
    assert a.clock() == b.clock() and a.clock()[1] == 5 + 11 + 7
    sd = b.state_dict()  # taken with the device clock on: carries the clock
    assert np.array_equal(a.state_dict()["blob"], sd["blob"])
    b.set_device_clock(False)  # back to the host clock: the counters were read back
    for k in range(23, 27):
        both(lambda s: tuple(t.clone() for t in s.step(dev[k])))
    b.set_device_clock(True)
    b.load_state_dict(sd)  # rewind b to step 23 while the device clock is on
    a.load_state_dict(sd)
    for k in range(23, 30):
        both(lambda s: tuple(t.clone() for t in s.step(dev[k])))
    assert a.clock() == b.clock()
    for s in (a, b):
        s.close()


def test_captured_closed_loop_steps_match_the_eager_loop(torch_cuda):
    """env.capture_steps: K x (policy, env.step) in ONE CUDA graph (device-resident clock); three replays against the same closed loop run
    step by step on a second env — every recorded step, the clock and the persistent state afterwards, and ordinary steps that follow."""
    torch = torch_cuda
    import gym_electric_motor_b200 as gem

    n, k_steps = 4096, 8
    mk = lambda: gem.make("Cont-CC-PMSM-v0", num_envs=n, ode_solver=gem.physical_systems.RK4Solver(), autoreset="same_step", seed=5)  # noqa: E731
    e1, e2 = mk(), mk()
    (s1, r1), _ = e1.reset()
    e2.reset()
    idx = torch.as_tensor([e1.physical_system.state_names.index(nm) for nm in e1.reference_generator.reference_names], device="cuda")

    def policy(state, ref):  # a P controller on the referenced currents, spread over the three phases
        err = (ref - state.index_select(1, idx)) * 3.0
        return torch.stack([err[:, 0], err[:, 1], -(err[:, 0] + err[:, 1])], dim=1).clamp(-1.0, 1.0).contiguous()

    cap = e2.capture_steps(policy, k_steps, record=True)
    launches0 = e2.sim.launch_count
    for rep in range(3):
        (st, rf), rw, tm = cap.replay()
        for k in range(k_steps):
            (s1, r1), w1, t1, _, _ = e1.step(policy(s1, r1))
            assert torch.equal(cap.states[k], s1) and torch.equal(cap.references[k], r1), (rep, k)
            assert torch.equal(cap.rewards[k], w1) and torch.equal(cap.terminateds[k], t1), (rep, k)
        assert torch.equal(st, s1) and torch.equal(rw, w1) and torch.equal(tm, t1)
    assert e2.sim.launch_count == launches0, "a replay goes through no library call"
    assert e2.physical_system.k == e1.physical_system.k == 3 * k_steps
    cap.release()
    assert e1.sim.clock() == e2.sim.clock()
    assert np.array_equal(e1.sim.state_dict()["blob"], e2.sim.state_dict()["blob"])
    a = torch.rand((n, 3), device="cuda") * 2 - 1
    (x1, y1), w1, t1, _, _ = e1.step(a)
    (x2, y2), w2, t2, _, _ = e2.step(a)
    assert torch.equal(x1, x2) and torch.equal(y1, y2) and torch.equal(w1, w2) and torch.equal(t1, t2)
    e1.close()
    e2.close()


def test_peer_store_path_with_one_rank_matches_plain_steps(torch_cuda):
    """distributed.PeerGather with a single rank: the step kernel writes its outputs through the multi-destination store path
    (gemb200_bind_peers, here one destination: the library-allocated gather buffer) — the same bits as an ordinary step of a second
    handle; the flag protocol (signal / wait kernels) runs as with N ranks.  The N-rank form needs torchrun: tools/peer_gather_check.py."""
    torch = torch_cuda
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.distributed import PeerGather

    n = 3000
    mk = lambda: gem.make("Cont-CC-PMSM-v0", num_envs=n, ode_solver=gem.physical_systems.RK4Solver(), autoreset="same_step", seed=9)  # noqa: E731
    e1, e2 = mk(), mk()
    e1.reset()
    e2.reset()
    pg = PeerGather(e2.sim, torch.float32)
    acts = torch.rand((7, n, 3), device="cuda") * 2 - 1
    for k in range(7):
        obs, ref, rew, term = e1.sim.step(acts[k])
        b = pg.step(acts[k])
        pg.finish()
        g_obs, g_ref, g_rew, g_term = pg.views(b)
        assert g_obs.shape[0] == 1
        assert torch.equal(g_obs[0], obs) and torch.equal(g_ref[0], ref) and torch.equal(g_rew[0], rew) and torch.equal(g_term[0], term), k
    pg.check()
    pg.release()
    a = torch.rand((n, 3), device="cuda") * 2 - 1  # unbound again: the specialised single-destination kernels
    o1, o2 = e1.sim.step(a), e2.sim.step(a)
    for x, y in zip(o1, o2):
        assert torch.equal(x, y)
    e1.close()
    e2.close()


def test_env_rollout_public_api(torch_cuda):
    """`env.rollout(actions)` of the batched environment == K x `env.step`, incl. the state filter"""
    torch = torch_cuda
    import gym_electric_motor_b200 as gem

    n, k_total = 2048, 16
    mk = lambda: gem.make("Cont-CC-PMSM-v0", num_envs=n, ode_solver=gem.physical_systems.RK4Solver(), autoreset="same_step", seed=3,  # noqa: E731
                          state_filter=["omega", "i_sd", "i_sq", "epsilon"])
    e1, e2 = mk(), mk()
    e1.reset()
    e2.reset()
    acts = torch.rand((k_total, n, 3), device="cuda") * 2 - 1
    (st, rf), rw, tm = e2.rollout(acts, record_every=1)
    assert st.shape == (k_total, n, 4) and rf.shape == (k_total, n, 2) and tm.dtype == torch.bool
    for k in range(k_total):
        (s1, r1), w1, t1, _, _ = e1.step(acts[k])
        assert torch.equal(s1, st[k]) and torch.equal(r1, rf[k]) and torch.equal(w1, rw[k]) and torch.equal(t1, tm[k])
    assert e2.physical_system.k == k_total
    e1.close()
    e2.close()


def test_full_size_rollout_replication_property(torch_cuda):
    """BASELINE size (N = 2^20, Cont-CC-PMSM-v0, RK4), 16 fused steps: 1024 action streams replicated 1024 times across the grid;
    every replica must be bit-identical to its prototype at every recorded step, and the last step must equal 16 single-step
    launches of a second handle."""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g = load_golden("pmsm_cc_rk4")
    n, proto, k_total = 1 << 20, 1024, 16
    cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=g["reset_ode"], dtype=K.F32, solver="rk4", ref_kind=K.REF_CONST)
    for r in range(cfg.n_ref):
        cfg.ref_value[r] = 0.1 * (r + 1)
    a, b = VectorSim(cfg), VectorSim(cfg)
    a.reset()
    b.reset()
    acts = (torch.rand((k_total, proto, 3), device="cuda") * 2 - 1).repeat(1, n // proto, 1).contiguous()
    obs, ref, rew, term = b.rollout(acts, record_every=4)
    for j in range(k_total // 4):
        v = obs[j].view(n // proto, proto, -1)
        assert torch.equal(v, v[0:1].expand_as(v))
    for k in range(k_total):
        last = a.step(acts[k])
    assert torch.equal(last[0], obs[-1]) and torch.equal(last[2], rew[-1]) and torch.equal(last[3], term[-1])


@pytest.mark.parametrize("dtype,tol", [(K.F64, 1e-9), (K.F32, 1e-5)], ids=["f64", "f32"])
@pytest.mark.parametrize("env_id", ["Cont-SC-PMSM-v0", "Cont-CC-SCIM-v0", "Finite-CC-EESM-v0", "Cont-SC-SeriesDc-v0"])
def test_per_env_parameter_blocks_match_single_parameter_oracles(torch_cuda, oracle_lib, env_id, dtype, tol):
    """Domain randomisation (gemb200_set_env_params): G groups of envs with G different motor / load parameter sets in ONE batch must equal
    G oracle runs, each configured with its group's parameters through the ordinary shared-parameter path (same global env indices -> same
    random streams).  Also: the fused rollout with per-env blocks is bit-identical to single steps, and dropping the blocks restores the
    shared-parameter results bit for bit."""
    torch = torch_cuda
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.vector_sim import VectorSim

    groups, per, steps = 5, 96, 50
    n = groups * per
    mk = lambda: gem.make(env_id, num_envs=n, ode_solver=gem.physical_systems.RK4Solver(), autoreset="same_step", seed=13,  # noqa: E731
                          dtype="float64" if dtype == K.F64 else "float32", env_index_offset=5000)
    env = mk()
    base = env.build_config()
    rng = np.random.default_rng(21)
    mp = np.tile(np.array(list(base.motor_param)), (n, 1))
    lp = np.tile(np.array(list(base.load_param)), (n, 1))
    scale_m = rng.uniform(0.7, 1.4, size=(groups, K.MAX_MOTOR_PARAM))
    scale_m[:, K.MP_P] = 1.0  # pole pairs stay integral (and enter the limits)
    scale_l = rng.uniform(0.7, 1.4, size=(groups, 8))
    scale_l[:, K.LP_TAU_DECAY] = 1.0
    for g in range(groups):
        mp[g * per:(g + 1) * per] *= scale_m[g]
        lp[g * per:(g + 1) * per] *= scale_l[g]
    env.sim.set_env_params(mp, lp)
    oras = []
    for g in range(groups):
        cfg = mk().build_config()
        cfg.n_envs, cfg.dtype, cfg.env_index_offset = per, K.F64, 5000 + g * per
        for j in range(K.MAX_MOTOR_PARAM):
            cfg.motor_param[j] = mp[g * per, j]
        for j in range(8):
            cfg.load_param[j] = lp[g * per, j]
        oras.append(oracle_lib.Oracle(cfg, nthreads=4))
    (s0, _), _ = env.reset()
    for g, ora in enumerate(oras):
        o_obs, _ = ora.reset()
        assert np.abs(s0[g * per:(g + 1) * per].double().cpu().numpy() - o_obs).max() < 1e-6
    sp = env.action_space
    alive = np.ones(n, dtype=bool)
    acts = []
    scim = "SCIM" in env_id
    for k in range(steps):
        a = rng.uniform(-1, 1, size=(n, len(sp.low))) if hasattr(sp, "low") else np.stack([rng.integers(0, int(m), size=n) for m in sp.nvec], axis=1).astype(np.int32)
        acts.append(a)
        (s, r), rew, term, _, _ = env.step(torch.as_tensor(a, device="cuda"))
        s, rew, term = s.double().cpu().numpy(), rew.double().cpu().numpy(), term.cpu().numpy().astype(np.uint8)
        for g, ora in enumerate(oras):
            sl = slice(g * per, (g + 1) * per)
            psi = ora.get_ode_state()[:, 3:5] if scim else None
            o_obs, o_ref, o_rew, o_term = ora.step(a[sl])
            alive[sl] &= ~(o_term != term[sl])
            d, o = s[sl].copy(), o_obs.copy()
            if scim:  # field frame undefined while the flux is ~0 (DESIGN.md finding 3)
                weak = np.hypot(psi[:, 0], psi[:, 1]) < 1e-3
                for arr in (d, o):
                    for p_, q_ in ((5, 6), (10, 11)):
                        arr[weak, p_] = np.hypot(arr[weak, p_], arr[weak, q_])
                        arr[weak, q_] = 0.0
            diff = np.abs(d - o)
            if "epsilon" in env.state_names:
                j = env.state_names.index("epsilon")
                diff[:, j] = np.abs((d[:, j] - o[:, j] + 1.0) % 2.0 - 1.0)
            m = alive[sl] & ~(o_term > 0)
            assert diff[m].max(initial=0.0) < 20 * tol, (g, k)
            assert np.abs(rew[sl] - o_rew)[alive[sl]].max(initial=0.0) < 200 * tol, (g, k)
    assert alive.mean() > 0.98
    # groups really differ: the same action sequence drives group 0 and group 1 to different states
    assert np.abs(s[:per] - s[per:2 * per]).max() > 1e-3
    # fused rollout with per-env blocks == single steps with per-env blocks
    e1, e2 = mk(), mk()
    for e in (e1, e2):
        e.sim.set_env_params(mp, lp)
        e.reset()
    dev = torch.as_tensor(np.array(acts[:12]), device="cuda").to(e1.sim.act_dtype).contiguous()
    (st, rf), rw, tm = e2.rollout(dev, record_every=1)
    for k in range(12):
        (s1, r1), w1, t1, _, _ = e1.step(dev[k])
        assert torch.equal(s1, st[k]) and torch.equal(r1, rf[k]) and torch.equal(w1, rw[k]) and torch.equal(t1, tm[k])
    # back to the shared parameters: bit-identical to an env that never had blocks
    e1.set_env_parameters()
    e3 = mk()
    e1.reset(seed=13)
    e3.reset(seed=13)
    for k in range(5):
        a1, a3 = e1.step(dev[k]), e3.step(dev[k])
        assert torch.equal(a1[0][0], a3[0][0]) and torch.equal(a1[1], a3[1])
