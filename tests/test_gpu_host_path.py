"""The host-buffer entry points (gemb200_step_host / gemb200_reset_host) against the device path (gemb200_step / gemb200_reset on the
current stream) of a twin handle of the same configuration, and against the float64 oracle.

From 2^16 envs on, a row-per-env handle's gemb200_step_host cuts the batch into 4 chunks of whole 256-env blocks that flow through three
streams (H2D, launch over the chunk's env range, D2H), all four sharing one RNG call id; below that it is one launch.  A chunk split that
drops envs, a launch over a sub-range that indexes wrongly or a chunk that draws other random numbers shows up here as a row that differs
from the twin's, or as a row the call never wrote: every host buffer is filled with a sentinel (NaN, 0xAB) before each call.  The host
calls are synchronous; they must also see every call queued before them on any stream (the ordering tests queue a spin first, so that
the earlier work is certainly still pending when the host call starts)."""
import ctypes as C

import numpy as np
import pytest

from gym_electric_motor_b200 import _cabi as K
from gpu_helpers import _draws, launch_sizes, torch_cuda  # noqa: F401
from helpers import _mk

pytestmark = pytest.mark.gpu

PIPE = 1 << 16  # gemb200_step_host pipelines row-per-env batches from this size on
STEPS = 24  # with the starts below: terminations, same-step resets and new reference sub-episodes in every chunk
SIZES = [PIPE - 1, PIPE, PIPE + 1, PIPE + 3, PIPE + 37, (1 << 18) + 4099, 1 << 20, (1 << 20) + 3]
SMALL = SIZES[:5]
BENCH = ("pmsm", "fin_sc_pmsm", "fin_sc_pmsm_il")
# general instantiations with side state: dead-time ring, RC supply and dq actions; observation wider than the state; speed profile; AC
# supply; an action width decided at run time
GENERAL = ("eesm_cc_rc_dq_dead1_rk4", "scim_sc_flux_cossin_dead1_rk4", "pmsm_cc_extspeed_rk4", "pmsm_cc_ac_rk4", "extex_cc_rk4")
FP64 = ("eesm_cc_rc_dq_dead1_rk4", "scim_sc_flux_cossin_dead1_rk4")
SPIN = 20_000_000  # clock cycles of the spin kernel queued ahead of a stream-ordered call (~10 ms)


def _chunks(n):
    """[begin, end) of the launches gemb200_step_host makes for a row-per-env handle of n envs"""
    if n < PIPE:
        return [(0, n)]
    per = ((n + 3) // 4 + 255) // 256 * 256
    return [(b, min(b + per, n)) for b in range(0, n, per)]


def _sampler(n, n_act, dtype, finite_hi=None, nonneg=False, seed=0):
    """act(k): the seeded actions of step k, [n, n_act] in the handle's action dtype, made on demand (2^20 envs x 25 steps would not
    fit comfortably at once): switching states below finite_hi per slot, or duty cycles = half a per-env constant plus half noise"""
    hold = np.random.default_rng([seed, 1 << 30]).uniform(-1, 1, size=(n, n_act))

    def act(k):
        rng = np.random.default_rng([seed, k])
        if finite_hi is not None:
            return (rng.random((n, n_act)) * np.asarray(finite_hi)).astype(np.int32)
        a = 0.5 * rng.uniform(-1, 1, size=(n, n_act)) + 0.5 * hold
        return (np.abs(a) if nonneg else a).astype(dtype)

    return act


def _bench_case(name, n, dtype=K.F32):
    """the bench's configuration `name` at n envs, with the motor current started near its limit and reference sub-episodes of 3-9
    steps (the kernel instantiation does not depend on either)"""
    import bench

    env = bench.make_env(name, n)
    cfg = env.build_config()
    cfg.dtype = dtype
    names = list(env.state_names)
    cur = names.index("i_sd") if "i_sd" in names else names.index("i_a")
    cfg.init_ode[1] = (0.97 if cfg.finite else 0.9) * cfg.limits[cur]
    for r in range(cfg.n_ref):
        cfg.ref_len_lo[r], cfg.ref_len_hi[r] = 3, 9
    sp = env.action_space
    np_dt = np.float32 if dtype == K.F32 else np.float64
    if hasattr(sp, "nvec"):
        act = _sampler(n, len(sp.nvec), np_dt, finite_hi=np.asarray(sp.nvec))
    elif hasattr(sp, "n"):
        act = _sampler(n, 1, np_dt, finite_hi=[int(sp.n)])
    else:
        act = _sampler(n, len(sp.low), np_dt, nonneg=bool(np.min(sp.low) >= 0))
    return cfg, act, names


def _golden_case(name, n, dtype=K.F32):
    """test_gpu_rollout's configuration of golden `name` (Wiener references, same-step auto-reset) with _random_actions' action ranges"""
    g, cfg = _mk(name, n, dtype, K.LAYOUT_AOS)
    a = g["actions"]
    np_dt = np.float32 if dtype == K.F32 else np.float64
    if a.ndim == 1:
        act = _sampler(n, 1, np_dt, finite_hi=[max(int(a.max()) + 1, 2)])
    elif a.dtype.kind == "i":
        act = _sampler(n, a.shape[1], np_dt, finite_hi=a.max(axis=0) + 1)
    else:
        act = _sampler(n, a.shape[1], np_dt, nonneg=bool(a.min() >= 0))
    return cfg, act, list(g["meta"]["state_names"])


def _sentinel(sim):
    """host output buffers (obs, ref, reward, terminated) holding NaN / 0xAB"""
    return (np.full(sim._shape(sim.n_state), np.nan, sim.np_dtype), np.full(sim._shape(sim.n_ref), np.nan, sim.np_dtype),
            np.full(sim.n, np.nan, sim.np_dtype), np.full(sim.n, 0xAB, np.uint8))


def _refill(bufs):
    for b in bufs[:3]:
        b.fill(np.nan)
    bufs[3].fill(0xAB)


def _same_bits(x, y, what):
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    assert x.shape == y.shape and x.dtype == y.dtype, (what, x.shape, y.shape, x.dtype, y.dtype)
    if x.size == 0:
        return
    xb, yb = x.view(np.uint8).reshape(x.shape[0], -1), y.view(np.uint8).reshape(y.shape[0], -1)
    bad = np.flatnonzero((xb != yb).any(axis=1))
    assert bad.size == 0, f"{what}: {bad.size} rows differ, first {bad[:8]}, last {bad[-1]} of {x.shape[0]}"


def _host(t):
    return t.cpu().numpy()


def _dev(torch, sim, a):
    return torch.from_numpy(a).to(sim.device)


def _state(sim, kind):
    """everything the handle owns: the checkpoint blob, or, where checkpoints are refused (parameters drawn per reset, adopted RNG
    identities), the packed env rows with their parameters or identities; and the clock"""
    if kind == "draws":
        s = sim.snapshot(params=True)
        return [_host(s.rows), _host(s.params), _host(sim.env_params())], sim.clock()
    if kind == "rng_ids":
        s = sim.snapshot(rng=True)
        return [_host(s.rows), _host(s.rng)], sim.clock()
    return [sim.state_dict()["blob"]], sim.clock()


def _assert_same_state(host, twin, kind, what):
    (sh, ch), (st, ct) = _state(host, kind), _state(twin, kind)
    assert ch == ct, (what, "clock", ch, ct)
    for j, (x, y) in enumerate(zip(sh, st)):
        _same_bits(x, y, f"{what} state {j}")


def _step_twins(torch, host, twin, act, ks, what, launches=None):
    """step k of `host` through gemb200_step_host and of `twin` through gemb200_step, for k in ks: every output bit for bit, and the
    launches the host call makes (default: one per chunk); returns the terminations per env summed over the steps"""
    out = _sentinel(host)
    n_launch = len(_chunks(host.n)) if launches is None else launches
    term = np.zeros(host.n, dtype=np.int64)
    for k in ks:
        a = act(k)
        _refill(out)
        l0 = host.launch_count
        host.step_host(a, out)
        assert host.launch_count - l0 == n_launch, (what, k, "launches", host.launch_count - l0)
        want = [_host(t) for t in twin.step(_dev(torch, twin, a))]
        for q, nm in enumerate(("obs", "ref", "reward", "terminated")):
            _same_bits(out[q], want[q], f"{what} step {k} {nm}")
        term += out[3]
    return term


def _case(kind, name, dtype, n):
    return _bench_case(name, n, dtype) if kind == "bench" else _golden_case(name, n, dtype)


def _pipeline_cases():
    out = []
    for n in SIZES:
        out += [pytest.param("bench", b, K.F32, n, id=f"{b}-{n}") for b in BENCH]
    out += [pytest.param("bench", "scim", K.F32, n, id=f"scim-{n}") for n in SIZES[-2:]]
    # NHOST (gpu_helpers.launch_sizes): the chunks launch 64-thread blocks while the twin's full-batch step launches 128, so the two sides
    # run one configuration at two launch shapes
    out += [pytest.param("bench", b, K.F32, "NHOST", id=f"{b}-NHOST") for b in BENCH]
    for n in SMALL + ["NHOST"]:
        out += [pytest.param("golden", g, K.F32, n, id=f"{g}-{n}") for g in GENERAL]
        out += [pytest.param("golden", g, K.F64, n, id=f"{g}-f64-{n}") for g in FP64]
        out += [pytest.param("draws", "pmsm_cc_rk4", K.F32, n, id=f"envp_draws-{n}"), pytest.param("rng_ids", "pmsm_cc_rk4", K.F32, n, id=f"rng_ids-{n}")]
    return out


# ---------------------------------------------------------------------------------------------------- 1. pipelined step == device step
@pytest.mark.parametrize("kind,name,dtype,n", _pipeline_cases())
def test_step_host_equals_device_step(torch_cuda, kind, name, dtype, n):
    """24 + 1 steps through the host buffers against the device path of a twin: obs, ref, reward and terminated of every env in every
    step, the state afterwards, the launches per call (4 chunk launches from 2^16 envs on, else 1).  Every chunk must see terminations.
    draws: per-env parameter blocks that also draw R_s, L_d, L_q, psi_p and J at every reset; rng_ids: every env has adopted another env's
    state and RNG identity (restore(..., rng="source"))."""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    n = launch_sizes()[n] if n == "NHOST" else n
    cfg, act, _ = _case("bench" if kind == "bench" else "golden", name, dtype, n)
    host, twin = VectorSim(cfg), VectorSim(cfg)
    rng = np.random.default_rng(n)
    if kind == "draws":
        mp = np.tile(np.array(list(cfg.motor_param)), (n, 1))
        lp = np.tile(np.array(list(cfg.load_param)), (n, 1))
        mp[:, K.MP_R_S] *= rng.uniform(0.8, 1.2, size=n)
        lp[:, K.LP_J_LOAD] *= rng.uniform(0.8, 1.2, size=n)
    perm = rng.permutation(n)
    for s in (host, twin):
        if kind == "draws":
            s.set_env_params(mp, lp)
            s.set_param_randomization(*_draws(cfg))
        s.reset()
        if kind == "rng_ids":
            s.restore(s.snapshot(rng=True), rows=perm, rng="source")
    torch.cuda.synchronize()
    term = _step_twins(torch, host, twin, act, range(STEPS), name)
    for b, e in _chunks(n):
        assert term[b:e].sum() > 0, (name, n, "no termination in chunk", b, e)
    _assert_same_state(host, twin, kind, name)
    _step_twins(torch, host, twin, act, [STEPS], f"{name} after")
    host.close()
    twin.close()


def test_pinned_host_buffers_give_the_same_bits(torch_cuda):
    """the bench's e2e route (page-locked torch tensors through step_host_ptr) against pageable numpy buffers, at 2^20 envs"""
    torch = torch_cuda
    from gym_electric_motor_b200 import hostmem
    from gym_electric_motor_b200.vector_sim import VectorSim

    n = 1 << 20
    cfg, act, _ = _bench_case("pmsm", n)
    pin, page = VectorSim(cfg), VectorSim(cfg)
    for s in (pin, page):
        s.reset()
    torch.cuda.synchronize()
    h_act = hostmem.pinned_empty((n, pin.n_act), torch.float32)
    h_out = [hostmem.pinned_empty((n, pin.n_state), torch.float32), hostmem.pinned_empty((n, pin.n_ref), torch.float32),
             hostmem.pinned_empty((n,), torch.float32), hostmem.pinned_empty((n,), torch.uint8)]
    out = _sentinel(page)
    for k in range(8):
        a = act(k)
        h_act.numpy()[:] = a
        for t in h_out[:3]:
            t.fill_(float("nan"))
        h_out[3].fill_(0xAB)
        _refill(out)
        pin.step_host_ptr(h_act.data_ptr(), *[t.data_ptr() for t in h_out])
        page.step_host(a, out)
        for q in range(4):
            _same_bits(h_out[q].numpy(), out[q], f"pinned step {k} output {q}")
    _assert_same_state(pin, page, "plain", "pinned")
    pin.close()
    page.close()


# ---------------------------------------------------------------------------------------------------- 2. oracle windows
@pytest.mark.parametrize("n", [PIPE + 37, (1 << 20) + 3])
@pytest.mark.parametrize("name", ["pmsm", "eesm_cc_rc_dq_dead1_rk4"])
def test_chunk_boundaries_match_the_oracle(torch_cuda, oracle_lib, name, n):
    """128-env windows across every chunk boundary of the pipelined host step, and the last 128 envs, against float64 oracles at the
    same global env indices; the bar of test_rollout_matches_oracle (fp32: 1e-5 of the column scale; an env whose termination differs
    from the oracle's has left the oracle's episode and is dropped, at most 0.5 % may)"""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    tol, w = 1e-5, 128
    cfg, act, names = _bench_case(name, n) if name in BENCH else _golden_case(name, n)
    sim = VectorSim(cfg)
    starts = [b - w // 2 for b, _ in _chunks(n)[1:]] + [n - w]
    assert len(starts) == 4
    oras = []
    for s0 in starts:
        c = type(cfg).from_buffer_copy(cfg)
        c.n_envs, c.dtype, c.env_index_offset = w, K.F64, cfg.env_index_offset + s0
        oras.append(oracle_lib.Oracle(c, nthreads=4))
    sim.reset()
    for o in oras:
        o.reset()
    torch.cuda.synchronize()
    ang = [j for j, nm in enumerate(names) if nm == "epsilon"]
    alive = [np.ones(w, dtype=bool) for _ in starts]
    scale = [None] * len(starts)
    out = _sentinel(sim)
    for k in range(STEPS):
        a = act(k)
        _refill(out)
        sim.step_host(a, out)
        for j, (s0, o) in enumerate(zip(starts, oras)):
            sl = slice(s0, s0 + w)
            o_obs, o_ref, o_rew, o_term = o.step(a[sl].astype(np.float64) if a.dtype.kind == "f" else a[sl])
            d_obs = out[0][sl].astype(np.float64)
            assert np.isin(out[3][sl], (0, 1)).all(), (name, n, s0, k, "rows the call did not write")
            alive[j] &= o_term == out[3][sl]
            scale[j] = np.full(d_obs.shape[1], 1e-3) if scale[j] is None else scale[j]
            scale[j] = np.maximum(scale[j], np.abs(o_obs[alive[j]]).max(axis=0, initial=0.0))
            diff = np.abs(d_obs - o_obs)
            for c_ in ang:
                diff[:, c_] = np.abs((d_obs[:, c_] - o_obs[:, c_] + 1.0) % 2.0 - 1.0)
            assert (diff[alive[j]] / scale[j]).max(initial=0.0) < tol, (name, n, s0, k)
            assert np.abs(out[2][sl] - o_rew)[alive[j]].max(initial=0.0) < 20 * tol, (name, n, s0, k)
            if out[1].shape[-1]:
                assert np.abs(out[1][sl] - o_ref)[alive[j]].max(initial=0.0) < 20 * tol, (name, n, s0, k)
    assert np.concatenate(alive).mean() > 0.995
    sim.close()


# ---------------------------------------------------------------------------------------------------- 3. NULL outputs
@pytest.mark.parametrize("n", [300, PIPE + 37])
@pytest.mark.parametrize("name", ["pmsm_cc_rk4", "eesm_cc_rc_dq_dead1_rk4"])  # PLAIN and general instantiation
def test_step_host_with_null_outputs(torch_cuda, name, n):
    """every output of gemb200_step_host may be NULL: the requested ones carry the bits of the twin's all-outputs step, the others keep
    their sentinel, and the clock and random streams advance as in a full call (the full step that follows equals the twin's)"""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    k_masked = 6
    cfg, act, _ = _golden_case(name, n)
    twin = VectorSim(cfg)
    twin.reset()
    want = [[_host(t) for t in twin.step(_dev(torch, twin, act(k)))] for k in range(k_masked + 1)]
    blob = twin.state_dict()["blob"]
    vp = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)  # noqa: E731
    for mask in (0b1111, 0b0000, 0b0001, 0b0010, 0b0100, 0b1000):
        sim = VectorSim(cfg)
        sim.reset()
        torch.cuda.synchronize()
        out = _sentinel(sim)
        for k in range(k_masked):
            _refill(out)
            sel = [o if (mask >> q) & 1 else None for q, o in enumerate(out)]
            a = act(k)
            K.check(sim._lib.gemb200_step_host(sim._h, vp(a), vp(sel[0]), vp(sel[1]) if sim.n_ref else None, vp(sel[2]), vp(sel[3])),
                    "gemb200_step_host")
            for q in range(4):
                if (mask >> q) & 1:
                    _same_bits(out[q], want[k][q], f"{name} mask {mask:04b} step {k} output {q}")
                else:
                    _same_bits(out[q], _sentinel(sim)[q], f"{name} mask {mask:04b} step {k} output {q} written although not requested")
        full = sim.step_host(act(k_masked))
        for q in range(4):
            _same_bits(full[q], want[k_masked][q], f"{name} mask {mask:04b} full step {q}")
        assert np.array_equal(sim.state_dict()["blob"], blob), (name, mask)
        sim.close()
    twin.close()


# ---------------------------------------------------------------------------------------------------- 4. masked reset_host
@pytest.mark.parametrize("n", [300, PIPE + 3])
@pytest.mark.parametrize("name", ["pmsm_cc_rk4", "eesm_cc_rc_dq_dead1_rk4"])
def test_masked_reset_host_keeps_the_callers_rows(torch_cuda, name, n):
    """gemb200_reset_host with a mask: masked rows equal the twin's gemb200_reset(mask), unmasked rows of the caller's obs / ref buffers
    keep what the caller had in them, and the state afterwards (and the step after it) equals the twin's"""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    cfg, act, _ = _golden_case(name, n)
    host, twin = VectorSim(cfg), VectorSim(cfg)
    for s in (host, twin):
        s.reset()
    torch.cuda.synchronize()
    _step_twins(torch, host, twin, act, range(5), name)
    mask = np.zeros(n, dtype=np.uint8)
    mask[::3] = 1
    rng = np.random.default_rng(4)
    obs = rng.standard_normal(host._shape(host.n_state)).astype(host.np_dtype)
    ref = rng.standard_normal(host._shape(host.n_ref)).astype(host.np_dtype)
    obs0, ref0 = obs.copy(), ref.copy()
    vp = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
    K.check(host._lib.gemb200_reset_host(host._h, vp(mask), vp(obs), vp(ref) if host.n_ref else None), "gemb200_reset_host")
    w_obs, w_ref = [_host(t) for t in twin.reset(torch.as_tensor(mask, device=twin.device))]
    m = mask.astype(bool)
    _same_bits(obs[m], w_obs[m], f"{name} reset obs (masked rows)")
    _same_bits(obs[~m], obs0[~m], f"{name} reset obs (unmasked rows)")
    if host.n_ref:
        _same_bits(ref[m], w_ref[m], f"{name} reset ref (masked rows)")
        _same_bits(ref[~m], ref0[~m], f"{name} reset ref (unmasked rows)")
    _assert_same_state(host, twin, "plain", name)
    _step_twins(torch, host, twin, act, [5], f"{name} after")
    host.close()
    twin.close()


# ---------------------------------------------------------------------------------------------------- 5. ordering
ORDER_CASES = ["reset", "reset_then_reset_host", "step", "rollout", "reseed", "restore"]


def _queue(case, sim, dev_acts, snap):
    if case.startswith("reset"):
        sim.reset()
    elif case == "step":
        sim.step(dev_acts[0])
    elif case == "rollout":
        sim.rollout(dev_acts[1:5], record_every=1)
    elif case == "reseed":
        sim.reseed(991)
    elif case == "restore":
        sim.restore(snap)


@pytest.mark.parametrize("side", [False, True], ids=["default_stream", "side_stream"])
@pytest.mark.parametrize("case", ORDER_CASES)
def test_host_calls_wait_for_earlier_stream_ordered_calls(torch_cuda, case, side):
    """a stream-ordered call X still pending behind a spin on the launching stream, then at once step_host (or reset_host): the result
    must be that of X followed by the host call, as the twin gets it by doing X, synchronising, then the same call on the device path"""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    n = PIPE + 37
    cfg, act, _ = _golden_case("pmsm_cc_rk4", n)
    host, twin = VectorSim(cfg), VectorSim(cfg)
    dev_acts = torch.as_tensor(np.stack([act(k) for k in range(6)]), device=host.device).contiguous()
    snaps = []
    for s in (host, twin):
        s.reset()
        snaps.append(s.snapshot())
        s.step(dev_acts[5])
    torch.cuda.synchronize()
    a = act(6)
    _queue(case, twin, dev_acts, snaps[1])
    torch.cuda.synchronize()
    want = [_host(t) for t in (twin.reset() if case == "reset_then_reset_host" else twin.step(_dev(torch, twin, a)))]
    stream = torch.cuda.Stream() if side else torch.cuda.current_stream()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(SPIN)
        _queue(case, host, dev_acts, snaps[0])
        got = host.reset_host() if case == "reset_then_reset_host" else host.step_host(a)
    torch.cuda.synchronize()
    for q, (x, y) in enumerate(zip(got, want)):
        _same_bits(x, y, f"{case} output {q}")
    _assert_same_state(host, twin, "plain", case)
    host.close()
    twin.close()


def test_device_calls_after_a_host_call_see_its_results(torch_cuda):
    """the reverse order: step_host, then device-path calls on a side stream, against a twin that does everything on the device path"""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    n = PIPE + 37
    cfg, act, _ = _golden_case("pmsm_cc_rk4", n)
    host, twin = VectorSim(cfg), VectorSim(cfg)
    for s in (host, twin):
        s.reset()
    torch.cuda.synchronize()
    dev_acts = torch.as_tensor(np.stack([act(k) for k in range(1, 5)]), device=host.device).contiguous()
    _step_twins(torch, host, twin, act, [0], "host step")
    want = [t.clone() for t in twin.rollout(dev_acts, record_every=1)]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        got = host.rollout(dev_acts, record_every=1)
    torch.cuda.synchronize()
    for q, (x, y) in enumerate(zip(got, want)):
        assert torch.equal(x, y), q
    _assert_same_state(host, twin, "plain", "reverse")
    host.close()
    twin.close()


# ---------------------------------------------------------------------------------------------------- 6. device clock
def test_step_host_under_the_device_clock_below_the_pipeline(torch_cuda):
    """below 2^16 envs the host step is one launch, which the device-resident clock allows: the same bits as the device step (the
    dead-time ring position comes from the device clock too)"""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    n = PIPE - 1
    cfg, act, _ = _golden_case("eesm_cc_rc_dq_dead1_rk4", n)
    cfg.dead_time_steps = 3
    host, twin = VectorSim(cfg), VectorSim(cfg)
    for s in (host, twin):
        s.reset()
        s.set_device_clock(True)
    torch.cuda.synchronize()
    _step_twins(torch, host, twin, act, range(12), "device clock", launches=2)  # the step and the clock tick
    _assert_same_state(host, twin, "plain", "device clock")
    host.close()
    twin.close()


def test_pipelined_step_host_refuses_the_device_clock(torch_cuda):
    """from 2^16 envs on the host step is refused while the device clock is on, and the refused call changes nothing: with the clock off
    again the state and the next step equal those of a twin that never made the call"""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    n = PIPE + 37
    cfg, act, _ = _golden_case("eesm_cc_rc_dq_dead1_rk4", n)
    host, twin = VectorSim(cfg), VectorSim(cfg)
    for s in (host, twin):
        s.reset()
    torch.cuda.synchronize()
    _step_twins(torch, host, twin, act, range(3), "before")
    host.set_device_clock(True)
    with pytest.raises(K.GemB200Error, match="device-resident clock"):
        host.step_host(act(3))
    host.set_device_clock(False)
    torch.cuda.synchronize()
    _assert_same_state(host, twin, "plain", "after the refused call")
    _step_twins(torch, host, twin, act, range(3, 6), "after")
    host.close()
    twin.close()
