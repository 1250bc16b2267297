"""Windows of a large batch against small handles, bit for bit: the step and rollout kernels at the launch shapes of large batches.

The step and rollout kernels choose their block size from the batch size (pick_block, DESIGN.md §2 "Launch shapes"): one warp per block
below 8 blocks of 64 threads per SM, 128 threads from 8 blocks of 128 per SM on.  The code that only matters with several warps in a block
(each warp's staging rows in shared memory, make_out's per-warp first env and valid count, the inactive lanes of per-env blocks, the L2
prefetch) therefore runs only at large N.  Every env is independent and keyed by its global index, and the library is built with
-fmad=false, so envs [s, s + w) of a handle of N envs must give exactly what a handle of w envs with env_index_offset + s gives on the same
action rows; the small handles always launch one-warp blocks.  N64 and N128 (gpu_helpers.launch_sizes) launch 64 and 128 threads
(test_gpu_launch_mode.test_launch_blocks).

Each case runs a reset, 3 steps, rollouts of 6 steps (every step recorded), 7 (every third) and 4 (last only), a seeded masked reset of about
a tenth of the envs and 2 more steps, compares every output of every window and then the window's packed env rows (same clock on both
sides).  The last test checks that misaligned caller buffers are refused before any launch."""
import ctypes as C

import numpy as np
import pytest

from gpu_helpers import _dev_actions, _draws, _eq, launch_sizes, torch_cuda  # noqa: F401
from helpers import ENV_PARAM_CASES, LP_SLOT, MOTOR_SLOTS, MP_SLOT, ROLLOUT_CASES, _mk, _random_actions, motor_of
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

STEPS = 22  # 3 steps, rollouts of 6, 7 and 4 steps, 2 steps after the masked reset
SIZES = ["N64", "N128"]
# one per-env parameter case per motor family, the finite B6 bridge with interlocking time and dq actions on the FluxObserver's angle
ENVP_CASES = ["sc-permex", "sc-extex", "sc-pmsm", "sc-eesm", "sc-scim", "cc-dfim", "fin-sc-pmsm-interlock", "cc-scim-observer-dq"]


def _windows(n, pf):
    """[start, end) of the compared windows: the first blocks' warp slots, 200 mid-batch envs off the warp grid, the prefetch distance, the
    last block, the last env alone and 33 envs from an odd start"""
    mid, odd = 128 * (n // 256) + 77, 3 * (n // 7) | 1
    return [(0, 256), (mid, mid + 200), (pf - 40, min(pf + 40, n)), (n - 300, n), (n - 1, n), (odd, odd + 33)]


def _cut(t, s, e, soa, stacked):
    """envs [s, e) of an output, an action or a feed tensor: [..., N] (SoA rows, per-env scalars) or [(K,) N, ...] (row-per-env)"""
    if t.dim() - stacked == 1 or soa:
        return t[..., s:e]
    return t[:, s:e] if stacked else t[s:e]


def _clone(ts):
    return tuple(t.clone() for t in ts)


def _drive(sim, acts, mask, refs=None, returns=False, prep=None):
    """the sequence of the module docstring on `sim`: [(what, tensors, stacked)] of every output.  refs: a reference feed of STEPS steps
    (step(reference=...) and rollout(references=...)); returns: the 4-step rollout is rollout_returns(discount=0.9); prep(sim): runs right
    after the first reset"""
    feed = (lambda a, b: None) if refs is None else (lambda a, b: refs[a:b])
    one = (lambda k: None) if refs is None else (lambda k: refs[k])
    out = [("reset", _clone(sim.reset()), 0)]
    if prep is not None:
        prep(sim)
    for k in range(3):
        out.append((f"step {k}", _clone(sim.step(acts[k], reference=one(k))), 0))
    out.append(("rollout K=6 every 1", sim.rollout(acts[3:9], 1, feed(3, 9)), 1))
    out.append(("rollout K=7 every 3", sim.rollout(acts[9:16], 3, feed(9, 16)), 1))
    if returns:
        ret, end, (obs, ref) = sim.rollout_returns(acts[16:20], 0.9, feed(16, 20))
        out.append(("rollout_returns K=4", (ret, end, obs.clone(), ref.clone()), 0))
    else:
        out.append(("rollout K=4 every 0", _clone(sim.rollout(acts[16:20], 0, feed(16, 20))), 0))
    out.append(("masked reset", _clone(sim.reset(mask)), 0))
    for k in (20, 21):
        out.append((f"step {k}", _clone(sim.step(acts[k], reference=one(k))), 0))
    return out


def _rows(sim):
    """everything a snapshot packs of every env: state rows, effective RNG identities and (row-per-env) physical parameters"""
    snap = sim.snapshot(rng=True, params=not sim.soa)
    return [snap.rows, snap.rng] + ([snap.params] if snap.params is not None else [])


def _compare_windows(torch, cfg_of, n, acts, setup=None, refs=None, returns=False, prep=None):
    """the big handle of n envs against one small handle per window (cfg_of(w, s): the configuration of w envs from global env s on);
    acts: the actions of all n envs, or a function of the big handle that makes them; setup(sim, s, e) gives both the window's per-env
    state before the sequence, prep(sim, s, e) right after the first reset"""
    from gym_electric_motor_b200.vector_sim import VectorSim

    sz = launch_sizes()
    mask = torch.as_tensor(np.random.default_rng([n, 7]).random(n) < 0.1, device="cuda").to(torch.uint8)
    big = VectorSim(cfg_of(n, 0))
    soa = big.soa
    if callable(acts):
        acts = acts(big)
    if setup is not None:
        setup(big, 0, n)
    want = _drive(big, acts, mask, refs, returns, None if prep is None else (lambda sim: prep(sim, 0, n)))
    want_rows = _rows(big)
    for s, e in _windows(n, sz["PF"]):
        small = VectorSim(cfg_of(e - s, s))
        if setup is not None:
            setup(small, s, e)
        got = _drive(small, _cut(acts, s, e, soa, 1).contiguous(), mask[s:e].contiguous(),
                     None if refs is None else _cut(refs, s, e, soa, 1).contiguous(), returns,
                     None if prep is None else (lambda sim: prep(sim, s, e)))
        for (what, ws, stacked), (_, gs, _) in zip(want, got):
            for j, (w, g) in enumerate(zip(ws, gs)):
                _eq(torch, _cut(w, s, e, soa, stacked), g, (n, (s, e), what, j))
        for j, (w, g) in enumerate(zip(want_rows, _rows(small))):
            _eq(torch, w[s:e], g, (n, (s, e), "snapshot", j))
        small.close()
    big.close()


# ------------------------------------------------------------------------------------------------------ (a) the instantiation matrix
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("layout", [K.LAYOUT_AOS, K.LAYOUT_SOA], ids=["aos", "soa"])
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ROLLOUT_CASES)
def test_windows_match_small_handles(torch_cuda, name, dtype, layout, size):
    """test_gpu_rollout's configurations (every family; PLAIN, general, interlocking, integrating-load, wrapper, dead-time, RC, AC and
    external-speed instantiations) at N64 / N128 against small handles"""
    torch = torch_cuda
    n = launch_sizes()[size]

    def cfg_of(w, s):
        _, cfg = _mk(name, w, dtype, layout)
        cfg.env_index_offset += s
        return cfg

    g, _ = _mk(name, 1, dtype, layout)
    _compare_windows(torch, cfg_of, n, lambda big: _dev_actions(torch, big, _random_actions(np.random.default_rng(5), g, n, STEPS)))


# ------------------------------------------------------------------------------------------------------ (b) per-env blocks, (b') RNG identities
def _env_cfg(case, dtype, layout="aos"):
    """cfg_of(w, s) of a per-env parameter case, and its action space"""
    import gym_electric_motor_b200 as gem

    env_id, kw = ENV_PARAM_CASES[case]()
    env = gem.make(env_id, num_envs=1, dtype="float64" if dtype == K.F64 else "float32", layout=layout, autoreset="same_step", seed=11,
                   env_index_offset=4321, **kw)
    space = env.action_space

    def cfg_of(w, s):
        cfg = env.build_config()
        cfg.n_envs, cfg.env_index_offset = w, cfg.env_index_offset + s
        return cfg

    return env_id, cfg_of, space


def _space_actions(torch, space, n, dtype, seed):
    """[STEPS, N, n_act] seeded actions of an action space: uniform duty cycles, or switching states below nvec / n"""
    rng = np.random.default_rng(seed)
    if hasattr(space, "nvec"):
        a = np.stack([rng.integers(0, int(m), size=(STEPS, n)) for m in space.nvec], axis=2).astype(np.int32)
        return torch.as_tensor(a, device="cuda").contiguous()
    if hasattr(space, "n"):
        return torch.as_tensor(rng.integers(0, int(space.n), size=(STEPS, n, 1)).astype(np.int32), device="cuda").contiguous()
    lo, hi = np.broadcast_to(space.low, (len(space.low),)), np.broadcast_to(space.high, (len(space.high),))
    a = rng.uniform(lo, hi, size=(STEPS, n, len(lo)))
    return torch.as_tensor(a, dtype=torch.float64 if dtype == K.F64 else torch.float32, device="cuda").contiguous()


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", ENVP_CASES)
def test_per_env_blocks_match_small_handles(torch_cuda, case, dtype, size):
    """per-env parameter rows (seeded, +-20 % on the family's slots and the load inertia) and parameter draws at every reset: the ENVP
    instantiations at N64 / N128 against small handles that hold their window's rows (the draws are keyed by the global env index)"""
    torch = torch_cuda
    n = launch_sizes()[size]
    env_id, cfg_of, space = _env_cfg(case, dtype)
    base = cfg_of(1, 0)
    rng = np.random.default_rng(17)
    mp = np.tile(np.array(list(base.motor_param)), (n, 1))
    lp = np.tile(np.array(list(base.load_param)), (n, 1))
    for nm in MOTOR_SLOTS[motor_of(env_id)]:
        mp[:, MP_SLOT[nm]] *= rng.uniform(0.8, 1.2, size=n)
    lp[:, LP_SLOT["j_load"]] *= rng.uniform(0.8, 1.2, size=n)
    draws = _draws(base)

    def setup(sim, s, e):
        sim.set_env_params(mp[s:e], lp[s:e])
        sim.set_param_randomization(*draws)

    _compare_windows(torch, cfg_of, n, _space_actions(torch, space, n, dtype, 3), setup=setup)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", ["sc-pmsm", "sc-scim", "cc-dfim", "fin-sc-pmsm-interlock"])
def test_adopted_rng_identities_match_small_handles(torch_cuda, case, dtype, size):
    """the rows of a 64-env source handle fanned out into every env with their RNG identities (restore(..., rng="source")) by a seeded row
    map, right after the first reset; each small handle adopts the same rows for its window, so both sides run the ENVP instantiations"""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    n = launch_sizes()[size]
    _, cfg_of, space = _env_cfg(case, dtype)
    src_cfg = cfg_of(64, 0)
    src_cfg.env_index_offset = 777_777
    src = VectorSim(src_cfg)
    src.reset()
    src.step(_space_actions(torch, space, 64, dtype, 1)[0])
    snap = src.snapshot(rng=True)
    row_map = torch.as_tensor(np.random.default_rng(23).integers(0, 64, size=n), dtype=torch.int32, device="cuda")

    def prep(sim, s, e):
        sim.restore(snap, rows=row_map[s:e], rng="source")

    _compare_windows(torch, cfg_of, n, _space_actions(torch, space, n, dtype, 4), prep=prep)
    src.close()


# ------------------------------------------------------------------------------------------------------ (c) reference feed and returns
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("layout", ["aos", "soa"])
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
def test_reference_feed_and_returns_match_small_handles(torch_cuda, dtype, layout, size):
    """an External-reference PMSM fed through step(reference=r) and rollout(references=R), and rollout_returns(discount=0.9) with its
    returns and end steps, at N64 / N128 against small handles"""
    torch = torch_cuda
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.reference_generators import ExternalReferenceGenerator as Ext, MultipleReferenceGenerator

    n = launch_sizes()[size]
    env = gem.make("Cont-CC-PMSM-v0", num_envs=1, dtype="float64" if dtype == K.F64 else "float32", layout=layout, autoreset="same_step",
                   seed=5, env_index_offset=999, reference_generator=MultipleReferenceGenerator([Ext("i_sd"), Ext("i_sq")]))

    def cfg_of(w, s):
        cfg = env.build_config()
        cfg.n_envs, cfg.env_index_offset = w, cfg.env_index_offset + s
        return cfg

    tdt = torch.float64 if dtype == K.F64 else torch.float32
    rng = np.random.default_rng(31)
    shape = (STEPS, 2, n) if layout == "soa" else (STEPS, n, 2)
    refs = torch.as_tensor(rng.uniform(-0.6, 0.6, size=shape), dtype=tdt, device="cuda").contiguous()
    a = rng.uniform(-1, 1, size=(STEPS, 3, n) if layout == "soa" else (STEPS, n, 3))
    acts = torch.as_tensor(a, dtype=tdt, device="cuda").contiguous()
    _compare_windows(torch, cfg_of, n, acts, refs=refs, returns=True)


# ------------------------------------------------------------------------------------------------------ misaligned caller buffers
def _refused(sim, rc, name):
    assert rc == K.E_INVALID, (name, rc)
    msg = K.load_library().gemb200_last_error().decode()
    assert name in msg, (name, msg)


@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
def test_misaligned_buffers_are_refused(torch_cuda, dtype):
    """every entry point that takes caller device buffers refuses one that is off its alignment (gemb200.h, "Alignment"): the fp32 row-per-env
    reference output of 2 slots (stored as one float2 per env) offset by 4 bytes, and every fp64 buffer offset by 4 bytes.  A refused call
    launches nothing and leaves the clock alone: the aligned calls after it give a twin handle's bits.  Aligned views (the step slices of an
    action or output tensor) are accepted."""
    torch = torch_cuda
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.vector_sim import VectorSim, _ptr

    n, k = 1000, 4
    env = gem.make("Cont-CC-PMSM-v0", num_envs=n, dtype="float64" if dtype == K.F64 else "float32", autoreset="same_step", seed=3,
                   ode_solver=gem.physical_systems.RK4Solver())
    cfg = env.build_config()
    sim, twin = VectorSim(cfg), VectorSim(cfg)
    assert sim.n_ref == 2
    lib, h, st = sim._lib, sim._h, sim._stream()
    tdt = sim.dtype
    acts = (torch.rand((k + 3, n, 3), device="cuda", dtype=tdt) * 2 - 1).contiguous()
    obs, ref, rew, term = sim._alloc_stacked(k)
    big = torch.zeros(ref.numel() + 64, dtype=tdt, device="cuda")  # 256-byte aligned: big[1:] is 4 bytes off in fp32
    off4 = lambda t: C.c_void_p(t.data_ptr() + 4)  # noqa: E731
    bad = off4(ref)  # ref_out: fp32 needs 8 bytes (float2 per env), fp64 needs 8 bytes (its element)
    feed = torch.zeros((k, n, 2), dtype=tdt, device="cuda")
    nx, nu, ww = sim.return_grad_dims()
    ret = torch.empty(n, dtype=tdt, device="cuda")
    end = torch.empty(n, dtype=torch.int32, device="cuda")
    ws = torch.empty(k * n * ww, dtype=tdt, device="cuda")
    ga, gx = torch.empty((k, n, nu), dtype=tdt, device="cuda"), torch.empty((n, nx), dtype=tdt, device="cuda")
    jx, ju = torch.empty((k, n, nx, nx), dtype=tdt, device="cuda"), torch.empty((k, n, nx, nu), dtype=tdt, device="cuda")
    slots = (C.c_int32 * 1)(K.MP_R_S)
    sio, so = torch.zeros((n, nx, 1), dtype=tdt, device="cuda"), torch.empty((k, n, nx, 1), dtype=tdt, device="cuda")
    a = _ptr(acts)
    calls = [
        ("gemb200_reset", "ref_out", lambda: lib.gemb200_reset(h, None, _ptr(obs[0]), bad, st)),
        ("gemb200_step", "ref_out", lambda: lib.gemb200_step(h, a, _ptr(obs[0]), bad, _ptr(rew[0]), _ptr(term[0]), st)),
        ("gemb200_rollout_record", "ref_out", lambda: lib.gemb200_rollout_record(h, a, k, 1, _ptr(obs), bad, _ptr(rew), _ptr(term), st)),
        ("gemb200_rollout_record_ref", "ref_out",
         lambda: lib.gemb200_rollout_record_ref(h, a, _ptr(feed), k, 1, _ptr(obs), bad, _ptr(rew), _ptr(term), st)),
        ("gemb200_rollout_returns", "ref_out", lambda: lib.gemb200_rollout_returns(h, a, None, k, 0.9, _ptr(ret), _ptr(end), _ptr(obs[0]), bad, st)),
        ("gemb200_rollout_jacobians", "ref_out",
         lambda: lib.gemb200_rollout_jacobians(h, a, None, k, _ptr(jx), _ptr(ju), _ptr(obs), bad, _ptr(rew), _ptr(term), st)),
        ("gemb200_rollout_return_grads", "ref_out",
         lambda: lib.gemb200_rollout_return_grads(h, a, None, k, 0.9, None, _ptr(ws), ws.numel() * ws.element_size(), _ptr(ret), _ptr(end), _ptr(ga),
                                                  _ptr(gx), _ptr(obs[0]), bad, st)),
        ("gemb200_rollout_param_sens", "ref_out",
         lambda: lib.gemb200_rollout_param_sens(h, a, None, k, 1, slots, _ptr(sio), _ptr(so), _ptr(obs), bad, _ptr(rew), _ptr(term), st)),
    ]
    if dtype == K.F64:  # every fp64 buffer is refused 4 bytes off: a few of each kind
        calls += [
            ("gemb200_step", "action", lambda: lib.gemb200_step(h, off4(acts), None, None, None, None, st)),
            ("gemb200_step", "obs_out", lambda: lib.gemb200_step(h, a, off4(obs), None, None, None, st)),
            ("gemb200_step", "reward_out", lambda: lib.gemb200_step(h, a, None, None, off4(rew), None, st)),
            ("gemb200_reset", "obs_out", lambda: lib.gemb200_reset(h, None, off4(obs), None, st)),
            ("gemb200_rollout_record_ref", "references", lambda: lib.gemb200_rollout_record_ref(h, a, off4(feed), k, 1, None, None, None, None, st)),
            ("gemb200_rollout_returns", "return_out", lambda: lib.gemb200_rollout_returns(h, a, None, k, 0.9, off4(ret), None, None, None, st)),
            ("gemb200_rollout_jacobians", "jac_x_out", lambda: lib.gemb200_rollout_jacobians(h, a, None, k, off4(jx), None, None, None, None, None, st)),
            ("gemb200_rollout_return_grads", "workspace",
             lambda: lib.gemb200_rollout_return_grads(h, a, None, k, 0.9, None, off4(ws), ws.numel() * ws.element_size(), _ptr(ret), None, _ptr(ga),
                                                      _ptr(gx), None, None, st)),
            ("gemb200_rollout_return_grads", "grad_a_out",
             lambda: lib.gemb200_rollout_return_grads(h, a, None, k, 0.9, None, _ptr(ws), ws.numel() * ws.element_size(), _ptr(ret), None, off4(ga),
                                                      _ptr(gx), None, None, st)),
            ("gemb200_rollout_param_sens", "sens_io", lambda: lib.gemb200_rollout_param_sens(h, a, None, k, 1, slots, off4(sio), None, None, None, None, None, st)),
        ]
    for s in (sim, twin):
        s.reset()
    torch.cuda.synchronize()
    launches, clock = sim.launch_count, sim.clock()
    for what, name, call in calls:
        _refused(sim, call(), name)
        assert sim.launch_count == launches and sim.clock() == clock, (what, name)
    delta = (C.c_int64 * 1)(8)
    _refused(sim, lib.gemb200_bind_peers(h, 1, C.cast(delta, C.c_void_p)), "dst_delta[0]")
    if dtype == K.F32:  # the Python layer passes caller tensors on: a reference view one element off its allocation is refused there too
        with pytest.raises(K.GemB200Error, match="ref_out"):
            sim.rollout_into(acts[:k], k, 1, obs, big[1:1 + ref.numel()].view(ref.shape), rew, term)
        assert sim.launch_count == launches and sim.clock() == clock
    # aligned calls, slices of the action tensor among them: the bits of a twin that never saw the refused calls
    for j in range(2):
        for q, (x, y) in enumerate(zip(_clone(sim.step(acts[j])), twin.step(acts[j]))):
            _eq(torch, x, y, ("step", j, q))
    for x, y in zip(sim.rollout(acts[2:2 + k], 1), twin.rollout(acts[2:2 + k], 1)):
        _eq(torch, x, y, "rollout")
    for x, y in zip(sim.rollout_returns(acts[2:2 + k], 0.9)[:2], twin.rollout_returns(acts[2:2 + k], 0.9)[:2]):
        _eq(torch, x, y, "returns")
    assert sim.clock() == twin.clock()
    env.close()
    sim.close()
    twin.close()
