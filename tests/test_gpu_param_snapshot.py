"""Per-env physical parameters in snapshots on the device (gemb200_pack_envs_params / gemb200_unpack_envs_params): a restored env that takes
its source's parameters runs its episode on the source's plant, so together with the source's RNG identity it replays the source bit for
bit under per-episode domain randomisation — copy.deepcopy(env) of the reference for domain-randomised batches."""
import ctypes as C

import numpy as np
import pytest

from gym_electric_motor_b200 import _cabi as K
from gpu_helpers import _MOTOR_SLOTS, SCIM_RANDOM, _acts, _dev_actions, _draws, _random_cfg, _run, _same_outputs, torch_cuda  # noqa: F401

pytestmark = pytest.mark.gpu

CASES_P = ["pmsm_cc_rk4", "eesm_cc_rk4", "permex_cc_rk4", "scim_cc_rk4", SCIM_RANDOM, "dfim_cc_rk4"]
CROSS_RESETS = ("pmsm_cc_rk4", "eesm_cc_rk4", "permex_cc_rk4")


def _config_row(cfg):
    return np.r_[np.array(list(cfg.motor_param)), np.array(list(cfg.load_param))]


def _warm(torch, sim, g, rng, k):
    for x in _dev_actions(torch, sim, _acts(rng, g, sim, k)):
        sim.step(x)


def _randomised_pair(torch, name, dtype, m=120, n_a=301, n_b=403):
    """A (seed 77, offset 12345) and B (seed 5, offset 999, other N), both drawing the same parameters at every reset, with different
    histories; A's envs src are then deep-copied into B's envs dst (state, RNG identity and parameters)"""
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, cfg_a = _random_cfg(name, n_a, dtype)
    _, cfg_b = _random_cfg(name, n_b, dtype, seed=5, offset=999)
    a, b = VectorSim(cfg_a), VectorSim(cfg_b)
    for s in (a, b):
        s.set_param_randomization(*_draws(s.cfg))
        s.reset()
    rng = np.random.default_rng(3)
    src, dst = rng.permutation(n_a)[:m], rng.permutation(n_b)[:m]
    _warm(torch, a, g, rng, 7)
    _warm(torch, b, g, rng, 12)
    b.restore(a.snapshot(src, rng=True, params=True), idx=torch.as_tensor(dst, device=b.device), rng="source", params="source")
    return g, a, b, src, dst, rng


def _same_actions(torch, g, a, b, src, dst, rng, steps=24):
    acts_a, acts_b = _acts(rng, g, a, steps), _acts(rng, g, b, steps)
    acts_b[:, dst] = acts_a[:, src]
    return _dev_actions(torch, a, acts_a), _dev_actions(torch, b, acts_b)


def _same_params(torch, a, b, src, dst, what):
    pa, pb = a.env_params(), b.env_params()
    assert torch.equal(pa[:, torch.as_tensor(src, device=a.device)], pb[:, torch.as_tensor(dst, device=b.device)]), what


# ---------------------------------------------------------------------------------------------------- 1. deep copy under draws
@pytest.mark.parametrize("mode", ["step", "rollout", "graph"])
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", CASES_P)
def test_deep_copy_under_draws_replays_the_source(torch_cuda, name, dtype, mode):
    torch = torch_cuda
    g, a, b, src, dst, rng = _randomised_pair(torch, name, dtype)
    _same_params(torch, a, b, src, dst, "right after the restore")
    da, db = _same_actions(torch, g, a, b, src, dst, rng)
    si, di = torch.as_tensor(src, device=a.device), torch.as_tensor(dst, device=b.device)
    if mode == "step":  # the drawn parameters after every step, so after every in-kernel reset
        out_a, out_b = [], []
        for k in range(da.shape[0]):
            out_a.append(tuple(t[si].clone() for t in a.step(da[k])))
            out_b.append(tuple(t[di].clone() for t in b.step(db[k])))
            _same_params(torch, a, b, src, dst, ("step", k))
    else:
        out_a, out_b = _run(torch, a, da, mode, si), _run(torch, b, db, mode, di)
        _same_params(torch, a, b, src, dst, mode)
    _same_outputs(torch, out_a, out_b, (name, mode))
    if name in CROSS_RESETS:
        assert sum(int(o[3].sum().item()) for o in out_a) > 0, "the case is meant to cross terminations + in-kernel resets after the restore"
    ra, rb = a.reset(), b.reset()  # an explicit reset draws the source's values as well
    assert torch.equal(ra[0][si], rb[0][di]) and torch.equal(ra[1][si], rb[1][di])
    _same_params(torch, a, b, src, dst, "reset")
    a.close()
    b.close()


# ---------------------------------------------------------------------------------------------------- 2. the source's parameters, own draws
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
def test_own_identity_with_source_parameters_draws_its_own_at_the_next_reset(torch_cuda, dtype):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    name = "pmsm_cc_rk4"
    g, cfg_a = _random_cfg(name, 301, dtype)
    _, cfg_b = _random_cfg(name, 403, dtype, seed=5, offset=999)
    a, b, twin = VectorSim(cfg_a), VectorSim(cfg_b), VectorSim(cfg_b)
    for s in (a, b, twin):
        s.set_param_randomization(*_draws(s.cfg))
        s.reset()
    rng = np.random.default_rng(4)
    src, dst = rng.permutation(a.n)[:64], rng.permutation(b.n)[:64]
    _warm(torch, a, g, rng, 5)
    acts = _dev_actions(torch, b, _acts(rng, g, b, 9))
    for x in acts:
        b.step(x)
        twin.step(x)
    b.restore(a.snapshot(src, params=True), idx=dst, params="source")
    _same_params(torch, a, b, src, dst, "the source's until the first reset")
    rb, rt = b.reset(), twin.reset()  # the same calls on B and its twin: every env of B draws what the twin's env draws
    assert torch.equal(rb[0], rt[0]) and torch.equal(rb[1], rt[1])
    assert torch.equal(b.env_params(), twin.env_params())
    everyone = torch.arange(b.n, device=b.device)
    da = _dev_actions(torch, b, _acts(rng, g, b, 12))
    _same_outputs(torch, _run(torch, b, da, "step", everyone), _run(torch, twin, da, "step", everyone), "after the reset")
    for s in (a, b, twin):
        s.close()


# ---------------------------------------------------------------------------------------------------- 3. host-set blocks into shared coefficients
def _obs_close(torch, x, y, dtype, what):
    """the reset observation of a constant initial state of an induction motor: derived on the device for per-env blocks, on the host for the
    shared coefficients (DESIGN.md §4), equal up to a few units in the last place"""
    eps = torch.finfo(x.dtype).eps
    tol = 4 * eps * torch.clamp(y.abs(), min=1.0)
    assert bool(((x - y).abs() <= tol).all()), (what, float((x - y).abs().max()))


@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ["pmsm_cc_rk4", "eesm_cc_rk4", "scim_cc_rk4", "dfim_cc_rk4"])
def test_host_set_blocks_restored_into_shared_coefficients(torch_cuda, name, dtype):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, cfg_a = _random_cfg(name, 301, dtype)
    _, cfg_b = _random_cfg(name, 403, dtype, seed=5, offset=999)
    a, b, twin = VectorSim(cfg_a), VectorSim(cfg_b), VectorSim(cfg_b)
    rng = np.random.default_rng(5)
    mp = np.tile(np.array(list(cfg_a.motor_param)), (a.n, 1))
    for s in _MOTOR_SLOTS[cfg_a.motor_kind]:
        mp[:, s] *= rng.uniform(0.8, 1.2, size=a.n)
    a.set_env_params(mp, None)
    for s in (a, b, twin):
        s.reset()
    _warm(torch, a, g, rng, 6)
    acts = _dev_actions(torch, b, _acts(rng, g, b, 4))
    for x in acts:
        b.step(x)
        twin.step(x)
    src, dst = rng.permutation(a.n)[:80], rng.permutation(b.n)[:80]
    snap = a.snapshot(src, rng=True, params=True)
    assert np.array_equal(snap.params[:, :K.MAX_MOTOR_PARAM].cpu().numpy(), mp[src])  # the host rows, exactly
    b.restore(snap, idx=dst, rng="source", params="source")
    da, db = _same_actions(torch, g, a, b, src, dst, rng, steps=24)
    everyone = torch.arange(b.n, device=b.device)
    out_a = _run(torch, a, da, "step", torch.as_tensor(src, device=a.device))
    out_b = _run(torch, b, db, "step", everyone)
    out_t = _run(torch, twin, db, "step", everyone)
    di = torch.as_tensor(dst, device=b.device)
    _same_outputs(torch, out_a, [tuple(t[di] for t in o) for o in out_b], "the restored envs replay their sources")
    keep = torch.ones(b.n, dtype=torch.bool, device=b.device)
    keep[di] = False
    induction = name.startswith(("scim", "dfim"))
    for k, (ob, ot) in enumerate(zip(out_b, out_t)):
        for q, nm in enumerate(("obs", "ref", "reward", "terminated")):
            x, y = ob[q][keep], ot[q][keep]
            if nm == "obs" and induction:
                _obs_close(torch, x, y, dtype, (name, k))
            else:
                assert torch.equal(x, y), (name, nm, k)
    for s in (a, b, twin):
        s.close()


# ---------------------------------------------------------------------------------------------------- 4. random-shooting MPC on randomised plants
def test_mpc_step_on_randomised_plants_matches_its_best_branch(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    plants, cand, horizon = 16, 32, 6
    g, cfg_p = _random_cfg("pmsm_cc_rk4", plants, K.F32)
    _, cfg_m = _random_cfg("pmsm_cc_rk4", plants * cand, K.F32, seed=8, offset=0)
    p, mdl = VectorSim(cfg_p), VectorSim(cfg_m)
    for s in (p, mdl):
        s.set_param_randomization(*_draws(s.cfg))
        s.reset()
    rng = np.random.default_rng(6)
    _warm(torch, p, g, rng, 3)
    ridx = torch.arange(plants, device=p.device, dtype=torch.int32).repeat_interleave(cand)
    for _ in range(3):  # three control steps
        acts = _dev_actions(torch, mdl, _acts(rng, g, mdl, horizon))
        mdl.restore(p.snapshot(rng=True, params=True), rows=ridx, rng="source", params="source")
        assert torch.equal(mdl.env_params(), p.env_params()[:, ridx.long()])
        obs, ref, rew, term = mdl.rollout(acts, record_every=1)
        r = ref[0].view(plants, cand, -1)
        assert torch.equal(r, r[:, :1].expand_as(r))
        best = rew.sum(0).view(plants, cand).argmax(1) + torch.arange(plants, device=p.device) * cand
        o, rf, w, t = (x.clone() for x in p.step(acts[0, best].contiguous()))
        assert torch.equal(o, obs[0, best]) and torch.equal(rf, ref[0, best]) and torch.equal(w, rew[0, best]) and torch.equal(t, term[0, best])
    p.close()
    mdl.close()


# ---------------------------------------------------------------------------------------------------- 5. edited parameters
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
def test_edited_parameters_equal_host_set_rows(torch_cuda, dtype):
    """B's env dst takes A's env src with an edited r_s; A's twin C gets the same row through gemb200_set_env_params: same bits"""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, cfg_a = _random_cfg("pmsm_cc_rk4", 301, dtype)
    _, cfg_b = _random_cfg("pmsm_cc_rk4", 403, dtype, seed=5, offset=999)
    a, c, b = VectorSim(cfg_a), VectorSim(cfg_a), VectorSim(cfg_b)
    for s in (a, b, c):
        s.reset()
    rng = np.random.default_rng(7)
    acts = _dev_actions(torch, a, _acts(rng, g, a, 6))
    for x in acts:
        a.step(x)
        c.step(x)
    _warm(torch, b, g, rng, 3)
    src, dst = rng.permutation(a.n)[:50], rng.permutation(b.n)[:50]
    snap = a.snapshot(src, rng=True, params=True)
    assert torch.equal(snap.params.cpu(), torch.as_tensor(np.tile(_config_row(cfg_a), (len(src), 1))))  # no blocks: the configuration's
    snap.params[:, K.MP_R_S] *= torch.linspace(0.7, 1.3, len(src), dtype=torch.float64, device=snap.params.device)
    b.restore(snap, idx=dst, rng="source", params="source")
    mp = np.tile(np.array(list(cfg_a.motor_param)), (a.n, 1))
    mp[src] = snap.params[:, :K.MAX_MOTOR_PARAM].cpu().numpy()
    c.set_env_params(mp, None)
    da = _acts(rng, g, a, 24)
    db = _acts(rng, g, b, 24)
    db[:, dst] = da[:, src]
    out_c = _run(torch, c, _dev_actions(torch, c, da), "step", torch.as_tensor(src, device=c.device))
    out_b = _run(torch, b, _dev_actions(torch, b, db), "step", torch.as_tensor(dst, device=b.device))
    _same_outputs(torch, out_c, out_b, "edited r_s")
    for s in (a, b, c):
        s.close()


# ---------------------------------------------------------------------------------------------------- 6. round trip, no-block pack
def test_pack_without_blocks_and_round_trip(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, cfg = _random_cfg("eesm_cc_rk4", 257, K.F64)
    h, twin = VectorSim(cfg), VectorSim(cfg)
    snap = h.snapshot(params=True)
    assert snap.pole_pairs == cfg.motor_param[K.MP_P]
    assert torch.equal(snap.params.cpu(), torch.as_tensor(np.tile(_config_row(cfg), (h.n, 1))))
    for s in (h, twin):
        s.set_param_randomization(*_draws(s.cfg))
        s.reset()
    rng = np.random.default_rng(8)
    acts = _dev_actions(torch, h, _acts(rng, g, h, 30))
    for x in acts[:10]:
        h.step(x)
        twin.step(x)
    h.restore(h.snapshot(params=True), params="source")  # every env into itself
    assert torch.equal(h.env_params(), twin.env_params())
    everyone = torch.arange(h.n, device=h.device)
    _same_outputs(torch, _run(torch, h, acts[10:], "step", everyone), _run(torch, twin, acts[10:], "step", everyone), "round trip")
    assert torch.equal(h.env_params(), twin.env_params())
    h.close()
    twin.close()


# ---------------------------------------------------------------------------------------------------- 7. capture
def test_captured_pack_and_unpack_give_the_eager_bits(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, cfg = _random_cfg("pmsm_cc_rk4", 300, K.F32)
    eager, cap = VectorSim(cfg), VectorSim(cfg)
    rng = np.random.default_rng(9)
    acts = _dev_actions(torch, eager, _acts(rng, g, eager, 30))
    src = torch.arange(0, 40, device=eager.device, dtype=torch.int32)
    dst = torch.arange(100, 140, device=eager.device, dtype=torch.int32)
    for s in (eager, cap):
        s.set_param_randomization(*_draws(s.cfg))
        s.set_device_clock(True)
        s.reset()
        for x in acts[:8]:
            s.step(x)
        s.restore(s.snapshot(src[:1], rng=True, params=True), idx=src[1:2], rng="source", params="source")  # identities in use before capture
    eager.restore(eager.snapshot(src, rng=True, params=True), idx=dst, rng="source", params="source")
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        snap = cap.snapshot(src, rng=True, params=True)
        cap.restore(snap, idx=dst, rng="source", params="source")
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager.env_params(), cap.env_params())
    everyone = torch.arange(cap.n, device=cap.device)
    _same_outputs(torch, _run(torch, eager, acts[8:], "step", everyone), _run(torch, cap, acts[8:], "step", everyone), "captured pack / unpack")
    assert torch.equal(eager.env_params(), cap.env_params())
    eager.close()
    cap.close()


# ---------------------------------------------------------------------------------------------------- refusals that stay
def test_paths_without_params_stay_refused_under_draws(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    _, cfg = _random_cfg("pmsm_cc_rk4", 64, K.F32)
    d = VectorSim(cfg)
    d.set_param_randomization(*_draws(d.cfg))
    d.reset()
    snap = d.snapshot(np.arange(4), rng=True, params=True)
    for call in (lambda: d.snapshot([0]), lambda: d.restore(snap, idx=np.arange(4)), lambda: d.restore(snap, idx=np.arange(4), rng="source"), d.state_dict):
        with pytest.raises(NotImplementedError):
            call()
    rows = torch.empty_like(snap.rows)
    assert d._lib.gemb200_pack_envs(d._h, None, 4, C.c_void_p(rows.data_ptr()), d._stream()) == K.E_INVALID
    assert d._lib.gemb200_adopt_rng_ids(d._h, C.c_void_p(snap.rng.data_ptr()), 4, None, None, 4, d._stream()) == K.E_INVALID
    assert d._lib.gemb200_pack_envs_params(d._h, None, 4, C.c_void_p(rows.data_ptr()), None, d._stream()) == K.E_INVALID  # params required
    d.close()
