"""Adopted RNG identities on the device (gemb200_pack_rng_ids / gemb200_adopt_rng_ids / gemb200_clear_rng_ids): a restored env that
adopts its source's identity repeats the source's random draws, so under the same actions it gives the source's outputs bit for bit —
copy.deepcopy(env) of the reference, for a batch.  Every case switches its random parts on: Wiener references, random initial states,
state noise and, where the case has one, the AC supply's random phase."""
import ctypes as C

import numpy as np
import pytest

from gpu_helpers import DEAD3, SCIM_RANDOM, SWITCHED, _acts, _dev_actions, _random_cfg, _run, _same_outputs, torch_cuda  # noqa: F401
from helpers import ROLLOUT_CASES
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

CROSS_RESETS = ("pmsm_cc_rk4", "eesm_cc_rk4", "permex_cc_rk4")
ALL = ROLLOUT_CASES + [DEAD3, SWITCHED, SCIM_RANDOM]
# Per-env blocks set from the host derive a constant initial state's reset observation on the device, which differs in the last bits from
# the host-derived one of the shared-coefficient kernels for the induction motors (DESIGN.md §4); blocks made by an adoption use the latter.
HOST_EXACT = [c for c in ALL if not c.startswith(("scim", "dfim"))]


def _branch_pair(torch, name, dtype, m=120, n_a=301, n_b=403, k1=7, k2=12):
    """A (seed 77, offset 12345) and B (seed 5, offset 999, other N): A's envs src restored with their identities into B's envs dst"""
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, cfg_a = _random_cfg(name, n_a, dtype)
    _, cfg_b = _random_cfg(name, n_b, dtype, seed=5, offset=999)
    a, b = VectorSim(cfg_a), VectorSim(cfg_b)
    rng = np.random.default_rng(3)
    src, dst = rng.permutation(n_a)[:m], rng.permutation(n_b)[:m]
    a.reset()
    b.reset()
    for acts, s, k in ((_acts(rng, g, a, k1), a, k1), (_acts(rng, g, b, k2), b, k2)):
        da = _dev_actions(torch, s, acts)
        for j in range(k):
            s.step(da[j])
    b.restore(a.snapshot(src, rng=True), idx=torch.as_tensor(dst, device=b.device), rng="source")
    return g, a, b, src, dst, rng


def _same_actions(torch, g, a, b, src, dst, rng, steps=24):
    acts_a, acts_b = _acts(rng, g, a, steps), _acts(rng, g, b, steps)
    acts_b[:, dst] = acts_a[:, src]
    return _dev_actions(torch, a, acts_a), _dev_actions(torch, b, acts_b)


# ---------------------------------------------------------------------------------------------------- the property the replay tests rest on
@pytest.mark.parametrize("blocks", ["host_blocks", "self_adopted"])
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ALL)
def test_per_env_blocks_of_the_shared_parameters_match_the_shared_kernels(torch_cuda, name, dtype, blocks):
    """Handle B runs its per-env parameter instantiations; with blocks that hold the shared parameters (derived on the host, or filled on
    the device by an adoption — here of every env's own identity) it gives the bits of the shared-coefficient kernels of an equal handle."""
    if blocks == "host_blocks" and name not in HOST_EXACT:
        pytest.skip("host-set blocks of an induction motor: reset observation derived on the device (DESIGN.md §4)")
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, cfg = _random_cfg(name, 257, dtype)
    a, b = VectorSim(cfg), VectorSim(cfg)
    if blocks == "host_blocks":
        b.set_env_params(np.tile(np.array(list(cfg.motor_param)), (b.n, 1)), np.tile(np.array(list(cfg.load_param)), (b.n, 1)))
    else:
        b.restore(b.snapshot(rng=True), rng="source")
    ra, rb = a.reset(), b.reset()
    assert torch.equal(ra[0], rb[0]) and torch.equal(ra[1], rb[1])
    acts = _dev_actions(torch, a, _acts(np.random.default_rng(1), g, a, 24))
    everyone = torch.arange(a.n, device=a.device)
    _same_outputs(torch, _run(torch, a, acts[:12], "step", everyone), _run(torch, b, acts[:12], "step", everyone), "step")
    _same_outputs(torch, _run(torch, a, acts[12:], "rollout", everyone), _run(torch, b, acts[12:], "rollout", everyone), "rollout")
    a.close()
    b.close()


# ---------------------------------------------------------------------------------------------------- exact replay
@pytest.mark.parametrize("mode", ["step", "rollout", "graph"])
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ALL)
def test_adopted_identity_replays_the_source(torch_cuda, name, dtype, mode):
    torch = torch_cuda
    g, a, b, src, dst, rng = _branch_pair(torch, name, dtype)
    da, db = _same_actions(torch, g, a, b, src, dst, rng)
    out_a = _run(torch, a, da, mode, torch.as_tensor(src, device=a.device))
    out_b = _run(torch, b, db, mode, torch.as_tensor(dst, device=b.device))
    _same_outputs(torch, out_a, out_b, (name, mode))
    if name in CROSS_RESETS:
        assert sum(int(o[3].sum().item()) for o in out_a) > 0, "the case is meant to cross terminations + in-kernel resets after the restore"
    a.close()
    b.close()


def test_masked_reset_draws_with_the_identity(torch_cuda):
    torch = torch_cuda
    g, a, b, src, dst, rng = _branch_pair(torch, "pmsm_cc_rk4", K.F32)
    ma, mb = torch.zeros(a.n, dtype=torch.uint8, device=a.device), torch.zeros(b.n, dtype=torch.uint8, device=b.device)
    ma[src[::2]] = 1
    mb[dst[::2]] = 1
    oa, ob = a.reset(ma), b.reset(mb)
    s2, d2 = torch.as_tensor(src[::2], device=a.device), torch.as_tensor(dst[::2], device=b.device)
    assert torch.equal(oa[0][s2], ob[0][d2]) and torch.equal(oa[1][s2], ob[1][d2])
    da, db = _same_actions(torch, g, a, b, src, dst, rng, steps=8)
    _same_outputs(torch, _run(torch, a, da, "step", torch.as_tensor(src, device=a.device)), _run(torch, b, db, "step", torch.as_tensor(dst, device=b.device)), "after")
    a.close()
    b.close()


# ---------------------------------------------------------------------------------------------------- same handle, fan-out, composition
def test_fan_out_on_one_handle(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, cfg = _random_cfg("pmsm_cc_rk4", 300, K.F32)
    h = VectorSim(cfg)
    rng = np.random.default_rng(9)
    h.reset()
    for a in _dev_actions(torch, h, _acts(rng, g, h, 5)):
        h.step(a)
    src, cand = 3, np.arange(100, 132)
    h.restore(h.snapshot([src], rng=True), idx=cand, rows=np.zeros(len(cand), dtype=np.int64), rng="source")
    same = _acts(rng, g, h, 16)
    same[:, cand] = same[:, src][:, None]
    out = _run(torch, h, _dev_actions(torch, h, same), "step", torch.as_tensor(np.r_[src, cand], device=h.device))
    for k, o in enumerate(out):  # identical actions: the source and its 32 copies are one trajectory
        for q in range(4):
            assert torch.equal(o[q], o[q][:1].expand_as(o[q])), (k, q)
    # different actions: the references are the source's until the candidate (or the source) terminates
    h.restore(h.snapshot([src], rng=True), idx=cand, rows=np.zeros(len(cand), dtype=np.int64), rng="source")
    out = _run(torch, h, _dev_actions(torch, h, _acts(rng, g, h, 16)), "step", torch.as_tensor(np.r_[src, cand], device=h.device))
    ref = torch.stack([o[1] for o in out]).cpu()  # [k, 1 + C, n_ref]
    term = torch.stack([o[3] for o in out]).cpu().bool()
    checked = 0
    for c in range(1, 1 + len(cand)):
        for k in range(len(out)):
            if term[k, 0] or term[k, c]:
                break
            assert torch.equal(ref[k, c], ref[k, 0]), (c, k)
            checked += 1
    assert checked > len(cand)
    h.close()


@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
def test_branch_of_a_branch_replays_the_original(torch_cuda, dtype):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, a, b, src, dst, rng = _branch_pair(torch, "pmsm_cc_rk4", dtype)
    _, cfg_c = _random_cfg("pmsm_cc_rk4", 97, dtype, seed=11, offset=3)
    c = VectorSim(cfg_c)
    c.reset()
    for x in _dev_actions(torch, c, _acts(rng, g, c, 4)):
        c.step(x)
    da, db = _same_actions(torch, g, a, b, src, dst, rng, steps=6)
    for k in range(6):
        a.step(da[k])
        b.step(db[k])
    m = 40
    cdst = rng.permutation(c.n)[:m]
    c.restore(b.snapshot(dst[:m], rng=True), idx=cdst, rng="source")
    acts_a, acts_c = _acts(rng, g, a, 24), _acts(rng, g, c, 24)
    acts_c[:, cdst] = acts_a[:, src[:m]]
    out_a = _run(torch, a, _dev_actions(torch, a, acts_a), "step", torch.as_tensor(src[:m], device=a.device))
    out_c = _run(torch, c, _dev_actions(torch, c, acts_c), "step", torch.as_tensor(cdst, device=c.device))
    _same_outputs(torch, out_a, out_c, "A -> B -> C")
    for s in (a, b, c):
        s.close()


# ---------------------------------------------------------------------------------------------------- the ways back to the own identity
def test_default_restore_returns_to_the_own_draws(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, a, b, src, dst, rng = _branch_pair(torch, "pmsm_cc_rk4", K.F32)
    b2 = VectorSim(_random_cfg("pmsm_cc_rk4", b.n, K.F32, seed=5, offset=999)[1])  # B's twin: the same clock, no identities adopted
    acts = _dev_actions(torch, b, _acts(rng, g, b, 36))
    b2.reset()
    for k in range(24):
        b2.step(acts[k])
    for k in range(12):  # B: 12 steps before the adoption (in _branch_pair), 12 after
        b.step(acts[k])
    b2.restore(b.snapshot())  # the same states everywhere; every env of b2 draws its own numbers
    snap = a.snapshot(src)
    ii = torch.as_tensor(dst, device=b.device)
    b.restore(snap, idx=ii)
    b2.restore(snap, idx=ii)
    everyone = torch.arange(b.n, device=b.device)
    _same_outputs(torch, _run(torch, b, acts[24:], "step", everyone), _run(torch, b2, acts[24:], "step", everyone), "default restore")
    for s in (a, b, b2):
        s.close()


def test_reseed_after_adoption_is_a_fresh_handle(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, a, b, src, dst, rng = _branch_pair(torch, "pmsm_cc_rk4", K.F32)
    b.reseed(4242)
    _, cfg_f = _random_cfg("pmsm_cc_rk4", b.n, K.F32, seed=4242, offset=999)
    f = VectorSim(cfg_f)
    acts = _dev_actions(torch, b, _acts(rng, g, b, 24))
    everyone = torch.arange(b.n, device=b.device)
    rb, rf = b.reset(), f.reset()
    assert torch.equal(rb[0], rf[0]) and torch.equal(rb[1], rf[1])
    _same_outputs(torch, _run(torch, b, acts, "rollout", everyone), _run(torch, f, acts, "rollout", everyone), "reseed")
    assert np.array_equal(b.state_dict()["blob"], f.state_dict()["blob"])  # checkpoints work again
    for s in (a, b, f):
        s.close()


def test_clear_returns_every_env_to_its_own_draws(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, a, b, src, dst, rng = _branch_pair(torch, "pmsm_cc_rk4", K.F64)
    b2 = VectorSim(_random_cfg("pmsm_cc_rk4", b.n, K.F64, seed=5, offset=999)[1])  # B's twin: the same clock, the same states, its own identities
    b2.reset()
    for x in _dev_actions(torch, b2, _acts(rng, g, b2, 12)):
        b2.step(x)
    b2.restore(b.snapshot())
    b.clear_rng_ids()
    acts = _dev_actions(torch, b, _acts(rng, g, b, 24))
    everyone = torch.arange(b.n, device=b.device)
    _same_outputs(torch, _run(torch, b, acts, "step", everyone), _run(torch, b2, acts, "step", everyone), "clear")
    for s in (a, b, b2):
        s.close()


# ---------------------------------------------------------------------------------------------------- refusals
def test_refusals(torch_cuda):
    torch = torch_cuda
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, a, b, src, dst, rng = _branch_pair(torch, "pmsm_cc_rk4", K.F32, m=8)
    ids = a.snapshot(src, rng=True).rng
    # checkpoints do not carry identities
    for call in (b.state_dict, lambda: b.load_state_dict(a.state_dict())):
        with pytest.raises(NotImplementedError, match="identities"):
            call()
    assert b._lib.gemb200_checkpoint_save(b._h, C.c_void_p(np.empty(b._lib.gemb200_checkpoint_size(b._h), np.uint8).ctypes.data)) == K.E_INVALID
    # SoA layout
    _, cfg_s = _random_cfg("pmsm_cc_rk4", 64, K.F32)
    cfg_s.layout = K.LAYOUT_SOA
    s = VectorSim(cfg_s)
    snap = a.snapshot(src, rng=True)
    with pytest.raises(ValueError, match="row-per-env"):
        s.restore(snap, idx=np.arange(8), rng="source")
    assert s._lib.gemb200_adopt_rng_ids(s._h, C.c_void_p(ids.data_ptr()), 8, None, None, 8, s._stream()) == K.E_INVALID
    # parameter draws on
    _, cfg_d = _random_cfg("pmsm_cc_rk4", 64, K.F32)
    d = VectorSim(cfg_d)
    d.set_param_randomization([K.MP_R_S], [K.DIST_UNIFORM], [0.1], [0.2])
    assert d._lib.gemb200_adopt_rng_ids(d._h, C.c_void_p(ids.data_ptr()), 8, None, None, 8, d._stream()) == K.E_INVALID
    with pytest.raises(NotImplementedError):
        d.restore(snap, idx=np.arange(8), rng="source")
    # CapturedSteps with warm-up steps saves a checkpoint
    env = gem.make("Cont-CC-PMSM-v0", num_envs=64)
    env.reset()
    env.restore_envs(env.snapshot_envs([0], rng=True), idx=[5], rng="source")
    with pytest.raises(NotImplementedError):
        env.capture_steps(lambda st, rf: torch.zeros((64, 3), device=st.device), 2, warmup=1)
    env.clear_rng_identities()
    env.state_dict()  # allowed again
    env.close()
    for x in (a, b, s, d):
        x.close()


# ---------------------------------------------------------------------------------------------------- random-shooting MPC with common random numbers
def test_mpc_step_with_identities_matches_its_best_branch(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    plants, cand, horizon = 16, 32, 6
    g, cfg_p = _random_cfg("pmsm_cc_rk4", plants, K.F32)
    _, cfg_m = _random_cfg("pmsm_cc_rk4", plants * cand, K.F32, seed=8, offset=0)
    p, mdl = VectorSim(cfg_p), VectorSim(cfg_m)
    rng = np.random.default_rng(6)
    p.reset()
    mdl.reset()
    warm = _dev_actions(torch, p, _acts(rng, g, p, 3))
    for k in range(3):
        p.step(warm[k])
    ridx = torch.arange(plants, device=p.device, dtype=torch.int32).repeat_interleave(cand)
    for _ in range(3):  # three control steps
        acts = _dev_actions(torch, mdl, _acts(rng, g, mdl, horizon))
        mdl.restore(p.snapshot(rng=True), rows=ridx, rng="source")
        obs, ref, rew, term = mdl.rollout(acts, record_every=1)
        r = ref[0].view(plants, cand, -1)
        assert torch.equal(r, r[:, :1].expand_as(r))  # every candidate of a plant sees the same next reference
        best = rew.sum(0).view(plants, cand).argmax(1) + torch.arange(plants, device=p.device) * cand
        o, rf, w, t = (x.clone() for x in p.step(acts[0, best].contiguous()))
        assert torch.equal(o, obs[0, best]) and torch.equal(rf, ref[0, best]) and torch.equal(w, rew[0, best]) and torch.equal(t, term[0, best])
    p.close()
    mdl.close()
