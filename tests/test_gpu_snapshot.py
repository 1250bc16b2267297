"""Per-env state snapshots on the device (gemb200_pack_envs / gemb200_unpack_envs): a restored env is physically its source.  The bar is
the one `copy.deepcopy(env)` sets in the reference — the copy continues exactly like the original — for every deterministic quantity, bit
for bit; random draws are keyed by (seed, global env index), so a restored env draws its own numbers from then on."""
import ctypes as C

import numpy as np
import pytest

from helpers import switched_config
from gym_electric_motor_b200 import _cabi as K
from gpu_helpers import _dev_actions, torch_cuda  # noqa: F401
from helpers import ROLLOUT_CASES, _mk, _random_actions

pytestmark = pytest.mark.gpu

DEAD3 = "pmsm_cc_rk4_dead3"  # every configuration in ROLLOUT_CASES has a dead time of 0 or 1: a ring of 1 cannot show a rotation error


def _cfg(name, n, dtype, layout, deterministic, seed=77, offset=12345):
    g, cfg = _mk(name.replace("_dead3", ""), n, dtype, layout, ref_kind=K.REF_CONST if deterministic else K.REF_WIENER)
    if name == DEAD3:
        cfg.dead_time_steps = 3
    if cfg.supply_kind == K.SUPPLY_AC1:
        cfg.supply_param[2] = 1.0  # fixed phase: a random phase at the in-kernel resets would be a random draw
    cfg.seed, cfg.env_index_offset = seed, offset
    return g, cfg


def _rows(t, idx, soa):
    """rows of envs idx of an output tensor ([N, k] / [N] in AoS, [k, N] in SoA)"""
    if t.dim() == 1:
        return t[idx]
    return t[:, idx].T if soa else t[idx]


def _branch(torch, name, dtype, layout, deterministic):
    from gym_electric_motor_b200.vector_sim import VectorSim

    n_a, n_b, k1, k2, k_after, m = 301, 403, 7, 12, 24, 120
    g, cfg_a = _cfg(name, n_a, dtype, layout, deterministic)
    _, cfg_b = _cfg(name, n_b, dtype, layout, deterministic, seed=5, offset=999)
    a, b = VectorSim(cfg_a), VectorSim(cfg_b)
    soa = a.soa
    rng = np.random.default_rng(3)
    acts_a = _random_actions(rng, g, n_a, k1 + k_after)
    acts_b = _random_actions(rng, g, n_b, k2 + k_after)
    src = rng.permutation(n_a)[:m]
    dst = rng.permutation(n_b)[:m]
    acts_b[k2:, dst] = acts_a[k1:, src]  # a restored env gets its source's actions from then on
    da, db = _dev_actions(torch, a, acts_a), _dev_actions(torch, b, acts_b)
    a.reset()
    b.reset()
    for k in range(k1):
        a.step(da[k])
    for k in range(k2):
        b.step(db[k])
    others = np.setdiff1d(np.arange(n_b), dst)
    before = b.snapshot().rows.clone()
    b.restore(a.snapshot(src), idx=torch.as_tensor(dst, device=b.device))
    after = b.snapshot().rows
    assert torch.equal(after[others], before[others]), "envs that were not restored changed"
    out_a, out_b = [], []
    for k in range(k_after):
        out_a.append(tuple(_rows(t, src, soa).clone() for t in a.step(da[k1 + k])))
        out_b.append(tuple(_rows(t, dst, soa).clone() for t in b.step(db[k2 + k])))
    n_term = sum(int(o[3].sum().item()) for o in out_a)
    for s in (a, b):
        s.close()
    return out_a, out_b, n_term


@pytest.mark.parametrize("deterministic", [True, False], ids=["const", "wiener"])
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", ROLLOUT_CASES + [DEAD3])
def test_branch_continues_like_its_source(torch_cuda, name, dtype, deterministic):
    out_a, out_b, n_term = _branch(torch_cuda, name, dtype, K.LAYOUT_AOS, deterministic)
    torch = torch_cuda
    for k, (oa, ob) in enumerate(zip(out_a, out_b)):
        assert torch.equal(oa[0], ob[0]), (name, "obs", k)
        assert torch.equal(oa[3], ob[3]), (name, "terminated", k)
        if deterministic:
            assert torch.equal(oa[1], ob[1]), (name, "ref", k)
            assert torch.equal(oa[2], ob[2]), (name, "reward", k)
    assert torch.equal(out_a[0][2], out_b[0][2]), (name, "reward of the first step after the restore")
    if name in ("pmsm_cc_rk4", "eesm_cc_rk4", "permex_cc_rk4"):
        assert n_term > 0, "the case is meant to cross terminations + in-kernel resets after the restore"


@pytest.mark.parametrize("deterministic", [True, False], ids=["const", "wiener"])
def test_branch_soa_layout(torch_cuda, deterministic):
    out_a, out_b, _ = _branch(torch_cuda, "pmsm_cc_rk4", K.F32, K.LAYOUT_SOA, deterministic)
    for k, (oa, ob) in enumerate(zip(out_a, out_b)):
        for q in (0, 3) + ((1, 2) if deterministic else ()):
            assert torch_cuda.equal(oa[q], ob[q]), (k, q)


@pytest.mark.parametrize("name", ["pmsm_cc_rk4", "eesm_cc_rc_dq_dead1_rk4", "scim_sc_flux_cossin_dead1_rk4", DEAD3, "pmsm_cc_extspeed_rk4",
                                  "permex_fin_sc_rc_interlock_rk4", "pmsm_cc_ac_rk4"])
@pytest.mark.parametrize("dtype", [K.F32, K.F64], ids=["f32", "f64"])
def test_round_trips(torch_cuda, name, dtype):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g, cfg = _cfg(name, 200, dtype, K.LAYOUT_AOS, deterministic=False)
    s = VectorSim(cfg)
    acts = _dev_actions(torch, s, _random_actions(np.random.default_rng(8), g, 200, 16))
    s.reset()
    for k in range(5):
        s.step(acts[k])
    blob = s.state_dict()["blob"]
    snap = s.snapshot()
    s.restore(snap)  # same envs, no step in between: nothing changes
    assert np.array_equal(s.state_dict()["blob"], blob)
    for k in range(5, 16):
        s.step(acts[k])
    s.restore(snap)  # eleven steps later: the clock-relative fields are re-based on the later clock
    assert torch.equal(s.snapshot().rows, snap.rows)
    s.close()


def test_clock_relative_fields_follow_the_destination_clock(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    # sub-episodes of 2..5 steps inside super-episodes of 5..11: both kinds of ends happen many times in 40 steps
    kinds = [dict(kind=K.REF_WIENER, margin=(-0.5, 0.5), length=(2, 6)), dict(kind=K.REF_SINUS, length=(2, 6)),
             dict(kind=K.REF_STEP, amp=(0.05, 0.2), length=(2, 6))]
    cfg_a = switched_config(64, kinds, [1.0 / 3] * 3, (5, 12), seed=21, dtype=K.F32)
    cfg_b = switched_config(50, kinds, [1.0 / 3] * 3, (5, 12), seed=99, dtype=K.F32)
    a, b = VectorSim(cfg_a), VectorSim(cfg_b)
    # row of a DC motor with one switched slot, fp32: hot [i, ref] | cold [omega, sigma or periodic start, sub-episode end] | swst [entry, end]
    assert a.record_layout()[0] == 7
    W_END, W_SWEND = 4, 6
    src, dst = np.arange(32), np.arange(10, 42)
    a.reset()
    b.reset()
    za, zb = torch.zeros((64, 1), device=a.device), torch.zeros((50, 1), device=b.device)
    for _ in range(5):
        a.step(za)
    for _ in range(13):
        b.step(zb)
    b.restore(a.snapshot(src), idx=dst)
    hist_a, hist_b, kinds_a = [], [], []
    for _ in range(40):
        ra, rb = a.snapshot(src).rows, b.snapshot(dst).rows
        hist_a.append(ra[:, [W_END, W_SWEND]].cpu().numpy().astype(np.int64))
        hist_b.append(rb[:, [W_END, W_SWEND]].cpu().numpy().astype(np.int64))
        kinds_a.append(ra[:, 5].cpu().numpy())
        a.step(za)
        b.step(zb)
    ha, hb = np.stack(hist_a), np.stack(hist_b)  # [step, env, field]: steps remaining until the (super-)episode ends
    steps = ha.shape[0]

    def first_break(x):  # first row whose value is not the previous one minus 1: a new (super-)episode started in that step
        br = np.nonzero(np.diff(x) != -1)[0]
        return br[0] + 1 if len(br) else steps

    ended = 0
    for e in range(len(src)):
        sa, sb, ea, eb = ha[:, e, 1], hb[:, e, 1], ha[:, e, 0], hb[:, e, 0]
        # super-episode: it ends when at most one step remains, and the next one is 5..11 steps long
        j1 = first_break(sa)
        assert np.array_equal(sa[:j1], sb[:j1]), ("super-episode", e)
        if j1 < steps:
            ended += 1
            assert sa[j1 - 1] <= 1 and sb[j1] > sb[j1 - 1], ("the destination's super-episode did not end on the same step", e)
        # sub-episode: compared until it ends by itself; a super-episode switch restarts it with a length of the env's own draw
        j0 = first_break(ea)
        stop = min(j0, j1)
        assert np.array_equal(ea[:stop], eb[:stop]), ("sub-episode", e)
        if j0 < j1:
            ended += 1
            assert ea[j0 - 1] <= 1 and eb[j0] > eb[j0 - 1], ("the destination's sub-episode did not end on the same step", e)
    assert ended > len(src)
    assert len(np.unique(np.stack(kinds_a))) > 1
    a.close()
    b.close()


def test_fan_out_in_a_cuda_graph(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    plants, cand, horizon = 64, 256, 4
    g, cfg_p = _cfg("pmsm_cc_rk4", plants, K.F32, K.LAYOUT_AOS, deterministic=False)
    _, cfg_m = _cfg("pmsm_cc_rk4", plants * cand, K.F32, K.LAYOUT_AOS, deterministic=False, seed=3, offset=0)
    sims = [VectorSim(c) for c in (cfg_p, cfg_m, cfg_p, cfg_m)]
    p, mdl, p_e, m_e = sims
    rng = np.random.default_rng(4)
    acts_p = _dev_actions(torch, p, _random_actions(rng, g, plants, 6))
    acts_m = _dev_actions(torch, mdl, _random_actions(rng, g, plants * cand, horizon))
    ridx = torch.arange(plants, device=p.device, dtype=torch.int32).repeat_interleave(cand)
    for s in sims:
        s.reset()
    for k in range(6):
        p.step(acts_p[k])
        p_e.step(acts_p[k])
    for s in sims:
        s.set_device_clock(True)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        snap = p.snapshot()
        mdl.restore(snap, rows=ridx)
        out = mdl.rollout(acts_m, record_every=1)
    for _ in range(2):
        graph.replay()
        snap_e = p_e.snapshot()
        m_e.restore(snap_e, rows=ridx)
        ref_out = m_e.rollout(acts_m, record_every=1)
        torch.cuda.synchronize()
        for q in range(4):
            assert torch.equal(out[q], ref_out[q]), q
        assert torch.equal(snap.rows, snap_e.rows)
    assert mdl.clock() == m_e.clock()
    for s in sims:
        s.close()


def test_mpc_step_matches_its_best_branch(torch_cuda):
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    plants, cand, horizon = 16, 32, 6
    g, cfg_p = _cfg("pmsm_cc_rk4", plants, K.F32, K.LAYOUT_AOS, deterministic=True)
    _, cfg_m = _cfg("pmsm_cc_rk4", plants * cand, K.F32, K.LAYOUT_AOS, deterministic=True, seed=8, offset=0)
    p, mdl = VectorSim(cfg_p), VectorSim(cfg_m)
    rng = np.random.default_rng(6)
    p.reset()
    mdl.reset()
    warm = _dev_actions(torch, p, _random_actions(rng, g, plants, 3))
    for k in range(3):
        p.step(warm[k])
    ridx = torch.arange(plants, device=p.device, dtype=torch.int32).repeat_interleave(cand)
    for _ in range(3):  # three control steps
        acts = _dev_actions(torch, mdl, _random_actions(rng, g, plants * cand, horizon))
        mdl.restore(p.snapshot(), rows=ridx)
        obs, ref, rew, term = mdl.rollout(acts, record_every=1)
        best = rew.sum(0).view(plants, cand).argmax(1) + torch.arange(plants, device=p.device) * cand
        o, r, w, t = (x.clone() for x in p.step(acts[0, best].contiguous()))
        assert torch.equal(o, obs[0, best]) and torch.equal(r, ref[0, best]) and torch.equal(w, rew[0, best]) and torch.equal(t, term[0, best])
    p.close()
    mdl.close()


@pytest.mark.parametrize("other", ["synrm", "dead_time"])
def test_rows_of_another_layout_are_refused(torch_cuda, other):
    from gym_electric_motor_b200.vector_sim import VectorSim

    _, cfg = _cfg("pmsm_cc_rk4", 32, K.F32, K.LAYOUT_AOS, deterministic=True)
    if other == "synrm":
        _, cfg_o = _cfg("synrm_cc_rk4", 32, K.F32, K.LAYOUT_AOS, deterministic=True)
    else:
        _, cfg_o = _cfg("pmsm_cc_rk4", 32, K.F32, K.LAYOUT_AOS, deterministic=True)
        cfg_o.dead_time_steps = 2
    s, o = VectorSim(cfg), VectorSim(cfg_o)
    snap = s.snapshot()
    with pytest.raises(ValueError):
        o.restore(snap)
    rc = o._lib.gemb200_unpack_envs(o._h, C.c_void_p(snap.rows.data_ptr()), len(snap), C.c_uint64(snap.layout_id), None, None, len(snap), o._stream())
    assert rc == K.E_INVALID
    s.close()
    o.close()
