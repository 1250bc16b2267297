"""Reference feed on the device: `rollout(actions, references=R)` gives exactly the outputs, final state and clock of K iterations of
`set_reference(R[k]); step(actions[k])`, bit for bit; `step(action, reference=r)` is `set_reference(r); step(action)`; a captured closed
loop reads row k of its static feed in step k of every replay.  The feed overwrites every reference slot, External or not."""
import numpy as np
import pytest

from helpers import col_rel_err, config_from_meta, golden_names, load_golden, replay_golden
from gpu_helpers import torch_cuda  # noqa: F401
from helpers import DeviceAdapter, _tol
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

N = 384  # three blocks, the last one partly inactive for the 128-thread block
KSTEPS = 24


def _make(torch, family, dtype, layout="aos", seed=5):
    import gym_electric_motor_b200 as gem
    from gym_electric_motor_b200.reference_generators import ExternalReferenceGenerator as Ext, MultipleReferenceGenerator, \
        WienerProcessReferenceGenerator

    env_id, names = {"pmsm": ("Cont-CC-PMSM-v0", ("i_sd", "i_sq")), "permex_sc": ("Cont-SC-PermExDc-v0", ("omega",)),
                     "scim": ("Cont-CC-SCIM-v0", ("i_sd", "i_sq")), "eesm": ("Cont-CC-EESM-v0", ("i_sd", "i_sq")),
                     "pmsm_finite": ("Finite-CC-PMSM-v0", ("i_sd", "i_sq")), "pmsm_mixed": ("Cont-CC-PMSM-v0", ("i_sd", "i_sq"))}[family]
    if family == "pmsm_mixed":  # a Wiener slot next to an External one: the feed overwrites both
        rg = MultipleReferenceGenerator([WienerProcessReferenceGenerator(reference_state="i_sd", sigma_range=(1e-2, 1e-1)), Ext("i_sq")])
    else:
        rg = Ext(names[0]) if len(names) == 1 else MultipleReferenceGenerator([Ext(n) for n in names])
    env = gem.make(env_id, num_envs=N, device="cuda", dtype=dtype, layout=layout, reference_generator=rg, autoreset="same_step", seed=seed)
    env.reset()
    return env


def _actions(torch, env, k, seed=0):
    """saturating actions, constant per env for stretches of 6 steps: currents leave their limits within a few steps, so envs terminate
    and auto-reset inside the launch.  Finite B6 (tau = 1e-5): one active voltage vector per env for the whole run, which first trips the
    current limit after ~50 steps"""
    sim = env.sim
    rng = np.random.default_rng(seed)
    lead = (k,) + sim._shape(sim.n_act)
    if sim.finite:
        a = np.broadcast_to(rng.integers(1, 7, size=lead[1:]), lead)
        return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.int32, device="cuda")
    a = np.repeat(rng.choice([-1.0, 1.0], size=((k + 5) // 6,) + lead[1:]), 6, axis=0)[:k] * rng.uniform(0.6, 1.0, size=lead)
    return torch.as_tensor(a, dtype=sim.dtype, device="cuda").contiguous()


def _feed(torch, env, k, seed=1):
    sim = env.sim
    r = np.random.default_rng(seed).uniform(-0.9, 0.9, size=(k,) + sim._shape(sim.n_ref))
    return torch.as_tensor(r, dtype=sim.dtype, device="cuda").contiguous()


def _set_ref(env, row):
    """the sequential spec's set_reference of one feed row (the host API takes [N, n_ref] in either layout)"""
    env.set_reference((row.t() if env.sim.soa else row).double())


def _sequential(torch, env, actions, refs, every):
    """K iterations of set_reference + step; the outputs a rollout with record_every = every returns"""
    k, rec = int(actions.shape[0]), []
    for j in range(k):
        _set_ref(env, refs[j])
        (o, r), w, t, _, _ = env.step(actions[j])
        rec.append((o.clone(), r.clone(), w.clone(), t.clone()))
    if every == 0:
        return rec[-1]
    sel = rec[every - 1::every]
    return tuple(torch.stack([s[q] for s in sel]) for q in range(4))


def _fused(env, actions, refs, every):
    (o, r), w, t = env.rollout(actions, record_every=every, references=refs)
    return o, r, w, t


def _assert_same(torch, got, want, what):
    for name, a, b in zip(("obs", "ref", "reward", "terminated"), got, want):
        a = a.view(torch.uint8) if a.dtype == torch.bool else a
        b = b.view(torch.uint8) if b.dtype == torch.bool else b
        assert a.shape == b.shape and torch.equal(a, b), (what, name, (a.double() - b.double()).abs().max().item())


def _blob(env):
    return env.sim.state_dict()["blob"]


FAMILIES = ["pmsm", "permex_sc", "scim", "eesm", "pmsm_finite", "pmsm_mixed"]


@pytest.mark.parametrize("clock", ["host", "device"])
@pytest.mark.parametrize("every", [0, 1, 3])
@pytest.mark.parametrize("layout", ["aos", "soa"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("family", FAMILIES)
def test_rollout_feed_equals_set_reference_and_step(torch_cuda, family, dtype, layout, every, clock):
    torch = torch_cuda
    seq, fus = _make(torch, family, dtype, layout), _make(torch, family, dtype, layout)
    if clock == "device":
        seq.sim.set_device_clock(True)
        fus.sim.set_device_clock(True)
    k = 64 if family == "pmsm_finite" else KSTEPS
    acts, refs = _actions(torch, seq, k), _feed(torch, seq, k)
    want = _sequential(torch, seq, acts, refs, every)
    got = _fused(fus, acts, refs, every)
    _assert_same(torch, got, want, (family, dtype, layout, every, clock))
    if every == 1:
        assert bool(want[3].any()), "no env terminated: the auto-reset inside the launch is not exercised"
    assert seq.sim.clock() == fus.sim.clock()
    assert np.array_equal(_blob(seq), _blob(fus))


def test_fed_values_reach_the_reward(torch_cuda):
    """sanity of the spec itself: a different feed gives different rewards and External ref outputs"""
    torch = torch_cuda
    a, b = _make(torch, "pmsm", "float32"), _make(torch, "pmsm", "float32")
    acts = _actions(torch, a, 6)
    ra, rb = _feed(torch, a, 6, seed=1), _feed(torch, a, 6, seed=2)
    (_, ref_a), rew_a, term_a = a.rollout(acts, record_every=1, references=ra)
    (_, ref_b), rew_b, _ = b.rollout(acts, record_every=1, references=rb)
    assert not torch.equal(rew_a, rew_b)
    keep = ~term_a[0]
    assert torch.equal(ref_a[0][keep], ra[0][keep])  # an External slot reports the value its step was scored against


def test_step_with_reference(torch_cuda):
    torch = torch_cuda
    for family, dtype, layout in (("pmsm", "float32", "aos"), ("pmsm_mixed", "float64", "soa"), ("pmsm_finite", "float32", "aos")):
        seq, fed = _make(torch, family, dtype, layout), _make(torch, family, dtype, layout)
        acts, refs = _actions(torch, seq, 8), _feed(torch, seq, 8)
        for j in range(8):
            _set_ref(seq, refs[j])
            (o1, r1), w1, t1, _, _ = seq.step(acts[j])
            (o2, r2), w2, t2, _, _ = fed.step(acts[j], reference=refs[j])
            _assert_same(torch, (o2, r2, w2, t2), (o1, r1, w1, t1), (family, j))
        assert np.array_equal(_blob(seq), _blob(fed))


def test_per_env_blocks_and_draws(torch_cuda):
    torch = torch_cuda
    for mode in ("blocks", "draws"):
        seq, fus = _make(torch, "pmsm_mixed", "float32"), _make(torch, "pmsm_mixed", "float32")
        r_s = float(seq.sim.cfg.motor_param[K.MP_R_S])
        for env in (seq, fus):
            if mode == "blocks":
                env.set_env_parameters(motor_parameter={"r_s": r_s * np.linspace(0.8, 1.2, N)})
            else:
                env.randomize_env_parameters(motor_parameter={"r_s": (0.8 * r_s, 1.2 * r_s)})
                env.reset()
        acts, refs = _actions(torch, seq, KSTEPS), _feed(torch, seq, KSTEPS)
        want = _sequential(torch, seq, acts, refs, 1)
        got = _fused(fus, acts, refs, 1)
        _assert_same(torch, got, want, mode)
        assert bool(want[3].any())
        if mode == "draws":  # every in-kernel reset drew the same new parameters
            assert torch.equal(seq.env_parameters()["r_s"], fus.env_parameters()["r_s"])
            seq.randomize_env_parameters()
            fus.randomize_env_parameters()
        assert torch.equal(seq.snapshot_envs().rows, fus.snapshot_envs().rows)


def test_adopted_rng_identities(torch_cuda):
    torch = torch_cuda
    seq, fus = _make(torch, "pmsm_mixed", "float32"), _make(torch, "pmsm_mixed", "float32")
    for env in (seq, fus):
        env.step(_actions(torch, env, 1, seed=3)[0])
        env.restore_envs(env.snapshot_envs(list(range(8)), rng=True), idx=list(range(100, 164)), rows=np.repeat(np.arange(8), 8), rng="source")
    acts, refs = _actions(torch, seq, KSTEPS), _feed(torch, seq, KSTEPS)
    want = _sequential(torch, seq, acts, refs, 1)
    got = _fused(fus, acts, refs, 1)
    _assert_same(torch, got, want, "identities")
    assert torch.equal(seq.snapshot_envs(rng=True).rows, fus.snapshot_envs(rng=True).rows)
    assert torch.equal(seq.snapshot_envs(rng=True).rng, fus.snapshot_envs(rng=True).rng)


def test_capture_steps_with_a_feed(torch_cuda):
    torch = torch_cuda
    n_steps = 6
    eager, cap_env = _make(torch, "pmsm", "float32"), _make(torch, "pmsm", "float32")

    def policy(s, r):  # closed loop on the fed reference
        return torch.cat([r - s[:, 5:7], torch.zeros_like(r[:, :1])], dim=1).mul(4.0).clamp(-1.0, 1.0).contiguous()

    feed = _feed(torch, eager, n_steps, seed=11)
    static = feed.clone()
    (st, rf), _ = eager.reset()
    cap_env.reset()
    cap = cap_env.capture_steps(policy, n_steps, record=True, references=static)
    for rnd, seed in enumerate((11, 12, 13)):
        if rnd:
            feed = _feed(torch, eager, n_steps, seed=seed)
            static.copy_(feed)  # refilled in place between replays
        rec = []
        for j in range(n_steps):
            a = policy(st, rf)
            _set_ref(eager, feed[j])
            (st, rf), w, t, _, _ = eager.step(a)
            rec.append((st.clone(), rf.clone(), w.clone(), t.clone()))
        cap.replay()
        for j in range(n_steps):
            _assert_same(torch, (cap.states[j], cap.references[j], cap.rewards[j], cap.terminateds[j]), rec[j], (rnd, j))
    cap.release()
    assert np.array_equal(_blob(eager), _blob(cap_env))


def _golden_feed_cases():
    out = []
    for name in golden_names():
        g = load_golden(name)
        if g["meta"]["reference_names"] and g["meta"]["case"]["solver"] != "dopri5":
            out.append(name)
    return out


@pytest.mark.parametrize("name", _golden_feed_cases())
def test_golden_segments_in_one_launch(torch_cuda, name):
    """each stretch between the reference harness's resets in one fused launch with its recorded refs_used: the bits of the per-step
    replay (helpers.replay_golden), fp64"""
    torch = torch_cuda
    from gym_electric_motor_b200.vector_sim import VectorSim

    g = load_golden(name)
    meta = g["meta"]
    cfg = config_from_meta(meta, reset_ode=g["reset_ode"], dtype=K.F64, solver=meta["case"]["solver"])
    step_out = replay_golden(DeviceAdapter(cfg), g)
    sim = VectorSim(config_from_meta(meta, reset_ode=g["reset_ode"], dtype=K.F64, solver=meta["case"]["solver"]))
    ref_idx = [meta["state_names"].index(n) for n in meta["reference_names"]]
    sim.reset()
    k_all = len(g["actions"])
    states, rewards, terms = [], [], []
    begin = 0
    ends = [int(k) for k in np.nonzero(g["terminated"])[0]] + [k_all - 1]
    for end in ends:
        if end < begin:
            continue
        seg = slice(begin, end + 1)
        acts = g["actions"][seg]
        acts = acts.reshape(len(acts), 1, -1)
        refs = torch.as_tensor(np.ascontiguousarray(g["refs_used"][seg][:, ref_idx]).reshape(end + 1 - begin, 1, len(ref_idx)),
                               dtype=torch.float64, device="cuda")
        o, _, w, t = sim.rollout(acts, 1, references=refs)
        states.append(o[:, 0].cpu().numpy())
        rewards.append(w[:, 0].cpu().numpy())
        terms.append(t[:, 0].cpu().numpy())
        if g["terminated"][end]:
            sim.reset()
        begin = end + 1
    states, rewards, terms = np.concatenate(states), np.concatenate(rewards), np.concatenate(terms)
    assert np.array_equal(states, step_out["states"]) and np.array_equal(rewards, step_out["rewards"])
    assert np.array_equal(terms, step_out["terminated"])
    if meta["motor_class"] not in ("SquirrelCageInductionMotor", "DoublyFedInductionMotor"):  # those: the weak-flux rule of test_gpu_parity
        tol = _tol(name, K.F64)
        assert col_rel_err(states, g["states"]) < tol and np.abs(rewards - g["rewards"]).max() < 10 * tol

