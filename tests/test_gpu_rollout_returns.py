"""Discounted returns on the device: `rollout_returns(actions, discount)` scores K steps in one launch.  Twin handles with equal seeds: A runs
`rollout(actions, record_every=1)`, B runs `rollout_returns`.  B's returns must be, bit for bit, the recurrence below run in torch over A's
recorded rewards and terminations in the env's dtype; its end steps A's first terminations; its (obs, ref) A's last recorded row; and
both handles must end in the same persistent state (checkpoint blob, or snapshot rows and the next steps where checkpoints are refused)."""
import numpy as np
import pytest

from gpu_helpers import ENV_IDS, N, _actions, _bits, _blob, _eq, _ext_env, _make, _next_steps, _same, torch_cuda  # noqa: F401
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

HORIZONS = (64, 7, 1)
DISCOUNTS = (1.0, 0.9, 0.0)

def _spec(torch, rew, term, discount):
    """the documented recurrence over recorded [K, N] rewards / terminations: w = 1, G = 0; G = G + (w * r_k) while not yet terminated;
    w = w * gamma after each step (gamma = discount rounded to the dtype).  Two separate torch ops per update: two roundings, no FMA."""
    k = rew.shape[0]
    t = term.view(torch.bool) if term.dtype == torch.uint8 else term
    gamma = torch.tensor(discount, dtype=rew.dtype, device=rew.device)
    w = torch.ones((), dtype=rew.dtype, device=rew.device)
    g = torch.zeros(rew.shape[1], dtype=rew.dtype, device=rew.device)
    alive = torch.ones(rew.shape[1], dtype=torch.bool, device=rew.device)
    for j in range(k):
        g = torch.where(alive, g + w * rew[j], g)
        alive = alive & ~t[j]
        w = w * gamma
    end = torch.where(t.any(0), t.int().argmax(0), torch.full_like(t[0], k, dtype=torch.int64)).to(torch.int32)
    return g, end


def _pair(torch, a_env, b_env, acts, discount, refs=None, what=""):
    """A: recorded rollout, B: rollout_returns with the same actions; checks returns, end steps and the last outputs.  Returns B's
    returns and end steps."""
    k = int(acts.shape[0])
    (obs, ref), rew, term = a_env.rollout(acts, record_every=1, references=refs)
    ret, end, (o_b, r_b) = b_env.rollout_returns(acts, discount=discount, references=refs)
    assert ret.shape == (a_env.sim.n,) and end.dtype == torch.int32 and ret.dtype == a_env.sim.dtype
    g, e = _spec(torch, rew, term, discount)
    _eq(torch, end, e, (what, "end_step"))
    _eq(torch, ret, g, (what, "returns"))
    _same(torch, o_b, obs[k - 1], (what, "obs"))
    _same(torch, r_b, ref[k - 1], (what, "ref"))
    return ret, end


def _assert_terminations(torch, end, k, what):
    """a sizeable share of envs terminates, at several distinct steps below K: the stop rule is exercised"""
    stopped = end[end < k]
    assert stopped.numel() >= end.numel() // 10, (what, "terminated envs", stopped.numel(), end.numel())
    assert torch.unique(stopped).numel() >= 3, (what, "distinct end steps", torch.unique(stopped).tolist())


@pytest.mark.parametrize("autoreset", ["same_step", "none"])
@pytest.mark.parametrize("layout", ["aos", "soa"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("family", list(ENV_IDS))
def test_returns_equal_recorded_rollout(torch_cuda, family, dtype, layout, autoreset):
    """every horizon and discount on one pair of twins, one after the other (under autoreset none both are reset before each launch, so
    every launch starts inside the limits)"""
    torch = torch_cuda
    a_env, b_env = _make(family, dtype, layout, autoreset), _make(family, dtype, layout, autoreset)
    seed = 0
    for k in HORIZONS:
        for discount in DISCOUNTS:
            if autoreset == "none":
                a_env.reset()
                b_env.reset()
            acts = _actions(torch, a_env, k, seed=seed)
            seed += 1
            what = (family, dtype, layout, autoreset, k, discount)
            _, end = _pair(torch, a_env, b_env, acts, discount, what=what)
            if k == 64:
                _assert_terminations(torch, end, k, what)
            assert a_env.sim.clock() == b_env.sim.clock(), what
    assert np.array_equal(_blob(a_env), _blob(b_env))
    _next_steps(torch, a_env, b_env)


@pytest.mark.parametrize("layout", ["aos", "soa"])
def test_reference_feed(torch_cuda, layout):
    torch = torch_cuda
    a_env, b_env = _ext_env(layout), _ext_env(layout)
    sim = a_env.sim
    for k, discount in ((64, 0.9), (7, 1.0)):
        acts = _actions(torch, a_env, k, seed=k)
        refs = torch.as_tensor(np.random.default_rng(k).uniform(-0.9, 0.9, size=(k,) + sim._shape(sim.n_ref)), dtype=sim.dtype, device="cuda")
        _, end = _pair(torch, a_env, b_env, acts, discount, refs=refs.contiguous(), what=("feed", layout, k))
        if k == 64:
            _assert_terminations(torch, end, k, "feed")
    assert a_env.sim.clock() == b_env.sim.clock()
    assert np.array_equal(_blob(a_env), _blob(b_env))


def test_per_env_parameter_blocks(torch_cuda):
    torch = torch_cuda
    a_env, b_env = _make("pmsm"), _make("pmsm")
    r_s = float(a_env.sim.cfg.motor_param[K.MP_R_S])
    for env in (a_env, b_env):
        env.set_env_parameters(motor_parameter={"r_s": r_s * np.linspace(0.8, 1.2, N)})
    for k, discount in ((64, 0.9), (7, 0.0)):
        _, end = _pair(torch, a_env, b_env, _actions(torch, a_env, k, seed=k), discount, what=("blocks", k))
        if k == 64:
            _assert_terminations(torch, end, k, "blocks")
    assert np.array_equal(_blob(a_env), _blob(b_env))
    _next_steps(torch, a_env, b_env)


def test_per_reset_draws(torch_cuda):
    torch = torch_cuda
    a_env, b_env = _make("pmsm"), _make("pmsm")
    r_s = float(a_env.sim.cfg.motor_param[K.MP_R_S])
    for env in (a_env, b_env):
        env.randomize_env_parameters(motor_parameter={"r_s": (0.8 * r_s, 1.2 * r_s)})
        env.reset()
    for k, discount in ((64, 1.0), (7, 0.9)):
        _, end = _pair(torch, a_env, b_env, _actions(torch, a_env, k, seed=k), discount, what=("draws", k))
        if k == 64:
            _assert_terminations(torch, end, k, "draws")
    # every in-kernel reset drew the same new parameters; checkpoints and snapshots are refused while drawing
    assert torch.equal(a_env.env_parameters()["r_s"], b_env.env_parameters()["r_s"])
    _next_steps(torch, a_env, b_env)  # with draws on: later resets draw alike too
    for env in (a_env, b_env):
        env.randomize_env_parameters()
    assert torch.equal(a_env.snapshot_envs().rows, b_env.snapshot_envs().rows)


def test_adopted_rng_identities(torch_cuda):
    torch = torch_cuda
    a_env, b_env = _make("pmsm"), _make("pmsm")
    for env in (a_env, b_env):
        env.step(_actions(torch, env, 1, seed=3)[0])
        env.restore_envs(env.snapshot_envs(list(range(8)), rng=True), idx=list(range(100, 164)), rows=np.repeat(np.arange(8), 8), rng="source")
    for k, discount in ((64, 0.9), (7, 1.0), (1, 0.0)):
        _pair(torch, a_env, b_env, _actions(torch, a_env, k, seed=k), discount, what=("identities", k))
    assert torch.equal(a_env.snapshot_envs(rng=True).rows, b_env.snapshot_envs(rng=True).rows)
    assert torch.equal(a_env.snapshot_envs(rng=True).rng, b_env.snapshot_envs(rng=True).rng)
    _next_steps(torch, a_env, b_env)


def test_mpc_fan_out(torch_cuda):
    """random-shooting MPC: each plant's state and random stream fanned out to its candidates (rng="source"); candidates of one plant
    given the same actions score the same return and end step"""
    torch = torch_cuda
    plants, cands, k = 6, 50, 16
    plant = _make("pmsm", n=plants, seed=1)
    plant.step(_actions(torch, plant, 1, seed=5)[0])
    snap = plant.snapshot_envs(rng=True)
    rows = np.repeat(np.arange(plants), cands)
    a_env, b_env = _make("pmsm", n=plants * cands, seed=2), _make("pmsm", n=plants * cands, seed=2)
    for env in (a_env, b_env):
        env.restore_envs(snap, rows=rows, rng="source")
    per_plant = _actions(torch, plant, k, seed=6)  # [K, plants, 3]
    acts = per_plant.repeat_interleave(cands, dim=1).contiguous()
    ret, end = _pair(torch, a_env, b_env, acts, 0.9, what="fan-out")
    ret2, end2, _ = b_env.rollout_returns(acts, discount=0.9)  # a second horizon from where the first left off
    for x in (ret, end, ret2, end2):
        x = _bits(torch, x).view(plants, cands)
        assert torch.equal(x, x[:, :1].expand_as(x))
    # and across plants the returns differ: the fan-out did not collapse everything into one env
    assert torch.unique(_bits(torch, ret)).numel() > 1


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_cuda_graph_capture(torch_cuda, dtype):
    """under the device clock rollout_returns_into is stream-ordered and capturable: replays of the captured launch equal eager calls on a
    twin, round after round, with the actions refilled in place"""
    torch = torch_cuda
    k, discount = 12, 0.9
    eager, cap = _make("pmsm", dtype), _make("pmsm", dtype)
    for env in (eager, cap):
        env.sim.set_device_clock(True)
    sim = cap.sim
    static = _actions(torch, cap, k, seed=0).clone()
    ret = torch.empty(N, dtype=sim.dtype, device="cuda")
    end = torch.empty(N, dtype=torch.int32, device="cuda")
    obs = torch.empty(sim._shape(sim.n_state), dtype=sim.dtype, device="cuda")
    ref = torch.empty(sim._shape(sim.n_ref), dtype=sim.dtype, device="cuda")
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        sim.rollout_returns_into(static, k, discount, ret, end, obs, ref)
    terminated = 0
    for rnd in range(4):
        acts = _actions(torch, eager, k, seed=10 + rnd)
        static.copy_(acts)
        graph.replay()
        g, e, (o, r) = eager.sim.rollout_returns(acts, discount)
        _eq(torch, ret, g, (rnd, "returns"))
        _eq(torch, end, e, (rnd, "end_step"))
        _eq(torch, obs, o, (rnd, "obs"))
        _eq(torch, ref, r, (rnd, "ref"))
        terminated += int((e < k).sum())
    assert terminated > 0
    assert eager.sim.clock() == cap.sim.clock()
    assert np.array_equal(_blob(eager), _blob(cap))
