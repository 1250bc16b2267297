"""Cost of scoring action sequences: discounted returns from one fused launch against the per-step outputs it replaces, in one process.

    python tools/rollout_returns_bench.py [--envs 1048576] [--horizons 8 64] [--reps 20] [--runs 3] [--plants 1024] [--mpc-horizon 8]

Cont-CC-PMSM-v0, fp32, row-per-env (AoS) layout, auto-reset on, U(-1, 1) actions drawn once up front, discount 0.99.  For each horizon K
and two coefficient modes, `shared` (shared coefficients) and `ids` (every env adopts another env's RNG identity, which puts every launch on
the ENVP instantiation), three arms take turns rep by rep:
  (a) returns   rollout_returns_into: returns, end steps and the last step's obs / ref (gemb200_rollout_returns);
  (b) last      rollout(record_every=0): the last step's obs / ref / reward / terminated, no score;
  (c) recorded  rewards and terminations recorded every step, then the termination-aware discounted sum and the first-termination index
                in torch (the score (a) computes in registers).
Reported: microseconds per env step of the whole batch, the median over --reps of CUDA-event timings, for each of --runs runs, and the
median and spread (max - min) over the runs.
Then the random-shooting MPC control step of tools/branch_bench.py, --plants plants x (--envs / --plants) candidates x --mpc-horizon steps,
rng="source" (every candidate adopts its plant's identity): snapshot the plants, fan them out, score the candidates, argmax per plant, step
the plants with the first action of their best candidate.  Scored by (a) and by (c), alternating, timed the same way.
Before timing, (a) is checked against (c)'s recorded rewards run through the exact recurrence of gemb200_rollout_returns on a twin
handle.  Prints the GPU name and power limit first.  Run from the repository root after the build; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import gym_electric_motor_b200 as gem  # noqa: E402
from gym_electric_motor_b200.vector_sim import VectorSim  # noqa: E402

DISCOUNT = 0.99


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=20).stdout.strip()
        name, plimit = [x.strip() for x in out.split(",")[:2]]
        return name, plimit
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def sim_of(n, seed=0):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=n)
    cfg = env.build_config()
    cfg.seed = seed
    s = VectorSim(cfg)
    s.reset()
    return s


def adopt_rotated_ids(s):
    """every env adopts the identity of its neighbour: all envs read an identity row, as after an MPC fan-out with rng="source" """
    s.restore(s.snapshot(rng=True), rows=torch.roll(torch.arange(s.n, device=s.device, dtype=torch.int32), 1), rng="source")


def torch_score(rew, term, weights):
    """termination-aware discounted return and first-termination index of recorded [K, N] rewards / terminations"""
    t = term.view(torch.bool)
    ti = t.to(torch.int32)
    alive = (ti.cumsum(0) - ti) == 0  # no termination before step k
    g = (rew * weights.view(-1, 1) * alive).sum(0)
    end = torch.where(t.any(0), ti.argmax(0), torch.full_like(ti[0], rew.shape[0]))
    return g, end


def exact_check(n, k, acts):
    """(a) against the recurrence over recorded rewards (two handles with equal seeds), bit for bit"""
    a, b = sim_of(n, seed=5), sim_of(n, seed=5)
    _, _, rew, term = a.rollout(acts, 1)
    ret, end, _ = b.rollout_returns(acts, DISCOUNT)
    gamma = torch.tensor(DISCOUNT, dtype=rew.dtype, device=rew.device)
    w = torch.ones((), dtype=rew.dtype, device=rew.device)
    g = torch.zeros(n, dtype=rew.dtype, device=rew.device)
    alive = torch.ones(n, dtype=torch.bool, device=rew.device)
    t = term.view(torch.bool)
    for j in range(k):
        g = torch.where(alive, g + w * rew[j], g)
        alive = alive & ~t[j]
        w = w * gamma
    e = torch.where(t.any(0), t.to(torch.int32).argmax(0), torch.full_like(end, k))
    ok = bool(torch.equal(g.view(torch.int32), ret.view(torch.int32)) and torch.equal(e.to(torch.int32), end))
    return ok, float((end < k).float().mean())


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def alternate(arms, reps, steps, warmup=3):
    """arms take turns rep by rep; median microseconds per env step of each"""
    for _ in range(warmup):
        for fn in arms.values():
            fn()
    torch.cuda.synchronize()
    ev = {a: [] for a in arms}
    for _ in range(reps):
        for a, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            ev[a].append((e0, e1))
    torch.cuda.synchronize()
    return {a: median([x.elapsed_time(y) for x, y in ev[a]]) * 1e3 / steps for a in arms}


def summarize(per_run):
    out = {}
    for a in per_run[0]:
        v = [r[a] for r in per_run]
        out[a] = dict(runs=[round(x, 3) for x in v], median=round(median(v), 3), spread=round(max(v) - min(v), 3))
    return out


def rollout_arms(args, k, mode):
    n = args.envs
    s = sim_of(n, seed=1)
    if mode == "ids":
        adopt_rotated_ids(s)
    g = torch.Generator(device="cuda").manual_seed(k)
    acts = (torch.rand((k, n, 3), device="cuda", generator=g) * 2 - 1).contiguous()
    ret = torch.empty(n, dtype=s.dtype, device="cuda")
    end = torch.empty(n, dtype=torch.int32, device="cuda")
    obs = torch.empty((n, s.n_state), dtype=s.dtype, device="cuda")
    ref = torch.empty((n, s.n_ref), dtype=s.dtype, device="cuda")
    rew1 = torch.empty(n, dtype=s.dtype, device="cuda")
    term1 = torch.empty(n, dtype=torch.uint8, device="cuda")
    rew = torch.empty((k, n), dtype=s.dtype, device="cuda")
    term = torch.empty((k, n), dtype=torch.uint8, device="cuda")
    weights = DISCOUNT ** torch.arange(k, device="cuda", dtype=torch.float64)
    weights = weights.to(s.dtype)

    def returns():
        s.rollout_returns_into(acts, k, DISCOUNT, ret, end, obs, ref)

    def last():
        s.rollout_into(acts, k, 0, obs, ref, rew1, term1)

    def recorded():
        s.rollout_into(acts, k, 1, None, None, rew, term)
        return torch_score(rew, term, weights)

    arms = dict(returns=returns, last=last, recorded=recorded)
    per_run = [alternate(arms, args.reps, k) for _ in range(args.runs)]
    del s, acts, rew, term
    torch.cuda.empty_cache()
    return summarize(per_run)


def mpc(args):
    p_n, h = args.plants, args.mpc_horizon
    c = args.envs // p_n
    plant, model = sim_of(p_n, seed=1), sim_of(p_n * c, seed=2)
    g = torch.Generator(device="cuda").manual_seed(0)
    cand = (torch.rand((h, p_n * c, model.n_act), device="cuda", generator=g) * 2 - 1).contiguous()
    ridx = torch.arange(p_n, device="cuda", dtype=torch.int32).repeat_interleave(c)
    base = torch.arange(p_n, device="cuda") * c
    ret = torch.empty(p_n * c, dtype=model.dtype, device="cuda")
    rew = torch.empty((h, p_n * c), dtype=model.dtype, device="cuda")
    term = torch.empty((h, p_n * c), dtype=torch.uint8, device="cuda")
    weights = (DISCOUNT ** torch.arange(h, device="cuda", dtype=torch.float64)).to(model.dtype)

    def control_step(score):
        model.restore(plant.snapshot(rng=True), rows=ridx, rng="source")
        best = score().view(p_n, c).argmax(1) + base
        plant.step(cand[0].index_select(0, best))

    def by_returns():
        model.rollout_returns_into(cand, h, DISCOUNT, ret)
        return ret

    def by_recorded():
        model.rollout_into(cand, h, 1, None, None, rew, term)
        return torch_score(rew, term, weights)[0]

    arms = dict(returns=lambda: control_step(by_returns), recorded=lambda: control_step(by_recorded))
    per_run = [alternate(arms, args.reps, 1) for _ in range(args.runs)]  # "per step" = per control step here: microseconds
    return p_n, c, h, summarize(per_run)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1 << 20)
    ap.add_argument("--horizons", type=int, nargs="+", default=[8, 64])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--plants", type=int, default=1024)
    ap.add_argument("--mpc-horizon", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    name, plimit = gpu_info()
    print(f"GPU: {name}, power limit {plimit}", flush=True)
    for k in args.horizons:
        gk = torch.Generator(device="cuda").manual_seed(100 + k)
        ok, share = exact_check(1 << 16, k, (torch.rand((k, 1 << 16, 3), device="cuda", generator=gk) * 2 - 1).contiguous())
        if not ok:
            raise SystemExit(f"K = {k}: rollout_returns differs from the recurrence over recorded rewards")
        for mode in ("shared", "ids"):
            res = rollout_arms(args, k, mode)
            print(json.dumps(dict(what="rollout_returns", env="Cont-CC-PMSM-v0", envs=args.envs, steps=k, mode=mode, dtype="float32",
                                  discount=DISCOUNT, exact_check=ok, terminated_share_in_check=round(share, 4), us_per_env_step=res)), flush=True)
    p_n, c, h, res = mpc(args)
    print(json.dumps(dict(what="mpc_control_step", rng="source", plants=p_n, candidates=c, horizon=h, discount=DISCOUNT, us_per_control_step=res)),
          flush=True)


if __name__ == "__main__":
    main()
