"""Cost of linearising the plant along a rollout: the fused Jacobian launch against the recorded rollout alone and against finite differences.

    python tools/jacobian_bench.py [--envs 1048576] [--horizons 8 64] [--reps 10] [--runs 2] [--motors PMSM SCIM]

Cont-CC-<motor>-v0, fp32, row-per-env layout, auto-reset on, U(-0.8, 0.8) actions drawn once up front.  For each motor and horizon K three
arms take turns rep by rep:
  (a) jacobians  rollout_jacobians_into: jac_x, jac_u and every step's obs / ref / reward / terminated (gemb200_rollout_jacobians);
  (b) recorded   rollout_into(record_every=1): the same outputs without the Jacobians;
  (c) fd         forward differences through the env itself: (n_x + n_u + 1) copies of every env in one handle, and per step one read of the
                 ODE state, one restore of the perturbed copies (set_ode_state), one step with the perturbed actions and one read of the result.
                 It runs on --envs // (n_x + n_u + 1) base envs (the copies fill the handle) and its time is scaled to --envs base envs.
Reported: microseconds per step of --envs envs, the median over --reps of CUDA-event timings, for each of --runs runs, and the median and
spread over the runs, plus the Jacobian bytes per env step.  Prints the GPU name and power limit first.  Writes nothing.
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


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=20).stdout.strip()
        name, plimit = [x.strip() for x in out.split(",")[:2]]
        return name, plimit
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def sim_of(motor, n, seed=0):
    cfg = gem.make(f"Cont-CC-{motor}-v0", num_envs=n).build_config()
    cfg.seed = seed
    s = VectorSim(cfg)
    s.reset()
    return s


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def timed(arms, reps, warmup=2):
    for _ in range(warmup):
        for fn, _ in arms.values():
            fn()
    torch.cuda.synchronize()
    ev = {a: [] for a in arms}
    for _ in range(reps):
        for a, (fn, _) in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            ev[a].append((e0, e1))
    torch.cuda.synchronize()
    return {a: median([x.elapsed_time(y) for x, y in ev[a]]) * 1e3 * arms[a][1] for a in arms}


def arms_for(motor, n, k):
    s = sim_of(motor, n)
    nx, nu = s.jacobian_dims()
    acts = (torch.rand((k, n, s.n_act), device=s.device) * 1.6 - 0.8).contiguous()
    jx = torch.empty((k, n, nx, nx), device=s.device)
    ju = torch.empty((k, n, nx, nu), device=s.device)
    obs = torch.empty((k, n, s.n_state), device=s.device)
    ref = torch.empty((k, n, max(s.n_ref, 1)), device=s.device)
    rew = torch.empty((k, n), device=s.device)
    term = torch.empty((k, n), dtype=torch.uint8, device=s.device)
    r = sim_of(motor, n)
    # finite differences: (nx + nu + 1) copies per base env
    c = nx + nu + 1
    p = n // c
    f = sim_of(motor, p * c)
    fa = (torch.rand((k, p, s.n_act), device=s.device) * 1.6 - 0.8)
    eye = torch.eye(c - 1, device=s.device, dtype=torch.float64) * 1e-3

    def fd():
        for j in range(k):
            y = f.get_ode_state().view(p, c, nx)
            y = y[:, :1].expand(p, c, nx).clone()  # every copy restarts from its base env
            y[:, 1:1 + nx] += eye[:nx, :nx]
            a = fa[j].unsqueeze(1).expand(p, c, s.n_act).clone()
            a[:, 1 + nx:] += eye[nx:, nx:].float()
            f.set_ode_state(y.view(p * c, nx))
            f.step(a.view(p * c, s.n_act))
            y1 = f.get_ode_state().view(p, c, nx)
            _ = (y1[:, 1:] - y1[:, :1]) * 1e3

    arms = {
        "jacobians": (lambda: s.rollout_jacobians_into(acts, k, jx, ju, obs, ref if s.n_ref else None, rew, term), 1.0 / k),
        "recorded": (lambda: r.rollout_into(acts, k, 1, obs, ref if s.n_ref else None, rew, term), 1.0 / k),
        "fd": (fd, 1.0 / k * n / p),
    }
    return arms, (nx, nu)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1 << 20)
    ap.add_argument("--horizons", type=int, nargs="+", default=[8, 64])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--motors", nargs="+", default=["PMSM", "SCIM"])
    args = ap.parse_args()
    name, plimit = gpu_info()
    print(json.dumps(dict(gpu=name, power_limit=plimit)))
    for motor in args.motors:
        for k in args.horizons:
            arms, (nx, nu) = arms_for(motor, args.envs, k)
            runs = [timed(arms, args.reps) for _ in range(args.runs)]
            res = {a: dict(runs=[round(r[a], 2) for r in runs], median=round(median([r[a] for r in runs]), 2),
                           spread=round(max(r[a] for r in runs) - min(r[a] for r in runs), 2)) for a in arms}
            print(json.dumps(dict(motor=motor, K=k, envs=args.envs, jac_bytes_per_env_step=4 * nx * (nx + nu), us_per_step=res)))
            del arms
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
