"""Cost of per-episode domain randomisation in the fused rollout: three arms alternating in one process.

    python tools/randomization_bench.py [--envs 1048576] [--steps 32] [--reps 20] [--env Cont-CC-PMSM-v0 ...]

Per env id (default Cont-CC-PMSM-v0 and Cont-CC-SCIM-v0), fp32, row-per-env (AoS) layout, auto-reset on, fused rollouts of --steps steps
with every step recorded and U(-1, 1) actions drawn once up front:
  shared      the shared constant-bank coefficients (the default path);
  envp        per-env parameter blocks set on the host (gemb200_set_env_params, every non-zero motor parameter except the pole pairs
              drawn once from +-20 % around its value);
  randomized  the same blocks with those parameters drawn again at every reset (gemb200_set_param_randomization), so every
              auto-reset inside the rollout pays the draw and the double-precision derivation.
The arms take turns rollout by rollout; each rollout is timed with CUDA events and the median over --reps is reported as microseconds
per env step of the whole batch, with the share of env steps that ended in a reset.  Also prints the wall time of the host call
gemb200_set_env_params at this size.  Prints the GPU name and power limit first.  Run from the repository root after the build; writes
nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import gym_electric_motor_b200 as gem  # noqa: E402
from gym_electric_motor_b200 import _cabi as K  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=20).stdout.strip()
        name, plimit = [x.strip() for x in out.split(",")[:2]]
        return name, plimit
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def spec_of(env):
    """every non-zero motor parameter except the pole pairs: name -> (0.8 v, 1.25 v)"""
    cfg, spec, used = env.build_config(), {}, set()
    for name, slot in env._MP_SLOT.items():
        v = cfg.motor_param[slot]
        if slot == K.MP_P or slot in used or v == 0:
            continue
        used.add(slot)
        spec[name] = tuple(sorted((0.8 * v, 1.25 * v)))
    return spec


def bench_env(env_id, n, steps, reps):
    mk = lambda: gem.make(env_id, num_envs=n, autoreset="same_step", seed=1, dtype="float32")  # noqa: E731
    arms = {"shared": mk(), "envp": mk(), "randomized": mk()}
    spec = spec_of(arms["shared"])
    rng = np.random.default_rng(0)
    rows = {name: rng.uniform(lo, hi, size=n) for name, (lo, hi) in spec.items()}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    arms["envp"].set_env_parameters(motor_parameter=rows)
    host_set_s = time.perf_counter() - t0
    arms["randomized"].set_env_parameters(motor_parameter=rows)
    arms["randomized"].randomize_env_parameters(motor_parameter=spec)
    for env in arms.values():
        env.reset()
    n_act = len(arms["shared"].action_space.low)
    acts = (torch.rand((steps, n, n_act), device="cuda", generator=torch.Generator(device="cuda").manual_seed(0)) * 2 - 1).contiguous()
    for _ in range(3):
        for env in arms.values():
            env.rollout(acts, record_every=1)
    torch.cuda.synchronize()
    ev = {a: [] for a in arms}
    resets = {a: 0 for a in arms}
    for _ in range(reps):
        for a, env in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _, _, term = env.rollout(acts, record_every=1)
            e1.record()
            ev[a].append((e0, e1))
            resets[a] += int(term.sum())
    torch.cuda.synchronize()
    out = dict(what="randomization_rollout", env=env_id, envs=n, steps=steps, reps=reps, dtype="float32", layout="aos",
               drawn=sorted(spec), host_set_env_params_s=round(host_set_s, 3))
    for a in arms:
        ms = sorted(x.elapsed_time(y) for x, y in ev[a])
        out[f"us_per_step_{a}"] = round(ms[len(ms) // 2] * 1e3 / steps, 3)
        out[f"reset_share_{a}"] = round(resets[a] / (reps * steps * n), 5)
    out["randomized_over_envp"] = round(out["us_per_step_randomized"] / out["us_per_step_envp"], 4)
    out["envp_over_shared"] = round(out["us_per_step_envp"] / out["us_per_step_shared"], 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--env", action="append", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    name, plimit = gpu_info()
    print(f"GPU: {name}, power limit {plimit}")
    for env_id in args.env or ["Cont-CC-PMSM-v0", "Cont-CC-SCIM-v0"]:
        print(json.dumps(bench_env(env_id, args.envs, args.steps, args.reps)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
