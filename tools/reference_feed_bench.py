"""Cost of a caller-supplied reference trajectory: the reference feed against the per-step set_reference path, in one process.

    python tools/reference_feed_bench.py [--envs 1048576] [--steps 32] [--reps 20] [--graph-envs 65536]

Cont-CC-PMSM-v0, fp32, row-per-env (AoS) layout, auto-reset on, U(-1, 1) actions and U(-0.9, 0.9) references drawn once up front.
Arms (a) to (c) run --envs envs with --steps steps, every step recorded; the reference generator is two ExternalReferenceGenerator
slots on i_sd and i_sq, except in (c):
  (a) feed        one fused rollout with the reference feed (gemb200_rollout_record_ref);
  (b) per_step    the same steps as set_reference(R[k]) + step(actions[k]) per step (R already in float64: the conversion is not timed);
  (c) wiener      the default env (Wiener references) in one PLAIN fused rollout: the ceiling of (a);
  (d) graph_feed  --graph-envs envs, --steps closed-loop steps with a constant-action policy and a reference feed, captured once with
                  capture_steps(..., references=R) and replayed.
The arms take turns rep by rep; each rep is timed with CUDA events (for (b) the events enclose the host loop, whose set_reference
synchronises every step) and the median over --reps is reported as microseconds per env step of the whole batch.  (a) and (b) are
checked to give identical outputs first.  Prints the GPU name and power limit first.  Run from the repository root after the build;
writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import gym_electric_motor_b200 as gem  # noqa: E402
from gym_electric_motor_b200.reference_generators import ExternalReferenceGenerator, MultipleReferenceGenerator  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=20).stdout.strip()
        name, plimit = [x.strip() for x in out.split(",")[:2]]
        return name, plimit
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def make(n, external=True):
    rg = MultipleReferenceGenerator([ExternalReferenceGenerator("i_sd"), ExternalReferenceGenerator("i_sq")]) if external else None
    env = gem.make("Cont-CC-PMSM-v0", num_envs=n, autoreset="same_step", seed=1, dtype="float32", reference_generator=rg)
    env.reset()
    return env


def median_us_per_step(pairs, steps):
    ms = sorted(a.elapsed_time(b) for a, b in pairs)
    return round(ms[len(ms) // 2] * 1e3 / steps, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--graph-envs", type=int, default=1 << 16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    name, plimit = gpu_info()
    print(f"GPU: {name}, power limit {plimit}")
    n, k = args.envs, args.steps
    g = torch.Generator(device="cuda").manual_seed(0)
    acts = (torch.rand((k, n, 3), device="cuda", generator=g) * 2 - 1).contiguous()
    refs = (torch.rand((k, n, 2), device="cuda", generator=g) * 1.8 - 0.9).contiguous()
    refs64 = refs.double()
    feed, per_step, wiener = make(n), make(n), make(n, external=False)

    def run_feed():
        return feed.rollout(acts, record_every=1, references=refs)

    def run_per_step():
        for j in range(k):
            per_step.set_reference(refs64[j])
            per_step.step(acts[j])

    def run_wiener():
        return wiener.rollout(acts, record_every=1)

    # same outputs: the fused feed against the per-step path, from the same start
    (s_a, r_a), w_a, t_a = run_feed()
    last = None
    for j in range(k):
        per_step.set_reference(refs64[j])
        last = per_step.step(acts[j])
    (s_b, r_b), w_b, t_b, _, _ = last
    same = bool(torch.equal(s_a[-1], s_b) and torch.equal(r_a[-1], r_b) and torch.equal(w_a[-1], w_b) and torch.equal(t_a[-1], t_b))
    if not same:
        raise SystemExit("the fused feed and the per-step path disagree")

    gn = args.graph_envs
    genv = make(gn)
    grefs = (torch.rand((k, gn, 2), device="cuda", generator=g) * 1.8 - 0.9).contiguous()
    const = torch.full((gn, 3), 0.1, device="cuda")
    cap = genv.capture_steps(lambda s, r: const, k, references=grefs)

    arms = {"feed": run_feed, "per_step": run_per_step, "wiener": run_wiener, "graph_feed": cap.replay}
    for _ in range(3):
        for fn in arms.values():
            fn()
    torch.cuda.synchronize()
    ev = {a: [] for a in arms}
    for _ in range(args.reps):
        for a, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            ev[a].append((e0, e1))
    torch.cuda.synchronize()
    cap.release()
    out = dict(what="reference_feed", env="Cont-CC-PMSM-v0", envs=n, graph_envs=gn, steps=k, reps=args.reps, dtype="float32", layout="aos",
               outputs_identical=same)
    for a in arms:
        out[f"us_per_step_{a}"] = median_us_per_step(ev[a], k)
    out["per_step_over_feed"] = round(out["us_per_step_per_step"] / out["us_per_step_feed"], 3)
    out["feed_over_wiener"] = round(out["us_per_step_feed"] / out["us_per_step_wiener"], 4)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
