"""Time rollout_return_grads against rollout_jacobians and rollout_returns on one GPU (CUDA events, warm-up, repeated runs).

    python tools/return_grad_bench.py [--n 1048576] [--reps 5] [--out results/return_grad_bench.json]

Per motor (PMSM, SCIM), fp32, N envs and K in {8, 64}: microseconds per env-step of the whole batch (median and spread of `reps` runs) for
(a) rollout_return_grads, (b) rollout_jacobians, (c) rollout_returns, and (d) central differences of (c), which need
2 (n_x + K n_u) + 1 copies of every plant: (c) times that count, the fan-out itself not included.  The card name and power limit are read in
the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import gym_electric_motor_b200 as gem

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"card": card, "n": args.n, "dtype": "float32", "rows": []}
    for env_id in ("Cont-CC-PMSM-v0", "Cont-CC-SCIM-v0"):
        env = gem.make(env_id, num_envs=args.n, device="cuda", dtype="float32", autoreset="same_step", seed=0)
        env.reset()
        sim = env.sim
        nx, nu, ww = sim.return_grad_dims()
        for k in (8, 64):
            acts = (torch.rand(k, args.n, nu, device="cuda") * 1.6 - 0.8).contiguous()
            ret = torch.empty(args.n, device="cuda")
            end = torch.empty(args.n, dtype=torch.int32, device="cuda")
            ga = torch.empty(k, args.n, nu, device="cuda")
            gx = torch.empty(args.n, nx, device="cuda")
            ws = torch.empty(k * args.n * ww, device="cuda")
            jx = torch.empty(k, args.n, nx, nx, device="cuda")
            ju = torch.empty(k, args.n, nx, nu, device="cuda")
            calls = {
                "a_return_grads": lambda: sim.rollout_return_grads_into(acts, k, 0.99, ws, ret, end, ga, gx),
                "b_jacobians": lambda: sim.rollout_jacobians_into(acts, k, jx, ju),
                "c_returns": lambda: sim.rollout_returns_into(acts, k, 0.99, ret, end),
            }
            row = {"env": env_id, "K": k, "ws_bytes": k * args.n * ww * 4}
            for name, fn in calls.items():
                fn()
                torch.cuda.synchronize()
                ts = []
                for _ in range(args.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn()
                    e1.record()
                    torch.cuda.synchronize()
                    ts.append(e0.elapsed_time(e1) * 1e3 / k)  # us per env-step of the whole batch
                ts.sort()
                row[name] = {"median_us": ts[len(ts) // 2], "min_us": ts[0], "max_us": ts[-1]}
            copies = 2 * (nx + k * nu) + 1
            row["d_central_differences_us"] = row["c_returns"]["median_us"] * copies
            row["fd_copies"] = copies
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
        del env, sim
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps({"card": card}))


if __name__ == "__main__":
    main()
