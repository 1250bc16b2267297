"""Time the fused rollout (Cont-CC-PMSM-v0) for any set of builds of the library, such as the parent commit and a change, each built
with gym_electric_motor_b200.build.build(out=...).
usage: python tools/rollout_variant_bench.py parent/libgemb200.so change/libgemb200.so     (each build in its own subprocess: GEMB200_LIB override)"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r'''
import sys, json, os
sys.path.insert(0, %r)
import torch
import gym_electric_motor_b200 as gem
import bench
cfgname = os.environ.get("GEMB200_BENCH_CONFIG", "pmsm")
out = {"lib": os.path.basename(os.environ.get("GEMB200_LIB", "default")), "config": cfgname}
for n, k in ((1 << 20, 16), (1 << 16, 64)):
    envs = [bench.make_env(cfgname, n, 0, r) for r in range(2)]
    for e in envs: e.reset()
    sim = envs[0].sim
    dev = sim.device
    if sim.finite:
        acts = [torch.randint(0, 8, (k, n, sim.n_act), device=dev, dtype=torch.int32) for _ in range(2)]
    else:
        acts = [torch.rand((k, n, sim.n_act), device=dev) * 2 - 1 for _ in range(2)]
    outs = [(torch.empty((k, n, sim.n_state), device=dev), torch.empty((k, n, max(sim.n_ref, 1)), device=dev), torch.empty((k, n), device=dev), torch.empty((k, n), dtype=torch.uint8, device=dev)) for _ in range(2)]
    for every in (1, 0):
        for r in range(3): envs[r %% 2].sim.rollout_into(acts[r %% 2], k, every, *outs[r %% 2])
        torch.cuda.synchronize()
        reps = max(8, 512 // k)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for r in range(reps): envs[r %% 2].sim.rollout_into(acts[r %% 2], k, every, *outs[r %% 2])
        e1.record(); torch.cuda.synchronize()
        out[f"us_step_n{n}_k{k}_rec{every}"] = round(1e3 * e0.elapsed_time(e1) / reps / k, 3)
    # single-step launches, rotating replicas
    pool = [acts[0][j] for j in range(8)]
    for r in range(8): envs[r %% 2].step(pool[r %% 8])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for r in range(200): envs[r %% 2].step(pool[r %% 8])
    e1.record(); torch.cuda.synchronize()
    out[f"us_step_n{n}_single"] = round(1e3 * e0.elapsed_time(e1) / 200, 3)
    for e in envs: e.close()
print(json.dumps(out))
''' % ROOT

for lib in sys.argv[1:] or [""]:
    env = dict(os.environ)
    if lib:
        env["GEMB200_LIB"] = os.path.abspath(lib)
    r = subprocess.run([sys.executable, "-c", CHILD], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    print(r.stdout.strip() or ("FAILED " + lib + " " + r.stderr[-400:]), flush=True)
