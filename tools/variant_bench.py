"""Time the headline kernel for any set of builds of the library, such as the parent commit and a change, each built with
gym_electric_motor_b200.build.build(out=...).
usage: python tools/variant_bench.py parent/libgemb200.so change/libgemb200.so     (each run in a subprocess: GEMB200_LIB override)"""
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
n = 1 << 20
env = gem.make(os.environ.get("GEMB200_ENV", "Cont-CC-PMSM-v0"), num_envs=n, ode_solver=gem.physical_systems.RK4Solver(), autoreset="same_step", seed=0)
env.reset()
sim = env.sim
dev = sim.device
pool = [torch.rand((n, sim.n_act), device=dev) * 2 - 1 for _ in range(8)]
K = 64
roll = torch.stack([pool[k %% 8] for k in range(K)]).contiguous()
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
for k in range(10): env.step(pool[k %% 8])
torch.cuda.synchronize()
# (a) per-step events with L2 flush
evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(100)]
for k in range(100):
    flush.zero_(); evs[k][0].record(); env.step(pool[k %% 8]); evs[k][1].record()
torch.cuda.synchronize()
ms_ev = sum(a.elapsed_time(b) for a, b in evs) / 100
# (b) back-to-back launches from C (gemb200_rollout), events around K steps
best = 1e9
for rep in range(5):
    sim.time_begin(); sim.rollout(roll); ms = sim.time_end() / K
    best = min(best, ms)
# (c) host cost of one env.step call (tiny batch)
import time
small = gem.make(os.environ.get("GEMB200_ENV", "Cont-CC-PMSM-v0"), num_envs=256, ode_solver=gem.physical_systems.RK4Solver(), autoreset="same_step")
small.reset(); a = torch.zeros((256, small.sim.n_act), device=dev)
for _ in range(200): small.step(a)
torch.cuda.synchronize(); t0 = time.perf_counter()
for _ in range(2000): small.step(a)
torch.cuda.synchronize(); host_us = (time.perf_counter() - t0) / 2000 * 1e6
print(json.dumps({"lib": os.path.basename(os.environ.get("GEMB200_LIB", "default")), "ms_events_flush": ms_ev, "ms_rollout_back_to_back": best,
                  "steps_per_s_rollout": n / (best * 1e-3), "host_us_per_step_call": host_us}))
''' % ROOT

for lib in sys.argv[1:] or [""]:
    env = dict(os.environ)
    if lib:
        env["GEMB200_LIB"] = os.path.abspath(lib)
    r = subprocess.run([sys.executable, "-c", CHILD], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    print(r.stdout.strip() or ("FAILED " + lib + " " + r.stderr[-400:]), flush=True)
