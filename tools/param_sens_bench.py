"""Cost of parameter sensitivities along a rollout: the fused launch against the Jacobian launch, the recorded rollout alone and central
differences over perturbed env copies.

    python tools/param_sens_bench.py [--envs 1048576] [--horizons 8 64] [--reps 10] [--runs 2]

fp32, row-per-env layout, auto-reset on, U(-0.8, 0.8) actions drawn once up front.  Cases: Cont-CC-PMSM-v0 with (r_s, l_d, l_q, psi_p)
and Cont-CC-SCIM-v0 with (r_s, r_r, l_m, l_sigs, l_sigr).  For each case and horizon K five arms take turns rep by rep:
  (a) sens       rollout_param_sens_into with S recorded after every step, and every step's obs / ref / reward / terminated;
  (b) sens_io    the same with only sens_io (S_K), no recorded S;
  (c) jacobians  rollout_jacobians_into: jac_x, jac_u and the recorded outputs;
  (d) recorded   rollout_into(record_every=1): the outputs alone;
  (e) cd         central differences: a recorded rollout of a handle whose envs are 2 n_p + 1 copies of --envs // (2 n_p + 1) base envs with
                 per-env parameter blocks (theta, theta_j (1 +- h)); its time is scaled to --envs base envs.
Reported: microseconds per step of --envs envs, the median over --reps of CUDA-event timings, for each of --runs runs, and over the runs
the upper median (with two runs: the larger one) and the spread.  Prints the GPU name and power limit first.  Writes nothing.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from jacobian_bench import gpu_info, median, sim_of, timed  # noqa: E402
from gym_electric_motor_b200 import _cabi as K  # noqa: E402
from gym_electric_motor_b200.core import ElectricMotorEnvironment  # noqa: E402

CASES = {"PMSM": ["r_s", "l_d", "l_q", "psi_p"], "SCIM": ["r_s", "r_r", "l_m", "l_sigs", "l_sigr"]}


def arms_for(motor, n, k):
    names = CASES[motor]
    slots = [ElectricMotorEnvironment._MP_SLOT[nm] for nm in names]
    n_p = len(slots)
    s = sim_of(motor, n)
    nx = s.param_sens_dims(slots)
    _, nu = s.jacobian_dims()
    acts = (torch.rand((k, n, s.n_act), device=s.device) * 1.6 - 0.8).contiguous()
    sio = torch.zeros((n, nx, n_p), device=s.device)  # arms (a) and (b) carry S on in it from rep to rep: the cost does not depend on S
    so = torch.empty((k, n, nx, n_p), device=s.device)
    obs = torch.empty((k, n, s.n_state), device=s.device)
    ref = torch.empty((k, n, max(s.n_ref, 1)), device=s.device)
    rew = torch.empty((k, n), device=s.device)
    term = torch.empty((k, n), dtype=torch.uint8, device=s.device)
    b = sim_of(motor, n)
    j = sim_of(motor, n)
    jx = torch.empty((k, n, nx, nx), device=s.device)
    ju = torch.empty((k, n, nx, nu), device=s.device)
    r = sim_of(motor, n)
    c = 2 * n_p + 1
    p = n // c
    f = sim_of(motor, p * c)
    mp = np.tile(np.array(list(f.cfg.motor_param)), (p * c, 1))
    for q, slot in enumerate(slots):
        mp[(1 + 2 * q) * p:(2 + 2 * q) * p, slot] *= 1 + 1e-3
        mp[(2 + 2 * q) * p:(3 + 2 * q) * p, slot] *= 1 - 1e-3
    f.set_env_params(mp, None)
    fa = acts[:, :p].repeat(1, c, 1).contiguous()
    fobs = torch.empty((k, p * c, s.n_state), device=s.device)
    fref = torch.empty((k, p * c, max(s.n_ref, 1)), device=s.device)
    frew = torch.empty((k, p * c), device=s.device)
    fterm = torch.empty((k, p * c), dtype=torch.uint8, device=s.device)
    arms = {
        "sens": (lambda: s.rollout_param_sens_into(acts, k, slots, sio, so, obs, ref if s.n_ref else None, rew, term), 1.0 / k),
        "sens_io": (lambda: b.rollout_param_sens_into(acts, k, slots, sio, None, obs, ref if s.n_ref else None, rew, term), 1.0 / k),
        "jacobians": (lambda: j.rollout_jacobians_into(acts, k, jx, ju, obs, ref if s.n_ref else None, rew, term), 1.0 / k),
        "recorded": (lambda: r.rollout_into(acts, k, 1, obs, ref if s.n_ref else None, rew, term), 1.0 / k),
        "cd": (lambda: f.rollout_into(fa, k, 1, fobs, fref if s.n_ref else None, frew, fterm), 1.0 / k * n / p),
    }
    return arms, (nx, n_p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1 << 20)
    ap.add_argument("--horizons", type=int, nargs="+", default=[8, 64])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--motors", nargs="+", default=list(CASES))
    args = ap.parse_args()
    name, plimit = gpu_info()
    print(json.dumps(dict(gpu=name, power_limit=plimit)))
    for motor in args.motors:
        for k in args.horizons:
            arms, (nx, n_p) = arms_for(motor, args.envs, k)
            runs = [timed(arms, args.reps) for _ in range(args.runs)]
            res = {a: dict(runs=[round(r[a], 2) for r in runs], upper_median=round(median([r[a] for r in runs]), 2),
                           spread=round(max(r[a] for r in runs) - min(r[a] for r in runs), 2)) for a in arms}
            print(json.dumps(dict(motor=motor, K=k, envs=args.envs, n_p=n_p, sens_bytes_per_env_step=4 * nx * n_p, us_per_step=res)))
            del arms
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
