"""Per-env snapshot throughput (gemb200_pack_envs / gemb200_unpack_envs) and a random-shooting MPC control step built on it.

    python tools/branch_bench.py [--envs 1048576] [--reps 20] [--rng own|source] [--params]

Prints the GPU name and power limit, then one JSON line per measurement (CUDA events, median over --reps):
  1. pack and unpack of all envs of Cont-CC-PMSM-v0 (fp32: 11 words = 44 B per env), bytes moved and the fraction of the H100 SXM data-sheet
     bandwidth (3.35 TB/s);
  2. fan-out unpack of 1024 rows into all envs (row_idx: every row into envs/1024 consecutive envs);
  3. a random-shooting MPC control step, 1024 plants x 1024 candidates x horizon 8: pack the plants, fan them out into the model handle,
     rollout recording only the rewards, sum over the horizon, argmax per plant, step the plants with the first action of their best
     branch.  The candidate actions are drawn once up front (their generation is the policy's cost, not the simulator's).
--rng source (copy.deepcopy semantics: every candidate adopts its plant's RNG identity, so all candidates of a plant are scored against
the same future reference) packs the identities with the rows and adopts them with the fan-out, in 1.-3. alike.  Before timing it checks
that the candidates of every plant record identical reference trajectories until they terminate.  It then prints a fourth line:
  4. microseconds per env step of a fused rollout of --envs envs recording every step for 32 steps, auto-reset on, in three arms taking
     turns: shared coefficients, per-env parameter blocks that hold the shared parameters, and the same blocks with adopted identities.
--params measures snapshots that carry the physical parameters (gemb200_pack_envs_params / gemb200_unpack_envs_params) instead, each
line with a state-only arm (no parameter draws, gemb200_pack_envs / _unpack_envs) and a params arm (r_s, l_d, l_q, psi_p and j_rotor drawn
+-20 % at every reset; 192 B parameter row per env): 1. pack and 2. unpack of all envs, 3. fan-out of 1024 rows into all envs, and
4. the MPC control step with rng="source" (identity only, shared plants) against rng="source", params="source" on randomised plants (the
model handle draws from the same distribution).
Run from the repository root after the build; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import gym_electric_motor_b200 as gem  # noqa: E402
from gym_electric_motor_b200.vector_sim import VectorSim  # noqa: E402

PEAK = 3.35e12  # H100 SXM data-sheet HBM3 bandwidth, B/s


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=20).stdout.strip()
        name, plimit = [x.strip() for x in out.split(",")[:2]]
        return name, plimit
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def timed(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return ms[len(ms) // 2]


def sim_of(n, seed=0):
    env = gem.make("Cont-CC-PMSM-v0", num_envs=n)
    cfg = env.build_config()
    cfg.seed = seed
    return VectorSim(cfg)


DRAWN = ("r_s", "l_d", "l_q", "psi_p", "j_rotor")


def randomised(sim):
    """draw DRAWN +-20 % around the configuration's values at every reset of `sim`"""
    from gym_electric_motor_b200 import _cabi as K

    slots = [dict(r_s=K.MP_R_S, l_d=K.MP_L_D, l_q=K.MP_L_Q, psi_p=K.MP_PSI_P, j_rotor=K.MP_J_ROTOR)[x] for x in DRAWN]
    v = [sim.cfg.motor_param[s] for s in slots]
    sim.set_param_randomization(slots, [K.DIST_UNIFORM] * len(slots), [0.8 * x for x in v], [1.2 * x for x in v])
    return sim


def line(**kw):
    for arm in ("state", "params"):
        if f"bytes_{arm}" in kw and f"ms_{arm}" in kw:
            kw[f"tb_s_{arm}"] = round(kw[f"bytes_{arm}"] / kw[f"ms_{arm}"] / 1e9, 3)
            kw[f"frac_datasheet_{arm}"] = round(kw[f"bytes_{arm}"] / kw[f"ms_{arm}"] / 1e-3 / PEAK, 3)
    print(json.dumps(kw))


def params_main(args):
    """--params: snapshots with physical parameters against state-only snapshots, and the MPC step on randomised plants"""
    mode = args.rng
    ids = mode == "source"
    n, m = args.envs, 1024
    state, drawn = sim_of(n, seed=0), randomised(sim_of(n, seed=0))
    for s in (state, drawn):
        s.reset()
    words, _ = state.record_layout()
    rec, idb, prb = 4 * words, (4 * 8 if ids else 0), 8 * 24  # state row, identity row, parameter row (bytes per env)
    envp_b = 30 * 4  # fp32 envp column
    snap_s, snap_p = state.snapshot(rng=ids), drawn.snapshot(rng=ids, params=True)
    torch.cuda.synchronize()
    ms_s = timed(lambda: state.snapshot(rng=ids), args.reps)
    ms_p = timed(lambda: drawn.snapshot(rng=ids, params=True), args.reps)
    line(what="pack", rng=mode, envs=n, ms_state=round(ms_s, 4), ms_params=round(ms_p, 4), bytes_state=2 * (rec + idb) * n,
         bytes_params=2 * (rec + idb + prb) * n)
    ms_s = timed(lambda: state.restore(snap_s, rng=mode), args.reps)
    ms_p = timed(lambda: drawn.restore(snap_p, rng=mode, params="source"), args.reps)
    # params: the rows read, 23 praw slots written, the pole-pair slot read, the envp column written
    line(what="unpack", rng=mode, envs=n, ms_state=round(ms_s, 4), ms_params=round(ms_p, 4), bytes_state=2 * (rec + idb) * n,
         bytes_params=2 * (rec + idb) * n + (prb + prb + envp_b) * n)
    few_s, few_p = snap_s[:m], snap_p[:m]
    ridx = torch.arange(m, device=state.device, dtype=torch.int32).repeat_interleave(n // m)
    ms_s = timed(lambda: state.restore(few_s, rows=ridx, rng=mode), args.reps)
    ms_p = timed(lambda: drawn.restore(few_p, rows=ridx, rng=mode, params="source"), args.reps)
    b_s = (rec + 4) * n + rec * m + ((2 * idb + 4) * n + idb * m if ids else 0)
    b_p = b_s + (prb + envp_b + 4) * n + prb * m  # 23 praw slots written + the pole-pair slot read, envp written, the row index again
    line(what="fan_out_unpack", rng=mode, rows=m, envs=n, ms_state=round(ms_s, 4), ms_params=round(ms_p, 4), bytes_state=b_s, bytes_params=b_p)
    del state, drawn, snap_s, snap_p, few_s, few_p
    torch.cuda.empty_cache()

    p_n, h = args.plants, args.horizon
    c = n // p_n
    out = dict(what="mpc_control_step_params", plants=p_n, candidates=c, horizon=h)
    for arm in ("identity_only", "params_randomised"):
        plant, model = sim_of(p_n, seed=1), sim_of(p_n * c, seed=2)
        if arm == "params_randomised":
            randomised(plant)
            randomised(model)
        plant.reset()
        model.reset()
        gen = torch.Generator(device=plant.device).manual_seed(0)
        cand = (torch.rand((h, p_n * c, model.n_act), device=plant.device, generator=gen) * 2 - 1).contiguous()
        rew = torch.empty((h, p_n * c), dtype=model.dtype, device=plant.device)
        ridx = torch.arange(p_n, device=plant.device, dtype=torch.int32).repeat_interleave(c)
        base = torch.arange(p_n, device=plant.device) * c
        kw = dict(params=True) if arm == "params_randomised" else {}
        kr = dict(params="source") if arm == "params_randomised" else {}

        def control_step():
            model.restore(plant.snapshot(rng=True, **kw), rows=ridx, rng="source", **kr)
            model.rollout_into(cand, h, 1, None, None, rew, None)
            plant.step(cand[0].index_select(0, rew.sum(0).view(p_n, c).argmax(1) + base))

        ms = timed(control_step, args.reps)
        out[f"ms_{arm}"] = round(ms, 4)
        out[f"env_steps_per_s_{arm}"] = round(p_n * c * h / ms * 1e3, 1)
        del plant, model, cand, rew
        torch.cuda.empty_cache()
    out["params_over_identity_only"] = round(out["ms_params_randomised"] / out["ms_identity_only"], 3)
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--plants", type=int, default=1024)
    ap.add_argument("--horizon", type=int, default=8)
    ap.add_argument("--rng", choices=("own", "source"), default="own")
    ap.add_argument("--params", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    if args.params:
        name, plimit = gpu_info()
        print(f"GPU: {name}, power limit {plimit}")
        params_main(args)
        return
    ids = args.rng == "source"
    name, plimit = gpu_info()
    print(f"GPU: {name}, power limit {plimit}")
    n = args.envs
    sim = sim_of(n)
    sim.reset()
    words, _ = sim.record_layout()
    rec_bytes = 4 * words
    mode = "source" if ids else "own"
    id_bytes = 4 * 8 if ids else 0  # GEMB200_RNG_ID_WORDS words per env: identity array and identity rows
    snap = sim.snapshot(rng=ids)
    torch.cuda.synchronize()

    ms = timed(lambda: sim.snapshot(rng=ids), args.reps)
    moved = 2 * (rec_bytes + id_bytes) * n  # state (and identities) read + rows written
    print(json.dumps(dict(what="pack", rng=mode, envs=n, words=words, ms=round(ms, 4), bytes=moved, tb_s=round(moved / ms / 1e9, 3),
                          frac_datasheet=round(moved / ms / 1e-3 / PEAK, 3))))
    ms = timed(lambda: sim.restore(snap, rng=mode), args.reps)
    print(json.dumps(dict(what="unpack", rng=mode, envs=n, words=words, ms=round(ms, 4), bytes=moved, tb_s=round(moved / ms / 1e9, 3),
                          frac_datasheet=round(moved / ms / 1e-3 / PEAK, 3))))

    m = 1024
    few = snap[:m]
    ridx = torch.arange(m, device=sim.device, dtype=torch.int32).repeat_interleave(n // m)
    ms = timed(lambda: sim.restore(few, rows=ridx, rng=mode), args.reps)
    # state written + row index read + the (L2-resident) rows once; with identities the own identity written by the unpack, then the
    # adopted one (index read again)
    moved_f = (rec_bytes + 4) * n + rec_bytes * m + ((2 * id_bytes + 4) * n + id_bytes * m if ids else 0)
    print(json.dumps(dict(what="fan_out_unpack", rng=mode, rows=m, envs=n, ms=round(ms, 4), bytes=moved_f, tb_s=round(moved_f / ms / 1e9, 3),
                          frac_datasheet=round(moved_f / ms / 1e-3 / PEAK, 3))))
    del sim, snap, few

    # random-shooting MPC: P plants x C candidates x horizon H
    p_n, h = args.plants, args.horizon
    c = n // p_n
    plant, model = sim_of(p_n, seed=1), sim_of(p_n * c, seed=2)
    plant.reset()
    model.reset()
    gen = torch.Generator(device=plant.device).manual_seed(0)
    cand = (torch.rand((h, p_n * c, model.n_act), device=plant.device, generator=gen) * 2 - 1).contiguous()
    rew = torch.empty((h, p_n * c), dtype=model.dtype, device=plant.device)
    ridx = torch.arange(p_n, device=plant.device, dtype=torch.int32).repeat_interleave(c)
    base = torch.arange(p_n, device=plant.device) * c
    marks = []

    def control_step(record=False):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(6)] if record else None
        if record:
            e[0].record()
        s = plant.snapshot(rng=ids)
        if record:
            e[1].record()
        model.restore(s, rows=ridx, rng=mode)
        if record:
            e[2].record()
        model.rollout_into(cand, h, 1, None, None, rew, None)
        if record:
            e[3].record()
        best = rew.sum(0).view(p_n, c).argmax(1) + base
        act = cand[0].index_select(0, best)
        if record:
            e[4].record()
        plant.step(act)
        if record:
            e[5].record()
            marks.append(e)

    if ids:  # common random numbers: the candidates of a plant see one reference trajectory until they terminate
        model.restore(plant.snapshot(rng=True), rows=ridx, rng="source")
        _, ref, _, term = model.rollout(cand, record_every=1)
        ref, term = ref.view(h, p_n, c, -1), term.view(h, p_n, c).bool()
        alive = term.int().cumsum(0) == 0  # no termination up to and including this step (a terminating step records the ref after its reset)
        alive = alive & alive[:, :, :1]
        same = (ref == ref[:, :, :1]).all(-1) | ~alive
        if not bool(same.all()):
            raise SystemExit("candidates of one plant recorded different reference trajectories with rng=source")
        print(json.dumps(dict(what="common_reference_check", plants=p_n, candidates=c, horizon=h, compared_steps=int(alive.sum()), ok=True)))

    for _ in range(3):
        control_step()
    torch.cuda.synchronize()
    for _ in range(args.reps):
        control_step(record=True)
    torch.cuda.synchronize()
    split = {}
    for k, lab in enumerate(["pack", "fan_out", "rollout", "select", "plant_step"]):
        v = sorted(e[k].elapsed_time(e[k + 1]) for e in marks)
        split[lab] = round(v[len(v) // 2], 4)
    tot = sorted(e[0].elapsed_time(e[5]) for e in marks)
    tot_ms = tot[len(tot) // 2]
    print(json.dumps(dict(what="mpc_control_step", rng=mode, plants=p_n, candidates=c, horizon=h, ms=round(tot_ms, 4), control_steps_per_s=round(1e3 / tot_ms, 1),
                          env_steps_per_s=round(p_n * c * h / tot_ms * 1e3, 1), split_ms=split)))
    del plant, model, cand, rew
    if ids:
        torch.cuda.empty_cache()
        print(json.dumps(rollout_arms(n, 32, args.reps)))


def rollout_arms(n, steps, reps):
    """us per env step of a recorded rollout: shared coefficients / per-env blocks of the shared parameters / the same with identities"""
    arms = {a: sim_of(n, seed=3) for a in ("shared", "envp", "envp_ids")}
    cfg = arms["envp"].cfg
    mp = np.tile(np.array(list(cfg.motor_param)), (n, 1))
    lp = np.tile(np.array(list(cfg.load_param)), (n, 1))
    arms["envp"].set_env_params(mp, lp)
    for s in arms.values():
        s.reset()
    s = arms["envp_ids"]  # every env adopts the identity of another env of the handle (a rotation): all of them read an identity row
    s.restore(s.snapshot(rng=True), rows=torch.roll(torch.arange(n, device=s.device, dtype=torch.int32), 1), rng="source")
    acts = (torch.rand((steps, n, s.n_act), device=s.device, generator=torch.Generator(device=s.device).manual_seed(0)) * 2 - 1).contiguous()
    for _ in range(3):
        for s in arms.values():
            s.rollout(acts, record_every=1)
    torch.cuda.synchronize()
    ev = {a: [] for a in arms}
    for _ in range(reps):
        for a, s in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            s.rollout(acts, record_every=1)
            e1.record()
            ev[a].append((e0, e1))
    torch.cuda.synchronize()
    out = dict(what="identity_rollout", env="Cont-CC-PMSM-v0", envs=n, steps=steps, reps=reps, dtype="float32", layout="aos")
    for a in arms:
        ms = sorted(x.elapsed_time(y) for x, y in ev[a])
        out[f"us_per_step_{a}"] = round(ms[len(ms) // 2] * 1e3 / steps, 3)
    out["envp_ids_over_envp"] = round(out["us_per_step_envp_ids"] / out["us_per_step_envp"], 4)
    return out


if __name__ == "__main__":
    main()
