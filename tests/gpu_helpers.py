"""Device-side test helpers: the `torch_cuda` fixture, env makers and action generators, the equality checks of the twin-handle tests,
the stepping modes of the replay tests and the kernel-name parser of the launch-mode tests.

Test modules import the fixture by name (`from gpu_helpers import torch_cuda  # noqa: F401`) so that pytest finds it there."""
import re

import numpy as np
import pytest

from helpers import _mk, _random_actions, load_golden, switched_config
from gym_electric_motor_b200 import _cabi as K


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    return torch


# ------------------------------------------------------------------------------------------------------------ launch shapes
def launch_block(n, sms):
    """threads per block of a step / rollout launch over n envs on a device with `sms` SMs: pick_block in csrc/gemb200_launch.cuh (128,
    halved while the grid would have fewer than 8 blocks per SM, down to 32)"""
    block = 128
    while block > 32 and (n + block - 1) // block < sms * 8:
        block //= 2
    return block


def launch_sizes():
    """the batch sizes of the launch-shape tests, from the SM count S of cuda:0 (S = 132 on an H100 SXM: 67 617, 135 205, 67 584, 405 581):
    N64 = 512 S + 33 launches 64-thread blocks, the last one a full warp and a warp with 1 env; N128 = 1024 S + 37 launches 128-thread
    blocks, the last one a full warp, a warp with 5 envs and two empty warps; PF = 512 S is the step kernel's L2 prefetch distance (both
    sizes exceed it); NHOST = 3072 S + 77: the pipelined host step's chunks launch 64 threads, a full-batch device step 128"""
    import torch

    s = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = dict(S=s, N64=512 * s + 33, N128=1024 * s + 37, PF=512 * s, NHOST=3072 * s + 77)
    assert (launch_block(N, s), launch_block(sizes["N64"], s), launch_block(sizes["N128"], s), launch_block(sizes["NHOST"], s)) == (32, 64, 128, 128)
    return sizes


# ------------------------------------------------------------------------------------------------------------ env makers and actions
N = 300  # not a multiple of 128: the last block and its last warp are partly inactive

ENV_IDS = {"permex": "Cont-CC-PermExDc-v0", "extex": "Cont-CC-ExtExDc-v0", "pmsm": "Cont-CC-PMSM-v0", "eesm": "Cont-CC-EESM-v0",
           "scim": "Cont-CC-SCIM-v0", "dfim": "Cont-CC-DFIM-v0", "pmsm_finite": "Finite-CC-PMSM-v0"}


def _make(family, dtype="float32", layout="aos", autoreset="same_step", seed=7, n=N, **kw):
    import gym_electric_motor_b200 as gem

    env = gem.make(ENV_IDS[family], num_envs=n, device="cuda", dtype=dtype, layout=layout, autoreset=autoreset, seed=seed, **kw)
    env.reset()
    return env


def _ext_env(layout="aos", dtype="float32", n=N):
    from gym_electric_motor_b200.reference_generators import ExternalReferenceGenerator as Ext, MultipleReferenceGenerator

    return _make("pmsm", dtype, layout, n=n, reference_generator=MultipleReferenceGenerator([Ext("i_sd"), Ext("i_sq")]))


def _actions(torch, env, k, seed=0):
    """saturating actions with a per-env magnitude, constant in sign for stretches of 6 steps: currents leave their limits after a number
    of steps that differs from env to env.  Finite B6: one active voltage vector per env, after a stretch of zero voltage of its own
    length."""
    sim = env.sim
    rng = np.random.default_rng(seed)
    lead = (k,) + sim._shape(sim.n_act)
    if sim.finite:  # the zero vector (0) for each env's first 0 .. 8 steps staggers the steps at which the currents trip
        a = np.array(np.broadcast_to(rng.integers(1, 7, size=lead[1:]), lead))
        start = rng.integers(0, 9, size=lead[1:])
        a[np.arange(k).reshape((k,) + (1,) * (len(lead) - 1)) < start] = 0
        return torch.as_tensor(a, dtype=torch.int32, device="cuda").contiguous()
    mag = rng.uniform(0.3, 1.0, size=(1,) + lead[1:])
    a = np.repeat(rng.choice([-1.0, 1.0], size=((k + 5) // 6,) + lead[1:]), 6, axis=0)[:k] * mag
    return torch.as_tensor(a, dtype=sim.dtype, device="cuda").contiguous()


def _dev_actions(torch, sim, acts):
    """[K, N, n_act] numpy -> device tensor in the sim's layout and action dtype"""
    a = np.asarray(acts).reshape(acts.shape[0], sim.n, sim.n_act)
    if sim.soa:
        a = np.ascontiguousarray(a.transpose(0, 2, 1))
    return torch.as_tensor(a, device=sim.device).to(sim.act_dtype).contiguous()


# ------------------------------------------------------------------------------------------------------------ equality checks
def _bits(torch, x):
    """bit pattern of a tensor (NaN-safe equality)"""
    if x.dtype == torch.float32:
        return x.contiguous().view(torch.int32)
    if x.dtype == torch.float64:
        return x.contiguous().view(torch.int64)
    return x.contiguous().view(torch.uint8) if x.dtype == torch.bool else x


def _eq(torch, a, b, what):
    """bit equality"""
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    assert torch.equal(_bits(torch, a), _bits(torch, b)), (what, (a.double() - b.double()).abs().nan_to_num(1e300).max().item())


def _same(torch, a, b, what):
    """equal values (NaN equals NaN).  For the outputs of A's PLAIN kernel against B's general one: the instantiations agree value for
    value but may differ in the sign of a zero (the equality the other rollout tests check with torch.equal)"""
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    ok = (a == b) | (torch.isnan(a) & torch.isnan(b)) if a.is_floating_point() else a == b
    assert bool(ok.all()), (what, (a.double() - b.double()).abs().nan_to_num(1e300).max().item())


def _same_outputs(torch, out_a, out_b, what):
    """torch.equal of every (obs, ref, reward, terminated) of two lists of per-step outputs (`_run`)"""
    for k, (oa, ob) in enumerate(zip(out_a, out_b)):
        for q, nm in enumerate(("obs", "ref", "reward", "terminated")):
            assert torch.equal(oa[q], ob[q]), (what, nm, k)


def _blob(env):
    return env.sim.state_dict()["blob"]


def _next_steps(torch, a_env, b_env, n=3, seed=99):
    """the outputs of a few more steps on both handles: the same persistent state where no checkpoint can tell"""
    acts = _actions(torch, a_env, n, seed=seed)
    for j in range(n):
        (o1, r1), w1, t1, _, _ = a_env.step(acts[j])
        (o2, r2), w2, t2, _, _ = b_env.step(acts[j])
        for name, x, y in (("obs", o1, o2), ("ref", r1, r2), ("reward", w1, w2), ("terminated", t1, t2)):
            _same(torch, y, x, ("next step", j, name))


# ------------------------------------------------------------------------------------------------------------ replays with random parts
DEAD3 = "pmsm_cc_rk4_dead3"
SWITCHED = "switched_periodic"
SCIM_RANDOM = "scim_random_init"


def _randomise(g, cfg):
    """random initial states on omega and the first currents (induction motors: their flux limits come from the env's initializer, see
    SCIM_RANDOM), and normal state noise on the first two states"""
    init = [cfg.init_ode[j] for j in range(8)]
    lim = np.array(g["meta"]["limits"])
    n_ode = len(g["reset_ode"])
    if cfg.motor_kind not in (K.MOTOR_SCIM, K.MOTOR_DFIM):
        cfg.init_random = 1
        for j in range(n_ode):
            span = (0.2 * lim[0] if j == 0 else 0.3 * lim[2]) if j < 3 else 0.0
            cfg.init_lo[j], cfg.init_hi[j] = init[j] - span, init[j] + span
    if cfg.n_state_ops < K.MAX_STATE_OPS:
        k = cfg.n_state_ops
        cfg.n_state_ops = k + 1
        cfg.sop_kind[k], cfg.sop_idx[k][0], cfg.sop_mask[k] = K.SOP_NOISE, K.NOISE_NORMAL, 0b11
        cfg.sop_param[k][0], cfg.sop_param[k][1] = 0.0, 0.01


def _random_cfg(name, n, dtype, seed=77, offset=12345):
    """(golden or None, config) of a case with its random parts on"""
    if name == SWITCHED:
        kinds = [dict(kind=K.REF_WIENER, margin=(-0.5, 0.5), length=(2, 6)), dict(kind=K.REF_SINUS, length=(2, 6)),
                 dict(kind=K.REF_STEP, amp=(0.05, 0.2), length=(2, 6)), dict(kind=K.REF_TRIANGULAR, length=(3, 7))]
        cfg = switched_config(n, kinds, [0.25] * 4, (5, 12), seed=seed, dtype=dtype)
        cfg.env_index_offset = offset
        return load_golden("permex_sc_euler3"), cfg
    if name == SCIM_RANDOM:
        import gym_electric_motor_b200 as gem

        cfg = gem.make("Cont-CC-SCIM-v0", num_envs=n, motor=dict(motor_initializer=dict(random_init="uniform"))).build_config()
        assert cfg.init_im_valid == 1
        cfg.dtype, cfg.seed, cfg.env_index_offset = dtype, seed, offset
        return None, cfg
    g, cfg = _mk(name.replace("_dead3", ""), n, dtype, K.LAYOUT_AOS)
    if name == DEAD3:
        cfg.dead_time_steps = 3
    _randomise(g, cfg)  # (_mk already leaves the AC supply's phase random)
    cfg.seed, cfg.env_index_offset = seed, offset
    return g, cfg


def _acts(rng, g, sim, steps):
    if g is None:
        return rng.uniform(-1, 1, size=(steps, sim.n, sim.n_act))
    return _random_actions(rng, g, sim.n, steps)


def _run(torch, sim, acts, mode, idx):
    """outputs of envs idx over len(acts) steps: eager steps, one recorded rollout, or steps captured in a CUDA graph (device clock)"""
    k = acts.shape[0]
    if mode == "rollout":
        o = sim.rollout(acts, record_every=1)
        return [tuple(t[j][idx].clone() for t in o) for j in range(k)]
    if mode == "graph":
        sim.set_device_clock(True)
        torch.cuda.synchronize()
        graph, rec = torch.cuda.CUDAGraph(), []
        with torch.cuda.graph(graph):
            for j in range(k):
                rec.append(tuple(t.clone() for t in sim.step(acts[j])))
        graph.replay()
        torch.cuda.synchronize()
        return [tuple(t[idx] for t in r) for r in rec]
    return [tuple(t[idx].clone() for t in sim.step(acts[j])) for j in range(k)]


_MOTOR_SLOTS = {  # parameters drawn per reset, +-20 % around the configuration's value (induction motors: no flux-limit slots with random init)
    K.MOTOR_PMSM: (K.MP_R_S, K.MP_L_D, K.MP_L_Q, K.MP_PSI_P, K.MP_J_ROTOR),
    K.MOTOR_EESM: (K.MP_R_S, K.MP_L_D, K.MP_L_Q, K.MP_R_E, K.MP_J_ROTOR),
    K.MOTOR_PERMEX_DC: (K.MP_R_A, K.MP_L_A, K.MP_PSI_E, K.MP_J_ROTOR),
    K.MOTOR_EXTEX_DC: (K.MP_R_A, K.MP_L_A, K.MP_R_E, K.MP_L_E, K.MP_J_ROTOR),
    K.MOTOR_SCIM: (K.MP_J_ROTOR,),
    K.MOTOR_DFIM: (K.MP_R_S, K.MP_L_M, K.MP_J_ROTOR),
}


def _draws(cfg):
    slots = [s for s in _MOTOR_SLOTS[cfg.motor_kind] if cfg.motor_param[s] > 0]
    return (slots, [K.DIST_UNIFORM] * len(slots), [0.8 * cfg.motor_param[s] for s in slots], [1.2 * cfg.motor_param[s] for s in slots])


# ------------------------------------------------------------------------------------------------------------ launch modes
# tangent kernel -> index of the template argument that selects its per-env (ENVP) variant; step_kernel and rollout_kernel: PLAIN is the
# 6th and ENVP the 8th
_TANGENT_ENVP_ARG = {"jacobian_kernel": 4, "param_sens_kernel": 4, "return_grad_kernel": 3}


def _mode(name):
    """(kernel, mode) of a step, rollout, Jacobian, parameter-sensitivity or return-gradient kernel name, or None for any other kernel"""
    m = re.search(r"(return_grad_kernel|param_sens_kernel|jacobian_kernel|step_kernel|rollout_kernel)<([^>]*)>", name)
    if not m:
        return None
    kernel = m.group(1)
    on = [a.strip() in ("true", "(bool)1", "1") for a in m.group(2).split(",")]
    if kernel in ("step_kernel", "rollout_kernel"):
        return kernel, "PLAIN" if on[5] else ("ENVP" if on[7] else "general")
    return kernel, "ENVP" if on[_TANGENT_ENVP_ARG[kernel]] else "shared"


def _kernels(torch, fn):
    """(kernel, mode) of every step, rollout, Jacobian, parameter-sensitivity and return-gradient kernel that fn() launches, in launch
    order, read from the kernel names torch.profiler records.  Step and rollout kernels: "PLAIN", "ENVP" or "general"; the tangent
    kernels: "ENVP" or "shared"."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [km for km in (_mode(e.name) for e in prof.events()) if km]


def _launches(torch, fn, tmp_path):
    """(kernel, mode, threads per block, blocks) of every kernel of `_kernels` that fn() launches, in launch order, read from the "block" and
    "grid" fields of the kernel events in the exported profiler trace"""
    import json

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = tmp_path / "trace.json"
    prof.export_chrome_trace(str(path))
    out = []
    for e in sorted(json.loads(path.read_text())["traceEvents"], key=lambda e: e.get("ts", 0)):
        km = _mode(e.get("name", "")) if e.get("cat") == "kernel" else None
        if km:
            args = e.get("args", {})
            assert "block" in args and "grid" in args, ("the trace has no launch shape for", e["name"][:80], sorted(args))
            out.append(km + (int(args["block"][0]), int(args["grid"][0])))
    return out
