"""Parameter sensitivities on the device (`rollout_param_sens`) against central differences of the float64 oracle.

The device runs one K-step launch from a common x0 and records S after every step.  Every perturbed copy theta_j (1 +- h) is its own oracle
instance with the device's configuration (the one parameter changed), seed and env_index_offset, driven from the same x0 with the same
actions; its ODE state is read after every step.  The oracle is an independent float64 implementation of the reference's models, so the
check does not rest on the device's own primal step.  Per case:
  * the primal: the device's state after K steps must be the unperturbed oracle's (1e-9 of the row scale);
  * every entry of S[k] must match the oracle's central differences within 1e-6 of its column's scale plus the row's own rounding floor
    64 eps (|x_r| + 1) / h; stencils whose forward and backward differences disagree (a kink crossed between the copies) are counted, <= 1 %;
  * a parameter that does not enter the model (the mechanical ones under a constant-speed load) gives exact 0 on both sides."""
import numpy as np
import pytest

from fd_helpers import SLOT, _oracle_states, _wrap, build_up_flux, sens_check
from gpu_helpers import torch_cuda  # noqa: F401
from gym_electric_motor_b200 import _cabi as K

pytestmark = pytest.mark.gpu

OFFSET = 7000  # global index of env 0, on the device and in every oracle copy
TOL = 1e-6
REL_H = 1e-4  # truncation of the K = 8 differences stays below 1e-7 of the column scale; the rounding floor is 10x lower than at 1e-5
MOTORS = {
    "pmsm": ("Cont-CC-PMSM-v0", ["r_s", "l_d", "l_q", "psi_p", "j_rotor", "a", "b", "c", "j_load"]),
    "scim": ("Cont-CC-SCIM-v0", ["r_s", "r_r", "l_m", "l_sigs", "l_sigr", "j_rotor", "b", "c", "j_load"]),
    "dfim": ("Cont-CC-DFIM-v0", ["r_s", "r_r", "l_m", "l_sigs", "l_sigr", "j_rotor", "b", "c"]),
    "eesm": ("Cont-CC-EESM-v0", ["r_s", "l_d", "l_q", "r_e", "l_m", "l_e", "j_rotor", "b", "c"]),
    "extex": ("Cont-CC-ExtExDc-v0", ["r_a", "l_a", "r_e", "l_e", "l_e_prime", "j_rotor", "a", "b", "c", "j_load"]),
}
MECH = ("j_rotor", "a", "b", "c", "j_load")
_KEEP = []


def _config(env_id, m, load):
    import gym_electric_motor_b200 as gem

    env = gem.make(env_id, num_envs=m, dtype="float64", autoreset="none", seed=13, env_index_offset=OFFSET)
    _KEEP.append(env)
    cfg = env.build_config()
    cfg.dtype = K.F64
    if load == "poly":
        cfg.load_kind = K.LOAD_POLY_STATIC
        cfg.load_param[K.LP_A], cfg.load_param[K.LP_B], cfg.load_param[K.LP_C] = 0.01, 0.02, 1e-4
        cfg.load_param[K.LP_J_LOAD] = 1e-3
    else:
        cfg.load_kind = K.LOAD_CONST_SPEED
    return cfg


@pytest.mark.parametrize("load", ["poly", "const"])
@pytest.mark.parametrize("motor", list(MOTORS))
def test_against_central_differences_of_the_oracle(torch_cuda, motor, load):
    from gym_electric_motor_b200.vector_sim import VectorSim

    torch = torch_cuda
    env_id, names = MOTORS[motor]
    m, k = 12, 8
    cfg = _config(env_id, m, load)
    slots = [SLOT[nm] for nm in names]
    sim = VectorSim(cfg)
    sim.reset()
    rng = np.random.default_rng(3)
    x0 = sim.get_ode_state().cpu().numpy()
    x0[:, 0] = np.linspace(-150, 150, m)  # running speeds of both signs, outside the static-friction band
    has_eps = cfg.motor_kind >= K.MOTOR_PMSM
    build_up_flux(rng, cfg, x0)
    if has_eps:
        x0[:, -1] = rng.uniform(-2.5, 2.5, m)
    sim.set_ode_state(x0)
    a = rng.uniform(-0.9, 0.9, (k, m, sim.n_act))
    acts = torch.as_tensor(a, dtype=torch.float64, device="cuda").contiguous()
    (so, _), _ = sim.rollout_param_sens(acts, slots)
    s = so.cpu().numpy()  # [K, m, n_x, n_p]
    x_dev = sim.get_ode_state().cpu().numpy()

    mid = _oracle_states(cfg, x0, a)
    d = x_dev - mid[-1]
    if has_eps:
        d[:, -1] = _wrap(d[:, -1])
    assert np.all(np.abs(d) <= 1e-9 * (np.abs(mid[-1]).max(axis=0) + 1)), (motor, load, "primal", np.abs(d).max())

    row = np.array(list(cfg.motor_param) + list(cfg.load_param))
    kinks = total = 0
    for j, (nm, slot) in enumerate(zip(names, slots)):
        h = REL_H * (abs(row[slot]) if row[slot] != 0 else 1.0)
        side = []
        for sign in (1.0, -1.0):
            c = type(cfg).from_buffer_copy(cfg)
            if slot < K.MAX_MOTOR_PARAM:
                c.motor_param[slot] = row[slot] + sign * h
            else:
                c.load_param[slot - K.MAX_MOTOR_PARAM] = row[slot] + sign * h
            side.append(_oracle_states(c, x0, a))
        dup, ddn = side[0] - mid, mid - side[1]
        if has_eps:
            dup[..., -1], ddn[..., -1] = _wrap(dup[..., -1]), _wrap(ddn[..., -1])
        fd, scale, err, kink, bad = sens_check(s[..., j], dup, ddn, mid, h, TOL)  # [K, m, n_x]
        if load == "const" and nm in MECH:
            assert np.all(s[..., j] == 0) and np.all(fd == 0), (motor, nm, "a parameter that does not enter: exact 0")
            continue
        assert scale.max() > 0, (motor, nm, "the parameter moves the trajectory")
        kinks += int(kink.sum())
        total += kink.size
        worst = (err / np.maximum(scale, 1e-300)).max(axis=2)
        assert not bad.any(), (motor, load, nm, worst[bad].max())
        print(f"{motor}-{load} {nm}: worst {worst[~kink].max():.2e} of the column scale")
    assert kinks <= 0.01 * max(total, 1), (motor, load, kinks, total)
