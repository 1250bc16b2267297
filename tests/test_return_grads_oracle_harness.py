"""The oracle central-difference harness of fd_helpers.py (used by test_gpu_return_grads_oracle.py) against a closed form, without a GPU.

PMSM at constant speed, RK4 with one step per tau, continuous B6 bridge with actions inside the clip range, constant references on i_sd and
i_sq and reward exponent 2, no constraint hit: the step is affine in (x, a),
    i_k+1 = Phi i_k + Gamma (B(eps_k) a_k + e),   eps_k+1 = eps_k + p omega tau,
with Phi, Gamma the RK4 step maps of the dq current dynamics and B(eps) = diag(1/l_d, 1/l_q) rot(-eps) T23 u_sup / 2 (the matrices
test_known_answer_linear_current_dynamics builds), and the return sum gamma^k r(i_k+1) is quadratic.  Its gradient with respect to the
initial currents and every action follows from those matrices; the harness's oracle central differences must match it."""
import math

import numpy as np

from fd_helpers import oracle_fd
from gym_electric_motor_b200 import _cabi as K


def _config(m):
    import gym_electric_motor_b200 as gem

    cfg = gem.make("Cont-CC-PMSM-v0", num_envs=m, dtype="float64", autoreset="none", seed=3).build_config()
    cfg.dtype, cfg.load_kind, cfg.solver_kind, cfg.solver_nsteps = K.F64, K.LOAD_CONST_SPEED, K.SOLVER_RK4, 1
    for r, v in enumerate((0.3, -0.2)):
        cfg.ref_kind[r], cfg.ref_value[r] = K.REF_CONST, v
    for j in range(K.MAX_STATE):
        cfg.reward_power[j] = 2.0
    return cfg


def test_harness_central_differences_match_the_closed_form(oracle_lib):
    m, k_steps, gamma = 6, 4, 0.9
    cfg = _config(m)
    ora = oracle_lib.Oracle(cfg)
    _, ref0 = ora.reset()
    assert ora.n_ref == 2 and list(cfg.ref_state[:2]) == [5, 6]
    rng = np.random.default_rng(0)
    warm = rng.uniform(-0.3, 0.3, (2, m, 3))
    x0 = np.zeros((m, 4))
    x0[:, 0] = rng.uniform(-300, 300, m)
    x0[:, 1:3] = rng.uniform(-0.3, 0.3, (m, 2)) * np.array([cfg.limits[5], cfg.limits[6]])
    x0[:, 3] = rng.uniform(-2.5, 2.5, m)
    acts = rng.uniform(-0.6, 0.6, (k_steps, m, 3))
    fd = oracle_fd(lambda: [(oracle_lib.Oracle(cfg), slice(None))], warm, x0, acts, gamma, ref0=ref0, angle=True)
    assert (fd["end"] == k_steps).all()

    mp = cfg.motor_param
    p, r, ld, lq, psi = mp[K.MP_P], mp[K.MP_R_S], mp[K.MP_L_D], mp[K.MP_L_Q], mp[K.MP_PSI_P]
    h = cfg.tau
    t23 = np.array([[2 / 3, -1 / 3, -1 / 3], [0.0, 1 / np.sqrt(3), -1 / np.sqrt(3)]])
    lim, ln, wt = np.array([cfg.limits[5], cfg.limits[6]]), np.array([cfg.state_length[5], cfg.state_length[6]]), np.array([cfg.reward_weight[5], cfg.reward_weight[6]])
    ncol = 4 + k_steps * 3
    worst = 0.0
    for i in range(m):
        w = x0[i, 0]
        mm = np.array([[-r / ld, p * w * lq / ld], [-p * w * ld / lq, -r / lq]])
        phi = sum(np.linalg.matrix_power(h * mm, j) / math.factorial(j) for j in range(5))
        gam = sum(h ** j * np.linalg.matrix_power(mm, j - 1) / math.factorial(j) for j in range(1, 5))
        e = np.array([0.0, -p * w * psi / lq])
        z, zs, bs, ret = x0[i, 1:3].copy(), [], [], 0.0
        for k in range(k_steps):
            eps = x0[i, 3] + k * p * w * h
            c, s = np.cos(eps), np.sin(eps)
            b = np.diag([1 / ld, 1 / lq]) @ np.array([[c, s], [-s, c]]) @ t23 * (0.5 * cfg.u_sup)
            z = phi @ z + gam @ (b @ acts[k, i] + e)
            zs.append(z)
            bs.append(b)
            ret += gamma ** k * (cfg.reward_bias - (wt * ((z / lim - ref0[i]) / ln) ** 2).sum())
        # the primal: the affine recursion is the oracle's trajectory
        assert abs(ret - fd["ret"][i]) <= 1e-10 * max(1.0, abs(ret)), (i, ret, fd["ret"][i])
        assert np.abs(zs[-1] - fd["xk"][i, 1:3]).max() <= 1e-10 * np.abs(lim).max()
        dr = [-2 * wt * (zk / lim - ref0[i]) / (ln * ln * lim) for zk in zs]  # d r_k / d i_k+1
        g = np.full(ncol, np.nan)  # the omega and angle columns are not affine: left out
        g[1:3] = sum(gamma ** k * np.linalg.matrix_power(phi, k + 1).T @ dr[k] for k in range(k_steps))
        for j in range(k_steps):
            g[4 + 3 * j: 7 + 3 * j] = sum(gamma ** k * (np.linalg.matrix_power(phi, k - j) @ gam @ bs[j]).T @ dr[k] for k in range(j, k_steps))
        cd = (fd["plus"][i] - fd["minus"][i]) / (2 * fd["h"])
        cols = ~np.isnan(g)
        scale = np.abs(g[cols]).max()
        assert scale > 0
        worst = max(worst, np.abs(cd[cols] - g[cols]).max() / scale)
    print(f"harness vs closed form: worst {worst:.2e}")
    assert worst < 1e-7, worst
