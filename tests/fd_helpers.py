"""Central-difference test helpers: the configurations, base points and +-h stencils of the Jacobian, return-gradient and
parameter-sensitivity tests, the stencil rules those tests share, and the float64 oracle runs they difference."""
import numpy as np

from gym_electric_motor_b200 import _cabi as K
from gym_electric_motor_b200.core import ElectricMotorEnvironment

# parameter name -> slot in the row of motor parameters followed by load parameters
SLOT = {**{nm: s for nm, s in ElectricMotorEnvironment._MP_SLOT.items()},
        **{nm: K.MAX_MOTOR_PARAM + s for nm, s in ElectricMotorEnvironment._LP_SLOT.items()}}
# switching states per converter kind: a finite action of a slot is drawn in 0 .. N_SWITCH - 1
N_SWITCH = {K.CONV_B6: 8, K.CONV_4QC: 4, K.CONV_2QC: 3, K.CONV_1QC: 2, K.CONV_NONE: 1}
_KEEP = []


def _wrap(d):
    return (d + np.pi) % (2 * np.pi) - np.pi


def _profile(t, amplitude, frequency):
    return amplitude * np.sin(2 * np.pi * frequency * t)


def _cfg(env_id, n, dtype, solver=K.SOLVER_RK4, nsteps=1, load=None, supply=None, action_dq=0, til=None, til1=None, autoreset="none"):
    import gym_electric_motor_b200 as gem

    kw = {}
    if load == "ext":  # a speed profile the load follows with its time constant (ExternalSpeedLoad)
        kw["load"] = gem.physical_systems.ExternalSpeedLoad(speed_profile=_profile, speed_profile_kwargs=dict(amplitude=120.0, frequency=7.0),
                                                          tau=1e-4, horizon_steps=2000)
    env = gem.make(env_id, num_envs=n, dtype=dtype, autoreset=autoreset, seed=11, **kw)
    _KEEP.append(env)  # the config points into the load's speed table, which the env owns
    cfg = env.build_config()
    cfg.solver_kind, cfg.solver_nsteps = solver, nsteps
    if load == "const":
        cfg.load_kind = K.LOAD_CONST_SPEED
    elif load == "poly":
        cfg.load_kind = K.LOAD_POLY_STATIC
        cfg.load_param[K.LP_A], cfg.load_param[K.LP_B], cfg.load_param[K.LP_C] = 0.01, 0.02, 1e-4
        cfg.load_param[K.LP_J_LOAD] = 1e-3
    if supply == "ac1":
        cfg.supply_kind, cfg.supply_param[0], cfg.supply_param[1], cfg.supply_param[2] = K.SUPPLY_AC1, 50.0, 0.3, 1.0
    if action_dq:
        cfg.action_dq = action_dq
    if til is not None:
        cfg.interlocking_time = til
    if til1 is not None:
        cfg.interlocking_time1 = til1
    return cfg


# ------------------------------------------------------------------------------------------------------------------ base points
# Each helper edits x0 [m, n_x] in place and draws from rng only where it applies, so callers keep their own order of draws.
def clip_angle(cfg, x0):
    """the angle kept away from the wrap at +-pi"""
    if cfg.motor_kind >= K.MOTOR_PMSM:
        x0[:, -1] = np.clip(x0[:, -1], -2.5, 2.5)


def build_up_flux(rng, cfg, x0):
    """induction motors: a built-up rotor flux, so that the field frame is defined (near zero the field angle turns with any
    perturbation)"""
    if cfg.motor_kind in (K.MOTOR_SCIM, K.MOTOR_DFIM):
        m = x0.shape[0]
        mag, ang = rng.uniform(0.2, 0.8, m), rng.uniform(-np.pi, np.pi, m)
        x0[:, 3], x0[:, 4] = mag * np.cos(ang), mag * np.sin(ang)


def currents_off_zero(rng, cfg, x0):
    """finite converters: no current exactly at 0, where a leg waiting in its interlock state switches its voltage with the current's
    sign"""
    if cfg.finite:
        cur = slice(1, 3 if cfg.motor_kind >= K.MOTOR_PMSM else x0.shape[1])
        x0[:, cur] += rng.choice([-1.0, 1.0], x0[:, cur].shape) * rng.uniform(0.5, 2.0, x0[:, cur].shape)


def switching_states(rng, cfg, shape):
    """finite actions [..., n_act]: a switching state per converter slot, within the slot's range"""
    hi = np.array([N_SWITCH[cfg.converter_kind[j]] for j in range(shape[-1])])
    return rng.integers(0, hi, shape)


# ------------------------------------------------------------------------------------------------------------------ +-h stencils
def fd_steps(x0, ncol):
    """the step h of every column of (x0, a_0 .. a_K-1): 1e-6 times a state column's largest magnitude (at least 1), 1e-6 for actions"""
    nx = x0.shape[1]
    return np.array([1e-6 * max(1.0, float(np.abs(x0[:, c]).max())) if c < nx else 1e-6 for c in range(ncol)])


def shift(xs, acts, c, dh, rows=slice(None)):
    """adds dh to column c of (x0, a_0 .. a_K-1) in the env rows `rows` of xs [envs, n_x] and acts [K, envs, n_u]"""
    nx = xs.shape[1]
    if c < nx:
        xs[rows, c] += dh
    else:
        kk, u = divmod(c - nx, acts.shape[2])
        acts[kk, rows, u] += dh


def stencil(x0, acts, nu):
    """every base env repeated reps = 2 n_col + 1 times as envs of one handle: copy 0 the base point, copies 2c + 1 and 2c + 2 with
    column c moved by +h_c and -h_c; the columns are the n_x states, then the nu action entries of every step (nu = 0: states only).
    Returns (xs [m reps, n_x], acts [K, m reps, n_act], h [n_col], reps)."""
    nx = x0.shape[1]
    ncol = nx + acts.shape[0] * nu
    reps = 2 * ncol + 1
    xs, a = np.repeat(x0, reps, axis=0), np.repeat(acts, reps, axis=1)
    h = fd_steps(x0, ncol)
    for c in range(ncol):
        shift(xs, a, c, h[c], slice(2 * c + 1, None, reps))
        shift(xs, a, c, -h[c], slice(2 * c + 2, None, reps))
    return xs, a, h, reps


def compare_fd(name, grad, fd, tol):
    """worst |grad - central difference| relative to each env's gradient scale, over the stencils that stay on one branch: a stencil is
    excluded when its end steps differ from the unperturbed run's or its one-sided differences disagree by more than 1e-4 of the scale
    (a termination, a clip, |e|^p at e = 0 on one side).  fd: dict(target [m], end [m], plus, minus, end_p, end_m [m, n_col], h [n_col]).
    Returns (worst, excluded, total)."""
    m, ncol = grad.shape
    worst, excluded = 0.0, 0
    for b in range(m):
        scale = max(np.abs(grad[b]).max(), 1e-12)
        for c in range(ncol):
            hc = fd["h"][c]
            right, left = (fd["plus"][b, c] - fd["target"][b]) / hc, (fd["target"][b] - fd["minus"][b, c]) / hc
            if fd["end_p"][b, c] != fd["end"][b] or fd["end_m"][b, c] != fd["end"][b] or abs(right - left) > 1e-4 * scale:
                excluded += 1
                continue
            worst = max(worst, abs(grad[b, c] - (fd["plus"][b, c] - fd["minus"][b, c]) / (2 * hc)) / scale)
    print(f"{name}: {m * ncol} perturbations, {excluded} excluded, worst {worst:.2e}")
    return worst, excluded, m * ncol


def sens_check(s, dup, ddn, mid, h, tol, d2h=None):
    """parameter sensitivities s [..., n_x] against the central difference d = (dup + ddn) / 2h of one parameter, row by row (last axis).
    Each entry may miss d by tol of its row's scale plus the reference's own error: the rounding floor 64 eps (|mid| + 1) / h and, with
    the 2h difference d2h, twice the distance to it.  A row whose forward and backward differences dup / h and ddn / h disagree by more
    than 1e-2 of the scale plus the rounding floor crossed a kink (a clip, a current sign, a friction branch, a termination) and is
    excluded.  Returns (d, scale, err, kink, bad): kink and bad per row, bad excluding the kinks."""
    d = (dup + ddn) / (2 * h)
    rnd = 64 * 2.2e-16 * (np.abs(mid) + 1) / h
    floor = rnd if d2h is None else rnd + 2 * np.abs(d - d2h)
    scale = np.abs(d).max(axis=-1, keepdims=True)
    kink = (np.abs(dup - ddn) / h > 1e-2 * scale + rnd).any(axis=-1)
    err = np.abs(s - d)
    bad = (err > tol * scale + floor).any(axis=-1) & ~kink
    return d, scale, err, kink, bad


# ------------------------------------------------------------------------------------------------------------------ the oracle side
def discount_power(gamma, k):
    w = 1.0
    for _ in range(k):
        w *= gamma
    return w


def oracle_run(make_oracles, warm, x0, ref0, acts, gamma):
    """the float64 oracle from reset through the warm-up actions, then from (x0, ref0) through acts [K, m, nu]: (returns, end steps, x_K).
    make_oracles() -> [(Oracle, slice of the m envs)]; returns sum gamma^k r_k up to and including the first termination (end = K: none)."""
    oras = make_oracles()
    for o, _ in oras:
        o.reset()
    for a in warm:
        for o, sl in oras:
            o.step(a[sl])
    for o, sl in oras:
        o.set_ode_state(x0[sl])
        if o.n_ref:
            o.set_reference(ref0[sl])
    k_steps, m = acts.shape[0], acts.shape[1]
    ret, end, w = np.zeros(m), np.full(m, k_steps), 1.0
    for k in range(k_steps):
        rew, term = np.zeros(m), np.zeros(m, dtype=bool)
        for o, sl in oras:
            _, _, rew[sl], t = o.step(acts[k][sl])
            term[sl] = t.astype(bool)
        alive = end == k_steps
        ret[alive] = ret[alive] + w * rew[alive]
        end[alive & term] = k
        w = w * gamma
    return ret, end, np.concatenate([o.get_ode_state() for o, _ in oras])


def oracle_fd(make_oracles, warm, x0, acts, gamma, ref0=None, value_grad=None, angle=False):
    """central differences of the oracle's returns over every column of (x0, a_0 .. a_K-1): one oracle instance set per stencil point.
    With value_grad [m, n_x], the target is returns + gamma^K value_grad . x_K for the envs with end == K (the angle of x_K unwrapped
    relative to the unperturbed run).  Returns dict(ret, end, xk, plus, minus, end_p, end_m, h) with [m, n_col] stencil arrays."""
    m, nx = x0.shape
    k_steps, _, nu = acts.shape
    ref0 = np.zeros((m, 0)) if ref0 is None else ref0
    gk = discount_power(gamma, k_steps)
    base = oracle_run(make_oracles, warm, x0, ref0, acts, gamma)

    def target(res):
        ret, end, xk = res
        if value_grad is None:
            return ret
        xk = xk.copy()
        if angle:
            d = xk[:, -1] - base[2][:, -1]
            xk[:, -1] = base[2][:, -1] + (d + np.pi) % (2 * np.pi) - np.pi
        return np.where(end == k_steps, ret + gk * (value_grad * xk).sum(1), ret)

    ncol = nx + k_steps * nu
    plus, minus = np.zeros((m, ncol)), np.zeros((m, ncol))
    end_p, end_m = np.zeros((m, ncol), dtype=int), np.zeros((m, ncol), dtype=int)
    h = fd_steps(x0, ncol)
    for c in range(ncol):
        for sign, val, ends in ((1.0, plus, end_p), (-1.0, minus, end_m)):
            xs, a = x0.copy(), acts.copy()
            shift(xs, a, c, sign * h[c])
            res = oracle_run(make_oracles, warm, xs, ref0, a, gamma)
            val[:, c] = target(res)
            ends[:, c] = res[1]
    return dict(ret=base[0], end=base[1], xk=base[2], target=target(base), plus=plus, minus=minus, end_p=end_p, end_m=end_m, h=h)


def _oracle_states(cfg, x0, acts):
    """the oracle's ODE state after every step from x0: [K, m, n_x]"""
    from oracle.gem_oracle import Oracle

    o = Oracle(cfg)
    o.reset()
    o.set_ode_state(x0)
    xs = []
    for a in acts:
        o.step(a)
        xs.append(o.get_ode_state())
    return np.stack(xs)
