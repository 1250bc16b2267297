#!/usr/bin/env python
"""Generate tests/golden/jacobians/system_jacobians.npz from the UNMODIFIED reference (CPU only; needs the reference sources, like make_golden.py).

For each of the nine motors under a constant-speed and a polynomial static load (the reference's Cont-CC-<motor>-v0 defaults otherwise),
at seeded points of its ODE state (the states a short random-action run visits) and seeded input voltages, the fixture holds:
  <case>/x      [P, n_ode]          the ODE state (reference order and units: [load states | motor states], the angle last)
  <case>/u      [P, n_u]            the voltages simulate() hands to the solver (the motor's VOLTAGES frame)
  <case>/jac    [P, n_ode, n_ode]   SCMLSystem._system_jacobian at (x, u)
  <case>/fd     [P, n_ode, n_ode]   central differences of SCMLSystem._system_equation at (x, u)
  <case>/tau    scalar              the env's sampling time
Usage:  python tests/golden/make_system_jacobians.py
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_ROOT = "/root/reference"
sys.dont_write_bytecode = True
try:
    import gymnasium  # noqa: F401
except ImportError:
    sys.path.insert(0, os.path.join(HERE, "..", "_shims"))
sys.path.insert(0, os.path.join(REF_ROOT, "src"))
warnings.filterwarnings("ignore")

import gym_electric_motor as gem  # noqa: E402
from gym_electric_motor import physical_systems as ps  # noqa: E402
from gym_electric_motor.core import ElectricMotorVisualization  # noqa: E402

MOTORS = {"PermExDc": 1, "ExtExDc": 2, "SeriesDc": 1, "ShuntDc": 1, "PMSM": 2, "SynRM": 2, "EESM": 3, "SCIM": 2, "DFIM": 4}
POLY = dict(a=0.01, b=0.02, c=1e-4, j_load=1e-3)
POINTS = 6


class NoViz(ElectricMotorVisualization):
    pass


def case(motor, load, seed):
    ld = ps.ConstantSpeedLoad(omega_fixed=80.0) if load == "const" else ps.PolynomialStaticLoad(load_parameter=dict(POLY))
    env = gem.make(f"Cont-CC-{motor}-v0", load=ld, visualization=NoViz())
    env.reset(seed=seed)
    sysm = env.physical_system.unwrapped
    rng = np.random.default_rng(seed)
    u_sup = float(sysm.supply.u_nominal)
    xs, us, jacs, fds = [], [], [], []
    for _ in range(POINTS):
        for _ in range(int(rng.integers(2, 12))):
            _, _, term, _, _ = env.step(env.action_space.sample())
            if term:
                env.reset()
        x = np.array(sysm._ode_solver.y, dtype=float)
        if load == "poly":  # a short run barely spins the load up: half the points at a running speed, half inside the static-friction band
            x[0] = rng.uniform(-250.0, 250.0) if rng.random() < 0.5 else rng.uniform(-1e-3, 1e-3) * POLY["a"]
        u = rng.uniform(-0.5, 0.5, MOTORS[motor]) * u_sup
        t = 0.0
        # the solver's parameter as simulate() passes it: the DFIM takes [[u_s alpha, u_s beta], [u_r alpha, u_r beta]]
        arg = np.array([u[:2], u[2:]]) if motor == "DFIM" else list(u)
        jac = np.array(sysm._system_jacobian(t, x, arg), dtype=float)
        fd = np.zeros_like(jac)
        for j in range(x.size):
            h = 1e-7 * max(1.0, abs(x[j]))
            xp, xm = x.copy(), x.copy()
            xp[j] += h
            xm[j] -= h
            fp = np.array(sysm._system_equation(t, xp, arg), dtype=float).copy()
            fm = np.array(sysm._system_equation(t, xm, arg), dtype=float).copy()
            fd[:, j] = (fp - fm) / (2 * h)
        xs.append(x), us.append(u), jacs.append(jac), fds.append(fd)
    return dict(x=np.array(xs), u=np.array(us), jac=np.array(jacs), fd=np.array(fds), tau=np.array(float(sysm.tau)))


def main():
    out = {}
    for k, motor in enumerate(MOTORS):
        for load in ("const", "poly"):
            for key, val in case(motor, load, 100 + 2 * k + (load == "poly")).items():
                out[f"{motor}_{load}/{key}"] = val
    path = os.path.join(HERE, "jacobians", "system_jacobians.npz")  # a directory of its own: the trajectory goldens are every *.npz above
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez_compressed(path, **out)
    print("wrote", path, len(out) // 5, "cases")


if __name__ == "__main__":
    main()
