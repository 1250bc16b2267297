"""ctypes wrapper of oracle/gem_oracle.c — TEST INFRASTRUCTURE, never imported by the product package.

The oracle takes the same POD `gemb200_config` as the C-ABI (struct definition only; see include/gemb200.h).
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_build", "libgem_oracle.so")
SOLVER_DOPRI5 = 100  # oracle-only solver kind
_lib = None


def build(force=False):
    src = os.path.join(HERE, "gem_oracle.c")
    hdr = os.path.join(HERE, "..", "include", "gemb200.h")
    stale = (not os.path.exists(LIB)) or any(
        os.path.exists(p) and os.path.getmtime(p) > os.path.getmtime(LIB) for p in (src, hdr)
    )
    if force or stale:
        subprocess.check_call(["make", "-C", HERE, "-B" if force else "-s"], stdout=subprocess.DEVNULL)
    return LIB


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(LIB)
        _lib.gem_oracle_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        _lib.gem_oracle_destroy.argtypes = [C.c_void_p]
        _lib.gem_oracle_dims.argtypes = [C.c_void_p] + [C.POINTER(C.c_int32)] * 4
        _lib.gem_oracle_reset.argtypes = [C.c_void_p] * 4
        _lib.gem_oracle_step.argtypes = [C.c_void_p] * 6 + [C.c_int]
        _lib.gem_oracle_rollout.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.c_int]
        for n in ("get_ode_state", "set_ode_state", "get_reference", "set_reference"):
            getattr(_lib, "gem_oracle_" + n).argtypes = [C.c_void_p, C.c_void_p]
        _lib.gem_oracle_get_ref_aux.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.gem_oracle_philox.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
        _lib.gem_oracle_probe_set_action.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double]
        _lib.gem_oracle_probe_convert.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
        _lib.gem_oracle_probe_conv_reset.argtypes = [C.c_void_p, C.c_void_p]
        _lib.gem_oracle_probe_i_sup.argtypes = [C.c_void_p, C.c_void_p]
        _lib.gem_oracle_probe_i_sup.restype = C.c_double
        _lib.gem_oracle_probe_mechanical_ode.argtypes = [C.c_void_p, C.c_double, C.c_double]
        _lib.gem_oracle_probe_mechanical_ode.restype = C.c_double
        _lib.gem_oracle_probe_mechanical_ode_ext.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double]
        _lib.gem_oracle_probe_mechanical_ode_ext.restype = C.c_double
        _lib.gem_oracle_probe_rc_supply_rhs.argtypes = [C.c_double] * 5
        _lib.gem_oracle_probe_rc_supply_rhs.restype = C.c_double
        _lib.gem_oracle_probe_ac1_voltage.argtypes = [C.c_double] * 4
        _lib.gem_oracle_probe_ac1_voltage.restype = C.c_double
        _lib.gem_oracle_probe_walk.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_int, C.c_void_p]
        _lib.gem_oracle_probe_wrap_action.argtypes = [C.c_void_p] * 5
        _lib.gem_oracle_probe_wrap_action.restype = C.c_int
        _lib.gem_oracle_probe_constraints.argtypes = [C.c_void_p, C.c_void_p]
        _lib.gem_oracle_probe_constraints.restype = C.c_double
        _lib.gem_oracle_probe_reward.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double]
        _lib.gem_oracle_probe_reward.restype = C.c_double
        _lib.gem_oracle_probe_euler.argtypes = [C.c_int, C.c_void_p, C.c_double, C.c_double, C.c_void_p]
        _lib.gem_oracle_set_clock.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
        _lib.gem_oracle_get_clock.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        _lib.gem_oracle_set_time_grid.argtypes = [C.c_void_p, C.c_int]
        _lib.gem_oracle_periodic_block.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Oracle:
    """N-env float64 CPU oracle with the env.reset / env.step contract of the reference (core.py:300-371)."""

    def __init__(self, cfg, nthreads=1):
        self._lib = lib()
        self.cfg = cfg
        self.n = int(cfg.n_envs)
        self.nthreads = int(nthreads)
        h = C.c_void_p()
        rc = self._lib.gem_oracle_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise ValueError(f"gem_oracle_create rc={rc}")
        self._h = h
        d = [C.c_int32() for _ in range(4)]
        self._lib.gem_oracle_dims(h, *[C.byref(x) for x in d])
        self.n_state, self.n_ode, self.n_act, self.n_ref = [x.value for x in d]
        self.finite = bool(cfg.finite)

    def __del__(self):
        if getattr(self, "_h", None):
            self._lib.gem_oracle_destroy(self._h)
            self._h = None

    def reset(self, mask=None):
        obs = np.zeros((self.n, self.n_state))
        ref = np.zeros((self.n, self.n_ref))
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        self._lib.gem_oracle_reset(self._h, _p(m), _p(obs), _p(ref))
        return obs, ref

    def step(self, action):
        if self.finite:
            a = np.ascontiguousarray(np.asarray(action).reshape(self.n, self.n_act), dtype=np.int32)
        else:
            a = np.ascontiguousarray(np.asarray(action, dtype=np.float64).reshape(self.n, self.n_act))
        obs = np.zeros((self.n, self.n_state))
        ref = np.zeros((self.n, self.n_ref))
        rew = np.zeros(self.n)
        term = np.zeros(self.n, dtype=np.uint8)
        self._lib.gem_oracle_step(self._h, _p(a), _p(obs), _p(ref), _p(rew), _p(term), self.nthreads)
        return obs, ref, rew, term

    def rollout(self, action_pool, n_steps):
        """n_steps consecutive steps, step k using action_pool[k % len(action_pool)]; returns the last step's outputs.  Identical results
        to n_steps calls of step(); the worker threads persist over the rollout (what bench.py's CPU arm times)."""
        dt = np.int32 if self.finite else np.float64
        pool = np.ascontiguousarray(np.asarray(action_pool, dtype=dt).reshape(len(action_pool), self.n, self.n_act))
        obs = np.zeros((self.n, self.n_state))
        ref = np.zeros((self.n, self.n_ref))
        rew = np.zeros(self.n)
        term = np.zeros(self.n, dtype=np.uint8)
        self._lib.gem_oracle_rollout(self._h, _p(pool), pool.strides[0], pool.shape[0], int(n_steps), _p(obs), _p(ref), _p(rew), _p(term), self.nthreads)
        return obs, ref, rew, term

    def set_clock(self, call_id, n_steps):
        """Jump to the clock (call id of the last API call, step calls so far) that VectorSim.clock() reports; reset afterwards."""
        self._lib.gem_oracle_set_clock(self._h, int(call_id), int(n_steps))

    def clock(self):
        a, b = C.c_uint64(), C.c_uint64()
        self._lib.gem_oracle_get_clock(self._h, C.byref(a), C.byref(b))
        return int(a.value), int(b.value)

    def set_time_grid(self, exact):
        """exact=False (default): the reference's grid, t accumulated with t += tau; exact=True: the device's, step k over [k tau, (k+1) tau]."""
        self._lib.gem_oracle_set_time_grid(self._h, 1 if exact else 0)

    def get_ode_state(self):
        out = np.zeros((self.n, self.n_ode))
        self._lib.gem_oracle_get_ode_state(self._h, _p(out))
        return out

    def set_ode_state(self, y):
        y = np.ascontiguousarray(np.asarray(y, dtype=np.float64).reshape(self.n, self.n_ode))
        self._lib.gem_oracle_set_ode_state(self._h, _p(y))

    def get_reference(self):
        out = np.zeros((self.n, self.n_ref))
        self._lib.gem_oracle_get_reference(self._h, _p(out))
        return out

    def set_reference(self, r):
        r = np.ascontiguousarray(np.asarray(r, dtype=np.float64).reshape(self.n, self.n_ref))
        self._lib.gem_oracle_set_reference(self._h, _p(r))

    def periodic_block(self, slot, kind, b, c, length):
        b = np.ascontiguousarray(b, dtype=np.uint32)
        c = np.ascontiguousarray(c, dtype=np.uint32)
        vals, par = np.zeros(length), np.zeros(5)
        self._lib.gem_oracle_periodic_block(self._h, slot, kind, _p(b), _p(c), length, _p(vals), _p(par))
        return vals, par

    # ---- component-level probes (env 0) for tests/test_oracle_known_answers.py
    def probe_set_action(self, action, t):
        if self.finite:
            a = np.ascontiguousarray(np.atleast_1d(action), dtype=np.int32)
            return self._lib.gem_oracle_probe_set_action(self._h, None, _p(a), float(t))
        a = np.ascontiguousarray(np.atleast_1d(action), dtype=np.float64)
        return self._lib.gem_oracle_probe_set_action(self._h, _p(a), None, float(t))

    def probe_convert(self, i_out, t):
        i = np.zeros(6)
        i[: len(np.atleast_1d(i_out))] = np.atleast_1d(i_out)
        u = np.zeros(6)
        self._lib.gem_oracle_probe_convert(self._h, _p(i), float(t), _p(u))
        return u

    def probe_i_sup(self, i_out):
        i = np.zeros(6)
        i[: len(np.atleast_1d(i_out))] = np.atleast_1d(i_out)
        return self._lib.gem_oracle_probe_i_sup(self._h, _p(i))

    def probe_conv_reset(self):
        u = np.zeros(6)
        self._lib.gem_oracle_probe_conv_reset(self._h, _p(u))
        return u

    def probe_mechanical_ode(self, omega, torque):
        return self._lib.gem_oracle_probe_mechanical_ode(self._h, float(omega), float(torque))

    def probe_mechanical_ode_ext(self, omega, torque, profile_value):
        return self._lib.gem_oracle_probe_mechanical_ode_ext(self._h, float(omega), float(torque), float(profile_value))

    def probe_walk(self, entry, start, increments):
        inc = np.ascontiguousarray(increments, dtype=np.float64)
        out = np.zeros(len(inc))
        self._lib.gem_oracle_probe_walk(self._h, int(entry), float(start), _p(inc), len(inc), _p(out))
        return out

    def probe_wrap_action(self, action):
        """the action-side wrappers (dead-time FIFO, dq -> abc) of env 0 as one more step call; returns the inner system's action"""
        out_f, out_i = np.zeros(8), np.zeros(2, dtype=np.int32)
        if self.finite:
            a = np.ascontiguousarray(np.atleast_1d(action), dtype=np.int32)
            n = self._lib.gem_oracle_probe_wrap_action(self._h, None, _p(a), _p(out_f), _p(out_i))
            return out_i[:n].copy()
        a = np.ascontiguousarray(np.atleast_1d(action), dtype=np.float64)
        n = self._lib.gem_oracle_probe_wrap_action(self._h, _p(a), None, _p(out_f), _p(out_i))
        return out_f[:n].copy()

    def probe_constraints(self, state):
        s = np.zeros(32)
        s[: len(state)] = state
        return self._lib.gem_oracle_probe_constraints(self._h, _p(s))

    def probe_reward(self, state, reference, violation):
        s, r = np.zeros(32), np.zeros(32)
        s[: len(state)] = state
        r[: len(reference)] = reference
        return self._lib.gem_oracle_probe_reward(self._h, _p(s), _p(r), float(violation))

    def get_ref_aux(self):
        sigma = np.zeros((self.n, self.n_ref))
        left = np.zeros((self.n, self.n_ref), dtype=np.int32)
        self._lib.gem_oracle_get_ref_aux(self._h, _p(sigma), _p(left))
        return sigma, left


def probe_euler(nsteps, y0, dt, u):
    """the oracle's EulerSolver stepping on the reference's test system (tests/conf.py:418-434)"""
    y0 = np.ascontiguousarray(y0, dtype=np.float64)
    out = np.zeros(2)
    lib().gem_oracle_probe_euler(int(nsteps), _p(y0), float(dt), float(u), _p(out))
    return out


def probe_rc_supply_rhs(u_sup, u_0, i_sup, r, c):
    return lib().gem_oracle_probe_rc_supply_rhs(float(u_sup), float(u_0), float(i_sup), float(r), float(c))


def probe_ac1_voltage(u_nominal, f, phi, t):
    return lib().gem_oracle_probe_ac1_voltage(float(u_nominal), float(f), float(phi), float(t))


def philox(counter, key):
    c = np.array(counter, dtype=np.uint32)
    lib().gem_oracle_philox(_p(c), int(key[0]), int(key[1]))
    return c
