import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from helpers import *
from gym_electric_motor_b200 import _cabi as K
from oracle.gem_oracle import Oracle
g = load_golden("pmsm_cc_rk4")
n = 600
for kinds in [(K.REF_LAPLACE, K.REF_WIENER), (K.REF_SINUS, K.REF_STEP), (K.REF_SAWTOOTH, K.REF_TRIANGULAR)]:
    def mk(dt):
        cfg = config_from_meta(g["meta"], n_envs=n, reset_ode=g["reset_ode"], dtype=dt, solver="rk4", ref_kind=K.REF_WIENER, autoreset=K.AUTORESET_SAME_STEP, seed=4242)
        for r in range(2):
            cfg.ref_kind[r] = kinds[r]
            cfg.ref_margin_lo[r], cfg.ref_margin_hi[r] = -0.6, 0.6
            cfg.ref_init_lo[r], cfg.ref_init_hi[r] = -0.6, 0.6
            cfg.ref_amp_lo[r], cfg.ref_amp_hi[r] = 0.05, 0.6
            cfg.ref_freq_lo[r], cfg.ref_freq_hi[r] = 20.0, 400.0
            cfg.ref_off_lo[r], cfg.ref_off_hi[r] = -0.6, 0.6
            cfg.ref_len_lo[r], cfg.ref_len_hi[r] = 7, 45
        return cfg
    dev = DeviceAdapter(mk(K.F64)); ora = Oracle(mk(K.F64), nthreads=8)
    _, o_ref = ora.reset(); _, d_ref = dev.reset()
    print(kinds, "reset diff per slot", np.abs(d_ref - o_ref).max(axis=0))
    rng = np.random.default_rng(1)
    for k in range(60):
        a = rng.uniform(-0.3, 0.3, size=(n, 3))
        _, o_ref, _, o_term = ora.step(a); _, d_ref, _, d_term = dev.step(a)
        d = np.abs(d_ref - o_ref)
        if d.max() > 1e-9:
            i = np.unravel_index(np.argmax(d), d.shape)
            print("  step", k, "max diff per slot", d.max(axis=0), "n_bad", (d > 1e-9).sum(axis=0), "worst env/slot", i, d_ref[i], o_ref[i], "term", o_term.sum(), d_term.sum())
            if k > 12: break
