"""Diagnostic: replay one golden on the device and print per-column errors and where they peak."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from helpers import *
from gym_electric_motor_b200 import _cabi as K

for name in sys.argv[1:]:
    g = load_golden(name)
    for dt in (K.F32, K.F64):
        cfg = config_from_meta(g["meta"], reset_ode=g["reset_ode"], dtype=dt, solver=g["meta"]["case"]["solver"])
        out = replay_golden(DeviceAdapter(cfg), g)
        d = np.abs(out["states"] - g["states"])
        scale = np.maximum(np.abs(g["states"]).max(axis=0), 1e-12)
        print(name, "f32" if dt == K.F32 else "f64")
        print("  names", g["meta"]["state_names"])
        print("  colrel", np.array2string(d.max(axis=0) / scale, precision=1))
        k = int(np.argmax((d / scale).max(axis=1)))
        print("  worst step", k, "ode before", g["ode_states"][k - 1] if k else g["reset_ode"])
        print("  dev", np.array2string(out["states"][k], precision=6))
        print("  ref", np.array2string(g["states"][k], precision=6))
