"""ctypes binding of the C-ABI declared in include/gemb200.h.

The shared library (gym_electric_motor_b200/libgemb200.so) is built in-tree by `__graft_entry__.build()` /
`python -m gym_electric_motor_b200.build` with nvcc for sm_90a.  There is NO fallback: if the library is missing
or cannot be loaded, `load_library()` raises — the product path never routes through a CPU implementation.
"""
import ctypes as C
import os

ABI_VERSION = 10
MAX_STATE, MAX_ODE, MAX_ACT, MAX_REF, MAX_CONSTRAINTS, MAX_MOTOR_PARAM, MAX_STATE_OPS = 28, 8, 6, 4, 4, 16, 4
MAX_REF_ENTRIES = 12  # generator parameter entries: output slots + switched sub-generators

# enums (include/gemb200.h)
MOTOR_PERMEX_DC, MOTOR_SERIES_DC, MOTOR_SHUNT_DC, MOTOR_EXTEX_DC, MOTOR_PMSM, MOTOR_SYNRM, MOTOR_EESM, MOTOR_SCIM, MOTOR_DFIM = range(9)
(MP_P, MP_R_S, MP_L_D, MP_L_Q, MP_PSI_P, MP_J_ROTOR, MP_R_A, MP_L_A, MP_PSI_E, MP_R_E, MP_L_E, MP_L_E_PRIME, MP_L_M,
 MP_K, MP_L_SIGS, MP_L_SIGR) = range(16)
CONV_NONE, CONV_1QC, CONV_2QC, CONV_4QC, CONV_B6 = range(5)
LOAD_CONST_SPEED, LOAD_POLY_STATIC, LOAD_EXT_SPEED = 0, 1, 2
LP_A, LP_B, LP_C, LP_J_LOAD, LP_TAU_DECAY, LP_TAU_LOAD = range(6)
SOLVER_EULER, SOLVER_RK4 = 0, 1
CONSTRAINT_LIMIT, CONSTRAINT_SQUARED = 0, 1
REF_CONST, REF_WIENER, REF_EXTERNAL, REF_LAPLACE, REF_SINUS, REF_STEP, REF_SAWTOOTH, REF_TRIANGULAR = range(8)
F32, F64 = 0, 1
LAYOUT_AOS, LAYOUT_SOA = 0, 1
AUTORESET_NONE, AUTORESET_SAME_STEP = 0, 1
SOP_NONE, SOP_COS_SIN, SOP_FLUX_OBSERVER, SOP_NOISE, SOP_CURRENT_SUM = range(5)
NOISE_NORMAL, NOISE_UNIFORM, NOISE_LAPLACE = range(3)
SUPPLY_IDEAL, SUPPLY_RC, SUPPLY_AC1 = 0, 1, 2
DIST_UNIFORM, DIST_LOG_UNIFORM = 0, 1
MAX_DRAW = MAX_MOTOR_PARAM + 8  # parameter slots of gemb200_set_param_randomization: motor slots, then load slots
RNG_ID_WORDS = 8  # GEMB200_RNG_ID_WORDS: words of one RNG identity row (gemb200_pack_rng_ids)
ENV_PARAM_SLOTS = MAX_DRAW  # GEMB200_ENV_PARAM_SLOTS: float64 slots of one parameter row (gemb200_pack_envs_params), the order of MAX_DRAW

E_INVALID, E_CUDA, E_NOMEM, E_ABI = -1, -2, -3, -4


class GemB200Config(C.Structure):
    """Mirror of `struct gemb200_config` (field order and types must match include/gemb200.h exactly;
    tests/test_cabi.py checks sizeof against the library)."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("abi_version", C.c_int32),
        ("n_envs", C.c_int32),
        ("device", C.c_int32),
        ("dtype", C.c_int32),
        ("layout", C.c_int32),
        ("autoreset", C.c_int32),
        ("finite", C.c_int32),
        ("motor_kind", C.c_int32),
        ("converter_kind", C.c_int32 * 2),
        ("load_kind", C.c_int32),
        ("solver_kind", C.c_int32),
        ("solver_nsteps", C.c_int32),
        ("tau", C.c_double),
        ("interlocking_time", C.c_double),
        ("u_sup", C.c_double),
        ("motor_param", C.c_double * MAX_MOTOR_PARAM),
        ("load_param", C.c_double * 8),
        ("limits", C.c_double * MAX_STATE),
        ("init_ode", C.c_double * MAX_ODE),
        ("n_constraints", C.c_int32),
        ("constraint_kind", C.c_int32 * MAX_CONSTRAINTS),
        ("constraint_mask", C.c_uint32 * MAX_CONSTRAINTS),
        ("reward_weight", C.c_double * MAX_STATE),
        ("reward_power", C.c_double * MAX_STATE),
        ("state_length", C.c_double * MAX_STATE),
        ("reward_bias", C.c_double),
        ("violation_reward", C.c_double),
        ("n_ref", C.c_int32),
        ("ref_kind", C.c_int32 * MAX_REF_ENTRIES),
        ("ref_state", C.c_int32 * MAX_REF_ENTRIES),
        ("ref_value", C.c_double * MAX_REF_ENTRIES),
        ("ref_margin_lo", C.c_double * MAX_REF_ENTRIES),
        ("ref_margin_hi", C.c_double * MAX_REF_ENTRIES),
        ("ref_init_lo", C.c_double * MAX_REF_ENTRIES),
        ("ref_init_hi", C.c_double * MAX_REF_ENTRIES),
        ("ref_sigma_lo", C.c_double * MAX_REF_ENTRIES),
        ("ref_sigma_hi", C.c_double * MAX_REF_ENTRIES),
        ("ref_len_lo", C.c_int32 * MAX_REF_ENTRIES),
        ("ref_len_hi", C.c_int32 * MAX_REF_ENTRIES),
        ("seed", C.c_uint64),
        ("env_index_offset", C.c_int64),
        ("action_dq", C.c_int32),
        ("dead_time_steps", C.c_int32),
        ("dead_time_outer", C.c_int32),
        ("init_random", C.c_int32),
        ("angle_advance", C.c_double),
        ("init_lo", C.c_double * MAX_ODE),
        ("init_hi", C.c_double * MAX_ODE),
        ("ref_amp_lo", C.c_double * MAX_REF_ENTRIES),
        ("ref_amp_hi", C.c_double * MAX_REF_ENTRIES),
        ("ref_freq_lo", C.c_double * MAX_REF_ENTRIES),
        ("ref_freq_hi", C.c_double * MAX_REF_ENTRIES),
        ("ref_off_lo", C.c_double * MAX_REF_ENTRIES),
        ("ref_off_hi", C.c_double * MAX_REF_ENTRIES),
        ("n_state_ops", C.c_int32),
        ("sop_kind", C.c_int32 * MAX_STATE_OPS),
        ("sop_idx", (C.c_int32 * 4) * MAX_STATE_OPS),
        ("sop_mask", C.c_uint32 * MAX_STATE_OPS),
        ("sop_param", (C.c_double * 8) * MAX_STATE_OPS),
        ("init_dist", C.c_int32 * MAX_ODE),
        ("init_mu", C.c_double * MAX_ODE),
        ("init_sigma", C.c_double * MAX_ODE),
        ("ref_sw_count", C.c_int32 * MAX_REF),
        ("ref_sw_first", C.c_int32 * MAX_REF),
        ("ref_sw_len_lo", C.c_int32 * MAX_REF),
        ("ref_sw_len_hi", C.c_int32 * MAX_REF),
        ("ref_sw_cdf", C.c_double * MAX_REF_ENTRIES),
        ("ext_speed_table", C.c_void_p),
        ("ext_speed_len", C.c_int32),
        ("supply_kind", C.c_int32),
        ("supply_param", C.c_double * 4),
        ("init_im_valid", C.c_int32),
        ("init_im", C.c_double * 8),
        ("interlocking_time1", C.c_double),
    ]


def new_config():
    """Python-side equivalent of gemb200_config_init (usable without the library, e.g. to drive the test oracle)."""
    cfg = GemB200Config()
    cfg.struct_size = C.sizeof(GemB200Config)
    cfg.abi_version = ABI_VERSION
    cfg.n_envs = 1
    cfg.solver_kind = SOLVER_RK4
    cfg.solver_nsteps = 1
    cfg.tau = 1e-4
    cfg.load_param[LP_TAU_DECAY] = 1e-3
    cfg.interlocking_time1 = -1.0
    for i in range(MAX_STATE):
        cfg.limits[i] = 1.0
        cfg.state_length[i] = 2.0
        cfg.reward_power[i] = 1.0
    for r in range(MAX_REF_ENTRIES):
        cfg.ref_len_lo[r], cfg.ref_len_hi[r] = 500, 2000
        cfg.ref_sigma_lo[r], cfg.ref_sigma_hi[r] = 1e-3, 1e-1
        cfg.ref_margin_lo[r], cfg.ref_margin_hi[r] = -1.0, 1.0
        cfg.ref_init_lo[r], cfg.ref_init_hi[r] = -1.0, 1.0
    return cfg


LIB_NAME = "libgemb200.so"
_lib = None

SYMBOLS = [
    "gemb200_version", "gemb200_last_error", "gemb200_config_init", "gemb200_query_dims", "gemb200_create",
    "gemb200_destroy", "gemb200_reset", "gemb200_step", "gemb200_step_host", "gemb200_reset_host", "gemb200_rollout", "gemb200_rollout_record",
    "gemb200_rollout_record_ref", "gemb200_rollout_returns", "gemb200_query_jacobian_dims", "gemb200_rollout_jacobians",
    "gemb200_query_return_grad_dims", "gemb200_rollout_return_grads", "gemb200_query_param_sens_dims", "gemb200_coef_tangents",
    "gemb200_rollout_param_sens",
    "gemb200_get_ode_state", "gemb200_set_ode_state", "gemb200_get_reference", "gemb200_set_reference",
    "gemb200_reseed", "gemb200_set_device_clock", "gemb200_get_clock", "gemb200_set_env_params", "gemb200_peer_buffer_alloc", "gemb200_peer_buffer_open", "gemb200_peer_buffer_close",
    "gemb200_peer_buffer_free", "gemb200_bind_peers", "gemb200_peer_signal", "gemb200_peer_wait", "gemb200_checkpoint_size", "gemb200_checkpoint_save", "gemb200_checkpoint_load", "gemb200_query_env_record",
    "gemb200_pack_envs", "gemb200_unpack_envs", "gemb200_set_param_randomization", "gemb200_get_env_params", "gemb200_launch_count",
    "gemb200_kernel_time_begin", "gemb200_kernel_time_end", "gemb200_pack_rng_ids", "gemb200_adopt_rng_ids", "gemb200_clear_rng_ids",
    "gemb200_pack_envs_params", "gemb200_unpack_envs_params",
]


def library_path():
    # GEMB200_LIB: developer override used by tools/variant_bench.py to load an experimental build of the SAME library
    return os.environ.get("GEMB200_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), LIB_NAME)


class GemB200Error(RuntimeError):
    pass


def load_library():
    """Load libgemb200.so and declare prototypes.  Raises GemB200Error when the extension is missing."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        raise GemB200Error(
            f"{path} not found: the CUDA extension is not built. Run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback."
        )
    try:
        lib = C.CDLL(path)
    except OSError as e:  # pragma: no cover - depends on the box
        raise GemB200Error(f"cannot load {path}: {e}") from e
    vp, i32p = C.c_void_p, C.POINTER(C.c_int32)
    cfgp = C.POINTER(GemB200Config)
    lib.gemb200_version.restype = C.c_int
    lib.gemb200_last_error.restype = C.c_char_p
    lib.gemb200_config_init.argtypes = [cfgp]
    lib.gemb200_query_dims.argtypes = [cfgp, i32p, i32p, i32p, i32p]
    lib.gemb200_create.argtypes = [cfgp, C.POINTER(vp)]
    lib.gemb200_destroy.argtypes = [vp]
    lib.gemb200_reset.argtypes = [vp, vp, vp, vp, vp]
    lib.gemb200_step.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.gemb200_step_host.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.gemb200_reset_host.argtypes = [vp, vp, vp, vp]
    lib.gemb200_rollout.argtypes = [vp, vp, C.c_int32, vp, vp, vp, vp, vp]
    lib.gemb200_rollout_record.argtypes = [vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp, vp]
    lib.gemb200_rollout_record_ref.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp, vp]
    lib.gemb200_rollout_returns.argtypes = [vp, vp, vp, C.c_int32, C.c_double, vp, vp, vp, vp, vp]
    lib.gemb200_query_jacobian_dims.argtypes = [cfgp, i32p, i32p]
    lib.gemb200_rollout_jacobians.argtypes = [vp, vp, vp, C.c_int32, vp, vp, vp, vp, vp, vp, vp]
    lib.gemb200_query_return_grad_dims.argtypes = [cfgp, i32p, i32p, i32p]
    lib.gemb200_rollout_return_grads.argtypes = [vp, vp, vp, C.c_int32, C.c_double, vp, vp, C.c_uint64, vp, vp, vp, vp, vp, vp, vp]
    lib.gemb200_query_param_sens_dims.argtypes = [cfgp, C.c_int32, i32p, i32p]
    lib.gemb200_coef_tangents.argtypes = [cfgp, vp, vp, C.c_int32, i32p, vp]
    lib.gemb200_rollout_param_sens.argtypes = [vp, vp, vp, C.c_int32, C.c_int32, i32p, vp, vp, vp, vp, vp, vp, vp]
    lib.gemb200_get_ode_state.argtypes = [vp, vp, vp]
    lib.gemb200_set_ode_state.argtypes = [vp, vp, vp]
    lib.gemb200_get_reference.argtypes = [vp, vp, vp]
    lib.gemb200_set_reference.argtypes = [vp, vp, vp]
    lib.gemb200_reseed.argtypes = [vp, C.c_uint64, vp]
    lib.gemb200_set_device_clock.argtypes = [vp, C.c_int32, vp]
    lib.gemb200_get_clock.argtypes = [vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), vp]
    lib.gemb200_set_env_params.argtypes = [vp, vp, vp]
    lib.gemb200_set_param_randomization.argtypes = [vp, C.c_int32, vp, vp, vp, vp]
    lib.gemb200_get_env_params.argtypes = [vp, vp, vp]
    lib.gemb200_peer_buffer_alloc.argtypes = [C.c_int32, C.c_int64, C.POINTER(vp), vp]
    lib.gemb200_peer_buffer_open.argtypes = [C.c_int32, vp, C.POINTER(vp)]
    lib.gemb200_peer_buffer_close.argtypes = [C.c_int32, vp]
    lib.gemb200_peer_buffer_free.argtypes = [C.c_int32, vp]
    lib.gemb200_bind_peers.argtypes = [vp, C.c_int32, vp]
    lib.gemb200_peer_signal.argtypes = [vp, C.c_int32, vp, C.c_uint32, vp]
    lib.gemb200_peer_wait.argtypes = [vp, C.c_int32, vp, C.c_uint32, vp, vp]
    lib.gemb200_checkpoint_size.argtypes = [vp]
    lib.gemb200_checkpoint_size.restype = C.c_int64
    lib.gemb200_checkpoint_save.argtypes = [vp, vp]
    lib.gemb200_checkpoint_load.argtypes = [vp, vp]
    lib.gemb200_query_env_record.argtypes = [cfgp, i32p, C.POINTER(C.c_uint64)]
    lib.gemb200_pack_envs.argtypes = [vp, vp, C.c_int32, vp, vp]
    lib.gemb200_unpack_envs.argtypes = [vp, vp, C.c_int32, C.c_uint64, vp, vp, C.c_int32, vp]
    lib.gemb200_pack_rng_ids.argtypes = [vp, vp, C.c_int32, vp, vp]
    lib.gemb200_adopt_rng_ids.argtypes = [vp, vp, C.c_int32, vp, vp, C.c_int32, vp]
    lib.gemb200_clear_rng_ids.argtypes = [vp, vp]
    lib.gemb200_pack_envs_params.argtypes = [vp, vp, C.c_int32, vp, vp, vp]
    lib.gemb200_unpack_envs_params.argtypes = [vp, vp, vp, vp, C.c_int32, C.c_uint64, vp, vp, C.c_int32, vp]
    lib.gemb200_launch_count.argtypes = [vp]
    lib.gemb200_launch_count.restype = C.c_int64
    lib.gemb200_kernel_time_begin.argtypes = [vp, vp]
    lib.gemb200_kernel_time_end.argtypes = [vp, vp, C.POINTER(C.c_float)]
    for name in SYMBOLS:
        fn = getattr(lib, name)
        if fn.restype is C.c_int and name not in ("gemb200_version",):
            fn.restype = C.c_int
    _lib = lib
    return lib


def check(rc, what="gemb200 call"):
    if rc != 0:
        lib = load_library()
        msg = lib.gemb200_last_error()
        raise GemB200Error(f"{what} failed (rc={rc}): {msg.decode() if msg else ''}")
