"""Low-level handle wrapper: one `VectorSim` = one gemb200_handle = N envs of one motor/converter/load/solver
combination on one CUDA device.  Tensors are torch tensors on that device (torch is plumbing: memory + streams);
all compute happens in libgemb200.so through the C-ABI (include/gemb200.h).

This is the batched counterpart of the reference's `SCMLSystem` + the per-step part of `ElectricMotorEnvironment`
(physical_systems.py:13-287, core.py:300-371).
"""
import ctypes as C

import numpy as np
import torch

from . import _cabi as K


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class VectorSim:
    def __init__(self, cfg, reuse_outputs=True):
        self._lib = K.load_library()
        if not torch.cuda.is_available():
            raise K.GemB200Error("no CUDA device visible: the CUDA path has no CPU fallback")
        self.cfg = cfg
        self.device = torch.device("cuda", int(cfg.device))
        d = [C.c_int32() for _ in range(4)]
        K.check(self._lib.gemb200_query_dims(C.byref(cfg), *[C.byref(x) for x in d]), "gemb200_query_dims")
        self.n_state, self.n_ode, self.n_act, self.n_ref = [x.value for x in d]
        self.n = int(cfg.n_envs)
        self.finite = bool(cfg.finite)
        self.soa = cfg.layout == K.LAYOUT_SOA
        self.dtype = torch.float32 if cfg.dtype == K.F32 else torch.float64
        self.np_dtype = np.float32 if cfg.dtype == K.F32 else np.float64
        self.act_dtype = torch.int32 if self.finite else self.dtype
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            K.check(self._lib.gemb200_create(C.byref(cfg), C.byref(h)), "gemb200_create")
        self._h = h
        self._reuse = reuse_outputs
        self._out = None

    # ------------------------------------------------------------------ lifecycle
    def close(self):
        if getattr(self, "_h", None):
            self._lib.gemb200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ helpers
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _shape(self, k):
        return (k, self.n) if self.soa else (self.n, k)

    def _ref_ptr(self, ref):
        """the reference output of a launch: NULL without reference slots"""
        return _ptr(ref) if self.n_ref else None

    def _alloc_outputs(self):
        if self._reuse and self._out is not None:
            return self._out
        self._out_ptrs = None
        out = (
            torch.empty(self._shape(self.n_state), dtype=self.dtype, device=self.device),
            torch.empty(self._shape(self.n_ref), dtype=self.dtype, device=self.device),
            torch.empty(self.n, dtype=self.dtype, device=self.device),
            torch.empty(self.n, dtype=torch.uint8, device=self.device),
        )
        if self._reuse:
            self._out = out
        return out

    def _alloc_stacked(self, s):
        """(obs, ref, reward, terminated) of s recorded steps, stacked on a leading axis"""
        return (
            torch.empty((s,) + self._shape(self.n_state), dtype=self.dtype, device=self.device),
            torch.empty((s,) + self._shape(self.n_ref), dtype=self.dtype, device=self.device),
            torch.empty((s, self.n), dtype=self.dtype, device=self.device),
            torch.empty((s, self.n), dtype=torch.uint8, device=self.device),
        )

    def bind_outputs(self, obs, ref, reward, terminated):
        """Let the step / reset launches write into caller-owned tensors (e.g. the sections of a packed all-gather buffer,
        distributed.PackedStepOutputs).  Shapes, dtypes and device must match what `step` returns."""
        exp = (self._shape(self.n_state), self._shape(self.n_ref), (self.n,), (self.n,))
        for t, shp, dt in zip((obs, ref, reward, terminated), exp, (self.dtype, self.dtype, self.dtype, torch.uint8)):
            if tuple(t.shape) != tuple(shp) or t.dtype != dt or t.device != self.device or not t.is_contiguous():
                raise ValueError(f"output tensor mismatch: need {tuple(shp)} {dt} contiguous on {self.device}, got {tuple(t.shape)} {t.dtype} on {t.device}")
            if t.data_ptr() % 16:
                raise ValueError("output tensors must be 16-byte aligned")
        self._reuse, self._out, self._out_ptrs = True, (obs, ref, reward, terminated), None

    def _as_action(self, action):
        if isinstance(action, torch.Tensor) and action.dtype == self.act_dtype and action.device == self.device and action.is_contiguous() \
                and action.numel() == self.n * self.n_act:
            return action  # fast path: nothing to convert (the launch only needs the pointer)
        a = torch.as_tensor(action, device=self.device)
        if a.dtype != self.act_dtype:
            a = a.to(self.act_dtype)
        a = a.reshape(self._shape(self.n_act))
        return a.contiguous()

    # ------------------------------------------------------------------ env API (device tensors)
    def reset(self, mask=None):
        """env.reset for all (mask=None) or the masked envs; returns (obs, ref_next) device tensors.
        With a mask, rows of unmasked envs keep their previous content."""
        obs, ref, _, _ = self._alloc_outputs()
        m = None
        if mask is not None:
            m = torch.as_tensor(mask, device=self.device).to(torch.uint8).contiguous()
        K.check(self._lib.gemb200_reset(self._h, _ptr(m), _ptr(obs), self._ref_ptr(ref), self._stream()), "gemb200_reset")
        return obs, ref

    def reseed(self, seed):
        """re-key the RNG streams and start the handle over (gemb200_reseed): equal seeds -> identical episodes"""
        K.check(self._lib.gemb200_reseed(self._h, C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), self._stream()), "gemb200_reseed")
        self.cfg.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        self._ids_adopted = False  # the reseed gives every env its own RNG identity back

    def set_device_clock(self, enable=True):
        """Device-resident clock (gemb200_set_device_clock): while on, step / rollout / reset launches read the RNG call id, the step count
        and the dead-time ring position from device memory and advance them with a one-thread kernel, so the launches can be captured in a
        CUDA graph and replayed (graph.CapturedSteps).  Same results as with the host clock, bit for bit."""
        K.check(self._lib.gemb200_set_device_clock(self._h, 1 if enable else 0, self._stream()), "gemb200_set_device_clock")

    def clock(self):
        """(number of API calls that drew random numbers, number of env steps) so far; synchronises when the device clock is on"""
        a, b = C.c_uint64(), C.c_uint64()
        K.check(self._lib.gemb200_get_clock(self._h, C.byref(a), C.byref(b), self._stream()), "gemb200_get_clock")
        return int(a.value), int(b.value)

    def set_env_params(self, motor_param=None, load_param=None):
        """Per-env parameter blocks (gemb200_set_env_params): motor_param [N, 16] / load_param [N, 8] float64 host arrays in the slot order of
        `_cabi.MP_*` / `_cabi.LP_*`; None keeps the configuration's values; both None: back to the shared coefficients.  Every motor row must
        keep the configuration's pole pairs (ValueError): the angle increments are prepared per handle."""
        mp = None if motor_param is None else np.ascontiguousarray(motor_param, dtype=np.float64).reshape(self.n, K.MAX_MOTOR_PARAM)
        lp = None if load_param is None else np.ascontiguousarray(load_param, dtype=np.float64).reshape(self.n, 8)
        if mp is not None:
            from .randomization import check_pole_pairs

            check_pole_pairs(mp[:, K.MP_P], self.cfg.motor_param[K.MP_P])
        vp = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)  # noqa: E731
        K.check(self._lib.gemb200_set_env_params(self._h, vp(mp), vp(lp)), "gemb200_set_env_params")
        if mp is None and lp is None:
            self._draw_slots = ()

    _draw_slots = ()

    @property
    def randomized_slots(self):
        """parameter slots drawn at every reset (gemb200_set_param_randomization), in the order of `env_params` rows"""
        return self._draw_slots

    def set_param_randomization(self, slots=(), kinds=(), lo=(), hi=()):
        """Per-episode domain randomisation (gemb200_set_param_randomization): from now on every reset of an env draws new values for the
        parameter slots (`_cabi.MP_*`, or `_cabi.MAX_MOTOR_PARAM + _cabi.LP_*`) from kinds[j] (`_cabi.DIST_*`) on [lo[j], hi[j]].  Draws
        nothing by itself; empty arguments stop drawing (the envs keep their last values)."""
        n = len(slots)
        if not (len(kinds) == len(lo) == len(hi) == n):
            raise ValueError("slots, kinds, lo and hi must have the same length")
        m = max(n, 1)
        K.check(self._lib.gemb200_set_param_randomization(self._h, n, (C.c_int32 * m)(*slots), (C.c_int32 * m)(*kinds),
                                                         (C.c_double * m)(*lo), (C.c_double * m)(*hi)), "gemb200_set_param_randomization")
        self._draw_slots = tuple(int(s) for s in slots)

    def env_params(self):
        """stored values of the drawn parameters, [len(randomized_slots), N] device tensor in the handle's dtype (stream-ordered copy)"""
        if not self._draw_slots:
            raise RuntimeError("no parameters are drawn per reset (set_param_randomization)")
        out = torch.empty((len(self._draw_slots), self.n), dtype=self.dtype, device=self.device)
        K.check(self._lib.gemb200_get_env_params(self._h, _ptr(out), self._stream()), "gemb200_get_env_params")
        return out

    _ids_adopted = False

    def _refuse_with_identities(self, what):
        if self._ids_adopted:
            raise NotImplementedError(f"{what} is not available while envs hold adopted RNG identities (restore(..., rng='source')): the "
                                      "checkpoint does not carry them (DESIGN.md §7); clear_rng_ids() or reseed first")

    def _refuse_while_drawing(self, what):
        if self._draw_slots:
            raise NotImplementedError(f"{what} is not available while parameters are drawn per reset: the drawn parameters are per-episode "
                                      "state that neither checkpoints nor snapshot rows carry (DESIGN.md §7); stop the draws first")

    def _as_feed(self, references, k):
        """check a reference feed of k steps: a contiguous device tensor of the handle's dtype, shaped [k, N, n_ref] (SoA: [k, n_ref, N]);
        k = None: one step, [N, n_ref] (SoA: [n_ref, N]).  Nothing is converted: a feed is read in place by the launch (and by every replay
        of a captured one).  No feed (None) stays None."""
        if references is None:
            return None
        if not self.n_ref:
            raise ValueError("a reference feed needs reference slots: this configuration has n_ref == 0")
        shape = self._shape(self.n_ref) if k is None else (int(k),) + self._shape(self.n_ref)
        if not isinstance(references, torch.Tensor):
            raise ValueError(f"references must be a {self.dtype} tensor of shape {shape} on {self.device}")
        if references.dtype != self.dtype or references.device != self.device or tuple(references.shape) != shape:
            raise ValueError(f"references must be {shape} {self.dtype} on {self.device}, got {tuple(references.shape)} {references.dtype} "
                             f"on {references.device}")
        if not references.is_contiguous():
            raise ValueError("references must be contiguous")
        return references

    def step(self, action, reference=None):
        """env.step: returns (obs, ref_next, reward, terminated) device tensors (views of reused buffers unless
        reuse_outputs=False).  reference ([N, n_ref], SoA [n_ref, N], the handle's dtype, on the device): first overwrite the stored value
        of every reference slot with it — `set_reference(reference); step(action)` in one stream-ordered, capturable launch (a K = 1
        rollout with a reference feed)."""
        if reference is not None:
            r = self._as_feed(reference, None)
            a = self._as_action(action)
            obs, ref, rew, term = out = self._alloc_outputs()
            self.rollout_into(a, 1, 0, obs, ref, rew, term, r[None])  # the K = 1 feed is a view: a captured step reads the caller's tensor
            return out
        a = self._as_action(action)
        out = self._alloc_outputs()
        if self._reuse:
            if getattr(self, "_out_ptrs", None) is None:
                obs, ref, rew, term = out
                self._out_ptrs = (_ptr(obs), self._ref_ptr(ref), _ptr(rew), _ptr(term))
            po, pr, pw, pt = self._out_ptrs
        else:
            obs, ref, rew, term = out
            po, pr, pw, pt = _ptr(obs), self._ref_ptr(ref), _ptr(rew), _ptr(term)
        rc = self._lib.gemb200_step(self._h, a.data_ptr(), po, pr, pw, pt, torch.cuda.current_stream(self.device).cuda_stream)
        if rc:
            K.check(rc, "gemb200_step")
        return out

    def rollout(self, actions, record_every=0, references=None):
        """K open-loop env.step calls fused into ONE launch (gemb200_rollout_record_ref): every env's record stays in registers for all K
        steps; bit-identical to K calls of `step`.  actions: [K, N, n_act] (SoA layout: [K, n_act, N]).
        record_every = 0 -> the outputs of the last step (obs, ref, reward, terminated), shapes as `step`;
        record_every = m >= 1 -> the outputs of steps m, 2m, ... stacked on a leading axis of length K // m (m = 1: full trajectory).
        references ([K, N, n_ref], SoA [K, n_ref, N], the handle's dtype, on the device; None: no feed): step k first overwrites the stored
        value of EVERY reference slot with references[k] — the same as K iterations of `set_reference(references[k]); step(actions[k])`."""
        a = actions if (isinstance(actions, torch.Tensor) and actions.dtype == self.act_dtype and actions.device == self.device and actions.is_contiguous()) \
            else torch.as_tensor(actions, device=self.device).to(self.act_dtype).contiguous()
        k = int(a.shape[0])
        if a.numel() != k * self.n * self.n_act:
            raise ValueError(f"actions must hold K x {self.n} x {self.n_act} values")
        r = self._as_feed(references, k)
        m = int(record_every)
        obs, ref, rew, term = self._alloc_outputs() if m == 0 else self._alloc_stacked(k // m)
        self.rollout_into(a, k, m, obs, ref, rew, term, r)
        return obs, ref, rew, term

    def rollout_into(self, actions, n_steps, record_every, obs, ref, rew, term, references=None):
        """Raw variant for benchmarking: caller-owned output tensors (any may be None), no allocation, no conversion.  references: the
        reference feed of `rollout`, checked like there."""
        r = self._as_feed(references, n_steps)
        K.check(self._lib.gemb200_rollout_record_ref(self._h, _ptr(actions), _ptr(r), int(n_steps), int(record_every), _ptr(obs), self._ref_ptr(ref),
                                                     _ptr(rew), _ptr(term), self._stream()),
                "gemb200_rollout_record" if r is None else "gemb200_rollout_record_ref")  # without a feed this is gemb200_rollout_record

    def _as_actions(self, actions):
        """check the actions of a fused launch: a contiguous device tensor of the action dtype, shaped [K, N, n_act] (SoA: [K, n_act, N])
        with K >= 1.  Nothing is converted."""
        if not isinstance(actions, torch.Tensor) or actions.dim() != 3:
            raise ValueError(f"actions must be a [K, {', '.join(map(str, self._shape(self.n_act)))}] {self.act_dtype} tensor on {self.device}")
        shape = (int(actions.shape[0]),) + self._shape(self.n_act)
        if actions.dtype != self.act_dtype or actions.device != self.device or tuple(actions.shape) != shape:
            raise ValueError(f"actions must be [K, {', '.join(map(str, shape[1:]))}] {self.act_dtype} on {self.device}, got "
                             f"{tuple(actions.shape)} {actions.dtype} on {actions.device}")
        if shape[0] < 1:
            raise ValueError("a rollout needs K >= 1 steps")
        if not actions.is_contiguous():
            raise ValueError("actions must be contiguous")
        return actions

    @staticmethod
    def _as_discount(discount):
        g = float(discount)
        if not (0.0 <= g <= 1.0):  # NaN fails both comparisons
            raise ValueError(f"discount must be a finite number in [0, 1], got {discount!r}")
        return g

    def rollout_returns(self, actions, discount=1.0, references=None):
        """K open-loop steps fused into ONE launch that hands back each env's discounted return instead of per-step outputs
        (gemb200_rollout_returns).  Returns (returns [N] in the handle's dtype, end_step [N] int32, (obs, ref) of the last step):
        end_step[i] = index of env i's first terminated step (K: none); returns[i] = sum of gamma^k * reward_k over k <= min(end_step, K - 1),
        gamma = discount rounded to the handle's dtype.  The final state, clock and RNG position are those of
        `rollout(actions, 1, references)`, bit for bit.  actions: [K, N, n_act] (SoA: [K, n_act, N]) in the action dtype on the device;
        references: the reference feed of `rollout`.  Bad actions, discount or feed: ValueError before any launch."""
        a = self._as_actions(actions)
        k = int(a.shape[0])
        g = self._as_discount(discount)
        r = self._as_feed(references, k)
        obs, ref, _, _ = self._alloc_outputs()
        ret = torch.empty(self.n, dtype=self.dtype, device=self.device)
        end = torch.empty(self.n, dtype=torch.int32, device=self.device)
        self.rollout_returns_into(a, k, g, ret, end, obs, ref, r)
        return ret, end, (obs, ref)

    def rollout_returns_into(self, actions, n_steps, discount, ret, end=None, obs=None, ref=None, references=None):
        """Raw variant of `rollout_returns` for benchmarking: caller-owned outputs (all but `ret` may be None), no allocation, no
        conversion.  The discount and the reference feed are checked like there."""
        g = self._as_discount(discount)
        r = self._as_feed(references, n_steps)
        K.check(self._lib.gemb200_rollout_returns(self._h, _ptr(actions), _ptr(r), int(n_steps), g, _ptr(ret), _ptr(end), _ptr(obs),
                                                  self._ref_ptr(ref), self._stream()), "gemb200_rollout_returns")

    def _query_dims(self, query, n_out, *args):
        """n_out int32 results of the configuration query `query` (no handle, no launch); NotImplementedError with the library's message
        for a configuration the launch refuses"""
        lib = K.load_library()
        out = [C.c_int32() for _ in range(n_out)]
        if getattr(lib, query)(C.byref(self.cfg), *args, *[C.byref(x) for x in out]):
            raise NotImplementedError(lib.gemb200_last_error().decode())
        return tuple(x.value for x in out)

    def jacobian_dims(self):
        """(n_x, n_u) of `rollout_jacobians`: n_x = n_ode, n_u = n_act (0 for finite converters).  NotImplementedError for a configuration the
        launch refuses (DESIGN.md §7)."""
        return self._query_dims("gemb200_query_jacobian_dims", 2)

    def rollout_jacobians(self, actions, references=None):
        """K open-loop steps in ONE launch that also linearise the plant (gemb200_rollout_jacobians).  Returns ((jac_x, jac_u), (obs, ref, rew,
        term)): jac_x [K, N, n_x, n_x] = d x_{k+1} / d x_k, jac_u [K, N, n_x, n_u] = d x_{k+1} / d a_k (None when n_u == 0), both in the
        handle's dtype, x = the ODE state of `get_ode_state` (the angle in radians), a = the caller's action; the outputs of every step exactly
        as `rollout(actions, record_every=1, references=references)` returns them, and the same final state, clock and RNG position.
        Refused configurations: NotImplementedError (DESIGN.md §7); bad actions or feed: ValueError before any launch."""
        nx, nu = self.jacobian_dims()
        a = self._as_actions(actions)
        k = int(a.shape[0])
        r = self._as_feed(references, k)
        jx = torch.empty((k, self.n, nx, nx), dtype=self.dtype, device=self.device)
        ju = torch.empty((k, self.n, nx, nu), dtype=self.dtype, device=self.device) if nu else None
        obs, ref, rew, term = self._alloc_stacked(k)
        self.rollout_jacobians_into(a, k, jx, ju, obs, ref, rew, term, r)
        return (jx, ju), (obs, ref, rew, term)

    def rollout_jacobians_into(self, actions, n_steps, jac_x, jac_u=None, obs=None, ref=None, rew=None, term=None, references=None):
        """Raw variant of `rollout_jacobians` for benchmarking: caller-owned outputs (all but `jac_x` may be None), no allocation, no
        conversion.  The reference feed is checked like there."""
        r = self._as_feed(references, n_steps)
        K.check(self._lib.gemb200_rollout_jacobians(self._h, _ptr(actions), _ptr(r), int(n_steps), _ptr(jac_x), _ptr(jac_u), _ptr(obs),
                                                    self._ref_ptr(ref), _ptr(rew), _ptr(term), self._stream()),
                "gemb200_rollout_jacobians")

    def return_grad_dims(self):
        """(n_x, n_u, ws_words) of `rollout_return_grads`: n_x = n_ode, n_u = n_act, ws_words = n_x (n_x + n_u) + n_x + n_u, the workspace
        words per env and step.  NotImplementedError for a configuration the launch refuses (DESIGN.md §7)."""
        return self._query_dims("gemb200_query_return_grad_dims", 3)

    def _as_tensor(self, t, name, shape):
        """check `t` (None stays None): a contiguous tensor of `shape` in the handle's dtype on its device.  Nothing is converted."""
        if t is not None and (not isinstance(t, torch.Tensor) or t.dtype != self.dtype or t.device != self.device or tuple(t.shape) != shape
                              or not t.is_contiguous()):
            got = f"{tuple(t.shape)} {t.dtype} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f"{name} must be a contiguous [{', '.join(map(str, shape))}] {self.dtype} tensor on {self.device}, got {got}")
        return t

    def rollout_return_grads(self, actions, discount=1.0, references=None, value_grad=None):
        """`rollout_returns` with the gradients of the returns (gemb200_rollout_return_grads), in ONE launch.  Returns (returns, end_step,
        (obs, ref), grad_a, grad_x0): the first three exactly as `rollout_returns(actions, discount, references)` returns them (and the
        same final state, clock and RNG position); grad_a [K, N, n_u] = d returns[i] / d a_k[i] for the caller's action, 0 for
        k >= end_step[i]; grad_x0 [N, n_x] = d returns[i] / d x_0[i], x the ODE state of `get_ode_state` (the angle last, in radians).
        value_grad [N, n_x] (handle dtype) adds discount^K value_grad[i] to the adjoint of every env with end_step == K.  The workspace,
        K * N * ws_words words, is a torch allocation of this call.  Refused configurations: NotImplementedError (DESIGN.md §7); bad
        actions, discount, feed or value_grad: ValueError before any launch."""
        nx, nu, ww = self.return_grad_dims()
        a = self._as_actions(actions)
        k = int(a.shape[0])
        g = self._as_discount(discount)
        r = self._as_feed(references, k)
        vg = self._as_tensor(value_grad, "value_grad", (self.n, nx))
        obs, ref, _, _ = self._alloc_outputs()
        ret = torch.empty(self.n, dtype=self.dtype, device=self.device)
        end = torch.empty(self.n, dtype=torch.int32, device=self.device)
        ga = torch.empty((k, self.n, nu), dtype=self.dtype, device=self.device)
        gx = torch.empty((self.n, nx), dtype=self.dtype, device=self.device)
        ws = torch.empty(k * self.n * ww, dtype=self.dtype, device=self.device)
        self.rollout_return_grads_into(a, k, g, ws, ret, end, ga, gx, obs, ref, r, vg)
        return ret, end, (obs, ref), ga, gx

    def rollout_return_grads_into(self, actions, n_steps, discount, workspace, ret, end, grad_a, grad_x0, obs=None, ref=None, references=None,
                                  value_grad=None):
        """Raw variant of `rollout_return_grads` for benchmarking: caller-owned outputs and workspace (a device tensor of at least
        n_steps * N * ws_words elements of the handle's dtype; `end`, `obs`, `ref` and `value_grad` may be None), no allocation, no
        conversion.  The discount and the reference feed are checked like there."""
        g = self._as_discount(discount)
        r = self._as_feed(references, n_steps)
        K.check(self._lib.gemb200_rollout_return_grads(self._h, _ptr(actions), _ptr(r), int(n_steps), g, _ptr(value_grad), _ptr(workspace),
                                                       workspace.numel() * workspace.element_size(), _ptr(ret), _ptr(end), _ptr(grad_a),
                                                       _ptr(grad_x0), _ptr(obs), self._ref_ptr(ref), self._stream()),
                "gemb200_rollout_return_grads")

    @staticmethod
    def _slot_array(slots):
        slots = [int(v) for v in slots]
        return (C.c_int32 * max(len(slots), 1))(*slots), len(slots)

    def param_sens_dims(self, slots):
        """n_x of `rollout_param_sens` for the parameter slots `slots` (GEMB200_MP_* / GEMB200_MAX_MOTOR_PARAM + GEMB200_LP_*): n_ode.
        NotImplementedError for a refused configuration or slot list (DESIGN.md §7)."""
        arr, n_p = self._slot_array(slots)
        return self._query_dims("gemb200_query_param_sens_dims", 1, n_p, arr)[0]

    def coef_tangents(self, slots, motor_param=None, load_param=None):
        """d (coefficient block) / d theta for the slots at a parameter row (the configuration's when None): float64 [n_p, 30] in the word
        order of the per-env coefficient block (gemb200_coef_tangents; no GPU)."""
        lib = K.load_library()
        arr, n_p = self._slot_array(slots)
        out = np.zeros((n_p, 30), dtype=np.float64)
        mp = None if motor_param is None else np.ascontiguousarray(motor_param, dtype=np.float64)
        lp = None if load_param is None else np.ascontiguousarray(load_param, dtype=np.float64)
        K.check(lib.gemb200_coef_tangents(C.byref(self.cfg), None if mp is None else mp.ctypes.data, None if lp is None else lp.ctypes.data, n_p, arr,
                                          out.ctypes.data), "gemb200_coef_tangents")
        return out

    def rollout_param_sens(self, actions, slots, references=None, sens0=None, record=True):
        """K open-loop steps in ONE launch that also carry the parameter sensitivities S = d x / d theta (gemb200_rollout_param_sens).
        Returns ((sens, sens_last), (obs, ref, rew, term)): sens [K, N, n_x, n_p] = d x_{k+1} / d theta after every step (None when
        record=False), sens_last [N, n_x, n_p] = the carried S after the last step (0 for an env reset in it), in the handle's dtype; the
        outputs of every step exactly as `rollout(actions, record_every=1, references=references)` returns them.  sens0 [N, n_x, n_p]: S at
        the start (None: zeros); it is not modified.  Refused configurations or slots: NotImplementedError (DESIGN.md §7); bad actions, feed
        or sens0: ValueError before any launch."""
        nx = self.param_sens_dims(slots)
        n_p = len(slots)
        a = self._as_actions(actions)
        k = int(a.shape[0])
        r = self._as_feed(references, k)
        sio = (torch.zeros((self.n, nx, n_p), dtype=self.dtype, device=self.device) if sens0 is None
               else self._as_tensor(sens0, "sens0", (self.n, nx, n_p)).clone())
        so = torch.empty((k, self.n, nx, n_p), dtype=self.dtype, device=self.device) if record else None
        obs, ref, rew, term = self._alloc_stacked(k)
        self.rollout_param_sens_into(a, k, slots, sio, so, obs, ref, rew, term, r)
        return (so, sio), (obs, ref, rew, term)

    def rollout_param_sens_into(self, actions, n_steps, slots, sens_io, sens_out=None, obs=None, ref=None, rew=None, term=None, references=None):
        """Raw variant of `rollout_param_sens` for benchmarking: caller-owned outputs (all but `sens_io` may be None; sens_io is read as S_0
        and overwritten with S_K), no allocation, no conversion.  The reference feed is checked like there."""
        r = self._as_feed(references, n_steps)
        arr, n_p = self._slot_array(slots)
        K.check(self._lib.gemb200_rollout_param_sens(self._h, _ptr(actions), _ptr(r), int(n_steps), n_p, arr, _ptr(sens_io), _ptr(sens_out), _ptr(obs),
                                                     self._ref_ptr(ref), _ptr(rew), _ptr(term), self._stream()),
                "gemb200_rollout_param_sens")

    # ------------------------------------------------------------------ host-buffer API (numpy)
    def step_host(self, action, out=None):
        """Same step through HOST buffers (the C-ABI does H2D, launch, D2H, sync).  `out` = tuple of numpy arrays to
        fill (obs, ref, reward, terminated); allocated when None."""
        a = np.ascontiguousarray(action, dtype=np.int32 if self.finite else self.np_dtype).reshape(self._shape(self.n_act))
        if out is None:
            out = (np.empty(self._shape(self.n_state), self.np_dtype), np.empty(self._shape(self.n_ref), self.np_dtype),
                   np.empty(self.n, self.np_dtype), np.empty(self.n, np.uint8))
        obs, ref, rew, term = out
        vp = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
        K.check(self._lib.gemb200_step_host(self._h, vp(a), vp(obs), vp(ref) if self.n_ref else None, vp(rew), vp(term)), "gemb200_step_host")
        return out

    def step_host_ptr(self, a_ptr, obs_ptr, ref_ptr, rew_ptr, term_ptr):
        """Raw-pointer variant for pinned torch host tensors (bench e2e leg)."""
        K.check(self._lib.gemb200_step_host(self._h, a_ptr, obs_ptr, ref_ptr, rew_ptr, term_ptr), "gemb200_step_host")

    def reset_host(self, mask=None):
        obs = np.zeros(self._shape(self.n_state), self.np_dtype)
        ref = np.zeros(self._shape(self.n_ref), self.np_dtype)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        vp = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)  # noqa: E731
        K.check(self._lib.gemb200_reset_host(self._h, vp(m), vp(obs), vp(ref) if self.n_ref else None), "gemb200_reset_host")
        return obs, ref

    # ------------------------------------------------------------------ state access
    def get_ode_state(self):
        out = torch.empty((self.n, self.n_ode), dtype=torch.float64, device=self.device)
        K.check(self._lib.gemb200_get_ode_state(self._h, _ptr(out), self._stream()), "gemb200_get_ode_state")
        return out

    def set_ode_state(self, y):
        y = torch.as_tensor(y, dtype=torch.float64, device=self.device).reshape(self.n, self.n_ode).contiguous()
        K.check(self._lib.gemb200_set_ode_state(self._h, _ptr(y), self._stream()), "gemb200_set_ode_state")
        torch.cuda.current_stream(self.device).synchronize()  # y may be a temporary

    def get_reference(self):
        out = torch.empty((self.n, self.n_ref), dtype=torch.float64, device=self.device)
        if self.n_ref:
            K.check(self._lib.gemb200_get_reference(self._h, _ptr(out), self._stream()), "gemb200_get_reference")
        return out

    def set_reference(self, r):
        if not self.n_ref:
            return
        r = torch.as_tensor(r, dtype=torch.float64, device=self.device).reshape(self.n, self.n_ref).contiguous()
        K.check(self._lib.gemb200_set_reference(self._h, _ptr(r), self._stream()), "gemb200_set_reference")
        torch.cuda.current_stream(self.device).synchronize()

    def state_dict(self):
        self._refuse_while_drawing("state_dict")
        self._refuse_with_identities("state_dict")
        size = self._lib.gemb200_checkpoint_size(self._h)
        buf = np.empty(size, dtype=np.uint8)
        K.check(self._lib.gemb200_checkpoint_save(self._h, buf.ctypes.data_as(C.c_void_p)), "gemb200_checkpoint_save")
        return {"blob": buf}

    def load_state_dict(self, sd):
        self._refuse_while_drawing("load_state_dict")
        self._refuse_with_identities("load_state_dict")
        buf = np.ascontiguousarray(sd["blob"], dtype=np.uint8)
        if buf.size != self._lib.gemb200_checkpoint_size(self._h):
            raise ValueError("checkpoint size mismatch")
        K.check(self._lib.gemb200_checkpoint_load(self._h, buf.ctypes.data_as(C.c_void_p)), "gemb200_checkpoint_load")

    # ------------------------------------------------------------------ per-env snapshots (snapshot.py)
    def record_layout(self):
        """(words per env of a packed record, layout id) of this handle's configuration (gemb200_query_env_record)"""
        if getattr(self, "_record", None) is None:
            w, lid = C.c_int32(), C.c_uint64()
            K.check(self._lib.gemb200_query_env_record(C.byref(self.cfg), C.byref(w), C.byref(lid)), "gemb200_query_env_record")
            self._record = (int(w.value), int(lid.value))
        return self._record

    def _dev_index(self, idx):
        if idx is None:
            return None
        t = idx if isinstance(idx, torch.Tensor) else torch.as_tensor(np.asarray(idx, dtype=np.int64).reshape(-1))
        return t.to(device=self.device, dtype=torch.int32).reshape(-1).contiguous()

    def snapshot(self, idx=None, rng=False, params=False):
        """Pack the persistent state of envs `idx` (None: all) into an EnvSnapshot (gemb200_pack_envs; stream-ordered, no host sync).
        Row j holds env idx[j]; a device index entry out of range leaves its row uninitialised.  rng=True also packs the envs' effective
        RNG identities (gemb200_pack_rng_ids) into `snap.rng`, for restore(..., rng="source").  params=True also packs their physical
        parameters (gemb200_pack_envs_params) into `snap.params`, for restore(..., params="source"); allowed while parameters are drawn."""
        from .snapshot import EnvSnapshot, check_params_layout

        if params:
            check_params_layout(self.soa)
        else:
            self._refuse_while_drawing("snapshot")
        words, lid = self.record_layout()
        ii = self._dev_index(idx)
        m = self.n if ii is None else int(ii.numel())
        rows = torch.empty((m, words), dtype=torch.int32, device=self.device)
        prm = None
        if params:
            prm = torch.empty((m, K.ENV_PARAM_SLOTS), dtype=torch.float64, device=self.device)
            K.check(self._lib.gemb200_pack_envs_params(self._h, _ptr(ii), m, _ptr(rows), _ptr(prm), self._stream()), "gemb200_pack_envs_params")
        else:
            K.check(self._lib.gemb200_pack_envs(self._h, _ptr(ii), m, _ptr(rows), self._stream()), "gemb200_pack_envs")
        ids = None
        if rng:
            ids = torch.empty((m, K.RNG_ID_WORDS), dtype=torch.int32, device=self.device)
            K.check(self._lib.gemb200_pack_rng_ids(self._h, _ptr(ii), m, _ptr(ids), self._stream()), "gemb200_pack_rng_ids")
        return EnvSnapshot(rows, lid, self.dtype, ids, prm, float(self.cfg.motor_param[K.MP_P]) if params else None)

    def clear_rng_ids(self):
        """every env draws with its own RNG identity again (gemb200_clear_rng_ids; stream-ordered)"""
        K.check(self._lib.gemb200_clear_rng_ids(self._h, self._stream()), "gemb200_clear_rng_ids")
        self._ids_adopted = False

    def restore(self, snap, idx=None, rows=None, rng="own", params="own"):
        """Env idx[j] (None: j) takes the state of snapshot row rows[j] (None: j) (gemb200_unpack_envs; stream-ordered, no host sync).
        `rows` fans one snapshot out: restore(snap, idx=range(C * m), rows=np.repeat(range(m), C)) copies every row into C envs.
        Device index entries out of range are skipped.  rng="own": the envs draw their own random numbers from then on; rng="source": they
        adopt the snapshot's RNG identities (gemb200_adopt_rng_ids) and repeat their sources' draws.  params="own": the envs keep their
        physical parameters; params="source": they take the snapshot's (gemb200_unpack_envs_params, one call with the state and, with
        rng="source", the identities), which is allowed while parameters are drawn per reset."""
        from .snapshot import check_layout, check_params_mode, check_rng_mode

        take = check_params_mode(snap, params, self.soa, self.cfg.motor_param[K.MP_P])
        if not take:
            self._refuse_while_drawing("restore")
        words, lid = self.record_layout()
        check_layout(snap, words, lid)
        adopt = check_rng_mode(snap, rng, self.soa)
        ii, rr = self._dev_index(idx), self._dev_index(rows)
        if ii is not None and rr is not None and ii.numel() != rr.numel():
            raise ValueError(f"idx ({ii.numel()}) and rows ({rr.numel()}) must have the same length")
        m = int(ii.numel()) if ii is not None else (int(rr.numel()) if rr is not None else min(len(snap), self.n))
        if snap.rows.device != self.device or (adopt and snap.rng.device != self.device) or (take and snap.params.device != self.device):
            raise ValueError(f"snapshot rows are on {snap.rows.device}, this handle on {self.device}: move the rows first")
        data = snap.rows.contiguous()
        if take:
            prm = snap.params.contiguous()
            ids = snap.rng.contiguous() if adopt else None
            K.check(self._lib.gemb200_unpack_envs_params(self._h, _ptr(data), _ptr(prm), _ptr(ids), len(snap), C.c_uint64(lid), _ptr(rr), _ptr(ii), m,
                                                         self._stream()), "gemb200_unpack_envs_params")
            if adopt:
                self._ids_adopted = True
            return
        K.check(self._lib.gemb200_unpack_envs(self._h, _ptr(data), len(snap), C.c_uint64(lid), _ptr(rr), _ptr(ii), m, self._stream()),
                "gemb200_unpack_envs")
        if adopt:
            ids = snap.rng.contiguous()
            K.check(self._lib.gemb200_adopt_rng_ids(self._h, _ptr(ids), len(snap), _ptr(rr), _ptr(ii), m, self._stream()), "gemb200_adopt_rng_ids")
            self._ids_adopted = True

    # ------------------------------------------------------------------ measurement helpers
    @property
    def launch_count(self):
        return int(self._lib.gemb200_launch_count(self._h))

    def time_begin(self):
        K.check(self._lib.gemb200_kernel_time_begin(self._h, self._stream()))

    def time_end(self):
        ms = C.c_float()
        K.check(self._lib.gemb200_kernel_time_end(self._h, self._stream(), C.byref(ms)))
        return ms.value
