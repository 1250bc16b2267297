"""Batched `ElectricMotorEnvironment` — the drop-in for reference core.py:53-392.

`reset()` / `step()` keep the reference's return structure
    reset -> ((state, reference_observation), info)
    step  -> ((state, reference_observation), reward, terminated, truncated, info)
with a leading env dimension N on every array (torch tensors on the CUDA device).  With `num_envs=None` the
environment runs ONE env and converts to the reference's scalar contract (numpy vectors, float reward, bool
terminated, assertion on stepping a terminated env, core.py:341).

The whole step — physical system, reference lookup, constraint check, reward, next reference — is one CUDA launch
through the C-ABI (include/gemb200.h: gemb200_step); see DESIGN.md.
"""
import numpy as np
import torch

from . import _cabi as K
from .constraints import Constraint, ConstraintMonitor
from .reference_generators import ReferenceGenerator
from .reward_functions import RewardFunction
from .spaces import Box, Tuple

try:  # a gymnasium.Env when gymnasium is installed, so that gymnasium.Wrapper / TimeLimit / FlattenObservation accept the scalar env
    from gymnasium import Env as _EnvBase  # pragma: no cover - this image has no gymnasium
except ImportError:
    _EnvBase = object


class Callback:
    """reference core.py:708-740 (hooks receive batched tensors)"""

    _env = None

    def set_env(self, env):
        self._env = env

    def on_reset_begin(self):
        pass

    def on_reset_end(self, state, reference):
        pass

    def on_step_begin(self, k, action):
        pass

    def on_step_end(self, k, state, reference, reward, terminated):
        pass

    def on_close(self):
        pass


class ElectricMotorVisualization(Callback):
    """reference core.py:743-753.  Plotting is host-side and out of scope; subclasses may still hook in."""

    def render(self):
        pass


class ElectricMotorEnvironment(_EnvBase):
    """See module docstring.  Constructor signature follows reference core.py:197-209 plus the batch options
    `num_envs`, `autoreset` ('same_step' | None), `seed`."""

    metadata = {}
    render_mode = None
    env_id = None

    def __init__(self, physical_system, reference_generator, reward_function, visualization=(), state_filter=None, callbacks=(),
                 constraints=(), physical_system_wrappers=(), scale_plots=False, num_envs=None, autoreset=None, seed=None, **kwargs):
        physical_system.apply_wrappers(tuple(physical_system_wrappers))  # fused into the kernel (physical_system_wrappers.py)
        if not isinstance(reference_generator, ReferenceGenerator):
            raise TypeError("reference_generator must be a built-in gym_electric_motor_b200 ReferenceGenerator")
        if not isinstance(reward_function, RewardFunction):
            raise TypeError("reward_function must be a built-in gym_electric_motor_b200 RewardFunction")
        self._scalar = num_envs is None
        if self._scalar and getattr(physical_system, "_layout", K.LAYOUT_AOS) == K.LAYOUT_SOA:
            raise ValueError("layout='soa' needs a batched environment (num_envs=...): the scalar contract returns one row per step")
        self._physical_system = physical_system
        self._reference_generator = reference_generator
        self._reward_function = reward_function
        self.num_envs = physical_system.num_envs
        if isinstance(constraints, ConstraintMonitor):
            cm = constraints
        else:
            limit_constraints = [c for c in constraints if isinstance(c, str)]
            additional = [c for c in constraints if isinstance(c, Constraint)]
            bad = [c for c in constraints if not isinstance(c, (str, Constraint))]
            if bad:
                raise TypeError("callable constraints are host code and cannot be fused into the kernel epilogue")
            cm = ConstraintMonitor(limit_constraints, additional)
        self._constraint_monitor = cm
        self._reference_generator.set_modules(self._physical_system)
        self._constraint_monitor.set_modules(self._physical_system)
        self._reward_function.set_modules(self._physical_system, self._reference_generator, self._constraint_monitor)
        ps = self._physical_system
        state_filter = state_filter or ps.state_names
        self.state_filter = [ps.state_names.index(s) for s in state_filter]
        self._filter_identity = self.state_filter == list(range(len(ps.state_names)))
        state_space = Box(ps.state_space.low[self.state_filter], ps.state_space.high[self.state_filter], dtype=np.float64)
        self.observation_space = Tuple((state_space, self._reference_generator.reference_space))
        self.action_space = ps.action_space
        self.reward_range = self._reward_function.reward_range
        self._terminated = True
        self._truncated = False
        self.scale_plots = scale_plots
        if isinstance(visualization, ElectricMotorVisualization):
            visualization = [visualization]
        self._visualizations = [v for v in (visualization or []) if isinstance(v, ElectricMotorVisualization)]
        self._callbacks = list(callbacks) + list(self._visualizations)
        if not self._visualizations:  # the reference's envs default to a MotorDashboard (user code reads env.visualizations[0]); here an
            from .visualization import MotorDashboard  # inert one that is not even registered as a callback (nothing to call per step)

            self._visualizations = [MotorDashboard(_quiet=True)]
        self._autoreset = K.AUTORESET_SAME_STEP if (autoreset in ("same_step", True, K.AUTORESET_SAME_STEP)) else K.AUTORESET_NONE
        self._seed_value = 0 if seed is None else int(seed)
        self._sim = None
        self._filter_index = None
        self._call_callbacks("set_env", self)

    # ------------------------------------------------------------------ reference-compatible properties
    @property
    def physical_system(self):
        return self._physical_system

    @property
    def reference_generator(self):
        return self._reference_generator

    @reference_generator.setter
    def reference_generator(self, reference_generator):
        """reference core.py:132-142: a new generator, then a reset is required.  Here the generator is part of the device handle's
        configuration, so the handle is dropped and rebuilt at the next reset."""
        if not isinstance(reference_generator, ReferenceGenerator):
            raise TypeError("reference_generator must be a built-in gym_electric_motor_b200 ReferenceGenerator")
        self._reference_generator = reference_generator
        self._reference_generator.set_modules(self._physical_system)
        self._reward_function.set_modules(self._physical_system, self._reference_generator, self._constraint_monitor)
        self.observation_space = Tuple((self.observation_space.spaces[0], self._reference_generator.reference_space))
        self._drop_handle()

    @property
    def reward_function(self):
        return self._reward_function

    @reward_function.setter
    def reward_function(self, reward_function):
        """reference core.py:153-162"""
        if not isinstance(reward_function, RewardFunction):
            raise TypeError("reward_function must be a built-in gym_electric_motor_b200 RewardFunction")
        self._reward_function = reward_function
        self._reward_function.set_modules(self._physical_system, self._reference_generator, self._constraint_monitor)
        self.reward_range = self._reward_function.reward_range
        self._drop_handle()

    def _drop_handle(self):
        self._terminated = True
        if self._sim is not None:
            self._sim.close()
            self._sim = None
            self._physical_system.attach(None)

    @property
    def constraint_monitor(self):
        return self._constraint_monitor

    @property
    def visualizations(self):
        """reference core.py:140-143 (agents look for a MotorDashboard in this list)"""
        return self._visualizations

    @property
    def limits(self):
        """limits of the states the env returns, i.e. after the state filter (reference core.py:169-174)"""
        return self._physical_system.limits[self.state_filter]

    @property
    def state_names(self):
        return [self._physical_system.state_names[s] for s in self.state_filter]

    @property
    def reference_names(self):
        return self._reference_generator.reference_names

    @property
    def nominal_state(self):
        return self._physical_system.nominal_state[self.state_filter]

    @property
    def unwrapped(self):
        return self

    @property
    def sim(self):
        """The underlying device handle wrapper (VectorSim)."""
        return self._ensure_sim()

    # ------------------------------------------------------------------ device handle
    def build_config(self):
        cfg = self._physical_system.fill_config(K.new_config())
        self._constraint_monitor.fill_config(cfg)
        self._reward_function.fill_config(cfg)
        self._reference_generator.fill_config(cfg)
        cfg.autoreset = self._autoreset
        cfg.seed = self._seed_value & 0xFFFFFFFFFFFFFFFF
        return cfg

    def _ensure_sim(self):
        if self._sim is None:
            from .vector_sim import VectorSim

            self._sim = VectorSim(self.build_config())
            self._physical_system.attach(self._sim)
        return self._sim

    def _call_callbacks(self, func_name, *args):
        for callback in self._callbacks:
            getattr(callback, func_name)(*args)

    def _filter(self, obs):
        if self._filter_identity:
            return obs
        import torch

        if self._filter_index is None:
            self._filter_index = torch.as_tensor(self.state_filter, device=obs.device)
        dim = 0 if self._sim.soa else 1
        return obs.index_select(dim, self._filter_index)

    # ------------------------------------------------------------------ gym API
    def reset(self, seed=None, options=None, mask=None, *_, **__):
        """core.py:300-319.  `seed` re-keys the device RNG streams (new handle state); `mask` (batched mode only)
        resets a subset of envs and returns the full observation tensors."""
        reseed = seed is not None and self._sim is not None
        if seed is not None:
            self._seed_value = int(seed)
        sim = self._ensure_sim()
        if reseed:  # the reference re-seeds every component on EVERY seeded reset (core.py:300-304): equal seeds, identical episodes
            sim.reseed(self._seed_value)
        self._call_callbacks("on_reset_begin")
        obs, ref = sim.reset(mask)
        self._terminated = False
        self._physical_system._k = 0
        state = self._filter(obs)
        self._call_callbacks("on_reset_end", state, ref)
        if self._scalar:
            return (state.double().cpu().numpy()[0], ref.double().cpu().numpy()[0]), {}
        return (state, ref), {}

    def step(self, action, reference=None):
        """core.py:328-371.  reference (batched mode only): this step's reference feed, [N, n_ref] (SoA: [n_ref, N]) in the env's dtype on
        its device.  It overwrites the stored value of EVERY reference slot before the step, exactly like `set_reference(reference)` before
        `step(action)`, but in the step's own launch: no host synchronisation, so a captured closed loop (`capture_steps(...,
        references=...)`) can track a caller-given reference.  Wrong shape, dtype or device: ValueError."""
        if reference is not None and self._scalar:
            raise TypeError("step(action, reference=...) needs a batched environment (num_envs=...); a scalar env takes set_reference()")
        sim = self._ensure_sim()
        if self._scalar:
            assert not self._terminated, "A reset is required before the environment can perform further steps"
            if not hasattr(self.action_space, "low"):  # finite converters assert their action (converters.py:204-206, :356-358, :827-829)
                candidate = np.asarray(action)
                candidate = int(candidate.reshape(-1)[0]) if candidate.size == 1 and hasattr(self.action_space, "n") else candidate.reshape(-1)
                assert self.action_space.contains(candidate), \
                    f"The selected action {action} is not a valid element of the action space {self.action_space}."
            action = np.asarray(action).reshape(1, -1)
        if self._callbacks:
            self._call_callbacks("on_step_begin", self._physical_system.k, action)
        obs, ref, reward, terminated = sim.step(action) if reference is None else sim.step(action, reference)
        self._physical_system._k += 1
        state = obs if self._filter_identity else self._filter(obs)
        if self._callbacks:
            self._call_callbacks("on_step_end", self._physical_system.k, state, ref, reward, terminated)
        if self._scalar:
            term = bool(terminated[0].item())
            self._terminated = term and self._autoreset == K.AUTORESET_NONE
            return (state.double().cpu().numpy()[0], ref.double().cpu().numpy()[0]), float(reward[0].item()), term, self._truncated, {}
        return (state, ref), reward, terminated.view(torch.bool), self._truncated, {}  # uint8 0/1 reinterpreted, no kernel

    def rollout(self, actions, record_every=1, references=None):
        """K consecutive `step` calls with pre-computed actions [K, N, n_act] in ONE kernel launch (open loop; bit-identical to calling
        `step` K times, core.py:328-371).  Returns ((states, references), rewards, terminateds) with a leading axis of K // record_every
        recorded steps (record_every = 0: only the last step, without the leading axis).  Batched mode only; callbacks see no
        per-step hooks.
        references: a reference feed [K, N, n_ref] (SoA: [K, n_ref, N]) in the env's dtype on its device — a drive cycle, a test profile,
        a recorded trajectory or the known future reference of an MPC horizon.  Step k first overwrites the stored value of EVERY reference
        slot (not only the ExternalReferenceGenerator ones) with references[k]: the result is exactly that of K iterations of
        `set_reference(references[k]); step(actions[k])`.  The returned reference of step k is what that loop returns: for an External
        slot the value step k was scored against (the reset value on an env that was auto-reset in step k).  A policy that needs a preview
        reads it from `references` itself.  Wrong shape, dtype, device or K: ValueError."""
        if self._scalar:
            raise TypeError("rollout() needs a batched environment (num_envs=...)")
        sim = self._ensure_sim()
        obs, ref, reward, terminated = sim.rollout(actions, record_every) if references is None else sim.rollout(actions, record_every, references)
        k = int(actions.shape[0]) if hasattr(actions, "shape") else len(actions)
        self._physical_system._k += k
        if not self._filter_identity:
            if self._filter_index is None:
                self._filter_index = torch.as_tensor(self.state_filter, device=obs.device)
            dim = (0 if sim.soa else 1) + (1 if record_every else 0)
            obs = obs.index_select(dim, self._filter_index)
        return (obs, ref), reward, terminated.view(torch.bool)

    def rollout_returns(self, actions, discount=1.0, references=None):
        """Score an action sequence: K steps with pre-computed actions [K, N, n_act] (SoA: [K, n_act, N]) in ONE kernel launch that hands
        back each env's discounted return instead of its per-step rewards.  Returns (returns, end_step, (state, reference)):
        end_step: int32 [N], the index of each env's first terminated step, K if it does not terminate within the launch;
        returns: [N] in the env's dtype, sum of discount^k * reward_k over the steps up to and including that first termination (the
        violation reward counts, nothing after it does, whatever the autoreset mode makes of the env afterwards);
        (state, reference): the last step's outputs as `rollout(actions, record_every=0)` returns them, to bootstrap the envs with
        end_step == K.  The env ends in exactly the state of `rollout(actions, references=references)`.  discount: finite, in [0, 1].
        references: the reference feed of `rollout`.  Batched mode only; bad actions, discount or feed: ValueError before any launch."""
        if self._scalar:
            raise TypeError("rollout_returns() needs a batched environment (num_envs=...)")
        sim = self._ensure_sim()
        ret, end, (obs, ref) = sim.rollout_returns(actions, discount, references)
        self._physical_system._k += int(actions.shape[0])
        if not self._filter_identity:
            if self._filter_index is None:
                self._filter_index = torch.as_tensor(self.state_filter, device=obs.device)
            obs = obs.index_select(0 if sim.soa else 1, self._filter_index)
        return ret, end, (obs, ref)

    def rollout_jacobians(self, actions, references=None):
        """Linearise the plant along an action sequence: K steps with pre-computed actions [K, N, n_act] in ONE kernel launch that also
        returns, per step k and env i, jac_x[k, i] = d x_{k+1} / d x_k ([n_x, n_x]) and jac_u[k, i] = d x_{k+1} / d a_k ([n_x, n_u]; None
        for finite converters).  x is the ODE state of `get_ode_state` ([load states | motor states], the angle last, in radians), a the
        action as passed to `step`.  Returns ((jac_x, jac_u), ((states, references), rewards, terminateds)), the second part exactly as
        `rollout(actions, record_every=1, references=references)` returns it; the env ends in that call's state.  A terminating step reports
        the Jacobian of the physical step it took.  `calc_jacobian` does not switch this on or off.  Refused configurations (dead time, RC
        supply, dq actions on the observer angle, SoA): NotImplementedError (DESIGN.md §7).
        Batched mode only; bad actions or feed: ValueError before any launch."""
        if self._scalar:
            raise TypeError("rollout_jacobians() needs a batched environment (num_envs=...)")
        sim = self._ensure_sim()
        (jx, ju), (obs, ref, reward, terminated) = sim.rollout_jacobians(actions, references)
        self._physical_system._k += int(actions.shape[0])
        if not self._filter_identity:
            if self._filter_index is None:
                self._filter_index = torch.as_tensor(self.state_filter, device=obs.device)
            obs = obs.index_select(2, self._filter_index)
        return (jx, ju), ((obs, ref), reward, terminated.view(torch.bool))

    def rollout_return_grads(self, actions, discount=1.0, references=None, value_grad=None):
        """Score an action sequence and differentiate the score: `rollout_returns` plus, from the same launch, grad_a [K, N, n_u] =
        d returns[i] / d a_k[i] (a = the action as passed to `step`, dq actions included; exactly 0 for k >= end_step[i]) and grad_x0 [N, n_x]
        = d returns[i] / d x_0[i] (x = the ODE state of `get_ode_state`, the angle last, in radians).  Returns (returns, end_step,
        (state, reference), grad_a, grad_x0), the first three as `rollout_returns(actions, discount, references)` returns them; the env
        ends in that call's state.  value_grad [N, n_x] (env dtype): the gradient of a bootstrap value V(x_K), added as discount^K *
        value_grad[i] to the adjoint of the envs with end_step == K (returns itself does not include V).  Non-smooth points take the
        one-sided derivative of the branch the step took, and termination has derivative 0: the gradient does not see a constraint a
        perturbed sequence would hit (DESIGN.md §7).  Refused configurations (those of `rollout_jacobians`, finite converters, a reward on
        an entry a state wrapper appends): NotImplementedError.  Batched mode only; bad actions, discount, feed or value_grad: ValueError
        before any launch."""
        if self._scalar:
            raise TypeError("rollout_return_grads() needs a batched environment (num_envs=...)")
        sim = self._ensure_sim()
        ret, end, (obs, ref), ga, gx = sim.rollout_return_grads(actions, discount, references, value_grad)
        self._physical_system._k += int(actions.shape[0])
        if not self._filter_identity:
            if self._filter_index is None:
                self._filter_index = torch.as_tensor(self.state_filter, device=obs.device)
            obs = obs.index_select(1, self._filter_index)
        return ret, end, (obs, ref), ga, gx

    def differentiable_returns(self, actions, discount=1.0, references=None):
        """`rollout_returns(actions, discount, references)[0]` as a torch autograd function of `actions`: the forward pass runs ONE
        `rollout_return_grads` launch and ADVANCES the env by K steps like `rollout_returns`; the backward pass returns
        grad_output[None, :, None] * grad_a.  So an action sequence that is an `nn.Parameter`, or the output of a policy, can be optimised
        with a torch optimiser.  Every call starts from the env's current state: to evaluate the same start again, branch the envs first
        (`snapshot_envs`) and put them back with `restore_envs(..., rng="source")` before the next call."""
        if self._scalar:
            raise TypeError("differentiable_returns() needs a batched environment (num_envs=...)")
        if not isinstance(actions, torch.Tensor):
            raise ValueError(f"actions must be a torch tensor, got {type(actions).__name__}")
        return _DifferentiableReturns.apply(actions, self, discount, references)

    def param_slots(self, params):
        """The parameter-row slots of the names `params` (the names of `set_env_parameters`): KeyError for an unknown name, ValueError for
        the pole pairs `p`, the EESM's `k` (DESIGN.md §7), an empty list or a parameter named twice (`r_r` is `r_e`)."""
        if isinstance(params, str):
            params = [params]
        slots = []
        for name in params:
            if name in self._MP_SLOT:
                if name in ("p", "k"):
                    raise ValueError(f"parameter sensitivities with respect to {name!r} are not provided: "
                                     + ("the angle increments are prepared per env handle" if name == "p" else "the EESM's coefficients are invariant in k")
                                     + " (DESIGN.md §7)")
                slot = self._MP_SLOT[name]
            elif name in self._LP_SLOT:
                slot = K.MAX_MOTOR_PARAM + self._LP_SLOT[name]
            else:
                raise KeyError(f"unknown parameter {name!r}")
            if slot in slots:
                raise ValueError(f"parameter {name!r} is named twice")
            slots.append(slot)
        if not 1 <= len(slots) <= 12:
            raise ValueError(f"parameter sensitivities take 1 to 12 parameters, got {len(slots)}")
        return slots

    def rollout_param_sensitivities(self, actions, params, references=None, sens0=None, record=True):
        """Parameter sensitivities along an action sequence: K steps with pre-computed actions [K, N, n_act] in ONE kernel launch that also
        carries, per env i, S = d x / d theta[i] with respect to the env's OWN physical parameters `params` (a list of the names
        `set_env_parameters` takes; `p` and `k` are refused).  x is the ODE state of `get_ode_state` (the angle last, in radians).  Returns
        ((sens, sens_last), ((states, references), rewards, terminateds)): sens [K, N, n_x, n_p] = d x_{k+1} / d theta after every step
        (None when record=False), sens_last [N, n_x, n_p] the carried S after the last step, to pass as `sens0` of the next call; the second
        part exactly as `rollout(actions, record_every=1, references=references)` returns it, and the env ends in that call's state.  sens0:
        S at the start (None: zeros, the sensitivity of the trajectory from the current state).  A terminating step reports the sensitivity
        of the physical step it took; an env auto-reset in it carries S = 0 from there.  Refused configurations (those of
        `rollout_jacobians`) and parameter draws at resets: NotImplementedError (DESIGN.md §7).  Batched mode only; bad actions, feed or
        sens0: ValueError before any launch."""
        if self._scalar:
            raise TypeError("rollout_param_sensitivities() needs a batched environment (num_envs=...)")
        slots = self.param_slots(params)
        sim = self._ensure_sim()
        if getattr(self, "_randomized_names", ()):
            raise NotImplementedError("parameter sensitivities are refused while parameter draws at resets are on (DESIGN.md §7)")
        (so, sl), (obs, ref, reward, terminated) = sim.rollout_param_sens(actions, slots, references, sens0, record)
        self._physical_system._k += int(actions.shape[0])
        if not self._filter_identity:
            if self._filter_index is None:
                self._filter_index = torch.as_tensor(self.state_filter, device=obs.device)
            obs = obs.index_select(2, self._filter_index)
        return (so, sl), ((obs, ref), reward, terminated.view(torch.bool))

    def capture_steps(self, policy, n_steps, record=False, warmup=1, references=None):
        """`n_steps` closed-loop steps — action = policy(state, reference); env.step(action) — captured ONCE in a CUDA graph (graph.py);
        `.replay()` of the returned object runs them with a single call.  Batched mode only.  references: a static reference feed
        [n_steps, N, n_ref] (SoA: [n_steps, n_ref, N]); step k of every replay is `step(action, reference=references[k])`, so refilling
        the tensor in place between replays makes the next replay track the new values."""
        from .graph import CapturedSteps

        return CapturedSteps(self, policy, n_steps, record=record, warmup=warmup, references=references)

    _MP_SLOT = dict(p=K.MP_P, r_s=K.MP_R_S, l_d=K.MP_L_D, l_q=K.MP_L_Q, psi_p=K.MP_PSI_P, j_rotor=K.MP_J_ROTOR, r_a=K.MP_R_A, l_a=K.MP_L_A, psi_e=K.MP_PSI_E,
                    r_e=K.MP_R_E, l_e=K.MP_L_E, l_e_prime=K.MP_L_E_PRIME, l_m=K.MP_L_M, k=K.MP_K, l_sigs=K.MP_L_SIGS, l_sigr=K.MP_L_SIGR, r_r=K.MP_R_E)
    _LP_SLOT = dict(a=K.LP_A, b=K.LP_B, c=K.LP_C, j_load=K.LP_J_LOAD)

    def set_env_parameters(self, motor_parameter=None, load_parameter=None):
        """Domain randomisation: give every env of the batch its own physical parameters — the batched counterpart of constructing N
        reference envs with N `motor_parameter` / `load_parameter` dicts (electric_motor.py:118-131, polynomial_static_load.py:46-64).
        Both arguments are dicts  name -> array of N values  with the reference's parameter names (`r_s`, `l_d`, `psi_p`, `j_rotor`, ...;
        `a`, `b`, `c`, `j_load`); parameters that are not named keep the value the env was made with.  Limits, nominal values and the
        normalisation stay those of the env.  `set_env_parameters()` without arguments returns to the shared parameters.  Pole pairs `p` may
        be named only with the env's own value (ValueError otherwise: the angle increments are prepared per handle); the flux limits of an
        induction motor's random initial states and the FluxObserver's constants stay those of the env's nominal motor (DESIGN.md §7)."""
        if self._scalar:
            raise TypeError("set_env_parameters() needs a batched environment (num_envs=...)")
        sim = self._ensure_sim()
        if not motor_parameter and not load_parameter:
            sim.set_env_params(None, None)
            return
        cfg = sim.cfg
        mp = np.tile(np.array(list(cfg.motor_param), dtype=np.float64), (sim.n, 1))
        lp = np.tile(np.array(list(cfg.load_param), dtype=np.float64), (sim.n, 1))
        for name, vals in (motor_parameter or {}).items():
            if name not in self._MP_SLOT:
                raise KeyError(f"unknown motor parameter {name!r}")
            mp[:, self._MP_SLOT[name]] = np.broadcast_to(np.asarray(vals, dtype=np.float64), (sim.n,))
        for name, vals in (load_parameter or {}).items():
            if name not in self._LP_SLOT:
                raise KeyError(f"unknown load parameter {name!r}")
            lp[:, self._LP_SLOT[name]] = np.broadcast_to(np.asarray(vals, dtype=np.float64), (sim.n,))
        from .randomization import check_pole_pairs

        check_pole_pairs(mp[:, K.MP_P], cfg.motor_param[K.MP_P])
        sim.set_env_params(mp, lp)

    def randomize_env_parameters(self, motor_parameter=None, load_parameter=None):
        """Per-episode domain randomisation: from now on EVERY reset of an env — `reset()`, with or without a mask, and the in-kernel
        auto-reset of `step`, `rollout` and captured graphs — draws new values for the named parameters from the env's own random stream.
        Both arguments are dicts  name -> distribution  with the names of `set_env_parameters`; a distribution is `(lo, hi)` (uniform) or
        `("uniform" | "log_uniform", lo, hi)`.  A drawn value is rounded to the env's dtype; the new episode's dynamics and its reset
        observation use it.  Parameters that are not named keep their current value.  Draws are reproducible: equal seeds give equal
        sequences, independent of sharding.  The call itself draws nothing (the usual pattern is this call, then `reset()`);
        `randomize_env_parameters()` without arguments stops drawing and the envs keep their last values.  Pole pairs cannot be drawn
        (ValueError); nor, for induction motors with random initial states, the parameters of their flux limits (NotImplementedError).
        Needs the row-per-env (AoS) layout (ValueError).  While draws are on, checkpoints are refused, and so are snapshots and restores
        unless they carry the parameters (`snapshot_envs(..., params=True)`, `restore_envs(..., params="source")`; DESIGN.md §7)."""
        if self._scalar:
            raise TypeError("randomize_env_parameters() needs a batched environment (num_envs=...)")
        from .randomization import encode_distributions

        cfg = self._sim.cfg if self._sim is not None else self.build_config()
        if cfg.layout == K.LAYOUT_SOA and (motor_parameter or load_parameter):
            raise ValueError("per-env parameter draws need the row-per-env layout (layout='aos')")
        names, slots, kinds, lo, hi = encode_distributions(motor_parameter, load_parameter, self._MP_SLOT, self._LP_SLOT,
                                                           flux_limits=bool(cfg.init_im_valid))
        self._ensure_sim().set_param_randomization(slots, kinds, lo, hi)
        self._randomized_names = tuple(names)

    _randomized_names = ()

    def env_parameters(self):
        """{name: tensor[N]} on the device: the stored values (env dtype) of the parameters drawn at every reset."""
        sim = self._ensure_sim()
        if not sim.randomized_slots:
            return {}
        vals = sim.env_params()
        return {name: vals[j] for j, name in enumerate(self._randomized_names)}

    def snapshot_envs(self, idx=None, rng=False, params=False):
        """Branching support, the batched counterpart of `copy.deepcopy(env)`: the complete persistent state of envs `idx` (None: all;
        list, numpy array or tensor) as an `EnvSnapshot` of packed device rows, taken without a host synchronisation.  Host-side
        indices are range-checked (IndexError); a device index tensor is taken as given.  rng=True also takes the envs' RNG identities
        (seed, global index and where their random streams stand), which `restore_envs(..., rng="source")` hands on.  params=True also
        takes their physical parameters (`snap.params`, float64 [m, 24] in the slot order of `_cabi.MP_*`, then `MAX_MOTOR_PARAM + LP_*`:
        per-env values, drawn or set from the host, or the env's own), which `restore_envs(..., params="source")` hands on; it is allowed
        while parameters are drawn per reset and needs the row-per-env layout (ValueError).  Batched mode only."""
        if self._scalar:
            raise TypeError("snapshot_envs() needs a batched environment (num_envs=...)")
        from .snapshot import check_host_index, check_params_layout

        sim = self._ensure_sim()
        idx = check_host_index(idx, sim.n, "idx")
        if params:
            check_params_layout(sim.soa)
            return sim.snapshot(idx, rng=bool(rng), params=True)
        return sim.snapshot(idx, rng=True) if rng else sim.snapshot(idx)

    def clear_rng_identities(self):
        """Every env draws its own random numbers again (drops the identities adopted with `restore_envs(..., rng="source")`); afterwards
        the envs draw exactly what they would have drawn had they never adopted one, and the env runs its shared-coefficient kernels again
        unless it has per-env parameters of its own.  Batched mode only."""
        if self._scalar:
            raise TypeError("clear_rng_identities() needs a batched environment (num_envs=...)")
        self._ensure_sim().clear_rng_ids()

    def restore_envs(self, snapshot, idx=None, rows=None, rng="own", params="own"):
        """Env idx[j] (None: env j) takes the state of snapshot row rows[j] (None: row j): physically the source env, continuing bit for
        bit except for the random numbers, which by default (rng="own") are the restored env's own from then on (its Wiener increments,
        periodic-generator parameters, switching choices, noise and later random resets).  `rows` fans one snapshot out to many envs without copying it.
        The snapshot may come from another env of the same kind and record layout (other num_envs or seed); another layout raises
        ValueError, host-side indices out of range IndexError.  Returns nothing: the observation rows of the restored envs are the
        caller's to keep (the next step's outputs are computed from the restored state).  Batched mode only.
        rng="source" (a snapshot taken with rng=True) gives `copy.deepcopy(env)` semantics instead: every restored env adopts its source's
        RNG identity and repeats the source's random numbers — same actions, same outputs, bit for bit, across terminations and resets.
        A later restore with rng="own", `clear_rng_identities()` or `reset(seed=...)` drops the identity.  It needs the row-per-env layout
        (ValueError); while identities are adopted, `state_dict` / `load_state_dict` raise NotImplementedError (DESIGN.md §7).
        params="source" (a snapshot taken with params=True) gives every restored env its row's physical parameters: it runs its current
        episode on the source's plant, and with parameter draws on its next reset draws new values (with rng="source": the source's).  This
        is what branching domain-randomised envs needs, and it is allowed while parameters are drawn per reset.  The values of
        `snapshot.params` are used as given, so an edited copy restores an ensemble of plants; the pole-pair slot is ignored, and pole pairs
        differing from this env's raise ValueError.  Afterwards the env runs per-env parameter blocks (DESIGN.md §7)."""
        if self._scalar:
            raise TypeError("restore_envs() needs a batched environment (num_envs=...)")
        from .snapshot import check_host_index, check_layout, check_params_mode, check_rng_mode

        sim = self._ensure_sim()
        words, lid = sim.record_layout()
        check_layout(snapshot, words, lid)
        idx = check_host_index(idx, sim.n, "idx")
        rows = check_host_index(rows, len(snapshot), "rows")
        take = check_params_mode(snapshot, params, sim.soa, sim.cfg.motor_param[K.MP_P])
        adopt = check_rng_mode(snapshot, rng, sim.soa)
        if take:
            sim.restore(snapshot, idx, rows, rng="source" if adopt else "own", params="source")
        elif adopt:
            sim.restore(snapshot, idx, rows, rng="source")
        else:
            sim.restore(snapshot, idx, rows)

    def set_reference(self, values):
        """Push reference values [N, n_ref] for ExternalReferenceGenerator slots (used by the next step's reward)."""
        self._ensure_sim().set_reference(values)

    def state_dict(self):
        return self._ensure_sim().state_dict()

    def load_state_dict(self, sd):
        self._ensure_sim().load_state_dict(sd)

    def render(self, *_, **__):
        for v in self._visualizations:
            v.render()

    def close(self):
        self._call_callbacks("on_close")
        self._reward_function.close()
        self._reference_generator.close()
        if self._sim is not None:
            self._sim.close()
            self._sim = None
        self._physical_system.attach(None)


class _DifferentiableReturns(torch.autograd.Function):
    """returns = env.rollout_return_grads(actions, ...)[0]; d returns / d actions from the same launch"""

    @staticmethod
    def forward(ctx, actions, env, discount, references):
        ret, _, _, ga, _ = env.rollout_return_grads(actions.detach(), discount, references)
        ctx.save_for_backward(ga)
        return ret

    @staticmethod
    def backward(ctx, grad_output):
        (ga,) = ctx.saved_tensors
        return grad_output[None, :, None] * ga, None, None, None
