"""Closed-loop control steps in a CUDA graph.

The reference's control loop is  `action = controller(state, reference); (state, reference), reward, terminated, ... = env.step(action)`
per step (core.py:328-371), i.e. at small N a sequence of launches whose cost is the host's submission path (Python -> ctypes -> launch),
not the kernels.  With pre-computed actions the fused rollout kernel removes that
(`env.rollout`); with a policy in the loop the remedy is a CUDA graph: K x (policy, env.step) captured once, replayed with one call.
What made a step uncapturable — every launch carrying its own clock (RNG call id, step count, dead-time ring position) in its kernel
parameters — is lifted by the device-resident clock of the C-ABI (`gemb200_set_device_clock`).
"""
import torch


class CapturedSteps:
    """`n_steps` closed-loop steps of a batched env, captured once, replayed by `replay()`.

    policy(state, reference) -> action tensor  ([N, n_act] float, or int32 switching states for finite converters); it is called
    `n_steps` times DURING CAPTURE ONLY, so it must consist of CUDA work on the current stream (torch ops / modules) without host
    synchronisation.  The first call sees `state0`, `reference0` (default: the env's current observation buffers, i.e. what the last
    reset / step returned).  After every `replay()` the attributes `state`, `reference`, `reward`, `terminated` hold the outputs of the
    last step (static tensors, overwritten by the next replay); with record=True `states`, `references`, `rewards`, `terminateds`
    hold all `n_steps` of them.  Bit-identical to running the same loop eagerly.

    references: a static reference feed [n_steps, N, n_ref] (SoA: [n_steps, n_ref, N]) in the env's dtype on its device.  Step k of every
    replay runs `env.step(action, reference=references[k])`, reading row k where the tensor stands at replay time: refill it in place
    between replays (never reallocate it) to track a new reference."""

    def __init__(self, env, policy, n_steps, record=False, warmup=1, references=None):
        if getattr(env, "_scalar", True):
            raise TypeError("CapturedSteps needs a batched environment (num_envs=...)")
        self.env, self.n_steps = env, int(n_steps)
        sim = env._ensure_sim()
        self._sim = sim
        self.reference_feed = None if references is None else sim._as_feed(references, self.n_steps)
        feed = (lambda k: None) if references is None else (lambda k: self.reference_feed[k])
        dev = sim.device
        obs, ref, _, _ = sim._alloc_outputs()
        if warmup:  # lazy initialisation inside the policy (cuBLAS workspaces, autotuning) must not happen during capture; the warm-up steps
            sd = sim.state_dict()  # are undone afterwards: records, clock, observation buffers
            o0, r0 = obs.clone(), ref.clone()
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                for j in range(int(warmup)):
                    (st, rf), _, _, _, _ = env.step(policy(env._filter(obs), ref), feed(j % self.n_steps))
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            sim.load_state_dict(sd)
            obs.copy_(o0)
            ref.copy_(r0)
            env._physical_system._k -= int(warmup)
        env._filter(obs)  # builds the state-filter index (a host-to-device copy) outside the capture
        sim.set_device_clock(True)
        self.graph = torch.cuda.CUDAGraph()
        rec = [] if record else None
        with torch.cuda.graph(self.graph):
            st, rf = env._filter(obs), ref
            for k in range(self.n_steps):
                (st, rf), rw, tm, _, _ = env.step(policy(st, rf), feed(k))
                if record:
                    rec.append((st.clone(), rf.clone(), rw.clone(), tm.clone()))
        env._physical_system._k -= self.n_steps  # capture ran the host side of env.step without executing anything
        self.state, self.reference, self.reward, self.terminated = st, rf, rw, tm
        if record:
            self.states, self.references, self.rewards, self.terminateds = ([r[q] for r in rec] for q in range(4))

    def replay(self):
        """run the captured steps once more from the env's current state (stream-ordered on the current stream)"""
        if self.graph is None:
            raise RuntimeError("CapturedSteps.replay() after release(): the captured launches read the device-resident clock, which is off")
        self.graph.replay()
        self.env._physical_system._k += self.n_steps
        return (self.state, self.reference), self.reward, self.terminated

    def release(self):
        """back to host-clocked launches (reads the clock back: synchronises)"""
        self._sim.set_device_clock(False)
        self.graph = None
