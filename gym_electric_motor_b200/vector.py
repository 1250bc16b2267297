"""`gymnasium.vector`-style facade over the batched environment (SURVEY.md §8f row 4).

    venv = gem.vector.make_vec("Cont-CC-PMSM-v0", num_envs=1 << 16)
    obs, info = venv.reset(seed=0)
    obs, rewards, terminations, truncations, infos = venv.step(actions)

Follows gymnasium's VectorEnv conventions: `num_envs`, `single_observation_space` / `single_action_space`, batched
`observation_space` / `action_space`, `AutoresetMode.SAME_STEP` semantics (a terminated env is reset inside the same step and
the returned observation is the first one of the new episode — done in-kernel).  Observations are the reference's tuple
`(state, reference)`; `flatten_obs=True` concatenates them to one `[N, n_state + n_ref]` tensor for learners that want a Box.
"""
import numpy as np

from .envs import make
from .spaces import Box, Tuple


def _batch_box(space, n):
    return Box(np.repeat(space.low[None], n, axis=0), np.repeat(space.high[None], n, axis=0), dtype=space.dtype)


class GemVectorEnv:
    metadata = {"autoreset_mode": "same_step"}

    def __init__(self, env_id, num_envs, flatten_obs=False, **kwargs):
        kwargs.setdefault("autoreset", "same_step")
        self.env = make(env_id, num_envs=num_envs, **kwargs)
        self.num_envs = int(num_envs)
        self.flatten_obs = bool(flatten_obs)
        state_space, ref_space = self.env.observation_space.spaces
        if self.flatten_obs:
            self.single_observation_space = Box(np.concatenate([state_space.low, ref_space.low]), np.concatenate([state_space.high, ref_space.high]),
                                                dtype=np.float32)
            self.observation_space = _batch_box(self.single_observation_space, self.num_envs)
        else:
            self.single_observation_space = self.env.observation_space
            self.observation_space = Tuple((_batch_box(state_space, self.num_envs), _batch_box(ref_space, self.num_envs)))
        self.single_action_space = self.env.action_space
        self.action_space = _batch_box(self.env.action_space, self.num_envs) if hasattr(self.env.action_space, "low") else self.env.action_space
        self.closed = False

    def _obs(self, state, ref):
        if not self.flatten_obs:
            return state, ref
        import torch

        return torch.cat([state, ref], dim=1)

    def reset(self, *, seed=None, options=None):
        (state, ref), info = self.env.reset(seed=seed, options=options)
        return self._obs(state, ref), info

    def step(self, actions, reference=None):
        """reference: this step's reference feed (ElectricMotorEnvironment.step), or None"""
        import torch

        (state, ref), reward, terminated, truncated, info = self.env.step(actions) if reference is None else self.env.step(actions, reference)
        truncations = torch.zeros_like(terminated)
        return self._obs(state, ref), reward, terminated, truncations, info

    def close(self):
        if not self.closed:
            self.env.close()
            self.closed = True

    @property
    def unwrapped(self):
        return self


def make_vec(env_id, num_envs, **kwargs):
    return GemVectorEnv(env_id, num_envs, **kwargs)
