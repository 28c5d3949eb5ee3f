"""Vector adapter over the batched env (SURVEY.md section 8b item 4; reference `rl4rs/utils/rllib_vector_env.py:9-69`).

The reference wraps ONE batched `RecEnvBase` as an RLlib `VectorEnv` of `batch_size` sub-envs so that RLlib's sampler
can drive it.  ray is not part of this image and the GPU trainer does not need it (`rl4rs_b200.trainer` consumes the
batched env directly), so this class keeps the reference's method names and semantics without the ray base class:

* `vector_reset()`             -> `env.reset()`                                  (rllib_vector_env.py:26-32)
* `reset_at(i)`                -> resets the WHOLE batch when `i == 0`, serves row `i` of that cached reset otherwise
                                  (rllib_vector_env.py:34-45; RLlib resets finished sub-envs in index order)
* `vector_step(actions)`       -> `env.step(np.array(actions))`                  (rllib_vector_env.py:47-60)
* `get_unwrapped()`            -> the one underlying env repeated `num_envs` times (rllib_vector_env.py:62-68)
* `try_render_at(i)`           -> `env.render()`                                 (rllib_vector_env.py:71-77)
"""
import numpy as np


class MyVectorEnvWrapper(object):
    def __init__(self, env, batch_size):
        self.env = env
        self.reset_cache = []
        self.observation_space = env.observation_space
        self.action_space = env.action_space
        self.num_envs = batch_size

    def vector_reset(self):
        return self.env.reset()

    def reset_at(self, index=None):
        if index == 0:
            self.reset_cache = self.env.reset()
        return self.reset_cache[index]

    def vector_step(self, actions):
        return self.env.step(np.array(actions))

    def get_unwrapped(self):
        return [self.env, ] * self.num_envs

    def try_render_at(self, index=None):
        return self.env.render()
