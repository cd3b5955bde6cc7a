"""HistoryWrapper (reference go1_gym/envs/wrappers/history_wrapper.py:6-44): rolling window of the last
`num_observation_history` observations, produced by the go1_history_roll kernel (ping-pong buffers instead of
a fresh torch.cat allocation per step).  As in the reference the history is NOT cleared when an env resets.

Each buffer is [num_envs][capi.history_pitch(K0)] and obs_history is its [:, :K0] view (K0 = num_obs_history): contiguous when K0 is a
multiple of 4 floats, otherwise rows padded to a 16-byte multiple so that the learner's tensor-core products read them in place.  The
padding columns stay zero."""
import torch

from go1_b200 import capi


class HistoryWrapper:
    def __init__(self, env):
        self.env = env
        self.obs_history_length = self.env.cfg.env.num_observation_history
        self.num_obs_history = self.obs_history_length * self.env.num_obs
        K0 = self.num_obs_history
        self._pitch = capi.history_pitch(K0)
        z = lambda: torch.zeros(self.env.num_envs, self._pitch, dtype=torch.float, device=self.env.device, requires_grad=False)[:, :K0]
        self._bufs = [z(), z()]
        self._cur = 0
        self.obs_history = self._bufs[0]
        self.num_privileged_obs = self.env.num_privileged_obs

    def __getattr__(self, name):          # gym.Wrapper-style forwarding
        if name.startswith("_") or name == "env":
            raise AttributeError(name)
        return getattr(self.env, name)

    def __setattr__(self, name, value):
        # attributes the Runner writes through the wrapper (episode_length_buf) belong to the env
        if name in ("episode_length_buf", "commands"):
            setattr(self.env, name, value)
        else:
            object.__setattr__(self, name, value)

    def _roll(self, obs):
        src, dst = self._bufs[self._cur], self._bufs[self._cur ^ 1]
        if self._pitch == self.num_obs_history:
            capi.check(capi.lib().go1_history_roll(capi.ptr(src), capi.ptr(obs), capi.ptr(dst), self.env.num_envs, self.env.num_obs,
                                                   self.obs_history_length, capi.stream_ptr()), "go1_history_roll")
        else:
            capi.check(capi.lib().go1_history_roll_pitched(capi.ptr(src), self._pitch, capi.ptr(obs), capi.ptr(dst), self._pitch, self.env.num_envs,
                                                           self.env.num_obs, self.obs_history_length, capi.stream_ptr()), "go1_history_roll_pitched")
        self._cur ^= 1
        self.obs_history = dst

    def step(self, action):
        obs, rew, done, info = self.env.step(action)
        privileged_obs = info["privileged_obs"]
        self._roll(obs)
        return {'obs': obs, 'privileged_obs': privileged_obs, 'obs_history': self.obs_history}, rew, done, info

    def get_observations(self):
        obs = self.env.get_observations()
        privileged_obs = self.env.get_privileged_observations()
        self._roll(obs)
        return {'obs': obs, 'privileged_obs': privileged_obs, 'obs_history': self.obs_history}

    def reset_idx(self, env_ids):
        ret = self.env.reset_idx(env_ids)
        self.obs_history[env_ids, :] = 0
        return ret

    def reset(self):
        ret = self.env.reset()
        privileged_obs = self.env.get_privileged_observations()
        self.obs_history[:, :] = 0
        return {"obs": ret, "privileged_obs": privileged_obs, "obs_history": self.obs_history}
