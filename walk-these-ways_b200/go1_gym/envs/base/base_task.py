"""BaseTask (reference go1_gym/envs/base/base_task.py:14-137): sizes, device, reset() contract."""
import torch


class BaseTask:
    def __init__(self, cfg, sim_params, physics_engine, sim_device, headless, eval_cfg=None):
        self.sim_params = sim_params
        self.physics_engine = physics_engine
        self.sim_device = sim_device
        self.headless = headless
        if not str(sim_device).startswith("cuda"):
            raise RuntimeError("go1_gym (CUDA build) runs on CUDA devices only: there is no CPU simulator")
        self.device = sim_device
        self.num_obs = cfg.env.num_observations
        self.num_privileged_obs = cfg.env.num_privileged_obs
        self.num_actions = cfg.env.num_actions
        if eval_cfg is not None:           # base_task.py:43-50: eval envs are appended after the train envs
            self.num_eval_envs = eval_cfg.env.num_envs
            self.num_train_envs = cfg.env.num_envs
            self.num_envs = self.num_eval_envs + self.num_train_envs
        else:
            self.num_eval_envs = 0
            self.num_train_envs = cfg.env.num_envs
            self.num_envs = cfg.env.num_envs
        self.extras = {}
        self.create_sim()
        self.enable_viewer_sync = True
        self.viewer = None

    def get_observations(self):
        return self.obs_buf

    def get_privileged_observations(self):
        return self.privileged_obs_buf

    def reset_idx(self, env_ids):
        raise NotImplementedError

    def reset(self):
        self.reset_idx(torch.arange(self.num_envs, device=self.device))
        obs, privileged_obs, _, _, _ = self.step(torch.zeros(self.num_envs, self.num_actions, device=self.device, requires_grad=False))
        return obs, privileged_obs

    def step(self, actions):
        raise NotImplementedError

    def render_gui(self, sync_frame_time=True):
        pass

    def close(self):
        pass
