"""CoRLRewards: the reward container of walk-these-ways (`Cfg.rewards.reward_container_name = "CoRLRewards"`).

Every built-in term is a `BuiltinReward` marker: the fused step kernel computes it.  To add a term, subclass the container,
write a method `_reward_<name>(self)` that reads `self.env` and returns a [num_envs] float32 tensor on the env's device, give
it a nonzero `Cfg.reward_scales.<name>`, and register the class in `REWARD_CONTAINERS`.  A method with the name of a built-in
term replaces the kernel's version.  The four task terms feed the command curriculum and `termination` is added after the
combination, so those five cannot be replaced.

During a term, `self.env` is the env as compute_reward sees it: after physics, before resets, and with last_actions,
last_last_actions, last_dof_vel, last_joint_pos_target and last_last_joint_pos_target as they were before this step's rolls.

The training rollout captures the env step, user terms included, in a CUDA graph and replays it; a replay re-runs the device work
the term queued at capture time, not its Python.  So a term must be a pure function of device tensors: host-side state it reads
(`self.env.common_step_counter`, a Python branch on values, an attribute rebound on the host) keeps its capture-time value.
`GO1_STEP_GRAPH=0` runs the rollout launch by launch instead."""
from go1_b200 import capi


class BuiltinReward:
    """Marker for the reward term `name` that the fused step kernel computes."""
    __slots__ = ("builtin_term",)

    def __init__(self, name):
        self.builtin_term = name

    def __repr__(self):
        return f"BuiltinReward({self.builtin_term!r})"


class CoRLRewards:
    def __init__(self, env):
        self.env = env

    def load_env(self, env):
        self.env = env


for _name in capi.REWARD_TERMS:
    setattr(CoRLRewards, "_reward_" + _name, BuiltinReward(_name))
del _name
