from .corl_rewards import BuiltinReward, CoRLRewards

# Cfg.rewards.reward_container_name -> container class.  Add your own container classes here.
REWARD_CONTAINERS = {"CoRLRewards": CoRLRewards}
