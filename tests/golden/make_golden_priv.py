#!/usr/bin/env python
"""Generates tests/golden/ppo_priv.npz by running the REFERENCE's own ActorCritic / PPO / RolloutStorage (imported through
tests/_stubs, the recipe of make_golden.make_ppo) once per privileged-observation width on the default network:

    python tests/golden/make_golden_priv.py

history 2100, actor / critic hidden [512, 256, 128], adaptation module [256, 128], 16 envs x 24 steps (minibatches of 96 rows), one
full act -> process_env_step -> compute_returns -> update cycle for num_privileged_obs = 5, 18 and 45, and 45 again with
PPO_Args.selective_adaptation_module_loss.  The inputs are priv_obs_util.inputs() (re-created by the tests, not stored); per case `c`
the file holds "c/storage/...", "c/update/losses", "c/update/learning_rate" and "c/final/<parameter>" (strided samples + sum + sum of
squares, ppo_golden_util.sample_tensor with priv_obs_util.sample_stride).  The initial weights are ppo_golden_util.seeded_weights.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))      # ppo_golden_util, priv_obs_util
import make_golden  # noqa: E402,F401  (puts the stubs and the reference on sys.path)
import torch  # noqa: E402

import priv_obs_util as U  # noqa: E402


def run(case, out, inputs):
    from go1_gym_learn.ppo_cse.actor_critic import ActorCritic
    from go1_gym_learn.ppo_cse.ppo import PPO, PPO_Args
    from ppo_golden_util import seeded_weights, sample_tensor
    import torch.distributions.normal as tn
    E, selective = U.CASES[case]
    PPO_Args.selective_adaptation_module_loss = selective
    torch.manual_seed(0)
    ac = ActorCritic(U.NOBS, E, U.NH, U.NA)
    with torch.no_grad():
        for k, v in seeded_weights({k: tuple(v.shape) for k, v in ac.state_dict().items()}).items():
            ac.state_dict()[k].copy_(torch.from_numpy(v))
    alg = PPO(ac, device="cpu")
    alg.init_storage(U.N, U.T, [U.NOBS], [E], [U.NH], [U.NA])
    C = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    for t in range(U.T):
        eps = C(inputs["in/eps"][t])
        orig = tn.Normal.sample
        tn.Normal.sample = lambda self, sample_shape=torch.Size(): (self.mean + self.stddev * eps).detach()
        try:
            with torch.inference_mode():
                alg.act(C(inputs["in/obs"][t]), C(inputs["in/priv"][t][:, :E]), C(inputs["in/hist"][t]))
        finally:
            tn.Normal.sample = orig
        infos = {"env_bins": torch.zeros(U.N), "time_outs": torch.zeros(U.N, dtype=torch.bool)}
        with torch.inference_mode():
            alg.process_env_step(C(inputs["in/rew"][t]), C(inputs["in/done"][t]), infos)
    with torch.inference_mode():
        alg.compute_returns(C(inputs["last/hist"]), C(inputs["last/priv"][:, :E]))
    st = alg.storage
    for n in ("actions", "values", "actions_log_prob", "mu", "returns", "advantages"):
        out[f"{case}/storage/{n}"] = getattr(st, n).detach().numpy().copy()
    perm = C(inputs["in/perm"])
    orig_rp = torch.randperm
    torch.randperm = lambda n, **k: perm
    try:
        losses = alg.update()
    finally:
        torch.randperm = orig_rp
        PPO_Args.selective_adaptation_module_loss = False
    out[f"{case}/update/losses"] = np.array(losses, dtype=np.float64)
    out[f"{case}/update/learning_rate"] = np.array(alg.learning_rate)
    for k, v in ac.state_dict().items():
        out[f"{case}/final/{k}"] = sample_tensor(v.detach().numpy(), stride=U.sample_stride(v.numel()))
    print(case, "losses", [round(float(x), 5) for x in losses[:6]], "lr", alg.learning_rate)


def main():
    torch.set_num_threads(8)
    inputs = U.inputs()
    out = {}
    for case in U.CASES:
        run(case, out, inputs)
    path = os.path.join(HERE, "ppo_priv.npz")
    np.savez_compressed(path, **out)
    print("ppo_priv.npz:", len(out), "arrays,", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
