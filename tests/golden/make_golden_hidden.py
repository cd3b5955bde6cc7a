#!/usr/bin/env python
"""Generates tests/golden/ppo_hidden.npz by running the REFERENCE's own ActorCritic / PPO / RolloutStorage (imported through
tests/_stubs, the recipe of make_golden.make_ppo) on a SMALL network with non-default AC_Args hidden dims:

    python tests/golden/make_golden_hidden.py

history 5 x 70, actor / critic hidden [64, 50, 36, 20] (four hidden layers: two run one by one, the last two and the head as a fused
tail; 50 is not a multiple of 4 floats), adaptation module [40, 25], ELU, 4 envs x 24 steps, one full
act -> process_env_step -> compute_returns -> update cycle.  The file holds the inputs ("in/...", "last/..."), "elu/storage/...",
"elu/update/losses", "elu/update/learning_rate" and "elu/final/<parameter>" (strided samples + sum + sum of squares,
ppo_golden_util.sample_tensor), and "meta/dims" = [N, T, NOBS, NH, NP, NA, number of actor / critic hidden layers, their widths...,
the adaptation module's widths...].  The initial weights are ppo_golden_util.seeded_weights (not stored).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))      # ppo_golden_util
import make_golden  # noqa: E402,F401  (puts the stubs and the reference on sys.path)
import torch  # noqa: E402

ACTIVATIONS = ("elu",)
N, T, NOBS, NH, NP, NA = 4, 24, 70, 350, 2, 12
HIDDEN, ADAPT_HIDDEN = [64, 50, 36, 20], [40, 25]
STRIDE = 3


def run(activation, out, inputs):
    from go1_gym_learn.ppo_cse.actor_critic import ActorCritic, AC_Args
    from go1_gym_learn.ppo_cse.ppo import PPO
    from ppo_golden_util import seeded_weights, sample_tensor
    import torch.distributions.normal as tn
    AC_Args.activation = activation
    AC_Args.actor_hidden_dims, AC_Args.critic_hidden_dims, AC_Args.adaptation_module_branch_hidden_dims = HIDDEN, HIDDEN, ADAPT_HIDDEN
    torch.manual_seed(0)
    ac = ActorCritic(NOBS, NP, NH, NA)
    with torch.no_grad():
        for k, v in seeded_weights({k: tuple(v.shape) for k, v in ac.state_dict().items()}).items():
            ac.state_dict()[k].copy_(torch.from_numpy(v))
    alg = PPO(ac, device="cpu")
    alg.init_storage(N, T, [NOBS], [NP], [NH], [NA])
    C = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    for t in range(T):
        eps = C(inputs["in/eps"][t])
        orig = tn.Normal.sample
        tn.Normal.sample = lambda self, sample_shape=torch.Size(): (self.mean + self.stddev * eps).detach()
        try:
            with torch.inference_mode():
                alg.act(C(inputs["in/obs"][t]), C(inputs["in/priv"][t]), C(inputs["in/hist"][t]))
        finally:
            tn.Normal.sample = orig
        infos = {"env_bins": torch.zeros(N), "time_outs": torch.zeros(N, dtype=torch.bool)}
        with torch.inference_mode():
            alg.process_env_step(C(inputs["in/rew"][t]), C(inputs["in/done"][t]), infos)
    with torch.inference_mode():
        alg.compute_returns(C(inputs["last/hist"]), C(inputs["last/priv"]))
    st = alg.storage
    for n in ("actions", "values", "actions_log_prob", "mu", "returns", "advantages"):
        out[f"{activation}/storage/{n}"] = getattr(st, n).detach().numpy().copy()
    perm = C(inputs["in/perm"])
    orig_rp = torch.randperm
    torch.randperm = lambda n, **k: perm
    try:
        losses = alg.update()
    finally:
        torch.randperm = orig_rp
    out[f"{activation}/update/losses"] = np.array(losses, dtype=np.float64)
    out[f"{activation}/update/learning_rate"] = np.array(alg.learning_rate)
    for k, v in ac.state_dict().items():
        out[f"{activation}/final/{k}"] = sample_tensor(v.detach().numpy(), stride=STRIDE)
    print(activation, "losses", [round(float(x), 5) for x in losses[:3]], "lr", alg.learning_rate)


def main():
    g = torch.Generator().manual_seed(11)
    R = lambda *s: torch.randn(*s, generator=g)
    inputs = {"in/obs": R(T, N, NOBS), "in/hist": R(T, N, NH) * 0.5, "in/priv": R(T, N, NP), "in/eps": R(T, N, NA), "in/rew": R(T, N),
              "last/hist": R(N, NH) * 0.5, "last/priv": R(N, NP)}
    inputs = {k: v.numpy().copy() for k, v in inputs.items()}
    inputs["in/done"] = (torch.rand(T, N, generator=g) < 0.1).numpy().copy()
    inputs["in/perm"] = torch.randperm(N * T, generator=g).numpy().copy()
    out = dict(inputs)
    out["meta/dims"] = np.array([N, T, NOBS, NH, NP, NA, len(HIDDEN)] + HIDDEN + ADAPT_HIDDEN, dtype=np.int64)
    for a in ACTIVATIONS:
        run(a, out, inputs)
    path = os.path.join(HERE, "ppo_hidden.npz")
    np.savez_compressed(path, **out)
    print("ppo_hidden.npz:", len(out), "arrays,", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
