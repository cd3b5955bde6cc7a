"""CPU side of num_privileged_obs > 4: the autograd oracle (oracle/ppo_oracle.py) against vectors produced by the reference's own ppo_cse
code with 5, 18 and 45 privileged observations and with selective_adaptation_module_loss (tests/golden/ppo_priv.npz, written by
tests/golden/make_golden_priv.py), and ActorCritic's limit on the width."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "walk-these-ways_b200", "compat"))      # params_proto, ml_logger
import priv_obs_util as U
from oracle import ppo_oracle
from oracle.ppo_oracle import ActorCriticOracle, PPOOracle, gae
from ppo_golden_util import seeded_weights, sample_tensor

HERE = os.path.dirname(os.path.abspath(__file__))


def _selective_mse(monkeypatch):
    """The reference's selective_adaptation_module_loss (ppo.py:177-183): the adaptation MSE of privileged column 0 only."""
    monkeypatch.setattr(ppo_oracle, "F", types.SimpleNamespace(mse_loss=lambda a, b: F.mse_loss(a[:, 0], b[:, 0])))


@pytest.mark.parametrize("case", list(U.CASES))
def test_oracle_reproduces_reference_ppo_cycle(case, monkeypatch):
    torch.set_num_threads(4)
    g = np.load(os.path.join(HERE, "golden", "ppo_priv.npz"))
    E, selective = U.CASES[case]
    if selective:
        _selective_mse(monkeypatch)
    inp = U.inputs()
    ac = ActorCriticOracle(num_obs=U.NOBS, num_priv=E, num_hist=U.NH, num_actions=U.NA)
    w = seeded_weights({k: tuple(v.shape) for k, v in ac.state_dict().items()})
    ac.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    T_ = lambda k: torch.from_numpy(np.ascontiguousarray(inp[k]))
    hist, priv, eps = T_("in/hist"), T_("in/priv")[..., :E].contiguous(), T_("in/eps")
    with torch.no_grad():
        acts, vals, logps, mus = [], [], [], []
        for t in range(U.T):
            d = ac.dist(hist[t])
            a = d.mean + d.stddev * eps[t]
            acts.append(a); vals.append(ac.value(hist[t], priv[t])); logps.append(d.log_prob(a).sum(-1, keepdim=True)); mus.append(d.mean)
        actions, values, logp, mu = torch.stack(acts), torch.stack(vals), torch.stack(logps), torch.stack(mus)
        last_v = ac.value(T_("last/hist"), T_("last/priv")[:, :E])
        returns, adv = gae(T_("in/rew").unsqueeze(-1), T_("in/done").unsqueeze(-1), values, last_v)
    for name, got in (("actions", actions), ("values", values), ("actions_log_prob", logp), ("mu", mu), ("returns", returns), ("advantages", adv)):
        assert np.allclose(got.numpy(), g[f"{case}/storage/{name}"], rtol=1e-4, atol=2e-5), name
    f = lambda x: x.flatten(0, 1)
    ppo = PPOOracle(ac)
    vl, sl, al, atl = ppo.update(f(hist), f(priv), f(actions), f(values), f(returns), f(adv), f(logp), f(mu), torch.ones_like(f(mu)),
                                 torch.from_numpy(inp["in/perm"]))
    ref = g[f"{case}/update/losses"]
    assert abs(vl - ref[0]) < 1e-3 * abs(ref[0]) and abs(sl - ref[1]) < 1e-3 and abs(al - ref[2]) < 1e-3 * abs(ref[2]) and abs(atl - ref[5]) < 1e-3 * abs(ref[5])
    assert abs(ppo.lr - float(g[f"{case}/update/learning_rate"])) < 1e-12
    for k, v in ac.state_dict().items():
        got, want = sample_tensor(v.numpy(), stride=U.sample_stride(v.numel())), g[f"{case}/final/{k}"]
        assert np.allclose(got[:-2], want[:-2], atol=2e-4), k


def test_selective_loss_changes_only_the_adaptation_step():
    """The selective case differs from the full one in the adaptation losses and weights, not in the PPO step's first minibatch inputs."""
    g = np.load(os.path.join(HERE, "golden", "ppo_priv.npz"))
    for n in ("actions", "values", "returns"):
        assert np.array_equal(g[f"e45/storage/{n}"], g[f"e45sel/storage/{n}"]), n
    assert abs(g["e45/update/losses"][2] - g["e45sel/update/losses"][2]) > 1e-3


@pytest.mark.parametrize("E", [0, 65, 100])
def test_actor_critic_rejects_unsupported_width_at_construction(E):
    from go1_gym_learn.ppo_cse.actor_critic import ActorCritic
    with pytest.raises(ValueError, match="1..64"):
        ActorCritic(70, E, 140, 12)


@pytest.mark.parametrize("E", [1, 5, 45, 64])
def test_actor_critic_accepts_supported_widths(E):
    from go1_gym_learn.ppo_cse.actor_critic import ActorCritic
    ac = ActorCritic(70, E, 140, 12)
    assert ac.adaptation_module[-1].out_features == E and ac.actor_body[0].in_features == 140 + E and ac.critic_body[0].in_features == 140 + E
