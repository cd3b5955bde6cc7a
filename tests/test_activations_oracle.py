"""CPU side of the AC_Args.activation family: the autograd oracle against vectors produced by the reference's own ppo_cse code for
every activation name (tests/golden/ppo_activations.npz, written by tests/golden/make_golden_activations.py), the name -> module
table, and the derivative-from-output formulas that the CUDA kernels restate (csrc/activation.cuh)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "walk-these-ways_b200", "compat"))      # params_proto, ml_logger
from activation_test_util import DERIV_FROM_OUTPUT, KINDS, MODULES, NAMES, header_enum, oracle_actor_critic
from oracle.ppo_oracle import PPOOracle, gae
from ppo_golden_util import seeded_weights, sample_tensor

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize("activation", NAMES)
def test_oracle_reproduces_reference_ppo_cycle(activation):
    torch.set_num_threads(4)
    g = np.load(os.path.join(HERE, "golden", "ppo_activations.npz"))
    N, T, NOBS, NH, NP, NA, h1, h2, ha = (int(x) for x in g["meta/dims"])
    ac = oracle_actor_critic(activation, NP, NH, NA, [h1, h2], [ha])
    w = seeded_weights({k: tuple(v.shape) for k, v in ac.state_dict().items()})
    ac.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
    T_ = lambda k: torch.from_numpy(np.ascontiguousarray(g[k]))
    hist, priv, eps = T_("in/hist"), T_("in/priv"), T_("in/eps")
    with torch.no_grad():
        acts, vals, logps, mus = [], [], [], []
        for t in range(T):
            d = ac.dist(hist[t])
            a = d.mean + d.stddev * eps[t]
            acts.append(a); vals.append(ac.value(hist[t], priv[t])); logps.append(d.log_prob(a).sum(-1, keepdim=True)); mus.append(d.mean)
        actions, values, logp, mu = torch.stack(acts), torch.stack(vals), torch.stack(logps), torch.stack(mus)
        last_v = ac.value(T_("last/hist"), T_("last/priv"))
        returns, adv = gae(T_("in/rew").unsqueeze(-1), T_("in/done").unsqueeze(-1), values, last_v)
    for name, got in (("actions", actions), ("values", values), ("actions_log_prob", logp), ("mu", mu), ("returns", returns), ("advantages", adv)):
        assert np.allclose(got.numpy(), g[f"{activation}/storage/{name}"], rtol=1e-4, atol=2e-5), name
    f = lambda x: x.flatten(0, 1)
    ppo = PPOOracle(ac)
    vl, sl, al, atl = ppo.update(f(hist), f(priv), f(actions), f(values), f(returns), f(adv), f(logp), f(mu), torch.ones_like(f(mu)),
                                 torch.from_numpy(g["in/perm"]))
    ref = g[f"{activation}/update/losses"]
    assert abs(vl - ref[0]) < 1e-3 * abs(ref[0]) and abs(sl - ref[1]) < 1e-3 and abs(al - ref[2]) < 1e-3 * abs(ref[2]) and abs(atl - ref[5]) < 1e-3 * abs(ref[5])
    assert abs(ppo.lr - float(g[f"{activation}/update/learning_rate"])) < 1e-12
    for k, v in ac.state_dict().items():
        got, want = sample_tensor(v.numpy(), stride=3), g[f"{activation}/final/{k}"]
        assert np.allclose(got[:-2], want[:-2], atol=2e-4), k


def test_crelu_is_relu_in_the_reference_vectors():
    g = np.load(os.path.join(HERE, "golden", "ppo_activations.npz"))
    for k in g.files:
        if k.startswith("crelu/"):
            assert np.array_equal(g[k], g["relu/" + k[len("crelu/"):]]), k


def test_get_activation_table_and_enum():
    from go1_b200 import capi
    from go1_gym_learn.ppo_cse.actor_critic import get_activation
    for name in NAMES:
        assert type(get_activation(name)) is MODULES[name], name
    assert type(get_activation("crelu")) is torch.nn.ReLU
    with pytest.raises(ValueError, match="sigmoid"):
        get_activation("gelu")
    enum = header_enum()
    assert enum["GO1_ACT_ELU"] == 0 and len(enum) == 6
    assert set(capi.ACTIVATIONS) == set(NAMES)
    for name, kind in capi.ACTIVATIONS.items():
        assert enum["GO1_ACT_" + ("RELU" if name == "crelu" else name.upper())] == kind, name
    assert capi.act_arg(capi.ACTIVATIONS["tanh"], 1) == (4 << 8) | 1


def test_actor_critic_rejects_unknown_activation_and_builds_the_modules():
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args, ActorCritic
    old = AC_Args.activation
    try:
        AC_Args.activation = "gelu"
        with pytest.raises(ValueError, match="gelu"):
            ActorCritic(70, 2, 140, 12)
        AC_Args.activation = "lrelu"
        ac = ActorCritic(70, 2, 140, 12)
        for seq in (ac.adaptation_module, ac.actor_body, ac.critic_body):
            assert all(type(m) is torch.nn.LeakyReLU for m in list(seq)[1::2])
        assert ac.act_kind == 3
    finally:
        AC_Args.activation = old


@pytest.mark.parametrize("kind", KINDS)
def test_derivative_from_output_matches_autograd(kind):
    """f'(v) computed from y = f(v) alone equals torch.autograd's derivative in fp64, kinks included (v = 0: relu 0, lrelu 0.01,
    elu / selu the left branch)."""
    v = torch.cat((torch.linspace(-30, 30, 2401, dtype=torch.float64), torch.tensor([0.0, -0.0, 1e-9, -1e-9, 30.0, -30.0], dtype=torch.float64)))
    v.requires_grad_(True)
    y = MODULES[kind]()(v)
    y.sum().backward()
    got = DERIV_FROM_OUTPUT[kind](y.detach())
    assert torch.allclose(got, v.grad, rtol=1e-12, atol=1e-12), float((got - v.grad).abs().max())
    at0 = float(DERIV_FROM_OUTPUT[kind](MODULES[kind]()(torch.zeros(1, dtype=torch.float64)))[0])
    assert at0 == {"elu": 1.0, "selu": SELU_AT_0, "relu": 0.0, "lrelu": 0.01, "tanh": 1.0, "sigmoid": 0.25}[kind]


SELU_AT_0 = 1.0507009873554805 * 1.6732632423543772
