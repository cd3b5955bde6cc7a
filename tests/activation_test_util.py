"""Helpers shared by the activation tests (tests/test_activations_oracle.py, tests/test_activations_gpu.py)."""
import os
import re

import torch
import torch.nn as nn

from oracle.ppo_oracle import ActorCriticOracle

HERE = os.path.dirname(os.path.abspath(__file__))
NAMES = ("elu", "selu", "relu", "crelu", "lrelu", "tanh", "sigmoid")          # every name AC_Args.activation accepts
KINDS = ("elu", "selu", "relu", "lrelu", "tanh", "sigmoid")                   # the six kernels behind them (crelu is relu)
MODULES = {"elu": nn.ELU, "selu": nn.SELU, "relu": nn.ReLU, "crelu": nn.ReLU, "lrelu": nn.LeakyReLU, "tanh": nn.Tanh, "sigmoid": nn.Sigmoid}
SELU_LAMBDA, SELU_ALPHA = 1.0507009873554805, 1.6732632423543772

# f'(v) as a function of the saved output y = f(v): the table the kernels restate (csrc/activation.cuh)
DERIV_FROM_OUTPUT = {
    "elu": lambda y: torch.where(y > 0, torch.ones_like(y), y + 1),
    "selu": lambda y: torch.where(y > 0, torch.full_like(y, SELU_LAMBDA), y + SELU_LAMBDA * SELU_ALPHA),
    "relu": lambda y: (y > 0).to(y.dtype),
    "lrelu": lambda y: torch.where(y > 0, torch.ones_like(y), torch.full_like(y, 0.01)),
    "tanh": lambda y: 1 - y * y,
    "sigmoid": lambda y: y * (1 - y),
}


def header_enum():
    """{GO1_ACT_*: value} of enum Go1Activation in include/go1_b200.h."""
    txt = open(os.path.join(os.path.dirname(HERE), "include", "go1_b200.h")).read()
    body = re.search(r"typedef enum Go1Activation \{(.*?)\}", txt, re.S).group(1)
    out, nxt = {}, 0
    for item in body.split(","):
        name, _, val = item.strip().partition("=")
        nxt = int(val) if val.strip() else nxt
        out[name.strip()] = nxt
        nxt += 1
    return out


def _mlp(i, hidden, o, activation):
    layers, d = [], i
    for h in hidden:
        layers += [nn.Linear(d, h), MODULES[activation]()]
        d = h
    return nn.Sequential(*layers, nn.Linear(d, o))


def oracle_actor_critic(activation, num_priv, num_hist, num_actions, hidden, adapt_hidden):
    """oracle.ppo_oracle.ActorCriticOracle with the given activation and layer widths (its dist / value methods unchanged)."""
    ac = ActorCriticOracle(num_priv=num_priv, num_hist=8, num_actions=num_actions)
    ac.adaptation_module = _mlp(num_hist, adapt_hidden, num_priv, activation)
    ac.actor_body = _mlp(num_hist + num_priv, hidden, num_actions, activation)
    ac.critic_body = _mlp(num_hist + num_priv, hidden, 1, activation)
    return ac
