"""AC_Args hidden-layer shapes on the host (no GPU needed): ActorCritic rejects hidden lists the kernels cannot run, and capi.row_pitch is
the one rule for the row pitch of the learner's hidden activation and gradient buffers."""
import copy
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "walk-these-ways_b200", "compat"))      # params_proto, ml_logger

FIELDS = ("actor_hidden_dims", "critic_hidden_dims", "adaptation_module_branch_hidden_dims")


@pytest.fixture(autouse=True)
def _restore_ac_args():
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    keep = {k: copy.copy(getattr(AC_Args, k)) for k in FIELDS}
    yield
    for k, v in keep.items():
        setattr(AC_Args, k, v)


@pytest.mark.parametrize("dims", [[], [0], [256, -3], [128, 0, 64], [64.0]])
@pytest.mark.parametrize("field", FIELDS)
def test_bad_hidden_dims_raise_value_error_naming_the_field(field, dims):
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    setattr(AC_Args, field, dims)
    with pytest.raises(ValueError, match=f"AC_Args.{field}"):
        ActorCritic(70, 2, 2100, 12)


@pytest.mark.parametrize("dims", [[1], [36], [500, 250, 125], [512, 256, 128, 64]])
def test_good_hidden_dims_build_the_reference_modules(dims):
    """Any non-empty list of positive widths builds the reference's nn.Sequential (Linear, activation, ..., Linear)."""
    import torch.nn as nn
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    for f in FIELDS:
        setattr(AC_Args, f, list(dims))
    ac = ActorCritic(70, 2, 2100, 12)
    for seq, i, o in ((ac.actor_body, 2102, 12), (ac.critic_body, 2102, 1), (ac.adaptation_module, 2100, 2)):
        lins = [m for m in seq if isinstance(m, nn.Linear)]
        assert [(m.in_features, m.out_features) for m in lins] == list(zip([i] + dims, dims + [o]))


@pytest.mark.parametrize("width,pitch", [(512, 512), (256, 256), (128, 128), (4, 4), (500, 500), (250, 256), (125, 128), (36, 36),
                                         (1, 32), (2, 32), (13, 32), (33, 64)])
def test_row_pitch(width, pitch):
    from go1_b200 import capi
    assert capi.row_pitch(width) == pitch


def test_row_pitch_is_the_history_rule():
    """One rule for every TMA-read buffer: widths that are multiples of 4 floats keep their width, the others get the next multiple of 32
    floats (128-byte rows); capi.history_pitch is the same rule."""
    from go1_b200 import capi
    for w in range(1, 128 * 33):
        p = capi.row_pitch(w)
        assert p >= w and p % 4 == 0
        assert p == w if w % 4 == 0 else (p % 32 == 0 and p - w < 32)
        assert capi.history_pitch(w) == p


@pytest.mark.parametrize("hidden,start", [([512, 256, 128], 1), ([256, 128], 1), ([1024, 512, 256], 2), ([256, 128, 64], 1),
                                          ([512, 256, 128, 64], 2), ([500, 250, 125], 1), ([250, 125], 1), ([256], None), ([512, 512], None),
                                          ([256, 256, 256], 2)])
def test_tail_start(hidden, start):
    """Where the fused tail begins: the last two hidden layers when they are at most 256 and 128 wide, else the last one when it is at
    most 256 wide; a one-hidden-layer net has no tail."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.actor_hidden_dims = list(hidden)
    ac = ActorCritic(70, 2, 2100, 12)
    ac.flatten()
    assert ac._nets["actor"].tail_start == start
