"""AC_Args.deterministic without a GPU: the C ABI pair and its ctypes binding, the switch read at ActorCritic construction (default from
GO1_DETERMINISTIC, or torch.use_deterministic_algorithms), and learners of both modes side by side with the library mode stubbed."""
import os
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in ("walk-these-ways_b200", os.path.join("walk-these-ways_b200", "compat")):
    sys.path.insert(0, os.path.join(ROOT, _p))


def test_abi_pair_is_declared_and_bound():
    from go1_b200 import capi
    syms = capi.exported_symbols()
    for name in ("go1_set_deterministic", "go1_deterministic", "go1_deterministic_workspace_bytes"):
        assert name in syms
    hdr = open(os.path.join(ROOT, "include", "go1_b200.h")).read()
    assert "void go1_set_deterministic(int on);" in hdr and "int go1_deterministic(void);" in hdr
    if os.path.exists(capi.LIB_PATH):
        L = capi.lib()
        assert L.go1_deterministic() == 0
        L.go1_set_deterministic(1)
        assert L.go1_deterministic() == 1
        L.go1_set_deterministic(0)
        assert L.go1_deterministic() == 0 and L.go1_deterministic_workspace_bytes() >= 0


def _ac():
    from go1_gym_learn.ppo_cse import ActorCritic
    return ActorCritic(70, 2, 2100, 12)


def test_switch_is_read_at_construction(monkeypatch):
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    monkeypatch.setattr(AC_Args, "deterministic", True)
    ac = _ac()
    monkeypatch.setattr(AC_Args, "deterministic", False)
    assert ac.deterministic and not _ac().deterministic
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        assert _ac().deterministic
    finally:
        torch.use_deterministic_algorithms(prev)


@pytest.mark.parametrize("env,want", [(None, False), ("0", False), ("1", True)])
def test_environment_variable_sets_the_default(env, want):
    e = {k: v for k, v in os.environ.items() if k != "GO1_DETERMINISTIC"}
    if env is not None:
        e["GO1_DETERMINISTIC"] = env
    code = ("import sys; sys.path[:0] = ['walk-these-ways_b200', 'walk-these-ways_b200/compat']\n"
            "from go1_gym_learn.ppo_cse.actor_critic import AC_Args; print(AC_Args.deterministic)")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=e, capture_output=True, text=True, check=True).stdout.split()
    assert out[-1] == str(want)


class _FakeLib:
    """The two mode functions of the library, recording every change."""

    def __init__(self):
        self.mode, self.sets = 0, []

    def go1_deterministic(self):
        return self.mode

    def go1_set_deterministic(self, on):
        self.sets.append(on)
        self.mode = on


def test_learners_of_both_modes_coexist(monkeypatch):
    from go1_b200 import capi
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args, in_mode
    from go1_gym_learn.ppo_cse.rollout_storage import RolloutStorage
    fake = _FakeLib()
    monkeypatch.setattr(capi, "_lib", fake)
    monkeypatch.setattr(capi, "lib", lambda: fake)
    monkeypatch.setattr(AC_Args, "deterministic", True)
    det = _ac()
    monkeypatch.setattr(AC_Args, "deterministic", False)
    default = _ac()
    seen = []

    class Probe:
        def __init__(self, ac):
            self.deterministic = ac.deterministic

        @in_mode
        def launch(self, inner=None):
            seen.append(fake.mode)
            if inner is not None:
                inner.launch()

    Probe(det).launch()
    Probe(default).launch()
    Probe(det).launch(inner=Probe(default))
    Probe(default).launch(inner=Probe(det))
    assert seen == [1, 0, 1, 0, 0, 1] and fake.mode == 0
    assert fake.sets == [1, 0, 1, 0, 1, 0, 1, 0]
    fake.sets.clear()
    Probe(default).launch()             # the library is already in the default mode: no call at all
    assert fake.sets == []
    # the public entry points run in their learner's mode, and so does the storage its PPO hands the mode to
    for name in ("forward_all", "backward_ppo", "backward_adaptation", "adaptation_forward", "evaluate", "act_student", "act_teacher"):
        assert getattr(type(det), name).__wrapped__
    assert RolloutStorage.compute_returns.__wrapped__ and RolloutStorage.deterministic is False
