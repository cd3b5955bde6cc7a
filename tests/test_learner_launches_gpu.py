"""The learner's launch trace against tests/golden/launches.json.gz (see launch_trace_util): for each case, forward_all / backward_ppo
(without and with a caller-built hT), adaptation_forward / backward_adaptation, act_student / act_teacher / evaluate and the packed-copy
refresh, or one PPO act -> store -> compute_returns -> update cycle, launch the same entry points, in the same order, with the same
arguments, on the same streams."""
import pytest

import launch_trace_util as lt

pytestmark = pytest.mark.gpu

_GOLD = {}


def _gold():
    if not _GOLD:
        _GOLD.update(lt.load()["cases"])
    return _GOLD


def test_fixture_covers_every_case():
    assert set(_gold()) == set(lt.CASES)


@pytest.mark.parametrize("name", list(lt.CASES))
def test_learner_launches_match_fixture(name, monkeypatch):
    want, got = _gold()[name], lt.trace(name, monkeypatch)
    for k, (w, g) in enumerate(zip(want, got)):
        assert w == g, f"launch {k} of {len(want)}:\n  fixture {w}\n  traced  {g}"
    assert len(got) == len(want), (len(got), len(want), got[len(want):len(want) + 3], want[len(got):len(got) + 3])
