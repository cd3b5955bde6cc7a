"""capi.history_pitch: the one rule for the row pitch of observation-history buffers (no GPU needed)."""
import pytest


@pytest.mark.parametrize("width,pitch", [(2100, 2100), (2112, 2112), (4, 4), (1050, 1056), (2130, 2144), (2201, 2208), (2263, 2272),
                                         (1, 32), (42, 64), (70, 96), (71, 96), (73, 96)])
def test_history_pitch(width, pitch):
    from go1_b200 import capi
    assert capi.history_pitch(width) == pitch


def test_history_pitch_rule_over_every_width():
    """Multiples of 4 floats keep their width; every other width gets the next multiple of 32 floats (128-byte rows)."""
    from go1_b200 import capi
    for w in range(1, 128 * 33):
        p = capi.history_pitch(w)
        assert p >= w and p % 4 == 0
        assert p == w if w % 4 == 0 else (p % 32 == 0 and p - w < 32)
