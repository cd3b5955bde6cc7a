"""CPU checks of AC_Args.gemm_impl = 2's host side: the BF16 row pitch, the C-ABI mirror of the BF16 entry points, the mode's validation."""
import ctypes
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))


def test_bf16_pitch():
    from go1_b200 import capi
    assert [capi.bf16_pitch(w) for w in (8, 16, 2104, 24576)] == [8, 16, 2104, 24576]
    assert [capi.bf16_pitch(w) for w in (1, 70, 2100, 2105, 2130, 24613)] == [64, 128, 2112, 2112, 2176, 24640]
    assert all(capi.bf16_pitch(w) * 2 % 16 == 0 and capi.bf16_pitch(w) >= w for w in range(1, 3000))


def test_header_declares_bf16_entry_points_and_epilogue_tail():
    from go1_b200 import capi
    names = capi.exported_symbols()
    for n in ("go1_gemm_bf16_ex", "go1_convert_bf16", "go1_gather_rows_bf16", "go1_transpose_to_bf16", "go1_transpose_bf16", "go1_rollout_store_rows_bf16"):
        assert n in names
    # the BF16 output sits at the END of Go1GemmEpilogue: zero-initialised structs of existing callers keep their meaning
    fields = [f[0] for f in capi.Go1GemmEpilogue._fields_]
    assert fields[-3:] == ["store_transposed", "out_bf16", "ld_out_bf16"]
    hdr = open(os.path.join(os.path.dirname(HERE), "include", "go1_b200.h")).read()
    body = hdr[hdr.index("typedef struct Go1GemmEpilogue"):hdr.index("} Go1GemmEpilogue;")]
    assert body.rindex("out_bf16") > body.rindex("store_transposed") and "ld_out_bf16" in body
    assert ctypes.sizeof(capi.Go1GemmEpilogue) % 8 == 0


def test_gemm_impl_values_are_checked():
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    ac = ActorCritic(70, 2, 2100, 12)
    saved = AC_Args.gemm_impl
    try:
        for impl in (0, 1, 2):
            AC_Args.gemm_impl = impl
            assert ac._impl() == impl
        AC_Args.gemm_impl = 3
        with pytest.raises(ValueError):
            ac._impl()
    finally:
        AC_Args.gemm_impl = saved
