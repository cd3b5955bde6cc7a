"""CPU checks of AC_Args.bf16_backward's host side: the flag's validation, the new entry points in the header and the library, their
ctypes signatures."""
import ctypes
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))

NEW = ("go1_gemm_bf16_mn", "go1_gemm_bf16_grouped", "go1_convert_bf16_segments", "go1_skinny_dgrad_act_bf16")


def test_bf16_backward_needs_gemm_impl_2():
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    ac = ActorCritic(70, 2, 2100, 12)
    saved = (AC_Args.gemm_impl, AC_Args.bf16_backward)
    assert AC_Args.bf16_backward is False
    try:
        AC_Args.bf16_backward = True
        for impl in (0, 1):
            AC_Args.gemm_impl = impl
            with pytest.raises(ValueError, match="gemm_impl = 2"):
                ac._impl()
        AC_Args.gemm_impl = 2
        assert ac._impl() == 2 and ac._bf16_backward()
        AC_Args.bf16_backward = False
        assert not ac._bf16_backward()
    finally:
        AC_Args.gemm_impl, AC_Args.bf16_backward = saved


def test_header_and_library_declare_the_new_entry_points():
    from go1_b200 import capi
    names = capi.exported_symbols()
    for n in NEW:
        assert n in names
    L = capi.lib()
    for n in NEW:
        assert hasattr(L, n)
    hdr = open(os.path.join(os.path.dirname(HERE), "include", "go1_b200.h")).read()
    body = hdr[hdr.index("typedef struct Go1Bf16Seg"):hdr.index("} Go1Bf16Seg;")]
    assert [f[0] for f in capi.Go1Bf16Seg._fields_] == ["src", "lds", "dst", "ldd", "rows", "cols"]
    assert all(f in body for f in ("src", "lds", "dst", "ldd", "rows", "cols"))


def test_ctypes_signatures():
    from go1_b200 import capi
    L = capi.lib()
    vp, ip = ctypes.c_void_p, ctypes.c_int
    mn = L.go1_gemm_bf16_mn
    assert mn.restype is ip and len(mn.argtypes) == 14
    assert mn.argtypes[:11] == [ip, ip, ip, ip, ip, vp, ip, vp, ip, vp, ip] and mn.argtypes[11] is ip and mn.argtypes[13] is vp
    assert mn.argtypes[12]._type_ is capi.Go1GemmEpilogue
    gr = L.go1_gemm_bf16_grouped
    pvp = ctypes.POINTER(vp)
    assert gr.restype is ip and gr.argtypes == [ip, ip, ip, ip, ip, ip, pvp, ip, pvp, ip, pvp, ip, ip, vp]
    assert L.go1_skinny_dgrad_act_bf16.argtypes == L.go1_skinny_dgrad_act.argtypes and L.go1_skinny_dgrad_act_bf16.restype is ip
    seg = L.go1_convert_bf16_segments
    assert seg.restype is ip and seg.argtypes[0]._type_ is capi.Go1Bf16Seg and seg.argtypes[1:] == [ip, vp]
