"""The first-layer weight gradients with K-major operands: the transposed epilogue store of go1_gemm_ex (store_transposed), the
K-major fused first-layer wgrad over the transposed history (history_kmajor) against fp64 autograd, and the split-K count picked for
the two production products."""
import csv
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))


def _gemm_ex(ta, tb, M, N, K, A, B, C, ldc, ep):
    from go1_b200 import capi
    capi.check(capi.lib().go1_gemm_ex(ta, tb, M, N, K, capi.ptr(A), A.stride(0), capi.ptr(B), B.stride(0), capi.ptr(C), ldc, ep, 1, capi.stream_ptr()), "gemm_ex")


@pytest.mark.parametrize("kind", [0, 4])         # GO1_ACT_ELU, GO1_ACT_TANH
@pytest.mark.parametrize("act", [0, 2])
@pytest.mark.parametrize("M,N", [(1000, 300), (4096, 512), (24576 + 37, 256)])
def test_transposed_store_matches_row_major(M, N, act, kind):
    """The dgrad shape (dz [M][K] times W given as [K][N], times f'(y) for act 2): the transposed store holds exactly the row-major
    result, with the fused column sums unchanged, and leaves the pitch padding of C^T alone beyond M rounded up to 4."""
    from go1_b200 import capi
    torch.manual_seed(M + N + act + kind)
    K = 256                                      # 8 k-blocks: never split, so both stores see the same accumulation order
    A = torch.randn(M, K, device="cuda")
    B = torch.randn(K, N, device="cuda")
    y = torch.rand(M, N, device="cuda") * 1.6 - 0.8
    ep = capi.Go1GemmEpilogue()
    ep.act, ep.act_kind = act, kind
    if act == 2:
        ep.dact_y, ep.ld_dact_y = y.data_ptr(), y.stride(0)
    cs_row, cs_t = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    ep.colsum = cs_row.data_ptr()
    C = torch.empty(M, N, device="cuda")
    _gemm_ex(0, 0, M, N, K, A, B, C, N, ep)
    MP = (M + 31) // 32 * 32 + 32
    CT = torch.full((N, MP), 7.0, device="cuda")
    ep.colsum, ep.store_transposed = cs_t.data_ptr(), 1
    _gemm_ex(0, 0, M, N, K, A, B, CT, MP, ep)
    torch.cuda.synchronize()
    assert torch.equal(CT[:, :M].t(), C)
    assert bool((CT[:, (M + 3) // 4 * 4:] == 7.0).all())       # the TMA store writes 16-byte chunks: padding past them is untouched
    # atomic column sums: same values, another order of the per-warp partial sums
    assert float((cs_t - cs_row).abs().max()) <= 1e-5 * float(cs_row.abs().max())
    ref = A.double() @ B.double()
    if act == 2:
        yd = y.double()
        ref = ref * (torch.where(yd > 0, 1.0, yd + 1.0) if kind == 0 else 1.0 - yd * yd)
    tol = 2.0 ** -9 * (A.abs().double() @ B.abs().double()) + 1e-4
    assert bool(((C.double() - ref).abs() <= tol).all())


def test_transposed_store_rejects_unsupported_layouts():
    from go1_b200 import capi
    A, B = torch.randn(16, 64, device="cuda"), torch.randn(64, 64, device="cuda")
    CT = torch.empty(64, 32, device="cuda")
    ep = capi.Go1GemmEpilogue()
    ep.store_transposed = 1
    with pytest.raises(capi.Go1Error):          # M < 32: no 32 x 32 block of C^T for the TMA store
        _gemm_ex(0, 0, 16, 64, 64, A, B, CT, 32, ep)
    with pytest.raises(capi.Go1Error):          # the fp32 CUDA-core path has no transposed store
        capi.check(capi.lib().go1_gemm_ex(0, 0, 16, 64, 64, capi.ptr(A), 64, capi.ptr(B), 64, capi.ptr(CT), 32, ep, 0, capi.stream_ptr()), "gemm_ex")


@pytest.mark.parametrize("M", [1000, 4096])
def test_kmajor_first_layer_wgrad_matches_autograd(M):
    """backward_ppo and backward_adaptation with the transposed history a caller keeps (RolloutStorage): every gradient, the first
    layers' bias and trailing-input (priv / latent) columns included, against fp64 autograd at the TF32 tolerance."""
    import copy
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args, history_kmajor
    AC_Args.gemm_impl, AC_Args.activation = 1, "elu"
    torch.manual_seed(5)
    NOBS, NH, NP, NA = 70, 2100, 2, 12
    ac = ActorCritic(NOBS, NP, NH, NA).to("cuda:0")
    ac.flatten()
    hb = torch.randn(M, 2112, device="cuda") * 0.3          # the minibatch row buffer: 2112-float pitch
    h = hb[:, :NH]
    priv = torch.randn(M, NP, device="cuda")
    hT = history_kmajor(h, priv, torch.empty(NH + 1 + 2 * NP, (M + 31) // 32 * 32, device="cuda"))
    dmean, dvalue, dstd = torch.randn(M, NA, device="cuda") / M, torch.randn(M, 1, device="cuda") / M, torch.randn(NA, device="cuda")
    ac.forward_all(h, priv, tag="train")
    ac.flat_grads.fill_(3.0)                                     # overwritten, not accumulated into
    ac.backward_ppo(h, priv, dmean, dvalue, dstd, hT=hT)
    torch.cuda.synchronize()
    g = ac.flat_grads.clone()
    assert torch.equal(hT[NH + 1 + NP:, :M].t(), ac._latent)     # the latent rows were written
    ref = {k: copy.deepcopy(getattr(ac, k)).double() for k in ("adaptation_module", "actor_body", "critic_body")}
    hd, pd = h.double(), priv.double()
    lat = ref["adaptation_module"](hd)
    ((ref["actor_body"](torch.cat((hd, lat), -1)) * dmean.double()).sum() + (ref["critic_body"](torch.cat((hd, pd), -1)) * dvalue.double()).sum()).backward()

    def check(grads, mods, what):
        for name in mods:
            for (pn, p_ref), p in zip(ref[name].named_parameters(), getattr(ac, name).parameters()):
                off = (p.data_ptr() - ac.flat_params.data_ptr()) // 4
                got = grads[off: off + p.numel()].view_as(p)
                err = (got.double() - p_ref.grad).abs().max() / (p_ref.grad.abs().max() + 1e-12)
                assert float(err) < 5e-3, (what, name, pn, float(err))        # TF32 products: 2^-11 per operand

    check(g, ref, "backward_ppo")
    for mod in ref.values():
        mod.zero_grad()
    outs = ac.adaptation_forward(h)
    dpred = torch.randn(M, NP, device="cuda") / M
    ac.flat_grads.fill_(3.0)                                     # overwritten, not accumulated into
    ac.backward_adaptation(h, outs, dpred, hT=hT)
    torch.cuda.synchronize()
    (ref["adaptation_module"](hd) * dpred.double()).sum().backward()
    check(ac.flat_grads, ("adaptation_module",), "backward_adaptation")


def test_split_count_of_production_wgrads(tmp_path, monkeypatch):
    """The fused first-layer wgrad (1280 x 2105 x 24576: 170 tiles) and the adaptation step's (256 x 2101 x 24576: 34 tiles) with
    K-major operands are split by the wave-quantised makespan: 3 and 11 splits on a 132-SM H100 SXM."""
    from go1_b200 import capi
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != 132:
        pytest.skip(f"split counts are stated for 132 SMs, this device has {sms}")
    L = capi.lib()
    M = 24576
    B = torch.randn(2105, M, device="cuda")
    out = tmp_path / "gemm.csv"
    monkeypatch.setenv("GO1_GEMM_TIMING_CSV", str(out))
    capi.check(L.go1_gemm_timing(1, None, None, None), "timing")
    for rows, n in ((1280, 2105), (256, 2101)):
        A = torch.randn(rows, M, device="cuda")
        C = torch.empty(rows, 2112, device="cuda")
        capi.check(L.go1_gemm(0, 1, rows, n, M, capi.ptr(A), M, capi.ptr(B), M, capi.ptr(C), 2112, None, 0, 0, 1, capi.stream_ptr()), "gemm")
    capi.check(L.go1_gemm_timing(0, None, None, None), "timing")
    rows = list(csv.DictReader(open(out)))
    got = {(int(r["M"]), int(r["N"])): (int(r["splits"]), int(r["a_mn_major"]), int(r["b_mn_major"])) for r in rows}
    assert got == {(1280, 2105): (3, 0, 0), (256, 2101): (11, 0, 0)}
