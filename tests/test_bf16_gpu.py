"""AC_Args.gemm_impl = 2: the learner's observation-history products on BF16 tensor cores (go1_gemm_bf16_ex), the BF16 transposed dgrad
store and the converting data movement, against fp64 references on the same BF16-rounded operands and bit for bit against torch."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))

ACTS = ["elu", "selu", "relu", "lrelu", "tanh", "sigmoid"]
F64 = {"elu": torch.nn.functional.elu, "selu": torch.selu, "relu": torch.relu, "lrelu": lambda v: torch.nn.functional.leaky_relu(v, 0.01),
       "tanh": torch.tanh, "sigmoid": torch.sigmoid}


def _bf16(shape, pitch=None, seed=0, scale=1.0):
    """A BF16 CUDA matrix with row pitch `pitch` (default capi.bf16_pitch) and its fp64 values."""
    from go1_b200 import capi
    g = torch.Generator(device="cuda").manual_seed(seed)
    rows, cols = shape
    buf = torch.zeros(rows, pitch or capi.bf16_pitch(cols), device="cuda", dtype=torch.bfloat16)
    x = buf[:, :cols]
    x.copy_((torch.randn(rows, cols, device="cuda", generator=g) * scale).to(torch.bfloat16))
    return x, x.double()


def _gemm16(M, N, K, A, B, C, ep):
    from go1_b200 import capi
    capi.check(capi.lib().go1_gemm_bf16_ex(0, 1, M, N, K, capi.ptr(A), A.stride(0), capi.ptr(B), B.stride(0), capi.ptr(C), C.stride(0) if C is not None else 0,
                                           ep, capi.stream_ptr()), "go1_gemm_bf16_ex")


def _bound(A64, B64, K):
    """fp32-accumulation bound on identical operands: c K 2^-24 (|A| |B|^T), c = 4 (split-K partial sums and the epilogue's few fp32 adds)."""
    return 4.0 * K * 2.0 ** -24 * (A64.abs() @ B64.abs().t()) + 1e-30


@pytest.mark.parametrize("M,N,K", [(4096, 1280, 2100), (24576, 1280, 2100), (24576 + 37, 256, 2130), (300, 96, 70), (33, 40, 8)])
def test_bf16_gemm_matches_fp64_on_rounded_operands(M, N, K):
    from go1_b200 import capi
    A, A64 = _bf16((M, K), seed=1)
    B, B64 = _bf16((N, K), seed=2)
    C = torch.full((M, N + 5), 7.0, device="cuda")
    ep = capi.Go1GemmEpilogue()
    _gemm16(M, N, K, A, B, C[:, :N], ep)
    ref = A64 @ B64.t()
    err = (C[:, :N].double() - ref).abs()
    assert (err <= _bound(A64, B64, K)).all(), float((err / _bound(A64, B64, K)).max())
    assert (C[:, N:] == 7.0).all()        # ldc padding untouched


def test_bf16_gemm_kmajor_wgrad_split_k():
    """The fused first-layer weight gradient of scripts/train.py: [1280][2105] = dz1T [1280][24576] hT [2105][24576]^T (split-K partial
    tiles reduced in C)."""
    from go1_b200 import capi
    M, N, K = 1280, 2105, 24576
    A, A64 = _bf16((M, K), seed=3)
    B, B64 = _bf16((N, K), seed=4)
    C = torch.empty(M, 2112, device="cuda")
    ep = capi.Go1GemmEpilogue()
    _gemm16(M, N, K, A, B, C[:, :N], ep)
    err = (C[:, :N].double() - A64 @ B64.t()).abs()
    assert (err <= _bound(A64, B64, K)).all()


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("nex", [1, 2, 3, 4])
def test_bf16_gemm_fused_epilogues(act, nex):
    """bias + activation on the leading columns, 1..4 trailing-input columns on the same ones (fp32 operands), as the fused first-layer
    forward of ActorCritic uses them; then accumulate."""
    from go1_b200 import capi
    M, N, K, lead = 1000, 384, 2100, 256
    A, A64 = _bf16((M, K), seed=5, scale=0.05)
    B, B64 = _bf16((N, K), seed=6, scale=0.05)
    g = torch.Generator(device="cuda").manual_seed(7)
    bias = torch.randn(N, device="cuda", generator=g)
    ex = torch.randn(M, nex, device="cuda", generator=g)
    wex = torch.randn(N, nex, device="cuda", generator=g)
    C = torch.empty(M, N, device="cuda")
    ep = capi.Go1GemmEpilogue()
    ep.bias, ep.act, ep.act_kind, ep.lead_cols = bias.data_ptr(), 1, capi.ACTIVATIONS[act], lead
    ep.extra, ep.ld_extra, ep.w_extra, ep.ld_w_extra, ep.num_extra = ex.data_ptr(), nex, wex.data_ptr(), nex, nex
    _gemm16(M, N, K, A, B, C, ep)
    z = A64 @ B64.t() + bias.double()
    z[:, :lead] += ex.double() @ wex.double()[:lead].t()
    ref = z.clone()
    ref[:, :lead] = F64[act](z[:, :lead])
    # the activation is applied in fp32 (act_fast): a few fp32 ulps of z, times |f'| <= 1.06 (selu)
    tol = 1.1 * _bound(A64, B64, K) + 4e-6 * (1 + z.abs())
    assert ((C.double() - ref).abs() <= tol).all(), float((C.double() - ref).abs().max())
    # accumulate (no activation): C += A B^T
    ep2 = capi.Go1GemmEpilogue()
    ep2.accumulate = 1
    C0 = C.clone()
    _gemm16(M, N, K, A, B, C, ep2)
    assert ((C.double() - (C0.double() + A64 @ B64.t())).abs() <= _bound(A64, B64, K) + 2e-7 * (1 + C0.double().abs())).all()


def test_bf16_gemm_rejects_bad_layouts():
    from go1_b200 import capi
    A, _ = _bf16((256, 100), pitch=104)
    B, _ = _bf16((128, 100), pitch=104)
    C = torch.empty(256, 128, device="cuda")
    ep = capi.Go1GemmEpilogue()
    L, st = capi.lib(), capi.stream_ptr()
    for ta, tb in ((1, 1), (0, 0), (1, 0)):        # MN-major operands are not taken
        assert L.go1_gemm_bf16_ex(ta, tb, 256, 128, 100, capi.ptr(A), A.stride(0), capi.ptr(B), B.stride(0), capi.ptr(C), 128, ep, st) != 0
    assert L.go1_gemm_bf16_ex(0, 1, 256, 128, 100, capi.ptr(A), 100, capi.ptr(B), 104, capi.ptr(C), 128, ep, st) != 0     # lda % 8 != 0
    # a BF16 output needs store_transposed
    out = torch.empty(128, 256, device="cuda", dtype=torch.bfloat16)
    ep.out_bf16, ep.ld_out_bf16 = out.data_ptr(), 256
    assert L.go1_gemm_bf16_ex(0, 1, 256, 128, 100, capi.ptr(A), 104, capi.ptr(B), 104, capi.ptr(C), 128, ep, st) != 0


@pytest.mark.parametrize("M", [24576, 1000, 33])
def test_bf16_transposed_dgrad_store_is_bitwise_rne_of_fp32_store(M):
    """The layer-2 dgrad with store_transposed and out_bf16 writes exactly torch's .to(bfloat16) of what the fp32 transposed store writes
    (same kernel, same sums), and the fp32-side reductions (column sums, trailing-input terms) are unchanged."""
    from go1_b200 import capi
    N, K = 512, 256           # dz1 [M][512] = (dz2 [M][256] W2 [256][512]) * f'(y1)
    g = torch.Generator(device="cuda").manual_seed(M)
    dz2 = torch.randn(M, K, device="cuda", generator=g)
    W2 = torch.randn(K, N, device="cuda", generator=g) * 0.05
    y1 = torch.randn(M, N, device="cuda", generator=g)
    ex = torch.randn(M, 2, device="cuda", generator=g)
    wex = torch.randn(N, 2, device="cuda", generator=g)
    outs = []
    for bf16 in (False, True):
        dx = torch.zeros(M, 2, device="cuda")
        ep = capi.Go1GemmEpilogue()
        ep.act, ep.dact_y, ep.ld_dact_y, ep.store_transposed = 2, y1.data_ptr(), N, 1
        ep.bwd_extra, ep.ld_bwd_extra, ep.bwd_w_extra, ep.ld_bwd_w_extra, ep.d_extra, ep.ld_d_extra, ep.num_bwd_extra = \
            ex.data_ptr(), 2, wex.data_ptr(), 2, dx.data_ptr(), 2, 2
        P = capi.bf16_pitch(M) if bf16 else capi.row_pitch(M)
        if bf16:
            T = torch.full((N, P), 3.0, device="cuda", dtype=torch.bfloat16)
            ep.out_bf16, ep.ld_out_bf16 = T.data_ptr(), P
            C = None
        else:
            T = torch.zeros(N, P, device="cuda")
            C = T
        capi.check(capi.lib().go1_gemm_ex(0, 0, M, N, K, capi.ptr(dz2), K, capi.ptr(W2), N, capi.ptr(C), P, ep, 1, capi.stream_ptr()), "dgrad")
        outs.append((T, dx))
    (T32, dx32), (T16, dx16) = outs
    assert torch.equal(T16[:, :M].view(torch.int16), T32[:, :M].to(torch.bfloat16).view(torch.int16))
    M8 = (M + 7) // 8 * 8        # the TMA store writes whole 16-byte chunks (8 BF16): padding beyond them stays untouched
    assert (T16[:, M8:] == 3.0).all()
    assert torch.allclose(dx16, dx32, rtol=1e-5, atol=1e-5)     # (atomic order)


def test_bf16_converters_are_bitwise_torch_rounding():
    from go1_b200 import capi
    L, st = capi.lib(), capi.stream_ptr()
    g = torch.Generator(device="cuda").manual_seed(11)
    src = torch.randn(300, 2130, device="cuda", generator=g) * torch.logspace(-30, 30, 2130, device="cuda")
    src[0, :8] = torch.tensor([0.0, -0.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, float("inf"), -float("inf"), 3.0e38, 1e-40], device="cuda")
    want = src.to(torch.bfloat16).view(torch.int16)
    P = capi.bf16_pitch(2130)
    # convert
    dst = torch.full((300, P), 5.0, device="cuda", dtype=torch.bfloat16)
    capi.check(L.go1_convert_bf16(capi.ptr(src), 2130, capi.ptr(dst), P, 300, 2130, st), "convert")
    assert torch.equal(dst[:, :2130].view(torch.int16), want) and (dst[:, 2130:] == 5.0).all()
    # the rollout's store into slot *slot_dev of a BF16 slab [T][rows][pitch], then the minibatch gather from it (both copy)
    T = 3
    slab = torch.full((T, 300, P), 5.0, device="cuda", dtype=torch.bfloat16)
    slot = torch.tensor([2], dtype=torch.int32, device="cuda")
    src16 = src.to(torch.bfloat16)
    capi.check(L.go1_rollout_store_rows_bf16(capi.ptr(src16), 2130, capi.ptr(slab), P, capi.ptr(slot), 300, 2130, st), "store_rows")
    assert torch.equal(slab[2, :, :2130].view(torch.int16), want) and (slab[2, :, 2130:] == 5.0).all() and (slab[:2] == 5.0).all()
    idx = (600 + torch.randperm(300, device="cuda", generator=g)[:200]).contiguous()
    dst = torch.full((200, P), 5.0, device="cuda", dtype=torch.bfloat16)
    capi.check(L.go1_gather_rows_bf16(capi.ptr(slab), P, capi.ptr(idx), capi.ptr(dst), P, 200, 2130, st), "gather")
    assert torch.equal(dst[:, :2130].view(torch.int16), want[idx - 600]) and (dst[:, 2130:] == 5.0).all()
    # transposes: fp32 -> BF16 (rounded), BF16 -> BF16 (copied)
    Mp = capi.bf16_pitch(300)
    dT = torch.full((2130, Mp + 8), 5.0, device="cuda", dtype=torch.bfloat16)
    capi.check(L.go1_transpose_to_bf16(capi.ptr(src), 2130, capi.ptr(dT), Mp + 8, 300, 2130, st), "transpose_to_bf16")
    assert torch.equal(dT[:, :300].view(torch.int16), want.t()) and (dT[:, 300:] == 5.0).all()
    s16 = src.to(torch.bfloat16)
    dT2 = torch.full((2130, Mp + 8), 5.0, device="cuda", dtype=torch.bfloat16)
    capi.check(L.go1_transpose_bf16(capi.ptr(s16), 2130, capi.ptr(dT2), Mp + 8, 300, 2130, st), "transpose_bf16")
    assert torch.equal(dT2, dT)
    assert L.go1_convert_bf16(capi.ptr(src), 2130, capi.ptr(dst), 100, 300, 2130, st) != 0      # ldd < cols


# ------------------------------------------------------------------------------------------------------------ ActorCritic at impl 2
def _ac_case(K0, E, hidden, act, M, seed=0):
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    saved = (AC_Args.actor_hidden_dims, AC_Args.critic_hidden_dims, AC_Args.activation)
    AC_Args.actor_hidden_dims = AC_Args.critic_hidden_dims = hidden
    AC_Args.activation = act
    torch.manual_seed(seed)
    try:
        ac = ActorCritic(70, E, K0, 12).cuda()
    finally:
        AC_Args.actor_hidden_dims, AC_Args.critic_hidden_dims, AC_Args.activation = saved
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    h = torch.randn(M, K0, device="cuda", generator=g)
    priv = torch.randn(M, E, device="cuda", generator=g)
    dmean = torch.randn(M, 12, device="cuda", generator=g) / M
    dvalue = torch.randn(M, 1, device="cuda", generator=g) / M
    return ac, h, priv, dmean, dvalue


def _reference(ac, h, priv, dmean, dvalue, act, rounded):
    """fp64 forward / backward of the three MLPs.  rounded: the history, the first-layer weight blocks W[:, :K0] and the first-layer dz (for
    the weight gradients, whose augmented operand rows -- ones, priv, latent -- are rounded too) in BF16 exactly where the kernels round them."""
    r = (lambda t: t.to(torch.bfloat16).double()) if rounded else (lambda t: t.double())
    K0 = h.shape[1]
    f = F64[act]
    hr = r(h)
    params = {k: v.detach().double().clone().requires_grad_(True) for k, v in ac.state_dict().items() if k != "std"}
    pre = {}

    def mlp(prefix, x_extra):
        idx = sorted({int(k.split(".")[1]) for k in params if k.startswith(prefix + ".")})
        W0, b0 = params[f"{prefix}.{idx[0]}.weight"], params[f"{prefix}.{idx[0]}.bias"]
        W0k = W0[:, :K0]
        Wr = W0k + (r(W0k.detach()) - W0k.detach())       # the rounded values, the gradient of W0k
        z = hr @ Wr.t() + b0
        if x_extra is not None:
            z = z + x_extra @ W0[:, K0:].t()
        z.retain_grad()
        pre[prefix] = (z, x_extra)
        y = f(z)
        for j, li in enumerate(idx[1:]):
            y = y @ params[f"{prefix}.{li}.weight"].t() + params[f"{prefix}.{li}.bias"]
            if j < len(idx) - 2:
                y = f(y)
        return y

    latent = mlp("adaptation_module", None)
    mean = mlp("actor_body", latent)
    value = mlp("critic_body", priv.double())
    (mean * dmean.double()).sum().backward(retain_graph=True)
    (value * dvalue.double()).sum().backward()
    grads = {k: v.grad for k, v in params.items()}
    for prefix, (z, xe) in pre.items():        # the first-layer weight / bias gradients as the K-major BF16 product forms them
        idx = min(int(k.split(".")[1]) for k in params if k.startswith(prefix + "."))
        dz = r(z.grad)
        grads[f"{prefix}.{idx}.bias"] = dz.sum(0)
        gW = dz.t() @ hr
        if xe is not None:
            gW = torch.cat([gW, dz.t() @ r(xe.detach())], 1)
        grads[f"{prefix}.{idx}.weight"] = gW
    return mean.detach(), value.detach(), grads


@pytest.mark.parametrize("K0,E,hidden,act", [(2100, 2, [512, 256, 128], "elu"), (2130, 45, [512, 256, 128], "elu"),
                                              (2100, 2, [130, 70, 33], "tanh")])
def test_actor_critic_impl2_matches_fp64_reference(K0, E, hidden, act):
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    M = 4096
    ac, h, priv, dmean, dvalue = _ac_case(K0, E, hidden, act, M)
    AC_Args.gemm_impl = 2
    try:
        mean, value = ac.forward_all(h, priv, tag="train")
        mean, value = mean.clone(), value.clone()
        ac.backward_ppo(h, priv, dmean, dvalue, torch.zeros(12, device="cuda"))
        torch.cuda.synchronize()
    finally:
        AC_Args.gemm_impl = 1
    flatg = ac.flat_grads
    got = {}
    for name, p in ac.named_parameters():
        if name == "std":
            continue
        off = (p.data_ptr() - ac.flat_params.data_ptr()) // 4
        got[name] = flatg[off:off + p.numel()].view(p.shape).double()
    rel = lambda a, b: float((a - b).abs().max() / (b.abs().max() + 1e-30))
    errs = {}
    for rounded in (True, False):
        rm, rv, rg = _reference(ac, h, priv, dmean, dvalue, act, rounded)
        errs[rounded] = {"mean": rel(mean.double(), rm), "value": rel(value.double(), rv), **{n: rel(got[n], w) for n, w in rg.items()}}
    print("max relative error against the BF16-rounded / the unrounded fp64 reference:",
          {n: (round(errs[True][n], 5), round(errs[False][n], 5)) for n in errs[True]})
    # against the reference that rounds where the kernels round, only the hidden layers' TF32 (2^-11 relative per operand) and fp32
    # accumulation remain: impl 1's bounds.  Against the unrounded reference BF16's operand rounding (unit roundoff 2^-9, 4x TF32's) adds
    # to that: the bound is 4x, and the errors there must be the larger ones on the history products' outputs (what BF16 costs).
    for n, e in errs[True].items():
        assert e < (2e-2 if n in ("mean", "value") else 3e-2), (n, errs[True])
    for n, e in errs[False].items():
        assert e < 4 * (2e-2 if n in ("mean", "value") else 3e-2), (n, errs[False])


def test_rollout_ratio_consistency_impl2():
    """The rollout's policy evaluation and the update's first minibatch read the same BF16 history and weights: the recomputed log pi of the
    stored actions equals the stored one up to fp32 accumulation order (|d log pi| < 2e-3 over 12 actions) and the KL is ~0 (< 1e-6)."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.ppo import PPO
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    N, T, NOBS, NH, NP, NA = 1024, 4, 70, 2100, 2, 12
    AC_Args.gemm_impl = 2
    try:
        torch.manual_seed(0)
        ac = ActorCritic(NOBS, NP, NH, NA)
        alg = PPO(ac, device="cuda:0")
        alg.init_storage(N, T, [NOBS], [NP], [NH], [NA])
        g = torch.Generator(device="cuda").manual_seed(3)
        for t in range(T):
            obs = torch.randn(N, NOBS, device="cuda", generator=g)
            priv = torch.randn(N, NP, device="cuda", generator=g)
            hist = torch.randn(N, NH, device="cuda", generator=g)
            alg.act(obs, priv, hist)
            alg.process_env_step(torch.randn(N, device="cuda", generator=g), torch.zeros(N, dtype=torch.bool, device="cuda"),
                                 {"env_bins": torch.zeros(N, device="cuda"), "time_outs": torch.zeros(N, dtype=torch.bool, device="cuda")})
        batch = next(alg.storage.mini_batch_generator(4, 1))
        hist_b, priv_b, actions_b, old_logp_b, old_mu_b = batch[3], batch[2], batch[4], batch[8], batch[9]
        assert hist_b.dtype == torch.bfloat16
        mean, _ = ac.forward_all(hist_b, priv_b, tag="train")
        std = ac.std.detach()
        logp = (-(actions_b - mean) ** 2 / (2 * std ** 2) - torch.log(std) - 0.9189385332046727).sum(-1)
        d = (logp - old_logp_b.view(-1)).abs().max().item()
        kl = (((mean - old_mu_b) ** 2) / (2 * std ** 2)).sum(-1).mean().item()
    finally:
        AC_Args.gemm_impl = 1
    assert d < 2e-3, d
    assert kl < 1e-6, kl


def test_full_ppo_cycle_matches_reference_golden_impl2():
    """test_full_ppo_cycle_matches_reference_golden at impl 2.  Its impl-1 factors (k = 250 on the rollout quantities, kl = 25 on the
    losses) come from TF32's 2^-10 unit roundoff; BF16's is 2^-8, 4x larger, on the history products, so the factors here are 4 x
    those: k = 1000, kl = 100, and the weight comparison bounds are 4 x impl 1's.  The golden run has 4 envs x 24 steps, so its
    minibatches have 24 rows: the forward passes (rollout and update) run the BF16 history products, but the update's backward takes the
    CUDA-core path of minibatches under 64 rows on the BF16-rounded history in fp32.  The BF16 transposed dz store and the BF16
    first-layer weight gradients are covered by test_actor_critic_impl2_matches_fp64_reference and the Runner test below."""
    from ppo_golden_util import seeded_weights, sample_tensor
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.ppo import PPO
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.gemm_impl = 2
    k, kl = 1000.0, 100.0
    try:
        g = np.load(os.path.join(HERE, "golden", "ppo.npz"))
        N, T, NOBS, NH, NP, NA = 4, 24, 70, 2100, 2, 12
        ac = ActorCritic(NOBS, NP, NH, NA)
        w = seeded_weights({kk: tuple(v.shape) for kk, v in ac.state_dict().items()})
        ac.load_state_dict({kk: torch.from_numpy(v) for kk, v in w.items()})
        alg = PPO(ac, device="cuda:0")
        alg.init_storage(N, T, [NOBS], [NP], [NH], [NA])
        C = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        for t in range(T):
            ac.injected_eps = C(g["in/eps"][t])
            alg.act(C(g["in/obs"][t]), C(g["in/priv"][t]), C(g["in/hist"][t]))
            infos = {"env_bins": torch.zeros(N, device="cuda"), "time_outs": torch.zeros(N, dtype=torch.bool, device="cuda")}
            alg.process_env_step(C(g["in/rew"][t]), C(g["in/done"][t]), infos)
        alg.compute_returns(C(g["last/hist"]), C(g["last/priv"]))
        st = alg.storage
        for name, tol in (("actions", 2e-5), ("values", 2e-5), ("actions_log_prob", 1e-4), ("mu", 2e-5), ("returns", 5e-5), ("advantages", 2e-4)):
            got, want = getattr(st, name).cpu().numpy(), g[f"storage/{name}"]
            assert np.allclose(got, want, rtol=1e-4 * k, atol=tol * k), (name, np.abs(got - want).max())
        alg.fixed_minibatch_indices = C(g["in/perm"])
        losses = alg.update()
    finally:
        AC_Args.gemm_impl = 1
    ref = g["update/losses"]
    assert abs(losses[0] - ref[0]) < 2e-3 * kl * abs(ref[0]) and abs(losses[1] - ref[1]) < 2e-3 * kl and abs(losses[2] - ref[2]) < 2e-3 * kl * abs(ref[2])
    assert abs(losses[5] - ref[5]) < 2e-3 * kl * abs(ref[5])
    for name_k, v in ac.state_dict().items():
        got, want = sample_tensor(v.cpu().numpy()), g[f"final/{name_k}"]
        d = np.abs(got[:-2] - want[:-2])
        assert np.quantile(d, 0.99) < 1.6e-2 and d.max() < 1.6e-1, (name_k, np.quantile(d, 0.99), d.max())
        assert abs(got[-1] - want[-1]) <= 2e-2 * max(1.0, abs(want[-1])), name_k


def test_graph_replayed_rollout_equals_eager_rollout_impl2(tmp_path, monkeypatch):
    """test_graph_replayed_rollout_equals_eager_rollout with the BF16 history products (the conversion of the history runs inside the
    captured policy evaluation)."""
    import test_runner_gpu
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    monkeypatch.setattr(AC_Args, "gemm_impl", 2)
    test_runner_gpu.test_graph_replayed_rollout_equals_eager_rollout(tmp_path, monkeypatch)


def test_runner_learn_impl2_checkpoint_loads_at_impl1(tmp_path, monkeypatch):
    """A few Runner.learn iterations at impl 2 on the scripts/train.py configuration (4096 envs): finite weights, the history slab in BF16,
    an fp32 state_dict.  The checkpoint loads into an impl-1 ActorCritic, and the TorchScript export that scripts/play.py loads
    (body_latest.jit behind adaptation_module_latest.jit) gives the impl-1 actions within the TF32 tolerance."""
    import test_runner_gpu
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    monkeypatch.chdir(tmp_path)                      # Runner.save writes ./tmp/legged_data like the reference
    monkeypatch.setattr(AC_Args, "gemm_impl", 2)
    env, Runner, RunnerArgs, logger = test_runner_gpu._make(tmp_path, n=4096)
    RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval = 24, 100, 100, 100
    RunnerArgs.resume = False
    runner = Runner(env, device="cuda:0")
    assert runner.alg.storage._hist_slab.element_size() == 2
    runner.learn(num_learning_iterations=3, init_at_random_ep_len=True, eval_freq=100)
    ac = runner.alg.actor_critic
    assert torch.isfinite(ac.flat_params).all()
    sd = ac.state_dict()
    assert all(v.dtype == torch.float32 for v in sd.values())
    hist = env.obs_history[:512, :env.num_obs_history].contiguous()
    monkeypatch.setattr(AC_Args, "gemm_impl", 1)
    ac1 = ActorCritic(env.num_obs, env.num_privileged_obs, env.num_obs_history, env.num_actions).cuda()
    ac1.load_state_dict(sd)
    want = ac1.act_student(hist).cpu()
    body = torch.jit.load(os.path.join("tmp", "legged_data", "body_latest.jit"))
    adapt = torch.jit.load(os.path.join("tmp", "legged_data", "adaptation_module_latest.jit"))
    h = hist.cpu()
    with torch.no_grad():
        got = body(torch.cat((h, adapt(h)), dim=-1))
    # TF32 (impl 1) against TorchScript's fp32: 2^-11 relative per operand over K0 = 2100 products, 4 layers deep
    assert torch.allclose(got, want, rtol=1e-2, atol=1e-2 * float(want.abs().max())), float((got - want).abs().max())
