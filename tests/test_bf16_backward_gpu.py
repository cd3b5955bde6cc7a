"""AC_Args.bf16_backward: the hidden layers' dgrads and weight gradients on BF16 tensor cores with MN-major operands read in place
(go1_gemm_bf16_mn / go1_gemm_bf16_grouped), the row-major BF16 store, the multi-segment conversion, and ActorCritic in the mode against
fp64 references."""
import csv
import itertools
import os
import sys

import pytest
import torch

from test_bf16_gpu import ACTS, F64, _bf16, _bound

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))


def _operand(ta, rows, cols, seed, scale=1.0):
    """A BF16 operand of logical shape [rows][cols] in the major `ta` asks for (1: stored transposed), its stored tensor and fp64 values."""
    if ta:
        t, t64 = _bf16((cols, rows), seed=seed, scale=scale)
        return t, t64.t()
    t, t64 = _bf16((rows, cols), seed=seed, scale=scale)
    return t, t64


def _mn(ta, tb, M, N, K, A, B, C, ep, c16=0, ldc=None):
    from go1_b200 import capi
    return capi.lib().go1_gemm_bf16_mn(ta, tb, M, N, K, capi.ptr(A), A.stride(0), capi.ptr(B), B.stride(0), capi.ptr(C),
                                       ldc if ldc is not None else (C.stride(0) if C is not None else 0), c16, ep, capi.stream_ptr())


def _case(ta, tb, M, N, K, seed=0, scale=1.0):
    # A is op(A) [M][K]: transA 0 = [M][K] stored, 1 = [K][M];  B is op(B)^T [N][K] logically: transB 1 = [N][K], 0 = [K][N]
    A, A64 = _operand(ta, M, K, seed + 1, scale)
    B, B64t = _operand(1 - tb, N, K, seed + 2, scale)      # B64t: [N][K]
    return A, A64, B, B64t


LAYOUTS = [(0, 0), (0, 1), (1, 0), (1, 1)]


@pytest.mark.parametrize("ta,tb", LAYOUTS)
@pytest.mark.parametrize("M,N,K", [(24576, 512, 256), (1000, 130, 250), (65, 12, 12), (24576, 256, 128), (1000, 256, 24576), (130, 512, 24576),
                                   (65, 130, 1000)])
def test_bf16_mn_gemm_matches_fp64_on_rounded_operands(ta, tb, M, N, K):
    """Every layout on ragged shapes (tiles and k-blocks partly beyond M, N, K read as zeros), BN = 32 / 64 / 128 and split-K (K = 24576)."""
    A, A64, B, B64 = _case(ta, tb, M, N, K)
    C = torch.full((M, N + 5), 7.0, device="cuda")
    from go1_b200 import capi
    assert _mn(ta, tb, M, N, K, A, B, C[:, :N], capi.Go1GemmEpilogue()) == 0
    err = (C[:, :N].double() - A64 @ B64.t()).abs()
    assert (err <= _bound(A64, B64, K)).all(), float((err / _bound(A64, B64, K)).max())
    assert (C[:, N:] == 7.0).all()


def _dgrad_ep(M, N, nbx, kind, seed, colsum=True):
    """The epilogue of a hidden-layer dgrad: act 2 from an fp32 saved output, column sums, nbx trailing-input terms."""
    from go1_b200 import capi
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.rand(M, N, device="cuda", generator=g) * 1.8 - 0.9       # inside every activation's range
    ex, wex = torch.randn(M, max(nbx, 1), device="cuda", generator=g), torch.randn(N, max(nbx, 1), device="cuda", generator=g)
    cs, gwx, dx = torch.zeros(N, device="cuda"), torch.zeros(N, max(nbx, 1), device="cuda"), torch.zeros(M, max(nbx, 1), device="cuda")
    ep = capi.Go1GemmEpilogue()
    ep.act, ep.act_kind, ep.dact_y, ep.ld_dact_y = 2, kind, y.data_ptr(), N
    if colsum:
        ep.colsum = cs.data_ptr()
    if nbx:
        ep.bwd_extra, ep.ld_bwd_extra, ep.bwd_w_extra, ep.ld_bwd_w_extra, ep.num_bwd_extra = ex.data_ptr(), nbx, wex.data_ptr(), nbx, nbx
        ep.g_w_extra, ep.ld_g_w_extra, ep.d_extra, ep.ld_d_extra = gwx.data_ptr(), nbx, dx.data_ptr(), nbx
    return ep, y, ex[:, :nbx], wex[:, :nbx], cs, gwx[:, :nbx], dx[:, :nbx]


def _deriv(act, y):
    """f'(z) from the output y = f(z), in fp64 (activation.cuh's act_deriv)."""
    return {"elu": lambda y: torch.where(y > 0, 1.0, y + 1.0), "selu": lambda y: torch.where(y > 0, 1.0507009873554805, y + 1.7580993408473766),
            "relu": lambda y: (y > 0).double(), "lrelu": lambda y: torch.where(y > 0, 1.0, 0.01), "tanh": lambda y: 1 - y * y,
            "sigmoid": lambda y: y * (1 - y)}[act](y)


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("ta,tb", [(0, 0), (1, 1)])
def test_bf16_mn_gemm_dgrad_epilogue(act, ta, tb):
    """act 2 with f' from the fp32 saved output for each activation kind, column sums, 1..4 trailing-input terms."""
    from go1_b200 import capi
    M, N, K = 3000, 300, 130
    nbx = 1 + ACTS.index(act) % 4
    A, A64, B, B64 = _case(ta, tb, M, N, K, seed=5, scale=0.3)
    ep, y, ex, wex, cs, gwx, dx = _dgrad_ep(M, N, nbx, capi.ACTIVATIONS[act], 6)
    C = torch.empty(M, N, device="cuda")
    assert _mn(ta, tb, M, N, K, A, B, C, ep) == 0
    v = (A64 @ B64.t()) * _deriv(act, y.double())
    tol = 1.1 * _bound(A64, B64, K) + 2e-6 * (1 + v.abs())
    assert ((C.double() - v).abs() <= tol).all(), float((C.double() - v).abs().max())
    rel = lambda a, b: float((a.double() - b).abs().max() / (b.abs().max() + 1e-30))
    assert rel(cs, v.sum(0)) < 1e-5
    assert rel(gwx, v.t() @ ex.double()) < 1e-5 and rel(dx, v @ wex.double()) < 1e-5


@pytest.mark.parametrize("M", [24576, 1000, 65])
def test_bf16_mn_transposed_bf16_store_is_bitwise_rne_of_fp32_store(M):
    """store_transposed + out_bf16 on the MN-major kernel (the layer-2 dgrad of AC_Args.bf16_backward: B = the BF16 W read MN-major)."""
    from go1_b200 import capi
    N, K = 512, 256
    A, A64, B, B64 = _case(0, 0, M, N, K, seed=M, scale=0.3)
    res = []
    for bf16 in (False, True):
        ep, *keep = _dgrad_ep(M, N, 2, 0, 9, colsum=False)      # (keep: the epilogue's operands stay allocated until the kernel has run)
        ep.store_transposed = 1
        if bf16:
            P = capi.bf16_pitch(M)
            T = torch.full((N, P), 3.0, device="cuda", dtype=torch.bfloat16)
            ep.out_bf16, ep.ld_out_bf16 = T.data_ptr(), P
            assert _mn(0, 0, M, N, K, A, B, None, ep) == 0
        else:
            T = torch.zeros(N, capi.row_pitch(M), device="cuda")
            assert _mn(0, 0, M, N, K, A, B, T, ep) == 0
        torch.cuda.synchronize()
        res.append(T)
    T32, T16 = res
    assert torch.equal(T16[:, :M].view(torch.int16), T32[:, :M].to(torch.bfloat16).view(torch.int16))
    assert (T16[:, (M + 7) // 8 * 8:] == 3.0).all()


@pytest.mark.parametrize("ta,tb", LAYOUTS)
@pytest.mark.parametrize("M,N,K", [(24576, 256, 512), (1000, 130, 70), (65, 12, 33), (300, 40, 24576)])
def test_bf16_mn_row_major_bf16_store_is_bitwise_rne_of_fp32_store(ta, tb, M, N, K):
    """c_bf16 = 1 writes exactly .to(torch.bfloat16) of what the fp32 output of the same call configuration holds (the same kernel, sums and
    epilogue), leaves the row padding beyond the written 16-byte chunks untouched, and its column sums see the fp32 values."""
    from go1_b200 import capi
    A, A64, B, B64 = _case(ta, tb, M, N, K, seed=3, scale=0.3)
    ep32, *keep32 = _dgrad_ep(M, N, 0, capi.ACTIVATIONS["tanh"], 4)      # (keep: the epilogue's operands stay allocated)
    cs32 = torch.zeros(N, device="cuda")
    ep32.colsum = cs32.data_ptr()
    C32 = torch.empty(M, N, device="cuda")
    assert _mn(ta, tb, M, N, K, A, B, C32, ep32) == 0
    ep16, *keep16 = _dgrad_ep(M, N, 0, capi.ACTIVATIONS["tanh"], 4)
    cs16 = torch.zeros(N, device="cuda")
    ep16.colsum = cs16.data_ptr()
    P = capi.bf16_pitch(N)
    C16 = torch.full((M, P + 8), 5.0, device="cuda", dtype=torch.bfloat16)
    assert _mn(ta, tb, M, N, K, A, B, C16, ep16, c16=1, ldc=P + 8) == 0
    torch.cuda.synchronize()
    assert torch.equal(C16[:, :N].view(torch.int16), C32.to(torch.bfloat16).view(torch.int16))
    assert (C16[:, (N + 7) // 8 * 8:] == 5.0).all()           # whole 16-byte chunks are written: padding beyond them is untouched
    # the column sums add the same fp32 values in another atomic order: M 2^-24 of the summed magnitudes
    assert ((cs16 - cs32).abs() <= M * 2.0 ** -24 * C32.abs().sum(0) + 1e-6).all()


def test_bf16_mn_rejects_bad_arguments():
    from go1_b200 import capi
    A, _ = _bf16((256, 100), pitch=104)
    B, _ = _bf16((128, 100), pitch=104)
    C = torch.empty(256, 128, device="cuda")
    ep = capi.Go1GemmEpilogue()
    L, st = capi.lib(), capi.stream_ptr()
    assert L.go1_gemm_bf16_mn(0, 1, 256, 128, 100, capi.ptr(A), 100, capi.ptr(B), 104, capi.ptr(C), 128, 0, ep, st) != 0     # lda % 8
    assert "multiples of 8 elements (TMA)" in L.go1_last_error().decode()
    assert L.go1_gemm_bf16_mn(2, 1, 256, 128, 100, capi.ptr(A), 104, capi.ptr(B), 104, capi.ptr(C), 128, 0, ep, st) != 0
    C16 = torch.empty(256, 132, device="cuda", dtype=torch.bfloat16)
    assert L.go1_gemm_bf16_mn(0, 1, 256, 128, 100, capi.ptr(A), 104, capi.ptr(B), 104, capi.ptr(C16), 132, 1, ep, st) != 0   # ldc % 8
    ep.accumulate = 1
    assert L.go1_gemm_bf16_mn(0, 1, 256, 128, 100, capi.ptr(A), 104, capi.ptr(B), 104, capi.ptr(C16), 128, 1, ep, st) != 0


@pytest.mark.parametrize("n", [2, 3, 4])
def test_bf16_grouped_equals_one_by_one(n):
    """The grouped weight gradients (dz^T y over the minibatch rows, both operands MN-major) against the same products launched one by one."""
    import ctypes as C
    from go1_b200 import capi
    M, N, K = 256, 512, 24576
    As, Bs = [_operand(1, M, K, 10 + p, 0.3)[0] for p in range(n)], [_operand(1, N, K, 20 + p, 0.3)[0] for p in range(n)]
    want = []
    for A, B in zip(As, Bs):
        Cw = torch.zeros(M, N, device="cuda")
        ep = capi.Go1GemmEpilogue()
        ep.accumulate = 1
        assert _mn(1, 0, M, N, K, A, B, Cw, ep) == 0
        want.append(Cw)
    got = [torch.zeros(M, N, device="cuda") for _ in range(n)]
    P = lambda ts: (C.c_void_p * n)(*[t.data_ptr() for t in ts])
    capi.check(capi.lib().go1_gemm_bf16_grouped(1, 0, M, N, K, n, P(As), As[0].stride(0), P(Bs), Bs[0].stride(0), P(got), N, 1, capi.stream_ptr()), "grouped")
    for A, B, g, w in zip(As, Bs, got, want):
        bound = _bound(A.double().t(), B.double().t(), K)
        assert ((g.double() - w.double()).abs() <= 2 * bound).all()


@pytest.mark.parametrize("o", [1, 2, 12])
def test_skinny_dgrad_bf16_is_bitwise_rne_of_fp32(o):
    """The head dgrad of the mode: go1_skinny_dgrad_act_bf16 stores exactly .to(torch.bfloat16) of go1_skinny_dgrad_act's fp32 output, its
    column sums equal the fp32 kernel's, and the row padding stays untouched."""
    from go1_b200 import capi
    L, st = capi.lib(), capi.stream_ptr()
    M, n = 24576, 128
    g = torch.Generator(device="cuda").manual_seed(o)
    dz, W = torch.randn(M, o, device="cuda", generator=g), torch.randn(o, n, device="cuda", generator=g)
    y = torch.rand(M, n, device="cuda", generator=g) * 1.8 - 0.9
    d32, cs32, cs16 = torch.empty(M, n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    d16 = torch.full((M, n + 8), 5.0, device="cuda", dtype=torch.bfloat16)
    kind = capi.ACTIVATIONS["tanh"]
    capi.check(L.go1_skinny_dgrad_act(capi.ptr(dz), o, capi.ptr(W), n, capi.ptr(y), n, capi.ptr(d32), n, capi.ptr(cs32), M, o, n, kind, st), "fp32")
    capi.check(L.go1_skinny_dgrad_act_bf16(capi.ptr(dz), o, capi.ptr(W), n, capi.ptr(y), n, capi.ptr(d16), n + 8, capi.ptr(cs16), M, o, n, kind, st), "bf16")
    torch.cuda.synchronize()
    assert torch.equal(d16[:, :n].view(torch.int16), d32.to(torch.bfloat16).view(torch.int16)) and (d16[:, n:] == 5.0).all()
    assert ((cs16 - cs32).abs() <= M * 2.0 ** -24 * d32.abs().sum(0) + 1e-6).all()
    assert L.go1_skinny_dgrad_act_bf16(capi.ptr(dz), o, capi.ptr(W), n, capi.ptr(y), n, capi.ptr(d16), n + 2, None, M, o, n, kind, st) != 0


def test_convert_bf16_segments_is_bitwise_torch_rounding():
    from go1_b200 import capi
    g = torch.Generator(device="cuda").manual_seed(2)
    big = torch.randn(700, 1300, device="cuda", generator=g) * 10
    srcs = [big[:, :512], big[:, 516:772], big[:300, 800:933], torch.randn(65, 33, device="cuda", generator=g)]
    dsts = [torch.full((s.shape[0], capi.bf16_pitch(s.shape[1])), 5.0, device="cuda", dtype=torch.bfloat16) for s in srcs]
    capi.convert_bf16_segments([(d[:, :s.shape[1]], s) for d, s in zip(dsts, srcs)])
    for d, s in zip(dsts, srcs):
        assert torch.equal(d[:, :s.shape[1]].view(torch.int16), s.to(torch.bfloat16).view(torch.int16)) and (d[:, s.shape[1]:] == 5.0).all()


# ------------------------------------------------------------------------------------------------------------ ActorCritic in the mode
def _ac_case(K0, E, hidden, act, M, seed=0):
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    saved = (AC_Args.actor_hidden_dims, AC_Args.critic_hidden_dims, AC_Args.adaptation_module_branch_hidden_dims, AC_Args.activation)
    AC_Args.actor_hidden_dims = AC_Args.critic_hidden_dims = hidden
    AC_Args.adaptation_module_branch_hidden_dims = hidden[1:] if len(hidden) > 2 else hidden
    AC_Args.activation = act
    torch.manual_seed(seed)
    try:
        ac = ActorCritic(70, E, K0, 12).cuda()
    finally:
        AC_Args.actor_hidden_dims, AC_Args.critic_hidden_dims, AC_Args.adaptation_module_branch_hidden_dims, AC_Args.activation = saved
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    h = torch.randn(M, K0, device="cuda", generator=g)
    priv = torch.randn(M, E, device="cuda", generator=g)
    dmean = torch.randn(M, 12, device="cuda", generator=g) / M
    dvalue = torch.randn(M, 1, device="cuda", generator=g) / M
    dpred = torch.randn(M, E, device="cuda", generator=g) / M
    return ac, h, priv, dmean, dvalue, dpred


def _mlp_ref(params, prefix, hr, x_extra, dout, act, r, K0):
    """fp64 forward and hand-written backward of one MLP, rounding (r) where AC_Args.bf16_backward rounds: the history and W1[:, :K0] (the
    forward's and the first-layer wgrad's operands), the head gradient of a head wider than 16 (a narrower one's skinny dgrad is fp32 and
    rounds its output), every hidden dz as stored, the hidden weights as the tensor-core dgrads read them,
    the layer inputs of the BF16 weight gradients, and the first-layer weight gradient's augmented columns.  The bias gradients, d(extra) and
    f' see unrounded values.  Returns (output, {name: grad}, d(extra))."""
    idx = sorted({int(k.split(".")[1]) for k in params if k.startswith(prefix + ".")})
    Ws = [params[f"{prefix}.{i}.weight"] for i in idx]
    bs = [params[f"{prefix}.{i}.bias"] for i in idx]
    f = F64[act]
    n = len(idx)
    z = hr @ r(Ws[0][:, :K0]).t() + bs[0]
    if x_extra is not None:
        z = z + x_extra @ Ws[0][:, K0:].t()
    ys = [f(z)]
    for li in range(1, n):
        v = ys[-1] @ Ws[li].t() + bs[li]
        ys.append(f(v) if li < n - 1 else v)
    g = {}
    o = Ws[-1].shape[0]
    g[f"{prefix}.{idx[-1]}.bias"] = dout.sum(0)
    d = r(dout)
    if o <= 16:
        g[f"{prefix}.{idx[-1]}.weight"] = dout.t() @ ys[-2]
    dextra = None
    for li in range(n - 1, 0, -1):
        if li < n - 1 or o > 16:
            g[f"{prefix}.{idx[li]}.weight"] = d.t() @ r(ys[li - 1])
        if li == n - 1 and o <= 16 and n > 2:       # the skinny head dgrad: fp32 dout and W, only its output is rounded
            dprev = (dout @ Ws[li]) * _deriv(act, ys[li - 1])
        else:
            dprev = (d @ r(Ws[li])) * _deriv(act, ys[li - 1])
        if li > 1:
            g[f"{prefix}.{idx[li - 1]}.bias"] = dprev.sum(0)
        elif x_extra is not None:
            dextra = dprev @ Ws[0][:, K0:]
        d = r(dprev)
    g[f"{prefix}.{idx[0]}.bias"] = d.sum(0)
    gW = d.t() @ hr
    if x_extra is not None:
        gW = torch.cat([gW, d.t() @ r(x_extra)], 1)
    g[f"{prefix}.{idx[0]}.weight"] = gW
    return ys[-1], g, dextra


def _reference(ac, h, priv, dmean, dvalue, dpred, act, rounded):
    r = (lambda t: t.to(torch.bfloat16).double()) if rounded else (lambda t: t.double())
    K0 = h.shape[1]
    params = {k: v.detach().double() for k, v in ac.state_dict().items() if k != "std"}
    hr = r(h)
    # the latent is an input of the actor; its gradient (d(extra) of the actor's first layer) is the adaptation module's head gradient
    lat = _mlp_ref(params, "adaptation_module", hr, None, torch.zeros_like(dpred, dtype=torch.float64), act, r, K0)[0]
    mean, gp, dlat = _mlp_ref(params, "actor_body", hr, lat, dmean.double(), act, r, K0)
    value, gc, _ = _mlp_ref(params, "critic_body", hr, priv.double(), dvalue.double(), act, r, K0)
    _, ga, _ = _mlp_ref(params, "adaptation_module", hr, None, dlat, act, r, K0)
    _, gad, _ = _mlp_ref(params, "adaptation_module", hr, None, dpred.double(), act, r, K0)
    return mean, value, {**ga, **gp, **gc}, gad


def _grads(ac, prefix=""):
    flatg = ac.flat_grads
    out = {}
    for name, p in ac.named_parameters():
        if name != "std" and name.startswith(prefix):
            off = (p.data_ptr() - ac.flat_params.data_ptr()) // 4
            out[name] = flatg[off:off + p.numel()].view(p.shape).double().clone()
    return out


@pytest.mark.parametrize("K0,E,hidden,act", [(k0, e, hd, a) for k0, e, hd, a in itertools.product(
    (2100, 2130), (2, 5, 45), ([512, 256, 128], [130, 70, 33], [256, 128, 64, 32]), ("elu", "tanh"))])
def test_actor_critic_bf16_backward_matches_fp64_reference(K0, E, hidden, act):
    """forward_all + backward_ppo and adaptation_forward + backward_adaptation with AC_Args.bf16_backward (the adaptation module's body is
    hidden[1:]: 256-128, 70-33, 128-64-32).  Against the reference that rounds where the kernels round only TF32 forward products and fp32
    accumulation remain: the bounds of test_actor_critic_impl2_matches_fp64_reference.  Against the unrounded reference every hidden dz,
    the hidden weights the dgrads read and the weight gradients' inputs are BF16 (unit roundoff 2^-9) as well as the history products: a
    gradient passes at most five such roundings on its way down the 4-layer bodies, each of relative size 2^-9 = 2e-3 and not all of one
    sign, so 4 x the rounded bound (0.08 / 0.12 of the largest entry) leaves a factor of about 10 over that worst case."""
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    M = 4096
    ac, h, priv, dmean, dvalue, dpred = _ac_case(K0, E, hidden, act, M)
    AC_Args.gemm_impl, AC_Args.bf16_backward = 2, True
    try:
        mean, value = ac.forward_all(h, priv, tag="train")
        mean, value = mean.clone(), value.clone()
        ac.backward_ppo(h, priv, dmean, dvalue, torch.zeros(12, device="cuda"))
        got = _grads(ac)
        outs = ac.adaptation_forward(h)
        ac.backward_adaptation(h, outs, dpred)
        got_ad = _grads(ac, "adaptation_module")
        torch.cuda.synchronize()
    finally:
        AC_Args.gemm_impl, AC_Args.bf16_backward = 1, False
    rel = lambda a, b: float((a - b).abs().max() / (b.abs().max() + 1e-30))
    errs = {}
    for rounded in (True, False):
        rm, rv, rg, rgad = _reference(ac, h, priv, dmean, dvalue, dpred, act, rounded)
        errs[rounded] = {"mean": rel(mean.double(), rm), "value": rel(value.double(), rv), **{n: rel(got[n], w) for n, w in rg.items()},
                         **{"adapt/" + n: rel(got_ad[n], w) for n, w in rgad.items()}}
    print("max relative error against the BF16-rounded / the unrounded fp64 reference:",
          {n: (round(errs[True][n], 5), round(errs[False][n], 5)) for n in errs[True]})
    for n, e in errs[True].items():
        assert e < (2e-2 if n in ("mean", "value") else 3e-2), (n, errs[True])
    for n, e in errs[False].items():
        assert e < 4 * (2e-2 if n in ("mean", "value") else 3e-2), (n, errs[False])


def test_no_backward_product_behind_the_first_layers_runs_on_tf32(tmp_path, monkeypatch):
    """Launch census of one minibatch's forward_all + backward_ppo in the mode (timing CSV): every product with an MN-major operand -- the
    dgrads and weight gradients -- is a BF16 go1_gemm_bf16_mn launch (bf16 = 2); the heads of at most 16 columns take their dgrad on the
    fp32 skinny kernel (no GEMM launch); the TF32 products left are the forward's (both operands K-major) and the fused tails."""
    from go1_b200 import capi
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    M = 4096
    ac, h, priv, dmean, dvalue, dpred = _ac_case(2100, 5, [512, 256, 128, 64], "elu", M)
    out = tmp_path / "gemm.csv"
    monkeypatch.setenv("GO1_GEMM_TIMING_CSV", str(out))
    monkeypatch.setattr(AC_Args, "gemm_impl", 2)
    monkeypatch.setattr(AC_Args, "bf16_backward", True)
    ac.forward_all(h, priv, tag="train")
    ac.backward_ppo(h, priv, dmean, dvalue, torch.zeros(12, device="cuda"))        # (builds the packed copies outside the timed window)
    L = capi.lib()
    capi.check(L.go1_gemm_timing(1, None, None, None), "timing")
    ac.forward_all(h, priv, tag="train")
    ac.backward_ppo(h, priv, dmean, dvalue, torch.zeros(12, device="cuda"))
    capi.check(L.go1_gemm_timing(0, None, None, None), "timing")
    rows = list(csv.DictReader(open(out)))
    bwd = [r for r in rows if r["a_mn_major"] == "1" or r["b_mn_major"] == "1"]
    assert bwd and all(r["bf16"] == "2" for r in bwd), [r for r in bwd if r["bf16"] != "2"]
    # 3 nets: a dgrad per hidden layer behind the first (3 + 3 + 2), a wgrad per hidden layer behind the first, grouped where shapes match
    assert sum(1 for r in bwd if r["b_mn_major"] == "1" and r["a_mn_major"] == "0") == 8
    assert all(r["bf16"] in ("0", "1") for r in rows if r not in bwd)


def test_full_ppo_cycle_matches_reference_golden_bf16_backward(monkeypatch):
    """test_full_ppo_cycle_matches_reference_golden_impl2 with the flag set, at impl 2's factors (k = 1000, kl = 100: 4 x impl 1's).  The
    golden minibatches have 24 rows, under the 64 at which the mode's products start: this checks that the flag leaves that path, and the
    rollout, exactly as at impl 2."""
    import test_bf16_gpu
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    monkeypatch.setattr(AC_Args, "bf16_backward", True)
    try:
        test_bf16_gpu.test_full_ppo_cycle_matches_reference_golden_impl2()
    finally:
        AC_Args.gemm_impl = 1


def _ppo_cycle(bf16_backward, N=512, T=24):
    """One rollout of random transitions and one PPO update (4 minibatches of N T / 4 rows, 5 epochs) from fixed weights and inputs."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.ppo import PPO
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    NOBS, NH, NP, NA = 70, 2100, 2, 12
    AC_Args.gemm_impl, AC_Args.bf16_backward = 2, bf16_backward
    try:
        torch.manual_seed(0)
        ac = ActorCritic(NOBS, NP, NH, NA)
        alg = PPO(ac, device="cuda:0")
        alg.init_storage(N, T, [NOBS], [NP], [NH], [NA])
        g = torch.Generator(device="cuda").manual_seed(5)
        for t in range(T):
            ac.injected_eps = torch.randn(N, NA, device="cuda", generator=g)
            alg.act(torch.randn(N, NOBS, device="cuda", generator=g), torch.randn(N, NP, device="cuda", generator=g),
                    torch.randn(N, NH, device="cuda", generator=g))
            alg.process_env_step(torch.randn(N, device="cuda", generator=g), torch.zeros(N, dtype=torch.bool, device="cuda"),
                                 {"env_bins": torch.zeros(N, device="cuda"), "time_outs": torch.zeros(N, dtype=torch.bool, device="cuda")})
        alg.compute_returns(torch.randn(N, NH, device="cuda", generator=g), torch.randn(N, NP, device="cuda", generator=g))
        alg.fixed_minibatch_indices = torch.randperm(N * T, device="cuda", generator=g)
        losses = alg.update()
        return losses, {k: v.detach().cpu().numpy() for k, v in ac.state_dict().items()}
    finally:
        AC_Args.gemm_impl, AC_Args.bf16_backward = 1, False


def test_full_ppo_cycle_bf16_backward_follows_impl2():
    """A PPO cycle whose minibatches have 3072 rows, so every backward runs the mode's products, against the same cycle at impl 2 (same
    weights, inputs, noise and minibatch order).  The two differ by the BF16 rounding of the hidden dz, weights and layer inputs in the
    gradients (2^-9 relative, where impl 2 has TF32's 2^-11): the losses, which the first minibatches' forward passes fix, agree to 2e-2
    relative, and the weights after 20 Adam steps (lr 1e-3, |step| <= lr) obey the golden tests' bounds on weights (99 % of the
    differences under 1.6e-2, all under 1.6e-1)."""
    import numpy as np
    l2, w2 = _ppo_cycle(False)
    lb, wb = _ppo_cycle(True)
    for i in (0, 1, 2, 5):
        assert abs(lb[i] - l2[i]) <= 2e-2 * max(abs(l2[i]), 1e-3), (i, lb[i], l2[i])
    for k in w2:
        d = np.abs(wb[k] - w2[k]).ravel()
        assert np.quantile(d, 0.99) < 1.6e-2 and d.max() < 1.6e-1, (k, np.quantile(d, 0.99), d.max())


def test_graph_replayed_rollout_equals_eager_rollout_bf16_backward(tmp_path, monkeypatch):
    import test_runner_gpu
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    monkeypatch.setattr(AC_Args, "gemm_impl", 2)
    monkeypatch.setattr(AC_Args, "bf16_backward", True)
    test_runner_gpu.test_graph_replayed_rollout_equals_eager_rollout(tmp_path, monkeypatch)


def test_runner_learn_bf16_backward_checkpoint_loads_at_impl1(tmp_path, monkeypatch):
    """test_runner_learn_impl2_checkpoint_loads_at_impl1 with the flag: 3 Runner.learn iterations at 4096 envs (minibatches of 24576 rows,
    so every update runs the mode's products) give finite fp32 weights, and the checkpoint and the TorchScript export act like an impl-1
    ActorCritic that loads it."""
    import test_runner_gpu
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(AC_Args, "gemm_impl", 2)
    monkeypatch.setattr(AC_Args, "bf16_backward", True)
    env, Runner, RunnerArgs, logger = test_runner_gpu._make(tmp_path, n=4096)
    RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval = 24, 100, 100, 100
    RunnerArgs.resume = False
    runner = Runner(env, device="cuda:0")
    runner.learn(num_learning_iterations=3, init_at_random_ep_len=True, eval_freq=100)
    ac = runner.alg.actor_critic
    assert torch.isfinite(ac.flat_params).all()
    sd = ac.state_dict()
    assert all(v.dtype == torch.float32 for v in sd.values())
    hist = env.obs_history[:512, :env.num_obs_history].contiguous()
    monkeypatch.setattr(AC_Args, "bf16_backward", False)
    monkeypatch.setattr(AC_Args, "gemm_impl", 1)
    ac1 = ActorCritic(env.num_obs, env.num_privileged_obs, env.num_obs_history, env.num_actions).cuda()
    ac1.load_state_dict(sd)
    want = ac1.act_student(hist).cpu()
    body = torch.jit.load(os.path.join("tmp", "legged_data", "body_latest.jit"))
    adapt = torch.jit.load(os.path.join("tmp", "legged_data", "adaptation_module_latest.jit"))
    h = hist.cpu()
    with torch.no_grad():
        got = body(torch.cat((h, adapt(h)), dim=-1))
    assert torch.allclose(got, want, rtol=1e-2, atol=1e-2 * float(want.abs().max())), float((got - want).abs().max())
