"""AC_Args.activation on the kernels: every Go1Activation through the C ABI (both GEMM impls, the bandwidth kernels, the fused tails),
through ActorCritic (gradients against fp64 autograd, a full PPO cycle against the reference's vectors) and through Runner.learn.
ELU is parametrised like the other kinds, as the control."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))
from activation_test_util import DERIV_FROM_OUTPUT, KINDS, MODULES, NAMES  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _restore_ac_args():
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    keep = {k: copy.copy(getattr(AC_Args, k)) for k in ("activation", "gemm_impl", "actor_hidden_dims", "critic_hidden_dims", "adaptation_module_branch_hidden_dims")}
    yield
    for k, v in keep.items():
        setattr(AC_Args, k, v)


def _kind(name):
    from go1_b200 import capi
    return capi.ACTIVATIONS[name]


def _f64(name, v):
    return MODULES[name]()(v.double())


def _gemm_ex(ta, tb, M, N, K, A, B, C, impl, kind, act, bias=None, dact_y=None, lead_cols=0):
    from go1_b200 import capi
    ep = capi.Go1GemmEpilogue()
    ep.act, ep.act_kind, ep.lead_cols = act, kind, lead_cols
    ep.bias = bias.data_ptr() if bias is not None else None
    if dact_y is not None:
        ep.dact_y, ep.ld_dact_y = dact_y.data_ptr(), dact_y.stride(0)
    return capi.lib().go1_gemm_ex(ta, tb, M, N, K, capi.ptr(A), A.stride(0), capi.ptr(B), B.stride(0), capi.ptr(C), C.stride(0), ep, impl, capi.stream_ptr())


def _tol_fast(ref):
    """act_fast's bound: 1e-6 absolute, plus the fp32 rounding of the result itself where it exceeds 1 (selu at large v)."""
    return 1e-6 + 2.0 ** -23 * ref.abs()


@pytest.mark.parametrize("name", KINDS)
def test_fast_activation_dense_sweep(name):
    """2^20 evenly spaced v in [-30, 30] (and the ends) through go1_mlp_extra_forward's float4 kernel, which applies act_fast with a zero
    trailing-input term: the error bound stated in csrc/activation.cuh, measured against fp64."""
    from go1_b200 import capi
    M, o, E = 4096, 256, 2
    v = torch.linspace(-30, 30, M * o, device="cuda", dtype=torch.float64).float().view(M, o).contiguous()
    y = v.clone()
    ex, w = torch.zeros(M, E, device="cuda"), torch.zeros(o, E, device="cuda")
    capi.check(capi.lib().go1_mlp_extra_forward(capi.ptr(y), o, capi.ptr(ex), E, capi.ptr(w), E, M, o, E, capi.act_arg(_kind(name), 1), capi.stream_ptr()), "extra_fwd")
    ref = _f64(name, v)
    err = (y.double() - ref).abs()
    assert bool((err <= _tol_fast(ref)).all()), float(err.max())
    near0 = v.abs() < 0.2      # the polynomial branches keep relative accuracy near 0 (tanh, elu, selu)
    if name in ("tanh", "elu", "selu"):
        rel = (err / ref.abs().clamp_min(1e-30))[near0 & (v != 0)]
        assert float(rel.max()) < 1e-6, float(rel.max())
    # the generic kernel (o % 4 != 0) uses the libm forms
    o2 = 37
    v2 = torch.linspace(-30, 30, 1000 * o2, device="cuda", dtype=torch.float64).float().view(1000, o2).contiguous()
    y2 = v2.clone()
    w2 = torch.zeros(o2, E, device="cuda")
    capi.check(capi.lib().go1_mlp_extra_forward(capi.ptr(y2), o2, capi.ptr(ex), E, capi.ptr(w2), E, 1000, o2, E, capi.act_arg(_kind(name), 1), capi.stream_ptr()), "extra_fwd")
    want = MODULES[name]()(v2)
    assert torch.allclose(y2, want, rtol=1e-6, atol=1e-7), float((y2 - want).abs().max())


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("name", KINDS)
def test_gemm_epilogue_sees_known_preactivations(name, impl):
    """A product with an identity operand: the epilogue's v is exactly the (TF32-representable) input, so act 1 / act 2 are checked on
    their own.  impl 0: 1e-6 relative against torch fp32; impl 1: act_fast's bound against fp64."""
    M, N = 300, 64
    torch.manual_seed(5)
    v = (torch.randint(-1920, 1921, (M, N), device="cuda").float() / 64.0).contiguous()      # multiples of 1/64 in [-30, 30]: 11 significant bits
    v[0, :8] = torch.tensor([0.0, -0.0, 1 / 64, -1 / 64, 30.0, -30.0, 0.25, -0.25], device="cuda")
    eye = torch.eye(N, device="cuda")
    out = torch.empty(M, N, device="cuda")
    assert _gemm_ex(0, 1, M, N, N, v, eye, out, impl, _kind(name), 1) == 0
    ref = _f64(name, v)
    if impl == 0:
        want = MODULES[name]()(v)
        assert torch.allclose(out, want, rtol=1e-6, atol=1e-7), float((out - want).abs().max())
    else:
        assert bool(((out.double() - ref).abs() <= _tol_fast(ref)).all()), float((out.double() - ref).abs().max())
    # act 2: dz = g * f'(y) from the saved output y
    y = MODULES[name]()(v / 8.0).contiguous()
    y[0, :4] = 0.0
    gq = (torch.randint(-512, 513, (M, N), device="cuda").float() / 256.0).contiguous()
    dz = torch.empty(M, N, device="cuda")
    assert _gemm_ex(0, 1, M, N, N, gq, eye, dz, impl, _kind(name), 2, dact_y=y) == 0
    want = (gq.double() * DERIV_FROM_OUTPUT[name](y.double()))
    assert torch.allclose(dz.double(), want, rtol=1e-6, atol=1e-7), float((dz.double() - want).abs().max())


@pytest.mark.parametrize("staged", [True, False])
@pytest.mark.parametrize("name", KINDS)
def test_gemm_tf32_epilogues_ragged_lead_cols(name, staged):
    """go1_gemm_ex impl 1 on ragged M / N with bias, the lead_cols split and act 1 / 2, through the staged (TMA store) and the direct
    epilogue (an output row stride that is not a multiple of 4 floats), against fp64 at TF32 accuracy."""
    M, N, K, lead = 300, 200, 72, 130
    torch.manual_seed(6)
    A, W, b = torch.randn(M, K, device="cuda"), torch.randn(N, K, device="cuda") / 4, torch.randn(N, device="cuda")
    ldc = N if staged else N + 1
    buf = torch.full((M, ldc), 7.0, device="cuda")
    out = buf[:, :N]
    assert _gemm_ex(0, 1, M, N, K, A, W, out, 1, _kind(name), 1, bias=b, lead_cols=lead) == 0
    z = A.double() @ W.double().t() + b.double()
    ref = torch.cat((_f64(name, z[:, :lead]), z[:, lead:]), 1)
    bound = 1.1 * 2.0 ** -9 * (A.abs().double() @ W.abs().double().t()) + 1e-5      # (selu stretches by lambda = 1.05)
    assert bool(((out.double() - ref).abs() <= bound).all()), float((out.double() - ref).abs().max())
    if not staged:
        assert bool((buf[:, N] == 7.0).all())
    # dgrad form: B = W as [K][N] (MN-major), times f'(saved output)
    y = MODULES[name]()(torch.randn(M, K, device="cuda") * 2)
    dzn = torch.randn(M, N, device="cuda")
    ldp = K if staged else K + 1
    pbuf = torch.zeros(M, ldp, device="cuda")
    dprev = pbuf[:, :K]
    assert _gemm_ex(0, 0, M, K, N, dzn, W, dprev, 1, _kind(name), 2, dact_y=y) == 0
    ref = (dzn.double() @ W.double()) * DERIV_FROM_OUTPUT[name](y.double())
    bound = 2.0 ** -9 * (dzn.abs().double() @ W.abs().double()) * DERIV_FROM_OUTPUT[name](y.double()).abs() + 1e-5
    assert bool(((dprev.double() - ref).abs() <= bound).all()), float((dprev.double() - ref).abs().max())


@pytest.mark.parametrize("name", KINDS)
def test_bandwidth_kernels(name):
    """go1_act_backward, go1_skinny_dgrad_act (float4 and scalar variants, with the fused column sums) and go1_mlp_extra_forward with a
    real trailing-input term, against torch."""
    from go1_b200 import capi
    L, st, kind = capi.lib(), capi.stream_ptr(), _kind(name)
    torch.manual_seed(7)
    y = MODULES[name]()(torch.randn(1000, 37, device="cuda") * 3)
    y[0, :5] = 0.0
    dy = torch.randn(1000, 37, device="cuda")
    dz = torch.empty_like(dy)
    capi.check(L.go1_act_backward(capi.ptr(y), 37, capi.ptr(dy), 37, capi.ptr(dz), 37, 1000, 37, kind, st), "act_backward")
    want = dy * DERIV_FROM_OUTPUT[name](y)
    assert torch.allclose(dz, want, rtol=1e-6, atol=1e-7)
    if name == "elu":
        dz2 = torch.empty_like(dy)
        capi.check(L.go1_elu_backward(capi.ptr(y), 37, capi.ptr(dy), 37, capi.ptr(dz2), 37, 1000, 37, st), "elu_backward")
        assert torch.equal(dz, dz2)
    for M, o, n in ((4097, 12, 128), (1000, 2, 256), (300, 3, 37)):
        d, W = torch.randn(M, o, device="cuda"), torch.randn(o, n, device="cuda")
        yp = MODULES[name]()(torch.randn(M, n, device="cuda") * 2)
        dprev = torch.empty(M, n, device="cuda")
        vec = n % 4 == 0
        cs = torch.zeros(n, device="cuda") if vec else None
        capi.check(L.go1_skinny_dgrad_act(capi.ptr(d), o, capi.ptr(W), n, capi.ptr(yp), n, capi.ptr(dprev), n, capi.ptr(cs), M, o, n, kind, st), "skinny_dgrad_act")
        ref = (d.double() @ W.double()) * DERIV_FROM_OUTPUT[name](yp.double())
        assert torch.allclose(dprev.double(), ref, rtol=1e-5, atol=1e-5), (M, o, n)
        if vec:
            assert torch.allclose(cs.double(), ref.sum(0), rtol=1e-4, atol=1e-3 * float(ref.abs().sum(0).max()) / M ** 0.5 + 1e-4), (M, o, n)
    M, o, E = 500, 512, 2
    yv, ex, w = torch.randn(M, o, device="cuda") * 2, torch.randn(M, E, device="cuda"), torch.randn(o, E + 3, device="cuda")
    ref = _f64(name, yv.double() + ex.double() @ w[:, :E].double().t())
    capi.check(L.go1_mlp_extra_forward(capi.ptr(yv), o, capi.ptr(ex), E, capi.ptr(w), E + 3, M, o, E, capi.act_arg(kind, 1), st), "extra_fwd")
    assert bool(((yv.double() - ref).abs() <= 4e-6 + 2e-6 * ref.abs()).all()), float((yv.double() - ref).abs().max())


def test_unknown_kind_is_rejected_before_launch():
    """Bad-argument cases stop on the host side of the ABI: non-zero return code and a go1_last_error() message."""
    from go1_b200 import capi
    L, st = capi.lib(), capi.stream_ptr()
    x = torch.zeros(128, 128, device="cuda")
    msg = lambda: L.go1_last_error().decode()
    for impl in (0, 1):
        assert _gemm_ex(0, 1, 128, 128, 128, x, x, x.clone(), impl, 6, 1) != 0 and "activation kind" in msg()
        assert _gemm_ex(0, 1, 128, 128, 128, x, x, x.clone(), impl, -1, 1) != 0 and "activation kind" in msg()
    assert L.go1_act_backward(capi.ptr(x), 128, capi.ptr(x), 128, capi.ptr(x), 128, 128, 128, 9, st) != 0 and "activation kind" in msg()
    assert L.go1_skinny_dgrad_act(capi.ptr(x), 128, capi.ptr(x), 128, capi.ptr(x), 128, capi.ptr(x), 128, None, 128, 4, 128, 6, st) != 0 and "activation kind" in msg()
    assert L.go1_mlp_extra_forward(capi.ptr(x), 128, capi.ptr(x), 2, capi.ptr(x), 2, 128, 128, 2, capi.act_arg(7, 1), st) != 0 and "activation kind" in msg()
    assert L.go1_gemm(0, 1, 128, 128, 128, capi.ptr(x), 128, capi.ptr(x), 128, capi.ptr(x.clone()), 128, None, capi.act_arg(6, 1), 0, 0, st) != 0
    q = (capi.Go1TailProblem * 1)()
    q[0].act_kind = 6
    assert L.go1_mlp_tail_forward_grouped(q, 1, 128, 512, 256, 128, st) != 0 and "activation kind" in msg()
    torch.cuda.synchronize()
    assert bool((x == 0).all())


def _ref_modules(ac):
    return {k: copy.deepcopy(getattr(ac, k)).double() for k in ("adaptation_module", "actor_body", "critic_body")}


@pytest.mark.parametrize("M", [100, 4096])
@pytest.mark.parametrize("name", KINDS)
def test_fused_tails_forward_match_layer_by_layer(name, M):
    """The fused forward tails (512-256-128-head grouped for actor + critic, 256-128-head for the adaptation module) against the
    layer-by-layer tensor-core path and fp64; M = 100 leaves guard rows in the last 64-row block, which must not leak into the rows
    that exist (sigmoid(0) = 0.5 would, if the guard relied on f(0) = 0)."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.gemm_impl, AC_Args.activation = 1, name
    torch.manual_seed(11)
    NOBS, NH, NP, NA = 70, 2100, 2, 12
    ac = ActorCritic(NOBS, NP, NH, NA).to("cuda:0")
    ac.flatten()
    with torch.no_grad():
        for p in ac.parameters():
            p.mul_(1.7)
    h, priv = torch.randn(M, NH, device="cuda") * 0.5, torch.randn(M, NP, device="cuda")
    res = {}
    for fuse in (False, True):
        ac.fuse_tail = fuse
        ac.forward_all(h, priv, tag="tailtest%d" % fuse)
        torch.cuda.synchronize()
        res[fuse] = [[t.clone() for t in outs] for outs in (ac._a_out, ac._p_out, ac._c_out)]
    hd = h.double()
    mods = list(_ref_modules(ac).values())
    lat = mods[0](hd)
    ins = [hd, torch.cat((hd, lat), -1), torch.cat((hd, priv.double()), -1)]
    for net in range(3):
        x, ref = ins[net], []
        for layer in mods[net]:
            x = layer(x)
            if not isinstance(layer, torch.nn.Linear) or layer is mods[net][-1]:
                ref.append(x)
        assert len(ref) == len(res[True][net]) == len(res[False][net])
        for li, (a, b, r) in enumerate(zip(res[False][net], res[True][net], ref)):
            r = r.detach()
            scale = float(r.abs().max()) + 1e-6
            assert torch.isfinite(b).all()
            assert float((b.double() - r).abs().max()) < 6e-3 * scale, (net, li, "fused vs fp64", float((b.double() - r).abs().max()), scale)
            assert float((a - b).abs().max()) < 4e-3 * scale, (net, li, "fused vs layered", float((a - b).abs().max()), scale)


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("name", KINDS)
def test_actor_critic_gradients_match_autograd(name, impl):
    """forward_all + backward_ppo + backward_adaptation at the train.py layer shapes (M = 4096 rows) against fp64 autograd through plain
    torch modules holding the same weights.  impl 0 at fp32 accuracy; impl 1 at its TF32 factor."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.gemm_impl, AC_Args.activation = impl, name
    torch.manual_seed(3)
    M, NOBS, NH, NP, NA = 4096, 70, 2100, 2, 12
    ac = ActorCritic(NOBS, NP, NH, NA).to("cuda:0")
    ac.flatten()
    h, priv = torch.randn(M, NH, device="cuda") * 0.3, torch.randn(M, NP, device="cuda")
    dmean, dvalue, dstd = torch.randn(M, NA, device="cuda") / M, torch.randn(M, 1, device="cuda") / M, torch.randn(NA, device="cuda")
    # Largest element error over the tensor's largest gradient.  impl 0: fp32 summation order (the two-element bias gradient of the latent
    # layer is a sum of 4096 rows that nearly cancels: observed up to 2e-3 for selu).  impl 1: 2^-11 per TF32 operand, and the
    # adaptation module's gradient comes through seven layers (actor body, latent, adaptation module); sigmoid's all-positive layer
    # outputs add a common-mode term that does not average out.  relu / lrelu: rounding flips the sign of the few pre-activations that lie
    # within it of 0 (fp32: a handful of the 5 M; TF32: ~1e-3 of them), and each flip switches a 0 / 1 derivative for a whole row.
    kinked = name in ("relu", "lrelu")
    tol = (2e-2 if kinked else 5e-3) if impl == 0 else (1e-1 if kinked else 5e-2)

    ac.flat_grads.zero_()
    mean, value = ac.forward_all(h, priv, tag="train")
    ac.backward_ppo(h, priv, dmean, dvalue, dstd)
    torch.cuda.synchronize()
    grads = ac.flat_grads.clone()
    ref = _ref_modules(ac)
    hd, pd = h.double(), priv.double()
    lat = ref["adaptation_module"](hd)
    mean_ref, value_ref = ref["actor_body"](torch.cat((hd, lat), -1)), ref["critic_body"](torch.cat((hd, pd), -1))
    assert float((mean.double() - mean_ref.detach()).abs().max()) < tol * (float(mean_ref.detach().abs().max()) + 1) * 2
    assert float((value.double() - value_ref.detach()).abs().max()) < tol * (float(value_ref.detach().abs().max()) + 1) * 2
    ((mean_ref * dmean.double()).sum() + (value_ref * dvalue.double()).sum()).backward()

    def check(g, what):
        for nm, mod in ref.items():
            for (pn, p_ref), p in zip(mod.named_parameters(), getattr(ac, nm).parameters()):
                off = (p.data_ptr() - ac.flat_params.data_ptr()) // 4
                got = g[off: off + p.numel()].view_as(p)
                err = (got.double() - p_ref.grad).abs().max() / (p_ref.grad.abs().max() + 1e-12)
                assert float(err) < tol, (what, nm, pn, float(err))

    check(grads, "backward_ppo")
    assert torch.equal(grads[ac.std_offset:ac.std_offset + NA], dstd)
    # adaptation step: MSE-like gradient dpred through the adaptation module alone
    for mod in ref.values():
        mod.zero_grad()
    outs = ac.adaptation_forward(h)
    dpred = torch.randn(M, NP, device="cuda") / M
    ac.flat_grads.zero_()
    ac.backward_adaptation(h, outs, dpred)
    torch.cuda.synchronize()
    (ref["adaptation_module"](hd) * dpred.double()).sum().backward()
    for (pn, p_ref), p in zip(ref["adaptation_module"].named_parameters(), ac.adaptation_module.parameters()):
        off = (p.data_ptr() - ac.flat_params.data_ptr()) // 4
        got = ac.flat_grads[off: off + p.numel()].view_as(p)
        err = (got.double() - p_ref.grad).abs().max() / (p_ref.grad.abs().max() + 1e-12)
        assert float(err) < tol, ("backward_adaptation", pn, float(err))


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("name", NAMES)
def test_full_ppo_cycle_matches_reference_vectors(name, impl):
    """act x24 -> process_env_step -> compute_returns -> update on the reference's own vectors for every activation name, on a small
    network (history 350, hidden [64, 32] / [32]): the layer-by-layer kernels with non-default hidden dims.  Tolerances as in
    test_ppo_gpu.test_full_ppo_cycle_matches_reference_golden (impl 1: TF32 factors k / kl)."""
    from ppo_golden_util import seeded_weights, sample_tensor
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.ppo import PPO
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    g = np.load(os.path.join(HERE, "golden", "ppo_activations.npz"))
    N, T, NOBS, NH, NP, NA, h1, h2, ha = (int(x) for x in g["meta/dims"])
    AC_Args.gemm_impl, AC_Args.activation = impl, name
    AC_Args.actor_hidden_dims, AC_Args.critic_hidden_dims, AC_Args.adaptation_module_branch_hidden_dims = [h1, h2], [h1, h2], [ha]
    k = 1.0 if impl == 0 else 250.0
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
    for nm, tol in (("actions", 2e-5), ("values", 2e-5), ("actions_log_prob", 1e-4), ("mu", 2e-5), ("returns", 5e-5), ("advantages", 2e-4)):
        got, want = getattr(st, nm).cpu().numpy(), g[f"{name}/storage/{nm}"]
        assert np.allclose(got, want, rtol=1e-4 * k, atol=tol * k), (nm, np.abs(got - want).max())
    alg.fixed_minibatch_indices = C(g["in/perm"])
    losses = alg.update()
    ref = g[f"{name}/update/losses"]
    kl = 1.0 if impl == 0 else 25.0
    assert abs(losses[0] - ref[0]) < 2e-3 * kl * abs(ref[0]) and abs(losses[1] - ref[1]) < 2e-3 * kl and abs(losses[2] - ref[2]) < 2e-3 * kl * abs(ref[2])
    assert abs(losses[5] - ref[5]) < 2e-3 * kl * abs(ref[5])
    if impl == 0:
        assert abs(alg.learning_rate - float(g[f"{name}/update/learning_rate"])) < 1e-12
    for name_k, v in ac.state_dict().items():
        got, want = sample_tensor(v.cpu().numpy(), stride=3), g[f"{name}/final/{name_k}"]
        if impl == 0:
            assert np.allclose(got[:-2], want[:-2], rtol=0, atol=3e-4), (name_k, np.abs(got[:-2] - want[:-2]).max())
        else:
            d = np.abs(got[:-2] - want[:-2])
            assert np.quantile(d, 0.99) < 4e-3 and d.max() < 4e-2, (name_k, np.quantile(d, 0.99), d.max())


def test_two_actor_critics_with_different_activations_coexist():
    """The kind is per instance (no process-global state): interleaved forward passes of a tanh and an ELU network stay their own."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.gemm_impl = 1
    nets = {}
    for name in ("tanh", "elu"):
        AC_Args.activation = name
        torch.manual_seed(1)
        nets[name] = ActorCritic(70, 2, 2100, 12).to("cuda:0")
    AC_Args.activation = "sigmoid"      # later changes of the global name do not reach existing instances
    h, priv = torch.randn(256, 2100, device="cuda") * 0.3, torch.randn(256, 2, device="cuda")
    for name, ac in nets.items():
        mean, value = ac.forward_all(h, priv)
        mods = _ref_modules(ac)
        hd = h.double()
        want = mods["actor_body"](torch.cat((hd, mods["adaptation_module"](hd)), -1))
        assert type(ac.actor_body[1]) is MODULES[name]
        want = want.detach()
    assert float((mean.double() - want).abs().max()) < 5e-3 * (float(want.abs().max()) + 1), name


def test_runner_learn_with_tanh_and_play_artifacts(tmp_path, monkeypatch):
    """AC_Args.activation = 'tanh' through the scripts/train.py flow: a short Runner.learn (graph-replayed rollout) trains, saves, and the
    TorchScript artefacts scripts/play.py loads carry nn.Tanh and reproduce the inference policy."""
    monkeypatch.chdir(tmp_path)
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.activation = "tanh"
    for m in [k for k in sys.modules if k.startswith("go1_gym.envs.base.legged_robot_config")]:
        del sys.modules[m]
    from go1_gym.envs.base.legged_robot_config import Cfg
    from go1_b200.train_config import apply_train_config
    from go1_gym.envs.go1.velocity_tracking import VelocityTrackingEasyEnv
    from go1_gym.envs.wrappers.history_wrapper import HistoryWrapper
    from go1_gym_learn.ppo_cse import Runner, RunnerArgs
    from ml_logger import logger
    apply_train_config(Cfg)
    Cfg.env.num_envs = 256
    logger.configure(prefix="run", root=str(tmp_path))
    env = HistoryWrapper(VelocityTrackingEasyEnv(sim_device="cuda:0", headless=True, cfg=Cfg))
    keep = (RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume)
    RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume = 8, 1, 1, 100, False
    try:
        runner = Runner(env, device="cuda:0")
        ac = runner.alg.actor_critic
        w0 = ac.flat_params.clone()
        runner.learn(num_learning_iterations=2, init_at_random_ep_len=True, eval_freq=100)
    finally:
        RunnerArgs.num_steps_per_env, RunnerArgs.save_interval, RunnerArgs.log_freq, RunnerArgs.save_video_interval, RunnerArgs.resume = keep
    assert torch.isfinite(ac.flat_params).all() and not torch.equal(ac.flat_params, w0)
    ck = os.path.join(str(tmp_path), "run", "checkpoints")
    body = torch.jit.load(os.path.join(ck, "body_latest.jit"))
    adapt = torch.jit.load(os.path.join(ck, "adaptation_module_latest.jit"))
    assert "Tanh" in str(body) and "ELU" not in str(body) and "Tanh" in str(adapt)
    h = torch.randn(5, env.num_obs_history) * 0.3
    policy = runner.get_inference_policy(device="cuda:0")
    AC_Args.gemm_impl = 0      # the exact-fp32 kernels against TorchScript's fp32 on the CPU
    want = policy({"obs_history": h.cuda()}).cpu()
    got = body(torch.cat((h, adapt(h)), dim=-1))
    assert torch.allclose(got, want, rtol=1e-4, atol=2e-5), float((got - want).abs().max())
