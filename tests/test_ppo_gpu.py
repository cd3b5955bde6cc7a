"""GPU parity tests of the learner kernels (through the C-ABI) against torch fp32 references and against the
vectors produced by the reference's own ppo_cse code (tests/golden/ppo.npz: BASELINE.json config 1)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))


def _gemm(ta, tb, M, N, K, A, lda, B, ldb, C, ldc, bias=None, act=0, acc=0, impl=0):
    from go1_b200 import capi
    capi.check(capi.lib().go1_gemm(ta, tb, M, N, K, capi.ptr(A), lda, capi.ptr(B), ldb, capi.ptr(C), ldc, capi.ptr(bias), act, acc, impl,
                                   capi.stream_ptr()), "gemm")


@pytest.mark.parametrize("ta,tb", [(0, 1), (0, 0), (1, 0), (1, 1)])
@pytest.mark.parametrize("M,N,K", [(4, 12, 128), (96, 2, 2100), (300, 257, 70), (129, 130, 2102), (512, 256, 4096)])
def test_gemm_fp32_matches_torch(ta, tb, M, N, K):
    torch.manual_seed(M + N + K)
    A = torch.randn((K, M) if ta else (M, K), device="cuda")
    B = torch.randn((N, K) if tb else (K, N), device="cuda")
    bias = torch.randn(N, device="cuda")
    ref = (A.t() if ta else A).double() @ (B.t() if tb else B).double()
    C = torch.full((M, N + 3), 7.0, device="cuda")            # ldc > N: the pad columns must stay untouched
    _gemm(ta, tb, M, N, K, A, A.stride(0), B, B.stride(0), C, N + 3)
    assert torch.allclose(C[:, :N].double(), ref, rtol=1e-4, atol=1e-3 * np.sqrt(K) / 30) and (C[:, N:] == 7.0).all()
    C2 = torch.randn(M, N, device="cuda"); C0 = C2.clone()
    _gemm(ta, tb, M, N, K, A, A.stride(0), B, B.stride(0), C2, N, bias=bias, act=1, acc=1)
    want = torch.nn.functional.elu(C0.double() + ref + bias.double())
    assert torch.allclose(C2.double(), want, rtol=1e-4, atol=1e-3 * np.sqrt(K) / 30)


def test_gemm_split_k_wgrad_shape():
    M, N, K = 256, 128, 24576          # dW of a 256->128 layer over a 24576-row minibatch
    A = torch.randn(K, M, device="cuda") * 0.1; B = torch.randn(K, N, device="cuda") * 0.1
    C = torch.zeros(M, N, device="cuda")
    _gemm(1, 0, M, N, K, A, M, B, N, C, N)
    assert torch.allclose(C.double(), A.t().double() @ B.double(), rtol=1e-4, atol=2e-3)


def test_elu_backward_colsum_gather():
    from go1_b200 import capi
    L, st = capi.lib(), capi.stream_ptr()
    y = torch.randn(1000, 37, device="cuda"); y = torch.nn.functional.elu(y); dy = torch.randn_like(y)
    dz = torch.empty_like(y)
    capi.check(L.go1_elu_backward(capi.ptr(y), 37, capi.ptr(dy), 37, capi.ptr(dz), 37, 1000, 37, st), "elu")
    assert torch.allclose(dz, dy * torch.where(y > 0, torch.ones_like(y), y + 1), atol=1e-6)
    out = torch.empty(37, device="cuda")
    capi.check(L.go1_colsum(capi.ptr(dz), 37, capi.ptr(out), 1000, 37, 0, st), "colsum")
    assert torch.allclose(out, dz.sum(0), rtol=1e-4, atol=1e-4)
    src = torch.randn(500, 2100, device="cuda"); idx = torch.randperm(500, device="cuda")[:200]
    dst = torch.empty(200, 2100, device="cuda")
    capi.check(L.go1_gather_rows(capi.ptr(src), capi.ptr(idx), capi.ptr(dst), 200, 2100, 2100, st), "gather")
    assert torch.equal(dst, src[idx])          # copies are bit-exact


@pytest.mark.parametrize("T,n", [(24, 4), (24, 4096), (70, 100), (5, 33)])
def test_gae_matches_reference_loop(T, n):
    """rollout_storage.py:74-88 restated as the literal reversed loop (fp32 torch) vs the warp-scan kernel."""
    from go1_b200 import capi
    torch.manual_seed(T * n)
    rew = torch.randn(T, n, 1, device="cuda"); val = torch.randn(T, n, 1, device="cuda"); last = torch.randn(n, 1, device="cuda")
    done = (torch.rand(T, n, 1, device="cuda") < 0.1).byte()
    ret = torch.zeros_like(rew); adv_k = torch.zeros_like(rew); stats = torch.zeros(2, dtype=torch.float64, device="cuda")
    L, st = capi.lib(), capi.stream_ptr()
    capi.check(L.go1_ppo_gae(capi.ptr(rew), capi.ptr(done), capi.ptr(val), capi.ptr(last), capi.ptr(ret), capi.ptr(adv_k), capi.ptr(stats), T, n, 0.99, 0.95, st), "gae")
    capi.check(L.go1_ppo_normalize_advantages(capi.ptr(adv_k), capi.ptr(stats), T * n, T * n, st), "norm")
    adv, returns = 0, torch.zeros_like(rew)
    for step in reversed(range(T)):
        nv = last if step == T - 1 else val[step + 1]
        nt = 1.0 - done[step].float()
        delta = rew[step] + nt * 0.99 * nv - val[step]
        adv = delta + nt * 0.99 * 0.95 * adv
        returns[step] = adv + val[step]
    a = returns - val
    a = (a - a.mean()) / (a.std() + 1e-8)
    assert torch.allclose(ret, returns, rtol=1e-5, atol=2e-5)
    assert torch.allclose(adv_k, a, rtol=1e-4, atol=2e-5)


def test_ppo_loss_kernel_matches_autograd():
    """Loss values and gradients of ppo.py:113-152 from torch autograd (the reference's own formulae)."""
    from go1_b200 import capi
    torch.manual_seed(0)
    n, A = 5000, 12
    mean = torch.randn(n, A, device="cuda", requires_grad=True); std = (torch.rand(A, device="cuda") + 0.5).requires_grad_()
    value = torch.randn(n, 1, device="cuda", requires_grad=True)
    actions = torch.randn(n, A, device="cuda"); old_mu = mean.detach() + 0.1 * torch.randn(n, A, device="cuda")
    old_sigma = (std.detach() * (1 + 0.05 * torch.randn(A, device="cuda"))).expand(n, A).contiguous()
    old_logp = torch.distributions.Normal(old_mu, old_sigma).log_prob(actions).sum(-1, keepdim=True)
    adv = torch.randn(n, 1, device="cuda"); returns = torch.randn(n, 1, device="cuda"); old_v = value.detach() + 0.3 * torch.randn(n, 1, device="cuda")
    dist = torch.distributions.Normal(mean, mean * 0. + std)
    logp = dist.log_prob(actions).sum(-1)
    ratio = torch.exp(logp - old_logp.squeeze())
    surr = torch.max(-adv.squeeze() * ratio, -adv.squeeze() * torch.clamp(ratio, 0.8, 1.2)).mean()
    vc = old_v + (value - old_v).clamp(-0.2, 0.2)
    vloss = torch.max((value - returns).pow(2), (vc - returns).pow(2)).mean()
    ent = dist.entropy().sum(-1).mean()
    loss = surr + 1.0 * vloss - 0.01 * ent
    loss.backward()
    kl = torch.sum(torch.log(std / old_sigma + 1.e-5) + (old_sigma ** 2 + (old_mu - mean) ** 2) / (2.0 * std ** 2) - 0.5, -1).mean()
    dmean = torch.empty(n, A, device="cuda"); dvalue = torch.empty(n, 1, device="cuda"); dstd = torch.empty(A, device="cuda"); sc = torch.empty(8, device="cuda")
    capi.check(capi.lib().go1_ppo_loss(capi.ptr(mean.detach()), A, capi.ptr(std.detach()), capi.ptr(value.detach()), capi.ptr(actions), capi.ptr(old_logp),
                                       capi.ptr(old_mu), capi.ptr(old_sigma), capi.ptr(adv), capi.ptr(returns), capi.ptr(old_v), capi.ptr(dmean), A,
                                       capi.ptr(dvalue), capi.ptr(dstd), capi.ptr(sc), n, A, 0.2, 1.0, 0.01, 1, 1.0 / n, capi.stream_ptr()), "loss")
    assert torch.allclose(sc[0], surr.detach(), rtol=1e-4, atol=1e-5) and torch.allclose(sc[1], vloss.detach(), rtol=1e-4)
    assert torch.allclose(sc[2], ent.detach(), rtol=1e-5) and torch.allclose(sc[3], kl.detach(), rtol=1e-4, atol=1e-5)
    assert torch.allclose(dmean, mean.grad, rtol=1e-4, atol=1e-7) and torch.allclose(dvalue, value.grad, rtol=1e-4, atol=1e-8)
    assert torch.allclose(dstd, std.grad, rtol=1e-3, atol=1e-5)


def test_clip_adam_matches_torch_optim():
    from go1_b200 import capi
    torch.manual_seed(1)
    p = torch.randn(100003, device="cuda"); ref = torch.nn.Parameter(p.clone()); opt = torch.optim.Adam([ref], lr=1e-3)
    m = torch.zeros_like(p); v = torch.zeros_like(p); gsq = torch.zeros(1, dtype=torch.float64, device="cuda")
    for t in range(1, 4):
        g = torch.randn_like(p) * 0.01 * t
        ref.grad = g.clone()
        torch.nn.utils.clip_grad_norm_([ref], 1.0)
        opt.step()
        capi.check(capi.lib().go1_ppo_grad_sqnorm(capi.ptr(g), g.numel(), capi.ptr(gsq), capi.stream_ptr()), "sq")
        capi.check(capi.lib().go1_ppo_adam_step(capi.ptr(p), capi.ptr(g), capi.ptr(m), capi.ptr(v), p.numel(), capi.ptr(gsq), 1.0, 1e-3, None, 0.9, 0.999, 1e-8, t,
                                                capi.stream_ptr()), "adam")
        assert torch.allclose(p, ref.detach(), rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("impl", [0, 1])
def test_full_ppo_cycle_matches_reference_golden(impl):
    """BASELINE config 1: act x24 -> process_env_step -> compute_returns -> update (5 epochs x 4 minibatches + adaptation
    steps) on the reference's own vectors.  impl 0: fp32 CUDA-core GEMMs (tolerances ~1e-4); impl 1: wgmma TF32 GEMMs
    (10-bit mantissa products: tolerances x250 on the rollout quantities, x25 on the losses, stated as `k` / `kl`)."""
    from ppo_golden_util import seeded_weights, sample_tensor
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.ppo import PPO
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.gemm_impl = impl
    k = 1.0 if impl == 0 else 250.0      # TF32: 2^-11 relative rounding per operand, K = 2100 products, 3-4 layers deep
    g = np.load(os.path.join(HERE, "golden", "ppo.npz"))
    N, T, NOBS, NH, NP, NA = 4, 24, 70, 2100, 2, 12
    ac = ActorCritic(NOBS, NP, NH, NA)
    w = seeded_weights({k: tuple(v.shape) for k, v in ac.state_dict().items()})
    ac.load_state_dict({k: torch.from_numpy(v) for k, v in w.items()})
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
    assert np.array_equal(st.dones.cpu().numpy(), g["storage/dones"])
    alg.fixed_minibatch_indices = C(g["in/perm"])
    losses = alg.update()
    ref = g["update/losses"]
    AC_Args.gemm_impl = 1      # back to the product default
    kl = 1.0 if impl == 0 else 25.0
    assert abs(losses[0] - ref[0]) < 2e-3 * kl * abs(ref[0]) and abs(losses[1] - ref[1]) < 2e-3 * kl and abs(losses[2] - ref[2]) < 2e-3 * kl * abs(ref[2])
    assert abs(losses[5] - ref[5]) < 2e-3 * kl * abs(ref[5])
    assert abs(alg.learning_rate - float(g["update/learning_rate"])) < 1e-12
    sd = ac.state_dict()
    for name_k, v in sd.items():
        got, want = sample_tensor(v.cpu().numpy()), g[f"final/{name_k}"]
        # 20 PPO + 20 adaptation Adam steps; lr <= 1e-3 so each weight moves <= ~0.02: compare the MOVED weights tightly
        if impl == 0:
            assert np.allclose(got[:-2], want[:-2], rtol=0, atol=3e-4), (name_k, np.abs(got[:-2] - want[:-2]).max())
            assert abs(got[-1] - want[-1]) <= 2e-4 * max(1.0, abs(want[-1])), name_k
        else:   # Adam normalises each gradient element, so TF32 noise can move individual weights by a few lr: compare in bulk
            d = np.abs(got[:-2] - want[:-2])
            assert np.quantile(d, 0.99) < 4e-3 and d.max() < 4e-2, (name_k, np.quantile(d, 0.99), d.max())
            assert abs(got[-1] - want[-1]) <= 5e-3 * max(1.0, abs(want[-1])), name_k


# ----------------------------------------------------------------------------------------------------------------
# TF32 tensor-core GEMM (impl=1; wgmma).  TF32 keeps 10 mantissa bits: |err| <= ~2^-10 * sum|a||b| per product, so the
# tolerance is stated relative to the fp64 reference of |A| |B|^T (torch 1.10, the reference's version, also ran its
# matmuls in TF32 by default on Ampere+).
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (128, 64, 64), (4096, 256, 2100), (300, 200, 70), (4, 512, 2100), (1000, 1280, 2100),
                                   (8000, 1280, 1056), (24576, 256, 1024),
                                   (3584, 1280, 1056), (24576, 1280, 1024), (3500, 1100, 2100),   # many tiles per CTA, long K
                                   (24576, 128, 256), (256, 128, 24576), (2100, 1280, 4096)])
def test_gemm_tcgen05_tf32(M, N, K):
    torch.manual_seed(M * 7 + N * 3 + K)
    ldk = (K + 3) // 4 * 4                               # TMA: row strides must be multiples of 16 bytes
    A = torch.randn(M, ldk, device="cuda")[:, :K]
    B = torch.randn(N, ldk, device="cuda")[:, :K]
    bias = torch.randn(N, device="cuda")
    ref = A.double() @ B.double().t()
    bound = (A.abs().double() @ B.abs().double().t()) * 2.0 ** -10 + 1e-6
    C = torch.full((M, N + 5), 3.0, device="cuda")
    _gemm(0, 1, M, N, K, A, ldk, B, ldk, C, N + 5, impl=1)
    torch.cuda.synchronize()
    err = (C[:, :N].double() - ref).abs()
    assert (err <= bound).all(), (float(err.max()), float((err / bound).max()))
    assert (C[:, N:] == 3.0).all()
    # must actually be TF32-accurate, not garbage-within-bound: relative Frobenius error ~1e-4..1e-3
    assert float(err.norm() / ref.norm()) < 2e-3
    C2 = torch.randn(M, N, device="cuda"); C0 = C2.clone()
    _gemm(0, 1, M, N, K, A, ldk, B, ldk, C2, N, bias=bias, act=1, acc=1, impl=1)
    want = torch.nn.functional.elu(C0.double() + ref + bias.double())
    assert ((C2.double() - want).abs() <= bound + 1e-5).all()


# Staged epilogue: 32 x 32 output blocks leave through shared memory + one TMA store per warp, the ELU' operand
# arrives through TMA loads (taken when C / dact_y are 16-byte aligned with row strides that are multiples of 4 floats, no accumulate, no split-K).
# Ragged M and N exercise the TMA clipping; the guard columns behind N and guard rows behind M must stay untouched.
@pytest.mark.parametrize("tb", [1, 0])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (24576, 512, 256), (24576, 256, 128), (1000, 200, 96), (4096 + 37, 128, 256), (300, 72, 40), (5000, 48, 512),
                                   (24576, 128, 12)])
def test_gemm_tcgen05_staged_epilogue(M, N, K, tb):
    import ctypes as C
    from go1_b200 import capi
    torch.manual_seed(M + 3 * N + 5 * K + tb)
    pad4 = lambda n: (n + 3) // 4 * 4
    A = torch.randn(M, pad4(K), device="cuda")[:, :K]
    if tb:
        Bs = torch.randn(N, pad4(K), device="cuda"); B = Bs[:, :K]
    else:
        Bs = torch.randn(K, pad4(N), device="cuda"); B = Bs[:, :N].t()
    ldc = pad4(N) + 8
    ref = A.double() @ B.double().t()
    bound = (A.abs().double() @ B.abs().double().t()) * 2.0 ** -9 + 1e-6
    bias = torch.randn(N, device="cuda")
    L = capi.lib()

    def call(ep, Cbuf):
        capi.check(L.go1_gemm_ex(0, tb, M, N, K, capi.ptr(A), A.stride(0), capi.ptr(Bs), Bs.stride(0), capi.ptr(Cbuf), ldc, C.byref(ep), 1, capi.stream_ptr()), "gemm_ex")
        torch.cuda.synchronize()

    # forward flavour: bias + ELU
    Cb = torch.full((M + 3, ldc), 3.0, device="cuda")
    ep = capi.Go1GemmEpilogue(); ep.bias = bias.data_ptr(); ep.act = 1
    call(ep, Cb)
    want = torch.nn.functional.elu(ref + bias.double())
    assert ((Cb[:M, :N].double() - want).abs() <= bound + 1e-5).all()
    assert (Cb[:M, N:] == 3.0).all() and (Cb[M:] == 3.0).all()
    # dgrad flavour: ELU' operand (row stride a multiple of 4 floats) + column sums
    y = torch.randn(M, pad4(N) + 4, device="cuda")
    cs = torch.zeros(N, device="cuda")
    Cb2 = torch.full((M + 3, ldc), 3.0, device="cuda")
    ep2 = capi.Go1GemmEpilogue(); ep2.act = 2; ep2.dact_y, ep2.ld_dact_y = y.data_ptr(), y.stride(0); ep2.colsum = cs.data_ptr()
    call(ep2, Cb2)
    fac = torch.where(y[:, :N] > 0, torch.ones_like(y[:, :N]), y[:, :N] + 1).double()
    want2 = ref * fac
    assert ((Cb2[:M, :N].double() - want2).abs() <= bound * fac.abs() + 1e-5).all()
    assert (Cb2[:M, N:] == 3.0).all() and (Cb2[M:] == 3.0).all()
    cs_ref = Cb2[:M, :N].double().sum(0)
    assert float((cs.double() - cs_ref).abs().max()) <= 1e-4 * float(Cb2[:M, :N].abs().double().sum(0).max()) + 1e-5
    # repeated launches reuse the staging buffers and barriers: same answer
    Cb3 = torch.full((M + 3, ldc), 3.0, device="cuda")
    ep2.colsum = None
    call(ep2, Cb3)
    assert torch.equal(Cb3[:M, :N], Cb2[:M, :N])


@pytest.mark.parametrize("n", [1, 2, 3, 4])
@pytest.mark.parametrize("M,N,K", [(128, 256, 24576), (256, 512, 8192), (100, 72, 500)])
def test_gemm_grouped_wgrads(M, N, K, n):
    """go1_gemm_grouped: n products of one shape in one grid (the equal-shape split-K wgrads of the three MLPs), accumulating into
    pre-filled outputs; each against its own fp64 reference."""
    import ctypes as C
    from go1_b200 import capi
    torch.manual_seed(M + N + K + n)
    pad = lambda v: (v + 3) // 4 * 4
    As = [torch.randn(K, pad(M), device="cuda") for _ in range(n)]      # dz as [K][M]
    Bs = [torch.randn(K, pad(N), device="cuda") for _ in range(n)]      # activations as [K][N]
    ldc = pad(N) + 4
    Cs = [torch.full((M, ldc), 0.5, device="cuda") for _ in range(n)]
    arr = lambda ts: (C.c_void_p * n)(*[t.data_ptr() for t in ts])
    capi.check(capi.lib().go1_gemm_grouped(1, 0, M, N, K, n, arr(As), pad(M), arr(Bs), pad(N), arr(Cs), ldc, 1, capi.stream_ptr()), "go1_gemm_grouped")
    torch.cuda.synchronize()
    for a, b, c in zip(As, Bs, Cs):
        A, B = a[:, :M].t().double(), b[:, :N].double()
        ref = 0.5 + A @ B
        bound = (A.abs() @ B.abs()) * 2.0 ** -9 + 1e-5
        assert ((c[:, :N].double() - ref).abs() <= bound).all()
        assert (c[:, N:] == 0.5).all()


# MN-major operands (dgrad: B = W as [K][N]; wgrad: A = dz as [K][M], B = activations as [K][N]) read straight from HBM
@pytest.mark.parametrize("ta,tb", [(0, 0), (1, 0), (1, 1)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (128, 32, 64), (300, 200, 72), (24576, 128, 12), (12, 128, 24576), (1280, 2100, 4096),
                                   (512, 256, 24576), (4096, 512, 256), (256, 2100, 24576), (256, 2100, 3000), (384, 1100, 2048)])
def test_gemm_tcgen05_tf32_mn_major(ta, tb, M, N, K):
    torch.manual_seed(M * 7 + N * 3 + K + ta * 2 + tb)
    pad = lambda n: (n + 3) // 4 * 4 + 4
    if ta:
        As = torch.randn(K, pad(M), device="cuda"); A = As[:, :M].t(); lda = As.stride(0)
    else:
        As = torch.randn(M, pad(K), device="cuda"); A = As[:, :K]; lda = As.stride(0)
    if tb:
        Bs = torch.randn(N, pad(K), device="cuda"); B = Bs[:, :K]; ldb = Bs.stride(0)
    else:
        Bs = torch.randn(K, pad(N), device="cuda"); B = Bs[:, :N].t(); ldb = Bs.stride(0)
    ref = A.double() @ B.double().t()
    # worst case per product: both operands truncated to 10 mantissa bits (2^-10 each); with K = 12 and 3M outputs the
    # tail of the distribution reaches ~1.4 * 2^-10 * sum|a||b|, so the hard bound is the two-operand one
    bound = (A.abs().double() @ B.abs().double().t()) * 2.0 ** -9 + 1e-6
    C = torch.full((M, N + 3), 3.0, device="cuda")
    _gemm(ta, tb, M, N, K, As, lda, Bs, ldb, C, N + 3, impl=1)
    torch.cuda.synchronize()
    err = (C[:, :N].double() - ref).abs()
    assert (err <= bound).all(), (float(err.max()), float((err / bound).max()))
    assert (C[:, N:] == 3.0).all()
    assert float(err.norm() / ref.norm()) < 2e-3
    C2 = torch.randn(M, N, device="cuda"); C0 = C2.clone()
    _gemm(ta, tb, M, N, K, As, lda, Bs, ldb, C2, N, acc=1, impl=1)
    assert ((C2.double() - (C0.double() + ref)).abs() <= bound + 1e-5).all()


def test_transpose_kernel():
    from go1_b200 import capi
    src = torch.randn(1000, 300, device="cuda")[:, :257]
    dst = torch.zeros(257, 1004, device="cuda")
    capi.check(capi.lib().go1_transpose(capi.ptr(src), 300, capi.ptr(dst), 1004, 1000, 257, capi.stream_ptr()), "transpose")
    assert torch.equal(dst[:, :1000], src.t()) and (dst[:, 1000:] == 0).all()


def test_gemm_tcgen05_rejects_unsupported_layouts():
    from go1_b200 import capi
    A = torch.randn(64, 70, device="cuda"); C = torch.zeros(64, 64, device="cuda")
    with pytest.raises(capi.Go1Error):
        _gemm(0, 1, 64, 64, 70, A, 70, A, 70, C, 64, impl=1)      # ld=70 floats: not a multiple of 16 bytes


# ----------------------------------------------------------------------------------------------------------------
# pieces of the fused first-layer forward and of the narrow-head backward
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,o,K", [(4, 12, 128), (4096, 1, 128), (24576 + 5, 2, 128), (1000, 16, 256)])
def test_skinny_forward_matches_fp64(M, o, K):
    """go1_skinny_forward (the 12 / 2 / 1-wide heads) against an fp64 matmul; x with a padded row stride, guard column in the output."""
    from go1_b200 import capi
    torch.manual_seed(M + o + K)
    xs = torch.randn(M, K + 8, device="cuda"); x = xs[:, :K]
    W = torch.randn(o, K, device="cuda"); b = torch.randn(o, device="cuda")
    out = torch.full((M, o + 1), 7.0, device="cuda")
    capi.check(capi.lib().go1_skinny_forward(capi.ptr(xs), xs.stride(0), capi.ptr(W), K, capi.ptr(b), capi.ptr(out), o + 1, M, o, K, capi.stream_ptr()), "skinny_forward")
    torch.cuda.synchronize()
    ref = x.double() @ W.double().t() + b.double()
    assert float((out[:, :o].double() - ref).abs().max()) < 1e-4
    assert (out[:, o] == 7.0).all()


@pytest.mark.parametrize("M,o,K", [(24576, 1, 128), (24576, 2, 128), (4097, 12, 128), (300, 16, 257)])
def test_skinny_wgrad_matches_fp64(M, o, K):
    from go1_b200 import capi
    torch.manual_seed(M + o + K)
    dz = torch.randn(M, o + 3, device="cuda")[:, :o]
    x = torch.randn(M, K + 4, device="cuda")[:, :K]
    g = torch.full((o, K + 2), 5.0, device="cuda")
    L = capi.lib()
    capi.check(L.go1_skinny_wgrad(capi.ptr(dz), dz.stride(0), capi.ptr(x), x.stride(0), capi.ptr(g), K + 2, M, o, K, 0, capi.stream_ptr()), "skinny_wgrad")
    ref = dz.double().t() @ x.double()
    tol = 1e-5 * (dz.abs().double().t() @ x.abs().double()) + 1e-6
    assert ((g[:, :K].double() - ref).abs() <= tol).all() and (g[:, K:] == 5.0).all()
    capi.check(L.go1_skinny_wgrad(capi.ptr(dz), dz.stride(0), capi.ptr(x), x.stride(0), capi.ptr(g), K + 2, M, o, K, 1, capi.stream_ptr()), "skinny_wgrad")
    assert ((g[:, :K].double() - 2 * ref).abs() <= 2 * tol).all()


def test_colsum_wide_and_narrow_paths():
    from go1_b200 import capi
    for M, N, ld in ((24576, 512, 1280), (1000, 256, 256), (777, 12, 12), (24576, 130, 132)):
        x = torch.randn(M, ld, device="cuda")
        out = torch.full((N,), 9.0, device="cuda")
        capi.check(capi.lib().go1_colsum(capi.ptr(x), ld, capi.ptr(out), M, N, 0, capi.stream_ptr()), "colsum")
        ref = x[:, :N].double().sum(0)
        assert ((out.double() - ref).abs() <= 1e-5 * x[:, :N].abs().double().sum(0) + 1e-6).all(), (M, N)


def test_fused_first_layer_epilogue_lead_cols_and_extra_forward():
    """One product for [lead | tail] output columns: bias everywhere, extra columns + ELU only on the leading ones; the tail
    is finished by go1_mlp_extra_forward (ActorCritic.forward_all)."""
    from go1_b200 import capi
    torch.manual_seed(5)
    M, K, lead, tail, E = 1000, 2100, 768, 512, 2
    A = torch.randn(M, K, device="cuda"); W = torch.randn(lead + tail, K, device="cuda") * 0.02
    bias = torch.randn(lead + tail, device="cuda"); ex = torch.randn(M, E, device="cuda")
    wx = torch.randn(lead, E, device="cuda"); wt = torch.randn(tail, E + 3, device="cuda"); lat = torch.randn(M, E, device="cuda")
    y = torch.zeros(M, lead + tail, device="cuda")
    ep = capi.Go1GemmEpilogue()
    ep.bias, ep.act, ep.accumulate = bias.data_ptr(), 1, 0
    ep.extra, ep.ld_extra, ep.w_extra, ep.ld_w_extra, ep.num_extra = ex.data_ptr(), E, wx.data_ptr(), E, E
    ep.dact_y, ep.lead_cols = None, lead
    L = capi.lib()
    capi.check(L.go1_gemm_ex(0, 1, M, lead + tail, K, capi.ptr(A), K, capi.ptr(W), K, capi.ptr(y), lead + tail, ep, 1, capi.stream_ptr()), "gemm_ex")
    pre = A.double() @ W.double().t() + bias.double()
    want_lead = torch.nn.functional.elu(pre[:, :lead] + ex.double() @ wx.double().t())
    tol = 2.0 ** -9 * (A.abs().double() @ W.abs().double().t()) + 1e-4
    assert ((y[:, :lead].double() - want_lead).abs() <= tol[:, :lead]).all()
    assert ((y[:, lead:].double() - pre[:, lead:]).abs() <= tol[:, lead:]).all()          # bias only, no activation
    yt = y[:, lead:]
    before = yt.clone()
    capi.check(L.go1_mlp_extra_forward(capi.ptr(yt), yt.stride(0), capi.ptr(lat), E, capi.ptr(wt), E + 3, M, tail, E, 1, capi.stream_ptr()), "extra_fwd")
    want_tail = torch.nn.functional.elu(before.double() + lat.double() @ wt[:, :E].double().t())
    assert ((yt.double() - want_tail).abs() <= 1e-5 * (1 + want_tail.abs())).all()
    with pytest.raises(capi.Go1Error):      # the fp32 CUDA-core path does not implement the split epilogue
        ep.lead_cols = lead
        capi.check(L.go1_gemm_ex(0, 1, M, lead + tail, K, capi.ptr(A), K, capi.ptr(W), K, capi.ptr(y), lead + tail, ep, 0, capi.stream_ptr()), "gemm_ex")


@pytest.mark.parametrize("M", [512, 2304, 1000, 24576 + 300])      # the last one: several row blocks per CTA and a change of problem inside a CTA's sequence
def test_fused_backward_epilogues_match_separate_kernels(M):
    """The bias gradients (column sums of dz) reduced inside the dgrad epilogues (GEMM atomics, or the skinny dgrad behind a narrow
    head) must equal the separate column-sum kernel over the dz buffer they were reduced from, up to the fp32 rounding of a different
    summation order; the whole flat gradient buffer is checked against an fp64 torch-autograd gradient of the same loss as well."""
    from go1_b200 import capi
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.gemm_impl = 1
    torch.manual_seed(3)
    NOBS, NH, NP, NA = 70, 2100, 2, 12
    ac = ActorCritic(NOBS, NP, NH, NA).to("cuda:0")
    ac.flatten()
    h = torch.randn(M, NH, device="cuda") * 0.3
    priv = torch.randn(M, NP, device="cuda")
    dmean = torch.randn(M, NA, device="cuda") / M
    dvalue = torch.randn(M, 1, device="cuda") / M
    dstd = torch.randn(NA, device="cuda")
    ac.flat_grads.zero_()
    ac.forward_all(h, priv, tag="train")
    ac.backward_ppo(h, priv, dmean, dvalue, dstd)
    torch.cuda.synchronize()
    a = ac.flat_grads.clone()
    scale = a.abs().max()
    L = capi.lib()
    for name in ("adapt", "actor", "critic"):
        net = ac._nets[name]
        for k in range(1, len(net.specs) - 1):          # the hidden layers behind the first one: their dz stays in a buffer of _Net
            dz = net.acts[("train", "d", k)][:M]
            _, bo, o, _ = net.specs[k]
            want = torch.empty(o, device="cuda")
            capi.check(L.go1_colsum(capi.ptr(dz), dz.stride(0), capi.ptr(want), M, o, 0, capi.stream_ptr()), "colsum")
            err = float((a[bo:bo + o] - want).abs().max())
            assert err <= 2e-5 * float(scale) + 1e-7, (name, k, err)
    # h as a view of a row buffer with a 2112-float pitch, the minibatch layout of RolloutStorage: same products, another order of the atomic sums
    hb = torch.zeros(M, NH + 12, device="cuda")
    hb[:, :NH] = h
    h2 = hb[:, :NH]
    ac.flat_grads.zero_()
    ac.forward_all(h2, priv, tag="train")
    ac.backward_ppo(h2, priv, dmean, dvalue, dstd)
    torch.cuda.synchronize()
    b = ac.flat_grads.clone()
    assert float((a - b).abs().max()) <= 3e-3 * float(scale) + 1e-7, float((a - b).abs().max())
    # fp64 autograd of sum(mean * dmean) + sum(value * dvalue) through plain torch modules holding the same weights
    import copy
    ref = {k: copy.deepcopy(getattr(ac, k)).double() for k in ("adaptation_module", "actor_body", "critic_body")}
    hd, pd = h.double(), priv.double()
    lat = ref["adaptation_module"](hd)
    loss = (ref["actor_body"](torch.cat((hd, lat), -1)) * dmean.double()).sum() + (ref["critic_body"](torch.cat((hd, pd), -1)) * dvalue.double()).sum()
    loss.backward()
    for name, mod in ref.items():
        for (pn, p_ref), p in zip(mod.named_parameters(), getattr(ac, name).parameters()):
            off = p.data_ptr() - ac.flat_params.data_ptr()
            g = b[off // 4: off // 4 + p.numel()].view_as(p)
            err = (g.double() - p_ref.grad).abs().max() / (p_ref.grad.abs().max() + 1e-12)
            assert float(err) < 5e-3, (name, pn, float(err))        # TF32 products: 2^-11 per operand


@pytest.mark.parametrize("M", [4, 100, 4096, 24576 + 37])
def test_fused_mlp_tail_forward_matches_layer_by_layer(M):
    """go1_mlp_tail_forward (layers behind the first one in ONE tensor-core launch, activations kept on the SM) against the
    layer-by-layer tensor-core path and an fp64 torch evaluation of the same modules: all three MLPs, every saved activation."""
    from go1_gym_learn.ppo_cse import ActorCritic
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    AC_Args.gemm_impl = 1
    torch.manual_seed(11)
    NOBS, NH, NP, NA = 70, 2100, 2, 12
    ac = ActorCritic(NOBS, NP, NH, NA).to("cuda:0")
    ac.flatten()
    with torch.no_grad():
        for p in ac.parameters():
            p.mul_(1.7)          # push some pre-activations well away from zero: both ELU branches in play
    h = torch.randn(M, NH, device="cuda") * 0.5
    priv = torch.randn(M, NP, device="cuda")
    res = {}
    for fuse in (False, True):
        ac.fuse_tail = fuse
        ac.forward_all(h, priv, tag="tailtest%d" % fuse)
        torch.cuda.synchronize()
        res[fuse] = [[t.clone() for t in outs] for outs in (ac._a_out, ac._p_out, ac._c_out)]
    import copy
    hd = h.double()
    mods = [copy.deepcopy(m).double() for m in (ac.adaptation_module, ac.actor_body, ac.critic_body)]
    lat = mods[0](hd)
    ins = [hd, torch.cat((hd, lat), -1), torch.cat((hd, priv.double()), -1)]
    for net in range(3):
        x, ref = ins[net], []
        for layer in mods[net]:
            x = layer(x)
            if isinstance(layer, torch.nn.ELU) or layer is mods[net][-1]:
                ref.append(x)
        assert len(ref) == len(res[True][net]) == len(res[False][net])
        for li, (a, b, r) in enumerate(zip(res[False][net], res[True][net], ref)):
            scale = float(r.abs().max()) + 1e-6
            assert torch.isfinite(b).all()
            assert float((b.double() - r).abs().max()) < 6e-3 * scale, (net, li, "fused vs fp64", float((b.double() - r).abs().max()), scale)
            assert float((a - b).abs().max()) < 4e-3 * scale, (net, li, "fused vs layered", float((a - b).abs().max()), scale)
