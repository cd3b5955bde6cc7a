"""AC_Args.deterministic / go1_set_deterministic: every learner entry point whose CTAs share a reduction target gives bit-identical outputs
for identical inputs (also while an unrelated product runs on another stream), within the fp64-reference bounds of the default mode; and
whole training iterations (rollout, returns, update) repeat bit for bit."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200"))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))

TF32 = 2.0 ** -9        # two operands rounded to TF32 (2^-11 relative each) and the fp32 sums of a split product, per |a||b| term


def _bits(t):
    return t.contiguous().view({torch.float32: torch.int32, torch.float64: torch.int64, torch.bfloat16: torch.int16}[t.dtype])


def _twice(run):
    """run() launches one entry point into fresh outputs and returns them; called twice in deterministic mode, the second time beside a
    large product on another stream (so the CTAs finish in another order), and the outputs must be bit-identical."""
    from go1_b200 import capi
    x = torch.randn(8192, 8192, device="cuda")
    with capi.deterministic(True):
        a = run()
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(4):
                x = x @ x.t() * 1e-4
        b = run()
        torch.cuda.synchronize()
    for u, v in zip(a, b):
        assert torch.equal(_bits(u), _bits(v)), float((u.double() - v.double()).abs().max())
    return a


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g) * scale


def _within(got, ref, bound):
    err = (got.double() - ref).abs()
    assert (err <= bound).all(), float((err / bound).max())


def _gemm_ex(ta, tb, M, N, K, A, B, C, ep, impl=1):
    from go1_b200 import capi
    capi.check(capi.lib().go1_gemm_ex(ta, tb, M, N, K, capi.ptr(A), A.stride(0), capi.ptr(B), B.stride(0), capi.ptr(C), C.stride(0), ep, impl,
                                      capi.stream_ptr()), "go1_gemm_ex")


@pytest.mark.parametrize("impl,M,N,K", [(1, 1280, 2105, 24576), (2, 1280, 2105, 24576), (1, 256, 2101, 24576), (1, 48, 512, 2105), (0, 48, 1280, 2105)])
def test_split_k_products_are_bitwise_repeatable(impl, M, N, K):
    """The first layers' fused weight gradient (170 tiles, 3 splits) at impl 1 and 2, the adaptation module's (34 tiles, 11 splits), a
    per-net first layer at 48 rows (forward, bias + activation after the split) on the tensor cores and on the CUDA cores (impl 0)."""
    from go1_b200 import capi
    fwd = K == 2105
    A = _rand(M, K, seed=1)
    B = _rand(N, K, seed=2, scale=K ** -0.5 if fwd else 1.0)
    bias = _rand(N, seed=3) if fwd else None
    if impl == 2:
        A16 = torch.zeros(M, capi.bf16_pitch(K), device="cuda", dtype=torch.bfloat16)[:, :K].copy_(A)
        B16 = torch.zeros(N, capi.bf16_pitch(K), device="cuda", dtype=torch.bfloat16)[:, :K].copy_(B)
        A, B = A16.double(), B16.double()

    def run():
        C = torch.empty(M, (N + 31) // 32 * 32, device="cuda")[:, :N]
        ep = capi.Go1GemmEpilogue()
        if fwd:
            ep.bias, ep.act = bias.data_ptr(), 1
        if impl == 2:
            capi.check(capi.lib().go1_gemm_bf16_ex(0, 1, M, N, K, capi.ptr(A16), A16.stride(0), capi.ptr(B16), B16.stride(0), capi.ptr(C), C.stride(0), ep,
                                                   capi.stream_ptr()), "go1_gemm_bf16_ex")
        else:
            Af = torch.empty(M, (K + 31) // 32 * 32, device="cuda")[:, :K].copy_(A)
            Bf = torch.empty(N, (K + 31) // 32 * 32, device="cuda")[:, :K].copy_(B)
            _gemm_ex(0, 1, M, N, K, Af, Bf, C, ep, impl)
        return [C]

    C, = _twice(run)
    A64, B64 = A.double(), B.double()
    ref = A64 @ B64.t()
    scale = A64.abs() @ B64.abs().t()
    if fwd:
        ref = torch.nn.functional.elu(ref + bias.double())
    k = TF32 if impl == 1 else 4.0 * K * 2.0 ** -24      # impl 2: the rounded operands exactly; impl 0: fp32 products
    _within(C, ref, k * scale + 1e-6)


@pytest.mark.parametrize("bf16", [False, True])
def test_grouped_wgrads_are_bitwise_repeatable(bf16):
    """Two 512 x 512 x 24576 weight gradients (MN-major dz and layer input) in one grouped grid, split along K."""
    import ctypes as C
    from go1_b200 import capi
    M, N, K = 512, 512, 24576
    dz = [_rand(K, M, seed=10 + p) for p in range(2)]
    x = [_rand(K, N, seed=20 + p) for p in range(2)]
    if bf16:
        dz, x = [t.to(torch.bfloat16) for t in dz], [t.to(torch.bfloat16) for t in x]

    def run():
        outs = [torch.zeros(M, N, device="cuda") for _ in range(2)]
        A = (C.c_void_p * 2)(*[t.data_ptr() for t in dz])
        B = (C.c_void_p * 2)(*[t.data_ptr() for t in x])
        Cc = (C.c_void_p * 2)(*[t.data_ptr() for t in outs])
        f = capi.lib().go1_gemm_bf16_grouped if bf16 else capi.lib().go1_gemm_grouped
        capi.check(f(1, 0, M, N, K, 2, A, M, B, N, Cc, N, 1, capi.stream_ptr()), "grouped")
        return outs

    outs = _twice(run)
    for p in range(2):
        A64, B64 = dz[p].double().t(), x[p].double().t()
        _within(outs[p], A64 @ B64.t(), (4.0 * K * 2.0 ** -24 if bf16 else TF32) * (A64.abs() @ B64.abs().t()) + 1e-6)


@pytest.mark.parametrize("M", [24576, 24000, 600])
def test_dgrad_epilogue_sums_are_bitwise_repeatable(M):
    """A hidden-layer dgrad with the derivative, the column sums (bias gradient) and two trailing inputs (their weight and input gradients)
    fused into its epilogue, and the 45-wide and 2-wide trailing-input backward kernels.  M = 24000 (4000 envs x 24 steps / 4 minibatches)
    and 600: the last 128-row tile ends in a 32-row block that lies wholly beyond M."""
    from go1_b200 import capi
    N, K, nbx = 512, 256, 2
    dzn = _rand(M, K, seed=1)
    W = _rand(K, N, seed=2, scale=K ** -0.5)
    y = torch.nn.functional.elu(_rand(M, N, seed=3))
    bx, bwx = _rand(M, nbx, seed=4), _rand(N, nbx, seed=5)

    def run():
        Cm = torch.empty(M, N, device="cuda")
        cs, gwx, dx = torch.zeros(N, device="cuda"), torch.zeros(N, nbx, device="cuda"), torch.zeros(M, nbx, device="cuda")
        ep = capi.Go1GemmEpilogue()
        ep.act, ep.dact_y, ep.ld_dact_y, ep.colsum = 2, y.data_ptr(), N, cs.data_ptr()
        ep.bwd_extra, ep.ld_bwd_extra, ep.num_bwd_extra = bx.data_ptr(), nbx, nbx
        ep.bwd_w_extra, ep.ld_bwd_w_extra, ep.g_w_extra, ep.ld_g_w_extra, ep.d_extra, ep.ld_d_extra = bwx.data_ptr(), nbx, gwx.data_ptr(), nbx, dx.data_ptr(), nbx
        _gemm_ex(0, 0, M, N, K, dzn, W, Cm, ep)
        return [Cm, cs, gwx, dx]

    Cm, cs, gwx, dx = _twice(run)
    fd = torch.where(y.double() > 0, 1.0, y.double() + 1.0)
    ref = (dzn.double() @ W.double()) * fd
    e = TF32 * (dzn.double().abs() @ W.double().abs()) * fd.abs() + 1e-7
    _within(Cm, ref, e)
    _within(cs, ref.sum(0), e.sum(0) + M * 2.0 ** -22 * ref.abs().sum(0))
    _within(gwx, ref.t() @ bx.double(), e.t() @ bx.double().abs() + M * 2.0 ** -22 * ref.abs().t() @ bx.double().abs())
    _within(dx, ref @ bwx.double(), e @ bwx.double().abs() + N * 2.0 ** -22 * ref.abs() @ bwx.double().abs())

    o = 512
    for E in (45, 2):
        dz, ex = _rand(M, o, seed=6), _rand(M, E, seed=7)

        def run_x():
            g = torch.empty(o, E, device="cuda")
            capi.check(capi.lib().go1_mlp_extra_backward(capi.ptr(dz), o, 0, capi.ptr(ex), E, None, 0, capi.ptr(g), E, None, 0, M, o, E, 0,
                                                         capi.stream_ptr()), "extra_backward")
            return [g]

        g, = _twice(run_x)
        r = dz.double().t() @ ex.double()
        _within(g, r, M * 2.0 ** -22 * (dz.double().abs().t() @ ex.double().abs()))


@pytest.mark.parametrize("K", [128, 130])
def test_skinny_kernels_and_colsum_are_bitwise_repeatable(K):
    """The narrow heads' weight gradient (with the fused bias gradient: shared-memory sums in warp order) and dgrad with column sums (fp32
    and BF16 output), and the column sums, on their vector (K = 128) and scalar (K = 130) paths."""
    from go1_b200 import capi
    L, st = capi.lib(), capi.stream_ptr
    M, o = 24576, 12
    dz, x = _rand(M, o, seed=1), _rand(M, K, seed=2)
    W, yp = _rand(o, 128, seed=3), torch.nn.functional.elu(_rand(M, 128, seed=4))

    def run():
        gW, gb = torch.empty(o, K, device="cuda"), torch.empty(o, device="cuda")
        capi.check(L.go1_skinny_wgrad_ex(capi.ptr(dz), o, capi.ptr(x), K, capi.ptr(gW), K, capi.ptr(gb) if K % 4 == 0 else None, M, o, K, 0, st()), "skinny_wgrad")
        cs = torch.empty(K, device="cuda")
        capi.check(L.go1_colsum(capi.ptr(x), K, capi.ptr(cs), M, K, 0, st()), "colsum")
        out = [gW, cs] + ([gb] if K % 4 == 0 else [])
        if K == 128:
            dp, c1 = torch.empty(M, 128, device="cuda"), torch.zeros(128, device="cuda")
            capi.check(L.go1_skinny_dgrad_act(capi.ptr(dz), o, capi.ptr(W), 128, capi.ptr(yp), 128, capi.ptr(dp), 128, capi.ptr(c1), M, o, 128, 0, st()), "dgrad")
            d16, c2 = torch.empty(M, 128, device="cuda", dtype=torch.bfloat16), torch.zeros(128, device="cuda")
            capi.check(L.go1_skinny_dgrad_act_bf16(capi.ptr(dz), o, capi.ptr(W), 128, capi.ptr(yp), 128, capi.ptr(d16), 128, capi.ptr(c2), M, o, 128, 0, st()),
                       "dgrad16")
            out += [dp, c1, d16, c2]
        return out

    out = _twice(run)
    d64, x64 = dz.double(), x.double()
    _within(out[0], d64.t() @ x64, M * 2.0 ** -22 * (d64.abs().t() @ x64.abs()))
    _within(out[1], x64.sum(0), M * 2.0 ** -22 * x64.abs().sum(0))
    if K == 128:
        _within(out[2], d64.sum(0), M * 2.0 ** -22 * d64.abs().sum(0))
        fd = torch.where(yp.double() > 0, 1.0, yp.double() + 1.0)
        ref = (d64 @ W.double()) * fd
        _within(out[3], ref, 1e-5 * (d64.abs() @ W.double().abs()) * fd.abs())
        for c in (out[4], out[6]):
            _within(c, ref.sum(0), M * 2.0 ** -22 * ref.abs().sum(0) + 1e-4)
        assert torch.equal(out[5], out[3].to(torch.bfloat16))


def test_loss_statistics_are_bitwise_repeatable():
    """The PPO loss scalars and std gradient, the adaptation MSE pair, the gradient norm and the advantage statistics at 4096 envs x 24
    steps (one 24576-row minibatch for the per-row kernels)."""
    from go1_b200 import capi
    L, st = capi.lib(), capi.stream_ptr
    n, na, T, N = 24576, 12, 24, 4096
    mean, old_mean = _rand(n, na, seed=1), _rand(n, na, seed=2)
    std, old_std = torch.rand(na, device="cuda") + 0.5, torch.rand(n, na, device="cuda") + 0.5
    actions = mean + std * _rand(n, na, seed=3)
    value, ret, oldv, adv, old_logp = (_rand(n, seed=s) for s in (4, 5, 6, 7, 8))
    pred, tgt = _rand(n, 2, seed=9), _rand(n, 2, seed=10)
    grad = _rand(3054619, seed=11)
    rew, vals, last = _rand(T, N, seed=12), _rand(T, N, seed=13), _rand(N, seed=14)
    dones = (torch.rand(T, N, device="cuda") < 0.05).to(torch.uint8)

    def run():
        dmean, dvalue, dstd, sc = torch.empty(n, na, device="cuda"), torch.empty(n, device="cuda"), torch.empty(na, device="cuda"), torch.empty(8, device="cuda")
        capi.check(L.go1_ppo_loss(capi.ptr(mean), na, capi.ptr(std), capi.ptr(value), capi.ptr(actions), capi.ptr(old_logp), capi.ptr(old_mean),
                                  capi.ptr(old_std), capi.ptr(adv), capi.ptr(ret), capi.ptr(oldv), capi.ptr(dmean), na, capi.ptr(dvalue), capi.ptr(dstd),
                                  capi.ptr(sc), n, na, 0.2, 1.0, 0.01, 1, 1.0 / n, st()), "loss")
        dpred, msc = torch.empty(n, 2, device="cuda"), torch.empty(2, device="cuda")
        capi.check(L.go1_ppo_mse(capi.ptr(pred), 2, capi.ptr(tgt), 2, capi.ptr(dpred), 2, capi.ptr(msc), n, n // 5 * 4, 2, st()), "mse")
        gsq = torch.empty(1, device="cuda", dtype=torch.float64)
        capi.check(L.go1_ppo_grad_sqnorm(capi.ptr(grad), grad.numel(), capi.ptr(gsq), st()), "sqnorm")
        R, A, stats = torch.empty(T, N, device="cuda"), torch.empty(T, N, device="cuda"), torch.empty(2, device="cuda", dtype=torch.float64)
        capi.check(L.go1_ppo_gae(capi.ptr(rew), capi.ptr(dones), capi.ptr(vals), capi.ptr(last), capi.ptr(R), capi.ptr(A), capi.ptr(stats), T, N, 0.99, 0.95,
                                 st()), "gae")
        return [dmean, dvalue, dstd, sc, dpred, msc, gsq, R, A, stats]

    out = _twice(run)
    default = run()          # the default mode: the same numerics up to the order of the sums
    for a, b in zip(out, default):
        assert torch.allclose(a.double(), b.double(), rtol=1e-5, atol=1e-6), float((a.double() - b.double()).abs().max())
    g64 = grad.double()
    assert abs(float(out[6]) - float((g64 * g64).sum())) <= 1e-9 * float((g64 * g64).sum())
    A64 = out[8].double()
    assert abs(float(out[9][0]) - float(A64.sum())) <= 1e-9 * float(A64.abs().sum())
    assert abs(float(out[9][1]) - float((A64 * A64).sum())) <= 1e-9 * float((A64 * A64).sum())
    d = pred.double() - tgt.double()
    ntr = n // 5 * 4
    assert abs(float(out[5][0]) - float((d[:ntr] ** 2).mean())) <= 1e-5 * float((d[:ntr] ** 2).mean())
    assert abs(float(out[5][1]) - float((d[ntr:] ** 2).mean())) <= 1e-5 * float((d[ntr:] ** 2).mean())


def _training_run(tmp_path, n, impl, bf16_backward, iters=3):
    """Runner rollout + compute_returns + update, `iters` times, from fixed seeds (as the graph-vs-eager rollout test reseeds), in
    deterministic mode: everything the run computed, on the host."""
    from test_runner_gpu import _make
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    saved = (AC_Args.gemm_impl, AC_Args.bf16_backward, AC_Args.deterministic)
    AC_Args.gemm_impl, AC_Args.bf16_backward, AC_Args.deterministic = impl, bf16_backward, True
    try:
        torch.manual_seed(0); np.random.seed(0)
        env, Runner, RunnerArgs, logger = _make(tmp_path, n=n)
        RunnerArgs.num_steps_per_env, RunnerArgs.resume = 24, False
        runner = Runner(env, device="cuda:0")
        alg, ac = runner.alg, runner.alg.actor_critic
        assert ac.deterministic
        g = torch.Generator().manual_seed(1)
        env.episode_length_buf = torch.randint(0, 1001, (n,), generator=g)
        od = env.get_observations()
        state = (od["obs"], od["privileged_obs"], od["obs_history"])
        snaps = []
        for it in range(iters):
            obs, priv, hist, infos = runner.rollout(*state)
            state = (obs, priv, hist)
            alg.compute_returns(hist, priv)
            st = alg.storage
            snap = {k: getattr(st, k).clone() for k in ("observations", "privileged_observations", "observation_histories", "actions", "rewards", "dones",
                                                        "values", "actions_log_prob", "mu", "sigma", "returns", "advantages")}
            snap["losses"] = torch.tensor(alg.update(), dtype=torch.float64)
            snap["lr"] = torch.tensor([alg.learning_rate], dtype=torch.float64)
            snap["params"] = ac.flat_params.clone()
            for name, opt in (("ppo", alg.optimizer), ("adapt", alg.adaptation_module_optimizer)):
                snap[name + "_m"], snap[name + "_v"] = opt.exp_avg.clone(), opt.exp_avg_sq.clone()
            env.env._curriculum_to_host(keep_device=True)
            snap["curriculum"] = torch.tensor(np.stack([c.weights for c in env.curricula]))
            snaps.append({k: v.cpu() for k, v in snap.items()})
        return snaps
    finally:
        AC_Args.gemm_impl, AC_Args.bf16_backward, AC_Args.deterministic = saved


@pytest.mark.parametrize("impl,bf16_backward,n", [(1, False, 1024), (2, False, 1024), (2, True, 1024), (0, False, 64)])
def test_training_iterations_are_bitwise_repeatable(tmp_path, monkeypatch, impl, bf16_backward, n):
    """Two runs of three training iterations in one process: parameters, both Adam moments, learning rate, losses, curriculum weights and
    the rollout storage are bit-identical (1024 envs: 6144-row minibatches, split-K products and the update's second stream)."""
    monkeypatch.chdir(tmp_path)
    a = _training_run(tmp_path, n, impl, bf16_backward)
    b = _training_run(tmp_path, n, impl, bf16_backward)
    for it, (x, y) in enumerate(zip(a, b)):
        for k in x:
            assert torch.equal(_bits(x[k]) if x[k].is_floating_point() else x[k], _bits(y[k]) if y[k].is_floating_point() else y[k]), (it, k)
    assert float(a[-1]["losses"][0]) != 0.0


@pytest.mark.parametrize("impl", [0, 1])
def test_golden_ppo_cycle_in_deterministic_mode(impl):
    """The golden PPO cycle (tests/golden/ppo.npz) in deterministic mode stays within the bounds of the default mode's test."""
    import test_ppo_gpu
    from go1_gym_learn.ppo_cse.actor_critic import AC_Args
    saved = AC_Args.deterministic
    AC_Args.deterministic = True
    try:
        test_ppo_gpu.test_full_ppo_cycle_matches_reference_golden(impl)
    finally:
        AC_Args.deterministic = saved
