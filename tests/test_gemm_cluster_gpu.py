"""The paired persistent GEMM: products with K-major operands whose 128 x 128 tile grid has an even tile count along N or M run in
clusters of two CTAs that share one operand box per k-block by TMA multicast.  Non-split products must equal, bit for bit, the same
product computed one output tile per launch (a single-tile launch has no pair); split-K products must meet the TF32 bound; the path is
taken only where it applies (the `kernel` column of the GO1_GEMM_TIMING_CSV dump) and works inside a captured CUDA graph."""
import csv
import ctypes as C
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "walk-these-ways_b200", "compat"))

K_IN = 2100                                   # the first layers' reduction (history width)
NEX = 2                                       # trailing priv columns of the fused first-layer forward


def _capi():
    from go1_b200 import capi
    return capi


def _ptr_at(t, row, col):
    return C.c_void_p(t.data_ptr() + (row * t.stride(0) + col) * t.element_size())


def _gemm_ex(ta, tb, M, N, K, A, lda, B, ldb, Cp, ldc, ep):
    capi = _capi()
    capi.check(capi.lib().go1_gemm_ex(ta, tb, M, N, K, A, lda, B, ldb, Cp, ldc, ep, 1, capi.stream_ptr()), "gemm_ex")


def _labels(tmp_path, monkeypatch, fn):
    """The `kernel` column of every product fn launches (eagerly)."""
    capi = _capi()
    out = tmp_path / "gemm.csv"
    monkeypatch.setenv("GO1_GEMM_TIMING_CSV", str(out))
    capi.check(capi.lib().go1_gemm_timing(1, None, None, None), "timing")
    fn()
    capi.check(capi.lib().go1_gemm_timing(0, None, None, None), "timing")
    return [r["kernel"] for r in csv.DictReader(open(out))]


class Fused:
    """The fused first-layer forward: C = f(A B^T + ex wex^T + bias) on columns < lead, A B^T + bias beyond; optionally stored as C^T."""

    def __init__(self, M, N, kind, ct, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        r = lambda *s: torch.randn(*s, device="cuda", generator=g)
        self.M, self.N, self.kind, self.ct = M, N, kind, ct
        self.A, self.B = r(M, K_IN) * 0.3, r(N, K_IN) * 0.05
        self.ex, self.wex, self.bias = r(M, NEX), r(N, NEX) * 0.1, r(N) * 0.1
        self.lead = N - 200                   # one tile straddles the lead, the last lies wholly past it
        self.ldc = (M + 3) // 4 * 4 if ct else N
        self.C = torch.full((N, self.ldc) if ct else (M, N), 7.0, device="cuda")
        self.ref = torch.full_like(self.C, 7.0)
        self.sink = torch.zeros(N, device="cuda")

    def _ep(self, i0, j0, tile):
        capi = _capi()
        ep = capi.Go1GemmEpilogue()
        ep.bias = self.bias.data_ptr() + 4 * j0
        ep.act_kind, ep.store_transposed = self.kind, self.ct
        lead = self.lead - j0
        if lead > 0:
            ep.act, ep.lead_cols = 1, lead
            ep.extra, ep.ld_extra = _ptr_at(self.ex, i0, 0).value, NEX
            ep.w_extra, ep.ld_w_extra, ep.num_extra = _ptr_at(self.wex, j0, 0).value, NEX, NEX
        if tile:                              # the column sums keep a one-tile product unsplit (they do not touch C)
            ep.colsum = self.sink.data_ptr()
        return ep

    def _out(self, C_, i0, j0):
        return _ptr_at(C_, j0, i0) if self.ct else _ptr_at(C_, i0, j0)

    def run(self):
        capi = _capi()
        _gemm_ex(0, 1, self.M, self.N, K_IN, capi.ptr(self.A), K_IN, capi.ptr(self.B), K_IN, capi.ptr(self.C), self.ldc, self._ep(0, 0, False))

    def run_tiles(self):
        for i0 in range(0, self.M, 128):
            mi = min(128, self.M - i0)
            for j0 in range(0, self.N, 128):
                nj = min(128, self.N - j0)
                _gemm_ex(0, 1, mi, nj, K_IN, _ptr_at(self.A, i0, 0), K_IN, _ptr_at(self.B, j0, 0), K_IN, self._out(self.ref, i0, j0), self.ldc,
                         self._ep(i0, j0, True))

    def check(self):
        self.run_tiles()
        torch.cuda.synchronize()
        assert torch.equal(self.C, self.ref)


@pytest.mark.parametrize("M,N,kind,ct", [
    (24576 + 37, 1280, 0, 0),                 # the fused forward of one update, pairs along N
    (24576 + 37, 1280, 4, 1),                 # tanh, stored transposed
    (4097, 1280, 0, 0),                       # the rollout's batch and one row more
    (4097, 1280, 1, 0),                       # selu
    (200, 1280, 0, 1),
    (24576, 384, 0, 0),                       # three column tiles: pairs along M
    (200, 384, 4, 1),
])
def test_paired_fused_forward_equals_tile_by_tile(tmp_path, monkeypatch, M, N, kind, ct):
    f = Fused(M, N, kind, ct, seed=M + N + kind + ct)
    assert _labels(tmp_path, monkeypatch, f.run) == ["p128c2"]
    f.check()
    if ct:                                    # the padding of C^T past M rounded up to 4 is left alone
        assert bool((f.C[:, (M + 3) // 4 * 4:] == 7.0).all())


@pytest.mark.parametrize("M,N", [(1280, 2105), (256, 2101), (512, 2048)])
def test_paired_split_k_wgrad_within_tf32_bound(tmp_path, monkeypatch, M, N):
    """The first-layer weight gradients (pairs along M: odd column-tile counts) and one with pairs along N, split along K."""
    capi = _capi()
    K = 24576
    g = torch.Generator(device="cuda").manual_seed(M + N)
    A = torch.randn(M, K, device="cuda", generator=g)
    B = torch.randn(N, K, device="cuda", generator=g)
    Cm = torch.full((M, N), 3.0, device="cuda")
    run = lambda: capi.check(capi.lib().go1_gemm(0, 1, M, N, K, capi.ptr(A), K, capi.ptr(B), K, capi.ptr(Cm), N, None, 0, 0, 1,
                                                 capi.stream_ptr()), "gemm")
    assert _labels(tmp_path, monkeypatch, run) == ["p128c2"]
    torch.cuda.synchronize()
    ref = A.double() @ B.double().t()
    tol = 2.0 ** -9 * (A.abs().double() @ B.abs().double().t()) + 1e-4
    assert bool(((Cm.double() - ref).abs() <= tol).all())


def test_pair_selection(tmp_path, monkeypatch):
    """Odd tile counts both ways, MN-major operands, grouped launches and the activation-derivative epilogue (act 2) keep one CTA per tile."""
    capi = _capi()
    L = capi.lib()
    A, B = torch.randn(1280, K_IN, device="cuda"), torch.randn(1280, K_IN, device="cuda")
    AT = torch.randn(K_IN, 1280, device="cuda")
    Cm = torch.empty(1280, 1280, device="cuda")
    arr = lambda ts: (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
    C2 = torch.zeros(1280, 1280, device="cuda")
    Y = torch.rand(1280, 1280, device="cuda")
    ep = capi.Go1GemmEpilogue()
    ep.act, ep.dact_y, ep.ld_dact_y = 2, Y.data_ptr(), 1280
    labels = _labels(tmp_path, monkeypatch, lambda: [
        capi.check(L.go1_gemm(0, 1, 384, 384, K_IN, capi.ptr(A), K_IN, capi.ptr(B), K_IN, capi.ptr(Cm), 1280, None, 0, 0, 1, capi.stream_ptr()), "odd"),
        capi.check(L.go1_gemm(1, 1, 1280, 1280, K_IN, capi.ptr(AT), 1280, capi.ptr(B), K_IN, capi.ptr(Cm), 1280, None, 0, 0, 1, capi.stream_ptr()), "mn"),
        capi.check(L.go1_gemm_grouped(0, 1, 1280, 1280, K_IN, 2, arr([A, B]), K_IN, arr([B, A]), K_IN, arr([Cm, C2]), 1280, 0,
                                      capi.stream_ptr()), "grouped"),
        _gemm_ex(0, 1, 1280, 1280, K_IN, capi.ptr(A), K_IN, capi.ptr(B), K_IN, capi.ptr(Cm), 1280, ep),
        capi.check(L.go1_gemm(0, 1, 1280, 1280, K_IN, capi.ptr(A), K_IN, capi.ptr(B), K_IN, capi.ptr(Cm), 1280, None, 0, 0, 1, capi.stream_ptr()), "paired"),
    ])
    assert labels == ["p128", "p128", "p128", "p128", "p128c2"]


def test_paired_product_in_cuda_graph():
    """The rollout's fused forward runs inside a captured graph: replaying it gives the eager result bit for bit."""
    f = Fused(4096, 1280, 0, 0, seed=11)
    f.run()
    torch.cuda.synchronize()
    eager = f.C.clone()
    f.C.fill_(7.0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        f.run()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(f.C, eager)


def test_back_to_back_pairs_along_n_and_m():
    """Two paired products on one stream without a synchronisation between them, one paired along N and one along M."""
    fn, fm = Fused(4097, 1280, 0, 0, seed=21), Fused(24576, 384, 0, 0, seed=22)
    fn.run()
    fm.run()
    fn.check()
    fm.check()
