"""ActorCritic of ppo_cse (reference go1_gym_learn/ppo_cse/actor_critic.py:19-147) on hand-written kernels.

Same public surface (AC_Args, ActorCritic(num_obs, num_privileged_obs, num_obs_history, num_actions),
.adaptation_module / .actor_body / .critic_body as nn.Sequential so checkpoints and TorchScript exports keep
the reference's names, .act / .evaluate / .act_student / .act_teacher / .get_actions_log_prob / .action_mean /
.action_std / .entropy), but:
  * all parameters are views into ONE flat fp32 buffer (adaptation module first), gradients into one flat
    gradient buffer -> one grad-norm, one Adam launch, one NCCL all-reduce per optimizer step;
  * forward and backward are explicit go1_gemm calls (fp32 CUDA-core or wgmma TF32) with fused
    bias+activation epilogues (AC_Args.activation: every name of the reference's get_activation); cat(obs_history, latent) is never materialised (the E = num_privileged_obs trailing
    input columns are added to the first layer's pre-activation: in the GEMM epilogue for E <= 4, by go1_mlp_extra_forward after
    the product for 4 < E <= 64);
  * no autograd graph: the backward pass is written out (see `backward_ppo`, `backward_adaptation`).
"""
import functools
import numbers
import os

import torch
import torch.nn as nn
from params_proto import PrefixProto

from go1_b200 import capi


class AC_Args(PrefixProto, cli=False):
    # policy
    init_noise_std = 1.0
    actor_hidden_dims = [512, 256, 128]
    critic_hidden_dims = [512, 256, 128]
    activation = 'elu'  # can be elu, relu, selu, crelu, lrelu, tanh, sigmoid (all run on the fused kernels; crelu is nn.ReLU, as in the reference)
    adaptation_module_branch_hidden_dims = [256, 128]
    use_decoder = False
    gemm_impl = 1       # 1 = wgmma TF32 tensor cores (default; torch 1.10, the reference's pin, also ran these matmuls in TF32), 0 = fp32 CUDA cores (exact),
                        # 2 = as 1, but the products that reduce over the observation history (the first layers) take BF16 operands (fp32 accumulation)
    bf16_backward = False   # with gemm_impl = 2 only: the hidden layers' dgrads and weight gradients run on BF16 too (MN-major operands read in place);
                            # hidden-layer dz is then held in BF16 (see ActorCritic.backward_ppo)
    deterministic = os.environ.get("GO1_DETERMINISTIC", "0") != "0"   # fixed-order learner reductions: bit-identical runs from identical inputs (go1_set_deterministic)


def in_mode(method):
    """Runs an ActorCritic / PPO / RolloutStorage method in the deterministic mode of the object (its `deterministic` attribute): the library
    mode is set around the call and restored afterwards, so that learners of either mode can be used side by side."""
    @functools.wraps(method)
    def wrapped(self, *a, **k):
        with capi.deterministic(self.deterministic):
            return method(self, *a, **k)
    return wrapped


def _mlp(in_dim, hidden, out_dim, activation):
    layers, d = [], in_dim
    for h in hidden:
        layers += [nn.Linear(d, h), get_activation(activation)]
        d = h
    layers.append(nn.Linear(d, out_dim))
    return nn.Sequential(*layers)


def _empty(*shape, device, dtype=torch.float32):
    """Scratch buffers outlive the Runner's torch.inference_mode() rollout block and are written again by the update,
    so they must be ordinary (non-inference) tensors whichever mode they are first needed in."""
    with torch.inference_mode(False):
        return torch.empty(*shape, device=device, dtype=dtype)


_TRANSPOSE = {(torch.float32, torch.float32): "go1_transpose", (torch.bfloat16, torch.bfloat16): "go1_transpose_bf16",
              (torch.float32, torch.bfloat16): "go1_transpose_to_bf16"}


def _transpose(x, out):
    """out[:cols][:M] = x^T for x [M][cols] (unit inner strides); an fp32 x into a BF16 out is rounded to nearest even."""
    name = _TRANSPOSE[(x.dtype, out.dtype)]
    capi.check(getattr(capi.lib(), name)(capi.ptr(x), x.stride(0), capi.ptr(out), out.stride(0), x.shape[0], x.shape[1], capi.stream_ptr()), name)


def _to_bf16(x, out):
    """out = x rounded to BF16 (nearest even) in one go1_convert_bf16 launch; x fp32 [rows][cols], out BF16, unit inner strides."""
    capi.check(capi.lib().go1_convert_bf16(capi.ptr(x), x.stride(0), capi.ptr(out), out.stride(0), x.shape[0], x.shape[1], capi.stream_ptr()), "convert_bf16")
    return out


def history_kmajor(h, priv, out):
    """The first layers' input transposed, K-major for their weight-gradient products: out[K0 + 1 + 2E][>= M] gets h's K0 columns as rows
    0..K0-1, ones in row K0 and priv's E columns in rows K0 + 1.. (priv None: only K0 + 1 rows).  Rows K0 + 1 + E.. are left for the
    latent, which ActorCritic.backward_ppo writes for each minibatch.  out is fp32 with h fp32 (row pitch a multiple of 4 floats), or BF16
    with the BF16 history of AC_Args.gemm_impl = 2 (row pitch a multiple of 8 elements): the history rows are copied, the ones row is
    exact and priv is rounded to BF16 (nearest even)."""
    M, K0 = h.shape[0], h.shape[1]
    _transpose(h, out)
    out[K0, :M].fill_(1.0)
    if priv is not None:
        _transpose(priv, out[K0 + 1:])
    return out


class _Net:
    """Forward/backward of one MLP whose first layer reads [x (K0 columns) | extra (E columns)].

    impl 0: every product is one fp32 CUDA-core go1_gemm.  impl 1: the large products run on the wgmma TF32 kernel,
    which reads its operands through TMA (16-byte aligned rows) in either major: forward K-major, dgrad with W as an
    MN-major B operand, wgrad with dz and the layer input as MN-major A and B operands -- except the first layers' wgrad, which
    ActorCritic runs K-major on transposed copies (history_kmajor, dz1T).  Hidden activations and their gradients live in buffers whose
    row pitch is capi.row_pitch(width) (_hbuf); a weight whose rows are not a multiple of 4 floats long (the first-layer block W[:, :K0],
    any hidden width that is not) is read through a packed TMA-readable copy, cached per weight version (_packed).

    The layers behind the first one run as a fused tail (go1_mlp_tail_forward_grouped) from layer `tail_start` on: the last two hidden
    layers and the head when their widths are at most 256 and 128, else the last hidden layer (up to 256 wide) and the head; earlier
    layers run one by one."""

    def __init__(self, seq, flat, grad, offsets, owner):
        self.linears = [m for m in seq if isinstance(m, nn.Linear)]
        self.specs = []                       # (w_off, b_off, out, in)
        for lin in self.linears:
            o, i = lin.weight.shape
            self.specs.append((offsets[id(lin.weight)], offsets[id(lin.bias)], o, i))
        last = self.linears[-1]
        self.end = offsets[id(last.bias)] + last.bias.numel()
        self.flat, self.grad, self.owner = flat, grad, owner
        self.acts = {}
        self._cache = {}
        self._ep = capi.Go1GemmEpilogue()
        self.kind = self._ep.act_kind = owner.act_kind      # Go1Activation of the hidden layers, passed to every kernel that applies f or f'
        hidden = [sp[2] for sp in self.specs[:-1]]
        if len(hidden) >= 3 and hidden[-2] <= 256 and hidden[-1] <= 128:
            self.tail_start = len(hidden) - 2
        elif len(hidden) >= 2 and hidden[-1] <= 256:
            self.tail_start = len(hidden) - 1
        else:
            self.tail_start = None

    def _buf(self, key, M, width, pitch=None, dtype=torch.float32):
        """[M][width] view of a cached buffer with row pitch `pitch` (default: width)."""
        pitch = width if pitch is None else pitch
        t = self.acts.get(key)
        if t is None or t.shape[0] < M or t.shape[1] != pitch or t.dtype != dtype:
            t = _empty(M, pitch, device=self.flat.device, dtype=dtype)
            self.acts[key] = t
        return t[:M, :width]

    def _buf16(self, key, M, width):
        """A BF16 operand buffer of AC_Args.gemm_impl = 2 (TMA-readable rows: capi.bf16_pitch)."""
        return self._buf(key, M, width, capi.bf16_pitch(width), torch.bfloat16)

    def _hbuf(self, key, M, width):
        """A hidden activation or gradient buffer: TMA-readable rows whatever the width."""
        return self._buf(key, M, width, capi.row_pitch(width))

    def _packed(self, li, K, dtype=torch.float32):
        """(copy, pitch): W[:, :K] of layer li in a TMA-readable copy, rebuilt once per weight version: fp32 with a row pitch that is a
        multiple of 128 bytes (any K: the kernels read the K tail as zeros), or BF16 (rounded to nearest even) with row pitch
        capi.bf16_pitch(K) (AC_Args.gemm_impl = 2: the first layers' operand; AC_Args.bf16_backward: the dgrads' MN-major B operand)."""
        W = self._cached((li, K, dtype), self._packer(li, K, dtype))
        return W, W.stride(0)

    def _packer(self, li, K, dtype):
        """The builder of _packed's cache entry.  pairs: a list that receives the BF16 conversion (dst, src) in place of launching it."""
        wo, bo, o, i = self.specs[li]
        W = self.flat[wo:wo + o * i].view(o, i)[:, :K]
        pitch = capi.bf16_pitch(K) if dtype == torch.bfloat16 else (K + 31) // 32 * 32

        def build(old, pairs=None):
            dst = old if old is not None else _empty(o, pitch, device=W.device, dtype=dtype)[:, :K]
            if dtype != torch.bfloat16:
                return dst.copy_(W)
            if pairs is None:
                return _to_bf16(W, dst)
            pairs.append((dst, W))
            return dst
        return build

    def packed16_pairs(self):
        """The (dst, src) conversions that bring the BF16 weight copies of layers 1.. (the MN-major B operands of the AC_Args.bf16_backward
        dgrads) up to the current weight version.  Their cache entries are marked current here; the caller launches the conversions
        (ActorCritic._convert_outputs: in the one launch that also makes the output copies, instead of one launch per layer)."""
        pairs = []
        for li in range(1, len(self.specs)):
            i = self.specs[li][3]
            self._cached((li, i, torch.bfloat16), self._packer(li, i, torch.bfloat16), pairs)
        return pairs

    def _weight_tma(self, li):
        """(W, row stride) of layer li for a TMA operand: in place when its rows allow it, else the packed copy."""
        wo, bo, o, i = self.specs[li]
        W = self.flat[wo:wo + o * i]
        return (W, i) if self._tma_ok(W, i) else self._packed(li, i)

    def _cached(self, key, build, pairs=None):
        """A packed copy of weights, keyed by (layer, K, dtype), rebuilt when the weights changed (weights_version).  The entry keeps its
        builder so that ActorCritic.ensure_packed() can refresh every copy eagerly before a CUDA graph that reads them is replayed: the
        graphs contain no packing kernels (the rollout replays one 24 times per weight version).  pairs: passed to the builder (_packer),
        which defers its BF16 conversion there."""
        ver = self.owner.weights_version
        hit = self._cache.get(key)
        if hit is None or hit[0] != ver:
            if torch.cuda.is_current_stream_capturing():
                raise capi.Go1Error("stale packed weights during graph capture: call ActorCritic.ensure_packed() first")
            old = hit[1] if hit else None
            hit = (ver, build(old) if pairs is None else build(old, pairs), build)
            self._cache[key] = hit
        return hit[1]

    def refresh_packed(self):
        ver = self.owner.weights_version
        for key, hit in list(self._cache.items()):
            if hit[0] != ver:
                self._cache[key] = (ver, hit[2](hit[1]), hit[2])

    @staticmethod
    def _p(x):
        return x.data_ptr() if torch.is_tensor(x) else x

    def _gemm(self, ta, tb, M, N, K, A, lda, B, ldb, Cm, ldc, impl=1, *, bias=None, act=0, acc=0, extra=None, w_extra=0, ld_w_extra=0, dact_y=None,
              lead_cols=0, colsum=None, bwd_extra=None, store_transposed=0, out16=None):
        """The entry point follows the operands: fp32 A and B -> go1_gemm_ex (impl 0 / 1); BF16 A and B, both K-major -> go1_gemm_bf16_ex;
        BF16 in any other major -> go1_gemm_bf16_mn (a BF16 Cm is stored row-major in BF16).  out16: a BF16 tensor that receives the
        transposed result (store_transposed) in place of Cm."""
        ep = self._ep
        ep.out_bf16, ep.ld_out_bf16 = (out16.data_ptr(), out16.stride(0)) if out16 is not None else (None, 0)
        ep.lead_cols = lead_cols
        ep.store_transposed = store_transposed
        ep.colsum = self._p(colsum) if colsum is not None else None
        if bwd_extra is not None:      # (extra [M][E], w_extra ptr, ld, g_w_extra ptr, ld, dextra [M][E] or None)
            ex, wex, ldw, gw, ldg, dex = bwd_extra
            ep.bwd_extra, ep.ld_bwd_extra, ep.num_bwd_extra = ex.data_ptr(), ex.stride(0), ex.shape[1]
            ep.bwd_w_extra, ep.ld_bwd_w_extra, ep.g_w_extra, ep.ld_g_w_extra = wex, ldw, gw, ldg      # gw None: no weight-gradient reduction
            ep.d_extra, ep.ld_d_extra = (dex.data_ptr(), dex.stride(0)) if dex is not None else (None, 0)
        else:
            ep.num_bwd_extra = 0
        ep.bias = self._p(bias) if bias is not None else None
        ep.act, ep.accumulate = act, acc
        if extra is not None:
            ep.extra, ep.ld_extra, ep.w_extra, ep.ld_w_extra, ep.num_extra = extra.data_ptr(), extra.stride(0), w_extra, ld_w_extra, extra.shape[1]
        else:
            ep.extra, ep.num_extra = None, 0
        if dact_y is not None:
            ep.dact_y, ep.ld_dact_y = dact_y.data_ptr(), dact_y.stride(0)
        else:
            ep.dact_y = None
        L, args = capi.lib(), (ta, tb, M, N, K, A.data_ptr(), lda, self._p(B), ldb, self._p(Cm), ldc)
        if A.dtype != torch.bfloat16:
            capi.check(L.go1_gemm_ex(*args, ep, impl, capi.stream_ptr()), "go1_gemm")
        elif (ta, tb) == (0, 1):
            capi.check(L.go1_gemm_bf16_ex(*args, ep, capi.stream_ptr()), "go1_gemm_bf16")
        else:
            c16 = 1 if torch.is_tensor(Cm) and Cm.dtype == torch.bfloat16 else 0
            capi.check(L.go1_gemm_bf16_mn(*args, c16, ep, capi.stream_ptr()), "go1_gemm_bf16_mn")

    @staticmethod
    def _tma_ok(x, ld):
        """TMA-readable K-major operand: 16-byte aligned base, row stride a multiple of 16 bytes."""
        p = x.data_ptr() if torch.is_tensor(x) else x
        return (p & 15) == 0 and (ld & 3) == 0

    def forward(self, x, ldx, K0, extra, M, impl, tag="a", first_out=None, defer_tail=False):
        """x: [M][K0] rows with stride ldx; extra: [M][E] contiguous or None. Returns list of layer outputs.
        first_out: the first layer's activated output if the caller already produced it (ActorCritic.forward_all).
        defer_tail: stop before the fused tail (the caller launches it, grouped with another net's) and return the outputs so far."""
        outs, inp, ld_in = [], x, ldx
        n = len(self.specs)
        for li, (wo, bo, o, i) in enumerate(self.specs):
            if li == 0 and first_out is not None:
                outs.append(first_out)
                inp, ld_in = first_out, first_out.stride(0)
                continue
            if li == self.tail_start and impl >= 1 and self._tail_ok() and self._tma_ok(inp, ld_in):
                return outs if defer_tail else outs + self._forward_tail(inp, ld_in, M, tag)
            y = self._hbuf((tag, li), M, o) if li < n - 1 else self._buf((tag, li), M, o)
            W = self.flat[wo:wo + o * i]
            b = self.flat[bo:bo + o]
            act = 1 if li < n - 1 else 0
            first_extra = li == 0 and extra is not None
            if impl >= 1 and li == n - 1 and li > 0 and o <= 16 and i % 4 == 0 and i <= 512 and self._tma_ok(inp, ld_in):
                # the narrow head: one bandwidth-bound pass instead of a padded tensor-core tile
                capi.check(capi.lib().go1_skinny_forward(self._p(inp), ld_in, W.data_ptr(), i, b.data_ptr(), capi.ptr(y), y.stride(0), M, o, i, capi.stream_ptr()), "skinny_forward")
                outs.append(y)
                continue
            K = K0 if first_extra else i
            Wm, ldw = W, i
            bf16 = li == 0 and impl == 2        # the history product: BF16 input (ActorCritic._model_input) and weights
            if li == 0 and (inp.dtype == torch.bfloat16) != bf16:
                raise capi.Go1Error("BF16 observation histories are the input of AC_Args.gemm_impl = 2 only")
            tc = impl >= 1 and self._tma_ok(inp, ld_in)
            if bf16:
                Wm, ldw = self._packed(li, K, torch.bfloat16)
            elif tc and (not self._tma_ok(W, i) or (li == 0 and K >= 1024 and i % 32 != 0)):
                # for the long first-layer rows the packed copy's aligned pitch alone is worth 30 % (misaligned 128-byte box rows cost an
                # extra L2 sector each)
                Wm, ldw = self._packed(li, K)
            ldy = y.stride(0)
            if first_extra and i - K0 > 4:      # wide trailing input: y = x W[:, :K0]^T + b, then y = act(y + extra W[:, K0:]^T)
                self._gemm(0, 1, M, o, K0, inp, ld_in, Wm, ldw, y, ldy, 1 if tc else 0, bias=b)
                capi.check(capi.lib().go1_mlp_extra_forward(capi.ptr(y), ldy, capi.ptr(extra), extra.stride(0), W.data_ptr() + 4 * K0, i, M, o, i - K0,
                                                            capi.act_arg(self.kind, act), capi.stream_ptr()), "go1_mlp_extra_forward")
            elif first_extra:   # y = act(x W[:, :K0]^T + extra W[:, K0:]^T + b): the (at most 4) trailing columns ride in the epilogue
                self._gemm(0, 1, M, o, K0, inp, ld_in, Wm, ldw, y, ldy, 1 if tc else 0, bias=b, act=act, extra=extra, w_extra=W.data_ptr() + 4 * K0, ld_w_extra=i)
            else:
                self._gemm(0, 1, M, o, K, inp, ld_in, Wm, ldw, y, ldy, 1 if tc else 0, bias=b, act=act)
            outs.append(y)
            inp, ld_in = y, y.stride(0)
        return outs

    def _tail_ok(self):
        """This net has a tail the fused kernel supports (hidden widths up to 256 behind the tail's input, a head of at most 12 columns)."""
        return self.owner.fuse_tail and self.tail_start is not None and self.specs[-1][2] <= 12

    def _tail_problem(self, x1, ldx1, M, tag):
        """(Go1TailProblem, [outputs of layers tail_start..]) of this net's tail for go1_mlp_tail_forward_grouped; x1 is the output of
        layer tail_start - 1."""
        ts, flat = self.tail_start, self.flat
        sp = self.specs[ts:]
        ptr = lambda off: flat.data_ptr() + 4 * off
        q = capi.Go1TailProblem()
        q.act_kind = self.kind
        (w2, b2, n2, k1) = sp[0]
        y2 = self._hbuf((tag, ts), M, n2)
        W2, q.ldw2 = self._weight_tma(ts)
        q.x, q.ldx, q.W2, q.b2, q.y2, q.ldy2 = self._p(x1), ldx1, self._p(W2), ptr(b2), y2.data_ptr(), y2.stride(0)
        if len(sp) == 3:
            (w3, b3, n3, _), (wh, bh, nh, _) = sp[1], sp[2]
            y3 = self._hbuf((tag, ts + 1), M, n3)
            out = self._buf((tag, ts + 2), M, nh)
            W3, q.ldw3 = self._weight_tma(ts + 1)
            q.W3, q.b3, q.y3, q.ldy3 = self._p(W3), ptr(b3), y3.data_ptr(), y3.stride(0)
            outs = [y2, y3, out]
        else:
            (wh, bh, nh, _) = sp[1]
            n3 = 0
            out = self._buf((tag, ts + 1), M, nh)
            q.W3, q.b3, q.y3, q.ldy3 = None, None, None, 0
            outs = [y2, out]
        q.Wh, q.bh, q.nh, q.out, q.ldout = ptr(wh), ptr(bh), nh, out.data_ptr(), out.stride(0)
        return q, outs, (k1, n2, n3)

    def _forward_tail(self, x1, ldx1, M, tag):
        """Layers tail_start.. (and the head) in ONE launch; returns their outputs in layer order."""
        q, outs, (k1, n2, n3) = self._tail_problem(x1, ldx1, M, tag)
        arr = (capi.Go1TailProblem * 1)(q)
        capi.check(capi.lib().go1_mlp_tail_forward_grouped(arr, 1, M, k1, n2, n3, capi.stream_ptr()), "go1_mlp_tail_forward")
        return outs

    def backward(self, x, ldx, K0, extra, outs, dout, M, impl, want_dextra=False, tag="a", dz1T=None, wgrads=None, y16=None):
        """dout: gradient w.r.t. the network output [M][out] (the last layer has no activation).  Adds the weight and bias gradients into
        the flat grad buffer, which the caller has zeroed (ActorCritic.backward_ppo / backward_adaptation): split-K partial tiles and the
        bias gradients reduced in epilogues are atomic sums.  dz of every hidden layer comes out of the dgrad GEMM already multiplied by
        the activation's derivative, computed from the saved layer output (fused epilogue).  dz1T: optional [o1][M] strided view; when
        given the first layer's dz is stored there transposed (K-major for the weight-gradient product) and that layer's wgrad, bias
        gradient and trailing-input weight gradients are left to the caller (ActorCritic._first_layer_wgrad: augmented rows of the
        transposed input).  A BF16 dz1T (AC_Args.gemm_impl = 2) receives the rounded dz; the bias, d(extra) and trailing-input reductions
        see the fp32 values.  wgrads: optional list that collects the tensor-core wgrads instead of launching them (ActorCritic._flush_wgrads
        launches equal shapes as grouped products).  Returns d(extra) [M][E] if requested.

        y16 (AC_Args.bf16_backward, M >= 64, with a BF16 dz1T): {layer: BF16 copy of outs[layer]} for the layers bf16_inputs lists
        (ActorCritic._convert_outputs).  Hidden-layer dz is then held in BF16: the head gradient is converted once the head's fp32 skinny
        kernels have read it (unless _skinny_head_dgrad), every dgrad behind it reads the BF16 copy of W (_packed) MN-major, multiplies by
        f'(y) from the fp32 saved output, reduces the bias gradient from the fp32 values and rounds the stored dz, and the weight
        gradients of the layers in y16 read the BF16 dz and layer input, both MN-major."""
        L, st = capi.lib(), capi.stream_ptr()
        n = len(self.specs)
        dz, dextra = dout, None
        bias_done = False      # this layer's bias gradient was reduced by the dgrad that made its dz, or is left to the caller
        extra_done = False     # likewise the first layer's trailing-input gradients
        dz1T16 = None          # a BF16 dz1T filled from the fp32 dz once go1_mlp_extra_backward has read that
        for li in range(n - 1, -1, -1):
            wo, bo, o, i = self.specs[li]
            W = self.flat[wo:wo + o * i]
            gW, gb = self.grad[wo:wo + o * i], self.grad[bo:bo + o]
            ldz = dz.stride(0)
            if li == 0:
                inp, ld_in, K = x, ldx, (K0 if extra is not None else i)
            else:
                inp, ld_in, K = outs[li - 1], outs[li - 1].stride(0), i
            wgrad_done = li == 0 and dz1T is not None       # made by the caller
            if y16 is None and impl >= 1 and M >= 64 and not self._tma_ok(dz, ldz) and (o > 16 or (li == 1 and dz1T is not None)):
                # a head gradient whose rows TMA cannot read ([M][1] values, [M][E] latents) where a tensor-core product must read it: the
                # wgrad and dgrad of a head wider than the skinny kernels take, or a one-hidden-layer net's dgrad that stores the first-layer
                # dz transposed
                dzp = self._buf((tag, "dhead"), M, o, capi.row_pitch(o))
                dzp.copy_(dz)
                dz, ldz = dzp, dzp.stride(0)
            # the narrow layers (heads): one bandwidth-bound pass instead of a padded GEMM tile; with y16 the layers listed there take
            # their wgrad on BF16 tensor cores whatever their width
            skinny = not wgrad_done and (o <= 16 if y16 is None else li - 1 not in y16)
            # ---- 1. bias gradient: reduced by the dgrad that made dz, by the skinny wgrad, or by go1_colsum
            if not bias_done:
                if skinny and K % 4 == 0 and self._tma_ok(inp, ld_in):
                    # weight AND bias gradient in one pass over the layer input
                    capi.check(L.go1_skinny_wgrad_ex(capi.ptr(dz), ldz, capi.ptr(inp), ld_in, gW.data_ptr(), i, gb.data_ptr(), M, o, K, 1, st), "skinny_wgrad")
                    wgrad_done = True
                else:
                    capi.check(L.go1_colsum(capi.ptr(dz), ldz, capi.ptr(gb), M, o, 0, st), "colsum")
            # ---- 2. wgrad: dW[o][K] = dz^T[o][M] inp[M][K]
            if skinny and not wgrad_done:
                capi.check(L.go1_skinny_wgrad(capi.ptr(dz), ldz, capi.ptr(inp), ld_in, gW.data_ptr(), i, M, o, K, 1, st), "skinny_wgrad")
                wgrad_done = True
            if y16 is not None and li == n - 1 and not self._skinny_head_dgrad(li, True):
                # the BF16 head gradient of the tensor-core products, once the fp32 kernels have read the fp32 one
                dz = self._buf16((tag, "dhead16"), M, o)
                capi.convert_bf16_segments([(dz, dout)])
                ldz = dz.stride(0)
            if not wgrad_done:      # both operands MN-major, read in place by the wgmma kernel; split-K partial tiles add into the zeroed gradient
                if y16 is not None:
                    inp, ld_in = y16[li - 1], y16[li - 1].stride(0)
                tc = impl >= 1 and M >= 64 and self._tma_ok(dz, ldz) and self._tma_ok(inp, ld_in)
                if tc and wgrads is not None:
                    wgrads.append((o, K, M, ldz, ld_in, i, dz, inp, gW))
                else:
                    self._gemm(1, 0, o, K, M, dz, ldz, inp, ld_in, gW, i, 1 if tc else 0, acc=1 if tc else 0)
            if li == 0:
                # trailing-input gradients the layer-2 dgrad epilogue did not reduce: d(extra) from dz in either layout, the weight
                # gradient only from a row-major dz (a transposed one is _first_layer_wgrad's augmented product)
                if extra is not None and not extra_done and (want_dextra or dz1T is None):
                    E = i - K0
                    if want_dextra:
                        dextra = self._buf((tag, "dextra"), M, E)
                    gwx = gW.data_ptr() + 4 * K0 if dz1T is None else None
                    capi.check(L.go1_mlp_extra_backward(capi.ptr(dz), ldz, 0 if dz1T is None else 1, capi.ptr(extra), extra.stride(0), W.data_ptr() + 4 * K0, i,
                                                        gwx, i, capi.ptr(dextra) if want_dextra else None, E, M, o, E, 0, st), "extra_backward")
                if dz1T16 is not None:
                    _to_bf16(dz, dz1T16)
                return dextra
            # ---- 3. dgrad (+ fused activation derivative): dz_prev[M][i] = (dz[M][o] W[o][i]) * f'(y_prev)
            pwo, pbo, po, pi = self.specs[li - 1]
            gb_prev, yprev = self.grad[pbo:pbo + po], outs[li - 1]
            to_T = li == 1 and dz1T is not None
            if to_T:
                dprev = dz1T
            elif y16 is not None:
                dprev = self._buf16((tag, "d16", li - 1), M, i)
            else:
                dprev = self._hbuf((tag, "d", li - 1), M, i)
            out16 = None
            if to_T and dz1T.dtype == torch.bfloat16:
                if extra is not None and pi - K0 > 4 and want_dextra:
                    # a wide trailing input's d(extra) is a pass over the stored dz (go1_mlp_extra_backward): fp32 first, the BF16 copy after it
                    dz1T16, dprev = dz1T, self._buf((tag, "dz1T32"), i, M, capi.row_pitch(M))
                else:
                    out16, dprev = dz1T, None
            ldp = dprev.stride(0) if dprev is not None else 0
            if impl >= 1 and self._tma_ok(dz, ldz) and M >= 64 and not self._skinny_head_dgrad(li, y16 is not None):
                # W read MN-major (in place, or its packed copy when its rows are not 16-byte multiples; with y16 its BF16 copy); the bias
                # gradient of layer li-1 (column sums of dprev) rides in the epilogue
                Wd, ldwd = self._weight_tma(li) if y16 is None else self._packed(li, i, torch.bfloat16)
                bx = None
                if li == 1 and extra is not None and 1 <= pi - K0 <= 4:
                    # dprev is the first layer's dz: d(extra), and the trailing-input weight gradient unless _first_layer_wgrad makes it,
                    # are reduced in this epilogue too
                    extra_done = True
                    if want_dextra:
                        dextra = self._buf((tag, "dextra"), M, pi - K0).zero_()
                    gwx = None if to_T else self.grad.data_ptr() + 4 * (pwo + K0)
                    if dextra is not None or gwx is not None:
                        bx = (extra, self.flat.data_ptr() + 4 * (pwo + K0), pi, gwx, pi, dextra)
                self._gemm(0, 0, M, i, o, dz, ldz, Wd, ldwd, dprev, ldp, 1, act=2, dact_y=yprev, colsum=None if to_T else gb_prev, bwd_extra=bx,
                           store_transposed=1 if to_T else 0, out16=out16)
                bias_done = True
            elif to_T:
                raise capi.Go1Error("transposed first-layer dz: the dgrad that produces it must be a tensor-core product")
            elif o <= 16:
                # the bias gradient of layer li-1 (column sums of dprev) is reduced in the same pass where the operands allow it
                bias_done = impl >= 1 and i % 4 == 0 and self._tma_ok(W, i) and self._tma_ok(dprev, ldp) and self._tma_ok(yprev, yprev.stride(0))
                if dprev.dtype == torch.bfloat16 and bias_done:
                    capi.check(L.go1_skinny_dgrad_act_bf16(capi.ptr(dz), ldz, capi.ptr(W), i, capi.ptr(yprev), yprev.stride(0), capi.ptr(dprev), ldp,
                                                           gb_prev.data_ptr(), M, o, i, self.kind, st), "skinny_dgrad_bf16")
                else:
                    d32 = self._hbuf((tag, "dskinny"), M, i) if dprev.dtype == torch.bfloat16 else dprev
                    capi.check(L.go1_skinny_dgrad_act(capi.ptr(dz), ldz, capi.ptr(W), i, capi.ptr(yprev), yprev.stride(0), capi.ptr(d32), d32.stride(0),
                                                      gb_prev.data_ptr() if bias_done else None, M, o, i, self.kind, st), "skinny_dgrad")
                    if d32 is not dprev:    # rows the vector kernel cannot read: the column sums and the BF16 copy of the fp32 dz
                        capi.check(L.go1_colsum(capi.ptr(d32), d32.stride(0), capi.ptr(gb_prev), M, i, 0, st), "colsum")
                        capi.convert_bf16_segments([(dprev, d32)])
                        bias_done = True
            else:
                self._gemm(0, 0, M, i, o, dz, ldz, W, i, dprev, ldp, 0, act=2, dact_y=yprev)
                bias_done = False
            dz = dprev if dprev is not None else out16

    def _skinny_head_dgrad(self, li, bf16):
        """With BF16 hidden-layer dz (AC_Args.bf16_backward) a head of at most 16 columns in a net of more than one hidden layer takes its
        dgrad on the skinny kernel, storing BF16: a K <= 16 tensor-core product pays for a whole 64-deep k-block and measured slower (35-45
        us per launch at M = 24576).  At gemm_impl 1 and 2 a head whose gradient rows TMA can read takes its dgrad on the tensor cores
        (the 12-wide actor head: 19 us there, 22 us on the skinny pass)."""
        n = len(self.specs)
        return bf16 and li == n - 1 and n > 2 and self.specs[li][2] <= 16

    def bf16_inputs(self, outs):
        """[(layer, width)] of the hidden outputs whose BF16 copies backward reads at AC_Args.bf16_backward: the input of every weight
        gradient behind the first layer that runs on BF16 (every hidden layer's, and the head's when it is wider than the skinny kernels'
        16 columns)."""
        n = len(self.specs)
        return [(li - 1, self.specs[li][3]) for li in range(1, n) if li < n - 1 or self.specs[li][2] > 16]


class ActorCritic(nn.Module):
    is_recurrent = False
    HEAD = 16          # floats reserved in front of the flat parameter / gradient buffers (see flatten())
    MAX_PRIVILEGED_OBS = 64     # widest trailing input the kernels take (go1_mlp_extra_forward / _backward); the eleven priv_observe_* groups give 45

    def __init__(self, num_obs, num_privileged_obs, num_obs_history, num_actions, **kwargs):
        if kwargs:
            print("ActorCritic.__init__ got unexpected arguments, which will be ignored: " + str([key for key in kwargs.keys()]))
        self.decoder = AC_Args.use_decoder
        super().__init__()
        activation = AC_Args.activation
        if activation not in capi.ACTIVATIONS:
            raise ValueError(f"AC_Args.activation = {activation!r}: expected one of {sorted(capi.ACTIVATIONS)}")
        self.act_kind = capi.ACTIVATIONS[activation]      # fixed per instance: it is baked into the captured CUDA graphs
        if not 1 <= num_privileged_obs <= self.MAX_PRIVILEGED_OBS:
            raise ValueError(f"num_privileged_obs = {num_privileged_obs}: the learner kernels take 1..{self.MAX_PRIVILEGED_OBS} privileged observations")
        self.num_obs_history, self.num_privileged_obs, self.num_actions = num_obs_history, num_privileged_obs, num_actions
        for field in ("adaptation_module_branch_hidden_dims", "actor_hidden_dims", "critic_hidden_dims"):
            dims = getattr(AC_Args, field)
            if len(dims) == 0 or not all(isinstance(d, numbers.Integral) and not isinstance(d, bool) and d > 0 for d in dims):
                raise ValueError(f"AC_Args.{field} = {dims!r}: expected a non-empty list of positive layer widths")
        self.adaptation_module = _mlp(num_obs_history, AC_Args.adaptation_module_branch_hidden_dims, num_privileged_obs, activation)
        self.actor_body = _mlp(num_privileged_obs + num_obs_history, AC_Args.actor_hidden_dims, num_actions, activation)
        self.critic_body = _mlp(num_privileged_obs + num_obs_history, AC_Args.critic_hidden_dims, 1, activation)
        self.std = nn.Parameter(AC_Args.init_noise_std * torch.ones(num_actions))
        self.distribution = None
        self._flat = self._grad = None
        self._mean = self._value = self._logp = None
        self._sample_counter = 0
        self._counter_dev = None
        self._packed_version = -1
        self.sample_seed = 0
        self.injected_eps = None      # parity tests inject the N(0,1) draws
        self.weights_version = 0      # bumped by every optimizer step / load: invalidates the packed first-layer weight copies
        self.update_streams = os.environ.get("GO1_UPDATE_STREAMS", "1") != "0"     # critic chain on a second stream during the update (measured -1.3 ms / iteration)
        self._side = None
        self.model_inputs = {}        # AC_Args.gemm_impl = 2: tag -> the BF16 history the last call with that tag read (see _model_input)
        self.fuse_tail = os.environ.get("GO1_FUSE_TAIL", "1") != "0"     # layers behind a first layer in one wgmma launch (go1_mlp_tail_forward_grouped: actor + critic bodies in one grid)
        # AC_Args.deterministic, or torch.use_deterministic_algorithms(True): every launch of this learner (and of its PPO and RolloutStorage)
        # sums its cross-CTA reductions in a fixed order (in_mode)
        self.deterministic = bool(AC_Args.deterministic) or torch.are_deterministic_algorithms_enabled()

    # ------------------------------------------------------------------ flat storage
    def _ordered_params(self):
        ps = []
        for seq in (self.adaptation_module, self.actor_body, self.critic_body):
            for m in seq:
                if isinstance(m, nn.Linear):
                    ps += [m.weight, m.bias]
        return ps + [self.std]

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._flat = None              # device / dtype changed: rebuild the flat views lazily
        return r

    def flatten(self):
        """(Re)build the flat parameter/gradient buffers and re-point every parameter at its slice."""
        if self._flat is not None:          # _apply() (device/dtype moves) resets it to None
            return
        ps = self._ordered_params()
        dev = ps[0].device
        # every tensor starts on a 16-byte boundary (zero padding in between: zero gradient, never moves) so that weights
        # are TMA-readable in place wherever their row length allows it
        # The first HEAD floats of both buffers belong to no parameter: in the gradient buffer they carry the loss scalars of the
        # minibatch (KL, surrogate / value loss, ... and the adaptation MSE pair), so that ONE all-reduce per optimizer step moves
        # gradients and scalars together; [HEAD : n_adapt_params] is the adaptation module (a prefix, so its own optimizer step
        # all-reduces the prefix [0 : n_adapt_params]: scalars + adaptation gradients).
        offsets, off = {}, self.HEAD
        for p in ps:
            off = (off + 3) // 4 * 4
            offsets[id(p)] = off
            off += p.numel()
        total = (off + 3) // 4 * 4
        flat = torch.zeros(total, device=dev, dtype=torch.float32)
        for p in ps:
            o, n = offsets[id(p)], p.numel()
            flat[o:o + n].copy_(p.data.reshape(-1))
            p.data = flat[o:o + n].view(p.shape)
        self._flat = flat
        self._packed_version = -1             # new _Net objects below: their packed weight copies do not exist yet
        self._grad = torch.zeros_like(flat)
        self.n_params = total                 # length of the flat buffers (HEAD + 3,054,619 parameters + alignment padding)
        self._nets = {}
        for name, seq in (("adapt", self.adaptation_module), ("actor", self.actor_body), ("critic", self.critic_body)):
            self._nets[name] = _Net(seq, self._flat, self._grad, offsets, self)
        self.n_adapt_params = (self._nets["adapt"].end + 3) // 4 * 4
        self.std_offset = offsets[id(self.std)]

    def ensure_packed(self):
        """Bring every packed weight copy (fused first-layer block, TMA-readable first-layer copies) up to date with the current weights.
        Called before a captured forward pass is replayed; a no-op while the weights are unchanged."""
        if self._flat is None or self._packed_version == self.weights_version:
            return
        for net in self._nets.values():
            net.refresh_packed()
        self._packed_version = self.weights_version

    @property
    def flat_params(self):
        self.flatten()
        return self._flat

    @property
    def flat_grads(self):
        self.flatten()
        return self._grad

    def load_state_dict(self, *a, **k):
        self.flatten()
        self.weights_version += 1
        return super().load_state_dict(*a, **k)

    # ------------------------------------------------------------------ reference API
    def reset(self, dones=None):
        pass

    def forward(self):
        raise NotImplementedError

    @property
    def action_mean(self):
        return self._mean

    @property
    def action_std(self):
        return self.std.detach().unsqueeze(0).expand_as(self._mean)

    @property
    def entropy(self):
        return (0.5 + 0.5 * torch.log(torch.tensor(2 * torch.pi)) + torch.log(self.std.detach())).sum().expand(self._mean.shape[0])

    def _impl(self):
        impl = int(AC_Args.gemm_impl)
        if impl not in (0, 1, 2):
            raise ValueError(f"AC_Args.gemm_impl = {AC_Args.gemm_impl!r}: expected 0 (fp32 CUDA cores), 1 (TF32 tensor cores) or 2 (BF16 history products)")
        if AC_Args.bf16_backward and impl != 2:
            raise ValueError(f"AC_Args.bf16_backward = True needs AC_Args.gemm_impl = 2 (it is {impl})")
        return impl

    def _bf16_backward(self):
        """AC_Args.bf16_backward, validated with the mode (_impl)."""
        return self._impl() == 2 and bool(AC_Args.bf16_backward)

    def _convert_outputs(self, named_outs, M, defer=False):
        """{net name: {layer: BF16 copy}} of the hidden outputs that the nets' BF16 weight gradients read (_Net.backward's y16), made together with the
        BF16 copies of the weights their dgrads read (stale after every optimizer step) by ONE go1_convert_bf16_segments launch per
        minibatch forward (two beyond 16 matrices; named_outs: [(net name, outs)]).  defer: only the weight copies are converted here;
        returns (copies, output pairs) and the caller converts the outputs (_backward_bodies: on the side stream, beside the dgrads)."""
        wpairs, ypairs, y16 = [], [], {}
        for name, outs in named_outs:
            net, y16[name] = self._nets[name], {}
            wpairs += net.packed16_pairs()
            for l, w in net.bf16_inputs(outs):
                y16[name][l] = net._buf16(("y16", name, l), M, w)
                ypairs.append((y16[name][l], outs[l]))
        if defer:
            if wpairs:
                capi.convert_bf16_segments(wpairs)
            return y16, ypairs
        if wpairs + ypairs:
            capi.convert_bf16_segments(wpairs + ypairs)
        return y16

    def _check_input(self, h):
        if not h.is_cuda:
            raise capi.Go1Error("ActorCritic runs on CUDA kernels only (no CPU fallback)")
        assert (h.dtype == torch.float32 or (h.dtype == torch.bfloat16 and self._impl() == 2)) and h.stride(1) == 1

    def _model_input(self, h, tag):
        """The observation history as the first layers read it: at AC_Args.gemm_impl = 2 in BF16 (rounded to nearest even, once per call, into a
        buffer kept per tag; a BF16 history -- RolloutStorage's minibatches -- is used as it is), else h itself.  The rollout's policy
        evaluation reads the copy that RolloutStorage then stores in its BF16 slab, so the update reads the identical operands."""
        self._check_input(h)
        if self._impl() != 2 or h.dtype == torch.bfloat16:
            return h
        M, K0 = h.shape[0], self.num_obs_history
        h16 = _to_bf16(h, self._nets["adapt"]._buf16((tag, "h16"), M, K0))
        self.model_inputs[tag] = h16
        return h16

    @in_mode
    def update_distribution(self, observation_history, tag="act"):
        self.flatten()
        h = self._model_input(observation_history, tag)
        M, K0 = h.shape[0], self.num_obs_history
        self._a_out = self._nets["adapt"].forward(h, h.stride(0), K0, None, M, self._impl(), tag)
        latent = self._a_out[-1]
        self._p_out = self._nets["actor"].forward(h, h.stride(0), K0, latent, M, self._impl(), tag)
        self._mean = self._p_out[-1]
        self._latent = latent

    @in_mode
    def forward_all(self, observation_history, privileged_observations, tag="act"):
        """update_distribution + evaluate in one pass.  With the tensor-core path the first layers of the three MLPs --
        which all read obs_history -- run as ONE product [M][256+512+512] = h Wcat^T: bias + activation (+ the critic's E <= 4
        privileged columns) ride in its epilogue for the adaptation/critic slices; the actor slice is finished
        (latent columns + activation) by go1_mlp_extra_forward once the adaptation module has produced the latent.  With E > 4 the
        epilogue finishes only the adaptation slice and go1_mlp_extra_forward also finishes the critic slice (priv columns)."""
        self.flatten()
        h, priv = self._model_input(observation_history, tag), privileged_observations.contiguous()
        M, K0, impl = h.shape[0], self.num_obs_history, self._impl()
        nets = self._nets
        na, npol, ncr = nets["adapt"], nets["actor"], nets["critic"]
        E = self.num_privileged_obs
        fused = impl >= 1 and _Net._tma_ok(h, h.stride(0)) and 1 <= E <= self.MAX_PRIVILEGED_OBS and \
            npol.specs[0][3] == K0 + E and ncr.specs[0][3] == K0 + E and na.specs[0][3] == K0
        if not fused:
            self.update_distribution(h, tag)
            return self._mean, self.evaluate(h, priv, tag)
        oa, op, oc = na.specs[0][2], npol.specs[0][2], ncr.specs[0][2]
        Pa, Pc = (oa + 3) // 4 * 4, (oc + 3) // 4 * 4     # the slices start on 16-byte boundaries (zero weight rows in between)
        NC = Pa + Pc + (op + 3) // 4 * 4
        flat = self._flat

        def w1(net):
            wo, bo, o, i = net.specs[0]
            return flat[wo:wo + o * i].view(o, i), flat[bo:bo + o]

        (Wa, ba), (Wp, bp), (Wc, bc) = w1(na), w1(npol), w1(ncr)

        KP = (K0 + 31) // 32 * 32      # 128-byte row pitch of the packed weights (aligned TMA box rows, see RolloutStorage.hist_pitch)

        def build_all(old):     # the packed block [adapt | critic | actor] x K0 (128-byte row pitch), its bias row and the trailing-input
            if old is None:     # weights of the leading (adaptation | critic) columns (zeros | Wc[:, K0:]): ONE launch for all seven pieces
                old = (_empty(NC, KP, device=flat.device)[:, :K0], _empty(1, NC, device=flat.device), _empty(Pa + Pc, E, device=flat.device).zero_())
                if NC != oa + oc + op:      # the padding rows between the slices stay zero
                    old[0].zero_()
                    old[1].zero_()
            W, b, x = old
            capi.copy_segments([(W[:oa], Wa), (W[Pa:Pa + oc], Wc[:, :K0]), (W[Pa + Pc:Pa + Pc + op], Wp[:, :K0]),
                                (b[:, :oa], ba.view(1, -1)), (b[:, Pa:Pa + oc], bc.view(1, -1)), (b[:, Pa + Pc:Pa + Pc + op], bp.view(1, -1)),
                                (x[Pa:Pa + oc], Wc[:, K0:])])
            return old

        Wcat, bcat, xcat = na._cached(("l1cat", K0, torch.float32), build_all)
        if impl == 2:           # the block in BF16 (rounded to nearest even; the padding rows stay zero), refreshed with the fp32 one
            Wcat = na._cached(("l1cat", K0, torch.bfloat16), lambda old: _to_bf16(
                na._cached(("l1cat", K0, torch.float32), build_all)[0],
                old if old is not None else _empty(NC, capi.bf16_pitch(K0), device=flat.device, dtype=torch.bfloat16)[:, :K0]))
        y = na._buf((tag, "y1cat"), M, NC)
        ya, yc, yp = y[:, :oa], y[:, Pa:Pa + oc], y[:, Pa + Pc:Pa + Pc + op]
        if E <= 4:
            na._gemm(0, 1, M, NC, K0, h, h.stride(0), Wcat, Wcat.stride(0), y, y.stride(0), bias=bcat, act=1,
                     extra=priv, w_extra=xcat.data_ptr(), ld_w_extra=E, lead_cols=Pa + Pc)
        else:       # wide privileged input: only the adaptation slice is finished in the epilogue; the critic slice gets priv here
            na._gemm(0, 1, M, NC, K0, h, h.stride(0), Wcat, Wcat.stride(0), y, y.stride(0), bias=bcat, act=1, lead_cols=Pa)
            capi.check(capi.lib().go1_mlp_extra_forward(capi.ptr(yc), yc.stride(0), capi.ptr(priv), priv.stride(0), Wc.data_ptr() + 4 * K0, K0 + E,
                                                        M, oc, E, capi.act_arg(self.act_kind, 1), capi.stream_ptr()), "go1_mlp_extra_forward")
        ts = npol.tail_start
        pair = npol._tail_ok() and ncr._tail_ok() and ts == ncr.tail_start and _Net._tma_ok(yp, yp.stride(0)) and _Net._tma_ok(yc, yc.stride(0)) and \
            [sp[2:] for sp in npol.specs[ts:-1]] == [sp[2:] for sp in ncr.specs[ts:-1]] and npol.specs[-1][2] + ncr.specs[-1][2] <= 16
        side = None if pair else self._side_stream(M)
        if side is not None:        # the critic's tail does not depend on the adaptation module: it runs beside adapt -> actor
            self._fork(side)
            with torch.cuda.stream(side):
                self._c_out = ncr.forward(h, h.stride(0), K0, priv, M, impl, tag, first_out=yc)
        self._a_out = na.forward(h, h.stride(0), K0, None, M, impl, tag, first_out=ya)
        latent = self._latent = self._a_out[-1]
        capi.check(capi.lib().go1_mlp_extra_forward(capi.ptr(yp), yp.stride(0), capi.ptr(latent), latent.stride(0), Wp.data_ptr() + 4 * K0, K0 + E,
                                                    M, op, E, capi.act_arg(self.act_kind, 1), capi.stream_ptr()), "go1_mlp_extra_forward")
        if pair:                    # the equal-shape tails of the actor and critic bodies in ONE grid (behind their layers before the tail)
            lead_p = npol.forward(h, h.stride(0), K0, latent, M, impl, tag, first_out=yp, defer_tail=True)
            lead_c = ncr.forward(h, h.stride(0), K0, priv, M, impl, tag, first_out=yc, defer_tail=True)
            qp, outs_p, shape = npol._tail_problem(lead_p[-1], lead_p[-1].stride(0), M, tag)
            qc, outs_c, _ = ncr._tail_problem(lead_c[-1], lead_c[-1].stride(0), M, tag)
            arr = (capi.Go1TailProblem * 2)(qp, qc)
            capi.check(capi.lib().go1_mlp_tail_forward_grouped(arr, 2, M, shape[0], shape[1], shape[2], capi.stream_ptr()), "go1_mlp_tail_forward")
            self._p_out, self._c_out = lead_p + outs_p, lead_c + outs_c
            self._mean, self._value = self._p_out[-1], self._c_out[-1]
            return self._mean, self._value
        self._p_out = npol.forward(h, h.stride(0), K0, latent, M, impl, tag, first_out=yp)
        self._mean = self._p_out[-1]
        if side is not None:
            self._join(side)
        else:
            self._c_out = ncr.forward(h, h.stride(0), K0, priv, M, impl, tag, first_out=yc)
        self._value = self._c_out[-1]
        return self._mean, self._value

    # ------------------------------------------------------------------ two-stream update (independent sub-chains side by side)
    def _side_stream(self, M):
        """A second stream for the critic's chain during the update (M = minibatch rows), or None: the mid-size products leave SMs
        idle at their ramp-up and tail (one 128 x 128 tile per CTA), which an independent chain on another stream fills."""
        if not self.update_streams or M < 4096 or torch.cuda.is_current_stream_capturing():
            return None
        if self._side is None:
            self._side = torch.cuda.Stream()
            self._ev_fork, self._ev_join = torch.cuda.Event(), torch.cuda.Event()
        return self._side

    def _fork(self, side):
        self._ev_fork.record()
        side.wait_event(self._ev_fork)

    def _join(self, side):
        self._ev_join.record(side)
        torch.cuda.current_stream().wait_event(self._ev_join)

    @in_mode
    def act_and_evaluate(self, observation_history, privileged_observations):
        """PPO.act's two calls (actor_critic.act + evaluate, ppo.py:67-68) on one fused forward pass."""
        self.forward_all(observation_history, privileged_observations, "act")
        return self._sample(observation_history), self._value

    # Normal-like accessors used through `self.distribution`
    @property
    def mean(self):
        return self._mean

    @property
    def stddev(self):
        return self.action_std

    @in_mode
    def act(self, observation_history, **kwargs):
        self.update_distribution(observation_history)
        return self._sample(observation_history)

    def _sample(self, observation_history):
        M = observation_history.shape[0]
        actions = torch.empty(M, self.num_actions, device=observation_history.device)
        self._logp = torch.empty(M, device=observation_history.device)
        eps = self.injected_eps
        if self._counter_dev is None or self._counter_dev.device != observation_history.device:
            with torch.inference_mode(False):
                self._counter_dev = torch.zeros(1, dtype=torch.int64, device=observation_history.device)
        capi.check(capi.lib().go1_ppo_sample_actions(capi.ptr(self._mean), self._mean.stride(0), capi.ptr(self.std.data),
                                                     capi.ptr(eps) if eps is not None else None, self.sample_seed, 0, capi.ptr(self._counter_dev),
                                                     capi.ptr(actions), capi.ptr(self._logp), M, self.num_actions, capi.stream_ptr()), "sample")
        self._last_actions = actions
        return actions

    def get_actions_log_prob(self, actions):
        last = getattr(self, "_last_actions", None)
        if last is not None and actions.data_ptr() == last.data_ptr() and actions.shape == last.shape:      # the sample kernel already produced it
            return self._logp
        d = actions - self._mean
        sd = self.std.detach()
        return (-(d * d) / (2 * sd * sd) - torch.log(sd) - 0.9189385332046727).sum(-1)

    def act_expert(self, ob, policy_info={}):
        return self.act_teacher(ob["obs_history"], ob["privileged_obs"])

    def act_inference(self, ob, policy_info={}):
        return self.act_student(ob["obs_history"], policy_info=policy_info)

    @in_mode
    def act_student(self, observation_history, policy_info={}):
        if observation_history.shape[0] == 0:
            return observation_history.new_zeros(0, self.num_actions)
        self.update_distribution(observation_history, tag="student")
        policy_info["latents"] = self._latent.detach().cpu().numpy()
        return self._mean

    @in_mode
    def act_teacher(self, observation_history, privileged_info, policy_info={}):
        if observation_history.shape[0] == 0:
            return observation_history.new_zeros(0, self.num_actions)
        self.flatten()
        h = self._model_input(observation_history, "teacher")
        out = self._nets["actor"].forward(h, h.stride(0), self.num_obs_history, privileged_info.contiguous(), h.shape[0], self._impl(), "teacher")
        policy_info["latents"] = privileged_info
        return out[-1]

    @in_mode
    def evaluate(self, observation_history, privileged_observations, tag="act", **kwargs):
        self.flatten()
        h = self._model_input(observation_history, tag)
        self._c_out = self._nets["critic"].forward(h, h.stride(0), self.num_obs_history, privileged_observations.contiguous(), h.shape[0], self._impl(), tag)
        self._value = self._c_out[-1]
        return self._value

    @in_mode
    def get_student_latent(self, observation_history):
        self.flatten()
        h = self._model_input(observation_history, "latent")
        return self._nets["adapt"].forward(h, h.stride(0), self.num_obs_history, None, h.shape[0], self._impl(), "latent")[-1]

    # ------------------------------------------------------------------ explicit backward passes (ppo.py:154-189)
    def _flush_wgrads(self, wgrads):
        """Launch the collected wgrads: equal shapes (same M, N, K and operand strides) as ONE grouped product (go1_gemm_grouped: up to
        four problems in one grid), the rest one by one.  All of them accumulate into the zeroed flat gradient buffer."""
        import ctypes as C
        groups = {}
        for it in wgrads:
            groups.setdefault(it[:6] + (it[6].dtype,), []).append(it)
        L, st = capi.lib(), capi.stream_ptr()
        for (o, K, M, ldz, ld_in, i, dt), items in groups.items():
            for k0 in range(0, len(items), 4):
                chunk = items[k0:k0 + 4]
                n = len(chunk)
                A = (C.c_void_p * n)(*[it[6].data_ptr() for it in chunk])
                B = (C.c_void_p * n)(*[it[7].data_ptr() for it in chunk])
                Cc = (C.c_void_p * n)(*[it[8].data_ptr() for it in chunk])
                if dt == torch.bfloat16:        # AC_Args.bf16_backward: BF16 dz and layer inputs, both MN-major
                    capi.check(L.go1_gemm_bf16_grouped(1, 0, o, K, M, n, A, ldz, B, ld_in, Cc, i, 1, st), "go1_gemm_bf16_grouped")
                else:
                    capi.check(L.go1_gemm_grouped(1, 0, o, K, M, n, A, ldz, B, ld_in, Cc, i, 1, st), "go1_gemm_grouped")

    def _first_layers_fusable(self, h, priv):
        """The first layers of the three nets can run their backward as one K-major product over hT (history_kmajor)."""
        nets, K0, E = self._nets, self.num_obs_history, self.num_privileged_obs
        return self._impl() >= 1 and h.shape[0] >= 64 and _Net._tma_ok(h, h.stride(0)) and 1 <= E <= self.MAX_PRIVILEGED_OBS and priv.shape[1] == E and \
            nets["actor"].specs[0][3] == K0 + E and nets["critic"].specs[0][3] == K0 + E and nets["adapt"].specs[0][3] == K0

    def _first_layer_wgrad(self, names, dz1T, hT, M, tag):
        """Weight gradients of the listed nets' first layers as ONE tensor-core product with both operands K-major,
        gcat[sum o][KA] = dz1T[sum o][M] hT[KA][M]^T (dz1T: the first-layer dz of the nets, stacked in `names` order, transposed by the
        dgrad epilogues that made it).  The augmented rows of hT make column K0 the bias gradient and columns K0 + 1.. the trailing-input
        weight gradients of the critic (priv) and the actor (latent); they are copied into the flat gradient buffer (overwriting).
        BF16 dz1T and hT (AC_Args.gemm_impl = 2): a BF16 product."""
        nets, K0, E = self._nets, self.num_obs_history, self.num_privileged_obs
        KA = hT.shape[0]
        KP = (KA + 31) // 32 * 32
        n0 = nets["adapt"]
        gcat = n0._buf((tag, "gWcat"), dz1T.shape[0], KP)
        n0._gemm(0, 1, dz1T.shape[0], KA, M, dz1T, dz1T.stride(0), hT, hT.stride(0), gcat, KP)
        row, pairs = 0, []
        for name in names:
            xcol = {"adapt": None, "actor": K0 + 1 + E, "critic": K0 + 1}[name]
            wo, bo, o, i = nets[name].specs[0]
            gW = self._grad[wo:wo + o * i].view(o, i)
            pairs.append((gW[:, :K0], gcat[row:row + o, :K0]))
            pairs.append((self._grad[bo:bo + o].view(o, 1), gcat[row:row + o, K0:K0 + 1]))
            if xcol is not None:
                pairs.append((gW[:, K0:K0 + E], gcat[row:row + o, xcol:xcol + E]))
            row += o
        capi.copy_segments(pairs)

    def _kmajor_buf(self, key, rows, M):
        """A [rows][M] K-major operand of the first layers' weight-gradient product: BF16 at AC_Args.gemm_impl = 2 (row pitch
        capi.bf16_pitch(M)), else fp32 (128-byte aligned rows)."""
        if self._impl() == 2:
            return self._nets["adapt"]._buf16(key, rows, M)
        return self._nets["adapt"]._buf(key, rows, M, (M + 31) // 32 * 32)

    @in_mode
    def backward_ppo(self, h, priv, dmean, dvalue, dstd, hT=None):
        """Gradients of the PPO loss into flat_grads[HEAD:] (overwrites; the loss scalars in the head are left alone). h/priv are the
        minibatch inputs of the forward pass just run with tag='train'; dmean [M,A], dvalue [M,1], dstd [A].
        hT: history_kmajor(h, priv) if the caller keeps one (RolloutStorage builds it once per update; BF16 at AC_Args.gemm_impl = 2,
        from the BF16 history); built here otherwise.  Its latent rows are written here."""
        M, K0 = h.shape[0], self.num_obs_history
        nets = self._nets
        self._grad[self.HEAD:].zero_()      # one fill; every kernel below adds into it (atomics in the epilogues and split-K products)
        if self._first_layers_fusable(h, priv):
            # the three first layers share their input: ONE transposed dz [o_a+o_p+o_c][M] (each net's layer-2 dgrad stores its
            # first-layer dz into its row slice) and ONE tensor-core wgrad with K-major operands (_first_layer_wgrad); at gemm_impl 2
            # both operands are BF16, the dz rounded by the dgrads that store it
            oa, op, oc = nets["adapt"].specs[0][2], nets["actor"].specs[0][2], nets["critic"].specs[0][2]
            E = self.num_privileged_obs
            if hT is None:
                hT = history_kmajor(self._model_input(h, "train"), priv, self._kmajor_buf(("train", "hT"), K0 + 1 + 2 * E, M))
            _transpose(self._latent, hT[K0 + 1 + E:])
            dz1 = nets["adapt"]._buf(("train", "dz1catT"), oa + op + oc, M, hT.stride(0), hT.dtype)
            named_outs = (("adapt", self._a_out), ("actor", self._p_out), ("critic", self._c_out))
            y16, ypairs = self._convert_outputs(named_outs, M, defer=True) if self._bf16_backward() else ({}, [])
            self._backward_bodies(h, priv, dmean, dvalue, dz1, oa, op, M, K0, y16, ypairs)
            self._first_layer_wgrad(("adapt", "actor", "critic"), dz1, hT, M, "train")
        else:
            impl = self._impl()
            if h.dtype == torch.bfloat16:      # (fewer than 64 rows: CUDA-core products, as at impl 1) the rounded history, exactly in fp32
                h = h.float()
            dlat = nets["actor"].backward(h, h.stride(0), K0, self._latent, self._p_out, dmean, M, impl, want_dextra=True, tag="train")
            nets["critic"].backward(h, h.stride(0), K0, priv, self._c_out, dvalue, M, impl, tag="train")
            nets["adapt"].backward(h, h.stride(0), K0, None, self._a_out, dlat, M, impl, tag="train")
        self._grad[self.std_offset:self.std_offset + self.num_actions].copy_(dstd)

    def _backward_bodies(self, h, priv, dmean, dvalue, dz1, oa, op, M, K0, y16, ypairs):
        """The three nets' backward passes down to their first-layer dz, stored transposed into the row slices of dz1 ([adapt | actor |
        critic] x M), and the tensor-core wgrads behind the first layers, launched as grouped products once all dz exist.  y16, ypairs:
        AC_Args.bf16_backward's {net name: BF16 output copies} and the conversions that make them (_convert_outputs(defer=True)), else
        empty.  Only the grouped wgrads read the copies, so the conversion runs first on the critic's side stream, beside the actor and
        adaptation dgrads (measured 2.2 ms of the 35 ms of kernel time of an update at 4096 envs, bandwidth-bound)."""
        nets, wgrads = self._nets, []

        def critic():
            nets["critic"].backward(h, h.stride(0), K0, priv, self._c_out, dvalue, M, 1, tag="train", dz1T=dz1[oa + op:], wgrads=wgrads,
                                    y16=y16.get("critic"))
        side = self._side_stream(M)
        if side is not None:    # critic chain beside actor -> adaptation chain
            self._fork(side)
            with torch.cuda.stream(side):
                if ypairs:
                    capi.convert_bf16_segments(ypairs)
                critic()
        elif ypairs:
            capi.convert_bf16_segments(ypairs)
        dlat = nets["actor"].backward(h, h.stride(0), K0, self._latent, self._p_out, dmean, M, 1, want_dextra=True, tag="train", dz1T=dz1[oa:oa + op],
                                      wgrads=wgrads, y16=y16.get("actor"))
        if side is None:
            critic()
        nets["adapt"].backward(h, h.stride(0), K0, None, self._a_out, dlat, M, 1, tag="train", dz1T=dz1[:oa], wgrads=wgrads, y16=y16.get("adapt"))
        if side is not None:
            self._join(side)
        self._flush_wgrads(wgrads)

    @in_mode
    def backward_adaptation(self, h, outs, dpred, hT=None):
        """Gradients of the adaptation module (overwrites its part of flat_grads, [HEAD:n_adapt_params]).  hT: history_kmajor(h, ..) if the
        caller keeps one (built here otherwise); the first layer's weight and bias gradients are the K-major product over its first K0 + 1 rows."""
        M, K0 = h.shape[0], self.num_obs_history
        net = self._nets["adapt"]
        self._grad[self.HEAD:self.n_adapt_params].zero_()
        if self._impl() >= 1 and M >= 64 and _Net._tma_ok(h, h.stride(0)) and net.specs[0][3] == K0:
            if hT is None:
                hT = history_kmajor(self._model_input(h, "adapt"), None, self._kmajor_buf(("adapt", "hT"), K0 + 1, M))
            dz1 = net._buf(("adapt", "dz1T"), net.specs[0][2], M, hT.stride(0), hT.dtype)
            y16 = self._convert_outputs((("adapt", outs),), M)["adapt"] if self._bf16_backward() else None
            net.backward(h, h.stride(0), K0, None, outs, dpred, M, 1, tag="adapt", dz1T=dz1, y16=y16)
            self._first_layer_wgrad(("adapt",), dz1, hT[:K0 + 1], M, "adapt")
        else:
            if h.dtype == torch.bfloat16:      # (fewer than 64 rows: CUDA-core products, as at impl 1) the rounded history, exactly in fp32
                h = h.float()
            net.backward(h, h.stride(0), K0, None, outs, dpred, M, self._impl(), tag="adapt")

    @in_mode
    def adaptation_forward(self, h):
        self.flatten()
        h = self._model_input(h, "adapt")
        return self._nets["adapt"].forward(h, h.stride(0), self.num_obs_history, None, h.shape[0], self._impl(), "adapt")


def get_activation(act_name):
    """The nn module of an AC_Args.activation name (reference actor_critic.py:149-166; an unknown name raises instead of returning None)."""
    table = {"elu": nn.ELU, "selu": nn.SELU, "relu": nn.ReLU, "crelu": nn.ReLU, "lrelu": nn.LeakyReLU, "tanh": nn.Tanh, "sigmoid": nn.Sigmoid}
    if act_name not in table:
        raise ValueError(f"invalid activation function {act_name!r}: expected one of {sorted(table)}")
    return table[act_name]()
