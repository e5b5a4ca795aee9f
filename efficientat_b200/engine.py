"""Execution engine: walks an MN module tree and launches the fused sm_90a kernels.

The module tree (efficientat_b200.models.mn) only *holds* parameters; this file is the forward /
backward pass.  Activations are NHWC ([B, F, T, C]) in fp32 or bf16; parameters are read in place
from the nn.Parameters (fp32) on every call, so optimiser steps and load_state_dict need no cache
invalidation.  Everything is enqueued on the current CUDA stream through the C ABI
(include/eat_b200.h); no torch compute op is on the path (torch supplies allocation only).

Data flow per InvertedResidual (reference models/mn/block_types.py:177-181):
  eval :  [pw-GEMM +BN+act] -> dw conv +BN+act (+SE squeeze) -> [SE MLP] -> pw-GEMM (SE gate on load)
          +BN (+residual)                       -- folded BatchNorm, 3-4 launches per block
  train:  conv kernels emit RAW outputs + per-channel batch statistics; the BatchNorm+activation
          of layer l is applied on the operand load of layer l+1, so no normalised tensor is written
          except the block output (BN3 + residual).
"""
import os

import torch

from ._lib import check_module_tensors, lib
from .models.common import head_dropout
from .models.mn.attention_pooling import MultiHeadAttentionPooling

ACT = {"none": 0, "relu": 1, "hswish": 2}
BN_EPS = 1e-3
BN_MOM = 0.01


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _stat_ptrs(stats):
    """(sum, sq) pointers of a statistics accumulator, or nulls when the forward runs on running statistics"""
    return (0, 0) if stats is None else (stats[0].data_ptr(), stats[1].data_ptr())


def _conv_out(n, k, s, d=1):
    return (n + 2 * ((k - 1) // 2) * d - d * (k - 1) - 1) // s + 1


class _Layer:
    """Plain record describing one block of the network for the launcher loops."""
    dil = 1             # depthwise dilation (MN's dilated tail: 2)


# one pass instead of two over the SE blocks' expanded tensors; EAT_SE_FUSED=0 restores the two-pass route
SE_FUSED_DEFAULT = "1"


DGRAD_BNRED_DEFAULT = "0"


# fp32 storage: the depthwise stage's backward below its BatchNorm (BN2 apply, weight and data gradient, expand-BatchNorm
# reduce) as one kernel, eat_dw_conv_bwd_fused; EAT_DW_BWD_FUSED=0 restores the four passes.  Routed (k, stride): at the
# mn10 B=256 shapes the fused kernel is 1.5-2.2x faster than the four passes for 3x3 and 5x5 stride 2, but 5x5 stride 1
# (blocks 5-6: 1.1x, blocks 14-15 at 4x32 pixels: 0.64x) loses in total, so those layers keep the passes
DW_BWD_FUSED_DEFAULT = "1"
DW_BWD_FUSED_SHAPES = ((3, 1), (3, 2), (5, 2))


# fp32 storage: the expand stage's backward below its BatchNorm (BN1 apply, weight and data gradient of the 1x1 conv) as one
# kernel, eat_pw_conv_bwd_fused, for the shapes its planner takes (cin <= 32, cexp <= 128: mn10 blocks 2-4, where it is
# 2.2-2.4x faster than the three passes at B=256); EAT_EXPAND_BWD_FUSED=0 restores the three passes
EXPAND_BWD_FUSED_DEFAULT = "1"


# fp32 storage: the project stage's backward below BN3 (BN3 apply, weight and data gradient of the 1x1 conv, BN2's reduce)
# as one kernel, eat_pw_proj_bwd_fused, for blocks without SE whose shapes its planner takes (cout <= 32, cexp <= 128:
# mn10 blocks 1-3); EAT_PROJ_BWD_FUSED=0 restores the separate passes
PROJ_BWD_FUSED_DEFAULT = "1"


# fp32 storage: the stem BatchNorm's backward apply on load in the stem weight gradient (eat_stem_wgrad with z), its only
# consumer, instead of a pass that writes dz0; EAT_STEM_BWD_FUSED=0 restores the apply pass
STEM_BWD_FUSED_DEFAULT = "1"


class _ZeroPool:
    """fp64 accumulators for BatchNorm statistics, carved from chunks that are zeroed with ONE fill each
    (a training step needs ~100 small zeroed buffers; one launch per buffer showed up as 250 tiny kernels)."""

    def __init__(self, chunk=1 << 16):
        self.chunk, self.buf, self.off = chunk, None, 0

    def take(self, rows, cols, dev):
        n = rows * cols
        if self.buf is None or self.off + n > self.buf.numel() or self.buf.device != dev:
            self.buf = torch.zeros(max(self.chunk, n), device=dev, dtype=torch.float64)
            self.off = 0
        v = self.buf[self.off:self.off + n].view(rows, cols)
        self.off += n
        return v


class _Fork:
    """Weight gradients are leaves of the backward graph: nothing downstream waits for them.  They are launched on a side
    stream so that they run beside the data-gradient / BatchNorm chain of the same block (in a captured CUDA graph the
    fork and join become graph edges): latency-bound tails of one kernel are filled by the other, and the two readers of
    a gradient tensor (weight- and data-gradient GEMM) sweep it together, so its second read tends to hit L2.
    Tensors the side stream reads are kept alive until `join`, after which the main stream may recycle them."""

    def __init__(self, device, enabled):
        self.enabled = enabled
        self.side = torch.cuda.Stream(device) if enabled else None
        self.keep = []

    def run(self, fn, *tensors):
        if not self.enabled:
            fn()
            return
        self.side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.side):
            fn()
        self.keep.extend(tensors)

    def join(self):
        if self.enabled:
            torch.cuda.current_stream().wait_stream(self.side)
            self.keep.clear()


class MNEngine:
    mha = None          # the MultiHeadAttentionPooling classifier, when the model has that head instead of 'mlp' (see _plan)
    # The saving forward and its backward in eval mode (input gradients): every BatchNorm runs on its running statistics,
    # whose backward is the batch-statistics formula with c1 = c2 = 0 (see _bn_bwd_coef)
    _bn_frozen = False
    _unwanted = frozenset()     # ids of gradient views no one asked for: the launches that only fill them are skipped

    def __init__(self, model):
        self.model = model
        self.precision = getattr(model, "precision", "fp32")
        if self.precision not in ("fp32", "bf16"):
            raise ValueError(f"precision must be 'fp32' or 'bf16', got {self.precision}")
        self.gemm_impl = os.environ.get("EAT_GEMM", "auto")     # auto | simt (exact-fp32 CUDA cores everywhere)
        self.tc_min_rows = 1024                                  # tiny GEMMs (classifier, SE) stay on CUDA cores
        self.pw_impl = "tc" if os.environ.get("EAT_PW_IMPL") == "tc" else "tma"
        # weight gradients on a side stream (see _Fork): both branches are HBM-bound, so it stays an opt-in experiment
        self.fork_wgrad = os.environ.get("EAT_FORK_WGRAD", "0") == "1"
        # SE blocks: squeeze-excitation reduce + BatchNorm-backward reduce of the depthwise output in one pass over the two
        # expanded tensors (eat_se_bn_bwd_reduce / _combine) instead of two (eat_se_bwd_reduce, eat_bn_bwd_reduce)
        self.se_fused = os.environ.get("EAT_SE_FUSED", SE_FUSED_DEFAULT) == "1"
        self.se_parts_per_sm = int(os.environ.get("EAT_SE_PARTS_PER_SM", "6"))
        # stride-2 blocks: the BatchNorm-backward reduce of the expand stage inside the depthwise data-gradient kernel that
        # produces its upstream gradient (eat_dw_conv_dgrad_bnred), fp32 storage
        self.dgrad_bnred = os.environ.get("EAT_DGRAD_BNRED", DGRAD_BNRED_DEFAULT) == "1"
        # fp32 storage: BN2-backward apply, depthwise weight and data gradient and the expand BatchNorm's reduce in one walk
        # (eat_dw_conv_bwd_fused); takes precedence over dgrad_bnred
        self.dw_bwd_fused = os.environ.get("EAT_DW_BWD_FUSED", DW_BWD_FUSED_DEFAULT) == "1"
        # fp32 storage: BN1-backward apply and both expand GEMMs in one pass (eat_pw_conv_bwd_fused)
        self.expand_bwd_fused = os.environ.get("EAT_EXPAND_BWD_FUSED", EXPAND_BWD_FUSED_DEFAULT) == "1"
        # fp32 storage, blocks without SE: BN3-backward apply, both project GEMMs and BN2's backward reduce in one pass
        # (eat_pw_proj_bwd_fused)
        self.proj_bwd_fused = os.environ.get("EAT_PROJ_BWD_FUSED", PROJ_BWD_FUSED_DEFAULT) == "1"
        # fp32 storage: the stem BatchNorm's backward apply inside the stem weight gradient (eat_stem_wgrad with z)
        self.stem_bwd_fused = os.environ.get("EAT_STEM_BWD_FUSED", STEM_BWD_FUSED_DEFAULT) == "1"
        self._pw_bwd_ok = {}
        self._fork = None
        self._se_scale = {}
        self._zero_pool = _ZeroPool()
        self._plan()

    # ------------------------------------------------------------------ structure
    def _plan(self):
        from .models.mn.block_types import ConcurrentSEBlock, ConvNormActivation, InvertedResidual
        feats = list(self.model.features)
        self.stem = feats[0]
        self.last = feats[-1]
        self.blocks = []
        for m in feats[1:-1]:
            assert isinstance(m, InvertedResidual)
            L = _Layer()
            subs = list(m.block)
            L.expand = L.se = None
            i = 0
            if len([s for s in subs if isinstance(s, ConvNormActivation)]) == 3:
                L.expand = subs[0]
                i = 1
            L.dw = subs[i]
            i += 1
            if isinstance(subs[i], ConcurrentSEBlock):
                L.se = subs[i].conc_se_layers[0]
                i += 1
            L.proj = subs[i]
            L.res = m.use_res_connect
            L.act = ACT["hswish"] if m.cnf.use_hs else ACT["relu"]
            L.k = m.cnf.kernel
            # a dilated depthwise conv runs at stride 1 (reference block_types.py:150); dilated layers go to the
            # eat_dw_conv_*_dil entry points, never to the fused depthwise backward or the dgrad + reduce kernel
            L.dil = m.cnf.dilation
            L.stride = 1 if L.dil > 1 else m.cnf.stride
            L.cin, L.cexp, L.cout = m.cnf.input_channels, m.cnf.expanded_channels, m.cnf.out_channels
            self.blocks.append(L)
        self.mha = self.model.classifier if isinstance(self.model.classifier, MultiHeadAttentionPooling) else None
        if self.mha is None:
            self.fc1 = self.model.classifier[2]
            self.fc2 = self.model.classifier[5]
        self.dropout_p = head_dropout(self.model)

    @property
    def tdtype(self):
        return torch.float32 if self.precision == "fp32" else torch.bfloat16

    @property
    def dcode(self):
        return 0 if self.precision == "fp32" else 1

    # ------------------------------------------------------------------ kernel wrappers
    def _gemm(self, a, w, out, M, N, K, in_sc=None, in_act=0, gate=None, rows_per_sample=1, sc=None, bias=None,
              act=0, res=None, stats=None, a_code=None, c_code=None, w_trans=False):
        """out[M,N] = epi(xf(a)[M,K] . w[N,K]^T).  in_sc: [2,K] (scale, shift) or None; sc: [2,N] or None;
        bias: [N] used as shift with scale None."""
        a_code = self.dcode if a_code is None else a_code
        c_code = self.dcode if c_code is None else c_code
        scale = _ptr(sc[0]) if sc is not None else 0
        shift = _ptr(sc[1]) if sc is not None else _ptr(bias)
        args = (a.data_ptr(), a_code, w.data_ptr(), 1 if w_trans else 0, out.data_ptr(), c_code, M, N, K,
                _ptr(in_sc[0]) if in_sc is not None else 0, _ptr(in_sc[1]) if in_sc is not None else 0, in_act,
                _ptr(gate), rows_per_sample, scale, shift, act, _ptr(res),
                _ptr(stats[0]) if stats is not None else 0, _ptr(stats[1]) if stats is not None else 0, _stream())
        L = lib()
        use_tc = (self.gemm_impl != "simt" and a_code == c_code and M >= self.tc_min_rows and K % 8 == 0
                  and N % 8 == 0 and act != 3 and in_act != 3)      # sigmoid epilogues (DyMN context nets) stay on CUDA cores
        if use_tc and a_code == 0 and self.pw_impl == "tma" and not (res is not None and act != 0):
            # fp32 storage: TMA-fed kernel; the weights are pre-split (bf16 hi|lo rows, BN scale folded, transposed for the
            # data gradient) once per launch into this scratch, so no CTA repeats that per tile
            ws = torch.empty(N * ((K + 31) // 32) * 128, device=w.device, dtype=torch.uint8)
            L.pw_tma_fwd(a.data_ptr(), w.data_ptr(), 1 if w_trans else 0, out.data_ptr(), M, N, K, args[9], args[10], in_act,
                         _ptr(gate), rows_per_sample, scale, shift, act, _ptr(res), args[18], args[19], ws.data_ptr(),
                         ws.numel(), _stream())
        elif use_tc:
            if w_trans:      # data gradient: feed W^T [N, K] as a K-major operand
                wt = torch.empty(N, K, device=w.device, dtype=torch.float32)
                L.transpose_f32(w.data_ptr(), wt.data_ptr(), K, N, _stream())
                args = (args[0], args[1], wt.data_ptr(), 0) + args[4:]
            L.pw_tc_fwd(*args)
        else:
            L.gemm_simt_fwd(*args)

    def _fold(self, bn, dev):
        c = bn.num_features
        sc = torch.empty(2, c, device=dev, dtype=torch.float32)
        lib().bn_fold(bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(),
                      bn.running_var.data_ptr(), bn.eps, sc[0].data_ptr(), sc[1].data_ptr(), c, _stream())
        return sc

    def _finalize(self, bn, stats, count, dev):
        """batch statistics -> (scale/shift [2,C], saved mean/invstd [2,C]); updates running buffers.
        On running statistics (_bn_frozen): the folded scale/shift and the running mean/invstd; no buffer changes."""
        if self._bn_frozen:
            return self._fold(bn, dev), torch.stack((bn.running_mean, torch.rsqrt(bn.running_var + bn.eps)))
        c = bn.num_features
        sc = torch.empty(2, c, device=dev, dtype=torch.float32)
        sv = torch.empty(2, c, device=dev, dtype=torch.float32)
        mom = bn.momentum if bn.momentum is not None else 0.1
        track = bn.track_running_stats and bn.running_mean is not None
        lib().bn_finalize(stats[0].data_ptr(), stats[1].data_ptr(), float(count), bn.weight.data_ptr(),
                          bn.bias.data_ptr(), bn.eps, mom, _ptr(bn.running_mean) if track else 0,
                          _ptr(bn.running_var) if track else 0, _ptr(bn.num_batches_tracked) if track else 0,
                          sc[0].data_ptr(), sc[1].data_ptr(), sv[0].data_ptr(), sv[1].data_ptr(), c, _stream())
        return sc, sv

    def _se_gate(self, se, pool, inv_count, B, C, dev, hidden=None):
        """Squeeze-excitation MLP (block_types.py:72-83) as two batched GEMMs: gate = sigmoid(W2 relu(W1 mean + b1) + b2)
        with mean = pool * inv_count folded into the first epilogue (scale = inv_count, shift = b1)."""
        S = se.fc1.out_features
        key = (S, float(inv_count), str(dev))
        sc = self._se_scale.get(key)
        if sc is None:
            sc = torch.full((S,), float(inv_count), device=dev, dtype=torch.float32)
            self._se_scale[key] = sc
        if hidden is None:
            hidden = torch.empty(B, S, device=dev, dtype=torch.float32)
        self._gemm(pool, se.fc1.weight, hidden, B, S, C, sc=(sc, se.fc1.bias), act=ACT["relu"], a_code=0, c_code=0)
        gate = torch.empty(B, C, device=dev, dtype=torch.float32)
        self._gemm(hidden, se.fc2.weight, gate, B, C, S, bias=se.fc2.bias, act=3, a_code=0, c_code=0)
        return gate, hidden

    def _dw_weights(self, conv, dev):
        c, k = conv.out_channels, conv.kernel_size[0]
        wt = torch.empty(k * k, c, device=dev, dtype=torch.float32)
        lib().dw_repack(conv.weight.data_ptr(), wt.data_ptr(), c, k, _stream())
        return wt

    # ------------------------------------------------------------------ forward
    def forward(self, x, return_fmaps=False, lengths=None):
        if not x.is_cuda:
            raise RuntimeError("efficientat_b200 models run on CUDA (sm_90a) only; got a CPU tensor")
        if x.dim() != 4 or x.shape[1] != 1:
            raise ValueError(f"expected input of shape [B, 1, F, T], got {tuple(x.shape)}")
        lengths = self._check_lengths(x, return_fmaps, lengths)
        check_module_tensors(self.model, x.device, type(self.model).__name__)
        self.dropout_p = head_dropout(self.model)                    # read at call time (it may be changed after engine())
        return self._dispatch(x, return_fmaps, lengths)

    def _check_lengths(self, x, return_fmaps, lengths):
        """`lengths` (clip b is x[b, :, :, :lengths[b]]) -> list of ints, or None.  The eval forward only: in training,
        BatchNorm's batch statistics would need the valid positions alone, which is a different semantics."""
        if lengths is None:
            return None
        from .packed import check_lengths
        if self.model.training:
            raise NotImplementedError("lengths: per-clip lengths are supported in eval() only")
        if x.requires_grad:
            raise NotImplementedError("lengths: per-clip lengths are not supported for an input that requires grad")
        if return_fmaps:
            raise NotImplementedError("lengths: return_fmaps is not supported with per-clip lengths")
        return check_lengths(lengths, x.shape[0], 1, x.shape[3])

    def _dispatch(self, x, return_fmaps, lengths=None):
        """train(): batch-statistics forward, with a graph when a parameter or the input requires grad.  eval(): the folded
        forward without a graph, unless the input requires grad: then the saving forward on running statistics."""
        from .autograd import mn_eval_grad_forward, mn_train_forward, mn_train_forward_fmaps
        grad_on = torch.is_grad_enabled()
        input_grad = grad_on and x.requires_grad
        needs_grad = input_grad or (grad_on and any(p.requires_grad for p in self.model.parameters()))
        with torch.cuda.device(x.device):                            # launches go to x's device, whatever is current
            if self.model.training:
                if return_fmaps:
                    logits, feat, fmaps = mn_train_forward_fmaps(self, x, needs_grad)
                    return self._squeeze(logits, feat) + (fmaps,)
                logits, feat = mn_train_forward(self, x, needs_grad)
                return self._squeeze(logits, feat) + (None,)
            if input_grad:
                if return_fmaps:
                    raise NotImplementedError("return_fmaps is not available when the input requires grad")
                logits, feat = mn_eval_grad_forward(self, x)
                return self._squeeze(logits, feat) + (None,)
            if lengths is not None:
                logits, feat, _ = self._forward_eval(x.detach(), lengths=lengths)
                return self._squeeze(logits, feat) + (None,)
            logits, feat, fmaps = self._forward_eval(x.detach(), return_fmaps)
            return self._squeeze(logits, feat) + (fmaps,)

    @staticmethod
    def _squeeze(logits, feat):
        # reference: `.squeeze()` then re-add the batch dim when B == 1 (mn/model.py:220-226); for B > 1
        # and num_classes > 1 the squeeze is a no-op, for B == 1 the unsqueeze restores [1, C].
        return logits, feat

    def _forward_eval(self, x, return_fmaps=False, lengths=None):
        L = lib()
        dev = x.device
        st = _stream()
        td, dc = self.tdtype, self.dcode
        x = x.float().contiguous()
        B, _, F, T = x.shape
        fmaps = [] if return_fmaps else None
        lens = None
        if lengths is not None:
            x, lens = self._lengths_input(x, lengths)

        def keep(t, f, tt, c):
            if fmaps is not None:   # NHWC storage -> logical NCHW view, like the reference's fmaps
                fmaps.append(t.view(B, f, tt, c).permute(0, 3, 1, 2))

        conv, bn = self.stem[0], self.stem[1]
        s0 = conv.stride[0]
        Fi, Ti = _conv_out(F, 3, s0), _conv_out(T, 3, s0)
        c0 = conv.out_channels
        a = torch.empty(B, Fi, Ti, c0, device=dev, dtype=td)
        sc = self._fold(bn, dev)
        L.stem_fwd(x.data_ptr(), conv.weight.data_ptr(), a.data_ptr(), dc, B, F, T, c0, s0, sc[0].data_ptr(),
                   sc[1].data_ptr(), ACT["hswish"], 0, 0, st)
        keep(a, Fi, Ti, c0)
        for i, blk in enumerate(self.blocks):
            a, Fi, Ti = self._ir_block_eval(blk, a, B, Fi, Ti, lens, i + 1)
            keep(a, Fi, Ti, blk.cout)
        logits, feat, z = self._head_eval(a, B, Fi, Ti, lens)
        keep(z, Fi, Ti, self.last[0].out_channels)
        return logits, feat, fmaps

    def _lengths_input(self, x, lengths):
        """-> (the stem's input with 0 past each clip's end, the call's StageLengths).  The stem reads its taps past a
        clip's end as that zero padding; the caller's tensor is never written."""
        from .packed import StageLengths
        B, _, F, T = x.shape
        lens = StageLengths(self, F, T, lengths, x.device)
        if lens.padded(0):
            x = x.clone()
            lib().time_pad_zero(x.data_ptr(), 0, B, F, T, 1, lens.ptr(0), _stream())
        return x, lens

    def _pad_zero(self, t, B, F, T, C, lens, s):
        """0 past each clip's end of stage s in the engine's own tensor t [B, F, T, C], before an op that mixes along time"""
        if lens.padded(s):
            lib().time_pad_zero(t.data_ptr(), self.dcode, B, F, T, C, lens.ptr(s), _stream())

    def _ir_block_eval(self, blk, a, B, Fi, Ti, lens=None, si=0):
        """one InvertedResidual with folded BatchNorm: 3-4 launches (reference block_types.py:177-181).
        lens: the call's StageLengths (clips of different lengths), with stage si the block's input; None otherwise."""
        L = lib()
        dev, st = a.device, _stream()
        td, dc = self.tdtype, self.dcode
        inp = a
        M = B * Fi * Ti
        if blk.expand is not None:
            e = torch.empty(B, Fi, Ti, blk.cexp, device=dev, dtype=td)
            self._gemm(inp, blk.expand[0].weight, e, M, blk.cexp, blk.cin, sc=self._fold(blk.expand[1], dev),
                       act=blk.act)
        else:
            e = inp
        if lens is not None:
            self._pad_zero(e, B, Fi, Ti, blk.cexp, lens, si)
        Fo, To = _conv_out(Fi, blk.k, blk.stride, blk.dil), _conv_out(Ti, blk.k, blk.stride, blk.dil)
        d = torch.empty(B, Fo, To, blk.cexp, device=dev, dtype=td)
        sc = self._fold(blk.dw[1], dev)
        # with lengths the squeeze is not fused into the depthwise epilogue: it would count the padded positions
        fused_pool = blk.se is not None and lens is None
        pool = torch.zeros(B, blk.cexp, device=dev, dtype=torch.float32) if fused_pool else None
        wt = self._dw_weights(blk.dw[0], dev)
        if blk.dil > 1:
            L.dw_conv_fwd_dil(e.data_ptr(), wt.data_ptr(), d.data_ptr(), dc, B, Fi, Ti, blk.cexp, blk.k, blk.stride, blk.dil,
                              0, 0, 0, sc[0].data_ptr(), sc[1].data_ptr(), blk.act, _ptr(pool), 0, 0, st)
        else:
            L.dw_conv_fwd(e.data_ptr(), wt.data_ptr(), d.data_ptr(), dc, B, Fi, Ti, blk.cexp, blk.k, blk.stride, 0, 0, 0,
                          sc[0].data_ptr(), sc[1].data_ptr(), blk.act, _ptr(pool), 0, 0, st)
        gate = None
        if blk.se is not None and lens is not None:
            pool = torch.empty(B, blk.cexp, device=dev, dtype=torch.float32)
            L.mean_len(d.data_ptr(), dc, pool.data_ptr(), B, Fo, To, blk.cexp, lens.ptr(si + 1), st)
            gate, _ = self._se_gate(blk.se, pool, 1.0, B, blk.cexp, dev)
        elif blk.se is not None:
            gate, _ = self._se_gate(blk.se, pool, 1.0 / (Fo * To), B, blk.cexp, dev)
        Mo = B * Fo * To
        o = torch.empty(B, Fo, To, blk.cout, device=dev, dtype=td)
        self._gemm(d, blk.proj[0].weight, o, Mo, blk.cout, blk.cexp, gate=gate, rows_per_sample=Fo * To,
                   sc=self._fold(blk.proj[1], dev), act=0, res=inp if blk.res else None)
        return o, Fo, To

    def _head_eval(self, a, B, Fi, Ti, lens=None):
        """last 1x1 conv + BN + Hardswish, global average pool, classifier MLP (mn/model.py:160-166,187-194,220-221).
        lens: the call's StageLengths; the pools then run over each clip's valid frames."""
        L = lib()
        dev, st = a.device, _stream()
        td, dc = self.tdtype, self.dcode
        conv, bn = self.last[0], self.last[1]
        cl = conv.out_channels
        M = B * Fi * Ti
        z = torch.empty(B, Fi, Ti, cl, device=dev, dtype=td)
        self._gemm(a, conv.weight, z, M, cl, conv.in_channels, sc=self._fold(bn, dev), act=ACT["hswish"])
        t_valid = None if lens is None else lens.ptr(lens.n - 1)
        if self.mha is not None:
            logits, feat, _ = self._mha_fwd(z, None, B, Fi, Ti, save=False, t_valid=t_valid)
            return logits, feat, z
        if t_valid is not None:
            feat = torch.empty(B, cl, device=dev, dtype=torch.float32)
            L.mean_len(z.data_ptr(), dc, feat.data_ptr(), B, Fi, Ti, cl, t_valid, st)
        else:
            feat = torch.zeros(B, cl, device=dev, dtype=torch.float32)
            L.bn_act_pool(z.data_ptr(), 0, 0, 0, feat.data_ptr(), 1.0 / (Fi * Ti), dc, B, Fi * Ti, cl, st)
        h = torch.empty(B, self.fc1.out_features, device=dev, dtype=torch.float32)
        self._gemm(feat, self.fc1.weight, h, B, self.fc1.out_features, cl, bias=self.fc1.bias, act=ACT["hswish"],
                   a_code=0, c_code=0)
        logits = torch.empty(B, self.fc2.out_features, device=dev, dtype=torch.float32)
        self._gemm(h, self.fc2.weight, logits, B, self.fc2.out_features, self.fc1.out_features, bias=self.fc2.bias,
                   a_code=0, c_code=0)
        return logits, feat, z

    # ------------------------------------------------------------------ training forward
    def _new_stats(self, c, dev):
        return None if self._bn_frozen else self._zero_pool.take(2, c, dev)

    def _forward_train(self, x, dropout_mask=None, frozen=False, fmaps=False):
        """Batch-statistics forward.  Returns (logits, feat, saved) where `saved` holds the raw conv outputs
        and BatchNorm statistics needed by `_backward` (activations are recomputed from them).
        frozen: the same forward with every BatchNorm on its running statistics (no buffer update) and no dropout --
        eval mode's forward when the input's gradient is wanted.
        fmaps: saved["fmaps"] holds the 17 feature maps (stem, blocks, last conv) as NHWC tensors [B, F, T, C]."""
        self._bn_frozen = frozen
        try:
            return self._forward_train_impl(x, dropout_mask, fmaps)
        finally:
            self._bn_frozen = False

    def _forward_train_impl(self, x, dropout_mask, fmaps=False):
        L = lib()
        dev = x.device
        st = _stream()
        td, dc = self.tdtype, self.dcode
        x = x.detach().float().contiguous()
        B, _, F, T = x.shape
        HS = ACT["hswish"]
        S = {"x": x, "B": B, "F": F, "T": T, "blocks": [], "frozen": self._bn_frozen, "fmaps": [] if fmaps else None}
        self._zero_pool = _ZeroPool()

        conv, bn = self.stem[0], self.stem[1]
        s0 = conv.stride[0]
        Fi, Ti = _conv_out(F, 3, s0), _conv_out(T, 3, s0)
        c0 = conv.out_channels
        z0 = torch.empty(B, Fi, Ti, c0, device=dev, dtype=td)
        stt = self._new_stats(c0, dev)
        L.stem_fwd(x.data_ptr(), conv.weight.data_ptr(), z0.data_ptr(), dc, B, F, T, c0, s0, 0, 0, 0, *_stat_ptrs(stt), st)
        sc0, sv0 = self._finalize(bn, stt, B * Fi * Ti, dev)
        a = torch.empty_like(z0)
        L.bn_apply(z0.data_ptr(), sc0[0].data_ptr(), sc0[1].data_ptr(), HS, 0, a.data_ptr(), dc, B * Fi * Ti, c0, st)
        S["stem"] = dict(z=z0, sc=sc0, sv=sv0, Fo=Fi, To=Ti)
        # the stem and block outputs are materialised anyway (each is the next stage's input): the maps are these tensors
        keep = S["fmaps"].append if fmaps else (lambda t: None)
        keep(a)
        for blk in self.blocks:
            a, Fi, Ti, R = self._block_train_fwd(blk, a, B, Fi, Ti)
            S["blocks"].append(R)
            keep(a)
        logits, feat = self._head_train_fwd(a, B, Fi, Ti, S, dropout_mask)
        return logits, feat, S

    def _block_train_fwd(self, blk, a, B, Fi, Ti):
        return self._ir_block_train_fwd(blk, a, B, Fi, Ti)

    def _ir_block_train_fwd(self, blk, a, B, Fi, Ti):
        L = lib()
        dev, st = a.device, _stream()
        td, dc = self.tdtype, self.dcode
        R = {"inp": a, "Fi": Fi, "Ti": Ti}
        inp = a
        M = B * Fi * Ti
        if blk.expand is not None:
            z1 = torch.empty(B, Fi, Ti, blk.cexp, device=dev, dtype=td)
            stt = self._new_stats(blk.cexp, dev)
            self._gemm(inp, blk.expand[0].weight, z1, M, blk.cexp, blk.cin, stats=stt)
            sc1, sv1 = self._finalize(blk.expand[1], stt, M, dev)
            R.update(z1=z1, sc1=sc1, sv1=sv1)
            dw_in, dw_sc = z1, sc1
        else:
            dw_in, dw_sc = inp, None
        Fo, To = _conv_out(Fi, blk.k, blk.stride, blk.dil), _conv_out(Ti, blk.k, blk.stride, blk.dil)
        Mo = B * Fo * To
        z2 = torch.empty(B, Fo, To, blk.cexp, device=dev, dtype=td)
        stt = self._new_stats(blk.cexp, dev)
        wt = self._dw_weights(blk.dw[0], dev)
        xf = (_ptr(dw_sc[0]) if dw_sc is not None else 0, _ptr(dw_sc[1]) if dw_sc is not None else 0,
              blk.act if dw_sc is not None else 0)
        if blk.dil > 1:
            L.dw_conv_fwd_dil(dw_in.data_ptr(), wt.data_ptr(), z2.data_ptr(), dc, B, Fi, Ti, blk.cexp, blk.k, blk.stride,
                              blk.dil, *xf, 0, 0, 0, 0, *_stat_ptrs(stt), st)
        else:
            L.dw_conv_fwd(dw_in.data_ptr(), wt.data_ptr(), z2.data_ptr(), dc, B, Fi, Ti, blk.cexp, blk.k, blk.stride, *xf,
                          0, 0, 0, 0, *_stat_ptrs(stt), st)
        sc2, sv2 = self._finalize(blk.dw[1], stt, Mo, dev)
        R.update(z2=z2, sc2=sc2, sv2=sv2, wt=wt, Fo=Fo, To=To)
        gate = None
        if blk.se is not None:
            Sq = blk.se.fc1.out_features
            pool = torch.zeros(B, blk.cexp, device=dev, dtype=torch.float32)
            L.bn_act_pool(z2.data_ptr(), sc2[0].data_ptr(), sc2[1].data_ptr(), blk.act, pool.data_ptr(),
                          1.0 / (Fo * To), dc, B, Fo * To, blk.cexp, st)
            gate, hidden = self._se_gate(blk.se, pool, 1.0, B, blk.cexp, dev)
            R.update(mean=pool, gate=gate, hidden=hidden)
        z3 = torch.empty(B, Fo, To, blk.cout, device=dev, dtype=td)
        stt = self._new_stats(blk.cout, dev)
        self._gemm(z2, blk.proj[0].weight, z3, Mo, blk.cout, blk.cexp, in_sc=sc2, in_act=blk.act, gate=gate,
                   rows_per_sample=Fo * To, stats=stt)
        sc3, sv3 = self._finalize(blk.proj[1], stt, Mo, dev)
        a = torch.empty(B, Fo, To, blk.cout, device=dev, dtype=td)
        L.bn_apply(z3.data_ptr(), sc3[0].data_ptr(), sc3[1].data_ptr(), 0, _ptr(inp) if blk.res else 0,
                   a.data_ptr(), dc, Mo, blk.cout, st)
        R.update(z3=z3, sc3=sc3, sv3=sv3)
        return a, Fo, To, R

    def _head_train_fwd(self, a, B, Fi, Ti, S, dropout_mask):
        L = lib()
        dev, st = a.device, _stream()
        td, dc = self.tdtype, self.dcode
        HS = ACT["hswish"]
        conv, bn = self.last[0], self.last[1]
        cl = conv.out_channels
        M = B * Fi * Ti
        zl = torch.empty(B, Fi, Ti, cl, device=dev, dtype=td)
        stt = self._new_stats(cl, dev)
        self._gemm(a, conv.weight, zl, M, cl, conv.in_channels, stats=stt)
        scl, svl = self._finalize(bn, stt, M, dev)
        S["last"] = dict(inp=a, z=zl, sc=scl, sv=svl, Fi=Fi, Ti=Ti)
        if S["fmaps"] is not None:
            # the heads apply the last BatchNorm + Hardswish on load and never store them: one pass when the map is asked for
            al = torch.empty_like(zl)
            L.bn_apply(zl.data_ptr(), scl[0].data_ptr(), scl[1].data_ptr(), HS, 0, al.data_ptr(), dc, M, cl, st)
            S["fmaps"].append(al)
        if self.mha is not None:
            logits, feat, S["head"] = self._mha_fwd(zl, scl, B, Fi, Ti, save=True)
            return logits, feat
        feat = torch.zeros(B, cl, device=dev, dtype=torch.float32)
        L.bn_act_pool(zl.data_ptr(), scl[0].data_ptr(), scl[1].data_ptr(), HS, feat.data_ptr(), 1.0 / (Fi * Ti), dc, B,
                      Fi * Ti, cl, st)
        # classifier: Linear -> Hardswish -> Dropout -> Linear.  The Hardswish and the dropout mask are applied on
        # the operand load of the second GEMM (in_act + per-row gate), so only the pre-activation is stored.
        n1 = self.fc1.out_features
        h_pre = torch.empty(B, n1, device=dev, dtype=torch.float32)
        self._gemm(feat, self.fc1.weight, h_pre, B, n1, cl, bias=self.fc1.bias, a_code=0, c_code=0)
        p = 0.0 if self._bn_frozen else self.dropout_p
        if dropout_mask is None and p > 0:
            dropout_mask = torch.empty(B, n1, device=dev, dtype=torch.float32).bernoulli_(1.0 - p).div_(1.0 - p)
        ident = self._ident(n1, dev)
        logits = torch.empty(B, self.fc2.out_features, device=dev, dtype=torch.float32)
        self._gemm(h_pre, self.fc2.weight, logits, B, self.fc2.out_features, n1, in_sc=ident, in_act=HS,
                   gate=dropout_mask, rows_per_sample=1, bias=self.fc2.bias, a_code=0, c_code=0)
        S["head"] = dict(feat=feat, h_pre=h_pre, mask=dropout_mask, ident=ident)
        return logits, feat

    def _mha_fwd(self, z, sc, B, Fi, Ti, save, t_valid=None):
        """multi-head attention pooling head (attention_pooling.py:40-56) on the last conv's output z [B, F, T, C]:
        frequency mean (with the BatchNorm + Hardswish applied on load when sc is given, i.e. z is raw), projection GEMM,
        attention pooling.  -> (logits [B, K], features [B, C], tensors the backward needs or None).
        t_valid: device row of each clip's valid frames (eval with lengths): features and the attention sums stop there."""
        L = lib()
        dev, st = z.device, _stream()
        head = self.mha
        C, H, K = z.shape[3], head.num_heads, head.out_dim
        m = torch.empty(B, Ti, C, device=dev, dtype=torch.float32)
        feat = torch.empty(B, C, device=dev, dtype=torch.float32)
        L.freq_pool(z.data_ptr(), self.dcode, _ptr(sc[0]) if sc is not None else 0, _ptr(sc[1]) if sc is not None else 0,
                    ACT["hswish"] if sc is not None else 0, m.data_ptr(), feat.data_ptr() if t_valid is None else 0, B, Fi,
                    Ti, C, st)
        if t_valid is not None:
            L.mean_len(z.data_ptr(), self.dcode, feat.data_ptr(), B, Fi, Ti, C, t_valid, st)
        P = torch.empty(B * Ti, 2 * H * K, device=dev, dtype=torch.float32)
        proj = head.subspace_proj
        self._gemm(m, proj.weight, P, B * Ti, 2 * H * K, C, bias=proj.bias, a_code=0, c_code=0)
        logits = torch.empty(B, K, device=dev, dtype=torch.float32)
        if t_valid is not None:
            L.att_pool_fwd_len(P.data_ptr(), head.head_weight.data_ptr(), head.epsilon, logits.data_ptr(), B, Ti, H, K,
                               t_valid, st)
            return logits, feat, None
        sa = r = None
        if save:
            sa = torch.empty(B, H, K, device=dev, dtype=torch.float32)
            r = torch.empty_like(sa)
        L.att_pool_fwd(P.data_ptr(), head.head_weight.data_ptr(), head.epsilon, logits.data_ptr(), _ptr(sa), _ptr(r), B, Ti,
                       H, K, st)
        return logits, feat, (dict(feat=feat, m=m, P=P, sa=sa, r=r) if save else None)

    def _mha_bwd(self, S, dlogits, G, fork):
        """backward of _mha_fwd down to the gradient at the last conv's BatchNorm + Hardswish output [B, F, T, C]
        (storage dtype); parameter gradients into G"""
        L = lib()
        dev, st = dlogits.device, _stream()
        head, Hd, Ls = self.mha, S["head"], S["last"]
        B, Fi, Ti = S["B"], Ls["Fi"], Ls["Ti"]
        C, H, K = Ls["z"].shape[3], head.num_heads, head.out_dim
        proj = head.subspace_proj
        dP = Hd["P"]                    # overwritten in place: P is not needed after this launch
        L.att_pool_bwd(dlogits.data_ptr(), Hd["P"].data_ptr(), dP.data_ptr(), head.head_weight.data_ptr(),
                       Hd["sa"].data_ptr(), Hd["r"].data_ptr(), head.epsilon, G[head.head_weight].data_ptr(),
                       G[proj.bias].data_ptr(), B, Ti, H, K, st)
        fork.run(lambda: self._wgrad(dP, Hd["m"], G[proj.weight], None, B * Ti, 2 * H * K, C, g_code=0, a_code=0), dP)
        dm = torch.empty(B, Ti, C, device=dev, dtype=torch.float32)
        self._gemm(dP, proj.weight, dm, B * Ti, C, 2 * H * K, a_code=0, c_code=0, w_trans=True)
        gA = torch.empty_like(Ls["z"])
        L.freq_pool_bwd(dm.data_ptr(), 1.0 / Fi, gA.data_ptr(), self.dcode, B, Fi, Ti, C, st)
        return gA

    def _ident(self, n, dev):
        t = torch.empty(2, n, device=dev, dtype=torch.float32)
        t[0].fill_(1.0)
        t[1].zero_()
        return t

    # ------------------------------------------------------------------ backward
    def _block_modules(self):
        return list(self.model.features)[1:-1]

    def param_list(self):
        return [p for p in self.model.parameters()]

    def _wanted(self, grad):
        """the gradient view, or None when its parameter's gradient was not asked for"""
        return None if grad is None or id(grad) in self._unwanted else grad

    def _wgrad(self, g, a, dW, db, M, N, K, in_sc=None, in_act=0, gate=None, rows_per_sample=1, g_code=None,
               a_code=None):
        if self._wanted(dW) is None and self._wanted(db) is None:
            return
        g_code = self.dcode if g_code is None else g_code
        a_code = self.dcode if a_code is None else a_code
        args = (g.data_ptr(), g_code, a.data_ptr(), a_code, dW.data_ptr(), _ptr(db), M, N, K,
                _ptr(in_sc[0]) if in_sc is not None else 0, _ptr(in_sc[1]) if in_sc is not None else 0,
                in_act, _ptr(gate), rows_per_sample, _stream())
        use_tc = (self.gemm_impl != "simt" and db is None and g_code == a_code and M >= self.tc_min_rows
                  and K % 8 == 0 and N % 8 == 0)
        if use_tc:
            lib().pw_tc_wgrad(*args)
        else:
            lib().gemm_simt_wgrad(*args)

    def _bn_bwd_coef(self, gA, gate, dpool, z, sc, sv, act, B, P, C, dgamma, dbeta, dev, code, sums):
        """BatchNorm-backward reduce (unless `sums` holds it already) + finalize -> the apply pass's (c1, c2) [2, C]"""
        L = lib()
        st = _stream()
        count = float(B * P)
        if self._bn_frozen:
            # running statistics do not depend on the batch: c1 = c2 = 0, and the apply is dz = scale * dy * act'.  The
            # reduce (against the running mean and invstd) only serves gamma's and beta's gradients; an infinite count
            # makes eat_bn_bwd_finalize's c1 = s1 / count and c2 = s2 / count zero
            dgamma, dbeta = self._wanted(dgamma), self._wanted(dbeta)
            if dgamma is None and dbeta is None:
                return torch.zeros(2, C, device=dev, dtype=torch.float32)
            count = float("inf")
        if sums is None:
            s = self._zero_pool.take(2, C, dev)
            L.bn_bwd_reduce(_ptr(gA), _ptr(gate), _ptr(dpool), z.data_ptr(), sc[0].data_ptr(), sc[1].data_ptr(),
                            sv[0].data_ptr(), sv[1].data_ptr(), act, code, B, P, C, s[0].data_ptr(), s[1].data_ptr(), st)
        else:
            s = sums
        coef = torch.empty(2, C, device=dev, dtype=torch.float32)
        L.bn_bwd_finalize(s[0].data_ptr(), s[1].data_ptr(), count, _ptr(dgamma), _ptr(dbeta),
                          coef[0].data_ptr(), coef[1].data_ptr(), C, st)
        return coef

    def _bn_bwd(self, gA, gate, dpool, z, sc, sv, act, B, P, C, dgamma, dbeta, dev, code=None, sums=None):
        """two-pass BatchNorm(+activation) backward -> dz (same dtype/shape as z).  `sums`: the (s1, s2) accumulators when
        the reduce pass already happened elsewhere (SE blocks: eat_se_bn_bwd_reduce + eat_se_bn_bwd_combine)."""
        code = self.dcode if code is None else code
        coef = self._bn_bwd_coef(gA, gate, dpool, z, sc, sv, act, B, P, C, dgamma, dbeta, dev, code, sums)
        return self._bn_bwd_apply(gA, gate, dpool, z, sc, sv, act, coef, B, P, C, code)

    def _bn_bwd_apply(self, gA, gate, dpool, z, sc, sv, act, coef, B, P, C, code):
        dz = torch.empty_like(z)
        lib().bn_bwd_apply(_ptr(gA), _ptr(gate), _ptr(dpool), z.data_ptr(), sc[0].data_ptr(), sc[1].data_ptr(),
                           sv[0].data_ptr(), sv[1].data_ptr(), act, coef[0].data_ptr(), coef[1].data_ptr(), dz.data_ptr(),
                           code, B, P, C, _stream())
        return dz

    def _block_bwd(self, blk, R, dy, G, B):
        return self._ir_block_bwd(blk, R, dy, G, B)

    def _ir_block_bwd(self, blk, R, dy, G, B):
        """backward of one InvertedResidual; returns the gradient w.r.t. the block input"""
        L = lib()
        st = _stream()
        dev = dy.device
        td, dc = self.tdtype, self.dcode
        Fi, Ti, Fo, To = R["Fi"], R["Ti"], R["Fo"], R["To"]
        Pi, Po = Fi * Ti, Fo * To
        gate = R.get("gate")
        # project: BN3 (no activation)
        fork = self._fork if self._fork is not None else _Fork(dev, False)
        dp = torch.empty_like(R["z2"])
        sums2 = None                                    # BN2's backward sums, when a kernel above the depthwise took them
        if (self.proj_bwd_fused and dc == 0 and blk.se is None
                and self._plan_takes("pw_proj_bwd_plan", B * Po, blk.cexp, blk.cout)):
            # dz3 is computed on load and never stored; one pass yields dp, the project weight's gradient and BN2's sums
            coef = self._bn_bwd_coef(dy, None, None, R["z3"], R["sc3"], R["sv3"], 0, B, Po, blk.cout,
                                     G[blk.proj[1].weight], G[blk.proj[1].bias], dev, 0, None)
            sums2 = self._zero_pool.take(2, blk.cexp, dev)
            sc3, sv3, sc2, sv2 = R["sc3"], R["sv3"], R["sc2"], R["sv2"]
            L.pw_proj_bwd_fused(dy.data_ptr(), R["z3"].data_ptr(), sc3[0].data_ptr(), sc3[1].data_ptr(), sv3[0].data_ptr(),
                                sv3[1].data_ptr(), coef[0].data_ptr(), coef[1].data_ptr(), R["z2"].data_ptr(),
                                sc2[0].data_ptr(), sc2[1].data_ptr(), sv2[0].data_ptr(), sv2[1].data_ptr(), blk.act,
                                blk.proj[0].weight.data_ptr(), dp.data_ptr(), G[blk.proj[0].weight].data_ptr(),
                                sums2[0].data_ptr(), sums2[1].data_ptr(), 0, B * Po, blk.cexp, blk.cout, st)
        else:
            dz3 = self._bn_bwd(dy, None, None, R["z3"], R["sc3"], R["sv3"], 0, B, Po, blk.cout,
                               G[blk.proj[1].weight], G[blk.proj[1].bias], dev)
            fork.run(lambda: self._wgrad(dz3, R["z2"], G[blk.proj[0].weight], None, B * Po, blk.cout, blk.cexp,
                                         in_sc=R["sc2"], in_act=blk.act, gate=gate, rows_per_sample=Po), dz3)
            self._gemm(dz3, blk.proj[0].weight, dp, B * Po, blk.cexp, blk.cout, w_trans=True)
        dpool = None
        if blk.se is not None:
            Sq = blk.se.fc1.out_features
            dgate = torch.zeros(B, blk.cexp, device=dev, dtype=torch.float32)
            if self.se_fused:
                # slices of a sample's pixels = CTAs per sample: ~EAT_SE_PARTS_PER_SM CTAs per SM over the batch, at least
                # ~16 pixels per slice.  Every slice writes 4 x C partial sums, so few, long slices are preferred.
                parts = max(1, min(32, (torch.cuda.get_device_properties(dev).multi_processor_count * self.se_parts_per_sm) // B, (Po + 15) // 16))
                part = torch.empty(parts, 4, B, blk.cexp, device=dev, dtype=torch.float32)
                L.se_bn_bwd_reduce(dp.data_ptr(), R["z2"].data_ptr(), R["sc2"][0].data_ptr(), R["sc2"][1].data_ptr(),
                                   R["sv2"][0].data_ptr(), blk.act, dgate.data_ptr(), part.data_ptr(), parts, dc, B, Po,
                                   blk.cexp, st)
            else:
                L.se_bwd_reduce(dp.data_ptr(), R["z2"].data_ptr(), R["sc2"][0].data_ptr(), R["sc2"][1].data_ptr(),
                                blk.act, dgate.data_ptr(), dc, B, Po, blk.cexp, st)
            du2 = torch.empty(B, blk.cexp, device=dev, dtype=torch.float32)
            du1 = torch.empty(B, Sq, device=dev, dtype=torch.float32)
            dpool = torch.empty(B, blk.cexp, device=dev, dtype=torch.float32)
            L.se_fc_bwd(dgate.data_ptr(), gate.data_ptr(), R["hidden"].data_ptr(), blk.se.fc1.weight.data_ptr(),
                        blk.se.fc2.weight.data_ptr(), 1.0 / Po, du2.data_ptr(), du1.data_ptr(), dpool.data_ptr(),
                        B, blk.cexp, Sq, st)
            fork.run(lambda: (self._wgrad(du2, R["hidden"], G[blk.se.fc2.weight], G[blk.se.fc2.bias], B, blk.cexp, Sq, g_code=0, a_code=0),
                              self._wgrad(du1, R["mean"], G[blk.se.fc1.weight], G[blk.se.fc1.bias], B, Sq, blk.cexp, g_code=0, a_code=0)),
                     du2, du1)
        # depthwise: BN2 + activation (+ SE gate / squeeze gradient composed on the fly)
        if blk.se is not None and self.se_fused:
            sums2 = self._zero_pool.take(2, blk.cexp, dev)
            L.se_bn_bwd_combine(part.data_ptr(), parts, gate.data_ptr(), dpool.data_ptr(), R["sv2"][1].data_ptr(), B,
                                blk.cexp, sums2[0].data_ptr(), sums2[1].data_ptr(), st)
        has_exp = blk.expand is not None
        dw_in = R["z1"] if has_exp else R["inp"]
        sc1 = R["sc1"] if has_exp else None
        if (self.dw_bwd_fused and dc == 0 and blk.dil == 1 and (blk.k, blk.stride) in DW_BWD_FUSED_SHAPES
                and blk.cexp % (4 if blk.k == 3 else 2) == 0):      # the kernel's channel vector: 4 (3x3) or 2 (5x5)
            # dz2 is computed on load and never stored; one walk yields the depthwise input gradient, the depthwise
            # weight gradient and the expand BatchNorm's backward sums
            coef = self._bn_bwd_coef(dp, gate, dpool, R["z2"], R["sc2"], R["sv2"], blk.act, B, Po, blk.cexp,
                                     G[blk.dw[1].weight], G[blk.dw[1].bias], dev, dc, sums2)
            da1 = torch.empty_like(dw_in)
            sums1 = self._zero_pool.take(2, blk.cexp, dev) if has_exp else None
            L.dw_conv_bwd_fused(dp.data_ptr(), _ptr(gate), _ptr(dpool), R["z2"].data_ptr(), R["sc2"][0].data_ptr(),
                                R["sc2"][1].data_ptr(), R["sv2"][0].data_ptr(), R["sv2"][1].data_ptr(), blk.act,
                                coef[0].data_ptr(), coef[1].data_ptr(), R["wt"].data_ptr(), dw_in.data_ptr(),
                                _ptr(sc1[0]) if has_exp else 0, _ptr(sc1[1]) if has_exp else 0, blk.act if has_exp else 0,
                                _ptr(dy) if (blk.res and not has_exp) else 0, da1.data_ptr(),
                                G[blk.dw[0].weight].data_ptr(), _ptr(R["sv1"][0]) if has_exp else 0,
                                _ptr(R["sv1"][1]) if has_exp else 0, _ptr(sums1[0]) if has_exp else 0,
                                _ptr(sums1[1]) if has_exp else 0, dc, B, Fi, Ti, blk.cexp, blk.k, blk.stride, st)
            return self._expand_bwd(blk, R, dy, G, B, da1, sums1)
        dz2 = self._bn_bwd(dp, gate, dpool, R["z2"], R["sc2"], R["sv2"], blk.act, B, Po, blk.cexp,
                           G[blk.dw[1].weight], G[blk.dw[1].bias], dev, sums=sums2)
        xf = (_ptr(sc1[0]) if has_exp else 0, _ptr(sc1[1]) if has_exp else 0, blk.act if has_exp else 0)
        if self._wanted(G[blk.dw[0].weight]) is None:
            pass                                        # the depthwise weight's gradient was not asked for
        elif blk.dil > 1:
            fork.run(lambda: L.dw_conv_wgrad_dil(dz2.data_ptr(), dw_in.data_ptr(), *xf, G[blk.dw[0].weight].data_ptr(), dc,
                                                 B, Fi, Ti, blk.cexp, blk.k, blk.stride, blk.dil, _stream()), dz2)
        else:
            fork.run(lambda: L.dw_conv_wgrad(dz2.data_ptr(), dw_in.data_ptr(), *xf, G[blk.dw[0].weight].data_ptr(), 0, dc,
                                             B, Fi, Ti, blk.cexp, blk.k, blk.stride, _stream()), dz2)
        da1 = torch.empty_like(dw_in)
        sums1 = None
        res = _ptr(dy) if (blk.res and not has_exp) else 0
        if blk.dil > 1:
            L.dw_conv_dgrad_dil(dz2.data_ptr(), R["wt"].data_ptr(), res, da1.data_ptr(), dc, B, Fi, Ti, blk.cexp, blk.k,
                                blk.stride, blk.dil, st)
        elif has_exp and self.dgrad_bnred and blk.stride == 2 and dc == 0 and blk.k in (3, 5):
            # the expand BatchNorm's reduce pass rides in the epilogue of the kernel that produces its upstream gradient
            sums1 = self._zero_pool.take(2, blk.cexp, dev)
            L.dw_conv_dgrad_bnred(dz2.data_ptr(), R["wt"].data_ptr(), 0, da1.data_ptr(), R["z1"].data_ptr(),
                                  R["sc1"][0].data_ptr(), R["sc1"][1].data_ptr(), R["sv1"][0].data_ptr(),
                                  R["sv1"][1].data_ptr(), blk.act, sums1[0].data_ptr(), sums1[1].data_ptr(), dc, B, Fi, Ti,
                                  blk.cexp, blk.k, blk.stride, st)
        else:
            # without an expand stage the depthwise input IS the block input: fold the residual gradient in
            L.dw_conv_dgrad(dz2.data_ptr(), R["wt"].data_ptr(), 0, res, da1.data_ptr(), dc, B, Fi, Ti, blk.cexp, blk.k,
                            blk.stride, st)
        return self._expand_bwd(blk, R, dy, G, B, da1, sums1)

    def _expand_bwd(self, blk, R, dy, G, B, da1, sums1):
        """expand stage (BN1 + 1x1 conv) from the depthwise input gradient da1; returns the gradient w.r.t. the block input.
        sums1: BN1's backward sums when the depthwise backward already took them (else None: a reduce pass)."""
        if blk.expand is None:
            return da1
        dev = da1.device
        Pi = R["Fi"] * R["Ti"]
        if self.expand_bwd_fused and self.dcode == 0 and self._plan_takes("pw_bwd_plan", B * Pi, blk.cexp, blk.cin):
            # dz1 is computed on load and never stored; one pass yields the block input's gradient and the expand weight's
            coef = self._bn_bwd_coef(da1, None, None, R["z1"], R["sc1"], R["sv1"], blk.act, B, Pi, blk.cexp,
                                     G[blk.expand[1].weight], G[blk.expand[1].bias], dev, 0, sums1)
            dinp = torch.empty_like(R["inp"])
            sc1, sv1 = R["sc1"], R["sv1"]
            lib().pw_conv_bwd_fused(da1.data_ptr(), R["z1"].data_ptr(), sc1[0].data_ptr(), sc1[1].data_ptr(),
                                    sv1[0].data_ptr(), sv1[1].data_ptr(), blk.act, coef[0].data_ptr(), coef[1].data_ptr(),
                                    R["inp"].data_ptr(), blk.expand[0].weight.data_ptr(), _ptr(dy) if blk.res else 0,
                                    dinp.data_ptr(), G[blk.expand[0].weight].data_ptr(), 0, B * Pi, blk.cexp, blk.cin,
                                    _stream())
            return dinp
        fork = self._fork if self._fork is not None else _Fork(dev, False)
        dz1 = self._bn_bwd(da1, None, None, R["z1"], R["sc1"], R["sv1"], blk.act, B, Pi, blk.cexp,
                           G[blk.expand[1].weight], G[blk.expand[1].bias], dev, sums=sums1)
        fork.run(lambda: self._wgrad(dz1, R["inp"], G[blk.expand[0].weight], None, B * Pi, blk.cexp, blk.cin), dz1)
        dinp = torch.empty_like(R["inp"])
        self._gemm(dz1, blk.expand[0].weight, dinp, B * Pi, blk.cin, blk.cexp, w_trans=True,
                   res=dy if blk.res else None)
        return dinp

    def _plan_takes(self, planner, M, cexp, cn):
        """whether the fused 1x1 backward kernel behind `planner` (pw_bwd_plan: expand stage, pw_proj_bwd_plan: project
        stage) accepts the shape (host-only, asked once per shape)"""
        key = (planner, M, cexp, cn)
        if key not in self._pw_bwd_ok:
            import ctypes
            from ._lib import EatError
            plan = (ctypes.c_int * 4)()
            try:
                getattr(lib(), planner)(M, cexp, cn, ctypes.addressof(plan))
                self._pw_bwd_ok[key] = True
            except EatError:
                self._pw_bwd_ok[key] = False
        return self._pw_bwd_ok[key]

    def _backward(self, S, dlogits, on_ready=None, input_grad=False, wanted=None, dembed=None, dfmaps=None):
        """-> dict {parameter: fp32 gradient view into one flat arena} (arena returned under key None).
        dlogits, dembed ([B, C] gradient of the embedding) and dfmaps (the 17 feature maps' gradients, [B, C, F, T] of any
        strides, fp32 or bf16; needs a forward with fmaps=True) may each be None, as may every entry of dfmaps: the
        gradients that are given are summed.  Without dlogits the classifier's backward is skipped and its views stay 0;
        stages no gradient reaches are skipped as well.
        on_ready(flat, i): called after each stage with the index i of the first parameter (model.parameters() order)
        whose gradient is final -- everything from i to the end is -- so a data-parallel trainer can start reducing.
        input_grad: the input spectrogram's gradient [B, 1, F, T] fp32 is returned under key "x".  wanted: the parameters
        whose gradients are needed (None: all); launches that only produce the others' gradients are skipped, so their
        views hold no gradient.  A forward on running statistics (S["frozen"]) gets the backward on them."""
        self._bn_frozen = S["frozen"]
        try:
            return self._backward_impl(S, dlogits, on_ready, input_grad, wanted, dembed, dfmaps)
        finally:
            self._bn_frozen = False
            self._unwanted = frozenset()

    def _add_fmap_grad(self, dy, g, shape, dtype=None):
        """dy (+)= g.  dy: the gradient at a map's NHWC tensor [B, F, T, C] (contiguous, `dtype`, by default the storage
        dtype), None when no gradient reached it: then a new tensor.  g: the map's own gradient [B, C, F, T] of any
        strides, fp32 or bf16; None when the loss does not use the map: then dy is returned as it is."""
        if g is None:
            return dy
        B, F, T, C = shape
        acc = dy is not None
        if dy is None:
            dy = torch.empty(B, F, T, C, device=g.device, dtype=dtype or self.tdtype)
        codes = {torch.float32: 0, torch.bfloat16: 1}
        lib().fmap_grad_nhwc(g.data_ptr(), codes[g.dtype], *g.stride(), dy.data_ptr(), codes[dy.dtype], B, C, F, T,
                             int(acc), _stream())
        return dy

    def _embed_grad(self, dembed, dfeat, B, C):
        """dfeat [B, C] fp32 (+)= dembed [B, C] (any strides); dfeat None: a new tensor"""
        return self._add_fmap_grad(dfeat, dembed[:, :, None, None], (B, 1, 1, C), torch.float32).view(B, C)

    def _backward_impl(self, S, dlogits, on_ready, input_grad, wanted, dembed=None, dfmaps=None):
        dev = S["x"].device
        B = S["B"]
        HS = ACT["hswish"]
        self._zero_pool = _ZeroPool()
        params = self.param_list()
        flat = torch.zeros(sum(p.numel() for p in params), device=dev, dtype=torch.float32)
        G, off = {}, 0
        for p in params:
            G[p] = flat[off:off + p.numel()].view_as(p)
            off += p.numel()
        if wanted is not None:
            wanted = {id(p) for p in wanted}
            self._unwanted = frozenset(id(G[p]) for p in params if id(p) not in wanted)
        if dlogits is not None:
            dlogits = dlogits.float().contiguous()
        fork = self._fork = _Fork(dev, self.fork_wgrad)
        pidx = {id(p): i for i, p in enumerate(params)}

        def done(module):
            fork.join()                                  # this stage's weight gradients are complete
            if on_ready is not None:
                on_ready(flat, min(pidx[id(p)] for p in module.parameters()))

        # ---- classifier
        Ls = S["last"]
        P = Ls["Fi"] * Ls["Ti"]
        conv, bn = self.last[0], self.last[1]
        cl = conv.out_channels
        last_shape = (B, Ls["Fi"], Ls["Ti"], cl)
        dlast = dfmaps[-1] if dfmaps is not None else None     # the last conv's activated output
        if self.mha is not None:
            gA = None
            if dlogits is not None:
                gA = self._mha_bwd(S, dlogits, G, fork)
                done(self.model.classifier)
            gA = self._add_fmap_grad(gA, dlast, last_shape)
            # the embedding is the global mean of the same activation: its gradient enters as the pool's
            dpool = self._embed_grad(dembed, None, B, cl).mul_(1.0 / P) if dembed is not None else None
            dz = None
            if gA is not None or dpool is not None:
                dz = self._bn_bwd(gA, None, dpool, Ls["z"], Ls["sc"], Ls["sv"], HS, B, P, cl, G[bn.weight], G[bn.bias],
                                  dev)
            return self._backward_trunk(S, G, flat, fork, done, dz, input_grad, dfmaps)
        dfeat = None
        if dlogits is not None:
            dfeat = self._classifier_bwd(S["head"], dlogits, G, fork, B, dev)
            done(self.fc1)
        if dembed is not None:
            dfeat = self._embed_grad(dembed, dfeat, B, cl)

        # ---- last 1x1 conv (+BN+Hardswish, global average pool)
        dpool = dfeat.mul_(1.0 / P) if dfeat is not None else None    # gradient of the spatial mean, broadcast inside the BN-backward kernels
        gA = self._add_fmap_grad(None, dlast, last_shape)
        dz = None
        if gA is not None or dpool is not None:
            dz = self._bn_bwd(gA, None, dpool, Ls["z"], Ls["sc"], Ls["sv"], HS, B, P, cl, G[bn.weight], G[bn.bias], dev)
        return self._backward_trunk(S, G, flat, fork, done, dz, input_grad, dfmaps)

    def _classifier_bwd(self, H, dlogits, G, fork, B, dev):
        """the MLP classifier's backward -> the embedding's gradient dfeat [B, C] fp32"""
        L = lib()
        st = _stream()
        HS = ACT["hswish"]
        n1, ncls, cl = self.fc1.out_features, self.fc2.out_features, self.fc1.in_features
        fork.run(lambda: self._wgrad(dlogits, H["h_pre"], G[self.fc2.weight], G[self.fc2.bias], B, ncls, n1, in_sc=H["ident"],
                                     in_act=HS, gate=H["mask"], rows_per_sample=1, g_code=0, a_code=0), dlogits)
        dh = torch.empty(B, n1, device=dev, dtype=torch.float32)
        self._gemm(dlogits, self.fc2.weight, dh, B, n1, ncls, a_code=0, c_code=0, w_trans=True)
        dpre = torch.empty_like(dh)
        L.act_bwd(dh.data_ptr(), H["h_pre"].data_ptr(), _ptr(H["mask"]), HS, dpre.data_ptr(), dh.numel(), st)
        fork.run(lambda: self._wgrad(dpre, H["feat"], G[self.fc1.weight], G[self.fc1.bias], B, n1, cl, g_code=0, a_code=0), dpre)
        dfeat = torch.empty(B, cl, device=dev, dtype=torch.float32)
        self._gemm(dpre, self.fc1.weight, dfeat, B, cl, n1, a_code=0, c_code=0, w_trans=True)
        return dfeat

    def _backward_trunk(self, S, G, flat, fork, done, dz, input_grad=False, dfmaps=None):
        """from the gradient dz at the last 1x1 conv's output (None: no gradient reached it) down to the stem; dfmaps[i]
        (None or an entry None: unused) is added to the gradient at the stem's (i = 0) or block i's output before that
        stage's backward.  A stage no gradient reaches is skipped: its parameters' views stay 0."""
        L = lib()
        st = _stream()
        dev = S["x"].device
        dc = self.dcode
        B = S["B"]
        HS = ACT["hswish"]
        Ls = S["last"]
        P = Ls["Fi"] * Ls["Ti"]
        conv = self.last[0]
        cl = conv.out_channels
        dy = None
        if dz is not None:
            fork.run(lambda: self._wgrad(dz, Ls["inp"], G[conv.weight], None, B * P, cl, conv.in_channels), dz)
            dy = torch.empty_like(Ls["inp"])
            self._gemm(dz, conv.weight, dy, B * P, conv.in_channels, cl, w_trans=True)
        done(self.last)

        # ---- blocks, last to first
        n = len(self.blocks)
        for i, (blk, R, mod) in enumerate(zip(reversed(self.blocks), reversed(S["blocks"]), reversed(self._block_modules()))):
            if dfmaps is not None:
                dy = self._add_fmap_grad(dy, dfmaps[n - i], (B, R["Fo"], R["To"], blk.cout))
            if dy is not None:
                dy = self._block_bwd(blk, R, dy, G, B)
            done(mod)
        # ---- stem
        St = S["stem"]
        conv, bn = self.stem[0], self.stem[1]
        c0 = conv.out_channels
        P0 = St["Fo"] * St["To"]
        if dfmaps is not None:
            dy = self._add_fmap_grad(dy, dfmaps[0], (B, St["Fo"], St["To"], c0))
        fused = self.stem_bwd_fused and dc == 0 and c0 <= 64 and c0 % 4 == 0 and conv.stride[0] in (1, 2)
        if dy is None:                                  # no gradient reached the stem
            if input_grad:
                G["x"] = torch.zeros(B, 1, S["F"], S["T"], device=dev, dtype=torch.float32)
        elif fused or input_grad:
            coef = self._bn_bwd_coef(dy, None, None, St["z"], St["sc"], St["sv"], HS, B, P0, c0, G[bn.weight], G[bn.bias],
                                     dev, dc, None)
            wgrad = self._wanted(G[conv.weight]) is not None
            if wgrad and fused:
                # dz0 is computed on load in its only consumer and never stored
                L.stem_wgrad(dy.data_ptr(), 0, S["x"].data_ptr(), G[conv.weight].data_ptr(), B, S["F"], S["T"], c0,
                             conv.stride[0], St["z"].data_ptr(), St["sc"][0].data_ptr(), St["sc"][1].data_ptr(),
                             St["sv"][0].data_ptr(), St["sv"][1].data_ptr(), HS, coef[0].data_ptr(), coef[1].data_ptr(), st)
            elif wgrad:
                dz0 = self._bn_bwd_apply(dy, None, None, St["z"], St["sc"], St["sv"], HS, coef, B, P0, c0, dc)
                L.stem_wgrad(dz0.data_ptr(), dc, S["x"].data_ptr(), G[conv.weight].data_ptr(), B, S["F"], S["T"], c0,
                             conv.stride[0], 0, 0, 0, 0, 0, 0, 0, 0, st)
            if input_grad:
                dx = torch.empty(B, 1, S["F"], S["T"], device=dev, dtype=torch.float32)
                L.stem_dgrad(dy.data_ptr(), dc, St["z"].data_ptr(), St["sc"][0].data_ptr(), St["sc"][1].data_ptr(),
                             St["sv"][0].data_ptr(), St["sv"][1].data_ptr(), HS, coef[0].data_ptr(), coef[1].data_ptr(),
                             conv.weight.data_ptr(), dx.data_ptr(), B, S["F"], S["T"], c0, conv.stride[0], st)
                G["x"] = dx
        else:
            dz0 = self._bn_bwd(dy, None, None, St["z"], St["sc"], St["sv"], HS, B, St["Fo"] * St["To"], c0, G[bn.weight],
                               G[bn.bias], dev)
            L.stem_wgrad(dz0.data_ptr(), dc, S["x"].data_ptr(), G[conv.weight].data_ptr(), B, S["F"], S["T"], c0,
                         conv.stride[0], 0, 0, 0, 0, 0, 0, 0, 0, st)
        fork.join()
        self._fork = None
        G[None] = flat
        return G
