"""DyMN execution engine: ContextGen -> DynamicConv 1x1 (wgmma, kernel mix fused into the weight staging) ->
BN+act -> DynamicConv depthwise (per-sample tap tables) + BN + DyReLU-B + CoordAtt -> DynamicConv 1x1 + BN
(+ residual).  Reference models/dymn/dy_block.py:390-409, models/dymn/model.py:157-200.

Eval: folded BatchNorm, DyReLU/CoordAtt fused into the depthwise epilogue.  Training: batch-statistics forward
(raw conv outputs + statistics, like MN) and a hand-written backward through every dynamic component:
DynamicConv data gradient with W^T banks, per-sample weight gradients S_b = G_b^T X_b on tensor cores from which
the bank gradients (sum_b alpha S_b) and the attention gradients (<S_b, W_k>) follow, DyReLU / CoordAtt
reductions, the coefficient / attention / coordinate nets, and the ContextGen pooling."""
import torch

from ._lib import check_module_tensors, lib
from .engine import ACT, MNEngine, _Layer, _conv_out, _ptr, _stat_ptrs, _stream


class DyMNEngine(MNEngine):
    def _plan(self):
        from .models.dymn.dy_block import DY_Block
        from .models.mn.block_types import ConvNormActivation, InvertedResidual
        m = self.model
        self.stem, self.last = m.in_c, m.out_c
        self.blocks = []
        for blk in m.layers:
            L = _Layer()
            L.dy = isinstance(blk, DY_Block)
            cnf = blk.cnf
            L.act = ACT["hswish"] if cnf.use_hs else ACT["relu"]
            L.k, L.stride = cnf.kernel, cnf.stride
            L.cin, L.cexp, L.cout = cnf.input_channels, cnf.expanded_channels, cnf.out_channels
            L.res = blk.use_res_connect
            if L.dy:
                L.m = blk
                L.has_exp = cnf.expanded_channels != cnf.input_channels
                L.H = blk.context_dim
            else:
                assert isinstance(blk, InvertedResidual)
                subs = [s for s in blk.block if isinstance(s, ConvNormActivation)]
                L.expand = subs[0] if len(subs) == 3 else None
                L.dw, L.proj, L.se = subs[-2], subs[-1], None
            self.blocks.append(L)
        self.fc1, self.fc2 = m.classifier[2], m.classifier[5]
        self.dropout_p = m.classifier[4].p

    dyn_tma_min_rps = int(__import__("os").environ.get("EAT_DYN_TMA_MIN_RPS", "400"))     # per-sample weights go through HBM: the TMA kernel pays off from ~400 rows per sample

    def _block_modules(self):
        return list(self.model.layers)

    def forward(self, x, return_fmaps=False, lengths=None):
        if not x.is_cuda:
            raise RuntimeError("efficientat_b200 models run on CUDA (sm_90a) only; got a CPU tensor")
        if x.dim() != 4 or x.shape[1] != 1:
            raise ValueError(f"expected input of shape [B, 1, F, T], got {tuple(x.shape)}")
        lengths = self._check_lengths(x, return_fmaps, lengths)
        check_module_tensors(self.model, x.device, type(self.model).__name__)
        self.dropout_p = float(self.model.classifier[4].p)
        return self._dispatch(x, return_fmaps, lengths)

    # ------------------------------------------------------------------ DynamicConv 1x1 dispatch
    def _mixed_weights(self, W, att, B, n):
        """[B, n] per-sample kernels sum_k att[b,k] W[k] (dy_block.py:111-117), exact fp32 (cross-check route only)"""
        nk = att.shape[1]
        out = torch.empty(B, n, device=att.device, dtype=torch.float32)
        lib().gemm_simt_fwd(att.data_ptr(), 0, W.data_ptr(), 1, out.data_ptr(), 0, B, n, nk, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0,
                            _stream())
        return out

    def _dyn_gemm(self, A, W, att, nk, C, M, N, K, rps, sc=None, act=0, res=None, stats=None):
        """C[M,N] = epi(A[M,K] . (sum_k att[b,k] W_k)[N,K]^T), rows of sample b use its own mixed kernel.
        Default: wgmma kernel with the mix fused into the weight staging.  EAT_GEMM=simt: the reference's own order
        of operations in exact fp32 (materialise the per-sample kernels, one CUDA-core GEMM per sample) -- the
        independent implementation the tensor-core path is checked against."""
        L = lib()
        dc = self.dcode
        if (self.gemm_impl != "simt" and dc == 0 and self.pw_impl == "tma" and rps >= self.dyn_tma_min_rps
                and not (res is not None and act != 0)):
            # fp32 storage, many rows per sample: the TMA kernel; per-sample kernels mixed + pre-split once per launch into
            # this scratch.  With few rows per sample the per-sample kernels (B * N * K floats through HBM) outweigh the
            # activations and the register-staged kernel, which mixes the L2-resident banks on the fly, is the better fit
            ws = torch.empty((M // rps) * N * ((K + 31) // 32) * 128, device=A.device, dtype=torch.uint8)
            L.pw_tma_dyn_fwd(A.data_ptr(), W.data_ptr(), att.data_ptr(), nk, 0, C.data_ptr(), M, N, K, rps,
                             _ptr(sc[0]) if sc is not None else 0, _ptr(sc[1]) if sc is not None else 0, act, _ptr(res),
                             _ptr(stats[0]) if stats is not None else 0, _ptr(stats[1]) if stats is not None else 0,
                             ws.data_ptr(), ws.numel(), _stream())
            return
        if self.gemm_impl != "simt":
            L.pw_tc_dyn_fwd(A.data_ptr(), dc, W.data_ptr(), att.data_ptr(), nk, C.data_ptr(), M, N, K, rps, 0, 0, 0,
                            _ptr(sc[0]) if sc is not None else 0, _ptr(sc[1]) if sc is not None else 0, act, _ptr(res),
                            _ptr(stats[0]) if stats is not None else 0, _ptr(stats[1]) if stats is not None else 0,
                            _stream())
            return
        B = M // rps
        Wm = self._mixed_weights(W, att, B, N * K)
        es = 4 if dc == 0 else 2
        for b in range(B):
            L.gemm_simt_fwd(A.data_ptr() + b * rps * K * es, dc, Wm.data_ptr() + 4 * b * N * K, 0,
                            C.data_ptr() + b * rps * N * es, dc, rps, N, K, 0, 0, 0, 0, 1,
                            _ptr(sc[0]) if sc is not None else 0, _ptr(sc[1]) if sc is not None else 0, act,
                            (res.data_ptr() + b * rps * N * es) if res is not None else 0,
                            _ptr(stats[0]) if stats is not None else 0, _ptr(stats[1]) if stats is not None else 0,
                            _stream())

    # ------------------------------------------------------------------
    def _dy_block_eval(self, blk, a, B, Fi, Ti, lens=None, si=0):
        """lens: the call's StageLengths (clips of different lengths), with stage si the block's input; None otherwise"""
        L = lib()
        st = _stream()
        dev = a.device
        td, dc = self.tdtype, self.dcode
        m = blk.m
        H = blk.H
        cg = m.context_gen
        P = Fi + Ti
        f32 = torch.float32
        # ---- ContextGen (dy_block.py:235-254)
        g = torch.empty(B, P, blk.cin, device=dev, dtype=f32)
        if lens is None:
            L.ctx_pool(a.data_ptr(), dc, g.data_ptr(), B, Fi, Ti, blk.cin, st)
        else:
            L.ctx_pool_len(a.data_ptr(), dc, g.data_ptr(), B, Fi, Ti, blk.cin, lens.ptr(si), st)
        hcat = torch.empty(B * P, H, device=dev, dtype=f32)
        self._gemm(g, cg.joint_conv.weight, hcat, B * P, H, blk.cin, sc=self._fold(cg.joint_norm, dev), act=ACT["hswish"],
                   a_code=0, c_code=0)
        if lens is None:
            h_c = torch.zeros(B, H, device=dev, dtype=f32)
            L.bn_act_pool(hcat.data_ptr(), 0, 0, 0, h_c.data_ptr(), 1.0 / P, 0, B, P, H, st)
        else:
            # the sequence of clip b is its first Fi + t_b rows: 0 beyond them is the time AvgPool's own zero padding
            h_c = torch.empty(B, H, device=dev, dtype=f32)
            if lens.padded(si):
                L.time_pad_zero(hcat.data_ptr(), 0, B, 1, P, H, lens.seq_ptr(si), st)
            L.mean_len(hcat.data_ptr(), 0, h_c.data_ptr(), B, 1, P, H, lens.seq_ptr(si), st)
        s = blk.stride
        Fo, To = _conv_out(Fi, blk.k, s), _conv_out(Ti, blk.k, s)
        hf = torch.empty(B, Fo, H, device=dev, dtype=f32)
        ht = torch.empty(B, To, H, device=dev, dtype=f32)
        L.seq_pool(hcat.data_ptr(), hf.data_ptr(), B, P, 0, Fi, H, s, 0, 0, 0, st)
        L.seq_pool(hcat.data_ptr(), ht.data_ptr(), B, P, Fi, Ti, H, s, 0, 0, 0, st)
        ca_f = torch.empty(B, Fo, blk.cexp, device=dev, dtype=f32)
        ca_t = torch.empty(B, To, blk.cexp, device=dev, dtype=f32)
        SIG = 3
        self._gemm(hf, cg.conv_f.weight, ca_f, B * Fo, blk.cexp, H, bias=cg.conv_f.bias, act=SIG, a_code=0, c_code=0)
        self._gemm(ht, cg.conv_t.weight, ca_t, B * To, blk.cexp, H, bias=cg.conv_t.bias, act=SIG, a_code=0, c_code=0)

        def attention(dc_mod):
            att = torch.empty(B, dc_mod.k, device=dev, dtype=f32)
            lin = dc_mod.residuals[0]
            L.dyconv_att(h_c.data_ptr(), lin.weight.data_ptr(), lin.bias.data_ptr(), float(dc_mod.temperature),
                         att.data_ptr(), B, H, dc_mod.k, st)
            return att

        # ---- expand: DynamicConv 1x1 + BN + act
        inp = a
        if blk.has_exp:
            att = attention(m.exp_conv)
            sc = self._fold(m.exp_norm, dev)
            e = torch.empty(B, Fi, Ti, blk.cexp, device=dev, dtype=td)
            self._dyn_gemm(inp, m.exp_conv.weight, att, m.exp_conv.k, e, B * Fi * Ti, blk.cexp, blk.cin, Fi * Ti, sc=sc,
                           act=blk.act)
        else:
            e = inp
        if lens is not None:
            self._pad_zero(e, B, Fi, Ti, blk.cexp, lens, si)
        # ---- depthwise DynamicConv + BN + DyReLU-B + CoordAtt
        att = attention(m.depth_conv)
        kk = blk.k * blk.k
        wt = torch.empty(B, kk, blk.cexp, device=dev, dtype=f32)
        L.dyconv_mix_dw(m.depth_conv.weight.data_ptr(), att.data_ptr(), wt.data_ptr(), B, blk.cexp, blk.k,
                        m.depth_conv.k, st)
        coef = m.depth_act.coef_net[0]
        npc = m.depth_act.M                                 # DyReLU-B pieces: theta [B, C, 2M]
        theta = torch.empty(B, 2 * npc * blk.cexp, device=dev, dtype=f32)
        self._gemm(h_c, coef.weight, theta, B, 2 * npc * blk.cexp, H, bias=coef.bias, act=SIG, a_code=0, c_code=0)
        sc = self._fold(m.depth_norm, dev)
        d = torch.empty(B, Fo, To, blk.cexp, device=dev, dtype=td)
        if npc == 2:
            L.dw_conv_fwd_dy(e.data_ptr(), wt.data_ptr(), kk * blk.cexp, d.data_ptr(), dc, B, Fi, Ti, blk.cexp, blk.k, s,
                             0, 0, 0, sc[0].data_ptr(), sc[1].data_ptr(), theta.data_ptr(), m.depth_act.lambdas.data_ptr(),
                             m.depth_act.init_v.data_ptr(), ca_f.data_ptr(), ca_t.data_ptr(), 0, 0, st)
        else:
            L.dw_conv_fwd_dy_m(e.data_ptr(), wt.data_ptr(), kk * blk.cexp, d.data_ptr(), dc, B, Fi, Ti, blk.cexp, blk.k, s,
                               0, 0, 0, sc[0].data_ptr(), sc[1].data_ptr(), theta.data_ptr(),
                               m.depth_act.lambdas.data_ptr(), m.depth_act.init_v.data_ptr(), ca_f.data_ptr(),
                               ca_t.data_ptr(), npc, 0, 0, st)
        # ---- project: DynamicConv 1x1 + BN (+ residual)
        att = attention(m.proj_conv)
        sc = self._fold(m.proj_norm, dev)
        o = torch.empty(B, Fo, To, blk.cout, device=dev, dtype=td)
        self._dyn_gemm(d, m.proj_conv.weight, att, m.proj_conv.k, o, B * Fo * To, blk.cout, blk.cexp, Fo * To, sc=sc,
                       res=inp if blk.res else None)
        return o, Fo, To

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
            if fmaps is not None:
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
            if blk.dy:
                a, Fi, Ti = self._dy_block_eval(blk, a, B, Fi, Ti, lens, i + 1)
            else:
                a, Fi, Ti = self._ir_block_eval(blk, a, B, Fi, Ti, lens, i + 1)
            keep(a, Fi, Ti, blk.cout)
        logits, feat, z = self._head_eval(a, B, Fi, Ti, lens)
        keep(z, Fi, Ti, self.last[0].out_channels)
        return logits, feat, fmaps

    # ------------------------------------------------------------------ training
    def _block_train_fwd(self, blk, a, B, Fi, Ti):
        if not blk.dy:
            return self._ir_block_train_fwd(blk, a, B, Fi, Ti)
        L = lib()
        st = _stream()
        dev = a.device
        td, dc = self.tdtype, self.dcode
        f32 = torch.float32
        m, H, cg = blk.m, blk.H, blk.m.context_gen
        P = Fi + Ti
        HS, SIG = ACT["hswish"], 3
        R = {"inp": a, "Fi": Fi, "Ti": Ti}
        inp = a
        # ---- ContextGen with batch-statistics BatchNorm on the joint sequence
        g = torch.empty(B, P, blk.cin, device=dev, dtype=f32)
        L.ctx_pool(a.data_ptr(), dc, g.data_ptr(), B, Fi, Ti, blk.cin, st)
        hraw = torch.empty(B * P, H, device=dev, dtype=f32)
        stt = self._new_stats(H, dev)
        self._gemm(g, cg.joint_conv.weight, hraw, B * P, H, blk.cin, stats=stt, a_code=0, c_code=0)
        scJ, svJ = self._finalize(cg.joint_norm, stt, B * P, dev)
        h_c = torch.zeros(B, H, device=dev, dtype=f32)
        L.bn_act_pool(hraw.data_ptr(), scJ[0].data_ptr(), scJ[1].data_ptr(), HS, h_c.data_ptr(), 1.0 / P, 0, B, P, H, st)
        s = blk.stride
        Fo, To = _conv_out(Fi, blk.k, s), _conv_out(Ti, blk.k, s)
        hf = torch.empty(B, Fo, H, device=dev, dtype=f32)
        ht = torch.empty(B, To, H, device=dev, dtype=f32)
        L.seq_pool(hraw.data_ptr(), hf.data_ptr(), B, P, 0, Fi, H, s, scJ[0].data_ptr(), scJ[1].data_ptr(), HS, st)
        L.seq_pool(hraw.data_ptr(), ht.data_ptr(), B, P, Fi, Ti, H, s, scJ[0].data_ptr(), scJ[1].data_ptr(), HS, st)
        ca_f = torch.empty(B, Fo, blk.cexp, device=dev, dtype=f32)
        ca_t = torch.empty(B, To, blk.cexp, device=dev, dtype=f32)
        self._gemm(hf, cg.conv_f.weight, ca_f, B * Fo, blk.cexp, H, bias=cg.conv_f.bias, act=SIG, a_code=0, c_code=0)
        self._gemm(ht, cg.conv_t.weight, ca_t, B * To, blk.cexp, H, bias=cg.conv_t.bias, act=SIG, a_code=0, c_code=0)
        R.update(g=g, hraw=hraw, scJ=scJ, svJ=svJ, h_c=h_c, hf=hf, ht=ht, ca_f=ca_f, ca_t=ca_t, Fo=Fo, To=To)

        def attention(dc_mod):
            att = torch.empty(B, dc_mod.k, device=dev, dtype=f32)
            lin = dc_mod.residuals[0]
            L.dyconv_att(h_c.data_ptr(), lin.weight.data_ptr(), lin.bias.data_ptr(), float(dc_mod.temperature),
                         att.data_ptr(), B, H, dc_mod.k, st)
            return att

        M = B * Fi * Ti
        if blk.has_exp:
            att_e = attention(m.exp_conv)
            z1 = torch.empty(B, Fi, Ti, blk.cexp, device=dev, dtype=td)
            stt = self._new_stats(blk.cexp, dev)
            self._dyn_gemm(inp, m.exp_conv.weight, att_e, m.exp_conv.k, z1, M, blk.cexp, blk.cin, Fi * Ti, stats=stt)
            sc1, sv1 = self._finalize(m.exp_norm, stt, M, dev)
            R.update(att_e=att_e, z1=z1, sc1=sc1, sv1=sv1)
            dw_in, dw_sc = z1, sc1
        else:
            dw_in, dw_sc = inp, None
        att_d = attention(m.depth_conv)
        kk = blk.k * blk.k
        wt = torch.empty(B, kk, blk.cexp, device=dev, dtype=f32)
        L.dyconv_mix_dw(m.depth_conv.weight.data_ptr(), att_d.data_ptr(), wt.data_ptr(), B, blk.cexp, blk.k,
                        m.depth_conv.k, st)
        coef = m.depth_act.coef_net[0]
        npc = m.depth_act.M                                 # DyReLU-B pieces: theta [B, C, 2M]
        theta = torch.empty(B, 2 * npc * blk.cexp, device=dev, dtype=f32)
        self._gemm(h_c, coef.weight, theta, B, 2 * npc * blk.cexp, H, bias=coef.bias, act=SIG, a_code=0, c_code=0)
        Mo = B * Fo * To
        z2 = torch.empty(B, Fo, To, blk.cexp, device=dev, dtype=td)
        stt = self._new_stats(blk.cexp, dev)
        xs = (_ptr(dw_sc[0]) if dw_sc is not None else 0, _ptr(dw_sc[1]) if dw_sc is not None else 0,
              blk.act if dw_sc is not None else 0)
        if npc == 2:
            L.dw_conv_fwd_dy(dw_in.data_ptr(), wt.data_ptr(), kk * blk.cexp, z2.data_ptr(), dc, B, Fi, Ti, blk.cexp, blk.k,
                             s, *xs, 0, 0, 0, 0, 0, 0, 0, *_stat_ptrs(stt), st)
        else:
            L.dw_conv_fwd_dy_m(dw_in.data_ptr(), wt.data_ptr(), kk * blk.cexp, z2.data_ptr(), dc, B, Fi, Ti, blk.cexp,
                               blk.k, s, *xs, 0, 0, 0, 0, 0, 0, 0, npc, *_stat_ptrs(stt), st)
        sc2, sv2 = self._finalize(m.depth_norm, stt, Mo, dev)
        p = torch.empty_like(z2)
        act_args = (z2.data_ptr(), p.data_ptr(), dc, sc2[0].data_ptr(), sc2[1].data_ptr(), theta.data_ptr(),
                    m.depth_act.lambdas.data_ptr(), m.depth_act.init_v.data_ptr(), ca_f.data_ptr(), ca_t.data_ptr())
        if npc == 2:
            L.dy_act_fwd(*act_args, B, Fo, To, blk.cexp, st)
        else:
            L.dy_act_fwd_m(*act_args, npc, B, Fo, To, blk.cexp, st)
        att_p = attention(m.proj_conv)
        z3 = torch.empty(B, Fo, To, blk.cout, device=dev, dtype=td)
        stt = self._new_stats(blk.cout, dev)
        self._dyn_gemm(p, m.proj_conv.weight, att_p, m.proj_conv.k, z3, Mo, blk.cout, blk.cexp, Fo * To, stats=stt)
        sc3, sv3 = self._finalize(m.proj_norm, stt, Mo, dev)
        out = torch.empty(B, Fo, To, blk.cout, device=dev, dtype=td)
        L.bn_apply(z3.data_ptr(), sc3[0].data_ptr(), sc3[1].data_ptr(), 0, _ptr(inp) if blk.res else 0, out.data_ptr(),
                   dc, Mo, blk.cout, st)
        R.update(att_d=att_d, wt=wt, theta=theta, z2=z2, sc2=sc2, sv2=sv2, p=p, att_p=att_p, z3=z3, sc3=sc3, sv3=sv3,
                 dw_in=dw_in, dw_sc=dw_sc)
        return out, Fo, To, R

    def _dyn1x1_bwd(self, conv, Gt, X, att, B, rps, N, K, G, res=None):
        """backward of a DynamicConv 1x1: returns (dX [B*rps, K], datt [B, k]); accumulates the bank gradients."""
        L = lib()
        st = _stream()
        dev = Gt.device
        dc = self.dcode
        M = B * rps
        nb = conv.k
        W = conv.weight
        if self.gemm_impl == "simt":
            return self._dyn1x1_bwd_exact(conv, Gt, X, att, B, rps, N, K, G, res)
        if dc == 0 and self.pw_impl == "tma" and rps >= self.dyn_tma_min_rps:
            # data gradient dX_b = G_b . W_b: the same dynamic GEMM with the banks read transposed (no W^T copies)
            dX = torch.empty(M, K, device=dev, dtype=self.tdtype)
            ws = torch.empty(B * K * ((N + 31) // 32) * 128, device=dev, dtype=torch.uint8)
            L.pw_tma_dyn_fwd(Gt.data_ptr(), W.data_ptr(), att.data_ptr(), nb, 1, dX.data_ptr(), M, K, N, rps, 0, 0, 0, _ptr(res),
                             0, 0, ws.data_ptr(), ws.numel(), st)
            S = torch.zeros(B, N * K, device=dev, dtype=torch.float32)             # per-sample weight gradients
            L.pw_tc_wgrad_persample(Gt.data_ptr(), X.data_ptr(), dc, S.data_ptr(), M, N, K, rps, st)
            datt = torch.empty(B, nb, device=dev, dtype=torch.float32)
            L.dyn_wgrad_mix(S.data_ptr(), att.data_ptr(), W.data_ptr(), G[W].data_ptr(), datt.data_ptr(), B, N * K, nb, st)
            return dX, datt
        Wt = torch.empty(nb, K, N, device=dev, dtype=torch.float32)           # W_k^T banks for the data gradient
        for j in range(nb):
            L.transpose_f32(W.data_ptr() + 4 * j * N * K, Wt.data_ptr() + 4 * j * N * K, N, K, st)
        dX = torch.empty(M, K, device=dev, dtype=self.tdtype)
        L.pw_tc_dyn_fwd(Gt.data_ptr(), dc, Wt.data_ptr(), att.data_ptr(), nb, dX.data_ptr(), M, K, N, rps, 0, 0, 0, 0, 0, 0,
                        _ptr(res), 0, 0, st)
        S = torch.zeros(B, N * K, device=dev, dtype=torch.float32)             # per-sample weight gradients
        L.pw_tc_wgrad_persample(Gt.data_ptr(), X.data_ptr(), dc, S.data_ptr(), M, N, K, rps, st)
        datt = torch.empty(B, nb, device=dev, dtype=torch.float32)
        L.dyn_wgrad_mix(S.data_ptr(), att.data_ptr(), W.data_ptr(), G[W].data_ptr(), datt.data_ptr(), B, N * K, nb, st)
        return dX, datt

    def _dyn1x1_bwd_exact(self, conv, Gt, X, att, B, rps, N, K, G, res):
        """exact-fp32 cross-check of _dyn1x1_bwd: per-sample CUDA-core GEMMs on the materialised mixed kernels"""
        L = lib()
        st = _stream()
        dev = Gt.device
        dc = self.dcode
        es = 4 if dc == 0 else 2
        M, nb, W = B * rps, conv.k, conv.weight
        Wm = self._mixed_weights(W, att, B, N * K)
        dX = torch.empty(M, K, device=dev, dtype=self.tdtype)
        S = torch.zeros(B, N * K, device=dev, dtype=torch.float32)
        for b in range(B):
            g_b, x_b = Gt.data_ptr() + b * rps * N * es, X.data_ptr() + b * rps * K * es
            L.gemm_simt_fwd(g_b, dc, Wm.data_ptr() + 4 * b * N * K, 1, dX.data_ptr() + b * rps * K * es, dc, rps, K, N,
                            0, 0, 0, 0, 1, 0, 0, 0, (res.data_ptr() + b * rps * K * es) if res is not None else 0, 0, 0, st)
            L.gemm_simt_wgrad(g_b, dc, x_b, dc, S.data_ptr() + 4 * b * N * K, 0, rps, N, K, 0, 0, 0, 0, 1, st)
        datt = torch.empty(B, nb, device=dev, dtype=torch.float32)
        L.dyn_wgrad_mix(S.data_ptr(), att.data_ptr(), W.data_ptr(), G[W].data_ptr(), datt.data_ptr(), B, N * K, nb, st)
        return dX, datt

    def _att_bwd(self, conv, datt, att, h_c, dh_c, G, B, H):
        lin = conv.residuals[0]
        lib().dyconv_att_bwd(datt.data_ptr(), att.data_ptr(), float(conv.temperature), h_c.data_ptr(),
                             lin.weight.data_ptr(), G[lin.weight].data_ptr(), G[lin.bias].data_ptr(), dh_c.data_ptr(),
                             B, H, conv.k, _stream())

    def _block_bwd(self, blk, R, dy, G, B):
        if not blk.dy:
            return self._ir_block_bwd(blk, R, dy, G, B)
        L = lib()
        st = _stream()
        dev = dy.device
        td, dc = self.tdtype, self.dcode
        f32 = torch.float32
        m, H, cg = blk.m, blk.H, blk.m.context_gen
        Fi, Ti, Fo, To = R["Fi"], R["Ti"], R["Fo"], R["To"]
        Pi, Po, P = Fi * Ti, Fo * To, Fi + Ti
        C = blk.cexp
        s = blk.stride
        HS = ACT["hswish"]
        h_c = R["h_c"]
        dh_c = torch.zeros(B, H, device=dev, dtype=f32)
        # ---- project: BN3, DynamicConv
        dz3 = self._bn_bwd(dy, None, None, R["z3"], R["sc3"], R["sv3"], 0, B, Po, blk.cout, G[m.proj_norm.weight],
                           G[m.proj_norm.bias], dev)
        dp, datt = self._dyn1x1_bwd(m.proj_conv, dz3, R["p"], R["att_p"], B, Po, blk.cout, C, G)
        self._att_bwd(m.proj_conv, datt, R["att_p"], h_c, dh_c, G, B, H)
        # ---- CoordAtt * DyReLU-B * BN2 backward
        dcaf = torch.zeros(B, Fo, C, device=dev, dtype=f32)
        dcat = torch.empty(B, To, C, device=dev, dtype=f32)
        act_mod = m.depth_act
        npc = act_mod.M                                     # DyReLU-B pieces: dcoef [B, C, 2M]
        dcoef = torch.zeros(B, C, 2 * npc, device=dev, dtype=f32)
        du = torch.empty_like(R["z2"])
        act_args = (dp.data_ptr(), R["z2"].data_ptr(), du.data_ptr(), dc, R["sc2"][0].data_ptr(), R["sc2"][1].data_ptr(),
                    R["theta"].data_ptr(), act_mod.lambdas.data_ptr(), act_mod.init_v.data_ptr(), R["ca_f"].data_ptr(),
                    R["ca_t"].data_ptr(), dcaf.data_ptr(), dcat.data_ptr(), dcoef.data_ptr())
        if npc == 2:
            L.dy_act_bwd(*act_args, B, Fo, To, C, st)
        else:
            L.dy_act_bwd_m(*act_args, npc, B, Fo, To, C, st)
        # DyReLU coefficient net
        coef = act_mod.coef_net[0]
        nco = 2 * npc * C
        dpre = torch.empty(B, nco, device=dev, dtype=f32)
        if npc == 2:
            L.dyrelu_coef_bwd(dcoef.data_ptr(), R["theta"].data_ptr(), act_mod.lambdas.data_ptr(), dpre.data_ptr(), B * nco, st)
        else:
            L.dyrelu_coef_bwd_m(dcoef.data_ptr(), R["theta"].data_ptr(), act_mod.lambdas.data_ptr(), dpre.data_ptr(),
                                B * nco, npc, st)
        self._wgrad(dpre, h_c, G[coef.weight], G[coef.bias], B, nco, H, g_code=0, a_code=0)
        dh_new = torch.empty_like(dh_c)
        self._gemm(dpre, coef.weight, dh_new, B, H, nco, a_code=0, c_code=0, w_trans=True, res=dh_c)
        dh_c = dh_new
        # coordinate-attention nets (conv_f / conv_t are Linear layers over the context dimension)
        dhcat = torch.empty(B, P, H, device=dev, dtype=f32)
        for dca, ca, hseq, conv, Lo, row0, Lin in ((dcaf, R["ca_f"], R["hf"], cg.conv_f, Fo, 0, Fi),
                                                   (dcat, R["ca_t"], R["ht"], cg.conv_t, To, Fi, Ti)):
            dgx = torch.empty_like(dca)
            L.sigmoid_bwd(dca.data_ptr(), ca.data_ptr(), dgx.data_ptr(), dca.numel(), st)
            self._wgrad(dgx, hseq, G[conv.weight], G[conv.bias], B * Lo, C, H, g_code=0, a_code=0)
            dhseq = torch.empty(B, Lo, H, device=dev, dtype=f32)
            self._gemm(dgx, conv.weight, dhseq, B * Lo, H, C, a_code=0, c_code=0, w_trans=True)
            L.seq_pool_bwd(dhseq.data_ptr(), dhcat.data_ptr(), B, P, row0, Lin, H, s, st)
        # ---- depthwise: BN2 (the activation was handled above), DynamicConv depthwise
        dz2 = self._bn_bwd(du, None, None, R["z2"], R["sc2"], R["sv2"], 0, B, Po, C, G[m.depth_norm.weight],
                           G[m.depth_norm.bias], dev)
        kk = blk.k * blk.k
        dw_in, dw_sc = R["dw_in"], R["dw_sc"]
        Sdw = torch.zeros(B, C * kk, device=dev, dtype=f32)
        L.dw_conv_wgrad(dz2.data_ptr(), dw_in.data_ptr(), _ptr(dw_sc[0]) if dw_sc is not None else 0,
                        _ptr(dw_sc[1]) if dw_sc is not None else 0, blk.act if dw_sc is not None else 0, Sdw.data_ptr(),
                        C * kk, dc, B, Fi, Ti, C, blk.k, s, st)
        datt = torch.empty(B, m.depth_conv.k, device=dev, dtype=f32)
        L.dyn_wgrad_mix(Sdw.data_ptr(), R["att_d"].data_ptr(), m.depth_conv.weight.data_ptr(),
                        G[m.depth_conv.weight].data_ptr(), datt.data_ptr(), B, C * kk, m.depth_conv.k, st)
        self._att_bwd(m.depth_conv, datt, R["att_d"], h_c, dh_c, G, B, H)
        da1 = torch.empty_like(dw_in)
        L.dw_conv_dgrad(dz2.data_ptr(), R["wt"].data_ptr(), kk * C, _ptr(dy) if (blk.res and not blk.has_exp) else 0,
                        da1.data_ptr(), dc, B, Fi, Ti, C, blk.k, s, st)
        if blk.has_exp:
            dz1 = self._bn_bwd(da1, None, None, R["z1"], R["sc1"], R["sv1"], blk.act, B, Pi, C, G[m.exp_norm.weight],
                               G[m.exp_norm.bias], dev)
            dinp, datt = self._dyn1x1_bwd(m.exp_conv, dz1, R["inp"], R["att_e"], B, Pi, C, blk.cin, G,
                                          res=dy if blk.res else None)
            dinp = dinp.view_as(R["inp"])
            self._att_bwd(m.exp_conv, datt, R["att_e"], h_c, dh_c, G, B, H)
        else:
            dinp = da1
        # ---- ContextGen: joint BN + Hardswish (gradient = sequence part + broadcast mean part), joint conv, pooling
        dpool = dh_c.mul_(1.0 / P)
        dhraw = self._bn_bwd(dhcat, None, dpool, R["hraw"], R["scJ"], R["svJ"], HS, B, P, H, G[cg.joint_norm.weight],
                             G[cg.joint_norm.bias], dev, code=0)
        self._wgrad(dhraw, R["g"], G[cg.joint_conv.weight], None, B * P, H, blk.cin, g_code=0, a_code=0)
        dg = torch.empty(B, P, blk.cin, device=dev, dtype=f32)
        self._gemm(dhraw, cg.joint_conv.weight, dg, B * P, blk.cin, H, a_code=0, c_code=0, w_trans=True)
        L.ctx_pool_bwd(dg.data_ptr(), dinp.data_ptr(), dc, B, Fi, Ti, blk.cin, st)
        return dinp
