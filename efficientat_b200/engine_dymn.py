"""DyMN execution engine: ContextGen -> DynamicConv 1x1 (wgmma, kernel mix fused into the weight staging) ->
BN+act -> DynamicConv depthwise (per-sample tap tables) + BN + DyReLU-B + CoordAtt -> DynamicConv 1x1 + BN
(+ residual).  Reference models/dymn/dy_block.py:390-409, models/dymn/model.py:157-200.

Eval: folded BatchNorm, DyReLU/CoordAtt fused into the depthwise epilogue.  Training: batch-statistics forward
(raw conv outputs + statistics, like MN) and a hand-written backward through every dynamic component:
DynamicConv data gradient with W^T banks, per-sample weight gradients S_b = G_b^T X_b on tensor cores from which
the bank gradients (sum_b alpha S_b) and the attention gradients (<S_b, W_k>) follow, DyReLU / CoordAtt
reductions, the coefficient / attention / coordinate nets, and the ContextGen pooling."""
import torch

from ._lib import lib
from .engine import ACT, MNEngine, _block_layer, _conv_out, _pair, _ptr, _stream, _xf

SIG = 3             # sigmoid epilogue of the context nets


class DyMNEngine(MNEngine):
    def _plan(self):
        from .models.dymn.dy_block import DY_Block
        from .models.mn.block_types import InvertedResidual
        m = self.model
        self.stem, self.last = m.in_c, m.out_c
        self.blocks = []
        for blk in m.layers:
            L = _block_layer(blk)
            L.dy = isinstance(blk, DY_Block)
            if L.dy:
                L.m = blk
                L.has_exp = L.cexp != L.cin
                L.H = blk.context_dim
            else:
                assert isinstance(blk, InvertedResidual)
            self.blocks.append(L)
        self.fc1, self.fc2 = m.classifier[2], m.classifier[5]
        self.dropout_p = m.classifier[4].p

    dyn_tma_min_rps = int(__import__("os").environ.get("EAT_DYN_TMA_MIN_RPS", "400"))     # per-sample weights go through HBM: the TMA kernel pays off from ~400 rows per sample

    def _block_modules(self):
        return list(self.model.layers)

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
            L.pw_tma_dyn_fwd(A.data_ptr(), W.data_ptr(), att.data_ptr(), nk, 0, C.data_ptr(), M, N, K, rps, *_pair(sc), act,
                             _ptr(res), *_pair(stats), ws.data_ptr(), ws.numel(), _stream())
            return
        if self.gemm_impl != "simt":
            L.pw_tc_dyn_fwd(A.data_ptr(), dc, W.data_ptr(), att.data_ptr(), nk, C.data_ptr(), M, N, K, rps, 0, 0, 0,
                            *_pair(sc), act, _ptr(res), *_pair(stats), _stream())
            return
        B = M // rps
        Wm = self._mixed_weights(W, att, B, N * K)
        es = 4 if dc == 0 else 2
        for b in range(B):
            L.gemm_simt_fwd(A.data_ptr() + b * rps * K * es, dc, Wm.data_ptr() + 4 * b * N * K, 0,
                            C.data_ptr() + b * rps * N * es, dc, rps, N, K, 0, 0, 0, 0, 1, *_pair(sc), act,
                            (res.data_ptr() + b * rps * N * es) if res is not None else 0, *_pair(stats), _stream())

    # ------------------------------------------------------------------ ContextGen (dy_block.py:235-254)
    def _attention(self, conv, h_c, B, H):
        """a DynamicConv's attention over its k kernels from the context h_c [B, H] -> [B, k]"""
        att = torch.empty(B, conv.k, device=h_c.device, dtype=torch.float32)
        lin = conv.residuals[0]
        lib().dyconv_att(h_c.data_ptr(), lin.weight.data_ptr(), lin.bias.data_ptr(), float(conv.temperature), att.data_ptr(),
                         B, H, conv.k, _stream())
        return att

    def _coord_att(self, blk, hseq, scJ, B, Fi, Ti, Fo, To):
        """the coordinate branch: the joint sequence hseq [B, Fi + Ti, H] split into its frequency and time parts, pooled
        to the depthwise output's Fo / To (with the joint BatchNorm + Hardswish on load when scJ is given, i.e. hseq is
        raw), and the conv_f / conv_t nets -> (hf [B, Fo, H], ht [B, To, H], ca_f [B, Fo, C], ca_t [B, To, C])"""
        L, st = lib(), _stream()
        dev, f32 = hseq.device, torch.float32
        cg, H, s = blk.m.context_gen, blk.H, blk.stride
        xf = _xf(scJ, ACT["hswish"])
        hf = torch.empty(B, Fo, H, device=dev, dtype=f32)
        ht = torch.empty(B, To, H, device=dev, dtype=f32)
        L.seq_pool(hseq.data_ptr(), hf.data_ptr(), B, Fi + Ti, 0, Fi, H, s, *xf, st)
        L.seq_pool(hseq.data_ptr(), ht.data_ptr(), B, Fi + Ti, Fi, Ti, H, s, *xf, st)
        ca_f = torch.empty(B, Fo, blk.cexp, device=dev, dtype=f32)
        ca_t = torch.empty(B, To, blk.cexp, device=dev, dtype=f32)
        self._gemm(hf, cg.conv_f.weight, ca_f, B * Fo, blk.cexp, H, bias=cg.conv_f.bias, act=SIG, a_code=0, c_code=0)
        self._gemm(ht, cg.conv_t.weight, ca_t, B * To, blk.cexp, H, bias=cg.conv_t.bias, act=SIG, a_code=0, c_code=0)
        return hf, ht, ca_f, ca_t

    # ------------------------------------------------------------------ eval
    def _block_eval(self, blk, a, B, Fi, Ti, lens=None, si=0):
        """lens: the call's StageLengths (clips of different lengths), with stage si the block's input; None otherwise"""
        if not blk.dy:
            return super()._block_eval(blk, a, B, Fi, Ti, lens, si)
        L = lib()
        st = _stream()
        dev = a.device
        td, dc = self.tdtype, self.dcode
        m = blk.m
        H = blk.H
        cg = m.context_gen
        P = Fi + Ti
        f32 = torch.float32
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
        _, _, ca_f, ca_t = self._coord_att(blk, hcat, None, B, Fi, Ti, Fo, To)

        # ---- expand: DynamicConv 1x1 + BN + act
        inp = a
        if blk.has_exp:
            att = self._attention(m.exp_conv, h_c, B, H)
            sc = self._fold(m.exp_norm, dev)
            e = torch.empty(B, Fi, Ti, blk.cexp, device=dev, dtype=td)
            self._dyn_gemm(inp, m.exp_conv.weight, att, m.exp_conv.k, e, B * Fi * Ti, blk.cexp, blk.cin, Fi * Ti, sc=sc,
                           act=blk.act)
        else:
            e = inp
        if lens is not None:
            self._pad_zero(e, B, Fi, Ti, blk.cexp, lens, si)
        # ---- depthwise DynamicConv + BN + DyReLU-B + CoordAtt
        att = self._attention(m.depth_conv, h_c, B, H)
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
        L.dw_conv_fwd_dy_m(e.data_ptr(), wt.data_ptr(), kk * blk.cexp, d.data_ptr(), dc, B, Fi, Ti, blk.cexp, blk.k, s,
                           0, 0, 0, *_pair(sc), theta.data_ptr(), m.depth_act.lambdas.data_ptr(),
                           m.depth_act.init_v.data_ptr(), ca_f.data_ptr(), ca_t.data_ptr(), npc, 0, 0, st)
        # ---- project: DynamicConv 1x1 + BN (+ residual)
        att = self._attention(m.proj_conv, h_c, B, H)
        sc = self._fold(m.proj_norm, dev)
        o = torch.empty(B, Fo, To, blk.cout, device=dev, dtype=td)
        self._dyn_gemm(d, m.proj_conv.weight, att, m.proj_conv.k, o, B * Fo * To, blk.cout, blk.cexp, Fo * To, sc=sc,
                       res=inp if blk.res else None)
        return o, Fo, To

    # ------------------------------------------------------------------ training
    def _block_train_fwd(self, blk, a, B, Fi, Ti):
        if not blk.dy:
            return super()._block_train_fwd(blk, a, B, Fi, Ti)
        L = lib()
        st = _stream()
        dev = a.device
        td, dc = self.tdtype, self.dcode
        f32 = torch.float32
        m, H, cg = blk.m, blk.H, blk.m.context_gen
        P = Fi + Ti
        HS = ACT["hswish"]
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
        L.bn_act_pool(hraw.data_ptr(), *_pair(scJ), HS, h_c.data_ptr(), 1.0 / P, 0, B, P, H, st)
        s = blk.stride
        Fo, To = _conv_out(Fi, blk.k, s), _conv_out(Ti, blk.k, s)
        hf, ht, ca_f, ca_t = self._coord_att(blk, hraw, scJ, B, Fi, Ti, Fo, To)
        R.update(g=g, hraw=hraw, scJ=scJ, svJ=svJ, h_c=h_c, hf=hf, ht=ht, ca_f=ca_f, ca_t=ca_t, Fo=Fo, To=To)

        M = B * Fi * Ti
        if blk.has_exp:
            att_e = self._attention(m.exp_conv, h_c, B, H)
            z1 = torch.empty(B, Fi, Ti, blk.cexp, device=dev, dtype=td)
            stt = self._new_stats(blk.cexp, dev)
            self._dyn_gemm(inp, m.exp_conv.weight, att_e, m.exp_conv.k, z1, M, blk.cexp, blk.cin, Fi * Ti, stats=stt)
            sc1, sv1 = self._finalize(m.exp_norm, stt, M, dev)
            R.update(att_e=att_e, z1=z1, sc1=sc1, sv1=sv1)
            dw_in, dw_sc = z1, sc1
        else:
            dw_in, dw_sc = inp, None
        att_d = self._attention(m.depth_conv, h_c, B, H)
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
        L.dw_conv_fwd_dy_m(dw_in.data_ptr(), wt.data_ptr(), kk * blk.cexp, z2.data_ptr(), dc, B, Fi, Ti, blk.cexp, blk.k, s,
                           *_xf(dw_sc, blk.act), 0, 0, 0, 0, 0, 0, 0, npc, *_pair(stt), st)
        sc2, sv2 = self._finalize(m.depth_norm, stt, Mo, dev)
        p = torch.empty_like(z2)
        L.dy_act_fwd_m(z2.data_ptr(), p.data_ptr(), dc, *_pair(sc2), theta.data_ptr(), m.depth_act.lambdas.data_ptr(),
                       m.depth_act.init_v.data_ptr(), ca_f.data_ptr(), ca_t.data_ptr(), npc, B, Fo, To, blk.cexp, st)
        att_p = self._attention(m.proj_conv, h_c, B, H)
        z3 = torch.empty(B, Fo, To, blk.cout, device=dev, dtype=td)
        stt = self._new_stats(blk.cout, dev)
        self._dyn_gemm(p, m.proj_conv.weight, att_p, m.proj_conv.k, z3, Mo, blk.cout, blk.cexp, Fo * To, stats=stt)
        sc3, sv3 = self._finalize(m.proj_norm, stt, Mo, dev)
        out = torch.empty(B, Fo, To, blk.cout, device=dev, dtype=td)
        L.bn_apply(z3.data_ptr(), *_pair(sc3), 0, _ptr(inp) if blk.res else 0, out.data_ptr(), dc, Mo, blk.cout, st)
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
        dX = torch.empty(M, K, device=dev, dtype=self.tdtype)
        if dc == 0 and self.pw_impl == "tma" and rps >= self.dyn_tma_min_rps:
            # data gradient dX_b = G_b . W_b: the same dynamic GEMM with the banks read transposed (no W^T copies)
            ws = torch.empty(B * K * ((N + 31) // 32) * 128, device=dev, dtype=torch.uint8)
            L.pw_tma_dyn_fwd(Gt.data_ptr(), W.data_ptr(), att.data_ptr(), nb, 1, dX.data_ptr(), M, K, N, rps, 0, 0, 0, _ptr(res),
                             0, 0, ws.data_ptr(), ws.numel(), st)
        else:
            Wt = torch.empty(nb, K, N, device=dev, dtype=torch.float32)           # W_k^T banks for the data gradient
            for j in range(nb):
                L.transpose_f32(W.data_ptr() + 4 * j * N * K, Wt.data_ptr() + 4 * j * N * K, N, K, st)
            L.pw_tc_dyn_fwd(Gt.data_ptr(), dc, Wt.data_ptr(), att.data_ptr(), nb, dX.data_ptr(), M, K, N, rps, 0, 0, 0, 0, 0,
                            0, _ptr(res), 0, 0, st)
        S = torch.zeros(B, N * K, device=dev, dtype=torch.float32)             # per-sample weight gradients
        L.pw_tc_wgrad_persample(Gt.data_ptr(), X.data_ptr(), dc, S.data_ptr(), M, N, K, rps, st)
        return dX, self._wgrad_mix(conv, S, att, B, N * K, G)

    def _dyn1x1_bwd_exact(self, conv, Gt, X, att, B, rps, N, K, G, res):
        """exact-fp32 cross-check of _dyn1x1_bwd: per-sample CUDA-core GEMMs on the materialised mixed kernels"""
        L = lib()
        st = _stream()
        dev = Gt.device
        dc = self.dcode
        es = 4 if dc == 0 else 2
        M = B * rps
        Wm = self._mixed_weights(conv.weight, att, B, N * K)
        dX = torch.empty(M, K, device=dev, dtype=self.tdtype)
        S = torch.zeros(B, N * K, device=dev, dtype=torch.float32)
        for b in range(B):
            g_b, x_b = Gt.data_ptr() + b * rps * N * es, X.data_ptr() + b * rps * K * es
            L.gemm_simt_fwd(g_b, dc, Wm.data_ptr() + 4 * b * N * K, 1, dX.data_ptr() + b * rps * K * es, dc, rps, K, N,
                            0, 0, 0, 0, 1, 0, 0, 0, (res.data_ptr() + b * rps * K * es) if res is not None else 0, 0, 0, st)
            L.gemm_simt_wgrad(g_b, dc, x_b, dc, S.data_ptr() + 4 * b * N * K, 0, rps, N, K, 0, 0, 0, 0, 1, st)
        return dX, self._wgrad_mix(conv, S, att, B, N * K, G)

    def _wgrad_mix(self, conv, S, att, B, n, G):
        """a DynamicConv's kernel-bank gradients (sum_b att[b, k] S_b, into G) and its attention's gradient
        (<S_b, W_k>, returned [B, k]) from the per-sample weight gradients S [B, n]"""
        datt = torch.empty(B, conv.k, device=S.device, dtype=torch.float32)
        lib().dyn_wgrad_mix(S.data_ptr(), att.data_ptr(), conv.weight.data_ptr(), G[conv.weight].data_ptr(), datt.data_ptr(),
                            B, n, conv.k, _stream())
        return datt

    def _att_bwd(self, conv, datt, att, h_c, dh_c, G, B, H):
        lin = conv.residuals[0]
        lib().dyconv_att_bwd(datt.data_ptr(), att.data_ptr(), float(conv.temperature), h_c.data_ptr(),
                             lin.weight.data_ptr(), G[lin.weight].data_ptr(), G[lin.bias].data_ptr(), dh_c.data_ptr(),
                             B, H, conv.k, _stream())

    def _block_bwd(self, blk, R, dy, G, B):
        if not blk.dy:
            return super()._block_bwd(blk, R, dy, G, B)
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
        L.dy_act_bwd_m(dp.data_ptr(), R["z2"].data_ptr(), du.data_ptr(), dc, *_pair(R["sc2"]), R["theta"].data_ptr(),
                       act_mod.lambdas.data_ptr(), act_mod.init_v.data_ptr(), R["ca_f"].data_ptr(), R["ca_t"].data_ptr(),
                       dcaf.data_ptr(), dcat.data_ptr(), dcoef.data_ptr(), npc, B, Fo, To, C, st)
        # DyReLU coefficient net
        coef = act_mod.coef_net[0]
        nco = 2 * npc * C
        dpre = torch.empty(B, nco, device=dev, dtype=f32)
        L.dyrelu_coef_bwd_m(dcoef.data_ptr(), R["theta"].data_ptr(), act_mod.lambdas.data_ptr(), dpre.data_ptr(), B * nco, npc,
                            st)
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
        L.dw_conv_wgrad(dz2.data_ptr(), dw_in.data_ptr(), *_xf(dw_sc, blk.act), Sdw.data_ptr(), C * kk, dc, B, Fi, Ti, C,
                        blk.k, s, st)
        datt = self._wgrad_mix(m.depth_conv, Sdw, R["att_d"], B, C * kk, G)
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
