"""SPADEResnetBlock — constructor, attribute names and state-dict keys of the reference's
models/networks/architecture.py:23-85; forward = fused sm_90a kernels.

Per block (x at 1/2^x_shift of the block's resolution; the nn.Upsample of generator.py:72 is folded
into the consumers' loads):

    stats(x)                                    one HBM pass, shared by norm_0 and norm_s
    actv_k  = relu(conv3x3(seg'))               thin direct conv, seg read through nearest resize
    h_k     = act(x_hat*(1+gamma)+beta)         wgmma implicit GEMM (K=9*128, N=2C) + SPADE epilogue
    conv_0 / conv_1 / conv_s                    wgmma implicit GEMM + bias / residual / blend epilogue
"""
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.utils.spectral_norm as spectral_norm

from .. import ops, precision
from .normalization import SPADE
from .prep import PackCache


class SPADEResnetBlock(nn.Module):
    def __init__(self, fin, fout, opt):
        super().__init__()
        self.learned_shortcut = (fin != fout)
        fmiddle = min(fin, fout)
        self.fin, self.fout, self.fmiddle = fin, fout, fmiddle
        self.conv_0 = nn.Conv2d(fin, fmiddle, kernel_size=3, padding=1)
        self.conv_1 = nn.Conv2d(fmiddle, fout, kernel_size=3, padding=1)
        if self.learned_shortcut:
            self.conv_s = nn.Conv2d(fin, fout, kernel_size=1, bias=False)
        if getattr(opt, "weight_norm_G", False):
            raise NotImplementedError("michigan_b200: --weight_norm_G is outside the hot path (SURVEY.md §2)")
        if "spectral" in opt.norm_G:
            self.conv_0 = spectral_norm(self.conv_0)
            self.conv_1 = spectral_norm(self.conv_1)
            if self.learned_shortcut:
                self.conv_s = spectral_norm(self.conv_s)
        norm_nc = opt.label_nc + (opt.orient_nc if not opt.no_orientation else 0) + \
            (opt.feat_num if opt.use_instance_feat else 0) + (3 if "spadebase" in opt.netG else 0)
        spade_config_str = opt.norm_G.replace("spectral", "")
        self.norm_0 = SPADE(spade_config_str, fin, norm_nc, getattr(opt, "weight_norm_G", False))
        self.norm_1 = SPADE(spade_config_str, fmiddle, norm_nc, getattr(opt, "weight_norm_G", False))
        if self.learned_shortcut:
            self.norm_s = SPADE(spade_config_str, fin, norm_nc, getattr(opt, "weight_norm_G", False))
        for c in (fin, fout, fmiddle):
            if c % 32 != 0:
                raise NotImplementedError("michigan_b200: channel counts must be multiples of 32 (got %d); use ngf %% 32 == 0" % c)
        self._cache = PackCache()

    # ------------------------------------------------------------------ operand preparation
    def sn_convs(self):
        cs = [self.conv_0, self.conv_1] + ([self.conv_s] if self.learned_shortcut else [])
        return [c for c in cs if hasattr(c, "weight_orig")]

    def _conv_pack(self, name, inv_sigma_of):
        conv = getattr(self, name)
        if hasattr(conv, "weight_orig"):
            w, isg = conv.weight_orig, inv_sigma_of[conv]
            # the scale depends on u, v as well: rebuilt whenever the spectral batch ran
            return precision.pack_conv(w.detach(), isg, precision.conv_fmt(w.shape[1]))
        fmt = precision.conv_fmt(conv.weight.shape[1])
        return self._cache.get((name, fmt), [conv.weight], lambda: precision.pack_conv(conv.weight.detach(), None, fmt))

    def _spade_pack(self, name, gfmt, gsplit):
        sp = getattr(self, name)
        c = self._cache
        if gfmt == ops.TF32:
            wgb = c.get(name + ".gb", [sp.mlp_gamma.weight, sp.mlp_beta.weight],
                        lambda: ops.pack_weight_gb(sp.mlp_gamma.weight.detach(), sp.mlp_beta.weight.detach()))
        else:
            wgb = c.get((name + ".gb16", gfmt, gsplit), [sp.mlp_gamma.weight, sp.mlp_beta.weight],
                        lambda: ops.pack_weight_gb16(sp.mlp_gamma.weight.detach(), sp.mlp_beta.weight.detach(), gfmt, gsplit))
        wsh = c.get((name + ".sh", ops.seg_tc_enabled()), [sp.mlp_shared[0].weight],
                    lambda: ops.pack_mlp_shared(sp.mlp_shared[0].weight.detach()))
        g1 = c.get(name + ".g1", [sp.mlp_gamma.bias], lambda: (sp.mlp_gamma.bias.detach() + 1.0).contiguous())
        return wsh, sp.mlp_shared[0].bias.detach(), wgb, g1, sp.mlp_beta.bias.detach()

    # ------------------------------------------------------------------ forward
    def forward_nhwc(self, x, x_shift, seg4, inv_sigma_of, blend=None, save=None):
        """x: [N, h>>x_shift, w>>x_shift, fin] NHWC; seg4: [N,Hs,Ws,4]; returns [N,h,w,fout].
        blend=(bf, hair, back, mask_stride) applies generator.py:186's background blend in the epilogue.
        save: a namespace to fill when the hand-written backward will run (autograd.block_bwd).  The arithmetic of the
        forward is the SAME in both modes (same operand formats, same kernels): training additionally keeps, per SPADE, the
        fp32 value of h = act(SPADE(x)) (operand of the weight-gradient GEMM) and 1 + gamma."""
        N, hs, ws, fin = x.shape
        h, w = hs << x_shift, ws << x_shift
        R = seg4.shape[1] // h
        if seg4.shape[1] != h * R or seg4.shape[2] != w * R:
            raise ValueError("segmap size must be an integer multiple of the feature size")
        extra = (self.norm_s.param_free_norm,) if self.learned_shortcut else ()
        if self.training:
            ns0, nh0, _, _ = self.norm_0.param_free_norm.scale_shift(x, x_shift, extra)
            nss, nhs = ns0, nh0
        else:
            if save is not None:
                raise RuntimeError("michigan_b200: the backward pass is implemented for train-mode batch statistics")
            ns0, nh0 = self.norm_0.param_free_norm.scale_shift(x)
            if self.learned_shortcut:
                nss, nhs = self.norm_s.param_free_norm.scale_shift(x)

        gfmt, gsplit = precision.gb_policy(R, self.training)

        def spade_act(name, src, shift, nscale, nshift, act):
            """-> (tensor-core operand (fmt, hi, lo) holding act(SPADE(src)) for the consumer conv, saved state | None)."""
            cfmt = precision.conv_fmt(src.shape[-1])
            wsh, bsh, wgb, g1b, bb = self._spade_pack(name, gfmt, gsplit)
            kw_a, get_a = precision.out_spec(gfmt, gsplit)
            actv = get_a(ops.mlp_shared(seg4, wsh, bsh, seg_resize=R, act=ops.ACT_RELU, out_hw=(h, w), **kw_a))
            c = src.shape[-1]
            sp_args = (src, shift, nscale, nshift, g1b, bb)
            if save is None:
                kw_h, get_h = precision.out_spec(cfmt, cfmt == ops.BF16)
                return get_h(precision.conv(actv, wgb, c, 3, 3, 1, 1, act=act, spade=sp_args, **kw_h)), None
            g1 = torch.empty((N, h, w, c), device=src.device, dtype=torch.float32)
            if cfmt == ops.TF32:
                h32 = precision.conv(actv, wgb, c, 3, 3, 1, 1, act=act, spade=sp_args, round_out=True, aux=g1)
                operand = (ops.TF32, h32, None)
            else:
                h32, hi, lo = precision.conv(actv, wgb, c, 3, 3, 1, 1, act=act, spade=sp_args, out16=(cfmt, True), aux=g1)
                operand = (cfmt, hi, lo)
            S = SimpleNamespace(sp=getattr(self, name), src=src, shift=shift, ns=nscale, nh=nshift, act=act, g1=g1, h=h32,
                                wsh=wsh, R=R, hw=(h, w))
            if cfmt == ops.BF16 and precision.conv_grad_fmt() == ops.BF16:
                S.h16 = operand[1]          # the forward's bf16 hi operand doubles as the weight-gradient GEMM's input
            return operand, S

        if save is not None:
            save.x, save.xs, save.blend, save.hw = x, x_shift, blend, (h, w)
        if self.learned_shortcut:
            hs_, sps = spade_act("norm_s", x, x_shift, nss, nhs, ops.ACT_NONE)
            x_s = precision.conv(hs_, self._conv_pack("conv_s", inv_sigma_of), self.fout, 1, 1, 1, 0)
            res, res_shift = x_s, 0
            del hs_
            if save is not None:
                save.sps = sps
        else:
            res, res_shift = x, x_shift
        h0, sp0 = spade_act("norm_0", x, x_shift, ns0, nh0, ops.ACT_LRELU)
        dx = precision.conv(h0, self._conv_pack("conv_0", inv_sigma_of), self.fmiddle, 3, 3, 1, 1, bias=self.conv_0.bias.detach())
        del h0
        ns1, nh1 = self.norm_1.param_free_norm.scale_shift(dx)[:2]
        h1, sp1 = spade_act("norm_1", dx, 0, ns1, nh1, ops.ACT_LRELU)
        out = precision.conv(h1, self._conv_pack("conv_1", inv_sigma_of), self.fout, 3, 3, 1, 1, bias=self.conv_1.bias.detach(),
                             res=res, res_shift=res_shift, blend=blend)
        if save is not None:
            save.sp0, save.sp1, save.dx = sp0, sp1, dx
        return out

    def forward(self, x, seg):
        """Reference signature (architecture.py:67): NCHW x and seg -> NCHW out."""
        from .prep import SpectralNormBatch
        if not hasattr(self, "_snb"):
            self._snb = SpectralNormBatch(self.sn_convs())
        inv = self._snb.run(self.training)
        inv_of = {c: inv[i:i + 1] for i, c in enumerate(self._snb.convs)}
        out = self.forward_nhwc(ops.nchw_to_nhwc(x.contiguous()), 0, ops.nchw_to_nhwc(seg.contiguous()), inv_of)
        return out.permute(0, 3, 1, 2)

    def shortcut(self, x, seg):
        raise RuntimeError("the shortcut branch is fused into forward()")

    def actvn(self, x):
        raise RuntimeError("LeakyReLU(0.2) is fused into the SPADE epilogue")
