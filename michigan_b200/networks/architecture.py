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

from .. import _lib, ops, precision
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


# ================================================================================================ VGG19
VGG19_WEIGHTS_FILE = "vgg19-dcbb9e9d.pth"
_VGG_CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, 256, "M", 512, 512, 512, 512, "M", 512]   # features[0:30]
_VGG_SLICES = [(0, 2), (2, 7), (7, 12), (12, 21), (21, 30)]                                   # ends: relu1_1 .. relu5_1


class VGGWeightsMissing(FileNotFoundError, NotImplementedError):
    """The ImageNet VGG19 weights are not available locally.  Nothing is downloaded; like every loss the stand-alone model
    cannot compute, it is refused (NotImplementedError), and the message names the file that would enable it."""


def vgg19_weights_path():
    """Where torchvision itself caches the VGG19 ImageNet weights (torchvision.models.VGG19_Weights.IMAGENET1K_V1)."""
    import os
    return os.path.join(torch.hub.get_dir(), "checkpoints", VGG19_WEIGHTS_FILE)


def _vgg_features():
    """torchvision.models.vgg19().features[0:30] as plain modules (same indices, so the same state-dict keys)."""
    layers, cin = [], 3
    for v in _VGG_CFG:
        if v == "M":
            layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
        else:
            layers += [nn.Conv2d(cin, v, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
            cin = v
    return layers


class VGG19(nn.Module):
    """architecture.py:160-190: torchvision's vgg19().features[0:30] in five slices ending at relu1_1 .. relu5_1, state-dict keys
    `sliceK.<feature index>.{weight,bias}`, frozen.  The weights are never downloaded: `state_dict` (torchvision layout
    `features.N.*`, or this module's own keys) or else the file torchvision would use (`vgg19_weights_path()`).

    On the sm_90a kernels: conv1_1 is a thin direct conv of the 4-channel padded image, every other conv the wgmma implicit GEMM
    (the 3x3 group kernel where the shape allows) with bias and ReLU fused, 16-bit operands in one pass (precision.gb_fmt);
    the max-pools read and write those operands (mg_maxpool2_nhwc).  Only the five taps are produced in fp32."""

    CONVS = [0, 2, 5, 7, 10, 12, 14, 16, 19, 21, 23, 25, 28]      # feature indices of the 13 convs
    POOLED = {2, 7, 16, 25}                                        # convs whose ReLU output is max-pooled
    TAPS = {0: 0, 5: 1, 10: 2, 19: 3, 28: 4}                       # convs whose ReLU output is a loss tap -> tap index

    def __init__(self, requires_grad=False, state_dict=None):
        super().__init__()
        if requires_grad:
            raise NotImplementedError("michigan_b200: VGG19 is frozen (the perceptual loss never trains it)")
        feats = _vgg_features()
        for k, (a, b) in enumerate(_VGG_SLICES):
            s = nn.Sequential()
            for x in range(a, b):
                s.add_module(str(x), feats[x])
            setattr(self, "slice%d" % (k + 1), s)
        if state_dict is None:
            import os
            path = vgg19_weights_path()
            if not os.path.exists(path):
                raise VGGWeightsMissing("michigan_b200: the VGG loss needs the ImageNet VGG19 weights at %s (torchvision's cache; "
                                        "nothing is downloaded) or an explicit state_dict" % path)
            state_dict = torch.load(path, map_location="cpu", weights_only=True)
        self.load_state_dict(self.from_torchvision(state_dict))
        for p in self.parameters():
            p.requires_grad_(False)
        self._cache = PackCache()

    @staticmethod
    def from_torchvision(sd):
        """torchvision `features.N.*` keys (N < 30) -> `sliceK.N.*`; a state dict already in this layout is returned as is."""
        if not any(k.startswith("features.") for k in sd):
            return sd
        out = {}
        for k, v in sd.items():
            if not k.startswith("features."):
                continue
            idx = int(k.split(".")[1])
            if idx >= 30:
                continue
            s = next(i for i, (a, b) in enumerate(_VGG_SLICES) if a <= idx < b)
            out["slice%d.%s" % (s + 1, k[len("features."):])] = v
        return out

    def conv(self, f):
        s = next(i for i, (a, b) in enumerate(_VGG_SLICES) if a <= f < b)
        return getattr(self, "slice%d" % (s + 1))[f - _VGG_SLICES[s][0]]

    # ------------------------------------------------------------------ operands
    def _fwd_pack(self, f, fmt):
        cv = self.conv(f)
        if f == 0:
            return self._cache.get("w0", [cv.weight], lambda: ops.pack_weight_thin(cv.weight.detach(), 4))
        if fmt == ops.TF32:
            return self._cache.get(("w", f, fmt), [cv.weight], lambda: ops.pack_weight(cv.weight.detach(), None, True))
        return self._cache.get(("w", f, fmt), [cv.weight], lambda: ops.pack_weight16(cv.weight.detach(), None, fmt, split=False))

    def _dgrad_pack(self, f, fmt):
        """Flipped / transposed 3x3 weights [Cin][9*Cout] of the data-gradient GEMM (ops.conv_dgrad's packing, kept)."""
        cv = self.conv(f)

        def build():
            O, I = cv.weight.shape[:2]
            wp = torch.empty((I, 9 * O), device=cv.weight.device, dtype=torch.float32)
            _lib.check(_lib.load().mg_pack_weight_dgrad(cv.weight.detach().data_ptr(), wp.data_ptr(), O, I, 3, 3, 1, 0, 3, 0, 3, None,
                                                        ops._stream()), "mg_pack_weight_dgrad")
            return wp if fmt == ops.TF32 else ops.cvt16(wp, fmt)
        return self._cache.get(("d", f, fmt), [cv.weight], build)

    # ------------------------------------------------------------------ forward / backward
    def run(self, x8, n_save=0):
        """x8: [B,H,W,4] NHWC image (channel 3 zero) -> (five fp32 NHWC taps, saved state or None).
        n_save > 0 keeps, for the first n_save images, what backward() needs: each ReLU output that is pooled or masked."""
        fmt = precision.gb_fmt(64)

        def kw(want_f32):
            if fmt == ops.TF32:
                return dict(round_out=True)
            return dict(out16=(fmt, False), want_f32=want_f32)

        taps, layers = [None] * 5, []
        opnd = None
        for i, f in enumerate(self.CONVS):
            cv = self.conv(f)
            tap = self.TAPS.get(f)
            last = f == self.CONVS[-1]
            if last and fmt != ops.TF32:
                k = {}
            else:
                k = kw(tap is not None)
            if f == 0:
                r = ops.conv_thin(x8, self._fwd_pack(0, fmt), cv.bias.detach(), 64, 3, 3, 1, 1, act=ops.ACT_RELU, **k)
            else:
                r = ops.conv_igemm(opnd, self._fwd_pack(f, fmt), cv.out_channels, 3, 3, 1, 1, bias=cv.bias.detach(), act=ops.ACT_RELU,
                                   a_fmt=fmt, **k)
            if fmt == ops.TF32 or last:
                a32, a16 = r, None
            else:
                a32, a16 = r[0], r[1]
            if tap is not None:
                taps[tap] = a32
            a = a32 if a32 is not None else a16          # the tensor the ReLU mask (and a pool's arg-max) is taken from
            if n_save:
                layers.append(SimpleNamespace(f=f, a=a[:n_save], tap=tap, pooled=f in self.POOLED, cin=cv.in_channels))
            opnd = a16 if a16 is not None else a32
            if f in self.POOLED:
                opnd = ops.maxpool2(opnd) if fmt == ops.TF32 else ops.maxpool2(opnd, out16=fmt, want_f32=False)[1]
        return taps, (SimpleNamespace(layers=layers, fmt=fmt) if n_save else None)

    def backward(self, S, gtaps, img_hw):
        """gtaps: fp32 NHWC gradients w.r.t. the five taps of the saved images -> d image [n,3,H,W] (NCHW fp32)."""
        g16 = precision.conv_grad_fmt() == ops.BF16
        d = None                                   # gradient w.r.t. the ReLU output of the current layer (or its pooled view)
        for L in reversed(S.layers):
            add = gtaps[L.tap] if L.tap is not None else None
            first = L.f == 0
            want16 = g16 and not first             # conv1_1's data gradient (thin_dgrad3) reads fp32
            if L.pooled:
                r = ops.maxpool2_relu_bwd(d, L.a, add=add, want_f32=not want16, want16=want16)
            elif d is None:
                r = ops.relu_bwd16(add, L.a, want_f32=not want16, want16=want16)
            else:
                r = ops.relu_bwd16(d, L.a, add=add, want_f32=not want16, want16=want16)
            dz = r[1] if want16 else r
            del d
            if first:
                n = dz.shape[0]
                dimg = torch.zeros((n, 3) + tuple(img_hw), device=dz.device, dtype=torch.float32)
                ops.thin_dgrad3(dz, self._fwd_pack(0, S.fmt), dimg, 3, 3, 1, 1, 0)
                return dimg
            _, Hh, Ww, _ = dz.shape
            gfmt = ops.BF16 if want16 else ops.TF32
            _, _, ph = ops.dgrad_geometry(3, 1, 1, 0)
            d = ops.conv_igemm(dz, self._dgrad_pack(L.f, gfmt), L.cin, 3, 3, 1, 0, out_hw=(Hh, Ww), a_fmt=gfmt,
                               _extra=dict(pad_h_extra=ph, pad_w_extra=ph, out_stride=1, OHF=Hh, OWF=Ww))
            del dz

    def forward(self, X):
        """Reference signature (architecture.py:182-189): NCHW image -> [h_relu1 .. h_relu5] (NCHW-shaped views of NHWC fp32).
        Gradients flow through VGGLoss only (its backward is hand-written)."""
        if torch.is_grad_enabled() and X.requires_grad:
            raise NotImplementedError("michigan_b200: differentiate through VGG19 via VGGLoss")
        taps, _ = self.run(ops.nchw_to_nhwc(X.contiguous(), 4))
        return [t.permute(0, 3, 1, 2) for t in taps]
