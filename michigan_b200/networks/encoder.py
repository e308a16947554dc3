"""Sub-networks instantiated inside SPADEBGenerator: the three reference-image encoders of --use_encoder
(--Image_encoder_mode partialconv: ImageEncoder3, reference models/networks/encoder.py:160-225, partialconv2d.py:15-85;
instance: ImageEncoder2, encoder.py:107-158; norm: ImageEncoder, encoder.py:61-105) and the background encoder
(encoder.py:271-341, MaskGAN_networks.py:114-173); and the --use_vae image encoder `ConvEncoder` (encoder.py:17-59, the
reference's netE).  Same constructors and state-dict keys; forward on the CUDA kernels, NHWC inside."""
import random
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn as nn

from .. import ops, precision
from .base_network import BaseNetwork
from .normalization import get_nonspade_norm_layer
from .prep import PackCache, SpectralNormBatch


class PartialConv2d(nn.Conv2d):
    """Parameter container with partialconv2d.py's constructor (multi_channel / return_mask kwargs)."""

    def __init__(self, *args, **kwargs):
        self.multi_channel = kwargs.pop("multi_channel", False)
        self.return_mask = kwargs.pop("return_mask", False)
        super().__init__(*args, **kwargs)
        if self.multi_channel:
            raise NotImplementedError("michigan_b200: multi-channel partial-conv masks are unused by spadeb")

    def forward(self, input, mask_in=None):
        raise RuntimeError("PartialConv2d is executed by ImageEncoder3's fused kernels")


class ImageEncoder3(BaseNetwork):
    """encoder.py:160-225 with norm_ref_encode='instance' (the default, base_options.py:94)."""

    def __init__(self, opt, sw, sh):
        super().__init__()
        kw = 3
        pw = int(np.ceil((kw - 1.0) / 2))
        ndf = opt.ngf
        self.sw, self.sh, self.opt = sw, sh, opt
        self.layer1 = PartialConv2d(3, ndf, kw, stride=2, padding=pw, return_mask=True)
        self.norm1 = nn.InstanceNorm2d(ndf, affine=False)
        self.layer2 = PartialConv2d(ndf * 1, ndf * 2, kw, stride=2, padding=pw, return_mask=True)
        self.norm2 = nn.InstanceNorm2d(ndf * 2, affine=False)
        self.layer3 = PartialConv2d(ndf * 2, ndf * 4, kw, stride=2, padding=pw, return_mask=True)
        self.norm3 = nn.InstanceNorm2d(ndf * 4, affine=False)
        self.layer4 = PartialConv2d(ndf * 4, ndf * 8, kw, stride=2, padding=pw, return_mask=True)
        self.norm4 = nn.InstanceNorm2d(ndf * 8, affine=False)
        self.layer5 = PartialConv2d(ndf * 8, ndf * 16, kw, stride=2, padding=pw, return_mask=True)
        self.norm5 = nn.InstanceNorm2d(ndf * 16, affine=False)
        self.actvn = nn.LeakyReLU(0.2, False)
        if "instance" not in opt.norm_ref_encode:
            raise NotImplementedError("michigan_b200: norm_ref_encode must be 'instance'")
        if ndf % 32 != 0:
            raise NotImplementedError("michigan_b200: ngf must be a multiple of 32")
        self._cache = PackCache()

    def forward_nhwc(self, image_ref, label_ref0, label_tag0, save=None):
        """image_ref [N,3,H,W] NCHW, label_* [N,1,H,W] -> [N,sh,sw,16*ngf] NHWC.
        save: namespace filled with what autograd.fc_bwd needs (same arithmetic either way)."""
        N, _, H, W = image_ref.shape
        mref = label_ref0.reshape(N, H, W).contiguous()
        mtag = label_tag0.reshape(N, H, W).contiguous()
        c = self._cache
        # layer 1: thin direct conv on image*mask
        x0 = ops.nchw_to_nhwc(image_ref.contiguous(), 4, pmul=mref)
        ratio, upd = ops.partial_mask(mref, 3, 2, 1)
        w1 = c.get("l1", [self.layer1.weight], lambda: ops.pack_weight_thin(self.layer1.weight.detach(), 4))
        x = ops.conv_thin(x0, w1, self.layer1.bias.detach(), self.layer1.out_channels, 3, 3, 2, 1, pscale=ratio, pmul=upd)
        if save is not None:
            save.mref, save.mtag, save.x0, save.wt1, save.layers = mref, mtag, x0, w1, []
            save.l1 = SimpleNamespace(ratio=ratio, upd=upd, y=x)
        for i in range(2, 6):
            # lrelu(IN(x)) * mask as a tensor-core operand of the next partial conv (partialconv2d.py:69)
            fmt = precision.conv_fmt(x.shape[-1])
            if save is None:
                kw_o, get_o = precision.out_spec(fmt, fmt == ops.BF16)
                xo = get_o(ops.instance_norm_act(x, ops.ACT_LRELU, 1e-5, pmul=upd, **kw_o))
            elif fmt == ops.TF32:
                a32, ss = ops.instance_norm_act_fwd(x, ops.ACT_LRELU, 1e-5, round_out=True, pmul=upd)
                xo = (ops.TF32, a32, None)
            else:
                a32, ss, hi, lo = ops.instance_norm_act_fwd(x, ops.ACT_LRELU, 1e-5, pmul=upd, out16=(fmt, True))
                xo = (fmt, hi, lo)
            ratio, upd_next = ops.partial_mask(upd, 3, 2, 1)
            layer = getattr(self, "layer%d" % i)
            wp = c.get(("l%d" % i, fmt), [layer.weight], lambda layer=layer: precision.pack_conv(layer.weight.detach(), None, fmt))
            y = precision.conv(xo, wp, layer.out_channels, 3, 3, 2, 1, bias=layer.bias.detach(), pscale=ratio, pmul=upd_next)
            if save is not None:
                save.layers.append(SimpleNamespace(layer=layer, a=a32, ss=ss, y_in=x, pm_in=upd, ratio=ratio, upd=upd_next))
            x, upd = y, upd_next
        if save is None:
            a6 = ops.instance_norm_act(x, ops.ACT_LRELU, 1e-5)
        else:
            a6, ss6 = ops.instance_norm_act_fwd(x, ops.ACT_LRELU, 1e-5)
            save.y5, save.ss6 = x, ss6
        out = ops.masked_mean_bcast(a6, mref, mtag)
        if save is not None:
            save.mhw = (out.shape[1], out.shape[2])
        if self.sh != out.shape[1]:
            out = ops.resize_bilinear(out, self.sh, self.sw)
        return out

    def backward_nhwc(self, G, S, dout):
        """Parameter gradients into G (autograd._Grads) given dout, the gradient of forward_nhwc's output."""
        from .autograd import fc_bwd
        fc_bwd(G, self, S, dout)

    def forward(self, x, label_ref0, label_tag0):
        return self.forward_nhwc(x, label_ref0, label_tag0).permute(0, 3, 1, 2)


class ConvBlock(nn.Module):
    """MaskGAN_networks.py:114-173, the configuration BackgroundEncode2 uses (norm='none', reflect pad)."""

    def __init__(self, input_dim, output_dim, kernel_size, stride, padding=0, norm="none", activation="relu", pad_type="zero"):
        super().__init__()
        if norm != "none" or activation != "relu" or pad_type != "reflect":
            raise NotImplementedError("michigan_b200: ConvBlock supports norm='none', activation='relu', pad_type='reflect'")
        self.use_bias = True
        self.pad = nn.ReflectionPad2d(padding)
        self.norm = None
        self.activation = nn.ReLU(inplace=True)
        self.conv = nn.Conv2d(input_dim, output_dim, kernel_size, stride, bias=self.use_bias)
        self.padding, self.kernel_size, self.stride = padding, kernel_size, stride


class BackgroundEncode2(BaseNetwork):
    """encoder.py:271-341 (num_upsampling_layers != 'most')."""

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        self.ngf = opt.ngf
        if opt.num_upsampling_layers == "most":
            raise NotImplementedError("michigan_b200: num_upsampling_layers='most' is not on the benchmark path")
        self.conv1 = ConvBlock(3, self.ngf, 7, 1, 3, norm="none", activation="relu", pad_type="reflect")
        self.layer1 = ConvBlock(self.ngf, 2 * self.ngf, 4, 2, 1, norm="none", activation="relu", pad_type="reflect")
        self.layer2 = ConvBlock(2 * self.ngf, 4 * self.ngf, 4, 2, 1, norm="none", activation="relu", pad_type="reflect")
        self.layer3 = ConvBlock(4 * self.ngf, 8 * self.ngf, 4, 2, 1, norm="none", activation="relu", pad_type="reflect")
        # present in the reference's state dict, never executed (encoder.py:284 vs 323-330)
        self.layer4 = ConvBlock(8 * self.ngf, 16 * self.ngf, 4, 2, 1, norm="none", activation="relu", pad_type="reflect")
        self._cache = PackCache()

    def back_mask(self, mask):
        """[N,H,W] complement of the dilated hair mask (encoder.py:286-316).  The train/eval switch is
        opt.isTrain, as in the reference; the dilation size is drawn with Python's `random` there too."""
        opt = self.opt
        hair = mask[:, 1].contiguous()
        if opt.isTrain:
            if opt.random_expand_mask:
                mh = hair.shape[1]
                th = int(mh * opt.random_expand_th)
                th = th if th % 2 == 1 else th + 1
                k = random.choice([max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4])
                return ops.maxpool_mask(hair, k, invert=True)
            return mask[:, 0].contiguous()
        if opt.expand_mask_be:
            k = opt.expand_th
            if opt.add_feat_zeros:
                th = opt.add_th
                H = W = opt.crop_size
                o = int(th / 2)
                inner = ops.maxpool_mask(hair[:, o:o + H, o:o + W].contiguous(), k, invert=False)
                e = torch.zeros_like(hair)
                e[:, o:o + H, o:o + W] = inner
                return (1 - e).contiguous()
            return ops.maxpool_mask(hair, k, invert=True)
        return mask[:, 0].contiguous()

    def forward_nhwc(self, image, mask, noise, save=None):
        """Returns ([x3,x2,x1,x0] NHWC features, back_mask [N,H,W]).  save: namespace for autograd.bg_bwd."""
        back = self.back_mask(mask)
        if self.opt.random_noise_background:
            inp = ops.nchw_to_nhwc(noise.contiguous(), 4)
        else:
            inp = ops.prep_bginput(image.contiguous(), noise.contiguous(), back)
        c = self._cache
        w1 = c.get("c1", [self.conv1.conv.weight], lambda: ops.pack_weight_thin(self.conv1.conv.weight.detach(), 4))
        x0 = ops.conv_thin(inp, w1, self.conv1.conv.bias.detach(), self.ngf, 7, 7, 1, 3, pad_mode=1, act=ops.ACT_RELU)
        if save is not None:
            save.inp, save.wt1, save.x0, save.layers = inp, w1, x0, []
        feats = [x0]
        x = x0
        for name in ("layer1", "layer2", "layer3"):
            blk = getattr(self, name)
            fmt = precision.conv_fmt(x.shape[-1])
            wp = c.get((name, fmt), [blk.conv.weight], lambda blk=blk: precision.pack_conv(blk.conv.weight.detach(), None, fmt))
            if fmt == ops.TF32:
                xp32 = ops.reflect_pad(x, 1, round_tf32=True)
                xp = (ops.TF32, xp32, None)
            else:
                xp32, hi, lo = ops.reflect_pad(x, 1, out16=(fmt, True), want_f32=save is not None)
                xp = (fmt, hi, lo)
            x = precision.conv(xp, wp, blk.conv.out_channels, 4, 4, 2, 0, bias=blk.conv.bias.detach(), act=ops.ACT_RELU)
            if save is not None:
                save.layers.append(SimpleNamespace(blk=blk, xp=xp32, y=x))
            feats.append(x)
        return feats[::-1], back

    def forward(self, image, mask, noise):
        feats, back = self.forward_nhwc(image, mask, noise)
        import torch.nn.functional as F
        bm = back.unsqueeze(1)
        sh, sw = bm.shape[2:]
        masks = [F.interpolate(bm, size=(int(sh / d), int(sw / d)), mode="nearest") for d in (8, 4, 2)] + [bm]
        return [f.permute(0, 3, 1, 2) for f in feats], masks


def norm_act(y, fmt, saving):
    """lrelu(IN(y)) as a tensor-core operand of `fmt` -> (operand, fp32 value, IN table); the last two only when saving
    (what the backward reads), else None."""
    if not saving:
        kw_o, get_o = precision.out_spec(fmt, fmt == ops.BF16)
        return get_o(ops.instance_norm_act(y, ops.ACT_LRELU, 1e-5, **kw_o)), None, None
    if fmt == ops.TF32:
        a32, ss = ops.instance_norm_act_fwd(y, ops.ACT_LRELU, 1e-5, round_out=True)
        return (ops.TF32, a32, None), a32, ss
    a32, ss, hi, lo = ops.instance_norm_act_fwd(y, ops.ACT_LRELU, 1e-5, out16=(fmt, True))
    return (fmt, hi, lo), a32, ss


class SNConvStack(BaseNetwork):
    """The layer stack ConvEncoder, ImageEncoder and ImageEncoder2 share (encoder.py:46-51, 89-94, 136-140): `layerK` =
    norm_E(Conv2d(k3, s2, p1)), i.e. spectral norm, bias removed, InstanceNorm2d without affine; LeakyReLU 0.2 between
    layers.  Layer 1 is the thin direct conv (its 3-channel input is too narrow for the implicit GEMM), the others the
    implicit-GEMM conv under the precision.conv_fmt policy.  Training runs one in-place power iteration of every conv in
    convs() per forward, as torch's spectral_norm hook does (also under no_grad); eval uses the stored u, v.  The
    backward is autograd.sn_conv_stack_bwd."""

    n_stack = 0   # layer1 .. layer<n_stack> run; anything after them (ImageEncoder.layer6) is only in the state dict

    def _check_opt(self, opt):
        if opt.norm_E not in ("spectralinstance", "instance"):
            raise NotImplementedError("michigan_b200: norm_E '%s' has no CUDA kernel (supported: [spectral]instance)" % opt.norm_E)
        if opt.ngf % 32 != 0:
            raise NotImplementedError("michigan_b200: ngf must be a multiple of 32")

    def convs(self):
        return [getattr(self, "layer%d" % i)[0] for i in range(1, self.n_stack + 1)]

    def spectral_batch(self):
        if getattr(self, "_snb", None) is None:
            self._snb = SpectralNormBatch([c for c in self.convs() if hasattr(c, "weight_orig")])
        return self._snb

    def run_stack(self, x, save):
        """x: the NHWC image, 4 channels (4th zero) -> the raw [N,h,w,C] output of the last conv, before its InstanceNorm.
        save: namespace filled with what autograd.sn_conv_stack_bwd needs (same arithmetic either way)."""
        snb = self.spectral_batch()
        inv = snb.run(self.training)
        # the backward keeps this forward's 1/sigma: the D step's no-grad forward re-runs the power iteration before it
        inv_of = {cv: (inv[i:i + 1].clone() if save is not None else inv[i:i + 1]) for i, cv in enumerate(snb.convs)}

        def weight(conv):
            return (conv.weight_orig, inv_of[conv]) if hasattr(conv, "weight_orig") else (conv.weight, None)

        convs = self.convs()
        w1, isg1 = weight(convs[0])
        # W / sigma of a 27*ngf-element weight, scaled on the device before packing (the thin conv has no sigma input)
        wt1 = ops.pack_weight_thin(w1.detach() * isg1 if isg1 is not None else w1.detach(), 4)
        y = ops.conv_thin(x, wt1, None, convs[0].out_channels, 3, 3, 2, 1)
        if save is not None:
            save.x0, save.inv_of, save.layers = x, inv_of, []
            save.y1 = y
        for conv in convs[1:]:
            fmt = precision.conv_fmt(y.shape[-1])
            xo, a32, ss = norm_act(y, fmt, save is not None)
            w, isg = weight(conv)
            wp = precision.pack_conv(w.detach(), isg, fmt)
            y_next = precision.conv(xo, wp, conv.out_channels, 3, 3, 2, 1)
            if save is not None:
                save.layers.append(SimpleNamespace(conv=conv, a=a32, ss=ss, y_in=y))
            y = y_next
        return y

    def last_norm_act(self, y, save):
        """lrelu(IN(y)) in fp32 after the last conv of the stack (the pooled encoders' tail); save keeps y and its IN table."""
        if save is None:
            return ops.instance_norm_act(y, ops.ACT_LRELU, 1e-5)
        a, ss = ops.instance_norm_act_fwd(y, ops.ACT_LRELU, 1e-5)
        save.y_last, save.ss_last = y, ss
        return a


def latent_weight(cache, fc, sh, sw):
    """fc.weight [O, K] (Linear) or [O, K, 1, 1] (1x1 Conv2d), O = C*sh*sw, with its rows permuted from the NCHW order
    (c, h, w) of the reference's view to the NHWC order (h, w, c) of the map, TF32-packed as a 1x1 conv; and the bias
    permuted alike (cached in `cache` until they change)."""
    def build():
        hw, k = sh * sw, fc.weight.shape[1]
        w = fc.weight.detach().reshape(-1, hw, k).transpose(0, 1).reshape(-1, k, 1, 1)
        b = fc.bias.detach().view(-1, hw).t().contiguous().view(-1)
        return ops.pack_weight(w.contiguous(), None, True), b
    return cache.get("fc", [fc.weight, fc.bias], build)


def latent_head(cache, fc, z, sh, sw, save):
    """fc(z) viewed as [N, C, sh, sw] (generator.py:110-116, encoder.py:99-101), written as the [N,sh,sw,C] NHWC map: one
    1x1 GEMM over the N rows of z [N, K] with the permuted weight and the bias in its epilogue.  save: keeps z and the
    packed weight for autograd.latent_bwd."""
    N = z.shape[0]
    z4 = z.detach().float().contiguous().view(N, 1, 1, -1)
    wp, b = latent_weight(cache, fc, sh, sw)
    x = ops.conv_igemm(z4, wp, wp.shape[0], 1, 1, 1, 0, bias=b).view(N, sh, sw, -1)
    if save is not None:
        save.z4, save.wp = z4, wp
    return x


class ImageEncoder(SNConvStack):
    """encoder.py:61-105, --Image_encoder_mode norm: the image is resized to 256x256 (bilinear, align_corners=False), five
    layers give a [N, 16ngf, 8, 8] map, then LeakyReLU, AdaptiveAvgPool2d(1) and fc = Conv2d(16ngf, 16ngf*sh*sw, 1), viewed
    as [N, 16ngf, sh, sw].  The labels are ignored.  layer6 (crop_size >= 256) is in the reference's state dict but never
    runs: its u, v never change and its gradient stays None.  On the kernels: the pool is mg_masked_mean_bcast without
    masks, fc the latent head's 1x1 GEMM over the N pooled rows (latent_head)."""

    n_stack = 5

    def __init__(self, opt, sw, sh):
        super().__init__()
        self._check_opt(opt)
        kw = 3
        pw = int(np.ceil((kw - 1.0) / 2))
        ndf = opt.ngf
        self.sw, self.sh, self.opt = sw, sh, opt
        norm_layer = get_nonspade_norm_layer(opt, opt.norm_E)
        self.layer1 = norm_layer(nn.Conv2d(3, ndf, kw, stride=2, padding=pw))
        self.layer2 = norm_layer(nn.Conv2d(ndf * 1, ndf * 2, kw, stride=2, padding=pw))
        self.layer3 = norm_layer(nn.Conv2d(ndf * 2, ndf * 4, kw, stride=2, padding=pw))
        self.layer4 = norm_layer(nn.Conv2d(ndf * 4, ndf * 8, kw, stride=2, padding=pw))
        self.layer5 = norm_layer(nn.Conv2d(ndf * 8, ndf * 16, kw, stride=2, padding=pw))
        if opt.crop_size >= 256:
            self.layer6 = norm_layer(nn.Conv2d(ndf * 8, ndf * 8, kw, stride=2, padding=pw))
        self.so = 4
        self.adaptivepool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Conv2d(ndf * 16, ndf * 16 * self.sw * self.sh, 1, 1, 0)
        self.actvn = nn.LeakyReLU(0.2, False)
        self._snb = None
        self._cache = PackCache()

    def forward_nhwc(self, image_ref, label_ref0=None, label_tag0=None, save=None):
        """image_ref [N,3,H,W] NCHW -> [N,sh,sw,16ngf] NHWC.  save: namespace for backward_nhwc."""
        _, _, H, W = image_ref.shape
        x = ops.nchw_to_nhwc(image_ref.detach().contiguous(), 4)
        if (H, W) != (256, 256):
            x = ops.resize_bilinear(x, 256, 256)                               # encoder.py:86-87
        a = self.last_norm_act(self.run_stack(x, save), save)
        pooled = ops.masked_mean_bcast(a, None, None)[:, 0, 0]                 # AdaptiveAvgPool2d(1): [N, 16ngf]
        return latent_head(self._cache, self.fc, pooled, self.sh, self.sw, save)

    def backward_nhwc(self, G, S, dout):
        """Parameter gradients into G (autograd._Grads) given dout, the gradient of forward_nhwc's output."""
        from .autograd import latent_bwd, sn_conv_stack_bwd
        dpooled = latent_bwd(G, self.fc, S, dout)
        N, h, w, C = S.y_last.shape
        dmap = torch.zeros((N, h, w, C), device=dout.device, dtype=torch.float32)
        dmap[:, 0, 0] = dpooled           # the adjoint of taking pixel (0, 0) of the broadcast mean
        da = ops.masked_mean_bcast_bwd(dmap, None, None)
        sn_conv_stack_bwd(G, self.convs(), S, ops.in_bwd(da, S.y_last, S.ss_last, ops.ACT_LRELU, round_tf32=True))

    def forward(self, x, label_ref=None, label_tag=None):
        return self.forward_nhwc(x).permute(0, 3, 1, 2)


class ImageEncoder2(SNConvStack):
    """encoder.py:107-158, --Image_encoder_mode instance: five layers take the image from H to H/32 (no resize), then
    LeakyReLU; per image and channel the mean over the reference hair, sum(x * ref) / max(sum(ref), 1), or the plain spatial
    mean under --ref_global_pool, broadcast onto the target hair.  Both labels are nearest-resized to the map; the result is
    nearest-resized to (sh, sw) when sh differs from the map's height.  On the kernels: mg_masked_mean_bcast, whose mask reads
    are that nearest resize, and a strided pick for the second one (an integer multiple is required)."""

    n_stack = 5

    def __init__(self, opt, sw, sh):
        super().__init__()
        self._check_opt(opt)
        kw = 3
        pw = int(np.ceil((kw - 1.0) / 2))
        ndf = opt.ngf
        self.sw, self.sh, self.opt = sw, sh, opt
        norm_layer = get_nonspade_norm_layer(opt, opt.norm_E)
        self.layer1 = norm_layer(nn.Conv2d(3, ndf, kw, stride=2, padding=pw))
        self.layer2 = norm_layer(nn.Conv2d(ndf * 1, ndf * 2, kw, stride=2, padding=pw))
        self.layer3 = norm_layer(nn.Conv2d(ndf * 2, ndf * 4, kw, stride=2, padding=pw))
        self.layer4 = norm_layer(nn.Conv2d(ndf * 4, ndf * 8, kw, stride=2, padding=pw))
        self.layer5 = norm_layer(nn.Conv2d(ndf * 8, ndf * 16, kw, stride=2, padding=pw))
        self.actvn = nn.LeakyReLU(0.2, False)
        self._snb = None

    def _pick(self, xh, xw):
        """The integer stride of the nearest resize from the (xh, xw) map to (sh, sw), or None when there is none."""
        if self.sh == xh:
            return None
        if xh % self.sh or xw % self.sw:
            raise NotImplementedError("michigan_b200: ImageEncoder2's %dx%d map is not an integer multiple of the %dx%d "
                                      "latent size" % (xh, xw, self.sh, self.sw))
        return xh // self.sh, xw // self.sw

    def forward_nhwc(self, image_ref, label_ref0, label_tag0, save=None):
        """image_ref [N,3,H,W] NCHW, label_* [N,1,H,W] -> [N,sh,sw,16ngf] NHWC.  save: namespace for backward_nhwc."""
        N, _, H, W = image_ref.shape
        x = ops.nchw_to_nhwc(image_ref.detach().contiguous(), 4)
        a = self.last_norm_act(self.run_stack(x, save), save)
        pick = self._pick(a.shape[1], a.shape[2])
        mref = None if getattr(self.opt, "ref_global_pool", False) else label_ref0.reshape(N, H, W).contiguous()
        mtag = label_tag0.reshape(N, H, W).contiguous()
        out = ops.masked_mean_bcast(a, mref, mtag)
        if save is not None:
            save.mref, save.mtag, save.pick = mref, mtag, pick
        if pick is not None:
            out = out[:, ::pick[0], ::pick[1]].contiguous()
        return out

    def backward_nhwc(self, G, S, dout):
        """Parameter gradients into G (autograd._Grads) given dout, the gradient of forward_nhwc's output."""
        from .autograd import sn_conv_stack_bwd
        d = dout
        if S.pick is not None:
            d = torch.zeros(S.y_last.shape, device=dout.device, dtype=torch.float32)
            d[:, ::S.pick[0], ::S.pick[1]] = dout
        da = ops.masked_mean_bcast_bwd(d, S.mref, S.mtag)
        sn_conv_stack_bwd(G, self.convs(), S, ops.in_bwd(da, S.y_last, S.ss_last, ops.ACT_LRELU, round_tf32=True))

    def forward(self, x, label_ref, label_tag):
        return self.forward_nhwc(x, label_ref, label_tag).permute(0, 3, 1, 2)


class ConvEncoder(SNConvStack):
    """encoder.py:17-59, the --use_vae encoder: image -> (mu, logvar), each [N, 256].

    The image is resized to 256x256 (bilinear, align_corners=False), then six k3 s2 p1 convs, each normalised by
    `norm_E` (spectral norm, bias removed, InstanceNorm2d without affine) and followed by LeakyReLU 0.2, give a
    [N, 8ngf, 4, 4] map; fc_mu and fc_var read it flattened in NCHW order.  On the kernels: the six layers are SNConvStack's,
    and fc_mu | fc_var one 1x1 implicit GEMM whose rows are the images, with the two weights concatenated and their columns
    permuted once into the NHWC order of the map (cached until the weights change).  The backward is
    autograd.conv_encoder_bwd; the image gets no gradient (the reference encodes image_ref.clone() of a tensor that needs
    none)."""

    n_stack = 6

    def __init__(self, opt):
        super().__init__()
        if opt.crop_size < 256:
            raise NotImplementedError("michigan_b200: --use_vae needs crop_size >= 256: below it the reference's ConvEncoder "
                                      "has no layer6 and fc_mu does not match its 8x8 map")
        if opt.z_dim != 256:
            raise NotImplementedError("michigan_b200: --use_vae needs z_dim 256: the reference's fc_mu / fc_var have 256 "
                                      "outputs whatever z_dim says")
        self._check_opt(opt)
        kw = 3
        pw = int(np.ceil((kw - 1.0) / 2))
        ndf = opt.ngf
        norm_layer = get_nonspade_norm_layer(opt, opt.norm_E)
        self.layer1 = norm_layer(nn.Conv2d(3, ndf, kw, stride=2, padding=pw))
        self.layer2 = norm_layer(nn.Conv2d(ndf * 1, ndf * 2, kw, stride=2, padding=pw))
        self.layer3 = norm_layer(nn.Conv2d(ndf * 2, ndf * 4, kw, stride=2, padding=pw))
        self.layer4 = norm_layer(nn.Conv2d(ndf * 4, ndf * 8, kw, stride=2, padding=pw))
        self.layer5 = norm_layer(nn.Conv2d(ndf * 8, ndf * 8, kw, stride=2, padding=pw))
        self.layer6 = norm_layer(nn.Conv2d(ndf * 8, ndf * 8, kw, stride=2, padding=pw))
        self.so = s0 = 4
        self.fc_mu = nn.Linear(ndf * 8 * s0 * s0, 256)
        self.fc_var = nn.Linear(ndf * 8 * s0 * s0, 256)
        self.actvn = nn.LeakyReLU(0.2, False)
        self.opt = opt
        self._snb = None
        self._cache = PackCache()

    def grad_stages(self):
        """One gradient all-reduce stage: the whole encoder is finished together (autograd.conv_encoder_bwd)."""
        return [list(self.parameters())]

    def fc_weight(self):
        """[512, 16C, 1, 1] fp32: fc_mu | fc_var with the columns in the NHWC order (h, w, c) of the 4x4 map."""
        def build():
            c = self.fc_mu.in_features // 16
            w = torch.cat([self.fc_mu.weight.detach(), self.fc_var.weight.detach()])
            return w.view(512, c, 16).transpose(1, 2).reshape(512, 16 * c, 1, 1).contiguous()
        return self._cache.get("fc_w", [self.fc_mu.weight, self.fc_var.weight], build)

    def forward(self, x):
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            from .autograd import conv_encoder_forward_autograd
            return conv_encoder_forward_autograd(self, x)
        return self.run(x, None)

    def run(self, image, save):
        """The one forward implementation: image [N,3,H,W] NCHW -> (mu, logvar).  save: namespace filled with what
        autograd.conv_encoder_bwd needs (same arithmetic either way)."""
        N, _, H, W = image.shape
        x = ops.nchw_to_nhwc(image.detach().contiguous(), 4)
        if (H, W) != (256, 256):
            x = ops.resize_bilinear(x, 256, 256)                               # encoder.py:42-43
        y = self.run_stack(x, save)
        # encoder.py:52-57: lrelu(IN(layer6)), flattened; fc_mu | fc_var as one GEMM over the N images
        K = y[0].numel()
        fmt = precision.conv_fmt(K)
        xo, a32, ss = norm_act(y, fmt, save is not None)
        xo = (xo[0], xo[1].view(N, 1, 1, K), None if xo[2] is None else xo[2].view(N, 1, 1, K))
        wf = self.fc_weight()
        wp = self._cache.get(("fc", fmt), [self.fc_mu.weight, self.fc_var.weight], lambda: precision.pack_conv(wf, None, fmt))
        bias = self._cache.get("fc_b", [self.fc_mu.bias, self.fc_var.bias],
                               lambda: torch.cat([self.fc_mu.bias.detach(), self.fc_var.bias.detach()]).contiguous())
        out = precision.conv(xo, wp, 512, 1, 1, 1, 0, bias=bias).view(N, 512)
        if save is not None:
            save.y6, save.ss6, save.a6 = y, ss, a32.view(N, 1, 1, K)
        return out[:, :256].contiguous(), out[:, 256:].contiguous()
