"""MultiscaleDiscriminator / NLayerDiscriminator — constructors, option hooks, forward signature and
state-dict layout of the reference's models/networks/discriminator.py:14-120 (norm_D =
'spectralinstance'); forward on the sm_90a kernels:

    model0      7->64 k4 s2 p2 + bias + LeakyReLU           thin direct conv (channels padded to 8)
    model1..3   SN conv k4 (s2,s2,s1) p2, no bias           wgmma implicit GEMM (stride via TMA elementStrides)
                InstanceNorm2d(affine=False) + LeakyReLU     per-(n,c) stats pass + normalise pass
    model4      512->1 k4 s1 p2 + bias                       warp-per-pixel dot product
    downsample  avg_pool2d(3, 2, 1, count_include_pad=False) on the 8-channel NHWC input
"""
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn as nn

from .. import ops, precision
from .base_network import BaseNetwork
from .normalization import get_nonspade_norm_layer
from .prep import PackCache, SpectralNormBatch


class NLayerDiscriminator(BaseNetwork):
    @staticmethod
    def modify_commandline_options(parser, is_train):
        parser.add_argument("--n_layers_D", type=int, default=4, help="# layers in each discriminator")
        return parser

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        kw = 4
        padw = int(np.ceil((kw - 1.0) / 2))
        nf = opt.ndf
        input_nc = self.compute_D_input_nc(opt)
        if input_nc > 8:
            raise NotImplementedError("michigan_b200: discriminator input has %d channels (max 8)" % input_nc)
        if nf % 32 != 0:
            raise NotImplementedError("michigan_b200: ndf must be a multiple of 32")
        norm_layer = get_nonspade_norm_layer(opt, opt.norm_D)
        sequence = [[nn.Conv2d(input_nc, nf, kernel_size=kw, stride=2, padding=padw), nn.LeakyReLU(0.2, False)]]
        self._strides = [2]
        for n in range(1, opt.n_layers_D):
            nf_prev = nf
            nf = min(nf * 2, 512)
            stride = 1 if n == opt.n_layers_D - 1 else 2
            self._strides.append(stride)
            sequence += [[norm_layer(nn.Conv2d(nf_prev, nf, kernel_size=kw, stride=stride, padding=padw)),
                          nn.LeakyReLU(0.2, False)]]
        sequence += [[nn.Conv2d(nf, 1, kernel_size=kw, stride=1, padding=padw)]]
        for n in range(len(sequence)):
            self.add_module("model" + str(n), nn.Sequential(*sequence[n]))
        self.n_layers = opt.n_layers_D
        self.padw = padw
        if "instance" not in opt.norm_D:
            raise NotImplementedError("michigan_b200: norm_D must be [spectral]instance")
        self._cache = PackCache()

    def compute_D_input_nc(self, opt):
        input_nc = opt.label_nc + opt.output_nc + opt.orient_nc
        if opt.contain_dontcare_label:
            input_nc += 1
        if not opt.no_instance:
            input_nc += 1
        return input_nc

    def mid_convs(self):
        """The (possibly spectrally-normalised) convs of model1..model{n-1}."""
        return [getattr(self, "model%d" % n)[0][0] for n in range(1, self.n_layers)]

    def forward_nhwc(self, x8, inv_sigma_of, save=None):
        """x8: [B,H,W,8] -> list of NHWC tensors (all intermediates + logits).
        save: namespace filled with what autograd._d_scale_bwd needs; the arithmetic is the same either way."""
        c = self._cache
        conv0 = self.model0[0]
        w0 = c.get("m0", [conv0.weight], lambda: ops.pack_weight_thin(conv0.weight.detach(), 8))
        # one-pass fp16 (or TF32): the discriminator is not under the generator's image-error bound

        def kw_for(fmt):
            return dict(round_out=True) if fmt == ops.TF32 else dict(out16=(fmt, False))

        def operand(r, fmt):
            """(feature fp32, tensor-core operand) from a producer's return value (fp32 | (fp32, hi, lo))."""
            return (r, (ops.TF32, r, None)) if fmt == ops.TF32 else (r[0], (fmt, r[1], None))

        fmt = precision.gb_fmt(conv0.out_channels)
        x, xo = operand(ops.conv_thin(x8, w0, conv0.bias.detach(), conv0.out_channels, 4, 4, 2, self.padw, act=ops.ACT_LRELU,
                                      **kw_for(fmt)), fmt)
        if save is not None:
            save.x8, save.wt0, save.f0, save.layers = x8, w0, x, []
        outs = [x]
        for n, conv in zip(range(1, self.n_layers), self.mid_convs()):
            if hasattr(conv, "weight_orig"):
                wp = ops.pack_weight(conv.weight_orig.detach(), inv_sigma_of[conv], True) if fmt == ops.TF32 else \
                    ops.pack_weight16(conv.weight_orig.detach(), inv_sigma_of[conv], fmt, split=False)
            elif fmt == ops.TF32:
                wp = c.get("m%d" % n, [conv.weight], lambda conv=conv: ops.pack_weight(conv.weight.detach(), None, True))
            else:
                wp = c.get(("m%d" % n, fmt), [conv.weight], lambda conv=conv: ops.pack_weight16(conv.weight.detach(), None, fmt, split=False))
            raw = precision.conv(xo, wp, conv.out_channels, 4, 4, self._strides[n], self.padw)
            fmt = precision.gb_fmt(conv.out_channels)
            f_in = x
            if save is None:
                x, xo = operand(ops.instance_norm_act(raw, ops.ACT_LRELU, 1e-5, **kw_for(fmt)), fmt)
            else:
                r = ops.instance_norm_act_fwd(raw, ops.ACT_LRELU, 1e-5, **kw_for(fmt))
                x, xo = operand(r[0] if fmt == ops.TF32 else (r[0], r[2], r[3]), fmt)
                save.layers.append(SimpleNamespace(conv=conv, stride=self._strides[n], f_in=f_in, raw=raw, ss=r[1]))
            outs.append(x)
        last = getattr(self, "model%d" % self.n_layers)[0]
        outs.append(ops.conv_to1(x, last.weight.detach(), last.bias.detach(), self.padw))
        if save is not None:
            save.f_last, save.last = x, last
        return outs

    def forward(self, input):
        snb = SpectralNormBatch([cv for cv in self.mid_convs() if hasattr(cv, "weight_orig")])
        inv = snb.run(self.training)
        inv_of = {cv: inv[i:i + 1] for i, cv in enumerate(snb.convs)}
        outs = [o.permute(0, 3, 1, 2) for o in self.forward_nhwc(ops.nchw_to_nhwc(input.contiguous(), 8), inv_of)]
        return outs if not self.opt.no_ganFeat_loss else outs[-1]


class MultiscaleDiscriminator(BaseNetwork):
    @staticmethod
    def modify_commandline_options(parser, is_train):
        parser.add_argument("--netD_subarch", type=str, default="n_layer", help="architecture of each discriminator")
        parser.add_argument("--num_D", type=int, default=2, help="number of discriminators to be used in multiscale")
        opt, _ = parser.parse_known_args()
        if opt.netD_subarch != "n_layer":
            raise ValueError("unrecognized discriminator subarchitecture %s" % opt.netD_subarch)
        NLayerDiscriminator.modify_commandline_options(parser, is_train)
        return parser

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        for i in range(opt.num_D):
            self.add_module("discriminator_%d" % i, self.create_single_discriminator(opt))
        self._snb = None

    def create_single_discriminator(self, opt):
        if opt.netD_subarch == "n_layer":
            return NLayerDiscriminator(opt)
        raise ValueError("unrecognized discriminator subarchitecture %s" % opt.netD_subarch)

    def grad_stages(self):
        """Gradient all-reduce stages in backward order (autograd._DiscriminatorFn.backward: coarsest scale first)."""
        return [list(D.parameters()) for _, D in reversed(list(self.named_children()))]

    def spectral_batch(self):
        if self._snb is None:
            convs = []
            for _, D in self.named_children():
                convs += [cv for cv in D.mid_convs() if hasattr(cv, "weight_orig")]
            self._snb = SpectralNormBatch(convs)
        return self._snb

    def forward(self, input):
        """input: [B,7,H,W] NCHW (fake||real on the batch, pix2pix_model.py:566).  Returns
        list[num_D] of list[n_layers_D+1] of NCHW-shaped (channels-last memory) tensors, or
        list of [logits] when --no_ganFeat_loss (discriminator.py:53-63)."""
        if torch.is_grad_enabled() and (input.requires_grad or any(p.requires_grad for p in self.parameters())):
            from .autograd import discriminator_forward_autograd
            return discriminator_forward_autograd(self, input)
        return self.forward_nograd(input)

    def forward_nograd(self, input):
        return self.run(input, None)

    def run(self, input, save):
        """The one forward implementation (save=None: no-grad; save=list to fill with per-scale state for the backward)."""
        snb = self.spectral_batch()
        inv = snb.run(self.training)
        if inv is None:
            inv_of = {}
        else:
            inv_of = {cv: (inv[i:i + 1].clone() if save is not None else inv[i:i + 1]) for i, cv in enumerate(snb.convs)}
        x8 = ops.nchw_to_nhwc(input.contiguous(), 8)
        get_feats = not self.opt.no_ganFeat_loss or save is not None
        result = []
        children = [D for _, D in self.named_children()]
        for i, D in enumerate(children):
            S = SimpleNamespace() if save is not None else None
            outs = [o.permute(0, 3, 1, 2) for o in D.forward_nhwc(x8, inv_of, save=S)]
            result.append(outs if get_feats else [outs[-1]])
            if save is not None:
                save.append(S)
            if i + 1 < len(children):
                x8 = ops.avgpool3s2(x8)
        return (result, inv_of) if save is not None else result
