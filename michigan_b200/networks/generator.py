"""SPADEBGenerator (`--netG spadeb`) — constructor, forward signature and state-dict layout of the
reference's models/networks/generator.py:19-230; the forward runs on the sm_90a kernels.

Data layout: every internal activation is NHWC fp32 in HBM; tensors that feed a tensor-core conv are
written TF32-rounded by their producer; the 2x nearest upsamples (generator.py:72,163-210) and the
hair/background mask pyramids (generator.py:149-159, encoder.py:332-336) are never materialised -
consumers index the low-resolution tensor / full-resolution mask directly.
"""
import os
from types import SimpleNamespace

import torch

from .. import ops
from .architecture import SPADEResnetBlock
from .base_network import BaseNetwork
from .encoder import BackgroundEncode2, ImageEncoder, ImageEncoder2, ImageEncoder3, latent_head
from .prep import PackCache, SpectralNormBatch

# MICHIGAN_B200_OVERLAP=1: background encoder on a second stream (off by default: the low-resolution blocks are short and the
# encoder's one-CTA-per-SM kernels cannot share an SM with a large-smem GEMM CTA anyway).
_OVERLAP = os.environ.get("MICHIGAN_B200_OVERLAP", "0") == "1"


# --Image_encoder_mode -> the reference-image encoder of --use_encoder (generator.py:38-44)
IMAGE_ENCODERS = {"partialconv": ImageEncoder3, "instance": ImageEncoder2, "norm": ImageEncoder}


class SPADEBGenerator(BaseNetwork):
    @staticmethod
    def modify_commandline_options(parser, is_train):
        parser.set_defaults(norm_G="spectralspadesyncbatch3x3")
        return parser

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        nf = opt.ngf
        self.sw, self.sh = self.compute_latent_vector_size(opt)
        if not getattr(opt, "use_vae", False):
            if not opt.use_encoder:
                raise NotImplementedError("michigan_b200: spadeb is implemented for --use_vae and for --use_encoder (the "
                                          "deterministic head has no kernels)")
            if opt.Image_encoder_mode not in IMAGE_ENCODERS:
                raise NotImplementedError("michigan_b200: --Image_encoder_mode '%s' is not one of %s"
                                          % (opt.Image_encoder_mode, ", ".join(IMAGE_ENCODERS)))
        if not opt.noise_background:
            raise NotImplementedError("michigan_b200: spadeb is implemented for --noise_background (BackgroundEncode2)")
        if opt.num_upsampling_layers != "more":
            raise NotImplementedError("michigan_b200: num_upsampling_layers must be 'more' (the default)")
        if getattr(opt, "no_orientation", False):
            raise NotImplementedError("michigan_b200: the orientation map is required")
        if getattr(opt, "bf_direct_add", False):
            raise NotImplementedError("michigan_b200: --bf_direct_add is not implemented")
        if getattr(opt, "use_vae", False):
            # generator.py:33-35: z -> the 16nf x sh x sw map (run(): one 1x1 GEMM over the N rows of z)
            if opt.z_dim % 32 != 0:
                raise NotImplementedError("michigan_b200: z_dim must be a multiple of 32")
            self.fc = torch.nn.Linear(opt.z_dim, 16 * nf * self.sw * self.sh)
        else:
            self.fc = IMAGE_ENCODERS[opt.Image_encoder_mode](opt, self.sw, self.sh)
        self.head_0 = SPADEResnetBlock(16 * nf, 16 * nf, opt)
        self.G_middle_0 = SPADEResnetBlock(16 * nf, 16 * nf, opt)
        self.G_middle_1 = SPADEResnetBlock(16 * nf, 16 * nf, opt)
        self.up_0 = SPADEResnetBlock(16 * nf, 8 * nf, opt)
        self.up_1 = SPADEResnetBlock(8 * nf, 4 * nf, opt)
        self.up_2 = SPADEResnetBlock(4 * nf, 2 * nf, opt)
        self.up_3 = SPADEResnetBlock(2 * nf, 1 * nf, opt)
        final_nc = nf
        self.conv_img = torch.nn.Conv2d(final_nc, 3, 3, padding=1)
        self.up = torch.nn.Upsample(scale_factor=2)
        self.backgroud_enc = BackgroundEncode2(opt)  # (sic) the reference's attribute name
        self._blocks = ["head_0", "G_middle_0", "G_middle_1", "up_0", "up_1", "up_2", "up_3"]
        self._snb = None
        self._cache = PackCache()
        self.last_taps = None
        self.collect_taps = False

    def compute_latent_vector_size(self, opt):
        n_up = {"normal": 5, "more": 6, "most": 7}.get(opt.num_upsampling_layers)
        if n_up is None:
            raise ValueError("opt.num_upsampling_layers [%s] not recognized" % opt.num_upsampling_layers)
        if opt.add_feat_zeros:
            sw = (opt.crop_size + opt.add_th) // (2 ** n_up)
        else:
            sw = opt.crop_size // (2 ** n_up)
        sh = round(sw / opt.aspect_ratio)
        return sw, sh

    # Gradient all-reduce stages, in the order the backward finalises them (autograd._GeneratorFn.backward): the key is the
    # block after whose backward the stage is complete.  Sizes (ngf 64): 30 / 54 / 94 / 94 / 94 / 36 MB - the three 94 MB
    # stages come out while only the cheap low-resolution blocks are left to compute.
    GRAD_STAGE_AFTER_BLOCK = {"up_1": 0, "up_0": 1, "G_middle_1": 2, "G_middle_0": 3, "head_0": 4}

    def grad_stages(self):
        def ps(*mods):
            return [p for m in mods for p in m.parameters()]
        return [ps(self.conv_img, self.up_3, self.up_2, self.up_1), ps(self.up_0), ps(self.G_middle_1), ps(self.G_middle_0),
                ps(self.head_0), ps(self.fc, self.backgroud_enc)]

    def _side_stream(self):
        dev = torch.cuda.current_device()
        st = getattr(self, "_side", None)
        if st is None or st.device.index != dev:
            st = torch.cuda.Stream(device=dev)
            self._side = st
        return st

    def spectral_batch(self):
        if self._snb is None:
            convs = []
            for b in self._blocks:
                convs += getattr(self, b).sn_convs()
            self._snb = SpectralNormBatch(convs)
        return self._snb

    def forward(self, input=None, z=None, orient_mask=None, image_ref=None, input_tag=None, noise=None, image_tag=None):
        """generator.py:107-230.  All arguments NCHW CUDA tensors; returns the [N,3,H,W] image in [-1,1]."""
        opt = self.opt
        if getattr(opt, "orient_random_disturb", False) or getattr(opt, "use_clip", False):
            raise NotImplementedError("michigan_b200: orient_random_disturb / use_clip are debugging paths")
        grad_z = z is not None and z.requires_grad
        if torch.is_grad_enabled() and (grad_z or any(p.requires_grad for p in self.parameters())):
            from .autograd import generator_forward_autograd
            return generator_forward_autograd(self, input, orient_mask, image_ref, input_tag, noise, image_tag, z=z)
        return self.forward_nograd(input, orient_mask, image_ref, input_tag, noise, image_tag, z=z)

    def forward_nograd(self, input, orient_mask, image_ref, input_tag, noise, image_tag, z=None):
        return self.run(input, orient_mask, image_ref, input_tag, noise, image_tag, None, z=z)

    def latent_head(self, z, N, device, save):
        """generator.py:110-116: x = view(fc(z)) as [N,sh,sw,16nf] NHWC (encoder.latent_head); z None -> sampled from
        N(0, I) on the device."""
        if z is None:
            z = torch.randn(N, self.opt.z_dim, dtype=torch.float32, device=device)
        return latent_head(self._cache, self.fc, z, self.sh, self.sw, save)

    def run(self, input, orient_mask, image_ref, input_tag, noise, image_tag, save, z=None):
        """The one forward implementation.  save=None: inference / no-grad; save=namespace: the autograd Function's forward,
        which keeps per-block state for the hand-written backward (networks/autograd.py) - identical arithmetic."""
        opt = self.opt
        if opt.bf_direct_add:
            raise NotImplementedError("michigan_b200: --bf_direct_add is not implemented")
        N, _, H, W = input_tag.shape
        input_tag = input_tag.contiguous()
        seg4 = ops.prep_seg(input_tag, orient_mask.contiguous())          # generator.py:129-142
        ins_ref = input[:, 1:2]
        ins_tag = input_tag[:, 1:2]
        sv = (lambda: SimpleNamespace()) if save is not None else (lambda: None)
        Sfc, Sbg = sv(), sv()
        # The background encoder (generator.py:144-147; full-resolution maps, one-CTA-per-SM kernels) is independent of the reference
        # encoder and of head_0 / G_middle_0 / G_middle_1, whose 8x8..32x32 maps give the persistent GEMM kernels only 16..128 tiles:
        # it runs on a second stream and fills the SMs those kernels leave idle; the main stream joins before up_0's blend.
        overlap = _OVERLAP and input_tag.is_cuda
        if overlap:
            main = torch.cuda.current_stream()
            side = self._side_stream()
            side.wait_event(main.record_event())
            with torch.cuda.stream(side):
                feats, back = self.backgroud_enc.forward_nhwc(image_tag, input_tag, noise, save=Sbg)
                bg_done = side.record_event()
        else:
            feats, back = self.backgroud_enc.forward_nhwc(image_tag, input_tag, noise, save=Sbg)  # generator.py:144-147
        if getattr(opt, "use_vae", False):
            x = self.latent_head(z, N, input_tag.device, Sfc)                        # generator.py:110-116
        else:
            x = self.fc.forward_nhwc(image_ref, ins_ref, ins_tag, save=Sfc)          # generator.py:117-123
        hair = input_tag[:, 1].contiguous()
        snb = self.spectral_batch()
        inv = snb.run(self.training)
        # training keeps private copies: the D step's no-grad forward re-runs the power iteration before this backward is gone
        inv_of = {c: (inv[i:i + 1].clone() if save is not None else inv[i:i + 1]) for i, c in enumerate(snb.convs)}
        taps = {} if self.collect_taps else None
        if taps is not None:
            taps["fc"] = x
            for i, f in enumerate(feats):
                taps["bg%d" % i] = f
        saved = []
        for idx, name in enumerate(self._blocks):
            blk = getattr(self, name)
            S = sv()
            if idx < 3:
                x = blk.forward_nhwc(x, 0 if idx == 0 else 1, seg4, inv_of, save=S)
            else:
                if overlap and idx == 3:
                    main.wait_event(bg_done)
                i = idx - 3
                ms = 8 >> i  # hair_masks / back_masks pyramid level == stride into the full-resolution masks
                x = blk.forward_nhwc(x, 1, seg4, inv_of, blend=(feats[i], hair, back, ms), save=S)
            saved.append(S)
            if taps is not None:
                taps[name] = x
        out = ops.conv_img(x, self.conv_img.weight.detach(), self.conv_img.bias.detach())  # generator.py:227-228
        self.last_taps = taps
        if save is not None:
            save.seg4, save.inv_of, save.saved, save.Sfc, save.Sbg, save.x_last, save.out = seg4, inv_of, saved, Sfc, Sbg, x, out
        return out
