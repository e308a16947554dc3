"""Pix2PixModel — the mode-dispatching caller of the hot path, mirroring the reference's
models/pix2pix_model.py (forward 62-122, create_optimizers 124-152, preprocess_input 209-254,
compute_generator_loss 257-365, compute_discriminator_loss 367-398, generate_fake 505-541,
discriminate 546-594) for the in-scope configuration: netG=spadeb, netD=multiscale, the GAN loss of any --gan_mode +
GAN feature loss and, each behind its --no_* flag, every other term of the reference's curr_step-1 objective (VGG
perceptual, style / content, background and rgb L1, Lab colour, Gabor orientation / confidence).  With the reference checkout
present, `michigan_b200.install()` lets the reference's own Pix2PixModel/Pix2PixTrainer drive these networks instead (INTEGRATION.md); this class is the
stand-alone equivalent used by bench.py and the tests on machines without the reference.
"""
import os

import torch
import torch.nn.functional as F

from . import networks, ops
from .networks.loss import (GANFeatLoss, GANLoss, KLDLoss, LabColorLoss, RGBBackgroundL1Loss, RGBL1Loss, StyleContentLoss,
                            VGGLoss, vgg_objective)


class Pix2PixModel(torch.nn.Module):
    @staticmethod
    def modify_commandline_options(parser, is_train):
        networks.modify_commandline_options(parser, is_train)
        return parser

    def __init__(self, opt):
        super().__init__()
        self.opt = opt
        if len(opt.gpu_ids) == 0:
            raise RuntimeError("michigan_b200 has no CPU path: gpu_ids must name a CUDA device")
        for flag in ("use_blender", "use_instance_feat", "unpairTrain"):
            if getattr(opt, flag, False):
                raise NotImplementedError("michigan_b200: --%s is outside the hot path (SURVEY.md §8)" % flag)
        # Every term of the reference's generator objective for curr_step 1 (pix2pix_model.py:296-345) is computed here: GAN
        # (any --gan_mode), GAN_Feat, VGG, content, style, background, rgb, lab, ORIENT, CONFIDENCE, each dropped by its --no_*
        # flag.  GANLoss and GANFeatLoss take --remove_background; VGGLoss and StyleContentLoss take it together with
        # mask_vgg_losses (the reference's hair-masked terms, networks.loss.masked_vgg_losses) and refuse it alone; LabColorLoss
        # takes --balance_Lab when opt.weight_dir names the count table (networks.loss.balanced_lab) and refuses it without.
        self.netIG = None
        if getattr(opt, "use_ig", False):
            self.netIG = networks.define_IG(opt)
            self._load_inpainting_network(opt)
        self.netG = networks.define_G(opt)
        self.netD = networks.define_D(opt) if opt.isTrain else None
        # --use_vae (pix2pix_model.py:42-43, 172): netE encodes image_ref to (mu, logvar), z = mu + eps exp(logvar / 2) drives
        # the generator's latent head, and the G step adds KLD first in G_losses
        self.netE = networks.define_E(opt) if getattr(opt, "use_vae", False) else None
        if opt.isTrain:
            if self.netE is not None:
                self.KLDLoss = KLDLoss()
            self.criterionGAN = GANLoss(opt.gan_mode, opt=opt)
            self.criterionGANFeat = GANFeatLoss(opt)
            if not getattr(opt, "no_vgg_loss", False):
                self.criterionVGG = VGGLoss(opt)
            if not (getattr(opt, "no_style_loss", False) and getattr(opt, "no_content_loss", False)):
                # one VGG19 instance for the perceptual and the style / content losses (they share one pass, _vgg_terms)
                shared = self.criterionVGG.vgg if hasattr(self, "criterionVGG") else None
                self.criterionStyleContent = StyleContentLoss(opt, vgg=shared)
            if not getattr(opt, "no_background_loss", False):
                self.criterionBackground = RGBBackgroundL1Loss()
            if not getattr(opt, "no_rgb_loss", False):
                self.criterionRGBL1 = RGBL1Loss()
            if not getattr(opt, "no_lab_loss", False):
                self.criterionLabL1 = LabColorLoss(opt)
            if not getattr(opt, "no_orient_loss", False):
                from .networks.loss import L1OLoss
                self.criterionOrient = L1OLoss(opt)
        if not opt.isTrain or getattr(opt, "continue_train", False):
            self._maybe_load(opt)

    # ------------------------------------------------------------------ checkpoints (util.py:195-231 layout)
    def _ckpt_path(self, label, epoch):
        return os.path.join(self.opt.checkpoints_dir, self.opt.name, "%s_net_%s.pth" % (epoch, label))

    def _maybe_load(self, opt):
        if not hasattr(opt, "checkpoints_dir"):
            return
        epoch = getattr(opt, "which_epoch", "latest")
        path = self._ckpt_path("G", epoch)
        if os.path.exists(path):
            load_weights(self.netG, torch.load(path, map_location="cpu"))
            if opt.isTrain and os.path.exists(self._ckpt_path("D", epoch)):
                load_weights(self.netD, torch.load(self._ckpt_path("D", epoch), map_location="cpu"))
            if self.netE is not None:
                load_weights(self.netE, torch.load(self._ckpt_path("E", epoch), map_location="cpu"))

    def save(self, epoch):
        """<checkpoints_dir>/<name>/<epoch>_net_{G,D,E}.pth (E with --use_vae, pix2pix_model.py:157-158), CPU state dicts with
        the reference's keys (util.py:195-200):
        rank 0 writes (snapshot copied on a side stream, serialised by a background thread), all ranks meet at a barrier."""
        from . import checkpoint
        checkpoint.save_state_dict(self.netG, self._ckpt_path("G", epoch))
        if self.netD is not None:
            checkpoint.save_state_dict(self.netD, self._ckpt_path("D", epoch))
        if self.netE is not None:
            checkpoint.save_state_dict(self.netE, self._ckpt_path("E", epoch))

    def _load_inpainting_network(self, opt):
        """util.load_inpainting_network (util.py:245-257): <checkpoints_dir>/<name>/<ig_model_name> = {'generator': state_dict}."""
        path = os.path.join(getattr(opt, "checkpoints_dir", "."), getattr(opt, "name", ""), getattr(opt, "ig_model_name", "InpaintingModel_gen.pth"))
        data = torch.load(path, map_location="cpu")
        self.netIG.load_state_dict(data["generator"])
        self.netIG.eval()

    def inpainting_orient(self, hole, orient_rgb, noise, mask):
        """pix2pix_model.py:407-429: fill the hole of the orientation RGB map with the frozen net (run at 256x256, nearest
        resize both ways) and derive the generator's 2-channel orientation input, masked by the hair mask."""
        inp = torch.cat([orient_rgb * (1 - hole) + noise * hole, hole], dim=1)
        if self.opt.crop_size != 256:
            inp = F.interpolate(inp, size=(256, 256), mode="nearest")
        out = self.netIG(inp)
        if self.opt.crop_size != 256:
            out = F.interpolate(out, size=(self.opt.crop_size, self.opt.crop_size), mode="nearest")
        out = out * hole + orient_rgb * (1 - hole)
        o2 = (out[:, :-1] - 0.5) * 2
        return out, (torch.stack([o2[:, 1], o2[:, 0]], dim=1) * mask).contiguous()

    def train(self, mode=True):
        """The orientation-inpainting net is frozen: it stays in eval mode whatever the model's mode (pix2pix_model.py:196-198)."""
        super().train(mode)
        if self.netIG is not None:
            self.netIG.eval()
        return self

    # ------------------------------------------------------------------ entry point
    def forward(self, data, mode):
        input_ref, input_tag, image_ref, image_tag, orient_mask, noise = self.preprocess_input(data)
        if self.netIG is not None:
            # pix2pix_model.py:260-263 / 370-372: the 2-channel inpainted orientation replaces the 1-channel angle map
            dev = input_tag.device
            with torch.no_grad():
                _, orient_mask = self.inpainting_orient(data["hole"].to(dev).float(), data["orient_rgb"].to(dev).float(), noise,
                                                        input_tag[:, 1:2])
        if mode == "generator":
            return self.compute_generator_loss(input_ref, input_tag, image_ref, image_tag, orient_mask, noise)
        if mode == "discriminator":
            return self.compute_discriminator_loss(input_ref, input_tag, image_ref, image_tag, orient_mask, noise)
        if mode == "encode_only":
            _, mu, logvar = self.encode_z(image_ref)
            return mu, logvar
        if mode == "inference":
            with torch.no_grad():
                return self.generate_fake(input_ref, image_ref, orient_mask, input_tag, image_tag, noise)
        raise ValueError("|mode| is invalid")

    def create_optimizers(self, opt):
        G_params = list(self.netG.parameters())
        if self.netE is not None:
            G_params += list(self.netE.parameters())
        D_params = list(self.netD.parameters()) if opt.isTrain else []
        if opt.no_TTUR:
            beta1, beta2 = opt.beta1, opt.beta2
            G_lr, D_lr = opt.lr, opt.lr
        else:
            beta1, beta2 = 0.0, 0.9
            G_lr, D_lr = opt.lr / 2, opt.lr * 2
        optimizer_G = torch.optim.Adam(G_params, lr=G_lr, betas=(beta1, beta2))
        optimizer_D = torch.optim.Adam(D_params, lr=D_lr, betas=(beta1, beta2))
        return optimizer_G, optimizer_D

    # ------------------------------------------------------------------ helpers
    def preprocess_input(self, data):
        """pix2pix_model.py:209-254: host->device copies and the one-hot label maps."""
        dev = _device()

        def dv(t):
            return t.to(dev, non_blocking=True)

        label_ref = dv(data["label_ref"]).long()
        label_tag = dv(data["label_tag"]).long()
        nc = self.opt.label_nc + 1 if self.opt.contain_dontcare_label else self.opt.label_nc
        bs, _, h, w = label_ref.shape
        input_ref = torch.zeros(bs, nc, h, w, device=dev).scatter_(1, label_ref, 1.0)
        input_tag = torch.zeros(bs, nc, h, w, device=dev).scatter_(1, label_tag, 1.0)
        return (input_ref, input_tag, dv(data["image_ref"]).float(), dv(data["image_tag"]).float(),
                dv(data["orient"]).float(), dv(data["noise"]).float())

    def zeros_padding(self, t):
        N, Cc, H, W = t.shape
        th = self.opt.add_th
        out = torch.zeros(N, Cc, H + th, W + th, device=t.device, dtype=t.dtype)
        o = int(th / 2)
        out[:, :, o:o + H, o:o + W] = t
        return out

    def encode_z(self, real_image):
        """pix2pix_model.py:400-403, 604-607: (z, mu, logvar).  The reparameterisation acts on N x 256 elements and stays torch
        arithmetic, as the reference's own Pix2PixModel.reparameterize does when install() drives it."""
        mu, logvar = self.netE(real_image)
        std = torch.exp(0.5 * logvar)
        eps = torch.randn_like(std)
        return eps.mul(std) + mu, mu, logvar

    def generate_fake(self, input_ref, image_ref, orient_mask, input_tag, image_tag, noise, z=None):
        """pix2pix_model.py:505-541; with --use_vae and no z given, z is encoded from image_ref (every mode, as the reference)."""
        if self.netE is not None and z is None:
            z, _, _ = self.encode_z(image_ref.clone())
        if self.opt.add_feat_zeros:
            input_ref, image_ref, orient_mask, input_tag, image_tag, noise = [
                self.zeros_padding(t) for t in (input_ref, image_ref, orient_mask, input_tag, image_tag, noise)]
        return self.netG(input_ref, z=z, orient_mask=orient_mask, image_ref=image_ref, input_tag=input_tag, noise=noise,
                         image_tag=image_tag)

    def discriminate(self, input_tag, fake_image, real_image, orient_mask):
        """pix2pix_model.py:546-594 (the 7-channel fake||real batch)."""
        seg4 = ops.prep_seg(input_tag.contiguous(), orient_mask.contiguous())
        cond = seg4.permute(0, 3, 1, 2)
        fake_concat = torch.cat([cond, fake_image], dim=1)
        real_concat = torch.cat([cond, real_image], dim=1)
        out = self.netD(torch.cat([fake_concat, real_concat], dim=0))
        fake = [[t[: t.size(0) // 2] for t in p] for p in out]
        real = [[t[t.size(0) // 2:] for t in p] for p in out]
        return fake, real

    def compute_generator_loss(self, input_ref, input_tag, image_ref, image_tag, orient_mask, noise):
        G_losses = {}
        z = None
        if self.netE is not None:
            # pix2pix_model.py:266-271, 505-511: KLD is the first key
            z, mu, logvar = self.encode_z(image_ref.clone())
            G_losses["KLD"] = self.KLDLoss(mu, logvar) * self.opt.lambda_kld
        fake_image = self.generate_fake(input_ref, image_ref, orient_mask, input_tag, image_tag, noise, z=z)
        # The discriminator's parameters are constants of the generator's objective: the reference back-propagates into
        # them anyway and discards the result (optimizer_D.zero_grad() precedes their only use, pix2pix_trainer.py:62-69).
        with _frozen(self.netD):
            pred_fake, pred_real = self.discriminate(input_tag, fake_image, image_tag, orient_mask)
        label_tag = input_tag[:, 1:2]
        if not self.opt.no_gan_loss:
            G_losses["GAN"] = self.criterionGAN(pred_fake, True, for_discriminator=False, label=label_tag)
        ref_is_tag = bool(torch.sum(input_tag[:, 1] - input_ref[:, 1]) == 0)
        if self.opt.curr_step == 1 and not self.opt.no_ganFeat_loss and ref_is_tag:
            G_losses["GAN_Feat"] = self.criterionGANFeat(pred_fake, pred_real, label_tag)
        # pix2pix_model.py:300-340, in the reference's key order (GAN, GAN_Feat, VGG, content, style, background, rgb, lab, ORIENT,
        # CONFIDENCE): VGG, background, rgb and lab only when ref is tag, content and style whenever curr_step is 1
        if self.opt.curr_step == 1:
            vgg, content, style = self._vgg_terms(fake_image, image_ref, image_tag, ref_is_tag, label_tag, input_ref[:, 1:2])
            if vgg is not None:
                G_losses["VGG"] = vgg * self.opt.lambda_vgg
            if content is not None:
                G_losses["content"] = content * self.opt.lambda_content
            if style is not None:
                G_losses["style"] = style * self.opt.lambda_style
        if self.opt.curr_step == 1 and not getattr(self.opt, "no_background_loss", False) and ref_is_tag:
            G_losses["background"] = self.criterionBackground(fake_image, input_tag, image_tag) * self.opt.lambda_background
        if self.opt.curr_step == 1 and not getattr(self.opt, "no_rgb_loss", False) and ref_is_tag:
            G_losses["rgb"] = self.criterionRGBL1(fake_image, image_tag.detach()) * self.opt.lambda_rgb
        if self.opt.curr_step == 1 and not getattr(self.opt, "no_lab_loss", False) and ref_is_tag:
            G_losses["lab"] = self.criterionLabL1(fake_image, image_tag.detach(), label_tag) * self.opt.lambda_lab
        if not getattr(self.opt, "no_orient_loss", False):
            # pix2pix_model.py:340-347
            orient_loss, confidence_loss = self.criterionOrient(fake_image, orient_mask, input_tag)
            G_losses["ORIENT"] = orient_loss * self.opt.lambda_orient
            if not getattr(self.opt, "no_confidence_loss", False):
                G_losses["CONFIDENCE"] = confidence_loss * self.opt.lambda_confidence
        return G_losses, fake_image

    def _vgg_terms(self, fake_image, image_ref, image_tag, ref_is_tag, label_tag, label_ref):
        """(VGG, content, style), None for a term that is off: one VGG19 pass over fake || tag (|| ref, unless it equals tag) for
        all of them (networks.loss.vgg_objective); VGG alone goes through criterionVGG, as before.  Under --remove_background
        the terms are masked by the tag's hair label, and the fake's style statistics by the reference's (pix2pix_model.py:
        303-315: label_tag, style_label = input_ref[:, 1], content_label = input_tag[:, 1])."""
        l1 = not getattr(self.opt, "no_vgg_loss", False) and ref_is_tag
        content = not getattr(self.opt, "no_content_loss", False)
        style = not getattr(self.opt, "no_style_loss", False)
        masked = self.criterionStyleContent.masked if (content or style) else False
        if not (content or style):
            return (self.criterionVGG(fake_image, image_tag, label_tag) if l1 else None), None, None
        crit = self.criterionStyleContent
        return vgg_objective(crit.vgg, fake_image, image_tag, image_ref, l1=l1, content=content, style=style,
                             weights=self.criterionVGG.weights if l1 else None, label=label_tag if masked else None,
                             style_label=label_ref if masked else None)

    def compute_discriminator_loss(self, input_ref, input_tag, image_ref, image_tag, orient_mask, noise):
        with torch.no_grad():
            fake_image = self.generate_fake(input_ref, image_ref, orient_mask, input_tag, image_tag, noise)
        fake_image = fake_image.detach().requires_grad_()
        pred_fake, pred_real = self.discriminate(input_tag, fake_image, image_tag, orient_mask)
        label_tag = input_tag[:, 1:2]
        return {"D_Fake": self.criterionGAN(pred_fake, False, for_discriminator=True, label=label_tag),
                "D_real": self.criterionGAN(pred_real, True, for_discriminator=True, label=label_tag)}

    def use_gpu(self):
        return True


def _device():
    """This process's CUDA device (tests/dryrun.py substitutes the CPU for host-logic tests)."""
    return torch.device("cuda", torch.cuda.current_device())


class _frozen:
    """with _frozen(net): parameters temporarily do not require grad (their gradients are neither computed nor reduced)."""

    def __init__(self, net):
        self.flags = [(p, p.requires_grad) for p in net.parameters()]

    def __enter__(self):
        for p, _ in self.flags:
            p.requires_grad_(False)

    def __exit__(self, *exc):
        for p, r in self.flags:
            p.requires_grad_(r)
        return False


def train_iteration(model, optimizer_G, optimizer_D, data):
    """One generator update followed by one discriminator update on `data` (what train.py's inner loop does per batch,
    train.py:94-101, with D_steps_per_G = 1): returns (g_losses, d_losses, generated).  `model` may be wrapped in
    DataParallelWithCallback; gradients are already rank-averaged when backward() returns."""
    optimizer_G.zero_grad(set_to_none=True)
    g_losses, generated = model(data, mode="generator")
    torch.stack([v.mean() for v in g_losses.values()]).sum().backward()
    optimizer_G.step()
    optimizer_D.zero_grad(set_to_none=True)
    d_losses = model(data, mode="discriminator")
    torch.stack([v.mean() for v in d_losses.values()]).sum().backward()
    optimizer_D.step()
    return g_losses, d_losses, generated


def load_weights(net, pretrained):
    """util.load_weights (util.py:202-218): strip a leading 'module.', copy only keys the model has."""
    own = net.state_dict()
    for k, v in pretrained.items():
        k = k[len("module."):] if k.startswith("module.") else k
        if k in own:
            own[k].copy_(v)
    return net
