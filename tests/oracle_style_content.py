"""CPU oracle of the remaining terms of the reference's generator objective, in plain fp32 PyTorch on top of
oracle_vgg_lab.vgg19_features, restating the reference exactly (remove_background=False):

  * calc_mean_std (models/networks/loss.py:624-632): per (n, c) mean and sqrt(unbiased variance + 1e-5);
  * StyleContentLoss (loss.py:656-711): loss_c = MSE(relu5_1(fake), relu5_1(content).detach()), loss_s = sum over the five taps of
    MSE(mu_fake, mu_style) + MSE(sigma_fake, sigma_style), the style taps detached;
  * RGBBackgroundL1Loss (loss.py:388-400): L1(fake * m, tag.detach() * m), m = input_semantics[:, 0:1];
  * the rgb loss, nn.L1Loss()(fake, tag.detach()) (pix2pix_model.py:51, 328-333);
  * compute_generator_loss with the reference's default loss set for curr_step 1 (pix2pix_model.py:257-347): GAN, GAN_Feat, VGG,
    content, style, background, rgb, lab, ORIENT, CONFIDENCE, in that order.

Pinned against the live reference by tests/golden/make_golden_style_content.py (tests/golden/golden_style_content.npz)."""
import torch
import torch.nn.functional as F

import michigan_oracle as orc
import oracle_vgg_lab as ovl


def calc_mean_std(feat, eps=1e-5):
    N, C = feat.shape[:2]
    var = feat.reshape(N, C, -1).var(dim=2) + eps
    return feat.reshape(N, C, -1).mean(dim=2).view(N, C, 1, 1), var.sqrt().view(N, C, 1, 1)


def style_loss(fake_feats, style_feats):
    loss = 0
    for f, s in zip(fake_feats, style_feats):
        mf, sf = calc_mean_std(f)
        ms, ss = calc_mean_std(s.detach())
        loss = loss + F.mse_loss(mf, ms) + F.mse_loss(sf, ss)
    return loss


def content_loss(fake_feats, content_feats):
    return F.mse_loss(fake_feats[-1], content_feats[-1].detach())


def style_content_loss(fake, style_image, content_image, sd):
    """StyleContentLoss.forward(fake, style_image, content_image) -> (loss_c, loss_s)."""
    ff = ovl.vgg19_features(fake, sd)
    return content_loss(ff, ovl.vgg19_features(content_image, sd)), style_loss(ff, ovl.vgg19_features(style_image, sd))


def background_loss(fake, input_semantics, image_tag):
    m = input_semantics[:, 0:1]
    return F.l1_loss(fake * m, (image_tag * m).detach())


def rgb_loss(fake, image_tag):
    return F.l1_loss(fake, image_tag.detach())


def compute_generator_loss_default(sdG, sdD, sd_vgg, opt, data, **kw):
    """compute_generator_loss with the reference's default loss set (options/train_options.py: every no_* off, all lambdas 1 except
    lambda_orient 10 and lambda_confidence 100), curr_step 1.  Returns (losses dict in the reference's key order, fake image)."""
    losses, fake = orc.compute_generator_loss(sdG, sdD, opt, data, **kw)
    ref_is_tag = bool(torch.sum(data["input_tag"][:, 1] - data["input_ref"][:, 1]) == 0)
    tag = data["image_tag"]
    ff = ovl.vgg19_features(fake, sd_vgg)
    tf = ovl.vgg19_features(tag, sd_vgg)
    if ref_is_tag:
        loss = 0
        for w, a, b in zip(ovl.VGG_WEIGHTS, ff, tf):
            loss = loss + w * F.l1_loss(a, b.detach())
        losses["VGG"] = loss * getattr(opt, "lambda_vgg", 1.0)
    losses["content"] = content_loss(ff, tf) * getattr(opt, "lambda_content", 1.0)
    losses["style"] = style_loss(ff, ovl.vgg19_features(data["image_ref"], sd_vgg)) * getattr(opt, "lambda_style", 1.0)
    if ref_is_tag:
        losses["background"] = background_loss(fake, data["input_tag"], tag) * getattr(opt, "lambda_background", 1.0)
        losses["rgb"] = rgb_loss(fake, tag) * getattr(opt, "lambda_rgb", 1.0)
        losses["lab"] = ovl.lab_loss(fake, tag.detach()) * getattr(opt, "lambda_lab", 1.0)
    lo, lc = orc.orient_loss_gabor(fake, data["orient_mask"], data["input_tag"])
    losses["ORIENT"] = lo * getattr(opt, "lambda_orient", 10.0)
    losses["CONFIDENCE"] = lc * getattr(opt, "lambda_confidence", 100.0)
    return losses, fake
