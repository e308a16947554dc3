"""CPU oracle of the reference's --remove_background VGG terms, in plain fp32 PyTorch on top of oracle_vgg_lab.vgg19_features,
restating the reference exactly (models/networks/loss.py, remove_background=True); every label is resized to each tap with
F.interpolate(mode='nearest'):

  * VGGLoss.L1_loss_mask (loss.py:187-207): sum_i w_i * sum |x_i l - y_i.detach() l| / (sum(l) * c + 1e-5);
  * calc_content_loss (loss.py:664-677): sum (x_5 l - t_5.detach() l)^2 / (sum(l) * c + 1e-5), l the content (tag) label;
  * calc_mean_std_mask (loss.py:634-654): mu = sum(x m) / (sum(m) + eps), sigma = sqrt(sum(((x m - mu) m)^2) / (sum(m) + eps) +
    eps) per (n, c) - a biased variance with eps twice;
  * calc_style_loss (loss.py:679-694) over the five taps: MSE(mu_f, mu_s) + MSE(sigma_f, sigma_s), where the fake features are
    masked by style_label (the style image's hair) and the style image's features by content_label (the tag's hair): the
    reference passes the labels crossed, and this restates the crossing.

Pinned against the live reference by tests/golden/make_golden_remove_background.py (tests/golden/golden_remove_background.npz)."""
import torch
import torch.nn.functional as F

import oracle_vgg_lab as ovl

EPS = 1e-5


def _resize(label, feat):
    return F.interpolate(label, size=feat.shape[2:], mode="nearest")


def l1_loss_mask(x, y, label):
    lab = _resize(label, x)
    return (x * lab - y.detach() * lab).abs().sum() / (lab.sum() * x.shape[1] + EPS)


def vgg_loss(x, y, label, sd):
    loss = 0
    for w, a, b in zip(ovl.VGG_WEIGHTS, ovl.vgg19_features(x, sd), ovl.vgg19_features(y, sd)):
        loss = loss + w * l1_loss_mask(a, b, label)
    return loss


def calc_mean_std_mask(feat, mask, eps=EPS):
    N, C = feat.shape[:2]
    m = mask.reshape(N, 1, -1)
    f = feat.reshape(N, C, -1) * m
    mean = (f.sum(2) / (m.sum(2) + eps)).view(N, C, 1)
    var = (((f - mean) * m) ** 2).sum(2) / (m.sum(2) + eps) + eps
    return mean.view(N, C, 1, 1), var.sqrt().view(N, C, 1, 1)


def content_loss(fake_feats, content_feats, content_label):
    x, t = fake_feats[-1], content_feats[-1].detach()
    lab = _resize(content_label, x)
    return ((x * lab - t * lab) ** 2).sum() / (lab.sum() * x.shape[1] + EPS)


def style_loss(fake_feats, style_feats, style_label, content_label):
    loss = 0
    for f, s in zip(fake_feats, style_feats):
        mf, sf = calc_mean_std_mask(f, _resize(style_label, f))
        ms, ss = calc_mean_std_mask(s.detach(), _resize(content_label, f))
        loss = loss + F.mse_loss(mf, ms) + F.mse_loss(sf, ss)
    return loss


def style_content_loss(fake, style_image, content_image, style_label, content_label, sd):
    """StyleContentLoss.forward(fake, style_image, content_image, style_label, content_label) -> (loss_c, loss_s)."""
    ff = ovl.vgg19_features(fake, sd)
    return (content_loss(ff, ovl.vgg19_features(content_image, sd), content_label),
            style_loss(ff, ovl.vgg19_features(style_image, sd), style_label, content_label))
