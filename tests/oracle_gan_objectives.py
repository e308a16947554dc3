"""CPU oracle of the reference's adversarial losses in every configuration, in plain PyTorch (any float dtype), restating
models/networks/loss.py:

  * GANLoss (19-140): per discriminator scale (the last tensor of each list), 'original' = BCE with logits and 'ls' = MSE
    against the constant target_real_label / target_fake_label, 'w' = -mean(x) for real and mean(x) for fake, 'hinge' =
    -mean(min(+-x - 1, 0)) on the discriminator side (times the wide-edge weight map when wide_edge > 1) and -mean(x) for the
    generator; under --remove_background the hinge terms are masked by the hair label resized (nearest) to the scale,
    label1: -sum(min((+-x - 1) label1, 0)) and -sum(x label1), each over sum(label1) * c + 1e-5.  The scale losses are
    averaged over the discriminators; a list input gives a [1] tensor.
  * GANFeatLoss (144-175): sum over discriminators and intermediate features of lambda_feat / num_D times L1(fake, real) or,
    under --remove_background, sum |fake label1 - real label1| / (sum(label1) * c + 1e-5), real detached.

Pinned against the live reference by tests/golden/make_golden_gan_objectives.py (tests/golden/golden_gan_objectives.npz)."""
import torch
import torch.nn.functional as F

import michigan_oracle as orc

GAN_MODES = ("ls", "original", "w", "hinge")


def resized_label(label, x):
    return F.interpolate(label.to(x.dtype), size=tuple(x.shape[2:]), mode="nearest")


def _masked_den(label1, c):
    return label1.sum() * c + 1e-5


def gan_scale_loss(x, target_is_real, for_discriminator, label, gan_mode, wide_edge=1.0, remove_background=False,
                   real_label=1.0, fake_label=0.0):
    """One discriminator scale's loss (loss.py:80-124), a 0-dim tensor."""
    if gan_mode in ("original", "ls"):
        t = torch.full_like(x, float(torch.tensor(real_label if target_is_real else fake_label, dtype=torch.float32)))
        return F.binary_cross_entropy_with_logits(x, t) if gan_mode == "original" else F.mse_loss(x, t)
    if gan_mode == "w":
        return -x.mean() if target_is_real else x.mean()
    zero = torch.zeros_like(x)
    arg = (x - 1) if target_is_real else (-x - 1)
    if remove_background:
        label1 = resized_label(label, x)
        den = _masked_den(label1, x.shape[1])
        if not for_discriminator:
            return -(x * label1).sum() / den
        return -torch.min(arg * label1, zero).sum() / den
    if not for_discriminator:
        return -x.mean()
    minval = torch.min(arg, zero)
    if wide_edge > 1.0:
        minval = minval * orc.wide_edge_weight(x, label.to(x.dtype), wide_edge)
    return -minval.mean()


def gan_loss(preds, target_is_real, for_discriminator, label, gan_mode, wide_edge=1.0, remove_background=False,
             real_label=1.0, fake_label=0.0):
    """GANLoss.__call__ (loss.py:126-140) over a list of discriminators (each a list of features, the logits last)."""
    if gan_mode not in GAN_MODES:
        raise ValueError("Unexpected gan_mode {}".format(gan_mode))
    total = 0
    for pred in preds:
        x = pred[-1] if isinstance(pred, list) else pred
        loss = gan_scale_loss(x, target_is_real, for_discriminator, label, gan_mode, wide_edge, remove_background, real_label,
                              fake_label)
        total = total + loss.reshape(1, -1).mean(dim=1)
    return total / len(preds)


def gan_feat_loss(pred_fake, pred_real, label, lambda_feat, remove_background=False):
    """GANFeatLoss.forward (loss.py:163-175), a [1] tensor."""
    num_D = len(pred_fake)
    loss = torch.zeros(1, dtype=pred_fake[0][0].dtype, device=pred_fake[0][0].device)
    for i in range(num_D):
        for j in range(len(pred_fake[i]) - 1):
            f, r = pred_fake[i][j], pred_real[i][j].detach()
            if remove_background:
                label1 = resized_label(label, f)
                term = (f * label1 - r * label1).abs().sum() / _masked_den(label1, f.shape[1])
            else:
                term = F.l1_loss(f, r)
            loss = loss + term * lambda_feat / num_D
    return loss
