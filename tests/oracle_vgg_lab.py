"""CPU oracle of the VGG19 perceptual loss and the Lab colour loss, in plain fp32 PyTorch (F.conv2d / F.max_pool2d, torch.where
for the Lab branches; no torchvision), restating the reference exactly:

  * VGG19 (models/networks/architecture.py:160-190): vgg19().features[0:30] in five slices ending at relu1_1 .. relu5_1, the image
    fed in [-1, 1] without ImageNet normalisation;
  * VGGLoss (loss.py:178-207, remove_background=False): sum_i w_i * mean |x_i - y_i.detach()|, w = 1/32, 1/16, 1/8, 1/4, 1;
  * LabColorLoss (loss.py:403-531, balance_Lab=False): L1 between the a, b channels of xyz2lab(rgb2xyz((img + 1) / 2));
  * the generator objective of the README's training command: hinge GAN + GAN_Feat (michigan_oracle.compute_generator_loss)
    + VGG + lab (pix2pix_model.py:300-307, 335-340) + ORIENT (340-347).

Pinned against the live reference by tests/golden/make_golden_vgg_lab.py (tests/golden/golden_vgg_lab.npz)."""
import torch
import torch.nn.functional as F

import michigan_oracle as orc

VGG_WEIGHTS = (1.0 / 32, 1.0 / 16, 1.0 / 8, 1.0 / 4, 1.0)
_CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, 256, "M", 512, 512, 512, 512, "M", 512]   # features[0:30]
_TAP_AFTER = {1, 6, 11, 20, 29}                                                             # relu1_1 .. relu5_1


def vgg19_features(x, sd):
    """sd: torchvision layout (features.N.weight / .bias) -> [h_relu1 .. h_relu5]."""
    out, i = [], 0
    for v in _CFG:
        if v == "M":
            x = F.max_pool2d(x, kernel_size=2, stride=2)
            i += 1
            continue
        x = F.conv2d(x, sd["features.%d.weight" % i], sd["features.%d.bias" % i], padding=1)
        x = F.relu(x)
        if i + 1 in _TAP_AFTER:
            out.append(x)
        i += 2
    return out


def vgg_loss(x, y, sd):
    xs, ys = vgg19_features(x, sd), vgg19_features(y, sd)
    loss = 0
    for w, a, b in zip(VGG_WEIGHTS, xs, ys):
        loss = loss + w * F.l1_loss(a, b.detach())
    return loss


_M = torch.tensor([[0.412453, 0.357580, 0.180423], [0.212671, 0.715160, 0.072169], [0.019334, 0.119193, 0.950227]])


def rgb2lab(img):
    """loss.py:441-485 on an image in [-1, 1]: (L, a, b) with the threshold branches as torch.where (the cube-root branch
    evaluated on clamped values, so that its derivative is finite where the other branch is taken)."""
    rgb = (img + 1) / 2.0
    xyz = torch.einsum("nc,bchw->bnhw", _M, rgb) / _M.sum(dim=1).view(1, 3, 1, 1)
    th = 0.008856
    f = torch.where(xyz > th, xyz.clamp(min=th).pow(1 / 3), 7.787 * xyz + 0.137931)
    y = xyz[:, 1]
    L = torch.where(y > th, 116 * f[:, 1] - 16, 903.3 * y)
    a = 500 * (f[:, 0] - f[:, 1])
    b = 200 * (f[:, 1] - f[:, 2])
    return torch.stack([L, a, b], 1)


def lab_loss(fake, real):
    return F.l1_loss(rgb2lab(fake)[:, 1:], rgb2lab(real)[:, 1:].detach())


def compute_generator_loss_readme(sdG, sdD, sd_vgg, opt, data, **kw):
    """compute_generator_loss with the README's loss set: GAN, GAN_Feat, VGG, lab, ORIENT (no confidence loss), in the
    reference's key order (options/train_options.py defaults: curr_step 1, lambda_vgg 1, lambda_lab 1, lambda_orient 10).
    Returns (losses dict, fake image)."""
    losses, fake = orc.compute_generator_loss(sdG, sdD, opt, data, **kw)
    ref_is_tag = bool(torch.sum(data["input_tag"][:, 1] - data["input_ref"][:, 1]) == 0)
    if getattr(opt, "curr_step", 1) == 1 and ref_is_tag:
        losses["VGG"] = vgg_loss(fake, data["image_tag"], sd_vgg) * getattr(opt, "lambda_vgg", 1.0)
        losses["lab"] = lab_loss(fake, data["image_tag"].detach()) * getattr(opt, "lambda_lab", 1.0)
    lo, _ = orc.orient_loss_gabor(fake, data["orient_mask"], data["input_tag"])
    losses["ORIENT"] = lo * getattr(opt, "lambda_orient", 10.0)
    return losses, fake
