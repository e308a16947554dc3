"""CPU oracle of the reference's unpaired training stage (--unpairTrain, curr_step 2), in plain fp32 PyTorch, restating the
reference exactly:

  * HairAvgLabLoss (models/networks/loss.py:534-621, balance_Lab=False): Lab of fake and real as LabColorLoss computes it
    (oracle_vgg_lab.rgb2lab), cal_hair_avg = sum(Lab * m) / sum(m) per image with a mask sum of 0 replaced by 1, then
    nn.L1Loss over the a, b averages against the detached real ones;
  * compute_generator_loss for curr_step 2 (pix2pix_model.py:280-363): GAN from the second discriminator (netD2,
    pix2pix_model.py:568-572), ORIENT / CONFIDENCE when on, hairAvgLab of fake against the reference image with the tag's and
    the reference's hair masks, background; in that key order.  GAN_Feat, VGG, style, content, rgb and lab belong to
    curr_step 1 and are absent.

Pinned against the live reference by tests/golden/make_golden_hair_avg_lab.py (tests/golden/golden_hair_avg_lab.npz)."""
import torch
import torch.nn.functional as F

import michigan_oracle as orc
import oracle_style_content as osc
import oracle_vgg_lab as ovl


def cal_hair_avg(lab, mask):
    s = (lab * mask).sum(dim=(2, 3), keepdim=True)
    cnt = mask.sum(dim=(2, 3), keepdim=True)
    return s / torch.where(cnt == 0, torch.ones_like(cnt), cnt)


def hair_avg_lab_loss(fake, real, mask_fake, mask_real):
    avg_f = cal_hair_avg(ovl.rgb2lab(fake), mask_fake)
    avg_r = cal_hair_avg(ovl.rgb2lab(real), mask_real)
    return F.l1_loss(avg_f[:, 1:], avg_r[:, 1:].detach())


def compute_generator_loss_unpaired(sdG, sdD2, opt, data, **kw):
    """The generator objective of the unpaired stage (curr_step 2).  sdD2: the second discriminator's state dict.
    Returns (losses dict in the reference's key order, fake image)."""
    fake = orc.generate_fake(sdG, opt, data, True, **kw)
    pred_fake, _ = orc.discriminate(sdD2, opt, data["input_tag"], fake, data["image_tag"], data["orient_mask"], True)
    losses = {}
    if not getattr(opt, "no_gan_loss", False):
        losses["GAN"] = orc.gan_loss_hinge(pred_fake, True, False, data["input_tag"][:, 1:2], opt)
    if not getattr(opt, "no_orient_loss", True):
        lo, lc = orc.orient_loss_gabor(fake, data["orient_mask"], data["input_tag"])
        losses["ORIENT"] = lo * getattr(opt, "lambda_orient", 10.0)
        if not getattr(opt, "no_confidence_loss", True):
            losses["CONFIDENCE"] = lc * getattr(opt, "lambda_confidence", 100.0)
    losses["hairAvgLab"] = hair_avg_lab_loss(fake, data["image_ref"], data["input_tag"][:, 1:2],
                                             data["input_ref"][:, 1:2]) * getattr(opt, "lambda_hairavglab", 1.0)
    losses["background"] = osc.background_loss(fake, data["input_tag"], data["image_tag"]) * getattr(opt, "lambda_background", 1.0)
    return losses, fake
