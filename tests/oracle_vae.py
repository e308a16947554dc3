"""Torch restatement of the reference's --use_vae pieces (CPU or GPU, any dtype), pinned to tests/golden/golden_vae.npz by
tests/test_oracle_vae.py:

  * ConvEncoder.forward (models/networks/encoder.py:41-59, norm_E 'spectralinstance');
  * KLDLoss (loss.py:211-213);
  * SPADEBGenerator.forward with use_vae (generator.py:110-116): x = fc(z).view(-1, 16 ngf, sh, sw), then the blocks of
    michigan_oracle.generator_forward.
"""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import michigan_oracle as orc  # noqa: E402


def conv_encoder(sd, image, training, prefix=""):
    """encoder.py:41-59 with the state dict `sd` (power iteration in place on sd's u, v when training)."""
    x = image
    if x.shape[2] != 256 or x.shape[3] != 256:
        x = F.interpolate(x, size=(256, 256), mode="bilinear")
    for i in range(1, 7):
        if i > 1:
            x = orc.lrelu(x)
        w = orc.conv_weight(sd, prefix + "layer%d.0" % i, training)
        x = F.instance_norm(F.conv2d(x, w, None, stride=2, padding=1))
    x = orc.lrelu(x).reshape(x.shape[0], -1)
    mu = F.linear(x, sd[prefix + "fc_mu.weight"], sd[prefix + "fc_mu.bias"])
    logvar = F.linear(x, sd[prefix + "fc_var.weight"], sd[prefix + "fc_var.bias"])
    return mu, logvar


def kld(mu, logvar):
    return -0.5 * torch.sum(1 + logvar - mu.pow(2) - logvar.exp())


def latent_head(sd, opt, z):
    sw, sh = orc.latent_size(opt)
    return F.linear(z, sd["fc.weight"], sd["fc.bias"]).view(-1, 16 * opt.ngf, sh, sw)


def generator_forward(sd, opt, z, input_tag, image_tag, orient_mask, noise, training, rng_k=None):
    """generator.py:107-230 with use_vae: the partial-conv encoder replaced by the latent head."""
    x = latent_head(sd, opt, z)
    hair = input_tag[:, 1:2]
    seg = torch.cat([input_tag, orient_mask if opt.use_ig else orc.orient_channels(orient_mask, hair, opt)], dim=1)
    back_feats, back_masks = orc.background_encode2(image_tag, input_tag, noise, sd, "backgroud_enc", opt, rng_k)
    H, W = hair.shape[2:]
    hair_masks = [F.interpolate(hair, size=(int(H / d), int(W / d)), mode="nearest") for d in (8, 4, 2)] + [hair]

    def up(t):
        return F.interpolate(t, scale_factor=2, mode="nearest")

    x = orc.spade_resnet_block(x, seg, sd, "head_0", training)
    x = orc.spade_resnet_block(up(x), seg, sd, "G_middle_0", training)
    x = orc.spade_resnet_block(up(x), seg, sd, "G_middle_1", training)
    for i in range(4):
        x = orc.spade_resnet_block(up(x), seg, sd, "up_%d" % i, training)
        x = back_feats[i] * (1 - hair_masks[i]) + x * (1 - back_masks[i])
    x = F.conv2d(orc.lrelu(x), sd["conv_img.weight"], sd["conv_img.bias"], padding=1)
    return torch.tanh(x)


def encode_z(sdE, image_ref, eps):
    """Pix2PixModel.encode_z + reparameterize (pix2pix_model.py:400-403, 604-607) with a given eps."""
    mu, logvar = conv_encoder(sdE, image_ref, True)
    return eps * torch.exp(0.5 * logvar) + mu, mu, logvar


def compute_generator_loss(sdG, sdD, sdE, opt, pre, eps, rng_k=None):
    """Pix2PixModel.compute_generator_loss with --use_vae and the GAN + GAN_Feat terms (pix2pix_model.py:257-297): KLD
    first.  Returns (losses, fake, mu, logvar)."""
    z, mu, logvar = encode_z(sdE, pre["image_ref"], eps)
    losses = {"KLD": kld(mu, logvar) * opt.lambda_kld}
    fake = generator_forward(sdG, opt, z, pre["input_tag"], pre["image_tag"], pre["orient_mask"], pre["noise"], True, rng_k)
    pred_fake, pred_real = orc.discriminate(sdD, opt, pre["input_tag"], fake, pre["image_tag"], pre["orient_mask"], True)
    label_tag = pre["input_tag"][:, 1:2]
    losses["GAN"] = orc.gan_loss_hinge(pred_fake, True, False, label_tag, opt)
    if not opt.no_ganFeat_loss and torch.sum(pre["input_tag"][:, 1] - pre["input_ref"][:, 1]) == 0:
        losses["GAN_Feat"] = orc.gan_feat_loss(pred_fake, pred_real, opt)
    return losses, fake, mu, logvar


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_vae.npz")


def fixture_inputs():
    """(z npz, cfg, sdG, sdD, sdE, pre, eps, k) of golden_vae.npz, rebuilt without the reference: the state dicts take their
    key layout from michigan_b200's own classes (equal to the reference's, tests/test_vae_glue.py) and the values from
    fill_state_dict; the inputs from synthetic_batch; k is the dilation make_golden_vae.py drew."""
    import json

    import numpy as np
    from michigan_b200 import networks
    from michigan_b200.options import make_opt
    from michigan_b200.synth import fill_state_dict, synthetic_batch
    z = np.load(GOLDEN)
    c = json.loads(bytes(z["config"]).decode())
    opt = make_opt(ngf=c["ngf"], ndf=c["ndf"], crop_size=c["size"], gpu_ids=[], use_vae=True)
    sds = []
    for net, seed in ((networks.SPADEBGenerator(opt), c["seed_G"]), (networks.MultiscaleDiscriminator(opt), c["seed_D"]),
                      (networks.ConvEncoder(opt), c["seed_E"])):
        sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
        fill_state_dict(sd, seed)
        sds.append(sd)
    data = synthetic_batch(c["batch"], c["size"], c["data_seed"])
    pre = dict(input_ref=orc.one_hot(data["label_ref"]), input_tag=orc.one_hot(data["label_tag"]), image_ref=data["image_ref"],
               image_tag=data["image_tag"], orient_mask=data["orient"], noise=data["noise"])
    import random
    random.seed(c["py_seed"])
    th = int(c["size"] * 0.05)
    th = th if th % 2 == 1 else th + 1
    k = random.choice([max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4])
    return z, c, sds[0], sds[1], sds[2], data, pre, torch.from_numpy(z["eps"]), k
