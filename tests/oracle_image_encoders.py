"""Torch restatement of the reference's pooled appearance encoders (CPU or GPU, any dtype), pinned to
tests/golden/golden_image_encoders.npz by tests/test_oracle_image_encoders.py:

  * ImageEncoder.forward, --Image_encoder_mode norm (models/networks/encoder.py:89-105);
  * ImageEncoder2.forward, --Image_encoder_mode instance, with and without --ref_global_pool (encoder.py:132-158);
  * SPADEBGenerator.forward with either of them as `fc` (generator.py:117-123), then the blocks of
    michigan_oracle.generator_forward.
"""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import michigan_oracle as orc  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_image_encoders.npz")
# fixture case -> (Image_encoder_mode, ref_global_pool)
CASES = {"instance": ("instance", False), "instance_global": ("instance", True), "norm": ("norm", False)}


def sn_stack(sd, prefix, x, training):
    """layer1 .. layer5, each norm_E = spectral-norm conv k3 s2 p1 without bias + InstanceNorm, LeakyReLU before layers 2-5
    and after layer 5 (power iteration in place on sd's u, v when training)."""
    for i in range(1, 6):
        if i > 1:
            x = orc.lrelu(x)
        w = orc.conv_weight(sd, prefix + "layer%d.0" % i, training)
        x = F.instance_norm(F.conv2d(x, w, None, stride=2, padding=1))
    return orc.lrelu(x)


def image_encoder(sd, prefix, image_ref, ngf, sh, sw, training):
    """encoder.py:89-105: resize to 256x256, five layers, global average pool, 1x1 fc viewed as [N, 16 ngf, sh, sw]."""
    x = image_ref
    if x.shape[2] != 256 or x.shape[3] != 256:
        x = F.interpolate(x, size=(256, 256), mode="bilinear")
    x = sn_stack(sd, prefix, x, training)
    x = x.mean(dim=(2, 3), keepdim=True)
    x = F.conv2d(x, sd[prefix + "fc.weight"], sd[prefix + "fc.bias"])
    return x.view(x.shape[0], 16 * ngf, sh, sw)


def image_encoder2(sd, prefix, image_ref, label_ref, label_tag, ref_global_pool, sh, sw, training):
    """encoder.py:132-158: five layers at full resolution, then per image the reference-hair (or global) mean broadcast
    onto the target hair, nearest-resized to (sh, sw) when the map's height differs."""
    x = sn_stack(sd, prefix, image_ref, training)
    xh, xw = x.shape[2:]
    lr = F.interpolate(label_ref, size=(xh, xw), mode="nearest")
    lt = F.interpolate(label_tag, size=(xh, xw), mode="nearest")
    if ref_global_pool:
        mean = x.mean(dim=(2, 3), keepdim=True)
    else:
        count = lr.sum(dim=(2, 3), keepdim=True)
        mean = (x * lr).sum(dim=(2, 3), keepdim=True) / torch.clamp(count, min=1)
    out = mean * lt
    if sh != xh:
        out = F.interpolate(out, size=(sh, sw), mode="nearest")
    return out


def encode(sd, opt, mode, ref_global_pool, input_ref, input_tag, image_ref, training):
    """generator.py:117-123: the fc branch of --use_encoder for `mode`."""
    sw, sh = orc.latent_size(opt)
    if mode == "norm":
        return image_encoder(sd, "fc.", image_ref, opt.ngf, sh, sw, training)
    return image_encoder2(sd, "fc.", image_ref, input_ref[:, 1:2], input_tag[:, 1:2], ref_global_pool, sh, sw, training)


def generator_forward(sd, opt, mode, ref_global_pool, input_ref, input_tag, image_ref, image_tag, orient_mask, noise, training,
                      rng_k=None):
    """generator.py:107-230 with --use_encoder and --Image_encoder_mode `mode`."""
    x = encode(sd, opt, mode, ref_global_pool, input_ref, input_tag, image_ref, training)
    hair = input_tag[:, 1:2]
    seg = torch.cat([input_tag, orc.orient_channels(orient_mask, hair, opt)], dim=1)
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


def compute_generator_loss(sdG, sdD, opt, mode, ref_global_pool, pre, rng_k=None):
    """Pix2PixModel.compute_generator_loss with the GAN + GAN_Feat terms (pix2pix_model.py:257-297).  Returns (losses, fake)."""
    fake = generator_forward(sdG, opt, mode, ref_global_pool, pre["input_ref"], pre["input_tag"], pre["image_ref"],
                             pre["image_tag"], pre["orient_mask"], pre["noise"], True, rng_k)
    pred_fake, pred_real = orc.discriminate(sdD, opt, pre["input_tag"], fake, pre["image_tag"], pre["orient_mask"], True)
    label_tag = pre["input_tag"][:, 1:2]
    losses = {"GAN": orc.gan_loss_hinge(pred_fake, True, False, label_tag, opt)}
    if not opt.no_ganFeat_loss and torch.sum(pre["input_tag"][:, 1] - pre["input_ref"][:, 1]) == 0:
        losses["GAN_Feat"] = orc.gan_feat_loss(pred_fake, pred_real, opt)
    return losses, fake


def shifted_ref(data, shift):
    """Image 1's reference hair moved `shift` pixels right: the two masks differ at the encoder's map grid, their areas (so
    sum(tag - ref), pix2pix_model.py:286) do not, and GAN_Feat stays in the objective."""
    out = dict(data)
    lab = data["label_ref"].clone()
    lab[1] = torch.roll(lab[1], shifts=shift, dims=-1)
    out["label_ref"] = lab
    return out


def fixture_inputs(case):
    """(npz, cfg, sdG, sdD, data, pre, k) of one case of golden_image_encoders.npz, rebuilt without the reference: the state
    dicts take their key layout from michigan_b200's own classes (equal to the reference's, tests/test_image_encoders_glue.py)
    and the values from fill_state_dict; the inputs from synthetic_batch and shifted_ref; k is the dilation
    make_golden_image_encoders.py drew."""
    import json
    import random

    import numpy as np
    from michigan_b200 import networks
    from michigan_b200.options import make_opt
    from michigan_b200.synth import fill_state_dict, synthetic_batch
    z = np.load(GOLDEN)
    c = json.loads(bytes(z["config"]).decode())
    mode, gp = CASES[case]
    opt = make_opt(ngf=c["ngf"], ndf=c["ndf"], crop_size=c["size"], gpu_ids=[], Image_encoder_mode=mode, ref_global_pool=gp)
    sds = []
    for net, seed in ((networks.SPADEBGenerator(opt), c["seed_G"]), (networks.MultiscaleDiscriminator(opt), c["seed_D"])):
        sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
        fill_state_dict(sd, seed)
        sds.append(sd)
    data = shifted_ref(synthetic_batch(c["batch"], c["size"], c["data_seed"]), c["shift"])
    pre = dict(input_ref=orc.one_hot(data["label_ref"]), input_tag=orc.one_hot(data["label_tag"]), image_ref=data["image_ref"],
               image_tag=data["image_tag"], orient_mask=data["orient"], noise=data["noise"])
    random.seed(c["py_seed"])
    th = int(c["size"] * 0.05)
    th = th if th % 2 == 1 else th + 1
    k = random.choice([max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4])
    return z, c, sds[0], sds[1], data, pre, k
