"""Deterministic synthetic weights and inputs (there is no network for checkpoints or datasets).

* `fill_state_dict` fills any state dict with values that depend only on (seed, key, shape), so that
  the reference networks (in tests/golden/make_golden.py), the CPU oracle and the CUDA modules can be
  given bit-identical weights without shipping a 438 MB checkpoint.  numpy's legacy RandomState is
  used on purpose: its stream is frozen across numpy versions.
* `synthetic_batch` builds the `data` dict consumed by Pix2PixModel.forward with the shapes and value
  ranges of the reference's data loader (data/base_dataset.py:149-159, data/pix2pix_dataset.py:178-188;
  SURVEY.md §8d).
"""
import zlib

import numpy as np
import torch


def _rs(seed, key):
    return np.random.RandomState((zlib.crc32(key.encode()) ^ (seed * 2654435761)) & 0x7FFFFFFF)


def fill_state_dict(sd, seed=0, power_iters=30):
    """In-place deterministic fill.  Conv weights ~ N(0, 1/(3 fan_in)) - the variance of PyTorch's default
    Conv2d init (kaiming_uniform, a=sqrt(5)), the regime in which SURVEY.md quotes the 1e-3 output bound
    (output std ~ 0.1) - biases ~ N(0, 0.02^2); spectral-norm
    u, v are the converged power-iteration vectors of the filled weight (so eval-mode W/sigma is
    well-scaled, unlike a never-trained random u, v: SURVEY.md §7 'random-init eval is degenerate');
    BN running stats: mean 0, var 1 (calibrate them with a train-mode forward if needed)."""
    for key in list(sd.keys()):
        t = sd[key]
        if key.endswith("num_batches_tracked"):
            t.zero_()
            continue
        r = _rs(seed, key)
        if key.endswith("running_mean"):
            t.zero_()
        elif key.endswith("running_var"):
            t.fill_(1.0)
        elif key.endswith("weight_u") or key.endswith("weight_v"):
            continue  # after the weights
        elif key.endswith("bias"):
            t.copy_(torch.from_numpy((r.standard_normal(tuple(t.shape)) * 0.02).astype(np.float32)))
        elif t.dim() >= 2:
            fan_in = int(np.prod(t.shape[1:]))
            t.copy_(torch.from_numpy((r.standard_normal(tuple(t.shape)) / np.sqrt(3.0 * fan_in)).astype(np.float32)))
        else:
            t.copy_(torch.from_numpy(r.standard_normal(tuple(t.shape)).astype(np.float32)))
    for key in list(sd.keys()):
        if key.endswith("weight_u"):
            base = key[: -len("weight_u")]
            w = sd[base + "weight_orig"].detach().double().cpu()
            # torch's spectral_norm flattens around dim 0, or dim 1 for ConvTranspose (InpaintGenerator's decoder,
            # generator.py:539-545): recognisable by the length of the stored u
            if sd[key].numel() != w.shape[0] and w.dim() > 1 and sd[key].numel() == w.shape[1]:
                w = w.transpose(0, 1)
            mat = w.reshape(w.shape[0], -1)
            u = torch.from_numpy(_rs(seed, key).standard_normal(mat.shape[0]))
            u = u / u.norm()
            for _ in range(power_iters):
                v = mat.t() @ u
                v = v / v.norm()
                u = mat @ v
                u = u / u.norm()
            sd[key].copy_(u.float())
            sd[base + "weight_v"].copy_(v.float())
    return sd


def vgg19_state_dict(seed=0):
    """A deterministic stand-in for the ImageNet VGG19 weights in torchvision's layout (`features.N.{weight,bias}`, the 16 convs
    of vgg19().features; the classifier is not needed): He-normal weights N(0, 2/fan_in), so that ReLU activations stay O(1)
    through the 13 convs the perceptual loss uses, and biases N(0, 0.01^2)."""
    sd, cin, i = {}, 3, 0
    for v in [64, 64, "M", 128, 128, "M", 256, 256, 256, 256, "M", 512, 512, 512, 512, "M", 512, 512, 512, 512, "M"]:
        if v == "M":
            i += 1
            continue
        key = "features.%d" % i
        sd[key + ".weight"] = torch.from_numpy((_rs(seed, key + ".weight").standard_normal((v, cin, 3, 3)) *
                                                np.sqrt(2.0 / (9 * cin))).astype(np.float32))
        sd[key + ".bias"] = torch.from_numpy((_rs(seed, key + ".bias").standard_normal(v) * 0.01).astype(np.float32))
        cin = v
        i += 2
    return sd


def synthetic_batch(n, size=512, seed=1234, use_ig=False, device="cpu"):
    """The data dict of SURVEY.md §8d: hair = axis-aligned box (~23 % of pixels), ref == tag so that the
    GAN-feature loss is active (pix2pix_model.py:286-297)."""
    g = torch.Generator().manual_seed(seed)
    s = size / 512.0
    label = torch.zeros(n, 1, size, size)
    label[:, :, int(102 * s):int(307 * s), int(102 * s):int(410 * s)] = 1.0
    image = torch.rand(n, 3, size, size, generator=g) * 2 - 1
    orient = torch.floor(torch.rand(n, 1, size, size, generator=g) * 255) * label
    noise = torch.rand(n, 3, size, size, generator=g)
    data = {
        "label_ref": label.clone(), "label_tag": label.clone(), "instance": torch.zeros(n),
        "image_ref": image.clone(), "image_tag": image.clone(), "orient": orient, "noise": noise,
        "hole": torch.zeros(n, 1, size, size), "orient_rgb": torch.zeros(n, 3, size, size),
        "path": ["synthetic_%d" % i for i in range(n)],
    }
    if use_ig:
        yy, xx = torch.meshgrid(torch.arange(size), torch.arange(size), indexing="ij")
        disk = (((yy - size * 0.4) ** 2 + (xx - size * 0.5) ** 2) < (size * 0.15) ** 2).float()
        data["hole"] = (label * disk.view(1, 1, size, size)).contiguous()
        th = orient / 255.0 * np.pi
        data["orient_rgb"] = torch.cat([(torch.cos(2 * th) + 1) / 2, (torch.sin(2 * th) + 1) / 2,
                                        torch.full_like(th, 0.5)], 1) * label
    if device != "cpu":
        data = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in data.items()}
    return data
