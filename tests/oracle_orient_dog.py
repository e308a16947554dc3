"""Torch restatement of the reference's DoG orientation loss (models/networks/loss.py:245-271 DoG_fn, 320-385 L1OLoss with an
orient_filter other than 'gabor'), and the fixed inputs of its tests.

The confidence of every pixel is its clamped maximum response times the hair mask, divided by M, the maximum of that product
over the whole batch; pixels where the quotient is <= 0 get 0.  ORIENT is the mean over N*2*H*W of |orient*hair - label2*hair|
and CONFIDENCE = sum |conf*hair - hair| / (sum hair + 1e-5).  The gradient of M (torch splits it evenly among tied maxima)
reaches the image through the 17x17 footprint of the maximising pixel.
"""
import math

import torch
import torch.nn.functional as F

CASES = ("angle", "use_ig", "one_empty", "tie", "no_hair", "fractional")
NON_TIE = ("angle", "use_ig", "one_empty", "fractional")


def gray_of(img):
    f = (img + 1) / 2.0 * 255
    return (0.299 * f[:, 0] + 0.587 * f[:, 1] + 0.144 * f[:, 2]).unsqueeze(1)


def responses(img, bank):
    """[N,32,H,W] responses of the [17*17][32] bank on the image's gray (fp32 conv, pad 8)."""
    w = bank.t().reshape(32, 1, 17, 17).to(img.dtype)
    return F.conv2d(gray_of(img), w, padding=8)


def orient_loss_dog(img, label, sem, use_ig, bank):
    """(ORIENT, CONFIDENCE) of img [N,3,H,W] in [-1,1]; label: the [N,1,H,W] angle map (0..255) or, with use_ig, the
    [N,2,H,W] (sin 2t, cos 2t) map; sem [N,2,H,W] with the hair mask in channel 1."""
    hair = sem[:, 1:2]
    r, idx = responses(img, bank).clamp(min=0).max(dim=1, keepdim=True)
    conf = r * hair
    conf = conf / conf.max()
    conf = conf * (~(conf <= 0)).to(conf.dtype)
    a = idx.float() * math.pi / 32
    orient = torch.cat([torch.sin(2 * a), torch.cos(2 * a)], dim=1).to(conf.dtype) * conf
    if use_ig:
        label2 = label
    else:
        t = label / 255 * math.pi
        label2 = torch.cat([torch.sin(2 * t), torch.cos(2 * t)], dim=1)
    lo = (orient * hair - label2 * hair).abs().mean()
    lc = (conf * hair - hair).abs().sum() / (hair.sum() + 1e-5)
    return lo, lc


def cases():
    """name -> (img, label, sem, use_ig): the inputs of tests/test_gpu_orient.py (2 x 96^2) and five variants."""
    from test_gpu_orient import _inputs
    img, orient, sem = _inputs()
    g = torch.Generator().manual_seed(7)
    out = {"angle": (img, orient, sem, False)}
    out["use_ig"] = (img, torch.rand(img.shape[0], 2, *img.shape[2:], generator=g) * 2 - 1, sem, True)
    s1 = sem.clone()
    s1[1, 1] = 0
    s1[1, 0] = 1
    out["one_empty"] = (img, orient, s1, False)
    it = img.clone()
    it[1] = it[0]
    st = sem.clone()
    st[1] = st[0]
    out["tie"] = (it, orient, st, False)
    s0 = sem.clone()
    s0[:, 1] = 0
    s0[:, 0] = 1
    out["no_hair"] = (img, orient, s0, False)
    sf = sem.clone()
    sf[:, 1] = sem[:, 1] * torch.rand(sem.shape[0], *sem.shape[2:], generator=g).clamp(min=0.05)
    out["fractional"] = (img, orient, sf, False)
    return out


def top_products(img, sem, bank, k=3):
    """The k largest values of r * hair over the batch (fp32), to check that a case's maximiser is unique."""
    r = responses(img, bank).clamp(min=0).max(dim=1, keepdim=True)[0]
    return (r * sem[:, 1:2]).flatten().topk(k).values
