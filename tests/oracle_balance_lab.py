"""CPU oracle of the count-balanced Lab losses of --balance_Lab, in plain fp32 PyTorch, restating the reference:

  * the weight (cal_weight, models/networks/loss.py:487-513, 578-597): the count table T in fp32 with T == 0 -> 1, max(T) / T,
    clamped at Lab_weight_th, read by grid_sample (mode 'nearest', torch's defaults) at ((int bins of (b, a) + 128, clamped
    to [0, 255]) - 127.5) / 127.5, per pixel of the real image (LabColorLoss) or per image of its hair averages
    (HairAvgLabLoss);
  * LabColorLoss (loss.py:515-531): w = lookup * mask with 0 -> 1, mean(w |ab_fake - ab_real|) over N x 2 x H x W;
  * HairAvgLabLoss (loss.py:599-621): w = lookup (no mask, no 0 -> 1), mean(w |avg_ab_fake - avg_ab_real|) over N x 2.

`count_table(seed)` is the synthetic colour-count table the tests use in place of the reference's data/ab_count.npy.
Pinned against the live reference by tests/golden/make_golden_balance_lab.py (tests/golden/golden_balance_lab.npz)."""
import numpy as np
import torch
import torch.nn.functional as F

import oracle_vgg_lab as ovl
from oracle_unpaired import cal_hair_avg

TABLE_SEED = 20
THRESHOLDS = (10.0, 2.5)


def count_table(seed=TABLE_SEED):
    """[256,256] float64 counts: log-uniform over 1 .. 1e8 (so that the clamp at Lab_weight_th bites), a third of them 0, and
    no symmetry between the a (row) and b (column) bins."""
    g = np.random.default_rng(seed)
    t = np.floor(10.0 ** g.uniform(0.0, 8.0, size=(256, 256)))
    t[g.random((256, 256)) < 0.33] = 0.0
    return t


def weight_map(table, th):
    """The reference's processed table, [1,1,256,256] fp32."""
    w = torch.tensor(table, dtype=torch.float32).view(1, 1, 256, 256)
    w[w == 0] = 1
    w = w.max() / w
    w[w > th] = th
    return w


def lookup(w, a, b):
    """grid_sample of the processed table w at the bins of a and b ([N,1,H,W] fp32) -> [N,1,H,W]."""
    m = (torch.cat([b, a], 1) + 128).clamp(0, 255).int().float()
    grid = ((m - 127.5) / 127.5).permute(0, 2, 3, 1)
    return F.grid_sample(w.expand(a.shape[0], 1, 256, 256), grid, mode="nearest", padding_mode="zeros", align_corners=False)


def lab_color_loss_balanced(fake, real, mask, w):
    lf, lr = ovl.rgb2lab(fake), ovl.rgb2lab(real).detach()
    wm = lookup(w, lr[:, 1:2], lr[:, 2:3]) * mask
    wm = torch.where(wm == 0, torch.ones_like(wm), wm)
    return (wm * (lf[:, 1:] - lr[:, 1:]).abs()).mean()


def hair_avg_lab_loss_balanced(fake, real, mask_fake, mask_real, w):
    af = cal_hair_avg(ovl.rgb2lab(fake), mask_fake)
    ar = cal_hair_avg(ovl.rgb2lab(real), mask_real).detach()
    wm = lookup(w, ar[:, 1:2], ar[:, 2:3])
    return (wm * (af[:, 1:] - ar[:, 1:]).abs()).mean()


def _lab64(img):
    rgb = (img.double() + 1) / 2
    M = ovl._M.double()
    xyz = torch.einsum("nc,bchw->bnhw", M, rgb) / M.sum(dim=1).view(1, 3, 1, 1)
    f = torch.where(xyz > 0.008856, xyz.clamp(min=0.008856).pow(1 / 3), 7.787 * xyz + 0.137931)
    return torch.stack([500 * (f[:, 0] - f[:, 1]), 200 * (f[:, 1] - f[:, 2])], 1)


def _near_integer(v, margin):
    return ((v + 128) - (v + 128).round()).abs() < margin


def golden_inputs(seed=11, n=2, size=32, margin=1e-3):
    """name -> (fake, real, mask_fake, mask_real), real drawn by rejection so that every pixel's a + 128, b + 128 and every
    image's hair-averaged a + 128, b + 128 (with mask_real) lie at least `margin` from an integer in float64: the bins do not
    depend on rounding.  Cases: partial hair (different tag and reference masks), an image without hair in either mask (its
    average is 0, bin 128), all hair."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(size).float(), torch.arange(size).float(), indexing="ij")
    blob_f = ((((yy - 0.4 * size) / (0.3 * size)) ** 2 + ((xx - 0.5 * size) / (0.35 * size)) ** 2) <= 1).float()
    blob_r = ((((yy - 0.55 * size) / (0.25 * size)) ** 2 + ((xx - 0.45 * size) / (0.4 * size)) ** 2) <= 1).float()
    masks = {"partial": (blob_f.expand(n, 1, size, size).clone(), blob_r.expand(n, 1, size, size).clone())}
    mf, mr = masks["partial"][0].clone(), masks["partial"][1].clone()
    mf[1] = 0
    mr[1] = 0
    masks["no_hair"] = (mf, mr)
    masks["all_hair"] = (torch.ones(n, 1, size, size), torch.ones(n, 1, size, size))
    out = {}
    for name, (mf, mr) in masks.items():
        fake = torch.rand(n, 3, size, size, generator=g) * 2 - 1
        real = torch.rand(n, 3, size, size, generator=g) * 2 - 1
        for _ in range(10000):
            ab = _lab64(real)
            bad = _near_integer(ab, margin).any(1)                       # [n, H, W]
            cnt = mr.double().sum((2, 3))
            avg = (ab * mr.double()).sum((2, 3)) / torch.where(cnt == 0, torch.ones_like(cnt), cnt)
            bad_avg = _near_integer(avg, margin).any(1) & (cnt[:, 0] > 0)
            for i in torch.nonzero(bad_avg).flatten().tolist():
                # redraw one random hair pixel of that image
                k = int(torch.randint(int(cnt[i, 0]), (1,), generator=g))
                y, x = torch.nonzero(mr[i, 0])[k].tolist()
                bad[i, y, x] = True
            if not bool(bad.any()):
                break
            fresh = torch.rand(n, 3, size, size, generator=g) * 2 - 1
            real = torch.where(bad.unsqueeze(1), fresh, real)
        else:
            raise RuntimeError("rejection sampling did not converge")
        out[name] = (fake.contiguous(), real.contiguous(), mf, mr)
    return out
