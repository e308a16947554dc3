"""The adversarial-loss oracle (tests/oracle_gan_objectives.py) against the outputs of the reference's own GANLoss and
GANFeatLoss on the same inputs (tests/golden/golden_gan_objectives.npz, written by tests/golden/make_golden_gan_objectives.py):
every gan_mode, non-default target labels, the wide-edge weight map, and --remove_background with a hair label, a full one
and an empty one.  CPU only."""
import os

import numpy as np
import pytest
import torch

import oracle_gan_objectives as og

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_gan_objectives.npz")
LABEL_SIZE = 48


def _label(n, kind):
    if kind == "empty":
        return torch.zeros(n, 1, LABEL_SIZE, LABEL_SIZE)
    if kind == "full":
        return torch.ones(n, 1, LABEL_SIZE, LABEL_SIZE)
    yy, xx = torch.meshgrid(torch.arange(LABEL_SIZE).float(), torch.arange(LABEL_SIZE).float(), indexing="ij")
    m = ((((yy - 21) / 13) ** 2 + ((xx - 25) / 16) ** 2) <= 1).float()
    out = m.expand(n, 1, LABEL_SIZE, LABEL_SIZE).clone()
    out[1:, :, :, :5] = 1
    return out


def inputs(n=2, seed=5):
    """(pred_fake, pred_real): two discriminators, each [features [n,4,h,w], logits [n,1,h',w']] at 37x37 / 35x35 and 9x9 / 5x5
    (odd ratios to the 48x48 label; the wide-edge pooling window is 2 at 35x35); logits with planted values 1, -1 and 0 (hinge ties, BCE at 0) and a few of |x| = 30."""
    g = torch.Generator().manual_seed(seed)

    def disc():
        out = []
        for (fh, lh) in ((37, 35), (9, 5)):
            f = torch.randn(n, 4, fh, fh, generator=g) * 1.5
            x = torch.randn(n, 1, lh, lh, generator=g) * 1.5
            flat = x.view(-1)
            flat[0::7], flat[1::7], flat[2::7] = 1.0, -1.0, 0.0
            flat[3::11] = 30.0 * torch.sign(flat[3::11])
            out.append([f, x])
        return out
    fake, real = disc(), disc()
    real[0][0].view(-1)[::5] = fake[0][0].view(-1)[::5]          # L1 ties
    return fake, real


# name -> (gan_mode, target_is_real, for_discriminator, wide_edge, remove_background, real_label, fake_label, label kind)
GAN_CASES = {}
for _mode in ("ls", "original", "w"):
    for _tag, _tir, _fd in (("d_real", True, True), ("d_fake", False, True), ("g", True, False)):
        GAN_CASES["%s_%s" % (_mode, _tag)] = (_mode, _tir, _fd, 1.0, False, 1.0, 0.0, "blob")
for _mode in ("ls", "original"):
    GAN_CASES["%s_targets_d_real" % _mode] = (_mode, True, True, 1.0, False, 0.9, 0.2, "blob")
    GAN_CASES["%s_targets_d_fake" % _mode] = (_mode, False, True, 1.0, False, 0.9, 0.2, "blob")
    GAN_CASES["%s_remove_background_ignored" % _mode] = (_mode, True, True, 2.0, True, 1.0, 0.0, "blob")
GAN_CASES.update({
    "hinge_wide_edge_d_real": ("hinge", True, True, 2.0, False, 1.0, 0.0, "blob"),
    "hinge_wide_edge_d_fake": ("hinge", False, True, 2.0, False, 1.0, 0.0, "blob"),
    "hinge_g": ("hinge", True, False, 2.0, False, 1.0, 0.0, "blob"),
    "hinge_d_real": ("hinge", True, True, 1.0, False, 1.0, 0.0, "blob"),
    "hinge_rb_d_real": ("hinge", True, True, 2.0, True, 1.0, 0.0, "blob"),
    "hinge_rb_d_fake": ("hinge", False, True, 2.0, True, 1.0, 0.0, "blob"),
    "hinge_rb_g": ("hinge", True, False, 2.0, True, 1.0, 0.0, "blob"),
    "hinge_rb_full_d_fake": ("hinge", False, True, 1.0, True, 1.0, 0.0, "full"),
    "hinge_rb_empty_d_real": ("hinge", True, True, 1.0, True, 1.0, 0.0, "empty"),
    "hinge_rb_empty_g": ("hinge", True, False, 1.0, True, 1.0, 0.0, "empty"),
})
# name -> (remove_background, label kind); lambda_feat 10
FEAT_CASES = {"feat": (False, "blob"), "feat_rb": (True, "blob"), "feat_rb_full": (True, "full"), "feat_rb_empty": (True, "empty")}
LAMBDA_FEAT = 10.0


def run_gan(case, crit_fn):
    """crit_fn(mode, real_label, fake_label, wide_edge, remove_background) -> a GANLoss-like callable; returns (loss, grad of
    the logits of both discriminators, flattened)."""
    mode, tir, fd, we, rb, rl, fl, kind = GAN_CASES[case]
    fake, real = inputs()
    preds = fake if not tir else real
    preds = [[t.clone().requires_grad_() for t in p] for p in preds]
    loss = crit_fn(mode, rl, fl, we, rb)(preds, tir, for_discriminator=fd, label=_label(2, kind))
    loss.sum().backward()
    return loss.detach(), torch.cat([p[-1].grad.reshape(-1) for p in preds])


def run_feat(case, crit_fn):
    rb, kind = FEAT_CASES[case]
    fake, real = inputs()
    fake = [[t.clone().requires_grad_() for t in p] for p in fake]
    loss = crit_fn(rb)(fake, real, _label(2, kind))
    loss.sum().backward()
    return loss.detach(), torch.cat([t.grad.reshape(-1) for p in fake for t in p[:-1]])


def oracle_gan(mode, rl, fl, we, rb):
    return lambda preds, tir, for_discriminator, label: og.gan_loss(preds, tir, for_discriminator, label, mode, we, rb, rl, fl)


def oracle_feat(rb):
    return lambda fake, real, label: og.gan_feat_loss(fake, real, label, LAMBDA_FEAT, rb)


def _check(name, loss, grad, z):
    want = float(z[name + "_loss"])
    gref = torch.from_numpy(z[name + "_grad"])
    assert loss.numel() == 1
    assert abs(float(loss) - want) <= 1e-6 * abs(want) + 1e-12, (name, float(loss), want)
    assert grad.shape == gref.shape
    assert float((grad - gref).abs().max()) <= 1e-6 * float(gref.abs().max()) + 1e-12, name


@pytest.mark.parametrize("case", list(GAN_CASES))
def test_gan_loss_oracle_matches_reference(case):
    z = np.load(GOLDEN)
    loss, grad = run_gan(case, oracle_gan)
    _check(case, loss, grad, z)
    if GAN_CASES[case][4] and GAN_CASES[case][0] == "hinge" and GAN_CASES[case][7] == "empty":
        assert float(loss) == 0.0 and float(grad.abs().max()) == 0.0


@pytest.mark.parametrize("case", list(FEAT_CASES))
def test_gan_feat_loss_oracle_matches_reference(case):
    z = np.load(GOLDEN)
    loss, grad = run_feat(case, oracle_feat)
    _check(case, loss, grad, z)
    if FEAT_CASES[case] == (True, "empty"):
        assert float(loss) == 0.0 and float(grad.abs().max()) == 0.0


def test_unknown_gan_mode_is_refused():
    from michigan_b200.networks.loss import GANLoss
    with pytest.raises(ValueError, match="Unexpected gan_mode"):
        GANLoss("wgan-gp")
    with pytest.raises(ValueError, match="Unexpected gan_mode"):
        og.gan_loss([torch.zeros(1, 1, 2, 2)], True, True, None, "softplus")
