"""The VGG19 perceptual / Lab colour loss oracle (tests/oracle_vgg_lab.py) against the outputs of the reference's own classes on
the same inputs (tests/golden/golden_vgg_lab.npz, written by tests/golden/make_golden_vgg_lab.py).  CPU only."""
import os

import numpy as np
import torch

import oracle_vgg_lab as ovl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_vgg_lab.npz")


def _inputs(n=2, size=64, seed=0):
    """fake, real: [n,3,size,size] in (-1, 1), smooth structure plus noise (the golden fixture's inputs)."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(size).float(), torch.arange(size).float(), indexing="ij")
    base = torch.stack([torch.sin(0.21 * xx + 0.1 * yy), torch.cos(0.13 * yy), torch.sin(0.05 * (xx + yy))]).unsqueeze(0) * 0.6
    fake = (base + 0.25 * torch.randn(n, 3, size, size, generator=g)).clamp(-0.98, 0.98)
    real = (base.flip(-1) + 0.25 * torch.randn(n, 3, size, size, generator=g)).clamp(-0.98, 0.98)
    return fake, real


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def test_vgg_loss_oracle_matches_reference():
    from michigan_b200.synth import vgg19_state_dict
    z = np.load(GOLDEN)
    fake, real = _inputs()
    x = fake.clone().requires_grad_()
    loss = ovl.vgg_loss(x, real, vgg19_state_dict(int(z["vgg_seed"])))
    loss.backward()
    assert abs(float(loss) - float(z["vgg_loss"])) <= 1e-5 * abs(float(z["vgg_loss"]))
    assert _rel(x.grad, torch.from_numpy(z["vgg_grad"])) <= 1e-4


def test_lab_loss_oracle_matches_reference():
    z = np.load(GOLDEN)
    fake, real = _inputs()
    x = fake.clone().requires_grad_()
    loss = ovl.lab_loss(x, real)
    loss.backward()
    assert abs(float(loss) - float(z["lab_loss"])) <= 1e-5 * abs(float(z["lab_loss"]))
    assert _rel(x.grad, torch.from_numpy(z["lab_grad"])) <= 1e-5


def test_lab_oracle_gradient_is_finite_at_saturated_pixels():
    """fake = -1 exactly gives X = Y = Z = 0: the cube-root branch is not taken and its derivative must not leak a NaN."""
    fake, real = _inputs(n=1, size=16)
    fake[:, :, :4] = -1.0
    fake[:, :, 4:8] = 1.0
    x = fake.clone().requires_grad_()
    ovl.lab_loss(x, real).backward()
    assert torch.isfinite(x.grad).all()
    assert x.grad[:, :, :4].abs().sum() > 0
