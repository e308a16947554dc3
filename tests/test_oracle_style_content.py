"""The style / content / background / rgb oracle (tests/oracle_style_content.py) against the outputs of the reference's own
classes on the same inputs (tests/golden/golden_style_content.npz, written by tests/golden/make_golden_style_content.py).
CPU only."""
import os

import numpy as np
import torch

import oracle_style_content as osc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_style_content.npz")


def _inputs(n=2, size=64, seed=0):
    """fake, ref, tag [n,3,size,size] in (-1, 1) with ref != tag, and the one-hot [n,2,size,size] label (channel 1 = an elliptic
    hair region, channel 0 = background): the golden fixture's inputs."""
    from test_oracle_vgg_lab import _inputs as images
    fake, tag = images(n, size, seed)
    _, ref = images(n, size, seed + 1)
    yy, xx = torch.meshgrid(torch.arange(size).float(), torch.arange(size).float(), indexing="ij")
    hair = torch.stack([(((yy - size * (0.4 + 0.1 * i)) / (0.3 * size)) ** 2 + ((xx - size / 2) / (0.35 * size)) ** 2 < 1).float()
                        for i in range(n)])
    sem = torch.stack([1 - hair, hair], 1)
    return fake, ref, tag, sem


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _check(name, loss, grad, z, tol_loss=1e-5, tol_grad=1e-4):
    ref = float(z[name + "_loss"])
    assert abs(float(loss) - ref) <= tol_loss * abs(ref), (name, float(loss), ref)
    assert _rel(grad, torch.from_numpy(z[name + "_grad"])) <= tol_grad, name


def test_style_content_oracle_matches_reference():
    from michigan_b200.synth import vgg19_state_dict
    z = np.load(GOLDEN)
    fake, ref, tag, _ = _inputs()
    sd = vgg19_state_dict(int(z["vgg_seed"]))
    for i, name in enumerate(("content", "style")):
        x = fake.clone().requires_grad_()
        loss = osc.style_content_loss(x, ref, tag, sd)[i]
        loss.backward()
        _check(name, loss, x.grad, z)


def test_background_and_rgb_oracle_match_reference():
    z = np.load(GOLDEN)
    fake, _, tag, sem = _inputs()
    x = fake.clone().requires_grad_()
    loss = osc.background_loss(x, sem, tag)
    loss.backward()
    _check("background", loss, x.grad, z)
    x = fake.clone().requires_grad_()
    loss = osc.rgb_loss(x, tag)
    loss.backward()
    _check("rgb", loss, x.grad, z)


def test_style_oracle_is_nan_free_with_dead_and_constant_channels():
    """calc_mean_std's eps keeps sigma > 0 for an all-zero channel (a dead ReLU) and for a constant one."""
    g = torch.Generator().manual_seed(0)
    f = torch.relu(torch.randn(2, 8, 4, 4, generator=g))
    f[:, 0] = 0.0
    f[:, 1] = 0.37
    s = torch.relu(torch.randn(2, 8, 4, 4, generator=g))
    x = f.clone().requires_grad_()
    osc.style_loss([x], [s]).backward()
    assert torch.isfinite(x.grad).all()
