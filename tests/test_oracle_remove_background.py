"""The --remove_background oracle (tests/oracle_remove_background.py) against the outputs of the reference's own VGGLoss and
StyleContentLoss with remove_background=True on the same inputs (tests/golden/golden_remove_background.npz, written by
tests/golden/make_golden_remove_background.py).  CPU only."""
import os

import numpy as np
import pytest
import torch

import oracle_remove_background as orb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_remove_background.npz")
CASES = ("crossed", "no_tag_hair", "no_ref_hair", "full")


def _ellipse(size, cy, cx, ry, rx):
    yy, xx = torch.meshgrid(torch.arange(size).float(), torch.arange(size).float(), indexing="ij")
    return ((((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2) < 1).float()


def _inputs(case, n=2, size=64):
    """fake, ref, tag [n,3,size,size] in (-1, 1) with ref != tag, and the [n,1,size,size] hair labels of the reference image
    (style_label) and of the tag (content_label), which differ in every case but 'full':
      crossed      two different ellipses per image;
      no_tag_hair  image 0's tag label is empty;
      no_ref_hair  image 1's reference label is empty;
      full         both labels all hair."""
    from test_oracle_style_content import _inputs as images
    fake, ref, tag, sem = images(n, size)
    lab_tag = sem[:, 1:2].clone()
    lab_ref = torch.stack([_ellipse(size, size * (0.55 - 0.1 * i), size * (0.4 + 0.15 * i), 0.25 * size, 0.3 * size)
                           for i in range(n)])[:, None]
    if case == "no_tag_hair":
        lab_tag[0] = 0.0
    elif case == "no_ref_hair":
        lab_ref[1] = 0.0
    elif case == "full":
        lab_tag = torch.ones_like(lab_tag)
        lab_ref = torch.ones_like(lab_ref)
    return fake, ref, tag, lab_ref, lab_tag


def oracle_terms(sd, fake, ref, tag, lab_ref, lab_tag):
    """name -> callable of the fake image: the three losses the golden fixture stores."""
    return {
        "vgg": lambda x: orb.vgg_loss(x, tag, lab_tag, sd),
        "content": lambda x: orb.style_content_loss(x, ref, tag, lab_ref, lab_tag, sd)[0],
        "style": lambda x: orb.style_content_loss(x, ref, tag, lab_ref, lab_tag, sd)[1],
    }


def _rel(a, b):
    return float((a - b).norm() / b.norm()) if float(b.norm()) > 0 else float(a.norm())


@pytest.mark.parametrize("case", CASES)
def test_remove_background_oracle_matches_reference(case):
    from michigan_b200.synth import vgg19_state_dict
    z = np.load(GOLDEN)
    sd = vgg19_state_dict(int(z["vgg_seed"]))
    fake, ref, tag, lab_ref, lab_tag = _inputs(case)
    for name, fn in oracle_terms(sd, fake, ref, tag, lab_ref, lab_tag).items():
        x = fake.clone().requires_grad_()
        loss = fn(x)
        loss.backward()
        want = float(z["%s/%s_loss" % (case, name)])
        assert abs(float(loss) - want) <= 1e-5 * abs(want), (case, name, float(loss), want)
        assert _rel(x.grad, torch.from_numpy(z["%s/%s_grad" % (case, name)])) <= 1e-4, (case, name)


def test_masked_statistics_of_an_empty_mask():
    """No mask pixel: mu = 0, sigma = sqrt(eps), and no gradient reaches the features."""
    g = torch.Generator().manual_seed(0)
    f = torch.relu(torch.randn(2, 8, 4, 4, generator=g)).requires_grad_()
    m = torch.zeros(2, 1, 4, 4)
    m[1, :, 1:3] = 1.0
    mu, sigma = orb.calc_mean_std_mask(f, m)
    assert float(mu[0].abs().max()) == 0.0
    assert torch.allclose(sigma[0], torch.full_like(sigma[0], orb.EPS ** 0.5))
    (mu.sum() + sigma.sum()).backward()
    assert float(f.grad[0].abs().max()) == 0.0 and float(f.grad[1].abs().max()) > 0.0
