"""The hair-average Lab loss oracle (tests/oracle_unpaired.py) against the outputs of the reference's own HairAvgLabLoss on the
same inputs (tests/golden/golden_hair_avg_lab.npz, written by tests/golden/make_golden_hair_avg_lab.py).  CPU only."""
import os

import numpy as np
import pytest
import torch

import oracle_unpaired as ou
from test_oracle_vgg_lab import _inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_hair_avg_lab.npz")
CASES = ("ref_not_tag", "empty_tag_hair", "empty_ref_hair")


def _blob(n, size, cy, cx, ry, rx):
    yy, xx = torch.meshgrid(torch.arange(size).float(), torch.arange(size).float(), indexing="ij")
    m = (((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1).float()
    return m.expand(n, 1, size, size).clone()


def cases(n=2, size=48):
    """name -> (fake, real, mask_fake, mask_real): images in (-1, 1), binary hair masks [n,1,size,size] of different shapes for
    the tag (mask_fake) and the reference (mask_real); one image of the second case has no tag hair, one of the third no
    reference hair."""
    fake, real = _inputs(n, size, seed=3)
    mf = _blob(n, size, 0.40 * size, 0.50 * size, 0.30 * size, 0.35 * size)
    mr = _blob(n, size, 0.55 * size, 0.45 * size, 0.25 * size, 0.40 * size)
    out = {"ref_not_tag": (fake, real, mf, mr)}
    e = mf.clone()
    e[1] = 0
    out["empty_tag_hair"] = (fake, real, e, mr)
    e = mr.clone()
    e[0] = 0
    out["empty_ref_hair"] = (fake, real, mf, e)
    return out


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("case", CASES)
def test_hair_avg_lab_oracle_matches_reference(case):
    z = np.load(GOLDEN)
    fake, real, mf, mr = cases()[case]
    x = fake.clone().requires_grad_()
    loss = ou.hair_avg_lab_loss(x, real, mf, mr)
    loss.backward()
    assert abs(float(loss) - float(z[case + "_loss"])) <= 1e-6 * abs(float(z[case + "_loss"]))
    ref_grad = torch.from_numpy(z[case + "_grad"])
    assert _rel(x.grad, ref_grad) <= 1e-5
    if case == "empty_tag_hair":
        # a mask sum of 0 counts as 1: that image's average is 0 and it receives no gradient
        assert float(x.grad[1].abs().max()) == 0.0 and float(ref_grad[1].abs().max()) == 0.0
