"""The DoG orientation loss restatement (tests/oracle_orient_dog.py) against the reference's own L1OLoss (orient_filter 'dog'),
stored by tests/golden/make_golden_orient_dog.py, and networks.loss.dog_bank against the reference's DoG_fn, bit for bit."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import oracle_orient_dog as od

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import ref_shims  # noqa: E402


@pytest.mark.parametrize("case", od.CASES)
def test_oracle_matches_the_reference_golden(case):
    from michigan_b200.networks.loss import dog_bank
    z = np.load(os.path.join(ROOT, "tests", "golden", "golden_orient_dog.npz"))
    img, label, sem, use_ig = od.cases()[case]
    x = img.clone().requires_grad_()
    lo, lc = od.orient_loss_dog(x, label, sem, use_ig, dog_bank("cpu"))
    (lo * 10.0 + lc * 100.0).backward()
    g = torch.from_numpy(z[case + "_g"])
    if case == "no_hair":
        assert math.isnan(float(z[case + "_lo"])) and math.isnan(float(lo)) and math.isnan(float(lc))
        assert torch.isnan(g).all() and torch.isnan(x.grad).all()
        return
    assert abs(float(lo) - float(z[case + "_lo"])) <= 1e-6 * abs(float(z[case + "_lo"]))
    assert abs(float(lc) - float(z[case + "_lc"])) <= 1e-6 * abs(float(z[case + "_lc"]))
    assert float((x.grad - g).norm() / g.norm()) <= 1e-5
    if case == "one_empty":
        assert float(x.grad[1].abs().max()) == 0.0 and float(g[1].abs().max()) == 0.0


@pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")
def test_dog_bank_is_the_reference_dog_fn_bit_for_bit():
    from make_golden_orient_dog import cuda_is_identity
    from michigan_b200.networks.loss import dog_bank
    ref_shims.import_reference()
    loss_mod = __import__("models.networks.loss", fromlist=["DoG_fn"])
    bank = dog_bank("cpu")
    assert bank.shape == (289, 32) and bank.dtype == torch.float32
    with cuda_is_identity():
        for k in range(32):
            theta = torch.nn.Parameter(torch.ones(1) * (math.pi * k / 32), requires_grad=False)
            ref = loss_mod.DoG_fn(17, 1, 1, theta).float().reshape(289)
            assert torch.equal(bank[:, k], ref), k
