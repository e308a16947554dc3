"""CPU: the --use_vae oracle (tests/oracle_vae.py) pinned to the reference's own generator step (tests/golden/golden_vae.npz)."""
import json

import numpy as np
import torch

import michigan_oracle as orc
import oracle_vae as ov
from helpers import assert_summary_close


def test_oracle_matches_reference_generator_step():
    z, c, sdG, sdD, sdE, _, pre, eps, k = ov.fixture_inputs()
    opt = orc.default_opt(ngf=c["ngf"], ndf=c["ndf"], crop_size=c["size"], isTrain=True)
    opt.lambda_kld = 0.05
    for sd in (sdG, sdE):
        for n, v in sd.items():
            if v.is_floating_point() and not n.endswith(("weight_u", "weight_v")):
                v.requires_grad_(True)
    losses, fake, mu, logvar = ov.compute_generator_loss(sdG, sdD, sdE, opt, pre, eps, rng_k=k)
    assert list(losses) == json.loads(bytes(z["loss_keys"]).decode()) == ["KLD", "GAN", "GAN_Feat"]
    for key, v in losses.items():
        assert abs(float(v.detach().mean()) - float(z["loss_" + key])) <= 1e-5 * max(1.0, abs(float(z["loss_" + key]))), key
    orc.trainer_loss(losses).backward()
    np.testing.assert_allclose(mu.detach().numpy(), z["mu"], rtol=0, atol=1e-5 * np.abs(z["mu"]).max())
    np.testing.assert_allclose(logvar.detach().numpy(), z["logvar"], rtol=0, atol=1e-5 * np.abs(z["logvar"]).max())
    g1 = z["grad_layer1.0.weight_orig"]
    np.testing.assert_allclose(sdE["layer1.0.weight_orig"].grad.numpy(), g1, rtol=0, atol=1e-4 * np.abs(g1).max())
    assert_summary_close("fake", fake, z["fake"], 1e-4)
    assert_summary_close("fc_mu.weight grad", sdE["fc_mu.weight"].grad, z["grad_fc_mu.weight"], 1e-4)
    assert_summary_close("G fc.weight grad", sdG["fc.weight"].grad, z["grad_G_fc.weight"], 1e-4)
    assert_summary_close("G fc.bias grad", sdG["fc.bias"].grad, z["grad_G_fc.bias"], 1e-4)
    for i in range(1, 7):
        for uv in ("u", "v"):
            np.testing.assert_allclose(sdE["layer%d.0.weight_%s" % (i, uv)].numpy(), z["post_layer%d.weight_%s" % (i, uv)],
                                       rtol=0, atol=1e-6)


def test_kld_is_a_sum_over_batch_and_z():
    mu, logvar = torch.randn(3, 256, dtype=torch.float64), torch.randn(3, 256, dtype=torch.float64)
    full = ov.kld(mu, logvar)
    assert torch.allclose(full, sum(ov.kld(mu[i:i + 1], logvar[i:i + 1]) for i in range(3)))
    assert torch.allclose(full, 0.5 * (mu ** 2).sum() + 0.5 * torch.expm1(logvar).sub(logvar).sum())
