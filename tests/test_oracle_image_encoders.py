"""CPU: the torch restatement of ImageEncoder / ImageEncoder2 and the generator step around them (tests/oracle_image_encoders.py)
against the fixture of the live reference's Pix2PixTrainer (tests/golden/make_golden_image_encoders.py)."""
import json

import numpy as np
import pytest
import torch

import michigan_oracle as orc
import oracle_image_encoders as oie


@pytest.mark.parametrize("case", list(oie.CASES))
def test_oracle_generator_step_matches_the_reference(case):
    z, c, sdG, sdD, data, pre, k = oie.fixture_inputs(case)
    mode, gp = oie.CASES[case]
    p = case + "/"
    opt = orc.default_opt(ngf=c["ngf"], ndf=c["ndf"], crop_size=c["size"], isTrain=True)
    for name, v in sdG.items():
        if not name.endswith(("weight_u", "weight_v", "running_mean", "running_var", "num_batches_tracked")):
            v.requires_grad_(True)
    losses, fake = oie.compute_generator_loss(sdG, sdD, opt, mode, gp, pre, rng_k=k)
    assert list(losses) == json.loads(bytes(z[p + "loss_keys"]).decode())
    for key, v in losses.items():
        assert abs(float(v.detach().mean()) - float(z[p + "loss_" + key])) <= 1e-5 * max(1.0, abs(float(z[p + "loss_" + key])))
    orc.trainer_loss(losses).backward()
    from helpers import summary
    got = summary(fake)
    assert np.abs(got - z[p + "fake"]).max() <= 1e-4 * float(z[p + "fake"][2])
    r = torch.as_tensor(z[p + "grad_fc.layer1.0.weight_orig"])
    assert float((sdG["fc.layer1.0.weight_orig"].grad - r).abs().max() / r.abs().max()) <= 1e-2
    if mode == "norm":
        r = torch.as_tensor(z[p + "grad_fc.fc.bias"])
        assert float((sdG["fc.fc.bias"].grad - r).abs().max() / r.abs().max()) <= 1e-2
    for i in range(1, 6):
        for uv in ("u", "v"):
            key = "fc.layer%d.0.weight_%s" % (i, uv)
            np.testing.assert_allclose(sdG[key].detach().numpy(), z[p + "post_" + key], rtol=0, atol=1e-6)
    if mode == "norm":   # layer6 is never run: the stored u, v are the initial ones
        for uv in ("u", "v"):
            key = "fc.layer6.0.weight_" + uv
            np.testing.assert_array_equal(sdG[key].detach().numpy(), z[p + "post_" + key])


def test_the_fixture_has_differing_masks_and_gan_feat():
    z, c, sdG, sdD, data, pre, k = oie.fixture_inputs("instance")
    assert not torch.equal(pre["input_ref"][1, 1], pre["input_tag"][1, 1])
    assert torch.equal(pre["input_ref"][0, 1], pre["input_tag"][0, 1])
    assert "GAN_Feat" in json.loads(bytes(z["instance/loss_keys"]).decode())
