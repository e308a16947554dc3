"""Host-code tests of the VGG perceptual and Lab colour losses on the CPU-only build box: the stand-alone trainer iteration with
the README's loss set on the no-op library (tests/dryrun.py), the weight sources of VGG19 and its refusals, and install()'s
rebinding of both loss classes in an unmodified reference checkout.  Numerics are tests/test_gpu_vgg_lab.py's job."""
import os
import random
import sys

import pytest
import torch

from dryrun import dry_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import ref_shims  # noqa: E402


@pytest.fixture
def vgg_hub(tmp_path):
    """A torch hub directory holding seeded stand-in VGG19 weights under torchvision's file name."""
    from michigan_b200.networks.architecture import VGG19_WEIGHTS_FILE
    from michigan_b200.synth import vgg19_state_dict
    old = torch.hub.get_dir()
    os.makedirs(tmp_path / "checkpoints")
    torch.save(vgg19_state_dict(0), tmp_path / "checkpoints" / VGG19_WEIGHTS_FILE)
    torch.hub.set_dir(str(tmp_path))
    yield tmp_path
    torch.hub.set_dir(old)


def test_vgg19_weights_layout_and_sources(vgg_hub, tmp_path_factory):
    from michigan_b200.networks import VGG19
    from michigan_b200.networks.architecture import VGGWeightsMissing
    from michigan_b200.synth import vgg19_state_dict
    sd = vgg19_state_dict(0)
    explicit = VGG19(state_dict=sd)
    cached = VGG19()
    keys = list(explicit.state_dict())
    assert keys[:2] == ["slice1.0.weight", "slice1.0.bias"] and keys[-2:] == ["slice5.28.weight", "slice5.28.bias"]
    assert len(keys) == 26
    for k, v in explicit.state_dict().items():
        assert torch.equal(v, cached.state_dict()[k])
    assert torch.equal(getattr(explicit.slice4, "19").weight, sd["features.19.weight"])
    assert explicit.conv(19) is getattr(explicit.slice4, "19")
    assert not any(p.requires_grad for p in explicit.parameters())
    with pytest.raises(NotImplementedError):
        VGG19(requires_grad=True, state_dict=sd)
    empty = tmp_path_factory.mktemp("empty_hub")
    torch.hub.set_dir(str(empty))
    with pytest.raises(VGGWeightsMissing, match="vgg19-dcbb9e9d.pth") as e:
        VGG19()
    assert isinstance(e.value, FileNotFoundError)


def test_loss_options_outside_the_kernels_are_refused():
    from michigan_b200.networks.loss import LabColorLoss, VGGLoss
    from michigan_b200.options import make_opt
    from michigan_b200.synth import vgg19_state_dict
    with pytest.raises(NotImplementedError):
        VGGLoss(make_opt(remove_background=True), state_dict=vgg19_state_dict(0))
    with pytest.raises(NotImplementedError):
        LabColorLoss(make_opt(balance_Lab=True))


@pytest.mark.parametrize("mode", ["mixed16", "tf32"])
def test_readme_loss_set_train_iteration_glue(vgg_hub, mode):
    """train_iteration with the README's loss set (hinge GAN, GAN_Feat, VGG, lab, ORIENT): every loss key in the reference's
    order, a gradient for every generator parameter, and the VGG19 weights never in an optimiser."""
    from michigan_b200 import precision
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel, train_iteration
    from michigan_b200.synth import synthetic_batch
    old = precision.mode()
    precision.set_mode(mode)
    try:
        with dry_run() as dr:
            opt = make_opt(is_train=True, ngf=64, ndf=64, crop_size=64, batchSize=2, no_vgg_loss=False, no_lab_loss=False,
                           no_orient_loss=False)
            model = Pix2PixModel(opt).train()
            optG, optD = model.create_optimizers(opt)
            vgg_params = {id(p) for p in model.criterionVGG.parameters()}
            assert vgg_params and not vgg_params & {id(p) for g in optG.param_groups + optD.param_groups for p in g["params"]}
            data = synthetic_batch(2, 64, 1)
            random.seed(0)
            g, d, img = train_iteration(model, optG, optD, dict(data))
            assert list(g) == ["GAN", "GAN_Feat", "VGG", "lab", "ORIENT"] and tuple(img.shape) == (2, 3, 64, 64)
            for name in ("mg_maxpool2_nhwc", "mg_maxpool2_relu_bwd", "mg_relu_bwd16", "mg_lab_loss_fwd", "mg_lab_loss_bwd",
                         "mg_loss_reduce_bwd", "mg_thin_dgrad3"):
                assert name in dr.lib.calls, name
            for name, p in model.netG.named_parameters():
                assert name.startswith("backgroud_enc.layer4") or p.grad is not None, name
    finally:
        precision.set_mode(old)


@pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")
def test_install_rebinds_vgg_and_lab_losses():
    import michigan_b200.networks.loss as mine
    from michigan_b200.install import install
    install(ref_shims.REF)
    import models.networks as pkg
    import models.networks.loss as los
    assert pkg.VGGLoss is mine.VGGLoss and los.VGGLoss is mine.VGGLoss
    assert pkg.LabColorLoss is mine.LabColorLoss and los.LabColorLoss is mine.LabColorLoss
    assert los.L1OLoss is not mine.L1OLoss       # the orientation loss keeps the reference's class under install()
