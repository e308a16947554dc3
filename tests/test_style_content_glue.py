"""Host-code tests of the style / content / background / rgb losses on the CPU-only build box: the stand-alone trainer iteration with
the reference's default loss set on the no-op library (tests/dryrun.py), the options it still refuses, the ABI record of the style
table, and install()'s rebinding of the loss classes in an unmodified reference checkout.  Numerics are
tests/test_gpu_style_content.py's job."""
import ctypes as C
import os
import random
import sys

import pytest
import torch

from dryrun import dry_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import ref_shims  # noqa: E402

DEFAULT_LOSSES = dict(no_vgg_loss=False, no_style_loss=False, no_content_loss=False, no_background_loss=False, no_rgb_loss=False,
                      no_lab_loss=False, no_orient_loss=False, no_confidence_loss=False)
DEFAULT_KEYS = ["GAN", "GAN_Feat", "VGG", "content", "style", "background", "rgb", "lab", "ORIENT", "CONFIDENCE"]


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


def test_style_tap_record_matches_the_library():
    from michigan_b200 import _lib, ops
    assert _lib.load().mg_style_tap_bytes() == C.sizeof(ops.StyleTap)


@pytest.mark.parametrize("mode", ["mixed16", "tf32"])
def test_default_loss_set_train_iteration_glue(vgg_hub, mode):
    """train_iteration with the reference's default loss set: the ten loss keys in the reference's order, a gradient for every
    generator parameter, the new kernels called, one VGG19 shared by the perceptual and style / content losses and in no
    optimiser."""
    from michigan_b200 import precision
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel, train_iteration
    from michigan_b200.synth import synthetic_batch
    old = precision.mode()
    precision.set_mode(mode)
    try:
        with dry_run() as dr:
            opt = make_opt(is_train=True, ngf=64, ndf=64, crop_size=64, batchSize=2, **DEFAULT_LOSSES)
            model = Pix2PixModel(opt).train()
            assert model.criterionStyleContent.vgg is model.criterionVGG.vgg
            optG, optD = model.create_optimizers(opt)
            vgg_params = {id(p) for p in model.criterionStyleContent.parameters()}
            assert vgg_params and not vgg_params & {id(p) for g in optG.param_groups + optD.param_groups for p in g["params"]}
            data = synthetic_batch(2, 64, 1)
            random.seed(0)
            g, d, img = train_iteration(model, optG, optD, dict(data))
            assert list(g) == DEFAULT_KEYS and tuple(img.shape) == (2, 3, 64, 64)
            for name in ("mg_in_stats", "mg_style_loss_fwd", "mg_style_tap_grad", "mg_pixel_l1_fwd", "mg_pixel_l1_bwd", "mg_loss_reduce",
                         "mg_loss_reduce_bwd", "mg_maxpool2_relu_bwd", "mg_thin_dgrad3"):
                assert name in dr.lib.calls, name
            assert dr.lib.calls.count("mg_style_loss_fwd") == 1 and dr.lib.calls.count("mg_style_tap_grad") == 5
            for name, p in model.netG.named_parameters():
                assert name.startswith("backgroud_enc.layer4") or p.grad is not None, name
    finally:
        precision.set_mode(old)


def test_style_and_content_are_computed_when_ref_is_not_tag(vgg_hub):
    """content and style do not depend on ref == tag (pix2pix_model.py:309-319); VGG, background, rgb and lab do."""
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel
    from michigan_b200.synth import synthetic_batch
    with dry_run():
        opt = make_opt(is_train=True, ngf=64, ndf=64, crop_size=64, batchSize=2, **DEFAULT_LOSSES)
        model = Pix2PixModel(opt).train()
        data = synthetic_batch(2, 64, 1)
        data["label_ref"] = 1 - data["label_tag"]
        random.seed(0)
        g, _ = model(dict(data), mode="generator")
    assert list(g) == ["GAN", "content", "style", "ORIENT", "CONFIDENCE"]


def test_style_image_equal_to_tag_runs_vgg_on_2n(vgg_hub):
    """The style image equal to the tag (paired training) is not run through VGG19 a second time."""
    from michigan_b200.networks import StyleContentLoss
    from michigan_b200.options import make_opt
    crit = StyleContentLoss(make_opt())
    fake, tag = torch.rand(2, 3, 64, 64), torch.rand(2, 3, 64, 64)
    seen = []
    orig = crit.vgg.run

    def run(x8, n_save=0):
        seen.append(x8.shape[0])
        return orig(x8, n_save)
    crit.vgg.run = run
    with dry_run():
        for style in (tag, tag.clone(), torch.rand(2, 3, 64, 64)):
            crit(fake.clone().requires_grad_(), style, tag)
    assert seen == [4, 4, 6]


def test_options_outside_the_kernels_are_refused(vgg_hub):
    from michigan_b200.networks import StyleContentLoss
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel
    with pytest.raises(NotImplementedError, match="remove_background"):
        StyleContentLoss(make_opt(remove_background=True))
    crit = StyleContentLoss(make_opt())
    for size in (16, 24, 31):
        with dry_run(), pytest.raises(NotImplementedError, match="crop_size >= 32"):
            crit(torch.rand(1, 3, size, size).requires_grad_(), torch.rand(1, 3, size, size), torch.rand(1, 3, size, size))
    with dry_run():
        crit(torch.rand(1, 3, 32, 32).requires_grad_(), torch.rand(1, 3, 32, 32), torch.rand(1, 3, 32, 32))
        for flag in ("remove_background", "balance_Lab", "unpairTrain", "use_vae", "use_blender"):
            with pytest.raises(NotImplementedError):
                Pix2PixModel(make_opt(is_train=True, ngf=64, ndf=64, crop_size=64, batchSize=2, **dict(DEFAULT_LOSSES, **{flag: True})))


@pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")
def test_install_rebinds_style_content_and_background_losses():
    import michigan_b200.networks.loss as mine
    from michigan_b200.install import install
    install(ref_shims.REF)
    import models.networks as pkg
    import models.networks.loss as los
    assert los.StyleContentLoss is mine.StyleContentLoss
    assert los.RGBBackgroundL1Loss is mine.RGBBackgroundL1Loss and pkg.RGBBackgroundL1Loss is mine.RGBBackgroundL1Loss
    # the package name is wrapped so that --no_style_loss --no_content_loss together build no VGG19 (michigan_b200.compat)
    assert pkg.StyleContentLoss is mine.StyleContentLoss or getattr(pkg.StyleContentLoss, "_mg_lazy", False)
    assert not isinstance(torch.nn.L1Loss(), mine.RGBL1Loss)
