"""Host-code tests of --remove_background with the reference's default objective on the CPU-only build box, against the no-op
library (tests/dryrun.py): the stand-alone train_iteration and, under install(), the reference's own Pix2PixTrainer run the
VGG, content and style losses hair-masked on the fused loss reductions (mg_loss_reduce ops 8, 9 and 10 and the masked mode of
mg_style_loss_fwd).  Numerics are tests/test_gpu_remove_background.py's job."""
import os
import random
import sys

import pytest

from dryrun import dry_run
from test_style_content_glue import DEFAULT_KEYS, DEFAULT_LOSSES, vgg_hub  # noqa: F401  (vgg_hub is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import ref_shims  # noqa: E402


class _OpLog:
    """Records the op of every loss-reduction term the losses put in a descriptor table, forward and backward."""

    def __init__(self, monkeypatch):
        import michigan_b200.networks.loss as los
        self.ops = []
        real = los._device_table

        def table(terms, device):
            self.ops.extend(int(t.op) for t in terms)
            return real(terms, device)
        monkeypatch.setattr(los, "_device_table", table)


def _check_grads(net):
    for name, p in net.named_parameters():
        assert name.startswith("backgroud_enc.layer4") or p.grad is not None, name


@pytest.mark.parametrize("mode", ["mixed16", "tf32"])
def test_default_loss_set_with_remove_background_train_iteration_glue(vgg_hub, monkeypatch, mode):
    """train_iteration with the reference's default loss set and --remove_background: the reference's ten keys in its order, a
    gradient for every generator parameter, the masked ops 8 (VGG L1), 9 (content) and 10 (style moments) forward and backward,
    one masked style launch and no unmasked style gradient."""
    from michigan_b200 import precision
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel, train_iteration
    from michigan_b200.synth import synthetic_batch
    log = _OpLog(monkeypatch)
    old = precision.mode()
    precision.set_mode(mode)
    try:
        with dry_run() as dr:
            opt = make_opt(is_train=True, ngf=64, ndf=64, crop_size=64, batchSize=2, remove_background=True, mask_vgg_losses=True,
                           **DEFAULT_LOSSES)
            model = Pix2PixModel(opt).train()
            optG, optD = model.create_optimizers(opt)
            data = synthetic_batch(2, 64, 1)
            random.seed(0)
            g, d, img = train_iteration(model, optG, optD, dict(data))
            assert list(g) == DEFAULT_KEYS and tuple(img.shape) == (2, 3, 64, 64)
            assert set(d) == {"D_Fake", "D_real"}
            _check_grads(model.netG)
            assert dr.lib.calls.count("mg_style_loss_fwd") == 1
            assert "mg_style_tap_grad" not in dr.lib.calls
    finally:
        precision.set_mode(old)
    # forward: one table with 5 L1 terms, 1 content term, 10 moment terms; backward: 5 x op 8, 5 x op 10, 1 x op 9
    for op, count in ((8, 5 + 5), (9, 1 + 1), (10, 10 + 5)):
        assert sum(1 for o in log.ops if o == op) >= count, (op, log.ops)


def test_masked_terms_are_an_explicit_opt_in(vgg_hub):
    """--remove_background alone is still refused by the VGG losses; with mask_vgg_losses they take the masked terms, and
    mask_vgg_losses without --remove_background changes nothing."""
    from michigan_b200.networks import StyleContentLoss, VGGLoss
    from michigan_b200.options import make_opt
    for cls in (VGGLoss, StyleContentLoss):
        with pytest.raises(NotImplementedError, match="remove_background"):
            cls(make_opt(remove_background=True))
        assert cls(make_opt(remove_background=True, mask_vgg_losses=True)).masked
        assert not cls(make_opt(mask_vgg_losses=True)).masked


def test_masked_losses_accept_crops_below_32(vgg_hub):
    """The masked style variance is biased (no division by M - 1), so a 1x1 relu5_1 map is not refused."""
    import torch
    from michigan_b200.networks import StyleContentLoss
    from michigan_b200.options import make_opt
    crit = StyleContentLoss(make_opt(remove_background=True, mask_vgg_losses=True))
    lab = torch.ones(1, 1, 16, 16)
    with dry_run():
        crit(torch.rand(1, 3, 16, 16).requires_grad_(), torch.rand(1, 3, 16, 16), torch.rand(1, 3, 16, 16), lab, lab)
        with pytest.raises(ValueError, match="hair label"):
            crit(torch.rand(1, 3, 16, 16).requires_grad_(), torch.rand(1, 3, 16, 16), torch.rand(1, 3, 16, 16))


@pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")
def test_reference_training_iteration_with_remove_background_runs_on_the_masked_losses(vgg_hub, tmp_path, monkeypatch):
    """The reference's unchanged Pix2PixTrainer under install() with its default objective and --remove_background."""
    import michigan_b200.networks.loss as mine
    from michigan_b200.install import install
    from michigan_b200.synth import synthetic_batch
    log = _OpLog(monkeypatch)
    # the VGG, content and style losses on (the shim's flags turn them off); the Gabor orientation loss stays off, as the
    # reference's own class builds its filters with .cuda()
    monkeypatch.setattr(ref_shims, "TRAIN_FLAGS", [f for f in ref_shims.TRAIN_FLAGS
                                                   if f not in ("--no_vgg_loss", "--no_style_loss", "--no_content_loss")])
    with dry_run() as dr:
        install(ref_shims.REF)
        opt = ref_shims.ref_options(True, ["--ngf", "64", "--ndf", "64", "--crop_size", "64", "--load_size", "64", "--batchSize", "2",
                                           "--checkpoints_dir", str(tmp_path), "--name", "rb", "--remove_background"])
        assert not (opt.no_vgg_loss or opt.no_style_loss or opt.no_content_loss)
        from trainers.pix2pix_trainer import Pix2PixTrainer
        trainer = Pix2PixTrainer(opt)
        model = trainer.pix2pix_model_on_one_gpu
        assert type(model.criterionVGG) is mine.VGGLoss and opt.mask_vgg_losses and model.criterionVGG.masked
        random.seed(0)
        data = synthetic_batch(2, 64, 1)
        trainer.run_generator_one_step(data)
        keys = list(trainer.g_losses)
        assert [k for k in DEFAULT_KEYS if k in keys] == keys and {"GAN", "GAN_Feat", "VGG", "content", "style"} <= set(keys), keys
        _check_grads(model.netG)
        trainer.run_discriminator_one_step(data)
        assert set(trainer.d_losses) == {"D_Fake", "D_real"}
        assert "mg_style_loss_fwd" in dr.lib.calls
    for op in (8, 9, 10):
        assert op in log.ops, (op, log.ops)
