"""CPU glue of the DoG orientation loss (dry run, tests/dryrun.py): L1OLoss with an orient_filter other than 'gabor' runs the
response pass (mg_conv_thin with the arg-max fields), mg_loss_reduce op 12, mg_loss_reduce_bwd op 12 and mg_orient_loss_bwd;
'gabor' keeps the Gabor entry points; the stand-alone model trains with --orient_filter dog under the same loss keys."""
import random

import pytest
import torch

from dryrun import dry_run


def _loss_inputs(n=2, size=16):
    img = torch.rand(n, 3, size, size) * 2 - 1
    sem = torch.zeros(n, 2, size, size)
    sem[:, 1, 4:12, 4:12] = 1
    sem[:, 0] = 1 - sem[:, 1]
    return img, torch.rand(n, 1, size, size) * 255, sem


@pytest.mark.parametrize("use_ig", [False, True])
def test_dog_loss_runs_through_the_dog_entry_points(use_ig):
    from michigan_b200.networks.loss import L1OLoss
    from michigan_b200.options import make_opt
    img, orient, sem = _loss_inputs()
    label = torch.rand(2, 2, 16, 16) * 2 - 1 if use_ig else orient
    with dry_run() as dr:
        crit = L1OLoss(make_opt(orient_filter="dog", use_ig=use_ig))
        x = img.clone().requires_grad_()
        lo, lc = crit(x, label, sem)
        assert lo.shape == () and lc.shape == ()
        (lo + lc).backward()
        assert dr.lib.calls == ["mg_conv_thin", "mg_loss_reduce", "mg_loss_reduce_bwd", "mg_orient_loss_bwd"]
        assert x.grad is not None and x.grad.shape == x.shape


@pytest.mark.parametrize("flt", ["gabor", "gabor_x"])
def test_gabor_keeps_its_entry_points(flt):
    from michigan_b200.networks.loss import L1OLoss
    from michigan_b200.options import make_opt
    img, orient, sem = _loss_inputs()
    with dry_run() as dr:
        x = img.clone().requires_grad_()
        lo, lc = L1OLoss(make_opt(orient_filter=flt))(x, orient, sem)
        (lo + lc).backward()
        assert dr.lib.calls == ["mg_orient_loss_fwd", "mg_orient_loss_bwd"]


def test_stand_alone_train_iteration_with_the_dog_filter():
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel, train_iteration
    from michigan_b200.synth import synthetic_batch
    with dry_run() as dr:
        opt = make_opt(is_train=True, ngf=64, ndf=64, crop_size=64, batchSize=2, no_orient_loss=False, no_confidence_loss=False,
                       orient_filter="dog")
        model = Pix2PixModel(opt).train()
        optG, optD = model.create_optimizers(opt)
        random.seed(0)
        g, d, img = train_iteration(model, optG, optD, dict(synthetic_batch(2, 64, 1)))
        assert list(g) == ["GAN", "GAN_Feat", "ORIENT", "CONFIDENCE"]
        assert "mg_orient_loss_fwd" not in dr.lib.calls and dr.lib.calls.count("mg_orient_loss_bwd") == 1
