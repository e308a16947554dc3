"""Host-code tests of --balance_Lab on the CPU-only build box: the weight table E against the reference's own lookup, the CPU
oracle against the reference's outputs (tests/golden/golden_balance_lab.npz), the opt-in and its refusals, and - against the
no-op library (tests/dryrun.py) - the stand-alone train_iteration and, under install(), the reference's own Pix2PixTrainer in
both training stages running the balanced losses.  Numerics of the kernels are tests/test_gpu_balance_lab.py's job."""
import os
import random
import sys

import numpy as np
import pytest
import torch

import oracle_balance_lab as obl
from dryrun import dry_run
from test_remove_background_glue import _OpLog

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_balance_lab.npz")
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import ref_shims  # noqa: E402


@pytest.fixture
def weight_dir(tmp_path):
    """The synthetic colour-count table of the golden fixture, saved where --weight_dir can name it."""
    path = tmp_path / "ab_count.npy"
    np.save(path, obl.count_table(obl.TABLE_SEED))
    return str(path)


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("th", obl.THRESHOLDS)
def test_weight_table_matches_the_oracle_lookup(weight_dir, th):
    """E[ka][kb] against grid_sample at every pair of bins (the oracle's restatement of cal_weight): bin 255 of either
    coordinate reads 0, every other bin its own entry of the processed table."""
    from michigan_b200.networks.loss import lab_weight_table
    E = lab_weight_table(weight_dir, th)
    assert E.shape == (256, 256) and E.dtype == torch.float32
    w = obl.weight_map(obl.count_table(obl.TABLE_SEED), th)
    k = torch.arange(256, dtype=torch.float32)
    a = k.view(1, 1, 256, 1).expand(1, 1, 256, 256) - 128 + 0.5
    b = k.view(1, 1, 1, 256).expand(1, 1, 256, 256) - 128 + 0.5
    assert torch.equal(E, obl.lookup(w, a, b)[0, 0])
    assert torch.equal(E[:255, :255], w[0, 0, :255, :255])
    assert bool((E[255] == 0).all()) and bool((E[:, 255] == 0).all())
    assert float(E.max()) == th and float(E[:255, :255].min()) >= 1.0
    assert not torch.equal(E, E.t())
    assert lab_weight_table(weight_dir, th) is E                        # read once per (path, th, device)


@pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")
@pytest.mark.parametrize("th", obl.THRESHOLDS)
def test_weight_table_matches_the_reference_cal_weight(weight_dir, th):
    """E against the reference's own HairAvgLabLoss.cal_weight (no mask, no 0 -> 1) on an image whose pixel (ka, kb) holds
    a = ka - 127.5, b = kb - 127.5: every pair of bins, bit for bit."""
    from make_golden_balance_lab import reference_losses
    from michigan_b200.networks.loss import lab_weight_table
    _, avg = reference_losses(weight_dir, th)
    k = torch.arange(256, dtype=torch.float32)
    img = torch.zeros(1, 3, 256, 256)
    img[0, 1] = k.view(256, 1) - 127.5
    img[0, 2] = k.view(1, 256) - 127.5
    assert torch.equal(lab_weight_table(weight_dir, th), avg.cal_weight(img)[0, 0])


@pytest.mark.parametrize("case", ["partial", "no_hair", "all_hair"])
@pytest.mark.parametrize("th", obl.THRESHOLDS)
def test_oracle_matches_reference_golden(case, th):
    z = np.load(GOLDEN)
    assert int(z["table_seed"]) == obl.TABLE_SEED
    fake, real, mf, mr = obl.golden_inputs()[case]
    w = obl.weight_map(obl.count_table(obl.TABLE_SEED), th)
    for cls, fn in (("lab", lambda x: obl.lab_color_loss_balanced(x, real, mf, w)),
                    ("avg", lambda x: obl.hair_avg_lab_loss_balanced(x, real, mf, mr, w))):
        key = "%s_%s_th%g" % (cls, case, th)
        x = fake.clone().requires_grad_()
        loss = fn(x)
        loss.backward()
        ref = float(z[key + "_loss"])
        assert abs(float(loss) - ref) <= 1e-6 * abs(ref), key
        assert _rel(x.grad, torch.from_numpy(z[key + "_grad"])) <= 1e-5, key


def test_balanced_losses_are_an_explicit_opt_in(weight_dir, tmp_path):
    """balance_Lab with weight_dir selects the balanced losses; balance_Lab alone is refused as before; weight_dir alone
    changes nothing; a missing file, a table of the wrong shape and a missing Lab_weight_th are handled."""
    from michigan_b200.networks.loss import LAB_WEIGHT_TH, HairAvgLabLoss, LabColorLoss
    from michigan_b200.options import make_opt
    assert not hasattr(make_opt(), "weight_dir")
    for cls in (LabColorLoss, HairAvgLabLoss):
        with pytest.raises(NotImplementedError, match="balance_Lab"):
            cls(make_opt(balance_Lab=True))
        assert cls(make_opt(weight_dir=weight_dir)).table_key is None
        assert cls(make_opt(balance_Lab=True, weight_dir=weight_dir, Lab_weight_th=2.5)).table_key == (weight_dir, 2.5)
        assert cls(make_opt(balance_Lab=True, weight_dir=weight_dir)).table_key == (weight_dir, LAB_WEIGHT_TH) == (weight_dir, 10.0)
        missing = str(tmp_path / "no_such_table.npy")
        with pytest.raises(FileNotFoundError, match="no_such_table.npy"):
            cls(make_opt(balance_Lab=True, weight_dir=missing))
        bad = str(tmp_path / "bad.npy")
        np.save(bad, np.ones((256, 255)))
        with pytest.raises(ValueError, match="256,256"):
            cls(make_opt(balance_Lab=True, weight_dir=bad))


def test_balanced_lab_color_loss_needs_the_hair_mask(weight_dir):
    from michigan_b200.networks.loss import LabColorLoss
    from michigan_b200.options import make_opt
    crit = LabColorLoss(make_opt(balance_Lab=True, weight_dir=weight_dir))
    x = torch.rand(2, 3, 8, 8)
    with dry_run():
        for mask in (None, torch.ones(2, 3, 8, 8), torch.ones(2, 1, 4, 4)):
            with pytest.raises(ValueError, match="hair mask"):
                crit(x.clone().requires_grad_(), x, mask)


def test_balanced_losses_issue_one_launch_each_way(weight_dir, monkeypatch):
    """LabColorLoss: one mg_loss_reduce of op 11 forward, one mg_loss_reduce_bwd backward, with a one-hot label view as the
    mask; HairAvgLabLoss: the unbalanced forward, one backward launch per image."""
    from michigan_b200.networks.loss import HairAvgLabLoss, LabColorLoss
    from michigan_b200.options import make_opt
    log = _OpLog(monkeypatch)
    opt = make_opt(balance_Lab=True, weight_dir=weight_dir)
    x, r = torch.rand(3, 3, 8, 8), torch.rand(3, 3, 8, 8)
    onehot = torch.zeros(3, 2, 8, 8)
    onehot[:, 1, 2:6, 2:6] = 1
    with dry_run() as dr:
        f = x.clone().requires_grad_()
        LabColorLoss(opt)(f, r, onehot[:, 1:2]).backward()
        assert dr.lib.calls == ["mg_loss_reduce", "mg_loss_reduce_bwd"] and log.ops == [11, 11]
        assert f.grad is not None and f.grad.shape == f.shape
        dr.lib.calls.clear()
        f = x.clone().requires_grad_()
        HairAvgLabLoss(opt)(f, r, onehot[:, 1:2], onehot[:, 1:2]).backward()
        assert dr.lib.calls == ["mg_hair_avg_lab_fwd"] + ["mg_hair_avg_lab_bwd"] * 3
        assert f.grad is not None and f.grad.shape == f.shape


@pytest.mark.parametrize("mode", ["mixed16", "tf32"])
def test_stand_alone_train_iteration_with_balance_lab(weight_dir, monkeypatch, mode):
    """The stand-alone model's train_iteration with the Lab loss on and --balance_Lab: the lab key, the balanced term (op 11)
    both ways and no unbalanced Lab kernel."""
    from michigan_b200 import precision
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel, train_iteration
    from michigan_b200.synth import synthetic_batch
    log = _OpLog(monkeypatch)
    old = precision.mode()
    precision.set_mode(mode)
    try:
        with dry_run() as dr:
            opt = make_opt(is_train=True, ngf=64, ndf=64, crop_size=64, batchSize=2, no_lab_loss=False, balance_Lab=True,
                           weight_dir=weight_dir)
            model = Pix2PixModel(opt).train()
            optG, optD = model.create_optimizers(opt)
            random.seed(0)
            g, d, img = train_iteration(model, optG, optD, dict(synthetic_batch(2, 64, 1)))
            assert list(g) == ["GAN", "GAN_Feat", "lab"] and tuple(img.shape) == (2, 3, 64, 64)
            assert "mg_lab_loss_fwd" not in dr.lib.calls and "mg_lab_loss_bwd" not in dr.lib.calls
            for name, p in model.netG.named_parameters():
                assert name.startswith("backgroud_enc.layer4") or p.grad is not None, name
    finally:
        precision.set_mode(old)
    assert log.ops.count(11) == 2, log.ops


@pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")
def test_reference_training_iteration_with_balance_lab(weight_dir, tmp_path, monkeypatch):
    """The reference's unchanged Pix2PixTrainer under install() with its Lab loss and --balance_Lab: the installed
    LabColorLoss reads the table named by --weight_dir and the lab term runs on op 11, not on mg_lab_loss_fwd."""
    import michigan_b200.networks.loss as mine
    from michigan_b200.install import install
    from michigan_b200.synth import synthetic_batch
    log = _OpLog(monkeypatch)
    monkeypatch.setattr(ref_shims, "TRAIN_FLAGS", [f for f in ref_shims.TRAIN_FLAGS if f != "--no_lab_loss"])
    with dry_run() as dr:
        install(ref_shims.REF)
        opt = ref_shims.ref_options(True, ["--ngf", "64", "--ndf", "64", "--crop_size", "64", "--load_size", "64", "--batchSize", "2",
                                           "--checkpoints_dir", str(tmp_path), "--name", "bl", "--balance_Lab", "--weight_dir",
                                           weight_dir, "--Lab_weight_th", "2.5"])
        from trainers.pix2pix_trainer import Pix2PixTrainer
        trainer = Pix2PixTrainer(opt)
        model = trainer.pix2pix_model_on_one_gpu
        assert type(model.criterionLabL1) is mine.LabColorLoss and model.criterionLabL1.table_key == (weight_dir, 2.5)
        random.seed(0)
        trainer.run_generator_one_step(synthetic_batch(2, 64, 1))
        assert "lab" in trainer.g_losses
        assert "mg_loss_reduce" in dr.lib.calls and "mg_lab_loss_fwd" not in dr.lib.calls
    assert log.ops.count(11) == 2, log.ops


@pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")
def test_reference_unpaired_stage_with_balance_lab(weight_dir, tmp_path, monkeypatch):
    """--unpairTrain --balance_Lab: the unpaired generator step's hairAvgLab is the balanced HairAvgLabLoss, one backward
    launch per image."""
    import michigan_b200.networks.loss as mine
    from test_unpaired_glue import UNPAIRED_KEYS, _opt, _unpaired_batch
    with dry_run() as dr:
        opt = _opt(tmp_path, "--balance_Lab", "--weight_dir", weight_dir)
        from trainers.pix2pix_trainer import Pix2PixTrainer
        trainer = Pix2PixTrainer(opt)
        model = trainer.pix2pix_model_on_one_gpu
        assert type(model.criterionHairAvgLab) is mine.HairAvgLabLoss
        assert model.criterionHairAvgLab.table_key == (weight_dir, 10.0)
        opt.curr_step = 2
        trainer.init_losses()
        random.seed(0)
        trainer.run_generator_one_step(_unpaired_batch())
        assert list(trainer.g_losses) == UNPAIRED_KEYS
        assert dr.lib.calls.count("mg_hair_avg_lab_fwd") == 1 and dr.lib.calls.count("mg_hair_avg_lab_bwd") == 2
