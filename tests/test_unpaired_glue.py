"""Host-code tests of the unpaired training stage (--unpairTrain, curr_step 2) on the CPU-only build box: the reference's own
Pix2PixTrainer / Pix2PixModel under install(), run against the no-op library (tests/dryrun.py).  What is checked is the
plumbing around the second discriminator and the hair-average Lab loss: which network judges the generator, which optimiser
steps, which parameters receive gradients, the loss keys, and the checkpoint files.  Numerics are
tests/test_gpu_hair_avg_lab.py's job."""
import os
import random
import sys

import pytest
import torch

from dryrun import dry_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import ref_shims  # noqa: E402

pytestmark = pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")

SIZE = 64
UNPAIRED_KEYS = ["GAN", "hairAvgLab", "background"]


def _opt(tmp_path, *extra):
    from michigan_b200.install import install
    install(ref_shims.REF)
    return ref_shims.ref_options(True, ["--unpairTrain", "--ngf", "64", "--ndf", "64", "--crop_size", str(SIZE), "--load_size",
                                        str(SIZE), "--batchSize", "2", "--checkpoints_dir", str(tmp_path), "--name", "unpaired"]
                                 + list(extra))


def _unpaired_batch():
    """Reference hair differs from the tag's (the unpaired loader's pairs)."""
    from michigan_b200.synth import synthetic_batch
    data = synthetic_batch(2, SIZE, 1)
    data["label_ref"] = torch.zeros_like(data["label_ref"])
    data["label_ref"][:, :, 10:40, 20:50] = 1.0
    data["image_ref"] = data["image_ref"].flip(-1).contiguous()
    return data


def _params(net):
    return [p for p in net.parameters()]


def test_unpaired_stage_runs_on_the_installed_classes(tmp_path):
    import michigan_b200.networks as mine
    from michigan_b200 import checkpoint
    with dry_run() as dr:
        opt = _opt(tmp_path)
        from trainers.pix2pix_trainer import Pix2PixTrainer
        trainer = Pix2PixTrainer(opt)
        model = trainer.pix2pix_model_on_one_gpu
        netD, netD2 = model.netD, model.netD2
        assert isinstance(netD2, mine.MultiscaleDiscriminator) and netD2 is not netD
        assert isinstance(model.criterionHairAvgLab, mine.loss.HairAvgLabLoss)
        # one spectral-norm batch per network, over that network's own convs
        assert netD.spectral_batch() is not netD2.spectral_batch()
        assert {id(c) for c in netD2.spectral_batch().convs} <= {id(m) for m in netD2.modules()}
        assert {id(p) for g in trainer.optimizer_D2.param_groups for p in g["params"]} == {id(p) for p in _params(netD2)}
        assert {id(p) for g in trainer.optimizer_D.param_groups for p in g["params"]} == {id(p) for p in _params(netD)}

        # ---- generator step of the unpaired stage: netD2 judges, neither discriminator gets a gradient
        opt.curr_step = 2
        trainer.init_losses()
        random.seed(0)
        seen = []
        hooks = [n.register_forward_hook(lambda m, i, o, name=name: seen.append(name)) for name, n in (("D", netD), ("D2", netD2))]
        trainer.run_generator_one_step(_unpaired_batch())
        assert list(trainer.g_losses) == UNPAIRED_KEYS
        assert seen == ["D2"]
        assert "mg_hair_avg_lab_fwd" in dr.lib.calls and "mg_hair_avg_lab_bwd" in dr.lib.calls
        assert all(p.grad is None for p in _params(netD) + _params(netD2))
        assert all(p.requires_grad for p in _params(netD) + _params(netD2))      # un-frozen again
        for name, p in model.netG.named_parameters():
            assert name.startswith("backgroud_enc.layer4") or p.grad is not None, name

        # ---- discriminator step: only optimizer_D2's parameters are stepped
        seen.clear()
        trainer.run_discriminator_one_step(_unpaired_batch())
        for h in hooks:
            h.remove()
        assert seen == ["D2"]
        assert all(p.grad is not None for p in _params(netD2)) and all(p.grad is None for p in _params(netD))
        assert all(len(trainer.optimizer_D2.state[p]) > 0 for p in _params(netD2))
        assert not trainer.optimizer_D.state

        # ---- checkpoints: save() writes D2 through the installed writer
        with torch.no_grad():
            for p in _params(netD2):
                p.fill_(0.25)
            for p in _params(netD):
                p.fill_(-0.5)
        trainer.save("latest")
        checkpoint.wait_pending()
    for label in ("G", "D", "D2"):
        assert os.path.isfile(tmp_path / "unpaired" / ("latest_net_%s.pth" % label)), label
    sd2 = torch.load(tmp_path / "unpaired" / "latest_net_D2.pth")
    assert list(sd2) == list(netD2.state_dict())


@pytest.mark.parametrize("same_netD_model", [False, True])
def test_continue_train_loads_both_discriminators(tmp_path, same_netD_model):
    """util.load_network (util.py:221-225) reads <epoch>_net_D2.pth for BOTH discriminators under --unpairTrain unless
    --same_netD_model is given, then <epoch>_net_D.pth for both (pix2pix_model.py:190-193)."""
    from michigan_b200 import checkpoint
    with dry_run():
        opt = _opt(tmp_path)
        from models.pix2pix_model import Pix2PixModel
        model = Pix2PixModel(opt)
        with torch.no_grad():
            for p in _params(model.netD2):
                p.fill_(0.25)
            for p in _params(model.netD):
                p.fill_(-0.5)
        model.save("latest")
        checkpoint.wait_pending()
        extra = ["--continue_train"] + (["--same_netD_model"] if same_netD_model else [])
        resumed = Pix2PixModel(_opt(tmp_path, *extra))
    want = -0.5 if same_netD_model else 0.25
    for net in (resumed.netD, resumed.netD2):
        assert all(bool((p == want).all()) for p in _params(net))
    assert resumed.netD is not resumed.netD2
