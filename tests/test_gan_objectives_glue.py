"""Host-code tests of the adversarial losses under install() on the CPU-only build box: the reference's own Pix2PixTrainer /
Pix2PixModel run one training iteration (generator step, then discriminator step) for every --gan_mode and for
--remove_background, against the no-op library (tests/dryrun.py), and must reach the fused loss reductions.  Numerics are
tests/test_gpu_gan_objectives.py's job."""
import os
import random
import sys

import pytest

from dryrun import dry_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import ref_shims  # noqa: E402

pytestmark = pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")

SIZE = 64


def test_install_rebinds_gan_losses():
    import michigan_b200.networks.loss as mine
    from michigan_b200.install import install
    install(ref_shims.REF)
    import models.networks as pkg
    import models.networks.loss as los
    for name in ("GANLoss", "GANFeatLoss"):
        assert getattr(pkg, name) is getattr(mine, name), name
        assert getattr(los, name) is getattr(mine, name), name


@pytest.mark.parametrize("flags", [["--gan_mode", "ls"], ["--gan_mode", "original"], ["--gan_mode", "w"], ["--gan_mode", "hinge"],
                                   ["--remove_background", "--no_vgg_loss", "--no_style_loss", "--no_content_loss"]],
                         ids=["ls", "original", "w", "hinge", "remove_background"])
def test_reference_training_iteration_runs_on_the_fused_losses(tmp_path, flags):
    import michigan_b200.networks.loss as mine
    from michigan_b200.install import install
    from michigan_b200.synth import synthetic_batch
    with dry_run() as dr:
        install(ref_shims.REF)
        opt = ref_shims.ref_options(True, ["--ngf", "64", "--ndf", "64", "--crop_size", str(SIZE), "--load_size", str(SIZE),
                                           "--batchSize", "2", "--checkpoints_dir", str(tmp_path), "--name", "gan"] + flags)
        from trainers.pix2pix_trainer import Pix2PixTrainer
        trainer = Pix2PixTrainer(opt)
        model = trainer.pix2pix_model_on_one_gpu
        assert type(model.criterionGAN) is mine.GANLoss and type(model.criterionGANFeat) is mine.GANFeatLoss
        assert model.criterionGAN.gan_mode == opt.gan_mode
        random.seed(0)
        data = synthetic_batch(2, SIZE, 1)
        trainer.run_generator_one_step(data)
        assert "GAN" in trainer.g_losses and "GAN_Feat" in trainer.g_losses
        trainer.run_discriminator_one_step(data)
        assert set(trainer.d_losses) == {"D_Fake", "D_real"}
        assert "mg_loss_reduce" in dr.lib.calls and "mg_loss_reduce_bwd" in dr.lib.calls
        assert ("mg_edge_weight" in dr.lib.calls) == (opt.gan_mode == "hinge" and not opt.remove_background and opt.wide_edge > 1)
