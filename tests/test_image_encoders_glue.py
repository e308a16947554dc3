"""CPU (dry run): the --Image_encoder_mode instance / norm glue - refusals, state-dict layout against the reference, install(),
the <epoch>_net_G.pth checkpoint and the data-parallel GradReducer of the generator."""
import os
import sys

import pytest
import torch

from dryrun import dry_run
from michigan_b200.options import make_opt

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import ref_shims  # noqa: E402

BASE = dict(is_train=True, ngf=32, ndf=32, crop_size=256, batchSize=2)


def test_refusals():
    from michigan_b200.networks import ImageEncoder, ImageEncoder2, SPADEBGenerator
    with pytest.raises(NotImplementedError, match="partialconv, instance, norm"):
        SPADEBGenerator(make_opt(**dict(BASE, Image_encoder_mode="normal")))
    with pytest.raises(NotImplementedError, match="deterministic"):
        SPADEBGenerator(make_opt(**dict(BASE, use_encoder=False)))
    for cls in (ImageEncoder, ImageEncoder2):
        with pytest.raises(NotImplementedError, match="norm_E"):
            cls(make_opt(**dict(BASE, norm_E="spectralbatch")), 4, 4)
        with pytest.raises(NotImplementedError, match="multiple of 32"):
            cls(make_opt(**dict(BASE, ngf=48)), 4, 4)
    # a 12x12 map (384 / 32) is not a multiple of a 5x5 latent size
    E = ImageEncoder2(make_opt(**BASE), 5, 5)
    with dry_run():
        x = torch.zeros(1, 3, 384, 384)
        m = torch.zeros(1, 1, 384, 384)
        with pytest.raises(NotImplementedError, match="integer multiple"):
            E.forward_nhwc(x, m, m)


@pytest.mark.parametrize("crop", [256, 128])
@pytest.mark.parametrize("mode", ["instance", "norm"])
@pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")
def test_state_dict_keys_match_the_reference(mode, crop):
    from michigan_b200 import networks
    ref_shims.import_reference()
    gen = __import__("models.networks.generator", fromlist=["SPADEBGenerator"])
    ropt = ref_shims.ref_options(True, ["--Image_encoder_mode", mode, "--ngf", "32", "--crop_size", str(crop),
                                        "--load_size", str(crop)])
    mine = networks.SPADEBGenerator(make_opt(**dict(BASE, crop_size=crop, Image_encoder_mode=mode)))
    r = {k: tuple(v.shape) for k, v in gen.SPADEBGenerator(ropt).state_dict().items()}
    m = {k: tuple(v.shape) for k, v in mine.state_dict().items()}
    assert list(m.items()) == list(r.items())
    assert any(k.startswith("fc.layer6.") for k in m) == (mode == "norm" and crop >= 256)


@pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")
def test_install_rebinds_and_the_reference_trainer_runs():
    import michigan_b200.networks as mine
    from michigan_b200.install import install
    install(ref_shims.REF)
    import models.networks.encoder as enc
    import models.networks.generator as gen
    for m in (enc, gen):
        assert m.ImageEncoder is mine.ImageEncoder and m.ImageEncoder2 is mine.ImageEncoder2
    ref_shims.patch_training()
    from michigan_b200.synth import synthetic_batch
    for mode, cls in (("instance", mine.ImageEncoder2), ("norm", mine.ImageEncoder)):
        ropt = ref_shims.ref_options(True, ["--Image_encoder_mode", mode, "--ngf", "32", "--ndf", "32", "--crop_size", "256",
                                            "--load_size", "256", "--batchSize", "2"])
        with dry_run():
            from trainers.pix2pix_trainer import Pix2PixTrainer
            trainer = Pix2PixTrainer(ropt)
            fc = trainer.pix2pix_model.netG.fc
            assert isinstance(fc, cls)
            trainer.run_generator_one_step(synthetic_batch(2, 256, 0))
            for n, p in fc.named_parameters():
                assert (p.grad is None) == n.startswith("layer6."), n
            trainer.run_discriminator_one_step(synthetic_batch(2, 256, 0))


@pytest.mark.parametrize("mode", ["instance", "norm"])
def test_checkpoint_round_trip(tmp_path, mode):
    from michigan_b200 import checkpoint
    from michigan_b200.pix2pix_model import Pix2PixModel
    opt = make_opt(**dict(BASE, Image_encoder_mode=mode, checkpoints_dir=str(tmp_path), name="enc"))
    with dry_run():
        m = Pix2PixModel(opt)
        os.makedirs(os.path.join(str(tmp_path), "enc"), exist_ok=True)
        with torch.no_grad():
            m.netG.fc.layer5[0].weight_orig.fill_(0.25)
        m.save("2")
    checkpoint.wait_pending()
    sd = torch.load(os.path.join(str(tmp_path), "enc", "2_net_G.pth"), map_location="cpu")
    assert list(sd) == list(m.netG.state_dict()) and torch.all(sd["fc.layer5.0.weight_orig"] == 0.25)
    with dry_run():
        m2 = Pix2PixModel(make_opt(**dict(BASE, Image_encoder_mode=mode, checkpoints_dir=str(tmp_path), name="enc",
                                          continue_train=True, which_epoch="2")))
        assert torch.all(m2.netG.fc.layer5[0].weight_orig == 0.25)


def _ddp_worker(rank, world, port, q):
    import torch.distributed as dist
    here = os.path.dirname(os.path.abspath(__file__))
    for p in (os.path.dirname(here), here):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from dryrun import dry_run
    from michigan_b200.networks import SPADEBGenerator
    from michigan_b200.networks.sync_batchnorm import DataParallelWithCallback
    from michigan_b200.synth import synthetic_batch
    torch.manual_seed(100 + rank)                # different weights per rank before the broadcast
    holder = torch.nn.Module()
    holder.netG = SPADEBGenerator(make_opt(**dict(BASE, Image_encoder_mode="norm")))
    wrapped = DataParallelWithCallback(holder, device_ids=[rank])
    G = holder.netG
    flat = torch.cat([t.detach().reshape(-1) for t in list(G.fc.parameters()) + list(G.fc.buffers())])
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    res = {"broadcast": bool(torch.equal(gathered[0], gathered[1])), "one_reducer": getattr(G.fc, "_grad_reducer", None) is None
           and any(r is G._grad_reducer for r in wrapped.reducers)}
    d = synthetic_batch(2, 256, 0)
    lab = torch.cat([1 - d["label_tag"], d["label_tag"]], 1)
    with dry_run():
        out = G(lab, orient_mask=d["orient"], image_ref=d["image_ref"], input_tag=lab, noise=d["noise"], image_tag=d["image_tag"])
        out.sum().backward()
    red = G._grad_reducer
    res["views"] = all((p.grad is None) if n.startswith("layer6.") else
                       (p.grad is not None and p.grad.data_ptr() == red.views[id(p)].data_ptr())
                       for n, p in G.fc.named_parameters())
    q.put((rank, res))
    dist.destroy_process_group()


def test_generator_with_norm_encoder_under_gloo():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_ddp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = dict(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=120)
    for r in range(2):
        assert out[r] == {"broadcast": True, "one_reducer": True, "views": True}, out
