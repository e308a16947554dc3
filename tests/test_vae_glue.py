"""CPU (dry run): the --use_vae glue - refusals, state-dict layout, install(), the reference's trainer, optimizer_G, the
<epoch>_net_E.pth checkpoint, encode_only, and the data-parallel GradReducer of netE."""
import os
import sys

import pytest
import torch

from dryrun import dry_run
from michigan_b200.options import make_opt

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import ref_shims  # noqa: E402

VAE = dict(is_train=True, ngf=32, ndf=32, crop_size=256, batchSize=2, use_vae=True)


def test_refusals():
    from michigan_b200.networks import ConvEncoder
    with pytest.raises(NotImplementedError, match="crop_size >= 256"):
        ConvEncoder(make_opt(**dict(VAE, crop_size=128)))
    with pytest.raises(NotImplementedError, match="z_dim 256"):
        ConvEncoder(make_opt(**dict(VAE, z_dim=128)))
    with pytest.raises(NotImplementedError, match="norm_E"):
        ConvEncoder(make_opt(**dict(VAE, norm_E="spectralbatch")))
    with dry_run():
        from michigan_b200.pix2pix_model import Pix2PixModel
        with pytest.raises(NotImplementedError, match="crop_size >= 256"):
            Pix2PixModel(make_opt(**dict(VAE, crop_size=64)))


@pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")
def test_state_dict_keys_match_the_reference():
    from michigan_b200 import networks
    ref = ref_shims.import_reference()
    enc = __import__("models.networks.encoder", fromlist=["ConvEncoder"])
    gen = __import__("models.networks.generator", fromlist=["SPADEBGenerator"])
    ropt = ref_shims.ref_options(True, ["--use_vae", "--ngf", "32", "--crop_size", "256", "--load_size", "256"])
    mine_opt = make_opt(**VAE)
    for ref_cls, mine in ((enc.ConvEncoder, networks.ConvEncoder(mine_opt)), (gen.SPADEBGenerator, networks.SPADEBGenerator(mine_opt))):
        r = {k: tuple(v.shape) for k, v in ref_cls(ropt).state_dict().items()}
        m = {k: tuple(v.shape) for k, v in mine.state_dict().items()}
        assert m == r
        assert list(m) == list(r)
    assert ref.KLDLoss is not None


@pytest.mark.skipif(not ref_shims.available(), reason="the reference checkout is absent")
def test_install_rebinds_and_reference_trainer_puts_kld_first():
    import michigan_b200.networks as mine
    from michigan_b200.install import install
    install(ref_shims.REF)
    import models.networks as pkg
    import models.networks.encoder as enc
    import models.networks.loss as los
    assert issubclass(enc.ConvEncoder, mine.ConvEncoder)
    assert los.KLDLoss is mine.loss.KLDLoss and pkg.KLDLoss is mine.loss.KLDLoss
    ref_shims.patch_training()
    ropt = ref_shims.ref_options(True, ["--use_vae", "--ngf", "32", "--ndf", "32", "--crop_size", "256", "--load_size", "256",
                                        "--batchSize", "2"])
    from michigan_b200.synth import synthetic_batch
    with dry_run():
        from trainers.pix2pix_trainer import Pix2PixTrainer
        trainer = Pix2PixTrainer(ropt)
        model = trainer.pix2pix_model
        assert isinstance(model.netE, mine.ConvEncoder)
        trainer.run_generator_one_step(synthetic_batch(2, 256, 0))
        assert list(trainer.g_losses)[0] == "KLD"
        assert all(p.grad is not None for p in model.netE.parameters())
        trainer.run_discriminator_one_step(synthetic_batch(2, 256, 0))


def test_optimizer_steps_netE_checkpoint_and_encode_only(tmp_path):
    from michigan_b200.pix2pix_model import Pix2PixModel, train_iteration
    from michigan_b200.synth import synthetic_batch
    opt = make_opt(**dict(VAE, checkpoints_dir=str(tmp_path), name="vae"))
    with dry_run():
        m = Pix2PixModel(opt)
        og, od = m.create_optimizers(opt)
        ids = {id(p) for g in og.param_groups for p in g["params"]}
        assert all(id(p) in ids for p in m.netE.parameters())
        assert all(id(p) in ids for p in m.netG.parameters())
        w = m.netE.fc_mu.weight
        g_losses, _, _ = train_iteration(m, og, od, synthetic_batch(2, 256, 0))
        assert list(g_losses)[0] == "KLD"
        assert w.grad is not None and og.state[w]["step"] == 1
        mu, logvar = m(synthetic_batch(2, 256, 0), mode="encode_only")
        assert mu.shape == logvar.shape == (2, 256)
        os.makedirs(os.path.join(str(tmp_path), "vae"), exist_ok=True)
        with torch.no_grad():
            m.netE.fc_var.bias.fill_(0.125)
        m.save("3")
    from michigan_b200 import checkpoint
    checkpoint.wait_pending()
    path = os.path.join(str(tmp_path), "vae", "3_net_E.pth")
    assert os.path.exists(path)
    sd = torch.load(path, map_location="cpu")
    assert set(sd) == set(m.netE.state_dict()) and torch.all(sd["fc_var.bias"] == 0.125)
    with dry_run():
        m2 = Pix2PixModel(make_opt(**dict(VAE, checkpoints_dir=str(tmp_path), name="vae", continue_train=True, which_epoch="3")))
        assert torch.all(m2.netE.fc_var.bias == 0.125)


def _ddp_worker(rank, world, port, q):
    import torch.distributed as dist
    here = os.path.dirname(os.path.abspath(__file__))
    for p in (os.path.dirname(here), here):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from dryrun import dry_run
    from michigan_b200.networks import ConvEncoder
    from michigan_b200.networks.sync_batchnorm import DataParallelWithCallback
    from michigan_b200.options import make_opt
    torch.manual_seed(100 + rank)                # different weights per rank before the broadcast
    holder = torch.nn.Module()
    holder.netE = ConvEncoder(make_opt(**VAE))
    wrapped = DataParallelWithCallback(holder, device_ids=[rank])
    E = holder.netE
    flat = torch.cat([t.detach().reshape(-1) for t in list(E.parameters()) + list(E.buffers())])
    gathered = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    res = {"broadcast": bool(torch.equal(gathered[0], gathered[1])), "reducer": getattr(E, "_grad_reducer", None) is not None,
           "in_wrapper": any(r is E._grad_reducer for r in wrapped.reducers)}
    with dry_run():
        mu, logvar = E(torch.rand(2, 3, 256, 256))
        (mu.sum() + logvar.sum()).backward()
    red = E._grad_reducer
    res["views"] = all(p.grad is not None and p.grad.data_ptr() == red.views[id(p)].data_ptr() for p in E.parameters())
    q.put((rank, res))
    dist.destroy_process_group()


def test_netE_gets_a_grad_reducer_and_rank0_weights_under_gloo():
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
        assert out[r] == {"broadcast": True, "reducer": True, "in_wrapper": True, "views": True}, out
