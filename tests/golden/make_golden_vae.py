"""Golden fixture of the reference's --use_vae generator step, generated on the CPU from the LIVE reference:

    python tests/golden/make_golden_vae.py [out.npz]

The unmodified Pix2PixTrainer / Pix2PixModel (--use_vae, crop 256, ngf 32, batch 2) runs one generator step on weights filled
by michigan_b200.synth.fill_state_dict and inputs from synthetic_batch.  Besides the training shims of ref_shims (no
arithmetic touched) there is one more: the reparameterisation's eps (pix2pix_model.py:604-607, torch.randn_like) is a fixed
tensor stored in the fixture, so the step is reproducible without the reference's RNG stream.

The oracle (tests/oracle_vae.py) must agree at fp32 noise level; then mu, logvar, the generated image, the losses (KLD first),
the gradients of netE.layer1.0.weight_orig, netE.fc_mu.weight, netG.fc.weight / bias, and netE's post-forward spectral-norm
u / v are stored (large tensors as tests/helpers.summary) in tests/golden/golden_vae.npz.
"""
import contextlib
import json
import os
import random
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ref_shims  # noqa: E402

CFG = dict(size=256, ngf=32, ndf=32, batch=2, seed_G=11, seed_D=12, seed_E=13, data_seed=5, eps_seed=7, py_seed=3)
BIG = ("fake", "grad_fc_mu.weight", "grad_G_fc.weight", "grad_G_fc.bias")


@contextlib.contextmanager
def fixed_eps(eps):
    """torch.randn_like(std) -> eps while the model runs (the only randn_like call of the step is reparameterize's)."""
    orig = torch.randn_like

    def randn_like(t, *a, **k):
        assert tuple(t.shape) == tuple(eps.shape)
        return eps.clone()

    torch.randn_like = randn_like
    try:
        yield
    finally:
        torch.randn_like = orig


def rng_k(size, py_seed):
    """The dilation size BackgroundEncode2 draws with Python's random (encoder.py:286-300)."""
    random.seed(py_seed)
    th = int(size * 0.05)
    th = th if th % 2 == 1 else th + 1
    return random.choice([max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4])


def main():
    out_path = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "golden_vae.npz"))
    import michigan_oracle as orc
    import oracle_vae as ov
    from helpers import summary
    from michigan_b200.synth import fill_state_dict, synthetic_batch
    warnings.filterwarnings("ignore")
    torch.set_num_threads(8)
    torch.manual_seed(0)
    ref_shims.patch_training()
    c = CFG
    size = c["size"]
    extra = ["--use_vae", "--ngf", str(c["ngf"]), "--ndf", str(c["ndf"]), "--crop_size", str(size), "--load_size", str(size),
             "--batchSize", str(c["batch"])]
    opt = ref_shims.ref_options(True, extra)
    from trainers.pix2pix_trainer import Pix2PixTrainer
    trainer = Pix2PixTrainer(opt)
    model = trainer.pix2pix_model
    netG, netD, netE = model.netG, model.netD, model.netE
    fill_state_dict(netG.state_dict(), c["seed_G"])
    fill_state_dict(netD.state_dict(), c["seed_D"])
    fill_state_dict(netE.state_dict(), c["seed_E"])
    sdG0 = {k: v.clone() for k, v in netG.state_dict().items()}
    sdD0 = {k: v.clone() for k, v in netD.state_dict().items()}
    sdE0 = {k: v.clone() for k, v in netE.state_dict().items()}
    eps = torch.from_numpy(np.random.RandomState(c["eps_seed"]).standard_normal((c["batch"], 256)).astype(np.float32))
    data = synthetic_batch(c["batch"], size, c["data_seed"])
    input_ref, input_tag, image_ref, image_tag, orient_mask, _, _, noise = model.preprocess_input(dict(data))
    pre = dict(input_ref=input_ref, input_tag=input_tag, image_ref=image_ref, image_tag=image_tag, orient_mask=orient_mask,
               noise=noise)

    seen = {}
    hook = netE.register_forward_hook(lambda m, i, o: seen.update(mu=o[0].detach().clone(), logvar=o[1].detach().clone()))
    gen_hook = netG.register_forward_hook(lambda m, i, o: seen.update(fake=o.detach().clone()))
    k = rng_k(size, c["py_seed"])
    random.seed(c["py_seed"])
    with fixed_eps(eps):
        trainer.run_generator_one_step(dict(data))
    hook.remove()
    gen_hook.remove()
    keys = list(trainer.g_losses.keys())
    assert keys[0] == "KLD", keys
    g_losses = {kk: float(v.mean()) for kk, v in trainer.g_losses.items()}
    res = {"config": np.frombuffer(json.dumps(c).encode(), dtype=np.uint8), "eps": eps.numpy(),
           "loss_keys": np.frombuffer(json.dumps(keys).encode(), dtype=np.uint8)}
    res["mu"], res["logvar"] = seen["mu"].numpy(), seen["logvar"].numpy()
    res["fake"] = seen["fake"]
    for kk, v in g_losses.items():
        res["loss_" + kk] = np.float64(v)
    res["grad_layer1.0.weight_orig"] = netE.layer1[0].weight_orig.grad.clone()
    res["grad_fc_mu.weight"] = netE.fc_mu.weight.grad.clone()
    res["grad_G_fc.weight"] = netG.fc.weight.grad.clone()
    res["grad_G_fc.bias"] = netG.fc.bias.grad.clone()
    for i in range(1, 7):
        for uv in ("u", "v"):
            res["post_layer%d.weight_%s" % (i, uv)] = getattr(netE, "layer%d" % i)[0].__getattr__("weight_" + uv).detach().numpy().copy()

    # the oracle on the same weights, inputs, eps and dilation
    oopt = orc.default_opt(ngf=c["ngf"], ndf=c["ndf"], crop_size=size, isTrain=True)
    oopt.lambda_kld = opt.lambda_kld
    sdG, sdD, sdE = [{kk: v.clone() for kk, v in sd.items()} for sd in (sdG0, sdD0, sdE0)]
    for sd, net in ((sdG, netG), (sdE, netE)):
        for n, _ in net.named_parameters():
            sd[n].requires_grad_(True)
    losses_o, fake_o, mu_o, lv_o = ov.compute_generator_loss(sdG, sdD, sdE, oopt, pre, eps, rng_k=k)
    orc.trainer_loss(losses_o).backward()
    assert list(losses_o.keys()) == keys, (list(losses_o.keys()), keys)
    for kk in keys:
        print("  G loss %-9s ref %.7f oracle %.7f" % (kk, g_losses[kk], float(losses_o[kk].mean())))
        assert abs(g_losses[kk] - float(losses_o[kk].mean())) <= 1e-5 * max(1.0, abs(g_losses[kk]))
    pairs = [("mu", mu_o), ("logvar", lv_o), ("fake", fake_o), ("grad_layer1.0.weight_orig", sdE["layer1.0.weight_orig"].grad),
             ("grad_fc_mu.weight", sdE["fc_mu.weight"].grad), ("grad_G_fc.weight", sdG["fc.weight"].grad),
             ("grad_G_fc.bias", sdG["fc.bias"].grad)]
    for name, o in pairs:
        r = torch.as_tensor(res[name])
        rel = float((o.detach() - r).abs().max() / r.abs().max())
        print("  %-26s max-abs rel %.2e" % (name, rel))
        assert rel <= 1e-4, name
    for i in range(1, 7):
        for uv in ("u", "v"):
            key = "layer%d.0.weight_%s" % (i, uv)
            assert torch.allclose(sdE[key], torch.as_tensor(res["post_" + key.replace(".0.", ".")]), atol=1e-6), key
    for name in BIG:
        res[name] = summary(torch.as_tensor(res[name]))
    res = {kk: (v.numpy() if torch.is_tensor(v) else v) for kk, v in res.items()}
    np.savez_compressed(out_path, **res)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main()
