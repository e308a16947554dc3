"""Golden fixture of the reference's generator step with the pooled appearance encoders, generated on the CPU from the LIVE
reference:

    python tests/golden/make_golden_image_encoders.py [out.npz]

For each case of oracle_image_encoders.CASES (--Image_encoder_mode instance, instance --ref_global_pool, norm) the unmodified
Pix2PixTrainer / Pix2PixModel (crop 256, ngf 32, batch 2) runs one generator step on weights filled by
michigan_b200.synth.fill_state_dict and inputs from synthetic_batch, with image 1's reference hair shifted
(oracle_image_encoders.shifted_ref) so that its reference and target masks differ.  Only the training shims of ref_shims
are applied (no arithmetic touched).

The oracle (tests/oracle_image_encoders.py) must agree at fp32 noise level; then, under "<case>/", the generated image, the
losses, the gradients of netG.fc.layer1.0.weight_orig, fc.layer5.0.weight_orig (and fc.fc.weight / bias for norm), and the
encoder's post-forward spectral-norm u / v are stored (large tensors as tests/helpers.summary) in
tests/golden/golden_image_encoders.npz.  layer6 of norm (in the state dict, never run) must keep its u / v.
"""
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

CFG = dict(size=256, ngf=32, ndf=32, batch=2, seed_G=31, seed_D=32, data_seed=6, py_seed=4, shift=40)
BIG = ("fake", "grad_fc.layer5.0.weight_orig", "grad_fc.fc.weight")


def rng_k(size, py_seed):
    """The dilation size BackgroundEncode2 draws with Python's random (encoder.py:286-300)."""
    random.seed(py_seed)
    th = int(size * 0.05)
    th = th if th % 2 == 1 else th + 1
    return random.choice([max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4])


def run_case(case, res):
    import michigan_oracle as orc
    import oracle_image_encoders as oie
    from michigan_b200.synth import fill_state_dict, synthetic_batch
    c = CFG
    size = c["size"]
    mode, gp = oie.CASES[case]
    extra = ["--Image_encoder_mode", mode, "--ngf", str(c["ngf"]), "--ndf", str(c["ndf"]), "--crop_size", str(size),
             "--load_size", str(size), "--batchSize", str(c["batch"])] + (["--ref_global_pool"] if gp else [])
    opt = ref_shims.ref_options(True, extra)
    from trainers.pix2pix_trainer import Pix2PixTrainer
    trainer = Pix2PixTrainer(opt)
    model = trainer.pix2pix_model
    netG, netD = model.netG, model.netD
    fill_state_dict(netG.state_dict(), c["seed_G"])
    fill_state_dict(netD.state_dict(), c["seed_D"])
    sdG0 = {k: v.clone() for k, v in netG.state_dict().items()}
    sdD0 = {k: v.clone() for k, v in netD.state_dict().items()}
    data = oie.shifted_ref(synthetic_batch(c["batch"], size, c["data_seed"]), c["shift"])
    input_ref, input_tag, image_ref, image_tag, orient_mask, _, _, noise = model.preprocess_input(dict(data))
    assert float(torch.sum(input_tag[:, 1] - input_ref[:, 1])) == 0 and not torch.equal(input_tag[1, 1], input_ref[1, 1])
    pre = dict(input_ref=input_ref, input_tag=input_tag, image_ref=image_ref, image_tag=image_tag, orient_mask=orient_mask,
               noise=noise)
    seen = {}
    hook = netG.register_forward_hook(lambda m, i, o: seen.update(fake=o.detach().clone()))
    k = rng_k(size, c["py_seed"])
    random.seed(c["py_seed"])
    trainer.run_generator_one_step(dict(data))
    hook.remove()
    keys = list(trainer.g_losses.keys())
    g_losses = {kk: float(v.mean()) for kk, v in trainer.g_losses.items()}
    p = case + "/"
    res[p + "loss_keys"] = np.frombuffer(json.dumps(keys).encode(), dtype=np.uint8)
    res[p + "fake"] = seen["fake"]
    for kk, v in g_losses.items():
        res[p + "loss_" + kk] = np.float64(v)
    names = ["fc.layer1.0.weight_orig", "fc.layer5.0.weight_orig"] + (["fc.fc.weight", "fc.fc.bias"] if mode == "norm" else [])
    params = dict(netG.named_parameters())
    for n in names:
        res[p + "grad_" + n] = params[n].grad.clone()
    if mode == "norm":
        assert params["fc.layer6.0.weight_orig"].grad is None
    sd_after = netG.state_dict()
    nl = 6 if mode == "norm" else 5
    for i in range(1, nl + 1):
        for uv in ("u", "v"):
            key = "fc.layer%d.0.weight_%s" % (i, uv)
            res[p + "post_" + key] = sd_after[key].detach().numpy().copy()
    if mode == "norm":
        for uv in ("u", "v"):
            key = "fc.layer6.0.weight_" + uv
            assert torch.equal(sd_after[key], sdG0[key]), key

    # the oracle on the same weights, inputs and dilation
    oopt = orc.default_opt(ngf=c["ngf"], ndf=c["ndf"], crop_size=size, isTrain=True)
    sdG = {kk: v.clone() for kk, v in sdG0.items()}
    sdD = {kk: v.clone() for kk, v in sdD0.items()}
    for n, _ in netG.named_parameters():
        sdG[n].requires_grad_(True)
    losses_o, fake_o = oie.compute_generator_loss(sdG, sdD, oopt, mode, gp, pre, rng_k=k)
    orc.trainer_loss(losses_o).backward()
    assert list(losses_o.keys()) == keys, (list(losses_o.keys()), keys)
    for kk in keys:
        print("  %-15s G loss %-9s ref %.7f oracle %.7f" % (case, kk, g_losses[kk], float(losses_o[kk].mean())))
        assert abs(g_losses[kk] - float(losses_o[kk].mean())) <= 1e-5 * max(1.0, abs(g_losses[kk]))
    pairs = [("fake", fake_o)] + [("grad_" + n, sdG[n].grad) for n in names]
    for name, o in pairs:
        r = torch.as_tensor(res[p + name])
        rel = float((o.detach() - r).abs().max() / r.abs().max())
        print("  %-15s %-30s max-abs rel %.2e" % (case, name, rel))
        # the encoder gradients cross five fp32 InstanceNorm backwards (the last on an 8x8 map) summed in two different
        # orders: a few 1e-3 of their largest element
        assert rel <= (1e-4 if name == "fake" else 1e-2), name
    for i in range(1, 6):
        for uv in ("u", "v"):
            key = "fc.layer%d.0.weight_%s" % (i, uv)
            assert torch.allclose(sdG[key], torch.as_tensor(res[p + "post_" + key]), atol=1e-6), key
    for name in BIG:
        if p + name in res:
            res[p + name] = summary_of(res[p + name])


def summary_of(t):
    from helpers import summary
    return summary(torch.as_tensor(t))


def main():
    out_path = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "golden_image_encoders.npz"))
    import oracle_image_encoders as oie
    warnings.filterwarnings("ignore")
    torch.set_num_threads(8)
    torch.manual_seed(0)
    ref_shims.patch_training()
    res = {"config": np.frombuffer(json.dumps(CFG).encode(), dtype=np.uint8)}
    for case in oie.CASES:
        run_case(case, res)
    res = {kk: (v.numpy() if torch.is_tensor(v) else v) for kk, v in res.items()}
    np.savez_compressed(out_path, **res)
    print("wrote", out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main()
