"""H100: --use_vae on the kernels - KLDLoss (mg_loss_reduce ops 3 and 13), ConvEncoder, the generator's latent head, the whole
stand-alone generator step against the oracle and the reference's fixture, one train iteration and sampling from the prior.

Bounds, from the operand formats (precision.py):
  * op 13 is fp32 per element (expm1f, <= 2 ulp) summed in fp64: per-element 1e-6 relative, sums 1e-6 relative.
  * ConvEncoder forward: layers 2-6 and fc_mu | fc_var run the three-pass bf16 split (~16 significand bits, 2^-16 relative per
    operand) on InstanceNorm-normalised maps; six layers of that stay well below 1e-3 relative L2 on mu and logvar.  Its
    gradients run TF32 (2^-11 relative per operand) through six InstanceNorm backwards: 1e-2 relative L2.
  * Latent head: one TF32 GEMM; z is read as TF32 (truncated to 10 bits, 2^-10) and the weight is rounded to TF32 (2^-11), so
    each output is within 2^-9 of sum |z_j w_kj| plus fp32 accumulation; the same per-element bound holds for dz, dW and db
    (db is the weight-gradient GEMM against a column of ones).
  * The whole step adds the generator's mixed-precision forward (DESIGN.md §5: image error ~1e-3 absolute) and its bf16
    gradient GEMMs (gradient cosine >= 0.999 against fp32, tests/test_gpu_parity.py): losses to 1e-2 relative, the image to
    1e-2 of its range, parameter gradients to cosine 0.99.
"""
import random

import numpy as np
import pytest
import torch

import michigan_oracle as orc
import oracle_vae as ov
from helpers import summary

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm())


def _cos(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float(a @ b / (a.norm() * b.norm()))


@pytest.mark.parametrize("n,z", [(8, 256), (3, 333), (1, 5)])
def test_kld_op13_elementwise(n, z):
    from michigan_b200.networks.loss import KLDLoss
    g = torch.Generator().manual_seed(n * 1000 + z)
    mu = (torch.randn(n, z, generator=g) * 2).to(DEV).requires_grad_()
    logvar = (torch.rand(n, z, generator=g) * 16 - 8).to(DEV).requires_grad_()
    loss = KLDLoss()(mu, logvar)
    m64, l64 = mu.detach().double(), logvar.detach().double()
    ref = 0.5 * (m64 ** 2).sum() + 0.5 * (torch.expm1(l64) - l64).sum()
    assert abs(float(loss.detach()) - float(ref)) <= 1e-6 * abs(float(ref))
    gup = 0.37
    (loss * gup).backward()
    np.testing.assert_allclose(mu.grad.double().cpu().numpy(), (gup * m64).cpu().numpy(), rtol=1e-6, atol=0)
    dl = gup * 0.5 * torch.expm1(l64)
    np.testing.assert_allclose(logvar.grad.double().cpu().numpy(), dl.cpu().numpy(), rtol=2e-6, atol=1e-12)


def _encoder(ngf, size):
    from michigan_b200 import networks
    from michigan_b200.options import make_opt
    from michigan_b200.synth import fill_state_dict
    E = networks.ConvEncoder(make_opt(ngf=ngf, crop_size=size, use_vae=True))
    sd = {k: v.detach().clone() for k, v in E.state_dict().items()}
    fill_state_dict(sd, 21)
    E.load_state_dict(sd)
    return E.to(DEV).train(), sd


def test_conv_encoder_forward_and_gradients_vs_fp64():
    torch.manual_seed(0)
    E, sd = _encoder(64, 512)
    img = (torch.rand(8, 3, 512, 512) * 2 - 1).to(DEV)
    mu, logvar = E(img)
    sd64 = {k: v.to(DEV).double() for k, v in sd.items()}
    for k, v in sd64.items():
        if not k.endswith(("weight_u", "weight_v")):
            v.requires_grad_(True)
    mu_o, lv_o = ov.conv_encoder(sd64, img.double(), True)
    assert _rel_l2(mu, mu_o) <= 1e-3 and _rel_l2(logvar, lv_o) <= 1e-3, (_rel_l2(mu, mu_o), _rel_l2(logvar, lv_o))
    for i in range(1, 7):          # the in-place power iteration of this forward
        for uv in ("u", "v"):
            got = getattr(E, "layer%d" % i)[0].__getattr__("weight_" + uv)
            assert _rel_l2(got, sd64["layer%d.0.weight_%s" % (i, uv)]) <= 1e-5
    dmu, dlv = torch.randn_like(mu), torch.randn_like(logvar)
    ((mu * dmu).sum() + (logvar * dlv).sum()).backward()
    ((mu_o * dmu.double()).sum() + (lv_o * dlv.double()).sum()).backward()
    for name, p in E.named_parameters():
        assert p.grad is not None, name
        err = _rel_l2(p.grad, sd64[name].grad)
        assert err <= 1e-2, (name, err)


def test_latent_head_vs_fp64():
    from michigan_b200 import networks
    from michigan_b200.networks.autograd import _Grads, latent_bwd
    from michigan_b200.options import make_opt
    torch.manual_seed(1)
    G = networks.SPADEBGenerator(make_opt(ngf=64, crop_size=512, use_vae=True)).to(DEV)
    with torch.no_grad():
        G.fc.weight.normal_(0, 0.05)
        G.fc.bias.normal_(0, 0.05)
    N = 8
    z = torch.randn(N, 256, device=DEV)
    S = type("S", (), {})()
    x = G.latent_head(z, N, DEV, S)
    W, b = G.fc.weight.detach().double(), G.fc.bias.detach().double()
    ref = (z.double() @ W.t() + b).view(N, 16 * 64, G.sh, G.sw).permute(0, 2, 3, 1)
    scale = (z.double().abs() @ W.abs().t()).view(N, 16 * 64, G.sh, G.sw).permute(0, 2, 3, 1)
    assert bool(((x.double() - ref).abs() <= 2.0 ** -9 * scale + 1e-6).all())
    dx = torch.randn_like(x)
    grads = _Grads()
    dz = latent_bwd(grads, G.fc, S, dx.contiguous())
    dy = dx.double().permute(0, 3, 1, 2).reshape(N, -1)          # the reference's NCHW row order
    dz_ref = dy @ W
    assert bool(((dz.double() - dz_ref).abs() <= 2.0 ** -9 * (dy.abs() @ W.abs()) + 1e-6).all())
    dW_ref = dy.t() @ z.double()
    dW = grads.get(G.fc.weight).double()
    assert bool(((dW - dW_ref).abs() <= 2.0 ** -9 * (dy.abs().t() @ z.double().abs()) + 1e-6).all())
    db = grads.get(G.fc.bias).double()
    assert bool(((db - dy.sum(0)).abs() <= 2.0 ** -9 * dy.abs().sum(0) + 1e-6).all())   # the same GEMM, against ones


def _fixture_model():
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel
    z, c, sdG, sdD, sdE, data, pre, eps, k = ov.fixture_inputs()
    opt = make_opt(is_train=True, ngf=c["ngf"], ndf=c["ndf"], crop_size=c["size"], batchSize=c["batch"], use_vae=True)
    model = Pix2PixModel(opt)
    model.netG.load_state_dict(sdG)
    model.netD.load_state_dict(sdD)
    model.netE.load_state_dict(sdE)
    return z, c, model, sdG, sdD, sdE, data, pre, eps, k


class _FixedEps:
    def __init__(self, eps):
        self.eps = eps

    def __enter__(self):
        self.orig = torch.randn_like
        torch.randn_like = lambda t, *a, **kw: self.eps.to(t.device).clone()

    def __exit__(self, *exc):
        torch.randn_like = self.orig
        return False


def test_generator_step_matches_oracle_and_fixture():
    z, c, model, sdG, sdD, sdE, data, pre, eps, k = _fixture_model()
    random.seed(c["py_seed"])
    with _FixedEps(eps):
        g_losses, fake = model(data, mode="generator")
    assert list(g_losses) == ["KLD", "GAN", "GAN_Feat"]
    sum(v.mean() for v in g_losses.values()).backward()
    # oracle in float64 on the CPU, same weights, inputs, eps and dilation
    opt = orc.default_opt(ngf=c["ngf"], ndf=c["ndf"], crop_size=c["size"], isTrain=True)
    opt.lambda_kld = 0.05
    sd64 = [{kk: v.double() for kk, v in sd.items()} for sd in (sdG, sdD, sdE)]
    for sd in (sd64[0], sd64[2]):
        for kk, v in sd.items():
            if not kk.endswith(("weight_u", "weight_v", "running_mean", "running_var", "num_batches_tracked")):
                v.requires_grad_(True)
    pre64 = {kk: v.double() for kk, v in pre.items()}
    losses_o, fake_o, mu_o, lv_o = ov.compute_generator_loss(sd64[0], sd64[1], sd64[2], opt, pre64, eps.double(), rng_k=k)
    orc.trainer_loss(losses_o).backward()
    for key in g_losses:
        got, o, ref = float(g_losses[key].detach().mean()), float(losses_o[key].detach().mean()), float(z["loss_" + key])
        assert abs(got - o) <= 1e-2 * max(abs(o), 0.1), (key, got, o)
        assert abs(got - ref) <= 1e-2 * max(abs(ref), 0.1), (key, got, ref)
    assert float((fake.detach().double().cpu() - fake_o.detach()).abs().max()) <= 1e-2 * 2
    got_s, ref_s = summary(fake), z["fake"]
    assert np.abs(got_s[4:] - ref_s[4:]).max() <= 1e-2 * 2
    E, G = model.netE, model.netG
    assert _cos(E.layer1[0].weight_orig.grad, sd64[2]["layer1.0.weight_orig"].grad) >= 0.99
    assert _cos(E.layer1[0].weight_orig.grad, torch.as_tensor(z["grad_layer1.0.weight_orig"])) >= 0.99
    for name, p in list(E.named_parameters()) + [("fc.weight", G.fc.weight), ("fc.bias", G.fc.bias)]:
        ref = (sd64[0] if p is G.fc.weight or p is G.fc.bias else sd64[2])[name].grad
        assert _cos(p.grad, ref) >= 0.99, (name, _cos(p.grad, ref))
    for i in range(1, 7):
        for uv in ("u", "v"):
            got = getattr(E, "layer%d" % i)[0].__getattr__("weight_" + uv).detach().cpu().numpy()
            np.testing.assert_allclose(got, z["post_layer%d.weight_%s" % (i, uv)], rtol=0, atol=1e-4)


def test_train_iteration_updates_netE():
    from michigan_b200.pix2pix_model import train_iteration
    z, c, model, *_ , data, pre, eps, k = _fixture_model()
    opt_g, opt_d = model.create_optimizers(model.opt)
    before = {n: p.detach().clone() for n, p in model.netE.named_parameters()}
    g_losses, d_losses, _ = train_iteration(model, opt_g, opt_d, data)
    assert "KLD" in g_losses and all(bool(torch.isfinite(v).all()) for v in list(g_losses.values()) + list(d_losses.values()))
    for n, p in model.netE.named_parameters():
        assert bool(torch.isfinite(p).all()), n
        assert not torch.equal(p.detach(), before[n]), n
    mu, logvar = model(data, mode="encode_only")
    assert mu.shape == logvar.shape == (c["batch"], 256)


def test_inference_samples_z_from_the_prior():
    z, c, model, *_ , data, pre, eps, k = _fixture_model()
    G = model.netG.eval()
    p = {kk: v.to(DEV) for kk, v in pre.items()}
    outs = []
    for seed in (0, 1):
        torch.manual_seed(seed)
        with torch.no_grad():
            outs.append(G(p["input_ref"], z=None, orient_mask=p["orient_mask"], image_ref=p["image_ref"], input_tag=p["input_tag"],
                          noise=p["noise"], image_tag=p["image_tag"]))
    assert all(bool(torch.isfinite(o).all()) for o in outs)
    assert float((outs[0] - outs[1]).abs().max()) > 1e-3
