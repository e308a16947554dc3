"""H100: --Image_encoder_mode instance and norm on the kernels - the unmasked and unbroadcast modes of mg_masked_mean_bcast
and its backward, ImageEncoder2 and ImageEncoder, the whole stand-alone generator step against the oracle and the reference's
fixture, one train iteration per mode and an eval forward.

Bounds, from the operand formats (precision.py):
  * The mean pair is fp32 per element: each channel's sum of h*w fp32 products, then one division and one product.  Against
    float64, per element (h*w + 2) * 2^-24 of the same expression on |x| (or |dout|).
  * Encoders: layers 2-5 run the three-pass bf16 split (~16 significand bits) on InstanceNorm-normalised maps; five layers
    of that stay well below 1e-3 relative L2 on the output.  norm's fc is the latent head's TF32 GEMM (2^-10 relative per
    product, DESIGN.md), also below 1e-3 relative L2.  Gradients run TF32 (2^-11 relative per operand) through five
    InstanceNorm backwards: 1e-2 relative L2, as for ConvEncoder (tests/test_gpu_vae.py).
  * The whole step adds the generator's mixed-precision forward (DESIGN.md §5: image error ~1e-3 absolute) and its bf16
    gradient GEMMs: losses to 1e-2 relative, the image to 1e-2 of its range, parameter gradients to cosine 0.99.
"""
import random

import numpy as np
import pytest
import torch

import michigan_oracle as orc
import oracle_image_encoders as oie
from helpers import summary
from michigan_b200 import ops

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm())


def _cos(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float(a @ b / (a.norm() * b.norm()))


def _mean_bcast64(x, mref, mtag):
    """float64 restatement on NCHW-free tensors: x [N,h,w,C], masks [N,MH,MW] or None."""
    N, h, w, C = x.shape
    if mref is None:
        r = torch.ones((N, h, w), dtype=torch.float64)
    else:
        r = mref[:, ::mref.shape[1] // h, ::mref.shape[2] // w].double()
    t = torch.ones((N, h, w), dtype=torch.float64) if mtag is None else mtag[:, ::mtag.shape[1] // h, ::mtag.shape[2] // w].double()
    mean = (x * r[..., None]).sum(dim=(1, 2)) / torch.clamp(r.sum(dim=(1, 2)), min=1)[:, None]
    return mean[:, None, None, :] * t[..., None]


@pytest.mark.parametrize("N,C,h,w,MH,MW,masks", [
    (2, 96, 8, 8, 8, 8, "none"), (3, 1024, 16, 16, 512, 512, "ref_none"), (1, 40, 5, 7, 20, 14, "tag_none"),
    (8, 1024, 8, 8, 256, 256, "none"), (4, 512, 18, 18, 576, 576, "ref_none"), (2, 64, 8, 8, 256, 256, "empty_ref"),
])
def test_masked_mean_null_modes_elementwise(N, C, h, w, MH, MW, masks):
    g = torch.Generator().manual_seed(N * 7 + C + h)
    x = torch.randn(N, h, w, C, generator=g, dtype=torch.float64)
    dout = torch.randn(N, h, w, C, generator=g, dtype=torch.float64)
    mref = (torch.rand(N, MH, MW, generator=g) < 0.4).float()
    mtag = (torch.rand(N, MH, MW, generator=g) < 0.6).float()
    if masks == "empty_ref":
        # image 0: hair only off the map's sampling grid, so its count at the grid is 0 (the max(count, 1) clamp)
        s = MH // h
        mref[0] = 0.
        mref[0, 1::s, 1::s] = 1.
    mref = None if masks in ("none", "ref_none") else mref
    mtag = None if masks in ("none", "tag_none") else mtag
    dm = [None if m is None else m.to(DEV) for m in (mref, mtag)]
    got = ops.masked_mean_bcast(x.float().to(DEV), *dm).double().cpu()
    xf = x.float().double()
    ref = _mean_bcast64(xf, mref, mtag)
    bound = (h * w + 2) * 2.0 ** -24 * _mean_bcast64(xf.abs(), mref, mtag) + 1e-30
    assert bool(((got - ref).abs() <= bound).all()), float((got - ref).abs().max())
    if masks == "empty_ref":
        assert float(got[0].abs().max()) == 0.0
    # backward: dx[q,c] = ref[q] / max(count, 1) * sum_p dout[p,c] tag[p]  (the adjoint of the forward)
    df = dout.float().double()
    dx = ops.masked_mean_bcast_bwd(dout.float().to(DEV), *dm).double().cpu()
    xr = xf.clone().requires_grad_(True)
    (_mean_bcast64(xr, mref, mtag) * df).sum().backward()
    xa = xf.abs().clone().requires_grad_(True)
    (_mean_bcast64(xa, mref, mtag) * df.abs()).sum().backward()
    bound = (h * w + 2) * 2.0 ** -24 * xa.grad + 1e-30
    assert bool(((dx - xr.grad).abs() <= bound).all()), float((dx - xr.grad).abs().max())


def test_masked_mean_refuses_mismatched_masks():
    x = torch.zeros(1, 8, 8, 32, device=DEV)
    with pytest.raises(Exception, match="multiple"):
        ops.masked_mean_bcast(x, None, torch.zeros(1, 12, 12, device=DEV))
    with pytest.raises(Exception, match="multiple"):
        ops.masked_mean_bcast_bwd(x, torch.zeros(1, 12, 12, device=DEV), None)


def _generator(mode, gp, ngf, size, seed=21):
    from michigan_b200 import networks
    from michigan_b200.options import make_opt
    from michigan_b200.synth import fill_state_dict
    G = networks.SPADEBGenerator(make_opt(ngf=ngf, ndf=ngf, crop_size=size, Image_encoder_mode=mode, ref_global_pool=gp))
    sd = {k: v.detach().clone() for k, v in G.state_dict().items()}
    fill_state_dict(sd, seed)
    G.load_state_dict(sd)
    return G.to(DEV).train(), sd


@pytest.mark.parametrize("case", list(oie.CASES))
def test_encoder_forward_and_gradients_vs_fp64(case):
    from michigan_b200.networks.autograd import _Grads
    mode, gp = oie.CASES[case]
    torch.manual_seed(0)
    G, sd = _generator(mode, gp, 64, 512)
    E = G.fc
    N, H = 8, 512
    img = (torch.rand(N, 3, H, H) * 2 - 1).to(DEV)
    lab_ref = torch.zeros(N, 1, H, H)
    lab_ref[:, :, 100:300, 90:420] = 1
    lab_ref[1] = torch.roll(lab_ref[1], 64, dims=-1)
    lab_tag = torch.zeros(N, 1, H, H)
    lab_tag[:, :, 120:330, 100:400] = 1
    lab_ref, lab_tag = lab_ref.to(DEV), lab_tag.to(DEV)
    S = type("S", (), {})()
    out = E.forward_nhwc(img, lab_ref, lab_tag, save=S)
    assert out.shape == (N, G.sh, G.sw, 16 * 64)
    sd64 = {k[3:]: v.to(DEV).double() for k, v in sd.items() if k.startswith("fc.")}
    for k, v in sd64.items():
        if not k.endswith(("weight_u", "weight_v")):
            v.requires_grad_(True)
    o64 = oie.encode({"fc." + k: v for k, v in sd64.items()}, orc.default_opt(ngf=64, crop_size=512), mode, gp,
                     torch.cat([1 - lab_ref, lab_ref], 1).double(), torch.cat([1 - lab_tag, lab_tag], 1).double(),
                     img.double(), True)
    got = out.permute(0, 3, 1, 2)
    assert _rel_l2(got, o64) <= 1e-3, _rel_l2(got, o64)
    for i in range(1, 6):          # the in-place power iteration of this forward
        for uv in ("u", "v"):
            assert _rel_l2(getattr(E, "layer%d" % i)[0].__getattr__("weight_" + uv), sd64["layer%d.0.weight_%s" % (i, uv)]) <= 1e-5
    dout = torch.randn_like(out)
    grads = _Grads()
    E.backward_nhwc(grads, S, dout.contiguous())
    (o64 * dout.permute(0, 3, 1, 2).double()).sum().backward()
    for name, p in E.named_parameters():
        if name.startswith("layer6."):
            assert grads.get(p) is None
            continue
        g = grads.get(p)
        assert g is not None, name
        err = _rel_l2(g.reshape(p.shape), sd64[name].grad)
        assert err <= 1e-2, (name, err)


def _fixture_model(case):
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel
    z, c, sdG, sdD, data, pre, k = oie.fixture_inputs(case)
    mode, gp = oie.CASES[case]
    opt = make_opt(is_train=True, ngf=c["ngf"], ndf=c["ndf"], crop_size=c["size"], batchSize=c["batch"], Image_encoder_mode=mode,
                   ref_global_pool=gp)
    model = Pix2PixModel(opt)
    model.netG.load_state_dict(sdG)
    model.netD.load_state_dict(sdD)
    return z, c, model, sdG, sdD, data, pre, k


@pytest.mark.parametrize("case", list(oie.CASES))
def test_generator_step_matches_oracle_and_fixture(case):
    z, c, model, sdG, sdD, data, pre, k = _fixture_model(case)
    mode, gp = oie.CASES[case]
    p = case + "/"
    random.seed(c["py_seed"])
    g_losses, fake = model(data, mode="generator")
    import json
    assert list(g_losses) == json.loads(bytes(z[p + "loss_keys"]).decode())
    sum(v.mean() for v in g_losses.values()).backward()
    opt = orc.default_opt(ngf=c["ngf"], ndf=c["ndf"], crop_size=c["size"], isTrain=True)
    sd64 = [{kk: v.double() for kk, v in sd.items()} for sd in (sdG, sdD)]
    for kk, v in sd64[0].items():
        if not kk.endswith(("weight_u", "weight_v", "running_mean", "running_var", "num_batches_tracked")):
            v.requires_grad_(True)
    pre64 = {kk: v.double() for kk, v in pre.items()}
    losses_o, fake_o = oie.compute_generator_loss(sd64[0], sd64[1], opt, mode, gp, pre64, rng_k=k)
    orc.trainer_loss(losses_o).backward()
    for key in g_losses:
        got, o, ref = float(g_losses[key].detach().mean()), float(losses_o[key].detach().mean()), float(z[p + "loss_" + key])
        assert abs(got - o) <= 1e-2 * max(abs(o), 0.1), (key, got, o)
        assert abs(got - ref) <= 1e-2 * max(abs(ref), 0.1), (key, got, ref)
    assert float((fake.detach().double().cpu() - fake_o.detach()).abs().max()) <= 1e-2 * 2
    assert np.abs(summary(fake)[4:] - z[p + "fake"][4:]).max() <= 1e-2 * 2
    G = model.netG
    params = dict(G.named_parameters())
    for name, prm in params.items():
        if not name.startswith("fc."):
            continue
        if name.startswith("fc.layer6."):
            assert prm.grad is None, name
            continue
        assert _cos(prm.grad, sd64[0][name].grad) >= 0.99, (name, _cos(prm.grad, sd64[0][name].grad))
    assert _cos(params["fc.layer1.0.weight_orig"].grad, torch.as_tensor(z[p + "grad_fc.layer1.0.weight_orig"])) >= 0.99
    if mode == "norm":
        assert _cos(params["fc.fc.bias"].grad, torch.as_tensor(z[p + "grad_fc.fc.bias"])) >= 0.99
    sd_after = G.state_dict()
    for i in range(1, 7 if mode == "norm" else 6):
        for uv in ("u", "v"):
            key = "fc.layer%d.0.weight_%s" % (i, uv)
            np.testing.assert_allclose(sd_after[key].detach().cpu().numpy(), z[p + "post_" + key], rtol=0, atol=1e-4)
    if mode == "norm":
        for uv in ("u", "v"):
            assert torch.equal(sd_after["fc.layer6.0.weight_" + uv].cpu(), sdG["fc.layer6.0.weight_" + uv])


@pytest.mark.parametrize("case", list(oie.CASES))
def test_train_iteration_updates_the_encoder(case):
    from michigan_b200.pix2pix_model import train_iteration
    z, c, model, *_, data, pre, k = _fixture_model(case)
    opt_g, opt_d = model.create_optimizers(model.opt)
    fc = model.netG.fc
    before = {n: p.detach().clone() for n, p in fc.named_parameters()}
    g_losses, d_losses, _ = train_iteration(model, opt_g, opt_d, data)
    assert all(bool(torch.isfinite(v).all()) for v in list(g_losses.values()) + list(d_losses.values()))
    for n, p in fc.named_parameters():
        assert bool(torch.isfinite(p).all()), n
        assert torch.equal(p.detach(), before[n]) == n.startswith("layer6."), n


@pytest.mark.parametrize("case", list(oie.CASES))
def test_eval_forward_keeps_u_v(case):
    z, c, model, sdG, sdD, data, pre, k = _fixture_model(case)
    mode, gp = oie.CASES[case]
    G = model.netG.eval()
    uv0 = {kk: v.detach().clone() for kk, v in G.state_dict().items() if kk.startswith("fc.") and kk.endswith(("_u", "_v"))}
    pd = {kk: v.to(DEV) for kk, v in pre.items()}
    with torch.no_grad():
        out = G(pd["input_ref"], orient_mask=pd["orient_mask"], image_ref=pd["image_ref"], input_tag=pd["input_tag"],
                noise=pd["noise"], image_tag=pd["image_tag"])
    for kk, v in G.state_dict().items():
        if kk in uv0:
            assert torch.equal(v, uv0[kk]), kk
    # the encoder's eval forward against the oracle's eval spectral norm (stored u, v: no power iteration)
    S = None
    x = G.fc.forward_nhwc(pd["image_ref"], pd["input_ref"][:, 1:2], pd["input_tag"][:, 1:2], save=S)
    sd64 = {kk: v.double() for kk, v in sdG.items()}
    o64 = oie.encode(sd64, orc.default_opt(ngf=c["ngf"], crop_size=c["size"]), mode, gp, pre["input_ref"].double(),
                     pre["input_tag"].double(), pre["image_ref"].double(), False)
    assert _rel_l2(x.permute(0, 3, 1, 2), o64) <= 1e-3
    assert bool(torch.isfinite(out).all())
