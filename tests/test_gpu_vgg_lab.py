"""VGG19 perceptual loss and Lab colour loss on the sm_90a kernels (csrc/mg_vgg.cu + the conv kernels) against the fp32 oracle
(tests/oracle_vgg_lab.py, itself pinned to the reference by tests/test_oracle_vgg_lab.py).

Bounds.  The VGG forward runs with fp16 operands (11-bit significand) and the backward with bf16 data gradients, so the loss
value is checked to 2e-3 relative (measured 1.3e-6 .. 6.5e-5 on an H100) and d fake by cosine >= 0.99 (measured 0.9939 ..
0.9956).  The L1 loss is piecewise linear, and with random VGG weights 30-46 % of the tap elements are exactly 0 in both fake
and real (dead ReLUs), where sign(x_i - y_i) = 0; one operand rounding turns many of them into +-1.  Rounding the operands of
the fp32 oracle's convs to fp16 reproduces the kernels' d fake error on its own (cosine 0.9958, relative L2 9.1 % at 64x64),
so the backward chain is also checked with fixed random gradients on the five taps, where no sign can flip.  There the fp16
forward still moves ReLU masks and pool arg-maxes of near-equal values: the fp16-rounded oracle alone is 3.9e-2 (relative L2
of d image, 64x64) from the fp32 one, the kernels 4.1e-2 (64x64) and 4.7e-2 (256x256); bound 8e-2.  The printed values are
the measurements; the bounds keep a margin over them."""
import os
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle_vgg_lab as ovl

pytestmark = pytest.mark.gpu


@pytest.fixture
def fp32_cudnn():
    """The oracle's convolutions on the GPU in true fp32 (cuDNN's TF32 default off for the test)."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def _images(n, size, seed=0):
    from test_oracle_vgg_lab import _inputs
    return _inputs(n, size, seed)


def _vgg(seed=0):
    from michigan_b200.networks import VGGLoss
    from michigan_b200.options import make_opt
    from michigan_b200.synth import vgg19_state_dict
    sd = vgg19_state_dict(seed)
    return VGGLoss(make_opt(), state_dict=sd), sd


def _cos(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float(a @ b / (a.norm() * b.norm()))


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


# ------------------------------------------------------------------------------------------------ max-pool / ReLU kernels
def _pool_input(n, h, w, c, seed):
    """ReLU-like NHWC tensor with planted ties (values on a 1/4 grid, whole windows equal) and zeros."""
    g = torch.Generator().manual_seed(seed)
    a = torch.relu(torch.randn(n, h, w, c, generator=g))
    a[:, ::3] = torch.round(a[:, ::3] * 4) / 4
    a[:, 0:2, 0:2] = 0.75
    a[0, :, :, :8] = 0.0
    return a.cuda()


@pytest.mark.parametrize("shape", [(2, 8, 10, 64), (1, 7, 9, 128), (2, 6, 5, 256)])
@pytest.mark.parametrize("in_dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_maxpool2_forward_backward_vs_torch(shape, in_dtype):
    from michigan_b200 import ops
    n, h, w, c = shape
    a = _pool_input(n, h, w, c, 1).to(in_dtype)
    af = a.float()
    ref = F.max_pool2d(af.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    y32, y16 = ops.maxpool2(a, out16=ops.F16)
    assert torch.equal(y32, ref)
    assert torch.equal(y16, ref.half())
    assert torch.equal(ops.maxpool2(a, out16=ops.BF16, want_f32=False)[1], ref.bfloat16())

    g = torch.Generator().manual_seed(2)
    dp = torch.randn(tuple(ref.shape), generator=g).cuda()
    add = torch.randn(tuple(a.shape), generator=g).cuda()
    at = af.permute(0, 3, 1, 2).clone().requires_grad_()
    F.max_pool2d(at, 2, 2).backward(dp.permute(0, 3, 1, 2))
    want = ((at.grad.permute(0, 2, 3, 1) + add) * (af > 0)).contiguous()
    dx32, dx16 = ops.maxpool2_relu_bwd(dp, a, add=add, want16=True)
    assert torch.equal(dx32, want)
    assert torch.equal(dx16, want.bfloat16())
    assert torch.equal(ops.maxpool2_relu_bwd(dp, a), (at.grad.permute(0, 2, 3, 1) * (af > 0)).contiguous())
    # `add` may be the output buffer itself (the tap gradient accumulated in place)
    buf = add.clone()
    ops._lib.check(ops._lib.load().mg_maxpool2_relu_bwd(dp.data_ptr(), af.contiguous().data_ptr(), None, 0, buf.data_ptr(), buf.data_ptr(),
                                                        None, n, h, w, c, ops._stream()), "mg_maxpool2_relu_bwd")
    assert torch.equal(buf, want)

    dy = torch.randn(tuple(a.shape), generator=g).cuda()
    dz32, dz16 = ops.relu_bwd16(dy, a, add=add, want16=True)
    r = ((dy + add) * (af > 0)).contiguous()
    assert torch.equal(dz32, r) and torch.equal(dz16, r.bfloat16())


# ------------------------------------------------------------------------------------------------ VGG loss
@pytest.mark.parametrize("size,mode", [(64, "mixed16"), (64, "tf32"), (512, "mixed16")])
def test_vgg_loss_value_and_grad_vs_oracle(size, mode, fp32_cudnn):
    from michigan_b200 import precision
    old = precision.mode()
    precision.set_mode(mode)
    try:
        crit, sd = _vgg()
        fake, real = _images(2, size)
        x = fake.cuda().requires_grad_()
        loss = crit(x, real.cuda())
        loss.backward()
        torch.cuda.synchronize()
    finally:
        precision.set_mode(old)
    sdc = {k: v.cuda() for k, v in sd.items()}
    xr = fake.cuda().requires_grad_()
    ref = ovl.vgg_loss(xr, real.cuda(), sdc)
    ref.backward()
    rel = abs(float(loss) - float(ref)) / abs(float(ref))
    cos = _cos(x.grad, xr.grad)
    print("VGG %d^2 %s: loss %.6f oracle %.6f rel %.2e; d fake cosine %.5f rel L2 %.3e"
          % (size, mode, float(loss), float(ref), rel, cos, _rel(x.grad, xr.grad)))
    assert torch.isfinite(x.grad).all()
    assert rel <= 2e-3
    assert cos >= 0.99


@pytest.mark.parametrize("size", [64, 256])
def test_vgg_backward_chain_vs_oracle_autograd(size, fp32_cudnn):
    """The hand-written VGG19 backward (ReLU / max-pool backward kernels, bf16 data-gradient GEMMs, thin_dgrad3) with fixed
    random upstream gradients on the five taps: smooth in the features, so no L1 sign can flip."""
    from michigan_b200 import ops
    crit, sd = _vgg()
    crit.vgg.cuda()
    fake, _ = _images(2, size)
    x = fake.cuda()
    taps, S = crit.vgg.run(ops.nchw_to_nhwc(x.contiguous(), 4), n_save=2)
    g = torch.Generator().manual_seed(5)
    gt = [torch.randn(tuple(t.shape), generator=g).cuda() for t in taps]
    dimg = crit.vgg.backward(S, gt, (size, size))
    sdc = {k: v.cuda() for k, v in sd.items()}
    xr = x.clone().requires_grad_()
    feats = ovl.vgg19_features(xr, sdc)
    sum((f * gg.permute(0, 3, 1, 2)).sum() for f, gg in zip(feats, gt)).backward()
    frel = max(_rel(t.permute(0, 3, 1, 2), f) for t, f in zip(taps, feats))
    rel = _rel(dimg, xr.grad)
    print("VGG chain %d^2: taps worst rel L2 %.3e; d image rel L2 %.3e" % (size, frel, rel))
    assert rel <= 8e-2


# ------------------------------------------------------------------------------------------------ Lab loss
def test_lab_loss_vs_oracle_with_saturated_pixels():
    from michigan_b200.networks import LabColorLoss
    from michigan_b200.options import make_opt
    fake, real = _images(2, 96)
    fake[:, :, :8] = -1.0                 # tanh saturated in fp32: X = Y = Z = 0
    fake[:, :, 8:16] = 1.0
    fake[0, 0, 20:30] = -1.0
    real[:, :, 40:44] = -1.0
    x = fake.cuda().requires_grad_()
    loss = LabColorLoss(make_opt())(x, real.cuda())
    (loss * 1.5).backward()
    xr = fake.clone().requires_grad_()
    ref = ovl.lab_loss(xr, real)
    (ref * 1.5).backward()
    rel = abs(float(loss) - float(ref)) / abs(float(ref))
    grel = _rel(x.grad.cpu(), xr.grad)
    print("Lab: loss %.7f oracle %.7f rel %.2e; d fake rel L2 %.3e" % (float(loss), float(ref), rel, grel))
    assert torch.isfinite(x.grad).all()
    assert rel <= 1e-5
    assert grel <= 1e-4


def test_losses_are_bit_reproducible():
    from michigan_b200.networks import LabColorLoss
    from michigan_b200.options import make_opt
    crit, _ = _vgg()
    lab = LabColorLoss(make_opt())
    fake, real = _images(2, 128, seed=3)
    outs = []
    for _ in range(2):
        x = fake.cuda().requires_grad_()
        lv, ll = crit(x, real.cuda()), lab(x, real.cuda())
        (lv + ll).backward()
        torch.cuda.synchronize()
        outs.append((lv.detach().clone(), ll.detach().clone(), x.grad.clone()))
    assert all(torch.equal(a, b) for a, b in zip(*outs))


# ------------------------------------------------------------------------------------------------ end to end
def test_generator_step_readme_losses_vs_oracle(tmp_path):
    """One generator step of Pix2PixModel with the README's loss set at the golden configuration (ngf 64, 128x128, batch 2)
    against the oracle's generator step with the same terms: losses within 1e-2 relative, per-tensor G-gradient cosine >= 0.998
    on the tensors the golden fixture samples."""
    import michigan_oracle as orc
    from helpers import load_golden, preprocessed, reference_layout_state, summary
    from michigan_b200.networks.architecture import VGG19_WEIGHTS_FILE
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel
    from michigan_b200.synth import synthetic_batch, vgg19_state_dict
    z, cfg = load_golden()
    sd_vgg = vgg19_state_dict(0)
    os.makedirs(tmp_path / "checkpoints")
    torch.save(sd_vgg, tmp_path / "checkpoints" / VGG19_WEIGHTS_FILE)
    old_hub = torch.hub.get_dir()
    torch.hub.set_dir(str(tmp_path))
    try:
        opt = make_opt(is_train=True, ngf=cfg["ngf"], ndf=cfg["ndf"], crop_size=cfg["size"], batchSize=cfg["batch"], no_vgg_loss=False,
                       no_lab_loss=False, no_orient_loss=False)
        model = Pix2PixModel(opt)
    finally:
        torch.hub.set_dir(old_hub)
    sdG = reference_layout_state("G", cfg, cfg["seed_G"])
    sdD = reference_layout_state("D", cfg, cfg["seed_D"])
    model.netG.load_state_dict(sdG)
    model.netD.load_state_dict(sdD)
    model.train()
    data = synthetic_batch(cfg["batch"], cfg["size"], cfg["data_seed"])
    random.seed(cfg["py_seed"])
    th = int(cfg["size"] * 0.05); th = th if th % 2 == 1 else th + 1
    k = random.choice([max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4])
    random.seed(cfg["py_seed"])
    g_losses, _ = model(dict(data), mode="generator")
    sum(v.mean() for v in g_losses.values()).backward()
    torch.cuda.synchronize()
    assert list(g_losses) == ["GAN", "GAN_Feat", "VGG", "lab", "ORIENT"]

    _, pre = preprocessed(cfg)
    oopt = orc.default_opt(ngf=cfg["ngf"], ndf=cfg["ndf"], crop_size=cfg["size"], isTrain=True)
    names = [n for n in sdG if not n.endswith(("running_mean", "running_var", "num_batches_tracked", "weight_u", "weight_v"))]
    for n in names:
        sdG[n].requires_grad_(True)
    losses_o, _ = ovl.compute_generator_loss_readme(sdG, sdD, sd_vgg, oopt, pre, rng_k=k)
    orc.trainer_loss(losses_o).backward()
    assert list(losses_o) == list(g_losses)
    for key in g_losses:
        a, b = float(g_losses[key].mean()), float(losses_o[key].mean())
        print("   %-9s %.6f  oracle %.6f" % (key, a, b))
        assert abs(a - b) <= 1e-2 * max(1.0, abs(b)), key
    named = dict(model.netG.named_parameters())
    worst = 1.0
    for key in z.files:
        if key.startswith("g_grad/") and not key.endswith("conv_0.bias"):   # bias before a batch-norm: gradient is exactly 0
            n = key[len("g_grad/"):]
            a, b = summary(named[n].grad, stride=101)[4:], summary(sdG[n].grad, stride=101)[4:]
            cos = float(np.dot(a.astype(np.float64), b) / (np.linalg.norm(a) * np.linalg.norm(b)))
            print("   %-45s cosine %.5f" % (n, cos))
            worst = min(worst, cos)
    assert worst >= 0.998, worst
