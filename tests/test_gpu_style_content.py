"""Style, content, background and rgb losses on the sm_90a kernels (mg_in_stats + mg_style_loss_fwd / mg_style_tap_grad, op 3 of
mg_loss_reduce, mg_pixel_l1_fwd / _bwd in csrc/mg_vgg.cu and csrc/mg_loss.cu) against float64 autograd at kernel level, and
against the fp32 oracle (tests/oracle_style_content.py, pinned to the reference by tests/test_oracle_style_content.py) end to end.

Kernel-level bounds follow tests/test_gpu_backward_kernels.py: |got - ref| <= k u R_abs, u = 2^-24, R_abs the same computation
on absolute values (for a difference a - b: |a| + |b|).  The style statistics are mg_in_stats' sums, fp32 over runs of 32 pixels
and fp64 above, so mu and sigma carry up to ~32 u of relative error before the fp64 loss arithmetic.  Each printed value is the
measurement; each bound keeps at least 3x over what an H100 measured."""
import os
import random

import numpy as np
import pytest
import torch

import oracle_style_content as osc

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
# k of the kernel-level checks (measured on an H100: see the printed values)
K_STYLE_LOSS, K_STYLE_GRAD, K_CONTENT, K_PIXEL = 2, 16, 8, 4


@pytest.fixture
def fp32_cudnn():
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def _cos(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float(a @ b / (a.norm() * b.norm()))


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _ratio(got, ref, rabs):
    """max |got - ref| / (u R_abs) (R_abs floored at the smallest normal, for elements that are exactly 0 in both)."""
    return float(((got.double().cpu() - ref.double().cpu()).abs() / (U * rabs.double().cpu().clamp_min(1e-300))).max())


# ------------------------------------------------------------------------------------------------ style kernels
def _tap_shapes(n, size):
    return [(n, size, size, 64), (n, size // 2, size // 2, 128), (n, size // 4, size // 4, 256), (n, size // 8, size // 8, 512),
            (n, size // 16, size // 16, 512)]


def _feature(shape, g):
    """ReLU-like NHWC fp32 map with a dead (all-zero) channel 0 and a constant channel 1 (0.37, not a binary fraction)."""
    f = torch.relu(torch.randn(shape, generator=g) * 0.8 + 0.2)
    f[..., 0] = 0.0
    f[..., 1] = 0.37
    return f


def _style_fp64(fs, ts, c4, gs, gc):
    """fp64 autograd of gs * sum_i [MSE(mu_f, mu_t) + MSE(sigma_f, sigma_t)] + gc * MSE(f_5, c4) -> (style loss, content loss,
    d/d f_i), calc_mean_std on NHWC maps."""
    xs = [f.double().requires_grad_() for f in fs]
    loss_s = 0
    for x, t in zip(xs, ts):
        n, h, w, c = x.shape
        xf, tf = x.reshape(n, h * w, c), t.double().reshape(n, h * w, c)
        loss_s = loss_s + ((xf.mean(1) - tf.mean(1)) ** 2).mean() + \
            (((xf.var(1) + 1e-5).sqrt() - (tf.var(1) + 1e-5).sqrt()) ** 2).mean()
    loss_c = ((xs[-1] - c4.double()) ** 2).mean()
    (gs * loss_s + gc * loss_c).backward()
    return loss_s.detach(), loss_c.detach(), [x.grad for x in xs]


@pytest.mark.parametrize("n,size", [(2, 64), (1, 64), (2, 32)])
def test_style_kernels_vs_fp64_autograd(n, size):
    """mg_in_stats -> mg_style_loss_fwd -> mg_style_tap_grad at the five tap shapes (size 32: a 2x2 relu5_1 map), with dead and
    constant channels, the VGG-L1 gradient as `add` aliasing the output, and the content gradient folded in at relu5_1."""
    from michigan_b200 import ops
    g = torch.Generator().manual_seed(n * 100 + size)
    shapes = _tap_shapes(n, size)
    fs = [_feature(s, g) for s in shapes]
    ts = [_feature(s, g) * 1.3 for s in shapes]
    c4 = _feature(shapes[-1], g)
    adds = [torch.randn(s, generator=g) * 1e-4 for s in shapes]
    gs, gc = 1.7, 0.6
    outs = []
    for _ in range(2):
        sums = [ops.channel_sums(torch.cat([f, t]).cuda()) for f, t in zip(fs, ts)]
        loss, coefs = ops.style_loss_fwd([(s[:n], s[n:], sh[1] * sh[2]) for s, sh in zip(sums, shapes)])
        gv = torch.tensor([gs, gc], device="cuda")
        grads = []
        for i, (f, a) in enumerate(zip(fs, adds)):
            out = a.cuda()
            ops.style_tap_grad(f.cuda(), gv, coef=coefs[i], content_t=c4.cuda() if i == 4 else None, add=out, out=out)
            grads.append(out)
        torch.cuda.synchronize()
        outs.append((loss.clone(), [c.clone() for c in coefs], grads))
    assert torch.equal(outs[0][0], outs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(outs[0][1] + outs[0][2], outs[1][1] + outs[1][2]))
    loss, _, grads = outs[0]

    ref_s, _, ref_g = _style_fp64(fs, ts, c4, gs, gc)
    r_loss = 0.0
    worst_g = 0.0
    for i, (f, t, a) in enumerate(zip(fs, ts, adds)):
        nn_, h, w, c = f.shape
        M = h * w
        fd, td = f.double().reshape(nn_, M, c), t.double().reshape(nn_, M, c)
        mf, mt = fd.mean(1), td.mean(1)
        sf, st = (fd.var(1) + 1e-5).sqrt(), (td.var(1) + 1e-5).sqrt()
        r_loss += float((((mf.abs() + mt.abs()) ** 2 + (sf + st) ** 2)).mean())
        NC = nn_ * c
        ka, kb = 2.0 / (NC * M), 2.0 / (NC * (M - 1))
        rs = (ka * (mf.abs() + mt.abs()))[:, None, :] + (kb * (sf + st) / sf)[:, None, :] * (fd.abs() + mf.abs()[:, None, :])
        rabs = a.double().abs() + gs * rs.reshape(f.shape)
        if i == 4:
            rabs = rabs + gc * 2.0 / f.numel() * (f.double().abs() + c4.double().abs())
        want = a.double() + ref_g[i]
        r = _ratio(grads[i], want, rabs)
        print("style tap %d %s: d tap max |err| / (u R_abs) = %.2f" % (i, tuple(f.shape), r))
        worst_g = max(worst_g, r)
    rl = abs(float(loss) - float(ref_s)) / (U * r_loss)
    print("style loss N=%d %d^2: %.8e fp64 %.8e, |err| / (u R_abs) = %.2f; worst d tap %.2f" % (n, size, float(loss), float(ref_s),
                                                                                                   rl, worst_g))
    assert rl <= K_STYLE_LOSS
    assert worst_g <= K_STYLE_GRAD


def test_style_loss_refuses_a_one_pixel_tap():
    from michigan_b200 import _lib, ops
    s = torch.zeros((1, 2, 512), device="cuda", dtype=torch.float64)
    with pytest.raises(_lib.MichiganNativeError, match="at least 2"):
        ops.style_loss_fwd([(s, s, 1)])


def test_content_op3_vs_fp64_autograd():
    """Op 3 of mg_loss_reduce (f = (a - b)^2, b detached) forward and backward at the relu5_1 shapes of 64^2 and 512^2, batch 2."""
    from michigan_b200.networks.loss import OP_SQ, _LossFn
    g = torch.Generator().manual_seed(7)
    for shape in [(2, 4, 4, 512), (2, 32, 32, 512), (3, 5, 7, 3)]:
        a = torch.relu(torch.randn(shape, generator=g))
        b = torch.relu(torch.randn(shape, generator=g))
        b[0, 0] = a[0, 0]                           # exact ties: zero contribution, zero gradient
        scale = 1.0 / a.numel()
        res = []
        for _ in range(2):
            x = a.cuda().requires_grad_()
            loss = _LossFn.apply([(OP_SQ, 0, b.cuda(), scale, 1.0, 0)], 1, x)
            (loss * 0.75).sum().backward()
            torch.cuda.synchronize()
            res.append((loss.detach().clone(), x.grad.clone()))
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
        xd = a.double().requires_grad_()
        ref = ((xd - b.double()) ** 2).sum() * scale
        (ref * 0.75).backward()
        rl = abs(float(res[0][0]) - float(ref)) / (U * float(((a.double().abs() + b.double().abs()) ** 2).sum() * scale))
        rg = _ratio(res[0][1], xd.grad, 0.75 * scale * 2 * (a.double().abs() + b.double().abs()))
        print("content op 3 %s: loss |err| / (u R_abs) %.2f, grad %.2f" % (shape, rl, rg))
        assert rl <= K_CONTENT and rg <= K_CONTENT
        assert float(res[0][1][0, 0].abs().max()) == 0.0


def _pixel_case(kind, n=2, h=40, w=56, seed=3):
    g = torch.Generator().manual_seed(seed)
    fake = torch.rand(n, 3, h, w, generator=g) * 2 - 1
    tag = torch.rand(n, 3, h, w, generator=g) * 2 - 1
    tag[:, :, :5] = fake[:, :, :5]                                  # exact ties: f == t gives 0
    if kind == "binary":
        mask = (torch.rand(n, h, w, generator=g) > 0.6).float()
    elif kind == "fractional":
        mask = torch.rand(n, h, w, generator=g)
        mask[:, 10:12] = 0.0
    else:
        mask = None
    return fake, tag, mask


@pytest.mark.parametrize("kind", ["binary", "fractional", "rgb"])
def test_pixel_l1_vs_fp64_autograd(kind):
    from michigan_b200 import ops
    fake, tag, mask = _pixel_case(kind)
    numel = fake.numel()
    gup = 1.3
    gscale = torch.tensor([gup / numel], dtype=torch.float32)
    res = []
    for _ in range(2):
        s = ops.pixel_l1_fwd(fake.cuda(), tag.cuda(), mask.cuda() if mask is not None else None)
        d = ops.pixel_l1_bwd(fake.cuda(), tag.cuda(), gscale.cuda(), mask.cuda() if mask is not None else None)
        torch.cuda.synchronize()
        res.append((s.clone(), d.clone()))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    s, d = res[0]
    m = mask.double()[:, None] if mask is not None else torch.ones(1, dtype=torch.float64)
    xd = fake.double().requires_grad_()
    ref = (xd * m - tag.double() * m).abs().sum()
    ref.backward(torch.tensor(float(gscale), dtype=torch.float64))
    rl = abs(float(s) - float(ref)) / (U * float(((fake.double().abs() + tag.double().abs()) * m).sum()))
    rg = _ratio(d, xd.grad, float(gscale) * m.expand_as(xd).abs() + 1e-300)
    print("pixel L1 %s: sum |err| / (u R_abs) %.2f, d fake %.2f" % (kind, rl, rg))
    assert rl <= K_PIXEL and rg <= K_PIXEL
    assert float(d[:, :, :5].abs().max()) == 0.0
    if mask is not None:
        assert bool((d.cpu()[(mask == 0)[:, None].expand_as(d)] == 0).all())


# ------------------------------------------------------------------------------------------------ losses end to end
def _vgg_sd(seed=0):
    from michigan_b200.synth import vgg19_state_dict
    return vgg19_state_dict(seed)


def _images(n, size):
    from test_oracle_style_content import _inputs
    return _inputs(n, size)


@pytest.mark.parametrize("size,mode", [(64, "mixed16"), (64, "tf32"), (512, "mixed16")])
def test_style_content_loss_vs_oracle(size, mode, fp32_cudnn):
    from michigan_b200 import precision
    from michigan_b200.networks import StyleContentLoss
    from michigan_b200.options import make_opt
    sd = _vgg_sd()
    fake, ref, tag, _ = _images(2, size)
    old = precision.mode()
    precision.set_mode(mode)
    try:
        crit = StyleContentLoss(make_opt(), state_dict=sd)
        got = []
        for i in range(2):
            x = fake.cuda().requires_grad_()
            lc, ls = crit(x, ref.cuda(), tag.cuda())
            (lc, ls)[i].backward()
            got.append((float(lc), float(ls), x.grad.clone()))
        torch.cuda.synchronize()
    finally:
        precision.set_mode(old)
    sdc = {k: v.cuda() for k, v in sd.items()}
    for i, name in enumerate(("content", "style")):
        xr = fake.cuda().requires_grad_()
        want = osc.style_content_loss(xr, ref.cuda(), tag.cuda(), sdc)[i]
        want.backward()
        rel = abs(got[i][i] - float(want)) / abs(float(want))
        cos, grel = _cos(got[i][2], xr.grad), _rel(got[i][2], xr.grad)
        print("%s %d^2 %s: loss %.7f oracle %.7f rel %.2e; d fake cosine %.6f rel L2 %.3e"
              % (name, size, mode, got[i][i], float(want), rel, cos, grel))
        assert torch.isfinite(got[i][2]).all()
        assert rel <= 1e-3
        assert cos >= 0.98


def test_combined_vs_separate_calls(fp32_cudnn):
    """One _VGGObjectiveFn call (VGG L1 + content + style, one VGG19 pass) against VGGLoss and StyleContentLoss called
    separately (two passes, the install() shape) on the same VGG19: same loss values, d fake of the summed objective."""
    from michigan_b200.networks import StyleContentLoss, VGGLoss
    from michigan_b200.networks.loss import vgg_objective
    from michigan_b200.options import make_opt
    sd = _vgg_sd()
    vggl = VGGLoss(make_opt(), state_dict=sd)
    sc = StyleContentLoss(make_opt(), vgg=vggl.vgg)
    fake, ref, tag, _ = _images(2, 128)
    x = fake.cuda().requires_grad_()
    l1, lc, ls = vgg_objective(vggl.vgg, x, tag.cuda(), ref.cuda(), l1=True, content=True, style=True)
    (l1 + lc + ls).backward()
    y = fake.cuda().requires_grad_()
    s1 = vggl(y, tag.cuda())
    sc_c, sc_s = sc(y, ref.cuda(), tag.cuda())
    (s1 + sc_c + sc_s).backward()
    torch.cuda.synchronize()
    rels = [abs(float(a) - float(b)) / abs(float(b)) for a, b in ((l1, s1), (lc, sc_c), (ls, sc_s))]
    grel = _rel(x.grad, y.grad)
    print("combined vs separate: loss rel (VGG, content, style) %.2e %.2e %.2e; d fake rel L2 %.3e" % (*rels, grel))
    assert max(rels) <= 1e-6
    assert grel <= 2e-2


def test_style_image_equal_to_tag_takes_the_2n_path():
    """ref == tag (same tensor, or equal values) runs VGG19 on 2N images; the result equals the 3N run with the tag passed as the
    style image."""
    from michigan_b200.networks import StyleContentLoss
    from michigan_b200.networks.loss import _VGGObjectiveFn
    from michigan_b200.options import make_opt
    crit = StyleContentLoss(make_opt(), state_dict=_vgg_sd())
    fake, _, tag, _ = _images(2, 64)
    tag = tag.cuda()
    seen = []
    orig = crit.vgg.run

    def run(x8, n_save=0):
        seen.append(x8.shape[0])
        return orig(x8, n_save)
    crit.vgg.run = run
    res = []
    for style in (tag, tag.clone()):
        x = fake.cuda().requires_grad_()
        lc, ls = crit(x, style, tag)
        (lc + ls).backward()
        res.append((float(lc), float(ls), x.grad.clone()))
    x = fake.cuda().requires_grad_()
    _, lc, ls = _VGGObjectiveFn.apply(crit.vgg, None, (False, True, True), x, tag, tag.clone())
    (lc + ls).backward()
    torch.cuda.synchronize()
    assert seen == [4, 4, 6]
    assert res[0][0] == res[1][0] and res[0][1] == res[1][1] and torch.equal(res[0][2], res[1][2])
    rel = max(abs(res[0][0] - float(lc)) / abs(float(lc)), abs(res[0][1] - float(ls)) / abs(float(ls)))
    grel = _rel(res[0][2], x.grad)
    print("2N vs 3N with style = tag: loss rel %.2e; d fake rel L2 %.3e" % (rel, grel))
    assert rel <= 1e-6 and grel <= 1e-5


@pytest.mark.parametrize("ref_is_tag", [True, False])
def test_generator_step_default_losses_vs_oracle(tmp_path, ref_is_tag):
    """One generator step of Pix2PixModel with the reference's default loss set at the golden configuration (ngf 64, 128x128,
    batch 2) against compute_generator_loss_default: every loss within 1e-2 relative, per-tensor G-gradient cosine >= 0.998.
    ref_is_tag False: image_ref differs from image_tag but the labels are equal, so every term is on and style runs on 3N."""
    import michigan_oracle as orc
    from helpers import load_golden, preprocessed, reference_layout_state, summary
    from michigan_b200.networks.architecture import VGG19_WEIGHTS_FILE
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel
    from michigan_b200.synth import synthetic_batch
    z, cfg = load_golden()
    sd_vgg = _vgg_sd()
    os.makedirs(tmp_path / "checkpoints")
    torch.save(sd_vgg, tmp_path / "checkpoints" / VGG19_WEIGHTS_FILE)
    old_hub = torch.hub.get_dir()
    torch.hub.set_dir(str(tmp_path))
    try:
        opt = make_opt(is_train=True, ngf=cfg["ngf"], ndf=cfg["ndf"], crop_size=cfg["size"], batchSize=cfg["batch"], no_vgg_loss=False,
                       no_style_loss=False, no_content_loss=False, no_background_loss=False, no_rgb_loss=False, no_lab_loss=False,
                       no_orient_loss=False, no_confidence_loss=False)
        model = Pix2PixModel(opt)
    finally:
        torch.hub.set_dir(old_hub)
    sdG = reference_layout_state("G", cfg, cfg["seed_G"])
    sdD = reference_layout_state("D", cfg, cfg["seed_D"])
    model.netG.load_state_dict(sdG)
    model.netD.load_state_dict(sdD)
    model.train()
    data = synthetic_batch(cfg["batch"], cfg["size"], cfg["data_seed"])
    _, pre = preprocessed(cfg)
    if not ref_is_tag:
        data["image_ref"] = data["image_tag"].flip(-1).contiguous()
        pre["image_ref"] = data["image_ref"]
    random.seed(cfg["py_seed"])
    th = int(cfg["size"] * 0.05); th = th if th % 2 == 1 else th + 1
    k = random.choice([max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4])
    random.seed(cfg["py_seed"])
    g_losses, _ = model(dict(data), mode="generator")
    sum(v.mean() for v in g_losses.values()).backward()
    torch.cuda.synchronize()
    assert list(g_losses) == ["GAN", "GAN_Feat", "VGG", "content", "style", "background", "rgb", "lab", "ORIENT", "CONFIDENCE"]

    oopt = orc.default_opt(ngf=cfg["ngf"], ndf=cfg["ndf"], crop_size=cfg["size"], isTrain=True)
    names = [n for n in sdG if not n.endswith(("running_mean", "running_var", "num_batches_tracked", "weight_u", "weight_v"))]
    for n in names:
        sdG[n].requires_grad_(True)
    losses_o, _ = osc.compute_generator_loss_default(sdG, sdD, sd_vgg, oopt, pre, rng_k=k)
    orc.trainer_loss(losses_o).backward()
    assert list(losses_o) == list(g_losses)
    for key in g_losses:
        a, b = float(g_losses[key].mean()), float(losses_o[key].mean())
        print("   %-10s %.6f  oracle %.6f  rel %.2e" % (key, a, b, abs(a - b) / max(abs(b), 1e-30)))
        if key in ("content", "style", "background", "rgb"):
            assert abs(a - b) <= 2e-4 * abs(b), key
        else:                                   # the terms of test_generator_step_readme_losses_vs_oracle, its bound
            assert abs(a - b) <= 1e-2 * max(1.0, abs(b)), key
    named = dict(model.netG.named_parameters())
    worst = 1.0
    for key in z.files:
        if key.startswith("g_grad/") and not key.endswith("conv_0.bias"):
            n = key[len("g_grad/"):]
            a, b = summary(named[n].grad, stride=101)[4:], summary(sdG[n].grad, stride=101)[4:]
            cos = float(np.dot(a.astype(np.float64), b) / (np.linalg.norm(a) * np.linalg.norm(b)))
            worst = min(worst, cos)
    print("   worst per-tensor G-gradient cosine %.5f" % worst)
    assert worst >= 0.998, worst

