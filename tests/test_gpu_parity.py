"""Parity of the CUDA path (through the C ABI) against the CPU oracle and the reference's golden
fixtures.  Tolerances: tensor-core convs read TF32 operands (10-bit mantissa, RN-rounded by the
producer) with fp32 accumulation, so feature maps are compared at 5e-3 of their abs-max and the
generator image against BASELINE.json's bound: max-abs <= 1e-3 (mean-abs reported, must be <= 2e-4)."""
import os
import random

import numpy as np
import pytest
import torch

import michigan_oracle as orc
from helpers import assert_summary_close, load_golden, max_mean_abs, preprocessed, reference_layout_state

pytestmark = pytest.mark.gpu

MAX_ABS = 1e-3
MEAN_ABS = 2e-4


def _cuda(d):
    return {k: v.cuda() for k, v in d.items()}


def _build_G(cfg, is_train, sd=None, **kw):
    from michigan_b200 import networks
    from michigan_b200.options import make_opt
    opt = make_opt(is_train=is_train, ngf=cfg["ngf"], ndf=cfg["ndf"], crop_size=cfg["size"], **kw)
    G = networks.SPADEBGenerator(opt)
    if sd is not None:
        missing = G.load_state_dict(sd, strict=True)
    return G.cuda(), opt


def _run_G(G, pre):
    p = _cuda(pre)
    with torch.no_grad():
        return G(p["input_ref"], orient_mask=p["orient_mask"], image_ref=p["image_ref"], input_tag=p["input_tag"],
                 noise=p["noise"], image_tag=p["image_tag"])


def test_generator_train_mode_vs_golden_and_oracle():
    z, cfg = load_golden()
    sd = reference_layout_state("G", cfg, cfg["seed_G"])
    G, opt = _build_G(cfg, True, sd)
    G.train()
    G.collect_taps = True
    _, pre = preprocessed(cfg)
    random.seed(cfg["py_seed"])  # the reference draws the dilation size with Python's `random` (encoder.py:294)
    out = _run_G(G, pre)
    torch.cuda.synchronize()
    ref = torch.from_numpy(z["g_train_out"])
    mx, mn = max_mean_abs(out, ref)
    print("G train-mode vs reference fixture: max-abs %.3e mean-abs %.3e" % (mx, mn))
    for name, t in G.last_taps.items():
        rel = assert_summary_close("tap " + name, t.permute(0, 3, 1, 2).contiguous(), z["tap/" + name], 5e-3)
        print("   tap %-12s rel err %.2e" % (name, rel))
    assert mx <= MAX_ABS and mn <= MEAN_ABS, (mx, mn)
    # side effects of a train-mode forward: running statistics and spectral-norm u, v
    got = G.state_dict()
    for k in z.files:
        if k.startswith("g_post/"):
            name = k[len("g_post/"):]
            r = torch.from_numpy(z[k])
            tol = 2e-3 if name.endswith(("running_mean", "running_var")) else 1e-4
            err = (got[name].cpu() - r).abs().max().item()
            assert err <= tol * max(1.0, r.abs().max().item()), (name, err)
    assert all(int(v) == 0 for k, v in got.items() if k.endswith("num_batches_tracked"))


def test_generator_training_forward_image_vs_golden():
    """The image returned by the TRAINING forward (grad enabled: the autograd Function that `mode='generator'` runs,
    pix2pix_model.py:505-541) against the reference's train-mode output, at the same bound as the no-grad forward:
    max-abs <= 1e-3, mean-abs <= 2e-4.  Both modes share one forward implementation and one operand policy."""
    z, cfg = load_golden()
    sd = reference_layout_state("G", cfg, cfg["seed_G"])
    G, opt = _build_G(cfg, True, sd)
    G.train()
    _, pre = preprocessed(cfg)
    p = _cuda(pre)
    random.seed(cfg["py_seed"])
    out = G(p["input_ref"], orient_mask=p["orient_mask"], image_ref=p["image_ref"], input_tag=p["input_tag"], noise=p["noise"],
            image_tag=p["image_tag"])
    assert out.requires_grad and out.grad_fn is not None
    mx, mn = max_mean_abs(out, torch.from_numpy(z["g_train_out"]))
    print("G TRAINING forward (autograd) vs reference fixture: max-abs %.3e mean-abs %.3e" % (mx, mn))
    assert mx <= MAX_ABS and mn <= MEAN_ABS, (mx, mn)
    # same kernels and operand formats as the no-grad forward from the same state; the only difference is the epilogue
    # variant of the gamma|beta GEMM (generic, also storing fp32 h and 1+gamma, vs the specialised bf16-only one), whose
    # fused multiply-adds are ordered differently: agreement to ~1e-5, two orders below the bound
    G2, _ = _build_G(cfg, True, sd)
    G2.train()
    random.seed(cfg["py_seed"])
    out2 = _run_G(G2, pre)
    d = (out.detach() - out2).abs().max().item()
    print("   training forward vs no-grad forward: max diff %.2e" % d)
    assert d <= 5e-5
    got = G.state_dict()
    for k in z.files:
        if k.startswith("g_post/"):
            name = k[len("g_post/"):]
            r = torch.from_numpy(z[k])
            tol = 2e-3 if name.endswith(("running_mean", "running_var")) else 1e-4
            assert (got[name].cpu() - r).abs().max().item() <= tol * max(1.0, r.abs().max().item()), name


def test_generator_eval_mode_vs_golden():
    z, cfg = load_golden()
    sd = reference_layout_state("G", cfg, cfg["seed_G"])
    for k in z.files:
        if k.startswith("g_post/"):
            sd[k[len("g_post/"):]] = torch.from_numpy(z[k]).clone()
    G, opt = _build_G(cfg, False, sd)
    G.eval()
    before = {k: v.clone() for k, v in G.state_dict().items()}
    _, pre = preprocessed(cfg)
    out = _run_G(G, pre)
    mx, mn = max_mean_abs(out, torch.from_numpy(z["g_eval_out"]))
    print("G eval-mode vs reference fixture: max-abs %.3e mean-abs %.3e" % (mx, mn))
    assert mx <= MAX_ABS and mn <= MEAN_ABS, (mx, mn)
    after = G.state_dict()
    assert all(torch.equal(before[k], after[k]) for k in before), "eval forward must not modify state"
    # repeatability: same inputs -> same result up to atomics ordering in the instance-norm statistics
    assert (out - _run_G(G, pre)).abs().max().item() <= 2e-6


def test_discriminator_vs_golden():
    from michigan_b200 import networks
    from michigan_b200.options import make_opt
    z, cfg = load_golden()
    sd = reference_layout_state("D", cfg, cfg["seed_D"])
    oopt = orc.default_opt(ngf=cfg["ngf"], ndf=cfg["ndf"], crop_size=cfg["size"])
    _, pre = preprocessed(cfg)
    fake = torch.from_numpy(z["g_train_out"])
    o = orc.orient_channels(pre["orient_mask"], pre["input_tag"][:, 1:2], oopt)
    x = torch.cat([torch.cat([pre["input_tag"], o, fake], 1), torch.cat([pre["input_tag"], o, pre["image_tag"]], 1)], 0)
    D = networks.MultiscaleDiscriminator(make_opt(ngf=cfg["ngf"], ndf=cfg["ndf"], crop_size=cfg["size"]))
    D.load_state_dict(sd, strict=True)
    D = D.cuda().train()
    with torch.no_grad():
        out = D(x.cuda())
    assert len(out) == 2 and all(len(o_) == 5 for o_ in out)
    for i in range(2):
        for j in range(5):
            t = out[i][j]
            assert t.shape[1] == (1 if j == 4 else min(cfg["ndf"] * 2 ** j, 512))
            if j == 4:
                r = torch.from_numpy(z["d/%d/4" % i])
                mx, mn = max_mean_abs(t, r)
                print("D[%d] logits max-abs %.3e (ref max %.2f)" % (i, mx, r.abs().max()))
                assert mx <= 5e-3 * r.abs().max().item()
            else:
                assert_summary_close("D[%d][%d]" % (i, j), t.contiguous(), z["d/%d/%d" % (i, j)], 5e-3)
    got = D.state_dict()
    for k in z.files:
        if k.startswith("d_post/"):
            r = torch.from_numpy(z[k])
            assert (got[k[len("d_post/"):]].cpu() - r).abs().max().item() <= 1e-4


def test_generator_full_size_vs_oracle():
    """BASELINE config shape (ngf 64, 512x512) at batch 1 against the oracle run on the host CPU."""
    cfg = dict(ngf=64, ndf=64, size=512, batch=1, data_seed=3)
    sd = reference_layout_state("G", cfg, 21)
    G, opt = _build_G(cfg, True, sd)
    G.train()
    _, pre = preprocessed(cfg)
    random.seed(9)
    th = int(512 * 0.05); th = th if th % 2 == 1 else th + 1
    k = random.choice([max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4])
    random.seed(9)
    out = _run_G(G, pre)
    oopt = orc.default_opt(isTrain=True)
    with torch.no_grad():
        ref = orc.generate_fake(sd, oopt, pre, True, rng_k=k)
    mx, mn = max_mean_abs(out, ref)
    print("G 512x512 ngf64 vs oracle: max-abs %.3e mean-abs %.3e (output std %.3f)" % (mx, mn, ref.std().item()))
    assert mx <= MAX_ABS and mn <= MEAN_ABS, (mx, mn)


def test_generator_batch8_train_mode_vs_oracle():
    """BASELINE.json configs[1]/[2] shape exactly: batch 8, 512x512, ngf 64, TRAIN-mode batch statistics over the 8
    samples, against the oracle on the host CPU (~25 s)."""
    cfg = dict(ngf=64, ndf=64, size=512, batch=8, data_seed=7)
    sd = reference_layout_state("G", cfg, 23)
    G, opt = _build_G(cfg, True, sd, batchSize=8)
    G.train()
    _, pre = preprocessed(cfg)
    g = torch.Generator().manual_seed(2)
    pre["image_ref"] = torch.rand(8, 3, 512, 512, generator=g) * 2 - 1     # a different image per sample
    pre["image_tag"] = pre["image_ref"].clone()
    random.seed(11)
    th = int(512 * 0.05); th = th if th % 2 == 1 else th + 1
    k = random.choice([max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4])
    random.seed(11)
    out = _run_G(G, pre)
    with torch.no_grad():
        ref = orc.generate_fake(sd, orc.default_opt(isTrain=True), pre, True, rng_k=k)
    mx, mn = max_mean_abs(out, ref)
    print("G batch 8 x 512x512 train-mode vs oracle: max-abs %.3e mean-abs %.3e (output std %.3f)" % (mx, mn, ref.std().item()))
    assert mx <= MAX_ABS and mn <= MEAN_ABS, (mx, mn)


def test_generator_add_feat_zeros_576_eval_vs_oracle():
    """BASELINE.json configs[0]'s geometry: inference with --add_feat_zeros => every input zero-padded by add_th/2 = 32
    on each side (pix2pix_model.py:240-254), the generator runs at 576x576 with a 9x9 latent (generator.py:79-96), and the
    eval-mode background mask dilates only inside the original window (encoder.py:301-314)."""
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel
    from michigan_b200.synth import synthetic_batch
    cfg = dict(ngf=64, ndf=64, size=512, batch=1, data_seed=13)
    sd = reference_layout_state("G", dict(cfg, size=512), 24)
    # Running statistics of a trained checkpoint describe the data it is used on; fill_state_dict leaves mean 0 / var 1,
    # and statistics from a different geometry make |x_hat| large (eval-mode BN does not re-normalise), which amplifies the
    # operand rounding of the gamma/beta GEMMs beyond anything a real checkpoint sees (measured: statistics of ONE other image -
    # 81 samples per channel in head_0 - leave a 2e-3 tail while the mean error stays at 1.4e-5).  So: one train-mode oracle
    # pass over FOUR other images of the same zero-padded 576x576 geometry, momentum 1, writes its batch statistics into sd.
    _, pre_cal = preprocessed(dict(cfg, data_seed=14, batch=4))
    g = torch.Generator().manual_seed(77)
    pre_cal["image_ref"] = torch.rand(4, 3, 512, 512, generator=g) * 2 - 1
    pre_cal["image_tag"] = pre_cal["image_ref"].clone()
    pre_cal["noise"] = torch.rand(4, 3, 512, 512, generator=g)
    with torch.no_grad():
        orc.generate_fake(sd, orc.default_opt(isTrain=True, add_feat_zeros=True), pre_cal, True, rng_k=5, momentum=1.0)
    assert float(sd["up_3.norm_0.param_free_norm.running_var"].mean()) != 1.0
    opt = make_opt(is_train=False, ngf=64, ndf=64, crop_size=512, add_feat_zeros=True, batchSize=1)
    model = Pix2PixModel(opt)
    assert (model.netG.sw, model.netG.sh) == (9, 9)
    model.netG.load_state_dict(sd, strict=True)
    model.eval()
    data = synthetic_batch(1, 512, 13)
    out = model(dict(data), mode="inference")
    assert tuple(out.shape) == (1, 3, 576, 576)
    _, pre = preprocessed(cfg)
    oopt = orc.default_opt(isTrain=False, add_feat_zeros=True)
    with torch.no_grad():
        ref = orc.generate_fake(sd, oopt, pre, False)
    mx, mn = max_mean_abs(out, ref)
    d = (out.cpu() - ref).abs()
    iy, ix = divmod(int(d[0].max(dim=0)[0].argmax()), 576)
    print("G 576x576 (--add_feat_zeros) eval vs oracle: max-abs %.3e mean-abs %.3e (at y=%d x=%d; inside the 512 window: %.3e; "
          "99.99th percentile %.3e)" % (mx, mn, iy, ix, float(d[..., 32:544, 32:544].max()), float(d.flatten().kthvalue(int(d.numel() * 0.9999))[0])))
    assert mx <= MAX_ABS and mn <= MEAN_ABS, (mx, mn)


def test_eval_batch_independence_at_benchmark_size():
    """Size-independent property at the BASELINE batch (N=8, 512x512): in eval mode every op is
    per-sample, so the batched result equals the per-image results (up to the summation order of the
    instance-norm statistics, whose fp64 partial sums are combined with atomics: <= 2e-5)."""
    cfg = dict(ngf=64, ndf=64, size=512, batch=8, data_seed=5)
    sd = reference_layout_state("G", cfg, 22)
    G, opt = _build_G(cfg, False, sd)
    G.eval()
    data, pre = preprocessed(cfg)
    # different image per sample so that samples are distinguishable
    g = torch.Generator().manual_seed(1)
    pre["image_ref"] = torch.rand(8, 3, 512, 512, generator=g) * 2 - 1
    pre["image_tag"] = pre["image_ref"].clone()
    out = _run_G(G, pre)
    for i in (0, 5):
        one = {k: v[i:i + 1].contiguous() for k, v in pre.items()}
        d = (out[i:i + 1] - _run_G(G, one)).abs().max().item()
        print("batched vs single, sample %d: max diff %.2e" % (i, d))
        assert d <= 2e-5, "sample %d differs between batched and single run: %g" % (i, d)
    assert torch.isfinite(out).all() and out.abs().max() <= 1.0


def _rel_l2(got_summary, ref_summary):
    a, b = got_summary[4:].astype(np.float64), ref_summary[4:].astype(np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-12))


def _cosine(got_summary, ref_summary):
    a, b = got_summary[4:].astype(np.float64), ref_summary[4:].astype(np.float64)
    return float(a @ b / max(np.linalg.norm(a) * np.linalg.norm(b), 1e-30))


def test_backward_chain_smooth_loss_vs_oracle():
    """Whole backward chain (generator -> discriminator) with a SMOOTH loss, against torch autograd on the
    CPU oracle: L = sum over the 10 discriminator outputs of mean(out^2).  Every parameter gradient of G and
    D is compared in relative L2.  Bound: 0.1 (measured <= 4e-2; round 1: 0.2).  The forward runs with TF32 operands (features accurate to
    ~5e-4), and LeakyReLU / ReLU derivatives jump at 0, so ~0.05 % of the activation-derivative masks differ
    from the fp32 oracle per layer: measured ~2e-2 per discriminator layer, ~1e-2 per SPADE block, compounding
    to ~0.12 at the reference encoder (7 blocks upstream).  Each backward stage on its own (every SPADE block, the
    encoders, the discriminator scales) is held to float64 autograd element by element, at the forward's own activation
    masks, by tests/test_gpu_backward_stages_fp64.py.  Tensors whose reference
    norm is below 1e-4 (1e-2 for 1-D sums) of the largest are measured against that floor."""
    from michigan_b200 import networks
    from michigan_b200.options import make_opt
    cfg = dict(ngf=64, ndf=64, size=128, batch=2, data_seed=9)
    sdG = reference_layout_state("G", cfg, 31)
    sdD = reference_layout_state("D", cfg, 32)
    _, pre = preprocessed(cfg)
    opt = make_opt(is_train=True, ngf=64, ndf=64, crop_size=128)
    G = networks.SPADEBGenerator(opt); G.load_state_dict(sdG); G = G.cuda().train()
    D = networks.MultiscaleDiscriminator(opt); D.load_state_dict(sdD); D = D.cuda().train()
    p = _cuda(pre)
    random.seed(4)
    th = int(128 * 0.05); th = th if th % 2 == 1 else th + 1
    k = random.choice([max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4])
    random.seed(4)
    fake = G(p["input_ref"], orient_mask=p["orient_mask"], image_ref=p["image_ref"], input_tag=p["input_tag"], noise=p["noise"],
             image_tag=p["image_tag"])
    oopt = orc.default_opt(ngf=64, ndf=64, crop_size=128, isTrain=True)
    cond = torch.cat([p["input_tag"], orc.orient_channels(pre["orient_mask"], pre["input_tag"][:, 1:2], oopt).cuda()], 1)
    x = torch.cat([torch.cat([cond, fake], 1), torch.cat([cond, p["image_tag"]], 1)], 0)
    outs = D(x)
    loss = sum((t * t).mean() for o_ in outs for t in o_)
    loss.backward()
    torch.cuda.synchronize()
    # oracle
    names_G = [n for n, _ in G.named_parameters()]
    names_D = [n for n, _ in D.named_parameters()]
    for n in names_G:
        sdG[n].requires_grad_(True)
    for n in names_D:
        sdD[n].requires_grad_(True)
    fake_o = orc.generate_fake(sdG, oopt, pre, True, rng_k=k)
    cond_o = torch.cat([pre["input_tag"], orc.orient_channels(pre["orient_mask"], pre["input_tag"][:, 1:2], oopt)], 1)
    x_o = torch.cat([torch.cat([cond_o, fake_o], 1), torch.cat([cond_o, pre["image_tag"]], 1)], 0)
    outs_o = orc.multiscale_discriminator(x_o, sdD, oopt, True)
    loss_o = sum((t * t).mean() for o_ in outs_o for t in o_)
    loss_o.backward()
    print("smooth loss: cuda %.6f oracle %.6f" % (float(loss), float(loss_o)))
    assert abs(float(loss) - float(loss_o)) <= 2e-3 * abs(float(loss_o))
    failures = []
    for label, net, sd, names in (("G", G, sdG, names_G), ("D", D, sdD, names_D)):
        named = dict(net.named_parameters())
        gmax = max(sd[n].grad.norm().item() for n in names if sd[n].grad is not None)
        rows = []
        for n in names:
            ref = sd[n].grad
            got = named[n].grad
            if ref is None:
                assert got is None or float(got.abs().max()) == 0.0, n
                continue
            assert got is not None, n
            # 1-D tensors (biases) are sums with heavy cancellation: floor their scale at 1 % of the largest gradient
            floor = (1e-2 if ref.dim() == 1 else 1e-4) * gmax
            rows.append(((got.cpu() - ref).norm().item() / max(ref.norm().item(), floor), n, ref.norm().item()))
        rows.sort(reverse=True)
        print("   %s: largest relative L2 gradient errors (gmax %.3e):" % (label, gmax))
        for e, n, rn in rows[:6]:
            print("      %-50s err %.3e  |ref| %.3e" % (n, e, rn))
        failures += [(label, n, e) for e, n, rn in rows if e > 0.1]
    assert not failures, failures[:10]


def test_train_iteration_losses_and_grads_vs_golden():
    """One generator step and one discriminator step through the hand-written backward (TF32 gradient
    GEMMs) against the reference trainer's losses and gradients stored in the golden fixture.
    Tolerances: losses 1e-2 relative (measured 5e-6); per-tensor gradient cosine similarity >= 0.998 on the stored
    strided samples (measured >= 0.9991 for G, >= 0.9995 for D; round 1: 0.98).  The hinge and L1 feature-matching losses are piecewise linear: a feature computed with an
    11-bit significand flips sign(f_fake - f_real) for ~0.1 % of the elements, which alone moves the
    gradient by several % in relative L2, so an exact-arithmetic bound is checked separately with a smooth
    loss in test_backward_chain_smooth_loss_vs_oracle."""
    from helpers import summary
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel
    from michigan_b200.synth import synthetic_batch
    z, cfg = load_golden()
    torch.manual_seed(0)
    opt = make_opt(is_train=True, ngf=cfg["ngf"], ndf=cfg["ndf"], crop_size=cfg["size"], batchSize=cfg["batch"])
    model = Pix2PixModel(opt)
    model.netG.load_state_dict(reference_layout_state("G", cfg, cfg["seed_G"]))
    model.netD.load_state_dict(reference_layout_state("D", cfg, cfg["seed_D"]))
    model.train()
    opt_G, opt_D = model.create_optimizers(opt)
    data = synthetic_batch(cfg["batch"], cfg["size"], cfg["data_seed"])

    random.seed(cfg["py_seed"])
    opt_G.zero_grad()
    g_losses, fake = model(dict(data), mode="generator")
    sum(g_losses.values()).mean().backward()
    torch.cuda.synchronize()
    got = [float(g_losses["GAN"].mean()), float(g_losses["GAN_Feat"].mean())]
    print("G losses", got, "reference", z["g_losses"].tolist())
    for a, b in zip(got, z["g_losses"]):
        assert abs(a - b) <= 1e-2 * max(1.0, abs(b)), (got, z["g_losses"])
    named = dict(model.netG.named_parameters())
    worst = 1.0
    for k in z.files:
        if k.startswith("g_grad/") and not k.endswith("conv_0.bias"):   # bias before a batch-norm: gradient is exactly 0
            p = named[k[len("g_grad/"):]]
            assert p.grad is not None, k
            cos = _cosine(summary(p.grad, stride=101), z[k])
            print("   %-45s cosine %.4f  rel L2 %.3e" % (k, cos, _rel_l2(summary(p.grad, stride=101), z[k])))
            worst = min(worst, cos)
    assert worst >= 0.998, worst
    assert named["backgroud_enc.layer4.conv.weight"].grad is None
    opt_G.step()

    # discriminator step from the INITIAL weights (decoupled from the generator's Adam update)
    model.netG.load_state_dict(reference_layout_state("G", cfg, cfg["seed_G"]))
    model.netD.load_state_dict(reference_layout_state("D", cfg, cfg["seed_D"]))
    random.seed(cfg["py_seed"] + 2)
    opt_D.zero_grad()
    d_losses = model(dict(data), mode="discriminator")
    sum(d_losses.values()).mean().backward()
    torch.cuda.synchronize()
    got = [float(d_losses["D_Fake"].mean()), float(d_losses["D_real"].mean())]
    print("D losses", got, "reference", z["d0_losses"].tolist())
    for a, b in zip(got, z["d0_losses"]):
        assert abs(a - b) <= 1e-2 * max(1.0, abs(b)), (got, z["d0_losses"])
    namedD = dict(model.netD.named_parameters())
    worst = 1.0
    for k in z.files:
        if k.startswith("d0_grad/"):
            cos = _cosine(summary(namedD[k[len("d0_grad/"):]].grad, stride=53), z[k])
            print("   %-45s cosine %.4f" % (k, cos))
            worst = min(worst, cos)
    assert worst >= 0.998, worst
    opt_D.step()


def test_inpaint_generator_vs_oracle():
    """InpaintGenerator (generator.py:490-575) composed from the main path's kernels vs the CPU oracle on identical
    deterministic weights; output in [0, 1], tolerance 1e-3 max-abs like the generator image."""
    from michigan_b200.networks.inpaint import InpaintGenerator
    from michigan_b200.synth import fill_state_dict
    net = InpaintGenerator()
    fill_state_dict(net.state_dict(), 21)
    g = torch.Generator().manual_seed(5)
    x = torch.rand(2, 4, 128, 128, generator=g)
    with torch.no_grad():
        ref = orc.inpaint_generator(x, {k: v.clone() for k, v in net.state_dict().items()})
    out = net.cuda()(x.cuda()).cpu()
    mx, mn = max_mean_abs(out, ref)
    print("InpaintGenerator vs oracle: max-abs %.3e mean-abs %.3e" % (mx, mn))
    assert mx <= MAX_ABS


def test_use_ig_train_iteration_vs_oracle_orientation_input(tmp_path):
    """BASELINE.json configs[4]'s model path: --use_ig.  The 2-channel orientation input the generator receives
    (Pix2PixModel.inpainting_orient, pix2pix_model.py:407-429: nearest 512->256, frozen InpaintGenerator, nearest back,
    hole blend, channel swap, hair mask) against the oracle, then one full train iteration with the orientation /
    confidence losses switched on (finite losses, gradients for every generator parameter)."""
    from michigan_b200.networks import InpaintGenerator
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel, train_iteration
    from michigan_b200.synth import fill_state_dict, synthetic_batch
    os.makedirs(tmp_path / "ig")
    ig = InpaintGenerator()
    fill_state_dict(ig.state_dict(), 2)
    sd_ig = {k: v.clone() for k, v in ig.state_dict().items()}
    torch.save({"generator": sd_ig}, tmp_path / "ig" / "InpaintingModel_gen.pth")
    opt = make_opt(is_train=True, ngf=64, ndf=64, crop_size=512, batchSize=2, use_ig=True, checkpoints_dir=str(tmp_path), name="ig",
                   ig_model_name="InpaintingModel_gen.pth", netIG="inpaint", no_orient_loss=False, no_confidence_loss=False)
    model = Pix2PixModel(opt).train()
    assert not model.netIG.training
    data = synthetic_batch(2, 512, 3, use_ig=True)
    hair = data["label_tag"]
    with torch.no_grad():
        _, o2 = model.inpainting_orient(data["hole"].cuda(), data["orient_rgb"].cuda(), data["noise"].cuda(), hair.cuda())
        _, o2_ref = orc.inpainting_orient(sd_ig, 512, data["hole"], data["orient_rgb"], data["noise"], hair)
    mx, mn = max_mean_abs(o2, o2_ref)
    print("inpainting_orient (2-channel orientation input) vs oracle: max-abs %.3e mean-abs %.3e" % (mx, mn))
    assert mx <= 2e-3           # (out - 0.5) * 2 doubles the InpaintGenerator's 1e-3 bound
    optG, optD = model.create_optimizers(opt)
    random.seed(0)
    g, d, img = train_iteration(model, optG, optD, dict(data))
    vals = {k: float(v.detach().mean()) for k, v in {**g, **d}.items()}
    print("use_ig train iteration losses:", vals)
    assert set(g) == {"GAN", "GAN_Feat", "ORIENT", "CONFIDENCE"} and all(np.isfinite(v) for v in vals.values())
    assert all(torch.isfinite(p).all() for p in model.netG.parameters())
