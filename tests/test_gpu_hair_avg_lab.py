"""The hair-average Lab loss of the unpaired stage on the sm_90a kernels (csrc/mg_vgg.cu: mg_hair_avg_lab_fwd / _bwd).

Kernels against float64 autograd, element by element:

    |got - ref| <= k * u * R_abs + tiny,   u = 2^-24

The kernels evaluate Lab per pixel in fp32 and sum in fp64, so R_abs is the sum behind each result of the magnitudes of the
terms whose rounding it inherits: for sum m a, sum 500 (|f(X)| + |f(Y)|) |m| (a is a difference of two f values; b, L likewise);
for d fake, the same chain rule as the gradient with every factor replaced by its magnitude.  The loss inherits its averages'
R_abs / cnt.  Measured on an H100 (|err| / (u R_abs), the four cases): sums 0.10-0.11, loss <= 0.01, d fake 3.0-4.6;
bounds K_SUMS = 1, K_GRAD = 8.  The module is also held to the reference's own outputs (tests/golden/golden_hair_avg_lab.npz)
and one generator step of the unpaired stage (curr_step 2) to tests/oracle_unpaired.py."""
import os
import random

import numpy as np
import pytest
import torch

import oracle_unpaired as ou

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
K_SUMS = 1
K_GRAD = 8
_M = [[0.412453, 0.357580, 0.180423], [0.212671, 0.715160, 0.072169], [0.019334, 0.119193, 0.950227]]
TH = 0.008856


def _case(n, h, w, kind, seed=5):
    """Images in (-1, 1) with a few saturated pixels; binary hair masks.  kind 'mixed': image 0 random masks, image 1 (if any) no
    tag hair, image 2 (if any) full tag hair and no reference hair; 'frac': fractional masks."""
    g = torch.Generator().manual_seed(seed)
    fake = torch.rand(n, 3, h, w, generator=g) * 2 - 1
    real = torch.rand(n, 3, h, w, generator=g) * 2 - 1
    fake[:, :, 0, :3] = -1.0                                       # X = Y = Z = 0: the linear branch and its slope
    if kind == "frac":
        mf, mr = torch.rand(n, 1, h, w, generator=g), torch.rand(n, 1, h, w, generator=g)
    else:
        mf = (torch.rand(n, 1, h, w, generator=g) > 0.6).float()
        mr = (torch.rand(n, 1, h, w, generator=g) > 0.5).float()
        if n > 1:
            mf[1] = 0
        if n > 2:
            mf[2] = 1
            mr[2] = 0
    return fake, real, mf, mr


def _lab64(img):
    """-> (xyz, f(xyz), L, a, b) in float64 from fp32 images, the M of the kernels (fp32 values, fp32 row sums)."""
    M = torch.tensor(_M, dtype=torch.float32)
    rs = ((M[:, 0] + M[:, 1]) + M[:, 2]).double()
    rgb = (img.double() + 1) / 2
    xyz = torch.einsum("kc,nchw->nkhw", M.double(), rgb) / rs.view(1, 3, 1, 1)
    f = torch.where(xyz > TH, xyz.clamp(min=TH).pow(1 / 3), 7.787 * xyz + 0.137931)
    y = xyz[:, 1]
    L = torch.where(y > TH, 116 * f[:, 1] - 16, 903.3 * y)
    return xyz, f, L, 500 * (f[:, 0] - f[:, 1]), 200 * (f[:, 1] - f[:, 2])


def _sums64(img, m):
    """-> ([N,4] sums m L, m a, m b, m;  [N,4] their R_abs)."""
    xyz, f, L, a, b = _lab64(img)
    m = m[:, 0].double()
    am = m.abs()
    s = torch.stack([(L * m).sum((1, 2)), (a * m).sum((1, 2)), (b * m).sum((1, 2)), m.sum((1, 2))], 1)
    rl = torch.where(xyz[:, 1] > TH, 116 * f[:, 1].abs() + 16, 903.3 * xyz[:, 1].abs())
    r = torch.stack([(rl * am).sum((1, 2)), (500 * (f[:, 0].abs() + f[:, 1].abs()) * am).sum((1, 2)),
                     (200 * (f[:, 1].abs() + f[:, 2].abs()) * am).sum((1, 2)), am.sum((1, 2))], 1)
    return s, r


def _loss64(fake, real, mf, mr):
    xd = fake.double().requires_grad_()
    _, _, L, a, b = _lab64(xd)
    _, _, Lr, ar, br = _lab64(real)

    def avg(ch, m):
        cnt = m.double().sum((1, 2, 3))
        return (ch * m[:, 0].double()).sum((1, 2)) / torch.where(cnt == 0, torch.ones_like(cnt), cnt)
    d = torch.stack([avg(a, mf) - avg(ar, mr), avg(b, mf) - avg(br, mr)], 1)
    loss = d.abs().mean()
    return xd, loss, d


def _grad_rabs(fake, mf, tab):
    """|chain rule|: d/d fake of sum m (|Ta| 500 (f(X) + f(Y)) + |Tb| 200 (f(Y) + f(Z))) with f' > 0, M > 0."""
    xd = fake.double().requires_grad_()
    _, f, _, _, _ = _lab64(xd)
    ta, tb = tab[:, 0].abs().view(-1, 1, 1), tab[:, 1].abs().view(-1, 1, 1)
    e = (ta * 500 * (f[:, 0] + f[:, 1]) + tb * 200 * (f[:, 1] + f[:, 2])) * mf[:, 0].double().abs()
    e.sum().backward()
    return xd.grad


def _ratio(got, ref, rabs):
    return float(((got.double().cpu() - ref.double()).abs() / (U * rabs.double().clamp_min(1e-300))).max())


@pytest.mark.parametrize("n,h,w,kind", [(3, 37, 53, "mixed"), (1, 29, 31, "mixed"), (2, 45, 61, "frac"), (8, 256, 256, "mixed")])
def test_hair_avg_lab_kernels_vs_fp64_autograd(n, h, w, kind):
    """Odd sizes, N = 1, empty and full masks; 8 x 256^2 runs several grid-stride passes per block."""
    from michigan_b200 import ops
    fake, real, mf, mr = _case(n, h, w, kind)
    gup = 0.7
    g = torch.tensor([gup], dtype=torch.float32).cuda()
    res = []
    for _ in range(2):
        s = ops.hair_avg_lab_fwd(fake.cuda(), real.cuda(), mf.cuda(), mr.cuda())
        d = ops.hair_avg_lab_bwd(fake.cuda(), mf.cuda(), s, g)
        torch.cuda.synchronize()
        res.append((s.clone(), d.clone()))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]), "second run differs"
    s, d = res[0]
    sf, rf = _sums64(fake, mf)
    sr, rr = _sums64(real, mr)
    ks = max(_ratio(s[:, 0], sf, rf), _ratio(s[:, 1], sr, rr))
    xd, loss, diff = _loss64(fake, real, mf, mr)
    loss.backward(torch.tensor(gup, dtype=torch.float64))
    # the module's loss from the same sums
    cnt = s[:, :, 3:]
    avg = s[:, :, 1:3] / torch.where(cnt == 0, torch.ones_like(cnt), cnt)
    got_loss = float((avg[:, 0] - avg[:, 1]).abs().mean())
    cf = torch.where(sf[:, 3] == 0, torch.ones_like(sf[:, 3]), sf[:, 3])
    cr = torch.where(sr[:, 3] == 0, torch.ones_like(sr[:, 3]), sr[:, 3])
    r_loss = float(((rf[:, 1:3] / cf[:, None]) + (rr[:, 1:3] / cr[:, None])).mean())
    kl = abs(got_loss - float(loss.detach())) / (U * r_loss)
    tab = gup / (2 * n) * torch.sign(diff.detach()) / cf[:, None]
    kg = _ratio(d, xd.grad, _grad_rabs(fake, mf, tab))
    print("hair-avg Lab %s %dx%dx%d: sums %.2f, loss %.2f, d fake %.2f  (|err| / (u R_abs))" % (kind, n, h, w, ks, kl, kg))
    assert ks <= K_SUMS and kl <= K_SUMS and kg <= K_GRAD
    if kind == "mixed":
        assert float(d.cpu()[(mf == 0).expand_as(d)].abs().max()) == 0.0           # no tag hair, no gradient
        if n > 1:
            assert float(s[1, 0].abs().max()) == 0.0


def test_hair_avg_lab_module_vs_reference_golden():
    """HairAvgLabLoss against the reference class's own loss and d fake (three cases of tests/test_oracle_unpaired.py)."""
    from michigan_b200.networks import HairAvgLabLoss
    from michigan_b200.options import make_opt
    from test_oracle_unpaired import CASES, GOLDEN, cases
    z = np.load(GOLDEN)
    crit = HairAvgLabLoss(make_opt())
    for name in CASES:
        fake, real, mf, mr = cases()[name]
        x = fake.cuda().requires_grad_()
        loss = crit(x, real.cuda(), mf.cuda(), mr.cuda())
        loss.backward()
        ref_l, ref_g = float(z[name + "_loss"]), torch.from_numpy(z[name + "_grad"]).double()
        rl = abs(float(loss) - ref_l) / abs(ref_l)
        rg = float((x.grad.cpu().double() - ref_g).norm() / ref_g.norm())
        print("   %-15s loss %.8f  reference %.8f  rel %.2e, d fake rel L2 %.2e" % (name, float(loss), ref_l, rl, rg))
        assert rl <= 1e-5 and rg <= 1e-5, name
    with pytest.raises(NotImplementedError, match="balance_Lab"):
        HairAvgLabLoss(make_opt(balance_Lab=True))


def test_unpaired_generator_step_vs_oracle():
    """One generator step of the unpaired stage (curr_step 2, pix2pix_model.py:280-363) assembled from the package's classes at
    the golden configuration (ngf 64, 128x128, batch 2): the generator and the stand-alone model's plumbing, a second
    discriminator's weights in the judging network, GANLoss, L1OLoss, HairAvgLabLoss and RGBBackgroundL1Loss, with the tag's
    and the reference's hair differing.  Against oracle_unpaired.compute_generator_loss_unpaired: every loss within its bound,
    a gradient for every generator parameter, per-tensor G-gradient cosine >= 0.998 on the tensors the golden fixture samples.
    Measured on an H100: hairAvgLab 2.4e-5 and background 1.1e-6 relative, the other terms within 1.7e-3, worst cosine 0.99994."""
    import michigan_oracle as orc
    from helpers import load_golden, reference_layout_state, summary
    from michigan_b200.networks import HairAvgLabLoss, RGBBackgroundL1Loss
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel, _frozen
    from michigan_b200.synth import synthetic_batch
    z, cfg = load_golden()
    opt = make_opt(is_train=True, ngf=cfg["ngf"], ndf=cfg["ndf"], crop_size=cfg["size"], batchSize=cfg["batch"], no_orient_loss=False,
                   no_confidence_loss=False)
    model = Pix2PixModel(opt)
    sdG = reference_layout_state("G", cfg, cfg["seed_G"])
    sdD2 = reference_layout_state("D", cfg, cfg["seed_D"] + 7)
    model.netG.load_state_dict(sdG)
    model.netD.load_state_dict(sdD2)
    model.train()
    data = synthetic_batch(cfg["batch"], cfg["size"], cfg["data_seed"])
    s = cfg["size"]
    data["label_ref"] = torch.zeros_like(data["label_ref"])
    data["label_ref"][:, :, s // 4:3 * s // 4, s // 8:s // 2] = 1.0
    data["image_ref"] = data["image_tag"].flip(-1).contiguous()
    random.seed(cfg["py_seed"])
    th = int(s * 0.05); th = th if th % 2 == 1 else th + 1
    k = random.choice([max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4])
    random.seed(cfg["py_seed"])
    input_ref, input_tag, image_ref, image_tag, orient_mask, noise = model.preprocess_input(dict(data))
    fake = model.generate_fake(input_ref, image_ref, orient_mask, input_tag, image_tag, noise)
    with _frozen(model.netD):
        pred_fake, _ = model.discriminate(input_tag, fake, image_tag, orient_mask)
    g = {"GAN": model.criterionGAN(pred_fake, True, for_discriminator=False, label=input_tag[:, 1:2])}
    g["ORIENT"], conf = model.criterionOrient(fake, orient_mask, input_tag)
    g["ORIENT"] = g["ORIENT"] * opt.lambda_orient
    g["CONFIDENCE"] = conf * opt.lambda_confidence
    g["hairAvgLab"] = HairAvgLabLoss(opt)(fake, image_ref, input_tag[:, 1:2], input_ref[:, 1:2]) * 1.0
    g["background"] = RGBBackgroundL1Loss()(fake, input_tag, image_tag) * 1.0
    sum(v.mean() for v in g.values()).backward()
    torch.cuda.synchronize()
    for name, p in model.netG.named_parameters():
        assert name.startswith("backgroud_enc.layer4") or p.grad is not None, name
    assert all(p.grad is None for p in model.netD.parameters())

    pre = dict(input_ref=orc.one_hot(data["label_ref"]), input_tag=orc.one_hot(data["label_tag"]), image_ref=data["image_ref"],
               image_tag=data["image_tag"], orient_mask=data["orient"], noise=data["noise"])
    oopt = orc.default_opt(ngf=cfg["ngf"], ndf=cfg["ndf"], crop_size=cfg["size"], isTrain=True)
    oopt.no_orient_loss, oopt.no_confidence_loss = False, False
    names = [n for n in sdG if not n.endswith(("running_mean", "running_var", "num_batches_tracked", "weight_u", "weight_v"))]
    for n in names:
        sdG[n].requires_grad_(True)
    losses_o, _ = ou.compute_generator_loss_unpaired(sdG, sdD2, oopt, pre, rng_k=k)
    orc.trainer_loss(losses_o).backward()
    assert list(losses_o) == list(g) == ["GAN", "ORIENT", "CONFIDENCE", "hairAvgLab", "background"]
    for key in g:
        a, b = float(g[key].mean()), float(losses_o[key].mean())
        print("   %-10s %.6f  oracle %.6f  rel %.2e" % (key, a, b, abs(a - b) / max(abs(b), 1e-30)))
        if key in ("hairAvgLab", "background"):
            assert abs(a - b) <= 1e-3 * abs(b), key
        else:                                   # the bound of the paired stage's generator-step tests
            assert abs(a - b) <= 1e-2 * max(1.0, abs(b)), key
    named = dict(model.netG.named_parameters())
    worst = 1.0
    for key in z.files:
        if key.startswith("g_grad/") and not key.endswith("conv_0.bias"):   # bias before a batch-norm: gradient is exactly 0
            n = key[len("g_grad/"):]
            a, b = summary(named[n].grad, stride=101)[4:], summary(sdG[n].grad, stride=101)[4:]
            cos = float(np.dot(a.astype(np.float64), b) / (np.linalg.norm(a) * np.linalg.norm(b)))
            worst = min(worst, cos)
    print("   worst per-tensor G-gradient cosine %.5f" % worst)
    assert worst >= 0.998, worst
