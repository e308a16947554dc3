"""The count-balanced Lab losses of --balance_Lab on the sm_90a kernels: mg_loss_reduce / mg_loss_reduce_bwd op 11 (LabColorLoss)
and the per-image weights of HairAvgLabLoss over mg_hair_avg_lab_fwd / _bwd.

Op 11 against float64 autograd, element by element, with the bins taken from the float64 Lab of the real image:

    |got - ref| <= bound,  u = 2^-24,

the forward sum's bound being sum over pixels of w (K_LAB u (R_a + R_b)) + 2 u w (|da| + |db|) (the Lab error of
test_gpu_loss_kernels_fp64.test_lab_loss_fwd_bwd carried through the weight, plus the two weighted products' roundings), and
d fake's (K_LAB + 2) u R_abs with R_abs the chain rule with magnitudes scaled by g w.  Where a real pixel's a + 128 or b + 128
lies within its error bound of an integer, the kernel may take either neighbouring bin: the forward bound then adds
(max - min of w over those bins) (|da| + |db|) and d fake of that pixel is waived, as is d fake where |da| or |db| is within its
bound (either sign) or t is within its bound of the threshold (either branch of f).

The whole classes are held to the reference's own outputs (tests/golden/golden_balance_lab.npz, rel 1e-5 for the loss and the
relative L2 error of d fake), the balanced loss with a uniform count table to the unbalanced one (fp64 summation rounding for
the loss, u |d fake| for the gradient), and one stand-alone train_iteration with the balanced Lab loss to the CPU oracle.

Measured on an H100 80GB HBM3 (700 W power limit): op 11 forward at most 0.0097 of its bound, d fake at most 0.30 of its
bound (8 x 512^2, 0.1-0.2 % of the pixels waived); the uniform table gave the same fp32 loss and d fake as the unbalanced
kernels; against the reference, loss rel <= 4.0e-7 and d fake rel L2 <= 1.6e-7; the train iteration's lab term equal to the
oracle's in fp32."""
import os

import numpy as np
import pytest
import torch

import oracle_balance_lab as obl
from test_gpu_loss_kernels_fp64 import (K_LAB, LAB_M, LAB_T, TINY, U, _gen, _lab_df, _lab_f, _lab_inputs, _lab_t,
                                        check_within)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_balance_lab.npz")
K_BAL = K_LAB + 2


def _table(g, zeros=True):
    """E: fp32 weights in [1, 10] with, optionally, a block of zero entries around the gray bins (a, b near 0) and bin 255."""
    E = 1 + 9 * torch.rand(256, 256, generator=g)
    if zeros:
        E[120:136, 124:132] = 0
        E[255] = 0
        E[:, 255] = 0
    return E


def _mask(kind, n, h, w, g):
    """[N,1,H,W] channel 1 of a two-channel map (image stride 2 H W, as the one-hot label's hair channel)."""
    m = torch.zeros(n, 2, h, w)
    if kind == "full":
        m[:, 1] = 1
    elif kind == "partial":
        m[:, 1] = (torch.rand(n, h, w, generator=g) > 0.4).float()
    elif kind == "nonbinary":
        m[:, 1] = torch.rand(n, h, w, generator=g) * 1.5
    return m


def _bins(x, bound):
    """Candidate bins of x = a + 128 (float64): (lo, hi), equal unless x lies within `bound` of an integer."""
    r = x.round()
    near = (x - r).abs() <= bound
    lo = torch.where(near, r - 1, x.floor()).clamp(0, 255).long()
    hi = torch.where(near, r, x.floor()).clamp(0, 255).long()
    return lo, hi


def _weights(E, ka, kb, l):
    w = E[ka, kb].double() * l
    return torch.where(w == 0, torch.ones_like(w), w)


def _op11(fake, real, mask, E, scale=1.0, gslot=1.0, add=None):
    """Run op 11 forward and backward on the GPU; -> (slot, d fake)."""
    from michigan_b200 import _lib, ops
    from michigan_b200.networks.loss import _Term, _balanced_lab_term, _device_table
    dev = torch.device("cuda")
    f, r, m, e = fake.to(dev), real.to(dev), mask.to(dev)[:, 1:2], E.to(dev)
    slots = torch.zeros(1, device=dev, dtype=torch.float64)
    t = _balanced_lab_term(f, r, m, e, None)
    t.scale = scale
    lib = _lib.load()
    assert lib.mg_loss_term_bytes() == __import__("ctypes").sizeof(_Term)
    _lib.check(lib.mg_loss_reduce(_device_table([t], dev).data_ptr(), 1, slots.data_ptr(), ops._stream()), "mg_loss_reduce")
    ga = torch.full_like(f, float("nan"))
    a = add.to(dev) if add is not None else None
    t = _balanced_lab_term(f, r, m, e, ga)
    t.scale = scale
    t.add = a.data_ptr() if a is not None else None
    g = torch.tensor([gslot], dtype=torch.float32, device=dev)
    _lib.check(lib.mg_loss_reduce_bwd(_device_table([t], dev).data_ptr(), 1, g.data_ptr(), ops._stream()), "mg_loss_reduce_bwd")
    torch.cuda.synchronize()
    return float(slots[0]), ga.cpu()


CASES = [(s, m) for s in [(1, 1, 1), (3, 17, 19), (2, 7, 1), (1, 1, 512 * 512 + 3)] for m in ("empty", "full", "partial", "nonbinary")]
CASES += [((8, 512, 512), "partial"), ((8, 512, 512), "nonbinary")]


@pytest.mark.parametrize("shape,mask_kind", CASES)
def test_op11_vs_float64(shape, mask_kind):
    n, h, w = shape
    name = "op11 %dx%dx%d %s" % (n, h, w, mask_kind)
    g = _gen(name)
    fake, real = _lab_inputs(n, h * w, g)
    fake, real = fake.view(n, 3, h, w), real.view(n, 3, h, w)
    mask = _mask(mask_kind, n, h, w, g)
    E = _table(g)
    scale, gslot = 0.75, 1.3 / (n * h * w)
    add = torch.randn(n, 3, h, w, generator=g) * 1e-3 if h == 17 else None
    got_s, got_g = _op11(fake, real, mask, E, scale, gslot, add)
    # float64 Lab, signs and bins
    tf, tr = _lab_t(fake), _lab_t(real)
    ff, fr = _lab_f(tf, tf > LAB_T), _lab_f(tr, tr > LAB_T)
    near_f = (tf - LAB_T).abs() <= K_LAB * U * tf
    jump = (_lab_f(tf, torch.ones_like(near_f)) - _lab_f(tf, torch.zeros_like(near_f))).abs()
    jump_f = torch.where(near_f, jump, torch.zeros_like(jump))
    near_r = (tr - LAB_T).abs() <= K_LAB * U * tr
    jump = (_lab_f(tr, torch.ones_like(near_r)) - _lab_f(tr, torch.zeros_like(near_r))).abs()
    jump_r = torch.where(near_r, jump, torch.zeros_like(jump))
    ar, br = 500 * (fr[:, 0] - fr[:, 1]), 200 * (fr[:, 1] - fr[:, 2])
    da, db = 500 * (ff[:, 0] - ff[:, 1]) - ar, 200 * (ff[:, 1] - ff[:, 2]) - br
    ra = 500 * (ff[:, 0].abs() + ff[:, 1].abs() + fr[:, 0].abs() + fr[:, 1].abs())
    rb = 200 * (ff[:, 1].abs() + ff[:, 2].abs() + fr[:, 1].abs() + fr[:, 2].abs())
    ba = K_LAB * U * ra + 500 * (jump_f[:, 0] + jump_f[:, 1] + jump_r[:, 0] + jump_r[:, 1])
    bb = K_LAB * U * rb + 200 * (jump_f[:, 1] + jump_f[:, 2] + jump_r[:, 1] + jump_r[:, 2])
    # the real pixel's a, b alone: its own share of the bound (fr terms and their jumps)
    bar = K_LAB * U * 500 * (fr[:, 0].abs() + fr[:, 1].abs()) + 500 * (jump_r[:, 0] + jump_r[:, 1])
    bbr = K_LAB * U * 200 * (fr[:, 1].abs() + fr[:, 2].abs()) + 200 * (jump_r[:, 1] + jump_r[:, 2])
    ka_lo, ka_hi = _bins(ar + 128, bar)
    kb_lo, kb_hi = _bins(br + 128, bbr)
    l = mask[:, 1].flatten(1).double()
    ws = torch.stack([_weights(E, a, b, l) for a in (ka_lo, ka_hi) for b in (kb_lo, kb_hi)])
    wmin, wmax = ws.min(0).values, ws.max(0).values
    wr = _weights(E, (ar + 128).floor().clamp(0, 255).long(), (br + 128).floor().clamp(0, 255).long(), l)
    assert bool(((ka_lo != ka_hi) | (kb_lo != kb_hi)).any()) or h * w < 64  # the gray pixels sit on bin boundary 128
    if mask_kind != "empty" and h * w >= 64:
        assert bool((E[ka_lo, kb_lo] == 0).any())                         # a zero table entry is read: w = 0 -> 1
    # forward
    ref = scale * (wr * (da.abs() + db.abs())).sum()
    bound = scale * (wmax * (ba + bb) + 2 * U * wmax * (da.abs() + db.abs()) + (wmax - wmin) * (da.abs() + db.abs())).sum()
    check_within(name + " fwd", torch.tensor([abs(got_s - float(ref))]), torch.tensor([float(bound) + 1e-12 * abs(float(ref))]))
    # backward
    gs = float(torch.tensor(gslot, dtype=torch.float32) * torch.tensor(scale, dtype=torch.float32))
    rs = ((LAB_M[:, 0] + LAB_M[:, 1]) + LAB_M[:, 2]).double()
    M = LAB_M.double()
    cube = tf > LAB_T
    dfk = torch.stack([500 * da.sign(), -500 * da.sign() + 200 * db.sign(), -200 * db.sign()], 1)
    dt = dfk * _lab_df(tf, cube) / rs.view(1, 3, 1)
    gw = (gs * wr).unsqueeze(1)
    want = gw * 0.5 * torch.einsum("nkp,kc->ncp", dt, M)
    rabs = gw.abs() * 0.5 * torch.einsum("nkp,kc->ncp", dt.abs(), M)
    got = got_g.flatten(2).double()
    extra = torch.zeros_like(want)
    if add is not None:
        a64 = add.flatten(2).double()
        want = want + a64
        extra = U * want.abs()
    waived = (da.abs() <= ba) | (db.abs() <= bb) | near_f.any(1) | (wmax != wmin)
    err = (got - want).abs()
    bound_g = K_BAL * U * rabs + extra + TINY
    ok = (err <= bound_g) | waived.unsqueeze(1)
    kept = (err / bound_g)[~waived.unsqueeze(1).expand_as(err)]
    print("%s bwd: max err / bound = %.3g, %d of %d pixels waived" % (name, float(kept.max()) if kept.numel() else 0.0,
                                                                       int(waived.sum()), waived.numel()))
    assert bool(torch.isfinite(got).all()), name
    assert bool(ok.all()), (name, "d fake out of bound")


def test_uniform_count_table_matches_the_unbalanced_loss(tmp_path):
    """A count table of ones gives w = 1 everywhere: the balanced LabColorLoss equals the unbalanced one up to fp64 summation
    rounding (the same per-pixel values summed in another order; the fp32 losses then differ by at most one rounding), its
    d fake up to fp32 rounding."""
    from michigan_b200.networks.loss import LabColorLoss
    from michigan_b200.options import make_opt
    path = str(tmp_path / "ones.npy")
    np.save(path, np.ones((256, 256)))
    g = _gen("uniform table")
    fake, real = _lab_inputs(4, 96 * 80, g)
    fake, real = fake.view(4, 3, 96, 80).cuda(), real.view(4, 3, 96, 80).cuda()
    mask = (torch.rand(4, 1, 96, 80, generator=g) > 0.5).float().cuda()
    out = []
    for opt in (make_opt(), make_opt(balance_Lab=True, weight_dir=path)):
        x = fake.clone().requires_grad_()
        loss = LabColorLoss(opt)(x, real, mask)
        (loss * 3.0).backward()
        out.append((float(loss), x.grad.cpu().double()))
    (l0, g0), (l1, g1) = out
    print("uniform table: loss %.10g vs %.10g, max |d fake diff| %.3g" % (l1, l0, float((g1 - g0).abs().max())))
    assert abs(l1 - l0) <= 2 * U * abs(l0)
    assert bool(((g1 - g0).abs() <= U * g0.abs() + TINY).all())


@pytest.mark.parametrize("th", obl.THRESHOLDS)
def test_balanced_losses_vs_reference_golden(tmp_path, th):
    """LabColorLoss and HairAvgLabLoss with --balance_Lab against the reference classes' own losses and d fake."""
    from michigan_b200.networks import HairAvgLabLoss, LabColorLoss
    from michigan_b200.options import make_opt
    z = np.load(GOLDEN)
    path = str(tmp_path / "ab_count.npy")
    np.save(path, obl.count_table(int(z["table_seed"])))
    opt = make_opt(balance_Lab=True, weight_dir=path, Lab_weight_th=th)
    lab, avg = LabColorLoss(opt), HairAvgLabLoss(opt)
    for case, (fake, real, mf, mr) in obl.golden_inputs().items():
        for cls, fn in (("lab", lambda x: lab(x, real.cuda(), mf.cuda())),
                        ("avg", lambda x: avg(x, real.cuda(), mf.cuda(), mr.cuda()))):
            key = "%s_%s_th%g" % (cls, case, th)
            x = fake.cuda().requires_grad_()
            loss = fn(x)
            loss.backward()
            ref_l, ref_g = float(z[key + "_loss"]), torch.from_numpy(z[key + "_grad"]).double()
            rl = abs(float(loss) - ref_l) / abs(ref_l)
            rg = float((x.grad.cpu().double() - ref_g).norm() / ref_g.norm())
            print("   %-22s loss %.8f  reference %.8f  rel %.2e, d fake rel L2 %.2e" % (key, float(loss), ref_l, rl, rg))
            assert rl <= 1e-5 and rg <= 1e-5, key


def test_stand_alone_train_iteration_with_balance_lab(tmp_path):
    """One stand-alone train_iteration with the Lab loss on and --balance_Lab (ngf 64, 64x64, batch 2): finite losses, a
    gradient for every generator parameter, and the lab term against the CPU oracle on the generated image (rel 1e-3: a real
    pixel on a bin boundary may take the neighbouring bin)."""
    import random
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel, train_iteration
    from michigan_b200.synth import synthetic_batch
    path = str(tmp_path / "ab_count.npy")
    np.save(path, obl.count_table(obl.TABLE_SEED))
    torch.manual_seed(0)
    opt = make_opt(is_train=True, ngf=64, ndf=64, crop_size=64, batchSize=2, no_lab_loss=False, balance_Lab=True,
                   weight_dir=path, Lab_weight_th=2.5)
    model = Pix2PixModel(opt).train()
    optG, optD = model.create_optimizers(opt)
    data = synthetic_batch(2, 64, 1)
    random.seed(0)
    g, d, img = train_iteration(model, optG, optD, dict(data))
    assert list(g) == ["GAN", "GAN_Feat", "lab"]
    assert all(bool(torch.isfinite(v).all()) for v in list(g.values()) + list(d.values()))
    for name, p in model.netG.named_parameters():
        assert name.startswith("backgroud_enc.layer4") or p.grad is not None, name
    ref = obl.lab_color_loss_balanced(img.detach().cpu().float(), data["image_tag"], data["label_tag"],
                                      obl.weight_map(obl.count_table(obl.TABLE_SEED), 2.5))
    rel = abs(float(g["lab"]) - float(ref)) / abs(float(ref))
    print("train_iteration lab %.8f, oracle %.8f, rel %.2e" % (float(g["lab"]), float(ref), rel))
    assert rel <= 1e-3
