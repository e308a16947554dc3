"""DoG orientation loss on the GPU (L1OLoss with an orient_filter other than 'gabor'), element by element against float64,
and the whole loss against the oracle (tests/oracle_orient_dog.py) and the reference's outputs (golden_orient_dog.npz).

Bounds, with u = 2^-24, k = 1.25 sqrt(289) + 8 and R_abs = sum over the taps of |gray| |K| (DESIGN.md §5):
  * response pass: each response within k u R_abs of float64 (gray from the fp32 image in float64); the arg-max is admissible
    when its float64 response is within 2 k u R_abs of the best; rh = r hair within the same bound times hair; M is the
    maximum of the kernel's own rh, bit for bit;
  * loss pass (op 12, given the kernel's idx and rh): the six slots against float64 of the formula, the four sums within
    1e-5 of the sum of their terms' magnitudes, the tie count exactly;
  * dL/dr (op 12 backward): every element within 1e-5 of the magnitude of its terms plus the share's bound, against float64
    autograd of the formula (torch's max() splits the M-gradient evenly among ties); the signs of |.| are taken from the fp32
    restatement of the kernel's arithmetic, so a value within rounding of 0 does not flip a whole term;
  * image gradient: the float64 transposed convolution of float64 dL/dr through the kernel's filters, within 2 k u of the
    transposed convolution of the magnitudes plus the dL/dr bound carried through |K|.
The worst measured ratio of error to bound is printed per test.
"""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle_orient_dog as od

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
KB = 1.25 * math.sqrt(289) + 8
SIZES = [(1, 1, 1), (1, 5, 7), (1, 16, 16), (1, 33, 47), (1, 17, 130), (3, 40, 24), (2, 512, 512)]


def _inputs(n, h, w, seed, frac=False, tie=False):
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(h).float(), torch.arange(w).float(), indexing="ij")
    base = torch.sin(0.7 * xx + 0.3 * yy).view(1, 1, h, w) * 0.5
    img = (base + 0.2 * torch.randn(n, 3, h, w, generator=g)).clamp(-1, 1)
    hair = (torch.rand(n, h, w, generator=g) < 0.7).float()
    if frac:
        hair = hair * torch.rand(n, h, w, generator=g)
    label2 = torch.rand(n, 2, h, w, generator=g) * 2 - 1
    if tie:                              # every image the same: the maximum ties across the batch, bit for bit
        img[1:], hair[1:], label2[1:] = img[:1].clone(), hair[:1].clone(), label2[:1].clone()
    return img.cuda(), hair.cuda().contiguous(), label2.cuda().contiguous()


def _bank():
    from michigan_b200.networks.loss import dog_bank
    return dog_bank("cuda")


def _resp64(img, bank):
    """float64 responses [N,32,H,W] and R_abs [N,32,H,W]."""
    gray = od.gray_of(img.double())
    w = bank.double().t().reshape(32, 1, 17, 17)
    return F.conv2d(gray, w, padding=8), F.conv2d(gray.abs(), w.abs(), padding=8)


def _response(img, hair, bank):
    from michigan_b200 import ops
    return ops.dog_response(img.contiguous(), bank, hair)


@pytest.mark.parametrize("size", SIZES)
def test_response_pass_vs_fp64(size):
    n, h, w = size
    bank = _bank()
    img, hair, _ = _inputs(n, h, w, seed=h * 131 + w, frac=(h == 33))
    idx, rh, m = _response(img, hair, bank)
    resp, rabs = _resp64(img, bank)
    tol = KB * U * rabs
    rc = resp.clamp(min=0)
    best, bi = rc.max(dim=1)
    il = idx.long().unsqueeze(1)
    sel, tsel = rc.gather(1, il)[:, 0], tol.gather(1, il)[:, 0]
    tbest = tol.gather(1, bi.unsqueeze(1))[:, 0]
    assert bool((sel >= best - tsel - tbest).all()), "inadmissible arg-max"
    err = (rh.double() - sel * hair.double()).abs()
    bound = tsel * hair.double() + 1e-30
    assert bool((err <= bound).all()), float((err / bound).max())
    assert float(m[0]) == float(rh.max())
    assert torch.equal(m.view(torch.int32)[0], rh.max().view(torch.int32))
    print("%s: rh err/bound %.3f" % (size, float((err / bound).max())))


def _op12(img, hair, label2, bank, sincos, go, gc):
    """The kernels' op 12 forward slots and backward dL/dr, with the response pass's idx, rh and M."""
    from michigan_b200 import _lib, ops
    from michigan_b200.networks.loss import DEN_EPS, _dog_term, _pinned_table
    idx, rh, m = _response(img, hair, bank)
    n, h, w = rh.shape
    slots = torch.zeros(6, device="cuda", dtype=torch.float64)
    t = _pinned_table(_dog_term(rh, label2, hair, idx, m, sincos, None), rh.device)
    _lib.check(_lib.load().mg_loss_reduce(t.data_ptr(), 1, slots.data_ptr(), ops._stream()), "mg_loss_reduce")
    god = torch.tensor(go, device="cuda", dtype=torch.float64) / (2.0 * n * h * w)
    gcd = torch.tensor(gc, device="cuda", dtype=torch.float64) / (slots[2] + DEN_EPS)
    gsl = torch.stack([god, gcd, (god * slots[3] + gcd * slots[4]) / slots[5]]).float().contiguous()
    dr = torch.empty_like(rh)
    t2 = _pinned_table(_dog_term(rh, label2, hair, idx, m, sincos, dr.data_ptr()), rh.device)
    _lib.check(_lib.load().mg_loss_reduce_bwd(t2.data_ptr(), 1, gsl.data_ptr(), ops._stream()), "mg_loss_reduce_bwd")
    torch.cuda.synchronize()
    return idx, rh, m, slots, dr


def _formula64(idx, rh, hair, label2, sincos, go, gc):
    """float64 autograd of the op 12 formula on rh (leaf), |.| signed as the kernel's fp32 arithmetic signs it."""
    x = rh.double().requires_grad_()
    h, l2 = hair.double(), label2.double()
    s = sincos[0][idx.long()].double()
    c = sincos[1][idx.long()].double()
    # fp32 restatement of the kernel's per-pixel values: only their signs are used
    q32 = rh / rh.max()
    conf32 = torch.where((q32 > 0) | torch.isnan(q32), q32, torch.zeros_like(q32))
    sg = [torch.sign(sincos[0][idx.long()] * conf32 * hair - label2[:, 0] * hair),
          torch.sign(sincos[1][idx.long()] * conf32 * hair - label2[:, 1] * hair), torch.sign(conf32 * hair - hair)]
    M = x.max()
    q = x / M
    conf = q * (~(q <= 0)).double()
    ds, dc, dcf = s * conf * h - l2[:, 0] * h, c * conf * h - l2[:, 1] * h, conf * h - h
    n, hh, ww = rh.shape
    lo = (ds * sg[0].double() + dc * sg[1].double()).sum() / (2.0 * n * hh * ww)
    lc = (dcf * sg[2].double()).sum() / (h.sum() + 1e-5)
    (go * lo + gc * lc).backward()
    with torch.no_grad():
        keep = (~(q <= 0)).double()
        Lo = keep * (sg[0].double() * s + sg[1].double() * c) * h
        Lc = keep * sg[2].double() * h
        dm = -x / (M * M)
        terms = {"fo": (ds.abs() + dc.abs()), "fc": dcf.abs(), "h": h, "so": Lo * dm, "sc": Lc * dm}
        ties = float((x == M).sum())
    return x.grad * h, terms, ties, Lo, Lc, float(M), lo, lc


def _dr_bound(rh, hair, terms, ties, Lo, Lc, M, go, gc):
    """Per-element bound of dL/dr: 1e-5 of the magnitude of its terms, plus at the maximisers the bound of the share, whose
    sums S carry 1e-5 of the magnitudes of their terms."""
    n, h, w = rh.shape
    god, gcd = go / (2.0 * n * h * w), gc / (float(terms["h"].sum()) + 1e-5)
    so, sc = terms["so"], terms["sc"]
    share = abs(god * float(so.sum()) + gcd * float(sc.sum())) / ties
    share_bound = (god * float(so.abs().sum()) + gcd * float(sc.abs().sum())) * 1e-5 / ties
    hh, at_m = hair.double(), (rh.double() == M).double()
    return 1e-5 * hh * ((god * Lo.abs() + gcd * Lc.abs()) / M + at_m * share) + hh * at_m * share_bound + 1e-30


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("kind", ["binary", "fractional", "tie"])
def test_loss_pass_and_dr_vs_fp64(size, kind):
    from michigan_b200.networks.loss import _orient_sincos
    n, h, w = size
    if kind == "tie" and n == 1:
        pytest.skip("a tie across images needs two")
    bank, sincos = _bank(), _orient_sincos("cuda")
    img, hair, label2 = _inputs(n, h, w, seed=7 * h + w, frac=kind == "fractional", tie=kind == "tie")
    go, gc = 10.0, 100.0
    idx, rh, m, slots, dr = _op12(img, hair, label2, bank, sincos, go, gc)
    if float(m[0]) == 0.0:
        assert torch.isnan(slots[:2]).all() and torch.isnan(dr).all()
        return
    ref_dr, terms, ties, Lo, Lc, M, _, _ = _formula64(idx, rh, hair, label2, sincos, go, gc)
    sl = slots.cpu()
    for k, key in enumerate(["fo", "fc", "h", "so", "sc"]):
        t = terms[key]
        ref, mag = float(t.sum()), float(t.abs().sum())
        assert abs(float(sl[k]) - ref) <= 1e-5 * mag + 1e-30, (key, float(sl[k]), ref, mag)
    assert float(sl[5]) == ties
    if kind == "tie":
        assert ties >= 2
    bound = _dr_bound(rh, hair, terms, ties, Lo, Lc, M, go, gc)
    err = (dr.double() - ref_dr).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    if kind == "tie":
        tied = dr[rh == rh.max()]
        assert bool((tied == tied[0]).all())
    print("%s %s: dL/dr err/bound %.3f, ties %d" % (size, kind, float((err / bound).max()), ties))


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("kind", ["binary", "fractional", "tie", "empty_image", "no_hair"])
def test_image_gradient_vs_fp64(size, kind):
    """The whole L1OLoss DoG backward element by element: the gather of dL/dr through the kernel's filters against the float64
    transposed convolution of float64 dL/dr, including the 17x17 footprint of the maximiser and the even split of a tie."""
    from michigan_b200.networks.loss import L1OLoss
    from michigan_b200.options import make_opt
    n, h, w = size
    if kind in ("tie", "empty_image") and n == 1:
        pytest.skip("needs two images")
    bank = _bank()
    img, hair, label2 = _inputs(n, h, w, seed=3 * h + w, frac=kind == "fractional", tie=kind == "tie")
    if kind == "empty_image":
        hair[1] = 0
    if kind == "no_hair":
        hair.zero_()
    sem = torch.stack([1 - hair, hair], dim=1)
    crit = L1OLoss(make_opt(orient_filter="dog", use_ig=True))
    x = img.clone().requires_grad_()
    lo, lc = crit(x, label2, sem)
    (lo * 10.0 + lc * 100.0).backward()
    if kind == "no_hair" or float(rh_max(img, hair, bank)) == 0.0:
        assert math.isnan(float(lo)) and math.isnan(float(lc)) and bool(torch.isnan(x.grad).all())
        return
    from michigan_b200.networks.loss import _orient_sincos
    sincos = _orient_sincos("cuda")
    idx, rh, m = _response(img, hair, bank)
    ref_dr, terms, ties, Lo, Lc, M, rlo, rlc = _formula64(idx, rh, hair, label2, sincos, 10.0, 100.0)
    bdr = _dr_bound(rh, hair, terms, ties, Lo, Lc, M, 10.0, 100.0)
    assert abs(float(lo) - float(rlo)) <= 1e-5 * abs(float(rlo)) + 1e-12
    assert abs(float(lc) - float(rlc)) <= 1e-5 * abs(float(rlc)) + 1e-12
    wk = bank.double().t().reshape(32, 1, 17, 17)
    D = torch.zeros(n, 32, h, w, device="cuda", dtype=torch.float64).scatter_(1, idx.long().unsqueeze(1), ref_dr.unsqueeze(1))
    dgray = F.conv_transpose2d(D, wk, padding=8)
    dabs = F.conv_transpose2d(D.abs(), wk.abs(), padding=8)
    coef = torch.tensor([0.299, 0.587, 0.144], device="cuda", dtype=torch.float64).view(1, 3, 1, 1) * 127.5
    ref = dgray * coef
    il = idx.long().unsqueeze(1)
    B = torch.zeros(n, 32, h, w, device="cuda", dtype=torch.float64).scatter_(1, il, bdr.unsqueeze(1))
    bound = (KB * 2 * U * dabs + F.conv_transpose2d(B, wk.abs(), padding=8)) * coef + 1e-30
    err = (x.grad.double() - ref).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    if kind == "empty_image":
        assert float(x.grad[1].abs().max()) == 0.0
    print("%s %s: d image err/bound %.3f" % (size, kind, float((err / bound).max())))


def rh_max(img, hair, bank):
    return _response(img, hair, bank)[2][0]


def test_loss_runs_without_host_synchronisation():
    from michigan_b200.networks.loss import L1OLoss
    from michigan_b200.options import make_opt
    img, hair, label2 = _inputs(2, 64, 64, seed=1)
    sem = torch.stack([1 - hair, hair], dim=1)
    crit = L1OLoss(make_opt(orient_filter="dog", use_ig=True))
    x = img.clone().requires_grad_()
    lo, lc = crit(x, label2, sem)            # builds the bank and the angle table
    (lo + lc).backward()
    torch.cuda.synchronize()
    x.grad = None
    torch.cuda.set_sync_debug_mode("error")
    try:
        lo, lc = crit(x, label2, sem)
        (lo * 10.0 + lc * 100.0).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert bool(torch.isfinite(x.grad).all())


def test_thin_convs_ignore_the_zeroed_argmax_fields():
    """The appended mg_thin_args fields are null in every ordinary thin conv: the conv writes what it wrote before (checked
    against float64) and bit for bit the same before and after an arg-max launch."""
    from michigan_b200 import ops
    torch.manual_seed(0)
    x = torch.randn(2, 20, 24, 4, device="cuda")
    wt = torch.randn(7 * 7 * 4 * 64, device="cuda") * 0.1
    bias = torch.randn(64, device="cuda")
    y0 = ops.conv_thin(x, wt, bias, 64, 7, 7, 1, 3)
    _response(*_inputs(1, 16, 16, seed=0)[:2], _bank())
    y1 = ops.conv_thin(x, wt, bias, 64, 7, 7, 1, 3)
    assert torch.equal(y0, y1)
    wk = wt.double().view(7, 7, 4, 64).permute(3, 2, 0, 1)
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), wk, bias.double(), padding=3).permute(0, 2, 3, 1)
    mag = F.conv2d(x.double().abs().permute(0, 3, 1, 2), wk.abs(), bias.double().abs(), padding=3).permute(0, 2, 3, 1)
    assert bool(((y0.double() - ref).abs() <= (1.25 * math.sqrt(196) + 8) * U * mag + 1e-30).all())


@pytest.mark.parametrize("case", od.CASES)
def test_dog_loss_vs_oracle_and_golden(case):
    """L1OLoss (DoG) against the oracle and the reference's own outputs, with the tolerances of test_gpu_orient.py."""
    from michigan_b200.networks.loss import L1OLoss, dog_bank
    from michigan_b200.options import make_opt
    z = np.load(os.path.join(ROOT, "tests", "golden", "golden_orient_dog.npz"))
    img, label, sem, use_ig = od.cases()[case]
    crit = L1OLoss(make_opt(orient_filter="dog", use_ig=use_ig))
    x = img.clone().cuda().requires_grad_()
    lo, lc = crit(x, label.cuda(), sem.cuda())
    (lo * 10.0 + lc * 100.0).backward()
    xr = img.clone().requires_grad_()
    ro, rc = od.orient_loss_dog(xr, label, sem, use_ig, dog_bank("cpu"))
    (ro * 10.0 + rc * 100.0).backward()
    g = x.grad.cpu()
    if case == "no_hair":
        assert math.isnan(float(lo)) and math.isnan(float(lc)) and bool(torch.isnan(g).all())
        return
    for ref_o, ref_c, ref_g in ((float(ro), float(rc), xr.grad), (float(z[case + "_lo"]), float(z[case + "_lc"]),
                                                                  torch.from_numpy(z[case + "_g"]))):
        assert abs(float(lo) - ref_o) <= 2e-4 * max(1.0, abs(ref_o))
        assert abs(float(lc) - ref_c) <= 1e-5 * max(1.0, abs(ref_c))
        rel = float((g - ref_g).norm() / ref_g.norm())
        assert rel <= 2e-2, rel
    print("%s: ORIENT %.6f (ref %.6f) CONFIDENCE %.6f (ref %.6f) grad rel L2 %.2e"
          % (case, float(lo), float(z[case + "_lo"]), float(lc), float(z[case + "_lc"]), rel))
    if case == "one_empty":
        assert float(g[1].abs().max()) == 0.0


def test_stand_alone_train_iteration_with_the_dog_filter():
    import random
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel, train_iteration
    from michigan_b200.synth import synthetic_batch
    torch.manual_seed(0)
    opt = make_opt(is_train=True, ngf=64, ndf=64, crop_size=64, batchSize=2, no_orient_loss=False, no_confidence_loss=False,
                   orient_filter="dog")
    model = Pix2PixModel(opt).train()
    optG, optD = model.create_optimizers(opt)
    random.seed(0)
    g, d, img = train_iteration(model, optG, optD, dict(synthetic_batch(2, 64, 1)))
    assert list(g) == ["GAN", "GAN_Feat", "ORIENT", "CONFIDENCE"]
    assert all(bool(torch.isfinite(v).all()) for v in list(g.values()) + list(d.values()))
    print("train_iteration: ORIENT %.5f CONFIDENCE %.5f" % (float(g["ORIENT"]), float(g["CONFIDENCE"])))
