"""The GAN-objective ops of the fused loss reductions (csrc/mg_loss.cu, mg_loss_reduce / mg_loss_reduce_bwd ops 4-8) and the
GANLoss / GANFeatLoss classes built on them, compared element by element with float64 autograd of the reference's own
expressions (models/networks/loss.py:80-124, 154-175), fed the kernels' exact fp32 inputs:

  op 4  BCE with logits against a constant target    gan_mode 'original'
  op 5  squared error against a constant target      gan_mode 'ls'
  op 6  a l                                          generator hinge, --remove_background
  op 7  min((sign a - 1) l, 0)                       discriminator hinge, --remove_background
  op 8  |a l - b l|                                  GANFeatLoss.L1_loss_mask

l is the [N,1,H,W] hair label read through the nearest resize to the term's (h, w); the masked ops also sum l over the
term's elements into a second slot, sum(label1) * c exactly.  Cases: the bench's logit sizes from a 512^2 label (67^2, 35^2,
batch 8) and odd ratios (48x80 -> 13x7, 17x19), hair / empty / full masks, planted ties at x = 1, -1, 0 (and a = b), logits
up to |x| = 100, targets 1, 0, 0.9, 0.2, NCHW and channels-last (NHWC permuted) layouts, labels read as the hair channel
of a one-hot map (image stride 3 H W).

Error model, as tests/test_gpu_loss_kernels_fp64.py: |got - ref| <= k u R_abs + tiny, u = 2^-24, R_abs the same formula on
absolute values (for BCE |(1 - t) x| + max(-x, 0) + log1p(exp(-|x|)) per element; for its gradient |sigmoid(x)| + |t|).
Each case prints its measured max |got - ref| / (u R_abs) next to k.  Bounds, and the largest value measured on an H100
80GB HBM3 (700 W power limit):

  * forward slot: k = L + 8, L the most elements one thread adds in fp32 (one per trip: ceil(n / (592 x 256))), + 8 for
    the per-element roundings of f (expf / log1pf within 2 ulp each, the products and adds): k = 9 .. 10, measured at most
    1.61.
  * label slot: exactly sum(label1) * c.
  * backward: K_GA = 8 on R_abs = |gslot scale| |f'| (MSE: 2 |gslot scale| (|x| + |t|)): measured 2.82 (op 5);
    BCE K_GA_BCE = 12 on |gslot scale| (sigmoid + |t|) (expf, 1 + e, the division, the difference with t, gslot * scale and
    the product, about 7 u): measured 3.57.  Ties as torch: the binary min gives each side half (times l, so 0 where the
    label is 0), |.| has gradient 0 at 0; the masked hinge's tie gradients are checked bit for bit.
  * whole classes against tests/oracle_gan_objectives.py in float64: loss K_CLASS = 64 on R_abs of all its terms (the masked
    terms' fp64 denominators add two roundings to the reduction's), measured 0.59; the input gradients K_GA (BCE K_GA_BCE),
    measured 2.32.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from test_gpu_loss_kernels_fp64 import TINY, U, _gen, check_close, d64

pytestmark = pytest.mark.gpu

dev = "cuda"
LOSS_BLOCKS, LOSS_THREADS = 592, 256
K_GA = 8.0
K_GA_BCE = 12.0
K_CLASS = 64.0
OP_BCE, OP_SQ_T, OP_WSUM, OP_HINGE_MASK, OP_L1_MASK = 4, 5, 6, 7, 8


def _label(n, H, W, kind, g):
    """The hair channel of an [n,3,H,W] one-hot label map (a view, image stride 3 H W): an ellipse per image plus noise
    specks, all 0 ('empty') or all 1 ('full')."""
    if kind == "empty":
        hair = torch.zeros(n, H, W)
    elif kind == "full":
        hair = torch.ones(n, H, W)
    else:
        yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
        hair = torch.zeros(n, H, W)
        for i in range(n):
            cy, cx = H * (0.3 + 0.4 * float(torch.rand(1, generator=g))), W * (0.3 + 0.4 * float(torch.rand(1, generator=g)))
            hair[i] = ((((yy - cy) / (0.3 * H)) ** 2 + ((xx - cx) / (0.25 * W)) ** 2) <= 1).float()
        hair = torch.maximum(hair, (torch.rand(n, H, W, generator=g) < 0.02).float())
    seg = torch.stack([1 - hair, hair, torch.zeros_like(hair)], 1).to(dev)
    return seg[:, 1:2]


def _on_device(x, layout):
    """x [N,C,h,w] on the device, NCHW contiguous or the NHWC-permuted view the discriminator returns."""
    if layout == "nchw":
        return x.to(dev).contiguous()
    return x.permute(0, 2, 3, 1).contiguous().to(dev).permute(0, 3, 1, 2)


def _logits(shape, g, big=False):
    x = torch.randn(*shape, generator=g) * 2.0
    flat = x.view(-1)
    flat[0::7], flat[1::7], flat[2::7] = 1.0, -1.0, 0.0             # hinge ties at +-1, BCE / sign at 0
    if big:
        flat[3::5] = (torch.rand(flat[3::5].numel(), generator=g) * 200 - 100)
        flat[4::13] = 100.0
        flat[5::13] = -100.0
    return x


def _per_thread(n):
    return -(-n // (LOSS_BLOCKS * LOSS_THREADS))


def _expr(op, x, b, l, sign, t):
    """The reference's per-element expression, differentiable in float64 (loss.py:83, 87, 110-117, 159)."""
    if op == OP_BCE:
        return F.binary_cross_entropy_with_logits(x, torch.full_like(x, t), reduction="none")
    if op == OP_SQ_T:
        return (x - t) ** 2
    if op == OP_WSUM:
        return x * l
    if op == OP_HINGE_MASK:
        return torch.min((sign * x - 1) * l, torch.zeros_like(x))
    return (x * l - b * l).abs()


def _fabs(op, x, b, l, sign, t):
    if op == OP_BCE:
        return ((1 - t) * x).abs() + (-x).clamp_min(0) + torch.log1p(torch.exp(-x.abs()))
    if op == OP_L1_MASK:
        return (x * l).abs() + (b * l).abs()
    return _expr(op, x, b, l, sign, t).abs()


def _dfabs(op, x, t, grad):
    """R_abs of one element's gradient, per unit coefficient where the derivative is not exact (BCE, MSE)."""
    if op == OP_BCE:
        return torch.sigmoid(x) + abs(t)
    if op == OP_SQ_T:
        return 2 * (x.abs() + abs(t))
    return None


MEASURED = {"fwd": 0.0, "bwd": 0.0}


def _run_op(name, op, a, b=None, label=None, sign=1.0, target=0.0, scale=None):
    """One term through mg_loss_reduce (slot 0, label sum in slot 1) and mg_loss_reduce_bwd; checks both against float64."""
    from michigan_b200 import _lib, ops
    from michigan_b200.networks.loss import _Spec, _device_table, _term
    lib = _lib.load()
    n = a.numel()
    if scale is None:
        scale = float(torch.tensor(-1.0 / (1.3 * n) if op != OP_L1_MASK else 0.9 / n, dtype=torch.float32))
    t32 = float(torch.tensor(target, dtype=torch.float32))
    spec = _Spec(op, 0, b, scale, sign, 0, target=t32, label=label)
    ga = torch.full_like(a, float("nan"))
    assert ga.stride() == a.stride()
    slots = torch.zeros(2, device=dev, dtype=torch.float64)
    tf = [_term(spec, a, b, None, 0, 1)]
    _lib.check(lib.mg_loss_reduce(_device_table(tf, a.device).data_ptr(), 1, slots.data_ptr(), ops._stream()), "mg_loss_reduce")
    gslot = 0.7
    gs = torch.tensor([gslot, 0.0], dtype=torch.float32, device=dev)
    tb = [_term(spec, a, b, ga.data_ptr(), 0, 1)]
    _lib.check(lib.mg_loss_reduce_bwd(_device_table(tb, a.device).data_ptr(), 1, gs.data_ptr(), ops._stream()), "mg_loss_reduce_bwd")
    x = d64(a).requires_grad_()
    bb = d64(b) if b is not None else None
    l = None
    if label is not None:
        l = d64(F.interpolate(label.float(), size=tuple(a.shape[2:]), mode="nearest"))
    f = _expr(op, x, bb, l, sign, t32)
    ref = f.sum() * scale
    rabs = _fabs(op, x.detach(), bb, l, sign, t32).sum() * abs(scale)
    k = _per_thread(n) + 8.0
    MEASURED["fwd"] = max(MEASURED["fwd"], check_close(name + " fwd", slots[0:1], ref.detach().view(1), rabs.view(1), k))
    if label is not None:
        assert float(slots[1]) == float(l.sum() * a.shape[1]), (name, float(slots[1]), float(l.sum() * a.shape[1]))
    # backward against float64 autograd of the reference expression
    (f.sum() * scale * gslot).backward()
    want = x.grad
    d = _dfabs(op, x.detach(), t32, want)
    r = want.abs() if d is None else abs(scale * gslot) * d
    MEASURED["bwd"] = max(MEASURED["bwd"], check_close(name + " bwd", ga, want, r, K_GA_BCE if op == OP_BCE else K_GA))
    return ga.cpu(), want, l, scale


BCE_SQ_CASES = [(op, shape, t, big) for op in (OP_BCE, OP_SQ_T)
                for shape, t, big in (((8, 1, 67, 67), 1.0, True), ((8, 1, 35, 35), 0.0, True), ((3, 1, 13, 7), 0.9, False),
                                      ((3, 1, 13, 7), 0.2, True), ((1, 1, 1, 1), 1.0, False))]


@pytest.mark.parametrize("op,shape,target,big", BCE_SQ_CASES)
def test_constant_target_ops(op, shape, target, big):
    name = "op%d %s t=%g%s" % (op, "x".join(map(str, shape)), target, " |x|<=100" if big else "")
    g = _gen(name)
    a = _logits(shape, g, big).to(dev)
    ga, _, _, scale = _run_op(name, op, a, target=target)
    assert bool(torch.isfinite(ga).all())
    if op == OP_BCE:
        # the BCE gradient is sigmoid(x) - t: at x = 0 exactly (0.5 - t) times the coefficient
        zero = a.cpu() == 0
        coef = torch.tensor(0.7, dtype=torch.float32) * torch.tensor(scale, dtype=torch.float32)
        assert bool((ga[zero] == coef * (0.5 - torch.tensor(target, dtype=torch.float32))).all())


# (op, N, C, h, w, H, W, mask, layout, sign)
MASK_CASES = [
    (OP_WSUM, 8, 1, 67, 67, 512, 512, "blob", "nchw", 1.0),
    (OP_WSUM, 8, 1, 35, 35, 512, 512, "blob", "nhwc", 1.0),
    (OP_HINGE_MASK, 8, 1, 67, 67, 512, 512, "blob", "nchw", 1.0),
    (OP_HINGE_MASK, 8, 1, 35, 35, 512, 512, "blob", "nchw", -1.0),
    (OP_HINGE_MASK, 3, 1, 13, 7, 48, 80, "empty", "nchw", 1.0),
    (OP_HINGE_MASK, 3, 1, 13, 7, 48, 80, "full", "nchw", -1.0),
    (OP_WSUM, 3, 1, 13, 7, 48, 80, "empty", "nchw", 1.0),
    (OP_HINGE_MASK, 2, 3, 17, 19, 48, 80, "blob", "nhwc", 1.0),
    (OP_WSUM, 2, 3, 17, 19, 48, 80, "blob", "nhwc", 1.0),
    (OP_L1_MASK, 8, 64, 129, 129, 512, 512, "blob", "nhwc", 1.0),
    (OP_L1_MASK, 2, 32, 35, 35, 512, 512, "blob", "nchw", 1.0),
    (OP_L1_MASK, 3, 5, 13, 7, 48, 80, "empty", "nhwc", 1.0),
    (OP_L1_MASK, 3, 5, 13, 7, 48, 80, "full", "nchw", 1.0),
    (OP_L1_MASK, 2, 7, 17, 19, 48, 80, "blob", "nhwc", 1.0),
]


@pytest.mark.parametrize("op,N,C,h,w,H,W,mask,layout,sign", MASK_CASES)
def test_masked_ops(op, N, C, h, w, H, W, mask, layout, sign):
    name = "op%d %dx%dx%dx%d from %dx%d %s %s sign %+g" % (op, N, C, h, w, H, W, mask, layout, sign)
    g = _gen(name)
    label = _label(N, H, W, mask, g)
    assert label.stride(0) == 3 * H * W
    x = _logits((N, C, h, w), g)
    b = None
    if op == OP_L1_MASK:
        bx = torch.randn(N, C, h, w, generator=g) * 2.0
        bx.view(-1)[::5] = x.view(-1)[::5]                            # a = b ties
        b = _on_device(bx, layout)
    a = _on_device(x, layout)
    ga, want, l, scale = _run_op(name, op, a, b, label, sign=sign)
    if mask == "empty":
        assert bool((ga == 0).all()), name
    if op == OP_HINGE_MASK:
        # a tie under the label gets half the gradient, and every masked-out element (a tie too) none
        le = l.expand_as(want)
        tie = ((sign * x.double() - 1) == 0) & (le != 0)
        if mask != "empty":
            assert int(tie.sum()) > 0
        gs = torch.tensor(0.7, dtype=torch.float32) * torch.tensor(scale, dtype=torch.float32)
        assert bool((ga[tie] == gs * (0.5 * sign) * le[tie].float()).all()), name
        assert bool((ga[(l == 0).expand_as(ga)] == 0).all()), name


# ---------------------------------------------------------------------------------------------------- whole classes
def _disc_outputs(n, g, layout):
    """pred_fake, pred_real as Pix2PixModel.discriminate slices them from one [2n] batch: two discriminators, features
    [16 @ 129^2, 32 @ 65^2] / [16 @ 65^2, 32 @ 33^2] and logits 67^2 / 35^2 (a 512^2 label)."""
    outs = []
    for sizes in (((16, 129), (32, 65), (1, 67)), ((16, 65), (32, 33), (1, 35))):
        d = []
        for c, s in sizes:
            t = _logits((2 * n, c, s, s), g) if c == 1 else torch.randn(2 * n, c, s, s, generator=g) * 1.5
            if c != 1:
                t[n:].view(-1)[::5] = t[:n].reshape(-1)[::5]
            d.append(_on_device(t, layout))
        outs.append(d)
    fake = [[t[:n] for t in p] for p in outs]
    real = [[t[n:] for t in p] for p in outs]
    return fake, real


def _d64_list(preds, grad=False):
    return [[d64(t).requires_grad_(grad) for t in p] for p in preds]


MEASURED_CLASS = {"loss": 0.0, "grad": 0.0}

CLASS_CASES = [  # (gan_mode, remove_background, target_is_real, for_discriminator, real_label, fake_label, mask, layout)
    ("original", False, True, True, 1.0, 0.0, "blob", "nhwc"), ("original", False, False, True, 0.9, 0.2, "blob", "nchw"),
    ("original", True, True, False, 1.0, 0.0, "blob", "nhwc"), ("ls", False, True, True, 0.9, 0.2, "blob", "nhwc"),
    ("ls", False, False, True, 1.0, 0.0, "blob", "nchw"), ("w", False, True, True, 1.0, 0.0, "blob", "nhwc"),
    ("w", False, False, True, 1.0, 0.0, "blob", "nhwc"), ("hinge", True, True, True, 1.0, 0.0, "blob", "nhwc"),
    ("hinge", True, False, True, 1.0, 0.0, "blob", "nchw"), ("hinge", True, True, False, 1.0, 0.0, "blob", "nhwc"),
    ("hinge", True, True, True, 1.0, 0.0, "empty", "nhwc"), ("hinge", True, False, True, 1.0, 0.0, "full", "nhwc"),
    ("hinge", False, True, True, 1.0, 0.0, "blob", "nhwc"),
]


@pytest.mark.parametrize("mode,rb,tir,fd,rl,fl,mask,layout", CLASS_CASES)
def test_gan_loss_class(mode, rb, tir, fd, rl, fl, mask, layout):
    import oracle_gan_objectives as og
    from michigan_b200.networks.loss import GANLoss
    from michigan_b200.options import make_opt
    name = "GANLoss %s rb=%d real=%d disc=%d targets %g/%g %s %s" % (mode, rb, tir, fd, rl, fl, mask, layout)
    g = _gen(name)
    n = 2
    fake, real = _disc_outputs(n, g, layout)
    preds = [[t.detach().requires_grad_(i == len(p) - 1) for i, t in enumerate(p)] for p in (real if tir else fake)]
    label = _label(n, 512, 512, mask, g)
    opt = make_opt(remove_background=rb, wide_edge=2.0)
    crit = GANLoss(mode, target_real_label=rl, target_fake_label=fl, opt=opt)
    loss = crit(preds, tir, for_discriminator=fd, label=label)
    assert tuple(loss.shape) == (1,)
    loss.sum().backward()
    p64 = [[d64(t).requires_grad_(i == len(p) - 1) for i, t in enumerate(p)] for p in preds]
    lab64 = d64(label)
    ref = og.gan_loss(p64, tir, fd, lab64, mode, 2.0, rb, rl, fl)
    ref.sum().backward()
    # R_abs: every scale's terms on absolute values, with its coefficient
    num = len(p64)
    rabs = 0.0
    for p in p64:
        x = p[-1].detach()
        t = float(torch.tensor(rl if tir else fl, dtype=torch.float32))
        sign = 1.0 if tir else -1.0
        if mode == "original":
            rabs += _fabs(OP_BCE, x, None, None, 1.0, t).mean() / num
        elif mode == "ls":
            rabs += ((x - t) ** 2).mean() / num
        elif mode == "w" or (mode == "hinge" and not rb and not fd):
            rabs += x.abs().mean() / num
        elif not rb:
            rabs += 2.0 * torch.min(sign * x - 1, torch.zeros_like(x)).abs().mean() / num
        else:
            l = og.resized_label(lab64, x)
            f = (x * l).abs() if not fd else ((sign * x - 1) * l).abs()
            rabs += f.sum() / (l.sum() * x.shape[1] + 1e-5) / num
    MEASURED_CLASS["loss"] = max(MEASURED_CLASS["loss"], check_close(name + " loss", loss.detach(), ref.detach(), rabs.view(1), K_CLASS))
    for p, q in zip(preds, p64):
        x, gref = q[-1].detach(), q[-1].grad
        if mode in ("original", "ls"):
            t = float(torch.tensor(rl if tir else fl, dtype=torch.float32))
            r = (torch.sigmoid(x) + abs(t) if mode == "original" else 2 * (x.abs() + abs(t))) / (x.numel() * num)
        else:
            r = gref.abs()
        k = K_GA_BCE if mode == "original" else K_GA
        MEASURED_CLASS["grad"] = max(MEASURED_CLASS["grad"], check_close(name + " grad", p[-1].grad, gref, r, k))
        if rb and mask == "empty":
            assert float(loss) == 0.0 and bool((p[-1].grad == 0).all())


@pytest.mark.parametrize("rb,mask,layout", [(False, "blob", "nhwc"), (True, "blob", "nhwc"), (True, "blob", "nchw"),
                                            (True, "empty", "nhwc"), (True, "full", "nchw")])
def test_gan_feat_loss_class(rb, mask, layout):
    import oracle_gan_objectives as og
    from michigan_b200.networks.loss import GANFeatLoss
    from michigan_b200.options import make_opt
    name = "GANFeatLoss rb=%d %s %s" % (rb, mask, layout)
    g = _gen(name)
    n = 2
    fake, real = _disc_outputs(n, g, layout)
    fake = [[t.detach().requires_grad_() for t in p] for p in fake]
    label = _label(n, 512, 512, mask, g)
    lam = 10.0
    crit = GANFeatLoss(make_opt(remove_background=rb, lambda_feat=lam))
    loss = crit(fake, real, label)
    loss.sum().backward()
    f64 = [[d64(t).requires_grad_() for t in p] for p in fake]
    r64 = _d64_list(real)
    lab64 = d64(label)
    ref = og.gan_feat_loss(f64, r64, lab64, lam, rb)
    ref.sum().backward()
    rabs = 0.0
    for pf, pr in zip(f64, r64):
        for f, r in zip(pf[:-1], pr[:-1]):
            if rb:
                l = og.resized_label(lab64, f)
                rabs += ((f.detach() * l).abs() + (r * l).abs()).sum() / (l.sum() * f.shape[1] + 1e-5) * lam / len(f64)
            else:
                rabs += (f.detach().abs() + r.abs()).mean() * lam / len(f64)
    MEASURED_CLASS["loss"] = max(MEASURED_CLASS["loss"], check_close(name + " loss", loss.detach(), ref.detach(), rabs.view(1), K_CLASS))
    for pf, pq in zip(fake, f64):
        for t, q in zip(pf[:-1], pq[:-1]):
            MEASURED_CLASS["grad"] = max(MEASURED_CLASS["grad"], check_close(name + " grad", t.grad, q.grad, q.grad.abs(), K_GA))
            if rb and mask == "empty":
                assert bool((t.grad == 0).all())
    if rb and mask == "empty":
        assert float(loss) == 0.0


def test_report_measured(capsys):
    """Prints the largest measured ratios of the cases run before it in this module."""
    print("measured: fwd %.3g bwd %.3g class loss %.3g class grad %.3g" % (MEASURED["fwd"], MEASURED["bwd"], MEASURED_CLASS["loss"],
                                                                           MEASURED_CLASS["grad"]))
