"""--remove_background in the VGG, content and style losses on the sm_90a kernels: mg_loss_reduce op 9 (masked squared
difference) and op 10 (masked channel moments), the accumulating backward (LossTerm.add) and the masked mode of
mg_style_loss_fwd, held element by element to float64 autograd of the reference's expressions (models/networks/loss.py:187-207,
634-711) fed the kernels' exact fp32 inputs; then VGGLoss and StyleContentLoss against the fp32 oracle
(tests/oracle_remove_background.py, pinned to the reference by tests/test_oracle_remove_background.py).

Error model, as tests/test_gpu_style_content.py: |got - ref| <= k u R_abs, u = 2^-24, R_abs the same computation on absolute
values.  Labels are the hair channel of a one-hot map (a non-contiguous view, image stride 3 H W), read through the nearest
resize from 512^2 (or 64^2) to taps of 512 ... 32 (... 4); dead (all-zero) and constant channels; empty and full masks; the
fake and target taps masked by different labels.  Each case prints its measured max |err| / (u R_abs).  Bounds, and the largest
value measured on an H100 80GB HBM3 (700 W power limit):

  * op 9 forward: k = L + 8 (L the most elements one thread adds in fp32), measured 0.02; label slot exact.  Backward with
    add: K_GA = 10 on |add| + |g| 2 (|a l| + |b l|) l (the products a l, b l, their difference, the factors 2, l and g, and
    the add: about 6 roundings), measured 3.11.
  * op 10 forward: K_MOM = 40 (fp32 runs of at most 32 elements, the square's rounding), measured 1.62; per-image label sums
    exact.
  * masked style loss (op 10 -> mg_style_loss_fwd masked): K_STYLE_LOSS = 8 on sum over taps of ((|mu_f| + |mu_t|)^2 +
    (sigma_f + sigma_t)^2) / (N C), measured 0.81; d tap (op 10 backward adding onto `add`): K_STYLE_GRAD = 16 on |add| + g l
    (2 (|mu_f| + |mu_t|) + 2 (sigma_f + sigma_t) / sigma_f (|a| + |mu'|)) / (N C (D + eps)), measured 2.34.
  * whole modules against the oracle, the bounds of the unmasked tests: VGG loss rel 2e-3 (measured 7.4e-5), d fake cosine
    0.99 (measured at least 0.9929); content and style rel 1e-3 (measured 3.3e-4), cosine 0.98 (measured at least 0.9940).
"""
import math

import pytest
import torch

import oracle_remove_background as orb
from test_gpu_loss_kernels_fp64 import TINY, U, check_close

pytestmark = pytest.mark.gpu

dev = "cuda"
LOSS_BLOCKS, LOSS_THREADS = 592, 256
K_GA = 10.0
K_MOM = 40.0
K_STYLE_LOSS = 8.0
K_STYLE_GRAD = 16.0
OP_SQ_MASK, OP_MOMENTS = 9, 10


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _label(n, H, W, kind, g):
    """The hair channel of an [n,3,H,W] one-hot map (a view, image stride 3 H W): an ellipse per image plus specks, or all 0
    ('empty'), all 1 ('full'), or image 0 empty and image 1 an ellipse ('half')."""
    yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    hair = torch.zeros(n, H, W)
    for i in range(n):
        cy, cx = H * (0.3 + 0.4 * float(torch.rand(1, generator=g))), W * (0.3 + 0.4 * float(torch.rand(1, generator=g)))
        hair[i] = ((((yy - cy) / (0.3 * H)) ** 2 + ((xx - cx) / (0.25 * W)) ** 2) <= 1).float()
    hair = torch.maximum(hair, (torch.rand(n, H, W, generator=g) < 0.02).float())
    if kind == "empty":
        hair.zero_()
    elif kind == "full":
        hair.fill_(1.0)
    elif kind == "half":
        hair[0] = 0.0
    seg = torch.stack([1 - hair, hair, torch.zeros_like(hair)], 1).to(dev)
    return seg[:, 1:2]


def _feature(shape, g):
    """ReLU-like NHWC fp32 tap with a dead channel 0 and a constant channel 1."""
    f = torch.relu(torch.randn(shape, generator=g) * 0.8 + 0.2)
    f[..., 0] = 0.0
    f[..., 1] = 0.37
    return f.to(dev)


def _tap_shapes(n, size):
    return [(n, size, size, 64), (n, size // 2, size // 2, 128), (n, size // 4, size // 4, 256), (n, size // 8, size // 8, 512),
            (n, size // 16, size // 16, 512)]


def _resized(label, tap):
    """[N,1,h,w] float64 nearest resize of the label to an NHWC tap, as NHWC [N,h,w,1]."""
    return torch.nn.functional.interpolate(label.double(), size=tap.shape[1:3], mode="nearest").permute(0, 2, 3, 1)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _launch(terms, nslots=None, gslots=None):
    from michigan_b200 import _lib, ops
    from michigan_b200.networks.loss import _device_table
    lib = _lib.load()
    table = _device_table(terms, torch.device(dev))
    if gslots is None:
        slots = torch.zeros(nslots, device=dev, dtype=torch.float64)
        _lib.check(lib.mg_loss_reduce(table.data_ptr(), len(terms), slots.data_ptr(), ops._stream()), "mg_loss_reduce")
        return slots
    _lib.check(lib.mg_loss_reduce_bwd(table.data_ptr(), len(terms), gslots.data_ptr(), ops._stream()), "mg_loss_reduce_bwd")


def _spec(op, label, scale=1.0):
    from michigan_b200.networks.loss import _Spec, _hair_label
    return _Spec(op, 0, None, scale, 1.0, 0, label=_hair_label(label, torch.empty(label.shape[0], 1, 1, 1)))


# ------------------------------------------------------------------------------------------------ op 9
OP9_CASES = [  # (N, label size, tap NHWC shape, label kind)
    (2, 512, (2, 32, 32, 512), "hair"),
    (2, 512, (2, 64, 64, 512), "half"),
    (2, 64, (2, 4, 4, 512), "empty"),
    (2, 64, (2, 4, 4, 512), "full"),
    (3, 48, (3, 5, 7, 8), "hair"),
]


@pytest.mark.parametrize("case", OP9_CASES, ids=lambda c: "%s_%dx%s" % (c[3], c[1], "x".join(map(str, c[2]))))
def test_op9_masked_squared_difference_vs_fp64(case):
    from michigan_b200.networks.loss import _term
    n, L, shape, kind = case
    g = _gen(sum(shape) + L)
    lab = _label(n, L, L, kind, g)
    a, b = _feature(shape, g), _feature(shape, g) * 1.1
    b[0, 0, 0] = a[0, 0, 0]                                      # ties: zero contribution, zero gradient
    sp = _spec(OP_SQ_MASK, lab, scale=0.75)
    slots = _launch([_term(sp, _nchw(a), b, None, 0, 1)], nslots=2)
    add = torch.randn(shape, generator=g).to(dev) * 1e-3
    ga = add.clone()
    gv = torch.tensor([1.3], device=dev)
    _launch([_term(sp, _nchw(a), b, ga.data_ptr(), 0, 1, add=ga.data_ptr())], gslots=gv)
    torch.cuda.synchronize()
    l = _resized(lab, a)
    x = a.double().requires_grad_()
    ref = 0.75 * ((x * l - b.double() * l) ** 2).sum()
    (1.3 * ref).backward()
    rabs = 0.75 * float((((a.double() * l).abs() + (b.double() * l).abs()) ** 2).sum())
    k = -(-a.numel() // (LOSS_BLOCKS * LOSS_THREADS)) + 8
    r = abs(float(slots[0]) - float(ref)) / (U * rabs + TINY)
    assert float(slots[1]) == float(l.sum()) * shape[3]
    rg = check_close("op 9 d a", ga, add.double() + x.grad,
                     add.double().abs() + 1.3 * 0.75 * 2 * ((a.double() * l).abs() + (b.double() * l).abs()) * l, K_GA)
    print("op 9 %s: fwd |err| / (u R_abs) %.2f (k %d), bwd %.2f" % (case, r, k, rg))
    assert r <= k


# ------------------------------------------------------------------------------------------------ op 10
def _moments_fp64(a, l):
    """(sum l a, sum l a^2) per (n, c) -> [N,2,C] and sum l per image -> [N], float64, l [N,h,w,1]."""
    ad = a.double()
    return torch.stack([(ad * l).sum((1, 2)), (ad * ad * l).sum((1, 2))], 1), l.sum((1, 2, 3))


def _moment_terms(pairs, offs):
    from michigan_b200.networks.loss import _term
    return [_term(_spec(OP_MOMENTS, lab), _nchw(a), None, None, o, o + 2 * a.shape[0] * a.shape[3]) for (a, lab), o in zip(pairs, offs)]


def _offsets(taps):
    offs, o = [], 0
    for t in taps:
        offs.append(o)
        o += 2 * t.shape[0] * t.shape[3] + t.shape[0]
    return offs, o


@pytest.mark.parametrize("n,L,size,kind", [(2, 512, 512, "hair"), (2, 512, 512, "half"), (2, 64, 64, "empty"), (2, 64, 64, "full"),
                                           (1, 48, 32, "hair")])
def test_op10_masked_moments_vs_fp64(n, L, size, kind):
    g = _gen(n * 7 + L + size)
    lab = _label(n, L, L, kind, g)
    taps = [_feature(s, g) for s in _tap_shapes(n, size)]
    offs, total = _offsets(taps)
    slots = _launch(_moment_terms([(t, lab) for t in taps], offs), nslots=total)
    torch.cuda.synchronize()
    worst = 0.0
    for t, o in zip(taps, offs):
        N, h, w, c = t.shape
        l = _resized(lab, t)
        sums, cnt = _moments_fp64(t, l)
        got = slots[o:o + 2 * N * c].view(N, 2, c)
        worst = max(worst, check_close("op 10 %s" % (tuple(t.shape),), got, sums, torch.stack([sums[:, 0].abs(), sums[:, 1]], 1), K_MOM))
        assert torch.equal(slots[o + 2 * N * c:o + 2 * N * c + N].cpu(), cnt.cpu()), (t.shape, kind)
    print("op 10 n=%d %d^2 -> %d^2 %s: max |err| / (u R_abs) %.2f" % (n, L, size, kind, worst))


# ------------------------------------------------------------------------------------------------ masked style, end to end
def _style_fp64(fs, ts, lf, lt, gs):
    """float64 autograd of gs * sum_i MSE(mu_f, mu_t) + MSE(sigma_f, sigma_t) with calc_mean_std_mask's expressions (fake masked
    by lf, targets by lt) on NHWC taps -> (loss, [d f_i], per tap (mu_f, mu_t, sigma_f, sigma_t, D_f, mu'))."""
    xs = [f.double().requires_grad_() for f in fs]
    loss = 0
    stats = []
    for x, t, mf_, mt_ in zip(xs, ts, lf, lt):
        def ms(feat, m):
            f = feat * m
            mean = f.sum((1, 2)) / (m.sum((1, 2)) + 1e-5)
            var = (((f - mean[:, None, None, :]) * m) ** 2).sum((1, 2)) / (m.sum((1, 2)) + 1e-5) + 1e-5
            return mean, var.sqrt()
        mu_f, s_f = ms(x, mf_)
        mu_t, s_t = ms(t.double(), mt_)
        loss = loss + ((mu_f - mu_t) ** 2).mean() + ((s_f - s_t) ** 2).mean()
        D = mf_.sum((1, 2))
        stats.append((mu_f.detach(), mu_t, s_f.detach(), s_t, D, mu_f.detach() * (1 + 1e-5 / (D + 1e-5))))
    (gs * loss).backward()
    return float(loss), [x.grad for x in xs], stats


@pytest.mark.parametrize("n,L,size,kinds", [(2, 512, 512, ("hair", "hair")), (2, 512, 512, ("half", "hair")), (2, 64, 64, ("hair", "empty")),
                                            (2, 64, 64, ("full", "full")), (1, 48, 16, ("hair", "hair"))])
def test_masked_style_loss_and_tap_gradient_vs_fp64(n, L, size, kinds):
    """op 10 over fake || target -> mg_style_loss_fwd (masked) -> op 10 backward adding onto the VGG-L1 gradient, with the
    fake masked by one label and the target by another (the reference's crossing); size 16 gives a 1x1 relu5_1 map, which
    the masked (biased) statistics accept."""
    from michigan_b200 import ops
    from michigan_b200.networks.loss import _term
    g = _gen(n * 11 + L + size + len(kinds[0]))
    lab_f, lab_t = _label(n, L, L, kinds[0], g), _label(n, L, L, kinds[1], g)
    shapes = _tap_shapes(n, size)
    fs = [_feature(s, g) for s in shapes]
    ts = [_feature(s, g) * 1.3 for s in shapes]
    adds = [torch.randn(s, generator=g).to(dev) * 1e-4 for s in shapes]
    gs = 1.7
    res = []
    for _ in range(2):
        pairs = [p for f, t in zip(fs, ts) for p in ((f, lab_f), (t, lab_t))]
        offs, total = _offsets([p[0] for p in pairs])
        slots = _launch(_moment_terms(pairs, offs), nslots=total)
        recs = []
        for k, s in enumerate(shapes):
            fo, to, N, c = offs[2 * k], offs[2 * k + 1], s[0], s[3]
            recs.append((slots[fo:fo + 2 * N * c].view(N, 2, c), slots[to:to + 2 * N * c].view(N, 2, c), s[1] * s[2],
                         slots[fo + 2 * N * c:fo + 2 * N * c + N], slots[to + 2 * N * c:to + 2 * N * c + N]))
        loss, coefs = ops.style_loss_fwd(recs)
        grads = [a.clone() for a in adds]
        terms = [_term(_spec(OP_MOMENTS, lab_f), _nchw(f), coefs[k], grads[k].data_ptr(), 0, 0, add=grads[k].data_ptr())
                 for k, f in enumerate(fs)]
        _launch(terms, gslots=torch.tensor([gs], device=dev))
        torch.cuda.synchronize()
        res.append((loss.clone(), grads))
    assert torch.equal(res[0][0], res[1][0]) and all(torch.equal(a, b) for a, b in zip(res[0][1], res[1][1]))
    loss, grads = res[0]
    lf = [_resized(lab_f, f) for f in fs]
    lt = [_resized(lab_t, f) for f in fs]
    ref, ref_g, stats = _style_fp64(fs, ts, lf, lt, gs)
    r_loss, worst = 0.0, 0.0
    for k, (f, a, (mu_f, mu_t, s_f, s_t, D, mup)) in enumerate(zip(fs, adds, stats)):
        NC = f.shape[0] * f.shape[3]
        r_loss += float(((mu_f.abs() + mu_t.abs()) ** 2 + (s_f + s_t) ** 2).mean())
        e = (NC * (D + 1e-5))[:, None, None, :]
        rs = (2 * (mu_f.abs() + mu_t.abs()))[:, None, None, :] / e + \
            (2 * (s_f + s_t) / s_f)[:, None, None, :] / e * (f.double().abs() + mup.abs()[:, None, None, :])
        rabs = a.double().abs() + gs * lf[k] * rs
        worst = max(worst, check_close("style tap %d" % k, grads[k], a.double() + ref_g[k], rabs, K_STYLE_GRAD))
        if kinds[0] in ("empty", "half"):
            assert torch.equal(grads[k][0], adds[k][0])              # no fake hair in image 0: no style gradient there
    rl = abs(float(loss) - ref) / (U * r_loss)
    print("masked style N=%d %d^2 -> %d^2 %s: loss %.8e fp64 %.8e |err| / (u R_abs) %.2f; worst d tap %.2f"
          % (n, L, size, kinds, float(loss), ref, rl, worst))
    assert math.isfinite(float(loss)) and rl <= K_STYLE_LOSS


def test_accumulating_backward_leaves_unmasked_ops_unchanged():
    """add null writes exactly what the parent wrote (g f'); add set adds onto it, bit for bit g f' + add in fp32."""
    from michigan_b200.networks.loss import OP_L1, OP_SQ, _Spec, _term
    g = _gen(5)
    a = torch.randn(3, 1000, generator=g).to(dev)
    b = torch.randn(3, 1000, generator=g).to(dev)
    add = torch.randn(3, 1000, generator=g).to(dev)
    for op in (OP_L1, OP_SQ):
        sp = _Spec(op, 0, b, 1.0 / a.numel(), 1.0, 0)
        plain, acc = torch.empty_like(a), add.clone()
        gv = torch.tensor([0.7], device=dev)
        _launch([_term(sp, a, b, plain.data_ptr(), 0, 0)], gslots=gv)
        _launch([_term(sp, a, b, acc.data_ptr(), 0, 0, add=acc.data_ptr())], gslots=gv)
        torch.cuda.synchronize()
        assert torch.equal(acc, add + plain), op


# ------------------------------------------------------------------------------------------------ modules against the oracle
@pytest.fixture
def fp32_cudnn():
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def _cos(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float(a @ b / (a.norm() * b.norm()))


@pytest.mark.parametrize("case", ["crossed", "no_tag_hair", "no_ref_hair", "full"])
@pytest.mark.parametrize("mode", ["mixed16", "tf32"])
def test_remove_background_modules_vs_oracle(case, mode, fp32_cudnn):
    from michigan_b200 import precision
    from michigan_b200.networks import StyleContentLoss, VGGLoss
    from michigan_b200.options import make_opt
    from michigan_b200.synth import vgg19_state_dict
    from test_oracle_remove_background import _inputs, oracle_terms
    sd = vgg19_state_dict(0)
    fake, ref, tag, lab_ref, lab_tag = _inputs(case)
    ref, tag, lab_ref, lab_tag = ref.cuda(), tag.cuda(), lab_ref.cuda(), lab_tag.cuda()
    old = precision.mode()
    precision.set_mode(mode)
    try:
        opt = make_opt(remove_background=True, mask_vgg_losses=True)
        vgg = VGGLoss(opt, state_dict=sd)
        sc = StyleContentLoss(opt, vgg=vgg.vgg)
        got = {}
        for name in ("vgg", "content", "style"):
            x = fake.cuda().requires_grad_()
            loss = vgg(x, tag, lab_tag) if name == "vgg" else sc(x, ref, tag, lab_ref, lab_tag)[name == "style"]
            loss.backward()
            got[name] = (float(loss), x.grad.clone())
        torch.cuda.synchronize()
    finally:
        precision.set_mode(old)
    sdc = {k: v.cuda() for k, v in sd.items()}
    for name, fn in oracle_terms(sdc, fake.cuda(), ref, tag, lab_ref, lab_tag).items():
        xr = fake.cuda().requires_grad_()
        want = fn(xr)
        want.backward()
        rel = abs(got[name][0] - float(want)) / abs(float(want))
        cos = _cos(got[name][1], xr.grad)
        print("%s %s %s: loss %.7f oracle %.7f rel %.2e; d fake cosine %.6f" % (case, mode, name, got[name][0], float(want), rel, cos))
        assert torch.isfinite(got[name][1]).all()
        assert rel <= (2e-3 if name == "vgg" else 1e-3), name
        assert cos >= (0.99 if name == "vgg" else 0.98), name
