"""The loss kernels of the generator and discriminator objectives, called directly and compared element by element with a
float64 CPU reference of the operation they compute, fed the kernels' exact fp32 inputs:

  * fused loss reductions   loss_reduce_kernel / loss_reduce_bwd_kernel (mg_loss_reduce, mg_loss_reduce_bwd): every hinge,
                            generator-hinge, GAN-feature, VGG L1 and content term, through descriptor tables built here
  * Gabor orientation loss  orient_fwd_kernel / orient_bwd_kernel (mg_orient_loss_fwd, mg_orient_loss_bwd)
  * Lab colour loss         lab_loss_fwd_kernel / lab_loss_bwd_kernel (mg_lab_loss_fwd, mg_lab_loss_bwd)
  * SPADE segmap MLP        seg_mlp_tc_kernel, pack_weight_seg_tc_kernel (mg_conv_seg_tc, mg_pack_weight_seg_tc)
  * generator output conv   conv_img (mg_conv_img)
  * input prologue, h != w  noise_pyramid_kernel, orient_rgb_kernel, hole_mask_kernel (mg_noise_pyramid, mg_orient_rgb,
                            mg_hole_mask)

Error model, where something sums:

    |got - ref| <= k * u * R_abs + tiny,      u = 2^-24,

R_abs = the same formula on absolute values.  Each case prints its measured max |got - ref| / (u R_abs) next to k.  Where a
bound is composed of several terms (the orientation loss's per-pixel outputs), the case prints the measured error as a
fraction of the bound instead.  Measured on an H100 80GB HBM3 (700 W power limit):

  * loss_reduce forward: k = L + 2, L the largest number of elements one thread adds in fp32 (from the launch geometry,
    592 blocks x 256 threads, 4 elements per trip on the float4 path), a worst-case bound: k = 3 .. 227, measured at most
    0.97 (k = 6, n = 4, a one-pass sum of 4 values).
  * loss_reduce backward: bit-exact against fp32 (gslot * scale) * f'(a).  At an exact tie the reference's derivative:
    0.5 sign w for the hinge (torch's binary min splits the gradient), 0 for |a - b| and (a - b)^2.  Also against float64
    autograd of the reference expression: measured 2.6, K_GA64 = 8.
  * Gabor responses: K_RESP = 1.25 sqrt(289) + 8 on R_abs = sum |gray| |K|.  The arg-max index must be admissible (within
    2 K_RESP u R_abs of the best clamped response; the chosen filter was at most 0.53 u R_abs below the best);
    dmax_l1, dmax_log and the three sums are recomputed in float64 from the kernel's index and held to the response bound
    propagated through tanh (|d^2 conf / d mx^2| <= 2 / (3 sqrt 3)): measured at most 0.15 of that bound.
  * Gabor backward: K_ORIENT_BWD = 36 on R_abs = coef 127.5 sum |g| |K|, with g's own fp32 rounding carried in R_abs;
    measured 10.4.
  * Lab: K_LAB = 16 per pixel on R_abs = 500 (|f_X| + |f_Y|) (a), 200 (|f_Y| + |f_Z|) (b) over fake and real, the chain
    rule with magnitudes for d fake; either branch of f where t is within the bound of the threshold (the branches differ by
    29 u in f and 650 u in f' there), either sign where |da| or |db| is.  Measured: d fake 4.4, the forward sum 0.03.
  * segmap MLP: the weight operand bit for bit against [W_hi | W_hi | W_lo | 0]; the output against float64 of exactly the
    three bf16 products the kernel forms, plus bias and act, K_SEG = 20 (measured 5.9); round_out, the 16-bit copies and the
    16-bit-only outputs under both epilogues bit for bit against the fp32 output.
  * conv_img: k = 1.25 sqrt(9 Cin) + 8 before tanh, carried through it (measured 6.1 against k = 38 at Cin 64).
  * noise pyramid: float64 INTER_LINEAR, bounded by each coordinate's fp32 rounding times the slopes plus the lerps'
    roundings (measured at most 0.25 of that bound); hole_mask bit for bit, orient_rgb too except within 1e-9 of
    an integer before truncation.
"""
import itertools
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

dev = "cuda"
U = 2.0 ** -24
TINY = 1e-30
# fused loss reductions (csrc/mg_loss.cu): grid (592, terms) x 256 threads
LOSS_BLOCKS, LOSS_THREADS = 592, 256
# float64 autograd of the reference expression against the kernel's fp32 gradient: three roundings (gslot * scale, a - b,
# the product) bound the error by 3 u |grad|; measured 2.6 (op 3), so k = 8 keeps 3x over the measurement.
K_GA64 = 8.0
# Gabor: sqrt(K) model of the 289-tap fp32 fma chain (as the conv tests), + 8 for gray's rounding and the epilogue
K_RESP = 1.25 * math.sqrt(289) + 8
# the backward gather sums up to 289 fma terms of both signs per pixel; measured 10.4 (2 x 512^2), k = 36 keeps 3x over it
K_ORIENT_BWD = 36.0
D2CONF = 2.0 / (3.0 * math.sqrt(3.0))          # max |d^2 conf / d mx^2|, conf = (tanh(mx) + 1) / 2
# Lab: (img + 1) / 2, three products and two adds, the row-sum division, powf (<= 4 ulp) or the linear branch, the
# differences and scales of a / b, or f' and the chain rule's products and sums
K_LAB = 16.0


def d64(t):
    return t.detach().cpu().double()


def check_close(name, got, ref, rabs, k, u=U):
    """|got - ref| <= k * u * rabs + TINY for every element; returns the measured max |got - ref| / (u R_abs)."""
    got, ref, rabs = d64(got), d64(ref), d64(rabs)
    assert got.shape == ref.shape == rabs.shape, (name, got.shape, ref.shape, rabs.shape)
    assert bool(torch.isfinite(got).all()), name
    err = (got - ref).abs()
    ratio = float((err / (u * rabs + TINY)).max()) if err.numel() else 0.0
    print("%s: max |got - ref| / (u R_abs) = %.3g (k = %g)" % (name, ratio, k))
    bad = err > k * u * rabs + TINY
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d elements out of bound; max ratio %.3g > k = %g; first at %s: got %r ref %r R_abs %r"
                             % (name, int(bad.sum()), bad.numel(), ratio, k, i, float(got[i]), float(ref[i]), float(rabs[i])))
    return ratio


def check_within(name, err, bound):
    """err <= bound + TINY element-wise (both float64, the bound composed per element); prints max err / bound."""
    ratio = float((err / (bound + TINY)).max()) if err.numel() else 0.0
    print("%s: max |got - ref| / bound = %.3g (must be <= 1)" % (name, ratio))
    bad = err > bound + TINY
    if bool(bad.any()):
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d elements out of bound (max ratio %.3g); first at %s: err %r bound %r"
                             % (name, int(bad.sum()), bad.numel(), ratio, i, float(err[i]), float(bound[i])))
    return ratio


def _bits(t):
    return t.view(torch.int64) if t.dtype == torch.float64 else t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def same_bits(name, a, b):
    a, b = a.detach().cpu(), b.detach().cpu()
    assert a.shape == b.shape and a.dtype == b.dtype, (name, a.shape, b.shape, a.dtype, b.dtype)
    neq = _bits(a) != _bits(b)
    if bool(neq.any()):
        i = tuple(neq.nonzero()[0].tolist())
        raise AssertionError("%s: %d of %d elements differ, first at %s: got %r want %r"
                             % (name, int(neq.sum()), neq.numel(), i, float(a[i]), float(b[i])))


def _gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def _lib():
    from michigan_b200 import _lib
    return _lib


def _ops():
    from michigan_b200 import ops
    return ops


# ============================================================================================== fused loss reductions
OP_HINGE_D, OP_SUM, OP_L1, OP_SQ = 0, 1, 2, 3


def T(op, n, slot=0, sign=1.0, w=False, a_off=0, b_off=0, ga=True, ties=True):
    """One term of a test table: op, n elements, output slot, hinge sign, weight map (op 0), a / b offset in floats (an
    offset of 1-3 floats sends the term down the scalar path), gradient wanted, planted ties."""
    return dict(op=op, n=n, slot=slot, sign=sign, w=w, a_off=a_off, b_off=b_off, ga=ga, ties=ties)


BIG = 33554432 + 5        # the finest VGG19 tap at batch 8, 512^2 (64 x 256^2 x 8 x 2 = 2^25), plus a ragged tail
ONE_PASS = LOSS_BLOCKS * LOSS_THREADS * 4
LOSS_CASES = {
    "hinge_real_weighted": [T(0, 1023, sign=1.0, w=True)],
    "hinge_fake_weighted": [T(0, 1023, sign=-1.0, w=True)],
    "hinge_real_n5": [T(0, 5, sign=1.0)],
    "hinge_fake_n3": [T(0, 3, sign=-1.0)],
    "hinge_n1_tie": [T(0, 1, sign=1.0)],
    "gen_hinge_n4": [T(1, 4)],
    "l1_n3": [T(2, 3)],
    "sq_n1": [T(3, 1)],
    "l1_one_pass": [T(2, ONE_PASS)],
    "l1_one_pass_plus_1": [T(2, ONE_PASS + 1)],
    "hinge_one_pass_plus_1": [T(0, ONE_PASS + 1, sign=-1.0, w=True)],
    "l1_sq_34M": [T(2, BIG, slot=0), T(3, BIG, slot=1)],
    "a_off1_l1": [T(2, 4099, a_off=1)],
    "a_off2_sq": [T(3, 1023, a_off=2)],
    "a_off3_hinge": [T(0, 1023, a_off=3, sign=1.0, w=True)],
    "a_off1_sum_one_pass_plus_1": [T(1, ONE_PASS + 1, a_off=1)],
    "b_off1_l1": [T(2, 4096, b_off=1)],
    "b_off3_sq": [T(3, 1025, b_off=3)],
    "table_7_terms_3_slots": [T(0, 4489, slot=0, sign=1.0, w=True), T(0, 1225, slot=0, sign=-1.0, w=True, a_off=1, ga=False),
                              T(2, 65536, slot=1), T(2, 1001, slot=1, b_off=2), T(3, 777, slot=2, ga=False),
                              T(1, 9, slot=2, a_off=3), T(3, 20000, slot=2)],
}


def _max_per_thread(n, vec):
    """L: the most elements one thread of loss_reduce_kernel adds in fp32 (float4 trips, then the scalar tail)."""
    stride = LOSS_BLOCKS * LOSS_THREADS
    if vec:
        n4 = n // 4
        return 4 * -(-n4 // stride) + (1 if n % 4 else 0)
    return -(-n // stride)


def _f64(op, a, b, sign):
    if op == OP_HINGE_D:
        return torch.clamp(sign * a - 1.0, max=0.0) * (b if b is not None else 1.0)
    if op == OP_SUM:
        return a
    if op == OP_L1:
        return (a - b).abs()
    return (a - b) ** 2


def _d_f32(op, a, b, sign):
    """f'(a) in fp32 as loss_reduce_bwd_kernel forms it; at a tie the reference's (torch's) derivative."""
    if op == OP_HINGE_D:
        m = sign * a - 1.0
        w = b if b is not None else torch.ones_like(a)
        sw = sign * w
        return torch.where(m < 0, sw, torch.where(m == 0, (0.5 * sign) * w, torch.zeros_like(a)))
    if op == OP_SUM:
        return torch.ones_like(a)
    if op == OP_L1:
        return torch.sign(a - b)
    return 2.0 * (a - b)


def _ref_expr(op, x, b, sign):
    """The reference's own expression per element (loss.py:92-100, 123-124, l1_loss, mse), differentiable in float64."""
    if op == OP_HINGE_D:
        m = torch.min(sign * x - 1, torch.zeros_like(x))
        return m * b if b is not None else m
    if op == OP_SUM:
        return x
    if op == OP_L1:
        return (x - b).abs()
    return (x - b) ** 2


@pytest.mark.parametrize("case", list(LOSS_CASES))
def test_loss_reduce_fwd_bwd(case):
    from michigan_b200.networks.loss import _Term, _device_table
    lib = _lib().load()
    ops = _ops()
    g = _gen(case)
    spec = LOSS_CASES[case]
    nslots = max(t["slot"] for t in spec) + 1
    terms_f, terms_b, host, keep = [], [], [], []
    gap = 4
    total = sum(t["n"] + gap for t in spec)
    sentinel = torch.tensor([0x7FC0DEAD], dtype=torch.int32).view(torch.float32)
    flat = sentinel.to(dev).repeat(total)
    off = 0
    for t in spec:
        n, op = t["n"], t["op"]
        a = torch.randn(n, generator=g) * 1.5
        b = None
        if op in (OP_L1, OP_SQ):
            b = torch.randn(n, generator=g) * 1.5
            if t["ties"]:
                b[::5] = a[::5]
        elif op == OP_HINGE_D and t["w"]:
            b = 1.0 + 2.0 * torch.rand(n, generator=g)
            b[::11] = 1.0
        if op == OP_HINGE_D and t["ties"]:
            a[::7] = t["sign"]                          # sign * a - 1 == 0 exactly
        da = torch.zeros(n + 4, device=dev)[t["a_off"]:t["a_off"] + n]
        da.copy_(a.to(dev))
        db = None
        if b is not None:
            db = torch.zeros(n + 4, device=dev)[t["b_off"]:t["b_off"] + n]
            db.copy_(b.to(dev))
        scale = float(torch.tensor(-1.0 / (n * 1.3) if op in (OP_HINGE_D, OP_SUM) else 0.9 / n, dtype=torch.float32))
        vec = (da.data_ptr() % 16 == 0) and (db is None or db.data_ptr() % 16 == 0)
        ga_ptr = flat.data_ptr() + 4 * off if t["ga"] else None
        terms_f.append(_Term(da.data_ptr(), db.data_ptr() if db is not None else None, None, n, scale, t["sign"], op, t["slot"]))
        terms_b.append(_Term(da.data_ptr(), db.data_ptr() if db is not None else None, ga_ptr, n, scale, t["sign"], op, t["slot"]))
        host.append((t, a, b, scale, off, _max_per_thread(n, vec)))
        keep += [da, db]
        off += n + gap
    # forward: each slot against the float64 sum of the formula times the fp32 scale
    slots = torch.zeros(nslots, device=dev, dtype=torch.float64)
    _lib().check(lib.mg_loss_reduce(_device_table(terms_f, torch.device(dev)).data_ptr(), len(terms_f), slots.data_ptr(),
                                    ops._stream()), "mg_loss_reduce")
    ref = torch.zeros(nslots, dtype=torch.float64)
    rabs = torch.zeros(nslots, dtype=torch.float64)
    kslot = [2.0] * nslots
    for t, a, b, scale, _, L in host:
        f = _f64(t["op"], a.double(), b.double() if b is not None else None, t["sign"])
        ref[t["slot"]] += f.sum() * scale
        rabs[t["slot"]] += f.abs().sum() * abs(scale)
        kslot[t["slot"]] = max(kslot[t["slot"]], L + 2.0)
    for s in range(nslots):
        check_close("%s fwd slot %d (L + 2)" % (case, s), slots[s:s + 1], ref[s:s + 1], rabs[s:s + 1], kslot[s])
    # backward: bit-exact against fp32 (gslot * scale) * f'(a); untouched where ga is null and between the terms
    gslots = torch.tensor([0.7, -1.3, 2.5][:nslots], dtype=torch.float32)
    _lib().check(lib.mg_loss_reduce_bwd(_device_table(terms_b, torch.device(dev)).data_ptr(), len(terms_b),
                                        gslots.to(dev).data_ptr(), ops._stream()), "mg_loss_reduce_bwd")
    got = flat.cpu()
    nties = 0
    for t, a, b, scale, o, _ in host:
        n, op, sign = t["n"], t["op"], t["sign"]
        same_bits("%s gap after term at %d" % (case, o), got[o + n:o + n + gap], sentinel.repeat(gap))
        if not t["ga"]:
            same_bits("%s ga = null term at %d untouched" % (case, o), got[o:o + n], sentinel.repeat(n))
            continue
        gs = gslots[t["slot"]] * torch.tensor(scale, dtype=torch.float32)
        want = gs * _d_f32(op, a, b, sign)
        same_bits("%s bwd term at %d" % (case, o), got[o:o + n], want)
        x = a.double().requires_grad_()
        (_ref_expr(op, x, b.double() if b is not None else None, sign).sum() * scale * float(gslots[t["slot"]])).backward()
        check_close("%s bwd term at %d vs fp64 autograd" % (case, o), got[o:o + n], x.grad, x.grad.abs(), K_GA64)
        if op == OP_HINGE_D and t["ties"]:
            tie = (sign * a.double() - 1) == 0
            nties += int(tie.sum())
            w = b.double() if b is not None else torch.ones(n, dtype=torch.float64)
            half = (0.5 * sign * w[tie]) * scale * float(gslots[t["slot"]])
            assert bool(((x.grad[tie] - half).abs() <= 1e-14 * half.abs()).all()), "autograd tie rule changed"
        elif op in (OP_L1, OP_SQ) and t["ties"]:
            tie = a == b
            nties += int(tie.sum())
            assert bool((got[o:o + n][tie] == 0).all()), case
    if any(t["ties"] and t["op"] != OP_SUM for t in spec):
        assert nties > 0, case


# ============================================================================================== Gabor orientation loss
COEF = [float(torch.tensor(c, dtype=torch.float32)) for c in (0.299, 0.587, 0.144)]


def _bank():
    from michigan_b200.networks.loss import gabor_bank
    return gabor_bank(torch.device(dev))


def _filters64(bank):
    """[17*17][32] bank -> conv2d weight [32, 1, 17, 17] (response[p] = sum_ij gray[p + (i, j) - 8] K[i][j])."""
    return d64(bank).t().reshape(32, 1, 17, 17).contiguous()


def _orient_inputs(n, h, w, form, g):
    """Dark, low-contrast texture (responses 0 < mx < 9, where the confidence gradient lives), a normal-contrast patch, a flat
    black band (every response 0) and hair over most of it; label2 from a 1-channel angle map or an unnormalised 2-channel
    (use_ig) map.  Where both sides are >= 17, a black 17 x 17 block in the top-right corner holds a ring of dim pixels at
    distance 2 .. 3.75 from its centre: every Gabor filter sums positive, so a flat gray region has positive responses, but at
    the ring's centre all 32 responses are negative (about -3.3 per gray level), which exercises the clamp to 0."""
    img = -1.0 + 0.008 * torch.rand(n, 3, h, w, generator=g)
    y0, x0 = h // 3, w // 3
    img[:, :, y0:y0 + max(1, h // 4), x0:x0 + max(1, w // 4)] = torch.rand(n, 3, max(1, h // 4), max(1, w // 4), generator=g) * 2 - 1
    img[:, :, (2 * h) // 3:(2 * h) // 3 + max(1, h // 8)] = -1.0
    if h >= 17 and w >= 17:
        yy, xx = torch.meshgrid(torch.arange(-8, 9.0), torch.arange(-8, 9.0), indexing="ij")
        d = (yy ** 2 + xx ** 2).sqrt()
        block = torch.where((d >= 2) & (d < 3.75), torch.tensor(-1.0 + 0.05), torch.tensor(-1.0))
        img[:, :, 0:17, w - 17:w] = block
    hair = (torch.rand(n, h, w, generator=g) < 0.8).float()
    if form == "angle":
        t = torch.floor(torch.rand(n, 1, h, w, generator=g) * 255) / 255 * math.pi
        label2 = torch.cat([torch.sin(2 * t), torch.cos(2 * t)], dim=1)
    else:
        label2 = torch.rand(n, 2, h, w, generator=g) * 2 - 1
    return img.float().contiguous(), label2.float().contiguous(), hair.contiguous()


def _orient_fwd(img, bank, label2, hair):
    lib = _lib().load()
    n, _, h, w = img.shape
    im, lb, hr = img.to(dev), label2.to(dev), hair.to(dev)
    idx = torch.empty((n, h, w), device=dev, dtype=torch.uint8)
    d1 = torch.empty((n, h, w), device=dev)
    d2 = torch.empty((n, h, w), device=dev)
    sums = torch.zeros(3, device=dev, dtype=torch.float64)
    _lib().check(lib.mg_orient_loss_fwd(im.data_ptr(), bank.data_ptr(), lb.data_ptr(), hr.data_ptr(), idx.data_ptr(), d1.data_ptr(),
                                        d2.data_ptr(), sums.data_ptr(), n, h, w, _ops()._stream()), "mg_orient_loss_fwd")
    return idx.cpu().long(), d1.cpu(), d2.cpu(), sums.cpu()


@pytest.mark.parametrize("n,h,w,form", [(1, 1, 1, "angle"), (2, 5, 7, "ig"), (1, 16, 16, "angle"), (2, 33, 47, "angle"),
                                        (1, 33, 47, "ig"), (1, 17, 130, "ig"), (3, 40, 24, "angle"), (2, 512, 512, "angle")])
def test_orient_loss_fwd(n, h, w, form):
    name = "orient_fwd %dx%dx%d %s" % (n, h, w, form)
    g = _gen(name)
    img, label2, hair = _orient_inputs(n, h, w, form, g)
    bank = _bank()
    idx, d1, d2, sums = _orient_fwd(img, bank, label2, hair)
    Wt = _filters64(bank)
    gray = sum(c * (img[:, i:i + 1].double() + 1) * 127.5 for i, c in enumerate(COEF))
    r = F.conv2d(gray, Wt, padding=8)
    rab = F.conv2d(gray.abs(), Wt.abs(), padding=8)
    rp = r.clamp_min(0)
    top = rp.max(1).values
    B = K_RESP * U * rab.max(1).values                          # response bound per pixel, the largest over the filters
    pick = rp.gather(1, idx.unsqueeze(1)).squeeze(1)
    need = float(((top - pick) / (U * rab.max(1).values + TINY)).max())
    print("%s: arg-max: max (best - chosen) / (u R_abs) = %.3g (admissible up to 2 k = %g)" % (name, need, 2 * K_RESP))
    assert bool((pick >= top - 2 * B).all()), (name, "inadmissible arg-max")
    adm = (rp >= top.unsqueeze(1) - 2 * B.unsqueeze(1)).sum(1)
    zero = rab.max(1).values == 0
    assert bool((idx[zero] == 0).all()), "all-zero responses must give index 0"
    assert bool((d1[zero] == 0).all() and (d2[zero] == 0).all()), "all-zero responses must give a zero gradient"
    neg = (r < -B.unsqueeze(1)).all(1)                          # every response negative beyond its bound, gray not all zero
    if h >= 17 and w >= 17:
        assert int((neg & ~zero).sum()) >= n, int((neg & ~zero).sum())
    assert bool((idx[neg] == 0).all()), "all-negative responses must give index 0"
    assert bool((d1[neg] == 0).all() and (d2[neg] == 0).all()), "all-negative responses must give a zero gradient"
    if h * w >= 256:
        assert float((adm == 1).double().mean()) > 0.5, "too few pixels with a unique winner: %g" % float((adm == 1).double().mean())
    # the kernel's index decides everything below; float64 from it
    hm = hair.double()
    mx = pick
    E = B
    th = torch.tanh(mx)
    conf = (th + 1) / 2
    dcd = (1 - th * th) / 2
    ang = 2.0 * idx.double() * math.pi / 32
    s, c = torch.sin(ang), torch.cos(ang)
    ls, lc = label2[:, 0].double() * hm, label2[:, 1].double() * hm
    ds, dc = s * conf * hm - ls, c * conf * hm - lc
    dconf = 0.5 * E + 4 * U
    ddcd = D2CONF * E + 4 * U
    Bs = hm.abs() * (16 * U + dconf) + 3 * U * (hm.abs() + ls.abs())
    Bc = hm.abs() * (16 * U + dconf) + 3 * U * (hm.abs() + lc.abs())
    # candidates: either sign where |ds| / |dc| is within its bound; dconf/dmax = 0 where the winner may have been clamped
    big = torch.full_like(mx, math.inf)
    err1, errl = big.clone(), big.clone()
    waived_sign = (ds.abs() <= Bs) | (dc.abs() <= Bc)
    waived_zero = (mx <= E) & (E > 0)
    for sgs, sgc, clamp in itertools.product((-1.0, 0.0, 1.0), (-1.0, 0.0, 1.0), (False, True)):
        ok = ((ds.sign() == sgs) | (ds.abs() <= Bs)) & ((dc.sign() == sgc) | (dc.abs() <= Bc))
        ok &= (~torch.tensor(clamp)) | (mx <= E)
        dd = torch.zeros_like(dcd) if clamp else dcd
        r1 = (sgs * s + sgc * c) * hm * dd
        rl = hm / conf * dd
        err1 = torch.where(ok, torch.minimum(err1, (d1.double() - r1).abs()), err1)
        errl = torch.where(ok, torch.minimum(errl, (d2.double() - rl).abs()), errl)
    b1 = hm.abs() * (2 * ddcd + dcd * 2 * 16 * U) + 6 * U * hm.abs() * dcd
    bl = hm.abs() * (2 * ddcd + 4 * dcd * dconf) + 6 * U * hm.abs() * dcd / conf
    check_within(name + " dmax_l1", err1, b1)
    check_within(name + " dmax_log", errl, bl)
    hairpx = hm != 0
    nw = int((waived_sign & hairpx).sum()) + int((waived_zero & hairpx).sum())
    print("%s: %d of %d hair pixels waived (sign or clamp)" % (name, nw, int(hairpx.sum())))
    assert nw <= max(2, 0.02 * int(hairpx.sum())), (name, nw)
    live = hairpx & (mx > 0) & (mx < 9)
    if min(h, w) >= 17:                                         # below that the bright patch reaches every pixel
        share = float(live.double().sum() / hairpx.double().sum())
        print("%s: %.2f of hair pixels have 0 < mx < 9" % (name, share))
        assert share > 0.3, share
        assert float((d1 != 0).double().mean()) > 0.2
    s0 = (ds.abs() + dc.abs()).sum()
    s1 = (torch.log(conf) * hm).sum()
    s2 = hm.sum()
    check_within(name + " sums[0]", (sums[0] - s0).abs().view(1), ((Bs + Bc).sum() + 1e-12 * s0.abs()).view(1))
    check_within(name + " sums[1]", (sums[1] - s1).abs().view(1),
                 ((hm.abs() * (2 * dconf + 3 * U * torch.log(conf).abs())).sum() + 1e-12 * s1.abs()).view(1))
    assert float(sums[2]) == float(s2), (name, float(sums[2]), float(s2))


def _orient_bwd(bank, idx, d1, d2, wts, n, h, w):
    lib = _lib().load()
    dimg = torch.full((n, 3, h, w), float("nan"), device=dev)
    i, a, b, ww = idx.to(dev).contiguous(), d1.to(dev).contiguous(), d2.to(dev).contiguous(), wts.to(dev).contiguous()
    _lib().check(lib.mg_orient_loss_bwd(bank.data_ptr(), i.data_ptr(), a.data_ptr(), b.data_ptr(), ww.data_ptr(), dimg.data_ptr(),
                                        n, h, w, _ops()._stream()), "mg_orient_loss_bwd")
    return dimg.cpu()


def _orient_bwd_ref(bank, idx, d1, d2, wts):
    """dimg[n,c,q] = coef_c 127.5 sum_p g[p] K_{idx[p]}[q - p + 8] in float64, and its R_abs (|g| from |w1 d1| + |w2 d2|)."""
    Wt = _filters64(bank)
    w1, w2 = float(wts[0]), float(wts[1])
    oh = F.one_hot(idx.long(), 32).permute(0, 3, 1, 2).double()
    g = w1 * d1.double() + w2 * d2.double()
    ga = (w1 * d1.double()).abs() + (w2 * d2.double()).abs()
    dg = F.conv_transpose2d(oh * g.unsqueeze(1), Wt, padding=8)
    ra = F.conv_transpose2d(oh * ga.unsqueeze(1), Wt.abs(), padding=8)
    ref = torch.cat([c * 127.5 * dg for c in COEF], 1)
    rabs = torch.cat([c * 127.5 * ra for c in COEF], 1)
    return ref, rabs


@pytest.mark.parametrize("n,h,w", [(1, 1, 1), (2, 5, 7), (1, 16, 16), (2, 33, 47), (1, 17, 130), (3, 40, 24), (2, 512, 512)])
def test_orient_loss_bwd(n, h, w):
    name = "orient_bwd %dx%dx%d" % (n, h, w)
    g = _gen(name)
    bank = _bank()
    idx = torch.randint(0, 32, (n, h, w), generator=g).to(torch.uint8)
    idx.view(-1)[:32] = torch.arange(32, dtype=torch.uint8)[:idx.numel()]
    d1 = torch.randn(n, h, w, generator=g) * (torch.rand(n, h, w, generator=g) > 0.3)
    d2 = torch.randn(n, h, w, generator=g) * (torch.rand(n, h, w, generator=g) > 0.3)
    wts = torch.tensor([0.37 / (n * h * w), -1.9 / max(1, n * h * w // 2)], dtype=torch.float32)
    got = _orient_bwd(bank, idx, d1, d2, wts, n, h, w)
    ref, rabs = _orient_bwd_ref(bank, idx, d1, d2, wts)
    check_close(name, got, ref, rabs, K_ORIENT_BWD)


def test_orient_loss_bwd_no_leak_between_images():
    """Image 0's upstream gradient is zero and image 1's large: image 0's d image must be exactly zero, halo included."""
    n, h, w = 2, 33, 47
    g = _gen("orient_leak")
    bank = _bank()
    idx = torch.randint(0, 32, (n, h, w), generator=g).to(torch.uint8)
    d1 = torch.randn(n, h, w, generator=g) * 1e3
    d2 = torch.randn(n, h, w, generator=g) * 1e3
    d1[0] = 0
    d2[0] = 0
    wts = torch.tensor([1.0, 1.0], dtype=torch.float32)
    got = _orient_bwd(bank, idx, d1, d2, wts, n, h, w)
    assert bool((got[0] == 0).all()), int((got[0] != 0).sum())
    assert bool((got[1] != 0).any())
    ref, rabs = _orient_bwd_ref(bank, idx, d1, d2, wts)
    check_close("orient_bwd leak case", got, ref, rabs, K_ORIENT_BWD)


# ============================================================================================== Lab colour loss
LAB_M = torch.tensor([[0.412453, 0.357580, 0.180423], [0.212671, 0.715160, 0.072169], [0.019334, 0.119193, 0.950227]],
                     dtype=torch.float32)
LAB_T = float(torch.tensor(0.008856, dtype=torch.float32))
LAB_A = float(torch.tensor(7.787, dtype=torch.float32))
LAB_B = float(torch.tensor(0.137931, dtype=torch.float32))


def _lab_t(img):
    """[N,3,H,W] fp32 -> xyz [N,3,HW] in float64 (fp32 M, its fp32 row sums, as the kernel)."""
    rs = ((LAB_M[:, 0] + LAB_M[:, 1]) + LAB_M[:, 2]).double()
    rgb = (img.double().flatten(2) + 1) / 2
    return torch.einsum("kc,ncp->nkp", LAB_M.double(), rgb) / rs.view(1, 3, 1)


def _lab_f(t, cube):
    return torch.where(cube, t.clamp(min=1e-300).pow(1.0 / 3), LAB_A * t + LAB_B)


def _lab_df(t, cube):
    return torch.where(cube, t.clamp(min=1e-300).pow(-2.0 / 3) / 3, torch.full_like(t, LAB_A))


def _lab_inputs(n, hw, g):
    """Random pixels, saturated -1 and +1 pixels (t = 0 and t = 1), gray pixels planted at t = T (1 + m 2^-e) for a range of
    m, e, on both sides of the threshold; real has its own planted pixels."""
    fake = torch.rand(n, 3, hw, generator=g) * 2 - 1
    real = torch.rand(n, 3, hw, generator=g) * 2 - 1
    if hw >= 7:
        fake[:, :, 0] = -1.0
        fake[:, :, 1] = 1.0
        real[:, :, 2] = -1.0
    plant = [LAB_T * (1 + m * 2.0 ** -e) for e in (8, 12, 16, 20, 22, 23) for m in (-3, -1, 1, 3)]
    for img, start in ((fake, 3), (real, 5)):
        for j, t in enumerate(plant):
            p = start + 2 * j
            if p < hw:
                img[:, :, p] = float(torch.tensor(2 * t - 1, dtype=torch.float32))
    return fake.contiguous(), real.contiguous()


@pytest.mark.parametrize("n,h,w", [(1, 1, 1), (3, 1, 7), (1, 7, 1), (3, 17, 19), (1, 1, 512 * 512 + 3), (3, 64, 96)])
def test_lab_loss_fwd_bwd(n, h, w):
    name = "lab %dx%dx%d" % (n, h, w)
    g = _gen(name)
    fake, real = _lab_inputs(n, h * w, g)
    fake, real = fake.view(n, 3, h, w), real.view(n, 3, h, w)
    ops = _ops()
    gscale = torch.tensor([0.83 / (n * h * w)], dtype=torch.float32)
    s = ops.lab_loss_fwd(fake.to(dev), real.to(dev)).cpu()
    dfake = ops.lab_loss_bwd(fake.to(dev), real.to(dev), gscale.to(dev)).cpu().flatten(2).double()
    tf, tr = _lab_t(fake), _lab_t(real)
    ff, fr = _lab_f(tf, tf > LAB_T), _lab_f(tr, tr > LAB_T)
    near_f = (tf - LAB_T).abs() <= K_LAB * U * tf
    near_r = (tr - LAB_T).abs() <= K_LAB * U * tr
    jump = (_lab_f(tf, torch.ones_like(near_f)) - _lab_f(tf, torch.zeros_like(near_f))).abs()
    jump_f = torch.where(near_f, jump, torch.zeros_like(jump))
    jump = (_lab_f(tr, torch.ones_like(near_r)) - _lab_f(tr, torch.zeros_like(near_r))).abs()
    jump_r = torch.where(near_r, jump, torch.zeros_like(jump))
    da = 500 * (ff[:, 0] - ff[:, 1]) - 500 * (fr[:, 0] - fr[:, 1])
    db = 200 * (ff[:, 1] - ff[:, 2]) - 200 * (fr[:, 1] - fr[:, 2])
    ra = 500 * (ff[:, 0].abs() + ff[:, 1].abs() + fr[:, 0].abs() + fr[:, 1].abs())
    rb = 200 * (ff[:, 1].abs() + ff[:, 2].abs() + fr[:, 1].abs() + fr[:, 2].abs())
    ba = K_LAB * U * ra + 500 * (jump_f[:, 0] + jump_f[:, 1] + jump_r[:, 0] + jump_r[:, 1])
    bb = K_LAB * U * rb + 200 * (jump_f[:, 1] + jump_f[:, 2] + jump_r[:, 1] + jump_r[:, 2])
    # forward: one fp64 sum of per-pixel fp32 values
    ref = (da.abs() + db.abs()).sum()
    check_within(name + " fwd sum", (s[0] - ref).abs().view(1), (ba + bb).sum().view(1) + 1e-12 * ref)
    print("%s fwd: |got - ref| / (u sum R_abs) = %.3g (k = %g)" % (name, float((s[0] - ref).abs() / (U * (ra + rb).sum())), K_LAB))
    # backward per pixel and channel
    gs = float(gscale[0])
    rs = ((LAB_M[:, 0] + LAB_M[:, 1]) + LAB_M[:, 2]).double()
    M = LAB_M.double()

    def dfake_of(sa, sb, cube):
        dfk = torch.stack([500 * sa, -500 * sa + 200 * sb, -200 * sb], 1)
        dt = dfk * _lab_df(tf, cube) / rs.view(1, 3, 1)
        out = gs * 0.5 * torch.einsum("nkp,kc->ncp", dt, M)
        rabs = abs(gs) * 0.5 * torch.einsum("nkp,kc->ncp", dt.abs(), M)
        return out, rabs

    cube = tf > LAB_T
    want, rabs = dfake_of(da.sign(), db.sign(), cube)
    waived = ((da.abs() <= ba) | (db.abs() <= bb) | near_f.any(1))
    bad = (dfake - want).abs() > K_LAB * U * rabs + TINY
    ok = ~waived.unsqueeze(1) & ~bad
    kept = ((dfake - want).abs() / (U * rabs + TINY))[~waived.unsqueeze(1).expand_as(dfake)]
    ratio = float(kept.max()) if kept.numel() else 0.0
    print("%s bwd: max |got - ref| / (u R_abs) = %.3g (k = %g), %d of %d pixels waived" % (name, ratio, K_LAB, int(waived.sum()),
                                                                                            waived.numel()))
    assert bool((ok | waived.unsqueeze(1)).all()), (name, "d fake out of bound", ratio)
    # waived pixels: some choice of signs (within their bound) and branches (near the threshold) must match
    for ni, p in waived.nonzero().tolist():
        sas = [-1.0, 0.0, 1.0] if abs(float(da[ni, p])) <= float(ba[ni, p]) else [float(da[ni, p].sign())]
        sbs = [-1.0, 0.0, 1.0] if abs(float(db[ni, p])) <= float(bb[ni, p]) else [float(db[ni, p].sign())]
        brs = [[bool(cube[ni, k, p])] if not bool(near_f[ni, k, p]) else [False, True] for k in range(3)]
        t1 = tf[ni:ni + 1, :, p:p + 1]
        best = math.inf
        for sa, sb, bx, by, bz in itertools.product(sas, sbs, *brs):
            cb = torch.tensor([bx, by, bz]).view(1, 3, 1)
            dfk = torch.tensor([500 * sa, -500 * sa + 200 * sb, -200 * sb], dtype=torch.float64).view(1, 3, 1)
            dt = dfk * _lab_df(t1, cb) / rs.view(1, 3, 1)
            o = gs * 0.5 * torch.einsum("nkp,kc->ncp", dt, M)
            ra_ = abs(gs) * 0.5 * torch.einsum("nkp,kc->ncp", dt.abs(), M)
            e = float(((dfake[ni:ni + 1, :, p:p + 1] - o).abs() / (K_LAB * U * ra_ + TINY)).max())
            best = min(best, e)
        assert best <= 1.0, (name, ni, p, best)
    assert int(waived.sum()) <= 4 * 24 * n + 2 * n + 0.001 * waived.numel(), (name, int(waived.sum()))


# ============================================================================================== SPADE segmap MLP (tensor cores)
# seg_mlp_tc_kernel (mg_conv_seg_tc) forms A_hi.W_hi + A_lo.W_hi + A_hi.W_lo of bf16 splits in one K = 128 wgmma chain over
# 36 taps x channels, on R_abs of the three products plus |bias|.  The conv tests' 1.25 sqrt(36) + 8 = 15.5 left less than
# 3x over the measured 5.9 (3 x 24 x 40, no seg_resize), so k = 2 sqrt(36) + 8 = 20.
K_SEG = 2 * math.sqrt(36) + 8


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def rna_tf32(t):
    """cvt.rna.tf32.f32 on finite fp32 values: round the magnitude to 10 stored mantissa bits, ties away from zero."""
    return ((t.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def split16(v32, fmt):
    """(hi, lo) = (cvt(v), cvt(v - float(hi))) as the kernels convert: round to nearest even, fp16 clamped to +-65504 (hi only)."""
    t = torch.float16 if fmt == "f16" else torch.bfloat16
    hi = (v32.clamp(-65504.0, 65504.0) if fmt == "f16" else v32).to(t)
    return hi, (v32 - hi.float()).to(t)


def _seg_pack_ref(w):
    """[128, Cin, 3, 3] fp32 -> the bf16 [128][128] operand: k = part * 36 + tap * 4 + ci, parts W_hi | W_hi | W_lo, zero tail."""
    wt = torch.zeros(128, 9, 4)
    wt[:, :, :w.shape[1]] = w.reshape(128, w.shape[1], 9).permute(0, 2, 1)
    hi, lo = split16(wt.reshape(128, 36), "bf16")
    return torch.cat([hi, hi, lo, torch.zeros(128, 20, dtype=torch.bfloat16)], 1).contiguous()


def _segmap(n, H, W, R, cin, g):
    """A realistic SPADE segmap at the input resolution (H R x W R): one-hot background / hair, then sin / cos of the
    orientation times hair (channel 3 zero when cin = 3)."""
    hr, wr = H * R, W * R
    hair = (torch.rand(n, 1, hr, wr, generator=g) < 0.6).float()
    ang = torch.rand(n, 1, hr, wr, generator=g) * math.pi
    seg = torch.cat([1 - hair, hair, torch.sin(2 * ang) * hair, torch.cos(2 * ang) * hair], 1)
    if cin == 3:
        seg[:, 3] = 0
    return nhwc(seg)


SEG_CASES = [  # (N, H, W, seg_resize, Cin, act, round_out)
    (1, 1, 1, 0, 4, 1, False), (3, 18, 9, 2, 4, 1, False), (2, 24, 40, 4, 3, 0, False), (1, 3, 130, 32, 4, 1, True),
    (2, 18, 9, 32, 3, 0, True), (3, 24, 40, 0, 4, 0, False), (1, 3, 130, 2, 3, 1, False), (2, 16, 16, 4, 4, 1, True),
]


@pytest.mark.parametrize("N,H,W,R,cin,act,round_out", SEG_CASES)
def test_seg_mlp_tc(N, H, W, R, cin, act, round_out):
    ops = _ops()
    name = "seg_mlp_tc N%d %dx%d R%d cin%d act%d round%d" % (N, H, W, R, cin, act, int(round_out))
    g = _gen(name)
    seg = _segmap(N, H, W, max(R, 1), cin, g)
    w = torch.randn(128, cin, 3, 3, generator=g) / 6
    b = torch.randn(128, generator=g)
    wpack = ops.pack_weight_seg_tc(w.to(dev))
    same_bits(name + " pack", wpack, _seg_pack_ref(w))
    sd, bd = seg.to(dev), b.to(dev)

    def run(**kw):
        out = ops.conv_seg_tc(sd, wpack, bd, seg_resize=R, act=act, out_hw=(H, W), **kw)
        torch.cuda.synchronize()
        return out

    got = run(round_out=round_out).cpu()
    # float64 of exactly the three products the kernel forms, from the bf16 splits of the nearest-resized segmap and of W
    a = seg[:, ::max(R, 1), ::max(R, 1), :][:, :H, :W]
    a_hi, a_lo = split16(a, "bf16")
    wt = torch.zeros(128, 4, 3, 3)
    wt[:, :cin] = w
    w_hi, w_lo = split16(wt, "bf16")
    pairs = [(a_hi, w_hi), (a_lo, w_hi), (a_hi, w_lo)]
    acc = sum(F.conv2d(nchw(d64(x)), d64(y), padding=1) for x, y in pairs)
    rabs = sum(F.conv2d(nchw(d64(x)).abs(), d64(y).abs(), padding=1) for x, y in pairs) + d64(b).abs().view(1, -1, 1, 1)
    ref = acc + d64(b).view(1, -1, 1, 1)
    if act == 1:
        ref = ref.clamp_min(0)
    if not round_out:
        check_close(name, nchw(got), ref, rabs, K_SEG)
    else:
        # round_out: the output is rna_tf32 of the unrounded value of the same accumulation
        same_bits(name + " round_out", got, rna_tf32(ops.conv_seg_tc(sd, wpack, bd, seg_resize=R, act=act, out_hw=(H, W)).cpu()))
        check_close(name + " (before round_out)",
                    nchw(ops.conv_seg_tc(sd, wpack, bd, seg_resize=R, act=act, out_hw=(H, W)).cpu()), ref, rabs, K_SEG)
    # 16-bit copies beside the fp32 output, and 16-bit-only outputs through both epilogues (MG_SEG_TMA 0 / 1): bit-identical to
    # the split of the fp32 output
    for fmt, fid in (("f16", ops.F16), ("bf16", ops.BF16)):
        o32, hi, lo = run(round_out=round_out, out16=(fid, True))
        want_hi, want_lo = split16(o32.cpu(), fmt)
        same_bits(name + " %s hi beside fp32" % fmt, hi, want_hi)
        same_bits(name + " %s lo beside fp32" % fmt, lo, want_lo)
        for knob in (0, 1):
            prev = _lib().set_tuning("MG_SEG_TMA", knob)
            try:
                _, h16, l16 = run(round_out=round_out, out16=(fid, True), want_f32=False)
                _, h16n, _ = run(round_out=round_out, out16=(fid, False), want_f32=False)
            finally:
                _lib().set_tuning("MG_SEG_TMA", prev)
            same_bits(name + " %s hi only, MG_SEG_TMA %d" % (fmt, knob), h16, want_hi)
            same_bits(name + " %s lo only, MG_SEG_TMA %d" % (fmt, knob), l16, want_lo)
            same_bits(name + " %s hi without lo, MG_SEG_TMA %d" % (fmt, knob), h16n, want_hi)


# ============================================================================================== conv_img (generator output conv)
# tanh(conv3x3(leaky_relu(x, 0.2)) + b): 9 Cin fp32 fmas per output, then tanhf.  Pre-activation model k = 1.25 sqrt(9 Cin) + 8
# on R_abs = sum |lrelu(x)| |w| + |b|, carried through tanh with its derivative 1 - y^2, plus tanhf's own 2 ulp.
@pytest.mark.parametrize("N,H,W,Cin", [(2, 37, 45, 64), (1, 8, 32, 32), (1, 1, 1, 16), (3, 9, 33, 4)])
def test_conv_img_forward_fp64(N, H, W, Cin):
    ops = _ops()
    name = "conv_img N%d %dx%d Cin%d" % (N, H, W, Cin)
    g = _gen(name)
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(3, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5
    b = torch.randn(3, generator=g) * 0.1
    got = ops.conv_img(nhwc(x).to(dev), w.to(dev), b.to(dev)).cpu()
    xa = F.leaky_relu(x.double(), 0.2)
    pre = F.conv2d(xa, w.double(), b.double(), padding=1)
    rpre = F.conv2d(xa.abs(), w.double().abs(), b.double().abs(), padding=1)
    ref = torch.tanh(pre)
    k = 1.25 * math.sqrt(9 * Cin) + 8
    rabs = (1 - ref * ref) * rpre + 2 * ref.abs() / k
    check_close(name, got, ref, rabs, k)


# ============================================================================================== input prologue, h != w
def _bilinear64(f, H, W):
    """cv2.resize(f, (W, H), interpolation=INTER_LINEAR) in float64 for an [h, w, 3] field: source coordinate
    (x + 0.5) * w / W - 0.5, clamped to the border.  Returns the value, and per pixel the coordinate of each axis and the
    largest |field| of the four taps (for the bound)."""
    h, w = f.shape[0], f.shape[1]

    def axis(n_out, n_in):
        fx = (torch.arange(n_out, dtype=torch.float64) + 0.5) * (n_in / n_out) - 0.5
        x0 = fx.floor()
        a = fx - x0
        a = torch.where(x0 < 0, torch.zeros_like(a), a)
        x0 = x0.clamp(min=0)
        a = torch.where(x0 >= n_in - 1, torch.zeros_like(a), a)
        x0 = x0.clamp(max=n_in - 1).long()
        return x0, (x0 + 1).clamp(max=n_in - 1), a, fx

    y0, y1, ay, fy = axis(H, h)
    x0, x1, ax, fx = axis(W, w)
    p00, p01 = f[y0][:, x0], f[y0][:, x1]
    p10, p11 = f[y1][:, x0], f[y1][:, x1]
    axv, ayv = ax.view(1, -1, 1), ay.view(-1, 1, 1)
    top = p00 + (p01 - p00) * axv
    bot = p10 + (p11 - p10) * axv
    m = torch.stack([p00.abs(), p01.abs(), p10.abs(), p11.abs()]).amax(0)
    return top + (bot - top) * ayv, fy, fx, m


def _fp32_coord(n_out, n_in):
    """The kernel's fp32 source coordinate ((x + 0.5) * (n_in / n_out) - 0.5, every step rounded to fp32)."""
    scale = torch.tensor(float(n_in), dtype=torch.float32) / torch.tensor(float(n_out), dtype=torch.float32)
    return ((torch.arange(n_out, dtype=torch.float32) + 0.5) * scale - 0.5).double()


@pytest.mark.parametrize("n,h,w", [(2, 48, 80), (1, 37, 64), (2, 80, 48), (1, 64, 37)])
def test_noise_pyramid_non_square(n, h, w):
    """Every octave of the noise pyramid resized to the full h x w with INTER_LINEAR and averaged.  The reference's
    generate_noise passes dsize = (height, width), which cv2 reads as (width, height), so it runs only at h = w; for h != w the
    kernel resizes each octave to h x w, which the float64 restatement below follows.  Bound per octave: the coordinate's
    fp32 rounding times the two slopes, plus 6 u of the taps' magnitude for the lerps; then the average's roundings."""
    from michigan_b200 import prologue
    g = _gen("noise %d %d %d" % (n, h, w))
    sizes = prologue.noise_octave_sizes(h, w)
    assert len(sizes) >= 3
    fields = [torch.randn(n, hh, ww, 3, generator=g) * 0.25 + 0.5 for hh, ww in sizes]
    got = prologue.noise_from_fields([f.to(dev) for f in fields], n, h, w).cpu()
    assert tuple(got.shape) == (n, 3, h, w)
    ref = torch.zeros(n, h, w, 3, dtype=torch.float64)
    bound = torch.zeros(n, h, w, 3, dtype=torch.float64)
    for l, (hh, ww) in enumerate(sizes):
        ey = (_fp32_coord(h, hh) - (torch.arange(h, dtype=torch.float64) + 0.5) * (hh / h) + 0.5).abs().view(-1, 1, 1)
        ex = (_fp32_coord(w, ww) - (torch.arange(w, dtype=torch.float64) + 0.5) * (ww / w) + 0.5).abs().view(1, -1, 1)
        for i in range(n):
            v, _, _, m = _bilinear64(d64(fields[l][i]), h, w)
            ref[i] += v
            bound[i] += (ex + ey) * 2 * m + 6 * U * m
    ref /= len(sizes)
    # the octave sum's adds (each within u of a partial sum <= levels * max |field|), then 1 / levels and the product
    bound = bound / len(sizes) + 2 * U * ref.abs() + len(sizes) * U * torch.stack([d64(f).abs().amax() for f in fields]).max()
    err = (d64(got) - nchw(ref)).abs()
    check_within("noise %dx%dx%d" % (n, h, w), err, nchw(bound))
    # the restatement is cv2's INTER_LINEAR where cv2 is available
    try:
        import cv2
    except ImportError:
        return
    import numpy as np
    v, _, _, _ = _bilinear64(d64(fields[1][0]), h, w)
    cv = cv2.resize(fields[1][0].double().numpy(), dsize=(w, h), interpolation=cv2.INTER_LINEAR)
    assert np.abs(cv - v.numpy()).max() <= 1e-6          # cv2 keeps its interpolation weights in fp32


@pytest.mark.parametrize("n,h,w", [(2, 48, 80), (1, 37, 64), (2, 80, 48)])
def test_orient_rgb_non_square(n, h, w):
    """trans_orient_to_rgb + ToTensor + mask: ((cos 2t + 1) / 2 m 255 -> uint8 -> / 255) m per channel, in float64 as numpy
    computes it.  Both sides evaluate cos / sin in float64; where an unmasked scaled value lies within 1e-9 of an integer,
    the truncation may land on either side."""
    from michigan_b200 import prologue
    g = _gen("orient_rgb %d %d %d" % (n, h, w))
    orient = torch.floor(torch.rand(n, 1, h, w, generator=g) * 256).clamp(max=255)
    orient.view(-1)[:256] = torch.arange(256.0)[:orient.numel()]
    label = (torch.rand(n, 1, h, w, generator=g) > 0.4).float()
    got = prologue.orient_rgb(orient.to(dev), label.to(dev)).cpu()
    t = orient.double() / 255.0 * math.pi
    m = label.double()
    v = torch.cat([(torch.cos(2 * t) + 1) / 2 * m * 255.0, (torch.sin(2 * t) + 1) / 2 * m * 255.0, 0.5 * m * 255.0], 1)
    q = torch.trunc(v)
    want = (q.float() / 255.0) * label
    alt = ((q - 1).clamp_min(0).float() / 255.0) * label
    alt2 = ((q + 1).float() / 255.0) * label
    near = ((v - v.round()).abs() <= 1e-9) & (m != 0)          # masked values are exactly 0 on both sides
    ok = (_bits(got) == _bits(want)) | (near & ((_bits(got) == _bits(alt)) | (_bits(got) == _bits(alt2))))
    assert bool(ok.all()), (int((~ok).sum()), tuple((~ok).nonzero()[0].tolist()))
    print("orient_rgb %dx%dx%d: %d of %d values within 1e-9 of an integer" % (n, h, w, int(near.sum()), near.numel()))
    assert int(near.sum()) <= 0.01 * near.numel() + 3 * n * 3


@pytest.mark.parametrize("n,h,w", [(3, 48, 80), (2, 37, 64), (2, 80, 48)])
def test_hole_mask_non_square(n, h, w):
    """generate_hole (base_dataset.py:335-361) restated in numpy per sample, bit for bit: the centre is the
    floor(u * count)-th nonzero pixel in row-major order, rr = int(int(th * count) / pi); an empty orientation mask is returned
    as it is."""
    import numpy as np
    from michigan_b200 import prologue
    g = _gen("hole %d %d %d" % (n, h, w))
    mask = torch.zeros(n, 1, h, w)
    mask[:, :, h // 6:(5 * h) // 6, w // 5:(4 * w) // 5] = 1
    omask = mask * (torch.rand(n, 1, h, w, generator=g) > 0.3).float()
    omask[-1] = 0
    th_u = torch.rand(n, generator=g) * 0.7 + 0.5
    idx_u = torch.rand(n, generator=g)
    got = prologue.hole_mask(mask.to(dev), omask.to(dev), th_u.to(dev), idx_u.to(dev)).cpu()
    for i in range(n):
        om = omask[i, 0].numpy()
        if np.abs(om).max() == 0:
            exp = om
        else:
            coord = np.where(om != 0)
            nums = len(coord[0])
            rr = int(int(float(th_u[i]) * nums) / math.pi)
            k = min(int(math.floor(np.float32(idx_u[i]) * np.float32(nums))), nums - 1)
            cy, cx = coord[0][k], coord[1][k]
            yy, xx = np.mgrid[0:h, 0:w]
            tmp = (((yy - cy) ** 2 + (xx - cx) ** 2) < rr).astype(np.float32)
            exp = om * tmp + (mask[i, 0].numpy() - om)
        same_bits("hole_mask %dx%dx%d image %d" % (n, h, w, i), got[i, 0], torch.from_numpy(np.ascontiguousarray(exp, dtype=np.float32)))
