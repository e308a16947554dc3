"""Every backward kernel called directly through its ops.* wrapper and compared with a float64 CPU reference: torch.autograd
applied to the forward op written in plain torch.nn.functional.  Forwards that have no parity test elsewhere are checked in
the same test, so each backward is held to the op its forward really computes.

Elementwise kernels that add nothing (act_bwd, blend_bwd, the TF32 rounding of in_bwd / instance_norm_act)
are compared bit for bit with fp32 torch evaluated in the kernel's own order of operations.

Everything that sums is compared element by element:

    |got - ref| <= k * u * R_abs + tiny

R_abs is the magnitude reference: the same fp64 computation on |inputs|, i.e. the sum of |a| |b| behind each output element
(for the normalisations, whose gradients cancel by construction, the explicit magnitude of each term; it is given in the
test).  u = 2^-24: the kernels accumulate in fp32, and the operands of the tensor-core GEMMs are rounded to the kernel's
format (TF32 RNA, bf16 RNE) on both sides first.  k comes from measurement on an H100: each case gives the largest measured
|got - ref| / (u * R_abs) next to its k.  A global max-error bound would hide a wrong border element whose values are small;
this bound does not.

Kernels that reduce across CTAs (through fp64 partial sums) are also run twice on the same inputs: the results must be
bit-identical.
"""
import pytest
import torch
import torch.nn.functional as F

from fp64ref import TINY, U, check_close, d64, nchw, nhwc, rna_tf32, vjp64

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(autouse=True)
def _fp32_reference():
    """Any on-device torch arithmetic must be true fp32 (the references below run on the CPU in float64)."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.fixture()
def gen():
    return torch.Generator(device="cpu").manual_seed(1234)


def _ops():
    from michigan_b200 import ops
    return ops


def _lib():
    from michigan_b200 import _lib
    return _lib


def check_rounded(name, got, ref, rabs, bits, k):
    """got = ref rounded to nearest at `bits` significant bits (TF32: 11, bf16: 8) up to k*u*R_abs of accumulated error:
    |got - ref| <= ulp(ref) / 2 + k u R_abs.  Truncation (up to a whole ulp) fails this."""
    got, ref, rabs = d64(got), d64(ref), d64(rabs)
    _, e = torch.frexp(ref)
    half_ulp = torch.ldexp(torch.ones_like(ref), (e - bits - 1).to(torch.int64))
    err = (got - ref).abs()
    ratio = float(((err - half_ulp).clamp_min(0) / (U * rabs + TINY)).max())
    print("%s: max (|got - ref| - ulp/2) / (u R_abs) = %.3g (k = %g)" % (name, ratio, k))
    bad = err > half_ulp + k * U * rabs + TINY
    assert not bool(bad.any()), (name, int(bad.sum()), ratio, k)


def up(t, s):
    """Nearest 2^s upsample of an NHWC tensor."""
    f = 1 << s
    return t.repeat_interleave(f, 1).repeat_interleave(f, 2) if s else t


# ============================================================================================== bit-exact elementwise kernels
@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("with_y,masks,rnd", [(True, "", False), (False, "pm1", False), (True, "pm2", True), (True, "pm1+pm2", False),
                                              (False, "pm1+pm2", True)])
def test_act_bwd_bit_exact(gen, act, with_y, masks, rnd):
    """act_bwd: dz = dy * act'(y) * (pm1 * pm2) with act' taken from the sign of the forward OUTPUT y (1 without y),
    optionally RNA-rounded to TF32, against the same products in fp32 torch: bit-equal.  y holds exact +0 and -0 (both take
    the negative branch), pm1 holds zeros."""
    ops = _ops()
    N, H, W, C = 2, 5, 7, 12
    dy = torch.randn(N, H, W, C, generator=gen)
    y = torch.randn(N, H, W, C, generator=gen)
    y.view(-1)[::7] = 0.0
    y.view(-1)[3::11] = -0.0
    pm1 = torch.rand(N, H, W, generator=gen) * 2
    pm1[torch.rand(N, H, W, generator=gen) < 0.25] = 0.0
    pm2 = torch.rand(N, H, W, generator=gen) + 0.5
    p1 = pm1 if "pm1" in masks else None
    p2 = pm2 if "pm2" in masks else None
    got = ops.act_bwd(dy.to(dev), y.to(dev) if with_y else None, act, pm1=None if p1 is None else p1.to(dev),
                      pm2=None if p2 is None else p2.to(dev), round_tf32=rnd)
    one, zero, slope = (torch.tensor(v, dtype=torch.float32) for v in (1.0, 0.0, 0.2))
    da = one
    if with_y and act == ops.ACT_RELU:
        da = torch.where(y > 0, one, zero)
    elif with_y and act == ops.ACT_LRELU:
        da = torch.where(y > 0, one, slope)
    m = torch.ones(N, H, W)
    if p1 is not None:
        m = m * p1
    if p2 is not None:
        m = m * p2
    ref = (dy * da) * m[..., None]
    if rnd:
        ref = rna_tf32(ref)
    assert torch.equal(got.cpu(), ref)


@pytest.mark.parametrize("ms,acc", [(1, False), (2, True), (8, False), (8, True)])
def test_blend_bwd_bit_exact(gen, ms, acc):
    """blend_bwd of out = bf*(1-hair) + y*(1-back) (generator.py:186) with full-resolution masks read every mask_stride-th
    pixel: dy = dout*(1-back), dbf (+)= dout*(1-hair), bit-equal to fp32 torch."""
    ops = _ops()
    N, h, w, C = 2, 6, 5, 8
    dout = torch.randn(N, h, w, C, generator=gen)
    hair = torch.rand(N, h * ms, w * ms, generator=gen)
    back = torch.rand(N, h * ms, w * ms, generator=gen)
    hair[:, ::3] = 1.0
    back[:, 1::4] = 0.0
    dbf0 = torch.randn(N, h, w, C, generator=gen)
    dy, dbf = ops.blend_bwd(dout.to(dev), hair.to(dev), back.to(dev), ms, dbf=dbf0.to(dev) if acc else None)
    hs, bs = hair[:, ::ms, ::ms], back[:, ::ms, ::ms]
    ref_dbf = dout * (1 - hs)[..., None]
    if acc:
        ref_dbf = ref_dbf + dbf0
    assert torch.equal(dy.cpu(), dout * (1 - bs)[..., None])
    assert torch.equal(dbf.cpu(), ref_dbf)


# ============================================================================================== pooling / pad / resize / masked mean
@pytest.mark.parametrize("H,W,C", [(10, 13, 4), (9, 8, 64), (7, 7, 4), (12, 10, 64)])
def test_avgpool3s2_fwd_bwd(gen, H, W, C):
    """avgpool3s2 and its backward vs F.avg_pool2d(3, 2, 1, count_include_pad=False): even and odd H, W independently (the
    last window is cut at odd and even edges differently), C 4 (the image path) and 64, and the backward's += into din.
    k = 12 (measured: forward 3.4, backward 1.8)."""
    ops = _ops()
    x = torch.randn(2, H, W, C, generator=gen)

    def pool(t):
        return nhwc(F.avg_pool2d(nchw(t), 3, 2, 1, count_include_pad=False))

    got = ops.avgpool3s2(x.to(dev))
    check_close("avgpool3s2", got, pool(d64(x)), pool(d64(x).abs()), 12)
    dout = torch.randn(got.shape, generator=gen)
    din0 = torch.randn(x.shape, generator=gen)
    din = ops.avgpool3s2_bwd(dout.to(dev), din0.to(dev))
    _, (g,) = vjp64(pool, [x], dout)
    _, (ga,) = vjp64(pool, [x.abs()], dout.abs())
    check_close("avgpool3s2_bwd", din, d64(din0) + g, d64(din0).abs() + ga, 12)


@pytest.mark.parametrize("H,W,pad", [(6, 9, 1), (2, 5, 1), (4, 4, 3), (9, 7, 3)])
def test_reflect_pad_fwd_bwd(gen, H, W, pad):
    """reflect_pad (bit-equal to F.pad(mode="reflect")) and its backward, which folds every mirrored copy back: pad 1 and 3,
    including H = pad + 1 (one row has mirrors on both sides), written and accumulated.  k = 8 (measured 1.9)."""
    ops = _ops()
    x = torch.randn(2, H, W, 8, generator=gen)

    def fwd(t):
        return nhwc(F.pad(nchw(t), (pad,) * 4, mode="reflect"))

    got = ops.reflect_pad(x.to(dev), pad)
    assert torch.equal(got.cpu(), fwd(x))
    dpad = torch.randn(got.shape, generator=gen)
    _, (g,) = vjp64(fwd, [x], dpad)
    _, (ga,) = vjp64(fwd, [x.abs()], dpad.abs())
    dx = ops.reflect_pad_bwd(dpad.to(dev), pad)
    check_close("reflect_pad_bwd", dx, g, ga, 8)
    dx0 = torch.randn(x.shape, generator=gen)
    dx = ops.reflect_pad_bwd(dpad.to(dev), pad, dx=dx0.to(dev))
    check_close("reflect_pad_bwd accumulate", dx, d64(dx0) + g, d64(dx0).abs() + ga, 8)


def _bilinear_src(n_in, n_out):
    """Source coordinate (align_corners=False, clamped at 0) and the two taps of each output row / column."""
    f = ((torch.arange(n_out, dtype=torch.float64) + 0.5) * (n_in / n_out) - 0.5).clamp_min(0.0)
    i0 = f.floor().long()
    return f, i0, torch.where(i0 < n_in - 1, i0 + 1, i0)


@pytest.mark.parametrize("H,W,OH,OW", [(32, 7, 9, 16), (7, 33, 16, 32), (33, 32, 32, 9)])
def test_resize_bilinear_fwd_bwd(gen, H, W, OH, OW):
    """resize_bilinear and its backward vs F.interpolate(bilinear, align_corners=False), down- and up-sampling at
    non-integer ratios in each direction; the backward (fp64 scatter) twice, bit-identical.
    The kernels compute the source coordinate f in fp32 (as torch's fp32 kernels do), which moves it by a few u (f + 1) and
    the result by that times the four taps: R_abs adds (fy + fx + 2) * sum of the four |taps| (and its adjoint in the
    backward).  k = 4 (measured: forward 0.6, backward 0.7)."""
    ops = _ops()
    C = 12
    x = torch.randn(2, H, W, C, generator=gen)
    fy, y0, y1 = _bilinear_src(H, OH)
    fx, x0, x1 = _bilinear_src(W, OW)

    def fwd(t):
        return nhwc(F.interpolate(nchw(t), size=(OH, OW), mode="bilinear", align_corners=False))

    def pos(t):
        taps = t[:, y0][:, :, x0] + t[:, y0][:, :, x1] + t[:, y1][:, :, x0] + t[:, y1][:, :, x1]
        return (fy[:, None] + fx[None, :] + 2)[None, :, :, None] * taps

    got = ops.resize_bilinear(x.to(dev), OH, OW)
    check_close("resize_bilinear", got, fwd(d64(x)), fwd(d64(x).abs()) + pos(d64(x).abs()), 4)
    dout = torch.randn(got.shape, generator=gen)
    din = ops.resize_bilinear_bwd(dout.to(dev), (H, W))
    _, (g,) = vjp64(fwd, [x], dout)
    _, (ga,) = vjp64(fwd, [x.abs()], dout.abs())
    _, (gp,) = vjp64(pos, [x.abs()], dout.abs())
    check_close("resize_bilinear_bwd", din, g, ga + gp, 4)
    assert torch.equal(din, ops.resize_bilinear_bwd(dout.to(dev), (H, W)))


@pytest.mark.parametrize("r,C", [(1, 40), (2, 64), (16, 20)])
def test_masked_mean_bcast_fwd_bwd(gen, r, C):
    """masked_mean_bcast (encoder.py:207-220): out = mtag * sum(x * mref) / max(sum(mref), 1) per sample and channel, masks at
    r times the map's resolution read by nearest sampling; the third sample's reference mask is empty; C is not a multiple
    of the kernel's 32-channel blocks.  Forward and backward vs fp64 autograd.  k = 8 (measured: forward 1.6, backward 1.3)."""
    ops = _ops()
    N, h, w = 3, 8, 6
    x = torch.randn(N, h, w, C, generator=gen)
    mref = (torch.rand(N, h * r, w * r, generator=gen) > 0.5).float()
    mtag = (torch.rand(N, h * r, w * r, generator=gen) > 0.4).float()
    mref[2] = 0.0
    mr = d64(mref[:, ::r, ::r])[..., None]
    mt = d64(mtag[:, ::r, ::r])[..., None]

    def fwd(t):
        return (t * mr).sum((1, 2), keepdim=True) / mr.sum((1, 2), keepdim=True).clamp_min(1.0) * mt

    got = ops.masked_mean_bcast(x.to(dev), mref.to(dev), mtag.to(dev))
    check_close("masked_mean_bcast", got, fwd(d64(x)), fwd(d64(x).abs()), 8)
    dout = torch.randn(x.shape, generator=gen)
    dx = ops.masked_mean_bcast_bwd(dout.to(dev), mref.to(dev), mtag.to(dev))
    _, (g,) = vjp64(fwd, [x], dout)
    _, (ga,) = vjp64(fwd, [x.abs()], dout.abs())
    check_close("masked_mean_bcast_bwd", dx, g, ga, 8)
    assert float(dx[2].abs().max()) == 0.0


# ============================================================================================== spectral norm
@pytest.mark.parametrize("shape", [(64, 3, 3, 3), (1024, 1024, 3, 3)])
def test_spectral_norm_bwd(gen, shape):
    """spectral_norm_bwd vs fp64 autograd of W / (u^T W v) with u, v constants (torch's spectral_norm): O x K = 64 x 27 and
    1024 x 9216, written and accumulated, and twice bit-identical.  R_abs = (|dWt| + |u||v|^T sum|dWt W| / sigma) / sigma.
    k = 8 (measured 1.9)."""
    ops = _ops()
    O, K = shape[0], shape[1] * shape[2] * shape[3]
    w = torch.randn(shape, generator=gen) / K ** 0.5
    v = torch.randn(K, generator=gen)
    v = v / v.norm()
    u = w.view(O, -1) @ v
    u = u / u.norm()
    sigma = float(u.double() @ w.view(O, -1).double() @ v.double())
    inv = torch.tensor([1.0 / sigma], dtype=torch.float32)
    dwt = torch.randn(shape, generator=gen)
    u64, v64 = d64(u), d64(v)
    _, (g,) = vjp64(lambda W: W / (u64 @ W.view(O, -1) @ v64), [w], dwt)
    s_abs = float((d64(dwt).abs() * d64(w).abs()).sum()) / sigma
    rabs = ((d64(dwt).abs().view(O, -1) + s_abs * u64.abs()[:, None] * v64.abs()[None]) / sigma).view(shape)
    args = [t.to(dev) for t in (dwt, w, u, v, inv)]
    got = ops.spectral_norm_bwd(*args)
    check_close("spectral_norm_bwd", got, g, rabs, 8)
    assert torch.equal(got, ops.spectral_norm_bwd(*args))
    out0 = torch.randn(shape, generator=gen)
    got = ops.spectral_norm_bwd(*args, out=out0.to(dev))
    check_close("spectral_norm_bwd accumulate", got, d64(out0) + g, d64(out0).abs() + rabs, 8)


# ============================================================================================== discriminator logits conv
@pytest.mark.parametrize("N,H", [(2, 19), (1, 35), (1, 67)])
def test_conv_to1_fwd_bwd(gen, N, H):
    """conv_to1 (PatchGAN logits: Cin 512 -> 1, k4, pad 2) and conv_to1_bwd vs fp64 autograd at the discriminator's odd
    sizes: dx accumulated onto a non-zero tensor, dw and db; want_dx=False leaves dx alone and gives the same dw, db
    (bit-identical: the weight gradient reduces through fp64).  k = 16 (measured: forward 0.4, dx 3.6, dw 0.2, db 0.02)."""
    ops = _ops()
    Cin, k, pad = 512, 4, 2
    x = torch.randn(N, H, H, Cin, generator=gen)
    w = torch.randn(1, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5
    b = torch.randn(1, generator=gen)

    def fwd(t, ww, bb):
        return nhwc(F.conv2d(nchw(t), ww, bb, padding=pad))

    got = ops.conv_to1(x.to(dev), w.to(dev), b.to(dev), pad)
    ref = fwd(d64(x), d64(w), d64(b))
    check_close("conv_to1", got, ref, fwd(d64(x).abs(), d64(w).abs(), d64(b).abs()), 16)
    dl = torch.randn(ref.shape, generator=gen)
    _, (gx, gw, gb) = vjp64(fwd, [x, w, b], dl)
    _, (ax, aw, ab) = vjp64(fwd, [x.abs(), w.abs(), b.abs()], dl.abs())
    dx0 = torch.randn(x.shape, generator=gen)
    dx, dw, db = ops.conv_to1_bwd(dl.to(dev), x.to(dev), w.to(dev), pad, dx=dx0.to(dev))
    check_close("conv_to1_bwd dx", dx, d64(dx0) + gx, d64(dx0).abs() + ax, 16)
    check_close("conv_to1_bwd dw", dw, gw, aw, 16)
    check_close("conv_to1_bwd db", db, gb, ab, 16)
    dx2, dw2, db2 = ops.conv_to1_bwd(dl.to(dev), x.to(dev), w.to(dev), pad, want_dx=False)
    assert dx2 is None
    assert torch.equal(dw, dw2) and torch.equal(db, db2)


# ============================================================================================== thin convs
@pytest.mark.parametrize("H,W,cin,cinp,k,s,p,c_lo", [(67, 35, 7, 8, 4, 2, 2, 4), (35, 67, 7, 8, 4, 2, 2, 4), (21, 19, 3, 4, 3, 1, 1, 0)])
def test_thin_dgrad3_adds_into_dimg(gen, H, W, cin, cinp, k, s, p, c_lo):
    """thin_dgrad3: the data gradient of a thin conv w.r.t. input channels [c_lo, c_lo+3) (the image inside the input), ADDED
    into a pre-filled NCHW dimg.  D model0 (k4 s2 p2, CinP 8, c_lo 4) at odd sizes and VGG conv1_1 (k3 s1 p1, CinP 4,
    c_lo 0).  k = 8 (measured 2.2)."""
    ops = _ops()
    N, Cout = 2, 64
    x = torch.randn(N, cin, H, W, generator=gen)
    w = torch.randn(Cout, cin, k, k, generator=gen) / (cin * k * k) ** 0.5

    def fwd(t, ww):
        return F.conv2d(t, ww, stride=s, padding=p)

    y = fwd(x, w)
    dz = torch.randn(y.shape, generator=gen)
    _, (gx, _) = vjp64(fwd, [x, w], dz)
    _, (ax, _) = vjp64(fwd, [x.abs(), w.abs()], dz.abs())
    dimg0 = torch.randn(N, 3, H, W, generator=gen)
    got = ops.thin_dgrad3(nhwc(dz).to(dev), ops.pack_weight_thin(w.to(dev), cinp), dimg0.to(dev), k, k, s, p, c_lo)
    check_close("thin_dgrad3", got, d64(dimg0) + gx[:, c_lo:c_lo + 3], d64(dimg0).abs() + ax[:, c_lo:c_lo + 3], 8)


# name, cin, cinp, cout, k, stride, pad, reflect, seg resize R.  cout32: a Cout the register-tiled kernel does not take,
# so mg_thin_wgrad runs its fallback kernel (thin_wgrad_kernel).
_THIN = [("mlp_shared", 4, 4, 128, 3, 1, 1, 0, 2), ("D_model0", 7, 8, 64, 4, 2, 2, 0, 1), ("bg_conv1", 3, 4, 64, 7, 1, 3, 1, 1),
         ("fc_layer1", 3, 4, 64, 3, 2, 1, 0, 1), ("cout32", 3, 4, 32, 3, 1, 1, 0, 1)]


@pytest.mark.parametrize("name,cin,cinp,cout,k,s,p,refl,R", _THIN, ids=[t[0] for t in _THIN])
def test_thin_wgrad(gen, name, cin, cinp, cout, k, s, p, refl, R):
    """Weight gradient of the thin convs at odd sizes on the fp32 CUDA-core kernels: twice, bit-identical, and vs fp64
    autograd.  k = 8 (measured 1.5)."""
    ops = _ops()
    N, H, W = 2, 21, 19
    xf = torch.randn(N, cinp, H * R, W * R, generator=gen)
    xf[:, cin:] = 0.0
    xr = xf[:, :cin, ::R, ::R].contiguous()
    xin = F.pad(xr, (p,) * 4, mode="reflect") if refl else xr
    pc = 0 if refl else p
    w = torch.randn(cout, cin, k, k, generator=gen) / (cin * k * k) ** 0.5

    def fwd(t, ww):
        return F.conv2d(t, ww, stride=s, padding=pc)

    dz = rna_tf32(torch.randn(fwd(xin, w).shape, generator=gen))
    xdev, dzdev = nhwc(xf).to(dev), nhwc(dz).to(dev)

    def oihw(dwt):
        return dwt.view(k, k, cinp, cout).permute(3, 2, 0, 1)[:, :cin]

    dwt = ops.thin_wgrad(xdev, dzdev, k, k, s, p, pad_mode=refl, seg_resize=R if R > 1 else 0, in_hw=(H, W))
    assert torch.equal(dwt, ops.thin_wgrad(xdev, dzdev, k, k, s, p, pad_mode=refl, seg_resize=R if R > 1 else 0, in_hw=(H, W)))
    _, (_, gw) = vjp64(fwd, [xin, w], dz)
    _, (_, aw) = vjp64(fwd, [xin.abs(), w.abs()], dz.abs())
    check_close(name + " thin_wgrad", oihw(dwt), gw, aw, 8)


# ============================================================================================== conv_img (generator output layer)
@pytest.mark.parametrize("Cin,H,W,act_in,act_out", [(32, 20, 45, 2, 3), (64, 9, 33, 2, 3), (128, 20, 45, 2, 3), (64, 17, 70, 0, 0),
                                                    (128, 9, 33, 0, 3), (32, 40, 64, 2, 0)])
def test_conv_img_bwd(gen, Cin, H, W, act_in, act_out):
    """conv_img_bwd vs fp64 autograd of tanh(conv3x3(lrelu(x)) + b) given the saved output y (as torch's tanh backward
    uses it: dz = dy (1 - y^2)): Cin 32/64/128, sizes ragged against the kernel's 8 x 32 tiles, act_in / act_out off.
    dw and db accumulate onto non-zero values (C ABI), and are bit-identical over two calls.  R_abs of dz is
    |dy| (1 + y^2).  k = 16 (measured: dx 4.5, dw 1.1, db 0.2)."""
    ops = _ops()
    N = 2
    x = torch.randn(N, Cin, H, W, generator=gen)
    w = torch.randn(3, Cin, 3, 3, generator=gen) / (Cin * 9) ** 0.5 * 0.7
    b = torch.randn(3, generator=gen) * 0.1

    def ain(t):
        return F.leaky_relu(t, 0.2) if act_in == ops.ACT_LRELU else t

    def pre(t, ww, bb):
        return F.conv2d(ain(t), ww, bb, padding=1)

    p64 = pre(d64(x), d64(w), d64(b))
    y = (torch.tanh(p64) if act_out == ops.ACT_TANH else p64).float()
    dy = torch.randn(y.shape, generator=gen)
    if act_out == ops.ACT_TANH:
        dz, dza = d64(dy) * (1 - d64(y) ** 2), d64(dy).abs() * (1 + d64(y) ** 2)
    else:
        dz, dza = d64(dy), d64(dy).abs()
    _, (gx, gw, gb) = vjp64(pre, [x, w, b], dz)
    _, (ax, aw, ab) = vjp64(pre, [x.abs(), w.abs(), b.abs()], dza)
    args = [t.to(dev) for t in (dy, y, nhwc(x), w)]
    dx, dw, db = ops.conv_img_bwd(*args, act_in=act_in, act_out=act_out)
    check_close("conv_img_bwd dx", dx, nhwc(gx), nhwc(ax), 16)
    check_close("conv_img_bwd dw", dw, gw, aw, 16)
    check_close("conv_img_bwd db", db, gb, ab, 16)
    dx2, dw2, db2 = ops.conv_img_bwd(*args, act_in=act_in, act_out=act_out)
    assert torch.equal(dw, dw2) and torch.equal(db, db2) and torch.equal(dx, dx2)
    # accumulation onto non-zero dw / db through the C ABI (the wrapper always starts from zeros)
    dw0, db0 = torch.randn(w.shape, generator=gen), torch.randn(3, generator=gen)
    dwa, dba = dw0.to(dev), db0.to(dev)
    ws, dxa = torch.empty(N, H, W, 4, device=dev), torch.empty(N, H, W, Cin, device=dev)
    _lib().check(_lib().load().mg_conv_img_bwd(*(ops._p(t) for t in (*args, ws, dxa, dwa, dba)), N, H, W, Cin, 3, act_in, act_out,
                                               ops._stream()), "mg_conv_img_bwd")
    check_close("conv_img_bwd dw accumulate", dwa, d64(dw0) + gw, d64(dw0).abs() + aw, 16)
    check_close("conv_img_bwd db accumulate", dba, d64(db0) + gb, d64(db0).abs() + ab, 16)
    assert torch.equal(dxa, dx)


def test_conv_img_bwd_rejects_cin_above_128():
    """conv_img_wgrad_kernel holds 5 tap slots per thread, which covers the 3x3 taps only while 256 / Cin >= 2, and its
    shared-memory tile outgrows the 200 KB it requests above Cin = 128: the launcher returns -2 before any launch."""
    ops, lib = _ops(), _lib()
    N, H, W, Cin = 1, 4, 8, 256
    t = [torch.zeros(s, device=dev) for s in ((N, 3, H, W), (N, 3, H, W), (N, H, W, Cin), (3, Cin, 3, 3), (N, H, W, 4),
                                             (N, H, W, Cin), (3, Cin, 3, 3), (3,))]
    rc = lib.load().mg_conv_img_bwd(*(ops._p(x) for x in t), N, H, W, Cin, 3, ops.ACT_LRELU, ops.ACT_TANH, ops._stream())
    assert rc == -2
    with pytest.raises(lib.MichiganNativeError, match=r"status -2"):
        ops.conv_img_bwd(t[0], t[1], t[2], t[3])
    torch.cuda.synchronize()


# ============================================================================================== instance norm
@pytest.mark.parametrize("N,H,W,C,pm", [(2, 8, 8, 64, False), (3, 40, 36, 64, True), (2, 12, 12, 512, True), (2, 24, 20, 128, False),
                                        (2, 5, 7, 256, True)])
def test_instance_norm_act_and_in_bwd(gen, N, H, W, C, pm):
    """instance_norm_act_fwd (y and the (rstd, -mean*rstd) table ss) and in_bwd vs fp64 autograd of
    lrelu(instance_norm(x)) * pmul: samples with different statistics, pmul with zeros, HW within one block and over many
    blocks per sample, C 64 .. 512; round_tf32 / round_out must equal RNA rounding of the unrounded result, and in_bwd is
    bit-identical over two calls.
    The variance comes from one-pass fp64 sums of fp32 partials (E[x^2] - mean^2), whose rounding is amplified by
    kappa = 1 + E[x^2] / var per (sample, channel); the magnitudes carry that factor:
    R_abs(rstd) = kappa rstd, R_abs(shift) = kappa (|mean| + E|x|) rstd, x-hat: xa = kappa (|x| + |mean| + E|x|) rstd,
    R_abs(y) = xa |pmul|, R_abs(dx) = kappa rstd (|g| + mean|g| + xa mean(|g| xa)) with |g| = |df pmul|.
    Elements whose x-hat lies within 8 u xa of 0 are left out of the dx check: there the LReLU branch is decided by rounding.
    k = 4 (measured: ss 0.6, y 0.8, dx 0.5)."""
    ops = _ops()
    scale = torch.rand(N, 1, 1, C, generator=gen) * 1.5 + 0.5
    shift = torch.randn(N, 1, 1, C, generator=gen) * 2
    x = torch.randn(N, H, W, C, generator=gen) * scale + shift
    pmul = torch.rand(N, H, W, generator=gen) + 0.5
    pmul[torch.rand(N, H, W, generator=gen) < 0.3] = 0.0
    pm_dev = pmul.to(dev) if pm else None
    pm64 = d64(pmul)[..., None] if pm else torch.ones((), dtype=torch.float64)
    xd = x.to(dev)
    y, ss = ops.instance_norm_act_fwd(xd, pmul=pm_dev)
    yr, ssr = ops.instance_norm_act_fwd(xd, pmul=pm_dev, round_out=True)
    assert torch.equal(ssr, ss) and torch.equal(yr, rna_tf32(y))

    x64 = d64(x)
    mean = x64.mean((1, 2), keepdim=True)
    var = x64.var((1, 2), unbiased=False, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    kappa = 1 + (x64 * x64).mean((1, 2), keepdim=True) / var
    ma = mean.abs() + x64.abs().mean((1, 2), keepdim=True)
    check_close("in ss rstd", ss[:, 0], rstd.view(N, C), (kappa * rstd).view(N, C), 4)
    check_close("in ss shift", ss[:, 1], (-mean * rstd).view(N, C), (kappa * ma * rstd).view(N, C), 4)

    def fwd(t):
        m = t.mean((1, 2), keepdim=True)
        r = 1.0 / torch.sqrt(t.var((1, 2), unbiased=False, keepdim=True) + 1e-5)
        return F.leaky_relu((t - m) * r, 0.2) * pm64

    xa = kappa * (x64.abs() + ma) * rstd
    check_close("in y", y, fwd(x64), xa * pm64.abs(), 4)
    df = torch.randn(x.shape, generator=gen)
    _, (g,) = vjp64(fwd, [x], df)
    ga = d64(df).abs() * pm64.abs()
    rabs = kappa * rstd * (ga + ga.mean((1, 2), keepdim=True) + xa * (ga * xa).mean((1, 2), keepdim=True))
    amb = ((x64 - mean) * rstd).abs() <= 8 * U * xa
    dx = ops.in_bwd(df.to(dev), xd, ss, ops.ACT_LRELU, pmul=pm_dev)
    check_close("in_bwd", dx, g, rabs, 4, skip=amb)
    assert torch.equal(dx, ops.in_bwd(df.to(dev), xd, ss, ops.ACT_LRELU, pmul=pm_dev))
    assert torch.equal(ops.in_bwd(df.to(dev), xd, ss, ops.ACT_LRELU, pmul=pm_dev, round_tf32=True), rna_tf32(dx))


# ============================================================================================== SPADE + batch norm backward
def _unpack_gb(dgb, C):
    """[N,H,W,2C] packed per GEMM N tile as [gamma(BN/2) | beta(BN/2)] -> (dgamma, dbeta) [N,H,W,C]."""
    ops = _ops()
    bn = ops.spade_bn(C)
    half = bn // 2
    t = dgb.float().cpu().view(*dgb.shape[:3], 2 * C // bn, 2, half)
    return t[..., 0, :].reshape(*dgb.shape[:3], C), t[..., 1, :].reshape(*dgb.shape[:3], C)


@pytest.mark.parametrize("C,xs,act,fmt", [(32, 0, 2, 0), (32, 1, 0, 2), (64, 1, 2, 2), (256, 1, 0, 0), (256, 0, 2, 2), (1024, 0, 2, 0),
                                          (1024, 1, 2, 2)])
def test_spade_bwd(gen, C, xs, act, fmt):
    """spade_bwd vs fp64 autograd of h = act(xhat * g1 + beta), xhat = up(x) * ns + nh, with act' read from the saved output h:
    C 32 / 64 (GEMM N tile 64 / 128, one tile), 256 and 1024 (4 and 16 tiles), x_shift 0/1, LReLU and none (norm_s).
    dgb is unpacked column by column; TF32 must be RNA-rounded and bf16 round-to-nearest (within half an ulp of the
    reference, plus k u R_abs).  dxhat, the BN sums (sum dxhat, sum dxhat xhat) and the bias sums (sum dgamma, sum dbeta)
    elementwise; sums and bias sums twice, bit-identical.  k = 4 (measured: dgb 0.7 beyond the half ulp, dxhat 1.0, sums 0.9,
    bias sums 0.5)."""
    ops = _ops()
    N = 2
    H, W = (8, 12) if C <= 256 else (4, 6)
    x = torch.randn(N, H >> xs, W >> xs, C, generator=gen)
    ns = torch.rand(C, generator=gen) + 0.5
    nh = torch.randn(C, generator=gen) * 0.3
    g1 = 1 + 0.3 * torch.randn(N, H, W, C, generator=gen)
    beta = 0.3 * torch.randn(N, H, W, C, generator=gen)
    xh64 = up(d64(x), xs) * d64(ns) + d64(nh)
    xha = up(d64(x).abs(), xs) * d64(ns) + d64(nh).abs()

    def fwd(xh, gg, bb):
        p = xh * gg + bb
        return F.leaky_relu(p, 0.2) if act == ops.ACT_LRELU else p

    h = fwd(xh64, d64(g1), d64(beta)).float()
    dh = torch.randn(N, H, W, C, generator=gen)
    _, (gxh, gg1, gbeta) = vjp64(fwd, [xh64, g1, beta], dh)
    _, (axh, ag1, abeta) = vjp64(lambda a, b_, c_: a * b_ + c_, [xha, g1.abs(), beta.abs()], dh.abs())
    args = [t.to(dev) for t in (dh, h, g1, x)]
    nsd, nhd = ns.to(dev), nh.to(dev)
    dgb, dxhat, sums, bsums = ops.spade_bwd(*args[:3], args[3], xs, nsd, nhd, act, dgb_fmt=fmt)
    assert dgb.dtype == (torch.float32 if fmt == ops.TF32 else torch.bfloat16)
    dg, db = _unpack_gb(dgb, C)
    if fmt == ops.TF32:
        assert int((dgb.view(torch.int32) & 0x1FFF).abs().max()) == 0
    bits = 11 if fmt == ops.TF32 else 8
    check_rounded("spade_bwd dgamma", dg, gg1, ag1, bits, 4)
    check_rounded("spade_bwd dbeta", db, gbeta, abeta, bits, 4)
    check_close("spade_bwd dxhat", dxhat, gxh, axh, 4)
    check_close("spade_bwd sums", sums[:2 * C], torch.cat([gxh.sum((0, 1, 2)), (gxh * xh64).sum((0, 1, 2))]),
                torch.cat([axh.sum((0, 1, 2)), (axh * xha).sum((0, 1, 2))]), 4)
    check_close("spade_bwd bias sums", bsums, torch.cat([gg1.sum((0, 1, 2)), gbeta.sum((0, 1, 2))]),
                torch.cat([ag1.sum((0, 1, 2)), abeta.sum((0, 1, 2))]), 4)
    _, _, sums2, bsums2 = ops.spade_bwd(*args[:3], args[3], xs, nsd, nhd, act, dgb_fmt=fmt)
    assert torch.equal(sums, sums2) and torch.equal(bsums, bsums2)


def _bn_stats(x64, xs):
    xu = up(x64, xs)
    mean = xu.mean((0, 1, 2))
    rstd = 1.0 / torch.sqrt(xu.var((0, 1, 2), unbiased=False) + 1e-5)
    return mean, rstd


def _bn(t, xs):
    xu = up(t, xs)
    return (xu - xu.mean((0, 1, 2))) / torch.sqrt(xu.var((0, 1, 2), unbiased=False) + 1e-5)


def _bn_rabs(x64, xs, ga):
    """Magnitude of rstd * sum_children(g - mean(g) - xhat mean(g xhat)) for |g| = ga (full resolution)."""
    mean, rstd = _bn_stats(x64, xs)
    xa = (up(x64, xs).abs() + mean.abs()) * rstd
    per = rstd * (ga + ga.mean((0, 1, 2)) + xa * (ga * xa).mean((0, 1, 2)))
    N, H, W, C = per.shape
    f = 1 << xs
    return per.view(N, H // f, f, W // f, f, C).sum((2, 4))


@pytest.mark.parametrize("xs,mode,acc", [(0, "count", False), (1, "count", True), (1, "device_count", False), (0, "device_count", True),
                                         (1, "plain", True), (0, "plain", False)])
def test_bn_bwd_apply(gen, xs, mode, acc):
    """bn_bwd_apply vs fp64 autograd of batch norm (batch statistics) through a nearest 2^x_shift upsample, given the BN
    sums (sum g, sum g xhat): the sample count passed in, or read from sums[2C] (count <= 0); sums=None is the plain
    child sum (the upsample backward of an identity shortcut); written or accumulated into a non-zero dx.
    R_abs = rstd sum_children(|g| + mean|g| + xa mean(|g| xa)) with xa = (|up(x)| + |mean|) rstd.  k = 8 (measured: 1.5 with
    statistics, 2.4 plain)."""
    ops = _ops()
    N, hs, ws, C = 2, 6, 5, 64
    H, W = hs << xs, ws << xs
    x = torch.randn(N, hs, ws, C, generator=gen) * 1.3 + 0.4
    g = torch.randn(N, H, W, C, generator=gen)
    dx0 = torch.randn(x.shape, generator=gen)
    x64, g64 = d64(x), d64(g)
    if mode == "plain":
        _, (ref,) = vjp64(lambda t: up(t, xs), [x], g)
        _, (rabs,) = vjp64(lambda t: up(t, xs), [x.abs()], g.abs())
        got = ops.bn_bwd_apply(g.to(dev), x.to(dev), xs, None, None, None, 1, dx=dx0.to(dev) if acc else None)
    else:
        mean, rstd = _bn_stats(x64, xs)
        ns, nh = rstd.float(), (-mean * rstd).float()
        xh = up(x64, xs) * d64(ns) + d64(nh)
        count = N * H * W
        sums = torch.cat([g64.sum((0, 1, 2)), (g64 * xh).sum((0, 1, 2)), torch.tensor([float(count)], dtype=torch.float64)])
        _, (ref,) = vjp64(lambda t: _bn(t, xs), [x], g)
        rabs = _bn_rabs(x64, xs, g64.abs())
        got = ops.bn_bwd_apply(g.to(dev), x.to(dev), xs, ns.to(dev), nh.to(dev), sums.to(dev), count if mode == "count" else 0,
                               dx=dx0.to(dev) if acc else None)
    if acc:
        ref, rabs = ref + d64(dx0), rabs + d64(dx0).abs()
    check_close("bn_bwd_apply " + mode, got, ref, rabs, 8)


def test_spade_bwd_then_bn_bwd_apply_chain(gen):
    """The train step's sequence for one SPADE: spade_bwd -> bn_bwd_apply (count read from sums[2C], as after the cross-rank
    all-reduce) against fp64 autograd w.r.t. x of lrelu(BN(up(x)) * g1 + beta) with batch statistics.  k = 8 (measured 1.2)."""
    ops = _ops()
    N, H, W, C, xs = 2, 8, 8, 64, 1
    x = torch.randn(N, H >> xs, W >> xs, C, generator=gen) * 0.8 - 0.3
    g1 = 1 + 0.3 * torch.randn(N, H, W, C, generator=gen)
    beta = 0.3 * torch.randn(N, H, W, C, generator=gen)
    x64 = d64(x)
    mean, rstd = _bn_stats(x64, xs)
    ns, nh = rstd.float(), (-mean * rstd).float()

    def fwd(t):
        return F.leaky_relu(_bn(t, xs) * d64(g1) + d64(beta), 0.2)

    h = fwd(x64).float()
    dh = torch.randn(N, H, W, C, generator=gen)
    _, (ref,) = vjp64(fwd, [x], dh)
    _, dxhat, sums, _ = ops.spade_bwd(dh.to(dev), h.to(dev), g1.to(dev), x.to(dev), xs, ns.to(dev), nh.to(dev), ops.ACT_LRELU)
    sums[2 * C] = float(N * H * W)
    got = ops.bn_bwd_apply(dxhat, x.to(dev), xs, ns.to(dev), nh.to(dev), sums, 0)
    check_close("spade_bwd -> bn_bwd_apply", got, ref, _bn_rabs(x64, xs, d64(dh).abs() * d64(g1).abs()), 8)


# ============================================================================================== gradient GEMMs
@pytest.mark.parametrize("C,fmt", [(32, 0), (32, 2), (128, 0), (128, 2), (512, 0), (512, 2)])
def test_gamma_beta_gradient_gemms(gen, C, fmt):
    """The two gradient GEMMs of SPADE's fused gamma|beta conv (autograd.py:101-112) vs fp64 autograd of
    conv2d(actv, cat(wg, wb), padding=1) on the kernels' operands: data gradient = conv_igemm on the packed dgb with
    pack_weight_dgrad_gb (TF32 RNA; bf16 = cvt16 of that), weight gradient = conv_wgrad / conv_wgrad16 + unpack_wgrad_gb.
    TF32 and bf16, C 32 (one 64-column tile), 128 and 512 (several 128-column tiles).
    The data gradient is a tensor-core GEMM of depth K = 9 * 2C whose error grows with K: k = 1.25 sqrt(K) (measured max
    ratio / sqrt(K): 0.28 TF32, 0.13 bf16).  The weight gradient reduces its split-K partials in fp64: k = 8 (measured 1.5)."""
    ops = _ops()
    N, H, W, I = 2, 10, 12, 128
    actv = F.relu(torch.randn(N, H, W, I, generator=gen))
    wg = torch.randn(C, I, 3, 3, generator=gen) / (I * 9) ** 0.5
    wb = torch.randn(C, I, 3, 3, generator=gen) / (I * 9) ** 0.5
    bn = ops.spade_bn(C)
    half = bn // 2
    dg, db = torch.randn(N, H, W, C, generator=gen), torch.randn(N, H, W, C, generator=gen)
    packed = torch.stack([dg.view(N, H, W, C // half, half), db.view(N, H, W, C // half, half)], dim=4).reshape(N, H, W, 2 * C)
    wdg = ops.pack_weight_dgrad_gb(wg.to(dev), wb.to(dev))
    if fmt == ops.TF32:
        aq, dq = rna_tf32(actv), rna_tf32(packed)
        wgq, wbq = rna_tf32(wg), rna_tf32(wb)
        dgb = dq.to(dev)
        dactv = ops.conv_igemm(dgb, wdg, I, 3, 3, 1, 1)
        dwp = ops.conv_wgrad(dgb, aq.to(dev), 3, 3, 1, 1)
    else:
        a16, d16 = actv.bfloat16(), packed.bfloat16()
        aq, dq = a16.float(), d16.float()
        wgq, wbq = rna_tf32(wg).bfloat16().float(), rna_tf32(wb).bfloat16().float()
        dgb = d16.to(dev)
        dactv = ops.conv_igemm(dgb, ops.cvt16(wdg, ops.BF16), I, 3, 3, 1, 1, a_fmt=ops.BF16)
        dwp = ops.conv_wgrad16(dgb, a16.to(dev), 3, 3, 1, 1)
    dwg, dwb = ops.unpack_wgrad_gb(dwp, C, I)
    dgq, dbq = _unpack_gb(dq, C)
    dgamma_beta = nchw(torch.cat([dgq, dbq], dim=-1))

    def fwd(a, wg_, wb_):
        return F.conv2d(nchw(a), torch.cat([wg_, wb_]), padding=1)

    _, (ga, gwg, gwb) = vjp64(fwd, [aq, wgq, wbq], dgamma_beta)
    _, (aa, awg, awb) = vjp64(fwd, [aq.abs(), wgq.abs(), wbq.abs()], dgamma_beta.abs())
    check_close("gamma|beta dgrad", dactv, ga, aa, 1.25 * (9 * 2 * C) ** 0.5)
    check_close("gamma|beta wgrad dwg", dwg, gwg, awg, 8)
    check_close("gamma|beta wgrad dwb", dwb, gwb, awb, 8)


# name, N, H, W, Cin, Cout, k, stride, pad: the networks' conv geometries at odd sizes
_GEOMS = [("k3s1p1", 2, 13, 11, 64, 64, 3, 1, 1), ("fc_k3s2p1", 2, 17, 15, 64, 128, 3, 2, 1), ("bg_k4s2p0", 2, 19, 17, 64, 128, 4, 2, 0),
          ("D_k4s2p2", 2, 35, 33, 64, 128, 4, 2, 2), ("D_k4s1p2", 1, 19, 21, 128, 64, 4, 1, 2)]
# k1 s2: the odd parity class has no taps at all (zeroed, or left alone when accumulating)
_DGRAD_GEOMS = _GEOMS + [("k1s2p0", 2, 15, 13, 64, 64, 1, 2, 0)]


@pytest.mark.parametrize("variant", ["fp32", "bf16", "fp32_sn_accumulate", "bf16_sn_out"])
@pytest.mark.parametrize("name,N,H,W,Cin,Cout,k,s,p", _DGRAD_GEOMS, ids=[g[0] for g in _DGRAD_GEOMS])
def test_conv_dgrad(gen, name, N, H, W, Cin, Cout, k, s, p, variant):
    """conv_dgrad (one implicit GEMM per output parity class on dY with flipped sub-kernels) vs fp64 autograd w.r.t. x on the
    kernel's operands: fp32 dY (TF32-exact) and the bf16 dy16 the mixed16 train step passes; inv_sigma (w * inv_sigma rounded
    to TF32, then bf16); out= over a non-zero tensor, overwritten or accumulated (the discriminator adds into the layer
    below).  Odd H, W leave some rows and columns without any output, and k1 s2 has a parity class without taps.
    The error of the tensor-core accumulation grows with the GEMM depth K = ceil(k / s)^2 * Cout of the largest parity
    class: k = 1.25 sqrt(K) (measured max ratio / sqrt(K): 0.36 TF32, 0.16 bf16)."""
    ops = _ops()
    x = torch.randn(N, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5
    bf16, sn = variant.startswith("bf16"), "_sn" in variant
    inv = torch.tensor([0.37], dtype=torch.float32)
    wq = rna_tf32(w * inv if sn else w)
    if bf16:
        wq = wq.bfloat16().float()

    def fwd(t, ww):
        return F.conv2d(t, ww, stride=s, padding=p)

    dy = torch.randn(fwd(x, w).shape, generator=gen)
    dy = dy.bfloat16().float() if bf16 else rna_tf32(dy)
    _, (gx, _) = vjp64(fwd, [x, wq], dy)
    _, (ax, _) = vjp64(fwd, [x.abs(), wq.abs()], dy.abs())
    gx, ax = nhwc(gx), nhwc(ax)
    out0 = torch.randn(N, H, W, Cin, generator=gen) * 10
    acc = variant.endswith("accumulate")
    out = out0.to(dev) if variant.endswith(("accumulate", "out")) else None
    dyd = nhwc(dy).to(dev)
    got = ops.conv_dgrad(dyd, w.to(dev), (H, W), s, p, inv_sigma=inv.to(dev) if sn else None, out=out, accumulate=acc,
                         dy16=dyd.bfloat16() if bf16 else None)
    if acc:
        gx, ax = gx + d64(out0), ax + d64(out0).abs()
    check_close("conv_dgrad %s %s" % (name, variant), got, gx, ax, 1.25 * (((k + s - 1) // s) ** 2 * Cout) ** 0.5)


@pytest.mark.parametrize("fmt", ["tf32", "bf16"])
@pytest.mark.parametrize("name,N,H,W,Cin,Cout,k,s,p", _GEOMS, ids=[g[0] for g in _GEOMS])
def test_conv_wgrad(gen, name, N, H, W, Cin, Cout, k, s, p, fmt):
    """conv_wgrad (TF32, mma.sync, split-K) and conv_wgrad16 (bf16, wgmma) + unpack_wgrad vs fp64 autograd w.r.t. w on the
    kernels' operands, at the networks' conv geometries with odd sizes; twice, bit-identical (the split-K partial sums go
    through fp64).  k = 8 (measured: TF32 1.7, bf16 1.4)."""
    ops = _ops()
    x = torch.randn(N, Cin, H, W, generator=gen)
    w = torch.randn(Cout, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5

    def fwd(t, ww):
        return F.conv2d(t, ww, stride=s, padding=p)

    dy = torch.randn(fwd(x, w).shape, generator=gen)
    if fmt == "tf32":
        xq, dq = rna_tf32(x), rna_tf32(dy)
        xa, da = nhwc(xq).to(dev), nhwc(dq).to(dev)
        dwp = ops.conv_wgrad(da, xa, k, k, s, p)
        again = ops.conv_wgrad(da, xa, k, k, s, p)
    else:
        xa, da = nhwc(x).bfloat16().to(dev), nhwc(dy).bfloat16().to(dev)
        xq, dq = x.bfloat16().float(), dy.bfloat16().float()
        dwp = ops.conv_wgrad16(da, xa, k, k, s, p)
        again = ops.conv_wgrad16(da, xa, k, k, s, p)
    assert torch.equal(dwp, again)
    dw = ops.unpack_wgrad(dwp, tuple(w.shape))
    _, (_, gw) = vjp64(fwd, [xq, w], dq)
    _, (_, aw) = vjp64(fwd, [xq.abs(), w.abs()], dq.abs())
    check_close("conv_wgrad %s %s" % (fmt, name), dw, gw, aw, 8)
