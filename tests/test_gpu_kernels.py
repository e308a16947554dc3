"""Kernel-level parity through the C ABI (ctypes -> libmichigan_sm90.so) against plain PyTorch fp32 references of
the same op on the same seeded inputs.  Tolerances (relative to the reference's abs-max) are stated per case:
operands pre-rounded to the kernel's input format are compared at fp32-accumulation accuracy (2e-5 .. 3e-5); the bf16
hi/lo split paths are compared against the UNROUNDED fp32 conv at 6e-5 (~16 significand bits)."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(autouse=True)
def _fp32_reference():
    """The PyTorch references must be true fp32: cuDNN/cuBLAS use TF32 for fp32 convs unless told otherwise."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _lib_mod():
    from michigan_b200 import _lib
    return _lib


def _ops():
    from michigan_b200 import ops
    return ops


def tf32_trunc(t):
    return (t.view(torch.int32) & ~0x1FFF).view(torch.float32)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def rel_err(got, ref):
    return float((got - ref).abs().max()) / max(float(ref.abs().max()), 1e-6)


@pytest.fixture()
def gen():
    return torch.Generator(device="cpu").manual_seed(1234)


@pytest.mark.parametrize("N,H,W,Cin,Cout,k,s,p", [
    (2, 32, 32, 64, 64, 3, 1, 1), (1, 16, 16, 32, 32, 1, 1, 0), (3, 8, 8, 64, 64, 3, 1, 1), (5, 4, 4, 64, 32, 3, 1, 1),
    (2, 33, 33, 64, 128, 4, 2, 2), (2, 65, 65, 64, 128, 4, 1, 2), (2, 64, 64, 64, 128, 3, 2, 1), (2, 24, 40, 128, 256, 3, 1, 1)])
def test_igemm_tf32_vs_conv2d(gen, N, H, W, Cin, Cout, k, s, p):
    """Implicit-GEMM conv (architecture.py:31-34, discriminator.py:84-96 geometries), TF32-exact operands: 2e-5."""
    ops = _ops()
    x = tf32_trunc(torch.randn(N, Cin, H, W, generator=gen).to(dev))
    w = tf32_trunc((torch.randn(Cout, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5).to(dev))
    b = torch.randn(Cout, generator=gen).to(dev)
    ref = F.leaky_relu(F.conv2d(x, w, b, stride=s, padding=p), 0.2)
    got = ops.conv_igemm(nhwc(x), ops.pack_weight(w, None, round_tf32=True), Cout, k, k, s, p, bias=b, act=ops.ACT_LRELU)
    assert rel_err(nchw(got), ref) <= 2e-5


@pytest.mark.parametrize("N,h,Cin,Cout,k,s,p", [(2, 32, 64, 64, 3, 1, 1), (2, 33, 128, 256, 4, 2, 2), (1, 64, 256, 128, 3, 1, 1),
                                              (3, 8, 64, 64, 1, 1, 0)])
def test_igemm_16bit_operands(gen, N, h, Cin, Cout, k, s, p):
    """fp16 one pass (exact on fp16-rounded operands) and bf16 hi/lo split (merged 2-MMA form for N <= 128, 3 passes
    otherwise; MG_MERGE=0 forces 3 passes) against the unrounded fp32 conv."""
    ops = _ops()
    x = torch.randn(N, Cin, h, h, generator=gen).to(dev)
    w = (torch.randn(Cout, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5).to(dev)
    b = torch.randn(Cout, generator=gen).to(dev)
    got = ops.conv_igemm(nhwc(x).half(), ops.pack_weight16(w, None, ops.F16, split=False), Cout, k, k, s, p, bias=b, a_fmt=ops.F16)
    assert rel_err(nchw(got), F.conv2d(x.half().float(), w.half().float(), b, stride=s, padding=p)) <= 2e-5
    xn = nhwc(x)
    hi = xn.bfloat16()
    lo = (xn - hi.float()).bfloat16()
    ref32 = F.conv2d(x, w, b, stride=s, padding=p)
    wp3 = ops.pack_weight16(w, None, ops.BF16, split=True)
    for merge in ("1", "0"):
        prev_knob = _lib_mod().set_tuning("MG_MERGE", int(merge))
        try:
            got = ops.conv_igemm(hi, wp3, Cout, k, k, s, p, bias=b, a_fmt=ops.BF16, x_lo=lo)
        finally:
            _lib_mod().set_tuning("MG_MERGE", prev_knob)
        assert rel_err(nchw(got), ref32) <= 6e-5, merge


@pytest.mark.parametrize("fmt", ["tf32", "bf3"])
def test_igemm_dual_pipelines(gen, fmt):
    """Persistent CTAs with several tiles each: max_ctas=3 gives 5 and 6 tiles per CTA (odd and even) through one stage ring
    and one accumulator tile.  MG_DUAL has no effect on sm_90a, so both runs take the same path: only the comparison with the
    fp32 conv2d is meaningful."""
    ops = _ops()
    N, h, Cin, Cout = 2, 32, 64, 64
    x = torch.randn(N, Cin, h, h, generator=gen).to(dev)
    w = (torch.randn(Cout, Cin, 3, 3, generator=gen) / 24).to(dev)
    b = torch.randn(Cout, generator=gen).to(dev)
    outs = {}
    for dual in ("1", "0"):
        prev_knob = _lib_mod().set_tuning("MG_DUAL", int(dual))
        try:
            if fmt == "tf32":
                xt, wt = tf32_trunc(x), tf32_trunc(w)
                ref = F.conv2d(xt, wt, b, padding=1)
                outs[dual] = ops.conv_igemm(nhwc(xt), ops.pack_weight(wt, None, round_tf32=True), Cout, 3, 3, 1, 1, bias=b, max_ctas=3)
                tol = 2e-5
            else:
                xn = nhwc(x)
                hi = xn.bfloat16()
                lo = (xn - hi.float()).bfloat16()
                ref = F.conv2d(x, w, b, padding=1)
                outs[dual] = ops.conv_igemm(hi, ops.pack_weight16(w, None, ops.BF16, split=True), Cout, 3, 3, 1, 1, bias=b, a_fmt=ops.BF16,
                                            x_lo=lo, max_ctas=3)
                tol = 6e-5
        finally:
            _lib_mod().set_tuning("MG_DUAL", prev_knob)
        assert rel_err(nchw(outs[dual]), ref) <= tol, dual
    assert torch.equal(outs["1"], outs["0"])   # same MMA order per output tile -> bit-identical


def test_igemm_halo_mode_matches_classic(gen):
    """MG_HALO=1 (one input patch per K chunk, taps through shifted UMMA descriptors) is an alternative schedule of the
    same GEMM: results must agree with the classic per-tap loads to accumulation-order noise."""
    ops = _ops()
    x = tf32_trunc(torch.randn(2, 64, 24, 40, generator=gen).to(dev))
    w = tf32_trunc((torch.randn(128, 64, 3, 3, generator=gen) / 24).to(dev))
    wp = ops.pack_weight(w, None, round_tf32=True)
    outs = []
    for halo in ("0", "1"):
        prev_knob = _lib_mod().set_tuning("MG_HALO", int(halo))
        try:
            outs.append(ops.conv_igemm(nhwc(x), wp, 128, 3, 3, 1, 1))
        finally:
            _lib_mod().set_tuning("MG_HALO", prev_knob)
    ref = F.conv2d(x, w, None, padding=1)
    assert rel_err(nchw(outs[0]), ref) <= 2e-5 and rel_err(nchw(outs[1]), ref) <= 2e-5
    assert rel_err(outs[1], outs[0]) <= 2e-6


@pytest.mark.parametrize("N,h,C,xs", [(2, 32, 64, 0), (2, 32, 128, 1), (1, 64, 32, 0), (3, 8, 256, 1)])
def test_fused_spade_epilogue(gen, N, h, C, xs):
    """normalization.py:110-116 + architecture.py:85 in one kernel: out = lrelu((x-mean)*rstd * (1+gamma) + beta) with
    gamma|beta = conv3x3(actv) in the accumulator, x read at half resolution when the upsample is folded (xs = 1)."""
    ops = _ops()
    actv = tf32_trunc(torch.randn(N, 128, h, h, generator=gen).to(dev))
    wg = tf32_trunc((torch.randn(C, 128, 3, 3, generator=gen) / 34.0).to(dev))
    wb = tf32_trunc((torch.randn(C, 128, 3, 3, generator=gen) / 34.0).to(dev))
    bg = torch.randn(C, generator=gen).to(dev) * 0.1
    bb = torch.randn(C, generator=gen).to(dev) * 0.1
    x = torch.randn(N, C, h >> xs, h >> xs, generator=gen).to(dev)
    mean = torch.randn(C, generator=gen).to(dev) * 0.1
    rstd = torch.rand(C, generator=gen).to(dev) + 0.5
    gamma = F.conv2d(actv, wg, bg, padding=1)
    beta = F.conv2d(actv, wb, bb, padding=1)
    xu = F.interpolate(x, scale_factor=2 ** xs, mode="nearest") if xs else x
    ref = F.leaky_relu((xu - mean.view(1, -1, 1, 1)) * rstd.view(1, -1, 1, 1) * (1 + gamma) + beta, 0.2)
    got = ops.conv_igemm(nhwc(actv), ops.pack_weight_gb(wg, wb), C, 3, 3, 1, 1, act=ops.ACT_LRELU,
                         spade=(nhwc(x), xs, rstd.contiguous(), (-mean * rstd).contiguous(), (1 + bg).contiguous(), bb))
    assert rel_err(nchw(got), ref) <= 3e-5


@pytest.mark.parametrize("N,H,W,R,cin", [(2, 32, 32, 1, 4), (1, 64, 64, 4, 4), (3, 16, 16, 2, 4), (2, 24, 40, 1, 3), (2, 18, 9, 4, 4)])
def test_seg_conv_tensor_core(gen, N, H, W, R, cin):
    """SPADE mlp_shared (normalization.py:92-96,110-111) as one K=128 bf16-split GEMM vs fp32 conv: 3e-5; the direct
    fp32 kernel (MG_SEG_TC=0 route) must agree as well."""
    ops = _ops()
    seg = torch.randn(N, 4, H * R, W * R, generator=gen).to(dev)
    seg[:, cin:] = 0
    w = (torch.randn(128, cin, 3, 3, generator=gen) / 6).to(dev)
    b = torch.randn(128, generator=gen).to(dev)
    ref = F.relu(F.conv2d(seg[:, :cin, ::R, ::R].contiguous(), w, b, padding=1))
    got = ops.conv_seg_tc(nhwc(seg), ops.pack_weight_seg_tc(w), b, seg_resize=R if R > 1 else 0, out_hw=(H, W))
    assert rel_err(nchw(got), ref) <= 3e-5
    direct = ops.conv_thin(nhwc(seg), ops.pack_weight_thin(w, 4), b, 128, 3, 3, 1, 1, seg_resize=R if R > 1 else 0, act=ops.ACT_RELU,
                           out_hw=(H, W))
    assert rel_err(nchw(direct), ref) <= 2e-5
    o32, hi, _ = ops.conv_seg_tc(nhwc(seg), ops.pack_weight_seg_tc(w), b, seg_resize=R if R > 1 else 0, out_hw=(H, W), out16=(ops.F16, False))
    assert torch.equal(hi.float(), o32.half().float())
    # 16-bit-only outputs leave through smem staging + TMA stores (MG_SEG_TMA=1, the default): bit-identical to the
    # register-store epilogue for both formats, on ragged tiles too (the TMA unit clips the part outside the image)
    from michigan_b200 import _lib
    for fmt, split in ((ops.F16, False), (ops.BF16, True)):
        outs = []
        for knob in (0, 1):
            prev = _lib.set_tuning("MG_SEG_TMA", knob)
            try:
                _, h16, l16 = ops.conv_seg_tc(nhwc(seg), ops.pack_weight_seg_tc(w), b, seg_resize=R if R > 1 else 0, out_hw=(H, W),
                                              out16=(fmt, split), want_f32=False)
                torch.cuda.synchronize()
            finally:
                _lib.set_tuning("MG_SEG_TMA", prev)
            outs.append((h16, l16))
        assert torch.equal(outs[0][0], outs[1][0])
        if split:
            assert torch.equal(outs[0][1], outs[1][1])
        recon = outs[1][0].float() + (outs[1][1].float() if split else 0)
        assert rel_err(nchw(recon), ref) <= (3e-5 if split else 1e-3)


@pytest.mark.parametrize("Cin,CinP,Cout,k,s,p,pm", [(4, 4, 128, 3, 1, 1, 0), (7, 8, 64, 4, 2, 2, 0), (3, 4, 64, 7, 1, 3, 1), (3, 4, 64, 3, 2, 1, 0)])
def test_thin_wgrad_vs_autograd(gen, Cin, CinP, Cout, k, s, p, pm):
    """Weight gradient of the thin convs (mlp_shared, D model0, bg conv1 with reflection padding, fc.layer1): fp32
    register-tiled kernel vs torch autograd, 2e-5 relative (summation order)."""
    ops = _ops()
    x = torch.randn(2, Cin, 32, 32, generator=gen).to(dev)
    w = (torch.randn(Cout, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5).to(dev).requires_grad_(True)
    xin = F.pad(x, (p, p, p, p), mode="reflect") if pm else x
    y = F.conv2d(xin, w, None, stride=s, padding=0 if pm else p)
    dz = torch.randn(y.shape, generator=gen).to(dev)
    y.backward(dz)
    dwt = ops.thin_wgrad(ops.nchw_to_nhwc(x, CinP), nhwc(dz), k, k, s, p, pad_mode=pm)
    dw = dwt.view(k, k, CinP, Cout)[:, :, :Cin].permute(3, 2, 0, 1)
    assert rel_err(dw, w.grad) <= 2e-5


def test_thin_wgrad_fused_relu_backward_and_bias(gen):
    """SPADE mlp_shared backward in one kernel: d actv * [actv > 0] applied on the fly, weight gradient over the nearest-resized
    segmap and the bias gradient (per-channel sums), against torch autograd of relu(conv3x3(resize(seg)))."""
    ops = _ops()
    N, hs, R = 2, 24, 2
    seg = torch.randn(N, 4, hs * R, hs * R, generator=gen).to(dev)
    w = (torch.randn(128, 4, 3, 3, generator=gen) / 6).to(dev).requires_grad_(True)
    b = (torch.randn(128, generator=gen) * 0.1).to(dev).requires_grad_(True)
    seg_r = seg[:, :, ::R, ::R]                                  # nearest resize to hs x hs (integer ratio: floor(dst * R))
    actv = F.relu(F.conv2d(seg_r, w, b, padding=1))
    dact = torch.randn(actv.shape, generator=gen).to(dev)
    actv.backward(dact)
    dwt, db = ops.thin_wgrad(nhwc(seg), nhwc(dact), 3, 3, 1, 1, seg_resize=R, in_hw=(hs, hs), relu_src=nhwc(actv.detach()), want_bias=True)
    dw = dwt.view(3, 3, 4, 128).permute(3, 2, 0, 1)
    assert rel_err(dw, w.grad) <= 2e-5
    assert rel_err(db, b.grad) <= 2e-5


@pytest.mark.parametrize("N,h,Cin,Cout,k,s,p", [(2, 32, 64, 64, 3, 1, 1), (2, 33, 64, 128, 4, 2, 2), (3, 8, 128, 64, 1, 1, 0), (2, 32, 64, 128, 3, 2, 1)])
def test_tensor_core_wgrad_and_dgrad(gen, N, h, Cin, Cout, k, s, p):
    """wgrad (both operands MN-major from NHWC, one filter row per CTA) and dgrad (the forward kernel on dY with per-parity
    flipped sub-filters) vs torch autograd on TF32-exact operands: 5e-5 (split-K atomics reorder the fp32 sums)."""
    ops = _ops()
    x = tf32_trunc(torch.randn(N, Cin, h, h, generator=gen).to(dev)).requires_grad_(True)
    w = tf32_trunc((torch.randn(Cout, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5).to(dev)).requires_grad_(True)
    y = F.conv2d(x, w, None, stride=s, padding=p)
    dy = tf32_trunc(torch.randn(y.shape, generator=gen).to(dev))
    y.backward(dy)
    dwp = ops.conv_wgrad(nhwc(dy), nhwc(x.detach()), k, k, s, p)
    dw = ops.unpack_wgrad(dwp, tuple(w.shape))
    assert rel_err(dw, w.grad) <= 5e-5
    dx = ops.conv_dgrad(nhwc(dy), w.detach(), (h, h), s, p)
    assert rel_err(nchw(dx), x.grad) <= 5e-5


@pytest.mark.parametrize("N,h,Cin,Cout,k,s,p", [(2, 32, 64, 64, 3, 1, 1), (2, 40, 128, 256, 3, 1, 1), (2, 33, 64, 128, 4, 2, 2), (3, 8, 128, 64, 1, 1, 0),
                                                   (2, 33, 256, 128, 4, 1, 2), (1, 20, 64, 64, 3, 1, 1)])
def test_wgrad_bf16_operands(gen, N, h, Cin, Cout, k, s, p):
    """The weight-gradient GEMM with bf16 operands (MN-major, plain 128B swizzle, K = 16 pixels per MMA) against torch autograd on
    bf16-exact operands (fp32 accumulation on both sides)."""
    ops = _ops()
    x = torch.randn(N, Cin, h, h, generator=gen).to(dev).bfloat16().float().requires_grad_(True)
    w = (torch.randn(Cout, Cin, k, k, generator=gen) / (Cin * k * k) ** 0.5).to(dev).requires_grad_(True)
    y = F.conv2d(x, w, None, stride=s, padding=p)
    dy = torch.randn(y.shape, generator=gen).to(dev).bfloat16().float()
    y.backward(dy)
    from michigan_b200 import _lib
    for halo in (0, 1):      # 1 (default): stride-1 layers load ONE input patch per stage, the KW taps read shifted views of it
        prev = _lib.set_tuning("MG_WGRAD_HALO", halo)
        try:
            dwp = ops.conv_wgrad16(nhwc(dy).bfloat16(), nhwc(x.detach()).bfloat16(), k, k, s, p)
            dw = ops.unpack_wgrad(dwp, tuple(w.shape))
        finally:
            _lib.set_tuning("MG_WGRAD_HALO", prev)
        assert rel_err(dw, w.grad) <= 5e-5, halo
    assert torch.equal(ops.cvt16(nhwc(dy)), nhwc(dy).bfloat16())
    sums, d16 = ops.chan_sum_cvt16(nhwc(dy))
    assert torch.equal(d16, nhwc(dy).bfloat16())
    assert rel_err(sums, dy.sum(dim=(0, 2, 3))) <= 1e-5


@pytest.mark.parametrize("fmt", ["tf32", "f16", "bf3"])
def test_igemm_dual_pipelines_n256(gen, fmt):
    """Same as test_igemm_dual_pipelines for a 256-column GEMM N (two 128-column tiles); again only the fp32 comparison is
    meaningful."""
    ops = _ops()
    N, h, Cin, Cout = 2, 32, 64, 256
    x = torch.randn(N, Cin, h, h, generator=gen).to(dev)
    w = (torch.randn(Cout, Cin, 3, 3, generator=gen) / 24).to(dev)
    b = torch.randn(Cout, generator=gen).to(dev)
    outs = {}
    for dual in ("2", "0"):
        prev_knob = _lib_mod().set_tuning("MG_DUAL", int(dual))
        try:
            if fmt == "tf32":
                xt, wt = tf32_trunc(x), tf32_trunc(w)
                ref, tol = F.conv2d(xt, wt, b, padding=1), 2e-5
                outs[dual] = ops.conv_igemm(nhwc(xt), ops.pack_weight(wt, None, round_tf32=True), Cout, 3, 3, 1, 1, bias=b, max_ctas=3)
            elif fmt == "f16":
                ref, tol = F.conv2d(x.half().float(), w.half().float(), b, padding=1), 2e-5
                outs[dual] = ops.conv_igemm(nhwc(x).half(), ops.pack_weight16(w, None, ops.F16, split=False), Cout, 3, 3, 1, 1, bias=b,
                                            a_fmt=ops.F16, max_ctas=3)
            else:
                xn = nhwc(x)
                hi = xn.bfloat16()
                lo = (xn - hi.float()).bfloat16()
                ref, tol = F.conv2d(x, w, b, padding=1), 6e-5
                outs[dual] = ops.conv_igemm(hi, ops.pack_weight16(w, None, ops.BF16, split=True), Cout, 3, 3, 1, 1, bias=b, a_fmt=ops.BF16,
                                            x_lo=lo, max_ctas=3)
        finally:
            _lib_mod().set_tuning("MG_DUAL", prev_knob)
        assert rel_err(nchw(outs[dual]), ref) <= tol, dual
    assert torch.equal(outs["2"], outs["0"])


def test_fused_loss_reductions_vs_reference_formulas(gen):
    """GANLoss (hinge, wide-edge weights, loss.py:60-140) and GANFeatLoss (loss.py:163-175) on the fused reduction kernels
    against the oracle's restatement of the reference formulas, values and gradients, at the discriminator's odd output
    sizes (67/35: even and odd pooling windows) and with channels-last feature slices as the discriminator produces them."""
    import michigan_oracle as orc
    from michigan_b200.networks.loss import GANFeatLoss, GANLoss
    from michigan_b200.options import make_opt
    opt = make_opt()
    oopt = orc.default_opt()
    N = 3
    label = torch.zeros(N, 1, 512, 512)
    label[:, :, 100:300, 120:400] = 1.0
    label[1, :, 50:90, 30:500] = 1.0
    sizes = [(67, 64), (35, 128)]

    def make(requires_grad):
        outs = []
        for h, c in sizes:
            feats = [torch.randn(2 * N, h, h, cc, generator=gen).permute(0, 3, 1, 2) for cc in (c, c)]
            outs.append(feats + [torch.randn(2 * N, h, h, 1, generator=gen).permute(0, 3, 1, 2) * 2])
        return outs

    cpu = make(True)
    ref_in = [[t.clone().requires_grad_(True) for t in o] for o in cpu]
    dev_in = [[t.clone().to(dev).requires_grad_(True) for t in o] for o in cpu]

    def halves(outs):
        return [[t[:N] for t in o] for o in outs], [[t[N:] for t in o] for o in outs]

    crit, critF = GANLoss("hinge", opt=opt), GANFeatLoss(opt)
    for name in ("d_fake", "d_real", "g", "feat"):
        rf, rr = halves(ref_in)
        df, dr = halves(dev_in)
        if name == "d_fake":
            ref, got = orc.gan_loss_hinge(rf, False, True, label, oopt), crit(df, False, for_discriminator=True, label=label.to(dev))
        elif name == "d_real":
            ref, got = orc.gan_loss_hinge(rr, True, True, label, oopt), crit(dr, True, for_discriminator=True, label=label.to(dev))
        elif name == "g":
            ref, got = orc.gan_loss_hinge(rf, True, False, label, oopt), crit(df, True, for_discriminator=False, label=label.to(dev))
        else:
            ref, got = orc.gan_feat_loss(rf, rr, oopt), critF(df, dr, label.to(dev))
        assert got.shape == (1,)
        assert abs(float(got) - float(ref)) <= 1e-5 * max(1.0, abs(float(ref))), (name, float(got), float(ref))
        for o in ref_in + dev_in:
            for t in o:
                t.grad = None
        (ref.sum() * 1.7).backward()
        (got.sum() * 1.7).backward()
        for ro, do in zip(ref_in, dev_in):
            for rt, dt in zip(ro, do):
                if rt.grad is None:
                    assert dt.grad is None or float(dt.grad.abs().max()) == 0.0
                else:
                    assert dt.grad is not None, name
                    assert (dt.grad.cpu() - rt.grad).abs().max().item() <= 1e-6 * max(1.0, rt.grad.abs().max().item()), name


@pytest.mark.parametrize("fmt,Cin,Cout,h,w", [("tf32", 64, 64, 48, 32), ("tf32", 32, 256, 40, 64), ("f16", 128, 128, 32, 32),
                                              ("bf3", 128, 64, 40, 48), ("bf3", 64, 128, 32, 32), ("bf3", 64, 256, 32, 32)])
def test_conv3x3_group_kernel_matches_per_tap_kernel(gen, fmt, Cin, Cout, h, w):
    """mg_conv3x3.cu (halo patches shared by two M tiles, one MMA-issuing thread per M tile) against the per-tap kernel and
    against torch, for every operand format and accumulator arrangement: TF32 (4 / 1x2 accumulators), fp16, bf16 hi+lo
    merged (Cout <= 128) and 3-pass (Cout 256); heights that are not a multiple of the 16-row tile; max_ctas forces several
    groups per CTA (ring wrap-around, accumulator double buffering)."""
    ops = _ops()
    N = 2
    x = torch.randn(N, Cin, h, w, generator=gen).to(dev)
    wt = (torch.randn(Cout, Cin, 3, 3, generator=gen) / (3 * Cin ** 0.5)).to(dev)
    b = torch.randn(Cout, generator=gen).to(dev)
    res = torch.randn(N, h, w, Cout, generator=gen).to(dev)

    def run():
        if fmt == "tf32":
            xt, wq = tf32_trunc(x), tf32_trunc(wt)
            return ops.conv_igemm(nhwc(xt), ops.pack_weight(wq, None, round_tf32=True), Cout, 3, 3, 1, 1, bias=b, res=res, act=2, max_ctas=5), \
                F.leaky_relu(F.conv2d(xt, wq, b, padding=1) + nchw(res), 0.2), 2e-5
        if fmt == "f16":
            return ops.conv_igemm(nhwc(x).half(), ops.pack_weight16(wt, None, ops.F16, split=False), Cout, 3, 3, 1, 1, bias=b, res=res, act=2,
                                  a_fmt=ops.F16, max_ctas=5), \
                F.leaky_relu(F.conv2d(x.half().float(), wt.half().float(), b, padding=1) + nchw(res), 0.2), 2e-5
        xn = nhwc(x)
        hi = xn.bfloat16()
        lo = (xn - hi.float()).bfloat16()
        return ops.conv_igemm(hi, ops.pack_weight16(wt, None, ops.BF16, split=True), Cout, 3, 3, 1, 1, bias=b, res=res, act=2, a_fmt=ops.BF16,
                              x_lo=lo, max_ctas=5), F.leaky_relu(F.conv2d(x, wt, b, padding=1) + nchw(res), 0.2), 6e-5

    outs = {}
    for g3 in (2, 0):
        prev = _lib_mod().set_tuning("MG_GROUP3", g3)
        try:
            outs[g3], ref, tol = run()
        finally:
            _lib_mod().set_tuning("MG_GROUP3", prev)
        assert rel_err(nchw(outs[g3]), ref) <= tol, (g3, rel_err(nchw(outs[g3]), ref))
    assert rel_err(outs[2], outs[0]) <= 2e-6


def test_conv3x3_group_kernel_spade_epilogue(gen):
    """The fused SPADE gamma|beta GEMM (fp16 operands, bf16 hi/lo output, folded 2x upsample of x) through the group kernel."""
    ops = _ops()
    N, C, h = 2, 64, 32
    actv = torch.randn(N, h, h, 128, generator=gen).to(dev)
    wg = (torch.randn(C, 128, 3, 3, generator=gen) / 34).to(dev)
    wb = (torch.randn(C, 128, 3, 3, generator=gen) / 34).to(dev)
    xs = torch.randn(N, h // 2, h // 2, C, generator=gen).to(dev)
    ns, nh, g1, bb = [torch.randn(C, generator=gen).to(dev) for _ in range(4)]
    wp = ops.pack_weight_gb16(wg, wb)
    outs = {}
    for g3 in (2, 0):
        prev = _lib_mod().set_tuning("MG_GROUP3", g3)
        try:
            _, hi, lo = ops.conv_igemm(actv.half(), wp, C, 3, 3, 1, 1, act=2, a_fmt=ops.F16, spade=(xs, 1, ns, nh, g1, bb),
                                       out16=(ops.BF16, True), want_f32=False, max_ctas=3)
            outs[g3] = hi.float() + lo.float()
        finally:
            _lib_mod().set_tuning("MG_GROUP3", prev)
    a16 = nchw(actv.half().float())
    gamma = F.conv2d(a16, wg.half().float(), None, padding=1)
    beta = F.conv2d(a16, wb.half().float(), None, padding=1)
    xh = F.interpolate(nchw(xs), scale_factor=2, mode="nearest") * ns.view(1, -1, 1, 1) + nh.view(1, -1, 1, 1)
    ref = F.leaky_relu(xh * (g1.view(1, -1, 1, 1) + gamma) + (bb.view(1, -1, 1, 1) + beta), 0.2)
    assert rel_err(nchw(outs[2]), ref) <= 1e-4 and rel_err(nchw(outs[0]), ref) <= 1e-4
    assert rel_err(outs[2], outs[0]) <= 2e-5


@pytest.mark.parametrize("N,h,w,C,xsh,act", [(2, 32, 32, 128, 1, 2), (1, 24, 40, 128, 0, 0), (2, 16, 48, 256, 1, 2)])
def test_spade_epilogue_tma_store(gen, N, h, w, C, xsh, act):
    """SPADE gamma|beta GEMM -> bf16 hi/lo operand (the SPEC 1/2 epilogue specialisations) against the fp32 formula; ragged tiles
    (24 x 40) exercise the edge masking.  MG_EPI_TMA has no effect on sm_90a: both settings take the same path, so only the
    fp32 comparison is meaningful."""
    ops = _ops()
    actv = torch.randn(N, h, w, 128, generator=gen).to(dev)
    wg = (torch.randn(C, 128, 3, 3, generator=gen) / 34).to(dev)
    wb = (torch.randn(C, 128, 3, 3, generator=gen) / 34).to(dev)
    xs = torch.randn(N, h >> xsh, w >> xsh, C, generator=gen).to(dev)
    ns, nh, g1, bb = [torch.randn(C, generator=gen).to(dev) for _ in range(4)]
    wp = ops.pack_weight_gb16(wg, wb)
    outs = {}
    for knob in (2, 1, 0):      # 2 = 1 + L1 prefetch of x ahead of the accumulator wait
        prev = _lib_mod().set_tuning("MG_EPI_TMA", knob)
        try:
            _, hi, lo = ops.conv_igemm(actv.half(), wp, C, 3, 3, 1, 1, act=act, a_fmt=ops.F16, spade=(xs, xsh, ns, nh, g1, bb),
                                       out16=(ops.BF16, True), want_f32=False, max_ctas=3)
            torch.cuda.synchronize()
            outs[knob] = hi.float() + lo.float()
        finally:
            _lib_mod().set_tuning("MG_EPI_TMA", prev)
    a16 = nchw(actv.half().float())
    gamma = F.conv2d(a16, wg.half().float(), None, padding=1)
    beta = F.conv2d(a16, wb.half().float(), None, padding=1)
    xu = F.interpolate(nchw(xs), scale_factor=2, mode="nearest") if xsh else nchw(xs)
    xh = xu * ns.view(1, -1, 1, 1) + nh.view(1, -1, 1, 1)
    ref = xh * (g1.view(1, -1, 1, 1) + gamma) + (bb.view(1, -1, 1, 1) + beta)
    if act == 2:
        ref = F.leaky_relu(ref, 0.2)
    assert rel_err(nchw(outs[1]), ref) <= 1e-4 and rel_err(nchw(outs[0]), ref) <= 1e-4
    assert torch.equal(outs[2], outs[1])
    assert rel_err(outs[1], outs[0]) <= 2e-5      # hi + lo carries 16 significand bits; the two epilogues contract their FMAs differently


@pytest.mark.parametrize("N,H,W,Cin", [(2, 32, 64, 64), (1, 20, 45, 64), (1, 9, 33, 32)])
def test_conv_img_forward(gen, N, H, W, Cin):
    """conv_img (generator.py:222-224: tanh(conv3x3(leaky_relu(x, 0.2)), Cin -> 3, NCHW output) against a float64 CPU evaluation of
    the same formula; ragged tiles (the kernel works on 8 x 32 pixel tiles with a one-pixel halo).  Bound 5e-5 on outputs in
    [-1, 1]: the kernel accumulates 9*Cin fp32 FMAs sequentially (measured 1.7e-6 against cuDNN's direct fp32 algorithm at 128x128;
    cuDNN itself is 1.2e-5 .. 1.4e-5 away on the small shapes, where it picks a transform-domain algorithm - hence the fp64 reference)."""
    ops = _ops()
    x = torch.randn(N, Cin, H, W, generator=gen)
    w = torch.randn(3, Cin, 3, 3, generator=gen) / (Cin * 9) ** 0.5
    b = torch.randn(3, generator=gen) * 0.1
    ref = torch.tanh(F.conv2d(F.leaky_relu(x.double(), 0.2), w.double(), b.double(), padding=1))
    got = ops.conv_img(nhwc(x.to(dev)), w.to(dev), b.to(dev))
    assert tuple(got.shape) == tuple(ref.shape)
    assert float((got.cpu().double() - ref).abs().max()) <= 5e-5


def test_input_prologue_kernels_vs_reference_formulas(gen):
    """The GPU input prologue (noise pyramid, orientation RGB, hole mask) against numpy/cv2 restatements of the reference's
    per-sample CPU functions (data/base_dataset.py:335-396) on identical random draws."""
    import math
    import cv2
    import numpy as np
    from michigan_b200 import prologue
    n, h, w = 2, 64, 64
    rs = np.random.RandomState(3)
    fields = [rs.normal(loc=0.5, scale=0.25, size=(n, hh, ww, 3)).astype(np.float32) for hh, ww in prologue.noise_octave_sizes(h, w)]
    assert len(fields) == 4
    ref = np.zeros((n, h, w, 3), np.float32)
    for i in range(n):
        acc = np.zeros((h, w, 3), np.float32)
        for f in fields:
            acc += cv2.resize(f[i].astype(np.float64), dsize=(h, w))          # generate_noise: float64 draws, INTER_LINEAR
        ref[i] = acc / len(fields)
    got = prologue.noise_from_fields([torch.from_numpy(f).to(dev) for f in fields], n, h, w)
    assert (got.cpu() - torch.from_numpy(ref).permute(0, 3, 1, 2)).abs().max().item() <= 2e-6
    assert abs(float(prologue.generate_noise(2, 128, 128, dev).mean()) - 0.5) < 0.02

    orient = torch.floor(torch.rand(n, 1, h, w, generator=gen) * 255)
    label = (torch.rand(n, 1, h, w, generator=gen) > 0.4).float()
    exp = torch.zeros(n, 3, h, w)
    for i in range(n):
        om = orient[i, 0].numpy().astype(np.float64) / 255.0 * math.pi
        rgb = np.zeros((h, w, 3))
        rgb[..., 1] = (np.sin(2 * om) + 1) / 2
        rgb[..., 0] = (np.cos(2 * om) + 1) / 2
        rgb[..., 2] = 0.5
        rgb *= label[i, 0].numpy()[..., np.newaxis]
        q = np.uint8(rgb * 255.0).astype(np.float32) / 255.0                 # PIL image -> ToTensor
        exp[i] = torch.from_numpy(q).permute(2, 0, 1) * label[i]
    got = prologue.orient_rgb(orient.to(dev), label.to(dev)).cpu()
    # cos/sin in double on both sides; a product landing within 1 ulp of an integer may truncate differently
    diff = (got - exp).abs()
    assert (diff > 1e-6).float().mean().item() < 1e-3 and diff.max().item() <= 1.0 / 255 + 1e-6

    mask = torch.zeros(n, 1, h, w)
    mask[:, :, 10:50, 12:40] = 1
    omask = mask.clone()
    omask[:, :, 10:20] = 0
    omask[1] = 0                                                              # empty orientation mask: returned as is
    th_u = torch.tensor([0.9, 0.7])
    idx_u = torch.tensor([0.37, 0.5])
    got = prologue.hole_mask(mask.to(dev), omask.to(dev), th_u.to(dev), idx_u.to(dev)).cpu()
    om0 = omask[0, 0].numpy()
    coord = np.where(om0 != 0)
    nums = len(coord[0])
    rr = int(int(0.9 * nums) / math.pi)
    k = min(int(math.floor(np.float32(0.37) * np.float32(nums))), nums - 1)
    cy, cx = coord[0][k], coord[1][k]
    yy, xx = np.mgrid[0:h, 0:w]
    tmp = (((yy - cy) ** 2 + (xx - cx) ** 2) < rr).astype(np.float32)
    exp0 = om0 * tmp + (mask[0, 0].numpy() - om0)
    assert np.array_equal(got[0, 0].numpy(), exp0)
    assert torch.equal(got[1], omask[1])
