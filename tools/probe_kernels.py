"""Development probe (GPU box): every C-ABI kernel against torch-on-GPU fp32 with TF32 disabled.

    python tools/probe_kernels.py <group>      groups: igemm igemm2 spade thin misc perf

Each group runs in its own process (a faulting kernel poisons the CUDA context).  Not a parity test:
tests/ compare against the CPU oracle; this is a fast bring-up/diagnostic tool.
"""
import sys
import os
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

from michigan_b200 import ops  # noqa: E402

dev = "cuda"
FAILS = []


def tf32_trunc(t):
    return (t.view(torch.int32) & ~0x1FFF).view(torch.float32)


def report(name, got, ref, tol):
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    ok = err <= tol * max(scale, 1e-6)
    print("%-58s max|err| %.3e  ref max %.3e  %s" % (name, err, scale, "OK" if ok else "FAIL"), flush=True)
    if not ok:
        FAILS.append(name)
        d = (got - ref).abs()
        idx = torch.nonzero(d > tol * max(scale, 1e-6))
        print("   bad elements: %d / %d ; first: %s" % (idx.shape[0], d.numel(), idx[:5].tolist()))


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


def igemm_case(N, H, W, Cin, Cout, k, s, p, bias=True, act=0, exact=True, tol=2e-5, bn=0, name=None):
    g = torch.Generator(device="cpu").manual_seed(N * 1000 + H * 10 + Cin + Cout + k)
    x = torch.randn(N, Cin, H, W, generator=g).to(dev)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).to(dev)
    b = torch.randn(Cout, generator=g).to(dev) if bias else None
    if exact:
        x = tf32_trunc(x)
        w = tf32_trunc(w)
    ref = F.conv2d(x, w, b, stride=s, padding=p)
    if act == 2:
        ref = F.leaky_relu(ref, 0.2)
    wp = ops.pack_weight(w, None, round_tf32=True)
    got = ops.conv_igemm(nhwc(x), wp, Cout, k, k, s, p, bias=b, act=act, bn=bn)
    torch.cuda.synchronize()
    report(name or "igemm N%d %dx%d %d->%d k%d s%d p%d bn%d" % (N, H, W, Cin, Cout, k, s, p, bn), nchw(got), ref, tol)


def group_igemm():
    igemm_case(2, 32, 32, 64, 64, 3, 1, 1)
    igemm_case(1, 16, 16, 32, 32, 1, 1, 0)
    igemm_case(2, 32, 32, 128, 256, 3, 1, 1)
    igemm_case(1, 64, 64, 64, 128, 3, 1, 1, bn=64)
    igemm_case(2, 16, 16, 256, 512, 3, 1, 1)


def group_igemm2():
    igemm_case(3, 8, 8, 64, 64, 3, 1, 1)          # two images per tile, ragged batch
    igemm_case(5, 4, 4, 64, 32, 3, 1, 1)          # eight images per tile
    igemm_case(2, 33, 33, 64, 128, 4, 2, 2, bias=False)   # PatchGAN geometry, stride 2 via elementStrides
    igemm_case(2, 65, 65, 64, 128, 4, 1, 2, bias=False)   # stride 1 pad 2 (model3)
    igemm_case(2, 66, 66, 64, 64, 4, 2, 1, bias=True, act=1 if False else 0)  # k4 s2 p1 (bg encoder after pad)
    igemm_case(2, 64, 64, 64, 128, 3, 2, 1)       # partial-conv geometry
    igemm_case(2, 32, 32, 64, 64, 3, 1, 1, exact=False, tol=3e-3, name="igemm unrounded inputs (tf32 hw rounding)")
    # larger: multiple tiles per CTA (persistence + ring wrap)
    igemm_case(4, 128, 128, 128, 256, 3, 1, 1)


def group_spade():
    g = torch.Generator(device="cpu").manual_seed(7)
    for (N, h, C, xs) in ((2, 32, 64, 0), (2, 32, 128, 1), (1, 64, 32, 0), (3, 8, 256, 1)):
        actv = tf32_trunc(torch.randn(N, 128, h, h, generator=g).to(dev))
        wg = tf32_trunc((torch.randn(C, 128, 3, 3, generator=g) / 34.0).to(dev))
        wb = tf32_trunc((torch.randn(C, 128, 3, 3, generator=g) / 34.0).to(dev))
        bg = torch.randn(C, generator=g).to(dev) * 0.1
        bb = torch.randn(C, generator=g).to(dev) * 0.1
        xh = h >> xs
        x = torch.randn(N, C, xh, xh, generator=g).to(dev)
        mean = torch.randn(C, generator=g).to(dev) * 0.1
        rstd = (torch.rand(C, generator=g).to(dev) + 0.5)
        gamma = F.conv2d(actv, wg, bg, padding=1)
        beta = F.conv2d(actv, wb, bb, padding=1)
        xu = F.interpolate(x, scale_factor=2 ** xs, mode="nearest") if xs else x
        ref = F.leaky_relu((xu - mean.view(1, -1, 1, 1)) * rstd.view(1, -1, 1, 1) * (1 + gamma) + beta, 0.2)
        wp = ops.pack_weight_gb(wg, wb)
        got = ops.conv_igemm(nhwc(actv), wp, C, 3, 3, 1, 1, act=2,
                             spade=(nhwc(x), xs, rstd.contiguous(), (-mean * rstd).contiguous(), (1 + bg).contiguous(), bb))
        torch.cuda.synchronize()
        report("spade N%d %dx%d C%d xshift%d" % (N, h, h, C, xs), nchw(got), ref, 3e-5)
    # residual (upsampled source) + blend epilogue
    N, h, Cin, Cout = 2, 32, 64, 64
    x = tf32_trunc(torch.randn(N, Cin, h, h, generator=g).to(dev))
    w = tf32_trunc((torch.randn(Cout, Cin, 3, 3, generator=g) / 24.0).to(dev))
    b = torch.randn(Cout, generator=g).to(dev)
    res = torch.randn(N, Cout, h // 2, h // 2, generator=g).to(dev)
    bf = torch.randn(N, Cout, h, h, generator=g).to(dev)
    hair = (torch.rand(N, 4 * h, 4 * h, generator=g) > 0.5).float().to(dev)
    back = (torch.rand(N, 4 * h, 4 * h, generator=g) > 0.5).float().to(dev)
    y = F.conv2d(x, w, b, padding=1) + F.interpolate(res, scale_factor=2, mode="nearest")
    hs = hair[:, ::4, ::4].unsqueeze(1)
    bs = back[:, ::4, ::4].unsqueeze(1)
    ref = bf * (1 - hs) + y * (1 - bs)
    got = ops.conv_igemm(nhwc(x), ops.pack_weight(w), Cout, 3, 3, 1, 1, bias=b, res=nhwc(res), res_shift=1,
                         blend=(nhwc(bf), hair, back, 4))
    torch.cuda.synchronize()
    report("igemm residual(up2)+blend", nchw(got), ref, 3e-5)
    # per-pixel scales (partial conv)
    ps = torch.rand(N, h, h, generator=g).to(dev) + 0.5
    pm = (torch.rand(N, h, h, generator=g) > 0.3).float().to(dev)
    ref = (F.conv2d(x, w, None, padding=1) * ps.unsqueeze(1) + b.view(1, -1, 1, 1)) * pm.unsqueeze(1)
    got = ops.conv_igemm(nhwc(x), ops.pack_weight(w), Cout, 3, 3, 1, 1, bias=b, pscale=ps, pmul=pm)
    torch.cuda.synchronize()
    report("igemm pscale/pmul (partial conv)", nchw(got), ref, 3e-5)


def group_thin():
    g = torch.Generator(device="cpu").manual_seed(11)
    # SPADE mlp_shared with nearest-resized seg
    N, Hf = 2, 64
    seg = torch.randn(N, 4, Hf, Hf, generator=g).to(dev)
    w = (torch.randn(128, 4, 3, 3, generator=g) / 6).to(dev)
    b = torch.randn(128, generator=g).to(dev)
    for h in (64, 32, 8):
        s_r = F.interpolate(seg, size=(h, h), mode="nearest")
        ref = F.relu(F.conv2d(s_r, w, b, padding=1))
        got = ops.conv_thin(nhwc(seg), ops.pack_weight_thin(w, 4), b, 128, 3, 3, 1, 1, seg_resize=Hf // h, act=1,
                            out_hw=(h, h))
        torch.cuda.synchronize()
        report("thin mlp_shared seg %d->%d" % (Hf, h), nchw(got), ref, 1e-5)
    # k7 reflect 3->64
    x = torch.randn(N, 3, 40, 40, generator=g).to(dev)
    w = (torch.randn(64, 3, 7, 7, generator=g) / 12).to(dev)
    b = torch.randn(64, generator=g).to(dev)
    ref = F.relu(F.conv2d(F.pad(x, (3, 3, 3, 3), mode="reflect"), w, b))
    got = ops.conv_thin(ops.nchw_to_nhwc(x, 4), ops.pack_weight_thin(w, 4), b, 64, 7, 7, 1, 3, pad_mode=1, act=1)
    torch.cuda.synchronize()
    report("thin k7 reflect 3->64", nchw(got), ref, 1e-5)
    # D layer 0: 7->64 k4 s2 p2 lrelu
    x = torch.randn(N, 7, 64, 64, generator=g).to(dev)
    w = (torch.randn(64, 7, 4, 4, generator=g) / 10).to(dev)
    b = torch.randn(64, generator=g).to(dev)
    ref = F.leaky_relu(F.conv2d(x, w, b, stride=2, padding=2), 0.2)
    got = ops.conv_thin(ops.nchw_to_nhwc(x, 8), ops.pack_weight_thin(w, 8), b, 64, 4, 4, 2, 2, act=2)
    torch.cuda.synchronize()
    report("thin D0 7->64 k4 s2 p2", nchw(got), ref, 1e-5)
    # partial conv layer 1: 3->64 k3 s2 p1
    x = torch.randn(N, 3, 64, 64, generator=g).to(dev)
    w = (torch.randn(64, 3, 3, 3, generator=g) / 5).to(dev)
    b = torch.randn(64, generator=g).to(dev)
    ref = F.conv2d(x, w, b, stride=2, padding=1)
    got = ops.conv_thin(ops.nchw_to_nhwc(x, 4), ops.pack_weight_thin(w, 4), b, 64, 3, 3, 2, 1)
    torch.cuda.synchronize()
    report("thin 3->64 k3 s2 p1", nchw(got), ref, 1e-5)


def group_misc():
    g = torch.Generator(device="cpu").manual_seed(13)
    N = 2
    x = torch.randn(N, 64, 48, 40, generator=g).to(dev)
    w = (torch.randn(3, 64, 3, 3, generator=g) / 24).to(dev)
    b = torch.randn(3, generator=g).to(dev)
    ref = torch.tanh(F.conv2d(F.leaky_relu(x, 0.2), w, b, padding=1))
    got = ops.conv_img(nhwc(x), w, b)
    torch.cuda.synchronize()
    report("conv_img", got, ref, 1e-5)
    x = torch.randn(N, 128, 18, 18, generator=g).to(dev)
    w = (torch.randn(1, 128, 4, 4, generator=g) / 45).to(dev)
    b = torch.randn(1, generator=g).to(dev)
    ref = F.conv2d(x, w, b, padding=2)
    got = ops.conv_to1(nhwc(x), w, b, 2)
    torch.cuda.synchronize()
    report("conv_to1", nchw(got), ref, 1e-5)
    # BN stats
    for C_, hw in ((64, 64), (1024, 8), (96, 20)):
        x = torch.randn(3, C_, hw, hw, generator=g).to(dev) * 2 + 0.7
        sums = ops.bn_sums(nhwc(x))
        cnt = 3 * hw * hw
        rm = torch.zeros(C_, device=dev); rv = torch.ones(C_, device=dev)
        nscale, nshift, mean, var = ops.bn_finalize(sums, cnt, cnt * 4, running_mean=rm, running_var=rv, want_stats=True)
        torch.cuda.synchronize()
        xd = x.double()
        m_ref = xd.mean(dim=(0, 2, 3)); v_ref = xd.var(dim=(0, 2, 3), unbiased=False)
        report("bn mean C%d" % C_, mean.double(), m_ref, 1e-6)
        report("bn var C%d" % C_, var.double(), v_ref, 1e-6)
        report("bn nscale C%d" % C_, nscale.double(), 1 / torch.sqrt(v_ref + 1e-5), 1e-6)
        report("bn running_var C%d" % C_, rv.double(), 0.9 + 0.1 * v_ref * (4 * cnt) / (4 * cnt - 1), 1e-6)
    # instance norm + lrelu
    x = torch.randn(3, 128, 33, 33, generator=g).to(dev) * 3 + 1
    ref = F.leaky_relu(F.instance_norm(x), 0.2)
    got = ops.instance_norm_act(nhwc(x))
    torch.cuda.synchronize()
    report("instance_norm+lrelu", nchw(got), ref, 1e-5)
    # prep
    tag = (torch.rand(N, 2, 32, 32, generator=g) > 0.5).float().to(dev)
    ori = torch.floor(torch.rand(N, 1, 32, 32, generator=g) * 255).to(dev)
    th = ori / 255.0 * 3.141592653589793
    ref = torch.cat([tag, torch.sin(2 * th) * tag[:, 1:2], torch.cos(2 * th) * tag[:, 1:2]], 1)
    seg4 = ops.prep_seg(tag, ori)
    torch.cuda.synchronize()
    report("prep_seg", nchw(seg4), ref, 2e-6)
    img = torch.randn(N, 3, 32, 32, generator=g).to(dev)
    d8 = ops.prep_dinput(seg4, img)
    report("prep_dinput", nchw(d8)[:, :7], torch.cat([ref, img], 1), 2e-6)
    noise = torch.rand(N, 3, 32, 32, generator=g).to(dev)
    hair = tag[:, 1].contiguous()
    back = ops.maxpool_mask(hair, 5, invert=True)
    ref_back = 1 - F.max_pool2d(hair.unsqueeze(1), 5, 1, 2)
    report("maxpool_mask", back.unsqueeze(1), ref_back, 0)
    bgin = ops.prep_bginput(img, noise, back)
    report("prep_bginput", nchw(bgin)[:, :3], img * ref_back + noise * (1 - ref_back), 1e-6)
    x8 = torch.randn(N, 8, 33, 31, generator=g).to(dev)
    ref = F.avg_pool2d(x8, 3, 2, [1, 1], count_include_pad=False)
    report("avgpool3s2", nchw(ops.avgpool3s2(nhwc(x8))), ref, 1e-6)
    report("nhwc_to_nchw", ops.nhwc_to_nchw(nhwc(x8)), x8, 0)


def group_f16():
    """16-bit operand paths: fp16 one pass (vs fp16-rounded inputs, exact) and bf16 three-pass split
    (vs full fp32 inputs: ~16-bit precision)."""
    g = torch.Generator(device="cpu").manual_seed(21)
    for (N, h, Cin, Cout, k, s_, p_) in ((2, 32, 64, 64, 3, 1, 1), (2, 33, 128, 256, 4, 2, 2), (1, 64, 256, 128, 3, 1, 1), (3, 8, 64, 64, 1, 1, 0)):
        x = torch.randn(N, Cin, h, h, generator=g).to(dev)
        w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).to(dev)
        b = torch.randn(Cout, generator=g).to(dev)
        # fp16 one pass
        xh = nhwc(x).half()
        wp = ops.pack_weight16(w, None, ops.F16, split=False)
        ref = F.conv2d(x.half().float(), w.half().float(), b, stride=s_, padding=p_)
        got = ops.conv_igemm(xh, wp, Cout, k, k, s_, p_, bias=b, a_fmt=ops.F16)
        torch.cuda.synchronize()
        report("fp16 1-pass N%d %d %d->%d k%d s%d" % (N, h, Cin, Cout, k, s_), nchw(got), ref, 2e-5)
        # bf16 split, operands produced by the kernels themselves
        xn = nhwc(x)
        hi = xn.bfloat16()
        lo = (xn - hi.float()).bfloat16()
        wp3 = ops.pack_weight16(w, None, ops.BF16, split=True)
        ref32 = F.conv2d(x, w, b, stride=s_, padding=p_)
        got = ops.conv_igemm(hi, wp3, Cout, k, k, s_, p_, bias=b, a_fmt=ops.BF16, x_lo=lo)
        torch.cuda.synchronize()
        report("bf16 3-pass N%d %d %d->%d k%d s%d (vs fp32)" % (N, h, Cin, Cout, k, s_), nchw(got), ref32, 6e-5)
    # 16-bit copies written by the epilogues / producers
    x = torch.randn(2, 64, 32, 32, generator=g).to(dev)
    w = (torch.randn(64, 64, 3, 3, generator=g) / 24).to(dev)
    o32, hi, lo = ops.conv_igemm(nhwc(tf32_trunc(x)), ops.pack_weight(tf32_trunc(w)), 64, 3, 3, 1, 1, out16=(ops.BF16, True))
    torch.cuda.synchronize()
    report("epilogue bf16 hi+lo reconstructs fp32", hi.float() + lo.float(), o32, 2e-5)
    o32, hi, lo = ops.conv_igemm(nhwc(tf32_trunc(x)), ops.pack_weight(tf32_trunc(w)), 64, 3, 3, 1, 1, out16=(ops.F16, False))
    report("epilogue fp16 hi", hi.float(), o32.half().float(), 0)
    y32, yh, yl = ops.instance_norm_act(nhwc(x), out16=(ops.BF16, True))
    report("instance_norm bf16 hi+lo", yh.float() + yl.float(), y32, 2e-5)
    p32, ph, pl = ops.reflect_pad(nhwc(x), 1, out16=(ops.BF16, True))
    report("reflect_pad bf16 hi+lo", ph.float() + pl.float(), p32, 2e-5)
    seg = torch.randn(2, 4, 64, 64, generator=g).to(dev)
    ws = (torch.randn(128, 4, 3, 3, generator=g) / 6).to(dev)
    bs = torch.randn(128, generator=g).to(dev)
    a32, ah, _ = ops.conv_thin(nhwc(seg), ops.pack_weight_thin(ws, 4), bs, 128, 3, 3, 1, 1, seg_resize=2, act=1, out_hw=(32, 32),
                               out16=(ops.F16, False))
    report("thin conv fp16 copy", ah.float(), a32.half().float(), 0)
    # SPADE fused, fp16 gamma/beta GEMM
    C = 128
    actv = torch.randn(2, 128, 32, 32, generator=g).to(dev).relu()
    wg = (torch.randn(C, 128, 3, 3, generator=g) / 34.0).to(dev)
    wb = (torch.randn(C, 128, 3, 3, generator=g) / 34.0).to(dev)
    xs = torch.randn(2, C, 32, 32, generator=g).to(dev)
    v1 = torch.ones(C, device=dev); v0 = torch.zeros(C, device=dev)
    a16 = nhwc(actv).half()
    gamma = F.conv2d(a16.float().permute(0, 3, 1, 2), wg.half().float(), None, padding=1)
    beta = F.conv2d(a16.float().permute(0, 3, 1, 2), wb.half().float(), None, padding=1)
    ref = F.leaky_relu(xs * (1 + gamma) + beta, 0.2)
    _, hi, lo = ops.conv_igemm(a16, ops.pack_weight_gb16(wg, wb), C, 3, 3, 1, 1, act=2, a_fmt=ops.F16,
                               spade=(nhwc(xs), 0, v1, v0, v1, v0), out16=(ops.BF16, True), want_f32=False)
    torch.cuda.synchronize()
    report("SPADE fp16 GEMM -> bf16 hi+lo", nchw(hi.float() + lo.float()), ref, 3e-5)


def group_halo(pw="16", bo="1"):
    """Halo mode of the implicit GEMM (3x3 s1 p1: one input patch per K chunk, taps through shifted descriptors).
    Run as halo_<PW>_<BO>; every case is also run with MG_HALO=0 and must agree with it bit for bit (same MMA order
    per output element is not guaranteed, so only closeness to the reference is asserted)."""
    os.environ["MG_HALO"] = "1"; os.environ["MG_HALO_PW"] = pw; os.environ["MG_HALO_BO"] = bo
    print("halo mode PW=%s base-offset=%s" % (pw, bo))
    igemm_case(2, 32, 32, 64, 64, 3, 1, 1)
    igemm_case(1, 16, 16, 32, 32, 3, 1, 1)
    igemm_case(2, 32, 32, 128, 256, 3, 1, 1)
    igemm_case(1, 64, 40, 64, 128, 3, 1, 1, bn=64)       # ragged width (40 = 5 tiles of 8), two N tiles
    igemm_case(2, 24, 20, 64, 64, 3, 1, 1)               # partial tiles in both directions
    igemm_case(4, 128, 128, 128, 256, 3, 1, 1)           # many tiles per CTA: ring wrap
    g = torch.Generator(device="cpu").manual_seed(21)
    for (N, h, Cin, Cout) in ((2, 32, 64, 64), (1, 64, 256, 128), (2, 48, 128, 256)):
        x = torch.randn(N, Cin, h, h, generator=g).to(dev)
        w = (torch.randn(Cout, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5).to(dev)
        b = torch.randn(Cout, generator=g).to(dev)
        xh = nhwc(x).half()
        ref = F.conv2d(x.half().float(), w.half().float(), b, padding=1)
        got = ops.conv_igemm(xh, ops.pack_weight16(w, None, ops.F16, split=False), Cout, 3, 3, 1, 1, bias=b, a_fmt=ops.F16)
        torch.cuda.synchronize()
        report("halo fp16 1-pass N%d %d %d->%d" % (N, h, Cin, Cout), nchw(got), ref, 2e-5)
        xn = nhwc(x)
        hi = xn.bfloat16()
        lo = (xn - hi.float()).bfloat16()
        ref32 = F.conv2d(x, w, b, padding=1)
        got = ops.conv_igemm(hi, ops.pack_weight16(w, None, ops.BF16, split=True), Cout, 3, 3, 1, 1, bias=b, a_fmt=ops.BF16, x_lo=lo)
        torch.cuda.synchronize()
        report("halo bf16 3-pass merged N%d %d %d->%d (vs fp32)" % (N, h, Cin, Cout), nchw(got), ref32, 6e-5)
    C = 128
    actv = torch.randn(2, 128, 32, 32, generator=g).to(dev).relu()
    wg = (torch.randn(C, 128, 3, 3, generator=g) / 34.0).to(dev)
    wb = (torch.randn(C, 128, 3, 3, generator=g) / 34.0).to(dev)
    xs = torch.randn(2, C, 16, 16, generator=g).to(dev)
    v1 = torch.ones(C, device=dev); v0 = torch.zeros(C, device=dev)
    a16 = nhwc(actv).half()
    gamma = F.conv2d(a16.float().permute(0, 3, 1, 2), wg.half().float(), None, padding=1)
    beta = F.conv2d(a16.float().permute(0, 3, 1, 2), wb.half().float(), None, padding=1)
    ref = F.leaky_relu(F.interpolate(xs, scale_factor=2, mode="nearest") * (1 + gamma) + beta, 0.2)
    _, hi, lo = ops.conv_igemm(a16, ops.pack_weight_gb16(wg, wb), C, 3, 3, 1, 1, act=2, a_fmt=ops.F16,
                               spade=(nhwc(xs), 1, v1, v0, v1, v0), out16=(ops.BF16, True), want_f32=False)
    torch.cuda.synchronize()
    report("halo SPADE fp16 GEMM -> bf16 hi+lo", nchw(hi.float() + lo.float()), ref, 3e-5)
    # SPADE with the 3-pass bf16 gamma/beta GEMM (policy for feature maps <= 64)
    ah = nhwc(actv).bfloat16(); al = (nhwc(actv) - ah.float()).bfloat16()
    gamma = F.conv2d(actv, wg, None, padding=1); beta = F.conv2d(actv, wb, None, padding=1)
    ref = F.leaky_relu(F.interpolate(xs, scale_factor=2, mode="nearest") * (1 + gamma) + beta, 0.2)
    got = ops.conv_igemm(ah, ops.pack_weight_gb16(wg, wb, ops.BF16, True), C, 3, 3, 1, 1, act=2, a_fmt=ops.BF16, x_lo=al,
                         spade=(nhwc(xs), 1, v1, v0, v1, v0))
    torch.cuda.synchronize()
    report("SPADE bf16 3-pass C128 (BN 256: classic path) (vs fp32)", nchw(got), ref, 6e-5)
    C2 = 64
    xs2 = xs[:, :C2].contiguous()
    gamma = F.conv2d(actv, wg[:C2], None, padding=1); beta = F.conv2d(actv, wb[:C2], None, padding=1)
    ref = F.leaky_relu(F.interpolate(xs2, scale_factor=2, mode="nearest") * (1 + gamma) + beta, 0.2)
    got = ops.conv_igemm(ah, ops.pack_weight_gb16(wg[:C2].contiguous(), wb[:C2].contiguous(), ops.BF16, True), C2, 3, 3, 1, 1, act=2,
                         a_fmt=ops.BF16, x_lo=al, spade=(nhwc(xs2), 1, v1[:C2].contiguous(), v0[:C2].contiguous(), v1[:C2].contiguous(), v0[:C2].contiguous()))
    torch.cuda.synchronize()
    report("halo SPADE bf16 3-pass merged C64 (vs fp32)", nchw(got), ref, 6e-5)
    # timing at the benchmark shapes (halo on vs off)
    for label, Cin, Cout, S, fmt in (("conv_0 up_3 bf16x3 128->64 512^2", 128, 64, 512, "bf3"), ("conv_1 up_3 bf16x3 64->64 512^2", 64, 64, 512, "bf3"),
                                     ("conv_0 up_2 bf16x3 256->128 256^2", 256, 128, 256, "bf3"), ("tf32 128->64 512^2", 128, 64, 512, "tf32")):
        x = torch.randn(8, S, S, Cin, device=dev)
        w = torch.randn(Cout, Cin, 3, 3, device=dev) / (Cin * 9) ** 0.5
        if fmt == "bf3":
            hi = x.bfloat16(); lo = (x - hi.float()).bfloat16()
            wp = ops.pack_weight16(w, None, ops.BF16, split=True)
            f = lambda: ops.conv_igemm(hi, wp, Cout, 3, 3, 1, 1, a_fmt=ops.BF16, x_lo=lo)
        else:
            wp = ops.pack_weight(w, None, round_tf32=True)
            f = lambda: ops.conv_igemm(x, wp, Cout, 3, 3, 1, 1)
        for halo in ("1", "0"):
            os.environ["MG_HALO"] = halo
            print("perf %-36s halo=%s: %.3f ms" % (label, halo, _time(f)), flush=True)
        del x
    os.environ["MG_HALO"] = "1"


def group_segtc():
    """SPADE mlp_shared on tensor cores (bf16 hi/lo split concatenated along K) vs fp32 conv and vs the direct kernel."""
    g = torch.Generator(device="cpu").manual_seed(5)
    for (N, H, W, R, cin) in ((2, 32, 32, 1, 4), (1, 64, 64, 4, 4), (3, 16, 16, 2, 4), (2, 24, 40, 1, 3), (2, 128, 128, 2, 4)):
        seg = torch.randn(N, 4, H * R, W * R, generator=g).to(dev)
        if cin < 4:
            seg[:, cin:] = 0
        w = (torch.randn(128, cin, 3, 3, generator=g) / 6).to(dev)
        b = torch.randn(128, generator=g).to(dev)
        segr = seg[:, :cin, ::R, ::R].contiguous()
        ref = F.relu(F.conv2d(segr, w, b, padding=1))
        wp = ops.pack_weight_seg_tc(w)
        got = ops.conv_seg_tc(nhwc(seg), wp, b, seg_resize=R if R > 1 else 0, out_hw=(H, W))
        torch.cuda.synchronize()
        report("seg_tc N%d %dx%d R%d cin%d fp32 out" % (N, H, W, R, cin), nchw(got), ref, 3e-5)
        o32, hi, lo = ops.conv_seg_tc(nhwc(seg), wp, b, seg_resize=R if R > 1 else 0, out_hw=(H, W), out16=(ops.F16, False))
        report("   fp16 copy", hi.float(), o32.half().float(), 0)
        _, hi, lo = ops.conv_seg_tc(nhwc(seg), wp, b, seg_resize=R if R > 1 else 0, out_hw=(H, W), out16=(ops.BF16, True), want_f32=False)
        report("   bf16 hi+lo", nchw(hi.float() + lo.float()), ref, 5e-5)
        got = ops.conv_seg_tc(nhwc(seg), wp, b, seg_resize=R if R > 1 else 0, out_hw=(H, W), round_out=True)
        report("   tf32-rounded out", nchw(got), ref, 6e-4)
    seg = torch.randn(8, 512, 512, 4, device=dev)
    w = torch.randn(128, 4, 3, 3, device=dev) / 6
    b = torch.randn(128, device=dev)
    wp, wt = ops.pack_weight_seg_tc(w), ops.pack_weight_thin(w, 4)
    for label, kw in (("fp16 out", dict(out16=(ops.F16, False), want_f32=False)), ("fp32 out", dict(round_out=True))):
        t1 = _time(lambda: ops.conv_seg_tc(seg, wp, b, **kw))
        t0 = _time(lambda: ops.conv_thin(seg, wt, b, 128, 3, 3, 1, 1, act=1, **kw))
        print("perf mlp_shared 8x512x512 %s: tensor-core %.3f ms, direct fp32 %.3f ms" % (label, t1, t0), flush=True)
    import ctypes
    from michigan_b200 import _lib
    names = ["mma total", "mma wait-acc-empty", "mma wait-operand", "builder total", "builder gather", "builder wait-empty", "builder store+fence",
             "epi total", "epi wait-acc-full", "epi tmem-ld", "epi transpose+stores"]
    for dbg in (16, 17, 18, 19):
        os.environ["MG_DBG"] = str(dbg)
        ops.conv_seg_tc(seg, wp, b, out16=(ops.F16, False), want_f32=False)
        buf = (ctypes.c_ulonglong * 16)()
        _lib.check(_lib.load().mg_debug_seg_prof(buf), "prof")
        print("seg_tc MG_DBG=%d cycles (CTA 0, 111 tiles): " % dbg + ", ".join("%s %d" % (n, buf[i]) for i, n in enumerate(names)), flush=True)
    os.environ["MG_DBG"] = "0"
    segf = torch.randn(8, 512, 512, 4, device=dev)
    t1 = _time(lambda: ops.conv_seg_tc(segf, wp, b, seg_resize=2, out_hw=(256, 256), out16=(ops.F16, False), want_f32=False))
    t0 = _time(lambda: ops.conv_thin(segf, wt, b, 128, 3, 3, 1, 1, act=1, seg_resize=2, out_hw=(256, 256), out16=(ops.F16, False), want_f32=False))
    print("perf mlp_shared 8x256x256 (R=2) fp16: tensor-core %.3f ms, direct fp32 %.3f ms" % (t1, t0), flush=True)


def group_bwd():
    """Tensor-core weight gradient (MN-major operands, split-K) and data gradient (transposed conv)."""
    g = torch.Generator(device="cpu").manual_seed(31)
    for (N, h, Cin, Cout, k, s_, p_) in ((2, 32, 64, 64, 3, 1, 1), (2, 32, 128, 256, 3, 1, 1), (2, 33, 64, 128, 4, 2, 2),
                                         (2, 65, 64, 128, 4, 1, 2), (2, 34, 64, 64, 4, 2, 0), (2, 32, 64, 128, 3, 2, 1),
                                         (3, 8, 128, 64, 1, 1, 0), (4, 64, 128, 128, 3, 1, 1)):
        x = tf32_trunc(torch.randn(N, Cin, h, h, generator=g).to(dev)).requires_grad_(True)
        w = tf32_trunc((torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).to(dev)).requires_grad_(True)
        y = F.conv2d(x, w, None, stride=s_, padding=p_)
        dy = tf32_trunc(torch.randn(y.shape, generator=g).to(dev))
        y.backward(dy)
        tag = "N%d %d %d->%d k%d s%d p%d" % (N, h, Cin, Cout, k, s_, p_)
        dwp = ops.conv_wgrad(nhwc(dy), nhwc(x.detach()), k, k, s_, p_)
        dw = ops.unpack_wgrad(dwp, tuple(w.shape))
        torch.cuda.synchronize()
        report("wgrad " + tag, dw, w.grad, 5e-5)
        dx = ops.conv_dgrad(nhwc(dy), w.detach(), (h, h), s_, p_)
        torch.cuda.synchronize()
        report("dgrad " + tag, nchw(dx), x.grad, 5e-5)


def group_bwd2():
    """Backward CUDA-core kernels against torch autograd (fp32, GPU)."""
    g = torch.Generator(device="cpu").manual_seed(41)
    # ---- SPADE elementwise backward + BN backward (through a folded 2x upsample)
    for (N, h, C, xs, act) in ((2, 16, 64, 0, 2), (2, 16, 128, 1, 2), (1, 8, 32, 1, 0)):
        hs = h >> xs
        x = torch.randn(N, C, hs, hs, generator=g).to(dev).requires_grad_(True)
        gamma = (torch.randn(N, C, h, h, generator=g).to(dev) * 0.3).requires_grad_(True)
        beta = (torch.randn(N, C, h, h, generator=g).to(dev) * 0.3).requires_grad_(True)
        xu = F.interpolate(x, scale_factor=2 ** xs, mode="nearest") if xs else x
        mean = xu.mean(dim=(0, 2, 3), keepdim=True)
        var = xu.var(dim=(0, 2, 3), unbiased=False, keepdim=True)
        rstd = 1 / torch.sqrt(var + 1e-5)
        xhat = (xu - mean) * rstd
        p_ = xhat * (1 + gamma) + beta
        hh = F.leaky_relu(p_, 0.2) if act == 2 else p_
        dh = torch.randn(N, C, h, h, generator=g).to(dev)
        hh.backward(dh)
        ns = rstd.view(-1).detach().contiguous()
        nh = (-mean.view(-1) * rstd.view(-1)).detach().contiguous()
        dgb, dxhat, sums, _bs = ops.spade_bwd(nhwc(dh), nhwc(hh.detach()), nhwc((1 + gamma).detach()), nhwc(x.detach()), xs, ns, nh, act)
        dx = ops.bn_bwd_apply(dxhat, nhwc(x.detach()), xs, ns, nh, sums, N * h * h)
        torch.cuda.synchronize()
        bn = ops.spade_bn(C); half = bn // 2
        ch = torch.arange(C, device=dev); gi = (ch // half) * bn + ch % half; bi = gi + half
        report("spade_bwd dgamma C%d xs%d" % (C, xs), nchw(dgb[..., gi].contiguous()), gamma.grad, 2e-3)
        report("spade_bwd dbeta  C%d xs%d" % (C, xs), nchw(dgb[..., bi].contiguous()), beta.grad, 2e-3)
        report("bn_bwd dx        C%d xs%d" % (C, xs), nchw(dx), x.grad, 2e-5)
    # ---- plain child-sum (upsample backward)
    gch = torch.randn(2, 32, 16, 16, generator=g).to(dev)
    ref = gch.view(2, 32, 8, 2, 8, 2).sum(dim=(3, 5))
    dxs = ops.bn_bwd_apply(nhwc(gch), nhwc(ref), 1, None, None, None, 1)
    report("upsample bwd (child sum)", nchw(dxs), ref, 1e-6)
    # ---- instance norm + lrelu (+mask) backward
    x = (torch.randn(3, 64, 17, 17, generator=g).to(dev) * 2 + 0.5).requires_grad_(True)
    pm = (torch.rand(3, 17, 17, generator=g) > 0.3).float().to(dev)
    y = F.leaky_relu(F.instance_norm(x), 0.2) * pm.unsqueeze(1)
    dy = torch.randn(3, 64, 17, 17, generator=g).to(dev)
    y.backward(dy)
    yf, ss = ops.instance_norm_act_fwd(nhwc(x.detach()), 2, 1e-5, pmul=pm)
    report("instance_norm_act_fwd", nchw(yf), y.detach(), 1e-5)
    report("in_bwd", nchw(ops.in_bwd(nhwc(dy), nhwc(x.detach()), ss, 2, pmul=pm)), x.grad, 2e-5)
    # ---- thin conv gradients
    for (Cin, CinP, Cout, k, s_, p_, pmode) in ((4, 4, 128, 3, 1, 1, 0), (7, 8, 64, 4, 2, 2, 0), (3, 4, 64, 7, 1, 3, 1), (3, 4, 64, 3, 2, 1, 0)):
        x = torch.randn(2, Cin, 32, 32, generator=g).to(dev).requires_grad_(True)
        w = (torch.randn(Cout, Cin, k, k, generator=g) / 6).to(dev).requires_grad_(True)
        xp = F.pad(x, (p_,) * 4, mode="reflect") if pmode else x
        y = F.conv2d(xp, w, None, stride=s_, padding=0 if pmode else p_)
        dz = torch.randn(y.shape, generator=g).to(dev)
        y.backward(dz)
        dwt = ops.thin_wgrad(ops.nchw_to_nhwc(x.detach(), CinP), nhwc(dz), k, k, s_, p_, pad_mode=pmode)
        dw = dwt.view(k, k, CinP, Cout).permute(3, 2, 0, 1)[:, :Cin]
        torch.cuda.synchronize()
        report("thin_wgrad %d->%d k%d s%d pm%d" % (Cin, Cout, k, s_, pmode), dw, w.grad, 2e-5)
        if Cin == 7:
            dimg = torch.zeros(2, 3, 32, 32, device=dev)
            ops.thin_dgrad3(nhwc(dz), ops.pack_weight_thin(w.detach(), 8), dimg, k, k, s_, p_, 4)
            report("thin_dgrad3 (image channels)", dimg, x.grad[:, 4:7], 2e-5)
    # seg_resize variant of thin_wgrad (mlp_shared)
    seg = torch.randn(2, 4, 64, 64, generator=g).to(dev)
    w = (torch.randn(128, 4, 3, 3, generator=g) / 6).to(dev).requires_grad_(True)
    y = F.conv2d(F.interpolate(seg, size=(16, 16), mode="nearest"), w, None, padding=1)
    dz = torch.randn(y.shape, generator=g).to(dev)
    y.backward(dz)
    dwt = ops.thin_wgrad(nhwc(seg), nhwc(dz), 3, 3, 1, 1, seg_resize=4, in_hw=(16, 16))
    report("thin_wgrad seg_resize", dwt.view(3, 3, 4, 128).permute(3, 2, 0, 1), w.grad, 2e-5)
    # timing at the training shapes
    for label, cinp, cout, k, s_, p_, pm, S_, Nn in (("bg conv1 3->64 k7 reflect 8x512^2", 4, 64, 7, 1, 3, 1, 512, 8),
                                                    ("D model0 7->64 k4 s2 16x512^2", 8, 64, 4, 2, 2, 0, 512, 16),
                                                    ("mlp_shared 4->128 k3 8x512^2", 4, 128, 3, 1, 1, 0, 512, 8)):
        xin = torch.randn(Nn, S_, S_, cinp, device=dev)
        oh = (S_ + 2 * p_ - k) // s_ + 1
        dzz = torch.randn(Nn, oh, oh, cout, device=dev)
        t_new = _time(lambda: ops.thin_wgrad(xin, dzz, k, k, s_, p_, pad_mode=pm))
        print("perf thin wgrad %-36s register-tiled %.3f ms" % (label, t_new), flush=True)
        del xin, dzz
    # ---- conv_img backward
    x = torch.randn(2, 64, 24, 40, generator=g).to(dev).requires_grad_(True)
    w = (torch.randn(3, 64, 3, 3, generator=g) / 24).to(dev).requires_grad_(True)
    b = torch.randn(3, generator=g).to(dev).requires_grad_(True)
    y = torch.tanh(F.conv2d(F.leaky_relu(x, 0.2), w, b, padding=1))
    dy = torch.randn(y.shape, generator=g).to(dev)
    y.backward(dy)
    dx, dw, db = ops.conv_img_bwd(dy, y.detach().contiguous(), nhwc(x.detach()), w.detach())
    torch.cuda.synchronize()
    report("conv_img_bwd dx", nchw(dx), x.grad, 2e-5)
    report("conv_img_bwd dw", dw, w.grad, 2e-5)
    report("conv_img_bwd db", db, b.grad, 2e-5)
    # ---- conv_to1 backward
    x = torch.randn(2, 128, 18, 18, generator=g).to(dev).requires_grad_(True)
    w = (torch.randn(1, 128, 4, 4, generator=g) / 45).to(dev).requires_grad_(True)
    b = torch.randn(1, generator=g).to(dev).requires_grad_(True)
    y = F.conv2d(x, w, b, padding=2)
    dl = torch.randn(y.shape, generator=g).to(dev)
    y.backward(dl)
    dx, dw, db = ops.conv_to1_bwd(nhwc(dl), nhwc(x.detach()), w.detach(), 2)
    torch.cuda.synchronize()
    report("conv_to1_bwd dx", nchw(dx), x.grad, 2e-5)
    report("conv_to1_bwd dw", dw, w.grad, 2e-5)
    report("conv_to1_bwd db", db, b.grad, 2e-5)
    # ---- avg-pool, reflect-pad, bilinear, masked-mean, blend backward
    x = torch.randn(2, 8, 33, 31, generator=g).to(dev).requires_grad_(True)
    y = F.avg_pool2d(x, 3, 2, [1, 1], count_include_pad=False)
    dy = torch.randn(y.shape, generator=g).to(dev)
    y.backward(dy)
    din = torch.zeros(2, 33, 31, 8, device=dev)
    ops.avgpool3s2_bwd(nhwc(dy), din)
    report("avgpool3s2_bwd", nchw(din), x.grad, 1e-5)
    x = torch.randn(2, 32, 12, 14, generator=g).to(dev).requires_grad_(True)
    y = F.pad(x, (1, 1, 1, 1), mode="reflect")
    dy = torch.randn(y.shape, generator=g).to(dev)
    y.backward(dy)
    report("reflect_pad_bwd", nchw(ops.reflect_pad_bwd(nhwc(dy), 1)), x.grad, 1e-5)
    x = torch.randn(2, 64, 16, 16, generator=g).to(dev).requires_grad_(True)
    y = F.interpolate(x, size=(8, 8), mode="bilinear")
    dy = torch.randn(y.shape, generator=g).to(dev)
    y.backward(dy)
    report("resize_bilinear_bwd", nchw(ops.resize_bilinear_bwd(nhwc(dy), (16, 16))), x.grad, 1e-5)
    x = torch.randn(2, 64, 4, 4, generator=g).to(dev).requires_grad_(True)
    mref = (torch.rand(2, 64, 64, generator=g) > 0.5).float().to(dev)
    mtag = (torch.rand(2, 64, 64, generator=g) > 0.5).float().to(dev)
    lr = mref[:, ::16, ::16].unsqueeze(1); lt = mtag[:, ::16, ::16].unsqueeze(1)
    y = ((x * lr).sum(dim=(2, 3), keepdim=True) / lr.sum(dim=(2, 3), keepdim=True).clamp(min=1)) * lt
    dy = torch.randn(y.shape, generator=g).to(dev)
    y.backward(dy)
    report("masked_mean_bcast_bwd", nchw(ops.masked_mean_bcast_bwd(nhwc(dy), mref, mtag)), x.grad, 1e-5)
    dout = torch.randn(2, 32, 16, 16, generator=g).to(dev)
    hair = (torch.rand(2, 64, 64, generator=g) > 0.5).float().to(dev)
    back = (torch.rand(2, 64, 64, generator=g) > 0.5).float().to(dev)
    dyb, dbf = ops.blend_bwd(nhwc(dout), hair, back, 4)
    report("blend_bwd dy", nchw(dyb), dout * (1 - back[:, ::4, ::4].unsqueeze(1)), 1e-6)
    report("blend_bwd dbf", nchw(dbf), dout * (1 - hair[:, ::4, ::4].unsqueeze(1)), 1e-6)
    # ---- spectral norm backward
    import torch.nn as nn
    conv = nn.utils.spectral_norm(nn.Conv2d(64, 32, 3, padding=1)).to(dev)
    conv.train()
    xin = torch.randn(2, 64, 8, 8, generator=g).to(dev)
    yy = conv(xin)
    dyy = torch.randn(yy.shape, generator=g).to(dev)
    yy.backward(dyy)
    with torch.no_grad():
        wmat = conv.weight_orig.reshape(32, -1)
        sigma = torch.dot(conv.weight_u, wmat @ conv.weight_v)
        wt = (conv.weight_orig / sigma).detach().requires_grad_(True)
    F.conv2d(xin, wt, conv.bias.detach(), padding=1).backward(dyy)
    inv = (1.0 / sigma).reshape(1).contiguous()
    got = ops.spectral_norm_bwd(wt.grad.contiguous(), conv.weight_orig.detach(), conv.weight_u, conv.weight_v, inv)
    report("spectral_norm_bwd", got, conv.weight_orig.grad, 2e-5)
    # ---- gamma|beta packed dgrad operand + packed wgrad unpack
    C = 64
    actv = tf32_trunc(torch.randn(2, 128, 16, 16, generator=g).to(dev)).requires_grad_(True)
    wg = tf32_trunc((torch.randn(C, 128, 3, 3, generator=g) / 34).to(dev)).requires_grad_(True)
    wb = tf32_trunc((torch.randn(C, 128, 3, 3, generator=g) / 34).to(dev)).requires_grad_(True)
    gam = F.conv2d(actv, wg, None, padding=1); bet = F.conv2d(actv, wb, None, padding=1)
    dgam = tf32_trunc(torch.randn(gam.shape, generator=g).to(dev)); dbet = tf32_trunc(torch.randn(bet.shape, generator=g).to(dev))
    (gam * dgam + bet * dbet).sum().backward()
    bn = ops.spade_bn(C); half = bn // 2
    ch = torch.arange(C, device=dev); gi = (ch // half) * bn + ch % half; bi = gi + half
    dgb = torch.zeros(2, 16, 16, 2 * C, device=dev)
    dgb[..., gi] = nhwc(dgam); dgb[..., bi] = nhwc(dbet)
    dactv = ops.conv_igemm(dgb, ops.pack_weight_dgrad_gb(wg.detach(), wb.detach()), 128, 3, 3, 1, 1)
    dwg, dwb = ops.unpack_wgrad_gb(ops.conv_wgrad(dgb, nhwc(actv.detach()), 3, 3, 1, 1), C, 128)
    torch.cuda.synchronize()
    report("gamma|beta dgrad (dactv)", nchw(dactv), actv.grad, 5e-5)
    report("gamma|beta wgrad dWg", dwg, wg.grad, 5e-5)
    report("gamma|beta wgrad dWb", dwb, wb.grad, 5e-5)


def _time(fn, iters=5):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def group_perf():
    """Headline GEMM shapes (N=8) in the three operand modes."""
    for (N, h, Cin, C, spade) in ((8, 512, 128, 128, True), (8, 512, 128, 64, False), (8, 256, 128, 256, True),
                                  (8, 256, 256, 128, False), (8, 64, 1024, 512, False)):
        x = torch.randn(N, h, h, Cin, device=dev)
        xs = torch.randn(N, h, h, C, device=dev)
        v = torch.ones(C, device=dev)
        w = torch.randn(C, Cin, 3, 3, device=dev) / 34
        b = torch.zeros(C, device=dev)
        if spade:
            flops = 2.0 * N * h * h * 9 * Cin * 2 * C
            wp32, wp16 = ops.pack_weight_gb(w, w), ops.pack_weight_gb16(w, w)
            x16 = x.half()
            t_tf32 = _time(lambda: ops.conv_igemm(x, wp32, C, 3, 3, 1, 1, act=2, spade=(xs, 0, v, v, v, v), round_out=True))
            t_f16 = _time(lambda: ops.conv_igemm(x16, wp16, C, 3, 3, 1, 1, act=2, spade=(xs, 0, v, v, v, v), a_fmt=ops.F16,
                                                 out16=(ops.BF16, True), want_f32=False))
            print("perf SPADE N%d %dx%d Cin%d C%d: tf32 %.3f ms %.0f TF/s | fp16->bf16 hi/lo %.3f ms %.0f TF/s" %
                  (N, h, h, Cin, C, t_tf32, flops / t_tf32 / 1e9, t_f16, flops / t_f16 / 1e9), flush=True)
        else:
            flops = 2.0 * N * h * h * 9 * Cin * C
            wp32, wp3 = ops.pack_weight(w), ops.pack_weight16(w, None, ops.BF16, True)
            hi = x.bfloat16(); lo = (x - hi.float()).bfloat16()
            t_tf32 = _time(lambda: ops.conv_igemm(x, wp32, C, 3, 3, 1, 1, bias=b))
            t_b3 = _time(lambda: ops.conv_igemm(hi, wp3, C, 3, 3, 1, 1, bias=b, a_fmt=ops.BF16, x_lo=lo))
            print("perf conv  N%d %dx%d Cin%d C%d: tf32 %.3f ms %.0f TF/s | bf16x3 %.3f ms %.0f TF/s (useful)" %
                  (N, h, h, Cin, C, t_tf32, flops / t_tf32 / 1e9, t_b3, flops / t_b3 / 1e9), flush=True)
    # thin convs
    seg = torch.randn(8, 512, 512, 4, device=dev)
    ws = ops.pack_weight_thin(torch.randn(128, 4, 3, 3, device=dev), 4)
    bs = torch.zeros(128, device=dev)
    t = _time(lambda: ops.conv_thin(seg, ws, bs, 128, 3, 3, 1, 1, seg_resize=1, act=1, out_hw=(512, 512), out16=(ops.F16, False), want_f32=False))
    print("perf mlp_shared 8x512x512 -> fp16: %.3f ms (%.2f TB/s written)" % (t, 8 * 512 * 512 * 128 * 2 / t / 1e9), flush=True)
    img = torch.randn(8, 512, 512, 4, device=dev)
    w7 = ops.pack_weight_thin(torch.randn(64, 3, 7, 7, device=dev), 4)
    t = _time(lambda: ops.conv_thin(img, w7, torch.zeros(64, device=dev), 64, 7, 7, 1, 3, pad_mode=1, act=1))
    print("perf bg conv1 k7 8x512x512: %.3f ms" % t, flush=True)
    # backward GEMMs
    dy = torch.randn(8, 256, 256, 128, device=dev)
    xa = torch.randn(8, 256, 256, 256, device=dev)
    wq = torch.randn(128, 256, 3, 3, device=dev) / 48
    flops = 2.0 * 8 * 256 * 256 * 9 * 256 * 128
    t = _time(lambda: ops.conv_wgrad(dy, xa, 3, 3, 1, 1))
    print("perf wgrad 8x256x256 256->128: %.3f ms %.0f TF/s" % (t, flops / t / 1e9), flush=True)
    t = _time(lambda: ops.conv_dgrad(dy, wq, (256, 256), 1, 1))
    print("perf dgrad 8x256x256 256->128: %.3f ms %.0f TF/s" % (t, flops / t / 1e9), flush=True)


if __name__ == "__main__":
    grp = sys.argv[1]
    if grp.startswith("halo_"):
        _, pw, bo = grp.split("_")
        group_halo(pw, bo)
        print("== group %s done, failures: %s" % (grp, FAILS))
        sys.exit(1 if FAILS else 0)
    t0 = time.time()
    print("== group %s on %s" % (grp, torch.cuda.get_device_name(0)), flush=True)
    globals()["group_" + grp]()
    torch.cuda.synchronize()
    print("== group %s done in %.1fs, failures: %s" % (grp, time.time() - t0, FAILS), flush=True)
    sys.exit(1 if FAILS else 0)
