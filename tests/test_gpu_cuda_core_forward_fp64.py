"""The CUDA-core forward kernels, called directly through their ops.* wrappers (or the C ABI where no wrapper exposes the
output) and compared element by element with a float64 CPU reference of the operation they compute, fed the kernel's exact
fp32 inputs:

  * BatchNorm statistics     chan_stats_kernel (mg_bn_stats, mg_bn_stats_cvt16), bn_finalize_kernel, bn_from_running_kernel
  * spectral norm            sn_wtu / sn_wv / sn_finish_kernel (mg_spectral_norm_batched, through SpectralNormBatch)
  * thin convs               thin_gemm_kernel, thin_conv_kernel (mg_conv_thin), every route MG_THIN_GEMM selects
  * partial-conv masks       partial_mask_kernel;  mask dilation: maxfilt_kernel (mg_maxpool_mask)
  * input preparation        prep_seg / prep_dinput / prep_bginput, nchw_to_nhwc, nhwc_to_nchw
  * attention softmax        softmax_rows_kernel;  hinge-loss weight map: edge_weight_kernel

Error model, where something sums:

    |got - ref| <= k * u * R_abs + tiny,      u = 2^-24,

R_abs = the same formula on absolute values (per case below).  Each case prints its measured max |got - ref| / (u R_abs)
next to k; k is at least 3x the value measured on an H100 80GB HBM3 (700 W power limit), given next to each constant.
Every output that is defined bit for bit (copies, max filters, masks, eager-order fp32 expressions of the reference, the
running-statistics update, 16-bit splits, round_out) is compared bit for bit.
"""
import math
import types
import zlib

import pytest
import torch
import torch.nn.functional as F

dev = "cuda"
U = 2.0 ** -24
TINY = 1e-30
# fp32 runs of 32 pixels, then fp64: a run's rounding error is at most 31 u sum|x| (Sigma x) / 32 u sum x^2 (Sigma x^2, one
# fma per pixel).  k is that worst-case bound; measured max ratio 2.7 (C 4096, P 7).  bn_finalize's bounds carry K_STATS
# through the variance (k = 1 there; measured 0.27).
K_STATS = 32.0
# sqrt(K) model of the fp32 dot products (thin convs, spectral norm), as tests/test_gpu_conv_forward_fp64.py.  Measured: thin
# convs 4.7 against k = 25.5 (K = 196) and 4.0 against k = 15.5 (K = 36, pscale), at most 1/3.8 of k in every case;
# spectral norm 0.094 sqrt(O + K).
C_DOT = 1.25
K_EPI = 8.0
# softmax: expf (<= 2 ulp), the rounded exponent argument (carried in R_abs), the row sum (sqrt(cols) model), one product.
# Measured max ratio 1.1 (cols 4096, k = 88).
K_SOFTMAX = 8.0


def _ops():
    from michigan_b200 import ops
    return ops


def _lib():
    from michigan_b200 import _lib
    return _lib


# ============================================================================================== helpers (as in the conv tests)
def rna_tf32(t):
    """cvt.rna.tf32.f32 on finite fp32 values: round the magnitude to 10 stored mantissa bits, ties away from zero."""
    return ((t.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def nchw(t):
    return t.permute(0, 3, 1, 2).contiguous()


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


def check_rounded(name, got, ref, rabs, bits, k):
    """got = ref rounded to nearest at `bits` significant bits up to k*u*R_abs of accumulated error."""
    got, ref, rabs = d64(got), d64(ref), d64(rabs)
    _, e = torch.frexp(ref)
    half_ulp = torch.ldexp(torch.ones_like(ref), (e - bits - 1).to(torch.int64))
    err = (got - ref).abs()
    ratio = float(((err - half_ulp).clamp_min(0) / (U * rabs + TINY)).max())
    print("%s: max (|got - ref| - ulp/2) / (u R_abs) = %.3g (k = %g)" % (name, ratio, k))
    bad = err > half_ulp + k * U * rabs + TINY
    assert not bool(bad.any()), (name, int(bad.sum()), ratio, k)
    return ratio


T16 = {"f16": torch.float16, "bf16": torch.bfloat16}
FMT = {"f16": 1, "bf16": 2}


def cvt16(v32, fmt):
    if fmt == "f16":
        v32 = v32.clamp(-65504.0, 65504.0)
    return v32.to(T16[fmt])


def split16(v32, fmt):
    """(hi, lo) = (cvt(v), cvt(v - float(hi))), as the kernels' split16."""
    hi = cvt16(v32, fmt)
    return hi, (v32 - hi.float()).to(T16[fmt])


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


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _launched(fn):
    """fn() under torch.profiler -> (result, names of the CUDA kernels launched)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = fn()
        torch.cuda.synchronize()
    return res, {ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA}


def _with_knobs(knobs, fn):
    lib, prev = _lib(), {}
    try:
        for k_, v_ in knobs.items():
            prev[k_] = lib.set_tuning(k_, v_)
        return fn()
    finally:
        for k_, v_ in reversed(list(prev.items())):
            lib.set_tuning(k_, v_)


# ============================================================================================== BatchNorm statistics
def _stats_step(P, C):
    """Pixel stride of one thread's 4-load group in chan_stats_kernel (launch_stats: rows of threads x blocks)."""
    tpr = min(C // 4, 256)
    rows = 256 // tpr
    want = min(max(-(-P // (rows * 8)), 1), _num_sms() * 3)
    return want * rows


def _stats_cases():
    """(C, P) pairs: rows = 256 (C 4), 85 rows of 3 threads = 255 of 256 threads (C 12), one row (C 1024), the channel-group
    loop running twice / four times (C 2048 / 4096); P = 1, 7, ~1e6, and P just below / at / above a multiple of the
    4-load group (4 x step) where the blocks per channel are capped at one wave."""
    return [(4, 1), (4, 7), (4, (1 << 20) + 3), (12, 7), (12, 1000), (64, 1), (64, 7), (1024, 1), (1024, 513),
            (2048, 33), (4096, 7), (4096, 300)]


STATS_CASES = _stats_cases() + [("group", C, d) for C in (12, 64) for d in (-1, 0, 1)]


def _stats_data(g, P, C, offset=True):
    x = torch.randn(P, C, generator=g)
    if offset:
        x = x * (0.1 + 2 * torch.rand(C, generator=g)) + 3 * torch.randn(C, generator=g)
    return x


def _call_stats(x, cvt16=False):
    """-> (sums [2C + 1] fp64, bf16 copy or None) through mg_bn_stats / mg_bn_stats_cvt16."""
    ops, lib = _ops(), _lib()
    C_ = x.shape[-1]
    if not cvt16:
        return ops.bn_sums(x).cpu(), None
    sums = torch.zeros(2 * C_ + 1, device=dev, dtype=torch.float64)
    out = torch.empty(x.shape, device=dev, dtype=torch.bfloat16)
    lib.check(lib.load().mg_bn_stats_cvt16(x.data_ptr(), x.numel() // C_, C_, sums.data_ptr(), out.data_ptr(),
                                           ops._stream()), "mg_bn_stats_cvt16")
    torch.cuda.synchronize()
    return sums.cpu(), out.cpu()


def _check_sums(name, sums, x):
    C_ = x.shape[-1]
    xd = x.double()
    r1 = check_close(name + ": sum x", sums[:C_], xd.sum(0), xd.abs().sum(0), K_STATS)
    r2 = check_close(name + ": sum x^2", sums[C_:2 * C_], (xd * xd).sum(0), (xd * xd).sum(0), K_STATS)
    assert float(sums[2 * C_]) == 0.0, name      # the count slot is the caller's
    return max(r1, r2)


@pytest.mark.gpu
@pytest.mark.parametrize("case", STATS_CASES, ids=lambda c: "C%d_P%s" % (c[1], "4step%+d" % c[2]) if c[0] == "group"
                         else "C%d_P%d" % c)
def test_bn_stats(case):
    if case[0] == "group":
        _, C_, d = case
        tpr = min(C_ // 4, 256)
        rows = 256 // tpr
        step = _num_sms() * 3 * rows
        P = 2 * 4 * step + d
        assert _stats_step(P, C_) == step
    else:
        C_, P = case
    name = "bn_stats C%d P%d" % (C_, P)
    x = _stats_data(_gen(name), P, C_)
    xg = x.to(dev)
    sums, _ = _call_stats(xg)
    ratio = _check_sums(name, sums, x)
    sums2, copy = _call_stats(xg, cvt16=True)
    _check_sums(name + " (cvt16)", sums2, x)
    same_bits(name + ": bf16 copy", copy, x.to(torch.bfloat16))
    # generator-like data: the fp32 runs and the fixed-order block reduction are deterministic, and the block partials add
    # exactly in fp64, so the atomics' order does not show
    same_bits(name + ": second run", _call_stats(xg)[0], sums)
    same_bits(name + ": cvt16 sums = plain sums", sums2, sums)
    print("CASE bn_stats C=%d P=%d max ratio %.3g (k %g)" % (C_, P, ratio, K_STATS))


@pytest.mark.gpu
def test_bn_stats_rejects_unsupported_channel_counts():
    lib = _lib()
    x = torch.zeros(8, 1028, device=dev)
    with pytest.raises(lib.MichiganNativeError, match=r"status -2"):
        _ops().bn_sums(x)


def _wide_range_channel(g, P):
    """|x| log-uniform over 2^-20 ... 2^10, random signs, in blocks of 4096 pixels of one decade each (so that whole
    fp32 runs - and whole CTA partials - sit at either end of the range)."""
    e = torch.empty(P)
    for i in range(0, P, 4096):
        lo = float(torch.randint(-20, 10, (1,), generator=g))
        e[i:i + 4096] = lo + torch.rand(min(4096, P - i), generator=g)
    s = torch.where(torch.rand(P, generator=g) < 0.5, -1.0, 1.0)
    return s * torch.exp2(e)


@pytest.mark.gpu
def test_bn_stats_reproducibility_wide_range():
    """Three runs on a channel whose values span 2^-20 ... 2^10.  The CTA partials then need more than fp64's 53 bits, so
    the order of the atomic adds can show in the last bits of the fp64 sums: the runs are held to the fp64 rounding of
    that order (a few u_64 * sum|x|), and to the fp32-run bound against the reference.  The fp32 results BatchNorm
    consumes (nscale, nshift, mean, var) can then differ by one rounding step: at most 1 fp32 ulp across the runs."""
    P, C_ = 1 << 20, 4
    g = _gen("wide")
    x = torch.stack([_wide_range_channel(g, P), torch.randn(P, generator=g), _wide_range_channel(g, P),
                     torch.randn(P, generator=g) * 1e3], 1).contiguous()
    xg = x.to(dev)
    runs = [_call_stats(xg)[0] for _ in range(3)]
    _check_sums("wide range", runs[0], x)
    xd = x.double()
    r_abs = torch.cat([xd.abs().sum(0), (xd * xd).sum(0)])
    u64 = 2.0 ** -53
    n_blocks = _num_sms() * 3
    differ = 0
    for r in runs[1:]:
        d = (r[:2 * C_] - runs[0][:2 * C_]).abs()
        differ += int((d != 0).sum())
        assert bool((d <= 2 * n_blocks * u64 * r_abs).all()), (d, r_abs)
    print("wide range: %d of %d fp64 sums differ between runs (allowed: fp64 rounding of the add order)" % (differ, 4 * C_))
    outs = []
    for r in runs:
        outs.append(_ops().bn_finalize(r.to(dev), float(P), want_stats=True))
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            a, b = d64(a), d64(b)
            _, e = torch.frexp(torch.maximum(a.abs(), b.abs()))
            ulp = torch.ldexp(torch.ones_like(a), (e - 24).to(torch.int64))
            assert bool(((a - b).abs() <= ulp).all()), ("wide range: fp32 statistics across runs differ by more than 1 ulp", a, b)


# ============================================================================================== bn_finalize / bn_from_running
def _finalize_ref(S, Q, n, eps, clamp_mode):
    mean = S / n
    var = (Q / n - mean * mean).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var.clamp_min(eps) if clamp_mode else var + eps)
    return mean, var, rstd


def _eager_running(running, stat32, momentum):
    """batchnorm.py:139-143 in fp32 eager order: (1 - m) * running + m * stat, each product rounded, then the add."""
    a = torch.tensor(1 - momentum, dtype=torch.float32)
    m = torch.tensor(momentum, dtype=torch.float32)
    return (a * running) + (m * stat32)


FIN_CASES = [
    # name, count mode, unbiased_mult, clamp_mode
    ("host_count", "host", 1, 0),
    ("device_count", "device", 1, 0),
    ("unbiased_x4", "host", 4, 0),
    ("unbiased_x16_device", "device", 16, 1),
    ("clamp_mode1", "host", 1, 1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", FIN_CASES, ids=lambda c: c[0])
def test_bn_finalize(case):
    name, cmode, mult, clamp = case
    ops = _ops()
    g = _gen("fin" + name)
    P, C_ = 3000, 16
    eps, momentum = 1e-5, 0.1
    eps64 = float(torch.tensor(eps, dtype=torch.float32))       # the kernel takes eps as a float
    x = torch.randn(P, C_, generator=g) * (0.5 + torch.rand(C_, generator=g)) + torch.randn(C_, generator=g)
    x[:, 1] = 0.1                                       # constant channel: var rounds to <= 0 and must clamp to 0
    x[:, 2] = 100.0 + 1.0 * torch.randn(P, generator=g)  # |mean| = 100 std: cancellation in E[x^2] - mean^2
    x[:, 3] *= 1e-3                                     # var < eps (clamp_mode 1 takes eps)
    sums = ops.bn_sums(x.to(dev))
    n = float(P)
    if cmode == "device":
        sums[2 * C_] = n
        count = 0.0
    else:
        count = n
    rm0 = torch.randn(C_, generator=g)
    rv0 = torch.rand(C_, generator=g) + 0.5
    # momentum 1: running = 0 * running + 1 * stat = the kernel's own fp32 mean and unbiased var, exactly
    rm1, rv1 = torch.zeros(C_, device=dev), torch.zeros(C_, device=dev)
    ops.bn_finalize(sums, count, unbiased_mult=mult, eps=eps, momentum=1.0, clamp_mode=clamp, running_mean=rm1, running_var=rv1)
    rm, rv = rm0.to(dev), rv0.to(dev)
    nscale, nshift, mean32, var32 = ops.bn_finalize(sums, count, unbiased_mult=mult, eps=eps, momentum=momentum,
                                                    clamp_mode=clamp, running_mean=rm, running_var=rv, want_stats=True)
    torch.cuda.synchronize()

    # fp64 reference from the data itself (two-pass variance), and the error the fp32 runs of Sigma x, Sigma x^2 carry in
    xd = x.double()
    mean, var, rstd = _finalize_ref(xd.sum(0), (xd * xd).sum(0), n, eps64, clamp)
    var2 = ((xd - mean) ** 2).mean(0)
    ex1, ex2 = xd.abs().mean(0), (xd * xd).mean(0)
    # |d var| <= K_STATS u (E[x^2] + 2 |mean| E|x|): relative to var this is ~ 3 mean^2 / var, the cancellation factor
    dvar = ex2 + 2 * mean.abs() * ex1
    assert float((var - var2).abs()[[0, 2, 4]].max()) < 1e-9 * float(ex2.max())
    vpe = (var.clamp_min(eps64) if clamp else var + eps64)
    r_scale = K_STATS * 0.5 * rstd * dvar / vpe + rstd          # second term: the fp32 rounding of the result
    r_shift = K_STATS * (ex1 * rstd + mean.abs() * 0.5 * rstd * dvar / vpe) + (mean * rstd).abs()
    rat = check_close(name + ": nscale", nscale, rstd, r_scale, 1.0)
    rat = max(rat, check_close(name + ": nshift", nshift, -mean * rstd, r_shift, 1.0))
    check_close(name + ": mean_out", mean32, mean, K_STATS * ex1 + mean.abs(), 1.0)
    check_close(name + ": var_out", var32, var, K_STATS * dvar + var, 1.0)
    c2 = float(dvar[2] / var[2])
    print("%s: large-offset channel (|mean| = %.0f std): var bound carries (E x^2 + 2|mean| E|x|) / var = %.3g"
          % (name, float(mean[2] / var[2].sqrt()), c2))
    assert c2 > 1e4
    assert float(var32[1]) == 0.0, float(var32[1])
    if clamp:
        # var < eps: rstd = 1 / sqrt(eps) exactly as fp64 rounds it
        same_bits(name + ": nscale where var < eps", nscale[[1, 3]].cpu(),
                  (1.0 / torch.tensor([eps64, eps64], dtype=torch.float64).sqrt()).float())
    # running statistics: the unbiased estimator with count * unbiased_mult samples, updated in the reference's fp32 order
    cu = n * mult
    unb = var * cu / (cu - 1)
    check_close(name + ": unbiased var (momentum 1)", rv1, unb, K_STATS * dvar * cu / (cu - 1) + unb, 1.0)
    same_bits(name + ": running mean (momentum 1) = mean_out", rm1, mean32)
    same_bits(name + ": running mean", rm, _eager_running(rm0, rm1.cpu(), momentum))
    same_bits(name + ": running var", rv, _eager_running(rv0, rv1.cpu(), momentum))
    print("CASE bn_finalize %s max ratio %.3g (k 1, bound carries K_STATS)" % (name, rat))


@pytest.mark.gpu
def test_bn_finalize_constant_channel_var_rounds_negative():
    """Sums of a constant channel whose Sigma x^2 came out one fp64 ulp low (as rounding can leave it): E[x^2] - mean^2 is
    negative with or without a fused product, and var clamps to exactly 0."""
    ops = _ops()
    n = 3000.0
    S = 0.1 * n
    m = S / n
    Q = m * m * n
    while not (Q / n - m * m < 0 and math.fsum([Q / n, -m * m]) < 0):
        Q = math.nextafter(Q, 0.0)
    sums = torch.tensor([S, Q, n], dtype=torch.float64, device=dev)
    rv = torch.ones(1, device=dev)
    _, nshift, mean32, var32 = ops.bn_finalize(sums, n, running_mean=torch.zeros(1, device=dev), running_var=rv,
                                               want_stats=True)
    assert float(var32) == 0.0
    same_bits("constant channel: running var", rv, _eager_running(torch.ones(1), torch.zeros(1), 0.1))


@pytest.mark.gpu
def test_bn_from_running():
    ops = _ops()
    g = _gen("from_running")
    C_ = 300
    rm = torch.randn(C_, generator=g) * 10
    rv = torch.rand(C_, generator=g) * 4
    rv[:5] = torch.tensor([0.0, 1e-7, 1e-5, 1e6, 3e-38])
    eps = 1e-5
    nscale, nshift = ops.bn_from_running(rm.to(dev), rv.to(dev), eps)
    # fp32: rstd = 1 / sqrtf(fl(rv + eps)), two correctly rounded operations
    base = (rv + torch.tensor(eps, dtype=torch.float32)).double()
    ref = 1.0 / base.sqrt()
    check_close("bn_from_running: nscale", nscale, ref, ref, 6.0)     # sqrtf and the divide: measured 1.43
    same_bits("bn_from_running: nshift = -rm * nscale", nshift, -rm * nscale.cpu())


# ============================================================================================== spectral norm
SN_LAYERS = [(3, 576), (64, 27), (64, 1152), (1024, 9216), (37, 1152), (1024, 27), (3, 9216)]


def _sn_convs(g):
    convs = []
    for O, K in SN_LAYERS:
        w = torch.randn(O, K, generator=g) / math.sqrt(K)
        u = F.normalize(torch.randn(O, generator=g), dim=0, eps=1e-12)
        v = F.normalize(torch.randn(K, generator=g), dim=0, eps=1e-12)
        convs.append(types.SimpleNamespace(weight_orig=w.reshape(O, K, 1, 1).to(dev), weight_u=u.to(dev), weight_v=v.to(dev)))
    return convs


def _sn_train_ref(w, u):
    """torch SpectralNorm.compute_weight, one power iteration, eps 1e-12 (architecture.py:38-42), in float64, with the R_abs
    of every intermediate."""
    W, u = w.double(), u.double()
    t = W.t() @ u
    nt = t.norm()
    v = t / max(nt, 1e-12)
    s = W @ v
    ns = s.norm()
    u_new = s / max(ns, 1e-12)
    sigma = u_new @ s
    Wa = W.abs()
    r_t = Wa.t() @ u.abs()
    r_v = r_t / nt + v.abs() * r_t.norm() / nt
    r_s = Wa @ (r_v + v.abs())
    r_u = r_s / ns + u_new.abs() * r_s.norm() / ns
    inv = 1.0 / sigma
    r_inv = inv * (r_s.norm() / ns + r_t.norm() / nt) + inv
    return dict(v=(v, r_v), u=(u_new, r_u), inv=(inv, r_inv))


@pytest.mark.gpu
def test_spectral_norm_batched():
    from michigan_b200.networks.prep import SpectralNormBatch
    g = _gen("sn")
    convs = _sn_convs(g)
    u0 = [c.weight_u.clone() for c in convs]
    v0 = [c.weight_v.clone() for c in convs]
    snb = SpectralNormBatch(convs)
    inv_t = snb.run(training=True).clone()
    torch.cuda.synchronize()
    assert not bool(snb.t_ws.any()), "the W^T u workspace must be left zeroed for the next call"
    worst = 0.0
    for i, (c, (O, K)) in enumerate(zip(convs, SN_LAYERS)):
        ref = _sn_train_ref(c.weight_orig.reshape(O, K).cpu(), u0[i].cpu())
        k = C_DOT * math.sqrt(O + K) + K_EPI
        nm = "sn O%d K%d" % (O, K)
        worst = max(worst, check_close(nm + ": v", c.weight_v, *ref["v"], k) / math.sqrt(O + K))
        worst = max(worst, check_close(nm + ": u", c.weight_u, *ref["u"], k) / math.sqrt(O + K))
        worst = max(worst, check_close(nm + ": inv_sigma", inv_t[i:i + 1], ref["inv"][0].reshape(1), ref["inv"][1].reshape(1), k)
                    / math.sqrt(O + K))
    # a second run from the same u, v gives the same bits (no split-K atomics)
    u1 = [c.weight_u.clone() for c in convs]
    v1 = [c.weight_v.clone() for c in convs]
    for c, a, b in zip(convs, u0, v0):
        c.weight_u.copy_(a)
        c.weight_v.copy_(b)
    inv_t2 = snb.run(training=True).clone()
    torch.cuda.synchronize()
    same_bits("sn: inv_sigma, second run", inv_t2, inv_t)
    for c, a, b in zip(convs, u1, v1):
        same_bits("sn: u, second run", c.weight_u, a)
        same_bits("sn: v, second run", c.weight_v, b)
    # eval mode: sigma = u . (W v) from the stored vectors, u and v untouched
    inv_e = snb.run(training=False).clone()
    torch.cuda.synchronize()
    for i, (c, (O, K)) in enumerate(zip(convs, SN_LAYERS)):
        same_bits("sn eval: u untouched", c.weight_u, u1[i])
        W, u, v = d64(c.weight_orig.reshape(O, K)), d64(c.weight_u), d64(c.weight_v)
        sigma = u @ (W @ v)
        r_sigma = u.abs() @ (W.abs() @ v.abs())
        inv = 1.0 / sigma
        k = C_DOT * math.sqrt(O + K) + K_EPI
        worst = max(worst, check_close("sn eval O%d K%d: inv_sigma" % (O, K), inv_e[i:i + 1], inv.reshape(1),
                                       (inv * inv * r_sigma + inv.abs()).reshape(1), k) / math.sqrt(O + K))
    assert not bool(snb.t_ws.any())
    print("CASE spectral_norm max ratio / sqrt(O + K) %.3g (C_DOT %g)" % (worst, C_DOT))


# ============================================================================================== thin convs
def thin_case(name, kernel, CinP, I, Cout, k, s, p, H, W, N=2, reflect=False, act=1, knobs=None, pscale=False, pmul=False,
              round_out=False, out16=None, want_f32=True, R=0):
    return dict(name=name, kernel=kernel, CinP=CinP, I=I, Cout=Cout, k=k, s=s, p=p, H=H, W=W, N=N, reflect=reflect, act=act,
                knobs=knobs or {}, pscale=pscale, pmul=pmul, round_out=round_out, out16=out16, want_f32=want_f32, R=R)


TG = "thin_gemm_kernel<%d,%d>"
TC = "thin_conv_kernel<%d,%d>"
THIN_CASES = [
    # ---- production geometries through the route that runs them (MG_THIN_GEMM = 1)
    thin_case("disc_model0_k4s2p2_lrelu", TG % (8, 4), 8, 7, 64, 4, 2, 2, 37, 29, act=2),
    thin_case("disc_model0_f16_out16", TG % (8, 4), 8, 7, 64, 4, 2, 2, 18, 22, act=2, out16=("f16", False), want_f32=False),
    thin_case("disc_model0_round", TG % (8, 4), 8, 7, 64, 4, 2, 2, 33, 35, act=2, round_out=True),
    thin_case("bgenc_conv1_k7_reflect3_relu", TG % (4, 4), 4, 3, 64, 7, 1, 3, 21, 35, reflect=True),
    thin_case("inpaint_k7_reflect3", TG % (4, 4), 4, 4, 64, 7, 1, 3, 17, 19, reflect=True, act=0),
    thin_case("imgenc_layer1_pscale_pmul", TC % (4, 4), 4, 3, 128, 3, 2, 1, 33, 31, act=0, pscale=True, pmul=True),
    thin_case("imgenc_layer1_bf16_split", TC % (4, 4), 4, 3, 128, 3, 2, 1, 16, 16, act=0, pscale=True, pmul=True,
              out16=("bf16", True)),
    thin_case("mlp_shared_seg_resize2", TC % (4, 4), 4, 4, 128, 3, 1, 1, 13, 9, R=2),
    thin_case("mlp_shared_round_f16_split", TC % (4, 4), 4, 4, 128, 3, 1, 1, 12, 20, round_out=True, out16=("f16", True)),
    thin_case("cout32_k3s1", TC % (4, 2), 4, 4, 32, 3, 1, 1, 9, 17, act=2),
    # ---- the other routes, held to the same bound at Cout 64 and 128
    thin_case("route0_cout64_k4s2_cin8", TC % (8, 2), 8, 7, 64, 4, 2, 2, 19, 17, act=2, knobs={"MG_THIN_GEMM": 0}),
    thin_case("route0_cout64_k7_reflect", TC % (4, 2), 4, 3, 64, 7, 1, 3, 11, 23, reflect=True, knobs={"MG_THIN_GEMM": 0}),
    thin_case("route2_cout128_cin4_pscale", TG % (4, 8), 4, 3, 128, 3, 2, 1, 33, 31, act=0, pscale=True, pmul=True,
              knobs={"MG_THIN_GEMM": 2}),
    thin_case("route2_cout128_cin8_round", TG % (8, 8), 8, 8, 128, 3, 1, 1, 10, 18, round_out=True, knobs={"MG_THIN_GEMM": 2}),
    thin_case("route2_cout128_seg_resize4", TG % (4, 8), 4, 4, 128, 3, 1, 1, 7, 5, R=4, knobs={"MG_THIN_GEMM": 2}),
    thin_case("route2_cout64_cin8_bf16", TG % (8, 4), 8, 8, 64, 3, 1, 1, 9, 9, out16=("bf16", True), knobs={"MG_THIN_GEMM": 2}),
    # ---- ragged and tiny maps
    thin_case("gemm_1x1_map", TG % (4, 4), 4, 4, 64, 3, 1, 1, 1, 1, N=3),
    thin_case("gemm_2x2_k4s2p2", TG % (8, 4), 8, 7, 64, 4, 2, 2, 2, 2, N=3, act=2),
    thin_case("conv_1x1_map", TC % (4, 4), 4, 4, 128, 3, 1, 1, 1, 1, N=3),
    thin_case("conv_odd_s2_2x3", TC % (4, 4), 4, 3, 128, 3, 2, 1, 3, 5, pscale=True),
    thin_case("gemm_reflect_2x2_k3", TG % (4, 4), 4, 3, 64, 3, 1, 1, 2, 2, reflect=True),
    thin_case("route0_reflect_k7_8x9", TC % (4, 2), 4, 3, 64, 7, 1, 3, 8, 9, reflect=True, knobs={"MG_THIN_GEMM": 0}),
]


def _thin_inputs(c):
    ops = _ops()
    g = _gen(c["name"])
    N, H, W, CinP, I, Cout, k = c["N"], c["H"], c["W"], c["CinP"], c["I"], c["Cout"], c["k"]
    R = c["R"] or 1
    x = torch.zeros(N, H * R, W * R, CinP)
    x[..., :I] = torch.randn(N, H * R, W * R, I, generator=g)
    w = torch.randn(Cout, I, k, k, generator=g) / math.sqrt(k * k * I)
    b = 0.3 * torch.randn(Cout, generator=g)
    Hp = H + 2 * c["p"]
    OH, OW = (Hp - k) // c["s"] + 1, (W + 2 * c["p"] - k) // c["s"] + 1
    ps = torch.rand(N, OH, OW, generator=g) * 3 + 0.5 if c["pscale"] else None
    pm = None
    if c["pmul"]:
        pm = (torch.rand(N, OH, OW, generator=g) > 0.3).float()
        pm[:, 0, :] = 0.0
    wt = ops.pack_weight_thin(w.to(dev), CinP)
    exp_wt = torch.zeros(k * k, CinP, Cout)
    exp_wt[:, :I] = w.permute(2, 3, 1, 0).reshape(k * k, I, Cout)
    same_bits(c["name"] + ": packed weights", wt, exp_wt)
    return dict(x=x, w=w, b=b, ps=ps, pm=pm, wt=wt, OH=OH, OW=OW)


def _thin_run(c, d, round_out=None, want_f32=None):
    ops = _ops()
    cu = lambda t: None if t is None else t.to(dev)
    o16 = None if c["out16"] is None else (FMT[c["out16"][0]], c["out16"][1])
    r = ops.conv_thin(d["x"].to(dev), d["wt"], d["b"].to(dev), c["Cout"], c["k"], c["k"], c["s"], c["p"],
                      pad_mode=int(c["reflect"]), seg_resize=c["R"], act=c["act"],
                      round_out=c["round_out"] if round_out is None else round_out, pscale=cu(d["ps"]), pmul=cu(d["pm"]),
                      out_hw=(c["H"], c["W"]) if c["R"] else None, out16=o16,
                      want_f32=c["want_f32"] if want_f32 is None else want_f32)
    torch.cuda.synchronize()
    out, hi, lo = r if isinstance(r, tuple) else (r, None, None)
    return {k_: v_.cpu() for k_, v_ in dict(out=out, hi=hi, lo=lo).items() if v_ is not None}


def _thin_ref(c, d):
    x = d64(d["x"])
    if c["R"]:
        x = x[:, ::c["R"], ::c["R"]]
    p = c["p"]
    xn = nchw(x)
    xp = F.pad(xn, (p, p, p, p), mode="reflect") if c["reflect"] else F.pad(xn, (p, p, p, p))
    w = torch.zeros(c["Cout"], c["CinP"], c["k"], c["k"], dtype=torch.float64)
    w[:, :c["I"]] = d64(d["w"])
    y, ra = nhwc(F.conv2d(xp, w, stride=c["s"])), nhwc(F.conv2d(xp.abs(), w.abs(), stride=c["s"]))
    b = d64(d["b"])
    if d["ps"] is not None:
        ps = d64(d["ps"])[..., None]
        y, ra = y * ps, ra * ps.abs()
    y, ra = y + b, ra + b.abs()
    if c["act"] == 1:
        y = y.clamp_min(0)
    elif c["act"] == 2:
        y = torch.where(y > 0, y, float(torch.tensor(0.2, dtype=torch.float32)) * y)
    if d["pm"] is not None:
        pm = d64(d["pm"])[..., None]
        y, ra = y * pm, ra * pm.abs()
    return y, ra


@pytest.mark.gpu
@pytest.mark.parametrize("c", [pytest.param(c, id=c["name"]) for c in THIN_CASES])
def test_conv_thin(c):
    d = _thin_inputs(c)
    r1, names = _with_knobs(c["knobs"], lambda: _launched(lambda: _thin_run(c, d)))
    thin = {n for n in names if "thin_" in n}
    assert any(c["kernel"] in n.replace(" ", "") for n in thin), (c["name"], c["kernel"], sorted(thin))
    assert len(thin) == 1, sorted(thin)
    r2 = _with_knobs(c["knobs"], lambda: _thin_run(c, d))
    for key in r1:
        same_bits("%s: %s, second run" % (c["name"], key), r1[key], r2[key])
    ref, rabs = _thin_ref(c, d)
    K = c["k"] * c["k"] * c["CinP"]
    k = C_DOT * math.sqrt(K) + K_EPI
    # the fp32 output: directly, or (16-bit-only calls) from the same call with want_f32
    out = r1["out"] if "out" in r1 else _with_knobs(c["knobs"], lambda: _thin_run(c, d, want_f32=True))["out"]
    if c["round_out"]:
        assert not bool((out.view(torch.int32) & 0x1FFF).any()), c["name"]
        plain = _with_knobs(c["knobs"], lambda: _thin_run(c, d, round_out=False))["out"]
        same_bits(c["name"] + ": round_out = rna_tf32 of the unrounded output", out, rna_tf32(plain))
        ratio = check_rounded(c["name"], out, ref, rabs, 11, k)
    else:
        ratio = check_close(c["name"], out, ref, rabs, k)
    if c["out16"]:
        hi, lo = split16(out, c["out16"][0])
        same_bits(c["name"] + ": hi = cvt(y32)", r1["hi"], hi)
        if c["out16"][1]:
            same_bits(c["name"] + ": lo = cvt(y32 - hi)", r1["lo"], lo)
        else:
            assert "lo" not in r1
    print("CASE %-32s %-24s K=%-4d max ratio %.3g / sqrt(K) %.3g  k %.1f" % (c["name"], c["kernel"], K, ratio,
                                                                            ratio / math.sqrt(K), k))


# ============================================================================================== partial-conv masks
def _partial_ref(mask, k, s, p):
    """partialconv2d.py:65-72 in fp32: um = conv2d(mask, ones), ratio = slide_winsize / (um + 1e-8) (a Python float over a
    tensor: reciprocal, then the product), update = clamp(um, 0, 1), ratio = ratio * update.  The masks here have window
    sums that are exact in fp32, so um is the same in any summation order (a sum of shifted slices)."""
    N, H, W = mask.shape
    mp = F.pad(mask, (p, p, p, p))
    OH, OW = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    um = torch.zeros(N, 1, OH, OW)
    for i in range(k):
        for j in range(k):
            um[:, 0] += mp[:, i:i + s * (OH - 1) + 1:s, j:j + s * (OW - 1) + 1:s]
    ratio = float(k * k) / (um + 1e-8)
    upd = torch.clamp(um, 0, 1)
    return torch.mul(ratio, upd)[:, 0], upd[:, 0]


def _holes(g, N, H, W):
    m = (torch.rand(N, H, W, generator=g) > 0.35).float()
    m[:, 0, :] = 0.0                  # holes along the borders
    m[:, :, -1] = 0.0
    m[:, 3:9, 2:7] = 0.0
    m[0, -4:, :4] = 0.0
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("geo", [(3, 2, 1, 33, 30), (3, 1, 1, 17, 18), (7, 1, 3, 20, 21), (4, 2, 1, 15, 16), (5, 3, 2, 23, 19)],
                         ids=lambda g: "k%d_s%d_p%d_%dx%d" % g)
def test_partial_mask(geo):
    k, s, p, H, W = geo
    g = _gen("pm%s" % (geo,))
    m = _holes(g, 3, H, W)
    # a soft mask of multiples of 2^-30: window sums near 1e-8, where um + 1e-8 is not max(um, 1e-8)
    m[2] = torch.randint(0, 256, (H, W), generator=g).float() * 2.0 ** -30
    ratio, upd = _ops().partial_mask(m.to(dev), k, s, p)
    rr, ru = _partial_ref(m, k, s, p)
    same_bits("partial_mask %s: update" % (geo,), upd, ru)
    same_bits("partial_mask %s: ratio" % (geo,), ratio, rr)


@pytest.mark.gpu
def test_partial_mask_image_encoder_chain():
    """The five partial convs of ImageEncoder3 (k3 s2 p1 each, encoder.py), each layer's update mask feeding the next."""
    g = _gen("pm_chain")
    m = _holes(g, 2, 128, 96)
    mg = m.to(dev)
    for i in range(5):
        ratio, upd = _ops().partial_mask(mg, 3, 2, 1)
        rr, ru = _partial_ref(m, 3, 2, 1)
        same_bits("layer%d: update" % (i + 1), upd, ru)
        same_bits("layer%d: ratio" % (i + 1), ratio, rr)
        m, mg = ru, upd


# ============================================================================================== mask dilation
def _maxpool_ref(m, k, invert):
    r = F.max_pool2d(m[:, None], k, 1, k // 2)[:, 0]
    return 1 - r if invert else r


def _random_expand_ks(size):
    th = int(size * 0.05)
    th = th if th % 2 == 1 else th + 1
    return sorted({max(th - 4, 1), max(th - 2, 1), th, th + 2, th + 4})


MAXPOOL_CASES = [(1, 9, 11), (3, 9, 11), (7, 5, 6), (9, 5, 3), (11, 40, 33)] + [(k, 128, 128) for k in _random_expand_ks(128)] + \
    [(k, 40, 37) for k in _random_expand_ks(512)]


@pytest.mark.gpu
@pytest.mark.parametrize("geo", MAXPOOL_CASES, ids=lambda g: "k%d_%dx%d" % g)
def test_maxpool_mask(geo):
    k, H, W = geo
    g = _gen("mp%s" % (geo,))
    m = (torch.rand(2, H, W, generator=g) > 0.8).float()
    m[1] = torch.rand(H, W, generator=g)              # non-binary values: the max itself is compared
    for inv in (False, True):
        got = _ops().maxpool_mask(m.to(dev), k, invert=inv)
        same_bits("maxpool_mask k%d invert=%d" % (k, inv), got, _maxpool_ref(m, k, inv))


@pytest.mark.gpu
def test_maxpool_mask_rejects_even_k():
    lib = _lib()
    with pytest.raises(lib.MichiganNativeError, match=r"status -2"):
        _ops().maxpool_mask(torch.zeros(1, 8, 8, device=dev), 4)


@pytest.mark.gpu
def test_back_mask_add_feat_zeros():
    """BackgroundEncode2.back_mask at inference with --add_feat_zeros: the dilation runs on the unpadded crop only
    (reference encoder.py:301-314)."""
    from michigan_b200.networks.encoder import BackgroundEncode2
    crop, th, k = 64, 8, 9
    g = _gen("afz")
    S = crop + th
    mask = torch.zeros(2, 2, S, S)
    mask[:, 1] = (torch.rand(2, S, S, generator=g) > 0.85).float()
    mask[:, 0] = 1 - mask[:, 1]
    opt = types.SimpleNamespace(isTrain=False, expand_mask_be=True, expand_th=k, add_feat_zeros=True, add_th=th,
                                crop_size=crop)
    got = BackgroundEncode2.back_mask(types.SimpleNamespace(opt=opt), mask.to(dev))
    hair = mask[:, 1:2]
    o = int(th / 2)
    e = hair * 0
    e[:, :, o:o + crop, o:o + crop] = F.max_pool2d(hair[:, :, o:o + crop, o:o + crop], kernel_size=k, stride=1, padding=k // 2)
    same_bits("back_mask add_feat_zeros", got, (1 - e)[:, 0])


# ============================================================================================== input preparation
@pytest.mark.gpu
def test_prep_seg_orientation_one_channel():
    """generator.py:131-133: th = orient / 255.0 * pi (fp32 divide, then the product), [sin 2th, cos 2th] * hair.  sinf /
    cosf of the kernel's fp32 2th within 4 ulp of fp64 (CUDA's sinf / cosf: <= 2 ulp), the product by the 0/1 mask exact."""
    g = _gen("prep_seg1")
    N, H, W = 2, 33, 47
    tag = torch.zeros(N, 2, H, W)
    tag[:, 1] = (torch.rand(N, H, W, generator=g) > 0.5).float()
    tag[:, 0] = 1 - tag[:, 1]
    orient = torch.randint(0, 256, (N, 1, H, W), generator=g).float()
    orient[1] = torch.rand(H, W, generator=g) * 255
    seg4 = _ops().prep_seg(tag.to(dev), orient.to(dev)).cpu()
    same_bits("prep_seg: tag channels", seg4[..., :2], nhwc(tag))
    th2 = 2 * d64(orient / 255.0 * math.pi)
    hair = d64(tag[:, 1:2])
    for i, fn in ((2, torch.sin), (3, torch.cos)):
        ref = nhwc(fn(th2) * hair)[..., 0]
        got = d64(seg4[..., i])
        _, e = torch.frexp(ref)
        ulp = torch.ldexp(torch.ones_like(ref), (e - 24).to(torch.int64))
        err = (got - ref).abs()
        ratio = float((err / ulp).max())
        print("prep_seg %s: max |got - ref| / ulp = %.3g (k = 4)" % (fn.__name__, ratio))   # measured 1.23
        assert bool((err <= 4 * ulp + 2.0 ** -149).all()), ratio


@pytest.mark.gpu
def test_prep_elementwise_bit_exact():
    ops = _ops()
    g = _gen("prep")
    N, H, W = 2, 19, 27
    tag = torch.randn(N, 2, H, W, generator=g)
    orient2 = torch.randn(N, 2, H, W, generator=g)
    seg4 = ops.prep_seg(tag.to(dev), orient2.to(dev))
    same_bits("prep_seg (2 orientation channels)", seg4, nhwc(torch.cat([tag, orient2], 1)))
    img = torch.randn(N, 3, H, W, generator=g)
    d8 = ops.prep_dinput(seg4, img.to(dev))
    same_bits("prep_dinput", d8, nhwc(torch.cat([tag, orient2, img, torch.zeros(N, 1, H, W)], 1)))
    # nchw_to_nhwc with channel padding and a per-pixel multiplier; nhwc_to_nchw dropping the padding
    x = torch.randn(N, 3, H, W, generator=g)
    pm = torch.rand(N, H, W, generator=g)
    pm[:, ::4] = 0.0
    got = ops.nchw_to_nhwc(x.to(dev), 4, pmul=pm.to(dev))
    same_bits("nchw_to_nhwc pmul cpad", got, nhwc(torch.cat([x * pm[:, None], torch.zeros(N, 1, H, W)], 1)))
    same_bits("nchw_to_nhwc", ops.nchw_to_nhwc(x.to(dev)), nhwc(x))
    y = torch.randn(N, H, W, 8, generator=g)
    same_bits("nhwc_to_nchw c=7 of 8", ops.nhwc_to_nchw(y.to(dev), 7), nchw(y)[:, :7])
    same_bits("nhwc_to_nchw", ops.nhwc_to_nchw(y.to(dev)), nchw(y))


@pytest.mark.gpu
def test_prep_bginput_eager_order():
    """encoder.py:321: image * back_mask + noise * (1 - back_mask), as eager fp32 ops: both products rounded, then the add.
    A non-binary mask makes the order visible (with a 0/1 mask every order gives the same bits)."""
    g = _gen("bginput")
    N, H, W = 2, 21, 30
    img = torch.randn(N, 3, H, W, generator=g)
    noise = torch.randn(N, 3, H, W, generator=g)
    back = torch.rand(N, H, W, generator=g)
    back[0] = (back[0] > 0.5).float()
    got = _ops().prep_bginput(img.to(dev), noise.to(dev), back.to(dev))
    bm = back[:, None]
    ref = img * bm + noise * (1 - bm)
    same_bits("prep_bginput", got, nhwc(torch.cat([ref, torch.zeros(N, 1, H, W)], 1)))


# ============================================================================================== softmax
def _softmax_rows_data(g, rows, cols):
    x = torch.randn(rows, cols, generator=g) * 3
    x[0] = torch.rand(cols, generator=g) * 80 - 40                 # scores over +-40: probabilities down to e^-80
    x[1] = 0.25                                                   # every score equal
    x[2, :] = torch.randn(cols, generator=g)
    x[2, ::3] = 5.0                                               # ties at the maximum
    x[3] = torch.randn(cols, generator=g) * 1e-3 + 1e4            # large offset: x - max carries the rounding of x
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("cols", [4, 12, 1000, 4096])
def test_softmax_rows(cols):
    ops = _ops()
    g = _gen("softmax%d" % cols)
    rows = 300 if cols <= 1000 else 96
    x = _softmax_rows_data(g, rows, cols)
    xg = x.to(dev)
    xd = x.double()
    m = xd.max(1, keepdim=True).values
    e = torch.exp(xd - m)
    ref = e / e.sum(1, keepdim=True)
    # expf's relative error + the rounding of x - m (|x - m| u) + the row sum; 1 for the product
    rabs = ref * (1 + (xd - m).abs())
    k = K_SOFTMAX + C_DOT * math.sqrt(cols)
    _, out, _ = ops.softmax_rows(xg)
    torch.cuda.synchronize()
    out = out.cpu()
    assert not bool((out.view(torch.int32) & 0x1FFF).any())
    ratio = check_rounded("softmax cols %d: TF32" % cols, out, ref, rabs, 11, k)
    _, out2, _ = ops.softmax_rows(xg)
    same_bits("softmax: second run", out2, out)
    for fmt in ("f16", "bf16"):
        bits = 11 if fmt == "f16" else 8
        tiny16 = 2.0 ** -25 if fmt == "f16" else 0.0
        _, hi, lo = ops.softmax_rows(xg, FMT[fmt], split=True)
        _, hi1, lo1 = ops.softmax_rows(xg, FMT[fmt], split=False)
        torch.cuda.synchronize()
        hi, lo, hi1 = hi.cpu(), lo.cpu(), hi1.cpu()
        assert lo1 is None
        same_bits("softmax %s: hi without lo" % fmt, hi1, hi)
        for nm, v, rel, t16 in (("hi", d64(hi), 2.0 ** -bits, tiny16), ("hi + lo", d64(hi) + d64(lo), 2.0 ** -(2 * bits),
                                                                        2 * tiny16)):
            err = (v - ref).abs()
            bound = k * U * rabs + rel * (ref + k * U * rabs) + t16 + TINY
            r = float(((err - rel * ref - t16).clamp_min(0) / (U * rabs + TINY)).max())
            print("softmax cols %d %s %s: max (|got - ref| - format rounding) / (u R_abs) = %.3g (k = %g)" % (cols, fmt, nm, r, k))
            assert not bool((err > bound).any()), (fmt, nm, int((err > bound).sum()))
    # rows of equal scores: exactly 1/cols where that is representable
    if cols & (cols - 1) == 0:
        assert bool((out[1] == 1.0 / cols).all())
    print("CASE softmax cols=%d max ratio %.3g (k %.1f)" % (cols, ratio, k))


# ============================================================================================== edge weight
def _edge_weight_ref(label, h, w, wide_edge):
    """loss.py:60-78 in fp32: nearest resize to the logits, max-pool edges, resize back, edges * wide_edge + (1 - edges)."""
    t = F.interpolate(label[:, None], size=(h, w), mode="nearest")
    k = max(1, int(h * 0.06))
    p = int(k / 2)
    out = F.max_pool2d(t, kernel_size=k, stride=1, padding=p)
    out2 = 1 - F.max_pool2d(1 - t, kernel_size=k, stride=1, padding=p)
    edges = F.interpolate(out - out2, size=(h, w), mode="nearest")
    return (edges * wide_edge + (1 - edges))[:, 0], k


@pytest.mark.gpu
@pytest.mark.parametrize("geo", [(128, 128, 66, 66), (128, 96, 35, 27), (512, 512, 34, 34), (256, 256, 18, 18),
                                 (128, 128, 10, 10), (512, 384, 50, 38)], ids=lambda g: "%dx%d_to_%dx%d" % g)
def test_edge_weight(geo):
    H, W, h, w = geo
    g = _gen("edge%s" % (geo,))
    lib = _lib()
    label = torch.zeros(2, H, W)
    label[:, H // 4:3 * H // 4, W // 5:W // 2] = 1.0
    label[1] = (torch.rand(H, W, generator=g) > 0.9).float()
    for wide_edge in (2.0, 3.7):
        out = torch.empty(2, h, w, device=dev)
        lg = label.to(dev)
        lib.check(lib.load().mg_edge_weight(lg.data_ptr(), out.data_ptr(), 2, H, W, h, w, wide_edge, _ops()._stream()),
                  "mg_edge_weight")
        ref, k = _edge_weight_ref(label, h, w, float(torch.tensor(wide_edge, dtype=torch.float32)))
        same_bits("edge_weight %s k=%d wide_edge %g" % (geo, k, wide_edge), out, ref)
