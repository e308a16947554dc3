"""Launch ONE kernel of the hot path a few times at its benchmark shape (N = 8, 512x512) - the target of `ncu --set full`
or of a profiler.  argv[1]: spade | group | wgrad16 | wgrad32 | seg | stats | spade_bwd | dconv"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from michigan_b200 import ops
which = sys.argv[1]
N, S, dev = 8, 512, "cuda"
g = torch.Generator(device="cuda").manual_seed(0)
r = lambda *s: torch.randn(*s, device=dev, generator=g)
if which == "spade":          # fused SPADE gamma|beta GEMM, up_3.norm_0 shape, fp16 operands -> bf16 hi/lo
    a16, wg, xs, v = r(N, S, S, 128).half(), r(128, 128, 3, 3) / 34, r(N, S // 2, S // 2, 128), torch.ones(128, device=dev)
    wp = ops.pack_weight_gb16(wg, wg)
    f = lambda: ops.conv_igemm(a16, wp, 128, 3, 3, 1, 1, act=2, a_fmt=ops.F16, spade=(xs, 1, v, v, v, v), out16=(ops.BF16, True), want_f32=False)
elif which == "group":        # up_3.conv_0: 3x3 128 -> 64, bf16 hi+lo split, M-tile-group kernel
    x, w, b = r(N, S, S, 128), r(64, 128, 3, 3) / 34, torch.zeros(64, device=dev)
    hi = x.bfloat16(); lo = (x - hi.float()).bfloat16(); wp = ops.pack_weight16(w, None, ops.BF16, split=True)
    f = lambda: ops.conv_igemm(hi, wp, 64, 3, 3, 1, 1, bias=b, a_fmt=ops.BF16, x_lo=lo)
elif which in ("wgrad16", "wgrad32"):   # gamma|beta weight gradient of up_3
    dy, x = r(N, S, S, 256), r(N, S, S, 128)
    if which == "wgrad16":
        dy16, x16 = dy.bfloat16(), x.bfloat16()
        f = lambda: ops.conv_wgrad16(dy16, x16, 3, 3, 1, 1)
    else:
        f = lambda: ops.conv_wgrad(dy, x, 3, 3, 1, 1)
elif which == "seg":          # SPADE mlp_shared 4 -> 128 at 512x512, fp16 output
    seg, w, b = r(N, S, S, 4), r(128, 4, 3, 3) / 6, torch.zeros(128, device=dev)
    wp = ops.pack_mlp_shared(w)
    o16 = (ops.BF16, True) if os.environ.get("MG_SEG_SPLIT") else (ops.F16, False)
    f = lambda: ops.mlp_shared(seg, wp, b, seg_resize=1, out_hw=(S, S), out16=o16, want_f32=False)
elif which == "stats":        # BN statistics of [8,512,512,64]
    x = r(N, S, S, 64)
    f = lambda: ops.bn_sums(x)
elif which == "spade_bwd":    # SPADE elementwise backward at the up_3.norm_1 shape (C = 64), bf16 dgamma|dbeta
    dh, h, g1, xs, v = r(N, S, S, 64), r(N, S, S, 64), r(N, S, S, 64), r(N, S, S, 64), torch.ones(64, device=dev)
    f = lambda: ops.spade_bwd(dh, h, g1, xs, 0, v, v, 2, dgb_fmt=ops.BF16)
elif which == "dconv":        # discriminator model3: 256 -> 512 k4 s1 p2 at 65x65, batch 16, fp16 operands
    x, w = r(16, 65, 65, 256).half(), r(512, 256, 4, 4) / 64
    wp = ops.pack_weight16(w, None, ops.F16, split=False)
    f = lambda: ops.conv_igemm(x, wp, 512, 4, 4, 1, 2, a_fmt=ops.F16)
else:
    raise SystemExit("unknown kernel " + which)
for _ in range(4):
    f()
torch.cuda.synchronize()
if os.environ.get("MG_TIME"):          # not under a profiler: average of 20 launches, CUDA events
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        f()
    e1.record()
    torch.cuda.synchronize()
    print("%s: %.4f ms/launch" % (which, e0.elapsed_time(e1) / 20))
print("done", which)
