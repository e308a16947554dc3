"""Where the epilogue of conv3x3_group_kernel spends its time: each benchmark-shape launch timed with the probe build's what-if
switches (MG_DBG) that skip parts of the register epilogue.

    python -m michigan_b200.build --probes
    MICHIGAN_B200_LIB=michigan_b200/lib/libmichigan_sm90_probes.so python tools/epilogue_split.py <out_dir> [--rounds R]

Shapes (N = 8, 512x512): the SPADE gamma|beta GEMM of up_3 (fp16 operands -> bf16 hi/lo, SPEC 1, BN 128; bench.py's
`roofline`), up_3.conv_0 (bf16 hi+lo merged, BN 64, bias -> fp32; `roofline_worst`) and up_3.conv_1 (bf16 hi+lo merged, BN 64,
bias + full-resolution residual + background blend -> fp32).  Probes (results are WRONG under 4, 8, 32, 64):
   0 unmodified   4 no epilogue   32 no 16-bit stores   64 no side loads   8 neither 16-bit stores nor side loads
The probes of one shape are interleaved round by round (median of the rounds, each round the mean of `launches` back-to-back
launches), and the card's name, power limit and SM clock are read in the same process.  Writes <out_dir>/epilogue_split.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from michigan_b200 import _lib, ops  # noqa: E402

PROBES = (0, 4, 32, 64, 8)
N, S = 8, 512


def shapes():
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    r = lambda *s: torch.randn(*s, device=dev, generator=g)
    out = {}
    a16, wg, xs, v = r(N, S, S, 128).half(), r(128, 128, 3, 3) / 34, r(N, S // 2, S // 2, 128), torch.ones(128, device=dev)
    wp = ops.pack_weight_gb16(wg, wg)
    out["spade_gb_up3"] = lambda: ops.conv_igemm(a16, wp, 128, 3, 3, 1, 1, act=2, a_fmt=ops.F16, spade=(xs, 1, v, v, v, v),
                                                 out16=(ops.BF16, True), want_f32=False)
    x, w0, b0 = r(N, S, S, 128), r(64, 128, 3, 3) / 34, torch.zeros(64, device=dev)
    hi0 = x.bfloat16(); lo0 = (x - hi0.float()).bfloat16(); wp0 = ops.pack_weight16(w0, None, ops.BF16, split=True)
    del x
    out["conv_0_up3"] = lambda: ops.conv_igemm(hi0, wp0, 64, 3, 3, 1, 1, bias=b0, a_fmt=ops.BF16, x_lo=lo0)
    h1 = r(N, S, S, 64); w1, b1 = r(64, 64, 3, 3) / 24, r(64)
    hi1 = h1.bfloat16(); lo1 = (h1 - hi1.float()).bfloat16(); wp1 = ops.pack_weight16(w1, None, ops.BF16, split=True)
    del h1
    res, bf = r(N, S, S, 64), r(N, S, S, 64)
    hair = (torch.rand(N, S, S, device=dev, generator=g) > 0.5).float()
    back = (torch.rand(N, S, S, device=dev, generator=g) > 0.5).float()
    out["conv_1_up3_res_blend"] = lambda: ops.conv_igemm(hi1, wp1, 64, 3, 3, 1, 1, bias=b1, a_fmt=ops.BF16, x_lo=lo1, res=res,
                                                         blend=(bf, hair, back, 1))
    return out


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        row = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [c.strip() for c in row.split(",")]))
    except Exception as e:  # the timings stand without it, but say so
        return {"name": torch.cuda.get_device_name(0), "error": str(e)}


def time_launches(f, launches):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=10)
    a = ap.parse_args()
    if "_probes" not in os.path.basename(_lib.LIB_PATH):
        raise SystemExit("MG_DBG switches exist only in the probe build: set MICHIGAN_B200_LIB to libmichigan_sm90_probes.so")
    os.makedirs(a.out_dir, exist_ok=True)
    res = {"gpu_before": gpu_info(), "lib": os.path.basename(_lib.LIB_PATH), "rounds": a.rounds, "launches": a.launches,
           "shapes": {}}
    for name, f in shapes().items():
        for d in PROBES:
            os.environ["MG_DBG"] = str(d)
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        times = {d: [] for d in PROBES}
        for _ in range(a.rounds):
            for d in PROBES:
                os.environ["MG_DBG"] = str(d)
                times[d].append(time_launches(f, a.launches))
        os.environ["MG_DBG"] = "0"
        med = {d: statistics.median(t) for d, t in times.items()}
        gap = med[0] - med[4]
        row = {"ms": {str(d): round(med[d], 4) for d in PROBES},
               "spread_ms": {str(d): round(max(t) - min(t), 4) for d, t in times.items()},
               "epilogue_ms": round(gap, 4),
               "stores16_ms": round(med[0] - med[32], 4),
               "side_loads_ms": round(med[0] - med[64], 4),
               "stores16_and_side_loads_ms": round(med[0] - med[8], 4),
               "rest_ms": round(med[8] - med[4], 4)}
        res["shapes"][name] = row
        print(name, json.dumps(row), flush=True)
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out_dir, "epilogue_split.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res["gpu_after"]))


if __name__ == "__main__":
    main()
