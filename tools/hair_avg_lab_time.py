"""Cost of the unpaired stage's colour term: HairAvgLabLoss forward + backward at batch 8, 512x512, on the kernels
(mg_hair_avg_lab_fwd / _bwd alone and through the autograd module), with the Lab colour loss of the paired stage for
context.

    python tools/hair_avg_lab_time.py OUT_DIR [--batch 8] [--reps 50] [--rounds 3]

Synthetic inputs: images uniform in (-1, 1), the tag's hair a box of ~23 % of the pixels, the reference's hair a shifted box.
Writes OUT_DIR/hair_avg_lab_time.json and prints one line per measurement (median of `reps` CUDA-event timings, each round
alternating the variants), headed by the GPU's name, power limit and maximum SM clock (read-only nvidia-smi query).
Algorithmic bytes: forward = both images and both masks read (32 B per pixel), backward = fake and its mask read plus d fake
written (28 B per pixel); pixels outside the masks are not loaded by the kernels, so the rate is an upper bound's share.
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)
import torch

from vgg_lab_time import gpu_info, timed

SIZE = 512
HBM_TBS = 3.35


def inputs(n, size, seed=0):
    g = torch.Generator().manual_seed(seed)
    fake = torch.rand(n, 3, size, size, generator=g) * 2 - 1
    real = torch.rand(n, 3, size, size, generator=g) * 2 - 1
    s = size / 512.0
    mf = torch.zeros(n, 1, size, size)
    mf[:, :, int(102 * s):int(307 * s), int(102 * s):int(410 * s)] = 1.0
    mr = torch.zeros(n, 1, size, size)
    mr[:, :, int(150 * s):int(380 * s), int(60 * s):int(330 * s)] = 1.0
    return [t.cuda() for t in (fake, real, mf, mr)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "hair_avg_lab_time.py needs a GPU"
    os.makedirs(a.out_dir, exist_ok=True)
    from michigan_b200 import ops
    from michigan_b200.networks import HairAvgLabLoss, LabColorLoss
    from michigan_b200.options import make_opt
    gpu = gpu_info()
    print("GPU:", gpu)
    n = a.batch
    fake, real, mf, mr = inputs(n, SIZE)
    crit, lab = HairAvgLabLoss(make_opt()), LabColorLoss(make_opt())
    sums = ops.hair_avg_lab_fwd(fake, real, mf, mr)
    g1 = torch.ones(1, device="cuda")

    def module():
        x = fake.detach().requires_grad_()
        crit(x, real, mf, mr).backward()

    def lab_module():
        x = fake.detach().requires_grad_()
        lab(x, real).backward()

    variants = {
        "hair_avg_lab_fwd kernels": lambda: ops.hair_avg_lab_fwd(fake, real, mf, mr),
        "hair_avg_lab_bwd kernel": lambda: ops.hair_avg_lab_bwd(fake, mf, sums, g1),
        "HairAvgLabLoss fwd+bwd": module,
        "LabColorLoss fwd+bwd": lab_module,
    }
    times = {k: [] for k in variants}
    for _ in range(a.rounds):
        for k, fn in variants.items():
            times[k].append(timed(fn, a.reps))
    px = n * SIZE * SIZE
    bytes_ = {"hair_avg_lab_fwd kernels": 32 * px, "hair_avg_lab_bwd kernel": 28 * px}
    hair = float(mf.mean()), float(mr.mean())
    res = {"gpu": gpu, "batch": n, "size": SIZE, "hair_fraction": hair, "ms": {}}
    print("batch %d, %dx%d, hair %.1f %% (tag) / %.1f %% (ref) of the pixels" % (n, SIZE, SIZE, 100 * hair[0], 100 * hair[1]))
    for k, ts in times.items():
        med = sorted(ts)[len(ts) // 2]
        res["ms"][k] = ts
        line = "%-28s %8.4f ms  (rounds: %s)" % (k, med, ", ".join("%.4f" % t for t in ts))
        if k in bytes_:
            line += "  %.0f GB/s algorithmic = %.1f %% of %.2f TB/s" % (bytes_[k] / med / 1e6, 100 * bytes_[k] / med / 1e9 / HBM_TBS,
                                                                        HBM_TBS)
        print(line)
    with open(os.path.join(a.out_dir, "hair_avg_lab_time.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
