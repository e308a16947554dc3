"""Cost of --balance_Lab: LabColorLoss forward + backward at batch 8, 512x512, balanced (mg_loss_reduce op 11 each way) and
unbalanced (mg_lab_loss_fwd / _bwd), next to an eager torch restatement of the reference's balanced loss (xyz2lab of both
images, grid_sample of the weight table, the weighted L1; autograd backward).

    python tools/lab_balance_time.py OUT_DIR [--batch 8] [--reps 50] [--rounds 3]

Synthetic inputs: images uniform in (-1, 1), the tag's hair a box of ~23 % of the pixels, the seeded count table of the tests
(tests/oracle_balance_lab.count_table) written to OUT_DIR.  Prints one line per measurement (median of `reps` CUDA-event
timings, each round alternating the variants), headed by the GPU's name, power limit and maximum SM clock (read-only
nvidia-smi query), and writes OUT_DIR/lab_balance_time.json.  Algorithmic bytes of op 11: forward = both images and the mask
read (28 B per pixel), backward = the same plus d fake written (40 B per pixel); the 256 KB table stays in cache.
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
import numpy as np
import torch

from hair_avg_lab_time import HBM_TBS, SIZE, inputs
from vgg_lab_time import gpu_info, timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "lab_balance_time.py needs a GPU"
    os.makedirs(a.out_dir, exist_ok=True)
    import oracle_balance_lab as obl
    import oracle_vgg_lab as ovl
    from michigan_b200.networks import LabColorLoss
    from michigan_b200.options import make_opt
    gpu = gpu_info()
    print("GPU:", gpu)
    n = a.batch
    fake, real, mask, _ = inputs(n, SIZE)
    path = os.path.join(a.out_dir, "ab_count.npy")
    table = obl.count_table(obl.TABLE_SEED)
    np.save(path, table)
    balanced = LabColorLoss(make_opt(balance_Lab=True, weight_dir=path))
    plain = LabColorLoss(make_opt())
    w = obl.weight_map(table, 10.0).cuda()
    ovl._M = ovl._M.cuda()                  # the oracle's RGB -> XYZ matrix, on the device of the eager restatement

    def run(fn):
        def go():
            x = fake.detach().requires_grad_()
            fn(x).backward()
        return go

    variants = {
        "LabColorLoss balanced fwd+bwd": run(lambda x: balanced(x, real, mask)),
        "LabColorLoss unbalanced fwd+bwd": run(lambda x: plain(x, real, mask)),
        "eager torch balanced fwd+bwd": run(lambda x: obl.lab_color_loss_balanced(x, real, mask, w)),
    }
    times = {k: [] for k in variants}
    for _ in range(a.rounds):
        for k, fn in variants.items():
            times[k].append(timed(fn, a.reps))
    px = n * SIZE * SIZE
    res = {"gpu": gpu, "batch": n, "size": SIZE, "hair_fraction": float(mask.mean()), "ms": {},
           "op11_bytes": {"fwd": 28 * px, "bwd": 40 * px}}
    print("batch %d, %dx%d, hair %.1f %% of the pixels; op 11 moves %.0f MB forward, %.0f MB backward (%.1f us at %.2f TB/s)"
          % (n, SIZE, SIZE, 100 * float(mask.mean()), 28 * px / 1e6, 40 * px / 1e6, 68 * px / HBM_TBS / 1e6, HBM_TBS))
    for k, ts in times.items():
        med = sorted(ts)[len(ts) // 2]
        res["ms"][k] = ts
        print("%-34s %8.4f ms  (rounds: %s)" % (k, med, ", ".join("%.4f" % t for t in ts)))
    with open(os.path.join(a.out_dir, "lab_balance_time.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
