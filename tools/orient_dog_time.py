"""Cost of --orient_filter dog: L1OLoss forward + backward at batch 8, 512x512 with the DoG filter (response pass, op 12 each
way, the gather), with the Gabor filter (mg_orient_loss_fwd / _bwd), and an eager torch restatement of the reference's DoG loss
(tests/oracle_orient_dog.py: one 32-filter conv, the batch-maximum normalisation and both losses; autograd backward).

    python tools/orient_dog_time.py OUT_DIR [--batch 8] [--reps 30] [--rounds 3]

Synthetic inputs: images uniform in (-1, 1), the hair a box of ~23 % of the pixels, angle labels.  Prints one line per
measurement (median of `reps` CUDA-event timings, each round alternating the variants), headed by the GPU's name, power limit
and maximum SM clock (read-only nvidia-smi query), and writes OUT_DIR/orient_dog_time.json.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "orient_dog_time.py needs a GPU"
    os.makedirs(a.out_dir, exist_ok=True)
    import oracle_orient_dog as od
    from michigan_b200.networks.loss import L1OLoss, dog_bank
    from michigan_b200.options import make_opt
    from michigan_b200.synth import synthetic_batch
    gpu = gpu_info()
    print("GPU:", gpu)
    n = a.batch
    data = synthetic_batch(n, SIZE, 1)
    img = data["image_tag"].cuda()
    label = data["orient"].cuda()
    hair = data["label_tag"].cuda()
    sem = torch.cat([1 - hair, hair], dim=1)
    dog, gabor = L1OLoss(make_opt(orient_filter="dog")), L1OLoss(make_opt(orient_filter="gabor"))
    bank = dog_bank("cuda")

    def run(fn):
        def go():
            x = img.detach().requires_grad_()
            lo, lc = fn(x)
            (lo * 10.0 + lc * 100.0).backward()
        return go

    variants = {
        "L1OLoss dog fwd+bwd": run(lambda x: dog(x, label, sem)),
        "L1OLoss gabor fwd+bwd": run(lambda x: gabor(x, label, sem)),
        "eager torch dog fwd+bwd": run(lambda x: od.orient_loss_dog(x, label, sem, False, bank)),
    }
    times = {k: [] for k in variants}
    for _ in range(a.rounds):
        for k, fn in variants.items():
            times[k].append(timed(fn, a.reps))
    res = {"gpu": gpu, "batch": n, "size": SIZE, "hair_fraction": float(hair.mean()), "ms": {}}
    print("batch %d, %dx%d, hair %.1f %% of the pixels" % (n, SIZE, SIZE, 100 * float(hair.mean())))
    for k, ts in times.items():
        med = sorted(ts)[len(ts) // 2]
        res["ms"][k] = ts
        print("%-26s %8.4f ms  (rounds: %s)" % (k, med, ", ".join("%.4f" % t for t in ts)))
    with open(os.path.join(a.out_dir, "orient_dog_time.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
