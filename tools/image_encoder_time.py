"""Cost of --Image_encoder_mode instance and norm at batch 8, 512x512, ngf 64: the stand-alone train step (train_iteration: G
step + D step) in each mode against partialconv (the default), alternated in one process, and each encoder's forward +
backward (forward_nhwc with saving, then backward_nhwc on a random output gradient).

    python tools/image_encoder_time.py OUT_DIR [--batch 8] [--reps 20] [--rounds 3]

Synthetic inputs (synthetic_batch) and the models' own initial weights.  Prints one line per measurement (median of `reps`
CUDA-event timings; each round alternates the train steps), headed by the GPU's name, power limit and maximum SM clock
(read-only nvidia-smi query), and writes OUT_DIR/image_encoder_time.json.
"""
import argparse
import json
import os
import sys
from types import SimpleNamespace

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)
import torch

from vgg_lab_time import gpu_info, timed

SIZE = 512
MODES = (("partialconv", False), ("instance", False), ("instance", True), ("norm", False))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "image_encoder_time.py needs a GPU"
    os.makedirs(a.out_dir, exist_ok=True)
    from michigan_b200.networks.autograd import _Grads
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel, train_iteration
    from michigan_b200.synth import synthetic_batch
    gpu = gpu_info()
    print("GPU:", gpu)
    n = a.batch
    data = synthetic_batch(n, SIZE, 1)
    steps, encs = {}, {}
    for mode, gp in MODES:
        name = mode + (" --ref_global_pool" if gp else "")
        m = Pix2PixModel(make_opt(is_train=True, batchSize=n, crop_size=SIZE, Image_encoder_mode=mode, ref_global_pool=gp))
        og, od = m.create_optimizers(m.opt)
        steps["train step " + name] = (lambda m=m, og=og, od=od: train_iteration(m, og, od, data))
        encs[name] = m.netG.fc
    img = data["image_ref"].cuda()
    lab = data["label_ref"].cuda()

    def enc_fb(E):
        S = SimpleNamespace()
        out = E.forward_nhwc(img, lab, lab, save=S)
        E.backward_nhwc(_Grads(), S, torch.ones_like(out))

    res = {"gpu": gpu, "batch": n, "size": SIZE, "ms": {}}
    for r in range(a.rounds):
        for name, fn in steps.items():
            t = timed(fn, a.reps)
            res["ms"].setdefault(name, []).append(t)
            print("round %d  %-44s %8.2f ms" % (r, name, t), flush=True)
    for name, E in encs.items():
        t = timed(lambda E=E: enc_fb(E), a.reps * 5)
        res["ms"]["encoder fwd+bwd " + name] = [t]
        print("%-52s %8.3f ms" % ("encoder fwd+bwd " + name, t), flush=True)
    with open(os.path.join(a.out_dir, "image_encoder_time.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
