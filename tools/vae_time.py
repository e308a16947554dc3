"""Cost of --use_vae at batch 8, 512x512, ngf 64: the stand-alone train step (train_iteration: G step + D step) with --use_vae
against the default partial-conv reference encoder, and the pieces --use_vae adds - ConvEncoder forward + backward, the
generator's latent head (forward, input gradient, weight gradient) and KLDLoss forward + backward.

    python tools/vae_time.py OUT_DIR [--batch 8] [--reps 20] [--rounds 3]

Synthetic inputs (synthetic_batch) and the models' own initial weights.  Prints one line per measurement (median of `reps`
CUDA-event timings; each round alternates the two train steps), headed by the GPU's name, power limit and maximum SM clock
(read-only nvidia-smi query), and writes OUT_DIR/vae_time.json.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "vae_time.py needs a GPU"
    os.makedirs(a.out_dir, exist_ok=True)
    from michigan_b200 import ops
    from michigan_b200.networks.autograd import _Grads, latent_bwd
    from michigan_b200.networks.loss import KLDLoss
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel, train_iteration
    from michigan_b200.synth import synthetic_batch
    gpu = gpu_info()
    print("GPU:", gpu)
    n = a.batch
    data = synthetic_batch(n, SIZE, 1)
    models, nets = {}, {}
    for name, vae in (("train step --use_vae", True), ("train step default encoder", False)):
        m = Pix2PixModel(make_opt(is_train=True, batchSize=n, crop_size=SIZE, use_vae=vae))
        og, od = m.create_optimizers(m.opt)
        models[name] = (lambda m=m, og=og, od=od: train_iteration(m, og, od, data))
        nets[vae] = m
    E, G = nets[True].netE, nets[True].netG
    img = data["image_ref"].cuda()

    def enc():
        mu, logvar = E(img)
        (mu.sum() + logvar.sum()).backward()

    z = torch.randn(n, 256, device="cuda")
    S = SimpleNamespace()
    x = G.latent_head(z, n, "cuda", S)
    dx = torch.randn_like(x)
    K = dx[0].numel()
    dy_ref = ops.nhwc_to_nchw(dx).view(n, 1, 1, K)
    za = torch.cat([z, torch.ones(n, 1, device="cuda"), torch.zeros(n, 31, device="cuda")], 1).view(n, 1, 1, 288)
    mu = torch.randn(n, 256, device="cuda", requires_grad=True)
    lv = torch.randn(n, 256, device="cuda", requires_grad=True)
    kld = KLDLoss()

    def kld_fb():
        kld(mu, lv).backward()

    pieces = {
        "ConvEncoder fwd+bwd": enc,
        "latent head fwd": lambda: G.latent_head(z, n, "cuda", None),
        "latent head input grad": lambda: ops.conv_dgrad(dx.view(n, 1, 1, K), S.wp.view(K, -1, 1, 1), (1, 1), 1, 0),
        "latent head weight + bias grad": lambda: ops.conv_wgrad(dy_ref, za, 1, 1, 1, 0),
        "latent head backward (latent_bwd)": lambda: latent_bwd(_Grads(), G.fc, S, dx),
        "KLDLoss fwd+bwd": kld_fb,
    }
    res = {"gpu": gpu, "batch": n, "size": SIZE, "ms": {}}
    for r in range(a.rounds):
        for name, fn in models.items():
            t = timed(fn, a.reps)
            res["ms"].setdefault(name, []).append(t)
            print("round %d  %-36s %8.2f ms" % (r, name, t), flush=True)
    for name, fn in pieces.items():
        t = timed(fn, a.reps * 5)
        res["ms"][name] = [t]
        print("%-44s %8.3f ms" % (name, t), flush=True)
    with open(os.path.join(a.out_dir, "vae_time.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
