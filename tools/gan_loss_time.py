"""Cost of the adversarial losses of one training iteration at the bench's shapes (batch 8, 512x512, num_D 2, ndf 64): the
generator's GAN + GAN_Feat terms and the discriminator's D_Fake + D_real terms, forward + backward, on the fused reduction
kernels (networks.loss.GANLoss / GANFeatLoss) against a torch restatement of the same losses on the same device
(tests/oracle_gan_objectives.py, eager ops as the reference runs them).

    python tools/gan_loss_time.py OUT_DIR [--batch 8] [--reps 30] [--rounds 3]

Configurations: hinge with --wide_edge 2 (the bench's), hinge with --remove_background, 'ls' and 'original'.  Synthetic
discriminator outputs with the multiscale discriminator's shapes at 512^2 (features 64 @ 257^2 ... 512 @ 66^2 and logits
67^2; 64 @ 129^2 ... 512 @ 34^2 and logits 35^2), stored NHWC and seen as NCHW views, sliced from one fake || real batch as
Pix2PixModel.discriminate does.  Writes OUT_DIR/gan_loss_time.json and prints one line per measurement (median of `reps`
CUDA-event timings, each round alternating kernels and torch), headed by the GPU's name, power limit and maximum SM clock
(read-only nvidia-smi query).
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
# (channels, side) of each discriminator's intermediate features and logits at 512^2, ndf 64, n_layers_D 4
SCALES = (((64, 257), (128, 129), (256, 65), (512, 66), (1, 67)), ((64, 129), (128, 65), (256, 33), (512, 34), (1, 35)))


def disc_outputs(n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    outs = []
    for scale in SCALES:
        d = []
        for c, s in scale:
            t = torch.randn(2 * n, s, s, c, device="cuda", generator=g).permute(0, 3, 1, 2)
            d.append(t)
        outs.append(d)
    return [[t[:n] for t in p] for p in outs], [[t[n:] for t in p] for p in outs]


def hair_label(n):
    seg = torch.zeros(n, 3, SIZE, SIZE, device="cuda")
    seg[:, 1, 100:380, 120:400] = 1.0
    seg[:, 0] = 1 - seg[:, 1]
    return seg[:, 1:2]


def iteration(gan, feat, fake, real, label):
    """GAN + GAN_Feat of the generator step, then D_Fake + D_real of the discriminator step, each backward."""
    f = [[t.detach().requires_grad_() for t in p] for p in fake]
    g = (gan(f, True, False, label) + feat(f, real, label)).sum()
    g.backward()
    fd = [[t.detach().requires_grad_() for t in p] for p in fake]
    rd = [[t.detach().requires_grad_() for t in p] for p in real]
    d = (gan(fd, False, True, label) + gan(rd, True, True, label)).sum()
    d.backward()


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import oracle_gan_objectives as og
    from michigan_b200.networks.loss import GANFeatLoss, GANLoss
    from michigan_b200.options import make_opt
    if not torch.cuda.is_available():
        raise SystemExit("gan_loss_time needs a CUDA device")
    info = gpu_info()
    print(info)
    fake, real = disc_outputs(a.batch)
    label = hair_label(a.batch)
    configs = [("hinge wide_edge 2", "hinge", False), ("hinge remove_background", "hinge", True), ("ls", "ls", False),
               ("original", "original", False)]
    res = {"gpu": info, "batch": a.batch, "size": SIZE, "unit": "ms per iteration (G: GAN + GAN_Feat, D: D_Fake + D_real, "
           "forward + backward)", "results": {}}
    for name, mode, rb in configs:
        opt = make_opt(gan_mode=mode, remove_background=rb, wide_edge=2.0, lambda_feat=10.0)
        crit, critF = GANLoss(mode, opt=opt), GANFeatLoss(opt)

        def kern():
            iteration(lambda p, tir, fd, lab: crit(p, tir, for_discriminator=fd, label=lab), critF, fake, real, label)

        def eager():
            iteration(lambda p, tir, fd, lab: og.gan_loss(p, tir, fd, lab, mode, 2.0, rb),
                      lambda f, r, lab: og.gan_feat_loss(f, r, lab, 10.0, rb), fake, real, label)
        tk, te = [], []
        for _ in range(a.rounds):
            tk.append(timed(kern, a.reps))
            te.append(timed(eager, a.reps))
        k, e = sorted(tk)[len(tk) // 2], sorted(te)[len(te) // 2]
        res["results"][name] = {"kernels_ms": k, "torch_ms": e, "speedup": e / k}
        print("%-26s kernels %.3f ms  torch %.3f ms  (%.2fx)" % (name, k, e, e / k))
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "gan_loss_time.json"), "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
