"""Cost of the paper's objective: the train step with the README's loss set (hinge GAN, GAN_Feat, VGG, lab, ORIENT) and with the
reference's default loss set (also content, style, background, rgb, CONFIDENCE) against the SURVEY §8d set (hinge GAN, GAN_Feat),
alternated in one process, plus the VGG and Lab loss kernels on their own and, for context, the oracle's VGG restatement run
eagerly on CUDA (cuDNN) with the same seeded weights.  The VGG terms of the default objective are timed as one combined pass
(VGG L1 + content + style, ref == tag and ref != tag) and as VGGLoss + StyleContentLoss called separately (what the reference's
Pix2PixModel does under install()), with the style statistics and tap-gradient kernels on their own.

    python tools/vgg_lab_time.py OUT_DIR [--batch 8] [--steps 5] [--rounds 3] [--remove_background]

--remove_background times only the hair-masked VGG terms: the combined VGG L1 + content + style pass (_VGGObjectiveFn, ref !=
tag, the tag and reference labels of the synthetic batch) and the default-objective train step, each masked against unmasked,
alternated in one process (OUT_DIR/vgg_lab_time_remove_background.json).

Batch 8, 512x512, synthetic inputs.  Writes OUT_DIR/vgg_lab_time.json and prints one line per measurement, headed by the GPU's
name, power limit and maximum SM clock (read-only nvidia-smi query).  Algorithmic rates: VGG = fake forward + real forward +
data gradient down to the image (3 x the forward's 2*MAC count per image, computed from the layer shapes); Lab = the bytes
of both images read by the forward and by the backward plus d fake written.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

SIZE = 512
_VGG_CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, 256, "M", 512, 512, 512, 512, "M", 512]


def vgg_forward_flop(size):
    """2 * MAC of VGG19 features[0:30] on one size x size image."""
    flop, cin, s = 0, 3, size
    for v in _VGG_CFG:
        if v == "M":
            s //= 2
            continue
        flop += 2 * 9 * cin * v * s * s
        cin = v
    return flop


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def timed(fn, reps, warmup=2):
    """Median of `reps` CUDA-event timings of fn() in ms."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--remove_background", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vgg_lab_time.py needs a CUDA device")
    if a.remove_background:
        return remove_background_times(a)
    import oracle_vgg_lab as ovl
    from kernel_times import DEFAULT_LOSSES, README_LOSSES, build_model
    from michigan_b200 import ops
    from michigan_b200.networks import LabColorLoss, StyleContentLoss, VGGLoss
    from michigan_b200.networks.loss import vgg_objective
    from michigan_b200.networks.sync_batchnorm import DataParallelWithCallback
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import train_iteration
    from michigan_b200.synth import synthetic_batch, vgg19_state_dict

    info = gpu_info()
    print("GPU:", info)
    n = a.batch
    data = synthetic_batch(n, SIZE, 1234)
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in data.items()}
    legs = {}
    for name, losses in (("8d", {}), ("readme", README_LOSSES), ("default", DEFAULT_LOSSES)):
        model = build_model(n, **losses)
        wrap = DataParallelWithCallback(model, device_ids=[0])
        optG, optD = model.create_optimizers(model.opt)
        legs[name] = (wrap, optG, optD)
    res = {"gpu": info, "batch": n, "size": SIZE, "images_per_s": {k: [] for k in legs}}
    for r in range(a.rounds):
        for name, (wrap, optG, optD) in legs.items():
            if r == 0:
                timed(lambda: train_iteration(wrap, optG, optD, dict(dev)), 1, warmup=2)
            t = timed(lambda: [train_iteration(wrap, optG, optD, dict(dev)) for _ in range(a.steps)], 1, warmup=0)
            res["images_per_s"][name].append(1e3 * n * a.steps / t)
            print("round %d  %-7s train step %.1f ms  %.2f images/s" % (r, name, t / a.steps, 1e3 * n * a.steps / t))
    del legs, wrap, optG, optD, model

    sd = vgg19_state_dict(0)
    crit = VGGLoss(make_opt(), state_dict=sd)
    g = torch.Generator().manual_seed(0)
    fake = (torch.rand(n, 3, SIZE, SIZE, generator=g) * 2 - 1).cuda()
    real = (torch.rand(n, 3, SIZE, SIZE, generator=g) * 2 - 1).cuda()

    def vgg_step():
        x = fake.detach().requires_grad_()
        crit(x, real).backward()

    flop = 3 * vgg_forward_flop(SIZE) * n
    ms = timed(vgg_step, 10)
    res["vgg_ms"], res["vgg_tflops"], res["vgg_gflop_per_image"] = ms, flop / ms / 1e9, flop / n / 1e9
    print("VGG loss fwd+bwd (ours): %.2f ms, %.1f GFLOP/img, %.0f TFLOP/s algorithmic" % (ms, flop / n / 1e9, flop / ms / 1e9))
    sdc = {k: v.cuda() for k, v in sd.items()}

    def vgg_oracle():
        x = fake.detach().requires_grad_()
        ovl.vgg_loss(x, real, sdc).backward()

    ms_o = timed(vgg_oracle, 5)
    res["vgg_cudnn_ms"] = ms_o
    print("VGG loss fwd+bwd (oracle, eager cuDNN, torch defaults): %.2f ms, %.0f TFLOP/s algorithmic" % (ms_o, flop / ms_o / 1e9))

    # the VGG terms of the default objective: one combined pass against the two loss classes called separately
    sc = StyleContentLoss(make_opt(), vgg=crit.vgg)
    ref = (torch.rand(n, 3, SIZE, SIZE, generator=g) * 2 - 1).cuda()

    def separate():
        x = fake.detach().requires_grad_()
        lc, ls = sc(x, real, real)
        (crit(x, real) + lc + ls).backward()

    def combined(style):
        x = fake.detach().requires_grad_()
        sum(vgg_objective(crit.vgg, x, real, style, l1=True, content=True, style=True)).backward()

    for r in range(a.rounds):
        for key, fn in (("separate", separate), ("combined", lambda: combined(real)), ("combined_ref_ne_tag", lambda: combined(ref))):
            ms = timed(fn, 5)
            res.setdefault("vgg_default_%s_ms" % key, []).append(ms)
            print("round %d  VGG + content + style fwd+bwd, %-20s %.2f ms" % (r, key, ms))
    taps, _ = crit.vgg.run(ops.nchw_to_nhwc(torch.cat([fake, real]).contiguous(), 4))
    gv = torch.ones(2, device="cuda")
    state = {}

    def style_fwd():
        sums = [ops.channel_sums(t) for t in taps]
        state["coefs"] = ops.style_loss_fwd([(s[:n], s[n:], t.shape[1] * t.shape[2]) for s, t in zip(sums, taps)])[1]

    def style_bwd():
        for i, t in enumerate(taps):
            ops.style_tap_grad(t[:n], gv, coef=state["coefs"][i], content_t=t[n:] if i == 4 else None)

    tap_bytes = sum(t.numel() * 4 for t in taps)
    ms_f, ms_b = timed(style_fwd, 20), timed(style_bwd, 20)
    res["style_stats_ms"], res["style_tap_grad_ms"] = ms_f, ms_b
    print("style statistics + loss (5 x mg_in_stats + mg_style_loss_fwd, %.2f GB of taps read): %.3f ms, %.0f GB/s"
          % (tap_bytes / 1e9, ms_f, tap_bytes / ms_f / 1e6))
    print("style tap gradients (5 x mg_style_tap_grad, fake half read + written, relu5_1 target read): %.3f ms, %.0f GB/s"
          % (ms_b, (tap_bytes + taps[4].numel() * 2) / ms_b / 1e6))

    lab = LabColorLoss(make_opt())

    def lab_step():
        x = fake.detach().requires_grad_()
        lab(x, real).backward()

    ms_l = timed(lab_step, 20)
    nbytes = n * SIZE * SIZE * 4 * (6 + 6 + 3)
    res["lab_ms"], res["lab_gbs"] = ms_l, nbytes / ms_l / 1e6
    print("Lab loss fwd+bwd: %.3f ms, %.0f GB/s algorithmic" % (ms_l, nbytes / ms_l / 1e6))
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "vgg_lab_time.json"), "w") as f:
        json.dump(res, f, indent=1)


def remove_background_times(a):
    """The masked VGG terms and the default-objective train step against the unmasked ones, alternated."""
    from kernel_times import DEFAULT_LOSSES, build_model
    from michigan_b200.networks import VGGLoss
    from michigan_b200.networks.loss import vgg_objective
    from michigan_b200.networks.sync_batchnorm import DataParallelWithCallback
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import train_iteration
    from michigan_b200.synth import synthetic_batch, vgg19_state_dict

    info = gpu_info()
    print("GPU:", info)
    n = a.batch
    data = synthetic_batch(n, SIZE, 1234)
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in data.items()}
    res = {"gpu": info, "batch": n, "size": SIZE}
    legs = {}
    for name, rb in (("default", False), ("default_remove_background", True)):
        model = build_model(n, remove_background=rb, mask_vgg_losses=rb, **DEFAULT_LOSSES)
        wrap = DataParallelWithCallback(model, device_ids=[0])
        optG, optD = model.create_optimizers(model.opt)
        legs[name] = (wrap, optG, optD)
    for r in range(a.rounds):
        for name, (wrap, optG, optD) in legs.items():
            if r == 0:
                timed(lambda: train_iteration(wrap, optG, optD, dict(dev)), 1, warmup=2)
            t = timed(lambda: [train_iteration(wrap, optG, optD, dict(dev)) for _ in range(a.steps)], 1, warmup=0)
            res.setdefault("train_step_ms/" + name, []).append(t / a.steps)
            print("round %d  %-26s train step %.1f ms  %.2f images/s" % (r, name, t / a.steps, 1e3 * n * a.steps / t))
    del legs, wrap, optG, optD, model

    crit = VGGLoss(make_opt(), state_dict=vgg19_state_dict(0))
    g = torch.Generator().manual_seed(0)
    fake, real, ref = [(torch.rand(n, 3, SIZE, SIZE, generator=g) * 2 - 1).cuda() for _ in range(3)]
    lab_tag, lab_ref = (dev["label_tag"] == 1).float(), (dev["label_ref"] == 1).float()      # the hair class

    def combined(masked):
        x = fake.detach().requires_grad_()
        kw = dict(label=lab_tag, style_label=lab_ref) if masked else {}
        sum(vgg_objective(crit.vgg, x, real, ref, l1=True, content=True, style=True, **kw)).backward()

    for r in range(a.rounds):
        for key, masked in (("unmasked", False), ("remove_background", True)):
            ms = timed(lambda: combined(masked), 5)
            res.setdefault("vgg_default_ref_ne_tag_ms/" + key, []).append(ms)
            print("round %d  VGG + content + style fwd+bwd, ref != tag, %-18s %.2f ms" % (r, key, ms))
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "vgg_lab_time_remove_background.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
