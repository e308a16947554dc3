"""Per-kernel GPU time of one generator-forward step and one train step at the benchmark configuration (batch 8, 512x512,
synthetic inputs, random-init weights), from torch.profiler CUDA activity.

    python tools/kernel_times.py OUT_DIR [--batch N] [--warmup W]

Writes OUT_DIR/kernel_times.md (one table per workload: kernel, launches, total ms, share of the step's kernel time) and
OUT_DIR/kernel_times.json.  Templated kernels are listed per instantiation, so the variant of each conv kernel is visible.
Selects the library like everything else (MICHIGAN_B200_LIB), which makes before/after tables of two builds comparable.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

SIZE = 512


def build_model(batch):
    import random
    from michigan_b200.options import make_opt
    from michigan_b200.pix2pix_model import Pix2PixModel
    from michigan_b200.synth import fill_state_dict
    random.seed(0)
    torch.manual_seed(0)
    opt = make_opt(is_train=True, gpu_ids=[0], batchSize=batch, niter=50, niter_decay=0)
    model = Pix2PixModel(opt)
    fill_state_dict(model.netG.state_dict(), 0)
    fill_state_dict(model.netD.state_dict(), 1)
    model.train()
    return model


def kernel_table(step, warmup):
    """Runs `step` warmup times, then once under the profiler -> [(kernel, launches, total_us)], longest first."""
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or ev.device_time_total <= 0:
            continue
        n, us = rows.get(ev.name, (0, 0.0))
        rows[ev.name] = (n + 1, us + ev.device_time_total)
    return sorted(((k, n, us) for k, (n, us) in rows.items()), key=lambda r: -r[2])


def markdown(title, rows):
    total = sum(us for _, _, us in rows)
    out = ["## %s: %.2f ms of kernel time" % (title, total / 1e3), "", "| kernel | launches | ms | share |", "|---|---|---|---|"]
    for name, n, us in rows:
        out.append("| `%s` | %d | %.3f | %.1f %% |" % (name.replace("|", "\\|"), n, us / 1e3, 100.0 * us / total))
    return "\n".join(out) + "\n"


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("out_dir")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kernel_times.py needs a CUDA device")
    from michigan_b200.networks.sync_batchnorm import DataParallelWithCallback
    from michigan_b200.pix2pix_model import train_iteration
    from michigan_b200.synth import synthetic_batch

    model = build_model(a.batch)
    data = synthetic_batch(a.batch, SIZE, 1234)
    dev = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in data.items()}
    tables = {}
    with torch.no_grad():
        pre = model.preprocess_input(dev)
        tables["generator forward"] = kernel_table(lambda: model.generate_fake(pre[0], pre[2], pre[4], pre[1], pre[3], pre[5]),
                                                   a.warmup)
    wrap = DataParallelWithCallback(model, device_ids=[0])
    optG, optD = model.create_optimizers(model.opt)
    tables["train step"] = kernel_table(lambda: train_iteration(wrap, optG, optD, dict(dev)), a.warmup)

    os.makedirs(a.out_dir, exist_ok=True)
    gpu = torch.cuda.get_device_name(0)
    with open(os.path.join(a.out_dir, "kernel_times.md"), "w") as f:
        f.write("# Per-kernel time, batch %d, %dx%d, %s\n\n" % (a.batch, SIZE, SIZE, gpu))
        for title, rows in tables.items():
            f.write(markdown(title, rows) + "\n")
    with open(os.path.join(a.out_dir, "kernel_times.json"), "w") as f:
        json.dump({"gpu": gpu, "batch": a.batch,
                   "tables": {t: [{"kernel": k, "launches": n, "us": us} for k, n, us in rows] for t, rows in tables.items()}}, f, indent=1)
    for title, rows in tables.items():
        print("%s: %.2f ms kernel time, %d kernels" % (title, sum(us for _, _, us in rows) / 1e3, len(rows)))


if __name__ == "__main__":
    main()
