"""Launcher: run an UNMODIFIED MichiGAN script (train.py / inference.py) on the sm_90a kernels, one process per GPU.

    python -m michigan_b200.launch <reference_root> inference.py --name MichiGAN --netG spadeb ...          # 1 GPU
    torchrun --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 -m michigan_b200.launch <reference_root> train.py \\
        --batchSize 4 <README flags>                                                                       # 8 GPUs

It replaces `--gpu_ids 0,1,...,7` + nn.DataParallel: `--batchSize` is per process, `--gpu_ids` is set to this process's
LOCAL_RANK (the reference then calls torch.cuda.set_device on it, options/base_options.py), a NCCL process group is
created for WORLD_SIZE > 1, `michigan_b200.install()` rebinds the hot-path classes, and the script runs via runpy from
the reference root (its relative paths - ./inference_samples, ./checkpoints - keep working).
"""
import os
import runpy
import sys


def main(argv=None, run_name="__main__"):
    argv = list(sys.argv[1:] if argv is None else argv)
    if len(argv) < 2:
        raise SystemExit("usage: python -m michigan_b200.launch <reference_root> <script.py> [script args...]")
    root, script, rest = os.path.abspath(argv[0]), argv[1], argv[2:]
    import torch
    import torch.distributed as dist
    local = int(os.environ.get("LOCAL_RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    if "--gpu_ids" in rest:
        i = rest.index("--gpu_ids")
        gpu_ids = rest[i + 1]
        del rest[i:i + 2]
    else:
        gpu_ids = None
    cpu_dry_run = gpu_ids == "-1"          # host-logic tests only (tests/dryrun.py); the product has no CPU path
    if not cpu_dry_run:
        if not torch.cuda.is_available():
            raise RuntimeError("michigan_b200.launch needs a CUDA device (no CPU path exists)")
        torch.cuda.set_device(local)
    if world > 1 and not dist.is_initialized():
        if cpu_dry_run:
            dist.init_process_group("gloo")
        else:
            dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import michigan_b200
    michigan_b200.install(root)
    old_argv, old_cwd = sys.argv, os.getcwd()
    sys.argv = [script] + rest + ["--gpu_ids", "-1" if cpu_dry_run else str(local)]
    os.chdir(root)
    try:
        return runpy.run_path(os.path.join(root, script), run_name=run_name)
    finally:
        sys.argv = old_argv
        os.chdir(old_cwd)
        from michigan_b200 import checkpoint
        checkpoint.wait_pending()


if __name__ == "__main__":
    main()
