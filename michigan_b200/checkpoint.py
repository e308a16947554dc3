"""Checkpoint I/O with the reference's file layout (util/util.py:195-231: `<checkpoints_dir>/<name>/<epoch>_net_<label>.pth`
= a CPU state dict with the network's own keys), device-side behaviour:

  * the reference's `save_network` moves the WHOLE network to the CPU and back in the middle of training
    (`net.cpu().state_dict()`; `net.cuda()`), on every DataParallel thread's shared module; here the parameters stay
    where they are: a snapshot is copied device -> pinned host memory on a side stream (the compute stream only waits
    for that copy, ~20 ms for the generator's 438 MB), and a background thread serialises it;
  * one writer: rank 0 (all ranks hold identical weights), written to a temporary file and renamed, followed by a
    barrier when a process group exists, so no rank can read or overwrite a half-written file.
"""
import atexit
import os
import threading

import torch
import torch.distributed as dist

_pending = {}          # path -> thread
_lock = threading.Lock()


def _rank_world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def wait_pending(path=None):
    """Block until the background writer(s) have finished (all of them, or the one for `path`)."""
    with _lock:
        items = [(p, t) for p, t in _pending.items() if path is None or p == path]
    for p, t in items:
        t.join()
        with _lock:
            if _pending.get(p) is t:
                del _pending[p]


atexit.register(wait_pending)


def _write(path, host_sd, event):
    if event is not None:
        event.synchronize()
    tmp = "%s.tmp.%d" % (path, os.getpid())
    torch.save(host_sd, tmp)
    os.replace(tmp, path)


def save_state_dict(net, path, asynchronous=True):
    """Write `net.state_dict()` (reference key layout) to `path`.  Rank 0 writes; every rank returns after the barrier.
    asynchronous=True: returns as soon as the snapshot copy is enqueued; `wait_pending()` (also run at exit and before the
    same path is written again) joins the writer."""
    rank, world = _rank_world()
    if rank == 0:
        wait_pending(path)
        os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
        sd = net.state_dict()
        on_gpu = any(v.is_cuda for v in sd.values())
        event = None
        if on_gpu:
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(cur)                        # snapshot = state after everything enqueued so far
            host = {}
            with torch.cuda.stream(side):
                for k, v in sd.items():
                    if v.is_cuda:
                        h = torch.empty(v.shape, dtype=v.dtype, device="cpu", pin_memory=True)
                        h.copy_(v.detach(), non_blocking=True)
                        host[k] = h
                    else:
                        host[k] = v.detach().clone()
                event = torch.cuda.Event()
                event.record(side)
            cur.wait_stream(side)                        # later optimizer steps must not overwrite what is being copied
        else:
            host = {k: v.detach().clone() for k, v in sd.items()}
        if asynchronous:
            t = threading.Thread(target=_write, args=(path, host, event), daemon=False)
            with _lock:
                _pending[path] = t
            t.start()
        else:
            _write(path, host, event)
    if world > 1:
        dist.barrier()


def network_path(opt, label, epoch):
    return os.path.join(opt.checkpoints_dir, opt.name, "%s_net_%s.pth" % (epoch, label))


def save_network(net, label, epoch, opt):
    """Signature of util.save_network (util/util.py:195-200); installed over it by michigan_b200.install()."""
    save_state_dict(net, network_path(opt, label, epoch))
