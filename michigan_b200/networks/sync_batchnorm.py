"""Replacement for the reference's vendored `models/networks/sync_batchnorm/` package.

The reference's data-parallel runtime is single-process torch.nn.DataParallel plus a Python
thread/queue master-slave SyncBN (batchnorm.py:51-145, comm.py:18-137, replicate.py:27-94).  The
The design is one process per GPU:

  * SyncBN statistics: every rank pushes its [sum | sum of squares | sample count] vector into all
    peers' symmetric buffers over NVLink and sums the world_size vectors in rank order inside ONE
    small kernel (`mg_peer_allreduce_f64`, csrc/mg_peer.cu) - no NCCL call, no host round trip, the
    result is bit-identical on every rank.  Without peer memory (gloo CPU tests, or when the
    symmetric-memory rendezvous is unavailable) the same vector goes through `dist.all_reduce`.
  * parameters and buffers are broadcast from rank 0 when the wrapper is built (nn.DataParallel
    re-replicates GPU 0's module on every forward, replicate.py:50-67, so replicas there can never
    differ; here they are made equal once and stay equal because every rank applies the same
    averaged gradient);
  * gradients: `GradReducer` - one flat fp32 buffer per network, filled stage by stage INSIDE the
    hand-written backward (autograd.py) and all-reduced (average) on NCCL's stream while the
    remaining stages still compute; `.grad` of every parameter is a view into the flat buffer.  The
    unchanged reference trainer (backward(); optimizer.step()) therefore needs no extra call.

The public names are kept so that `from models.networks.sync_batchnorm import
SynchronizedBatchNorm2d, DataParallelWithCallback` (normalization.py:10, pix2pix_trainer.py:6)
keeps working.
"""
import ctypes as C
import os

import torch
import torch.distributed as dist
import torch.nn as nn

from .. import _lib, ops


def _world():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _rank():
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


# ================================================================================================ statistics exchange
class _PeerExchange:
    """Symmetric exchange buffer of this process group + the call sequence number (see csrc/mg_peer.cu)."""

    def __init__(self, device):
        import torch.distributed._symmetric_memory as symm
        lib = _lib.load()
        world, rank = _world(), _rank()
        nbytes = int(lib.mg_peer_buffer_bytes(world))
        if nbytes <= 0:
            raise RuntimeError("world size %d not supported by the peer exchange" % world)
        self.buf = symm.empty((nbytes + 7) // 8, dtype=torch.float64, device=device)
        self.buf.zero_()
        self.hdl = symm.rendezvous(self.buf, dist.group.WORLD)
        ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        if len(ptrs) != world or int(self.hdl.rank) != rank:
            raise RuntimeError("symmetric-memory rendezvous returned %d peers for world %d" % (len(ptrs), world))
        self.ptrs = (C.c_void_p * world)(*ptrs)
        self.status = torch.zeros(1, device=device, dtype=torch.int32)
        self.world, self.rank, self.seq = world, rank, 0
        self.max_elems = int(lib.mg_peer_max_elems())
        torch.cuda.synchronize(device)   # every buffer is zeroed before the first push can land

    def allreduce(self, vec, tail):
        """In-place sum over ranks; element [-1] is replaced by `tail` (this rank's sample count) before the exchange."""
        self.seq += 1
        _lib.check(_lib.load().mg_peer_allreduce_f64(vec.data_ptr(), vec.numel(), self.ptrs, self.world, self.rank, self.seq,
                                                     1, float(tail), self.status.data_ptr(), ops._stream()), "mg_peer_allreduce_f64")

    def check(self):
        """Host-synchronising health check (tests / end of an epoch): did any exchange time out?"""
        if int(self.status.item()) != 0:
            raise RuntimeError("michigan_b200: a SyncBN peer exchange timed out (a rank died or the ranks' call sequences diverged)")


_exchange = {"state": None, "backend": None}   # state: None = not decided, False = use dist.all_reduce, _PeerExchange


def exchange_backend():
    """'peer' | 'collective' | None (single process / not decided yet) - reported by bench.py."""
    return _exchange["backend"]


def _peer_exchange_for(t):
    """Decide ONCE per process (collectively, so that all ranks agree) how statistics are exchanged."""
    st = _exchange["state"]
    if st is not None:
        return st or None
    ok = 0
    ex = None
    if t.is_cuda and dist.get_backend() == "nccl" and os.environ.get("MICHIGAN_B200_PEER_EXCHANGE", "1") != "0":
        try:
            ex = _PeerExchange(t.device)
            ok = 1
        except Exception as e:   # no symmetric memory on this platform: fall back to the collective (never to a CPU path)
            if _rank() == 0:
                print("michigan_b200: peer-memory statistics exchange unavailable (%s: %s); using dist.all_reduce" % (type(e).__name__, e))
    flag = torch.tensor([ok], device=t.device if t.is_cuda else "cpu", dtype=torch.int32)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)      # also the barrier that orders buffer zeroing before the first push
    if int(flag.item()) == 1:
        _exchange["state"], _exchange["backend"] = ex, "peer"
        return ex
    _exchange["state"], _exchange["backend"] = False, "collective"
    return None


def reset_exchange():
    """Forget the exchange state (tests that create several process groups in one process)."""
    _exchange["state"] = _exchange["backend"] = None


def allreduce_sums(sums, local_count):
    """Sum the per-rank statistics vector across the data-parallel group, in place, together with the per-rank sample
    count (batchnorm.py:119 `sum_size`).  sums: [2*C + 1] float64; element 2*C receives the count.
    Returns the `count` argument for mg_bn_finalize / mg_bn_bwd_apply: the host value when single-process, 0.0
    ("read sums[2*C] on the device") otherwise.  Replaces SyncMaster.run_master / SlavePipe.run_slave +
    ReduceAddCoalesced/Broadcast (batchnorm.py:105-126, comm.py:49-133)."""
    if _world() == 1:
        return float(local_count)
    ex = _peer_exchange_for(sums)
    if ex is not None and sums.numel() <= ex.max_elems:
        ex.allreduce(sums, local_count)
    else:
        sums[-1] = float(local_count)
        dist.all_reduce(sums, op=dist.ReduceOp.SUM)
    return 0.0


class SynchronizedBatchNorm2d(nn.Module):
    """Parameter/buffer container with the reference's state-dict layout (running_mean, running_var,
    num_batches_tracked, optional affine weight/bias) and its statistics semantics
    (batchnorm.py:63-93,128-145): train -> global batch statistics over all ranks, biased variance
    for normalisation, running stats updated with momentum 0.1 and the unbiased variance,
    num_batches_tracked never incremented (the reference's forward bypasses nn.BatchNorm.forward);
    eval -> running statistics.  1/sqrt(var+eps) is used in every mode (the reference's
    single-replica / CPU path, batchnorm.py:65-68); see DESIGN.md for the clamp variant.
    """

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True):
        super().__init__()
        self.num_features, self.eps, self.momentum, self.affine = num_features, eps, momentum, affine
        if affine:
            self.weight = nn.Parameter(torch.ones(num_features))
            self.bias = nn.Parameter(torch.zeros(num_features))
        else:
            self.register_parameter("weight", None)
            self.register_parameter("bias", None)
        self.register_buffer("running_mean", torch.zeros(num_features))
        self.register_buffer("running_var", torch.ones(num_features))
        self.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))

    def scale_shift(self, x_nhwc, upsample_shift=0, extra_running=()):
        """(nscale, nshift) such that x_hat = x*nscale + nshift, for an NHWC tensor.  `upsample_shift`:
        the reference normalises the 2^shift nearest-upsampled tensor - same mean/var, 4^shift more
        samples in the unbiased factor.  `extra_running`: other BN containers that see the same
        input (norm_s next to norm_0) and whose running buffers get the identical update."""
        if not self.training:
            return ops.bn_from_running(self.running_mean, self.running_var, self.eps)
        sums = ops.bn_sums(x_nhwc)
        local = x_nhwc.numel() // x_nhwc.shape[-1]
        mult = 4 ** upsample_shift
        if local * _world() * mult <= 1:
            raise ValueError("BatchNorm computes unbiased standard-deviation, which requires size > 1.")
        count = allreduce_sums(sums, local)
        out = ops.bn_finalize(sums, count, mult, self.eps, self.momentum, 0, self.running_mean, self.running_var, want_stats=True)
        for other in extra_running:
            ops.bn_finalize(sums, count, mult, other.eps, other.momentum, 0, other.running_mean, other.running_var)
        return out

    def forward(self, x):
        raise RuntimeError("SynchronizedBatchNorm2d is consumed by the fused SPADE kernels; it has no standalone forward")

    def extra_repr(self):
        return "{num_features}, eps={eps}, momentum={momentum}, affine={affine}".format(**self.__dict__)


SynchronizedBatchNorm1d = SynchronizedBatchNorm2d
SynchronizedBatchNorm3d = SynchronizedBatchNorm2d


# ================================================================================================ gradient averaging
class GradReducer:
    """Gradient all-reduce (mean over ranks) of one network, driven from inside its hand-written backward.

    All parameters live in ONE flat fp32 gradient buffer, laid out in the order the backward finalises them
    (`stages`: lists of parameters, first stage = first finished).  When a stage's gradients are complete the
    backward calls `reduce_stage(i, grads)`: they are written into the stage's slice (one multi-tensor copy) and
    the slice is all-reduced asynchronously on NCCL's stream while the next stage computes.  `finish()` makes the
    compute stream wait for the outstanding reductions and returns per-parameter VIEWS of the flat buffer, which
    autograd installs as `.grad` - so there is no per-parameter copy-back, no `torch.cat`, and the unchanged
    `loss.backward(); optimizer.step()` of pix2pix_trainer.py:42-58 sees averaged gradients.
    Replaces DataParallel's reduce-add of the replicas' gradients onto GPU 0 (replicate.py:50-67)."""

    def __init__(self, stages):
        self.stages = [[p for p in st if p.requires_grad] for st in stages]
        params = [p for st in self.stages for p in st]
        if not params:
            self.flat = None
            return
        dev = params[0].device
        total = sum(p.numel() for p in params)
        self.flat = torch.zeros(total, device=dev, dtype=torch.float32)
        self.views, self.slices = {}, []
        off = 0
        for st in self.stages:
            s0 = off
            for p in st:
                self.views[id(p)] = self.flat[off:off + p.numel()].view(p.shape)
                off += p.numel()
            self.slices.append((s0, off))
        self.handles = []
        self.avg_op = dist.ReduceOp.AVG if dist.get_backend() == "nccl" else None
        self.world = _world()

    def begin(self, params):
        """Called at the start of a backward.  If a previous backward's gradients are still installed as `.grad`
        (gradient accumulation without zero_grad(set_to_none=True)), the flat buffer cannot be overwritten: use a
        private buffer for this backward (rare path)."""
        self.handles = []
        self._private = None
        if any(p.grad is not None and p.grad.data_ptr() == self.views[id(p)].data_ptr() for p in params if id(p) in self.views):
            self._private = torch.empty_like(self.flat)

    def _target(self, p):
        v = self.views[id(p)]
        if self._private is None:
            return v
        off = (v.data_ptr() - self.flat.data_ptr()) // 4
        return self._private[off:off + p.numel()].view(p.shape)

    def reduce_stage(self, i, get_grad):
        """get_grad(p) -> finished gradient tensor of p or None.  Returns nothing; the views are handed out by finish()."""
        st = self.stages[i]
        if not st:
            return
        dst, src, zero = [], [], []
        for p in st:
            g = get_grad(p)
            if g is None:
                zero.append(self._target(p))
            else:
                dst.append(self._target(p))
                src.append(g.reshape(p.shape))
        if zero:
            torch._foreach_zero_(zero)
        if dst:
            torch._foreach_copy_(dst, src)
        a, b = self.slices[i]
        seg = (self.flat if self._private is None else self._private)[a:b]
        if self.avg_op is not None:
            self.handles.append((dist.all_reduce(seg, op=self.avg_op, async_op=True), None))
        else:
            self.handles.append((dist.all_reduce(seg, op=dist.ReduceOp.SUM, async_op=True), seg))

    def finish(self, params, get_grad):
        """-> tuple of gradients for `params` (views of the reduced flat buffer; None where no gradient exists)."""
        for h, seg in self.handles:
            h.wait()
            if seg is not None:
                seg.div_(self.world)
        self.handles = []
        # fresh view objects: autograd installs a returned gradient as `.grad` without copying only when nothing else
        # references the tensor object (AccumulateGrad's "steal" path)
        return tuple((self._target(p).view(p.shape) if (id(p) in self.views and get_grad(p) is not None) else None) for p in params)


class DataParallelWithCallback(nn.Module):
    """Drop-in for replicate.py:50-67 under one-process-per-GPU.  `device_ids` is accepted for
    signature compatibility; the wrapped module lives on this process's device.  Calls are forwarded
    unchanged (`wrapper(data, mode=...)`), the input is this rank's shard.

    On construction (world > 1): every parameter and buffer is broadcast from rank 0 (the reference's replicas
    are copies of GPU 0's module by construction), and every sub-network that runs a hand-written backward
    (`grad_stages()` protocol: SPADEBGenerator, MultiscaleDiscriminator) gets a GradReducer, so gradients are
    averaged across ranks inside backward()."""

    def __init__(self, module, device_ids=None, output_device=None, dim=0):
        super().__init__()
        self.module = module
        self.device_ids = list(device_ids) if device_ids is not None else []
        self.reducers = []
        if _world() > 1:
            self.broadcast_state()
            for m in module.modules():
                if hasattr(m, "grad_stages") and any(p.requires_grad for p in m.parameters()):
                    m._grad_reducer = GradReducer(m.grad_stages())
                    self.reducers.append(m._grad_reducer)

    def broadcast_state(self):
        """Rank 0's parameters and buffers (weights, spectral-norm u/v, BN running statistics) to every rank."""
        seen = set()
        for t in list(self.module.parameters()) + list(self.module.buffers()):
            if id(t) in seen:
                continue
            seen.add(id(t))
            dist.broadcast(t.data, src=0)

    def forward(self, *inputs, **kwargs):
        return self.module(*inputs, **kwargs)

    def attach_optimizer(self, optimizer):
        """Kept for round-1 callers: gradients are already averaged when backward() returns."""
        return optimizer


def patch_replication_callback(data_parallel):
    return data_parallel


def convert_model(module):
    return module


def patch_sync_batchnorm():
    import contextlib
    return contextlib.nullcontext()
