"""Per-forward weight preparation: batched spectral norm + operand packing for the tensor-core kernels.

State-dict tensors stay OIHW fp32 with the reference's key layout (`weight_orig/_u/_v`, SURVEY.md §5);
the packed copies (tap-major K, W/sigma applied, TF32-rounded) are transient device buffers that are
rebuilt whenever a parameter's version counter changes.
"""
import ctypes as C

import torch

from .. import _lib, ops


class _SnDesc(C.Structure):
    _fields_ = [("w", C.c_void_p), ("u", C.c_void_p), ("v", C.c_void_p), ("t", C.c_void_p), ("s", C.c_void_p),
                ("inv_sigma", C.c_void_p), ("O", C.c_int32), ("K", C.c_int32)]


def is_spectral(conv):
    return hasattr(conv, "weight_orig")


class SpectralNormBatch:
    """All spectrally-normalised convs of one network, processed by mg_spectral_norm_batched."""

    def __init__(self, convs):
        self.convs = list(convs)
        self._key = None
        self._descs = None
        self.inv_sigma = None

    def _build(self, device):
        n = len(self.convs)
        ks = [c.weight_orig[0].numel() for c in self.convs]
        os_ = [c.weight_orig.shape[0] for c in self.convs]
        self.max_K, self.max_O = max(ks), max(os_)
        self.t_ws = torch.zeros(sum(ks), device=device, dtype=torch.float32)
        self.s_ws = torch.zeros(sum(os_), device=device, dtype=torch.float32)
        self.inv_sigma = torch.zeros(n, device=device, dtype=torch.float32)
        arr = (_SnDesc * n)()
        ko = oo = 0
        for i, c in enumerate(self.convs):
            w = c.weight_orig
            if not w.is_contiguous():
                raise ValueError("weight_orig must be contiguous")
            arr[i].w, arr[i].u, arr[i].v = w.data_ptr(), c.weight_u.data_ptr(), c.weight_v.data_ptr()
            arr[i].t = self.t_ws.data_ptr() + 4 * ko
            arr[i].s = self.s_ws.data_ptr() + 4 * oo
            arr[i].inv_sigma = self.inv_sigma.data_ptr() + 4 * i
            arr[i].O, arr[i].K = os_[i], ks[i]
            ko += ks[i]
            oo += os_[i]
        raw = bytes(arr)
        host = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
        self._descs = host.to(device)
        self._key = tuple((c.weight_orig.data_ptr(), c.weight_u.data_ptr(), c.weight_v.data_ptr()) for c in self.convs)

    def run(self, training):
        """Power iteration (training) + sigma for every layer; returns the [L] inv_sigma tensor."""
        if not self.convs:
            return None
        dev = self.convs[0].weight_orig.device
        key = tuple((c.weight_orig.data_ptr(), c.weight_u.data_ptr(), c.weight_v.data_ptr()) for c in self.convs)
        if self._descs is None or key != self._key or self._descs.device != dev:
            self._build(dev)
        _lib.check(_lib.load().mg_spectral_norm_batched(self._descs.data_ptr(), len(self.convs), self.max_O, self.max_K,
                                                        int(training), 1e-12, ops._stream()),
                   "mg_spectral_norm_batched")
        return self.inv_sigma


class PackCache:
    """Caches packed operands keyed on the source tensors' (data_ptr, _version)."""

    def __init__(self):
        self._store = {}

    def get(self, name, tensors, build, volatile=False):
        key = tuple((t.data_ptr(), t._version) for t in tensors)
        hit = self._store.get(name)
        if not volatile and hit is not None and hit[0] == key:
            return hit[1]
        val = build()
        self._store[name] = (key, val)
        return val

    def clear(self):
        self._store.clear()
