"""One-process check of mg_conv_img: parity against torch (fp32) on three shapes, then CUDA-event timing at the benchmark
shape (8 x 512 x 512 x 64 -> 3)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from michigan_b200 import ops
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
dev = "cuda"
g = torch.Generator(device="cpu").manual_seed(7)
worst = 0.0
for N, H, W, C in ((2, 32, 64, 64), (1, 20, 45, 64), (1, 9, 33, 32), (1, 128, 128, 64)):
    x = torch.randn(N, C, H, W, generator=g).to(dev)
    w = (torch.randn(3, C, 3, 3, generator=g) / (C * 9) ** 0.5).to(dev)
    b = (torch.randn(3, generator=g) * 0.1).to(dev)
    ref = torch.tanh(F.conv2d(F.leaky_relu(x, 0.2), w, b, padding=1))
    got = ops.conv_img(x.permute(0, 2, 3, 1).contiguous(), w, b)
    err = float((got - ref).abs().max())
    worst = max(worst, err)
    print("conv_img %s max-abs err %.3e" % ((N, H, W, C), err), flush=True)
x = torch.randn(8, 512, 512, 64, device=dev)
w = torch.randn(3, 64, 3, 3, device=dev) / 24
b = torch.zeros(3, device=dev)
for _ in range(3):
    ops.conv_img(x, w, b)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(20):
    ops.conv_img(x, w, b)
e1.record(); torch.cuda.synchronize()
print("conv_img 8x512x512x64: %.4f ms/launch" % (e0.elapsed_time(e1) / 20))
print("PARITY_OK" if worst <= 1e-5 else "PARITY_FAIL", worst)
