"""Times the wgmma weight-gradient kernel alone on the heaviest training shapes."""
import sys, os
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from focoos_b200 import autograd_ops as A, ops

SHAPES = {"fpn_rep_3x3_80": (16, 80, 80, 256, 256, 3), "res3_3x3_80": (16, 80, 80, 128, 128, 3), "res2_1x1_160": (16, 160, 160, 64, 256, 1), "res5_1x1_20": (16, 20, 20, 2048, 512, 1),
          "dec_ffn_lin": (1, 1, 4800, 256, 1024, 1)}
names = sys.argv[1:] or list(SHAPES)
be = ops._be()
for n in names:
    B, H, W, Cin, Cout, k = SHAPES[n]
    x = torch.randn((B, H, W, Cin), device="cuda")
    dy = torch.randn((B, H, W, Cout), device="cuda")
    xp, dp = ops.split_pair(x), ops.split_pair(dy)
    dw = torch.empty((Cout, k, k, Cin), device="cuda")
    for _ in range(3):
        be.conv_wgrad_tc(xp, dp, k, k, 1, (k - 1) // 2, dw)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        be.conv_wgrad_tc(xp, dp, k, k, 1, (k - 1) // 2, dw)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    fl = 2.0 * B * H * W * Cin * Cout * k * k
    print(f"{n:16s} {ms * 1e3:8.1f} us  {fl / ms / 1e9:7.1f} TFLOP/s algorithmic (x3 products issued = {3 * fl / ms / 1e9:7.1f} on the tensor pipe)")
