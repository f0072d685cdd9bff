"""Times the five small-channel 3x3 fp32-accurate convs of every ResNet-vd forward (pair in, pair out, folded BN + ReLU) at bs=32 and writes their outputs.
Run on the GPU:  python tools/conv_smallc_micro.py [OUT_DIR]   (with OUT_DIR: one <layer>.npy per shape, the pair output for seeded inputs, so two
builds can be compared bit for bit)

Rows: conv1_2 and conv1_3 of the stem at 320x320 (Cin = 32) and branch2b of the three res2 blocks at 160x160 (the three share one shape).
Bytes are algorithmic (input pair, weight pair and output pair once each, 4 B per element); flops are those of the fp32 conv.  The tensor roof is a third of
the sustained fp16 rate (three products per algorithmic product)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from bench import measured_peaks
from focoos_b200 import ops
from focoos_b200.engine import _split3_weights

B = 32
SHAPES = [("conv1_2", 320, 320, 32, 32), ("conv1_3", 320, 320, 32, 64), ("res2_branch2b", 160, 160, 64, 64)]
LAUNCHES = {"res2_branch2b": 3}
ITERS, WARM = 20, 3

out_dir = sys.argv[1] if len(sys.argv) > 1 else None
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
pk = measured_peaks()
tensor = pk["tf_sustained"] * 1e12 / 3.0
hbm = pk["hbm_gbs"] * 1e9
print(f"{torch.cuda.get_device_name()}: tensor roof {tensor / 1e12:.0f} TFLOP/s algorithmic (sustained fp16 / 3), HBM {hbm / 1e9:.0f} GB/s; bs={B}, {ITERS} timed launches each")
print(f"{'layer':14} {'shape':22} {'us':>8} {'floor':>7} {'eff':>5} {'GB':>6} {'GFLOP':>7} {'GB/s':>6} {'TF/s':>6} bound")
total = floor_total = 0.0
for name, H, W, Cin, Cout in SHAPES:
    g = torch.Generator().manual_seed(H + Cin + Cout)
    x = (torch.rand(B, H, W, Cin, generator=g) * 3.0).cuda()
    w = (torch.randn(Cout, 3, 3, Cin, generator=g) / (9 * Cin) ** 0.5)
    sc, bi = torch.rand(Cout, generator=g) + 0.5, torch.randn(Cout, generator=g) * 0.2
    xp, w3, sc, bi = ops.to_pair(x), _split3_weights(w).cuda(), sc.cuda(), bi.cuda()
    out = ops.Pair.empty((B, H, W, Cout), x.device)
    run = lambda: ops.conv2d_pair(xp, w3, sc, bi, pad=1, act=ops.ACT_RELU, out=out)
    for _ in range(WARM):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(ITERS):
        run()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / ITERS
    if out_dir:
        np.save(os.path.join(out_dir, name + ".npy"), out.buf.cpu().numpy())
    flops = 2.0 * B * H * W * Cout * 9 * Cin
    byts = 4.0 * (B * H * W * Cin + Cout * 9 * Cin + B * H * W * Cout)
    floor = max(flops / tensor, byts / hbm) * 1e6
    n = LAUNCHES.get(name, 1)
    total += n * us
    floor_total += n * floor
    print(f"{name:14} {f'{H}x{W} {Cin}->{Cout}':22} {us:8.1f} {floor:7.1f} {floor / us:5.2f} {byts / 1e9:6.2f} {flops / 1e9:7.1f} {byts / us / 1e3:6.0f} {flops / us / 1e6:6.1f} "
          f"{'tensor' if flops / tensor > byts / hbm else 'HBM'}{f'  (x{n} per forward)' if n > 1 else ''}")
print(f"five launches per forward: {total:.1f} us, floor {floor_total:.1f} us")
