"""SHA-256 digests of the raw output bytes of the tensor-core kernels (conv_tc_kernel, conv_tc_smallc_kernel, wgrad_tc_kernel) on seeded inputs: one conv
per template instantiation and per feature of the epilogue, the producer and the host set-up.  The kernels are deterministic run to run (the row maximum is an
order-independent atomic max, the weight-gradient partials are reduced in a fixed order), so two builds that compute the same thing print the same JSON.
Run on the GPU:  python tools/conv_tc_digest.py [OUT.json]"""
import hashlib, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from focoos_b200 import ops
from focoos_b200.engine import _split3_weights

if not torch.cuda.is_available():
    sys.exit("conv_tc_digest: needs a CUDA device")
DEV = "cuda"
RELU, SILU, GELU, AFTER = ops.ACT_RELU, ops.ACT_SILU, ops.ACT_GELU, 16
F16, F32 = torch.float16, torch.float32
digests = {}
seed = [0]


def rnd(shape, dtype=F32, s=1.0):
    seed[0] += 1
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed[0])) * s).to(dtype).to(DEV)


def record(name, *tensors):
    torch.cuda.synchronize()
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.contiguous().cpu().numpy().tobytes())
    assert name not in digests, name
    digests[name] = h.hexdigest()


def folded_bn(Cout):
    return rnd((Cout,)).abs() + 0.5, rnd((Cout,), s=0.2)


def conv_f16(name, B, H, W, Cin, Cout, k, stride=1, act=RELU, out_dtype=F16, res=False, pad=None):
    """fp16 operands, one product (FS = false)"""
    pad = (k - 1) // 2 if pad is None else pad
    x, w = rnd((B, H, W, Cin), F16), rnd((Cout, k, k, Cin), F16, (k * k * Cin) ** -0.5)
    sc, bi = folded_bn(Cout)
    r = rnd((B, (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1, Cout), out_dtype) if res else None
    record(name, ops.conv2d(x, w, sc, bi, stride=stride, pad=pad, act=act, residual=r, out_dtype=out_dtype, algo=ops.ALGO_TCGEN05))


def conv_split(name, B, H, W, C, Cout, k, stride=1, act=RELU, out_pair=True, res=False):
    """split-precision operands, three products (FS = true, or the small-channel kernel), fp32 or pair output"""
    pad = (k - 1) // 2
    xp, w3 = ops.to_pair(rnd((B, H, W, C), s=3.0)), _split3_weights(rnd((Cout, k, k, C), s=(k * k * C) ** -0.5))
    sc, bi = folded_bn(Cout)
    r = rnd((B, (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1, Cout)) if res else None
    r = ops.to_pair(r) if res and out_pair else r
    out = ops.conv2d_pair(xp, w3, sc, bi, stride=stride, pad=pad, act=act, residual=r, out_pair=out_pair)
    record(name, out.buf if out_pair else out)


# ---- fp16 operands: BLOCK_K 64 / 32 x BLOCK_N 64 / 128 x fp16 / fp32 output
for odt in (F16, F32):
    o = "f16" if odt == F16 else "f32"
    conv_f16(f"f16_k64_n64_{o}", 2, 20, 20, 64, 64, 3, out_dtype=odt)
    conv_f16(f"f16_k64_n128_{o}", 2, 20, 20, 256, 256, 3, out_dtype=odt)
    conv_f16(f"f16_k32_n64_{o}", 2, 40, 40, 32, 64, 3, out_dtype=odt)
    conv_f16(f"f16_k32_n128_{o}", 2, 16, 16, 32, 128, 1, out_dtype=odt)
conv_f16("f16_gelu", 1, 1, 400, 256, 1024, 1, act=GELU)
conv_f16("f16_res_then_relu", 2, 20, 20, 256, 1024, 1, res=True)
conv_f16("f16_silu_then_res", 2, 20, 20, 256, 256, 3, act=SILU | AFTER, res=True)
conv_f16("f32_res_then_relu", 1, 1, 1000, 256, 512, 1, out_dtype=F32, res=True)
conv_f16("f16_k32_res_in_staging", 2, 40, 40, 32, 64, 3, res=True)          # 32-channel stages have no room for the residual: it lands in the staging buffer
conv_f16("f16_k32_res_in_staging_after", 2, 40, 40, 32, 128, 3, act=SILU | AFTER, res=True)
conv_f16("f16_s2_even", 2, 40, 40, 128, 128, 3, stride=2)
conv_f16("f16_s2_odd", 2, 33, 41, 64, 64, 3, stride=2)
conv_f16("f16_2x2_s2", 2, 40, 40, 256, 512, 2, stride=2, act=0, pad=0)
conv_f16("f32_cout_tail", 1, 1, 300, 256, 80, 1, out_dtype=F32)
conv_f16("f16_cout_tail", 1, 1, 300, 256, 200, 1)
conv_f16("f16_ragged_map", 2, 7, 9, 64, 64, 3)

# ---- split precision: fp32 and pair output, with and without residual, on every (BLOCK_K, BLOCK_N)
for pair in (False, True):
    o = "pair" if pair else "f32"
    conv_split(f"fs_k64_n128_{o}", 2, 20, 20, 256, 256, 3, out_pair=pair)
    conv_split(f"fs_k64_n64_{o}", 2, 40, 40, 64, 64, 3, out_pair=pair)
    conv_split(f"fs_k32_n128_{o}", 2, 40, 40, 32, 128, 3, out_pair=pair)
    conv_split(f"fs_k32_n64_{o}", 2, 20, 20, 96, 64, 3, out_pair=pair)
    conv_split(f"fs_k64_n128_{o}_res", 3, 20, 20, 512, 2048, 1, out_pair=pair, res=True)
    conv_split(f"fs_k64_n64_{o}_res", 2, 24, 40, 256, 64, 1, out_pair=pair, res=True)
    conv_split(f"fs_k32_n128_{o}_res_after", 2, 20, 20, 96, 128, 3, act=SILU | AFTER, out_pair=pair, res=True)
    conv_split(f"fs_s2_even_{o}", 2, 40, 40, 128, 128, 3, stride=2, out_pair=pair)
    conv_split(f"fs_s2_odd_{o}", 2, 33, 41, 64, 64, 3, stride=2, out_pair=pair)
    conv_split(f"fs_ragged_map_{o}", 2, 7, 9, 64, 128, 3, out_pair=pair, res=True)
    conv_split(f"smallc_32_{o}", 2, 40, 200, 32, 32, 3, out_pair=pair)
    conv_split(f"smallc_64_{o}", 1, 33, 130, 32, 64, 3, out_pair=pair)
conv_split("fs_cout_tail_f32", 1, 1, 300, 256, 80, 1, out_pair=False)

# channel slices of wider pair buffers: input = channels [0, C), residual = [C, 2C), output = a slice of another buffer
C = 128
yp = ops.to_pair(rnd((2, 20, 24, 2 * C), s=2.0))
dst = ops.Pair(torch.zeros((2, 20, 24, 4 * C), dtype=F16, device=DEV))
ops.conv2d_pair(yp.slice(0, C), _split3_weights(rnd((C, 3, 3, C), s=0.03)), None, rnd((C,), s=0.2), pad=1, act=SILU | AFTER, residual=yp.slice(C, 2 * C),
                out=dst.slice(C, 2 * C))
record("fs_pair_channel_slices", dst.buf)

# split-precision conv spelled through ops.conv2d (the dense [hi|lo] tensor, forwarded to conv2d_pair)
record("fs_conv2d_entry", ops.conv2d(ops.split_pair(rnd((2, 20, 20, 128), s=3.0)), _split3_weights(rnd((128, 3, 3, 128), s=0.03)), *folded_bn(128), pad=1, act=RELU,
                                     out_dtype=F32, algo=ops.ALGO_TCGEN05_SPLIT3))

# per-image weights (3-D weight map): fp16 and split precision
B, H, W, C, Q = 3, 40, 52, 256, 100
x, me = rnd((B, H, W, C)), rnd((B, Q, C), s=C ** -0.5)
out = torch.zeros((B, H, W, 104), dtype=F16, device=DEV)
ops.conv2d_per_image(x.half(), me.half().reshape(B, Q, 1, 1, C), out=out[..., :Q])
record("f16_per_image_weights", out)
out = torch.zeros((B, H, W, 104), dtype=F32, device=DEV)
ops.conv2d_per_image(ops.to_pair(x), _split3_weights(me).reshape(B, Q, 1, 1, 3 * C), out=out[..., :Q])
record("fs_per_image_weights", out)

# row-max-only epilogue
x, w, b = rnd((3, 1000, 256), s=2.0), rnd((365, 256), s=0.08), rnd((365,), s=2.0) - 3.0
record("f16_rowmax", ops.linear_rowmax(x.half(), w.half(), b))
record("fs_rowmax", ops.linear_rowmax_pair(ops.to_pair(x), _split3_weights(w), b))

# weight gradients: [hi | lo] pairs (three products) and plain fp16 (one product), stride 1 and 2, both tile widths
be = ops._be()
for name, B, H, W, Cin, Cout, k, stride in [("s1_n128", 2, 40, 40, 256, 256, 3, 1), ("s1_n64", 2, 23, 37, 64, 128, 3, 1), ("s1_lin", 1, 1, 600, 256, 1024, 1, 1),
                                            ("s2_n128", 2, 31, 45, 128, 256, 3, 2), ("s2_n64", 2, 40, 40, 64, 64, 3, 2)]:
    pad = (k - 1) // 2
    x, dy = rnd((B, H, W, Cin)), rnd((B, (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1, Cout))
    dw = torch.empty((Cout, k, k, Cin), device=DEV)
    be.conv_wgrad_tc(ops.split_pair(x), ops.split_pair(dy), k, k, stride, pad, dw)
    record(f"wgrad_pair_{name}", dw)
    be.conv_wgrad_tc_f16(x.half(), dy.half(), k, k, stride, pad, dw)
    record(f"wgrad_f16_{name}", dw)

text = json.dumps({"device": torch.cuda.get_device_name(), "digests": digests}, indent=1, sort_keys=True)
print(text)
if len(sys.argv) > 1:
    with open(sys.argv[1], "w") as f:
        f.write(text + "\n")
