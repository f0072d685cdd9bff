"""-m gpu: MaskFormer and BisenetFormer at image sizes that are not multiples of 32.

The stride-2 3x3 convs on odd maps load their A operand through a 4-D tensor map with traversal stride 2 (conv_tc.cu); even maps keep the 5-D parity view.
Every tensor-core configuration a stride-2 layer can reach is checked against an fp64 conv on odd maps, bit for bit against the same conv on the map
zero-extended to even size, and the engines are checked to launch the same conv kernels at odd sizes as at even ones.  The other kernels the odd maps reach
(stem, pools, nearest / bilinear upsamples) are checked at odd and non-x2 geometries, and both models end to end against goldens from the reference."""
import json
import math
import os
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from focoos_b200 import ops
from focoos_b200.bisenetformer import BisenetFormer, BisenetFormerConfig
from focoos_b200.engine import _split3_weights
from focoos_b200.fai_mf import FAIMaskFormer, MaskFormerConfig
from focoos_b200.processor import MaskFormerProcessor
from focoos_b200.utils.seeded_weights import seeded_state_dict
from oracle.gen_golden import synth_images
from tests.parity_utils import GOLDEN, load_golden, manifest_template, update_report

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
DEV = "cuda"
FAMILIES = {"mf": (FAIMaskFormer, MaskFormerConfig, "fai_mf_l_coco_ins"), "bisenet": (BisenetFormer, BisenetFormerConfig, "bisenetformer_l_ade")}


def rnd(shape, dtype, seed, s=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * s).to(dtype)


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def close(got, ref, tol, what):
    a, b = got.detach().double().cpu(), ref.detach().double().cpu()
    err, scale = float((a - b).abs().max()), max(1.0, float(b.abs().max()))
    assert err <= tol * scale, f"{what}: max|d|={err:.3e} scale={scale:.2e}"


def resize_tol(x_nchw, size):
    """bilinear resize at a non-integer ratio: the kernels compute the source coordinate (dst + 0.5) * (in / out) - 0.5 in fp32, like ATen, and the scale and
    the coordinate are rounded once each, so a value may move by up to two ulps of the largest coordinate times the largest step between neighbours"""
    step = max(float(x_nchw.diff(dim=-1).abs().max()) if x_nchw.shape[-1] > 1 else 0.0, float(x_nchw.diff(dim=-2).abs().max()) if x_nchw.shape[-2] > 1 else 0.0)
    return 2 * 2.0 ** -24 * max(size) * step


# ---- conv_tc: 3x3 stride-2 pad-1 convs on odd maps -------------------------------------------------------------------------------------------------------
# mode: "f16" = fp16 operands and output (fp16 precision); "fs32" / "pair" = fused split (fp32_tc) with fp32 / pair output.  Cin 32 -> 32-channel k-blocks,
# Cin >= 64 -> 64-channel k-blocks; Cout 64 -> N64 tiles, Cout 128 -> N128 tiles.
CONFIGS = [(mode, cin, cout) for mode in ("f16", "fs32", "pair") for cin, cout in ((32, 64), (32, 128), (64, 64), (128, 128))]
# the bars test_gpu_conv_tc.py holds the same configurations to on even maps
TOL = {"f16": 3e-3, "fs32": 2e-5, "pair": 2e-5}


def _conv_inputs(B, H, W, Cin, Cout, mode, seed):
    dt = torch.float16 if mode == "f16" else torch.float32
    x = rnd((B, H, W, Cin), dt, seed + 1, 1.0 if mode == "f16" else 3.0)
    w = rnd((Cout, 3, 3, Cin), dt, seed + 2, 1.0 / math.sqrt(9 * Cin))
    sc, bi = torch.rand(Cout, generator=torch.Generator().manual_seed(seed + 3)) + 0.5, rnd((Cout,), torch.float32, seed + 4, 0.2)
    return x, w, sc, bi


def _run_tc(x, w, sc, bi, mode):
    """the layer on the tensor cores (an unsupported shape raises: no CUDA-core fallback) -> fp32 NHWC on the host"""
    x, sc, bi = x.to(DEV), sc.to(DEV), bi.to(DEV)
    if mode == "f16":
        out = ops.conv2d(x, w.to(DEV), sc, bi, stride=2, pad=1, act=ops.ACT_RELU, out_dtype=torch.float16, algo=ops.ALGO_TCGEN05)
    elif mode == "fs32":
        out = ops.conv2d_pair(ops.to_pair(x), _split3_weights(w).to(DEV), sc, bi, stride=2, pad=1, act=ops.ACT_RELU, out_pair=False)
    else:
        out = ops.conv2d_pair(ops.Pair(ops.split_pair(x)), _split3_weights(w).to(DEV), sc, bi, stride=2, pad=1, act=ops.ACT_RELU, out_pair=True)
    torch.cuda.synchronize()
    return out.float().cpu()


def _ref64(x, w, sc, bi):
    y = F.conv2d(nchw(x.double()), nchw(w.double()), None, 2, 1) * sc.double().view(1, -1, 1, 1) + bi.double().view(1, -1, 1, 1)
    return nhwc(torch.relu(y))


@pytest.mark.parametrize("mode,Cin,Cout", CONFIGS)
@pytest.mark.parametrize("H,W", [(45, 62), (46, 61), (45, 61), (1, 1), (3, 3), (5, 7)])
def test_conv_s2_odd_maps_vs_fp64(mode, Cin, Cout, H, W):
    x, w, sc, bi = _conv_inputs(2, H, W, Cin, Cout, mode, seed=H * 100 + W)
    got = _run_tc(x, w, sc, bi, mode)
    ref = _ref64(x, w, sc, bi)
    assert got.shape == ref.shape == (2, (H - 1) // 2 + 1, (W - 1) // 2 + 1, Cout)
    close(got, ref, TOL[mode], f"{mode} {Cin}->{Cout} @{H}x{W}")


@pytest.mark.parametrize("mode,B,H,W,Cin,Cout", [("f16", 2, 45, 61, 256, 256), ("fs32", 2, 45, 61, 256, 256), ("pair", 2, 45, 61, 256, 256),   # ResNet-101 res5 branch2b
                                                  ("pair", 2, 90, 121, 128, 128), ("f16", 2, 23, 31, 512, 512), ("pair", 1, 23, 31, 512, 512),   # res3 / res5 branch2b
                                                  ("f16", 2, 179, 242, 32, 64), ("fs32", 2, 179, 242, 32, 64)])                                  # STDC stem2 ConvX
def test_conv_s2_shipped_odd_shapes_vs_fp64(mode, B, H, W, Cin, Cout):
    x, w, sc, bi = _conv_inputs(B, H, W, Cin, Cout, mode, seed=7)
    close(_run_tc(x, w, sc, bi, mode), _ref64(x, w, sc, bi), TOL[mode], f"{mode} {Cin}->{Cout} @{H}x{W}")


@pytest.mark.parametrize("mode,Cin,Cout", CONFIGS)
@pytest.mark.parametrize("H,W", [(45, 61), (45, 62), (46, 61), (3, 5)])
def test_conv_s2_odd_map_equals_zero_extended_even_map_bitwise(mode, Cin, Cout, H, W):
    """a (2k+1)-row map read through the strided view and the same map zero-extended to 2k+2 rows read through the parity view fill the same smem tiles:
    the outputs (same shape) are identical bit for bit"""
    x, w, sc, bi = _conv_inputs(2, H, W, Cin, Cout, mode, seed=3)
    He, We = H + H % 2, W + W % 2
    xe = torch.zeros((2, He, We, Cin), dtype=x.dtype)
    xe[:, :H, :W] = x
    odd, even = _run_tc(x, w, sc, bi, mode), _run_tc(xe, w, sc, bi, mode)
    assert odd.shape == even.shape
    assert torch.equal(odd, even), f"{mode} {Cin}->{Cout} @{H}x{W}: max|d|={float((odd - even).abs().max()):.3e}"


# ---- no stride-2 conv leaves the tensor cores at odd sizes ------------------------------------------------------------------------------------------------
def _model(family, precision):
    cls, cfg, manifest = FAMILIES[family]
    m = cls(cfg(), precision=precision)
    m.load_state_dict(seeded_state_dict(manifest_template(manifest), 0), strict=True)
    return m.cuda()


def _conv_kernel_sequence(m, x):
    from torch.profiler import ProfilerActivity, profile

    m(x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.2)  # kernels launched right as a session starts have been seen missing from its trace: start the work 0.2 s in
        m(x)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    return [e.name for e in ev if "conv" in e.name.lower()]


@pytest.mark.parametrize("precision", ["fp32_tc", "fp16"])
@pytest.mark.parametrize("family", ["mf", "bisenet"])
def test_odd_sizes_launch_the_conv_kernels_of_even_sizes(family, precision):
    """The ResNet branch2b convs (MaskFormer) and the STDC stem2 ConvX (BisenetFormer) run on odd maps at 357x483 and on even ones at 352x480: the sequence of
    conv kernels launched must be the same, so none of them drops to the CUDA-core conv"""
    m = _model(family, precision)
    seqs = {}
    for size in ((352, 480), (357, 483)):
        img = torch.from_numpy(synth_images(12, [size])[0]).unsqueeze(0).cuda()
        seqs[size] = _conv_kernel_sequence(m, img)
    even, odd = seqs[(352, 480)], seqs[(357, 483)]
    n_tc = sum("conv_tc_kernel" in n for n in even)
    assert n_tc > 0
    assert len(odd) == len(even) and odd == even, [(i, a, b) for i, (a, b) in enumerate(zip(even, odd)) if a != b][:5] or (len(even), len(odd))


# ---- the other kernels at odd and non-x2 geometries --------------------------------------------------------------------------------------------------------
def test_stem_from_uint8_on_odd_images():
    for (H, W) in ((357, 483), (45, 61), (3, 5)):
        img = torch.randint(0, 256, (2, H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(H))
        w, sc, bi = rnd((32, 3, 3, 3), torch.float32, 31, 0.2), torch.rand(32) + 0.5, rnd((32,), torch.float32, 32, 0.1)
        mean, std = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
        got = ops.stem_conv(img.to(DEV), w.to(DEV), sc.to(DEV), bi.to(DEV), mean, std, ops.ACT_RELU, torch.float32)
        xr = (nchw(img.double()) - torch.tensor(mean, dtype=torch.float64).view(1, 3, 1, 1)) / torch.tensor(std, dtype=torch.float64).view(1, 3, 1, 1)
        ref = nhwc(torch.relu(F.conv2d(xr, nchw(w.double()), None, 2, 1) * sc.double().view(1, -1, 1, 1) + bi.double().view(1, -1, 1, 1)))
        close(got, ref, 1e-5, f"stem {H}x{W}")
        pair = ops.stem_conv(img.to(DEV), w.to(DEV), sc.to(DEV), bi.to(DEV), mean, std, ops.ACT_RELU, out_pair=True)
        close(pair.float(), got.cpu(), 1e-6, f"stem pair {H}x{W}")


@pytest.mark.parametrize("H,W", [(179, 242), (45, 61), (23, 31), (90, 121), (5, 7), (1, 1)])
def test_tensor_and_pair_pools_on_odd_maps_vs_fp64(H, W):
    x = rnd((2, H, W, 64), torch.float32, H + W, 3.0)
    x64 = nchw(x.double())
    xg = x.to(DEV)
    close(ops.maxpool3x3s2(xg), nhwc(F.max_pool2d(x64, 3, 2, 1)), 1e-6, "maxpool3x3s2")
    close(ops.avgpool2x2(xg), nhwc(F.avg_pool2d(x64, 2, 2, 0, ceil_mode=True)), 1e-6, "avgpool2x2 ceil")
    close(ops.avgpool3x3s2(xg), nhwc(F.avg_pool2d(x64, 3, 2, 1)), 1e-6, "avgpool3x3s2")
    w9c, sc, bi = rnd((9, 64), torch.float32, 2, 0.3), torch.rand(64) + 0.5, rnd((64,), torch.float32, 3, 0.1)
    dw = F.conv2d(x64, w9c.double().t().reshape(64, 1, 3, 3), None, 2, 1, 1, 64) * sc.double().view(1, -1, 1, 1) + bi.double().view(1, -1, 1, 1)
    close(ops.dwconv3x3s2(xg, w9c.to(DEV), sc.to(DEV), bi.to(DEV)), nhwc(dw), 1e-5, "dwconv3x3s2")
    xp = ops.Pair(ops.split_pair(xg))
    close(ops.maxpool3x3s2(xp).float(), nhwc(F.max_pool2d(x64, 3, 2, 1)), 3e-6, "pair pool mode 0")
    close(ops.avgpool2x2(xp).float(), nhwc(F.avg_pool2d(x64, 2, 2, 0, ceil_mode=True)), 3e-6, "pair pool mode 1")
    size = (2 * H + 1, 2 * W - 1)
    ref = nhwc(F.interpolate(x64, size=size, mode="bilinear", align_corners=False))
    close(ops.resize_bilinear(xp, size).float(), ref, 3e-6 + resize_tol(x64, size) / max(1.0, float(ref.abs().max())), "pair pool mode 2")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("h,w,H,W", [(12, 16, 23, 31), (23, 31, 45, 61), (45, 61, 90, 121), (31, 61, 61, 121)])
def test_upsample_nearest_add_source_indices(dtype, h, w, H, W):
    """each output pixel takes the source pixel F.interpolate(mode="nearest") takes: the source values are their own flat indices (exact in fp16 below 2048)"""
    idx = torch.arange(h * w, dtype=torch.float32).reshape(1, h, w, 1)
    y = (idx % 2048).expand(2, h, w, 8).contiguous().to(dtype)
    cur = torch.zeros((2, H, W, 8), dtype=dtype)
    got = ops.upsample_nearest_add(y.to(DEV), cur.to(DEV)).cpu()
    ref = nhwc(F.interpolate(nchw(y.float()), size=(H, W), mode="nearest")).to(dtype)
    assert torch.equal(got, ref)
    cur = rnd((2, H, W, 8), dtype, 5)
    close(ops.upsample_nearest_add(y.to(DEV), cur.to(DEV)), ref.float() + cur.float(), 2e-3 if dtype == torch.float16 else 1e-6, "nearest + add")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_mask_upsampling_at_non_integer_ratios(dtype):
    """90x121 -> 357x483 (MaskFormer at 357x483), 45x61 -> 357x483 (BisenetFormer) and 270x480 -> 1080x1920: probabilities against torch, and the fused
    argmax / statistics / selection kernels against the materialised probabilities"""
    Q = 100
    for (h, w, H, W) in ((90, 121, 357, 483), (45, 61, 357, 483), (270, 480, 1080, 1920)):
        B = 2 if H < 1000 else 1
        x = (rnd((B, h, w, 104), torch.float32, h, 4.0)).to(dtype)
        ref = F.interpolate(torch.sigmoid(nchw(x.float()[..., :Q]).double()), size=(H, W), mode="bilinear", align_corners=False)
        xg = x.to(DEV)
        probs = ops.mask_sigmoid_upsample(xg, Q, (H, W))
        low = torch.sigmoid(nchw(x.float()[..., :Q]).double())
        close(probs, ref, 2e-6 + resize_tol(low, (H, W)), f"mask_sigmoid_upsample {h}x{w}->{H}x{W}")
        scores = torch.rand((B, Q), generator=torch.Generator().manual_seed(1)).to(DEV)
        l0, c0 = ops.mask_argmax(probs, scores)
        l1, c1 = ops.mask_sigmoid_upsample_argmax(xg, Q, (H, W), scores)
        assert torch.equal(l0, l1) and torch.equal(c0, c1), (h, w, H, W)
        n0, s0 = ops.mask_stats(probs, 0.5)
        n1, s1 = ops.mask_sigmoid_upsample_stats(xg, Q, (H, W), 0.5)
        # the two kernels may round a probability one ulp apart; over the 2 M pixels of a 1080x1920 plane a few sit that close to the threshold
        assert int((n0 - n1).abs().max()) <= (0 if H * W < 10 ** 6 else 4), (h, w, H, W, int((n0 - n1).abs().max()))
        assert float((s0 - s1).abs().max()) <= 1e-5 * float(s0.abs().max())
        bq = torch.tensor([[0, 3], [B - 1, 99], [0, 57]], dtype=torch.int32, device=DEV)
        sel = ops.mask_sigmoid_upsample_select(xg, bq, (H, W))
        for i, (b, q) in enumerate(bq.tolist()):
            assert torch.equal(sel[i], probs[b, q]), (h, w, H, W, b, q)
        del probs, sel
        torch.cuda.empty_cache()


# ---- end to end against the reference's goldens ------------------------------------------------------------------------------------------------------------
def _meta(name):
    with open(os.path.join(GOLDEN, "golden_meta_any_size.json")) as f:
        return json.load(f)[name]


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc", "fp16"])
@pytest.mark.parametrize("name", ["mf_l_coco_ins_b2_357x483", "mf_l_coco_ins_b1_720x1280", "bisenetformer_l_ade_b2_357x483", "bisenetformer_l_ade_b1_720x1280"])
def test_end_to_end_vs_reference_golden_at_any_size(name, precision):
    g, meta = load_golden(name), _meta(name)
    family = "mf" if name.startswith("mf") else "bisenet"
    m = _model(family, precision)
    imgs = synth_images(meta["image_seed"], [tuple(s) for s in g["sizes"].tolist()])
    x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs]).cuda()
    taps = {}
    out = m(x, taps=taps)
    torch.cuda.synchronize()
    scale = float(g["pred_masks_stat"][2])
    pm = taps["pred_masks"][..., :100].permute(0, 3, 1, 2)[:, ::10, ::2, ::2].float().cpu().numpy()
    e = {"mask_logits_max_abs": float(np.abs(pm - g["pred_masks_q10_s2"]).max()), "mask_logit_scale": scale,
         "class_prob_max_abs": float(np.abs(out.logits.cpu().numpy() - g["logits"]).max()),
         "mask_prob_max_abs": float(np.abs(out.masks[:, ::10, ::4, ::4].cpu().numpy() - g["masks_q10_s4"]).max())}
    dets = MaskFormerProcessor(m.config).postprocess(out, imgs, threshold=float(g["threshold"]))
    e["det_counts"], e["ref_counts"] = [len(d) for d in dets], g["det_count"].tolist()
    update_report("parity_report_any_size.json", {f"{name}/{precision}": e})
    print(name, precision, e)
    if precision == "fp16":
        # one fp16 tensor-core product per conv / linear and fp16 activations: the detections may differ.  Bars about twice what an H100 gave (MaskFormer:
        # logits 2.5e-2 relative, class / mask probabilities 0.12 / 0.29; BisenetFormer: 4.8e-3 relative, 0.019 / 0.018)
        lbar, cbar, mbar = (5e-2, 0.25, 0.5) if family == "mf" else (1e-2, 0.05, 0.05)
        assert e["mask_logits_max_abs"] <= lbar * scale and e["class_prob_max_abs"] <= cbar and e["mask_prob_max_abs"] <= mbar, e
        return
    # fp32: the bars of the golden tests at multiples of 32 (test_gpu_mf.py, test_gpu_bisenet.py).  MaskFormer fp32_tc: the pre-sigmoid logits are held to the
    # 1e-3 relative bar of test_gpu_mf.py; the probabilities to the 1e-2 of test_mf_full_size_batch_invariance_and_oracle, class probabilities to 5e-3 (3.5e-3
    # at 720x1280 on an H100): the 9-layer masked decoder's discrete attention masks flip on ~1e-5 differences, and more pixels give more flips
    if family == "mf":
        lbar, cbar, mbar = (1e-4, 1e-3, 1e-3) if precision == "fp32" else (1e-3, 5e-3, 1e-2)
    else:
        lbar, cbar, mbar = (1e-4 if precision == "fp32" else 2e-4), 1e-3, 1e-3
    assert e["mask_logits_max_abs"] <= lbar * scale and e["class_prob_max_abs"] <= cbar and e["mask_prob_max_abs"] <= mbar, e
    for i, d in enumerate(dets):
        n = int(g["det_count"][i])
        assert len(d) == n
        assert [x.cls_id for x in d.detections] == g["det_labels"][i, :n].tolist()
        if n:
            assert np.abs(np.array([x.conf for x in d.detections]) - g["det_scores"][i, :n]).max() <= cbar  # score = class probability x mask score
            # a box edge moves when one pixel's probability sits within ~1e-4 of the threshold: small pixel tolerance, as at multiples of 32
            assert np.abs(np.array([x.bbox for x in d.detections]) - g["det_boxes"][i, :n]).max() <= 3


@pytest.mark.parametrize("family", ["mf", "bisenet"])
def test_odd_size_image_alone_equals_inside_a_batch(family):
    m = _model(family, "fp32_tc")
    imgs = synth_images(21, [(357, 483)] * 4)
    x = torch.stack([torch.from_numpy(im).permute(2, 0, 1).float() for im in imgs]).cuda()
    out4 = m(x)
    out1 = m(x[2:3].contiguous())
    torch.cuda.synchronize()
    assert torch.equal(out4.logits[2:3], out1.logits), "class probabilities depend on the batch"
    assert torch.equal(out4.masks[2:3], out1.masks), "mask probabilities depend on the batch"


@pytest.mark.parametrize("name,manifest", [("fai-mf-l-coco-ins", "fai_mf_l_coco_ins"), ("bisenetformer-l-ade", "bisenetformer_l_ade")])
def test_focoos_model_720p_graph_replay_equals_eager(name, manifest):
    """ModelManager.get(...) -> FocoosModel.__call__ on one 720x1280 uint8 frame: the first call runs eagerly, the second replays the captured CUDA graph"""
    from focoos_b200 import ModelManager

    fm = ModelManager.get(name, state_dict=seeded_state_dict(manifest_template(manifest), 0), precision="fp32_tc")
    fm.model.cuda()
    imgs = synth_images(22, [(720, 1280)])
    runs = [fm(imgs, threshold=0.5, batched=True) for _ in range(2)]
    x = torch.from_numpy(imgs[0]).permute(2, 0, 1).float().unsqueeze(0).cuda()
    ref = fm.processor.postprocess(fm.model(x), imgs, threshold=0.5)
    key = lambda dets: [[(d.cls_id, tuple(d.bbox), d.mask) for d in r.detections] for r in dets]  # noqa: E731
    assert key(runs[0]) == key(runs[1]) == key(ref)
    assert np.allclose([d.conf for d in runs[1][0].detections], [d.conf for d in ref[0].detections], atol=1e-6)


@pytest.mark.timeout(1200)
def test_bisenet_1080p_vs_oracle():
    """one 1080x1920 image in the fp32-accurate mode against the CPU oracle: the bars of test_bisenet_full_size_batch_invariance_and_oracle"""
    from oracle import bisenet_oracle as O

    sd = seeded_state_dict(manifest_template("bisenetformer_l_ade"), 0)
    m = BisenetFormer(BisenetFormerConfig(), precision="fp32_tc")
    m.load_state_dict(sd, strict=True)
    m.cuda()
    x = torch.from_numpy(synth_images(23, [(1080, 1920)])[0]).permute(2, 0, 1).float().unsqueeze(0)
    out = m(x.cuda())
    torch.cuda.synchronize()
    with torch.no_grad():
        probs, masks = O.bisenet_forward(sd, x, O.BisenetOracleConfig())
    e_cls = float((out.logits.cpu() - probs).abs().max())
    e_mask = float((out.masks.cpu() - masks).abs().max())
    sem_g = (out.logits[0].max(-1).values.view(-1, 1, 1) * out.masks[0]).argmax(0).cpu()
    sem_o = (probs[0].max(-1).values.view(-1, 1, 1) * masks[0]).argmax(0)
    differ = float((sem_g != sem_o).float().mean())
    update_report("parity_report_any_size.json", {"bisenet_fp32_tc_1080x1920": {"class_prob_max_abs": e_cls, "mask_prob_max_abs": e_mask, "argmax_pixels_differing": differ}})
    assert e_cls <= 1e-3 and e_mask <= 1e-3, (e_cls, e_mask)
    assert differ <= 1e-4, differ
