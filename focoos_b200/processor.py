"""DETRProcessor — host-side mirror of `focoos/models/fai_detr/processor.py` + `focoos/processor/base_processor.py`.

preprocess: list of HWC uint8 / CHW tensors -> [B,3,S,S] fp32 on the device (H2D copy + per-image bilinear
resize to `im_size`, align_corners=False — Processor.get_torch_batch, base_processor.py:223-296).
postprocess: ONE fused kernel for the whole batch (top-k over Q*C, label/query decode, threshold, scale to the
original image, round-half-even), ONE device->host copy of the compacted result, then FocoosDet objects —
replacing the reference's per-image Python loop with 3 `.cpu().tolist()` syncs each (processor.py:183-217).
"""
from __future__ import annotations

import base64
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import ops
from .engine import _split3_weights
from .ports import Boxes, DETRConfig, DETRModelOutput, FocoosDet, FocoosDetections, Instances


def get_image_sizes(inputs) -> List[Tuple[int, int]]:
    """base_processor.py:176-221: (height, width) of every ORIGINAL input image."""
    if _is_u8_nhwc_batch(inputs):
        return [(int(inputs.shape[1]), int(inputs.shape[2]))] * int(inputs.shape[0])
    if _is_nchw_batch(inputs):
        return [(int(inputs.shape[2]), int(inputs.shape[3]))] * int(inputs.shape[0])
    if isinstance(inputs, (torch.Tensor, np.ndarray)) or not isinstance(inputs, (list, tuple)):
        inputs = [inputs]
    sizes = []
    for img in inputs:
        if isinstance(img, torch.Tensor):
            h, w = img.shape[-2:]
        elif isinstance(img, np.ndarray):
            h, w = img.shape[-3:-1] if img.ndim > 3 else img.shape[:2]
        elif hasattr(img, "size") and not callable(img.size):  # PIL
            w, h = img.size
        else:
            raise ValueError(f"Unsupported input type: {type(img)}")
        sizes.append((int(h), int(w)))
    return sizes


def _is_u8_nhwc_batch(x) -> bool:
    """Extension over the reference (which mis-stacks 4-D tensors, SURVEY §7): a uint8 [B,H,W,3] tensor is a batch."""
    return isinstance(x, torch.Tensor) and x.dim() == 4 and x.dtype == torch.uint8 and x.shape[-1] == 3


def _is_nchw_batch(x) -> bool:
    """a [B,3,H,W] tensor / array with B > 1 is a BATCH of images (SURVEY §8f.1; the reference stacks it into a 5-D tensor and fails)"""
    return isinstance(x, (torch.Tensor, np.ndarray)) and x.ndim == 4 and x.shape[1] == 3 and x.shape[0] > 1 and x.shape[-1] != 3


class DETRProcessor:
    def __init__(self, config: DETRConfig, image_size: Optional[Union[int, Tuple[int, int]]] = None):
        self.config = config
        self.image_size = image_size
        self.top_k = config.top_k
        self.threshold = config.threshold
        self.training = False

    def eval(self):
        self.training = False
        return self

    # -- preprocess -------------------------------------------------------------------------------
    def preprocess(self, inputs, device, dtype: torch.dtype = torch.float32):
        if self.training:
            raise ValueError("During training, inputs should be a list of DetectionDatasetDict")
        target = None
        if self.image_size is not None:
            target = (self.image_size, self.image_size) if isinstance(self.image_size, int) else tuple(self.image_size)
        return self.get_torch_batch(inputs, target, device, dtype), []

    def get_torch_batch(self, inputs, target_size, device, dtype):
        if _is_u8_nhwc_batch(inputs):  # one H2D copy for the whole batch
            x = inputs.to(device, non_blocking=True)
            if target_size is not None and tuple(x.shape[1:3]) != tuple(target_size):
                return ops.image_resize(x, target_size).to(dtype)  # one launch: uint8 NHWC batch -> resized float NCHW (the model's float input)
            return x.contiguous()  # FAIDetr's stem kernel reads uint8 NHWC directly (no float CHW copy)
        if _is_nchw_batch(inputs):  # one H2D copy, one batched resize
            x = (torch.from_numpy(np.ascontiguousarray(inputs)) if isinstance(inputs, np.ndarray) else inputs).to(device, non_blocking=True).to(dtype)
            if target_size is not None and tuple(x.shape[-2:]) != tuple(target_size):
                x = ops.image_resize(x.float(), target_size).to(dtype)
            return x.contiguous()
        if not isinstance(inputs, (list, tuple)):
            inputs = [inputs]
        outs = []
        for inp in inputs:
            if hasattr(inp, "size") and not isinstance(inp, (np.ndarray, torch.Tensor)):
                inp = np.array(inp)
            if isinstance(inp, np.ndarray):
                inp = torch.from_numpy(np.ascontiguousarray(inp))
            if inp.dim() == 3:
                inp = inp.unsqueeze(0)
            if inp.shape[1] != 3 and inp.shape[-1] == 3:
                inp = inp.permute(0, 3, 1, 2)
            if device is not None:
                inp = inp.to(device, non_blocking=True)
            inp = inp.to(dtype)
            if target_size is not None and tuple(inp.shape[-2:]) != tuple(target_size):
                inp = self._resize(inp, target_size)
            outs.append(inp.squeeze(0))
        return torch.stack(outs, 0).contiguous()

    @staticmethod
    def _resize(img_nchw: torch.Tensor, size):
        """bilinear, align_corners=False, via the NHWC resize kernel (channels padded 3 -> 4 for vector access)."""
        _, C, H, W = img_nchw.shape
        if C == 3 and img_nchw.dtype == torch.float32:
            return ops.image_resize(img_nchw, size)
        x = torch.zeros((1, H, W, 4), dtype=img_nchw.dtype, device=img_nchw.device)
        x[..., :C] = img_nchw.permute(0, 2, 3, 1)
        y = ops.resize_bilinear(x, size)
        return y[..., :C].permute(0, 3, 1, 2).contiguous()

    # -- postprocess ------------------------------------------------------------------------------
    def postprocess_tensors(self, output: DETRModelOutput, image_sizes: Sequence[Tuple[int, int]], top_k=None, threshold=None):
        top_k = top_k or self.top_k
        threshold = threshold or self.threshold  # `x or default` idiom of the reference (a falsy 0.0 -> default)
        sizes = torch.tensor(list(image_sizes), dtype=torch.int32).to(output.logits.device, non_blocking=True)
        return ops.detr_postprocess(output.logits, output.boxes, sizes, top_k, threshold)

    def postprocess_packed(self, output: DETRModelOutput, image_sizes, top_k=None, threshold=None, sizes_dev=None) -> torch.Tensor:
        """the fused post-process kernel + the packing of its five outputs into ONE int32 device tensor [B, K*7 + 1]
        (per detection: score bits, label, 4 box coords, query; then the keep count) - the single thing that travels to the host"""
        if sizes_dev is not None:
            s, l, b, q, c = ops.detr_postprocess(output.logits, output.boxes, sizes_dev, top_k or self.top_k, threshold or self.threshold)
        else:
            s, l, b, q, c = self.postprocess_tensors(output, image_sizes, top_k, threshold)
        B = s.shape[0]
        packed = torch.cat([s.view(torch.int32).unsqueeze(-1), l.unsqueeze(-1), b, q.unsqueeze(-1)], dim=-1)
        return torch.cat([packed.reshape(B, -1), c.unsqueeze(-1)], dim=1)

    @staticmethod
    def detections_from_packed(packed_h: np.ndarray, class_names: Sequence[str] = ()) -> List[FocoosDetections]:
        B = packed_h.shape[0]
        K = (packed_h.shape[1] - 1) // 7
        res = []
        for i in range(B):
            n = int(packed_h[i, -1])
            row = packed_h[i, :-1].reshape(K, 7)[:n]
            confs = row[:, 0].copy().view(np.float32).tolist()
            labels = row[:, 1].tolist()
            boxes = row[:, 2:6].tolist()
            res.append(FocoosDetections(detections=[
                FocoosDet(bbox=bx, conf=cf, cls_id=lb, label=class_names[lb] if class_names else None)
                for bx, cf, lb in zip(boxes, confs, labels)]))
        return res

    def postprocess(self, output: DETRModelOutput, inputs, class_names: Sequence[str] = (), top_k=None, threshold=None) -> List[FocoosDetections]:
        image_sizes = get_image_sizes(inputs)
        B = output.boxes.shape[0]
        assert len(image_sizes) == B, f"Expected image sizes {len(image_sizes)} to match batch size {B}"
        # one packed D2H copy: [B, K, 7] (score bits, label, 4 box coords, query) + counts
        return self.detections_from_packed(self.postprocess_packed(output, image_sizes, top_k, threshold).cpu().numpy(), class_names)

    def eval_postprocess(self, output: DETRModelOutput, batched_inputs, top_k: Optional[int] = None):
        """fai_detr/processor.py:121-144 (the evaluator path, trainer/evaluation/evaluator.py:179-190): per image top-k WITHOUT threshold, boxes scaled
        to the dataset entry's (height, width), clipped, empty ones dropped -> [{"instances": Instances(boxes, scores, classes)}].
        ONE kernel for the whole batch (the reference loops over images in Python) and one tiny D2H (the per-image counts); the instance tensors
        stay on the device, as the reference's do.  `batched_inputs[i]` needs `.height` / `.width` (DatasetEntry) or the same dict keys."""
        top_k = top_k or self.top_k
        def hw(e):
            h = e.get("height") if isinstance(e, dict) else getattr(e, "height", None)
            w = e.get("width") if isinstance(e, dict) else getattr(e, "width", None)
            return (int(h or 1), int(w or 1))  # `or 1` as the reference
        sizes = [hw(e) for e in batched_inputs]
        assert len(sizes) == output.logits.shape[0]
        sizes_dev = torch.tensor(sizes, dtype=torch.int32).to(output.logits.device, non_blocking=True)
        s, l, b, c = ops.detr_eval_postprocess(output.logits, output.boxes, sizes_dev, top_k)
        counts = c.cpu().tolist()
        return [{"instances": Instances(sizes[i], boxes=Boxes(b[i, :n]), scores=s[i, :n], classes=l[i, :n].long())} for i, n in enumerate(counts)]

    def export_postprocess(self, output, inputs, class_names=(), top_k=None, threshold: float = 0.5):
        """processor.py:219-236: output = (boxes, logits) of an exported graph."""
        boxes, logits = output[0], output[1]
        if isinstance(boxes, np.ndarray):
            boxes = torch.from_numpy(boxes)
        if isinstance(logits, np.ndarray):
            logits = torch.from_numpy(logits)
        return self.postprocess(DETRModelOutput(boxes=boxes, logits=logits, loss=None), inputs, class_names, 300 if top_k is None else top_k, threshold)


# ==================================================================================================
# MaskFormerProcessor — mirror of `focoos/models/fai_mf/processor.py` (SURVEY §8 a17), instance mode
# ==================================================================================================
def binary_mask_to_base64(mask: np.ndarray) -> str:
    """utils/vision.py:270-293: PNG (0/255, single channel) -> base64, encoded with OpenCV exactly as the reference does (`cv2.imencode(".png", mask * 255)`),
    so the string is byte-identical to the reference's (pinned by tests/test_png_tail.py against strings produced by the unmodified reference function).
    Without OpenCV the image is encoded with PIL: a different byte stream that decodes to the same mask."""
    import base64

    m = (np.asarray(mask) * 255).astype(np.uint8)
    try:
        import cv2
    except ImportError:  # pragma: no cover - the image ships OpenCV
        import io

        from PIL import Image

        buf = io.BytesIO()
        Image.fromarray(m, mode="L").save(buf, format="PNG")
        return base64.b64encode(buf.getvalue()).decode("utf-8")
    ok, enc = cv2.imencode(".png", m)
    if not ok:
        raise ValueError("Failed to encode image")
    return base64.b64encode(enc.tobytes()).decode("utf-8")


def base64_to_binary_mask(b64: str) -> np.ndarray:
    """inverse of binary_mask_to_base64 (utils/vision.py:296-320 decodes the same way for fai_detections_to_sv): PNG -> bool mask"""
    import base64
    import io

    from PIL import Image

    return np.array(Image.open(io.BytesIO(base64.b64decode(b64)))) > 0


_SEM_FMT = {"fp32": "fp32", "fp16": "fp16", "fp32_tc": "pair"}  # model precision -> operand format of the class x mask product


def _entry_get(e, name):
    return e[name] if isinstance(e, dict) else getattr(e, name)


class MaskFormerProcessor(DETRProcessor):
    """preprocess as the base Processor; postprocess = the reference's tensor pipeline as GPU reductions + one compaction:
    per (image, query): pixel count and probability mass of `prob >= mask_threshold` (ONE pass over the [B,Q,H,W] tensor),
    class score x mask score, threshold, then only the KEPT masks are binarised / resized to the original image size and
    boxed and PNG-encoded on the device; only the PNG files travel to the host, for base64.  Works for any batch size (the reference raises IndexError
    for B >= 2, SURVEY A.25): the batched result equals the concatenation of the reference's per-image results."""

    def __init__(self, config, image_size=None):
        self.config = config
        self.image_size = image_size
        self.top_k, self.threshold = config.top_k, config.threshold
        self.mask_threshold, self.use_mask_score, self.predict_all_pixels = config.mask_threshold, config.use_mask_score, config.predict_all_pixels
        self.training = False

    def eval_postprocess(self, output, batched_inputs, top_k: Optional[int] = None, precision: str = "fp32"):
        """fai_mf/processor.py:142-166 for semantic configs (BisenetFormer's processor is the same): per image the mask probabilities at the entry's
        (height, width) and sem_seg = einsum("qc,qhw->chw", logits, probs) (semantic_inference, :99-105) -> [{"sem_seg": [C,height,width] fp32}].
        `output.masks` must be the model's LazyMasks (`lazy_masks = True`).  Per run of entries with the same (height, width), three launches and no
        torch arithmetic: the NHWC probabilities [g,height,width,Qk] (mask_sigmoid_upsample_nhwc, then resize_bilinear when (height, width) is not the
        input size), and the product as a 1x1 conv with per-image weights W_b = logits[b]^T (C padded to Cp, Q to Qk with zeros) writing NHWC scores
        [g,height,width,Cp].  Each "sem_seg" is a [C,H,W] view of that buffer (a permute, channels >= C sliced off).  The reference's crop to the
        augmented size is a no-op here: the masks are at the input size, so its output stride is 1.  The product's arithmetic follows `precision`:
        CUDA-core fp32 ("fp32"), three fp16 tensor-core products on the [hi | lo] pair ("fp32_tc"), one fp16 product with fp32 accumulation ("fp16")."""
        if self.config.postprocessing_type != "semantic":
            raise NotImplementedError("focoos_b200: evaluation of instance-segmentation models (mask AP) is not built; only semantic configs can be evaluated")
        if precision not in _SEM_FMT:
            raise ValueError(f"precision must be one of {sorted(_SEM_FMT)} (got {precision!r})")
        lazy = output.masks
        if not hasattr(lazy, "materialize"):
            raise TypeError("MaskFormerProcessor.eval_postprocess reads the low-resolution mask logits: run the model with `lazy_masks = True`")
        logits = output.logits
        B, Q, C = logits.shape
        assert len(batched_inputs) == B, (len(batched_inputs), B)
        fmt = _SEM_FMT[precision]
        Qk, Cp = -(-Q // 32) * 32, -(-C // 8) * 8  # the tensor-core product takes channels in 32-wide chunks; fp32 rows of 8 channels are 32-byte aligned
        w = torch.zeros((B, Cp, Qk), dtype=torch.float32, device=logits.device)
        w[:, :C, :Q] = logits.transpose(1, 2)
        w = _split3_weights(w) if fmt == "pair" else w.to(torch.float16 if fmt == "fp16" else torch.float32)
        w = w.reshape(B, Cp, 1, 1, w.shape[-1])
        sizes = [(int(_entry_get(e, "height")), int(_entry_get(e, "width"))) for e in batched_inputs]
        results = []
        i = 0
        while i < B:
            j = i + 1
            while j < B and sizes[j] == sizes[i]:
                j += 1
            probs = ops.mask_sigmoid_upsample_nhwc(lazy.logits[i:j], Q, lazy.size, Qk, fmt)
            if sizes[i] != tuple(lazy.size):  # interpolate_image(mask, (height, width))
                probs = ops.resize_bilinear(probs, sizes[i])
            scores = ops.conv2d_per_image(probs, w[i:j], out_dtype=torch.float32)
            results += [{"sem_seg": scores[k, ..., :C].permute(2, 0, 1)} for k in range(j - i)]
            i = j
        return results

    def export_postprocess(self, output, inputs, class_names=(), top_k=None, threshold: float = 0.5):
        """fai_mf/processor.py:308-337: output = (masks, logits) of an exported graph."""
        from .fai_mf import MaskFormerModelOutput

        masks, logits = (torch.from_numpy(t) if isinstance(t, np.ndarray) else t for t in output[:2])
        return self.postprocess(MaskFormerModelOutput(masks=masks, logits=logits, loss=None), inputs, class_names, top_k, threshold)

    def postprocess_tensors(self, output, threshold=None, use_mask_score=None, predict_all_pixels=None):
        """-> list over images of (query idx [n], scores [n], labels [n]) on the host, plus the device masks tensor."""
        threshold = threshold or self.threshold
        use_mask_score = use_mask_score or self.use_mask_score
        predict_all_pixels = predict_all_pixels or self.predict_all_pixels  # fai_mf/processor.py:188-190: the argument ORs with the configured default
        self._labels = self._masks = self._lazy = None
        lazy = hasattr(output.masks, "materialize")  # fai_mf.LazyMasks: low-resolution logits, upsampling not done yet
        if predict_all_pixels and use_mask_score:
            # the reference's mask score of a semantic region is its mean probability over the argmax pixels (:249-257); the fused argmax kernels return pixel
            # counts only, so this combination (no shipped config uses it) is refused rather than scored differently
            raise NotImplementedError("focoos_b200: use_mask_score together with predict_all_pixels is not supported")
        if predict_all_pixels:  # semantic: every pixel goes to argmax_q(score_q * prob_q) (processor.py:208-220)
            scores_dev = output.logits.max(-1).values  # [B,Q]; tiny reduction, stays on the device for the argmax kernel
            if lazy:  # sigmoid + bilinear upsampling + argmax in one kernel: the [B,Q,H,W] tensor is never written
                self._labels, count = ops.mask_sigmoid_upsample_argmax(output.masks.logits, output.masks.num_queries, output.masks.size, scores_dev)
            else:
                self._labels, count = ops.mask_argmax(output.masks, scores_dev)
            psum = count.float()
        else:
            if lazy:  # counts / probability mass straight from the low-resolution logits; only the kept masks are upsampled later
                self._lazy = output.masks
                count, psum = ops.mask_sigmoid_upsample_stats(output.masks.logits, output.masks.num_queries, output.masks.size, float(self.mask_threshold))
            else:
                self._masks = output.masks  # never written back into `output` (it may be a CUDA-graph static)
                count, psum = ops.mask_stats(self._masks, float(self.mask_threshold))
        host = torch.cat([output.logits.reshape(output.logits.shape[0], -1), count.float(), psum], dim=1).cpu().numpy()  # one D2H
        B, Q, K = output.logits.shape
        res = []
        for b in range(B):
            logits = host[b, : Q * K].reshape(Q, K)
            cnt, ps = host[b, Q * K: Q * K + Q], host[b, Q * K + Q:]
            scores, labels = logits.max(-1), logits.argmax(-1)
            nz = np.nonzero(cnt > 1)[0]
            s = scores[nz]
            if use_mask_score:  # (sum 1e-3*m*p) / (sum 1e-3*m + 1e-5), fai_mf/processor.py:249-257
                s = s * ((np.float32(1e-3) * ps[nz]) / (np.float32(1e-3) * cnt[nz] + np.float32(1e-5)))
            keep = np.nonzero(s > threshold)[0] if threshold > 0 else np.arange(len(s))
            res.append((nz[keep].astype(np.int32), s[keep].astype(np.float32), labels[nz][keep].astype(np.int32)))
        return res

    @staticmethod
    def _crops_to_base64(m, box):
        """(boxes as a host array, base64 PNG of every crop m[i][y1:min(y2,H), x1:min(x2,W)]) - trim_mask + binary_mask_to_base64, utils/vision.py:264-293.
        Device masks are encoded on the device (ops.mask_png): only the files and their lengths reach the host.  Host masks come only from the CPU
        reference backend of the tests (every product op refuses host tensors) and are encoded by binary_mask_to_base64 itself."""
        H, W = m.shape[1:]
        if not m.is_cuda:
            mh, box_h = m.numpy().astype(bool), box.numpy()
            return box_h, [binary_mask_to_base64(mh[i][y1:min(y2, H), x1:min(x2, W)]) for i, (x1, y1, x2, y2) in enumerate(box_h.tolist())]
        png, lens = ops.mask_png(m, box)
        box_h, data = box.cpu().numpy(), png.cpu().numpy().tobytes()
        out, off = [], 0
        for (x1, y1, x2, y2), n in zip(box_h.tolist(), lens.tolist()):
            if n:
                out.append(base64.b64encode(data[off:off + n]).decode("utf-8"))
                off += n
            else:  # a crop with no rows or no columns: whatever binary_mask_to_base64 does with it
                out.append(binary_mask_to_base64(np.zeros((max(0, min(y2, H) - y1), max(0, min(x2, W) - x1)), dtype=bool)))
        return box_h, out

    def postprocess(self, output, inputs, class_names=(), top_k=None, threshold=None, use_mask_score=None, predict_all_pixels=None):
        image_sizes = get_image_sizes(inputs)
        B = output.logits.shape[0]
        assert len(image_sizes) == B, f"Expected image sizes {len(image_sizes)} to match batch size {B}"
        # top_k is accepted for signature compatibility: the reference's MaskFormerProcessor.postprocess never reads it either (fai_mf/processor.py:170-262)
        kept = self.postprocess_tensors(output, threshold, use_mask_score, predict_all_pixels)
        results = []
        for b, (q, s, l) in enumerate(kept):
            if len(q) == 0:
                results.append(FocoosDetections(detections=[]))
                continue
            bq = torch.tensor(np.stack([np.full_like(q, b), q], 1), dtype=torch.int32).to(output.logits.device)
            if self._labels is not None:
                m, box = ops.label_resize_bbox(self._labels, bq, image_sizes[b])
            else:
                if self._lazy is not None:  # upsample just this image's kept planes, then index them as a [n,1,H,W] batch
                    planes = ops.mask_sigmoid_upsample_select(self._lazy.logits, bq, self._lazy.size).unsqueeze(1)
                    idx = torch.stack([torch.arange(len(q), dtype=torch.int32), torch.zeros(len(q), dtype=torch.int32)], 1).to(planes.device)
                    m, box = ops.mask_resize_bbox(planes, idx, float(self.mask_threshold), image_sizes[b])
                else:
                    m, box = ops.mask_resize_bbox(self._masks, bq, float(self.mask_threshold), image_sizes[b])
            box_h, masks_b64 = self._crops_to_base64(m, box)
            dets = []
            for i in range(len(q)):
                x1, y1, x2, y2 = (int(v) for v in box_h[i])
                dets.append(FocoosDet(bbox=[x1, y1, x2, y2], conf=float(s[i]), cls_id=int(l[i]), mask=masks_b64[i],
                                      label=class_names[int(l[i])] if class_names else None))
            results.append(FocoosDetections(detections=dets))
        return results
