"""CPU reference of the box-AP matching operator (`CudaBackend._box_ap_match`, same signature).

TEST INFRASTRUCTURE — NOT PRODUCT CODE.  `BoxAPRefBackend` is the per-operator `RefBackend` plus this operator: `-m "not gpu"` tests install it as
`focoos_b200.ops._backend` to run DeviceBoxAPEvaluator's host logic on a GPU-less machine.  The matching is BoxAPEvaluator.evaluate's loop restated per
(image, class): detections in stable descending-score order, `cand = where(used, -1, iou)`, the first argmax, a hit iff `cand[j] >= t`.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.ops_ref import RefBackend


def iou_row(d: np.ndarray, g: np.ndarray) -> np.ndarray:
    """IoU of one box d [4] against g [n,4] with the arithmetic of trainer._iou_matrix (numpy promotion: fp32 x fp32 -> fp32, fp32 x fp64 -> fp64)"""
    a, b = d[None], g
    lt = np.maximum(a[:, None, :2], b[None, :, :2])
    rb = np.minimum(a[:, None, 2:], b[None, :, 2:])
    inter = np.clip(rb - lt, 0, None).prod(-1)
    aa = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    ab = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    return (inter / np.maximum(aa[:, None] + ab[None, :] - inter, 1e-12))[0]


def match_image(scores, classes, boxes, gt_boxes, gt_classes, thresholds, C) -> np.ndarray:
    """tp bits [n] of one image's detections (numpy arrays)"""
    bits = np.zeros(len(scores), dtype=np.int64)
    for c in range(C):
        gi = np.nonzero(gt_classes == c)[0]
        di = [i for i in sorted(range(len(scores)), key=lambda i: -float(scores[i])) if classes[i] == c]
        if not len(gi) or not di:
            continue
        g = gt_boxes[gi]
        ious = [iou_row(boxes[i], g) for i in di]
        for ti, t in enumerate(thresholds):
            used = np.zeros(len(gi), dtype=bool)
            for k, i in enumerate(di):
                cand = np.where(used, -1.0, ious[k])
                j = int(cand.argmax())
                if cand[j] >= t:
                    used[j] = True
                    bits[i] |= 1 << ti
    return bits


class BoxAPRefBackend(RefBackend):
    def _box_ap_match(self, scores, classes, boxes, counts, gt_boxes, gt_classes, gt_offsets, gt_offsets_host, thresholds_host, C, tp, gt_count):
        B, K = scores.shape
        off = gt_offsets_host.numpy()
        thr = thresholds_host.numpy()
        s, cl, bx, n = scores.numpy(), classes.numpy(), boxes.numpy(), counts.numpy()
        gb, gc = gt_boxes.numpy(), gt_classes.numpy()
        out = np.zeros((B, K), dtype=np.int64)
        for b in range(B):
            k = int(min(max(n[b], 0), K))
            out[b, :k] = match_image(s[b, :k], cl[b, :k], bx[b, :k], gb[off[b]:off[b + 1]], gc[off[b]:off[b + 1]], thr, C)
        tp.copy_(torch.from_numpy(out.astype(np.uint16).view(np.int16)))
        ok = (gc >= 0) & (gc < C)
        gt_count += torch.from_numpy(np.bincount(gc[ok], minlength=C).astype(np.int64))
