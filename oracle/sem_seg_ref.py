"""CPU references of the semantic-evaluation operators (`CudaBackend._mask_sigmoid_upsample_nhwc`, `CudaBackend._sem_seg_confusion`, same signatures).

TEST INFRASTRUCTURE — NOT PRODUCT CODE.  `SemSegRefBackend` is the per-operator `RefBackend` plus these two operators: `-m "not gpu"` tests install it as
`focoos_b200.ops._backend` to run MaskFormerProcessor.eval_postprocess and SemSegEvaluator on a GPU-less machine, and compare with the reference's goldens.
"""
from __future__ import annotations

import torch

from oracle.ops_ref import RefBackend


class SemSegRefBackend(RefBackend):
    def _mask_sigmoid_upsample_nhwc(self, x, Q, out):
        """the probabilities of mask_sigmoid_upsample (sigmoid, then F.interpolate), NHWC, channels Q.. zero; fp32 / fp16 or re-split into the pair"""
        B, H, W, Qo = out.shape
        probs = torch.empty((B, Q, H, W), dtype=torch.float32)
        self.mask_sigmoid_upsample(x, Q, probs)
        v = torch.zeros((B, H, W, Qo), dtype=torch.float32)
        v[..., :Q] = probs.permute(0, 2, 3, 1)
        if hasattr(out, "hi"):
            self._pair_write(out, v)
        else:
            out.copy_(v.to(out.dtype))

    def _sem_seg_confusion(self, scores, labels, C, ignore_label, conf, invalid):
        """the reference's arithmetic (sem_seg_evaluation.py:97-107): torch.argmax over the first C channels, ignore -> C, bincount; labels outside [0, C]
        are counted in `invalid` instead"""
        pred = scores[..., :C].argmax(-1).reshape(-1).long()
        gt = labels.reshape(-1).long()
        gt = torch.where(gt == ignore_label, torch.full_like(gt, C), gt)
        ok = (gt >= 0) & (gt <= C)
        conf += torch.bincount((C + 1) * pred[ok] + gt[ok], minlength=(C + 1) ** 2).reshape(C + 1, C + 1)
        invalid += int((~ok).sum())
