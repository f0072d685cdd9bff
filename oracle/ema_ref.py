"""CPU reference of the model-EMA operator (`CudaBackend._ema_update`, same signature).

TEST INFRASTRUCTURE — NOT PRODUCT CODE.  `EMARefBackend` is the per-operator `RefBackend` plus this operator: `-m "not gpu"` tests install it as
`focoos_b200.ops._backend` to run train_step.ModelEMA and the trainer's EMA path on a GPU-less machine, and compare with the reference's golden.
"""
from __future__ import annotations

import ctypes

import torch

from oracle.ops_ref import RefBackend


class EMARefBackend(RefBackend):
    def _ema_update(self, ema, params, chunks, decay, one_minus_decay):
        """fb200_ema_update on host tensors; the chunk table's addresses are read back as the tensors they point to.  fp32: fma(omd, p, fl(ema * d)),
        restated in double (the product is exact there; the sum is rounded twice, which can differ from one rounding only on an exact tie).
        int64: trunc(fp32(ema) * d + fp32(src) * omd) with fp32 products and sum."""
        d, omd = torch.tensor(decay, dtype=torch.float32), torch.tensor(one_minus_decay, dtype=torch.float32)

        def fp32_ema(e, p):
            t = (e * d).double()  # fp32 product, one rounding
            e.copy_((float(omd) * p.double() + t).float())

        if ema.numel():
            fp32_ema(ema, params)
        for src, dst, n, kind in chunks.tolist():
            dt, ct = (torch.int64, ctypes.c_int64) if kind == 1 else (torch.float32, ctypes.c_float)
            s = torch.frombuffer((ct * n).from_address(src), dtype=dt)
            e = torch.frombuffer((ct * n).from_address(dst), dtype=dt)
            if kind == 1:
                e.copy_((e.float() * d + s.float() * omd).long())
            else:
                fp32_ema(e, s)
