"""tests/golden/ema_updates.npz: the UNMODIFIED reference EMAUpdater (focoos/trainer/solver/ema.py:96-140) over a small seeded model holding
every kind of entry the fai-detr EMA sees - trainable fp32 parameters, a frozen parameter, BatchNorm running statistics and the int64
num_batches_tracked counter (started above 2^24, where its conversion to fp32 rounds) - for STEPS updates with ema_warmup = 2000 and 0.

Before update s the model's values are set to seeded new ones (the counter grows by one per step) and stored as `w<warmup>_model<s>_<name>`;
the EMA state after the update as `w<warmup>_ema<s>_<name>`; the initial EMA (EMAHook.before_train) as `w<warmup>_ema0_<name>`.

    python -m oracle.gen_golden_ema
"""
import os
import sys

import numpy as np
import torch

from oracle import ref_import

STEPS = 5
DECAY = 0.999
WARMUPS = (2000, 0)
COUNTER0 = (1 << 24) + 3


def make_model():
    """the model tests/test_ema_cpu.py builds too: a linear layer, a frozen conv, a BatchNorm"""
    m = torch.nn.Module()
    m.fc = torch.nn.Linear(37, 11)
    m.conv = torch.nn.Conv2d(3, 5, 3)
    m.conv.weight.requires_grad_(False)
    m.bn = torch.nn.BatchNorm2d(5)
    return m


def step_values(m, s):
    """seeded values of every entry before update s (1-based)"""
    g = torch.Generator().manual_seed(1000 + s)
    out = {}
    for n, t in list(m.named_parameters()) + list(m.named_buffers()):
        if t.dtype == torch.int64:
            out[n] = torch.full_like(t, COUNTER0 + s)
        elif "running_var" in n:
            out[n] = 0.5 + torch.rand(t.shape, generator=g)
        else:
            out[n] = torch.randn(t.shape, generator=g) * (0.1 * s)
    return out


def main():
    ref_import.install()
    sys.meta_path.append(ref_import._StubFinder(["iopath"]))  # imported by the hooks module ema.py pulls in, not by the EMA itself
    from focoos.trainer.solver.ema import EMAState, EMAUpdater

    arrays = {}
    for w in WARMUPS:
        torch.manual_seed(0)
        m = make_model()
        with torch.no_grad():
            m.bn.num_batches_tracked.fill_(COUNTER0)
            m.bn.running_mean.normal_()
        state = EMAState()
        upd = EMAUpdater(state, decay=DECAY, warmups=w)
        upd.init_state(m)
        for n, v in state.state.items():
            arrays[f"w{w}_ema0_{n}"] = v.numpy().copy()
        for s in range(1, STEPS + 1):
            vals = step_values(m, s)
            with torch.no_grad():
                for n, t in list(m.named_parameters()) + list(m.named_buffers()):
                    t.copy_(vals[n])
                    arrays[f"w{w}_model{s}_{n}"] = t.numpy().copy()
            upd.update(m)
            for n, v in state.state.items():
                arrays[f"w{w}_ema{s}_{n}"] = v.numpy().copy()
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ema_updates.npz")
    np.savez_compressed(out, steps=STEPS, decay=DECAY, warmups=np.array(WARMUPS), counter0=COUNTER0, **arrays)
    print(len(arrays), "arrays ->", out)


if __name__ == "__main__":
    main()
