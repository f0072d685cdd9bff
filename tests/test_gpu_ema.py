"""Model EMA on the H100: ops.ema_update over the full fai-detr-l-obj365 training state (frozen parameters, BatchNorm buffers and int64 counters
included) equals the reference's torch._foreach_mul_ / _foreach_add_ on the same device bit for bit; a step the loss scaler skipped still
updates it; FocoosModel.train with ema_enabled evaluates and saves the averaged weights, with one EMA launch per step."""
import math
from types import SimpleNamespace

import pytest
import torch
import torch.nn as nn

from focoos_b200 import DETRConfig, FAIDetr, ModelManager, ops
from focoos_b200.train_step import FlatAdamW, ModelEMA, TrainStep, freeze_backbone_at, get_optimizer_params
from focoos_b200.trainer import SyntheticDetectionDataset, TrainerArgs, inference_on_dataset
from focoos_b200.utils.seeded_weights import desaturate_classifiers
from tests.parity_utils import seeded_sd

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = torch.device("cuda", 0)
two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")


def _entries(m):
    return list(m.named_parameters()) + list(m.named_buffers())


def reference_update(state: dict, model: nn.Module, updates: int, decay: float, warmup: int):
    """EMAUpdater.update (focoos/trainer/solver/ema.py:112-140) on the device, on a {name: tensor} copy of the entries"""
    d = decay * (1 - math.exp(-updates / warmup)) if warmup > 0 else decay
    ema_list, vals = [], []
    for name, val in _entries(model):
        if val.dtype in (torch.float32, torch.float16):
            ema_list.append(state[name])
            vals.append(val)
        else:
            state[name].copy_(state[name] * d + val * (1.0 - d))
    torch._foreach_mul_(ema_list, d)
    torch._foreach_add_(ema_list, vals, alpha=1 - d)


def _assert_bitwise(ema: ModelEMA, state: dict, model: nn.Module, what: str):
    for name, t in _entries(model):
        got = ema.entries[id(t)]
        assert torch.equal(got, state[name]), f"{what}: {name} differs by {float((got.double() - state[name].double()).abs().max()):.3e}"


@pytest.mark.parametrize("warmup", [2000, 0])
def test_kernel_equals_torch_foreach_on_the_training_state(warmup):
    m = FAIDetr(DETRConfig(), precision="fp32")
    m.load_state_dict(desaturate_classifiers(seeded_sd(0)), strict=True)
    freeze_backbone_at(m, 1)  # the stem and the first stage are frozen parameters: they average outside the flat buffer
    m.to(DEV).train()
    g = torch.Generator(device=DEV).manual_seed(3)
    with torch.no_grad():
        for n, b in m.named_buffers():
            if b.dtype == torch.int64:
                b.fill_((1 << 24) + 5)  # above 2^24: the conversion to fp32 rounds
            elif "running" in n:
                b.copy_(torch.rand(b.shape, generator=g, device=DEV) + 0.5)
    opt = FlatAdamW(get_optimizer_params(m, 5e-4, 0.02))
    ema = ModelEMA(m, opt, decay=0.999, warmup=warmup)
    kinds = ema.chunks[:, 3].tolist()
    assert kinds.count(ModelEMA.KIND_INT64) == sum(b.dtype == torch.int64 for b in m.buffers()) > 0 and any(not p.requires_grad for p in m.parameters())
    state = {n: t.detach().clone() for n, t in _entries(m)}
    for u in range(1, 6):
        with torch.no_grad():  # what a step changes: every trainable parameter, the running statistics, the counters
            opt.flat_params.add_(torch.randn(opt.flat_params.shape, generator=g, device=DEV), alpha=1e-2)
            for n, b in m.named_buffers():
                if b.dtype == torch.int64:
                    b.add_(1)
                elif "running" in n:
                    b.mul_(0.9).add_(torch.rand(b.shape, generator=g, device=DEV), alpha=0.1)
        ema.update()
        reference_update(state, m, u, 0.999, warmup)
        _assert_bitwise(ema, state, m, f"update {u}")
    assert any(not torch.equal(state[n], t) for n, t in _entries(m))


class _TinyLoss(nn.Module):
    def __init__(self):
        super().__init__()
        self.backbone = nn.Linear(7, 13)
        self.head = nn.Linear(13, 3)
        self.register_buffer("calls", torch.tensor(0, dtype=torch.int64))

    def forward(self, x, y):
        self.calls += 1
        return SimpleNamespace(loss=((self.head(torch.relu(self.backbone(x))) - y) ** 2).mean())


def test_a_step_the_loss_scaler_skipped_still_updates_the_ema():
    torch.manual_seed(0)
    m = _TinyLoss().to(DEV)
    opt = FlatAdamW(get_optimizer_params(m, 5e-2, 0.02))
    ema = ModelEMA(m, opt, decay=0.9, warmup=0)
    step = TrainStep(m, opt, None, ema)
    state = {n: t.detach().clone() for n, t in _entries(m)}
    for it in range(3):
        x, y = torch.randn((4, 7), device=DEV), torch.randn((4, 3), device=DEV)
        if it == 1:
            y[0, 0] = float("inf")
        step(x, y)
        reference_update(state, m, it + 1, 0.9, 0)
        assert opt.stats()["found_inf"] == (1 if it == 1 else 0)
        _assert_bitwise(ema, state, m, f"step {it}")
    assert ema.updates == 3 and opt.stats()["step"] == 2


def test_train_evaluates_and_saves_the_ema(tmp_path, monkeypatch):
    fm = ModelManager.get("fai-detr-l-obj365")
    data = SyntheticDetectionDataset(n=4, size=256, num_classes=365)
    val = SyntheticDetectionDataset(n=4, size=256, num_classes=365, seed=9)
    states, calls = [], []
    init, update = ModelEMA.__init__, ModelEMA.update

    def rec_init(self, model, *a, **k):
        states.append({n: t.detach().clone() for n, t in _entries(model)})
        init(self, model, *a, **k)

    def rec_update(self):
        states.append({n: t.detach().clone() for n, t in _entries(self.model)})
        n0 = len(ops._trace)
        update(self)
        calls.append([name for name, *_ in ops._trace[n0:]])
    monkeypatch.setattr(ModelEMA, "__init__", rec_init)
    monkeypatch.setattr(ModelEMA, "update", rec_update)
    ops.enable_trace(True)
    try:
        args = TrainerArgs(run_name="ema", output_dir=str(tmp_path), num_gpus=1, max_iters=3, batch_size=2, log_period=1, eval_period=1, ema_enabled=True,
                           ema_decay=0.99, ema_warmup=2)
        info = fm.train(args, data, data_val=val)
    finally:
        ops.enable_trace(False)
    monkeypatch.undo()
    assert calls == [["fb200_ema_update"]] * args.max_iters, "one launch per step"
    # the reference's arithmetic on the device over the weights each update saw
    live = SimpleNamespace(named_parameters=lambda: [], named_buffers=lambda: [])
    state = {n: v.clone() for n, v in states[0].items()}
    for u, st in enumerate(states[1:], 1):
        live.named_parameters = lambda st=st: list(st.items())
        reference_update(state, live, u, args.ema_decay, args.ema_warmup)
    final = torch.load(tmp_path / "ema" / "model_final.pth", weights_only=True)["model"]
    for k, v in final.items():
        assert torch.equal(v, state[k].cpu()), f"model_final.pth: {k}"
    assert any(not torch.equal(final[k], states[-1][k].cpu()) for k in final)
    for k, v in fm.model.state_dict().items():
        assert torch.equal(v.cpu(), final[k]), f"the reloaded model: {k}"
    assert info["train_args"]["ema_enabled"] is True and info["weights_uri"].endswith("model_final.pth")
    evals = [h for h in info["training_history"] if "val_metrics" in h]
    assert [h["iter"] for h in evals] == [0, 1, 2]
    assert inference_on_dataset(fm, val, batch_size=2) == info["val_metrics"], "the final metrics are those of the averaged weights"


@two_gpus
def test_two_gpu_training_saves_the_ema(tmp_path):
    fm = ModelManager.get("fai-detr-l-obj365")
    data = SyntheticDetectionDataset(n=8, size=256, num_classes=365)
    val = SyntheticDetectionDataset(n=4, size=256, num_classes=365, seed=9)
    args = TrainerArgs(run_name="t", output_dir=str(tmp_path), num_gpus=2, max_iters=2, batch_size=2, log_period=1, master_port=29573, ema_enabled=True,
                       ema_decay=0.9, ema_warmup=0)
    info = fm.train(args, data, data_val=val)
    assert info["val_metrics"]["num_images"] == 4
    assert inference_on_dataset(fm, val, batch_size=2) == info["val_metrics"], "rank 0's EMA, evaluated on one GPU over all of data_val"
