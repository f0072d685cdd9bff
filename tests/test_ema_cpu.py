"""Model EMA (TrainerArgs.ema_enabled) without a GPU: train_step.ModelEMA on the CPU reference operators against the reference EMAUpdater's
golden, its apply / restore, and the trainer's use of it - evaluation on the averaged weights with training left bit-identical, model_final.pth
holding the EMA, ema_enabled=False unchanged, and two data-parallel ranks against one."""
import multiprocessing as mp
import os
import socket
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.nn as nn

from focoos_b200 import ops
from focoos_b200.train_step import FlatAdamW, GradBucketReducer, ModelEMA, TrainStep, get_optimizer_params
from focoos_b200.trainer import SyntheticDetectionDataset, TrainerArgs
from oracle.gen_golden_ema import make_model
from oracle.ema_ref import EMARefBackend

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ema_updates.npz")


@pytest.fixture()
def ref_backend():
    ops._backend = EMARefBackend()
    yield
    ops._backend = None


def _groups(m):
    return get_optimizer_params(m, base_lr=1e-3, weight_decay=0.02)


def _ulps(a: torch.Tensor, b: torch.Tensor) -> int:
    """largest distance in units in the last place between two fp32 tensors (same-sign values)"""
    return int((a.contiguous().view(torch.int32).long() - b.contiguous().view(torch.int32).long()).abs().max()) if a.numel() else 0


def _assert_ema_equal(got: dict, want: dict, what: str):
    assert sorted(got) == sorted(want), what
    for k in want:
        if want[k].dtype == torch.int64:
            assert torch.equal(got[k], want[k]), f"{what}: {k} {got[k]} vs {want[k]}"
        else:
            assert _ulps(got[k], want[k]) <= 1, f"{what}: {k} differs by {_ulps(got[k], want[k])} ulp"


@pytest.mark.parametrize("warmup", [2000, 0])
def test_model_ema_equals_the_reference_updater(ref_backend, warmup):
    z = np.load(GOLDEN)
    m = make_model()
    with torch.no_grad():
        for n, t in m.state_dict(keep_vars=True).items():
            t.copy_(torch.from_numpy(z[f"w{warmup}_ema0_{n}"]))
    opt = FlatAdamW(_groups(m), chunk_elems=16)
    ema = ModelEMA(m, opt, decay=float(z["decay"]), warmup=warmup, chunk_elems=7)  # several chunks per tensor
    assert len(ema.side) == 4 and ema.chunks.shape[0] > len(ema.side), "outside the flat buffer: the frozen conv weight and the 3 BatchNorm buffers"
    for s in range(1, int(z["steps"]) + 1):
        with torch.no_grad():
            for n, t in m.state_dict(keep_vars=True).items():
                t.copy_(torch.from_numpy(z[f"w{warmup}_model{s}_{n}"]))
        ema.update()
        _assert_ema_equal(ema.state_dict(), {n: torch.from_numpy(z[f"w{warmup}_ema{s}_{n}"]) for n in m.state_dict()}, f"update {s}")
    assert ema.updates == int(z["steps"])


def test_applied_restores_the_training_values_through_the_flat_buffer(ref_backend):
    torch.manual_seed(0)
    m = make_model()
    opt = FlatAdamW(_groups(m))
    ema = ModelEMA(m, opt, decay=0.9, warmup=0)
    with torch.no_grad():
        for t in m.state_dict(keep_vars=True).values():
            t.add_(3)
    ema.update()
    train = {k: v.detach().clone() for k, v in m.state_dict().items()}
    averaged = ema.state_dict()
    assert any(not torch.equal(train[k], averaged[k]) for k in train)
    with ema.applied():
        assert all(torch.equal(v, averaged[k]) for k, v in m.state_dict().items())
    assert all(torch.equal(v, train[k]) for k, v in m.state_dict().items()), "restored bit for bit"
    base = opt.flat_params.data_ptr()
    for p, o in zip(opt.params, opt.offsets):
        assert p.data_ptr() == base + 4 * o, "the parameters are still views of the optimiser's flat buffer"
    ema.apply()
    assert all(torch.equal(v, averaged[k]) for k, v in m.state_dict().items())
    with pytest.raises(NotImplementedError, match="float16"):
        m.register_buffer("fp16_buffer", torch.zeros(3, dtype=torch.float16))
        ModelEMA(m, opt)


def test_the_cuda_update_refuses_host_tensors():
    """no CPU fallback: without a reference backend installed, ops.ema_update only launches the kernel"""
    z = torch.zeros(8)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.ema_update(z, z.clone(), torch.zeros((0, 4), dtype=torch.int64), 0.9, 0.1)


# ---- the trainer -----------------------------------------------------------------------------------------------------------------------------
def _train(tmp_path, name, ema, period, record=None, monkeypatch=None):
    from tests.test_api_cpu import _fm
    torch.manual_seed(0)  # the same initial weights (the 5-class head is not in the seeded weights)
    fm = _fm(size=128, num_classes=5)
    data = SyntheticDetectionDataset(n=4, size=128, num_classes=5)
    val = SyntheticDetectionDataset(n=3, size=128, num_classes=5, seed=9)
    if record is not None:  # the model's state when EMAHook.before_train and every after_step see it
        init, update = ModelEMA.__init__, ModelEMA.update

        def rec_init(self, model, *a, **k):
            record.append({k_: v.detach().clone() for k_, v in model.state_dict().items()})
            init(self, model, *a, **k)

        def rec_update(self):
            record.append({k_: v.detach().clone() for k_, v in self.model.state_dict().items()})
            update(self)
        monkeypatch.setattr(ModelEMA, "__init__", rec_init)
        monkeypatch.setattr(ModelEMA, "update", rec_update)
    args = TrainerArgs(run_name=name, output_dir=str(tmp_path), num_gpus=1, max_iters=3, batch_size=2, log_period=1, eval_period=period, ema_enabled=ema,
                       ema_decay=0.9, ema_warmup=2)
    info = fm.train(args, data, data_val=val)
    final = torch.load(tmp_path / name / "model_final.pth", weights_only=True)["model"]
    if record is not None:
        monkeypatch.undo()
    return fm, args, val, info, final


def _reference_ema(states, decay, warmup):
    """EMAUpdater.update (ema.py:112-140) over the recorded states, with torch's own foreach ops"""
    import math
    ema = {k: v.clone() for k, v in states[0].items()}
    for u, st in enumerate(states[1:], 1):
        d = decay * (1 - math.exp(-u / warmup)) if warmup > 0 else decay
        fl = [k for k in ema if ema[k].dtype == torch.float32]
        torch._foreach_mul_([ema[k] for k in fl], d)
        torch._foreach_add_([ema[k] for k in fl], [st[k] for k in fl], alpha=1 - d)
        for k in ema:
            if ema[k].dtype != torch.float32:
                ema[k].copy_(ema[k] * d + st[k] * (1.0 - d))
    return ema


def test_trainer_evaluates_and_saves_the_ema(ref_backend, tmp_path, monkeypatch):
    states = []
    fm_b, args_b, val, info_b, final_b = _train(tmp_path, "ema", True, 0, record=states, monkeypatch=monkeypatch)
    _, _, _, info_a, final_a = _train(tmp_path, "ema_eval", True, 1)
    _, _, _, info_c, final_c = _train(tmp_path, "plain", False, 0)
    assert len(states) == 1 + args_b.max_iters, "one EMA snapshot at the start, one update per iteration"
    _assert_ema_equal(final_b, _reference_ema(states, args_b.ema_decay, args_b.ema_warmup), "model_final.pth")
    assert any(not torch.equal(final_b[k], states[-1][k]) for k in final_b), "the averaged weights differ from the last training weights"
    # periodic evaluation on the EMA leaves training (and so the EMA) bit-identical
    assert all(torch.equal(final_a[k], final_b[k]) for k in final_b)
    evals = [h for h in info_a["training_history"] if "val_metrics" in h]
    assert [h["iter"] for h in evals] == [0, 1, 2] and evals[-1]["val_metrics"] == info_a["val_metrics"] == info_b["val_metrics"]
    losses = [[h for h in i["training_history"] if "val_metrics" not in h] for i in (info_a, info_b, info_c)]
    assert losses[0] == losses[1] == losses[2], "the EMA does not touch the training step"
    # without the EMA, model_final.pth holds the training weights, which the EMA run trained to as well
    assert all(torch.equal(final_c[k], states[-1][k]) for k in final_c)
    assert {k: info_b["train_args"][k] for k in ("ema_enabled", "ema_decay", "ema_warmup")} == {"ema_enabled": True, "ema_decay": 0.9, "ema_warmup": 2}
    assert info_c["train_args"]["ema_enabled"] is False
    # the final metrics are those of the averaged weights, which FocoosModel.train reloaded
    assert all(torch.equal(v, final_b[k]) for k, v in fm_b.model.state_dict().items())
    assert fm_b.eval(args_b, val, save_json=False) == info_b["val_metrics"]


# ---- two data-parallel ranks ------------------------------------------------------------------------------------------------------------------
class _TinyLoss(nn.Module):
    """a frozen parameter and an int64 counter next to the trainable ones; forward(x, y) -> .loss as the model's training forward returns it"""

    def __init__(self):
        super().__init__()
        self.backbone = nn.Linear(7, 13)
        self.head = nn.Linear(13, 3)
        self.frozen = nn.Parameter(torch.randn(13), requires_grad=False)
        self.register_buffer("calls", torch.tensor(5, dtype=torch.int64))

    def forward(self, x, y):
        self.calls += 1
        return SimpleNamespace(loss=((self.head(torch.relu(self.backbone(x)) + self.frozen) - y) ** 2).mean())


def _data(it, rank):
    g = torch.Generator().manual_seed(100 * it + rank)
    return torch.randn((4, 7), generator=g), torch.randn((4, 3), generator=g)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _ddp_worker(rank, world, port, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ops._backend = EMARefBackend()
    torch.manual_seed(0)
    m = _TinyLoss()
    opt = FlatAdamW(get_optimizer_params(m, base_lr=5e-2, weight_decay=0.02), world_size=world, chunk_elems=16)
    red = GradBucketReducer(opt, bucket_bytes=256)
    red.attach_hooks()
    step = TrainStep(m, opt, red, ModelEMA(m, opt, decay=0.8, warmup=3))
    for it in range(4):
        step(*_data(it, rank))
    q.put((rank, {k: v.numpy().copy() for k, v in step.ema.state_dict().items()}))
    dist.destroy_process_group()


def test_two_ranks_keep_the_ema_of_one_rank_on_the_whole_batch():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_ddp_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = {r: {k: torch.from_numpy(a) for k, a in sd.items()} for r, sd in (q.get(timeout=150) for _ in range(world))}
    for p in procs:
        p.join(30)
        assert p.exitcode == 0
    ops._backend = EMARefBackend()
    try:
        torch.manual_seed(0)
        m = _TinyLoss()
        opt = FlatAdamW(get_optimizer_params(m, base_lr=5e-2, weight_decay=0.02), chunk_elems=16)
        step = TrainStep(m, opt, None, ModelEMA(m, opt, decay=0.8, warmup=3))
        for it in range(4):
            parts = [_data(it, r) for r in range(world)]
            step(torch.cat([x for x, _ in parts]), torch.cat([y for _, y in parts]))
        one = step.ema.state_dict()
    finally:
        ops._backend = None
    for rank in range(world):
        for k, v in one.items():
            if v.dtype == torch.int64:
                assert torch.equal(res[rank][k], v), k
            else:
                assert torch.allclose(res[rank][k], v, rtol=2e-6, atol=1e-7), (k, float((res[rank][k] - v).abs().max()))
    assert all(torch.equal(res[0][k], res[1][k]) for k in one), "every rank keeps the same EMA"
