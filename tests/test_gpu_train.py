"""-m gpu: one full fine-tune iteration of FAIDetr on the GPU (training-mode forward, criterion, backward through the hand-written
kernels, clipping, AdamW) against the golden of the unmodified reference's training step (oracle/gen_golden_train.py)."""
import numpy as np
import pytest
import torch

from focoos_b200 import DETRConfig, FAIDetr, ops
from focoos_b200.criterion import DETRTargets
from focoos_b200.train_step import FlatAdamW, TrainStep, get_optimizer_params
from oracle.gen_golden import synth_images
from oracle.gen_golden_train import synth_targets
from focoos_b200.utils.seeded_weights import desaturate_classifiers
from tests.parity_utils import load_golden, seeded_sd
from tests.test_train_graph_cpu import check_against_golden, check_amp_gradients, run_step

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = torch.device("cuda", 0)


@pytest.mark.parametrize("precision", ["fp32", "fp32_tc"])
def test_train_step_gradients_match_reference(precision):
    """fp32 (SIMT) reproduces the reference's discrete choices (top-k queries, 7 Hungarian assignments) and is compared end to end.
    The seeded, untrained decoder emits many near-duplicate queries, so the split-precision tensor-core mode (errors ~1e-5 instead of ~1e-6)
    can flip an assignment between two near-tied queries; it is compared with the reference's assignments teacher-forced, which keeps the
    comparison about the forward/backward kernels."""
    g = load_golden("detr_l_train_b2_192")
    m = FAIDetr(DETRConfig(), precision=precision)
    m.load_state_dict(desaturate_classifiers(seeded_sd(0)), strict=True)
    m.to(DEV)
    if precision == "fp32_tc":
        m.criterion().forced_match = torch.from_numpy(g["match_q"])
        m.train_graph().forced_topk = torch.from_numpy(g["topk_ind"])  # assignments index the ORDERED query list
    n0 = ops.launch_count()
    losses = run_step(m, g, DEV)
    torch.cuda.synchronize()
    got = m.criterion().last_match.cpu().numpy()
    same = int((got == g["match_q"]).sum())
    print(f"[{precision}] assignments equal to the reference: {same}/{got.size}")
    if precision == "fp32":
        assert same == got.size, "fp32 mode must reproduce every Hungarian assignment of the reference"
        assert sorted(m.train_graph().last_topk[0].tolist()) == sorted(g["topk_ind"][0].tolist()), "and the same query set"
    worst = check_against_golden(m, losses, g, loss_rtol=5e-4, grad_rtol=4e-3)
    print(f"[{precision}] worst gradient-norm error / tolerance: {worst}; kernels launched: {ops.launch_count() - n0}")


def test_train_step_amp_precision():
    """train_precision="amp" (TrainerArgs.amp_enabled, the reference's torch.autocast(fp16) arithmetic: one fp16 tensor-core product per conv/linear, fp32
    accumulation and storage) against the reference's fp32 training-step golden, assignments teacher-forced: losses within 2e-2 relative and gradient norms within 2e-2 (median) / 8e-2 (p90) - the fp16 operand-rounding class, not the fp32 bars of the other two modes."""
    g = load_golden("detr_l_train_b2_192")
    m = FAIDetr(DETRConfig(), precision="fp32_tc")
    m.train_precision = "amp"
    m.load_state_dict(desaturate_classifiers(seeded_sd(0)), strict=True)
    m.to(DEV)
    m.criterion().forced_match = torch.from_numpy(g["match_q"])
    m.train_graph().forced_topk = torch.from_numpy(g["topk_ind"])
    assert m.train_graph().prec == "amp"
    losses = run_step(m, g, DEV)
    torch.cuda.synchronize()
    keys = g["loss_keys"].tolist()
    got = np.array([float(losses[k].detach()) for k in keys])
    np.testing.assert_allclose(got, g["loss_values"], rtol=2e-2, atol=1e-4)
    params = dict(m.named_parameters())
    total = float(np.sqrt((g["grad_norm"] ** 2).sum()))
    errs = check_amp_gradients(params, g, total)
    print(f"[amp] losses {got} vs {g['loss_values']}; gradient-norm errors: median {errs[len(errs) // 2]:.3e}, p90 {errs[int(0.9 * len(errs))]:.3e}, max {errs[-1]:.3e}")


def test_full_iteration_on_gpu():
    g = load_golden("detr_l_train_b2_192")
    m = FAIDetr(DETRConfig(), precision="fp32")
    m.load_state_dict(desaturate_classifiers(seeded_sd(0)), strict=True)
    m.to(DEV).train()
    opt = FlatAdamW(get_optimizer_params(m, base_lr=5e-4, weight_decay=0.02, weight_decay_norm=0.0, backbone_multiplier=0.1), clip_gradients=0.1, amp=True)
    opt.track_unused_parameters()
    names = g["param_names"].tolist()
    before = opt.flat_params.clone()
    size, B = int(g["size"][0]), int(g["size"][1])
    x = torch.from_numpy(np.stack(synth_images(5, [(size, size)] * B))).permute(0, 3, 1, 2).float().to(DEV)
    targets = [DETRTargets(labels=t[0].to(DEV), boxes=t[1].to(DEV)) for t in synth_targets(6, B, m.config.num_classes)]
    step = TrainStep(m, opt)
    loss_dict = step(x, targets)
    torch.cuda.synchronize()
    st = opt.stats()
    assert st["found_inf"] == 0 and st["step"] == 1
    assert abs(st["grad_norm"] - float(g["total_grad_norm"])) <= 2e-3 * float(g["total_grad_norm"]), st  # loss scaling (2^10) must cancel exactly
    total = float(g["total_grad_norm"])
    delta = (opt.flat_params - before).cpu()
    for i, (n, has, dn, gn) in enumerate(zip(names, g["grad_has"], g["step_delta_norm"], g["grad_norm"])):
        o, cnt = opt.offsets[i], opt.params[i].numel()
        mine = float(delta[o:o + cnt].norm())
        if not has:
            assert mine == 0.0, n
        elif gn >= 1e-5 * total:
            assert abs(mine - dn) <= 3e-2 * dn + 1e-9, f"{n}: |delta| {mine:.4e} vs reference {dn:.4e}"
    # a second iteration runs (running statistics / moments / step counter advance) and the loss is finite
    l2 = step(x, targets)
    assert all(torch.isfinite(v).all() for v in l2.values()) and opt.stats()["step"] == 2
    # back to eval: the inference engine is re-packed from the updated parameters
    m.eval()
    out = m(x[:, :, :, :].contiguous())
    assert out.logits.shape[:2] == (B, 300) and torch.isfinite(out.logits).all()
