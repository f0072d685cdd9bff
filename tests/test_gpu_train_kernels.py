"""The fine-tune step's criterion (csrc/criterion.cu), optimiser step (csrc/optim.cu) and pool / resize backward kernels
(csrc/bwd_conv_norm.cu) against float64 references, at the fai-detr-l fine-tune shapes (bs=16, 640x640) and at the ties and borders where
these kernels apply special rules.

- Criterion: `detr_match_cost` against oracle/criterion_oracle.match_cost run on float64 tensors; the device assignment against scipy's
  optimum on the same fp32 costs (ties included: duplicated targets and queries); VFL / L1 / GIoU losses and d/dlogits, d/dboxes against
  fp64 autograd of oracle/criterion_oracle.layer_losses, with the matching forced onto identical, touching, disjoint, nested and
  out-of-frame box pairs and onto saturated logits.  Box corners are multiples of 1/64 (1/256 at full shape): x0 = cx - w/2 is then exact
  in fp32 and fp64 alike, so a tie in one precision is a tie in the other.
- Optimiser: a float64 replay of the reference's torch sequence (GradScaler.unscale_, clip_grad_norm_ twice, AdamW with per-tensor
  lr / weight decay, GradScaler.update; the sequence of oracle/optim_oracle.py) over the real 501-tensor fai-detr-l flat buffer plus
  synthetic chunk / padding edge tensors, with world_size = 8, unused tensors, a NaN, an inf and a loss-scale growth.
- Pool / resize backward: F.max_pool2d(3, 2, 1), F.avg_pool2d(2, 2, 0, ceil_mode=True) and F.interpolate(bilinear, align_corners=False)
  autograd on float64 NCHW CPU tensors.  Upstream gradients are small integers, so wherever the forward weights are dyadic (max-pool
  routing, average pool, 2x resizes) every sum is exact in fp32 and the kernels must match bit for bit: a gradient routed to the wrong
  tied input is an error of order 1.

Every tolerance is stated relative to the scale of its quantity, in units of U = 2^-24 (the fp32 unit roundoff), with its derivation
beside it.  The unmarked tests need no GPU: they check the fp64 references themselves."""
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F
from scipy.optimize import linear_sum_assignment

from focoos_b200 import DETRConfig, FAIDetr, ops
from focoos_b200 import autograd_ops as A
from focoos_b200 import criterion as K
from focoos_b200.train_step import FlatAdamW, get_optimizer_params
from oracle import criterion_oracle as CO
from oracle.optim_oracle import ReferenceStepper

pytestmark = pytest.mark.timeout(900)
gpu = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64
U = 2.0 ** -24  # fp32 unit roundoff


@pytest.fixture
def be():
    """the CUDA backend (never the CPU reference backend some host-graph tests install)"""
    b = ops._be()
    assert isinstance(b, ops.CudaBackend)
    return b


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# =====================================================================================================================================
# 1. Criterion
# =====================================================================================================================================
COST_W = (2.0, 5.0, 2.0)   # matcher: class, bbox, giou (fai_detr config)
COST_ALPHA = 0.25
LOSS_W = (1.0, 5.0, 2.0)   # loss_vfl, loss_bbox, loss_giou
VFL_ALPHA = 0.75
VFL_THREADS = 132 * 256    # loss_vfl_kernel: kNumSMs blocks of 256 threads per layer
L_FT, B_FT, Q_FT = 7, 16, 300   # six decoder layers + the encoder top-k; bs=16 per GPU; 300 queries
TIE_IMAGE = 4


def _grid_boxes(g, n, grid=256):
    """n boxes (cx, cy, w, h) float64 with cx, cy multiples of 1/grid and w, h even multiples: every corner is a multiple of 1/grid"""
    c = torch.randint(16, grid - 16, (n, 2), generator=g)
    wh = 2 * torch.randint(3, grid // 4, (n, 2), generator=g)
    return torch.cat([c, wh], 1).to(F64) / grid


def _full_case(C, seed):
    """L=7, B=16, Q=300 predictions and targets with per-image counts 0, 1, 100, 300 (square assignment), a tie image and 2..40 elsewhere.
    Every target has a planted near-hit query.  The tie image holds three identical targets and three identical queries sitting on them."""
    g = _gen(seed)
    counts = [0, 1, 100, 300] + torch.randint(2, 41, (B_FT - 4,), generator=g).tolist()
    counts[TIE_IMAGE] = max(counts[TIE_IMAGE], 6)
    targets = [(torch.randint(0, C, (n,), generator=g), _grid_boxes(g, n)) for n in counts]
    lab, tb = targets[TIE_IMAGE]
    lab[1:3], tb[1:3] = lab[0], tb[0]
    logits = torch.randn((L_FT, B_FT, Q_FT, C), generator=g, dtype=F64) * 2 - 3
    boxes = _grid_boxes(g, L_FT * B_FT * Q_FT).reshape(L_FT, B_FT, Q_FT, 4)
    for l in range(L_FT):
        for b, (lab, tb) in enumerate(targets):
            q = torch.randperm(Q_FT, generator=g)[:len(lab)]
            boxes[l, b, q] = tb + torch.randint(-2, 3, (len(lab), 4), generator=g).to(F64) * (2 / 256)
            logits[l, b, q, lab] += 4
        lab, tb = targets[TIE_IMAGE]
        boxes[l, TIE_IMAGE, 10] = tb[0]
        logits[l, TIE_IMAGE, 10, lab[0]] += 6
        boxes[l, TIE_IMAGE, 11:13] = boxes[l, TIE_IMAGE, 10]
        logits[l, TIE_IMAGE, 11:13] = logits[l, TIE_IMAGE, 10]
    return logits.float().to(F64), boxes, targets   # the logits the device receives, exactly


def _dev_targets(targets):
    return [K.DETRTargets(labels=t[0].to(DEV), boxes=t[1].to(device=DEV, dtype=torch.float32)) for t in targets]


def _criterion(gamma=2.0):
    m = K.BoxHungarianMatcher(cost_class=COST_W[0], cost_bbox=COST_W[1], cost_giou=COST_W[2], use_focal_loss=True, alpha=COST_ALPHA, gamma=2.0)
    return K.SetCriterion(num_classes=80, matcher=m, weight_dict={"loss_vfl": LOSS_W[0], "loss_bbox": LOSS_W[1], "loss_giou": LOSS_W[2]},
                          losses=["vfl", "boxes"], focal_alpha=VFL_ALPHA, focal_gamma=gamma)


def _cost_tol(logits, boxes, lab, tb, gamma):
    """per-element bound [Q, n] on |fp32 cost - fp64 cost| for one image.  The fp32 sigmoid carries three roundings (expf, 1 + e, 1 / .), so
    |dp| <= 4U p.  -log(1 - p + 1e-8) turns that absolute error into 4U p / (1 - p + 1e-8) and (1 - p)^gamma into a relative gamma 4U p / (1 - p);
    with the 2x margin these are the two singular terms.  Every other operation (box corners are exact, the GIoU division and the sums round a
    few times) stays within 16U of the sum S of the absolute values of the cost's terms (|GIoU| <= 1, plus 1 for its parts)."""
    p = torch.sigmoid(logits)[:, lab]
    neg = (1 - COST_ALPHA) * p ** gamma * -(1 - p + 1e-8).log()
    pos = COST_ALPHA * (1 - p) ** gamma * -(p + 1e-8).log()
    l1 = (boxes[:, None, :] - tb[None, :, :]).abs().sum(-1)
    S = COST_W[1] * l1 + COST_W[0] * (pos + neg) + 3 * COST_W[2]
    sing = (1 - COST_ALPHA) * p ** gamma * p / (1 - p + 1e-8) + COST_ALPHA * gamma * p * (1 - p) ** (gamma - 1) * -(p + 1e-8).log()
    return 16 * U * S + COST_W[0] * 8 * U * sing


def _pairs(bx, targets, idx):
    bi = torch.cat([torch.full_like(q, b) for b, (q, _) in enumerate(idx)])
    qi = torch.cat([q for q, _ in idx])
    tgt = torch.cat([t[1][j] for t, (_, j) in zip(targets, idx)], 0)
    lab = torch.cat([t[0][j] for t, (_, j) in zip(targets, idx)], 0)
    return bi, qi, bx[bi, qi], tgt, lab


def _loss_reference(lg, bx, targets, idx, nb, gamma):
    """one layer: fp64 (losses [3], dlogits, dboxes) by autograd of oracle/criterion_oracle.layer_losses, and the per-element tolerances"""
    lg, bx = lg.clone().requires_grad_(True), bx.clone().requires_grad_(True)
    losses = torch.stack(CO.layer_losses(lg, bx, targets, idx, nb, alpha=VFL_ALPHA, gamma=gamma, weights=LOSS_W))
    losses.sum().backward()
    dlg, dbx = lg.grad, bx.grad
    lg, bx = lg.detach(), bx.detach()
    B, Q, C = lg.shape
    bi, qi, src, tgt, lab = _pairs(bx, targets, idx)
    a, t = CO.cxcywh_to_xyxy(src), CO.cxcywh_to_xyxy(tgt)
    iou, uni = CO.pair_iou(a, t)
    giou = CO.pair_giou(a, t)
    ts = torch.zeros((B, Q, C), dtype=F64)
    onehot = torch.zeros((B, Q, C), dtype=F64)
    ts[bi, qi, lab] = iou
    onehot[bi, qi, lab] = 1.0
    p = torch.sigmoid(lg)
    w = VFL_ALPHA * p ** gamma * (1 - onehot) + ts
    bce = F.binary_cross_entropy_with_logits(lg, ts, reduction="none").abs()
    T = len(qi)
    # VFL sum: per-thread fp32 sums of B*Q*C / VFL_THREADS terms, a 256-way tree (8 levels) and 132 serial block partials, each adding <= U of the
    # running sum; each term w * bce carries <= 8U of w * (|x| + 1) from the cancellation inside (1 - ts) x - min(x, 0) + log1p(exp(-|x|))
    k_vfl = B * Q * C / VFL_THREADS + 8 + 132 + 8
    tol_vfl = LOSS_W[0] / nb * U * (k_vfl * (w * bce).sum() + 8 * (w * (lg.abs() + 1)).sum())
    # L1 / GIoU sums: per-thread sums of T / 256 terms and a 256-way tree; each 1 - GIoU term carries <= 16U (exact corners, ~4 roundings)
    k_box = T / 256 + 8 + 8
    tol_l1 = LOSS_W[1] / nb * U * k_box * (src - tgt).abs().sum()
    tol_giou = LOSS_W[2] / nb * U * (k_box * (1 - giou).abs().sum() + 16 * T)
    # dlogits = w (p - ts) / nb: p carries 4U p absolute (expf within 2 ulp, 1 + e, 1 / .), w = alpha p^gamma + ts about 14U relative
    # (gamma 4U, pow or square, two products), the scaling 2U: <= 20U w (p + ts), taken as 32U
    tol_dl = 32 * U * w * (p + ts) * LOSS_W[0] / nb + 1e-37
    # dboxes: every intermediate of the GIoU reverse pass is bounded by M = dg (2/U + I/U^2 + (U+eps)/Ae^2 + 1/Ae) x (sum of the box extents);
    # each is formed by <= 8 fp32 roundings from exact corners, so 64U M bounds the sum; the L1 part is sign(d) w / nb, one rounding
    iw = (torch.min(a[:, 2], t[:, 2]) - torch.max(a[:, 0], t[:, 0])).clamp(min=0)
    ih = (torch.min(a[:, 3], t[:, 3]) - torch.max(a[:, 1], t[:, 1])).clamp(min=0)
    ew = torch.max(a[:, 2], t[:, 2]) - torch.min(a[:, 0], t[:, 0])
    eh = torch.max(a[:, 3], t[:, 3]) - torch.min(a[:, 1], t[:, 1])
    I, Ae = iw * ih, ew * eh + 1e-5
    dg = LOSS_W[2] / nb
    M = dg * (2 / uni + I / uni ** 2 + (uni + 1e-5) / Ae ** 2 + 1 / Ae) * (iw + ih + ew + eh + (a[:, 2] - a[:, 0]) + (a[:, 3] - a[:, 1]))
    tol_db = torch.zeros((B, Q, 4), dtype=F64)
    tol_db[bi, qi] = (64 * U * M + 4 * U * LOSS_W[1] / nb)[:, None]
    return losses.detach(), dlg, dbx, torch.stack([tol_vfl, tol_l1, tol_giou]), tol_dl, tol_db


def _assert_within(got, ref, tol, what):
    err = (got.to(F64) - ref).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = tuple(int(v) for v in torch.nonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} elements out of bounds, first at {i}: got {float(got[i]):.9g}, fp64 {float(ref[i]):.9g}, "
                             f"tol {float(tol[i]):.3g} (max err/tol {float((err / tol.clamp(min=1e-300)).max()):.3g})")


def _check_layer_losses(table, dlogits, dboxes, logits, boxes, targets, idx, nb, gamma, what):
    """table [L,3], dlogits [L,B,Q,C], dboxes [L,B,Q,4] from the device against fp64 autograd, layer by layer"""
    for l in range(logits.shape[0]):
        ref, dl, db, tl, tdl, tdb = _loss_reference(logits[l], boxes[l], targets, idx[l], nb, gamma)
        _assert_within(table[l], ref, tl, f"{what} layer {l} losses (vfl, bbox, giou)")
        _assert_within(dlogits[l], dl, tdl, f"{what} layer {l} dlogits")
        _assert_within(dboxes[l], db, tdb, f"{what} layer {l} dboxes")


def _run_criterion(crit, logits, boxes, targets, nb=None):
    """the device criterion over all layers: (loss table [L,3], dlogits, dboxes) on the CPU"""
    L = logits.shape[0]
    lg = logits.to(device=DEV, dtype=torch.float32).requires_grad_(True)
    bx = boxes.to(device=DEV, dtype=torch.float32).requires_grad_(True)
    out = {"pred_logits": lg[0], "pred_boxes": bx[0], "aux_outputs": [{"pred_logits": lg[i], "pred_boxes": bx[i]} for i in range(1, L)]}
    crit.num_boxes_hint = nb
    losses = crit(out, _dev_targets(targets))
    table = torch.stack([torch.stack([losses["loss_vfl" + s], losses["loss_bbox" + s], losses["loss_giou" + s]])
                         for s in [""] + [f"_{i}" for i in range(L - 1)]])
    table.sum().backward()
    return table.detach().cpu(), lg.grad.cpu(), bx.grad.cpu()


@gpu
@pytest.mark.parametrize("C", [80, 365])
def test_criterion_cost_assignment_losses_at_finetune_shapes(be, C):
    """L=7, B=16, Q=300: the cost of every (layer, image) block against fp64, the device assignment's total cost against scipy's optimum on
    the same fp32 costs (and the assignment itself wherever the optimum is unique), then the losses and gradients of the whole criterion."""
    logits, boxes, targets = _full_case(C, seed=C)
    mq, cost = K.match(logits.float().to(DEV), boxes.float().to(DEV), _dev_targets(targets), *COST_W, COST_ALPHA, 2.0, return_cost=True)
    mq, cost = mq.cpu(), cost.cpu().to(F64)
    idx = [[] for _ in range(L_FT)]
    o = 0
    for b, (lab, tb) in enumerate(targets):
        n = len(lab)
        for l in range(L_FT):
            if n == 0:
                idx[l].append((torch.zeros(0, dtype=torch.int64), torch.zeros(0, dtype=torch.int64)))
                continue
            ref = CO.match_cost(logits[l, b], boxes[l, b], lab, tb, *COST_W, alpha=COST_ALPHA, gamma=2.0).T
            _assert_within(cost[l, o:o + n], ref, _cost_tol(logits[l, b], boxes[l, b], lab, tb, 2.0).T, f"cost layer {l} image {b}")
            blk = cost[l, o:o + n].numpy()
            r, c = linear_sum_assignment(blk)
            got = mq[l, o:o + n].numpy()
            assert got.min() >= 0 and got.max() < Q_FT and len(set(got.tolist())) == n, f"layer {l} image {b}: not a valid assignment"
            opt, dev = blk[r, c].sum(), blk[np.arange(n), got].sum()
            # the two totals are double sums of the same fp32 entries in different orders: they differ by <= n 2^-52 sum|c| unless the assignments differ
            assert abs(dev - opt) <= n * 2.0 ** -52 * np.abs(blk[r, c]).sum(), f"layer {l} image {b}: device total {dev!r} vs optimum {opt!r}"
            if b != TIE_IMAGE:  # continuous random costs: the optimum is unique
                assert np.array_equal(got, c), f"layer {l} image {b}: device assignment differs from scipy's"
            idx[l].append((torch.as_tensor(c, dtype=torch.int64), torch.as_tensor(r, dtype=torch.int64)))
        o += n
    crit = _criterion()
    table, dlg, dbx = _run_criterion(crit, logits, boxes, targets)
    assert torch.equal(crit.last_match.cpu(), mq), "the criterion's own matching differs from a second run of the matcher"
    nb = float(sum(len(t[0]) for t in targets))
    # the tie image: the device may pair the three identical targets with the three identical queries in another order than scipy does;
    # the losses and gradients are invariant under that exchange
    _check_layer_losses(table, dlg, dbx, logits, boxes, targets, idx, nb, 2.0, f"C={C}")


@gpu
def test_match_cost_gamma_powf_branch(be):
    """gamma = 1.5 runs the powf branch of the cost kernel (the shipped configs use 2)"""
    logits, boxes, targets = _full_case(80, seed=3)
    logits, boxes = logits[:2], boxes[:2]
    _, cost = K.match(logits.float().to(DEV), boxes.float().to(DEV), _dev_targets(targets), *COST_W, COST_ALPHA, 1.5, return_cost=True)
    cost = cost.cpu().to(F64)
    o = 0
    for b, (lab, tb) in enumerate(targets):
        n = len(lab)
        for l in range(2):
            if n:
                ref = CO.match_cost(logits[l, b], boxes[l, b], lab, tb, *COST_W, alpha=COST_ALPHA, gamma=1.5).T
                _assert_within(cost[l, o:o + n], ref, _cost_tol(logits[l, b], boxes[l, b], lab, tb, 1.5).T, f"gamma=1.5 cost layer {l} image {b}")
        o += n


# ---- forced matching onto the edge cases of the box losses -----------------------------------------------------------------------------------------
EDGE_KINDS = ("same", "touch_x", "touch_y", "disjoint", "nested", "nested_shared_edges", "contains_shared_edge", "shared_x1", "outside")


def _edge_pair(kind, g, t=None):
    """(pred, target, target corners) with pred in relation `kind` to the target (corners t, drawn when None); boxes are cxcywh float64 built
    from integer corners in units of 1/64"""
    def r(lo, hi):
        return int(torch.randint(lo, hi, (1,), generator=g))

    if t is None:
        tx0, ty0 = r(8, 28), r(8, 28)
        t = (tx0, ty0, tx0 + r(8, 24), ty0 + r(8, 24))
    tx0, ty0, tx1, ty1 = t
    if kind == "same":               # every max and min ties, GIoU = 1
        p = t
    elif kind == "touch_x":          # pred.x1 == tgt.x0: intersection width exactly 0, heights overlap
        y0 = ty0 + r(-4, 4)
        p = (tx0 - r(4, 12), y0, tx0, y0 + r(6, 16))
    elif kind == "touch_y":
        x0 = tx0 + r(-4, 4)
        p = (x0, ty1, x0 + r(6, 16), ty1 + r(4, 12))
    elif kind == "disjoint":
        x0, y0 = tx1 + r(1, 6), ty0 + r(-12, 12)
        p = (x0, y0, x0 + r(4, 12), y0 + r(4, 12))
    elif kind == "nested":           # pred strictly inside the target
        p = (tx0 + 2, ty0 + 2, tx1 - 2, ty1 - 3)
    elif kind == "nested_shared_edges":   # inside, sharing the left and top edges (min and max tie on x0 and y0)
        p = (tx0, ty0, tx1 - r(1, 6), ty1 - r(1, 6))
    elif kind == "contains_shared_edge":  # pred around the target, sharing its right edge
        p = (tx0 - r(1, 6), ty0 - r(1, 6), tx1, ty1 + r(1, 6))
    elif kind == "shared_x1":        # partial overlap with one equal coordinate
        p = (tx0 + r(1, 6), ty0 + r(1, 6), tx1, ty1 + r(1, 6))
    elif kind == "outside":          # pred reaching outside [0, 1] on three sides
        p = (-r(1, 16), ty0 - r(1, 6), 64 + r(1, 16), 64 + r(1, 16))
    else:
        raise ValueError(kind)

    def cxcywh(c):
        x0, y0, x1, y1 = c
        return torch.tensor([(x0 + x1) / 128, (y0 + y1) / 128, (x1 - x0) / 64, (y1 - y0) / 64], dtype=F64)

    return cxcywh(p), cxcywh(t), t


def _forced_case(seed, L=2, B=4, Q=300, C=80, per_kind=2):
    g = _gen(seed)
    logits = torch.randn((L, B, Q, C), generator=g, dtype=F64) * 2 - 3
    boxes = _grid_boxes(g, L * B * Q, grid=64).reshape(L, B, Q, 4)
    n = per_kind * len(EDGE_KINDS)
    targets, forced = [], [[] for _ in range(L)]
    for b in range(B):
        kinds = [k for k in EDGE_KINDS for _ in range(per_kind)]
        pairs = [_edge_pair(k, g) for k in kinds]
        lab = torch.randint(0, C, (n,), generator=g)
        targets.append((lab, torch.stack([t for _, t, _ in pairs])))
        for l in range(L):
            q = torch.randperm(Q, generator=g)[:n]
            if l:   # the other layers place new pred boxes in the same relations to the same targets
                pairs = [_edge_pair(k, g, tc) for k, (_, _, tc) in zip(kinds, pairs)]
            boxes[l, b, q] = torch.stack([p for p, _, _ in pairs])
            # saturated logits on the matched class: +30 (p rounds to 1 in fp32), -30 (BCE through log1pf), the rest unchanged
            sat = torch.tensor([30.0, -30.0, 0.0])[torch.arange(n) % 3]
            logits[l, b, q, lab] = torch.where(sat != 0, sat, logits[l, b, q, lab])
            # whole rows of unmatched queries at +-30
            free = torch.ones(Q, dtype=torch.bool)
            free[q] = False
            rows = torch.nonzero(free)[:6, 0]
            logits[l, b, rows] = torch.tensor([30.0, -30.0] * 3, dtype=F64)[:, None]
            forced[l].append(q)
    return logits.float().to(F64), boxes, targets, torch.stack([torch.cat(f) for f in forced])


@gpu
@pytest.mark.parametrize("gamma", [2.0, 1.5])
def test_criterion_forced_matching_edge_boxes(be, gamma):
    """matching forced onto identical / touching / disjoint / nested / out-of-frame pairs and saturated logits, with a fractional num_boxes
    (the rank average of 71 boxes over 8 ranks); gamma = 1.5 runs the VFL kernel's powf branch"""
    logits, boxes, targets, forced = _forced_case(seed=7 if gamma == 2.0 else 8)
    nb = 71 / 8
    crit = _criterion(gamma)
    crit.forced_match = forced
    table, dlg, dbx = _run_criterion(crit, logits, boxes, targets, nb=nb)
    counts = [len(t[0]) for t in targets]
    offs = np.cumsum([0] + counts)
    idx = [[(forced[l, offs[b]:offs[b + 1]].to(torch.int64), torch.arange(counts[b])) for b in range(len(targets))] for l in range(forced.shape[0])]
    _check_layer_losses(table, dlg, dbx, logits, boxes, targets, idx, nb, gamma, f"forced gamma={gamma}")


def test_edge_boxes_are_exact_in_fp32():
    """the corners the kernels derive in fp32 (cx -+ 0.5 w) equal the fp64 ones, so every designed tie and touch is one in both precisions"""
    g = _gen(0)
    for kind in EDGE_KINDS:
        for _ in range(20):
            p, t, _ = _edge_pair(kind, g)
            for box in (p, t):
                c64 = CO.cxcywh_to_xyxy(box[None])[0]
                c32 = CO.cxcywh_to_xyxy(box[None].float())[0]
                assert torch.equal(c32.to(F64), c64), (kind, box)
            a, b = CO.cxcywh_to_xyxy(p[None].float())[0], CO.cxcywh_to_xyxy(t[None].float())[0]
            rawiw = float(torch.min(a[2], b[2]) - torch.max(a[0], b[0]))
            rawih = float(torch.min(a[3], b[3]) - torch.max(a[1], b[1]))
            if kind == "same":
                assert torch.equal(a, b)
            elif kind == "touch_x":
                assert rawiw == 0.0 and rawih > 0
            elif kind == "touch_y":
                assert rawih == 0.0 and rawiw > 0
            elif kind == "disjoint":
                assert rawiw < 0
            elif kind == "outside":
                assert float(a[0]) < 0 and float(a[2]) > 1
            else:
                assert rawiw > 0 and rawih > 0


def test_giou_gradient_reference_matches_finite_differences():
    """fp64 autograd of 1 - GIoU (oracle/criterion_oracle.pair_giou) against central differences, for boxes in general position (no ties):
    the truncation error of a step h is ~h^2 |f'''| ~ 1e-12 and the rounding error ~1e-16 / h ~ 1e-10, far below the 1e-7 bound"""
    g = _gen(1)
    src = torch.cat([0.2 + 0.6 * torch.rand((64, 2), generator=g, dtype=F64), 0.05 + 0.4 * torch.rand((64, 2), generator=g, dtype=F64)], 1)
    tgt = (src + 0.08 * torch.randn((64, 4), generator=g, dtype=F64)).clamp(0.03, 0.97)

    def f(s):
        return (1 - CO.pair_giou(CO.cxcywh_to_xyxy(s), CO.cxcywh_to_xyxy(tgt))).sum()

    s = src.clone().requires_grad_(True)
    f(s).backward()
    h = 1e-6
    fd = torch.zeros_like(src)
    for i in range(src.shape[0]):
        for k in range(4):
            e = torch.zeros_like(src)
            e[i, k] = h
            fd[i, k] = (f(src + e) - f(src - e)) / (2 * h)
    assert float((s.grad - fd).abs().max()) <= 1e-7 * float(fd.abs().max())


# =====================================================================================================================================
# 2. Optimiser step
# =====================================================================================================================================
SYNTH_NUMELS = (65536, 65539, 1, 3, 5)   # padded lengths 65536 (one whole chunk), 65540 (a chunk + a 4-element chunk), 4, 4, 8
CLIP, BETAS, EPS, INIT_SCALE, GROWTH_INTERVAL, WORLD = 0.1, (0.9, 0.999), 1e-8, 2.0 ** 10, 3, 8
NORM_RTOL = 1e-6


class Replay64:
    """float64 replay over one flat buffer of the reference's step (oracle/optim_oracle.py: GradScaler.unscale_, clip_grad_norm_ twice, AdamW
    with per-tensor lr / weight decay, GradScaler.update), for gradients that hold loss scale x the SUM over `world` ranks.  lr / wd are per
    element; inactive elements belong to tensors whose .grad is None: no update, no decay, and clip_grad_norm_ does not see them."""

    def __init__(self, lr, wd, amp=True, world=1, scale=INIT_SCALE, growth_interval=GROWTH_INTERVAL):
        self.lr, self.wd, self.amp, self.world, self.growth_interval = lr, wd, amp, world, growth_interval
        self.scale, self.tracker, self.step_count = (scale if amp else 1.0), 0, 0

    def stats(self, g_sum):
        """(found_inf, grad norm, clip coefficient) of this step's gradients, as the torch sequence computes them"""
        found = not bool(torch.isfinite(g_sum).all())
        g = g_sum / self.world / self.scale
        norm = float(torch.linalg.vector_norm(g))
        coef = 1.0
        for _ in range(2):  # clip_grad_norm_ in TrainerLoop.clip_grads and in FullModelGradientClippingOptimizer.step
            c = min(CLIP / (float(torch.linalg.vector_norm(g)) + 1e-6), 1.0)
            g = g * c
            coef *= c
        return found, norm, coef

    def step(self, p, m, v, g_sum, active, coef):
        """new (p, m, v) from the state before the step, given the clip coefficient `coef`; then the scaler update.  Returns (p, m, v, found_inf)."""
        found = not bool(torch.isfinite(g_sum).all())
        self.step_scale = self.scale   # the loss scale this step's gradients carry (the update below may change self.scale)
        if not found:
            self.step_count += 1
            g = g_sum / self.world / self.scale * coef
            b1, b2 = BETAS
            pn = p * (1 - self.lr * self.wd)
            mn = m + (g - m) * (1 - b1)
            vn = v * b2 + (1 - b2) * g * g
            bc1, bc2 = 1 - b1 ** self.step_count, 1 - b2 ** self.step_count
            pn = pn - (self.lr / bc1) * mn / (vn.sqrt() / math.sqrt(bc2) + EPS)
            p, m, v = torch.where(active, pn, p), torch.where(active, mn, m), torch.where(active, vn, v)
        if self.amp:
            if found:
                self.scale, self.tracker = self.scale * 0.5, 0
            else:
                self.tracker += 1
                if self.tracker == self.growth_interval:
                    self.scale, self.tracker = self.scale * 2.0, 0
        return p, m, v, found

    def tolerances(self, p, m, v, g_sum, coef):
        """per-element bounds on the fp32 kernel's (p, m, v) after one step from the same fp32 state and the same clip coefficient.  The kernel
        rounds each operation once (lr, 1 - lr wd, lr / bc1, bc1, sqrt(bc2) and the gradient multiplier are fp32 too): <= 8 roundings on any
        path, so delta = 16U relative to the sum of the absolute values that enter it.  v' = b2 v + (1 - b2) g^2 has positive terms only.
        Call after step(): the bias corrections and the loss scale are those of the step just taken."""
        assert self.step_count > 0
        d = 16 * U
        g = (g_sum / self.world / self.step_scale * coef).abs()
        b1, b2 = BETAS
        step = self.step_count
        bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
        vn = v * b2 + (1 - b2) * g * g
        den = vn.sqrt() / math.sqrt(bc2) + EPS
        mabs = m.abs() + g
        return d * (p.abs() + (self.lr / bc1) * mabs / den), d * mabs, d * vn


def _fai_detr_groups():
    """(name, initial values on the CPU, lr, weight decay) of the fai-detr-l parameter groups, then the synthetic edge tensors"""
    model = FAIDetr(DETRConfig())
    groups = get_optimizer_params(model, base_lr=5e-4, weight_decay=0.02, backbone_multiplier=0.1)
    out = [(g["name"], g["params"][0].detach().clone(), g["lr"], g["weight_decay"]) for g in groups]
    gen = _gen(5)
    out += [(f"edge{i}", torch.randn(n, generator=gen) * 0.1, 5e-4, 0.02 * (i % 2)) for i, n in enumerate(SYNTH_NUMELS)]
    return out


def _flat_adamw(layout, device, amp=True, world=WORLD):
    params = [nn.Parameter(t.to(device)) for _, t, _, _ in layout]
    groups = [{"params": [p], "lr": lr, "weight_decay": wd, "name": name} for p, (name, _, lr, wd) in zip(params, layout)]
    opt = FlatAdamW(groups, betas=BETAS, eps=EPS, clip_gradients=CLIP, amp=amp, init_scale=INIT_SCALE, growth_interval=GROWTH_INTERVAL, world_size=world)
    opt.track_unused_parameters()
    return opt, params


def _per_element(opt, values, dtype=F64):
    out = torch.zeros(opt.total, dtype=dtype, device=opt.flat_params.device)
    for o, p, x in zip(opt.offsets, opt.params, values):
        out[o:o + p.numel()] = x
    return out


# the fine-tune leg's schedule of events over 8 steps: clipped, below the clip threshold, NaN, inf, then enough finite steps for a scale growth
PLAN = ("clip", "small", "nan_last", "clip", "inf_middle", "clip", "clip", "clip")


def _step_grads(opt, it, kind, device):
    """this step's flat gradient values (loss scale x sum over ranks is applied by the caller): per-tensor magnitudes spread over 1e-4..1e-1"""
    g = torch.Generator(device=device).manual_seed(100 + it)
    G = torch.randn(opt.total, generator=g, device=device)
    mag = torch.exp(torch.empty(len(opt.params), device=device).uniform_(math.log(1e-4), math.log(1e-1), generator=g))
    G *= torch.repeat_interleave(mag, torch.tensor([(p.numel() + 3) // 4 * 4 for p in opt.params], device=device))
    if kind == "small":
        G *= 1e-7 / float(torch.linalg.vector_norm(G.double()))  # the unscaled norm ends far below the 0.1 threshold: clip coefficient exactly 1
    elif kind == "nan_last":
        G[opt.offsets[-1] + opt.params[-1].numel() - 1] = float("nan")   # the last real element of the last tensor
    elif kind == "inf_middle":
        G[opt.total // 2] = float("inf")
    return G


def _backward(opt, params, G, active, scale):
    """gradients through autograd into the flat buffer (the post-accumulate hooks mark the tensors reached): d/dp of scale * sum(p * G) = scale * G"""
    opt.zero_grad()
    loss = sum((p * G[o:o + p.numel()].view_as(p)).sum() for i, (p, o) in enumerate(zip(params, opt.offsets)) if active[i])
    (loss * scale).backward()


def _run_plan(layout, inactive, check):
    opt, params = _flat_adamw(layout, DEV)
    active = [i not in inactive for i in range(len(params))]
    act_el = _per_element(opt, [1.0 if a else 0.0 for a in active]) > 0
    lr_el = _per_element(opt, [lr for _, _, lr, _ in layout])
    wd_el = _per_element(opt, [wd for _, _, _, wd in layout])
    rep = Replay64(lr_el, wd_el, world=WORLD)
    for it, kind in enumerate(PLAN):
        G = _step_grads(opt, it, kind, DEV)
        scale = float(opt.loss_scale)
        assert not check or scale == rep.scale, f"step {it}: loss scale {scale} vs {rep.scale}"
        _backward(opt, params, G, active, scale)
        p0, m0, v0 = opt.flat_params.double(), opt.exp_avg.double(), opt.exp_avg_sq.double()
        g = opt.flat_grads.double()
        opt.step()
        st = opt.stats()
        if not check:
            continue
        found, norm, coef = rep.stats(g)
        assert st["found_inf"] == int(found) == int(kind in ("nan_last", "inf_middle")), f"step {it} ({kind}): found_inf"
        if not found:
            # grad_stats: per-thread fp32 sums of ~81 float4 (326 squares) then a double reduction.  One thread's sum is within 326 U of its
            # value at worst, but the roundings are unbiased and independent across the 135 168 threads, so the total's relative error is
            # ~U sqrt(326 / 135168) ~ 3e-9; 1e-6 covers the final fp32 rounding of the norm (U / 2) with two orders of margin
            assert abs(st["grad_norm"] - norm) <= NORM_RTOL * norm, f"step {it}: grad_norm {st['grad_norm']!r} vs fp64 {norm!r}"
            # coef = min(0.1 / (norm + 1e-6), 1), twice: inherits the norm's relative error plus ~4 roundings; exactly 1 below the threshold
            assert abs(st["clip_coef"] - coef) <= (NORM_RTOL + 8 * U) * coef, f"step {it}: clip_coef {st['clip_coef']!r} vs fp64 {coef!r}"
            if kind == "small":
                assert st["clip_coef"] == 1.0 == coef
        # the buffers: one fp64 step from the kernel's own fp32 state, with the kernel's clip coefficient (checked just above)
        p1, m1, v1, _ = rep.step(p0, m0, v0, g, act_el, st["clip_coef"])
        tp, tm, tv = rep.tolerances(p0, m0, v0, g, st["clip_coef"])   # after rep.step: the bias corrections of this step
        for name, got, ref, tol in (("param", opt.flat_params, p1, tp), ("exp_avg", opt.exp_avg, m1, tm), ("exp_avg_sq", opt.exp_avg_sq, v1, tv)):
            err = (got.double() - ref).abs()
            if found:
                assert torch.equal(got.double(), {"param": p0, "exp_avg": m0, "exp_avg_sq": v0}[name]), f"step {it}: skipped step changed {name}"
            else:
                i = int(torch.argmax(err / tol.clamp(min=1e-300)))
                assert bool((err <= tol).all()), f"step {it} ({kind}) {name}[{i}]: {float(got[i])!r} vs fp64 {float(ref[i])!r} (tol {float(tol[i]):.3g})"
        for i in inactive:  # no gradient: parameters and moments bit-unchanged (weight decay included)
            o, n = opt.offsets[i], params[i].numel()
            assert torch.equal(opt.flat_params[o:o + n], p0[o:o + n].float()) and torch.equal(opt.exp_avg[o:o + n], m0[o:o + n].float()) \
                and torch.equal(opt.exp_avg_sq[o:o + n], v0[o:o + n].float()), f"step {it}: inactive tensor {layout[i][0]} changed"
        assert st["step"] == rep.step_count and st["scale"] == rep.scale and st["growth_tracker"] == rep.tracker, f"step {it}: {st}"
    return opt


@gpu
def test_optimizer_step_fai_detr_flat_buffer_vs_fp64_replay(be):
    """the real 501-tensor / 44.0 M-element fai-detr-l layout plus the chunk / padding edge tensors, world_size = 8, five tensors unused"""
    layout = _fai_detr_groups()
    n_real = len(layout) - len(SYNTH_NUMELS)
    assert n_real == 501
    inactive = {3, 120, 377, n_real, n_real + 2}   # three real tensors, the whole-chunk edge tensor and the 3-element one
    opt = _run_plan(layout, inactive, check=True)
    st = opt.stats()
    assert st["step"] == 6 and st["scale"] == INIT_SCALE * 0.25 * 2, st   # two skipped steps backed off twice; three finite steps in a row grew it once
    again = _run_plan(layout, inactive, check=False)
    for a, b in ((opt.flat_params, again.flat_params), (opt.exp_avg, again.exp_avg), (opt.exp_avg_sq, again.exp_avg_sq), (opt.ctrl, again.ctrl)):
        assert torch.equal(a, b), "two identical runs differ"


@gpu
def test_optimizer_without_scaler_skips_nonfinite_step(be):
    """amp=False: a non-finite gradient skips the step (FB200_CTRL_FOUND_INF); torch would write NaN into the parameters instead"""
    layout = [(f"t{i}", torch.randn(n, generator=_gen(i)) * 0.1, 1e-3, 0.02) for i, n in enumerate((7, 4099, 1))]
    opt, params = _flat_adamw(layout, DEV, amp=False, world=1)
    G = torch.randn(opt.total, generator=_gen(9)).to(DEV)
    _backward(opt, params, G, [True] * 3, 1.0)
    opt.step()
    before = [t.clone() for t in (opt.flat_params, opt.exp_avg, opt.exp_avg_sq)]
    G[5] = float("nan")
    _backward(opt, params, G, [True] * 3, 1.0)
    opt.step()
    st = opt.stats()
    assert st["found_inf"] == 1 and st["step"] == 1 and st["scale"] == 1.0
    for a, b in zip((opt.flat_params, opt.exp_avg, opt.exp_avg_sq), before):
        assert torch.equal(a, b)


def test_fp64_replay_matches_reference_stepper():
    """the fp64 replay against oracle/optim_oracle.ReferenceStepper (torch's own CPU classes) on a small layout: world_size = 8 (DDP's average
    before unscale_), one tensor without gradient, a NaN step, a below-threshold step and a scale growth.  fp32 tolerance as in the optimiser's
    existing parity test: 2e-6 of the parameter scale."""
    shapes = [(7,), (65, 33), (3, 3, 8, 5), (1,), (3000,)]
    inactive = 2
    init = [torch.randn(s, generator=_gen(20 + i)) * 0.1 for i, s in enumerate(shapes)]
    ref = [nn.Parameter(t.clone()) for t in init]
    groups = [{"params": [p], "lr": 1e-3 * (0.1 if i % 2 else 1.0), "weight_decay": 0.0 if i == 3 else 0.02, "name": f"p{i}"} for i, p in enumerate(ref)]
    stepper = ReferenceStepper(groups, lr=1e-3, weight_decay=0.02, clip=CLIP, growth_interval=GROWTH_INTERVAL)
    sizes = [t.numel() for t in init]
    lr = torch.cat([torch.full((n,), g["lr"], dtype=F64) for n, g in zip(sizes, groups)])
    wd = torch.cat([torch.full((n,), g["weight_decay"], dtype=F64) for n, g in zip(sizes, groups)])
    act = torch.cat([torch.full((n,), i != inactive) for i, n in enumerate(sizes)])
    rep = Replay64(lr, wd, world=WORLD)
    p = torch.cat([t.reshape(-1) for t in init]).to(F64)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    g = _gen(3)
    for it in range(8):
        mag = [1.0, 1e-6, 50.0, 1.0][it % 4]
        G = [torch.randn(s, generator=g) * mag for s in shapes]   # the sum over the 8 ranks
        if it == 2:
            G[4][17] = float("nan")
        assert stepper.scaler.get_scale() == rep.scale
        stepper.step(lambda: sum((q * Gi).sum() for i, (q, Gi) in enumerate(zip(ref, G)) if i != inactive),
                     world_grads=lambda ps: [q.grad.div_(WORLD) for q in ps if q.grad is not None])
        gs = torch.cat([Gi.reshape(-1) for Gi in G]).to(F64) * rep.scale * act
        _, _, coef = rep.stats(gs)
        p, m, v, _ = rep.step(p, m, v, gs, act, coef)
        got = torch.cat([q.detach().reshape(-1) for q in ref]).to(F64)
        assert float((got - p).abs().max()) <= 2e-6 * max(1.0, float(p.abs().max())), f"step {it}"
    assert stepper.scaler.get_scale() == rep.scale and rep.step_count == 7


# =====================================================================================================================================
# 3. Max-pool, average-pool and bilinear-resize backward
# =====================================================================================================================================
def _nchw64(t):
    return t.permute(0, 3, 1, 2).to(device="cpu", dtype=F64)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _int_grad(shape, seed):
    """upstream gradient of small non-zero integers (|dy| in 1..15): sums of up to 16 of them times dyadic weights are exact in fp32"""
    g = _gen(seed)
    mag = torch.randint(1, 16, shape, generator=g, dtype=torch.int32)
    return torch.where(torch.rand(shape, generator=g) < 0.5, -mag, mag).float()


def _misaligned_like(t):
    """an uninitialised tensor shaped like t whose data pointer is 4 bytes past a 16-byte boundary"""
    buf = torch.empty(t.numel() + 4, dtype=t.dtype, device=t.device)
    v = buf[1:1 + t.numel()].view(t.shape)
    assert v.data_ptr() % 16 == 4
    return v


MAXPOOL_CASES = {  # name: (B, H, W, C, input kind)
    "stem_relu": (16, 320, 320, 64, "relu"),        # the stem output at 640x640, bs=16: about half the values are exact zeros
    "stem_levels": (16, 320, 320, 64, "levels"),    # quantised to a few levels: positive values tie too
    "odd_45x61": (2, 45, 61, 64, "levels"),
    "one_pixel": (3, 1, 1, 64, "relu"),
    "map_2x3": (3, 2, 3, 64, "levels"),
}


@gpu
@pytest.mark.parametrize("case", list(MAXPOOL_CASES))
def test_maxpool_bwd_routes_ties_to_the_first_maximum(be, case):
    """max_pool2d(3, 2, 1) backward: the vector kernel (through A.MaxPoolFn), the scalar kernel on a misaligned dx and on C = 6.  With integer dy
    every dx is an exact fp32 sum, so the kernels must equal fp64 autograd bit for bit; aten's CPU kernel routes a tie to the first maximum in
    row-major window order, the rule the kernels implement."""
    B, H, W, C, kind = MAXPOOL_CASES[case]
    g = _gen(list(MAXPOOL_CASES).index(case))
    x = torch.randn((B, H, W, C), generator=g)
    x = torch.relu(x) if kind == "relu" else torch.relu(torch.round(2 * x)) / 2
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    dy = _int_grad((B, Ho, Wo, C), 1)
    xr = _nchw64(x).requires_grad_(True)
    yr = F.max_pool2d(xr, 3, 2, 1)
    yr.backward(_nchw64(dy))
    ref = _nhwc(xr.grad)
    xd, dyd = x.to(DEV), dy.to(DEV)
    xg = xd.clone().requires_grad_(True)
    y = A.MaxPoolFn.apply(xg)
    assert torch.equal(_nhwc(yr.detach()).float(), y.detach().cpu())
    y.backward(dyd)
    assert torch.equal(xg.grad.cpu().to(F64), ref), f"{case}: vector kernel, {int((xg.grad.cpu().to(F64) != ref).sum())} elements differ"
    first = xg.grad.clone()
    xg.grad = None
    A.MaxPoolFn.apply(xg).backward(dyd)
    assert torch.equal(xg.grad, first), "vector kernel: two runs differ"
    dx = _misaligned_like(xd)
    be.maxpool_bwd(xd, dyd, dx)
    assert torch.equal(dx.cpu().to(F64), ref), f"{case}: scalar kernel (misaligned dx)"
    x6, dy6 = xd[..., :6].contiguous(), dyd[..., :6].contiguous()
    dx6 = torch.empty_like(x6)
    be.maxpool_bwd(x6, dy6, dx6)
    assert torch.equal(dx6.cpu().to(F64), ref[..., :6]), f"{case}: scalar kernel (C = 6)"
    be.maxpool_bwd(x6, dy6, dx6)
    assert torch.equal(dx6.cpu().to(F64), ref[..., :6]), "scalar kernel: two runs differ"


AVGPOOL_CASES = {  # name: (B, H, W, C); the ResNet-vd shortcut pools of fai-detr-l at 640x640, bs=16, and odd maps
    "vd_160": (16, 160, 160, 256),
    "vd_80": (16, 80, 80, 512),
    "vd_40": (16, 40, 40, 1024),
    "odd_45x61": (2, 45, 61, 64),
    "one_pixel": (3, 1, 1, 64),
}


@gpu
@pytest.mark.parametrize("case", list(AVGPOOL_CASES))
def test_avgpool_ceil_bwd(be, case):
    """AvgPool2d(2, 2, 0, ceil_mode=True) backward: dy / (in-bounds window size 1, 2 or 4) is exact for integer dy, so bit-equal to fp64 autograd"""
    B, H, W, C = AVGPOOL_CASES[case]
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    dy = _int_grad((B, Ho, Wo, C), 2)
    xr = torch.zeros((B, C, H, W), dtype=F64, requires_grad=True)
    F.avg_pool2d(xr, 2, 2, 0, ceil_mode=True).backward(_nchw64(dy))
    ref = _nhwc(xr.grad)
    dyd = dy.to(DEV)
    dx = torch.empty((B, H, W, C), device=DEV)
    be.avgpool_bwd(dyd, dx)
    assert torch.equal(dx.cpu().to(F64), ref), f"{case}: {int((dx.cpu().to(F64) != ref).sum())} elements differ"
    dx2 = torch.empty_like(dx)
    be.avgpool_bwd(dyd, dx2)
    assert torch.equal(dx, dx2), "two runs differ"


RESIZE_CASES = {  # name: (B, H, W, Ho, Wo, C): the forward resizes (H, W) -> (Ho, Wo); the backward maps dy [B,Ho,Wo,C] to dx [B,H,W,C]
    "fpn_up_20_40": (16, 20, 20, 40, 40, 256),
    "fpn_up_40_80": (16, 40, 40, 80, 80, 256),
    "fpn_down_80_40": (16, 80, 80, 40, 40, 256),
    "fpn_down_40_20": (16, 40, 40, 20, 20, 256),
    "down_45x61_23x31": (4, 45, 61, 23, 31, 64),
    "up_23x31_45x61": (4, 23, 31, 45, 61, 64),
    "up_1x1_5x7": (4, 1, 1, 5, 7, 64),
    "down_7x5_1x1": (4, 7, 5, 1, 1, 64),
}


def _resize_tol(H, W, Ho, Wo, dy_max):
    """bound on |dx(fp32) - dx(fp64)|.  The kernel's source coordinate (ho + 0.5) sh - 0.5 with sh = fl(H / Ho) is off by <= (H + 1) U, and so is
    each 1-D weight; a product of two weights by <= (H + W + 3) U; at most n = (ceil(Ho / H) + 3)(ceil(Wo / W) + 3) candidates add to one dx,
    each |dy| <= dy_max, and their running sum rounds n more times.  Zero when every weight and sum is exact (2x ratios: weights in 1/16)."""
    if (Ho == 2 * H or H == 2 * Ho) and (Wo == 2 * W or W == 2 * Wo):
        return 0.0
    n = (math.ceil(Ho / H) + 3) * (math.ceil(Wo / W) + 3)
    return (H + W + 3 + n) * U * n * dy_max


@gpu
@pytest.mark.parametrize("case", list(RESIZE_CASES))
def test_resize_bilinear_bwd(be, case):
    """bilinear (align_corners=False) backward at the FPN shapes of fai-detr-l (bs=16, C=256) and at non-2x ratios, through A.ResizeFn and through
    the ABI with dy a channel slice of a wider NaN-filled buffer (dy_pitch > C): the other channels must not reach dx"""
    B, H, W, Ho, Wo, C = RESIZE_CASES[case]
    dy = _int_grad((B, Ho, Wo, C), 3)
    xr = torch.zeros((B, C, H, W), dtype=F64, requires_grad=True)
    F.interpolate(xr, size=(Ho, Wo), mode="bilinear", align_corners=False).backward(_nchw64(dy))
    ref = _nhwc(xr.grad)
    tol = _resize_tol(H, W, Ho, Wo, 15.0)
    xg = torch.zeros((B, H, W, C), device=DEV, requires_grad=True)
    dyd = dy.to(DEV)
    A.ResizeFn.apply(xg, (Ho, Wo)).backward(dyd)
    err = float((xg.grad.cpu().to(F64) - ref).abs().max())
    assert err <= tol, f"{case}: max |dx - fp64| = {err:.3g} > {tol:.3g}"
    wide = torch.full((B, Ho, Wo, C + 24), float("nan"), device=DEV)
    wide[..., 8:8 + C] = dyd
    dy_slice = wide[..., 8:8 + C]
    dx = torch.empty((B, H, W, C), device=DEV)
    be._call("fb200_resize_bilinear_bwd", ops._p(dy_slice), dy_slice.stride(2), B, H, W, C, Ho, Wo, ops._p(dx), ops._stream())
    assert torch.equal(dx, xg.grad), f"{case}: the pitched dy gives another dx (NaN channels read: {bool(dx.isnan().any())})"
    dx2 = torch.empty_like(dx)
    be.resize_bwd(dyd, dx2)
    assert torch.equal(dx2, xg.grad), "two runs differ"
