"""-m gpu: the training-mode BatchNorm kernels (bwd_conv_norm.cu) against torch fp64 on the CPU, at the row counts of real fine-tuning.

Each BatchNorm pass is routed by C and R = B*H*W to one of several kernels, and their unrolled main loops only run once the grid is
capped, i.e. at row counts far above the tiny shapes of the other training tests:
  column passes (statistics, backward sums)   col_partial4_kernel (C in {32, 64, 128} or C % 128 == 0), else the scalar col_partial_kernel;
                                              four-rows-per-iteration loop once R > 3 * 264 * RPB
  element-wise passes (apply, backward apply) the column-fixed *_cf_kernels when 256 % (C/4) == 0 or (C/4) % 256 == 0, else the generic
                                              bn_apply_kernel / bn_bwd_apply4_kernel; the cf two-rows-per-iteration loop once R*C/4 > 2112 * 256
The large row counts below are above both thresholds of their C and not a multiple of the loop's row step, so the unrolled loops and
their tails both run.  The SyncBatchNorm / FrozenBatchNorm phase kernels are checked the same way, with data-parallel ranks simulated
by splitting the rows on one GPU.

Every case has adversarial channels: a constant one (variance 0, rstd = 1/sqrt(eps)), one with mean >> sigma, and one whose row 0 -
the reference row of the kernels' single-pass sums - lies 40 sigma from the channel mean; the rest are N(0.5, 2).  (With row 0 as the
one pivot of all squared sums, that channel's variance lost ~1e-5 to fp32 cancellation and failed the 1e-6 running-statistics bar.)"""
import functools

import pytest
import torch
import torch.nn.functional as F

from focoos_b200 import autograd_ops as A
from focoos_b200 import ops

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]
DEV = "cuda"
EPS, MOMENTUM = 1e-5, 0.1
FWD_TOL, GRAD_TOL, RUN_TOL = 2e-5, 5e-5, 1e-6

# (name, activation, fused residual): the four combinations BatchNormTrainFn accepts
VARIANTS = [("none", ops.ACT_NONE, False), ("relu", ops.ACT_RELU, False), ("relu_res", ops.ACT_RELU, True), ("silu", ops.ACT_SILU, False)]
VID = [v[0] for v in VARIANTS]
ACT_FN = {ops.ACT_NONE: lambda t: t, ops.ACT_RELU: F.relu, ops.ACT_SILU: F.silu}

# C -> a row count above every loop threshold of that C (see the module docstring), and the kernels it selects:
LARGE_R = {
    12: 7001,     # scalar col_partial (RPB 8): 4-row loop for R > 6,336; generic bn_apply / bn_bwd_apply4 (C/4 = 3 does not divide 256)
    32: 71587,    # col_partial4 (RPB 32): R > 25,344; cf, C/4 = 8: 2-row loop for R > 67,584
    64: 36871,    # col_partial4 (RPB 16): R > 12,672; cf, C/4 = 16: R > 33,792
    256: 9013,    # col_partial4 (RPB 8): R > 6,336; cf, C/4 = 64: R > 8,448
    2048: 6421,   # col_partial4 (RPB 8, 16 channel chunks): R > 6,336; cf, C/4 = 512 (blocks rounded to pairs): R > 1,056
    96: 7001,     # scalar col_partial (RPB 8): R > 6,336; generic bn_apply / bn_bwd_apply4 (C/4 = 24 does not divide 256)
}
# tiny row counts: fewer rows than one block's row lanes (a single, partly idle row slice)
CASES = [(C, R) for C in LARGE_R for R in (2, 5, LARGE_R[C])]


def special_channels(C):
    """(constant, mean >> sigma, far pivot) channel indices, spread over different float4 lanes and blocks"""
    return 1, C // 2 + 2, C - 1


@functools.lru_cache(maxsize=4)
def bn_data(R, C, seed=0):
    g = torch.Generator().manual_seed(seed * 1000003 + R * 4099 + C)
    x = torch.randn((R, C), generator=g) * 2 + 0.5
    c_const, c_big, c_piv = special_channels(C)
    x[:, c_const] = 0.7
    x[:, c_big] = 50 + 0.05 * torch.randn(R, generator=g)
    x[0, c_piv] = 0.5 + 40 * 2.0
    res = torch.randn((R, C), generator=g)
    gamma = (torch.rand(C, generator=g) + 0.5) * torch.where(torch.rand(C, generator=g) < 0.25, -1.0, 1.0)
    beta = torch.randn(C, generator=g) * 0.5
    rm, rv = torch.randn(C, generator=g) * 0.1, torch.rand(C, generator=g) + 0.5
    dy = torch.randn((R, C), generator=g)
    return x, res, gamma, beta, rm, rv, dy


def masked_dy(dy, z, act):
    """dy with zeros where a ReLU's argument is within 1e-3 of 0: there the fp32 kernel and the fp64 reference may take different sides of the
    kink (a gradient of dy or 0), so neither choice is tested; everywhere else the mask is the same on both sides"""
    return torch.where(z.abs() < 1e-3, torch.zeros_like(dy), dy) if act == ops.ACT_RELU else dy


def ulp32(t):
    t = t.float()
    return (torch.nextafter(t.abs(), torch.tensor(float("inf"))) - t.abs()).double()


def check(got, ref, what, tol, extra=None, floor=None):
    """max |got - ref| within tol * max |ref|, taken PER CHANNEL (last dimension) for [R, C] tensors: the constant channel's rstd is
    1/sqrt(eps) ~ 316, so a tensor-wide scale would hide errors in every other channel.  `extra` [C] adds a per-channel allowance;
    `floor` [C] is a least scale, for results that are small only because larger terms cancel."""
    ref = ref.detach().double().reshape(-1, ref.shape[-1])
    got = got.detach().double().cpu().reshape(ref.shape)
    scale = ref.abs().amax(0).clamp_min(1e-6)
    if floor is not None:
        scale = torch.maximum(scale, floor)
    bar = tol * scale + (0.0 if extra is None else extra)
    err = (got - ref).abs().amax(0)
    c = int(torch.argmax(err / bar))
    assert bool((err <= bar).all()), f"{what}: channel {c}: max|d|={float(err[c]):.3e} > bar {float(bar[c]):.3e} (scale {float(scale[c]):.3e})"


def check_vec(got, ref, what, tol, extra=None):
    """[C] vectors (dgamma, dbeta, running_mean): within tol * max |ref| of the whole vector (a column sum of random gradients may be near 0)"""
    got, ref = got.detach().double().cpu().reshape(-1), ref.detach().double().reshape(-1)
    bar = tol * max(1e-6, float(ref.abs().max())) + (0.0 if extra is None else extra)
    err = (got - ref).abs()
    c = int(torch.argmax(err / bar))
    assert bool((err <= bar).all()), f"{what}: channel {c}: max|d|={float(err[c]):.3e} > bar {float(torch.as_tensor(bar).expand_as(err)[c]):.3e}"


def reference(x, res, gamma, beta, rm, rv, dy, act, with_res):
    """fp64 train-mode BatchNorm over the rows of [R, C] fp32 inputs (+ res, then act), its autograd gradients and the running statistics
    (momentum 0.1, unbiased variance); dy is masked around the ReLU kink (masked_dy).  Returns (dict of fp64 results, masked dy fp32); the dict
    also carries what the bars of check_all are derived from."""
    xd, gd, bd = (t.detach().double().requires_grad_(True) for t in (x, gamma, beta))
    rd = res.detach().double().requires_grad_(True) if with_res else None
    rmd, rvd = rm.double(), rv.double()
    zb = F.batch_norm(xd, rmd, rvd, gd, bd, training=True, momentum=MOMENTUM, eps=EPS)
    z = zb + rd if with_res else zb
    dy = masked_dy(dy, z.detach(), act)
    y = ACT_FN[act](z)
    y.backward(dy.double())
    xv = x.double()
    mean, var = xv.mean(0), xv.var(0, unbiased=False)
    rstd = (var + EPS).rsqrt()
    out = dict(y=y.detach(), dx=xd.grad, dgamma=gd.grad, dbeta=bd.grad, running_mean=rmd, running_var=rvd, mean=mean, rstd=rstd,
               R=x.shape[0], act=act, gamma=gamma.double(), dy=dy.double(), xhat_max=rstd * (xv - mean).abs().amax(0),
               # y = act(BN(x) + res) is small where the two cancel; its error is that of the terms
               y_floor=zb.detach().abs().amax(0) + (res.double().abs().amax(0) if with_res else 0.0))
    if with_res:
        out["dres"] = rd.grad
    return out, dy


def mean_rounding(ref, mean_ulps):
    """Allowances for the rounding of the kernel's mean to fp32.  However exact its sums are, (x - mean) carries that rounding, a shift
    d = rstd * ulp(mean) / 2 of every x_hat of the channel; for the mean >> sigma channel (50 + 0.05 N: ulp(50) / 2 = 1.9e-6, rstd = 20)
    that is 3.8e-5, above the forward bar.  (SyncBatchNorm combines per-rank means that are fp32 values themselves: up to one ulp.)
    To first order, with dz = |gamma| d and dg <= k |dy| dz (k = max |act''| = 1/2 for SiLU; 0 otherwise, the ReLU kink being masked),
    the shift moves
        y       by dz
        dbeta   by k dz sum|dy|                                                              (dbeta = sum g)
        dgamma  by d |dbeta| + k dz max|x_hat| sum|dy|                                       (dgamma = sum g * x_hat)
        dx      by |gamma| rstd (k dz max|dy| + (d_dbeta + d |dgamma| + max|x_hat| d_dgamma) / R)
    The same terms are added for every channel; they are negligible where |mean| is not large against sigma."""
    k = 0.5 if ref["act"] == ops.ACT_SILU else 0.0
    rstd, ga, xm = ref["rstd"], ref["gamma"].abs(), ref["xhat_max"]
    d = rstd * ulp32(ref["mean"]) * mean_ulps
    dz = ga * d
    db, dg = ref["dbeta"].abs(), ref["dgamma"].abs()
    dy_sum, dy_max = ref["dy"].abs().sum(0), ref["dy"].abs().amax(0)
    d_dbeta = k * dz * dy_sum
    d_dgamma = d * db + k * dz * xm * dy_sum
    return dict(y=dz, dbeta=d_dbeta, dgamma=d_dgamma, dx=ga * rstd * (k * dz * dy_max + (d_dbeta + d * dg + xm * d_dgamma) / ref["R"]))


def check_stats(mean, rstd, ref, what, target=None, mean_ulps=0.5):
    # the mean to the forward bar in units of sigma (its effect on x_hat), plus its own fp32 rounding; rstd relative, per channel
    target = ref if target is None else target
    err_m = (mean.double().cpu() - target["mean"].double()).abs()
    bar_m = FWD_TOL / ref["rstd"] + ulp32(ref["mean"]) * mean_ulps
    assert bool((err_m <= bar_m).all()), f"{what} mean: channel {int(torch.argmax(err_m / bar_m))} off by {float((err_m / bar_m).max()):.2f} x the bar"
    check(rstd.reshape(1, -1), target["rstd"].reshape(1, -1), f"{what} rstd", FWD_TOL)


def check_running(rm, rv, ref, what):
    check_vec(rm, ref["running_mean"], f"{what} running_mean", RUN_TOL)
    check(rv.reshape(1, -1), ref["running_var"].reshape(1, -1), f"{what} running_var", RUN_TOL)  # positive: relative per channel


def run_train_fn(x, res, gamma, beta, rm, rv, dy, act, with_res):
    """BatchNormTrainFn forward + backward on the GPU from fresh copies of the inputs; returns every output on the CPU"""
    xg, gg, bg = (t.to(DEV, copy=True).requires_grad_(True) for t in (x, gamma, beta))
    rg = res.to(DEV, copy=True).requires_grad_(True) if with_res else None
    rmg, rvg = rm.to(DEV, copy=True), rv.to(DEV, copy=True)
    yg = A.BatchNormTrainFn.apply(xg, gg, bg, rmg, rvg, rg, act, EPS, MOMENTUM)
    saved = yg.grad_fn.saved_tensors  # (x, gamma, beta, save_mean, save_rstd, y or None): what the backward pass consumes
    mean, rstd = saved[3].cpu(), saved[4].cpu()
    yg.backward(dy.to(DEV, copy=True))
    out = dict(y=yg.detach().cpu(), dx=xg.grad.cpu(), dgamma=gg.grad.cpu(), dbeta=bg.grad.cpu(), running_mean=rmg.cpu(), running_var=rvg.cpu(), mean=mean, rstd=rstd)
    if with_res:
        out["dres"] = rg.grad.cpu()
    return out


def check_all(got, ref, what, target=None, mean_ulps=0.5):
    """every output of one forward + backward against `target` (default: the fp64 reference; or another kernel path's outputs), with the bars
    derived from the fp64 reference `ref`"""
    t = ref if target is None else target
    mr = mean_rounding(ref, mean_ulps)
    check(got["y"], t["y"], f"{what} y", FWD_TOL, extra=mr["y"], floor=ref["y_floor"])
    # dx = gamma * rstd * (g - mean(g) - x_hat * mean(g * x_hat)) cancels to ~0 when R is tiny (R = 2: x_hat = +-1 and dx = 0 exactly without an
    # activation), so its scale is at least that of the terms: |gamma| * rstd * max |dy|
    check(got["dx"], t["dx"], f"{what} dx", GRAD_TOL, extra=mr["dx"], floor=ref["gamma"].abs() * ref["rstd"] * ref["dy"].abs().amax(0))
    if "dres" in ref:
        check(got["dres"], t["dres"], f"{what} dres", FWD_TOL)
    check_vec(got["dgamma"], t["dgamma"], f"{what} dgamma", GRAD_TOL, extra=mr["dgamma"])
    check_vec(got["dbeta"], t["dbeta"], f"{what} dbeta", GRAD_TOL, extra=mr["dbeta"])
    check_stats(got["mean"], got["rstd"], ref, what, t, mean_ulps)
    check_running(got["running_mean"], got["running_var"], t, what)


@pytest.mark.parametrize("name,act,with_res", VARIANTS, ids=VID)
@pytest.mark.parametrize("C,R", CASES, ids=[f"C{C}-R{R}" for C, R in CASES])
def test_batchnorm_train_matches_fp64(C, R, name, act, with_res):
    """bn_train_fwd / bn_train_bwd through BatchNormTrainFn: y, dx, dres, dgamma, dbeta, the saved mean / rstd and the running statistics"""
    x, res, gamma, beta, rm, rv, dy = bn_data(R, C)
    ref, dy = reference(x, res, gamma, beta, rm, rv, dy, act, with_res)
    got = run_train_fn(x, res, gamma, beta, rm, rv, dy, act, with_res)
    check_all(got, ref, f"C={C} R={R} {name}")


@pytest.mark.parametrize("C", list(LARGE_R))
def test_batchnorm_train_is_bitwise_reproducible(C):
    """No atomics anywhere in these reductions: the same inputs must give bit-identical outputs (catches races a tolerance can miss).
    ReLU with a residual: the branch that reads the saved forward output in backward."""
    R = LARGE_R[C]
    x, res, gamma, beta, rm, rv, dy = bn_data(R, C)
    a = run_train_fn(x, res, gamma, beta, rm, rv, dy, ops.ACT_RELU, True)
    b = run_train_fn(x, res, gamma, beta, rm, rv, dy, ops.ACT_RELU, True)
    for k in a:
        assert torch.equal(a[k], b[k]), f"C={C} R={R}: {k} differs between two identical runs"


# ---- SyncBatchNorm as its phase kernels, ranks simulated by splitting the rows ------------------------------------------------------------
SYNC_R = {64: 2 * LARGE_R[64], 96: 2 * LARGE_R[96]}  # C = 64: cf kernels, C = 96: scalar col_partial + generic element-wise kernels


def rank_rows(R, world):
    """row counts per simulated rank: one rank; two equal ranks (each above every loop threshold of its C); three unequal ranks, one of 7 rows"""
    if world == 1:
        return [R]
    if world == 2:
        return [R // 2, R - R // 2]
    return [7, R // 2, R - R // 2 - 7]


def sync_phases(xs, rs, dys, gamma, beta, rm, rv, act, with_res):
    """what SyncBatchNormTrainFn runs on each rank, with the collectives done in place: the [W, 2C+1] all-gather of [mean | biased var | count]
    rows, and the all-reduce of the backward sums as an fp32 sum over ranks"""
    be = ops._be()
    C = xs[0].shape[1]
    rows = []
    for x in xs:
        st = torch.empty(2 * C + 1, device=DEV)
        be.bn_stats(x, st[:C], st[C:2 * C])
        st[2 * C:].fill_(float(x.shape[0]))
        rows.append(st)
    allst = torch.stack(rows)
    mean, rstd, inv_total = torch.empty(C, device=DEV), torch.empty(C, device=DEV), torch.empty(1, device=DEV)
    be.bn_sync_combine(allst, EPS, MOMENTUM, rm, rv, mean, rstd, inv_total)
    keep_y = act != ops.ACT_NONE and with_res
    ys = []
    for x, r in zip(xs, rs):
        y = torch.empty_like(x)
        be.bn_apply(x, mean, rstd, gamma, beta, r if with_res else None, act, y)
        ys.append(y)
    local = []
    for x, dy, y in zip(xs, dys, ys):
        s = torch.empty((2, C), device=DEV)
        be.bn_bwd_reduce(x, dy, y if keep_y else None, gamma, beta, mean, rstd, act, s[0], s[1])
        local.append(s)
    sums = local[0].clone()
    for s in local[1:]:
        sums += s
    glob = sums * inv_total
    dxs, dress = [], []
    for x, dy, y in zip(xs, dys, ys):
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if with_res else None
        be.bn_bwd_apply(x, dy, y if keep_y else None, gamma, beta, mean, rstd, glob[0], glob[1], 1.0, act, dx, dres)
        dxs.append(dx)
        dress.append(dres)
    out = dict(y=torch.cat(ys).cpu(), dx=torch.cat(dxs).cpu(), dgamma=sums[1].cpu(), dbeta=sums[0].cpu(), running_mean=rm.cpu(), running_var=rv.cpu(),
               mean=mean.cpu(), rstd=rstd.cpu())
    if with_res:
        out["dres"] = torch.cat(dress).cpu()
    return out, allst, float(inv_total.item())


@pytest.mark.parametrize("name,act,with_res", VARIANTS, ids=VID)
@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("C", list(SYNC_R))
def test_sync_batchnorm_phases_match_full_batch(C, world, name, act, with_res):
    """W ranks x (their rows) through bn_stats / bn_sync_combine / bn_apply / bn_bwd_reduce / bn_bwd_apply == fp64 BatchNorm over all rows,
    and == bn_train_fwd / bn_train_bwd on the concatenated rows (the kernel-level form of "2 ranks x B/2 == 1 rank x B")"""
    R = SYNC_R[C]
    x, res, gamma, beta, rm, rv, dy = bn_data(R, C)
    ref, dy = reference(x, res, gamma, beta, rm, rv, dy, act, with_res)
    counts = rank_rows(R, world)
    xs, rs, dys = (list(t.to(DEV, copy=True).split(counts)) for t in (x, res, dy))
    gg, bg, rmg, rvg = gamma.to(DEV, copy=True), beta.to(DEV, copy=True), rm.to(DEV, copy=True), rv.to(DEV, copy=True)
    got, allst, inv_total = sync_phases(xs, rs, dys, gg, bg, rmg, rvg, act, with_res)
    what = f"C={C} ranks={counts} {name}"
    assert torch.equal(allst[:, 2 * C].cpu(), torch.tensor(counts, dtype=torch.float32))
    assert inv_total == float(torch.tensor(1.0 / R, dtype=torch.float32)), f"{what}: inv_total {inv_total!r} is not float32(1/{R})"
    # the combined mean is formed from per-rank fp32 means: up to one ulp (see mean_rounding)
    check_all(got, ref, what, mean_ulps=1.0)
    check_all(got, ref, f"{what} vs bn_train", target=run_train_fn(x, res, gamma, beta, rm, rv, dy, act, with_res), mean_ulps=1.0)


def test_sync_combine_without_running_stats_writes_only_its_outputs():
    """bn_sync_combine(running_mean = running_var = None): the same mean / rstd / 1 / total as with them, and nothing written outside those"""
    C, counts = 64, [7, 1000, 993]
    x = bn_data(sum(counts), C)[0].to(DEV, copy=True)
    be = ops._be()
    rows = []
    for xr in x.split(counts):
        st = torch.empty(2 * C + 1, device=DEV)
        be.bn_stats(xr, st[:C], st[C:2 * C])
        st[2 * C:].fill_(float(xr.shape[0]))
        rows.append(st)
    allst = torch.stack(rows)
    allst0 = allst.clone()
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    mean, rstd, inv_total = torch.empty(C, device=DEV), torch.empty(C, device=DEV), torch.empty(1, device=DEV)
    be.bn_sync_combine(allst, EPS, MOMENTUM, rm, rv, mean, rstd, inv_total)
    buf = torch.full((2, C + 8), float("nan"), device=DEV)  # outputs inside sentinel-filled buffers: a stray write shows up in the margins
    tbuf = torch.full((8,), float("nan"), device=DEV)
    be.bn_sync_combine(allst, EPS, MOMENTUM, None, None, buf[0, :C], buf[1, :C], tbuf[:1])
    assert torch.equal(buf[0, :C], mean) and torch.equal(buf[1, :C], rstd) and torch.equal(tbuf[:1], inv_total)
    assert bool(buf[:, C:].isnan().all()) and bool(tbuf[1:].isnan().all()), "bn_sync_combine wrote outside mean / rstd / inv_total"
    assert torch.equal(allst, allst0)


def test_sync_batchnorm_fn_on_one_gpu(tmp_path):
    """SyncBatchNormTrainFn over a world-size-1 NCCL group == BatchNormTrainFn: the device-side wiring (the count fill, the all_gather_into_tensor
    layout, sums * inv_total) that the CPU test with the gloo backend and the reference operators cannot reach"""
    import torch.distributed as dist

    if not dist.is_available() or not dist.is_nccl_available():
        pytest.skip("torch.distributed without NCCL")
    if dist.is_initialized():
        pytest.skip("a default process group already exists")
    C = 64
    R = LARGE_R[C]
    dist.init_process_group("nccl", store=dist.FileStore(str(tmp_path / "store"), 1), rank=0, world_size=1,
                            device_id=torch.device(DEV, torch.cuda.current_device()))
    try:
        for name, act, with_res in VARIANTS:
            x, res, gamma, beta, rm, rv, dy = bn_data(R, C)
            ref, dy = reference(x, res, gamma, beta, rm, rv, dy, act, with_res)
            full = run_train_fn(x, res, gamma, beta, rm, rv, dy, act, with_res)
            xg, gg, bg = (t.to(DEV, copy=True).requires_grad_(True) for t in (x, gamma, beta))
            rg = res.to(DEV, copy=True).requires_grad_(True) if with_res else None
            rmg, rvg = rm.to(DEV, copy=True), rv.to(DEV, copy=True)
            yg = A.SyncBatchNormTrainFn.apply(xg, gg, bg, rmg, rvg, rg, act, EPS, MOMENTUM, None)
            saved = yg.grad_fn.saved_tensors  # (x, gamma, beta, mean, rstd, y or None, inv_total)
            assert float(saved[6].item()) == float(torch.tensor(1.0 / R, dtype=torch.float32))
            yg.backward(dy.to(DEV, copy=True))
            got = dict(y=yg.detach().cpu(), dx=xg.grad.cpu(), dgamma=gg.grad.cpu(), dbeta=bg.grad.cpu(), running_mean=rmg.cpu(), running_var=rvg.cpu(),
                       mean=saved[3].cpu(), rstd=saved[4].cpu())
            if with_res:
                got["dres"] = rg.grad.cpu()
            check_all(got, ref, f"SyncBatchNormTrainFn {name} vs BatchNormTrainFn", target=full)
            check_all(got, ref, f"SyncBatchNormTrainFn {name}")
    finally:
        dist.destroy_process_group()


# ---- FrozenBatchNorm2d: the affine of the running statistics, nothing trained ------------------------------------------------------------
@pytest.mark.parametrize("name,act,with_res", VARIANTS, ids=VID)
@pytest.mark.parametrize("C", [64, 96])  # C = 64 at R = 36,871: the cf kernels with their 2-row loop; C = 96: the generic kernels
def test_frozen_batchnorm_matches_fp64(C, name, act, with_res):
    """FrozenBatchNormFn: y and dx against fp64 (x - running_mean) * gamma / sqrt(running_var + eps) + beta (+ res, then act); the running
    buffers stay bit-identical and weight / bias get no gradient"""
    R = LARGE_R[C]
    x, res, gamma, beta, rm, rv, dy = bn_data(R, C)
    xd, rd = x.double().requires_grad_(True), res.double().requires_grad_(True)
    zb = (xd - rm.double()) * (gamma.double() / (rv.double() + EPS).sqrt()) + beta.double()
    z = zb + rd if with_res else zb
    dy = masked_dy(dy, z.detach(), act)
    yr = ACT_FN[act](z)
    yr.backward(dy.double())
    bn = torch.nn.BatchNorm2d(C).to(DEV)
    with torch.no_grad():
        bn.weight.copy_(gamma)
        bn.bias.copy_(beta)
        bn.running_mean.copy_(rm)
        bn.running_var.copy_(rv)
    rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
    xg = x.to(DEV, copy=True).requires_grad_(True)
    rg = res.to(DEV, copy=True).requires_grad_(True) if with_res else None
    yg = A.batch_norm_train(xg.reshape(1, 1, R, C), bn, None if rg is None else rg.reshape(1, 1, R, C), act, frozen=True)
    yg.backward(dy.to(DEV, copy=True).reshape(1, 1, R, C))
    what = f"frozen C={C} R={R} {name}"
    check(yg.reshape(R, C), yr, f"{what} y", FWD_TOL, floor=zb.detach().abs().amax(0) + (res.double().abs().amax(0) if with_res else 0.0))
    check(xg.grad, xd.grad, f"{what} dx", GRAD_TOL)
    if with_res:
        check(rg.grad, rd.grad, f"{what} dres", FWD_TOL)
    assert torch.equal(bn.running_mean, rm0) and torch.equal(bn.running_var, rv0), "the running buffers must not change"
    assert int(bn.num_batches_tracked) == 0
    assert bn.weight.grad is None and bn.bias.grad is None
