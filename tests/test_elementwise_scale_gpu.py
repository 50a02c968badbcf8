"""The HBM-bound kernels (csrc/elementwise.cu, csrc/loss.cu) at the batch-32 sizes of the ResNet101-UNet at 320x320,
where every thread of their capped grid-stride loops runs several iterations.

Every case asserts, from the device's SM count and the launch model of oracle/elementwise_checks.py, that each thread
(or each pixel lane of a reduction block) owns at least 3 work items, and the cases marked ragged also assert a partial
last pass (for the BatchNorm kernels: a thread whose second group falls off the end).  Shapes are the network's layers
"C@HxW" at batch 32, or at a larger batch where 32 images do not give every thread 3 items; one tensor case lives in
device memory at a time.  References and bars: oracle/elementwise_checks.py."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import unet_oracle as O
from oracle.conv_checks import assert_bound, assert_exact, assert_same
from oracle.elementwise_checks import (ADAM_EPS, BETAS, BF, BN, CSUM, EPS, F64, GRAD_SCALE, LOSS_N, LOSS_S, POOL,
                                       SIZE_C, STEPS, WD, adam_lr, affine, assert_bf16, assert_reduce_regime,
                                       assert_stride_regime, bn_bwd_reduce_ref, bn_case, check_adam, check_bn_apply,
                                       check_bn_bwd_apply, check_fin, check_reduction, chunks, classifier_bwd_ref,
                                       classifier_fwd_ref, free_case, gen, ids, ints, loss_case, loss_ref, pool_ref,
                                       rand, randn, resnet101_unet_layout, with_ties)

pytestmark = pytest.mark.gpu


# =====================================================================================================================
# BatchNorm: train-apply (finalisation folded in), finalize + eval apply, backward apply and reduce, channel sums
BN_FWD = [(c, res, relu) for c in BN for res in (0, 1, 2) for relu in (True, False)]


@pytest.mark.parametrize("c,res,relu", [pytest.param(*p, id="%s-res%d-%s" % (ids([p[0]])[0], p[1], "relu" if p[2]
                                                                            else "linear")) for p in BN_FWD])
def test_bn_forward(mcb, cuda, c, res, relu):
    """bn_train_apply (statistics finalised in the apply pass, mean / invstd published, running statistics updated)
    and bn_finalize + bn_apply (the eval-mode apply), with no residual, an activation residual, or a downsample
    BatchNorm residual"""
    from mcb200 import ops
    n, h, w, ch = c["n"], c["h"], c["w"], c["c"]
    pixels = n * h * w
    assert_stride_regime(pixels * ch // 8, 256, pair=True, ragged=c.get("ragged", False))
    d = bn_case(c)
    z = d["z"]
    resid = d["r"] if res else None
    e = lambda: torch.empty(ch, device=cuda)
    # train-apply
    rm, rv, mean, inv = d["rm0"].clone(), d["rv0"].clone(), e(), e()
    tr = ops.make_bn_train(d["zstats"], d["gamma"], d["beta"], rm, rv, mean, inv)
    rtr = rbn = None
    if res == 2:
        rrm, rrv, rmean, rinv = d["rrm0"].clone(), d["rrv0"].clone(), e(), e()
        rtr = ops.make_bn_train(d["rstats"], d["rgamma"], d["rbeta"], rrm, rrv, rmean, rinv)
    y = torch.empty_like(z)
    ops.bn_train_apply(z, tr, y, relu, resid, rtr)
    check_fin(dict(mean=mean, invstd=inv, rm=rm, rv=rv), d["zstats"], pixels, d["rm0"], d["rv0"], "bn_train_apply")
    if res == 2:
        check_fin(dict(mean=rmean, invstd=rinv, rm=rrm, rv=rrv), d["rstats"], pixels, d["rrm0"], d["rrv0"],
                  "bn_train_apply residual BN")
        rbn = affine(d["rgamma"], d["rbeta"], rmean, rinv)
    check_bn_apply(y, z, affine(d["gamma"], d["beta"], mean, inv), relu, "bn_train_apply", resid, rbn)
    # finalize + eval apply
    rm, rv, mean, inv, scale, shift = d["rm0"].clone(), d["rv0"].clone(), e(), e(), e(), e()
    ops.bn_finalize(d["zstats"], pixels, d["gamma"], d["beta"], rm, rv, scale, shift, mean, inv)
    check_fin(dict(mean=mean, invstd=inv, rm=rm, rv=rv), d["zstats"], pixels, d["rm0"], d["rv0"], "bn_finalize")
    rscale = rshift = None
    if res == 2:
        rscale, rshift, rmean, rinv = e(), e(), e(), e()
        ops.bn_finalize(d["rstats"], pixels, d["rgamma"], d["rbeta"], None, None, rscale, rshift, rmean, rinv)
        rbn = (rscale, rshift, rshift.abs())
    y = torch.empty_like(z)
    ops.bn_apply(z, scale, shift, y, relu, resid, rscale, rshift)
    check_bn_apply(y, z, (scale, shift, shift.abs()), relu, "bn_apply", resid, rbn)


BN_BWD = [(c, mask, gout) for c in BN for mask, gout in ((False, "none"), (True, "none"), (True, "store"),
                                                         (True, "accumulate"), (False, "accumulate"))]


@pytest.mark.parametrize("c,mask,gout", [pytest.param(*p, id="%s-%s-gout_%s" % (ids([p[0]])[0], "mask" if p[1] else
                                                                                "nomask", p[2])) for p in BN_BWD])
def test_bn_bwd_apply(mcb, cuda, c, mask, gout):
    """dz = gamma invstd (g - dbeta / M - xhat dgamma / M), g = dy [* (y > 0)]; g_out = g stored or added"""
    from mcb200 import ops
    n, h, w, ch = c["n"], c["h"], c["w"], c["c"]
    pixels = n * h * w
    assert_stride_regime(pixels * ch // 8, 256, pair=True, ragged=c.get("ragged", False))
    d = bn_case(c)
    z, dy = d["z"], d["dy"]
    ym = d["ym"] if mask else None
    dz = torch.empty_like(z)
    g_out = {"none": None, "store": torch.empty_like(z), "accumulate": d["r"].clone()}[gout]
    ops.bn_bwd_apply(dy, ym, z, d["bmean"], d["binv"], d["bgamma"], d["dbeta"], d["dgamma"], dz, g_out,
                     gout == "accumulate")
    check_bn_bwd_apply(dz, dy, ym, z, d["bmean"], d["binv"], d["bgamma"], d["dbeta"], d["dgamma"], pixels,
                       "bn_bwd_apply dz")
    if gout != "none":
        g = dy.masked_fill(ym <= 0, 0) if mask else dy
        if gout == "accumulate":
            g = (d["r"].float() + g.float()).to(BF)
        assert_exact(g_out, g, "bn_bwd_apply g_out (%s)" % gout)


@pytest.mark.parametrize("c,kind", [pytest.param(c, k, id="%s-%s" % (i, k)) for c, i in zip(BN, ids(BN))
                                    for k in ("real-mask", "real-nomask", "exact")])
def test_bn_bwd_reduce(mcb, cuda, c, kind):
    """dbeta += sum g, dgamma += sum g xhat over the pixels (g = dy [* (y > 0)]) into prefilled outputs.  exact: dy in
    {-1, 0, 1}, z in {-2 .. 2}, mean 0, invstd 1, so xhat = z and every partial sum is an integer"""
    from mcb200 import ops
    n, h, w, ch = c["n"], c["h"], c["w"], c["c"]
    pixels = n * h * w
    assert_reduce_regime(pixels, ch, ragged=c.get("ragged", False))
    d = bn_case(c)
    g = gen("bnred", c["desc"], kind)
    ym = None if kind == "real-nomask" else d["ym"]
    if kind == "exact":
        dy, z = ints(g, -1, 1, n, h, w, ch).to(BF), ints(g, -2, 2, n, h, w, ch).to(BF)
        mean, inv = torch.zeros(ch, device=cuda), torch.ones(ch, device=cuda)
        pre_b, pre_g = ints(g, -50, 50, ch), ints(g, -50, 50, ch)
    else:
        dy, z, mean, inv = d["dy"], d["z"], d["bmean"], d["binv"]
        pre_b, pre_g = randn(g, ch) * 10, randn(g, ch) * 10
    runs = []
    for _ in range(2):
        db, dgm = pre_b.clone(), pre_g.clone()
        ops.bn_bwd_reduce(dy, ym, z, mean, inv, db, dgm)
        runs.append((db, dgm))
    sb, sg, ab, ag = bn_bwd_reduce_ref(dy, ym, z, mean, inv)
    (db, dgm), (db2, dgm2) = runs
    check_reduction(db, pre_b, sb, ab, kind == "exact", "dbeta")
    check_reduction(dgm, pre_g, sg, ag, kind == "exact", "dgamma")
    assert_same(db, db2, "dbeta")
    assert_same(dgm, dgm2, "dgamma")


@pytest.mark.parametrize("c,exact", [pytest.param(c, e, id="%s-%s" % (i, e)) for c, i in zip(CSUM, ids(CSUM))
                                     for e in ("real", "exact")])
def test_channel_sum(mcb, cuda, c, exact):
    """out += sum over pixels, into a prefilled out"""
    from mcb200 import ops
    n, h, w, ch = c["n"], c["h"], c["w"], c["c"]
    assert_reduce_regime(n * h * w, ch, ragged=c.get("ragged", False))
    g = gen("csum", c["desc"], exact)
    if exact == "exact":
        x, pre = ints(g, -1, 1, n, h, w, ch).to(BF), ints(g, -50, 50, ch)
    else:
        x, pre = randn(g, n, h, w, ch).to(BF), randn(g, ch) * 10
    runs = []
    for _ in range(2):
        out = pre.clone()
        ops.channel_sum(x, out)
        runs.append(out)
    v = x.view(-1, ch)
    check_reduction(runs[0], pre, v.sum(0, dtype=F64), v.abs().sum(0, dtype=F64), exact == "exact", "channel_sum")
    assert_same(runs[0], runs[1], "channel_sum")


# =====================================================================================================================
# synchronised BatchNorm on one device: two halves with the global statistics reproduce the full batch
SYNC = BN[1]   # 64@80x80, batch 32


def test_sync_bn_train_apply_halves(mcb, cuda):
    """what two ranks compute: bn_train_apply(count_scale=2) on each half with the all-reduced [sum, sumsq] equals the
    matching half of the full-batch run bitwise -- output, mean, invstd and running statistics, residual BN included"""
    from mcb200 import ops
    c = SYNC
    n, h, w, ch = c["n"], c["h"], c["w"], c["c"]
    assert n == 32
    assert_stride_regime(n // 2 * h * w * ch // 8, 256, pair=True)
    d = bn_case(c)
    z, r = d["z"], d["r"]

    def run(sl, scale):
        st = [d["rm0"].clone(), d["rv0"].clone()] + [torch.empty(ch, device=cuda) for _ in range(2)]
        rst = [d["rrm0"].clone(), d["rrv0"].clone()] + [torch.empty(ch, device=cuda) for _ in range(2)]
        tr = ops.make_bn_train(d["zstats"], d["gamma"], d["beta"], *st)
        rtr = ops.make_bn_train(d["rstats"], d["rgamma"], d["rbeta"], *rst)
        y = torch.empty_like(z[sl])
        ops.bn_train_apply(z[sl], tr, y, True, r[sl], rtr, count_scale=scale)
        return y, st + rst

    y, st = run(slice(0, n), 1)
    for k in range(2):
        sl = slice(k * n // 2, (k + 1) * n // 2)
        yk, stk = run(sl, 2)
        assert_same(yk, y[sl], "half %d output" % k)
        for name, a, b in zip(("running_mean", "running_var", "mean", "invstd") * 2, stk, st):
            assert_same(a, b, "half %d %s" % (k, name))


def test_sync_bn_bwd_apply_halves(mcb, cuda):
    """bn_bwd_apply(count_scale=2) on each half with the global dbeta / dgamma equals the matching half of the
    full-batch run bitwise (dz and the stored g_out)"""
    from mcb200 import ops
    c = SYNC
    n, h, w, ch = c["n"], c["h"], c["w"], c["c"]
    assert_stride_regime(n // 2 * h * w * ch // 8, 256, pair=True)
    d = bn_case(c)

    def run(sl, scale):
        dz, g = torch.empty_like(d["z"][sl]), torch.empty_like(d["z"][sl])
        ops.bn_bwd_apply(d["dy"][sl], d["ym"][sl], d["z"][sl], d["bmean"], d["binv"], d["bgamma"], d["dbeta"],
                         d["dgamma"], dz, g, False, count_scale=scale)
        return dz, g

    dz, g = run(slice(0, n), 1)
    for k in range(2):
        sl = slice(k * n // 2, (k + 1) * n // 2)
        dzk, gk = run(sl, 2)
        assert_same(dzk, dz[sl], "half %d dz" % k)
        assert_same(gk, g[sl], "half %d g_out" % k)


# =====================================================================================================================
def test_bn_eval_params_batched(mcb, cuda):
    """every BatchNorm of UNetResNet(101) in one launch equals per-BN bn_eval_params bitwise and leaves the floats past
    each BatchNorm's C untouched"""
    from mcb200 import _lib as L
    from mcb200 import ops
    _, widths = resnet101_unet_layout()
    assert len(widths) == 104 and min(widths) == 64 and max(widths) == 2048
    pad = 37
    offs, total = [], 0
    for ch in widths:
        offs.append(total)
        total += ch + pad
    g = gen("eval-batched")
    gamma, beta, rm, rv = rand(g, total) + 0.5, randn(g, total), randn(g, total), rand(g, total) + 0.05
    sentinel = 12345.5
    scale, shift, scale1, shift1 = (torch.full((total,), sentinel, device=cuda) for _ in range(4))
    rows = [[t.data_ptr() + 4 * o for t in (gamma, beta, rm, rv, scale, shift)] + [ch] for o, ch in zip(offs, widths)]
    table = torch.tensor(rows, dtype=torch.int64, device=cuda)
    L.fcall("mcb_bn_eval_params_batched", table.data_ptr(), len(widths), max(widths), EPS)
    for o, ch in zip(offs, widths):
        s = slice(o, o + ch)
        ops.bn_eval_params(gamma[s], beta[s], rm[s], rv[s], scale1[s], shift1[s], eps=EPS)
    torch.cuda.synchronize()
    assert_same(scale, scale1, "batched scale")
    assert_same(shift, shift1, "batched shift")
    for o, ch in zip(offs, widths):
        s = slice(o + ch, o + ch + pad)
        assert bool((scale[s] == sentinel).all() and (shift[s] == sentinel).all()), "bytes past C=%d written" % ch


# =====================================================================================================================
# 2x2 max-pool
@pytest.mark.parametrize("c", POOL, ids=ids(POOL))
def test_maxpool(mcb, cuda, c):
    """forward max, and the backward routing every gradient to the FIRST maximum of its window in scan order (pool_ref),
    stored (all four positions overwritten) or added to an existing gradient"""
    from mcb200 import ops
    n, h, w, ch = c["n"], c["h"], c["w"], c["c"]
    ho, wo = h // 2, w // 2
    assert_stride_regime(n * ho * wo * ch // 8, 256, ragged=c.get("ragged", False))
    g = gen("pool", c["desc"])
    tied = ints(g, 0, 2, n, h, w, ch) * 0.5                  # {0, 0.5, 1}: ties inside most windows
    x = torch.where(rand(g, n, h, w, ch) < 0.5, tied, randn(g, n, h, w, ch)).to(BF)
    x[0, 0:2, 0:2] = 1.5                                     # fully tied windows
    x[1 % n, 2:4, 2:4] = -0.75
    dy = randn(g, n, ho, wo, ch).to(BF)
    assert bool((x[:, 0::2, 0::2] == x[:, 0::2, 1::2]).any()), "no ties"
    m, routed = pool_ref(x, dy)
    assert_exact(ops.maxpool2_fwd(x), m, "maxpool2_fwd")
    del m
    dx = randn(g, n, h, w, ch).to(BF)
    ops.maxpool2_bwd(x, dy, dx, False)
    assert_exact(dx, routed, "maxpool2_bwd store")
    pre = randn(g, n, h, w, ch).to(BF)
    dx = pre.clone()
    ops.maxpool2_bwd(x, dy, dx, True)
    assert_exact(dx, (pre.float() + routed.float()).to(BF), "maxpool2_bwd accumulate")


# =====================================================================================================================
# the final 1x1 classifier (C = 32, K = 2) at 32 x 320 x 320
@pytest.mark.parametrize("exact", ["real", "exact"])
def test_final_conv(mcb, cuda, exact):
    """logits = W x + b; backward dx = (x > 0) W^T dlogits, dW += sum dlogits x^T, db += sum dlogits into prefilled
    dW / db.  exact: x in {0, 1, 2}, dlogits in {-1, 0, 1}, weights and bias in multiples of 1/8"""
    from mcb200 import ops
    n, h, w, ch, k = 32, 320, 320, 32, 2
    pixels = n * h * w
    assert_stride_regime(pixels, 256)                   # final_conv_fwd: grid_for(pixels, 256)
    assert_stride_regime(pixels, 128, 4, ragged=True)   # final_conv_bwd: grid_for(pixels, 128, 4)
    exact = exact == "exact"
    g = gen("final", exact)
    if exact:
        x = ints(g, 0, 2, n, h, w, ch).to(BF)
        wt, b = ints(g, -16, 16, k, ch) / 8, ints(g, -8, 8, k) / 8
        dl = ints(g, -1, 1, n, k, h, w)
        pre_w, pre_b = ints(g, -50, 50, k * ch), ints(g, -50, 50, k)
    else:
        x = randn(g, n, h, w, ch).clamp_min(0).to(BF)
        wt, b = randn(g, k, ch) * 0.2, randn(g, k)
        dl = randn(g, n, k, h, w)
        pre_w, pre_b = randn(g, k * ch), randn(g, k)
    logits = torch.empty(n, k, h, w, device=cuda)
    ops.final_conv_fwd(x, wt.view(-1), b, logits)
    runs = []
    for _ in range(2):
        dx, dw, db = torch.empty_like(x), pre_w.clone(), pre_b.clone()
        ops.final_conv_bwd(x, wt.view(-1), dl, dx, dw, db)
        runs.append((dx, dw, db))
    sw = sb = aw = ab = 0
    dx = runs[0][0]
    for sl in chunks(n, h * w * ch):
        lg, la = classifier_fwd_ref(x[sl], wt, b)
        gx, ga, *sums = classifier_bwd_ref(x[sl], wt, dl[sl])
        sw, aw, sb, ab = (u + v for u, v in zip((sw, aw, sb, ab), sums))
        what = " [images %d:%d]" % (sl.start, sl.stop)
        if exact:
            assert_exact(logits[sl], lg, "final_conv_fwd" + what)
            assert_exact(dx[sl], gx, "final_conv_bwd dx" + what)
        else:
            assert_bound(logits[sl], lg, la, "final_conv_fwd" + what, rel=0.0)
            assert_bf16(dx[sl], gx, ga, "final_conv_bwd dx" + what)
    (dx, dw, db), (dx2, dw2, db2) = runs
    check_reduction(dw, pre_w, sw, aw, exact, "final_conv_bwd dW")
    check_reduction(db, pre_b, sb, ab, exact, "final_conv_bwd db")
    assert_same(dx, dx2, "final_conv_bwd dx")
    assert_same(dw, dw2, "final_conv_bwd dW")
    assert_same(db, db2, "final_conv_bwd db")


# =====================================================================================================================
# losses at 32 x 320 x 320
@pytest.mark.parametrize("mode", [0, 1], ids=["weighted_ce_dice", "plain_ce"])
def test_loss(mcb, cuda, mode):
    """loss_partials (the four global sums) + loss_grad (loss, dlogits) against the float64 mixed_loss /
    plain_ce_loss and their autograd gradients"""
    from mcb200 import ops
    pixels = LOSS_N * LOSS_S * LOSS_S
    assert_stride_regime(pixels, 256, ragged=True)
    logits, t = loss_case()
    tgt = t if mode == 0 else t[:, :1].contiguous()
    assert bool((t[:, 1] == 0).any() and (t[:, 1] > 0).any() and (t[:, 2] == 0).any())
    cfg = dict(size_c=SIZE_C)
    runs = []
    for _ in range(2):
        sums = torch.zeros(4, dtype=F64, device=cuda)
        ops.loss_partials(logits, tgt, sums, mode=mode, **cfg)
        runs.append(sums)
    assert_same(runs[0], runs[1], "loss sums")
    sums = runs[0]
    dlog, loss = torch.empty_like(logits), torch.zeros((), device=cuda)
    ops.loss_grad(logits, tgt, sums, dlog, loss, mode=mode, **cfg)
    # float64 reference
    lg = logits.double().requires_grad_(True)
    t64 = t.double()
    if mode == 0:
        ref = O.mixed_loss(lg, t64, imsize=(LOSS_S, LOSS_S))
    else:
        ref = O.plain_ce_loss(lg, t64[:, :1])
    ref.backward()
    ref = ref.detach()
    ref_sums, p, tol = loss_ref(logits, t, mode)
    # every term is non-negative: A = ref
    assert_bound(sums, ref_sums, ref_sums, "loss sums [I, P, T, S]", rel=0.0)
    assert_exact(sums[2], ref_sums[2], "loss sum T")
    assert abs(float(loss) - float(ref)) <= 1e-6 * abs(float(ref)), (float(loss), float(ref))
    assert_bound(dlog, lg.grad, 0.0, "dlogits", rel=0.0, extra=tol)
    if mode == 0:
        assert_bound(ops.softmax2(logits), p, 0.0, "softmax2", rel=0.0, extra=2.0 ** -18 * p)


# =====================================================================================================================
# fused Adam over the ResNet101-UNet parameter arena
def adam_zero_block(n):
    """parameters that are zero with zero gradients: v stays 0, the denominator is eps, the update 0"""
    return slice(n // 3, n // 3 + 4097)


def adam_init(n):
    g = gen("adam-init")
    p = randn(g, n) * 0.05
    p[adam_zero_block(n)] = 0
    return p


def adam_grad(n, t):
    """gradient magnitudes spread over 1e-8 .. 1, random signs, 10% zeros"""
    g = gen("adam-grad", t)
    grad = torch.pow(10.0, rand(g, n) * 8 - 8) * (ints(g, 0, 1, n) * 2 - 1) * (rand(g, n) >= 0.1)
    grad[adam_zero_block(n)] = 0
    return grad


@pytest.mark.parametrize("entry", ["adam_step", "adam_step_dyn"])
def test_adam_arena(mcb, cuda, entry):
    """STEPS steps over a vector the length of UNetResNet(101)'s fp32 arena, each checked from the kernel's own state;
    adam_step_dyn reads {lr, 1 - beta1^t, sqrt(1 - beta2^t)} from the device, as the captured train step does"""
    from mcb200 import ops
    n, _ = resnet101_unet_layout()
    assert_stride_regime(n, 256, ragged=True)
    free_case()
    p = adam_init(n)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    p16 = torch.empty(n, dtype=BF, device=cuda)
    hyper = torch.empty(3, device=cuda)
    for t in range(1, STEPS + 1):
        grad = adam_grad(n, t)
        p0, m0, v0 = p.clone(), m.clone(), v.clone()
        if entry == "adam_step":
            ops.adam_step(p, grad, m, v, p16, t, adam_lr(t), BETAS, ADAM_EPS, WD, GRAD_SCALE)
        else:
            hyper.copy_(torch.tensor(ops.adam_hyper(adam_lr(t), BETAS, t)))
            ops.adam_step_dyn(p, grad, m, v, p16, hyper, BETAS, ADAM_EPS, WD, GRAD_SCALE)
        check_adam(t, adam_lr(t), p0, m0, v0, grad, p, m, v, entry)
        assert_same(p16, p.to(BF), "%s bf16 copy, step %d" % (entry, t))
        zb = adam_zero_block(n)
        assert not bool(p[zb].any() or m[zb].any() or v[zb].any())
        del p0, m0, v0, grad


def test_adam_dyn_segments_equal_adam_step(mcb, cuda):
    """one adam_step_dyn launch per arena slice (odd offsets), as the captured train step launches one per backward
    segment, with hyper computed as FusedTrainStep.step computes it, equals adam_step over the whole arena bitwise;
    the elements between and after the slices stay bitwise untouched"""
    from mcb200 import ops
    n, _ = resnet101_unet_layout()
    a, b = (n // 7) | 1, (n // 2) | 1
    c, e = b + 4099, n - 5
    slices, gaps = [(0, a), (a, b), (c, e)], [(b, c), (e, n)]
    for lo, hi in slices:
        assert_stride_regime(hi - lo, 256)
    free_case()
    pa = adam_init(n)
    ma, va, ha = torch.zeros_like(pa), torch.zeros_like(pa), torch.zeros(n, dtype=BF, device=cuda)
    pb, mb, vb, hb = pa.clone(), ma.clone(), va.clone(), ha.clone()
    hyper = torch.empty(3, device=cuda)
    for t in range(1, STEPS + 1):
        grad = adam_grad(n, t)
        ops.adam_step(pa, grad, ma, va, ha, t, adam_lr(t), BETAS, ADAM_EPS, WD, GRAD_SCALE)
        hyper.copy_(torch.tensor(ops.adam_hyper(adam_lr(t), BETAS, t)))
        before = [[x[lo:hi].clone() for x in (pb, mb, vb, hb)] for lo, hi in gaps]
        for lo, hi in slices:
            ops.adam_step_dyn(pb[lo:hi], grad[lo:hi], mb[lo:hi], vb[lo:hi], hb[lo:hi], hyper, BETAS, ADAM_EPS, WD,
                              GRAD_SCALE)
        for lo, hi in slices:
            for name, x, y in zip("pmvh", (pb, mb, vb, hb), (pa, ma, va, ha)):
                assert_same(x[lo:hi], y[lo:hi], "step %d slice %d:%d %s" % (t, lo, hi, name))
        for (lo, hi), old in zip(gaps, before):
            for name, x, y in zip("pmvh", (pb, mb, vb, hb), old):
                assert_same(x[lo:hi], y, "step %d gap %d:%d %s" % (t, lo, hi, name))
        del grad, before


# =====================================================================================================================
# layout conversion, stem im2col, fp32 -> bf16
def test_layout_conversions(mcb, cuda):
    from mcb200 import ops
    n, ch, h, w = 32, 3, 320, 320
    assert_stride_regime(n * ch * h * w, 256, ragged=True)
    free_case()
    g = gen("layout")
    x = with_ties(randn(g, n, ch, h, w), g)
    y = ops.nchw_to_nhwc_bf16(x)
    assert_same(y, x.permute(0, 2, 3, 1).to(BF), "nchw_f32_to_nhwc_bf16")
    assert_same(ops.nhwc_to_nchw_f32(y), y.permute(0, 3, 1, 2).float(), "nhwc_bf16_to_nchw_f32")


@pytest.mark.parametrize("w", [320, 300])
def test_stem_im2col(mcb, cuda, w):
    """col[n][oy][ox][k] = x[n][c][2 oy - 3 + ky][2 ox - 3 + kx] (zero outside), k = (ky * 7 + kx) * 3 + c < 147,
    zero for k in 147 .. 191.  Width 300: the last 32-pixel strip of each output row has 22 pixels"""
    from mcb200 import ops
    n, h = 32, 320
    wo = w // 2
    if w == 300:
        assert wo % 32
    free_case()
    g = gen("stem", w)
    x = with_ties(randn(g, n, 3, h, w), g)
    col = ops.stem_im2col(x)
    assert col.shape == (n, h // 2, wo, 192)
    for sl in chunks(n, 3 * h * w * 49 // 4):
        u = F.unfold(x[sl], 7, padding=3, stride=2)                     # (n, c * 49 + tap, pixels)
        ref = u.view(u.shape[0], 3, 49, h // 2, wo).permute(0, 3, 4, 2, 1).reshape(u.shape[0], h // 2, wo, 147)
        assert_same(col[sl, ..., :147], ref.to(BF), "stem_im2col [images %d:%d]" % (sl.start, sl.stop))
    assert not bool(col[..., 147:].any()), "stem_im2col: k >= 147 not zero"


def test_cast_f32_bf16(mcb, cuda):
    from mcb200 import ops
    n, _ = resnet101_unet_layout()
    assert_stride_regime(n, 256, ragged=True)
    free_case()
    g = gen("cast")
    x = with_ties(randn(g, n) * torch.pow(10.0, rand(g, n) * 6 - 3), g)
    assert_same(ops.cast_bf16(x, torch.empty(n, dtype=BF, device=cuda)), x.to(BF), "cast_f32_bf16")


# =====================================================================================================================
def test_host_rejections(mcb, cuda):
    """argument checks that return an error before any launch, leaving every output untouched"""
    from mcb200 import _lib as L
    from mcb200 import ops
    ch = 64
    z = torch.ones(2, 4, 4, ch, dtype=BF, device=cuda)
    pixels = z.numel() // ch
    stats = torch.cat([torch.full((ch,), float(pixels)), torch.full((ch,), float(pixels))]).to(cuda)
    vec = lambda v: torch.full((ch,), v, device=cuda)
    rm, rv, mean, inv = vec(7.0), vec(7.0), vec(7.0), vec(7.0)
    one, zero = vec(1.0), vec(0.0)
    tr = ops.make_bn_train(stats, one, zero, rm, rv, mean, inv)
    y = torch.full_like(z, 3.0)
    with pytest.raises(RuntimeError, match="stat_count"):
        L.fcall("mcb_bn_train_apply_global", z.data_ptr(), C.byref(tr), None, None, 1, y.data_ptr(), pixels,
                pixels - 1, ch, 0.1, 1e-5)
    with pytest.raises(RuntimeError, match="stat_count"):
        L.fcall("mcb_bn_bwd_apply_global", z.data_ptr(), None, z.data_ptr(), mean.data_ptr(), inv.data_ptr(),
                one.data_ptr(), zero.data_ptr(), zero.data_ptr(), y.data_ptr(), None, 0, pixels, pixels - 1, ch)
    with pytest.raises(RuntimeError, match="res_bn without residual"):
        ops.bn_train_apply(z, tr, y, True, None, tr)
    # C = 24: C / 8 = 3 does not divide 256
    z24, y24 = torch.ones(2, 4, 4, 24, dtype=BF, device=cuda), torch.full((2, 4, 4, 24), 3.0, dtype=BF, device=cuda)
    v24 = torch.ones(24, device=cuda)
    s24 = torch.ones(48, device=cuda)
    tr24 = ops.make_bn_train(s24, v24, v24, v24.clone(), v24.clone(), v24.clone(), v24.clone())
    with pytest.raises(RuntimeError, match="must divide 256"):
        ops.bn_apply(z24, v24, v24, y24, True)
    with pytest.raises(RuntimeError, match="must divide 256"):
        ops.bn_train_apply(z24, tr24, y24, True)
    with pytest.raises(RuntimeError, match="must divide 256"):
        ops.bn_bwd_apply(z24, None, z24, v24, v24, v24, v24, v24, y24)
    # the classifier backward is built for C = 32, K = 2 only
    x16 = torch.ones(1, 4, 4, 16, dtype=BF, device=cuda)
    dx16 = torch.full_like(x16, 3.0)
    dw, db = torch.full((32,), 3.0, device=cuda), torch.full((2,), 3.0, device=cuda)
    with pytest.raises(RuntimeError, match="32 -> 2"):
        ops.final_conv_bwd(x16, torch.ones(32, device=cuda), torch.ones(1, 2, 4, 4, device=cuda), dx16, dw, db)
    torch.cuda.synchronize()
    for name, t in (("y", y), ("y24", y24), ("dx", dx16), ("dw", dw), ("db", db)):
        assert bool((t == 3.0).all()), "%s written by a rejected call" % name
    for name, t in (("running_mean", rm), ("running_var", rv), ("mean", mean), ("invstd", inv)):
        assert bool((t == 7.0).all()), "%s written by a rejected call" % name
    assert bool((v24 == 1.0).all())
