"""NaN and +-Inf through the kernels of the train step and the inference forward, against torch.

A diverged run is only visible if its NaN travels: one NaN weight (what Adam leaves after one NaN gradient) must give a
NaN loss and NaN running statistics, as it does in the reference.  Every other test of the suite feeds finite operands,
so a kernel that quietly turns a NaN into 0 (fmaxf-based ReLU, a max-pool that skips NaN, a variance clamp) passes them.

assert_nonfinite_like: NaN, +Inf and -Inf of got sit at exactly ref's positions, and the finite elements meet the bar
the kernel already has in oracle/conv_checks.py or oracle/elementwise_checks.py.

A. Each kernel against torch, or against a float64 reference of oracle/elementwise_checks.py that follows torch's
   rules, the non-finite values planted in three kinds of place: inside the first tile or pass, in the ragged last tile
   or channel group, and in an element that the kernel's grid-stride loop (or persistent tile loop) reaches only on a
   later pass, at the batch-32 shapes of oracle/elementwise_checks.py.  torch's rules: relu(NaN) = NaN; max_pool2d's
   output is NaN if its window holds a NaN, and its index is the first maximum or the last NaN in scan order; a NaN
   BatchNorm variance makes invstd, scale, shift and the running variance NaN; relu's backward zeroes the gradient where
   y <= 0 only.
B. The whole network against the reference (baseline/torch_cudnn_unet.py in fp32, oracle.step_checks.reference_step):
   the eval forward with a NaN or +Inf input pixel or a NaN encoder weight, and the fused train step with a NaN encoder
   weight, eager and through the captured graph.
Signed zeros: for finite operands the kernels keep the bits they gave before NaN propagated (test_signed_zero).

Measured on an H100 80GB HBM3 at its 700 W power limit: the whole file takes about 2 minutes."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import conv_checks as CC
from oracle import elementwise_checks as EC
from oracle import make_golden_sigmoid_dice as SD
from oracle import step_checks as SC
from oracle.step_checks import no_tf32, rng_and_peak_memory  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

BF, F64 = torch.bfloat16, torch.float64
NAN, INF = float("nan"), float("inf")
NONFINITE = (NAN, INF, -INF)
_CACHE = {}   # conv_checks' references of CONV and GRAD


# ---------------------------------------------------------------------------------------------------------- helpers
def assert_nonfinite_like(got, ref, what, absref=None, rel=2.0 ** -8, extra=0.0, finite_ref=None):
    """NaN, +Inf, -Inf at exactly ref's positions; with absref given, conv_checks.assert_bound(absref, rel, extra) on
    the elements ref has finite, against finite_ref there if given.  The non-finite elements of absref and extra count
    as 0: a finite ref there is a ReLU or mask zero of a non-finite term, and got must equal it"""
    got = got.detach().double().cpu()
    ref = ref.detach().double().cpu()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    for name, kind in (("NaN", torch.isnan), ("+Inf", lambda t: t == INF), ("-Inf", lambda t: t == -INF)):
        g, r = kind(got), kind(ref)
        if not torch.equal(g, r):
            i = tuple(int(v) for v in (g != r).nonzero()[0])
            raise AssertionError("%s: %s at %d positions, the reference at %d; %d differ, first at %s: got %r, ref %r" % (
                what, name, int(g.sum()), int(r.sum()), int((g != r).sum()), i, float(got[i]), float(ref[i])))
    if absref is not None:
        keep = torch.isfinite(ref)
        fin = lambda t: t.detach().double().cpu().nan_to_num(0, 0, 0)[keep] if torch.is_tensor(t) else t
        want = ref if finite_ref is None else finite_ref.detach().double().cpu()
        CC.assert_bound(got[keep], want[keep], fin(absref), what, rel=rel, extra=fin(extra))


def plant(x, flat, values=NONFINITE):
    """x.view(-1)[flat[i]] = values[i % len(values)], in place"""
    v = x.view(-1)
    for i, f in enumerate(flat):
        v[f] = values[i % len(values)]
    return x


def cpu(t):
    return t.detach().cpu()


# =====================================================================================================================
# A. kernels
# =====================================================================================================================
# ---------------------------------------------------------------------------------- BatchNorm apply (train and eval)
BN_CASES = [EC.BN[1], EC.BN[10]]      # 64@80x80 at batch 32; 64@97x101 x31, a partial last pass


def poisoned_bn(c):
    def make():
        d = EC.bn_case(c)
        z, r = d["z"].clone(), d["r"].clone()
        ch = z.shape[-1]
        groups = EC.stride_places(z.numel() // 8, 256, pair=True)
        # the non-finite values of z at channels 1, 4, 6 of each 8-channel group, r's at 2, 5, 7: both in the last one
        plant(z, [g * 8 + j for g in groups for j in (1, 4, 6)])
        plant(r, [g * 8 + j for g in groups for j in (2, 5, 7)])
        plant(z, [z.numel() - ch + 3], (NAN,))          # the last pixel's first channel group
        return dict(d, z=z, r=r)
    return EC.cached(("nonfinite bn", c["desc"]), make)


@pytest.mark.parametrize("c,res,relu", [pytest.param(c, res, relu, id="%s-res%d-%s" % (
    c["desc"].replace(" ", "_"), res, "relu" if relu else "linear")) for c in BN_CASES for res in (0, 1, 2)
    for relu in (True, False)])
def test_bn_apply_nonfinite(mcb, cuda, c, res, relu):
    """bn_train_apply and bn_finalize + bn_apply with NaN / +-Inf in z (and in the residual): the statistics are those
    of the finite z, so only the planted elements are non-finite, and ReLU must keep each NaN a NaN"""
    from mcb200 import ops
    d = poisoned_bn(c)
    z, ch = d["z"], d["z"].shape[-1]
    resid = d["r"] if res else None
    e = lambda: torch.empty(ch, device=cuda)
    rm, rv, mean, inv = d["rm0"].clone(), d["rv0"].clone(), e(), e()
    tr = ops.make_bn_train(d["zstats"], d["gamma"], d["beta"], rm, rv, mean, inv)
    rtr = rbn = None
    if res == 2:
        rmean, rinv = e(), e()
        rtr = ops.make_bn_train(d["rstats"], d["rgamma"], d["rbeta"], d["rrm0"].clone(), d["rrv0"].clone(), rmean, rinv)
    y = torch.empty_like(z)
    ops.bn_train_apply(z, tr, y, relu, resid, rtr)
    if res == 2:
        rbn = EC.affine(d["rgamma"], d["rbeta"], rmean, rinv)
    ref, a = EC.bn_apply_ref(z, EC.affine(d["gamma"], d["beta"], mean, inv), relu, resid, rbn)
    assert_nonfinite_like(y, ref, "bn_train_apply", 0.0, extra=2.0 ** -20 * a)
    scale, shift = e(), e()
    ops.bn_finalize(d["zstats"], z.numel() // ch, d["gamma"], d["beta"], None, None, scale, shift, e(), e())
    rscale = rshift = None
    if res == 2:
        rscale, rshift = e(), e()
        ops.bn_finalize(d["rstats"], z.numel() // ch, d["rgamma"], d["rbeta"], None, None, rscale, rshift, e(), e())
        rbn = (rscale, rshift, rshift.abs())
    y = torch.empty_like(z)
    ops.bn_apply(z, scale, shift, y, relu, resid, rscale, rshift)
    ref, a = EC.bn_apply_ref(z, (scale, shift, shift.abs()), relu, resid, rbn)
    assert_nonfinite_like(y, ref, "bn_apply", 0.0, extra=2.0 ** -20 * a)


# ------------------------------------------------------------------------------ BatchNorm statistics finalisation
def bn_stats_case():
    """z (N, H, W, C) bf16 at 64@80x80, batch 32, with non-finite values in a few channels: one NaN (3), one +Inf (10),
    one -Inf (17), +Inf and -Inf (24: the sum reaches Inf - Inf), two +Inf (40), a NaN in the last channel (63)"""
    def make():
        d = EC.bn_case(EC.BN[1])
        z = d["z"].clone()
        n, h, w, ch = z.shape
        px = n * h * w
        at = lambda p, cc: p * ch + cc
        plant(z, [at(17, 3), at(px // 2, 10), at(px - 1, 17), at(100, 24), at(px - 7, 24), at(3, 40), at(px // 3, 40),
                  at(px - 1, 63)], (NAN, INF, -INF, INF, -INF, INF, INF, NAN))
        return dict(d, z=z, zstats=EC.channel_stats(z))
    return EC.cached(("nonfinite bnstats",), make)


def torch_bn_train(z, gamma, beta, rm0, rv0):
    """torch.native_batch_norm(training=True) in float64 on the CPU: y, mean, invstd, running mean and variance"""
    x = z.double().cpu().permute(0, 3, 1, 2)
    rm, rv = rm0.double().cpu().clone(), rv0.double().cpu().clone()
    y, mean, invstd = torch.native_batch_norm(x, gamma.double().cpu(), beta.double().cpu(), rm, rv, True, EC.MOM,
                                              EC.EPS)
    return y.permute(0, 2, 3, 1), mean, invstd, rm, rv


@pytest.mark.parametrize("entry", ["bn_finalize", "bn_train_apply"])
def test_bn_statistics_nonfinite(mcb, cuda, entry):
    """mean, invstd, scale, shift, running mean and variance of the finalisation (bn_finalize, and the copy folded into
    bn_train_apply through make_bn_train) against torch's training-mode batch_norm; bn_train_apply's output too"""
    from mcb200 import ops
    d = bn_stats_case()
    z, ch = d["z"], d["z"].shape[-1]
    pixels = z.numel() // ch
    e = lambda: torch.empty(ch, device=cuda)
    rm, rv, mean, inv = d["rm0"].clone(), d["rv0"].clone(), e(), e()
    ty, tmean, tinv, trm, trv = torch_bn_train(z, d["gamma"], d["beta"], d["rm0"], d["rv0"])
    if entry == "bn_finalize":
        scale, shift = e(), e()
        ops.bn_finalize(d["zstats"], pixels, d["gamma"], d["beta"], rm, rv, scale, shift, mean, inv)
    else:
        y = torch.empty_like(z)
        ops.bn_train_apply(z, ops.make_bn_train(d["zstats"], d["gamma"], d["beta"], rm, rv, mean, inv), y, False)
        scale = d["gamma"] * inv
        shift = d["beta"] - mean * scale
    fref, ftol = EC.fin_ref(d["zstats"], pixels, d["rm0"], d["rv0"])
    got = dict(mean=mean, invstd=inv, rm=rm, rv=rv)
    want = dict(mean=tmean, invstd=tinv, rm=trm, rv=trv)
    for k in got:
        assert_nonfinite_like(got[k], want[k], "%s %s" % (entry, k), 0.0, rel=0.0, extra=ftol[k], finite_ref=fref[k])
    tsc = d["gamma"].double().cpu() * tinv
    assert_nonfinite_like(scale, tsc, entry + " scale")
    assert_nonfinite_like(shift, d["beta"].double().cpu() - tmean * tsc, entry + " shift")
    assert bool(torch.isnan(rv[[3, 10, 17, 24, 40, 63]]).all()), "a non-finite channel's running_var must be NaN"
    if entry == "bn_train_apply":
        assert_nonfinite_like(y, ty, "bn_train_apply output")


# --------------------------------------------------------------------------------------------- conv forward epilogue
CONV = dict(desc="nonfinite 64->64 3x3 b32 24x24", n=32, h=24, w=24, c0=64, cout=64, k=3)   # 144+ tiles of <= 128 px


def conv_places(c):
    """(n, y, x) pixels inside the first tile, in a tile a persistent CTA reaches on its second round, and the last"""
    n, h, w = c["n"], c["h"], c["w"]
    p = [37, CC.sms() * 128 + 200, n * h * w - 1]
    assert p[1] < n * h * w - 128
    return [(q // (h * w), q // w % h, q % w) for q in p]


@pytest.mark.parametrize("where", ["x", "w", "scale", "bias", "residual"])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "linear"])
def test_conv_fwd_nonfinite(mcb, cuda, where, relu):
    """conv_fwd's epilogue y = [relu](acc scale + bias + residual), with NaN / +-Inf in the input activation, the
    weight, or the epilogue's scale, bias or residual; float64 reference of the same operation"""
    c = CONV
    x, wt, b, _, _ = CC.fwd_ref(c, False, _CACHE)
    x, wt, b = x.clone(), wt.clone(), b.clone()
    g = CC.gen("nonfinite conv epilogue", c["desc"])
    scale = torch.rand(c["cout"], generator=g) + 0.5
    res = CC.bf16r(torch.randn(c["n"], c["cout"], c["h"], c["w"], generator=g))
    places = conv_places(c)
    if where == "x":
        for (n, yy, xx), ch, v in zip(places, (3, 31, 63), NONFINITE):
            x[n, ch, yy, xx] = v
    elif where == "w":
        wt[5, 7, 1, 1], wt[40, 2, 0, 0], wt[63, 63, 2, 2] = NONFINITE
    elif where == "scale":
        scale[[5, 40, 63]] = torch.tensor(NONFINITE)
    elif where == "bias":
        b[[5, 40, 63]] = torch.tensor(NONFINITE)
    else:
        for (n, yy, xx), ch, v in zip(places, (3, 31, 63), NONFINITE):
            res[n, ch, yy, xx] = v
    conv = lambda a, v: F.conv2d(a.double(), v.double(), padding=c["k"] // 2)
    v = lambda t: t.double().view(1, -1, 1, 1)
    ref = conv(x, wt) * v(scale) + v(b) + res.double()
    ref = torch.relu(ref) if relu else ref
    A = conv(x.abs(), wt.abs()) * v(scale.abs()) + v(b.abs()) + res.double().abs()
    y = CC.run_fwd(c, x, wt, bias=b.cuda(), relu=relu, scale=scale.cuda(), residual=CC.dev(res))
    assert_nonfinite_like(CC.nchw(y), ref, "conv_fwd (%s non-finite)" % where, A)


# ----------------------------------------------------------------------------------------- conv data / weight gradient
GRAD = dict(desc="nonfinite grad 64->64 3x3 b32 24x24", n=32, h=24, w=24, cin=64, cout=64, k=3)


def test_conv_wgrad_nonfinite_input(mcb, cuda):
    """dW = sum dy x: a NaN in the input x makes every tap of its channel's weight gradient NaN (the pixel is interior,
    so every tap reaches it); +-Inf make them +-Inf or NaN as the float64 reference says"""
    from mcb200 import ops
    c = GRAD
    x, dy, _, _ = CC.wgrad_ref(c, False, _CACHE)
    x = x.clone()
    (n0, y0, x0), (n1, y1, x1), (n2, y2, x2) = conv_places(dict(c, c0=c["cin"]))
    x[n0, 9, 10, 10], x[n1, 20, y1, x1], x[n2, 63, y2, x2] = NONFINITE
    wg = lambda a, d: torch.nn.grad.conv2d_weight(a.double(), (c["cout"], c["cin"], 3, 3), d.double(), padding=1)
    ref, A = wg(x, dy), wg(x.abs(), dy.abs())
    dw = torch.zeros(9, c["cout"], c["cin"], device=cuda)
    ops.conv_wgrad(CC.dev(dy), CC.dev(x), dw, 3, 1)
    got = ops.unpack_conv_weight(dw, 3)
    assert_nonfinite_like(got, ref, "conv_wgrad", A, rel=0.0)
    assert bool(torch.isnan(got[:, 9]).all()), "the NaN input channel's weight gradient must be NaN at every tap"


def test_conv_dgrad_nonfinite(mcb, cuda):
    """dx = conv_transpose(dy, W) masked by the producing ReLU's output (relu_mask): NaN / +-Inf in dy spread over
    their footprint; a NaN (or +Inf) in the ReLU output passes the gradient, as torch's relu backward (zero where
    y <= 0) does"""
    from mcb200 import ops
    c = GRAD
    dy, wt, act, _, _, _ = CC.dgrad_ref(c, False, _CACHE)
    dy, act = dy.clone(), act.clamp_min(0)
    (n0, y0, x0), (n1, y1, x1), (n2, y2, x2) = conv_places(dict(c, c0=c["cin"]))
    dy[n0, 4, y0, x0], dy[n1, 30, y1, x1], dy[n2, 63, y2, x2] = NONFINITE
    act[n1, 5, 3, 3], act[0, 6, 10, 11], act[n2, 7, 0, 0] = NAN, INF, NAN
    dg = lambda v, d: torch.nn.grad.conv2d_input(act.shape, v.double(), d.double(), padding=1)
    full, A = dg(wt, dy), dg(wt.abs(), dy.abs())
    ref = torch.ops.aten.threshold_backward(full, act.double(), 0.0)
    got = ops.conv_dgrad(CC.dev(dy), CC.pack(wt), 3, 1, (c["h"], c["w"]), relu_mask=CC.dev(act))
    assert_nonfinite_like(CC.nchw(got), ref, "conv_dgrad", A)


# ---------------------------------------------------------------------------------------------------------- max-pool
# one window pattern per planted window, in scan order (0, 0), (0, 1), (1, 0), (1, 1)
WINDOWS = [(NAN, 1, 2, 3), (3, NAN, 2, 1), (1, 2, NAN, 3), (3, 2, 1, NAN),         # a NaN at each position
           (NAN, 5, NAN, 1), (1, NAN, 7, NAN),                                     # two NaNs
           (INF, 1, 2, 3), (1, 2, 3, INF), (-INF, -INF, -INF, -INF), (-INF, 0.5, -INF, 1),
           (INF, NAN, 1, 2), (-INF, 1, NAN, INF)]


def plant_windows(x, c8_places, windows=WINDOWS):
    """x (N, H, W, C) bf16; window k into the pooled item near places[k % len] (a pooled pixel and 8-channel group as
    the kernels count them), at channel k % 8 of the group"""
    n, h, w, ch = x.shape
    ho, wo, c8 = h // 2, w // 2, ch // 8
    total = n * ho * wo * c8
    out = []
    for k, pat in enumerate(windows):
        item = (c8_places[k % len(c8_places)] - 8 * (k // len(c8_places))) % total   # distinct items near each place
        cg, p = item % c8, item // c8
        ox, oy, nn = p % wo, p // wo % ho, p // (wo * ho)
        cc = cg * 8 + k % 8
        for q, v in enumerate(pat):
            x[nn, 2 * oy + q // 2, 2 * ox + q % 2, cc] = v
        out.append((nn, oy, ox, cc))
    return out


def test_maxpool_nonfinite(mcb, cuda):
    """maxpool2_fwd and maxpool2_bwd (store and accumulate) at 2048@10x10 -> 5x5, batch 160 (a partial last pass),
    with the windows of WINDOWS planted: the output as torch's max_pool2d, the gradient routed to torch's index
    (elementwise_checks.pool_ref)"""
    from mcb200 import ops
    c = EC.POOL[1]
    n, h, w, ch = c["n"], c["h"], c["w"], c["c"]
    g = EC.gen("nonfinite pool")
    x = EC.randn(g, n, h, w, ch).to(BF)
    total = n * (h // 2) * (w // 2) * ch // 8
    plant_windows(x, EC.stride_places(total, 256))
    dy = EC.randn(g, n, h // 2, w // 2, ch).to(BF)
    ref_y, routed = EC.pool_ref(x, dy)
    assert_nonfinite_like(ops.maxpool2_fwd(x), ref_y, "maxpool2_fwd", 0.0, rel=0.0)
    dx = torch.empty_like(x)
    ops.maxpool2_bwd(x, dy, dx, False)
    assert_nonfinite_like(dx, routed, "maxpool2_bwd store", 0.0, rel=0.0)
    pre = EC.randn(g, n, h, w, ch).to(BF)
    dx = pre.clone()
    ops.maxpool2_bwd(x, dy, dx, True)
    acc = (pre.float() + routed.float()).to(BF)
    assert_nonfinite_like(dx, acc, "maxpool2_bwd accumulate", 0.0, rel=0.0)


def test_maxpool_bwd_skip_relu_nonfinite(mcb, cuda):
    """maxpool2_bwd_skip_relu (the VGG encoders' pool over y = relu(conv + b) that also feeds a concat) at 64@80x80,
    batch 32: g = (y <= 0) ? 0 : bf16(g + routed dpool), routed to torch's index; db += per-channel sums of g"""
    from mcb200 import ops
    n, h, w, ch = 32, 80, 80, 64
    g = EC.gen("nonfinite skip pool")
    y = EC.randn(g, n, h, w, ch).clamp_min(0).to(BF)
    pooled = n * (h // 2) * (w // 2)
    grid, lanes = EC.reduce_grid(pooled, ch)
    second = grid * lanes + 3                               # a pooled pixel a lane reaches on its second pass
    # y is a ReLU output: the windows without -Inf
    plant_windows(y, [i * (ch // 8) for i in (5, second, pooled - 1)],
                  [p for p in WINDOWS if not any(v == -INF for v in p)])
    dpool = EC.randn(g, n, h // 2, w // 2, ch).to(BF)
    g0 = EC.randn(g, n, h, w, ch).to(BF)
    ref = EC.pool_skip_ref(y, g0, dpool)
    gg, db = g0.clone(), torch.zeros(ch, device=cuda)
    ops.maxpool2_bwd_skip_relu(y, dpool, gg, db)
    assert_nonfinite_like(gg, ref, "maxpool2_bwd_skip_relu g", 0.0, rel=0.0)
    stored = gg.double().cpu().view(-1, ch)
    CC.assert_bound(db, stored.sum(0), stored.abs().sum(0), "maxpool2_bwd_skip_relu db", rel=0.0)


# ---------------------------------------------------------------------------------------------- the 1x1 classifier
FINAL = (8, 320, 320, 32, 2)     # n, h, w, C, K: 819200 pixels, three passes of final_conv_fwd's grid-stride loop


@pytest.mark.parametrize("where", ["x", "w", "b"])
def test_final_conv_fwd_nonfinite(mcb, cuda, where):
    from mcb200 import ops
    n, h, w, ch, k = FINAL
    g = EC.gen("nonfinite final fwd")
    x = EC.randn(g, n, h, w, ch).clamp_min(0).to(BF)
    wt, b = EC.randn(g, k, ch) * 0.2, EC.randn(g, k)
    places = EC.stride_places(n * h * w, 256)
    if where == "x":
        plant(x, [p * ch + cc for p, cc in zip(places, (0, 9, 17, 31))], (NAN, INF, NAN, INF))
    elif where == "w":
        wt[1, 5], wt[0, 31] = NAN, INF
    else:
        b[0], b[1] = -INF, NAN
    logits = torch.empty(n, k, h, w, device=cuda)
    ops.final_conv_fwd(x, wt.reshape(-1), b, logits)
    ref, la = EC.classifier_fwd_ref(x.cpu(), wt.cpu(), b.cpu())
    assert_nonfinite_like(logits, ref, "final_conv_fwd (%s)" % where, la, rel=0.0)


def test_final_conv_bwd_nonfinite(mcb, cuda):
    """dx = (x > 0) W^T dlogits, dW += sum dlogits x^T, db += sum dlogits with NaN / +-Inf in dlogits"""
    from mcb200 import ops
    n, h, w, ch, k = FINAL
    g = EC.gen("nonfinite final bwd")
    x = EC.randn(g, n, h, w, ch).clamp_min(0).to(BF)
    wt = EC.randn(g, k, ch) * 0.2
    dl = EC.randn(g, n, k, h, w)
    for p, kk, v in zip(EC.stride_places(n * h * w, 128, 4), (0, 1, 1, 0), (NAN, INF, -INF, NAN)):
        dl[p // (h * w), kk, p // w % h, p % w] = v
    pre_w, pre_b = EC.randn(g, k * ch), EC.randn(g, k)
    dx, dw, db = torch.empty_like(x), pre_w.clone(), pre_b.clone()
    ops.final_conv_bwd(x, wt.reshape(-1), dl, dx, dw, db)
    gx, ga, sw, aw, sb, ab = EC.classifier_bwd_ref(x.cpu(), wt.cpu(), dl.cpu())
    assert_nonfinite_like(dx, gx, "final_conv_bwd dx", 0.0, extra=2.0 ** -20 * ga)
    pw, pb = pre_w.double().cpu(), pre_b.double().cpu()
    assert_nonfinite_like(dw, pw + sw, "final_conv_bwd dW", pw.abs() + aw, rel=0.0)
    assert_nonfinite_like(db, pb + sb, "final_conv_bwd db", pb.abs() + ab, rel=0.0)


# ------------------------------------------------------------------------------------------------ softmax and loss
@pytest.mark.parametrize("kind", ["nan", "+inf", "-inf"])
@pytest.mark.parametrize("act", ["softmax", "sigmoid"])
def test_loss_nonfinite_logit(mcb, cuda, kind, act):
    """loss_partials + loss_grad (weighted cross entropy + Dice with either activation) and softmax2 at 32 x 320 x 320
    with one non-finite logit at a pixel the grid-stride loop reaches on its second pass, and the same value in the
    last pixel's other class: the loss, the four sums and d(loss)/d(logits) against autograd of the reference's loss
    in float64 on the CPU"""
    from mcb200 import ops
    logits, t = EC.loss_case()
    z = logits.clone()
    v = {"nan": NAN, "+inf": INF, "-inf": -INF}[kind]
    n, _, s, _ = z.shape
    p = EC.stride_places(n * s * s, 256)[2]
    z[p // (s * s), 1, p // s % s, p % s] = v
    z[n - 1, 0, s - 1, s - 1] = v
    cfg = dict(size_c=EC.SIZE_C, dice_activation=act)
    sums = torch.zeros(4, dtype=F64, device=cuda)
    ops.loss_partials(z, t, sums, mode=0, **cfg)
    dlog, loss = torch.empty_like(z), torch.zeros((), device=cuda)
    ops.loss_grad(z, t, sums, dlog, loss, mode=0, **cfg)
    lg = z.double().cpu().requires_grad_(True)
    ref = SD.mixed_loss(lg, t.double().cpu(), imsize=(s, s), activation=act)
    ref.backward()
    assert_nonfinite_like(loss.reshape(1), ref.detach().reshape(1), "loss (%s)" % act)
    assert_nonfinite_like(dlog, lg.grad, "dlogits (%s)" % act)
    if act == "softmax":
        assert_nonfinite_like(ops.softmax2(z), torch.softmax(z.double().cpu(), 1), "softmax2")


# ------------------------------------------------------------------------------------------------------------- Adam
@pytest.mark.parametrize("entry", ["adam_step", "adam_step_dyn"])
def test_adam_nonfinite_gradient(mcb, cuda, entry):
    """one step with NaN and +-Inf gradients: p, m and v against torch.optim.Adam in float64 (L2 decay, the gradient
    scale applied first); the finite elements within elementwise_checks.check_adam's bounds; the bf16 copy of p
    non-finite where p is"""
    from mcb200 import ops
    threads = EC.grid_for(1 << 30, 256) * 256
    n = 3 * threads + 1001
    g = EC.gen("nonfinite adam")
    p = EC.randn(g, n) * 0.05
    m, v = EC.randn(g, n) * 1e-3, EC.rand(g, n) * 1e-6
    grad = EC.randn(g, n) * 1e-2
    places = EC.stride_places(n, 256)
    plant(grad, places + [q - 1 for q in places] + [q - 2 for q in places])
    t, lr = 3, EC.adam_lr(3)
    p0, m0, v0 = p.clone(), m.clone(), v.clone()
    p16 = torch.empty(n, dtype=BF, device=cuda)
    if entry == "adam_step":
        ops.adam_step(p, grad, m, v, p16, t, lr, EC.BETAS, EC.ADAM_EPS, EC.WD, EC.GRAD_SCALE)
    else:
        hyper = torch.tensor(ops.adam_hyper(lr, EC.BETAS, t), dtype=torch.float32, device=cuda)
        ops.adam_step_dyn(p, grad, m, v, p16, hyper, EC.BETAS, EC.ADAM_EPS, EC.WD, EC.GRAD_SCALE)
    tp = p0.double().cpu().requires_grad_(True)
    opt = torch.optim.Adam([tp], lr=lr, betas=EC.BETAS, eps=EC.ADAM_EPS, weight_decay=EC.WD)
    # the kernel's pre-step state: the step below runs at t
    opt.state[tp] = st = dict(step=torch.tensor(float(t - 1)), exp_avg=m0.double().cpu(), exp_avg_sq=v0.double().cpu())
    tp.grad = grad.double().cpu() * C.c_float(EC.GRAD_SCALE).value
    opt.step()
    keep = torch.isfinite(tp.detach()) & torch.isfinite(st["exp_avg"]) & torch.isfinite(st["exp_avg_sq"])
    for name, got, want in (("p", p, tp.detach()), ("m", m, st["exp_avg"]), ("v", v, st["exp_avg_sq"])):
        assert_nonfinite_like(got, want, "%s %s" % (entry, name))
    k = keep.to(cuda)
    EC.check_adam(t, lr, p0[k], m0[k], v0[k], grad[k], p[k], m[k], v[k], entry)
    assert_nonfinite_like(p16, p, entry + " bf16 copy")


# ------------------------------------------------------------------------------------ casts and layout kernels
BF16_MAX_BITS = 0x7F7F0000
OVER = [0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0xFF7F7FFF, 0xFF7F8000, 0xFF7FFFFF]   # below / at / above the tie to Inf


def with_extremes(x, flat):
    """NaN, +-Inf, and fp32 values beyond bf16's largest finite value (the tie rounds to even: Inf) at flat"""
    plant(x, flat)
    ext = torch.tensor([b - (1 << 32) if b >= 1 << 31 else b for b in OVER], dtype=torch.int32).view(torch.float32)
    v = x.view(-1)
    for i in range(len(OVER)):
        v[(flat[i % len(flat)] + 1 + i // len(flat)) % v.numel()] = float(ext[i])
    return x


def assert_cast_like(got, ref, what):
    assert_nonfinite_like(got, ref, what, 0.0, rel=0.0)


def test_cast_and_layout_nonfinite(mcb, cuda):
    """cast_bf16 and nchw_to_nhwc_bf16 / nhwc_to_nchw_f32 keep NaN and +-Inf, and round values beyond the bf16 range
    to +-Inf as tensor.to(torch.bfloat16) does; the largest finite value below the tie stays finite"""
    from mcb200 import ops
    n, ch, h, w = 32, 3, 320, 320
    g = EC.gen("nonfinite cast")
    x = EC.randn(g, n, ch, h, w)
    with_extremes(x, EC.stride_places(x.numel(), 256))
    ref = x.to(BF)
    assert bool(torch.isinf(ref).sum() >= 4) and int((ref.view(torch.int16) == 0x7F7F).sum()) >= 1
    assert_cast_like(ops.cast_bf16(x.view(-1), torch.empty(x.numel(), dtype=BF, device=cuda)), ref.view(-1),
                     "cast_f32_bf16")
    y = ops.nchw_to_nhwc_bf16(x)
    assert_cast_like(y, x.permute(0, 2, 3, 1).to(BF), "nchw_f32_to_nhwc_bf16")
    assert_cast_like(ops.nhwc_to_nchw_f32(y), y.permute(0, 3, 1, 2).float(), "nhwc_bf16_to_nchw_f32")


@pytest.mark.parametrize("entry", ["stem_im2col", "vgg_input_im2col"])
def test_im2col_nonfinite(mcb, cuda, entry):
    """the stem's 7x7/s2 and the VGG input conv's 3x3 im2col copy NaN, +-Inf and the rounded-to-Inf extremes into every
    column that reads them (F.unfold of the same image, then the bf16 cast)"""
    from mcb200 import ops
    n, h, w = 32, 320, 300          # width 300: a partial last strip
    g = EC.gen("nonfinite im2col", entry)
    x = EC.randn(g, n, 3, h, w)
    with_extremes(x, [3 * w + 7, (n // 2) * 3 * h * w + h * w + 5 * w + 100, x.numel() - 1])
    if entry == "stem_im2col":
        col = ops.stem_im2col(x)
        k, s, pad, taps, width = 7, 2, 3, 147, 192
    else:
        col = ops.vgg_input_im2col(x)
        k, s, pad, taps, width = 3, 1, 1, 27, 32
    ho, wo = h // s, w // s
    for sl in EC.chunks(n, 3 * h * w * k * k // (s * s)):
        u = F.unfold(x[sl].cpu(), k, padding=pad, stride=s)
        ref = u.view(u.shape[0], 3, k * k, ho, wo).permute(0, 3, 4, 2, 1).reshape(u.shape[0], ho, wo, taps)
        assert_cast_like(col[sl, ..., :taps], ref.to(BF), "%s [images %d:%d]" % (entry, sl.start, sl.stop))
    assert not bool(col[..., taps:width].any())


# ------------------------------------------------------------------------------------------ fixed-order finishing sum
def test_det_sum_nonfinite_rows(mcb, cuda):
    """mcb_det_sum_f32 over 70 rows: columns with one NaN, with +Inf and -Inf in different rows (Inf - Inf), with +Inf
    only; against the float32 re-summation in the library's order (elementwise_checks.reference_sum), bit for bit
    where finite"""
    rng = np.random.default_rng(70)
    nrows, n = 70, 1000
    rows = EC.wide_range_rows(rng, nrows, n)
    rows[3, 10] = np.nan
    rows[69, 999] = np.nan
    rows[0, 20], rows[45, 20] = np.inf, -np.inf
    rows[31, 21], rows[32, 21] = np.inf, -np.inf
    rows[7, 22], rows[8, 22] = np.inf, np.inf
    rows[33, 23] = -np.inf
    out0 = rng.standard_normal(n).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        want = (out0 + EC.reference_sum(rows)).astype(np.float32)
    got = EC.run_det_sum(rows, n, n, 0, out0)
    assert_nonfinite_like(torch.from_numpy(got), torch.from_numpy(want), "det_sum", 0.0, rel=0.0)
    assert np.isnan(got[[10, 20, 21, 999]]).all() and got[22] == np.inf and got[23] == -np.inf


# ------------------------------------------------------------------------------------------------------ signed zeros
def test_signed_zero(mcb, cuda):
    """-0.0 and +0.0 through the ReLU of bn_apply and of the conv epilogue and through the max-pool: the bits finite
    operands got before NaN propagated are kept (pinned below).  torch's relu and max_pool2d keep -0.0 in places where
    these kernels give +0.0; only the finite bits of the kernels themselves are pinned here"""
    from mcb200 import ops
    ch = 64
    full = lambda v: torch.full((ch,), v, device=cuda)
    z = torch.zeros(1, 2, 2, ch, dtype=BF, device=cuda)
    z[0, 0, 1], z[0, 1, 0] = -0.0, -0.0
    out = {}
    for relu in (True, False):
        for sh in ("+0", "-0"):
            y = torch.empty_like(z)
            ops.bn_apply(z, full(1.0), full(float(sh)), y, relu)      # z * 1 + shift: -0 only for z = -0, shift -0
            out["bn_apply relu=%d shift=%s" % (relu, sh)] = y[0, :, :, 0].reshape(-1)
    x = torch.zeros(2, 4, 4, ch, dtype=BF, device=cuda)
    wt = torch.zeros(9, ch, ch, dtype=BF, device=cuda)
    for relu in (True, False):
        y = ops.conv_fwd(x, wt, 3, 1, bias=torch.full((ch,), -0.0, device=cuda), relu=relu,
                         scale=torch.full((ch,), -1.0, device=cuda))
        out["conv_fwd relu=%d" % relu] = y[0, 0, :2, 0]
    p = torch.zeros(1, 2, 8, ch, dtype=BF, device=cuda)
    for win, pat in enumerate([(-0.0, -0.0, -0.0, -0.0), (-0.0, 0.0, -0.0, -0.0), (0.0, -0.0, -0.0, -0.0),
                               (-0.0, -0.0, -0.0, 0.0)]):
        for q, v in enumerate(pat):
            p[0, q // 2, 2 * win + q % 2] = v
    out["maxpool2_fwd"] = ops.maxpool2_fwd(p)[0, 0, :, 0]
    got = {k: [int(b) & 0xFFFF for b in v.contiguous().view(torch.int16).cpu()] for k, v in out.items()}
    assert got == SIGNED_ZERO_BITS, got


SIGNED_ZERO_BITS = {   # bf16 bits: relu(-0) is +0; the max of a window of zeros is -0 only if all four are -0
    "bn_apply relu=1 shift=+0": [0, 0, 0, 0], "bn_apply relu=1 shift=-0": [0, 0, 0, 0],
    "bn_apply relu=0 shift=+0": [0, 0, 0, 0], "bn_apply relu=0 shift=-0": [0, 0x8000, 0x8000, 0],
    "conv_fwd relu=1": [0, 0], "conv_fwd relu=0": [0x8000, 0x8000],
    "maxpool2_fwd": [0x8000, 0, 0, 0]}


# =====================================================================================================================
# B. the network
# =====================================================================================================================
EVAL_CASES = [("ResNet34", 2, 256), ("ResNet101", 64, 320)]    # the bench's infer workload: ResNet101, batch 64, 320
POISON = "encoder.layer2.0.conv1.weight"


def poison_index(shape):
    return (5, 3, shape[2] // 2, shape[3] // 2)


def poisoned_sd(sd):
    """sd with the NaN in POISON and in every key that aliases it (the reference's conv1 .. conv5 are the encoder's
    own modules, so a state_dict holds each of their weights twice, and loading one clean copy would undo the other)"""
    w = sd[POISON]
    out = {k: v.clone() for k, v in sd.items()}
    for k, v in sd.items():
        if v.shape == w.shape and torch.equal(v, w):
            out[k][poison_index(w.shape)] = NAN
    return out


def reference_eval(enc, sd, X):
    """baseline/torch_cudnn_unet.py in fp32 eval mode (BatchNorm from the running statistics) on the CPU"""
    from baseline.torch_cudnn_unet import UNetResNet
    net = UNetResNet(SC.DEPTH[enc])
    net.load_state_dict(sd, strict=True)
    net.eval()
    with torch.no_grad():
        return net(X.cpu())


@pytest.mark.parametrize("enc,n,s", EVAL_CASES, ids=["%s-b%d-%d" % c for c in EVAL_CASES])
def test_eval_forward_nonfinite(mcb, cuda, enc, n, s):
    """the eval forward (BatchNorm folded into the conv epilogues) of a model built as the benchmark builds it: the
    non-finite logits at the reference's positions, for a NaN input pixel, a +Inf input pixel and a NaN weight of an
    encoder conv.  The images of a batch are independent in eval mode, so the reference runs on the poisoned image and
    on the last one (and a clean image must stay finite)"""
    sd = SC.seeded_sd(enc)
    run = SC.BenchStep(enc, sd, cuda, 2, s)
    net = run.net
    net.eval()
    X = SC.batch(SC.SEED + 50, n, s)[0]
    last = n - 1
    for variant in ("nan pixel", "+inf pixel", "nan weight"):
        Xv, sdv = X.clone(), sd
        if variant == "nan weight":
            w = dict(net.named_parameters())[POISON]
            idx = poison_index(w.shape)
            saved = float(w.data[idx])
            with torch.no_grad():
                w.data[idx] = NAN
            sdv = poisoned_sd(sd)
        else:
            Xv[0, 1, s // 2 + 3, 17] = NAN if variant == "nan pixel" else INF
        with torch.no_grad():
            got = cpu(net(Xv.to(cuda)))
        if variant == "nan weight":
            with torch.no_grad():
                w.data[idx] = saved
        ref = reference_eval(enc, sdv, Xv[[0, last]])
        assert_nonfinite_like(got[[0, last]], ref, "%s eval logits (%s)" % (enc, variant))
        bad = (~torch.isfinite(got)).flatten(1).any(1)
        print("%s b%d %s: %d of %d logits of image 0 non-finite, images with a non-finite logit: %d" % (
            enc, n, variant, int((~torch.isfinite(got[0])).sum()), got[0].numel(), int(bad.sum())))
        if variant != "nan weight":
            assert bool(bad[0]) and not bool(bad[1:].any()), "only the poisoned image may hold non-finite logits"
    del run, net
    SC.free_device_memory()


TRAIN_CASES = [("ResNet34", 2, 256), ("ResNet101", SC.N, SC.S)]


def nan_params(named):
    return {k for k, v in named if bool(torch.isnan(v).any())}


def reference_after_step(enc, sd, X, T, adam):
    """reference_step's gradients and running statistics, and the parameters after torch.optim.Adam's step with the
    hyperparameters the fused step hands its Adam -> (loss, running statistics, names of parameters holding a NaN)"""
    ref = SC.reference_step(enc, sd, X, T, emulate_bf16=False)
    lr, betas, eps, wd = adam
    plain = SC.O.strip_module_prefix(sd)
    params = {k: plain[k].clone().double().requires_grad_(True) for k in ref["grads"]}
    opt = torch.optim.Adam(list(params.values()), lr=lr, betas=betas, eps=eps, weight_decay=wd)
    for k, p in params.items():
        p.grad = ref["grads"][k].double()
    opt.step()
    return ref["loss"], ref["stats"], nan_params((k, p.detach()) for k, p in params.items())


def check_poisoned_step(enc, loss, stats, params, ref):
    ref_loss, ref_stats, ref_nan = ref
    assert np.isnan(float(loss)) and np.isnan(ref_loss), (float(loss), ref_loss)
    for k in ref_stats:
        assert_nonfinite_like(stats[k], ref_stats[k], "%s %s" % (enc, k))
    nan_stats = [k for k in ref_stats if bool(torch.isnan(ref_stats[k]).any())]
    assert nan_stats, "the poisoned conv's BatchNorm must get NaN running statistics"
    got_nan = nan_params(params)
    assert got_nan == ref_nan, "parameters holding a NaN after the step differ: %s" % sorted(got_nan ^ ref_nan)
    print("%s: loss NaN, %d of %d running statistics and %d of %d parameter tensors hold a NaN, as in the reference" % (
        enc, len(nan_stats), len(ref_stats), len(got_nan), len(ref_nan | set(k for k, _ in params))))


def arena_params(net):
    return [(name, p.detach()) for name, p, _ in net._arena_params()]


def poison_arena(net):
    """a NaN into the fp32 master weight and its bf16 operand copy, as a step's Adam would leave it"""
    p = dict(net.named_parameters())[POISON]
    idx = poison_index(p.shape)
    with torch.no_grad():
        p.data[idx] = NAN
        k = p.shape[2]
        net._packed(p, net._w16)[idx[2] * k + idx[3], idx[0], idx[1]] = NAN


@pytest.mark.parametrize("enc,n,s", TRAIN_CASES, ids=["%s-b%d-%d" % c for c in TRAIN_CASES])
def test_train_step_nan_weight(mcb, cuda, no_tf32, enc, n, s):
    """_fit_loop's fused train step with one NaN encoder weight: a NaN loss, NaN running statistics where the
    reference's are NaN, and after Adam the same set of parameter tensors holding a NaN as the reference.  Then once
    more through the captured graph: a clean eager step, the NaN written into the weight, a graph replay -- equal, bit
    for bit, NaNs included, to the same launches in program order"""
    sd = SC.seeded_sd(enc)
    sdp = poisoned_sd(sd)
    X, T = (t.to(cuda) for t in SC.batch(SC.SEED + 60, n, s))
    run = SC.BenchStep(enc, sdp, cuda, n, s)
    adam = run.adam
    loss = run.step(X, T)
    got = (cpu(loss), SC.running_stats(run.net), [(k, cpu(v)) for k, v in arena_params(run.net)])
    del run
    SC.free_device_memory()
    ref = reference_after_step(enc, sdp, X, T, adam)
    check_poisoned_step(enc, *got, ref)
    del got

    # through the captured graph
    batches = [tuple(t.to(cuda) for t in SC.batch(SC.SEED + 61 + i, n, s)) for i in range(2)]
    run = SC.BenchStep(enc, sd, cuda, n, s)
    layout = SC.arena_layout(run.net)
    run.step(*batches[0])
    poison_arena(run.net)
    assert run.is_replay(*batches[1])
    graphed = SC.snapshot(run, run.step(*batches[1]))
    del run
    SC.free_device_memory()
    run = SC.BenchStep(enc, sd, cuda, n, s)
    steps = run.serial_steps(batches)
    next(steps)
    poison_arena(run.net)
    serial = SC.snapshot(run, next(steps))
    bad = SC.snapshot_mismatches(layout, graphed, serial)
    assert not bad, "%s graph replay against program order: %s" % (enc, "; ".join(bad))
    assert np.isnan(float(graphed["loss"]))
    assert any(bool(torch.isnan(v).any()) for v in graphed["stats"].values())
    assert bool(torch.isnan(graphed["p32"]).any())
    del run, graphed, serial
    SC.free_device_memory()
