"""TEST INFRASTRUCTURE -- the harness of the tests of the HBM-bound kernels (csrc/elementwise.cu, csrc/loss.cu) and of
the fixed-order finishing sum (csrc/detsum.cuh): tests/test_elementwise_gpu.py (small shapes),
tests/test_elementwise_scale_gpu.py (the batch-32 sizes, where every thread loops), tests/test_nonfinite_gpu.py (NaN and
+-Inf), tests/test_vgg_kernels_gpu.py (the pool of a skip connection) and tests/test_detsum_gpu.py.  Never imported by
the product path; mcb200 is imported inside the functions, once the mcb fixture has built it.

Operands are seeded on the device from a key (gen); cached keeps one case's tensors at a time, so device memory stays
bounded.  The launch model (grid_for, reduce_grid) restates the kernels' grid formulas, so that a case can assert the
regime it runs in: every thread (or pixel lane of a reduction block) owns at least 3 work items.

References are float64 from the bf16-rounded operands; A is the same operation on |operands|.  The bars are
oracle/conv_checks.py's assert_bound / assert_exact / assert_same, with each kernel's own allowance:
  bf16 outputs        |got - ref| <= 2^-8 |ref| (half a bf16 ulp) + 2^-20 A (assert_bf16);
  real-valued sums    |got - ref| <= 2^-16 A, and a second run repeats the first bitwise;
  integer-exact sums  bitwise, the sums < 2^24 (check_reduction); pure data movement (max-pool with torch's index rule,
                      layout conversions, im2col, fp32 -> bf16) bitwise;
  BatchNorm statistics within a few fp32 ulps of the float64 finalisation, scaled by the magnitudes the fp32 arithmetic
                      cancels (fin_ref);
  the loss            within 1e-6 relative; d(loss)/d(logits) per pixel within 2^-18 of that pixel's CE weight / M and
                      Dice term (loss_ref);
  Adam                one step from the kernel's own state: p within 2^-18 of the update size plus one fp32 ulp, m and v
                      within 2^-20 of their terms' magnitudes (check_adam);
  the finishing sum   bitwise against a float32 re-summation in the library's order (reference_sum)."""
import ctypes as C
import math
import zlib

import numpy as np
import torch

from oracle import synthetic
from oracle import unet_oracle as O
from oracle.conv_checks import assert_bound, assert_exact, sms

BF, F64 = torch.bfloat16, torch.float64
U = 2.0 ** -24                                            # fp32 unit roundoff
MOM, EPS = C.c_float(0.1).value, C.c_float(1e-5).value   # BatchNorm momentum / eps as the kernels receive them

_CASE = {}    # the current case's tensors
_LAYOUT = {}  # UNetResNet(101)'s arena length and BatchNorm widths


# -------------------------------------------------------------------------------------------------- seeded operands
def gen(*key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))


def randn(g, *shape):
    return torch.randn(shape, generator=g, device="cuda")


def rand(g, *shape):
    return torch.rand(shape, generator=g, device="cuda")


def ints(g, lo, hi, *shape):
    """integers in [lo, hi] as float32"""
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda", dtype=torch.int8).float()


def cached(key, make):
    """make(), kept under key until another key is asked for"""
    if key not in _CASE:
        _CASE.clear()
        _CASE[key] = make()
    return _CASE[key]


def free_case():
    _CASE.clear()


def chunks(n, per_image, limit=1 << 23):
    """batch slices of at most `limit` elements: bounds the float64 temporaries of a reference"""
    step = max(1, limit // per_image)
    return [slice(i, min(n, i + step)) for i in range(0, n, step)]


def with_ties(x, g):
    """plant fp32 values exactly halfway between two bf16 values (round to nearest even decides)"""
    k = min(x.numel(), 1 << 16)
    y = randn(g, k).to(BF).float()
    x.view(-1)[:k] = (y.view(torch.int32) | 0x8000).view(torch.float32)
    return x


def ids(cases):
    return [c["desc"].replace(" ", "_") for c in cases]


# ------------------------------------------------------------------------------------------------ launch-regime model
def grid_for(work, threads, per_sm=8):
    """elementwise.cu grid_for (also loss.cu loss_grid, with 256 threads)"""
    return max(1, min(-(-work // threads), sms() * per_sm))


def reduce_grid(pixels, c):
    """channel_reduce_kernel's launch (elementwise.cu reduce_cfg and its callers, the skip-connection pool's too):
    blocks of lanes x C/8 threads, 256 - 256 % (C/8) of them, grid min(pixels / (4 lanes), 4 x SMs) -> (grid, lanes)"""
    c8 = c // 8
    lanes = max(256 - 256 % c8, c8) // c8
    return max(1, min(-(-pixels // (lanes * 4)), sms() * 4)), lanes


def assert_stride_regime(work, threads, per_sm=8, ragged=False, pair=False):
    """a grid-stride loop over `work` items launched with grid_for: every thread owns at least 3 items; ragged: the last
    pass is partial.  pair: the BatchNorm apply kernels, launched over ceil(work / 2) items, take items i and
    i + stride per iteration -- ragged then means some thread's last iteration has no second item"""
    t = grid_for((work + 1) // 2 if pair else work, threads, per_sm) * threads
    assert work // t >= 3, "%d items over %d threads (%d SMs)" % (work, t, sms())
    if ragged:
        span = 2 * t if pair else t
        assert work % span, "%d items fill every pass of %d threads" % (work, span)


def assert_reduce_regime(pixels, c, ragged=False):
    """each pixel lane of reduce_grid owns at least 3 pixels; ragged: some lane's last iteration has no second pixel"""
    grid, lanes = reduce_grid(pixels, c)
    assert pixels // (grid * lanes) >= 3, "%d pixels over %d lanes (%d SMs)" % (pixels, grid * lanes, sms())
    if ragged:
        assert pixels % (2 * grid * lanes)


def stride_places(total, threads, per_sm=8, pair=False):
    """work-item indices of a grid_for grid-stride loop over `total` items: inside the first pass, on the second item of
    a pair (pair: the BatchNorm apply kernels take i and i + stride), on the second pass, and the last item"""
    t = grid_for((total + 1) // 2 if pair else total, threads, per_sm) * threads
    step = 2 * t if pair else t
    assert total > step + t, "%d items do not reach a second pass of %d threads" % (total, step)
    return [5, t + 3 if pair else 17, step + 11, total - 1]


# ---------------------------------------------------------------------------------------------------------- the bars
def assert_bf16(got, ref, absref, what):
    """a bf16 output: |got - ref| <= 2^-8 |ref| + 2^-20 A"""
    assert_bound(got, ref, 0.0, what, extra=2.0 ** -20 * absref)


def check_reduction(got, pre, s, a, exact, what):
    """got = pre + a sum s (A: a) into a prefilled output: bitwise when exact (the sums < 2^24), else within 2^-16 A"""
    ref, a = pre.double() + s, pre.double().abs() + a
    if exact:
        assert float(a.max()) < 2 ** 24
        assert_exact(got, ref, what)
    else:
        assert_bound(got, ref, a, what, rel=0.0)


# ------------------------------------------------------------------------------------------------------- BatchNorm
def channel_stats(x):
    """[sum, sumsq] per channel of an NHWC bf16 tensor, as the conv epilogue hands them over (fp32)"""
    v = x.view(-1, x.shape[-1])
    return torch.cat([v.sum(0, dtype=F64), (v.float() ** 2).sum(0, dtype=F64)]).float()


def fin_ref(stats, count, rm0, rv0):
    """float64 finalisation of fp32 [sum, sumsq] and bounds for the fp32 kernel: the variance E[x^2] - mean^2 cancels,
    so its error scales with E[x^2] + mean^2"""
    ch = stats.numel() // 2
    s = stats.double()
    mean, e2 = s[:ch] / count, s[ch:] / count
    var = (e2 - mean * mean).clamp_min(0)
    invstd = (var + EPS).rsqrt()
    unbiased = var * count / (count - 1)
    rm0, rv0 = rm0.double(), rv0.double()
    var_tol = 4 * U * (e2 + mean * mean)
    ref = dict(mean=mean, invstd=invstd, rm=(1 - MOM) * rm0 + MOM * mean, rv=(1 - MOM) * rv0 + MOM * unbiased)
    tol = dict(mean=2 * U * mean.abs(), invstd=invstd * (6 * U + 0.5 * var_tol / (var + EPS)),
               rm=4 * U * ((1 - MOM) * rm0.abs() + MOM * mean.abs()) + MOM * 2 * U * mean.abs(),
               rv=4 * U * ((1 - MOM) * rv0.abs() + MOM * unbiased) + MOM * var_tol * count / (count - 1))
    return ref, tol


def check_fin(got, stats, count, rm0, rv0, what):
    """got: any of mean, invstd, rm, rv (running mean, running variance) against fin_ref"""
    ref, tol = fin_ref(stats, count, rm0, rv0)
    for k, v in got.items():
        assert_bound(v, ref[k], 0.0, "%s %s" % (what, k), rel=0.0, extra=tol[k])


def affine(gamma, beta, mean, invstd):
    """a BatchNorm as z sc + sh, float64: (sc, sh, the magnitudes of the terms inside sh)"""
    sc = gamma.double() * invstd.double()
    return sc, beta.double() - mean.double() * sc, beta.double().abs() + (mean.double() * sc).abs()


def bn_apply_ref(z, bn, relu, r=None, rbn=None):
    """y = [relu](z sc + sh [+ r | + r rsc + rsh]) and A on z's device; bn, rbn: (sc, sh, A of sh) as affine gives
    them, rbn for a downsample BatchNorm residual"""
    v = lambda t: t.to(z.device, F64)
    sc, sh, sh_abs = map(v, bn)
    zz = z.double()
    f, a = zz * sc + sh, (zz * sc).abs() + sh_abs
    if r is not None:
        rr = r.double()
        if rbn is None:
            f, a = f + rr, a + rr.abs()
        else:
            rsc, rsh, rsh_abs = map(v, rbn)
            f, a = f + rr * rsc + rsh, a + (rr * rsc).abs() + rsh_abs
    return (torch.relu(f) if relu else f), a


def check_bn_apply(y, z, bn, relu, what, r=None, rbn=None):
    """bn_apply / bn_train_apply's y against bn_apply_ref, a batch chunk at a time"""
    for sl in chunks(z.shape[0], z[0].numel()):
        f, a = bn_apply_ref(z[sl], bn, relu, None if r is None else r[sl], rbn)
        assert_bf16(y[sl], f, a, "%s [images %d:%d]" % (what, sl.start, sl.stop))


def bn_grad(dy, ym):
    """g = dy [* (ym > 0)], float64"""
    return dy.double() if ym is None else dy.double() * (ym > 0)


def check_bn_bwd_apply(dz, dy, ym, z, mean, invstd, gamma, dbeta, dgamma, count, what):
    """dz = gamma invstd (g - dbeta / M - xhat dgamma / M), g = bn_grad(dy, ym), a batch chunk at a time"""
    mu, iv = mean.double(), invstd.double()
    a = gamma.double() * iv
    k1, k2 = dbeta.double() / count, dgamma.double() / count
    for sl in chunks(z.shape[0], z[0].numel()):
        gg, zz = bn_grad(dy[sl], None if ym is None else ym[sl]), z[sl].double()
        ref = a * (gg - k1 - (zz - mu) * iv * k2)
        A = a.abs() * (gg.abs() + k1.abs() + (zz.abs() + mu.abs()) * iv * k2.abs())
        assert_bf16(dz[sl], ref, A, "%s [images %d:%d]" % (what, sl.start, sl.stop))


def bn_bwd_reduce_ref(dy, ym, z, mean, invstd):
    """sum g and sum g xhat over the pixels per channel, and their A: (sb, sg, ab, ag)"""
    mu, iv = mean.double(), invstd.double()
    sb = sg = ab = ag = 0
    for sl in chunks(z.shape[0], z[0].numel()):
        gg, zz = bn_grad(dy[sl], None if ym is None else ym[sl]), z[sl].double()
        sb = sb + gg.sum((0, 1, 2))
        sg = sg + (gg * (zz - mu) * iv).sum((0, 1, 2))
        ab = ab + gg.abs().sum((0, 1, 2))
        ag = ag + (gg.abs() * (zz.abs() + mu.abs()) * iv).sum((0, 1, 2))
    return sb, sg, ab, ag


# BatchNorm layers of the ResNet101-UNet at 320x320, at batch 32 or at a larger batch where 32 images do not give every
# thread 3 items
BN = [
    dict(desc="64@160x160", c=64, h=160, w=160, n=32),      # the stem BatchNorm
    dict(desc="64@80x80", c=64, h=80, w=80, n=32),
    dict(desc="256@80x80", c=256, h=80, w=80, n=8),
    dict(desc="128@40x40", c=128, h=40, w=40, n=64),
    dict(desc="512@40x40", c=512, h=40, w=40, n=16),
    dict(desc="256@20x20", c=256, h=20, w=20, n=128),
    dict(desc="1024@20x20", c=1024, h=20, w=20, n=32),
    dict(desc="512@10x10", c=512, h=10, w=10, n=256),
    dict(desc="2048@10x10", c=2048, h=10, w=10, n=64),
    # odd pixel counts: the last pass is partial
    dict(desc="2048@10x10 x33", c=2048, h=10, w=10, n=33, ragged=True),
    dict(desc="64@97x101 x31", c=64, h=97, w=101, n=31, ragged=True),
]
CSUM = BN + [dict(desc="32@320x320", c=32, h=320, w=320, n=32, ragged=True)]   # dec0's bias gradient


def bn_case(c):
    def make():
        g = gen("bn", c["desc"])
        n, h, w, ch = c["n"], c["h"], c["w"], c["c"]
        s = rand(g, ch) * 1.5 + 0.5
        o = (rand(g, ch) - 0.5) * s                      # per-channel offsets, |mean| <= std / 2
        d = dict(z=(randn(g, n, h, w, ch) * s + o).to(BF), r=(randn(g, n, h, w, ch) * 1.2 - 0.1).to(BF),
                 dy=randn(g, n, h, w, ch).to(BF), ym=randn(g, n, h, w, ch).clamp_min(0).to(BF),
                 gamma=rand(g, ch) + 0.5, beta=randn(g, ch) * 0.3, rgamma=rand(g, ch) + 0.5, rbeta=randn(g, ch) * 0.3,
                 rm0=randn(g, ch) * 0.1, rv0=rand(g, ch) + 0.5, rrm0=randn(g, ch) * 0.1, rrv0=rand(g, ch) + 0.5)
        m = n * h * w
        # backward operands: the forward's saved mean / invstd, gamma and the global dbeta / dgamma
        d.update(bmean=randn(g, ch) * 0.2, binv=rand(g, ch) + 0.5, bgamma=randn(g, ch),
                 dbeta=randn(g, ch) * 0.3 * m, dgamma=randn(g, ch) * 0.3 * m)
        d["zstats"], d["rstats"] = channel_stats(d["z"]), channel_stats(d["r"])
        return d
    return cached(("bn", c["desc"]), make)


def resnet101_unet_layout():
    """(fp32 arena length, BatchNorm widths) of UNetResNet(101, 2)"""
    if not _LAYOUT:
        from mcb200 import unet_models
        net = unet_models.UNetResNet(101, 2, is_deconv=True)
        _LAYOUT["arena"] = net._p32.numel()
        _LAYOUT["bns"] = [m.num_features for m in net.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    return _LAYOUT["arena"], _LAYOUT["bns"]


# --------------------------------------------------------------------------------------------------- 2x2 max-pool
POOL = [dict(desc="64@160x160->80x80", c=64, h=160, w=160, n=32),     # after the stem
        dict(desc="2048@10x10->5x5", c=2048, h=10, w=10, n=160, ragged=True)]


def pool_ref(x, dy):
    """2x2 max-pool of NHWC x and its backward by torch's index rule: scanning a window in order (0,0), (0,1), (1,0),
    (1,1), a position takes over when it is greater than the current maximum or is NaN -- the first maximum, or the
    last NaN.  -> (the pooled max, dy routed to x's shape), in x's dtype (exact: every value is one of the operands)"""
    n, h, w, ch = x.shape
    xv = x.view(n, h // 2, 2, w // 2, 2, ch)
    m, best = xv[:, :, 0, :, 0], torch.zeros(dy.shape, dtype=torch.int8, device=x.device)
    for k in (1, 2, 3):
        v = xv[:, :, k // 2, :, k % 2]
        upd = (v > m) | v.isnan()
        m, best = torch.where(upd, v, m), torch.where(upd, torch.full_like(best, k), best)
    routed = torch.zeros(x.shape, dtype=dy.dtype, device=x.device)
    rv = routed.view(n, h // 2, 2, w // 2, 2, ch)
    for k in range(4):
        rv[:, :, k // 2, :, k % 2] = torch.where(best == k, dy, torch.zeros_like(dy))
    return m, routed


def pool_skip_ref(y, g, dpool):
    """maxpool2_bwd_skip_relu's g: (y <= 0) ? 0 : bf16(g + dpool routed by pool_ref), as torch's relu backward (a NaN y
    passes the gradient)"""
    t = (g.float() + pool_ref(y, dpool)[1].float()).to(BF)
    return torch.where(y <= 0, torch.zeros_like(t), t)


# ------------------------------------------------------------------------------------------------- 1x1 classifier
def classifier_fwd_ref(x, wt, b):
    """logits = W x + b (NHWC x, K x C weights) as NCHW float64, and A"""
    xs, w64, b64 = x.double(), wt.to(x.device, F64), b.to(x.device, F64).view(1, -1, 1, 1)
    return (torch.einsum("nhwc,kc->nkhw", xs, w64) + b64,
            torch.einsum("nhwc,kc->nkhw", xs.abs(), w64.abs()) + b64.abs())


def classifier_bwd_ref(x, wt, dl):
    """dx = (x > 0) W^T dlogits and A, dW = sum dlogits x^T and A (flattened K x C), db = sum dlogits and A"""
    xs, ds, w64 = x.double(), dl.to(x.device, F64), wt.to(x.device, F64)
    gx = torch.where(xs > 0, torch.einsum("nkhw,kc->nhwc", ds, w64), torch.zeros((), dtype=F64, device=x.device))
    return (gx, torch.einsum("nkhw,kc->nhwc", ds.abs(), w64.abs()),
            torch.einsum("nkhw,nhwc->kc", ds, xs).reshape(-1),
            torch.einsum("nkhw,nhwc->kc", ds.abs(), xs.abs()).reshape(-1),
            ds.sum((0, 2, 3)), ds.abs().sum((0, 2, 3)))


# ------------------------------------------------------------------------------------------------------------ loss
LOSS_N, LOSS_S = 32, 320
SIZE_C = math.sqrt(LOSS_S * LOSS_S) / 2.0   # the size weight's constant for 320 x 320 tiles


def loss_case():
    """logits (N, 2, S, S) and targets (N, 3, S, S) at the train step's batch 32 and 320 x 320"""
    def make():
        _, t = synthetic.train_batch(LOSS_N, LOSS_S, seed=320, n_rect=40)
        t = torch.from_numpy(t)
        t[:, 2, ::9, ::7] = 0                # size 0 (weight 1) pixels, inside and outside buildings
        t = t.to("cuda")
        g = gen("loss")
        logits = randn(g, LOSS_N, 2, LOSS_S, LOSS_S) * 2
        logits[:, 1] += 1.5 * (2 * t[:, 0] - 1)   # a partly trained net: mostly, not always, right
        return logits, t
    return cached(("loss",), make)


def loss_ref(logits, t, mode):
    """float64 for loss_partials / loss_grad, mode 0 (weighted CE + Dice) or 1 (plain CE): the four sums [I, P, T, S],
    the softmax, and the bound on d(loss)/d(logits) per pixel (N, 1, H, W): 2^-18 of its CE weight / M and Dice term"""
    s = logits.shape[-1]
    z, t64 = logits.double(), t.double()
    p = torch.softmax(z, 1)
    p0, p1 = p[:, 0], p[:, 1]
    t1 = (t64[:, 0].long() == 1).double()
    w = O.loss_weights(t64, imsize=(s, s)) if mode == 0 else torch.ones_like(p1)
    ce = torch.logsumexp(z, 1) - torch.where(t64[:, 0].long() != 0, z[:, 1], z[:, 0])
    sums = torch.stack([(p1 * t1).sum(), p1.sum(), t1.sum(), (w * ce).sum()])
    tol = w / p1.numel()
    if mode == 0:
        I, P, T = (float(v) for v in sums[:3])
        dn, num = P + T + 1.0 + 1e-7, 2 * I + 1.0
        tol = tol + 0.2 * (t1 * 2 / dn + num / dn ** 2) * p1 * p0
    return sums, p, 2.0 ** -18 * tol.unsqueeze(1)


# ------------------------------------------------------------------------------------------------------------ Adam
BETAS, ADAM_EPS, WD, GRAD_SCALE, STEPS = (0.9, 0.999), 1e-8, 1e-4, 0.3, 10


def adam_lr(t):
    return 5e-4 * (1 - 0.05 * t)


def ulp32(x):
    """spacing of fp32 at the fp32 value nearest x"""
    a = x.float().abs()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def check_adam(t, lr, p0, m0, v0, grad, p, m, v, what):
    """one step against float64 Adam (L2 decay folded into the gradient).  As in torch.optim.Adam, the bias
    corrections come from the caller's double betas; the moment updates, lr, eps, weight decay and gradient scale
    take the fp32 values the kernel receives"""
    f = lambda x: C.c_float(x).value
    b1, b2, lr, eps, wd, gs = f(BETAS[0]), f(BETAS[1]), f(lr), f(ADAM_EPS), f(WD), f(GRAD_SCALE)
    bc1, bc2s = 1 - BETAS[0] ** t, math.sqrt(1 - BETAS[1] ** t)
    step = 1 << 22
    for lo in range(0, p.numel(), step):
        s = slice(lo, lo + step)
        P0, M0, V0, G = p0[s].double(), m0[s].double(), v0[s].double(), grad[s].double()
        gi = G * gs + wd * P0
        gmag = (G * gs).abs() + (wd * P0).abs()
        mr = b1 * M0 + (1 - b1) * gi
        vr = b2 * V0 + (1 - b2) * gi * gi
        denom = vr.sqrt() / bc2s + eps
        pr = P0 - lr / bc1 * mr / denom
        mmag = b1 * M0.abs() + (1 - b1) * gmag
        vmag = b2 * V0 + (1 - b2) * gmag * gmag
        umag = lr / bc1 * mmag / denom
        at = " step %d [%d:%d]" % (t, lo, min(lo + step, p.numel()))
        assert_bound(m[s], mr, 0.0, what + " m" + at, rel=0.0, extra=2.0 ** -20 * mmag)
        assert_bound(v[s], vr, 0.0, what + " v" + at, rel=0.0, extra=2.0 ** -20 * vmag)
        assert_bound(p[s], pr, 0.0, what + " p" + at, rel=0.0, extra=2.0 ** -18 * umag + ulp32(pr))


# ---------------------------------------------------------------------------------------- fixed-order finishing sum
def reference_sum(rows):
    """float32, the library's order: rows [R, n] -> [n]; per lane l < 32 the rows l, l + 32, ... added in turn, then the
    lanes combined as a butterfly (16, 8, 4, 2, 1)"""
    lanes = []
    for l in range(32):
        t = np.zeros(rows.shape[1], np.float32)
        for r in range(l, rows.shape[0], 32):
            t = (t + rows[r]).astype(np.float32)
        lanes.append(t)
    o = 16
    while o:
        for l in range(o):
            lanes[l] = (lanes[l] + lanes[l + o]).astype(np.float32)
        o //= 2
    return lanes[0]


def wide_range_rows(rng, nrows, n):
    """magnitudes over six decades, so that a different association changes the rounding"""
    return (rng.standard_normal((nrows, n)) * 10.0 ** rng.uniform(-3, 3, (nrows, n))).astype(np.float32)


def run_det_sum(rows_h, n, inner, out_stride, out_h):
    """mcb_det_sum_f32 over the host rows into a device copy of out_h -> the result on the host"""
    from mcb200 import _lib as L
    rows = torch.from_numpy(rows_h).to("cuda")
    out = torch.from_numpy(out_h.copy()).to("cuda")
    L.fcall("mcb_det_sum_f32", rows.data_ptr(), rows_h.shape[0], rows_h.shape[1], n, inner, out.data_ptr(), out_stride)
    torch.cuda.synchronize()
    return out.cpu().numpy()
