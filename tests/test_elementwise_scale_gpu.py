"""The HBM-bound kernels (csrc/elementwise.cu, csrc/loss.cu) at the batch-32 sizes of the ResNet101-UNet at 320x320,
where every thread of their capped grid-stride loops runs several iterations.

grid_for() caps a grid at 8 x SMs blocks of 256 threads; the BatchNorm apply kernels handle two 16-byte groups (i,
i + stride) per iteration; channel_reduce_kernel and final_conv_bwd_kernel cap at 4 x SMs blocks and keep a private
partial per thread that detsum.cuh adds in block order; the loss kernels cap at 8 x SMs blocks.  Every case asserts,
from the device's SM count and these launch formulas, that each thread (or each pixel lane of a reduction block) owns
at least 3 work items, and the cases marked ragged also assert a partial last pass (for the BatchNorm kernels: a
thread whose second group falls off the end).  Shapes are the network's layers "C@HxW" at batch 32, or at a larger
batch where 32 images do not give every thread 3 items; one tensor case lives in device memory at a time.

References are float64 from the bf16-rounded operands; A is the same operation on |operands|.
  * integer-exact cases (channel sums, BatchNorm backward sums, the classifier) and pure data movement (max-pool with
    its first-maximum tie rule, layout conversions, stem im2col, fp32 -> bf16) must match exactly; sums stay < 2^24;
  * real-valued reductions: |got - ref| <= 2^-16 A, and a second run repeats the first bitwise;
  * bf16 outputs: |got - ref| <= 2^-8 |ref| (half a bf16 ulp) + 2^-20 A;
  * BatchNorm statistics (mean, invstd, running mean / unbiased running variance) within a few fp32 ulps of the
    float64 finalisation, scaled by the magnitudes the fp32 arithmetic cancels;
  * the loss within 1e-6 relative, d(loss)/d(logits) per pixel within 2^-18 of that pixel's own CE weight / M and
    Dice term;
  * Adam, one step at a time from the kernel's own state, within 2^-18 of the step's update size (magnitudes) plus
    one fp32 ulp of p; m and v within 2^-20 of their terms' magnitudes."""
import ctypes as C
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from oracle import synthetic
from oracle import unet_oracle as O

pytestmark = pytest.mark.gpu

BF, F64 = torch.bfloat16, torch.float64
U = 2.0 ** -24                       # fp32 unit roundoff
MOM, EPS = C.c_float(0.1).value, C.c_float(1e-5).value   # BatchNorm momentum / eps as the kernels receive them

_CASE = {}    # the current case's tensors: one case at a time, so device memory stays bounded
_LAYOUT = {}  # UNetResNet(101)'s arena length and BatchNorm widths


# ---------------------------------------------------------------------------------------------------------- helpers
def cached(key, make):
    if key not in _CASE:
        _CASE.clear()
        _CASE[key] = make()
    return _CASE[key]


def gen(*key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))


def randn(g, *shape):
    return torch.randn(shape, generator=g, device="cuda")


def rand(g, *shape):
    return torch.rand(shape, generator=g, device="cuda")


def ints(g, lo, hi, *shape):
    """integers in [lo, hi] as float32"""
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda", dtype=torch.int8).float()


def chunks(n, per_image, limit=1 << 23):
    """batch slices of at most `limit` elements: bounds the float64 temporaries of a reference"""
    step = max(1, limit // per_image)
    return [slice(i, min(n, i + step)) for i in range(0, n, step)]


def assert_bound(got, ref, tol, what):
    """|got - ref| <= tol element-wise (NaN counts as a failure)"""
    got = got.double()
    ref = ref.to(got.device, F64)
    err = (got - ref).abs()
    bad = ~(err <= tol)
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        t = float(tol[i]) if torch.is_tensor(tol) else tol
        raise AssertionError("%s: %d/%d elements off, max err %g; first at %s: got %r, ref %r, bound %g" % (
            what, int(bad.sum()), bad.numel(), float(err.nan_to_num(float("inf")).max()), i, float(got[i]),
            float(ref[i]), t))


def assert_exact(got, ref, what):
    """equal values (+0 and -0 alike)"""
    ref = ref.to(got.device)
    if got.dtype != ref.dtype:
        got, ref = got.double(), ref.double()
    bad = got != ref
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError("%s: %d/%d elements differ; first at %s: got %r, ref %r" % (
            what, int(bad.sum()), bad.numel(), i, float(got[i]), float(ref[i])))


def assert_same(a, b, what):
    """bitwise repeat of a run"""
    assert torch.equal(a, b), "%s: two runs differ in %d elements" % (what, int((a != b).sum()))


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid_for(work, threads, per_sm=8):
    """elementwise.cu grid_for (also loss.cu loss_grid with 256 threads)"""
    return max(1, min(-(-work // threads), sms() * per_sm))


def assert_stride_regime(work, threads, per_sm=8, ragged=False, pair=False):
    """a grid-stride loop over `work` items launched with grid_for: every thread owns at least 3 items; ragged: the last
    pass is partial.  pair: the BatchNorm apply kernels, launched over ceil(work / 2) items, take items i and
    i + stride per iteration -- ragged then means some thread's last iteration has no second item"""
    grid = grid_for((work + 1) // 2 if pair else work, threads, per_sm)
    t = grid * threads
    assert work // t >= 3, "%d items over %d threads (%d SMs)" % (work, t, sms())
    if ragged:
        span = 2 * t if pair else t
        assert work % span, "%d items fill every pass of %d threads" % (work, span)


def assert_reduce_regime(pixels, c, ragged=False):
    """channel_reduce_kernel: 256 - 256 % (C/8) threads = lanes x C/8, grid min(pixels / (4 lanes), 4 x SMs); each
    pixel lane owns at least 3 pixels; ragged: some lane's last iteration has no second pixel"""
    c8 = c // 8
    threads = max(256 - 256 % c8, c8)
    lanes = threads // c8
    grid = max(1, min(-(-pixels // (lanes * 4)), sms() * 4))
    assert pixels // (grid * lanes) >= 3, "%d pixels over %d lanes (%d SMs)" % (pixels, grid * lanes, sms())
    if ragged:
        assert pixels % (2 * grid * lanes)


def ulp32(x):
    """spacing of fp32 at the fp32 value nearest x"""
    a = x.float().abs()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def resnet101_unet_layout():
    """(fp32 arena length, BatchNorm widths) of UNetResNet(101, 2)"""
    if not _LAYOUT:
        from mcb200 import unet_models
        net = unet_models.UNetResNet(101, 2, is_deconv=True)
        _LAYOUT["arena"] = net._p32.numel()
        _LAYOUT["bns"] = [m.num_features for m in net.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    return _LAYOUT["arena"], _LAYOUT["bns"]


# =====================================================================================================================
# BatchNorm: train-apply (finalisation folded in), finalize + eval apply, backward apply and reduce, channel sums
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


def ids(cases):
    return [c["desc"].replace(" ", "_") for c in cases]


def channel_stats(x):
    """[sum, sumsq] per channel of an NHWC bf16 tensor, as the conv epilogue hands them over (fp32)"""
    v = x.view(-1, x.shape[-1])
    return torch.cat([v.sum(0, dtype=F64), (v.float() ** 2).sum(0, dtype=F64)]).float()


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
    ref, tol = fin_ref(stats, count, rm0, rv0)
    for k, v in got.items():
        assert_bound(v, ref[k], tol[k], "%s %s" % (what, k))


def check_apply(y, d, sc, sh, sh_abs, res, rsc, rsh, rsh_abs, relu, what):
    """y = [relu](z * sc + sh [+ r | + r * rsc + rsh]); sh_abs, rsh_abs: magnitudes of the terms inside the shifts"""
    z, r = d["z"], d["r"]
    n = z.shape[0]
    for sl in chunks(n, z[0].numel()):
        zz = z[sl].double()
        f = zz * sc + sh
        a = (zz * sc).abs() + sh_abs
        if res == 1:
            rr = r[sl].double()
            f, a = f + rr, a + rr.abs()
        elif res == 2:
            rr = r[sl].double()
            f, a = f + rr * rsc + rsh, a + (rr * rsc).abs() + rsh_abs
        if relu:
            f = f.clamp_min(0)
        assert_bound(y[sl], f, 2.0 ** -8 * f.abs() + 2.0 ** -20 * a, "%s [images %d:%d]" % (what, sl.start, sl.stop))


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
    rtr = None
    if res == 2:
        rrm, rrv, rmean, rinv = d["rrm0"].clone(), d["rrv0"].clone(), e(), e()
        rtr = ops.make_bn_train(d["rstats"], d["rgamma"], d["rbeta"], rrm, rrv, rmean, rinv)
    y = torch.empty_like(z)
    ops.bn_train_apply(z, tr, y, relu, resid, rtr)
    check_fin(dict(mean=mean, invstd=inv, rm=rm, rv=rv), d["zstats"], pixels, d["rm0"], d["rv0"], "bn_train_apply")
    sc = d["gamma"].double() * inv.double()
    sh, sh_abs = d["beta"].double() - mean.double() * sc, d["beta"].double().abs() + (mean.double() * sc).abs()
    rsc = rsh = rsh_abs = None
    if res == 2:
        check_fin(dict(mean=rmean, invstd=rinv, rm=rrm, rv=rrv), d["rstats"], pixels, d["rrm0"], d["rrv0"],
                  "bn_train_apply residual BN")
        rsc = d["rgamma"].double() * rinv.double()
        rsh = d["rbeta"].double() - rmean.double() * rsc
        rsh_abs = d["rbeta"].double().abs() + (rmean.double() * rsc).abs()
    check_apply(y, d, sc, sh, sh_abs, res, rsc, rsh, rsh_abs, relu, "bn_train_apply")
    # finalize + eval apply
    rm, rv, mean, inv, scale, shift = d["rm0"].clone(), d["rv0"].clone(), e(), e(), e(), e()
    ops.bn_finalize(d["zstats"], pixels, d["gamma"], d["beta"], rm, rv, scale, shift, mean, inv)
    check_fin(dict(mean=mean, invstd=inv, rm=rm, rv=rv), d["zstats"], pixels, d["rm0"], d["rv0"], "bn_finalize")
    rscale = rshift = None
    if res == 2:
        rscale, rshift, rmean, rinv = e(), e(), e(), e()
        ops.bn_finalize(d["rstats"], pixels, d["rgamma"], d["rbeta"], None, None, rscale, rshift, rmean, rinv)
        rsc, rsh, rsh_abs = rscale.double(), rshift.double(), rshift.double().abs()
    y = torch.empty_like(z)
    ops.bn_apply(z, scale, shift, y, relu, resid, rscale, rshift)
    check_apply(y, d, scale.double(), shift.double(), shift.double().abs(), res, rsc, rsh, rsh_abs, relu, "bn_apply")


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
    mu, iv = d["bmean"].double(), d["binv"].double()
    a = d["bgamma"].double() * iv
    k1, k2 = d["dbeta"].double() / pixels, d["dgamma"].double() / pixels
    for sl in chunks(n, z[0].numel()):
        gg = dy[sl].double()
        if mask:
            gg = gg * (ym[sl] > 0)
        zz = z[sl].double()
        ref = a * (gg - k1 - (zz - mu) * iv * k2)
        A = a.abs() * (gg.abs() + k1.abs() + (zz.abs() + mu.abs()) * iv * k2.abs())
        assert_bound(dz[sl], ref, 2.0 ** -8 * ref.abs() + 2.0 ** -20 * A, "bn_bwd_apply dz [images %d:%d]" % (
            sl.start, sl.stop))
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
    mu, iv = mean.double(), inv.double()
    sb = sg = ab = ag = 0
    for sl in chunks(n, z[0].numel()):
        gg = dy[sl].double()
        if ym is not None:
            gg = gg * (ym[sl] > 0)
        zz = z[sl].double()
        sb = sb + gg.sum((0, 1, 2))
        sg = sg + (gg * (zz - mu) * iv).sum((0, 1, 2))
        ab = ab + gg.abs().sum((0, 1, 2))
        ag = ag + (gg.abs() * (zz.abs() + mu.abs()) * iv).sum((0, 1, 2))
    (db, dgm), (db2, dgm2) = runs
    ref_b, ref_g = pre_b.double() + sb, pre_g.double() + sg
    ab, ag = ab + pre_b.double().abs(), ag + pre_g.double().abs()
    if kind == "exact":
        assert max(float(ab.max()), float(ag.max())) < 2 ** 24
        assert_exact(db, ref_b, "dbeta")
        assert_exact(dgm, ref_g, "dgamma")
    else:
        assert_bound(db, ref_b, 2.0 ** -16 * ab, "dbeta")
        assert_bound(dgm, ref_g, 2.0 ** -16 * ag, "dgamma")
    assert_same(db, db2, "dbeta")
    assert_same(dgm, dgm2, "dgamma")


CSUM = BN + [dict(desc="32@320x320", c=32, h=320, w=320, n=32, ragged=True)]   # dec0's bias gradient


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
    ref = pre.double() + v.sum(0, dtype=F64)
    A = pre.double().abs() + v.abs().sum(0, dtype=F64)
    if exact == "exact":
        assert float(A.max()) < 2 ** 24
        assert_exact(runs[0], ref, "channel_sum")
    else:
        assert_bound(runs[0], ref, 2.0 ** -16 * A, "channel_sum")
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
POOL = [dict(desc="64@160x160->80x80", c=64, h=160, w=160, n=32),     # after the stem
        dict(desc="2048@10x10->5x5", c=2048, h=10, w=10, n=160, ragged=True)]


@pytest.mark.parametrize("c", POOL, ids=ids(POOL))
def test_maxpool(mcb, cuda, c):
    """forward max, and the backward routing every gradient to the FIRST maximum of its window in scan order, stored
    (all four positions overwritten) or added to an existing gradient"""
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
    xv = x.view(n, ho, 2, wo, 2, ch)
    cands = [xv[:, :, ky, :, kx] for ky in (0, 1) for kx in (0, 1)]   # scan order
    m, best = cands[0], torch.zeros(cands[0].shape, dtype=torch.int8, device=cuda)
    for k in (1, 2, 3):
        upd = cands[k] > m
        m = torch.where(upd, cands[k], m)
        best = torch.where(upd, torch.full_like(best, k), best)
    assert bool((cands[0] == cands[1]).any()), "no ties"
    assert_exact(ops.maxpool2_fwd(x), m, "maxpool2_fwd")
    routed = torch.zeros_like(x)
    rv = routed.view(n, ho, 2, wo, 2, ch)
    for k in range(4):
        rv[:, :, k // 2, :, k % 2] = torch.where(best == k, dy, torch.zeros_like(dy))
    del best, m, cands
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
    w64, b64 = wt.double(), b.double().view(1, k, 1, 1)
    sw = sb = aw = ab = 0
    dx = runs[0][0]
    for sl in chunks(n, h * w * ch):
        xs, ds = x[sl].double(), dl[sl].double()
        lg = torch.einsum("nhwc,kc->nkhw", xs, w64) + b64
        la = torch.einsum("nhwc,kc->nkhw", xs.abs(), w64.abs()) + b64.abs()
        gx = torch.einsum("nkhw,kc->nhwc", ds, w64)
        gx = torch.where(xs > 0, gx, torch.zeros_like(gx))
        ga = torch.einsum("nkhw,kc->nhwc", ds.abs(), w64.abs())
        sw = sw + torch.einsum("nkhw,nhwc->kc", ds, xs)
        aw = aw + torch.einsum("nkhw,nhwc->kc", ds.abs(), xs.abs())
        sb, ab = sb + ds.sum((0, 2, 3)), ab + ds.abs().sum((0, 2, 3))
        what = " [images %d:%d]" % (sl.start, sl.stop)
        if exact:
            assert_exact(logits[sl], lg, "final_conv_fwd" + what)
            assert_exact(dx[sl], gx, "final_conv_bwd dx" + what)
        else:
            assert_bound(logits[sl], lg, 2.0 ** -16 * la, "final_conv_fwd" + what)
            assert_bound(dx[sl], gx, 2.0 ** -8 * gx.abs() + 2.0 ** -20 * ga, "final_conv_bwd dx" + what)
    ref_w, ref_b = pre_w.double() + sw.reshape(-1), pre_b.double() + sb
    aw, ab = pre_w.double().abs() + aw.reshape(-1), pre_b.double().abs() + ab
    (dx, dw, db), (dx2, dw2, db2) = runs
    if exact:
        assert max(float(aw.max()), float(ab.max())) < 2 ** 24
        assert_exact(dw, ref_w, "final_conv_bwd dW")
        assert_exact(db, ref_b, "final_conv_bwd db")
    else:
        assert_bound(dw, ref_w, 2.0 ** -16 * aw, "final_conv_bwd dW")
        assert_bound(db, ref_b, 2.0 ** -16 * ab, "final_conv_bwd db")
    assert_same(dx, dx2, "final_conv_bwd dx")
    assert_same(dw, dw2, "final_conv_bwd dW")
    assert_same(db, db2, "final_conv_bwd db")


# =====================================================================================================================
# losses at 32 x 320 x 320
LOSS_N, LOSS_S = 32, 320
SIZE_C = math.sqrt(LOSS_S * LOSS_S) / 2.0   # the size weight's constant for 320 x 320 tiles


def loss_case():
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
    with torch.no_grad():
        z = logits.double()
        p = torch.softmax(z, 1)
        p0, p1 = p[:, 0], p[:, 1]
        t1 = (t64[:, 0].long() == 1).double()
        w = O.loss_weights(t64, imsize=(LOSS_S, LOSS_S)) if mode == 0 else torch.ones_like(p1)
        ce = torch.logsumexp(z, 1) - torch.where(t64[:, 0].long() != 0, z[:, 1], z[:, 0])
        ref_sums = torch.stack([(p1 * t1).sum(), p1.sum(), t1.sum(), (w * ce).sum()])
    # every term is non-negative: A = ref
    assert_bound(sums, ref_sums, 2.0 ** -16 * ref_sums, "loss sums [I, P, T, S]")
    assert_exact(sums[2], ref_sums[2], "loss sum T")
    assert abs(float(loss) - float(ref)) <= 1e-6 * abs(float(ref)), (float(loss), float(ref))
    tol = w / pixels
    if mode == 0:
        I, P, T = (float(v) for v in ref_sums[:3])
        dn, num = P + T + 1.0 + 1e-7, 2 * I + 1.0
        tol = tol + 0.2 * (t1 * 2 / dn + num / dn ** 2) * p1 * p0
    assert_bound(dlog, lg.grad, 2.0 ** -18 * tol.unsqueeze(1), "dlogits")
    if mode == 0:
        pr = ops.softmax2(logits)
        assert_bound(pr, p, 2.0 ** -18 * p, "softmax2")


# =====================================================================================================================
# fused Adam over the ResNet101-UNet parameter arena
BETAS, ADAM_EPS, WD, GRAD_SCALE, STEPS = (0.9, 0.999), 1e-8, 1e-4, 0.3, 10


def adam_lr(t):
    return 5e-4 * (1 - 0.05 * t)


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
        assert_bound(m[s], mr, 2.0 ** -20 * mmag, what + " m" + at)
        assert_bound(v[s], vr, 2.0 ** -20 * vmag, what + " v" + at)
        assert_bound(p[s], pr, 2.0 ** -18 * umag + ulp32(pr), what + " p" + at)


@pytest.mark.parametrize("entry", ["adam_step", "adam_step_dyn"])
def test_adam_arena(mcb, cuda, entry):
    """STEPS steps over a vector the length of UNetResNet(101)'s fp32 arena, each checked from the kernel's own state;
    adam_step_dyn reads {lr, 1 - beta1^t, sqrt(1 - beta2^t)} from the device, as the captured train step does"""
    from mcb200 import ops
    n, _ = resnet101_unet_layout()
    assert_stride_regime(n, 256, ragged=True)
    _CASE.clear()
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
    _CASE.clear()
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
def with_ties(x, g):
    """plant fp32 values exactly halfway between two bf16 values (round to nearest even decides)"""
    k = min(x.numel(), 1 << 16)
    y = randn(g, k).to(BF).float()
    x.view(-1)[:k] = (y.view(torch.int32) | 0x8000).view(torch.float32)
    return x


def test_layout_conversions(mcb, cuda):
    from mcb200 import ops
    n, ch, h, w = 32, 3, 320, 320
    assert_stride_regime(n * ch * h * w, 256, ragged=True)
    _CASE.clear()
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
    _CASE.clear()
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
    _CASE.clear()
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
