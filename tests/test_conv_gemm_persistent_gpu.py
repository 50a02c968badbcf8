"""The convolution kernels in the persistent, multi-tile regime the full-size network runs.

conv_gemm_kernel is persistent: the grid is min(tiles, SMs) and each CTA walks tiles t = blockIdx.x, += gridDim.x,
carrying from one tile to the next the TMA ring position and mbarrier parity, the haloed A ring, the rotation of the
output staging buffers, the aux-tile prefetch of the next tile and the per-channel reduction registers (flushed when
the N tile changes).  wgrad_kernel runs its ring over many K blocks per CTA and adds into an existing dW.  Every
convolution case here puts at least two tiles on every CTA (asserted against the device's SM count) and sweeps the
existing knobs: MCB_FORCE_BN (N tile width), MCB_HALO (0 never, 1 wherever the haloed tile fits, 2 the default rule)
and MCB_WGRAD_SPLITS.  Shapes are layers of the ResNet101-UNet at 320x320 ("cin->cout kK sS @HxW"), at small batches;
the deep layers (20x20, 10x10) take more images so that the persistent grid still wraps.

References are float64 on the CPU from the bf16-rounded operands; A, the same op on |operands|, scales the fp32
accumulation error.  bf16 outputs: |got - ref| <= 2^-8 |ref| + 2^-16 A (half a bf16 ulp plus an accumulation
allowance far above the realistic ~2^-24 A, far below one dropped product term, tap or channel chunk).  fp32 weight
gradients: |got - ref| <= 2^-16 A.  Integer-exact variants (operands in {-1, 0, 1}, |ref| <= 256, sums < 2^24) must
match bitwise, fused reductions included; real-valued fused reductions must repeat bitwise from run to run."""
import itertools
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

_REF = {}  # references per case, shared by the knob sweeps


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def bf16r(x):
    return x.to(torch.bfloat16).to(torch.float32)


def dev(x):
    """NCHW float -> NHWC bf16 on the GPU"""
    return nhwc(x).to("cuda", torch.bfloat16)


def cached(key, make):
    if key not in _REF:
        _REF[key] = make()
    return _REF[key]


def gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def ints(g, shape, density=1.0):
    """values in {-1, 0, 1}; a nonzero with probability 2/3 * density"""
    v = torch.randint(-1, 2, shape, generator=g).float()
    return v * (torch.rand(shape, generator=g) < density).float() if density < 1 else v


def int_density(k_terms):
    """weight density for K-term integer dot products: E[v^2] = 16, so max|v| stays far below 256 and the per-channel
    sums of v^2 over <= 10^5 pixels below 2^24"""
    return min(1.0, 24.0 / k_terms)


def assert_bound(got, ref, absref, what, rel=2.0 ** -8, extra=0.0):
    """|got - ref| <= rel |ref| + 2^-16 absref + extra element-wise (rel = 0, absref = 0: exact)"""
    got = got.double()
    d = got.device
    ref = ref.to(d, torch.float64)
    absref = absref.to(d, torch.float64) if torch.is_tensor(absref) else absref
    extra = extra.to(d, torch.float64) if torch.is_tensor(extra) else extra
    err = (got - ref).abs()
    bad = ~(err <= rel * ref.abs() + 2.0 ** -16 * absref + extra)  # (NaN counts as bad)
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        a = float(absref[i]) if torch.is_tensor(absref) else absref
        raise AssertionError("%s: %d/%d elements off, max err %g; first at %s: got %r, ref %r, A %g" % (
            what, int(bad.sum()), bad.numel(), float(err.nan_to_num(float("inf")).max()), i, float(got[i]),
            float(ref[i]), a))


def assert_exact(got, ref, what):
    assert_bound(got, ref, 0.0, what, rel=0.0)


def assert_same(a, b, what):
    """bitwise repeat of a run"""
    assert torch.equal(a, b), "%s: two runs differ in %d elements" % (what, int((a != b).sum()))


def assert_multi_tile(n, hv, wv, n_extent, bn, phases=1):
    """at least two tiles on every CTA of the persistent grid.  A pixel tile has <= 128 rows, so
    ceil(pixels / 128) x N tiles x phases is a lower bound on the tile count.  A forced BN that does not divide the N
    extent is ignored by the host; the bound then takes the widest possible tile."""
    bn = bn if n_extent % bn == 0 else n_extent
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = -(-n * hv * wv // 128) * (n_extent // bn) * phases
    assert tiles >= 2 * sms, "only %d tiles (lower bound) for %d SMs" % (tiles, sms)


def set_knobs(monkeypatch, bn=None, halo=None, splits=None):
    for name, v in (("MCB_FORCE_BN", bn), ("MCB_HALO", halo), ("MCB_WGRAD_SPLITS", splits)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, str(v))


def sweep(cases, *axes, halo=False):
    """pytest params: case x its BN list x (halo: its MCB_HALO list, the default rule if it has none) x axes"""
    out = []
    for c in cases:
        for bn in c.get("bn", (None,)):
            for hm in c.get("halo", (2,)) if halo else (None,):
                for vs in itertools.product(*axes):
                    args = [c] + [a for a in (bn, hm) if a is not None] + list(vs)
                    parts = [c["desc"].replace(" ", "_")] + (["BN%d" % bn] if bn else []) + \
                        (["halo%d" % hm] if halo and "halo" in c else []) + list(vs)
                    out.append(pytest.param(*args, id="-".join(parts)))
    return out


# =====================================================================================================================
# forward (conv_fwd): bias; ReLU + BatchNorm statistics; concatenated inputs (c1 > 0)
FWD = [
    dict(desc="64->64 k3 s1 @80x80", n=6, h=80, w=80, c0=64, c1=0, cout=64, k=3, s=1, bn=(32, 64), halo=(2, 1)),
    dict(desc="64->256 k1 s1 @80x80", n=6, h=80, w=80, c0=64, c1=0, cout=256, k=1, s=1, bn=(32, 64, 128, 256)),
    dict(desc="128->128 k3 s2 @80x80", n=8, h=80, w=80, c0=128, c1=0, cout=128, k=3, s=2, bn=(32,)),
    dict(desc="256->512 k1 s2 @80x80", n=6, h=80, w=80, c0=256, c1=0, cout=512, k=1, s=2, bn=(32, 64, 128)),
    dict(desc="1024->256 k1 s1 @20x20", n=12, h=20, w=20, c0=1024, c1=0, cout=256, k=1, s=1, bn=(32,)),
    # several images per pixel tile, ragged tiles
    dict(desc="512->512 k3 s1 @10x10", n=22, h=10, w=10, c0=512, c1=0, cout=512, k=3, s=1, bn=(32,)),
    # the default rule takes the haloed tile here
    dict(desc="128->128 k3 s1 @160x160", n=2, h=160, w=160, c0=128, c1=0, cout=128, k=3, s=1, bn=(32, 64, 128),
         halo=(2, 0)),
    dict(desc="32->32 k3 s1 @320x320", n=1, h=320, w=320, c0=32, c1=0, cout=32, k=3, s=1, bn=(32,), halo=(2, 1)),
    dict(desc="256+64->128 k3 s1 @80x80", n=6, h=80, w=80, c0=256, c1=64, cout=128, k=3, s=1, bn=(32, 64, 128),
         halo=(2, 1)),
    dict(desc="512+256->256 k3 s1 @40x40", n=8, h=40, w=40, c0=512, c1=256, cout=256, k=3, s=1, bn=(32, 64),
         halo=(2, 1)),
    # haloed tile over two sources with unequal chunk counts (2 + 4)
    dict(desc="128+256->128 k3 s1 @32x48", n=11, h=32, w=48, c0=128, c1=256, cout=128, k=3, s=1, bn=(32, 64),
         halo=(1,)),
]
FWD_BY_DESC = {c["desc"]: c for c in FWD}


def fwd_ref(c, exact):
    def make():
        g = gen("fwd", c["desc"], exact)
        cin, k, cout = c["c0"] + c["c1"], c["k"], c["cout"]
        if exact:
            x = ints(g, (c["n"], cin, c["h"], c["w"]))
            wt = ints(g, (cout, cin, k, k), int_density(cin * k * k))
            b = torch.randint(-3, 4, (cout,), generator=g).float()
        else:
            x = bf16r(torch.randn(c["n"], cin, c["h"], c["w"], generator=g))
            wt = bf16r(torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5)
            b = torch.randn(cout, generator=g)
        conv = lambda a, v: F.conv2d(a.double(), v.double(), stride=c["s"], padding=k // 2)
        return x, wt, b, conv(x, wt), conv(x.abs(), wt.abs())
    return cached(("fwd", c["desc"], exact), make)


def run_fwd(c, x, wt, **kw):
    from mcb200 import ops
    c0 = c["c0"]
    x2 = dev(x[:, c0:]) if c["c1"] else None
    wp = ops.pack_conv_weight(wt).to("cuda", torch.bfloat16)
    return ops.conv_fwd(dev(x[:, :c0]), wp, c["k"], c["s"], x2=x2, **kw)


@pytest.mark.parametrize("c,bn,halo", sweep(FWD, halo=True))
def test_conv_fwd(mcb, cuda, monkeypatch, c, bn, halo):
    set_knobs(monkeypatch, bn=bn, halo=halo)
    cout = c["cout"]
    assert_multi_tile(c["n"], c["h"] // c["s"], c["w"] // c["s"], cout, bn)
    x, wt, b, ref, absref = fwd_ref(c, exact=False)
    bd = b.double().view(1, -1, 1, 1)
    y = run_fwd(c, x, wt, bias=b.to(cuda))
    assert_bound(nchw(y), ref + bd, absref + bd.abs(), "conv_fwd + bias")
    # fused ReLU + statistics, twice: the second run must repeat the first bitwise
    runs = []
    for _ in range(2):
        stats = torch.zeros(2 * cout, device=cuda)
        runs.append((run_fwd(c, x, wt, relu=True, stats=stats), stats))
    (y1, st1), (y2, st2) = runs
    assert_bound(nchw(y1), ref.clamp_min(0), absref, "conv_fwd relu")
    assert_same(y1, y2, "conv_fwd relu output")
    assert_same(st1, st2, "conv_fwd stats")
    # the statistics are defined on the STORED bf16 output
    yq = nchw(y1).double()
    sq = yq * yq
    assert_bound(st1[:cout], yq.sum((0, 2, 3)), yq.abs().sum((0, 2, 3)), "stats sum", rel=0.0)
    assert_bound(st1[cout:], sq.sum((0, 2, 3)), sq.sum((0, 2, 3)), "stats sum of squares", rel=0.0)


@pytest.mark.parametrize("c,bn,halo", sweep(FWD, halo=True))
def test_conv_fwd_integer_exact(mcb, cuda, monkeypatch, c, bn, halo):
    set_knobs(monkeypatch, bn=bn, halo=halo)
    cout = c["cout"]
    assert_multi_tile(c["n"], c["h"] // c["s"], c["w"] // c["s"], cout, bn)
    x, wt, b, ref, _ = fwd_ref(c, exact=True)
    ref = ref + b.double().view(1, -1, 1, 1)
    assert ref.abs().max() <= 256
    s1, s2 = ref.sum((0, 2, 3)), (ref * ref).sum((0, 2, 3))
    assert ref.abs().sum((0, 2, 3)).max() < 2 ** 24 and s2.max() < 2 ** 24
    stats = torch.zeros(2 * cout, device=cuda)
    y = run_fwd(c, x, wt, bias=b.to(cuda), stats=stats)
    assert_exact(nchw(y), ref, "conv_fwd")
    assert_exact(stats[:cout], s1, "stats sum")
    assert_exact(stats[cout:], s2, "stats sum of squares")


# =====================================================================================================================
# inference epilogue: v = relu(acc * scale + bias + residual), BatchNorm folded into scale / bias
EVAL = [dict(FWD_BY_DESC["64->256 k1 s1 @80x80"], bn=(64, 256)),  # bottleneck conv3
        dict(FWD_BY_DESC["64->64 k3 s1 @80x80"], bn=(32, 64))]    # BasicBlock conv2


@pytest.mark.parametrize("c,bn,exact", sweep(EVAL, ("real", "exact")))
def test_conv_fwd_eval_epilogue(mcb, cuda, monkeypatch, c, bn, exact):
    set_knobs(monkeypatch, bn=bn)
    exact = exact == "exact"
    n, h, w, cout = c["n"], c["h"], c["w"], c["cout"]
    assert_multi_tile(n, h, w, cout, bn)
    x, wt, _, conv, absconv = fwd_ref(c, exact)
    g = gen("eval", c["desc"], exact)
    if exact:  # power-of-two scales, integer bias and residual: every step is exact
        scale = 2.0 ** torch.randint(-1, 2, (cout,), generator=g).float() * (2 * torch.randint(0, 2, (cout,), generator=g) - 1)
        bias = torch.randint(-3, 4, (cout,), generator=g).float()
        res = torch.randint(-3, 4, (n, cout, h, w), generator=g).float()
    else:
        scale = torch.randn(cout, generator=g) * 0.5 + 1.0
        bias = torch.randn(cout, generator=g)
        res = bf16r(torch.randn(n, cout, h, w, generator=g))
    sd, bd = scale.double().view(1, -1, 1, 1), bias.double().view(1, -1, 1, 1)
    ref = (conv * sd + bd + res.double()).clamp_min(0)
    y = run_fwd(c, x, wt, scale=scale.to(cuda), bias=bias.to(cuda), residual=dev(res), relu=True)
    if exact:
        assert ref.abs().max() <= 256
        assert_exact(nchw(y), ref, "conv_fwd eval epilogue")
    else:
        assert_bound(nchw(y), ref, absconv * sd.abs() + bd.abs() + res.double().abs(), "conv_fwd eval epilogue")


# =====================================================================================================================
# data gradient (conv_dgrad): plain; ReLU-masked with the fused channel sum
DGRAD = [
    dict(desc="128->128 k3 s1 @160x160", n=2, h=160, w=160, cin=128, cout=128, k=3, s=1, bn=(32, 64, 128),
         halo=(2, 0)),
    dict(desc="64->64 k3 s1 @80x80", n=6, h=80, w=80, cin=64, cout=64, k=3, s=1, bn=(32, 64), halo=(2, 1)),
    dict(desc="256->64 k1 s1 @80x80", n=6, h=80, w=80, cin=256, cout=64, k=1, s=1, bn=(32, 64, 128, 256)),
    dict(desc="256->512 k1 s2 @80x80", n=6, h=80, w=80, cin=256, cout=512, k=1, s=2, bn=(32, 64)),
    dict(desc="128->128 k3 s2 @80x80", n=6, h=80, w=80, cin=128, cout=128, k=3, s=2, bn=(32, 64, 128)),
    dict(desc="256+64->128 k3 s1 @80x80", n=6, h=80, w=80, cin=320, cout=128, k=3, s=1, bn=(32, 64, 256),
         halo=(2, 0)),
]
DGRAD_BY_DESC = {c["desc"]: c for c in DGRAD}


def dgrad_ref(c, exact):
    def make():
        g = gen("dgrad", c["desc"], exact)
        n, cin, cout, k, s = c["n"], c["cin"], c["cout"], c["k"], c["s"]
        ho, wo = c["h"] // s, c["w"] // s
        if exact:
            dy = ints(g, (n, cout, ho, wo))
            wt = ints(g, (cout, cin, k, k), int_density(cout * k * k))
        else:
            dy = bf16r(torch.randn(n, cout, ho, wo, generator=g))
            wt = bf16r(torch.randn(cout, cin, k, k, generator=g) / (cout * k * k) ** 0.5)
        act = bf16r(torch.randn(n, cin, c["h"], c["w"], generator=g))  # ReLU output of the producing layer
        dg = lambda v, d: torch.nn.grad.conv2d_input((n, cin, c["h"], c["w"]), v.double(), d.double(), stride=s,
                                                     padding=k // 2)
        return dy, wt, act, dg(wt, dy), dg(wt.abs(), dy.abs())
    return cached(("dgrad", c["desc"], exact), make)


def pack(wt):
    from mcb200 import ops
    return ops.pack_conv_weight(wt).to("cuda", torch.bfloat16)


DGRAD_MASKED = [DGRAD_BY_DESC[d] for d in ("128->128 k3 s1 @160x160", "64->64 k3 s1 @80x80", "256->64 k1 s1 @80x80")]


@pytest.mark.parametrize("c,bn,halo,exact", sweep(DGRAD_MASKED, ("real", "exact"), halo=True))
def test_conv_dgrad_masked_channel_sum(mcb, cuda, monkeypatch, c, bn, halo, exact):
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn, halo=halo)
    exact = exact == "exact"
    n, h, w, cin, k, s = c["n"], c["h"], c["w"], c["cin"], c["k"], c["s"]
    assert_multi_tile(n, h, w, cin, bn)
    dy, wt, act, ref, absref = dgrad_ref(c, exact)
    check = (lambda got, r, a, what: assert_exact(got, r, what)) if exact else assert_bound
    if exact:
        assert ref.abs().max() <= 256
    dyd, wp, actd = dev(dy), pack(wt), dev(act)
    check(nchw(ops.conv_dgrad(dyd, wp, k, s, (h, w))), ref, absref, "conv_dgrad")
    mask = (act > 0).double()
    runs = []
    for _ in range(2):
        csum = torch.zeros(cin, device=cuda)
        runs.append((ops.conv_dgrad(dyd, wp, k, s, (h, w), relu_mask=actd, channel_sum=csum), csum))
    (dx1, cs1), (dx2, cs2) = runs
    check(nchw(dx1), ref * mask, absref * mask, "conv_dgrad masked")
    assert_same(dx1, dx2, "conv_dgrad masked")
    assert_same(cs1, cs2, "conv_dgrad channel_sum")
    gq = nchw(dx1).double()  # the channel sum is defined on the STORED gradient
    if exact:
        assert gq.abs().sum((0, 2, 3)).max() < 2 ** 24
        assert_exact(cs1, gq.sum((0, 2, 3)), "channel_sum")
    else:
        assert_bound(cs1, gq.sum((0, 2, 3)), gq.abs().sum((0, 2, 3)), "channel_sum", rel=0.0)


BNRED = [DGRAD_BY_DESC["128->128 k3 s2 @80x80"]]


@pytest.mark.parametrize("c,bn,exact", sweep(BNRED, ("real", "exact")))
def test_conv_dgrad_bn_reduce_stride2(mcb, cuda, monkeypatch, c, bn, exact):
    """the backward of the producing conv-BN-ReLU unit fused into a stride-2 data gradient: four phases, each with its
    own output and aux tensor maps, so the aux prefetch of the next tile crosses phases"""
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn)
    exact = exact == "exact"
    n, h, w, cin, k, s = c["n"], c["h"], c["w"], c["cin"], c["k"], c["s"]
    assert_multi_tile(n, h // 2, w // 2, cin, bn, phases=4)
    dy, wt, _, ref, absref = dgrad_ref(c, exact)
    g = gen("bnred", c["desc"], exact)
    if exact:  # power-of-two scales and integer shifts: the mask, xhat and both sums are exact
        z = torch.randint(-3, 4, (n, cin, h, w), generator=g).float()
        mean = torch.randint(-1, 2, (cin,), generator=g).float()
        invstd = 2.0 ** torch.randint(-1, 2, (cin,), generator=g).float()
        gamma = 2.0 ** torch.randint(-1, 2, (cin,), generator=g).float() * (2 * torch.randint(0, 2, (cin,), generator=g) - 1)
        beta = torch.randint(-1, 2, (cin,), generator=g).float()
    else:
        z = bf16r(torch.randn(n, cin, h, w, generator=g) * 1.5 + 0.3)
        mean, invstd = torch.randn(cin, generator=g) * 0.2, torch.rand(cin, generator=g) + 0.5
        gamma, beta = torch.randn(cin, generator=g), torch.randn(cin, generator=g) * 0.5
    v = lambda t: t.double().view(1, -1, 1, 1)
    sc = gamma * invstd
    yb = z.double() * v(sc) + v(beta - mean * sc)  # the producing unit's BatchNorm output
    xhat = (z.double() - v(mean)) * v(invstd)
    mask = (yb > 0).double()
    decided = torch.ones_like(mask) if exact else (yb.abs() > 1e-3).double()  # sign not hinging on fma rounding
    runs = []
    for _ in range(2):
        dbeta, dgamma = torch.zeros(cin, device=cuda), torch.zeros(cin, device=cuda)
        bnr = (dev(z), mean.to(cuda), invstd.to(cuda), gamma.to(cuda), beta.to(cuda), dbeta, dgamma)
        runs.append((ops.conv_dgrad(dev(dy), pack(wt), k, s, (h, w), bn_reduce=bnr), dbeta, dgamma))
    (dx, db, dgm), (dx2, db2, dgm2) = runs
    assert_same(dx, dx2, "dgrad bn-mask")
    assert_same(db, db2, "dbeta")
    assert_same(dgm, dgm2, "dgamma")
    gq = nchw(dx).double().cpu()
    if exact:
        assert ref.abs().max() <= 256
        assert_exact(gq, ref * mask, "dgrad bn-mask")
        assert (gq * xhat).abs().sum((0, 2, 3)).max() < 2 ** 22
        assert_exact(db, gq.sum((0, 2, 3)), "dbeta")
        assert_exact(dgm, (gq * xhat).sum((0, 2, 3)), "dgamma")
    else:
        assert_bound(gq * decided, ref * mask * decided, absref * decided, "dgrad bn-mask")
        assert_bound(db, gq.sum((0, 2, 3)), gq.abs().sum((0, 2, 3)), "dbeta", rel=0.0)
        assert_bound(dgm, (gq * xhat).sum((0, 2, 3)), (gq * xhat).abs().sum((0, 2, 3)), "dgamma", rel=0.0)


def assert_accumulated(got, pre, ref, absref, what):
    """got = bf16(pre + bf16(acc)): two roundings, so the bound gains the first one's 2^-8 |ref| (and its A term).
    Where ref and A are zero (pixels the kernel must not touch) this demands got == pre exactly."""
    assert_bound(got, pre.double() + ref, absref, what, extra=2.0 ** -8 * ref.abs() + 2.0 ** -16 * absref)


@pytest.mark.parametrize("c,bn", sweep([DGRAD_BY_DESC["256->512 k1 s2 @80x80"]]))
def test_conv_dgrad_1x1_stride2_accumulate(mcb, cuda, monkeypatch, c, bn):
    """only the even pixels of a 1x1 stride-2 conv's input receive gradient: without accumulate the rest is zero,
    with accumulate it keeps the existing gradient bitwise"""
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn)
    n, h, w, cin, k, s = c["n"], c["h"], c["w"], c["cin"], c["k"], c["s"]
    assert_multi_tile(n, h // 2, w // 2, cin, bn)
    dy, wt, _, ref, absref = dgrad_ref(c, exact=False)
    dyd, wp = dev(dy), pack(wt)
    assert_bound(nchw(ops.conv_dgrad(dyd, wp, k, s, (h, w))), ref, absref, "conv_dgrad 1x1 s2")
    pre = bf16r(torch.randn(n, cin, h, w, generator=gen("acc", c["desc"])))
    out = dev(pre)
    ops.conv_dgrad(dyd, wp, k, s, (h, w), accumulate=True, out=out)
    assert_accumulated(nchw(out), pre, ref, absref, "conv_dgrad 1x1 s2 accumulate")


@pytest.mark.parametrize("c,bn,halo", sweep([DGRAD_BY_DESC["256+64->128 k3 s1 @80x80"]], halo=True))
def test_conv_dgrad_concat_slices_accumulate(mcb, cuda, monkeypatch, c, bn, halo):
    """the gradient of a concatenated input, one source at a time (cin / ci_off select the weight columns), added to
    the gradient that source already has"""
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn, halo=halo)
    n, h, w, k = c["n"], c["h"], c["w"], c["k"]
    dy, wt, _, ref, absref = dgrad_ref(c, exact=False)
    dyd, wp = dev(dy), pack(wt)
    g = gen("concat-acc", c["desc"])
    for off, cin in ((0, 256), (256, 64)):
        assert_multi_tile(n, h, w, cin, bn)
        pre = bf16r(torch.randn(n, cin, h, w, generator=g))
        out = dev(pre)
        ops.conv_dgrad(dyd, wp, k, 1, (h, w), cin=cin, ci_off=off, accumulate=True, out=out)
        sl = slice(off, off + cin)
        assert_accumulated(nchw(out), pre, ref[:, sl], absref[:, sl], "dgrad slice %d:%d" % (off, off + cin))


# =====================================================================================================================
# transposed conv (k4 s2 p1): forward (4 phases), data gradient (16 taps, masked + channel sum), weight gradient
CONVT = [
    dict(desc="256->64 convt @40x40", n=6, h=40, w=40, cin=256, cout=64, bn=(32, 64)),
    dict(desc="128->32 convt @160x160", n=2, h=160, w=160, cin=128, cout=32, bn=(32, 64, 128)),
]


def convt_ref(c, exact):
    def make():
        g = gen("convt", c["desc"], exact)
        n, h, w, cin, cout = c["n"], c["h"], c["w"], c["cin"], c["cout"]
        if exact:
            x = ints(g, (n, cin, h, w))
            wt = ints(g, (cin, cout, 4, 4), int_density(16 * cout))  # = 4 cin terms forward, 16 cout backward
            dy = ints(g, (n, cout, 2 * h, 2 * w))
            b = torch.randint(-3, 4, (cout,), generator=g).float()
        else:
            x = bf16r(torch.randn(n, cin, h, w, generator=g))
            wt = bf16r(torch.randn(cin, cout, 4, 4, generator=g) / (cin * 4) ** 0.5)
            dy = bf16r(torch.randn(n, cout, 2 * h, 2 * w, generator=g))
            b = torch.randn(cout, generator=g)
        act = bf16r(torch.randn(n, cin, h, w, generator=g))

        def grads(xv, wv, dv):
            xr, wr = xv.double().requires_grad_(True), wv.double().requires_grad_(True)
            y = F.conv_transpose2d(xr, wr, stride=2, padding=1)
            y.backward(dv.double())
            return y.detach(), xr.grad, wr.grad
        return (x, wt, dy, b, act) + grads(x, wt, dy) + grads(x.abs(), wt.abs(), dy.abs())
    return cached(("convt", c["desc"], exact), make)


@pytest.mark.parametrize("c,bn,exact", sweep(CONVT, ("real", "exact")))
def test_convt(mcb, cuda, monkeypatch, c, bn, exact):
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn)
    exact = exact == "exact"
    n, h, w, cin, cout = c["n"], c["h"], c["w"], c["cin"], c["cout"]
    assert_multi_tile(n, h, w, cout, bn, phases=4)
    assert_multi_tile(n, h, w, cin, bn)
    x, wt, dy, b, act, y_ref, dx_ref, dw_ref, y_abs, dx_abs, dw_abs = convt_ref(c, exact)
    check = (lambda got, r, a, what, **kw: assert_exact(got, r, what)) if exact else assert_bound
    if exact:
        assert max(y_ref.abs().max(), dx_ref.abs().max()) <= 256 - 3
    wp = ops.pack_convt_weight(wt).to(cuda, torch.bfloat16)
    xd, dyd = dev(x), dev(dy)
    bd = b.double().view(1, -1, 1, 1)
    y = ops.convt_fwd(xd, wp, bias=b.to(cuda), relu=True)
    check(nchw(y), (y_ref + bd).clamp_min(0), y_abs + bd.abs(), "convt_fwd")
    check(nchw(ops.convt_dgrad(dyd, wp)), dx_ref, dx_abs, "convt_dgrad")
    mask = (act > 0).double()
    runs = []
    for _ in range(2):
        csum = torch.zeros(cin, device=cuda)
        runs.append((ops.convt_dgrad(dyd, wp, relu_mask=dev(act), channel_sum=csum), csum))
    (dx1, cs1), (dx2, cs2) = runs
    check(nchw(dx1), dx_ref * mask, dx_abs * mask, "convt_dgrad masked")
    assert_same(dx1, dx2, "convt_dgrad masked")
    assert_same(cs1, cs2, "convt_dgrad channel_sum")
    gq = nchw(dx1).double()
    if exact:
        assert_exact(cs1, gq.sum((0, 2, 3)), "convt channel_sum")
    else:
        assert_bound(cs1, gq.sum((0, 2, 3)), gq.abs().sum((0, 2, 3)), "convt channel_sum", rel=0.0)


# =====================================================================================================================
# weight gradients (conv_wgrad, convt_wgrad): dW += gradient, split-K over pixel tiles
WGRAD = [
    dict(desc="64->64 k3 s1 @80x80", n=2, h=80, w=80, cin=64, cout=64, k=3, s=1),
    dict(desc="256->512 k1 s2 @80x80", n=2, h=80, w=80, cin=256, cout=512, k=1, s=2),
    dict(desc="1024->256 k1 s1 @20x20", n=4, h=20, w=20, cin=1024, cout=256, k=1, s=1),
    dict(desc="128->128 k3 s1 @160x160", n=1, h=160, w=160, cin=128, cout=128, k=3, s=1),
    dict(desc="32->32 k3 s1 @320x320", n=1, h=320, w=320, cin=32, cout=32, k=3, s=1),
    # transposed (k4 s2 p1, s=0 here): dy at twice the input size; operands shared with test_convt
    dict(desc="256->64 convt @40x40", n=6, h=40, w=40, cin=256, cout=64, k=4, s=0),
    dict(desc="128->32 convt @160x160", n=2, h=160, w=160, cin=128, cout=32, k=4, s=0),
]
WGRAD_REGION = 4 << 20  # fp32 elements of one stream's split-K workspace: splits x taps x cout x cin


def pick_tile(wv, hv, n, max_rows, row_mult):
    """the host's pixel-box choice (conv_gemm.cu pick_tile); returns the tile count"""
    best, choice = -1.0, (1, 1, 1)
    for bw in range(1, min(max_rows, wv, 256) + 1):
        bh = 1
        while bw * bh <= max_rows and bh <= min(hv, 256):
            for bn in range(1, min(256, max_rows // (bw * bh)) + 1):
                if bn > n and row_mult == 1:
                    break
                if (bw * bh * bn) % row_mult:
                    continue
                tiles = -(-wv // bw) * -(-hv // bh) * -(-n // bn)
                score = wv * hv * n / (tiles * max_rows) + 1e-6 * bw + 1e-9 * bh
                if score > best:
                    best, choice = score, (bw, bh, bn)
            bh += 1
    bw, bh, bn = choice
    return -(-wv // bw) * -(-hv // bh) * -(-n // bn)


def ragged_splits(tiles):
    """a split count that does not divide the pixel tiles and leaves the last split(s) without any"""
    for s in range(3, tiles):
        per = -(-tiles // s)
        if tiles % s and -(-tiles // per) < s:
            return s
    raise AssertionError("no ragged split for %d tiles" % tiles)


def wgrad_ref(c, exact):
    if c["s"] == 0:
        x, _, dy, _, _, _, _, dw_ref, _, _, dw_abs = convt_ref(c, exact)
        return x, dy, pack_t(dw_ref), pack_t(dw_abs)

    def make():
        g = gen("wgrad", c["desc"], exact)
        n, h, w, cin, cout, k, s = c["n"], c["h"], c["w"], c["cin"], c["cout"], c["k"], c["s"]
        if exact:
            x, dy = ints(g, (n, cin, h, w)), ints(g, (n, cout, h // s, w // s))
        else:
            x = bf16r(torch.randn(n, cin, h, w, generator=g))
            dy = bf16r(torch.randn(n, cout, h // s, w // s, generator=g))
        wg = lambda a, d: torch.nn.grad.conv2d_weight(a.double(), (cout, cin, k, k), d.double(), stride=s,
                                                      padding=k // 2)
        return x, dy, pack_t(wg(x, dy), k), pack_t(wg(x.abs(), dy.abs()), k)
    return cached(("wgrad", c["desc"], exact), make)


def pack_t(wt, k=None):
    """weight gradient -> the library's (taps, cout, cin) layout (k None: a transposed conv's (cin, cout, 4, 4))"""
    if k is None:
        return wt.permute(2, 3, 1, 0).reshape(16, wt.shape[1], wt.shape[0])
    return wt.permute(2, 3, 0, 1).reshape(k * k, wt.shape[0], wt.shape[1])


@pytest.mark.parametrize("c,splits,exact", sweep(WGRAD, ("default", "1", "ragged"), ("real", "exact")))
def test_wgrad(mcb, cuda, monkeypatch, c, splits, exact):
    """dW (prefilled with random values) += gradient.  Splits: the default heuristic; one split (every pixel tile in
    one CTA: its ring wraps many times, red.add into dW); a ragged forced split (uneven shares, the last splits own no
    tile; the finisher adds the rows).  Conv weight gradients write a column slice of a wider dW (ci_off / cin_total,
    as for a concatenated input): the columns around it must stay bitwise unchanged."""
    from mcb200 import ops
    n, h, w, cin, cout, k, s = c["n"], c["h"], c["w"], c["cin"], c["cout"], c["k"], c["s"]
    convt = s == 0
    hv, wv = (h, w) if convt else (h // s, w // s)
    tiles = pick_tile(wv, hv, n, 64, 16)
    assert tiles > 8, "the ring (<= 8 stages) would not wrap"
    forced = {"default": None, "1": 1, "ragged": ragged_splits(tiles)}[splits]
    if forced is not None and forced > 1:
        assert forced * k * k * cout * cin <= WGRAD_REGION
    set_knobs(monkeypatch, splits=forced)
    x, dy, ref, absref = wgrad_ref(c, exact == "exact")
    ci_off, cin_total = (0, cin) if convt else (64, cin + 128)
    g = gen("wgrad-pre", c["desc"], exact)
    pre = torch.randint(-50, 51, (k * k, cout, cin_total), generator=g).float() if exact == "exact" else \
        torch.randn(k * k, cout, cin_total, generator=g)
    expect = pre.double()
    expect[:, :, ci_off:ci_off + cin] += ref
    bound = torch.zeros_like(expect)
    bound[:, :, ci_off:ci_off + cin] = absref + pre[:, :, ci_off:ci_off + cin].double().abs()
    xd, dyd = dev(x), dev(dy)
    runs = []
    for _ in range(1 if exact == "exact" else 2):
        dw = pre.to(cuda)
        if convt:
            ops.convt_wgrad(dyd, xd, dw)
        else:
            ops.conv_wgrad(dyd, xd, dw, k, s, ci_off=ci_off)
        runs.append(dw)
    if exact == "exact":
        assert expect.abs().max() < 2 ** 24
        assert_exact(runs[0], expect, "wgrad")
    else:
        assert_bound(runs[0], expect, bound, "wgrad", rel=0.0)  # (bound 0 outside the slice: bitwise unchanged)
        assert_same(runs[0], runs[1], "wgrad")


def test_wgrad_two_streams(mcb, cuda, monkeypatch):
    """two split-K weight gradients in flight on two streams at once: each stream has its own workspace region, so each
    result equals the same launch run alone, bitwise"""
    from mcb200 import ops
    set_knobs(monkeypatch, splits=8)
    cases = [WGRAD[0], WGRAD[1]]
    jobs = []
    for c in cases:
        x, dy, ref, absref = wgrad_ref(c, False)
        pre = torch.randn(c["k"] ** 2, c["cout"], c["cin"], generator=gen("streams", c["desc"]))
        jobs.append((c, dev(x), dev(dy), pre, ref, absref))
    alone = []
    for c, xd, dyd, pre, _, _ in jobs:
        alone.append(ops.conv_wgrad(dyd, xd, pre.to(cuda), c["k"], c["s"]))
    outs = [pre.to(cuda) for _, _, _, pre, _, _ in jobs]
    cur = torch.cuda.current_stream()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for st, (c, xd, dyd, _, _, _), dw in zip(streams, jobs, outs):
        st.wait_stream(cur)
        with torch.cuda.stream(st):
            ops.conv_wgrad(dyd, xd, dw, c["k"], c["s"])
    torch.cuda.synchronize()
    for (c, _, _, pre, ref, absref), a, dw in zip(jobs, alone, outs):
        assert_bound(dw, pre.double() + ref, absref + pre.double().abs(), "wgrad %s on a side stream" % c["desc"],
                     rel=0.0)
        assert_same(dw, a, "wgrad %s: two streams vs alone" % c["desc"])
