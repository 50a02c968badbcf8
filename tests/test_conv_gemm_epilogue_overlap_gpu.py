"""The hand-off between conv_gemm_kernel's MMA warpgroups and its epilogue warpgroup.

The MMA warpgroups write each tile to a bf16 staging buffer and go on to the next tile's main loop while the epilogue
warpgroup runs the second pass (statistics, masks, channel sums) and the TMA stores of the staged tile.  Two staging
buffers rotate when the operand ring still keeps three stages (BN <= 128 here), one otherwise (BN = 256 with 64-channel
K blocks); the aux tiles of the data gradients travel through a ring of two chunk buffers across tiles.  Every case
below puts at least three tiles on every CTA, so each buffer and each barrier phase is reused, and the channel sums are
carried across tiles and N tiles.  The tail cases run one tile per CTA (fewer tiles than SMs) and CTAs with unequal
tile counts; the last test runs the kernels next to a weight gradient on a second stream.

References are float64 on the CPU from the bf16-rounded operands, with the bars of test_conv_gemm_persistent_gpu.py:
|got - ref| <= 2^-8 |ref| + 2^-16 A for bf16 outputs (A: the same op on |operands|), channel sums against the float64
sum of the STORED output within 2^-16 of the sum of magnitudes.  Integer-exact variants (operands in {-1, 0, 1})
match bitwise, fused sums included."""
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

_REF = {}


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def bf16r(x):
    return x.to(torch.bfloat16).to(torch.float32)


def dev(x):
    return nhwc(x).to("cuda", torch.bfloat16)


def gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def ints(g, shape, density=1.0):
    v = torch.randint(-1, 2, shape, generator=g).float()
    return v * (torch.rand(shape, generator=g) < density).float() if density < 1 else v


def cached(key, make):
    if key not in _REF:
        _REF[key] = make()
    return _REF[key]


def assert_bound(got, ref, absref, what, rel=2.0 ** -8, extra=0.0):
    got = got.double()
    ref = ref.to(got.device, torch.float64)
    absref = absref.to(got.device, torch.float64) if torch.is_tensor(absref) else absref
    extra = extra.to(got.device, torch.float64) if torch.is_tensor(extra) else extra
    err = (got - ref).abs()
    bad = ~(err <= rel * ref.abs() + 2.0 ** -16 * absref + extra)
    assert not bad.any(), "%s: %d/%d elements off, max err %g" % (
        what, int(bad.sum()), bad.numel(), float(err.nan_to_num(float("inf")).max()))


def assert_exact(got, ref, what):
    assert_bound(got, ref, 0.0, what, rel=0.0)


def check_sums(got, stored, what, exact):
    """a fused per-channel sum against the float64 sum of what the kernel stored (stored: N, C, H, W float64)"""
    s, a = stored.sum((0, 2, 3)), stored.abs().sum((0, 2, 3))
    if exact:
        assert a.max() < 2 ** 24
        assert_exact(got, s, what)
    else:
        assert_bound(got, s, a, what, rel=0.0)


def pick_tiles(wv, hv, n, max_rows=128):
    """pixel tiles of the host's box choice (conv_gemm.cu pick_tile, row multiple 1)"""
    best, tiles = -1.0, 0
    for bw in range(1, min(max_rows, wv, 256) + 1):
        bh = 1
        while bw * bh <= max_rows and bh <= min(hv, 256):
            for bn in range(1, min(256, max_rows // (bw * bh)) + 1):
                if bn > n:
                    break
                t = -(-wv // bw) * -(-hv // bh) * -(-n // bn)
                score = wv * hv * n / (t * max_rows) + 1e-6 * bw + 1e-9 * bh
                if score > best:
                    best, tiles = score, t
            bh += 1
    return tiles


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def tile_count(hv, wv, n, n_extent, bn, phases=1):
    return pick_tiles(wv, hv, n) * (n_extent // bn) * phases


def set_bn(monkeypatch, bn):
    monkeypatch.setenv("MCB_FORCE_BN", str(bn))
    monkeypatch.delenv("MCB_HALO", raising=False)


def pack(wt):
    from mcb200 import ops
    return ops.pack_conv_weight(wt).to("cuda", torch.bfloat16)


# =====================================================================================================================
# forward with ReLU and BatchNorm statistics
FWD = [
    dict(desc="64->256 k1 @80x80", n=8, h=80, w=80, c0=64, c1=0, cout=256, k=1, bn=(32, 64, 128, 256)),
    dict(desc="64+64->256 k1 @80x80 concat", n=8, h=80, w=80, c0=64, c1=64, cout=256, k=1, bn=(64, 256)),
    # 37 images of 10x10: every tile is ragged (rows < 128), the last pixel tile of the batch partly empty
    dict(desc="128->1024 k1 @10x10 ragged", n=37, h=10, w=10, c0=128, c1=0, cout=1024, k=1, bn=(32, 64)),
    dict(desc="64->64 k3 @80x80", n=8, h=80, w=80, c0=64, c1=0, cout=64, k=3, bn=(32, 64)),
]


def fwd_ref(c, exact):
    def make():
        g = gen("fwd", c["desc"], exact)
        cin, k, cout = c["c0"] + c["c1"], c["k"], c["cout"]
        if exact:
            x = ints(g, (c["n"], cin, c["h"], c["w"]))
            wt = ints(g, (cout, cin, k, k), min(1.0, 24.0 / (cin * k * k)))
            b = torch.randint(-3, 4, (cout,), generator=g).float()
        else:
            x = bf16r(torch.randn(c["n"], cin, c["h"], c["w"], generator=g))
            wt = bf16r(torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5)
            b = torch.randn(cout, generator=g)
        conv = lambda a, v: F.conv2d(a.double(), v.double(), padding=k // 2)
        return x, wt, b, conv(x, wt), conv(x.abs(), wt.abs())
    return cached(("fwd", c["desc"], exact), make)


def run_fwd(c, x, wt, **kw):
    from mcb200 import ops
    c0 = c["c0"]
    x2 = dev(x[:, c0:]) if c["c1"] else None
    return ops.conv_fwd(dev(x[:, :c0]), pack(wt), c["k"], 1, x2=x2, **kw)


def fwd_params():
    return [pytest.param(c, bn, ex, id="%s-BN%d-%s" % (c["desc"].replace(" ", "_"), bn, ex))
            for c in FWD for bn in c["bn"] for ex in ("real", "exact")]


@pytest.mark.parametrize("c,bn,exact", fwd_params())
def test_fwd_stats(mcb, cuda, monkeypatch, c, bn, exact):
    set_bn(monkeypatch, bn)
    exact = exact == "exact"
    cout = c["cout"]
    assert tile_count(c["h"], c["w"], c["n"], cout, bn) >= 3 * sms()
    x, wt, b, ref, absref = fwd_ref(c, exact)
    bd = b.double().view(1, -1, 1, 1)
    stats = torch.zeros(2 * cout, device=cuda)
    y = nchw(run_fwd(c, x, wt, bias=b.to(cuda), relu=True, stats=stats)).double()
    want = (ref + bd).clamp_min(0)
    if exact:
        assert want.abs().max() <= 256
        assert_exact(y, want, "conv_fwd")
    else:
        assert_bound(y, want, absref + bd.abs(), "conv_fwd")
    check_sums(stats[:cout], y, "stats sum", exact)
    check_sums(stats[cout:], y * y, "stats sum of squares", exact)


# =====================================================================================================================
# data gradients: ReLU mask + channel sum (aux 1), BatchNorm-backward mask + dbeta / dgamma (aux 2), accumulate
DGRAD = [
    dict(desc="256<-64 k1 s1 @80x80", n=8, h=80, w=80, cin=256, cout=64, k=1, s=1, bn=(32, 64, 128, 256)),
    # four phases with their own output and aux tensor maps: the aux ring crosses phases
    dict(desc="128<-128 k3 s2 @80x80 phased", n=8, h=80, w=80, cin=128, cout=128, k=3, s=2, bn=(32, 64, 128)),
]


def dgrad_ref(c, exact):
    def make():
        g = gen("dgrad", c["desc"], exact)
        n, cin, cout, k, s = c["n"], c["cin"], c["cout"], c["k"], c["s"]
        ho, wo = c["h"] // s, c["w"] // s
        if exact:
            dy = ints(g, (n, cout, ho, wo))
            wt = ints(g, (cout, cin, k, k), min(1.0, 24.0 / (cout * k * k)))
            z = torch.randint(-3, 4, (n, cin, c["h"], c["w"]), generator=g).float()
            mean = torch.randint(-1, 2, (cin,), generator=g).float()
            invstd = 2.0 ** torch.randint(-1, 2, (cin,), generator=g).float()
            gamma = 2.0 ** torch.randint(-1, 2, (cin,), generator=g).float() * \
                (2 * torch.randint(0, 2, (cin,), generator=g) - 1)
            beta = torch.randint(-1, 2, (cin,), generator=g).float()
        else:
            dy = bf16r(torch.randn(n, cout, ho, wo, generator=g))
            wt = bf16r(torch.randn(cout, cin, k, k, generator=g) / (cout * k * k) ** 0.5)
            z = bf16r(torch.randn(n, cin, c["h"], c["w"], generator=g) * 1.5 + 0.3)
            mean, invstd = torch.randn(cin, generator=g) * 0.2, torch.rand(cin, generator=g) + 0.5
            gamma, beta = torch.randn(cin, generator=g), torch.randn(cin, generator=g) * 0.5
        dg = lambda v, d: torch.nn.grad.conv2d_input((n, cin, c["h"], c["w"]), v.double(), d.double(), stride=s,
                                                     padding=k // 2)
        return dy, wt, (z, mean, invstd, gamma, beta), dg(wt, dy), dg(wt.abs(), dy.abs())
    return cached(("dgrad", c["desc"], exact), make)


def bn_terms(bnp):
    z, mean, invstd, gamma, beta = bnp
    v = lambda t: t.double().view(1, -1, 1, 1)
    sc = gamma * invstd
    yb = z.double() * v(sc) + v(beta - mean * sc)
    return yb, (z.double() - v(mean)) * v(invstd)


def dgrad_params(modes):
    return [pytest.param(c, bn, m, ex, id="%s-BN%d-%s-%s" % (c["desc"].replace(" ", "_"), bn, m, ex))
            for c in DGRAD for bn in c["bn"] for m in modes for ex in ("real", "exact")]


@pytest.mark.parametrize("c,bn,mode,exact", dgrad_params(("relu", "bn")))
def test_dgrad_aux(mcb, cuda, monkeypatch, c, bn, mode, exact):
    from mcb200 import ops
    set_bn(monkeypatch, bn)
    exact = exact == "exact"
    n, h, w, cin, k, s = c["n"], c["h"], c["w"], c["cin"], c["k"], c["s"]
    phases = 4 if s == 2 else 1
    assert tile_count(h // s, w // s, n, cin, bn, phases) >= 3 * sms()
    dy, wt, bnp, ref, absref = dgrad_ref(c, exact)
    yb, xhat = bn_terms(bnp)
    if mode == "relu":
        # the ReLU output of the producing layer; its sign is yb's
        mask = (yb > 0).double()
        csum = torch.zeros(cin, device=cuda)
        dx = ops.conv_dgrad(dev(dy), pack(wt), k, s, (h, w), relu_mask=dev(yb.float()), channel_sum=csum)
        decided = torch.ones_like(mask)
    else:
        mask = (yb > 0).double()
        decided = torch.ones_like(mask) if exact else (yb.abs() > 1e-3).double()  # sign not hinging on fma rounding
        dbeta, dgamma = torch.zeros(cin, device=cuda), torch.zeros(cin, device=cuda)
        args = (dev(bnp[0]),) + tuple(t.to(cuda) for t in bnp[1:]) + (dbeta, dgamma)
        dx = ops.conv_dgrad(dev(dy), pack(wt), k, s, (h, w), bn_reduce=args)
    gq = nchw(dx).double().cpu()
    if exact:
        assert ref.abs().max() <= 256
        assert_exact(gq, ref * mask, "dgrad masked")
    else:
        assert_bound(gq * decided, ref * mask * decided, absref * decided, "dgrad masked")
    if mode == "relu":
        check_sums(csum, gq, "channel sum", exact)
    else:
        check_sums(dbeta, gq, "dbeta", exact)
        check_sums(dgamma, gq * xhat, "dgamma", exact)


@pytest.mark.parametrize("c,bn", [pytest.param(c, bn, id="%s-BN%d" % (c["desc"].replace(" ", "_"), bn))
                                  for c in DGRAD for bn in c["bn"]])
def test_dgrad_accumulate(mcb, cuda, monkeypatch, c, bn):
    """TMA reduce-add from the staging buffers: got = bf16(pre + bf16(acc))"""
    from mcb200 import ops
    set_bn(monkeypatch, bn)
    n, h, w, cin, k, s = c["n"], c["h"], c["w"], c["cin"], c["k"], c["s"]
    dy, wt, _, ref, absref = dgrad_ref(c, False)
    pre = bf16r(torch.randn(n, cin, h, w, generator=gen("acc", c["desc"])))
    out = dev(pre)
    ops.conv_dgrad(dev(dy), pack(wt), k, s, (h, w), accumulate=True, out=out)
    assert_bound(nchw(out), pre.double() + ref, absref, "dgrad accumulate",
                 extra=2.0 ** -8 * ref.abs() + 2.0 ** -16 * absref)


# =====================================================================================================================
# transposed conv: forward over four phases, data gradient masked with its channel sum
CONVT = dict(desc="128->32 convt @160x160", n=2, h=160, w=160, cin=128, cout=32)


def convt_ref(exact):
    def make():
        c = CONVT
        g = gen("convt", exact)
        n, h, w, cin, cout = c["n"], c["h"], c["w"], c["cin"], c["cout"]
        if exact:
            x, dy = ints(g, (n, cin, h, w)), ints(g, (n, cout, 2 * h, 2 * w))
            wt = ints(g, (cin, cout, 4, 4), min(1.0, 24.0 / (16 * cout)))
        else:
            x, dy = bf16r(torch.randn(n, cin, h, w, generator=g)), bf16r(torch.randn(n, cout, 2 * h, 2 * w, generator=g))
            wt = bf16r(torch.randn(cin, cout, 4, 4, generator=g) / (cin * 4) ** 0.5)
        act = bf16r(torch.randn(n, cin, h, w, generator=g))

        def grads(xv, wv, dv):
            xr = xv.double().requires_grad_(True)
            y = F.conv_transpose2d(xr, wv.double(), stride=2, padding=1)
            y.backward(dv.double())
            return y.detach(), xr.grad
        return (x, wt, dy, act) + grads(x, wt, dy) + grads(x.abs(), wt.abs(), dy.abs())
    return cached(("convt", exact), make)


@pytest.mark.parametrize("bn", (32, 64, 128))
@pytest.mark.parametrize("exact", ("real", "exact"))
def test_convt(mcb, cuda, monkeypatch, bn, exact):
    from mcb200 import ops
    set_bn(monkeypatch, bn)
    exact = exact == "exact"
    c = CONVT
    assert tile_count(c["h"], c["w"], c["n"], c["cin"], bn) >= 3 * sms()
    x, wt, dy, act, y_ref, dx_ref, y_abs, dx_abs = convt_ref(exact)
    check = (lambda got, r, a, what: assert_exact(got, r, what)) if exact else assert_bound
    wp = ops.pack_convt_weight(wt).to(cuda, torch.bfloat16)
    check(nchw(ops.convt_fwd(dev(x), wp, relu=True)), y_ref.clamp_min(0), y_abs, "convt_fwd")
    mask = (act > 0).double()
    csum = torch.zeros(c["cin"], device=cuda)
    dx = nchw(ops.convt_dgrad(dev(dy), wp, relu_mask=dev(act), channel_sum=csum)).double()
    check(dx, dx_ref * mask, dx_abs * mask, "convt_dgrad masked")
    check_sums(csum, dx, "convt channel sum", exact)


# =====================================================================================================================
# tails: one tile per CTA (fewer tiles than SMs), and CTAs with unequal tile counts, whose last drain overlaps no
# further main loop while the other CTAs still run one
TAIL = [
    dict(desc="fewer tiles than SMs", n=1, h=32, w=32, c=256, bn=64),
    dict(desc="uneven tiles per CTA", n=8, h=80, w=80, c=256, bn=256),
]


@pytest.mark.parametrize("c", TAIL, ids=lambda c: c["desc"].replace(" ", "_"))
def test_tails(mcb, cuda, monkeypatch, c):
    from mcb200 import ops
    set_bn(monkeypatch, c["bn"])
    n, h, w, ch, bn = c["n"], c["h"], c["w"], c["c"], c["bn"]
    tiles = tile_count(h, w, n, ch, bn)
    if c["desc"].startswith("fewer"):
        assert tiles < sms()
    else:
        assert tiles > 2 * sms() and tiles % sms() != 0
    g = gen("tail", c["desc"])
    x = bf16r(torch.randn(n, ch, h, w, generator=g))
    wt = bf16r(torch.randn(ch, ch, 1, 1, generator=g) / ch ** 0.5)
    ref, absref = (F.conv2d(a.double(), v.double()) for a, v in ((x, wt), (x.abs(), wt.abs())))
    stats = torch.zeros(2 * ch, device=cuda)
    y = nchw(ops.conv_fwd(dev(x), pack(wt), 1, 1, relu=True, stats=stats)).double()
    assert_bound(y, ref.clamp_min(0), absref, "conv_fwd")
    check_sums(stats[:ch], y, "stats sum", False)
    check_sums(stats[ch:], y * y, "stats sum of squares", False)
    # the data gradient of the same 1x1 conv with the BatchNorm-backward reductions
    z = bf16r(torch.randn(n, ch, h, w, generator=g))
    mean, invstd = torch.randn(ch, generator=g) * 0.2, torch.rand(ch, generator=g) + 0.5
    gamma, beta = torch.randn(ch, generator=g), torch.randn(ch, generator=g) * 0.5
    yb, xhat = bn_terms((z, mean, invstd, gamma, beta))
    decided = (yb.abs() > 1e-3).double()
    dref = torch.nn.grad.conv2d_input(x.shape, wt.double(), x.double())
    dabs = torch.nn.grad.conv2d_input(x.shape, wt.double().abs(), x.double().abs())
    dbeta, dgamma = torch.zeros(ch, device=cuda), torch.zeros(ch, device=cuda)
    args = (dev(z), mean.to(cuda), invstd.to(cuda), gamma.to(cuda), beta.to(cuda), dbeta, dgamma)
    gq = nchw(ops.conv_dgrad(dev(x), pack(wt), 1, 1, (h, w), bn_reduce=args)).double().cpu()
    mask = (yb > 0).double()
    assert_bound(gq * decided, dref * mask * decided, dabs * decided, "dgrad bn-mask")
    check_sums(dbeta, gq, "dbeta", False)
    check_sums(dgamma, gq * xhat, "dgamma", False)


# =====================================================================================================================
def test_bitwise_with_side_stream_wgrad(mcb, cuda, monkeypatch):
    """outputs and channel sums repeat bitwise when a weight gradient shares the SMs from a second stream"""
    from mcb200 import ops
    monkeypatch.delenv("MCB_FORCE_BN", raising=False)
    monkeypatch.delenv("MCB_HALO", raising=False)
    c, d = FWD[0], DGRAD[1]
    x, wt, b, _, _ = fwd_ref(c, False)
    dy, dwt, bnp, _, _ = dgrad_ref(d, False)
    xd, wp, bd = dev(x), pack(wt), b.to(cuda)
    dyd, dwp = dev(dy), pack(dwt)
    bn_dev = (dev(bnp[0]),) + tuple(t.to(cuda) for t in bnp[1:])
    # the side stream's work: the weight gradient of the forward conv
    wx = dev(bf16r(torch.randn(16, 256, 80, 80, generator=gen("side"))))
    wdy = dev(bf16r(torch.randn(16, 256, 80, 80, generator=gen("side-dy"))))

    def run():
        stats = torch.zeros(2 * c["cout"], device=cuda)
        dbeta, dgamma = torch.zeros(d["cin"], device=cuda), torch.zeros(d["cin"], device=cuda)
        y = ops.conv_fwd(xd, wp, 1, 1, bias=bd, relu=True, stats=stats)
        dx = ops.conv_dgrad(dyd, dwp, d["k"], d["s"], (d["h"], d["w"]), bn_reduce=bn_dev + (dbeta, dgamma))
        return y, stats, dx, dbeta, dgamma

    alone = run()
    torch.cuda.synchronize()
    cur, side = torch.cuda.current_stream(), torch.cuda.Stream()
    for _ in range(3):
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(4):
                ops.conv_wgrad(wdy, wx, torch.zeros(1, 256, 256, device=cuda), 1, 1)
        shared = run()
        torch.cuda.synchronize()
        for a, s_, what in zip(alone, shared, ("y", "stats", "dx", "dbeta", "dgamma")):
            assert torch.equal(a, s_), "%s differs next to a side-stream weight gradient" % what
