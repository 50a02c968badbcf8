"""The hand-off between conv_gemm_kernel's MMA warpgroups and its epilogue warpgroup.

The MMA warpgroups write each tile to a bf16 staging buffer and go on to the next tile's main loop while the epilogue
warpgroup runs the second pass (statistics, masks, channel sums) and the TMA stores of the staged tile.  Two staging
buffers rotate when the operand ring still keeps three stages (BN <= 128 here), one otherwise (BN = 256 with 64-channel
K blocks); the aux tiles of the data gradients travel through a ring of two chunk buffers across tiles.  Every case
below puts at least three tiles on every CTA, so each buffer and each barrier phase is reused, and the channel sums are
carried across tiles and N tiles.  The tail cases run one tile per CTA (fewer tiles than SMs) and CTAs with unequal
tile counts; the last test runs the kernels next to a weight gradient on a second stream.

References and bars: oracle/conv_checks.py, the same as test_conv_gemm_persistent_gpu.py's (float64 from the
bf16-rounded operands; bf16 outputs within 2^-8 |ref| + 2^-16 A, channel sums against the float64 sum of the STORED
output within 2^-16 A).  Integer-exact variants (operands in {-1, 0, 1}) match bitwise, fused sums included."""
import pytest
import torch
import torch.nn.functional as F

from oracle.conv_checks import (assert_accumulated, assert_bound, assert_exact, assert_tiles_per_cta, bf16r,
                                bn_operands, bn_reduce, bn_terms, check_sums, convt_ref, dev, dgrad_ref, fwd_ref, gen,
                                nchw, pack, pack_t, run_fwd, set_knobs, sms, sweep, tile_count)

pytestmark = pytest.mark.gpu

_REF = {}


# =====================================================================================================================
# forward with ReLU and BatchNorm statistics
FWD = [
    dict(desc="64->256 k1 @80x80", n=8, h=80, w=80, c0=64, c1=0, cout=256, k=1, bn=(32, 64, 128, 256)),
    dict(desc="64+64->256 k1 @80x80 concat", n=8, h=80, w=80, c0=64, c1=64, cout=256, k=1, bn=(64, 256)),
    # 37 images of 10x10: every tile is ragged (rows < 128), the last pixel tile of the batch partly empty
    dict(desc="128->1024 k1 @10x10 ragged", n=37, h=10, w=10, c0=128, c1=0, cout=1024, k=1, bn=(32, 64)),
    dict(desc="64->64 k3 @80x80", n=8, h=80, w=80, c0=64, c1=0, cout=64, k=3, bn=(32, 64)),
]


@pytest.mark.parametrize("c,bn,exact", sweep(FWD, ("real", "exact")))
def test_fwd_stats(mcb, cuda, monkeypatch, c, bn, exact):
    set_knobs(monkeypatch, bn=bn)
    exact = exact == "exact"
    cout = c["cout"]
    assert_tiles_per_cta(tile_count(c["n"], c["h"], c["w"], cout, bn), 3)
    x, wt, b, ref, absref = fwd_ref(c, exact, _REF)
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


@pytest.mark.parametrize("c,bn,mode,exact", sweep(DGRAD, ("relu", "bn"), ("real", "exact")))
def test_dgrad_aux(mcb, cuda, monkeypatch, c, bn, mode, exact):
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn)
    exact = exact == "exact"
    n, h, w, cin, k, s = c["n"], c["h"], c["w"], c["cin"], c["k"], c["s"]
    phases = 4 if s == 2 else 1
    assert_tiles_per_cta(tile_count(n, h // s, w // s, cin, bn, phases), 3)
    dy, wt, _, bnp, ref, absref = dgrad_ref(c, exact, _REF)
    yb, xhat = bn_terms(bnp)
    mask = (yb > 0).double()
    if mode == "relu":
        # the ReLU output of the producing layer; its sign is yb's
        csum = torch.zeros(cin, device=cuda)
        dx = ops.conv_dgrad(dev(dy), pack(wt), k, s, (h, w), relu_mask=dev(yb.float()), channel_sum=csum)
        decided = torch.ones_like(mask)
    else:
        decided = torch.ones_like(mask) if exact else (yb.abs() > 1e-3).double()  # sign not hinging on fma rounding
        args = bn_reduce(bnp)
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
        check_sums(args[-2], gq, "dbeta", exact)
        check_sums(args[-1], gq * xhat, "dgamma", exact)


@pytest.mark.parametrize("c,bn", sweep(DGRAD))
def test_dgrad_accumulate(mcb, cuda, monkeypatch, c, bn):
    """TMA reduce-add from the staging buffers: got = bf16(pre + bf16(acc))"""
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn)
    n, h, w, cin, k, s = c["n"], c["h"], c["w"], c["cin"], c["k"], c["s"]
    dy, wt, _, _, ref, absref = dgrad_ref(c, False, _REF)
    pre = bf16r(torch.randn(n, cin, h, w, generator=gen("acc", c["desc"])))
    out = dev(pre)
    ops.conv_dgrad(dev(dy), pack(wt), k, s, (h, w), accumulate=True, out=out)
    assert_accumulated(nchw(out), pre, ref, absref, "dgrad accumulate")


# =====================================================================================================================
# transposed conv: forward over four phases, data gradient masked with its channel sum
CONVT = dict(desc="128->32 convt @160x160", n=2, h=160, w=160, cin=128, cout=32)


@pytest.mark.parametrize("bn", (32, 64, 128))
@pytest.mark.parametrize("exact", ("real", "exact"))
def test_convt(mcb, cuda, monkeypatch, bn, exact):
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn)
    exact = exact == "exact"
    c = CONVT
    assert_tiles_per_cta(tile_count(c["n"], c["h"], c["w"], c["cin"], bn), 3)
    x, wt, dy, _, act, y_ref, dx_ref, _, y_abs, dx_abs, _ = convt_ref(c, exact, _REF)
    check = (lambda got, r, a, what: assert_exact(got, r, what)) if exact else assert_bound
    wp = pack_t(wt)
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
    set_knobs(monkeypatch, bn=c["bn"])
    n, h, w, ch, bn = c["n"], c["h"], c["w"], c["c"], c["bn"]
    tiles = tile_count(n, h, w, ch, bn)
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
    bnp = bn_operands(g, (n, ch, h, w), False)
    yb, xhat = bn_terms(bnp)
    decided = (yb.abs() > 1e-3).double()
    dref = torch.nn.grad.conv2d_input(x.shape, wt.double(), x.double())
    dabs = torch.nn.grad.conv2d_input(x.shape, wt.double().abs(), x.double().abs())
    args = bn_reduce(bnp)
    gq = nchw(ops.conv_dgrad(dev(x), pack(wt), 1, 1, (h, w), bn_reduce=args)).double().cpu()
    mask = (yb > 0).double()
    assert_bound(gq * decided, dref * mask * decided, dabs * decided, "dgrad bn-mask")
    check_sums(args[-2], gq, "dbeta", False)
    check_sums(args[-1], gq * xhat, "dgamma", False)


# =====================================================================================================================
def test_bitwise_with_side_stream_wgrad(mcb, cuda, monkeypatch):
    """outputs and channel sums repeat bitwise when a weight gradient shares the SMs from a second stream"""
    from mcb200 import ops
    set_knobs(monkeypatch)
    c, d = FWD[0], DGRAD[1]
    x, wt, b, _, _ = fwd_ref(c, False, _REF)
    dy, dwt, _, bnp, _, _ = dgrad_ref(d, False, _REF)
    xd, wp, bd = dev(x), pack(wt), b.to(cuda)
    dyd, dwp, bnr = dev(dy), pack(dwt), bn_reduce(bnp)[:-2]
    # the side stream's work: the weight gradient of the forward conv
    wx = dev(bf16r(torch.randn(16, 256, 80, 80, generator=gen("side"))))
    wdy = dev(bf16r(torch.randn(16, 256, 80, 80, generator=gen("side-dy"))))

    def run():
        stats = torch.zeros(2 * c["cout"], device=cuda)
        dbeta, dgamma = torch.zeros(d["cin"], device=cuda), torch.zeros(d["cin"], device=cuda)
        y = ops.conv_fwd(xd, wp, 1, 1, bias=bd, relu=True, stats=stats)
        dx = ops.conv_dgrad(dyd, dwp, d["k"], d["s"], (d["h"], d["w"]), bn_reduce=bnr + (dbeta, dgamma))
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
