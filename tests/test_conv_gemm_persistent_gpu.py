"""The convolution kernels in the persistent, multi-tile regime the full-size network runs.

conv_gemm_kernel is persistent: the grid is min(tiles, SMs) and each CTA walks tiles t = blockIdx.x, += gridDim.x,
carrying from one tile to the next the TMA ring position and mbarrier parity, the haloed A ring, the rotation of the
output staging buffers, the aux-tile prefetch of the next tile and the per-channel reduction registers (flushed when
the N tile changes).  wgrad_kernel runs its ring over many K blocks per CTA and adds into an existing dW.  Every
convolution case here puts at least two tiles on every CTA (asserted against the device's SM count) and sweeps the
existing knobs: MCB_FORCE_BN (N tile width), MCB_HALO (0 never, 1 wherever the haloed tile fits, 2 the default rule)
and MCB_WGRAD_SPLITS.  Shapes are layers of the ResNet101-UNet at 320x320 ("cin->cout kK sS @HxW"), at small batches;
the deep layers (20x20, 10x10) take more images so that the persistent grid still wraps.

References and bars: oracle/conv_checks.py (float64 from the bf16-rounded operands; bf16 outputs within 2^-8 |ref| +
2^-16 A, fp32 weight gradients and fused sums within 2^-16 A).  Integer-exact variants (operands in {-1, 0, 1}) must
match bitwise, fused reductions included; real-valued fused reductions must repeat bitwise from run to run."""
import pytest
import torch

from oracle.conv_checks import (assert_accumulated, assert_bound, assert_exact, assert_same, assert_tiles_per_cta,
                                bf16r, bn_reduce, bn_terms, check_sums, convt_ref, dev, dgrad_ref, fwd_ref, gen, nchw,
                                pack, pack_t, pick_tile, run_fwd, set_knobs, sweep, tile_count, wgrad_ref)

pytestmark = pytest.mark.gpu

_REF = {}  # references per case, shared by the knob sweeps


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


@pytest.mark.parametrize("c,bn,halo", sweep(FWD, halo=True))
def test_conv_fwd(mcb, cuda, monkeypatch, c, bn, halo):
    set_knobs(monkeypatch, bn=bn, halo=halo)
    cout = c["cout"]
    assert_tiles_per_cta(tile_count(c["n"], c["h"] // c["s"], c["w"] // c["s"], cout, bn, any_box=True), 2)
    x, wt, b, ref, absref = fwd_ref(c, False, _REF)
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
    check_sums(st1[:cout], yq, "stats sum", False)
    check_sums(st1[cout:], yq * yq, "stats sum of squares", False)


@pytest.mark.parametrize("c,bn,halo", sweep(FWD, halo=True))
def test_conv_fwd_integer_exact(mcb, cuda, monkeypatch, c, bn, halo):
    set_knobs(monkeypatch, bn=bn, halo=halo)
    cout = c["cout"]
    assert_tiles_per_cta(tile_count(c["n"], c["h"] // c["s"], c["w"] // c["s"], cout, bn, any_box=True), 2)
    x, wt, b, ref, _ = fwd_ref(c, True, _REF)
    ref = ref + b.double().view(1, -1, 1, 1)
    assert ref.abs().max() <= 256
    stats = torch.zeros(2 * cout, device=cuda)
    y = nchw(run_fwd(c, x, wt, bias=b.to(cuda), stats=stats)).double()
    assert_exact(y, ref, "conv_fwd")
    check_sums(stats[:cout], y, "stats sum", True)  # (y equals ref here)
    check_sums(stats[cout:], y * y, "stats sum of squares", True)


# =====================================================================================================================
# inference epilogue: v = relu(acc * scale + bias + residual), BatchNorm folded into scale / bias
EVAL = [dict(FWD_BY_DESC["64->256 k1 s1 @80x80"], bn=(64, 256)),  # bottleneck conv3
        dict(FWD_BY_DESC["64->64 k3 s1 @80x80"], bn=(32, 64))]    # BasicBlock conv2


@pytest.mark.parametrize("c,bn,exact", sweep(EVAL, ("real", "exact")))
def test_conv_fwd_eval_epilogue(mcb, cuda, monkeypatch, c, bn, exact):
    set_knobs(monkeypatch, bn=bn)
    exact = exact == "exact"
    n, h, w, cout = c["n"], c["h"], c["w"], c["cout"]
    assert_tiles_per_cta(tile_count(n, h, w, cout, bn, any_box=True), 2)
    x, wt, _, conv, absconv = fwd_ref(c, exact, _REF)
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


DGRAD_MASKED = [DGRAD_BY_DESC[d] for d in ("128->128 k3 s1 @160x160", "64->64 k3 s1 @80x80", "256->64 k1 s1 @80x80")]


@pytest.mark.parametrize("c,bn,halo,exact", sweep(DGRAD_MASKED, ("real", "exact"), halo=True))
def test_conv_dgrad_masked_channel_sum(mcb, cuda, monkeypatch, c, bn, halo, exact):
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn, halo=halo)
    exact = exact == "exact"
    n, h, w, cin, k, s = c["n"], c["h"], c["w"], c["cin"], c["k"], c["s"]
    assert_tiles_per_cta(tile_count(n, h, w, cin, bn, any_box=True), 2)
    dy, wt, act, _, ref, absref = dgrad_ref(c, exact, _REF)
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
    check_sums(cs1, nchw(dx1), "channel_sum", exact)  # the channel sum is defined on the STORED gradient


BNRED = [DGRAD_BY_DESC["128->128 k3 s2 @80x80"]]


@pytest.mark.parametrize("c,bn,exact", sweep(BNRED, ("real", "exact")))
def test_conv_dgrad_bn_reduce_stride2(mcb, cuda, monkeypatch, c, bn, exact):
    """the backward of the producing conv-BN-ReLU unit fused into a stride-2 data gradient: four phases, each with its
    own output and aux tensor maps, so the aux prefetch of the next tile crosses phases"""
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn)
    exact = exact == "exact"
    n, h, w, cin, k, s = c["n"], c["h"], c["w"], c["cin"], c["k"], c["s"]
    assert_tiles_per_cta(tile_count(n, h // 2, w // 2, cin, bn, 4, any_box=True), 2)
    dy, wt, _, bnp, ref, absref = dgrad_ref(c, exact, _REF)
    yb, xhat = bn_terms(bnp)
    mask = (yb > 0).double()
    decided = torch.ones_like(mask) if exact else (yb.abs() > 1e-3).double()  # sign not hinging on fma rounding
    runs = []
    for _ in range(2):
        bnr = bn_reduce(bnp)
        runs.append((ops.conv_dgrad(dev(dy), pack(wt), k, s, (h, w), bn_reduce=bnr),) + bnr[-2:])
    (dx, db, dgm), (dx2, db2, dgm2) = runs
    assert_same(dx, dx2, "dgrad bn-mask")
    assert_same(db, db2, "dbeta")
    assert_same(dgm, dgm2, "dgamma")
    gq = nchw(dx).double().cpu()
    if exact:
        assert ref.abs().max() <= 256
        assert_exact(gq, ref * mask, "dgrad bn-mask")
        assert (gq * xhat).abs().sum((0, 2, 3)).max() < 2 ** 22
    else:
        assert_bound(gq * decided, ref * mask * decided, absref * decided, "dgrad bn-mask")
    check_sums(db, gq, "dbeta", exact)
    check_sums(dgm, gq * xhat, "dgamma", exact)


@pytest.mark.parametrize("c,bn", sweep([DGRAD_BY_DESC["256->512 k1 s2 @80x80"]]))
def test_conv_dgrad_1x1_stride2_accumulate(mcb, cuda, monkeypatch, c, bn):
    """only the even pixels of a 1x1 stride-2 conv's input receive gradient: without accumulate the rest is zero,
    with accumulate it keeps the existing gradient bitwise"""
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn)
    n, h, w, cin, k, s = c["n"], c["h"], c["w"], c["cin"], c["k"], c["s"]
    assert_tiles_per_cta(tile_count(n, h // 2, w // 2, cin, bn, any_box=True), 2)
    dy, wt, _, _, ref, absref = dgrad_ref(c, False, _REF)
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
    dy, wt, _, _, ref, absref = dgrad_ref(c, False, _REF)
    dyd, wp = dev(dy), pack(wt)
    g = gen("concat-acc", c["desc"])
    for off, cin in ((0, 256), (256, 64)):
        assert_tiles_per_cta(tile_count(n, h, w, cin, bn, any_box=True), 2)
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


@pytest.mark.parametrize("c,bn,exact", sweep(CONVT, ("real", "exact")))
def test_convt(mcb, cuda, monkeypatch, c, bn, exact):
    from mcb200 import ops
    set_knobs(monkeypatch, bn=bn)
    exact = exact == "exact"
    n, h, w, cin, cout = c["n"], c["h"], c["w"], c["cin"], c["cout"]
    assert_tiles_per_cta(tile_count(n, h, w, cout, bn, 4, any_box=True), 2)
    assert_tiles_per_cta(tile_count(n, h, w, cin, bn, any_box=True), 2)
    x, wt, dy, b, act, y_ref, dx_ref, _, y_abs, dx_abs, _ = convt_ref(c, exact, _REF)
    check = (lambda got, r, a, what, **kw: assert_exact(got, r, what)) if exact else assert_bound
    if exact:
        assert max(y_ref.abs().max(), dx_ref.abs().max()) <= 256 - 3
    wp, xd, dyd = pack_t(wt), dev(x), dev(dy)
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
    check_sums(cs1, nchw(dx1), "convt channel_sum", exact)


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


def ragged_splits(tiles):
    """a split count that does not divide the pixel tiles and leaves the last split(s) without any"""
    for s in range(3, tiles):
        per = -(-tiles // s)
        if tiles % s and -(-tiles // per) < s:
            return s
    raise AssertionError("no ragged split for %d tiles" % tiles)


def wgrad_operands(c, exact):
    """x, dy, then the float64 dW and A in the library's (taps, cout, cin) layout"""
    from mcb200 import ops
    if c["s"] == 0:
        x, _, dy, _, _, _, _, dw, _, _, dw_abs = convt_ref(c, exact, _REF)
        return x, dy, ops.pack_convt_weight(dw), ops.pack_convt_weight(dw_abs)
    x, dy, dw, dw_abs = wgrad_ref(c, exact, _REF)
    return x, dy, ops.pack_conv_weight(dw), ops.pack_conv_weight(dw_abs)


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
    x, dy, ref, absref = wgrad_operands(c, exact == "exact")
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
        x, dy, ref, absref = wgrad_operands(c, False)
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
