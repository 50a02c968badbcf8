"""Parity of the wgmma convolution family (forward, data gradient, weight gradient, transposed conv) with the op the
reference calls (nn.Conv2d / nn.ConvTranspose2d, src/unet_models.py:21-34, 125-150; torchvision resnet blocks), on
bf16-rounded operands.  References and bars: oracle/conv_checks.py (float64, element-wise: bf16 outputs within
2^-8 |ref| + 2^-16 A, fp32 weight gradients within 2^-16 A); integer-valued cases must match exactly.  The
real-valued fused per-channel sums keep their allclose bars (rtol 1e-4) against the sum of the stored output.

These shapes are small: each CTA of the persistent conv kernel runs about one tile, and the weight-gradient ring does
not wrap.  test_conv_gemm_persistent_gpu.py covers the multi-tile regime of the full-size network (several tiles per
CTA, every N-tile width, accumulation into existing gradients)."""
import pytest
import torch

from oracle.conv_checks import (assert_accumulated, assert_bound, assert_exact, bf16r, bn_reduce, bn_terms,
                                check_sums, convt_ref, dev, dgrad_ref, fwd_ref, gen, nchw, pack, pack_t, run_fwd,
                                set_knobs, wgrad_ref)

pytestmark = pytest.mark.gpu


def case(n, h, w, cin, cout, k=3, s=1, c1=0):
    """a case dict of oracle/conv_checks.py, seeded by its shape"""
    return dict(desc=(n, h, w, cin, cout, k, s, c1), n=n, h=h, w=w, c0=cin - c1, c1=c1, cin=cin, cout=cout, k=k, s=s)


FWD_CASES = [
    # n, h, w, cin, cout, k, stride
    (2, 16, 16, 64, 64, 1, 1),
    (2, 16, 16, 64, 128, 3, 1),
    (3, 20, 20, 128, 256, 3, 1),
    (2, 20, 12, 256, 64, 1, 1),
    (2, 16, 16, 64, 128, 3, 2),
    (2, 24, 16, 128, 256, 1, 2),
    (4, 5, 5, 128, 512, 3, 1),
    (2, 10, 10, 512, 512, 3, 1),
    (1, 32, 32, 32, 32, 3, 1),
    (2, 8, 8, 1024, 256, 1, 1),
]


@pytest.mark.parametrize("n,h,w,cin,cout,k,stride", FWD_CASES)
def test_conv_fwd(mcb, cuda, n, h, w, cin, cout, k, stride):
    c = case(n, h, w, cin, cout, k, stride)
    x, wt, b, ref, absref = fwd_ref(c, False)
    bd = b.double().view(1, -1, 1, 1)
    y = run_fwd(c, x, wt, bias=b.to(cuda))
    assert_bound(nchw(y), ref + bd, absref + bd.abs(), "conv_fwd")
    # fused ReLU + no bias + statistics
    stats = torch.zeros(2 * cout, device=cuda)
    y2 = run_fwd(c, x, wt, relu=True, stats=stats)
    assert_bound(nchw(y2), ref.clamp_min(0), absref, "conv_fwd relu")
    yf = y2.float()
    s1 = yf.sum(dim=(0, 1, 2)).cpu()
    s2 = (yf * yf).sum(dim=(0, 1, 2)).cpu()
    st = stats.cpu()
    assert torch.allclose(st[:cout], s1, rtol=1e-4, atol=1e-2), (st[:cout] - s1).abs().max()
    assert torch.allclose(st[cout:], s2, rtol=1e-4, atol=1e-2), (st[cout:] - s2).abs().max()


def test_conv_fwd_integer_exact(mcb, cuda):
    """small-integer operands: every product and partial sum is exact in fp32 and the result fits bf16 exactly"""
    c = case(2, 12, 20, 64, 64)
    x, wt, _, ref, _ = fwd_ref(c, True)
    assert ref.abs().max() <= 256
    assert_exact(nchw(run_fwd(c, x, wt)), ref, "conv_fwd")


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 32, 16, 64, 128), (1, 32, 24, 128, 64), (1, 16, 16, 32, 32),
                                             (2, 20, 20, 64, 64)])
def test_conv3x3_haloed_tile_path(mcb, cuda, monkeypatch, n, h, w, cin, cout):
    _haloed_tile_checks(cuda, monkeypatch, n, h, w, cin, cout)


def _haloed_tile_checks(cuda, monkeypatch, n, h, w, cin, cout):
    """MCB_HALO=1 forces the haloed-tile 3x3 path (one TMA box per channel chunk serves the nine taps through
    row-shifted wgmma descriptors; default rule: >= 128 channels on large images): forward (+stats, integer-exact),
    plain / masked data gradient, against the same references as the per-tap path"""
    from mcb200 import ops
    set_knobs(monkeypatch, halo=1)
    c = case(n, h, w, cin, cout)
    x, wt, _, ref, _ = fwd_ref(c, True)
    stats = torch.zeros(2 * cout, device=cuda)
    y = nchw(run_fwd(c, x, wt, stats=stats))
    assert_exact(y, ref, "halo conv_fwd")
    check_sums(stats[:cout], y, "halo stats sum", True)
    dy, wr, act, _, dref, dabs = dgrad_ref(c, False)
    dyd, wrp = dev(dy), pack(wr)
    assert_bound(nchw(ops.conv_dgrad(dyd, wrp, 3, 1, (h, w))), dref, dabs, "halo dgrad")
    mask = (act > 0).double()
    dxm = ops.conv_dgrad(dyd, wrp, 3, 1, (h, w), relu_mask=dev(act))
    assert_bound(nchw(dxm), dref * mask, dabs * mask, "halo dgrad mask")


def test_conv_fwd_concat(mcb, cuda):
    c = case(2, 10, 10, 64 + 128, 128, c1=128)
    x, wt, b, ref, absref = fwd_ref(c, False)
    bd = b.double().view(1, -1, 1, 1)
    y = run_fwd(c, x, wt, bias=b.to(cuda), relu=True)
    assert_bound(nchw(y), (ref + bd).clamp_min(0), absref + bd.abs(), "conv_fwd concat")


DGRAD_CASES = [
    (2, 16, 16, 64, 64, 1, 1),
    (2, 16, 16, 64, 128, 3, 1),
    (2, 20, 20, 256, 128, 3, 1),
    (2, 16, 16, 64, 128, 3, 2),
    (2, 16, 24, 128, 256, 1, 2),
    (1, 32, 32, 32, 32, 3, 1),
    (4, 5, 5, 128, 512, 3, 1),
]


@pytest.mark.parametrize("n,h,w,cin,cout,k,stride", DGRAD_CASES)
def test_conv_dgrad(mcb, cuda, n, h, w, cin, cout, k, stride):
    from mcb200 import ops
    c = case(n, h, w, cin, cout, k, stride)
    dy, wt, act, _, ref, absref = dgrad_ref(c, False)
    wp, dyd = pack(wt), dev(dy)
    assert_bound(nchw(ops.conv_dgrad(dyd, wp, k, stride, (h, w))), ref, absref, "conv_dgrad")
    # relu mask
    mask = (act > 0).double()
    csum = torch.zeros(cin, device=cuda)
    dx2 = ops.conv_dgrad(dyd, wp, k, stride, (h, w), relu_mask=dev(act), channel_sum=csum)
    assert_bound(nchw(dx2), ref * mask, absref * mask, "conv_dgrad mask")
    # fused bias gradient of the producing layer = per-channel sum of the STORED masked gradient
    assert torch.allclose(csum.cpu(), nchw(dx2).float().cpu().sum(dim=(0, 2, 3)), rtol=1e-4, atol=1e-3)
    # accumulate on top of an existing gradient
    base = bf16r(torch.randn(n, cin, h, w, generator=gen("acc", c["desc"])))
    acc = dev(base)
    ops.conv_dgrad(dyd, wp, k, stride, (h, w), accumulate=True, out=acc)
    assert_accumulated(nchw(acc), base, ref, absref, "conv_dgrad accumulate")


@pytest.mark.parametrize("n,h,w,cin,cout,k,stride", [(2, 16, 16, 64, 128, 3, 1), (2, 20, 20, 256, 64, 1, 1),
                                                       (2, 16, 16, 128, 128, 3, 2), (4, 5, 5, 128, 512, 3, 1)])
def test_conv_dgrad_fused_bn_reductions(mcb, cuda, n, h, w, cin, cout, k, stride):
    """dgrad epilogue fused with the backward of the producing conv-BN-ReLU unit: ReLU mask recomputed from the BN input
    z (TMA-fetched tile), BatchNorm-backward sums of the stored gradient"""
    from mcb200 import ops
    dy, wt, _, bnp, ref, absref = dgrad_ref(case(n, h, w, cin, cout, k, stride), False)
    yb, xhat = bn_terms(bnp)
    decided = (yb.abs() > 1e-3).double()  # elements whose sign does not hinge on fma rounding
    args = bn_reduce(bnp)
    dx = nchw(ops.conv_dgrad(dev(dy), pack(wt), k, stride, (h, w), bn_reduce=args)).cpu()
    assert_bound(dx * decided, ref * (yb > 0).double() * decided, absref * decided, "dgrad bn-mask")
    gq = dx.float()  # the sums are defined on the STORED gradient
    dbeta, dgamma = args[-2].cpu(), args[-1].cpu()
    assert torch.allclose(dbeta, gq.sum(dim=(0, 2, 3)), rtol=1e-4, atol=1e-3)
    assert torch.allclose(dgamma, (gq * xhat.float()).sum(dim=(0, 2, 3)), rtol=1e-4, atol=2e-3)


def test_conv_dgrad_concat_slice(mcb, cuda):
    from mcb200 import ops
    n, h, w, c0, c1, cout = 2, 10, 10, 64, 128, 128
    dy, wt, _, _, ref, absref = dgrad_ref(case(n, h, w, c0 + c1, cout), False)
    wp, dyd = pack(wt), dev(dy)
    d0 = ops.conv_dgrad(dyd, wp, 3, 1, (h, w), cin=c0, ci_off=0)
    d1 = ops.conv_dgrad(dyd, wp, 3, 1, (h, w), cin=c1, ci_off=c0)
    assert_bound(nchw(d0), ref[:, :c0], absref[:, :c0], "dgrad slice 0")
    assert_bound(nchw(d1), ref[:, c0:], absref[:, c0:], "dgrad slice 1")


WGRAD_CASES = [
    (2, 16, 16, 64, 64, 1, 1),
    (2, 16, 16, 64, 128, 3, 1),
    (3, 20, 20, 128, 256, 3, 1),
    (2, 16, 16, 64, 128, 3, 2),
    (2, 16, 24, 128, 256, 1, 2),
    (1, 32, 32, 32, 32, 3, 1),
    (4, 5, 5, 128, 512, 3, 1),
    (2, 8, 8, 256, 64, 1, 1),
]


@pytest.mark.parametrize("n,h,w,cin,cout,k,stride", WGRAD_CASES)
def test_conv_wgrad(mcb, cuda, n, h, w, cin, cout, k, stride):
    from mcb200 import ops
    x, dy, ref, absref = wgrad_ref(case(n, h, w, cin, cout, k, stride), False)
    dw = torch.zeros(k * k, cout, cin, device=cuda)
    ops.conv_wgrad(dev(dy), dev(x), dw, k, stride)
    assert_bound(ops.unpack_conv_weight(dw, k), ref, absref, "conv_wgrad", rel=0.0)


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 8, 8, 64, 64), (2, 10, 10, 128, 256), (1, 16, 16, 128, 32),
                                             (3, 5, 5, 512, 256)])
def test_convt(mcb, cuda, n, h, w, cin, cout):
    from mcb200 import ops
    x, wt, dy, b, act, y_ref, dx_ref, dw_ref, y_abs, dx_abs, dw_abs = convt_ref(case(n, h, w, cin, cout, 4), False)
    bd = b.double().view(1, -1, 1, 1)
    wp, xd, dyd = pack_t(wt), dev(x), dev(dy)
    y = ops.convt_fwd(xd, wp, bias=b.to(cuda), relu=True)
    assert_bound(nchw(y), (y_ref + bd).clamp_min(0), y_abs + bd.abs(), "convt_fwd")
    # gradients
    assert_bound(nchw(ops.convt_dgrad(dyd, wp)), dx_ref, dx_abs, "convt_dgrad")
    mask = (act > 0).double()
    csum = torch.zeros(cin, device=cuda)
    dxm = ops.convt_dgrad(dyd, wp, relu_mask=dev(act), channel_sum=csum)
    assert_bound(nchw(dxm), dx_ref * mask, dx_abs * mask, "convt_dgrad mask")
    assert torch.allclose(csum.cpu(), nchw(dxm).float().cpu().sum(dim=(0, 2, 3)), rtol=1e-4, atol=1e-3)
    dw = torch.zeros(16, cout, cin, device=cuda)
    ops.convt_wgrad(dyd, xd, dw)
    assert_bound(ops.unpack_convt_weight(dw), dw_ref, dw_abs, "convt_wgrad", rel=0.0)
