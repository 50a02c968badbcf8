"""Parity of the wgmma convolution family (forward, data gradient, weight gradient, transposed conv) against
torch's fp32 CPU convolution — the op the reference calls (nn.Conv2d / nn.ConvTranspose2d, src/unet_models.py:21-34,
125-150; torchvision resnet blocks) — on bf16-rounded operands.

Tolerance: outputs are stored as bf16 (8 mantissa bits) after fp32 accumulation, so |err| <= 2^-8 |ref| + small
accumulation-order noise; integer-valued cases must match exactly.

These shapes are small: each CTA of the persistent conv kernel runs about one tile, and the weight-gradient ring does
not wrap.  test_conv_gemm_persistent_gpu.py covers the multi-tile regime of the full-size network (several tiles per
CTA, every N-tile width, accumulation into existing gradients) with element-wise float64 bounds."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def bf16r(x):
    return x.to(torch.bfloat16).to(torch.float32)


def assert_close_bf16(got, ref, what, extra=0.0):
    got = got.float().cpu()
    err = (got - ref).abs()
    tol = ref.abs() * 2.0 ** -7 + 2e-2 * ref.abs().mean() + 1e-3 + extra
    bad = (err > tol)
    assert not bad.any(), "%s: %d/%d elements off, max err %g (ref max %g)" % (
        what, int(bad.sum()), bad.numel(), float(err.max()), float(ref.abs().max()))


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
    from mcb200 import ops
    g = torch.Generator().manual_seed(1234 + h * w + cin)
    x = bf16r(torch.randn(n, cin, h, w, generator=g))
    wt = bf16r(torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5)
    b = torch.randn(cout, generator=g)
    ref = F.conv2d(x, wt, b, stride=stride, padding=k // 2)
    xd = nhwc(x).to(cuda, torch.bfloat16)
    wp = ops.pack_conv_weight(wt).to(cuda, torch.bfloat16)
    y = ops.conv_fwd(xd, wp, k, stride, bias=b.to(cuda))
    torch.cuda.synchronize()
    assert_close_bf16(nchw(y), ref, "conv_fwd")
    # fused ReLU + no bias + statistics
    stats = torch.zeros(2 * cout, device=cuda)
    y2 = ops.conv_fwd(xd, wp, k, stride, relu=True, stats=stats)
    torch.cuda.synchronize()
    ref2 = F.relu(F.conv2d(x, wt, None, stride=stride, padding=k // 2))
    assert_close_bf16(nchw(y2), ref2, "conv_fwd relu")
    yf = y2.float()
    s1 = yf.sum(dim=(0, 1, 2)).cpu()
    s2 = (yf * yf).sum(dim=(0, 1, 2)).cpu()
    st = stats.cpu()
    assert torch.allclose(st[:cout], s1, rtol=1e-4, atol=1e-2), (st[:cout] - s1).abs().max()
    assert torch.allclose(st[cout:], s2, rtol=1e-4, atol=1e-2), (st[cout:] - s2).abs().max()


def test_conv_fwd_integer_exact(mcb, cuda):
    """small-integer operands: every product and partial sum is exact in fp32 and the result fits bf16 exactly"""
    from mcb200 import ops
    g = torch.Generator().manual_seed(7)
    n, h, w, cin, cout, k = 2, 12, 20, 64, 64, 3
    x = torch.randint(-1, 2, (n, cin, h, w), generator=g).float()
    wt = (torch.rand(cout, cin, k, k, generator=g) < 0.1).float() * torch.randint(-1, 2, (cout, cin, k, k), generator=g)
    ref = F.conv2d(x, wt, None, padding=1)
    assert ref.abs().max() <= 256
    y = ops.conv_fwd(nhwc(x).to(cuda, torch.bfloat16), ops.pack_conv_weight(wt).to(cuda, torch.bfloat16), k)
    assert torch.equal(nchw(y).float().cpu(), ref)


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 32, 16, 64, 128), (1, 32, 24, 128, 64), (1, 16, 16, 32, 32),
                                             (2, 20, 20, 64, 64)])
def test_conv3x3_haloed_tile_path(mcb, cuda, monkeypatch, n, h, w, cin, cout):
    _haloed_tile_checks(cuda, monkeypatch, n, h, w, cin, cout)


def _haloed_tile_checks(cuda, monkeypatch, n, h, w, cin, cout):
    """MCB_HALO=1 forces the haloed-tile 3x3 path (one TMA box per channel chunk serves the nine taps through
    row-shifted wgmma descriptors; default rule: >= 128 channels on large images): forward (+stats, integer-exact),
    plain / masked data gradient, against the same references as the per-tap path"""
    from mcb200 import ops
    monkeypatch.setenv("MCB_HALO", "1")
    g = torch.Generator().manual_seed(11 + h + cin)
    x = torch.randint(-1, 2, (n, cin, h, w), generator=g).float()
    wt = (torch.rand(cout, cin, 3, 3, generator=g) < 0.1).float() * torch.randint(-1, 2, (cout, cin, 3, 3), generator=g)
    ref = F.conv2d(x, wt, None, padding=1)
    stats = torch.zeros(2 * cout, device=cuda)
    wp = ops.pack_conv_weight(wt).to(cuda, torch.bfloat16)
    y = ops.conv_fwd(nhwc(x).to(cuda, torch.bfloat16), wp, 3, stats=stats)
    assert torch.equal(nchw(y).float().cpu(), ref)
    assert torch.allclose(stats[:cout].cpu(), ref.sum(dim=(0, 2, 3)), atol=1e-2)
    dy = bf16r(torch.randn(n, cout, h, w, generator=g))
    wr = bf16r(torch.randn(cout, cin, 3, 3, generator=g) / (cout * 9) ** 0.5)
    dref = torch.nn.grad.conv2d_input((n, cin, h, w), wr, dy, padding=1)
    wrp = ops.pack_conv_weight(wr).to(cuda, torch.bfloat16)
    dyd = nhwc(dy).to(cuda, torch.bfloat16)
    assert_close_bf16(nchw(ops.conv_dgrad(dyd, wrp, 3, 1, (h, w))), dref, "halo dgrad")
    act = bf16r(torch.randn(n, cin, h, w, generator=g))
    dxm = ops.conv_dgrad(dyd, wrp, 3, 1, (h, w), relu_mask=nhwc(act).to(cuda, torch.bfloat16))
    assert_close_bf16(nchw(dxm), dref * (act > 0).float(), "halo dgrad mask")


def test_conv_fwd_concat(mcb, cuda):
    from mcb200 import ops
    g = torch.Generator().manual_seed(3)
    n, h, w, c0, c1, cout = 2, 10, 10, 64, 128, 128
    x0 = bf16r(torch.randn(n, c0, h, w, generator=g))
    x1 = bf16r(torch.randn(n, c1, h, w, generator=g))
    wt = bf16r(torch.randn(cout, c0 + c1, 3, 3, generator=g) / 40)
    b = torch.randn(cout, generator=g)
    ref = F.relu(F.conv2d(torch.cat([x0, x1], 1), wt, b, padding=1))
    y = ops.conv_fwd(nhwc(x0).to(cuda, torch.bfloat16), ops.pack_conv_weight(wt).to(cuda, torch.bfloat16), 3, 1,
                     bias=b.to(cuda), relu=True, x2=nhwc(x1).to(cuda, torch.bfloat16))
    assert_close_bf16(nchw(y), ref, "conv_fwd concat")


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
    g = torch.Generator().manual_seed(99 + h + cin + k)
    wt = bf16r(torch.randn(cout, cin, k, k, generator=g) / (cout * k * k) ** 0.5)
    dy = bf16r(torch.randn(n, cout, h // stride, w // stride, generator=g))
    ref = torch.nn.grad.conv2d_input((n, cin, h, w), wt, dy, stride=stride, padding=k // 2)
    wp = ops.pack_conv_weight(wt).to(cuda, torch.bfloat16)
    dyd = nhwc(dy).to(cuda, torch.bfloat16)
    dx = ops.conv_dgrad(dyd, wp, k, stride, (h, w))
    assert_close_bf16(nchw(dx), ref, "conv_dgrad")
    # relu mask
    act = bf16r(torch.randn(n, cin, h, w, generator=g))
    csum = torch.zeros(cin, device=cuda)
    dx2 = ops.conv_dgrad(dyd, wp, k, stride, (h, w), relu_mask=nhwc(act).to(cuda, torch.bfloat16), channel_sum=csum)
    assert_close_bf16(nchw(dx2), ref * (act > 0).float(), "conv_dgrad mask")
    # fused bias gradient of the producing layer = per-channel sum of the STORED masked gradient
    assert torch.allclose(csum.cpu(), nchw(dx2).float().cpu().sum(dim=(0, 2, 3)), rtol=1e-4, atol=1e-3)
    # accumulate on top of an existing gradient
    base = bf16r(torch.randn(n, cin, h, w, generator=g))
    acc = nhwc(base).to(cuda, torch.bfloat16)
    ops.conv_dgrad(dyd, wp, k, stride, (h, w), accumulate=True, out=acc)
    assert_close_bf16(nchw(acc), ref + base, "conv_dgrad accumulate", extra=2.0 ** -7 * float(base.abs().max()))


@pytest.mark.parametrize("n,h,w,cin,cout,k,stride", [(2, 16, 16, 64, 128, 3, 1), (2, 20, 20, 256, 64, 1, 1),
                                                       (2, 16, 16, 128, 128, 3, 2), (4, 5, 5, 128, 512, 3, 1)])
def test_conv_dgrad_fused_bn_reductions(mcb, cuda, n, h, w, cin, cout, k, stride):
    """dgrad epilogue fused with the backward of the producing conv-BN-ReLU unit: ReLU mask recomputed from the BN input
    z (TMA-fetched tile), BatchNorm-backward sums of the stored gradient"""
    from mcb200 import ops
    g = torch.Generator().manual_seed(5 + h + cin)
    wt = bf16r(torch.randn(cout, cin, k, k, generator=g) / (cout * k * k) ** 0.5)
    dy = bf16r(torch.randn(n, cout, h // stride, w // stride, generator=g))
    z = bf16r(torch.randn(n, cin, h, w, generator=g) * 1.5 + 0.3)
    mean, invstd = torch.randn(cin, generator=g) * 0.2, torch.rand(cin, generator=g) + 0.5
    gamma, beta = torch.randn(cin, generator=g), torch.randn(cin, generator=g) * 0.5
    sc = gamma * invstd
    sh = beta - mean * sc
    y = z * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)
    decided = (y.abs() > 1e-3).float()  # elements whose sign does not hinge on fma rounding
    ref = torch.nn.grad.conv2d_input((n, cin, h, w), wt, dy, stride=stride, padding=k // 2) * (y > 0).float()
    dbeta, dgamma = torch.zeros(cin, device=cuda), torch.zeros(cin, device=cuda)
    dx = ops.conv_dgrad(nhwc(dy).to(cuda, torch.bfloat16), ops.pack_conv_weight(wt).to(cuda, torch.bfloat16), k, stride,
                        (h, w), bn_reduce=(nhwc(z).to(cuda, torch.bfloat16), mean.to(cuda), invstd.to(cuda),
                                           gamma.to(cuda), beta.to(cuda), dbeta, dgamma))
    assert_close_bf16(nchw(dx) * decided.to(cuda), ref * decided, "dgrad bn-mask")
    gq = nchw(dx).float().cpu()  # the sums are defined on the STORED gradient
    xhat = (z - mean.view(1, -1, 1, 1)) * invstd.view(1, -1, 1, 1)
    assert torch.allclose(dbeta.cpu(), gq.sum(dim=(0, 2, 3)), rtol=1e-4, atol=1e-3)
    assert torch.allclose(dgamma.cpu(), (gq * xhat).sum(dim=(0, 2, 3)), rtol=1e-4, atol=2e-3)


def test_conv_dgrad_concat_slice(mcb, cuda):
    from mcb200 import ops
    g = torch.Generator().manual_seed(5)
    n, h, w, c0, c1, cout = 2, 10, 10, 64, 128, 128
    wt = bf16r(torch.randn(cout, c0 + c1, 3, 3, generator=g) / 30)
    dy = bf16r(torch.randn(n, cout, h, w, generator=g))
    ref = torch.nn.grad.conv2d_input((n, c0 + c1, h, w), wt, dy, padding=1)
    wp = ops.pack_conv_weight(wt).to(cuda, torch.bfloat16)
    dyd = nhwc(dy).to(cuda, torch.bfloat16)
    d0 = ops.conv_dgrad(dyd, wp, 3, 1, (h, w), cin=c0, ci_off=0)
    d1 = ops.conv_dgrad(dyd, wp, 3, 1, (h, w), cin=c1, ci_off=c0)
    assert_close_bf16(nchw(d0), ref[:, :c0], "dgrad slice 0")
    assert_close_bf16(nchw(d1), ref[:, c0:], "dgrad slice 1")


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
    g = torch.Generator().manual_seed(17 + h + cin + k)
    x = bf16r(torch.randn(n, cin, h, w, generator=g))
    dy = bf16r(torch.randn(n, cout, h // stride, w // stride, generator=g))
    ref = torch.nn.grad.conv2d_weight(x, (cout, cin, k, k), dy, stride=stride, padding=k // 2)
    dw = torch.zeros(k * k, cout, cin, device=cuda)
    ops.conv_wgrad(nhwc(dy).to(cuda, torch.bfloat16), nhwc(x).to(cuda, torch.bfloat16), dw, k, stride)
    got = ops.unpack_conv_weight(dw, k).cpu()
    err = (got - ref).abs().max()
    assert err <= 1e-3 * ref.abs().max() + 1e-3, "wgrad err %g (ref max %g)" % (err, ref.abs().max())


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 8, 8, 64, 64), (2, 10, 10, 128, 256), (1, 16, 16, 128, 32),
                                             (3, 5, 5, 512, 256)])
def test_convt(mcb, cuda, n, h, w, cin, cout):
    from mcb200 import ops
    g = torch.Generator().manual_seed(23 + h + cin)
    x = bf16r(torch.randn(n, cin, h, w, generator=g))
    wt = bf16r(torch.randn(cin, cout, 4, 4, generator=g) / (cin * 4) ** 0.5)
    b = torch.randn(cout, generator=g)
    ref = F.relu(F.conv_transpose2d(x, wt, b, stride=2, padding=1))
    wp = ops.pack_convt_weight(wt).to(cuda, torch.bfloat16)
    xd = nhwc(x).to(cuda, torch.bfloat16)
    y = ops.convt_fwd(xd, wp, bias=b.to(cuda), relu=True)
    assert_close_bf16(nchw(y), ref, "convt_fwd")
    # gradients
    dy = bf16r(torch.randn(n, cout, 2 * h, 2 * w, generator=g))
    xr = x.clone().requires_grad_(True)
    wr = wt.clone().requires_grad_(True)
    F.conv_transpose2d(xr, wr, None, stride=2, padding=1).backward(dy)
    dyd = nhwc(dy).to(cuda, torch.bfloat16)
    dx = ops.convt_dgrad(dyd, wp)
    assert_close_bf16(nchw(dx), xr.grad, "convt_dgrad")
    act = bf16r(torch.randn(*xr.shape, generator=g))
    csum = torch.zeros(xr.shape[1], device=cuda)
    dxm = ops.convt_dgrad(dyd, wp, relu_mask=nhwc(act).to(cuda, torch.bfloat16), channel_sum=csum)
    assert_close_bf16(nchw(dxm), xr.grad * (act > 0).float(), "convt_dgrad mask")
    assert torch.allclose(csum.cpu(), nchw(dxm).float().cpu().sum(dim=(0, 2, 3)), rtol=1e-4, atol=1e-3)
    dw = torch.zeros(16, cout, cin, device=cuda)
    ops.convt_wgrad(dyd, xd, dw)
    got = ops.unpack_convt_weight(dw).cpu()
    err = (got - wr.grad).abs().max()
    assert err <= 1e-3 * wr.grad.abs().max() + 1e-3, "convt wgrad err %g" % err
