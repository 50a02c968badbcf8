"""The 3x3 transposed conv of the UNet11 decoder (nn.ConvTranspose2d(kernel_size=3, stride=2, padding=1,
output_padding=1), reference src/unet_models.py:42-53) through mcb_convt_{fwd,dgrad,wgrad} with ksize = 3.

References and bars: oracle/conv_checks.py (float64; bf16 outputs within 2^-8 |ref| + 2^-16 A, fp32 dW within
2^-16 A); integer-exact variants (operands in {-1, 0, 1}, |ref| <= 256) must match bit for bit.  Shapes cover ragged
tiles (sides that are not tile multiples, where the d=+1 tap of output parity 1 reads the zero row past the edge) and a
persistent launch in which every CTA runs at least two tiles."""
import pytest
import torch

from oracle.conv_checks import (assert_accumulated, assert_bound, assert_exact, assert_same, assert_tiles_per_cta,
                                bf16r, check_sums, convt_ref, dev, gen, nchw, pack_t, tile_count)

pytestmark = pytest.mark.gpu


def case(n, h, w, cin, cout, k=3):
    return dict(desc=(n, h, w, cin, cout, k), n=n, h=h, w=w, cin=cin, cout=cout, k=k)


SHAPES = [(2, 8, 8, 64, 32), (3, 13, 7, 32, 64), (1, 11, 20, 128, 64), (2, 10, 10, 256, 128)]


@pytest.mark.parametrize("n,h,w,cin,cout", SHAPES)
def test_convt3_forward_dgrad_wgrad(mcb, cuda, n, h, w, cin, cout):
    from mcb200 import ops
    c = case(n, h, w, cin, cout)
    x, wt, dy, b, act, y_ref, dx_ref, dw_ref, y_abs, dx_abs, dw_abs = convt_ref(c, False)
    wp = pack_t(wt)
    assert wp.shape == (9, cout, cin)
    # forward, bias + ReLU epilogue
    bd = b.double().view(1, -1, 1, 1)
    y = ops.convt_fwd(dev(x), wp, bias=b.to(cuda), relu=True)
    assert y.shape == (n, 2 * h, 2 * w, cout)
    assert_bound(nchw(y), (y_ref + bd).clamp_min(0), y_abs + bd.abs(), "convt3 fwd")
    # data gradient, plain and with the producer's ReLU mask + its bias gradient (channel sum of the stored dx)
    assert_bound(nchw(ops.convt_dgrad(dev(dy), wp)), dx_ref, dx_abs, "convt3 dgrad")
    csum = torch.zeros(cin, dtype=torch.float32, device=cuda)
    stored = nchw(ops.convt_dgrad(dev(dy), wp, relu_mask=dev(act), channel_sum=csum)).double().cpu()
    mask = (act > 0).double()
    assert_bound(stored, dx_ref * mask, dx_abs * mask, "convt3 dgrad masked")
    assert torch.allclose(csum.double().cpu(), stored.sum(dim=(0, 2, 3)), rtol=1e-5,
                          atol=1e-5 * float(stored.abs().sum(dim=(0, 2, 3)).max()))
    # accumulate onto an existing gradient
    g = gen("pre", c["desc"])
    base = bf16r(torch.randn(n, cin, h, w, generator=g))
    dxa = dev(base)
    ops.convt_dgrad(dev(dy), wp, accumulate=True, out=dxa)
    assert_accumulated(nchw(dxa), base, dx_ref, dx_abs, "convt3 dgrad accumulate")
    # weight gradient added to a random dW
    dw0 = torch.randn(9, cout, cin, generator=g)
    dw = dw0.to(cuda)
    ops.convt_wgrad(dev(dy), dev(x), dw)
    unpack = lambda t: ops.unpack_convt_weight(t, 3).double()
    assert_bound(unpack(dw), unpack(dw0) + dw_ref, unpack(dw0.abs()) + dw_abs, "convt3 wgrad", rel=0.0)


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 9, 6, 64, 32), (2, 16, 16, 128, 64)])
def test_convt3_integer_exact(mcb, cuda, n, h, w, cin, cout):
    """operands in {-1, 0, 1}: every output, the channel sums and dW are exact in fp32 and bf16"""
    from mcb200 import ops
    c = case(n, h, w, cin, cout)
    x, wt, dy, _, act, ref, dx_ref, dw_ref, _, _, _ = convt_ref(c, True)
    wp = pack_t(wt)
    assert float(ref.abs().max()) <= 256
    assert_exact(nchw(ops.convt_fwd(dev(x), wp)), ref, "convt3 fwd")
    assert float(dx_ref.abs().max()) <= 256 and float(dw_ref.abs().max()) < 2 ** 23
    csum = torch.zeros(cin, dtype=torch.float32, device=cuda)
    dxm = nchw(ops.convt_dgrad(dev(dy), wp, relu_mask=dev(act), channel_sum=csum))
    assert_exact(dxm, dx_ref * (act > 0).double(), "convt3 dgrad masked")
    check_sums(csum, dxm, "convt3 channel sum", True)
    dw0 = torch.randint(-4, 5, (9, cout, cin), generator=gen("pre", c["desc"])).float()
    dw = dw0.to(cuda)
    ops.convt_wgrad(dev(dy), dev(x), dw)
    assert_exact(ops.unpack_convt_weight(dw, 3), ops.unpack_convt_weight(dw0, 3).double() + dw_ref, "convt3 wgrad")


def test_convt3_persistent_multi_tile(mcb, cuda):
    """enough tiles that every CTA of the persistent grid runs at least two (for any pixel box the host picks), so the
    TMA ring, the output-buffer rotation and the phase walk carry across tiles; the fused channel sum and the split-K
    weight gradient must give the same bits twice"""
    from mcb200 import ops
    n, h, w, cin, cout = 16, 48, 48, 128, 64
    assert_tiles_per_cta(tile_count(n, h, w, cout, None, 4, any_box=True), 2)
    assert_tiles_per_cta(tile_count(n, h, w, cin, None, any_box=True), 2)
    x, wt, dy, _, act, y_ref, dx_ref, dw_ref, y_abs, dx_abs, dw_abs = convt_ref(case(n, h, w, cin, cout), False)
    wp = pack_t(wt)
    assert_bound(nchw(ops.convt_fwd(dev(x), wp)), y_ref, y_abs, "convt3 fwd persistent")
    mask = (act > 0).double()
    sums, dws = [], []
    for _ in range(2):
        csum = torch.zeros(cin, dtype=torch.float32, device=cuda)
        dxm = ops.convt_dgrad(dev(dy), wp, relu_mask=dev(act), channel_sum=csum)
        dw = torch.zeros(9, cout, cin, dtype=torch.float32, device=cuda)
        ops.convt_wgrad(dev(dy), dev(x), dw)
        sums.append(csum)
        dws.append(dw)
    assert_bound(nchw(dxm), dx_ref * mask, dx_abs * mask, "convt3 dgrad persistent")
    assert_bound(ops.unpack_convt_weight(dws[0], 3), dw_ref, dw_abs, "convt3 wgrad persistent", rel=0.0)
    assert_same(sums[0], sums[1], "convt3 channel sum")
    assert_same(dws[0], dws[1], "convt3 wgrad")


def test_convt_ksize_zero_means_four(mcb, cuda):
    """a zeroed ksize field keeps the 4x4 kernel: the ABI of existing callers is unchanged"""
    from mcb200 import _lib as L
    from mcb200 import ops
    x, wt, _, _, _, ref, _, _, ref_abs, _, _ = convt_ref(case(1, 6, 6, 64, 32, k=4), False)
    wp = pack_t(wt)
    xd = dev(x)
    y = torch.empty(1, 12, 12, 32, dtype=torch.bfloat16, device=cuda)
    a = L.ConvtFwdArgs()
    a.x = xd.data_ptr(); a.n, a.h, a.w, a.cin = 1, 6, 6, 64
    a.weight = wp.data_ptr(); a.cout = 32; a.y = y.data_ptr()
    assert a.ksize == 0
    L.call("mcb_convt_fwd", a)
    assert torch.equal(y, ops.convt_fwd(xd, wp))
    assert_bound(nchw(y), ref, ref_abs, "convt4 fwd")
    a.ksize = 5
    with pytest.raises(RuntimeError, match="ksize"):
        L.call("mcb_convt_fwd", a)
