"""The kernels the VGG-encoder U-Nets (UNet11, UNetVGG16; reference src/unet_models.py:56-106, :224-312) add to the
H100 path:
  * the full-resolution 3-channel input conv, Conv2d(3, 64, 3, padding 1) + bias + ReLU, as an im2col (27 of 32
    columns, k = (ky*3 + kx)*3 + c) + the 1x1 GEMM, with its weight gradient unpacked into the [9][64][3] master slot;
  * the 32 + 64-channel concat conv of dec1 (ConvRelu(96, 32) over cat[dec2, conv1]): forward, the two segment data
    gradients (ci_off 0 / cin 32 and ci_off 32 / cin 64 of a 96-wide weight) and the two segment weight gradients;
  * the max-pool backward of a stage output that also feeds a decoder concat (mcb_maxpool2_bwd_skip_relu).

References and bars: oracle/conv_checks.py (float64 from the bf16-rounded operands, on the device for the input conv
and the pool; bf16 outputs within 2^-8 |ref| + 2^-16 A, fp32 sums and weight gradients within 2^-16 A); the pool's
routing and launch model: oracle/elementwise_checks.py.  Integer-valued variants must match bit for bit.  Every case
asserts its launch regime from the device's SM count."""
import pytest
import torch
import torch.nn.functional as F

from oracle.conv_checks import (assert_bound, assert_exact, assert_same, assert_tiles_per_cta, bf16r, check_sums, dev,
                                dgrad_ref, fwd_ref, nchw, pack, run_fwd, tile_count, wgrad_ref)
from oracle.elementwise_checks import pool_skip_ref, reduce_grid

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------- input conv
def _input_im2col_ref(x):
    """(n, 3, h, w) float64 -> (n, h, w, 32) with k = (ky*3 + kx)*3 + c, zero beyond 27 and outside the image"""
    n, _, h, w = x.shape
    xp = F.pad(x, (1, 1, 1, 1))
    col = torch.zeros(n, h, w, 32, dtype=x.dtype, device=x.device)
    for ky in range(3):
        for kx in range(3):
            for c in range(3):
                col[..., (ky * 3 + kx) * 3 + c] = xp[:, c, ky:ky + h, kx:kx + w]
    return col


INPUT_SHAPES = [(2, 8, 8), (3, 17, 100), (1, 31, 300), (32, 320, 320)]


@pytest.mark.parametrize("n,h,w", INPUT_SHAPES)
def test_input_conv_forward_and_weight_gradient(mcb, cuda, n, h, w):
    from mcb200 import ops
    if (n, h, w) == (32, 320, 320):
        assert_tiles_per_cta(tile_count(n, h, w, 64, None, any_box=True), 4)  # persistent: several pixel tiles per CTA
    if w % 64:
        assert w > 64 or n * h > 1                       # an im2col strip that the 64-pixel strip does not fill
    g = torch.Generator(device=cuda).manual_seed(n * 7 + h + w)
    x = torch.randn(n, 3, h, w, generator=g, device=cuda)
    col = ops.vgg_input_im2col(x)
    xr = bf16r(x).double()
    assert torch.equal(col.double(), _input_im2col_ref(xr))              # border pixels and pad columns included
    wt = torch.randn(64, 3, 3, 3, generator=g, device=cuda) / 27 ** 0.5
    slot = ops.pack_conv_weight(wt).reshape(-1).contiguous()             # master layout [9][64][3]
    w16 = torch.empty(1, 64, 32, dtype=torch.bfloat16, device=cuda)
    ops.vgg_input_pack_weight(slot, w16)
    wref = torch.zeros(64, 32, dtype=torch.float64, device=cuda)
    wr = bf16r(wt).double()
    wref[:, :27] = wr.permute(0, 2, 3, 1).reshape(64, 27)
    assert torch.equal(w16[0].double(), wref)
    bias = torch.randn(64, generator=g, device=cuda) * 0.1
    y = ops.conv_fwd(col, w16, 1, 1, bias=bias, relu=True)
    ref = torch.relu(F.conv2d(xr, wr, bias.double(), padding=1))
    acc = F.conv2d(xr.abs(), wr.abs(), bias.double().abs(), padding=1)
    assert_bound(nchw(y), ref, acc, "input conv fwd")
    # weight gradient: 1x1 wgrad over the im2col columns, then += into the master slot
    dy = bf16r(torch.randn(n, 64, h, w, generator=g, device=cuda)).double()
    gw = torch.zeros(1, 64, 32, dtype=torch.float32, device=cuda)
    ops.conv_wgrad(dev(dy), col, gw, 1, 1)
    assert bool((gw[0, :, 27:] == 0).all())
    base = torch.randn(9 * 64 * 3, generator=g, device=cuda)
    dw = base.clone()
    ops.vgg_input_unpack_wgrad(gw, dw)
    dref = torch.nn.grad.conv2d_weight(xr, wt.shape, dy, padding=1)
    dacc = torch.nn.grad.conv2d_weight(xr.abs(), wt.shape, dy.abs(), padding=1)
    got = ops.unpack_conv_weight((dw - base).view(9, 64, 3), 3)
    base_abs = ops.unpack_conv_weight(base.abs().double().view(9, 64, 3), 3)
    assert_bound(got, dref, dacc + base_abs, "input conv wgrad", rel=0.0)
    # run to run identical
    gw2 = torch.zeros_like(gw)
    ops.conv_wgrad(dev(dy), col, gw2, 1, 1)
    assert torch.equal(gw, gw2)


def test_input_conv_integer_exact(mcb, cuda):
    from mcb200 import ops
    n, h, w = 4, 64, 72
    g = torch.Generator(device=cuda).manual_seed(3)
    x = torch.randint(-2, 3, (n, 3, h, w), generator=g, device=cuda).float()
    wt = torch.randint(-1, 2, (64, 3, 3, 3), generator=g, device=cuda).float()
    bias = torch.randint(-2, 3, (64,), generator=g, device=cuda).float()
    col = ops.vgg_input_im2col(x)
    w16 = torch.empty(1, 64, 32, dtype=torch.bfloat16, device=cuda)
    ops.vgg_input_pack_weight(ops.pack_conv_weight(wt).reshape(-1).contiguous(), w16)
    y = ops.conv_fwd(col, w16, 1, 1, bias=bias, relu=True)
    ref = torch.relu(F.conv2d(x.double(), wt.double(), bias.double(), padding=1))
    assert_exact(nchw(y), ref, "input conv fwd")
    dy = torch.randint(-1, 2, (n, 64, h, w), generator=g, device=cuda).double()
    gw = torch.zeros(1, 64, 32, dtype=torch.float32, device=cuda)
    ops.conv_wgrad(dev(dy), col, gw, 1, 1)
    dw = torch.zeros(9 * 64 * 3, dtype=torch.float32, device=cuda)
    ops.vgg_input_unpack_wgrad(gw, dw)
    dref = torch.nn.grad.conv2d_weight(x.double(), wt.shape, dy, padding=1)
    assert torch.equal(ops.unpack_conv_weight(dw.view(9, 64, 3), 3).double(), dref)


def test_input_conv_rejects_bad_arguments(mcb, cuda):
    from mcb200 import _lib as L
    with pytest.raises(RuntimeError, match="null pointer"):
        L.fcall("mcb_vgg_input_im2col", None, None, 1, 8, 8)
    x = torch.zeros(1, 3, 8, 8, device=cuda)
    col = torch.zeros(1, 8, 8, 32, dtype=torch.bfloat16, device=cuda)
    with pytest.raises(RuntimeError, match="size"):
        L.fcall("mcb_vgg_input_im2col", x.data_ptr(), col.data_ptr(), 1, 0, 8)


# ---------------------------------------------------------------------------------------------------- 32 + 64 concat
def _concat_case(ops, cuda, n, h, w, cout, integer):
    c = dict(desc=(n, h, w, cout), n=n, h=h, w=w, c0=32, c1=64, cin=96, cout=cout, k=3)
    check = (lambda got, r, a, what, rel=0.0: assert_exact(got, r, what)) if integer else assert_bound
    # forward with bias + ReLU
    x, wt, b, ref, acc = fwd_ref(c, integer)
    assert pack(wt).shape == (9, cout, 96)
    bd = b.double().view(1, -1, 1, 1)
    y = run_fwd(c, x, wt, bias=b.to(cuda), relu=True)
    check(nchw(y), (ref + bd).clamp_min(0), acc + bd.abs(), "concat fwd")
    # the two segment data gradients, plain and with the producer's ReLU mask + bias gradient (channel sum)
    dy, wt, act, _, dx_ref, dx_acc = dgrad_ref(c, integer)
    w16, dyd = pack(wt), dev(dy)
    for lo, ch in ((0, 32), (32, 64)):
        seg, seg_acc, mask = dx_ref[:, lo:lo + ch], dx_acc[:, lo:lo + ch], dev(act[:, lo:lo + ch])
        dx = ops.conv_dgrad(dyd, w16, 3, 1, (h, w), cin=ch, ci_off=lo)
        assert dx.shape == (n, h, w, ch)
        check(nchw(dx), seg, seg_acc, "concat dgrad ci_off %d" % lo)
        sums = [torch.zeros(ch, dtype=torch.float32, device=cuda) for _ in range(2)]
        dxm = ops.conv_dgrad(dyd, w16, 3, 1, (h, w), cin=ch, ci_off=lo, relu_mask=mask, channel_sum=sums[0])
        ops.conv_dgrad(dyd, w16, 3, 1, (h, w), cin=ch, ci_off=lo, relu_mask=mask, channel_sum=sums[1])
        keep = (act[:, lo:lo + ch] > 0).double()
        check(nchw(dxm), seg * keep, seg_acc * keep, "concat dgrad masked ci_off %d" % lo)
        check_sums(sums[0], nchw(dxm), "concat dgrad channel sum", integer)
        assert_same(sums[0], sums[1], "concat dgrad channel sum")
    # the two segment weight gradients into one 96-wide dW
    x, dy, dw_ref, dw_acc = wgrad_ref(c, integer)
    dws = [torch.zeros(9, cout, 96, dtype=torch.float32, device=cuda) for _ in range(2)]
    for dw in dws:
        ops.conv_wgrad(dev(dy), dev(x[:, :32]), dw, 3, 1, ci_off=0)
        ops.conv_wgrad(dev(dy), dev(x[:, 32:]), dw, 3, 1, ci_off=32)
    check(ops.unpack_conv_weight(dws[0], 3), dw_ref, dw_acc, "concat wgrad", rel=0.0)
    assert_same(dws[0], dws[1], "concat wgrad")


CONCAT_SHAPES = [(2, 8, 8, 32), (3, 13, 7, 32), (1, 11, 20, 64), (2, 40, 48, 32)]


@pytest.mark.parametrize("n,h,w,cout", CONCAT_SHAPES)
def test_concat_32_64_real(mcb, cuda, n, h, w, cout):
    from mcb200 import ops
    _concat_case(ops, cuda, n, h, w, cout, integer=False)


@pytest.mark.parametrize("n,h,w,cout", [(2, 9, 14, 32), (1, 16, 16, 64)])
def test_concat_32_64_integer_exact(mcb, cuda, n, h, w, cout):
    from mcb200 import ops
    _concat_case(ops, cuda, n, h, w, cout, integer=True)


def test_concat_32_64_persistent(mcb, cuda):
    """dec1's shape class at full resolution: every CTA of the forward and the data gradients runs several tiles"""
    from mcb200 import ops
    n, h, w = 4, 128, 160
    assert_tiles_per_cta(tile_count(n, h, w, 32, None, any_box=True), 4)
    _concat_case(ops, cuda, n, h, w, 32, integer=False)


# ---------------------------------------------------------------------------------------------------- pool + skip
POOL_SHAPES = [(8, 320, 320, 64), (4, 160, 160, 128), (2, 40, 40, 256), (2, 20, 20, 512), (3, 6, 10, 64)]


@pytest.mark.parametrize("n,h,w,c", POOL_SHAPES)
def test_pool_skip_relu_integer_exact(mcb, cuda, n, h, w, c):
    from mcb200 import ops
    pooled = n * (h // 2) * (w // 2)
    grid, lanes = reduce_grid(pooled, c)
    if n * h * w * c >= 8 * 160 * 160 * 64:
        assert pooled / (grid * lanes) > 2               # every thread loops over several windows
    g = torch.Generator(device=cuda).manual_seed(n + h + c)
    # ReLU outputs in {0, 1, 2}: zeros (masked) and ties (first maximum) in most windows
    y = torch.randint(-2, 3, (n, c, h, w), generator=g, device=cuda).clamp_min(0).double()
    gskip = torch.randint(-4, 5, (n, c, h, w), generator=g, device=cuda).double()
    dpool = torch.randint(-4, 5, (n, c, h // 2, w // 2), generator=g, device=cuda).double()
    ref = nchw(pool_skip_ref(dev(y), dev(gskip), dev(dpool)))
    gd = dev(gskip)
    base = torch.randint(-8, 9, (c,), generator=g, device=cuda).float()
    db = base.clone()
    ops.maxpool2_bwd_skip_relu(dev(y), dev(dpool), gd, db)
    assert_exact(nchw(gd), ref, "pool skip")
    assert bool((nchw(gd)[y == 0] == 0).all())
    assert torch.equal(db.double(), base.double() + ref.sum(dim=(0, 2, 3), dtype=torch.float64))
    db2 = base.clone()
    gd2 = dev(gskip)
    ops.maxpool2_bwd_skip_relu(dev(y), dev(dpool), gd2, db2)
    assert torch.equal(gd, gd2) and torch.equal(db, db2)


@pytest.mark.parametrize("n,h,w,c", [(8, 320, 320, 64), (2, 40, 40, 512)])
def test_pool_skip_relu_real(mcb, cuda, n, h, w, c):
    """real values: g is the single bf16 rounding of the fp32 sum; the bias gradient sums the stored bf16 g"""
    from mcb200 import ops
    g = torch.Generator(device=cuda).manual_seed(c)
    y = bf16r(torch.relu(torch.randn(n, c, h, w, generator=g, device=cuda))).double()
    gskip = bf16r(torch.randn(n, c, h, w, generator=g, device=cuda)).double()
    dpool = bf16r(torch.randn(n, c, h // 2, w // 2, generator=g, device=cuda)).double()
    gd = dev(gskip)
    db = torch.zeros(c, dtype=torch.float32, device=cuda)
    ops.maxpool2_bwd_skip_relu(dev(y), dev(dpool), gd, db)
    assert torch.equal(gd, pool_skip_ref(dev(y), dev(gskip), dev(dpool)))   # the single rounding of the fp32 sum
    check_sums(db, nchw(gd), "pool skip bias gradient", False)
    db2 = torch.zeros_like(db)
    gd2 = dev(gskip)
    ops.maxpool2_bwd_skip_relu(dev(y), dev(dpool), gd2, db2)
    assert torch.equal(db, db2)


def test_pool_skip_relu_rejects_bad_arguments(mcb, cuda):
    from mcb200 import _lib as L
    from mcb200 import ops
    y = torch.zeros(1, 4, 4, 64, dtype=torch.bfloat16, device=cuda)
    g = torch.zeros_like(y)
    d = torch.zeros(1, 2, 2, 64, dtype=torch.bfloat16, device=cuda)
    db = torch.zeros(64, device=cuda)
    with pytest.raises(RuntimeError, match="null pointer"):
        L.fcall("mcb_maxpool2_bwd_skip_relu", y.data_ptr(), None, g.data_ptr(), db.data_ptr(), 1, 4, 4, 64)
    with pytest.raises(RuntimeError, match="alias"):
        L.fcall("mcb_maxpool2_bwd_skip_relu", y.data_ptr(), d.data_ptr(), y.data_ptr(), db.data_ptr(), 1, 4, 4, 64)
    with pytest.raises(AssertionError, match="alias"):
        ops.maxpool2_bwd_skip_relu(y, d, y, db)
    with pytest.raises(RuntimeError, match="size"):
        L.fcall("mcb_maxpool2_bwd_skip_relu", y.data_ptr(), d.data_ptr(), g.data_ptr(), db.data_ptr(), 1, 5, 4, 64)
    with pytest.raises(RuntimeError, match="channel"):
        L.fcall("mcb_maxpool2_bwd_skip_relu", y.data_ptr(), d.data_ptr(), g.data_ptr(), db.data_ptr(), 1, 4, 4, 60)
