"""The kernels the VGG-encoder U-Nets (UNet11, UNetVGG16; reference src/unet_models.py:56-106, :224-312) add to the
H100 path:
  * the full-resolution 3-channel input conv, Conv2d(3, 64, 3, padding 1) + bias + ReLU, as an im2col (27 of 32
    columns, k = (ky*3 + kx)*3 + c) + the 1x1 GEMM, with its weight gradient unpacked into the [9][64][3] master slot;
  * the 32 + 64-channel concat conv of dec1 (ConvRelu(96, 32) over cat[dec2, conv1]): forward, the two segment data
    gradients (ci_off 0 / cin 32 and ci_off 32 / cin 64 of a 96-wide weight) and the two segment weight gradients;
  * the max-pool backward of a stage output that also feeds a decoder concat (mcb_maxpool2_bwd_skip_relu).

References are float64 (on the device) from the bf16-rounded operands; A, the same op on |operands|, sets the
accumulation allowance: bf16 outputs |got - ref| <= 2^-8 |ref| + 2^-16 A, fp32 sums |got - ref| <= 2^-16 A.  Integer-
valued variants must match bit for bit.  Every case asserts its launch regime from the device's SM count."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).double()


def bf16r(x):
    return x.to(torch.bfloat16).double()


def dev16(t):
    return nhwc(t).to(torch.bfloat16)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def check_bf16(got, ref, acc, what):
    bad = (got - ref).abs() > ref.abs() * 2.0 ** -8 + acc * 2.0 ** -16
    assert not bool(bad.any()), (what, int(bad.sum()), float((got - ref).abs().max()))


def check_f32(got, ref, acc, what):
    bad = (got.double() - ref).abs() > acc * 2.0 ** -16
    assert not bool(bad.any()), (what, int(bad.sum()), float((got.double() - ref).abs().max()))


def conv_tiles(n, h, w):
    """lower bound of the implicit GEMM's 128-row pixel tiles"""
    return n * h * w // 128


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
        assert conv_tiles(n, h, w) >= 4 * sms()          # persistent: every CTA runs several pixel tiles
    if w % 64:
        assert w > 64 or n * h > 1                       # an im2col strip that the 64-pixel strip does not fill
    g = torch.Generator(device=cuda).manual_seed(n * 7 + h + w)
    x = torch.randn(n, 3, h, w, generator=g, device=cuda)
    col = ops.vgg_input_im2col(x)
    assert torch.equal(col.double(), _input_im2col_ref(bf16r(x)))      # border pixels and pad columns included
    wt = torch.randn(64, 3, 3, 3, generator=g, device=cuda) / 27 ** 0.5
    slot = ops.pack_conv_weight(wt).reshape(-1).contiguous()             # master layout [9][64][3]
    w16 = torch.empty(1, 64, 32, dtype=torch.bfloat16, device=cuda)
    ops.vgg_input_pack_weight(slot, w16)
    wref = torch.zeros(64, 32, dtype=torch.float64, device=cuda)
    wref[:, :27] = bf16r(wt).permute(0, 2, 3, 1).reshape(64, 27)
    assert torch.equal(w16[0].double(), wref)
    bias = torch.randn(64, generator=g, device=cuda) * 0.1
    y = ops.conv_fwd(col, w16, 1, 1, bias=bias, relu=True)
    xr, wr = bf16r(x), bf16r(wt)
    ref = torch.relu(F.conv2d(xr, wr, bias.double(), padding=1))
    acc = F.conv2d(xr.abs(), wr.abs(), bias.double().abs(), padding=1)
    check_bf16(nchw(y), ref, acc, "input conv fwd")
    # weight gradient: 1x1 wgrad over the im2col columns, then += into the master slot
    dy = bf16r(torch.randn(n, 64, h, w, generator=g, device=cuda))
    gw = torch.zeros(1, 64, 32, dtype=torch.float32, device=cuda)
    ops.conv_wgrad(dev16(dy), col, gw, 1, 1)
    assert bool((gw[0, :, 27:] == 0).all())
    base = torch.randn(9 * 64 * 3, generator=g, device=cuda)
    dw = base.clone()
    ops.vgg_input_unpack_wgrad(gw, dw)
    dref = torch.nn.grad.conv2d_weight(xr, wt.shape, dy, padding=1)
    dacc = torch.nn.grad.conv2d_weight(xr.abs(), wt.shape, dy.abs(), padding=1)
    got = ops.unpack_conv_weight((dw - base).view(9, 64, 3), 3)
    check_f32(got, dref, dacc + ops.unpack_conv_weight(base.abs().double().view(9, 64, 3), 3), "input conv wgrad")
    # run to run identical
    gw2 = torch.zeros_like(gw)
    ops.conv_wgrad(dev16(dy), col, gw2, 1, 1)
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
    assert torch.equal(nchw(y), ref)
    dy = torch.randint(-1, 2, (n, 64, h, w), generator=g, device=cuda).double()
    gw = torch.zeros(1, 64, 32, dtype=torch.float32, device=cuda)
    ops.conv_wgrad(dev16(dy), col, gw, 1, 1)
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
def _concat_operands(n, h, w, cout, cuda, seed, integer=False):
    g = torch.Generator(device=cuda).manual_seed(seed)
    if integer:
        rnd = lambda *s: torch.randint(-1, 2, s, generator=g, device=cuda).double()  # noqa: E731
        return rnd(n, 32, h, w), rnd(n, 64, h, w), rnd(cout, 96, 3, 3), rnd(cout), rnd(n, cout, h, w), \
            rnd(n, 32, h, w), rnd(n, 64, h, w)
    a = bf16r(torch.randn(n, 32, h, w, generator=g, device=cuda))
    b = bf16r(torch.randn(n, 64, h, w, generator=g, device=cuda))
    wt = bf16r(torch.randn(cout, 96, 3, 3, generator=g, device=cuda) / (96 * 9) ** 0.5)
    bias = torch.randn(cout, generator=g, device=cuda).float().double() * 0.1
    dy = bf16r(torch.randn(n, cout, h, w, generator=g, device=cuda))
    ma = bf16r(torch.randn(n, 32, h, w, generator=g, device=cuda))
    mb = bf16r(torch.randn(n, 64, h, w, generator=g, device=cuda))
    return a, b, wt, bias, dy, ma, mb


def _concat_case(ops, cuda, n, h, w, cout, seed, integer):
    a, b, wt, bias, dy, ma, mb = _concat_operands(n, h, w, cout, cuda, seed, integer)
    w16 = ops.pack_conv_weight(wt).to(torch.bfloat16)
    assert w16.shape == (9, cout, 96)
    x = torch.cat([a, b], 1)
    # forward with bias + ReLU
    y = ops.conv_fwd(dev16(a), w16, 3, 1, bias=bias.float(), relu=True, x2=dev16(b))
    ref = torch.relu(F.conv2d(x, wt, bias, padding=1))
    acc = F.conv2d(x.abs(), wt.abs(), bias.abs(), padding=1)
    if integer:
        assert torch.equal(nchw(y), ref)
    else:
        check_bf16(nchw(y), ref, acc, "concat fwd")
    # the two segment data gradients, plain and with the producer's ReLU mask + bias gradient (channel sum)
    dx_ref = torch.nn.grad.conv2d_input(x.shape, wt, dy, padding=1)
    dx_acc = torch.nn.grad.conv2d_input(x.shape, wt.abs(), dy.abs(), padding=1)
    for lo, c, mask in ((0, 32, ma), (32, 64, mb)):
        seg, seg_acc = dx_ref[:, lo:lo + c], dx_acc[:, lo:lo + c]
        dx = ops.conv_dgrad(dev16(dy), w16, 3, 1, (h, w), cin=c, ci_off=lo)
        assert dx.shape == (n, h, w, c)
        if integer:
            assert torch.equal(nchw(dx), seg), (lo, c)
        else:
            check_bf16(nchw(dx), seg, seg_acc, "concat dgrad ci_off %d" % lo)
        csum = torch.zeros(c, dtype=torch.float32, device=cuda)
        dxm = ops.conv_dgrad(dev16(dy), w16, 3, 1, (h, w), cin=c, ci_off=lo, relu_mask=dev16(mask), channel_sum=csum)
        keep = (mask > 0).double()
        stored = nchw(dxm)
        if integer:
            assert torch.equal(stored, seg * keep)
            assert torch.equal(csum.double(), stored.sum(dim=(0, 2, 3)))
        else:
            check_bf16(stored, seg * keep, seg_acc * keep, "concat dgrad masked ci_off %d" % lo)
            check_f32(csum, stored.sum(dim=(0, 2, 3)), stored.abs().sum(dim=(0, 2, 3)), "concat dgrad channel sum")
        csum2 = torch.zeros_like(csum)
        ops.conv_dgrad(dev16(dy), w16, 3, 1, (h, w), cin=c, ci_off=lo, relu_mask=dev16(mask), channel_sum=csum2)
        assert torch.equal(csum, csum2)
    # the two segment weight gradients into one 96-wide dW
    dw_ref = torch.nn.grad.conv2d_weight(x, wt.shape, dy, padding=1)
    dw_acc = torch.nn.grad.conv2d_weight(x.abs(), wt.shape, dy.abs(), padding=1)
    dw = torch.zeros(9, cout, 96, dtype=torch.float32, device=cuda)
    ops.conv_wgrad(dev16(dy), dev16(a), dw, 3, 1, ci_off=0)
    ops.conv_wgrad(dev16(dy), dev16(b), dw, 3, 1, ci_off=32)
    got = ops.unpack_conv_weight(dw, 3)
    if integer:
        assert torch.equal(got.double(), dw_ref)
    else:
        check_f32(got, dw_ref, dw_acc, "concat wgrad")
    dw2 = torch.zeros_like(dw)
    ops.conv_wgrad(dev16(dy), dev16(a), dw2, 3, 1, ci_off=0)
    ops.conv_wgrad(dev16(dy), dev16(b), dw2, 3, 1, ci_off=32)
    assert torch.equal(dw, dw2)


CONCAT_SHAPES = [(2, 8, 8, 32), (3, 13, 7, 32), (1, 11, 20, 64), (2, 40, 48, 32)]


@pytest.mark.parametrize("n,h,w,cout", CONCAT_SHAPES)
def test_concat_32_64_real(mcb, cuda, n, h, w, cout):
    from mcb200 import ops
    _concat_case(ops, cuda, n, h, w, cout, seed=n * 100 + h + w + cout, integer=False)


@pytest.mark.parametrize("n,h,w,cout", [(2, 9, 14, 32), (1, 16, 16, 64)])
def test_concat_32_64_integer_exact(mcb, cuda, n, h, w, cout):
    from mcb200 import ops
    _concat_case(ops, cuda, n, h, w, cout, seed=17 + h, integer=True)


def test_concat_32_64_persistent(mcb, cuda):
    """dec1's shape class at full resolution: every CTA of the forward and the data gradients runs several tiles"""
    from mcb200 import ops
    n, h, w = 4, 128, 160
    assert conv_tiles(n, h, w) >= 4 * sms()
    _concat_case(ops, cuda, n, h, w, 32, seed=5, integer=False)


# ---------------------------------------------------------------------------------------------------- pool + skip
def _pool_skip_ref(y, gskip, dpool):
    """float64 NCHW: g = (gskip + dpool routed to the first maximum of each window) * (y > 0)"""
    n, c, h, w = y.shape
    win = y.view(n, c, h // 2, 2, w // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, c, h // 2, w // 2, 4)
    first = F.one_hot(win.argmax(-1), 4).double()          # argmax returns the first maximal index
    routed = (first * dpool.unsqueeze(-1)).view(n, c, h // 2, w // 2, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(
        n, c, h, w)
    return (gskip + routed) * (y > 0).double()


def _pool_regime(n, h, w, c):
    """windows per thread of the capped grid (elementwise.cu reduce_cfg / mcb_maxpool2_bwd_skip_relu)"""
    c8 = c // 8
    threads = 256 - 256 % c8
    lanes = threads // c8
    pooled = n * (h // 2) * (w // 2)
    grid = max(1, min((pooled + lanes * 4 - 1) // (lanes * 4), sms() * 4))
    return pooled / (grid * lanes)


POOL_SHAPES = [(8, 320, 320, 64), (4, 160, 160, 128), (2, 40, 40, 256), (2, 20, 20, 512), (3, 6, 10, 64)]


@pytest.mark.parametrize("n,h,w,c", POOL_SHAPES)
def test_pool_skip_relu_integer_exact(mcb, cuda, n, h, w, c):
    from mcb200 import ops
    per = _pool_regime(n, h, w, c)
    if n * h * w * c >= 8 * 160 * 160 * 64:
        assert per > 2                                   # every thread loops over several windows
    g = torch.Generator(device=cuda).manual_seed(n + h + c)
    # ReLU outputs in {0, 1, 2}: zeros (masked) and ties (first maximum) in most windows
    y = torch.randint(-2, 3, (n, c, h, w), generator=g, device=cuda).clamp_min(0).double()
    gskip = torch.randint(-4, 5, (n, c, h, w), generator=g, device=cuda).double()
    dpool = torch.randint(-4, 5, (n, c, h // 2, w // 2), generator=g, device=cuda).double()
    ref = _pool_skip_ref(y, gskip, dpool)
    gd = dev16(gskip)
    base = torch.randint(-8, 9, (c,), generator=g, device=cuda).float()
    db = base.clone()
    ops.maxpool2_bwd_skip_relu(dev16(y), dev16(dpool), gd, db)
    assert torch.equal(nchw(gd), ref)
    assert bool((nchw(gd)[y == 0] == 0).all())
    assert torch.equal(db.double(), base.double() + ref.sum(dim=(0, 2, 3)))
    db2 = base.clone()
    gd2 = dev16(gskip)
    ops.maxpool2_bwd_skip_relu(dev16(y), dev16(dpool), gd2, db2)
    assert torch.equal(gd, gd2) and torch.equal(db, db2)


@pytest.mark.parametrize("n,h,w,c", [(8, 320, 320, 64), (2, 40, 40, 512)])
def test_pool_skip_relu_real(mcb, cuda, n, h, w, c):
    """real values: g is the single bf16 rounding of the fp32 sum; the bias gradient sums the stored bf16 g"""
    from mcb200 import ops
    g = torch.Generator(device=cuda).manual_seed(c)
    y = bf16r(torch.relu(torch.randn(n, c, h, w, generator=g, device=cuda)))
    gskip = bf16r(torch.randn(n, c, h, w, generator=g, device=cuda))
    dpool = bf16r(torch.randn(n, c, h // 2, w // 2, generator=g, device=cuda))
    ref = _pool_skip_ref(y, gskip, dpool)
    gd = dev16(gskip)
    db = torch.zeros(c, dtype=torch.float32, device=cuda)
    ops.maxpool2_bwd_skip_relu(dev16(y), dev16(dpool), gd, db)
    expect = nhwc(ref.float()).to(torch.bfloat16)        # fp32 sum of two bf16 values, one rounding
    assert torch.equal(gd, expect)
    stored = nchw(gd)
    check_f32(db, stored.sum(dim=(0, 2, 3)), stored.abs().sum(dim=(0, 2, 3)), "pool skip bias gradient")
    db2 = torch.zeros_like(db)
    gd2 = dev16(gskip)
    ops.maxpool2_bwd_skip_relu(dev16(y), dev16(dpool), gd2, db2)
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
