"""The 3x3 transposed conv of the UNet11 decoder (nn.ConvTranspose2d(kernel_size=3, stride=2, padding=1,
output_padding=1), reference src/unet_models.py:42-53) through mcb_convt_{fwd,dgrad,wgrad} with ksize = 3.

References are float64 on the CPU from the bf16-rounded operands; A, the same op on |operands|, sets the accumulation
allowance: bf16 outputs |got - ref| <= 2^-8 |ref| + 2^-16 A, fp32 dW |got - ref| <= 2^-16 A.  Integer-exact variants
(operands in {-1, 0, 1}, |ref| <= 256) must match bit for bit.  Shapes cover ragged tiles (sides that are not tile
multiples, where the d=+1 tap of output parity 1 reads the zero row past the edge) and a persistent launch in which
every CTA runs at least two tiles."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).double().cpu()


def bf16r(x):
    return x.to(torch.bfloat16).double()


def convt3(x, w):
    return F.conv_transpose2d(x, w, stride=2, padding=1, output_padding=1)


def convt3_grads(x, w, dy):
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    convt3(xr, wr).backward(dy)
    return xr.grad, wr.grad


def check_bf16(got, ref, acc, what):
    bad = (got - ref).abs() > ref.abs() * 2.0 ** -8 + acc * 2.0 ** -16
    assert not bool(bad.any()), (what, int(bad.sum()), float((got - ref).abs().max()))


def _operands(n, h, w, cin, cout, seed, integer=False):
    g = torch.Generator().manual_seed(seed)
    if integer:
        rnd = lambda *s: torch.randint(-1, 2, s, generator=g).double()  # noqa: E731
        return rnd(n, cin, h, w), rnd(cin, cout, 3, 3), rnd(n, cout, 2 * h, 2 * w), rnd(n, cin, h, w)
    x = bf16r(torch.randn(n, cin, h, w, generator=g))
    wt = bf16r(torch.randn(cin, cout, 3, 3, generator=g) / (cin * 2.25) ** 0.5)
    dy = bf16r(torch.randn(n, cout, 2 * h, 2 * w, generator=g))
    act = bf16r(torch.randn(n, cin, h, w, generator=g))
    return x, wt, dy, act


def _dev(t, cuda):
    return nhwc(t).to(cuda, torch.bfloat16)


SHAPES = [(2, 8, 8, 64, 32), (3, 13, 7, 32, 64), (1, 11, 20, 128, 64), (2, 10, 10, 256, 128)]


@pytest.mark.parametrize("n,h,w,cin,cout", SHAPES)
def test_convt3_forward_dgrad_wgrad(mcb, cuda, n, h, w, cin, cout):
    from mcb200 import ops
    x, wt, dy, act = _operands(n, h, w, cin, cout, seed=n * 1000 + h * 10 + cin)
    wp = ops.pack_convt_weight(wt).to(cuda, torch.bfloat16)
    assert wp.shape == (9, cout, cin)
    g = torch.Generator().manual_seed(7)
    bias = torch.randn(cout, generator=g) * 0.1
    # forward, bias + ReLU epilogue
    ref = torch.relu(convt3(x, wt) + bias.double().view(1, -1, 1, 1))
    acc = convt3(x.abs(), wt.abs()) + bias.double().abs().view(1, -1, 1, 1)
    y = ops.convt_fwd(_dev(x, cuda), wp, bias=bias.to(cuda), relu=True)
    assert y.shape == (n, 2 * h, 2 * w, cout)
    check_bf16(nchw(y), ref, acc, "convt3 fwd")
    # data gradient, plain and with the producer's ReLU mask + its bias gradient (channel sum of the stored dx)
    dx_ref, dw_ref = convt3_grads(x, wt, dy)
    dx_acc, dw_acc = convt3_grads(x.abs(), wt.abs(), dy.abs())
    dx = ops.convt_dgrad(_dev(dy, cuda), wp)
    check_bf16(nchw(dx), dx_ref, dx_acc, "convt3 dgrad")
    csum = torch.zeros(cin, dtype=torch.float32, device=cuda)
    dxm = ops.convt_dgrad(_dev(dy, cuda), wp, relu_mask=_dev(act, cuda), channel_sum=csum)
    mask = (act > 0).double()
    check_bf16(nchw(dxm), dx_ref * mask, dx_acc * mask, "convt3 dgrad masked")
    stored = nchw(dxm)
    assert torch.allclose(csum.double().cpu(), stored.sum(dim=(0, 2, 3)), rtol=1e-5,
                          atol=1e-5 * float(stored.abs().sum(dim=(0, 2, 3)).max()))
    # accumulate onto an existing gradient
    base = bf16r(torch.randn(n, cin, h, w, generator=g))
    dxa = _dev(base, cuda)
    ops.convt_dgrad(_dev(dy, cuda), wp, accumulate=True, out=dxa)
    # two bf16 roundings (<= 2^-8 relative each): the gradient is rounded, then the reduce-add rounds base + that
    got, want = nchw(dxa), base + dx_ref
    bound = dx_ref.abs() * 2.0 ** -8 + (want.abs() + dx_ref.abs() * 2.0 ** -8) * 2.0 ** -8 + dx_acc * 2.0 ** -16
    bad = (got - want).abs() > bound
    assert not bool(bad.any()), ("convt3 dgrad accumulate", int(bad.sum()), float((got - want).abs().max()))
    # weight gradient added to a random dW
    dw0 = torch.randn(9, cout, cin, generator=g)
    dw = dw0.to(cuda)
    ops.convt_wgrad(_dev(dy, cuda), _dev(x, cuda), dw)
    got = ops.unpack_convt_weight(dw.cpu(), 3).double()
    want = ops.unpack_convt_weight(dw0, 3).double() + dw_ref
    tol = (ops.unpack_convt_weight(dw0.abs(), 3).double() + dw_acc) * 2.0 ** -16 + 1e-30
    assert bool(((got - want).abs() <= tol).all()), float((got - want).abs().max())


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 9, 6, 64, 32), (2, 16, 16, 128, 64)])
def test_convt3_integer_exact(mcb, cuda, n, h, w, cin, cout):
    """operands in {-1, 0, 1}: every output, the channel sums and dW are exact in fp32 and bf16"""
    from mcb200 import ops
    x, wt, dy, act = _operands(n, h, w, cin, cout, seed=3, integer=True)
    wp = ops.pack_convt_weight(wt).to(cuda, torch.bfloat16)
    ref = convt3(x, wt)
    assert float(ref.abs().max()) <= 256
    assert torch.equal(nchw(ops.convt_fwd(_dev(x, cuda), wp)), ref)
    dx_ref, dw_ref = convt3_grads(x, wt, dy)
    assert float(dx_ref.abs().max()) <= 256 and float(dw_ref.abs().max()) < 2 ** 23
    csum = torch.zeros(cin, dtype=torch.float32, device=cuda)
    dxm = ops.convt_dgrad(_dev(dy, cuda), wp, relu_mask=_dev(act, cuda), channel_sum=csum)
    masked = dx_ref * (act > 0).double()
    assert torch.equal(nchw(dxm), masked)
    assert torch.equal(csum.double().cpu(), masked.sum(dim=(0, 2, 3)))
    dw0 = torch.randint(-4, 5, (9, cout, cin)).float()
    dw = dw0.to(cuda)
    ops.convt_wgrad(_dev(dy, cuda), _dev(x, cuda), dw)
    assert torch.equal(ops.unpack_convt_weight(dw.cpu(), 3).double(), ops.unpack_convt_weight(dw0, 3).double() + dw_ref)


def test_convt3_persistent_multi_tile(mcb, cuda):
    """enough tiles that every CTA of the persistent grid runs at least two (ceil(pixels / 128) x N tiles x phases is a
    lower bound of the tile count), so the TMA ring, the output-buffer rotation and the phase walk carry across tiles;
    the fused channel sum and the split-K weight gradient must give the same bits twice"""
    from mcb200 import ops
    n, h, w, cin, cout = 16, 48, 48, 128, 64
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    m_tiles = -(-n * h * w // 128)
    assert m_tiles * 4 >= 2 * sms and m_tiles * max(1, cin // 256) >= 2 * sms
    x, wt, dy, act = _operands(n, h, w, cin, cout, seed=11)
    wp = ops.pack_convt_weight(wt).to(cuda, torch.bfloat16)
    y = ops.convt_fwd(_dev(x, cuda), wp)
    check_bf16(nchw(y), convt3(x, wt), convt3(x.abs(), wt.abs()), "convt3 fwd persistent")
    dx_ref, dw_ref = convt3_grads(x, wt, dy)
    dx_acc, dw_acc = convt3_grads(x.abs(), wt.abs(), dy.abs())
    mask = (act > 0).double()
    sums, dws = [], []
    for _ in range(2):
        csum = torch.zeros(cin, dtype=torch.float32, device=cuda)
        dxm = ops.convt_dgrad(_dev(dy, cuda), wp, relu_mask=_dev(act, cuda), channel_sum=csum)
        dw = torch.zeros(9, cout, cin, dtype=torch.float32, device=cuda)
        ops.convt_wgrad(_dev(dy, cuda), _dev(x, cuda), dw)
        sums.append(csum.cpu())
        dws.append(dw.cpu())
    check_bf16(nchw(dxm), dx_ref * mask, dx_acc * mask, "convt3 dgrad persistent")
    got = ops.unpack_convt_weight(dws[0], 3).double()
    assert bool(((got - dw_ref).abs() <= dw_acc * 2.0 ** -16 + 1e-30).all()), float((got - dw_ref).abs().max())
    assert torch.equal(sums[0], sums[1]) and torch.equal(dws[0], dws[1])


def test_convt_ksize_zero_means_four(mcb, cuda):
    """a zeroed ksize field keeps the 4x4 kernel: the ABI of existing callers is unchanged"""
    from mcb200 import _lib as L
    from mcb200 import ops
    g = torch.Generator().manual_seed(5)
    x = bf16r(torch.randn(1, 64, 6, 6, generator=g))
    wt = bf16r(torch.randn(64, 32, 4, 4, generator=g) / 16)
    wp = ops.pack_convt_weight(wt).to(cuda, torch.bfloat16)
    xd = _dev(x, cuda)
    y = torch.empty(1, 12, 12, 32, dtype=torch.bfloat16, device=cuda)
    a = L.ConvtFwdArgs()
    a.x = xd.data_ptr(); a.n, a.h, a.w, a.cin = 1, 6, 6, 64
    a.weight = wp.data_ptr(); a.cout = 32; a.y = y.data_ptr()
    assert a.ksize == 0
    L.call("mcb_convt_fwd", a)
    assert torch.equal(y, ops.convt_fwd(xd, wp))
    ref = F.conv_transpose2d(x, wt, stride=2, padding=1)
    check_bf16(nchw(y), ref, F.conv_transpose2d(x.abs(), wt.abs(), stride=2, padding=1), "convt4 fwd")
    a.ksize = 5
    with pytest.raises(RuntimeError, match="ksize"):
        L.call("mcb_convt_fwd", a)
