"""Unit parity of the HBM-bound kernels (csrc/elementwise.cu, csrc/loss.cu) against torch fp32 on the CPU — the ops
the reference runs through torch (BatchNorm2d, MaxPool2d, Conv2d 7x7 / 1x1, CrossEntropy/Dice losses, Adam).
The batch-32 sizes, where every thread of the capped grid-stride loops runs several iterations, are tested in
tests/test_elementwise_scale_gpu.py."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import synthetic
from oracle import unet_oracle as O
from oracle.conv_checks import bf16r, nchw, nhwc

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def close(got, ref, rtol=2 ** -7, atol=1e-3):
    got, ref = got.float().cpu(), ref.float().cpu()
    err = (got - ref).abs()
    assert bool((err <= rtol * ref.abs() + atol).all()), "max err %g at ref %g" % (
        float(err.max()), float(ref.flatten()[err.argmax()]))


def test_layout_conversions_roundtrip(mcb, cuda):
    from mcb200 import ops
    x = torch.randn(3, 24, 10, 14)
    y = ops.nchw_to_nhwc_bf16(x.to(cuda))
    assert torch.equal(y.cpu(), nhwc(x).to(BF))
    z = ops.nhwc_to_nchw_f32(y)
    assert torch.equal(z.cpu(), bf16r(x))


def test_stem_im2col_gemm_equals_conv7x7(mcb, cuda):
    from mcb200 import ops
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 3, 64, 96, generator=g)
    w = torch.randn(64, 3, 7, 7, generator=g) * 0.1
    ref = F.conv2d(bf16r(x), bf16r(w), None, stride=2, padding=3)
    col = ops.stem_im2col(x.to(cuda))
    master = w.permute(2, 3, 0, 1).contiguous().to(cuda)  # [7][7][64][3], the arena layout
    wp = torch.zeros(1, 64, 192, dtype=BF, device=cuda)
    ops.stem_pack_weight(master.view(-1), wp)
    y = ops.conv_fwd(col, wp, 1, 1)
    close(nchw(y), ref, atol=2e-2)
    # weight-gradient path: wgrad on the im2col matrix, unpacked to the master layout
    dy = bf16r(torch.randn(2, 64, 32, 48, generator=g))
    gref = torch.nn.grad.conv2d_weight(bf16r(x), (64, 3, 7, 7), dy, stride=2, padding=3)
    gw = torch.zeros(1, 64, 192, device=cuda)
    ops.conv_wgrad(nhwc(dy).to(cuda, BF), col, gw, 1, 1)
    gm = torch.zeros(49 * 64 * 3, device=cuda)
    ops.stem_unpack_wgrad(gw, gm)
    got = gm.view(7, 7, 64, 3).permute(2, 3, 0, 1).cpu()
    assert (got - gref).abs().max() < 2e-3 * gref.abs().max()


@pytest.mark.parametrize("c,n,h,w,residual", [(64, 2, 8, 8, None), (256, 3, 5, 7, "act"), (1024, 2, 4, 4, "bn"),
                                               (2048, 2, 2, 2, "act"), (128, 1, 16, 16, "bn")])
def test_batchnorm_train_forward_backward(mcb, cuda, c, n, h, w, residual):
    """stats (as the conv epilogue produces them) -> finalize -> apply(+residual)+ReLU; backward reduce + apply,
    against torch.batch_norm autograd on the same bf16-rounded z"""
    from mcb200 import ops
    g = torch.Generator().manual_seed(c + h)
    z = bf16r(torch.randn(n, c, h, w, generator=g) * 2 + 0.5)
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.1
    r = bf16r(torch.randn(n, c, h, w, generator=g)) if residual else None
    rgamma, rbeta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.1
    dy = bf16r(torch.randn(n, c, h, w, generator=g))
    # reference
    zr = z.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    rm, rv = torch.zeros(c), torch.ones(c)
    y = F.batch_norm(zr, rm, rv, gr, br, True, 0.1, 1e-5)
    rr = None
    if residual == "act":
        rr = r.clone().requires_grad_(True)
        y = y + rr
    elif residual == "bn":
        rr = r.clone().requires_grad_(True)
        y = y + F.batch_norm(rr, None, None, rgamma, rbeta, True, 0.1, 1e-5)
    out = F.relu(y)
    out.backward(dy)
    # CUDA
    zd = nhwc(z).to(cuda, BF)
    stats = torch.cat([z.sum(dim=(0, 2, 3)), (z * z).sum(dim=(0, 2, 3))]).to(cuda)
    count = n * h * w
    gm, bt = gamma.to(cuda), beta.to(cuda)
    rmd, rvd = torch.zeros(c, device=cuda), torch.ones(c, device=cuda)
    scale, shift, mean, invstd = (torch.empty(c, device=cuda) for _ in range(4))
    ops.bn_finalize(stats, count, gm, bt, rmd, rvd, scale, shift, mean, invstd)
    assert torch.allclose(rmd.cpu(), rm, rtol=1e-4, atol=1e-5) and torch.allclose(rvd.cpu(), rv, rtol=1e-4, atol=1e-5)
    yd = torch.empty_like(zd)
    if residual == "bn":
        rd = nhwc(r).to(cuda, BF)
        rstats = torch.cat([r.sum(dim=(0, 2, 3)), (r * r).sum(dim=(0, 2, 3))]).to(cuda)
        rs_, rsh_, rmean, rinv = (torch.empty(c, device=cuda) for _ in range(4))
        ops.bn_finalize(rstats, count, rgamma.to(cuda), rbeta.to(cuda), None, None, rs_, rsh_, rmean, rinv)
        ops.bn_apply(zd, scale, shift, yd, True, rd, rs_, rsh_)
    elif residual == "act":
        rd = nhwc(r).to(cuda, BF)
        ops.bn_apply(zd, scale, shift, yd, True, rd)
    else:
        ops.bn_apply(zd, scale, shift, yd, True)
    close(nchw(yd), out.detach(), atol=1e-2)
    # fused finalize + apply (what the training plan launches) == the two-step path
    rm2, rv2 = torch.zeros(c, device=cuda), torch.ones(c, device=cuda)
    mean2, inv2 = torch.empty(c, device=cuda), torch.empty(c, device=cuda)
    tr = ops.make_bn_train(stats, gm, bt, rm2, rv2, mean2, inv2)
    y2 = torch.empty_like(zd)
    if residual == "bn":
        rg, rbt = rgamma.to(cuda), rbeta.to(cuda)
        rmean2, rinv2 = torch.empty(c, device=cuda), torch.empty(c, device=cuda)
        rtr = ops.make_bn_train(rstats, rg, rbt, None, None, rmean2, rinv2)
        ops.bn_train_apply(zd, tr, y2, True, rd, rtr)
        assert torch.allclose(rmean2, rmean) and torch.allclose(rinv2, rinv)
    elif residual == "act":
        ops.bn_train_apply(zd, tr, y2, True, rd)
    else:
        ops.bn_train_apply(zd, tr, y2, True)
    assert torch.equal(y2, yd)
    assert torch.allclose(mean2, mean) and torch.allclose(inv2, invstd)
    assert torch.allclose(rm2, rmd) and torch.allclose(rv2, rvd)
    # backward (mask from the stored bf16 output, like the plan does)
    dyd = nhwc(dy).to(cuda, BF)
    dbeta, dgamma = torch.zeros(c, device=cuda), torch.zeros(c, device=cuda)
    ops.bn_bwd_reduce(dyd, yd, zd, mean, invstd, dbeta, dgamma)
    dz = torch.empty_like(zd)
    g_out = torch.zeros_like(zd) if residual == "act" else None
    ops.bn_bwd_apply(dyd, yd, zd, mean, invstd, gm, dbeta, dgamma, dz, g_out, False)
    mask_ref = (out.detach() > 0)
    mask_got = nchw(yd).float().cpu() > 0
    agree = (mask_ref == mask_got)
    assert agree.float().mean() > 0.995  # outputs within a bf16 ulp of 0 may flip
    tolc = 3e-2 * float(gr.grad.abs().max()) + 1e-2
    assert (dgamma.cpu() - gr.grad).abs().max() < tolc * max(1.0, math.sqrt(count) / 4)
    assert (dbeta.cpu() - br.grad).abs().max() < tolc * max(1.0, math.sqrt(count) / 4)
    err = (nchw(dz).float().cpu() - zr.grad).abs()
    assert float((err * agree).max()) < 3e-2 * float(zr.grad.abs().max()) + 1e-2
    if residual == "act":
        errg = (nchw(g_out).float().cpu() - rr.grad).abs() * agree
        assert float(errg.max()) < 1e-2 * float(rr.grad.abs().max()) + 1e-3
        # accumulate mode adds on top
        ops.bn_bwd_apply(dyd, yd, zd, mean, invstd, gm, dbeta, dgamma, dz, g_out, True)
        errg2 = (nchw(g_out).float().cpu() - 2 * rr.grad).abs() * agree
        assert float(errg2.max()) < 3e-2 * float(rr.grad.abs().max()) + 1e-3


def test_batchnorm_eval_params(mcb, cuda):
    from mcb200 import ops
    c = 128
    g = torch.Generator().manual_seed(1)
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g)
    rm, rv = torch.randn(c, generator=g), torch.rand(c, generator=g) + 0.2
    z = bf16r(torch.randn(2, c, 6, 6, generator=g))
    ref = F.relu(F.batch_norm(z, rm, rv, gamma, beta, False, 0.1, 1e-5))
    scale, shift = torch.empty(c, device=cuda), torch.empty(c, device=cuda)
    ops.bn_eval_params(gamma.to(cuda), beta.to(cuda), rm.to(cuda), rv.to(cuda), scale, shift)
    zd = nhwc(z).to(cuda, BF)
    y = ops.bn_apply(zd, scale, shift, torch.empty_like(zd), True)
    close(nchw(y), ref)


def test_maxpool_forward_backward_with_ties(mcb, cuda):
    from mcb200 import ops
    g = torch.Generator().manual_seed(2)
    x = F.relu(bf16r(torch.randn(2, 64, 12, 20, generator=g)))  # many exact zeros -> ties inside windows
    x[0, :, 0:2, 0:2] = 1.5                                       # a fully tied window
    xr = x.clone().requires_grad_(True)
    y = F.max_pool2d(xr, 2, 2)
    dy = bf16r(torch.randn(y.shape, generator=g))
    y.backward(dy)
    xd = nhwc(x).to(cuda, BF)
    yd = ops.maxpool2_fwd(xd)
    assert torch.equal(nchw(yd).float().cpu(), y.detach())
    dx = torch.zeros_like(xd)
    ops.maxpool2_bwd(xd, nhwc(dy).to(cuda, BF), dx, False)
    assert torch.equal(nchw(dx).float().cpu(), xr.grad)
    ops.maxpool2_bwd(xd, nhwc(dy).to(cuda, BF), dx, True)
    close(nchw(dx), 2 * xr.grad, rtol=2 ** -7, atol=1e-6)


@pytest.mark.parametrize("c", [32, 64, 512, 2048])
def test_channel_sum(mcb, cuda, c):
    from mcb200 import ops
    x = bf16r(torch.randn(3, c, 9, 11))
    out = torch.zeros(c, device=cuda)
    ops.channel_sum(nhwc(x).to(cuda, BF), out)
    assert torch.allclose(out.cpu(), x.sum(dim=(0, 2, 3)), rtol=1e-4, atol=1e-3)


def test_final_conv_forward_backward(mcb, cuda):
    from mcb200 import ops
    g = torch.Generator().manual_seed(3)
    x = F.relu(bf16r(torch.randn(2, 32, 24, 40, generator=g)))
    w, b = torch.randn(2, 32, generator=g) * 0.2, torch.randn(2, generator=g)
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    y = F.conv2d(xr, wr.view(2, 32, 1, 1), br)
    dl = torch.randn(y.shape, generator=g)
    y.backward(dl)
    xd = nhwc(x).to(cuda, BF)
    logits = torch.empty(2, 2, 24, 40, device=cuda)
    ops.final_conv_fwd(xd, w.to(cuda).view(-1), b.to(cuda), logits)
    assert torch.allclose(logits.cpu(), y.detach(), rtol=1e-5, atol=1e-5)
    dx, dw, db = torch.empty_like(xd), torch.zeros(64, device=cuda), torch.zeros(2, device=cuda)
    ops.final_conv_bwd(xd, w.to(cuda).view(-1), dl.to(cuda), dx, dw, db)
    close(nchw(dx), xr.grad * (x > 0), atol=1e-3)
    assert torch.allclose(dw.cpu().view(2, 32), wr.grad, rtol=1e-4, atol=1e-3)
    assert torch.allclose(db.cpu(), br.grad, rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("n,s", [(2, 64), (3, 96)])
def test_loss_kernels_match_reference_formulas(mcb, cuda, n, s):
    from mcb200 import models, ops
    _, t = synthetic.train_batch(n, s, seed=s, n_rect=7)
    T = torch.from_numpy(t)
    logits = torch.randn(n, 2, s, s) * 2
    lr = logits.clone().requires_grad_(True)
    ref = O.mixed_loss(lr, T, imsize=(256, 256))
    ref.backward()
    lg = logits.to(cuda).requires_grad_(True)
    loss = models.mixed_dice_cross_entropy_loss(lg, T.to(cuda), dice_weight=0.2, cross_entropy_weight=1.0, smooth=1,
                                                w0=50, sigma=10, imsize=(256, 256))
    loss.backward()
    assert abs(float(loss) - float(ref)) < 1e-5 * abs(float(ref))
    assert torch.allclose(lg.grad.cpu(), lr.grad, rtol=1e-3, atol=1e-9)
    # plain CE (PyTorchUNet)
    lr2 = logits.clone().requires_grad_(True)
    ref2 = O.plain_ce_loss(lr2, T[:, :1])
    ref2.backward()
    lg2 = logits.to(cuda).requires_grad_(True)
    l2 = models.multiclass_segmentation_loss(lg2, T[:, :1].contiguous().to(cuda))
    l2.backward()
    assert abs(float(l2) - float(ref2)) < 1e-5 * abs(float(ref2))
    assert torch.allclose(lg2.grad.cpu(), lr2.grad, rtol=1e-3, atol=1e-10)
    # softmax used by transform()
    p = ops.softmax2(logits.to(cuda))
    assert torch.allclose(p.cpu(), torch.softmax(logits, 1), rtol=1e-5, atol=1e-7)


def test_adam_matches_torch_optim(mcb, cuda):
    from mcb200 import ops
    g = torch.Generator().manual_seed(4)
    p0 = torch.randn(10007, generator=g)
    p_ref = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p_ref], lr=5e-4, weight_decay=1e-4)
    p = p0.to(cuda)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    p16 = torch.empty(p.numel(), dtype=BF, device=cuda)
    for step in range(1, 6):
        grad = torch.randn(10007, generator=g) * (0.1 ** step)
        p_ref.grad = grad.clone()
        opt.step()
        ops.adam_step(p, grad.to(cuda), m, v, p16, step, 5e-4, (0.9, 0.999), 1e-8, 1e-4)
        assert torch.allclose(p.cpu(), p_ref.detach(), rtol=1e-5, atol=1e-7), step
    assert torch.equal(p16.cpu(), p.cpu().to(BF))
