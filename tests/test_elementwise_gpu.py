"""The HBM-bound kernels (csrc/elementwise.cu, csrc/loss.cu) at small shapes, against the float64 references and bars
of oracle/elementwise_checks.py (the stem's im2col GEMM against oracle/conv_checks.py's); the losses through autograd
and Adam over several steps against torch.  The batch-32 sizes, where every thread of the capped grid-stride loops
runs several iterations, are tested in tests/test_elementwise_scale_gpu.py."""
import pytest
import torch
import torch.nn.functional as F

from oracle import synthetic
from oracle import unet_oracle as O
from oracle.conv_checks import assert_bound, assert_exact, bf16r, nchw, nhwc
from oracle.elementwise_checks import (EPS, F64, affine, assert_bf16, bn_apply_ref, bn_bwd_reduce_ref, check_bn_apply,
                                       check_bn_bwd_apply, check_fin, classifier_bwd_ref, classifier_fwd_ref, pool_ref)

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def assert_sum(got, ref, absref, what, rtol, atol):
    """an fp32 sum at these small shapes: the harness bar, 2^-16 A, and the rtol |ref| + atol bound these tests have
    held since they compared with torch, now against the float64 reference; each element meets the tighter of the two"""
    assert_bound(got, ref, absref, what, rel=0.0)
    assert_bound(got, ref, 0.0, what, rel=rtol, extra=atol)


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
    xr, wr = bf16r(x).double(), bf16r(w).double()
    conv = lambda a, v: F.conv2d(a, v, stride=2, padding=3)
    col = ops.stem_im2col(x.to(cuda))
    master = w.permute(2, 3, 0, 1).contiguous().to(cuda)  # [7][7][64][3], the arena layout
    wp = torch.zeros(1, 64, 192, dtype=BF, device=cuda)
    ops.stem_pack_weight(master.view(-1), wp)
    y = ops.conv_fwd(col, wp, 1, 1)
    assert_bound(nchw(y), conv(xr, wr), conv(xr.abs(), wr.abs()), "stem conv_fwd")
    # weight-gradient path: wgrad on the im2col matrix, unpacked to the master layout
    dy = bf16r(torch.randn(2, 64, 32, 48, generator=g))
    wg = lambda a, d: torch.nn.grad.conv2d_weight(a, (64, 3, 7, 7), d.double(), stride=2, padding=3)
    gw = torch.zeros(1, 64, 192, device=cuda)
    ops.conv_wgrad(nhwc(dy).to(cuda, BF), col, gw, 1, 1)
    gm = torch.zeros(49 * 64 * 3, device=cuda)
    ops.stem_unpack_wgrad(gw, gm)
    got = gm.view(7, 7, 64, 3).permute(2, 3, 0, 1).cpu()
    assert_bound(got, wg(xr, dy), wg(xr.abs(), dy.abs()), "stem wgrad", rel=0.0)


@pytest.mark.parametrize("c,n,h,w,residual", [(64, 2, 8, 8, None), (256, 3, 5, 7, "act"), (1024, 2, 4, 4, "bn"),
                                               (2048, 2, 2, 2, "act"), (128, 1, 16, 16, "bn")])
def test_batchnorm_train_forward_backward(mcb, cuda, c, n, h, w, residual):
    """stats (as the conv epilogue produces them) -> finalize -> apply(+residual)+ReLU, the fused finalize + apply
    bitwise equal to the two steps; backward reduce + apply, the mask from the stored bf16 output as the plan does"""
    from mcb200 import ops
    g = torch.Generator().manual_seed(c + h)
    z = bf16r(torch.randn(n, c, h, w, generator=g) * 2 + 0.5)
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.1
    r = bf16r(torch.randn(n, c, h, w, generator=g)) if residual else None
    rgamma, rbeta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.1
    dy = bf16r(torch.randn(n, c, h, w, generator=g))
    zd = nhwc(z).to(cuda, BF)
    stats = torch.cat([z.sum(dim=(0, 2, 3)), (z * z).sum(dim=(0, 2, 3))]).to(cuda)
    count = n * h * w
    gm, bt, rg, rbt = gamma.to(cuda), beta.to(cuda), rgamma.to(cuda), rbeta.to(cuda)
    rm0, rv0 = torch.zeros(c, device=cuda), torch.ones(c, device=cuda)
    rmd, rvd = rm0.clone(), rv0.clone()
    scale, shift, mean, invstd = (torch.empty(c, device=cuda) for _ in range(4))
    ops.bn_finalize(stats, count, gm, bt, rmd, rvd, scale, shift, mean, invstd)
    check_fin(dict(mean=mean, invstd=invstd, rm=rmd, rv=rvd), stats, count, rm0, rv0, "bn_finalize")
    rd = nhwc(r).to(cuda, BF) if residual else None
    rs_ = rsh_ = rbn = None
    if residual == "bn":
        rstats = torch.cat([r.sum(dim=(0, 2, 3)), (r * r).sum(dim=(0, 2, 3))]).to(cuda)
        rs_, rsh_, rmean, rinv = (torch.empty(c, device=cuda) for _ in range(4))
        ops.bn_finalize(rstats, count, rg, rbt, None, None, rs_, rsh_, rmean, rinv)
        check_fin(dict(mean=rmean, invstd=rinv), rstats, count, rm0, rv0, "bn_finalize residual BN")
        rbn = affine(rg, rbt, rmean, rinv)
    yd = torch.empty_like(zd)
    ops.bn_apply(zd, scale, shift, yd, True, rd, rs_, rsh_)
    # against gamma, beta and the checked mean / invstd: bn_finalize's scale and shift are checked through yd
    check_bn_apply(yd, zd, affine(gm, bt, mean, invstd), True, "bn_apply", rd, rbn)
    # fused finalize + apply (what the training plan launches) == the two-step path
    rm2, rv2 = rm0.clone(), rv0.clone()
    mean2, inv2 = torch.empty(c, device=cuda), torch.empty(c, device=cuda)
    tr = ops.make_bn_train(stats, gm, bt, rm2, rv2, mean2, inv2)
    rtr = None
    if residual == "bn":
        rmean2, rinv2 = torch.empty(c, device=cuda), torch.empty(c, device=cuda)
        rtr = ops.make_bn_train(rstats, rg, rbt, None, None, rmean2, rinv2)   # keeps pointers: rg, rbt stay alive
    y2 = torch.empty_like(zd)
    ops.bn_train_apply(zd, tr, y2, True, rd, rtr)
    assert torch.equal(y2, yd)
    check_fin(dict(mean=mean2, invstd=inv2, rm=rm2, rv=rv2), stats, count, rm0, rv0, "bn_train_apply")
    if residual == "bn":
        check_fin(dict(mean=rmean2, invstd=rinv2), rstats, count, rm0, rv0, "bn_train_apply residual BN")
    # backward
    dyd = nhwc(dy).to(cuda, BF)
    dbeta, dgamma = torch.zeros(c, device=cuda), torch.zeros(c, device=cuda)
    ops.bn_bwd_reduce(dyd, yd, zd, mean, invstd, dbeta, dgamma)
    sb, sg, ab, ag = bn_bwd_reduce_ref(dyd, yd, zd, mean, invstd)
    assert_bound(dbeta, sb, ab, "bn_bwd_reduce dbeta", rel=0.0)
    assert_bound(dgamma, sg, ag, "bn_bwd_reduce dgamma", rel=0.0)
    dz = torch.empty_like(zd)
    g_out = torch.zeros_like(zd) if residual == "act" else None
    ops.bn_bwd_apply(dyd, yd, zd, mean, invstd, gm, dbeta, dgamma, dz, g_out, False)
    check_bn_bwd_apply(dz, dyd, yd, zd, mean, invstd, gm, dbeta, dgamma, count, "bn_bwd_apply dz")
    if residual == "act":
        gref = dyd.masked_fill(yd <= 0, 0)
        assert_exact(g_out, gref, "bn_bwd_apply g_out")
        # accumulate mode adds on top
        ops.bn_bwd_apply(dyd, yd, zd, mean, invstd, gm, dbeta, dgamma, dz, g_out, True)
        assert_exact(g_out, (2 * gref.float()).to(BF), "bn_bwd_apply g_out accumulate")


def test_batchnorm_eval_params(mcb, cuda):
    from mcb200 import ops
    c = 128
    g = torch.Generator().manual_seed(1)
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g)
    rm, rv = torch.randn(c, generator=g), torch.rand(c, generator=g) + 0.2
    z = bf16r(torch.randn(2, c, 6, 6, generator=g))
    scale, shift = torch.empty(c, device=cuda), torch.empty(c, device=cuda)
    ops.bn_eval_params(gamma.to(cuda), beta.to(cuda), rm.to(cuda), rv.to(cuda), scale, shift)
    zd = nhwc(z).to(cuda, BF)
    y = ops.bn_apply(zd, scale, shift, torch.empty_like(zd), True)
    ref, a = bn_apply_ref(zd, affine(gamma, beta, rm, (rv.double() + EPS).rsqrt()), True)
    assert_bf16(y, ref, a, "bn_eval_params + bn_apply")


def test_maxpool_forward_backward_with_ties(mcb, cuda):
    from mcb200 import ops
    g = torch.Generator().manual_seed(2)
    x = F.relu(bf16r(torch.randn(2, 64, 12, 20, generator=g)))  # many exact zeros -> ties inside windows
    x[0, :, 0:2, 0:2] = 1.5                                       # a fully tied window
    dy = bf16r(torch.randn(2, 64, 6, 10, generator=g))
    xd, dyd = nhwc(x).to(cuda, BF), nhwc(dy).to(cuda, BF)
    m, routed = pool_ref(xd, dyd)
    assert_exact(ops.maxpool2_fwd(xd), m, "maxpool2_fwd")
    dx = torch.zeros_like(xd)
    ops.maxpool2_bwd(xd, dyd, dx, False)
    assert_exact(dx, routed, "maxpool2_bwd store")
    ops.maxpool2_bwd(xd, dyd, dx, True)
    assert_exact(dx, (2 * routed.float()).to(BF), "maxpool2_bwd accumulate")


@pytest.mark.parametrize("c", [32, 64, 512, 2048])
def test_channel_sum(mcb, cuda, c):
    from mcb200 import ops
    x = bf16r(torch.randn(3, c, 9, 11))
    out = torch.zeros(c, device=cuda)
    xd = nhwc(x).to(cuda, BF)
    ops.channel_sum(xd, out)
    v = xd.view(-1, c)
    assert_sum(out, v.sum(0, dtype=F64), v.abs().sum(0, dtype=F64), "channel_sum", 1e-4, 1e-3)


def test_final_conv_forward_backward(mcb, cuda):
    from mcb200 import ops
    g = torch.Generator().manual_seed(3)
    x = F.relu(bf16r(torch.randn(2, 32, 24, 40, generator=g)))
    w, b = torch.randn(2, 32, generator=g) * 0.2, torch.randn(2, generator=g)
    dl = torch.randn(2, 2, 24, 40, generator=g)
    xd = nhwc(x).to(cuda, BF)
    logits = torch.empty(2, 2, 24, 40, device=cuda)
    ops.final_conv_fwd(xd, w.to(cuda).view(-1), b.to(cuda), logits)
    lg, la = classifier_fwd_ref(xd, w, b)
    assert_sum(logits, lg, la, "final_conv_fwd", 1e-5, 1e-5)
    dx, dw, db = torch.empty_like(xd), torch.zeros(64, device=cuda), torch.zeros(2, device=cuda)
    ops.final_conv_bwd(xd, w.to(cuda).view(-1), dl.to(cuda), dx, dw, db)
    gx, ga, sw, aw, sb, ab = classifier_bwd_ref(xd, w, dl)
    assert_bf16(dx, gx, ga, "final_conv_bwd dx")
    assert_sum(dw, sw, aw, "final_conv_bwd dW", 1e-4, 1e-3)
    assert_sum(db, sb, ab, "final_conv_bwd db", 1e-4, 1e-3)


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
    p = torch.softmax(logits.double(), 1)
    assert_bound(ops.softmax2(logits.to(cuda)), p, 0.0, "softmax2", rel=0.0, extra=2.0 ** -18 * p)


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
