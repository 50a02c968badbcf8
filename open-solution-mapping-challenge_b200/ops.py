"""Tensor-level wrappers over the C ABI (one function per entry point of include/mcb200.h).

All activations are torch CUDA tensors, NHWC (shape (N, H, W, C)), bf16, contiguous.  Conv weights are "packed":
bf16 (k*k, cout, cin).  These wrappers only marshal pointers and shapes; the arithmetic is in libmcb200.so."""
import ctypes as C

import torch

from . import _lib as L


def _chk(t, dtype=torch.bfloat16):
    assert t.is_cuda and t.is_contiguous() and t.dtype == dtype, (t.device, t.is_contiguous(), t.dtype)
    return t


def pack_conv_weight(w):
    """(cout, cin, kh, kw) -> (kh*kw, cout, cin), the library's tap-major layout"""
    co, ci, kh, kw = w.shape
    return w.permute(2, 3, 0, 1).reshape(kh * kw, co, ci).contiguous()


def unpack_conv_weight(wp, k):
    t, co, ci = wp.shape
    return wp.reshape(k, k, co, ci).permute(2, 3, 0, 1).contiguous()


def pack_convt_weight(w):
    """ConvTranspose2d weight (cin, cout, kh, kw) -> (kh*kw, cout, cin)"""
    ci, co, kh, kw = w.shape
    return w.permute(2, 3, 1, 0).reshape(kh * kw, co, ci).contiguous()


def unpack_convt_weight(wp, k=4):
    t, co, ci = wp.shape
    return wp.reshape(k, k, co, ci).permute(3, 2, 0, 1).contiguous()


def conv_fwd(x, w, ksize, stride=1, bias=None, relu=False, stats=None, x2=None, out=None, scale=None, residual=None):
    _chk(x); _chk(w)
    n, h, wd, c0 = x.shape
    c1 = 0
    if x2 is not None:
        _chk(x2)
        assert x2.shape[:3] == x.shape[:3]
        c1 = x2.shape[3]
    cout = w.shape[1]
    assert w.shape == (ksize * ksize, cout, c0 + c1), (w.shape, ksize, cout, c0, c1)
    if out is None:
        out = torch.empty((n, h // stride, wd // stride, cout), dtype=torch.bfloat16, device=x.device)
    a = L.ConvFwdArgs()
    a.x[0] = x.data_ptr(); a.x[1] = x2.data_ptr() if x2 is not None else None
    a.cin[0] = c0; a.cin[1] = c1
    a.n, a.h, a.w = n, h, wd
    a.weight = w.data_ptr(); a.cout = cout; a.ksize = ksize; a.stride = stride
    a.bias = _chk(bias, torch.float32).data_ptr() if bias is not None else None
    a.relu = int(relu)
    a.stats = _chk(stats, torch.float32).data_ptr() if stats is not None else None
    a.y = _chk(out).data_ptr()
    a.scale = _chk(scale, torch.float32).data_ptr() if scale is not None else None
    a.residual = _chk(residual).data_ptr() if residual is not None else None
    L.call("mcb_conv_fwd", a)
    return out


def conv_dgrad(dy, w, ksize, stride, in_hw, cin=None, ci_off=0, relu_mask=None, accumulate=False, out=None,
               bn_reduce=None, channel_sum=None):
    """bn_reduce = (z, mean, invstd, gamma, beta, dbeta, dgamma): fuse the backward of the conv-BN-ReLU unit that
    produced this conv's input into the epilogue (ReLU mask recomputed from z, BatchNorm-backward reductions);
    relu_mask must then be None"""
    _chk(dy); _chk(w)
    n = dy.shape[0]
    h, wd = in_hw
    cout, cin_total = w.shape[1], w.shape[2]
    cin = cin_total if cin is None else cin
    if out is None:
        assert not accumulate
        out = torch.empty((n, h, wd, cin), dtype=torch.bfloat16, device=dy.device)
    a = L.ConvDgradArgs()
    a.dy = dy.data_ptr(); a.n, a.h, a.w = n, h, wd
    a.weight = w.data_ptr(); a.cout = cout; a.cin_total = cin_total; a.ci_off = ci_off; a.cin = cin
    a.ksize = ksize; a.stride = stride
    a.dx = _chk(out).data_ptr()
    a.relu_mask = _chk(relu_mask).data_ptr() if relu_mask is not None else None
    a.accumulate = int(accumulate)
    if bn_reduce is not None:
        z, mean, invstd, gamma, beta, dbeta, dgamma = bn_reduce
        a.bn_z = _chk(z).data_ptr(); a.bn_mean = mean.data_ptr(); a.bn_invstd = invstd.data_ptr()
        a.bn_gamma = gamma.data_ptr(); a.bn_beta = beta.data_ptr()
        a.bn_dbeta = dbeta.data_ptr(); a.bn_dgamma = dgamma.data_ptr()
    if channel_sum is not None:
        a.dx_channel_sum = _chk(channel_sum, torch.float32).data_ptr()
    L.call("mcb_conv_dgrad", a)
    return out


def conv_wgrad(dy, x, dw, ksize, stride, ci_off=0):
    """dw (fp32, (k*k, cout, cin_total)) += wgrad"""
    _chk(dy); _chk(x); _chk(dw, torch.float32)
    n, h, wd, cin = x.shape
    a = L.ConvWgradArgs()
    a.dy = dy.data_ptr(); a.x = x.data_ptr(); a.n, a.h, a.w = n, h, wd
    a.cout = dw.shape[1]; a.cin_total = dw.shape[2]; a.ci_off = ci_off; a.cin = cin
    a.ksize = ksize; a.stride = stride; a.dw = dw.data_ptr()
    L.call("mcb_conv_wgrad", a)
    return dw


def _convt_ksize(taps):
    """packed transposed-conv weights hold k*k taps: 16 -> ConvTranspose2d(4, 2, 1), 9 -> ConvTranspose2d(3, 2, 1, 1)"""
    assert taps in (9, 16), taps
    return 3 if taps == 9 else 4


def convt_fwd(x, w, bias=None, relu=False, out=None):
    _chk(x); _chk(w)
    n, h, wd, cin = x.shape
    cout = w.shape[1]
    assert w.shape[1:] == (cout, cin), (w.shape, cin)
    if out is None:
        out = torch.empty((n, 2 * h, 2 * wd, cout), dtype=torch.bfloat16, device=x.device)
    a = L.ConvtFwdArgs()
    a.x = x.data_ptr(); a.n, a.h, a.w, a.cin = n, h, wd, cin
    a.weight = w.data_ptr(); a.cout = cout
    a.bias = _chk(bias, torch.float32).data_ptr() if bias is not None else None
    a.relu = int(relu); a.y = _chk(out).data_ptr(); a.ksize = _convt_ksize(w.shape[0])
    L.call("mcb_convt_fwd", a)
    return out


def convt_dgrad(dy, w, relu_mask=None, accumulate=False, out=None, channel_sum=None):
    _chk(dy); _chk(w)
    n, h2, w2, cout = dy.shape
    h, wd = h2 // 2, w2 // 2
    cin = w.shape[2]
    if out is None:
        assert not accumulate
        out = torch.empty((n, h, wd, cin), dtype=torch.bfloat16, device=dy.device)
    a = L.ConvtDgradArgs()
    a.dy = dy.data_ptr(); a.n, a.h, a.w, a.cin = n, h, wd, cin
    a.weight = w.data_ptr(); a.cout = cout; a.dx = _chk(out).data_ptr()
    a.relu_mask = _chk(relu_mask).data_ptr() if relu_mask is not None else None
    a.accumulate = int(accumulate)
    if channel_sum is not None:
        a.dx_channel_sum = _chk(channel_sum, torch.float32).data_ptr()
    a.ksize = _convt_ksize(w.shape[0])
    L.call("mcb_convt_dgrad", a)
    return out


def convt_wgrad(dy, x, dw):
    _chk(dy); _chk(x); _chk(dw, torch.float32)
    n, h, wd, cin = x.shape
    a = L.ConvtWgradArgs()
    a.dy = dy.data_ptr(); a.x = x.data_ptr(); a.n, a.h, a.w, a.cin = n, h, wd, cin
    a.cout = dw.shape[1]; a.dw = dw.data_ptr(); a.ksize = _convt_ksize(dw.shape[0])
    L.call("mcb_convt_wgrad", a)
    return dw


# ---------------------------------------------------------------------------------------------------------------------
# HBM-bound glue
# ---------------------------------------------------------------------------------------------------------------------
F32 = torch.float32


def nchw_to_nhwc_bf16(x, out=None):
    _chk(x, F32)
    n, c, h, w = x.shape
    if out is None:
        out = torch.empty((n, h, w, c), dtype=torch.bfloat16, device=x.device)
    L.fcall("mcb_nchw_f32_to_nhwc_bf16", x.data_ptr(), out.data_ptr(), n, c, h, w)
    return out


def nhwc_to_nchw_f32(x, out=None):
    _chk(x)
    n, h, w, c = x.shape
    if out is None:
        out = torch.empty((n, c, h, w), dtype=F32, device=x.device)
    L.fcall("mcb_nhwc_bf16_to_nchw_f32", x.data_ptr(), out.data_ptr(), n, c, h, w)
    return out


def stem_im2col(x, out=None):
    _chk(x, F32)
    n, c, h, w = x.shape
    assert c == 3
    if out is None:
        out = torch.empty((n, h // 2, w // 2, 192), dtype=torch.bfloat16, device=x.device)
    L.fcall("mcb_stem_im2col", x.data_ptr(), out.data_ptr(), n, h, w)
    return out


def stem_pack_weight(w49x64x3, out):
    L.fcall("mcb_stem_pack_weight", _chk(w49x64x3, F32).data_ptr(), _chk(out).data_ptr())
    return out


def stem_unpack_wgrad(dwp, dw):
    L.fcall("mcb_stem_unpack_wgrad", _chk(dwp, F32).data_ptr(), _chk(dw, F32).data_ptr())


def vgg_input_im2col(x, out=None):
    """fp32 NCHW image -> bf16 (N, H, W, 32) im2col of the 3x3 pad-1 VGG input conv (k = (ky*3 + kx)*3 + c)"""
    _chk(x, F32)
    n, c, h, w = x.shape
    assert c == 3
    if out is None:
        out = torch.empty((n, h, w, 32), dtype=torch.bfloat16, device=x.device)
    assert out.shape == (n, h, w, 32), out.shape
    L.fcall("mcb_vgg_input_im2col", x.data_ptr(), _chk(out).data_ptr(), n, h, w)
    return out


def vgg_input_pack_weight(w9x64x3, out):
    """fp32 [9][64][3] master slot -> bf16 (1, 64, 32) GEMM operand"""
    assert w9x64x3.numel() == 9 * 64 * 3 and out.shape == (1, 64, 32), (w9x64x3.shape, out.shape)
    L.fcall("mcb_vgg_input_pack_weight", _chk(w9x64x3, F32).data_ptr(), _chk(out).data_ptr())
    return out


def vgg_input_unpack_wgrad(dwp, dw):
    """dw ([9][64][3] fp32 slot) += the (1, 64, 32) fp32 weight gradient of the im2col GEMM"""
    assert dwp.shape == (1, 64, 32) and dw.numel() == 9 * 64 * 3, (dwp.shape, dw.shape)
    L.fcall("mcb_vgg_input_unpack_wgrad", _chk(dwp, F32).data_ptr(), _chk(dw, F32).data_ptr())


def bn_finalize(stats, count, gamma, beta, rm, rv, scale, shift, mean, invstd, momentum=0.1, eps=1e-5):
    c = gamma.numel()
    L.fcall("mcb_bn_finalize", stats.data_ptr(), int(count), gamma.data_ptr(), beta.data_ptr(), L.dp(rm), L.dp(rv),
            momentum, eps, scale.data_ptr(), shift.data_ptr(), mean.data_ptr(), invstd.data_ptr(), c)


def bn_eval_params(gamma, beta, rm, rv, scale, shift, eps=1e-5):
    L.fcall("mcb_bn_eval_params", gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(), eps,
            scale.data_ptr(), shift.data_ptr(), gamma.numel())


def bn_apply(z, scale, shift, out, relu=True, residual=None, res_scale=None, res_shift=None):
    _chk(z); _chk(out)
    c = z.shape[-1]
    L.fcall("mcb_bn_apply", z.data_ptr(), scale.data_ptr(), shift.data_ptr(), L.dp(residual), L.dp(res_scale),
            L.dp(res_shift), int(relu), out.data_ptr(), z.numel() // c, c)
    return out


def make_bn_train(stats, gamma, beta, rm, rv, mean, invstd):
    b = L.BNTrain()
    b.stats, b.gamma, b.beta = stats.data_ptr(), gamma.data_ptr(), beta.data_ptr()
    b.running_mean, b.running_var = L.dp(rm), L.dp(rv)
    b.mean, b.invstd = mean.data_ptr(), invstd.data_ptr()
    return b


def bn_train_apply(z, bn, out, relu=True, residual=None, res_bn=None, momentum=0.1, eps=1e-5, count_scale=1):
    """bn / res_bn: L.BNTrain structs (make_bn_train); statistics finalisation folded into the apply pass.
    count_scale = world size when the statistics have been all-reduced (synchronised BatchNorm)"""
    c = z.shape[-1]
    pixels = z.numel() // c
    L.fcall("mcb_bn_train_apply_global", _chk(z).data_ptr(), C.byref(bn), L.dp(residual),
            C.byref(res_bn) if res_bn is not None else None, int(relu), _chk(out).data_ptr(), pixels,
            pixels * int(count_scale), c, momentum, eps)
    return out


def bn_bwd_reduce(dy, y_mask, z, mean, invstd, dbeta, dgamma):
    c = z.shape[-1]
    L.fcall("mcb_bn_bwd_reduce", _chk(dy).data_ptr(), L.dp(y_mask), _chk(z).data_ptr(), mean.data_ptr(),
            invstd.data_ptr(), dbeta.data_ptr(), dgamma.data_ptr(), z.numel() // c, c)


def bn_bwd_apply(dy, y_mask, z, mean, invstd, gamma, dbeta, dgamma, dz, g_out=None, g_accumulate=False, count_scale=1):
    c = z.shape[-1]
    pixels = z.numel() // c
    L.fcall("mcb_bn_bwd_apply_global", _chk(dy).data_ptr(), L.dp(y_mask), _chk(z).data_ptr(), mean.data_ptr(),
            invstd.data_ptr(), gamma.data_ptr(), dbeta.data_ptr(), dgamma.data_ptr(), _chk(dz).data_ptr(), L.dp(g_out),
            int(g_accumulate), pixels, pixels * int(count_scale), c)


def channel_sum(x, out):
    c = x.shape[-1]
    L.fcall("mcb_channel_sum", _chk(x).data_ptr(), out.data_ptr(), x.numel() // c, c)


def maxpool2_fwd(x, out=None):
    _chk(x)
    n, h, w, c = x.shape
    if out is None:
        out = torch.empty((n, h // 2, w // 2, c), dtype=torch.bfloat16, device=x.device)
    L.fcall("mcb_maxpool2_fwd", x.data_ptr(), out.data_ptr(), n, h, w, c)
    return out


def maxpool2_bwd(x, dy, dx, accumulate=False):
    n, h, w, c = x.shape
    L.fcall("mcb_maxpool2_bwd", _chk(x).data_ptr(), _chk(dy).data_ptr(), _chk(dx).data_ptr(), int(accumulate), n, h, w, c)
    return dx


def maxpool2_bwd_skip_relu(y, dpool, g, db):
    """y = relu(conv + b) feeding pool(y) and a decoder concat; g (holding the concat's gradient) becomes
    (g + routed dpool) * (y > 0) in place, db += its per-channel sums"""
    n, h, w, c = y.shape
    assert g.shape == y.shape and dpool.shape == (n, h // 2, w // 2, c) and db.numel() == c
    assert g.data_ptr() not in (y.data_ptr(), dpool.data_ptr()), "g is rewritten in place: it must not alias y or dpool"
    L.fcall("mcb_maxpool2_bwd_skip_relu", _chk(y).data_ptr(), _chk(dpool).data_ptr(), _chk(g).data_ptr(),
            _chk(db, F32).data_ptr(), n, h, w, c)
    return g


def final_conv_fwd(x, w, b, logits):
    n, h, wd, c = x.shape
    k = b.numel()
    L.fcall("mcb_final_conv_fwd", _chk(x).data_ptr(), w.data_ptr(), b.data_ptr(), _chk(logits, F32).data_ptr(), n, h,
            wd, c, k)
    return logits


def final_conv_bwd(x, w, dlogits, dx, dw, db):
    n, h, wd, c = x.shape
    k = db.numel()
    L.fcall("mcb_final_conv_bwd", _chk(x).data_ptr(), w.data_ptr(), _chk(dlogits, F32).data_ptr(), _chk(dx).data_ptr(),
            dw.data_ptr(), db.data_ptr(), n, h, wd, c, k)


def adam_step(p, g, m, v, p_bf16, step, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, grad_scale=1.0):
    L.fcall("mcb_adam_step", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), L.dp(p_bf16), p.numel(), lr,
            betas[0], betas[1], eps, weight_decay, int(step), grad_scale)


def adam_hyper(lr, betas, step):
    """[lr, 1 - beta1^t, (1 - beta2^t)^0.5] for adam_step_dyn's `hyper`: torch.optim.Adam's bias corrections, in
    double from the caller's betas.  mcb_adam_step computes the same doubles on the host (pow(bc2, 0.5) included), so
    both entry points give the same bits once the values are rounded to fp32."""
    return [lr, 1.0 - betas[0] ** step, (1.0 - betas[1] ** step) ** 0.5]


def adam_step_dyn(p, g, m, v, p_bf16, hyper, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, grad_scale=1.0):
    """Adam over a (slice of the) flat arena with {lr, 1-b1^t, sqrt(1-b2^t)} read from the device tensor `hyper`"""
    L.fcall("mcb_adam_step_dyn", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), L.dp(p_bf16), p.numel(),
            hyper.data_ptr(), betas[0], betas[1], eps, weight_decay, grad_scale)


def cast_bf16(x, out):
    L.fcall("mcb_cast_f32_bf16", _chk(x, F32).data_ptr(), _chk(out).data_ptr(), x.numel())
    return out


DICE_ACTIVATIONS = ("softmax", "sigmoid")   # mcb_loss_args.dice_activation 0, 1


def dice_activation_code(name):
    """the mcb_loss_args.dice_activation of an activation name; the reference's error for any other
    (src/models.py:438-443)"""
    if name not in DICE_ACTIVATIONS:
        raise NotImplementedError('only sigmoid and softmax are implemented')
    return DICE_ACTIVATIONS.index(name)


def _loss_args(logits, target, mode, cfg):
    a = L.LossArgs()
    n, k, h, w = logits.shape
    assert k == 2, "the CUDA loss kernels implement the reference's 2-class configuration"
    assert target.shape == (n, 3 if mode == 0 else 1, h, w), target.shape
    a.logits = _chk(logits, F32).data_ptr(); a.target = _chk(target, F32).data_ptr()
    a.n, a.h, a.w, a.mode = n, h, w, mode
    a.w0 = cfg.get("w0", 50.0); a.sigma = cfg.get("sigma", 10.0); a.size_c = cfg.get("size_c", 128.0)
    a.dice_weight = cfg.get("dice_weight", 0.2); a.ce_weight = cfg.get("ce_weight", 1.0)
    a.dice_smooth = cfg.get("dice_smooth", 1.0)
    a.dice_activation = dice_activation_code(cfg.get("dice_activation", "softmax"))
    return a


def loss_partials(logits, target, sums, mode=0, **cfg):
    """sums: float64[4] on device, zeroed by the caller; += (sum p1*t, sum p1, sum t, sum w*ce)"""
    a = _loss_args(logits, target, mode, cfg)
    L.fcall("mcb_loss_partials", C.byref(a), sums.data_ptr())


def loss_grad(logits, target, sums, dlogits, loss_out, global_pixels=None, grad_scale=1.0, mode=0, **cfg):
    a = _loss_args(logits, target, mode, cfg)
    n, _, h, w = logits.shape
    L.fcall("mcb_loss_grad", C.byref(a), sums.data_ptr(), int(global_pixels or n * h * w), grad_scale,
            dlogits.data_ptr(), L.dp(loss_out))


def softmax2(logits, out=None):
    n, k, h, w = logits.shape
    assert k == 2
    if out is None:
        out = torch.empty_like(logits)
    L.fcall("mcb_softmax2", _chk(logits, F32).data_ptr(), out.data_ptr(), n, h, w)
    return out
