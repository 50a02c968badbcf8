"""Float64 references of single plan units on a plan's own buffers, shared by the unit tests of the train step
(tests/test_train_step_vgg_scale_gpu.py, oracle/resnet_step_units.py) and of the batch-64 inference forward
(tests/test_infer_forward_units_gpu.py).

Activations and gradients are the plan's NHWC bf16 buffers; every reference is evaluated in float64 on their device.
Bounds are element-wise, |got - ref| <= rel |ref| + acc A + extra, with A the same operation on absolute values."""
import torch
import torch.nn.functional as F

SAMPLE = (0, 10, 21, 31)  # images of the batch-32 train step's element-wise forward and data-gradient checks (the
#                           reductions take all 32); the first and the last image hold the batch's edge tiles
CHUNK = 8                 # images per float64 evaluation over a whole batch (sums over the chunks added in float64)
# accumulation allowance of the weight gradients.  Their reductions run over all 3.3 M pixels of the batch, and the
# split-K GEMM caps its splits at one wave of CTAs, so one fp32 accumulator chain adds up to k = 12800 pixel tiles x 4
# MMA steps (VGG's dec1: 4 splits).  The a-priori bound of such a chain, k 2^-24 A, is 2^-8.4 A, and the rounding
# outgrows the 2^-16 A that holds at the persistent-kernel test's shapes: measured worst 2^-10.9 A (VGG16's dec1).  A
# missing weight gradient is off by |ref|, up to about 2^-8 A here, at most elements.
WGRAD_ACC = 2.0 ** -9


def f64(t):
    return t.to(torch.float64)


def nchw(t):
    return t.permute(0, 3, 1, 2)


def grad_view(net, name):
    """the step's gradient of parameter `name` in the gradient arena, in the parameter's shape"""
    p = dict((n, p) for n, p, _ in net._arena_params())[name]
    return net._view(net._g32, net._slots[id(p)])


class Bounds:
    """element-wise |got - ref| <= rel |ref| + 2^-16 A + extra checks; keeps the worst |got - ref| / bound per kind"""

    def __init__(self):
        self.worst, self.fails, self.count = {}, [], 0

    def check(self, kind, what, got, ref, absref, rel=0.0, extra=0.0, acc=2.0 ** -16):
        got = f64(got)
        err = (got - ref).abs()
        lim = rel * ref.abs() + acc * absref + extra
        ok = err <= lim                              # (NaN counts as bad)
        ratio = torch.where(lim > 0, err / lim.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
        r = float(torch.where(torch.isnan(err), float("inf"), ratio).max())
        self.count += 1
        if r > self.worst.get(kind, (-1.0, ""))[0]:
            self.worst[kind] = (r, what)
        if not bool(ok.all()):
            i = tuple(int(j) for j in (~ok).nonzero()[0])
            self.fails.append("%s %s: %d of %d elements out of bounds, first at %s: got %r, ref %r, bound %r" % (
                what, kind, int((~ok).sum()), ok.numel(), i, float(got[i]), float(ref[i]), float(lim[i])))

    def zero_where_off(self, what, g, y):
        """the stored gradient g is masked by the unit's own ReLU: zero wherever the stored output y is"""
        self.count += 1
        n = int(((g != 0) & (y == 0)).sum())
        if n:
            self.fails.append("%s: %d stored gradient elements are nonzero where the ReLU output is 0" % (what, n))

    def report(self):
        for kind, (r, what) in sorted(self.worst.items()):
            print("  worst |got - ref| / bound, %-32s %.3f (%s)" % (kind, r, what))


def wgrad64(x, g, shape, **kw):
    """float64 conv2d weight gradient (and the same on absolute values) over the whole batch, CHUNK images at a time;
    x and g are NCHW views of stored bf16 tensors"""
    ref = absref = 0.0
    for i in range(0, x.shape[0], CHUNK):
        xi, gi = f64(x[i:i + CHUNK]), f64(g[i:i + CHUNK])
        ref = ref + torch.nn.grad.conv2d_weight(xi, shape, gi, **kw)
        absref = absref + torch.nn.grad.conv2d_weight(xi.abs(), shape, gi.abs(), **kw)
        del xi, gi
    return ref, absref


def check_bias(bd, what, got, g):
    """bias gradient = float64 channel sum of the stored (masked) bf16 output gradient g (NHWC), whole batch"""
    ref = absref = 0.0
    for i in range(0, g.shape[0], CHUNK):
        gi = f64(g[i:i + CHUNK])
        ref = ref + gi.sum((0, 1, 2))
        absref = absref + gi.abs().sum((0, 1, 2))
        del gi
    bd.check(what[0], what[1], got, ref, absref)


def conv_kw(conv):
    return dict(stride=conv.stride, padding=conv.padding)


def conv_ref(x, w, conv):
    """float64 conv2d of x with w as the nn.Conv2d `conv` runs it, and the same on absolute values"""
    kw = conv_kw(conv)
    return F.conv2d(x, w, **kw), F.conv2d(x.abs(), w.abs(), **kw)


def bn_affine(p, bn_name, mean, invstd):
    """float64 per-channel (scale, shift) of BatchNorm `bn_name` normalising with (mean, invstd); p: its fp32 gamma and
    beta (float64 on the device), by parameter name.  Training passes the batch statistics, inference the running ones"""
    sc = p[bn_name + ".weight"] * invstd
    return sc, p[bn_name + ".bias"] - mean * sc


def check_conv_forward(bd, prefix, x, y, w, b, transposed=False, images=SAMPLE):
    """forward of one conv (or stride-2 transposed conv) + bias + ReLU on `images`: x the NCHW bf16 input, y the NHWC
    stored output, w / b the bf16 weight and fp32 bias (float64 on the device).  |got - ref| <= 2^-8 |ref| + 2^-16 A"""
    xs = f64(x[list(images)])
    if transposed:
        op = dict(stride=2, padding=1, output_padding=1 if w.shape[-1] == 3 else 0)
        ref = F.conv_transpose2d(xs, w, b, **op)
        absref = F.conv_transpose2d(xs.abs(), w.abs(), b.abs(), **op)
    else:
        ref = F.conv2d(xs, w, b, padding=1)
        absref = F.conv2d(xs.abs(), w.abs(), b.abs(), padding=1)
    del xs
    bd.check("forward", prefix, nchw(y)[list(images)], ref.clamp_min(0), absref, rel=2.0 ** -8)
    del ref, absref


def check_conv_half(bd, net, w16, b32, prefix, wkey, bkey, x, y, g, bias_from, transposed=False, images=SAMPLE):
    """one conv (or stride-2 transposed conv) + bias + ReLU: x the NCHW bf16 input, y and g the NHWC stored output and
    output gradient; w16 / b32 the pre-step bf16 weight and fp32 bias (float64 on the device).  The forward is checked
    on `images`, the weight and bias gradients over the whole batch"""
    w = w16[wkey]
    check_conv_forward(bd, prefix, x, y, w, b32[bkey], transposed, images)
    bd.zero_where_off(prefix + " ReLU mask", g, y)
    if transposed:     # d conv_transpose2d(x, W) / dW = conv2d weight gradient of the conv from the output back to x
        ref, absref = wgrad64(nchw(g), x, w.shape, stride=2, padding=1)
    else:
        ref, absref = wgrad64(x, nchw(g), w.shape, padding=1)
    bd.check("weight gradient", wkey, grad_view(net, wkey), ref, absref, acc=WGRAD_ACC)
    del ref, absref
    check_bias(bd, ("bias gradient (%s)" % bias_from, bkey), grad_view(net, bkey), g)
