"""TEST INFRASTRUCTURE -- every unit of a ResNet U-Net train step against float64, at any batch and size: the model
built as bench.py builds it (oracle.step_checks.BenchStep: PyTorchUNetWeighted with bench.unet_config's settings, the
reference-like raw init).  tests/test_train_step_resnet_units_gpu.py runs it at batch 32 and 320x320 (ResNet101 and
ResNet34), tests/test_train_step_config5_gpu.py at BASELINE.json config 5's batch 16 and 512x512 (ResNet152).

Two steps run; the second, a graph replay, is checked on the step's own buffers (engine.Plan.block_parts,
Plan.stem_parts, Plan.dec_mid) against the pre-step weights, BatchNorm parameters and running statistics, which Adam
rewrites inside the step and are therefore snapshotted before it.  Each stored intermediate is checked against a
reference computed from the stored inputs of its own unit, so no error compounds from one unit into the next.  A is
the same operation on absolute values; `images` is a few images of the batch, the first and the last among them, and
the reductions take the whole batch:
  conv output z         float64 conv of the stored bf16 input with the bf16 weight       2^-8 |ref| + 2^-16 A   images
  BN mean, invstd       two-pass float64 mean and biased variance of the stored z        mean 2^-16 mean|z|, invstd
                                                                                         2^-12 relative
  running mean / var    (1 - m) pre-step + m (float64 mean, unbiased variance)           2^-12 of the terms (+ m x
                                                                                         the mean's allowance)
  BN apply y, block out from the stored z, the kernel's mean / invstd and pre-step       2^-8 |ref| + 2^-20 sum|terms|
                        gamma / beta, residual x or bn_d(z_d) with the downsample BN's
                        own statistics, ReLU
  stem max-pool         c1 = max_pool2d(a0); grad(a0) = grad(c1) routed to the first     bitwise
                        maximum of each window, as torch picks it
  dbeta, dgamma         sum g and sum g xhat, g = stored dy (stored y > 0)               2^-16 A
  dz                    gamma invstd (g - dbeta/M - xhat dgamma/M)                       2^-8 |ref| + 2^-16 A
  weight gradients      conv2d_weight of the stored dz and input (the stem: its unpacked  WGRAD_ACC A
                        7x7x3 slot)
  inner grad(y)         conv2d_input of the next conv's dz, masked by y > 0; zero        2^-8 |ref| + 2^-16 A   images
                        wherever y is
  block-input grads     every consumer: conv1's dgrad, the identity g or the downsample's as above + 2^-8 |partial|
                        dgrad, the decoder's skip dgrad for stage outputs (c5: the        for every bf16 write before
                        skip dgrad and the max-pool's routed gradient)                    the last, + 2^-8 |term| for
                                                                                          every dgrad added by TMA
                                                                                          reduce-add      images
  decoder halves, dec0  oracle.unit_checks.check_conv_half, as in test_train_step_vgg_scale_gpu.py
  final 1x1             dW, db of the stored dec0 output and plan.dlogits; dec0's        2^-16 A; 2^-8 |ref| + 2^-16 A
                        masked data gradient

The BatchNorm statistics are the point of the invstd bound: the conv epilogue sums z and z^2 in fp32 and the apply
pass finalises var = sumsq / M - mean^2, which loses about 2^-24 chain (1 + mean^2 / var) of the variance.  At 2^-12 the
normalised output moves by at most an eighth of bf16's half ulp, so the storage format hides the error; above it, it
does not.  The report prints, per BatchNorm, max |mean| / std over its channels and the worst relative invstd error."""
import torch
import torch.nn.functional as F

from oracle.step_checks import N, S, SEED, STATS, BenchStep, batch, free_device_memory, seeded_sd
from oracle.unit_checks import (CHUNK, SAMPLE, WGRAD_ACC, Bounds, bn_affine, check_conv_half, conv_kw, conv_ref, f64,
                                grad_view, nchw, wgrad64)

REL = 2.0 ** -8           # bf16 rounding of a stored output (and its share of what the reference rounds away)
TERMS = 2.0 ** -20        # fp32 rounding of the BN apply's affine terms
INVSTD_REL = 2.0 ** -12
MEAN_ACC = 2.0 ** -16


class Step:
    """the model after two train steps at batch n and sxs, with what the second step read before Adam rewrote it:
    pre-step bf16 weights and fp32 parameters (float64 on the device, by parameter name) and running statistics"""

    def __init__(self, enc, cuda, n, s, images):
        from mcb200 import engine
        self.momentum, self.eps = engine.BN_MOMENTUM, engine.BN_EPS
        self.images = list(images)
        run = BenchStep(enc, seeded_sd(enc), cuda, n, s)
        net = run.net
        X, T = (t.to(cuda) for t in batch(SEED, n, s))
        run.step(X, T)
        X, T = (t.to(cuda) for t in batch(SEED + 1, n, s))
        torch.cuda.synchronize()
        w16, p32 = net._w16.clone(), net._p32.clone()
        self.stats_pre = {k: f64(b) for k, b in net.named_buffers() if k.endswith(STATS)}
        run.step(X, T)
        torch.cuda.synchronize()
        assert run.fused.graphs is not None and run.fused.opt.t == 2, "the second step must be a graph replay"
        self.w = {name: f64(net._view(w16, net._slots[id(p)])) for name, p, _ in net._arena_params()}
        self.p = {name: f64(net._view(p32, net._slots[id(p)])) for name, p, _ in net._arena_params()}
        del w16, p32, X, T
        self.run, self.net, self.plan = run, net, run.fused.plan

    def mod(self, name):
        return self.net.get_submodule(name)

    def sample(self, t):
        """float64 NCHW copy of the sampled images of a stored NHWC tensor"""
        return f64(nchw(t)[self.images])


def dgrad_ref(shape, w, dz, conv):
    kw = conv_kw(conv)
    return (torch.nn.grad.conv2d_input(shape, w, dz, **kw),
            torch.nn.grad.conv2d_input(shape, w.abs(), dz.abs(), **kw))


def batch_stats(z):
    """two-pass float64 per-channel mean, biased variance and mean |z| of the stored NHWC z, CHUNK images at a time"""
    m = z.numel() // z.shape[3]
    s = a = q = 0.0
    for i in range(0, z.shape[0], CHUNK):
        zi = f64(z[i:i + CHUNK])
        s, a = s + zi.sum((0, 1, 2)), a + zi.abs().sum((0, 1, 2))
    mean = s / m
    for i in range(0, z.shape[0], CHUNK):
        q = q + ((f64(z[i:i + CHUNK]) - mean) ** 2).sum((0, 1, 2))
    return mean, q / m, a / m, m


def check_bn_forward(bd, st, report, bn_name, z, state):
    """the kernel's mean / invstd and the running statistics after the step against the two-pass float64 statistics"""
    mean, var, mean_abs, m = batch_stats(z)
    invstd = 1.0 / torch.sqrt(var + st.eps)
    bd.check("BN mean", bn_name, state.mean, mean, mean_abs, acc=MEAN_ACC)
    bd.check("BN invstd", bn_name, state.invstd, invstd, 0.0, rel=INVSTD_REL)
    report.append((bn_name, float((mean.abs() / var.sqrt().clamp_min(1e-300)).max()),
                   float(((f64(state.invstd) - invstd).abs() / invstd).max())))
    mo = st.momentum
    bnm = st.mod(bn_name)
    rm0, rv0 = st.stats_pre[bn_name + ".running_mean"], st.stats_pre[bn_name + ".running_var"]
    rm_terms = ((1 - mo) * rm0, mo * mean)
    bd.check("running mean", bn_name, bnm.running_mean, rm_terms[0] + rm_terms[1], 0.0,
             extra=INVSTD_REL * (rm_terms[0].abs() + rm_terms[1].abs()) + mo * MEAN_ACC * mean_abs)
    rv_ref = (1 - mo) * rv0 + mo * var * (m / (m - 1))
    bd.check("running var", bn_name, bnm.running_var, rv_ref, 0.0, rel=INVSTD_REL)


def step_affine(st, bn_name, state):
    """float64 (scale, shift) of a BatchNorm from the kernel's own mean / invstd and the pre-step gamma / beta"""
    return bn_affine(st.p, bn_name, f64(state.mean), f64(state.invstd))


def check_bn_backward(bd, st, part, dy, ymask):
    """dbeta, dgamma (whole batch) and dz of one conv + BN unit given its stored output gradient dy and ReLU output"""
    net, bn, z = st.net, part.state, part.z
    mu, istd = f64(bn.mean), f64(bn.invstd)
    db = dg = adb = adg = 0.0
    for i in range(0, z.shape[0], CHUNK):
        g = f64(dy[i:i + CHUNK]) * (ymask[i:i + CHUNK] > 0)
        xh = (f64(z[i:i + CHUNK]) - mu) * istd
        db, adb = db + g.sum((0, 1, 2)), adb + g.abs().sum((0, 1, 2))
        dg, adg = dg + (g * xh).sum((0, 1, 2)), adg + (g * xh).abs().sum((0, 1, 2))
        del g, xh
    bd.check("dbeta", part.bn, grad_view(net, part.bn + ".bias"), db, adb)
    bd.check("dgamma", part.bn, grad_view(net, part.bn + ".weight"), dg, adg)
    m = z.numel() // z.shape[3]
    k1, k2 = f64(grad_view(net, part.bn + ".bias")) / m, f64(grad_view(net, part.bn + ".weight")) / m
    a = st.p[part.bn + ".weight"] * istd
    g = f64(dy) * (ymask > 0)
    xh = (f64(z) - mu) * istd
    ref = a * (g - k1 - xh * k2)
    absref = a.abs() * (g.abs() + k1.abs() + (xh * k2).abs())
    del g, xh
    bd.check("dz", part.conv, part.dz, ref, absref, rel=REL)


def check_conv_bn(bd, st, report, part, dy, ymask, x_nchw=None):
    """conv output z (the sampled images), the BN statistics, the BN backward and the weight gradient of one conv + BN
    unit.  x_nchw: the conv's NCHW input when it is not part.x (the stem)"""
    conv = st.mod(part.conv)
    x = nchw(part.x) if x_nchw is None else x_nchw
    w = st.w[part.conv + ".weight"]
    ref, absref = conv_ref(f64(x[st.images]), w, conv)
    bd.check("conv output z", part.conv, st.sample(part.z), ref, absref, rel=REL)
    del ref, absref
    check_bn_forward(bd, st, report, part.bn, part.z, part.state)
    check_bn_backward(bd, st, part, dy, ymask)
    ref, absref = wgrad64(x, nchw(part.dz), w.shape, **conv_kw(conv))
    bd.check("weight gradient", part.conv, grad_view(st.net, part.conv + ".weight"), ref, absref, acc=WGRAD_ACC)
    del ref, absref


def check_apply(bd, st, what, kind, y, z, bn_name, state, residual=None):
    """y = relu(bn(z) [+ residual]) over the whole batch; residual = ("x", x) or ("bn", z_d, bn name, state)"""
    sc, sh = step_affine(st, bn_name, state)
    zz = f64(z)
    ref = zz * sc + sh
    terms = (zz * sc).abs() + (f64(state.mean) * sc).abs() + st.p[bn_name + ".bias"].abs()
    del zz
    if residual is not None and residual[0] == "x":
        r = f64(residual[1])
        ref, terms = ref + r, terms + r.abs()
        del r
    elif residual is not None:
        rsc, rsh = step_affine(st, residual[2], residual[3])
        r = f64(residual[1])
        ref = ref + r * rsc + rsh
        terms = terms + (r * rsc).abs() + (f64(residual[3].mean) * rsc).abs() + st.p[residual[2] + ".bias"].abs()
        del r
    bd.check(kind, what, y, ref.clamp_min(0), 0.0, rel=REL, extra=TERMS * terms)
    del ref, terms


def check_sum_of_writes(bd, kind, what, got, writes):
    """a stored gradient that several launches write in turn, the first storing, the others adding in bf16: writes =
    [(ref, absref, staged)] in write order.  Every write before the last rounds its partial sum to bf16, and a staged
    term (a conv dgrad's TMA reduce-add) is rounded to bf16 on its own before it is added"""
    ref = sum(r for r, _, _ in writes)
    absref = sum(a for _, a, _ in writes)
    extra, partial = 0.0, 0.0
    for j, (r, _, staged) in enumerate(writes):
        if j > 0 and staged:
            extra = extra + REL * r.abs()
        partial = partial + r
        if j < len(writes) - 1:
            extra = extra + REL * partial.abs()
    bd.check(kind, what, got, ref, absref, rel=REL, extra=extra)


def skip_dgrad(st, dec, x):
    """decoder `dec`'s data gradient into its skip input x (the sampled images): the dgrad of its middle gradient
    through the skip channels of its first conv, as a check_sum_of_writes entry"""
    prefix, ins, out = dec
    gm = st.sample(st.plan.grad[id(st.plan.dec_mid[id(out)])])
    w = st.w[prefix + ".block.0.conv.weight"][:, ins[0].shape[3]:]
    shape = (len(st.images), x.shape[3], x.shape[1], x.shape[2])
    return (torch.nn.grad.conv2d_input(shape, w, gm, padding=1),
            torch.nn.grad.conv2d_input(shape, w.abs(), gm.abs(), padding=1), True)


def routed(x, g):
    """the 2x2 max-pool gradient g routed to the first maximum of each window of x (float64 NCHW)"""
    _, where = F.max_pool2d(x, 2, 2, return_indices=True)
    return F.max_unpool2d(g, where, 2, 2, output_size=x.shape[2:])


def check_every_unit(enc, cuda, n=N, s=S, images=SAMPLE):
    """build `enc`'s U-Net as bench.py does at batch n and sxs, run two steps and check every unit of the second
    against float64 (the module docstring); print the check count, the worst |got - ref| / bound per kind and the
    BatchNorm report; assert the check count by formula and every bound.  The plan is released before this returns.
    -> (check count, conv + BN parts, report)"""
    assert images[0] == 0 and images[-1] == n - 1, "the sampled images hold the batch's first and last image"
    out = _check_every_unit(Step(enc, cuda, n, s, images), enc, n)
    free_device_memory()
    return out


def _check_every_unit(st, enc, n):
    images = st.images
    net, plan, sample = st.net, st.plan, st.sample
    bd, report = Bounds(), []
    blocks = [(prefix, ins[0], out) for kind, prefix, ins, out in plan.units if kind == "block"]
    decoders = [(prefix, ins, out) for kind, prefix, ins, out in plan.units if kind == "decoder"]
    skip_of = {id(ins[1]): (prefix, ins, out) for prefix, ins, out in decoders if len(ins) == 2}

    # ---- stem: 7x7/s2 conv (im2col + GEMM), BN, ReLU, 2x2 max-pool
    sp = plan.stem_parts
    from mcb200.engine import _ConvPart
    stem = _ConvPart("encoder.conv1", "encoder.bn1", None, sp["z0"], sp["a0"], sp["bn0"])
    stem.dz = sp["dz0"]
    x_stem = plan.x_in.to(torch.bfloat16)          # the im2col rounds the image to bf16
    d_a0 = plan.grad[id(sp["a0"])]
    check_conv_bn(bd, st, report, stem, d_a0, sp["a0"], x_nchw=x_stem)
    del x_stem
    check_apply(bd, st, "encoder.bn1", "BN apply y", sp["a0"], sp["z0"], "encoder.bn1", sp["bn0"])
    a0 = f64(nchw(sp["a0"]))
    bd.check("max-pool (bitwise)", "c1", nchw(sp["c1"]), F.max_pool2d(a0, 2, 2), 0.0)
    bd.check("max-pool (bitwise)", "grad(a0)", nchw(d_a0), routed(a0, f64(nchw(plan.grad[id(sp["c1"])]))), 0.0)
    del a0

    # ---- encoder blocks
    n_parts = n_inner = 0
    for prefix, x, out in blocks:
        parts = plan.block_parts[id(out)]
        down = parts[-1] if parts[-1].conv.endswith("downsample.0") else None
        last = parts[-2] if down is not None else parts[-1]
        inner = parts[:parts.index(last)]
        d_out = plan.grad[id(out)]
        n_parts += len(parts)
        n_inner += len(inner)
        for i, part in enumerate(inner):
            check_conv_bn(bd, st, report, part, plan.grad[id(part.y)], part.y)
            check_apply(bd, st, part.bn, "BN apply y", part.y, part.z, part.bn, part.state)
            nxt = parts[i + 1]
            conv = st.mod(nxt.conv)
            y = sample(part.y)
            ref, absref = dgrad_ref(tuple(y.shape), st.w[nxt.conv + ".weight"], sample(nxt.dz), conv)
            mask = (y > 0).double()
            bd.check("inner data gradient", part.conv + " output", sample(plan.grad[id(part.y)]), ref * mask,
                     absref * mask, rel=REL)
            bd.zero_where_off(part.conv + " output ReLU mask", plan.grad[id(part.y)], part.y)
            del y, ref, absref, mask
        for part in [last] + ([down] if down is not None else []):
            check_conv_bn(bd, st, report, part, d_out, out)
        res = ("x", x) if down is None else ("bn", down.z, down.bn, down.state)
        check_apply(bd, st, prefix, "block output", out, last.z, last.bn, last.state, res)

        # every consumer of the block input, in the order of its writes
        xs = (len(st.images), x.shape[3], x.shape[1], x.shape[2])
        writes = []
        if id(x) in skip_of:
            writes.append(skip_dgrad(st, skip_of[id(x)], x))
        if down is None:
            g = sample(d_out) * (sample(out) > 0)
            writes.append((g, g.abs(), False))     # bn_bwd_apply adds the exact bf16 g in fp32
        for part in [parts[0]] + ([down] if down is not None else []):
            writes.append(dgrad_ref(xs, st.w[part.conv + ".weight"], sample(part.dz), st.mod(part.conv)) + (True,))
        check_sum_of_writes(bd, "block-input gradient", prefix + " input", sample(plan.grad[id(x)]), writes)
        del writes

    # ---- c5: dec5's skip dgrad, then the centre max-pool's routed gradient
    c5 = blocks[-1][2]
    pool = decoders[0][1][0]
    writes = [skip_dgrad(st, skip_of[id(c5)], c5)]
    r = routed(sample(c5), sample(plan.grad[id(pool)]))
    writes.append((r, r.abs(), False))              # maxpool2_bwd adds the exact routed bf16 value in fp32
    check_sum_of_writes(bd, "block-input gradient", "c5 (dec5 skip + max-pool)", sample(plan.grad[id(c5)]), writes)
    del writes, r

    # ---- decoder blocks half by half, dec0 and the 1x1 classifier
    for prefix, ins, out in decoders:
        mid = plan.dec_mid[id(out)]
        x = torch.cat([nchw(a) for a in ins], 1) if len(ins) > 1 else nchw(ins[0])
        check_conv_half(bd, net, st.w, st.p, prefix + ".block.0", prefix + ".block.0.conv.weight",
                        prefix + ".block.0.conv.bias", x, mid, plan.grad[id(mid)], "convT dgrad epilogue",
                        images=images)
        src = "dgrad epilogue" if id(out) in plan.bias_fused else "channel_sum"
        check_conv_half(bd, net, st.w, st.p, prefix + ".block.1", prefix + ".block.1.weight",
                        prefix + ".block.1.bias", nchw(mid), out, plan.grad[id(out)], src, transposed=True,
                        images=images)
        del x
    d1, y0 = decoders[-1][2], plan.classifier_in
    g0 = plan.grad[id(y0)]
    check_conv_half(bd, net, st.w, st.p, "dec0", "dec0.conv.weight", "dec0.conv.bias", nchw(d1), y0, g0, "channel_sum",
                    images=images)
    dl = plan.dlogits
    k = dl.shape[1]
    dw = adw = db = adb = 0.0
    for i in range(0, n, CHUNK):
        yi, di = f64(y0[i:i + CHUNK]), f64(dl[i:i + CHUNK])
        dw, adw = dw + torch.einsum("nkhw,nhwc->kc", di, yi), adw + torch.einsum("nkhw,nhwc->kc", di.abs(), yi.abs())
        db, adb = db + di.sum((0, 2, 3)), adb + di.abs().sum((0, 2, 3))
        del yi, di
    bd.check("final 1x1 dW, db", "final.weight", grad_view(net, "final.weight").reshape(k, -1), dw, adw)
    bd.check("final 1x1 dW, db", "final.bias", grad_view(net, "final.bias"), db, adb)
    wf = st.p["final.weight"].reshape(k, -1)
    ds = f64(dl[st.images])
    mask = (sample(y0) > 0).double()
    ref = torch.einsum("nkhw,kc->nchw", ds, wf) * mask
    absref = torch.einsum("nkhw,kc->nchw", ds.abs(), wf.abs()) * mask
    bd.check("inner data gradient", "dec0 output (final 1x1)", sample(g0), ref, absref, rel=REL)
    del ds, mask, ref, absref

    print("%s: %d checks" % (enc, bd.count))
    bd.report()
    print("  BatchNorm statistics: max |mean| / std over the channels, worst relative invstd error (bound 2^-12)")
    for name, ratio, err in report:
        print("    %-36s max |mean|/std %8.2f   invstd error %.2e" % (name, ratio, err))
    worst = max(report, key=lambda r: r[2])
    print("  largest |mean| / std %.2f (%s); worst invstd error %.2e = 2^%.1f (%s)" % (
        max(r[1] for r in report), max(report, key=lambda r: r[1])[0], worst[2],
        torch.tensor(max(worst[2], 1e-300)).log2().item(), worst[0]))
    n_blocks = len(blocks)
    assert len(report) == n_parts + 1
    # 12 stem checks, 9 per conv + BN, 3 more per inner unit, 2 per block, c5, 4 per conv half, final 1x1's 3
    assert bd.count == 12 + 9 * n_parts + 3 * n_inner + 2 * n_blocks + 1 + 4 * (2 * len(decoders) + 1) + 3, bd.count
    assert not bd.fails, "\n".join(bd.fails[:20])
    return bd.count, n_parts, report
