"""The VGG-encoder U-Nets' train step end to end at the size bench_encoders.py publishes it: UNet11 (VGG11) and
UNetVGG16 (VGG16) at batch 32 and 320x320, built as bench_encoders.vgg_fused_step builds them (FusedTrainStep with
bench.unet_config's loss and Adam settings), and part A for the AlbuNet-wired ResNet34 plan through
PyTorchUNetWeighted._fit_loop.

At this size the VGG nets hold the largest tensors of the project: the 64-channel full-resolution activations have
2.1e8 elements, dec1's 96-channel concat input 3.1e8, and the implicit im2col of dec1's 3x3 conv spans 2.8e9 elements,
past 2^31; each per-channel bias sum runs over 3.3 M pixels.  Checked, per net:
  A. the captured step (side-stream weight gradients, per-segment Adam hooks inside the backward graph, graph replays)
     equals the same segments run eagerly in program order on one stream, bit for bit, for three distinct batches.
     In program order a segment's Adam hook runs exactly where it is issued, so a VGGPlan segment bound (decoder |
     conv5 | conv4 | rest) that takes in a parameter whose gradient is finished later fails here deterministically;
  B. every step's weights, Adam moments and bf16 operands are exactly Adam of that step's own gradients over the whole
     arena: segments that do not tile the arena, or a hook that reads its gradients before they have landed, break
     this;
  U. every unit of the plan against float64 on the step's own buffers (the CUDA path's bf16 inputs, the pre-step bf16
     weights and the stored output gradient), element-wise, with the bounds of test_conv_gemm_persistent_gpu.py
     (A is the same operation on absolute values):
       forward output   |got - ref| <= 2^-8 |ref| + 2^-16 A   (on images SAMPLE; ReLU applied)
       weight gradient  |got - ref| <= 2^-9 A                  (whole batch; unit_checks.WGRAD_ACC: why not 2^-16 A)
       bias gradient    float64 sum of the stored bf16 gradient, to 2^-16 A (whole batch): from the dgrad epilogue
                        (units inside a stage, decoder outputs), maxpool2_bwd_skip_relu (stage outputs), the
                        transposed conv's dgrad epilogue (decoder middles) and channel_sum (dec1)
     and every stored gradient is zero wherever its unit's stored ReLU output is.  The decoder blocks are checked half
     by half, element-wise: the plan keeps each block's middle activation (Plan.dec_mid) and its gradient.  dec1 is
     checked against cat[dec2, conv1] together with both data-gradient segments it writes: dec2's stored gradient,
     and conv1's, which also holds the pooled path (the first maximum of each 2x2 window, as torch picks it);
  D. step 1 against the fp32 reference (oracle.vgg_oracle on the GPU, TF32 off) with the rules of
     test_encoders_vgg_gpu.py::test_logits_loss_and_gradients_against_reference, the CUDA path measured against a
     bf16-storage emulation of the same step.

Exact equality is the bar of A and B: every cross-CTA sum of the step is added in a fixed order.  At most one batch-32
plan is alive at a time; what is compared across runs is kept on the host.

Measured on an H100 80GB HBM3 at its 700 W power limit: the file takes about 90 s and at most 27.3 GiB of device memory
(test D); U takes 6 s per net.  U's worst |got - ref| / bound: forward 0.99 (the bf16 rounding of the output itself),
weight gradients 0.27 (VGG16's dec1), bias gradients 0.003 whichever kernel sums them, dec1's data-gradient segments
0.99.  Step 1 against fp32: loss relative error 5.4e-6 (VGG11) and 3.4e-5 (VGG16), as the emulation's; training logits
max-abs 1.1e-3 and 1.2e-3 against the emulation's 1.1e-3 and 1.3e-3.  37 of UNet11's 40 gradient tensors and all 50 of
UNetVGG16's are bounded by the emulation; UNet11's centre block (emulated 0.058 .. 0.065) is held to finiteness."""
import gc
import time

import pytest
import torch
import torch.nn.functional as F

import bench
import bench_data
import bench_encoders
from oracle import unet_oracle as O
from oracle import vgg_oracle as V
from oracle.unit_checks import SAMPLE, Bounds, check_conv_half, f64, grad_view, nchw

pytestmark = pytest.mark.gpu

VGG = ["VGG11", "VGG16"]
N, S = 32, 320            # bench_encoders.py's batch and net input
SEED = 1234
LOGIT_TOL = 1e-3
REPRODUCIBLE_REL = 0.05   # test_encoders_vgg_gpu.py: emulated deviation up to which a gradient is bounded tightly
STATS = ("running_mean", "running_var")


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def _rng_and_peak_memory(cuda):
    """leave torch's generators as the other tests expect them; report the device and the peak memory of each test"""
    with torch.random.fork_rng(devices=[cuda]):
        torch.cuda.reset_peak_memory_stats(cuda)
        t0 = time.time()
        yield
    print("\n[%s] peak device memory %.1f GiB, %.0f s" % (torch.cuda.get_device_name(cuda),
                                                           torch.cuda.max_memory_allocated(cuda) / 2 ** 30,
                                                           time.time() - t0))


@pytest.fixture
def no_tf32():
    """a true fp32 reference: cuDNN convolutions default to TF32 (a 10-bit mantissa).  Deterministic cuDNN algorithms
    keep the reference's own rounding the same from run to run."""
    b = torch.backends
    saved = b.cudnn.allow_tf32, b.cuda.matmul.allow_tf32, b.cudnn.deterministic
    b.cudnn.allow_tf32 = b.cuda.matmul.allow_tf32 = False
    b.cudnn.deterministic = True
    yield
    b.cudnn.allow_tf32, b.cuda.matmul.allow_tf32, b.cudnn.deterministic = saved


def vgg_sd(enc):
    with torch.random.fork_rng(devices=[]):
        return V.make_reference_like_state_dict(enc, seed=SEED)


class VGGStep:
    """the fused train step bench_encoders.vgg_fused_step times, on a net loaded with sd"""

    def __init__(self, enc, sd, dev):
        from mcb200.models import FusedTrainStep
        self.cfg, self.lr, self.wd = bench_encoders.vgg_step_settings(enc)
        self.betas, self.eps = (0.9, 0.999), 1e-8          # FusedTrainStep.step's defaults, as the benchmark calls it
        net = bench_encoders.vgg_net(enc)
        net.load_state_dict(sd)
        self.net = net.to(dev)
        self.fused = FusedTrainStep(self.net, (N, 3, S, S), (N, 3, S, S), 0, self.cfg)

    def step(self, X, T):
        return self.fused.step(X, T, lr=self.lr, betas=self.betas, eps=self.eps, weight_decay=self.wd)

    def serial_steps(self, batches):
        """the fused step's own segments, run eagerly in program order on the current stream (see serial_steps below),
        with the Adam scalars FusedTrainStep.step sets.  Yields the loss of every step."""
        from mcb200 import ops
        fused = self.fused
        fused.plan._side = torch.cuda.current_stream()
        for X, T in batches:
            fused.opt.t += 1
            fused._adam_cfg = (self.betas, self.eps, self.wd)
            fused._hyper.copy_(torch.tensor(ops.adam_hyper(self.lr, self.betas, fused.opt.t), dtype=torch.float32))
            fused.plan.x_in.copy_(X)
            fused.target.copy_(T)
            fused._seg_forward()
            fused._loss_partials()
            fused._seg_backward()
            yield fused.loss.reshape(1).clone()


def free_device_memory():
    gc.collect()               # launch plans hold their closures in reference cycles
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def batch(seed, n=N):
    x, t = bench_data.train_batch(n, S, seed=seed)
    return torch.from_numpy(x), torch.from_numpy(t)


def bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float64: torch.int64}[t.dtype])


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(bits(a), bits(b))


def host(t):
    return t.detach().cpu().clone()


def arena_layout(net):
    """[(offset, numel, name)] of the parameter arena, top of the arena first.  The arena follows the forward order of
    the layers (input conv at 0, classifier on top), so this is the order in which the backward pass completes them."""
    return sorted(((net._slots[id(p)].off, p.numel(), name) for name, p, _ in net._arena_params()), reverse=True)


def arena_mismatch(layout, a, b):
    """None when the flat arena tensors a and b are bitwise equal; otherwise the parameter of the difference nearest the
    top of the arena -- the first differing tensor in backward order -- and how many elements differ"""
    ne = torch.nonzero(bits(a) != bits(b)).flatten()
    if ne.numel() == 0:
        return None
    i = int(ne.max())
    for off, numel, name in layout:
        if off <= i:
            inside = i < off + numel
            k = int(((ne >= off) & (ne < off + numel)).sum())
            return "%s (%d of its %d elements differ; %d in the whole arena)" % (
                name if inside else "the alignment padding after " + name, k, numel, ne.numel())
    return "arena element %d" % i


def running_stats(net):
    return {k: host(b) for k, b in net.named_buffers() if k.endswith(STATS)}


def snapshot(net, fused, opt, loss):
    """what one train step left behind, on the host"""
    torch.cuda.synchronize()
    return dict(loss=host(loss), logits=host(fused.plan.logits), g32=host(net._g32), p32=host(net._p32),
                m=host(opt.m), v=host(opt.v), w16=host(net._w16), stats=running_stats(net))


def snapshot_mismatches(layout, a, b):
    """every difference between two snapshots; arena tensors and running statistics named in backward order"""
    out = ["loss %r != %r" % (a["loss"], b["loss"])] if not same_bits(a["loss"], b["loss"]) else []
    if not same_bits(a["logits"], b["logits"]):
        out.append("logits: %d elements differ" % int((bits(a["logits"]) != bits(b["logits"])).sum()))
    for k in ("g32", "p32", "m", "v", "w16"):
        d = arena_mismatch(layout, a[k], b[k])
        if d:
            out.append("%s: first differing tensor %s" % (k, d))
    stats = [k for k in a["stats"] if not same_bits(a["stats"][k], b["stats"][k])]
    if stats:
        out.append("running statistics: %d differ, first in backward order %s" % (len(stats), stats[-1]))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# A. the captured step against the same launches in program order
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("enc", VGG)
def test_captured_step_equals_serial_launch_order(mcb, cuda, enc):
    sd = vgg_sd(enc)
    batches = [tuple(t.to(cuda) for t in batch(SEED + i)) for i in range(3)]

    run = VGGStep(enc, sd, cuda)
    layout = arena_layout(run.net)
    graphed = []
    for i, (X, T) in enumerate(batches):
        graphed.append(snapshot(run.net, run.fused, run.fused.opt, run.step(X, T)))
        assert run.fused.graphs is not None and run.fused.opt.t == i + 1
    del run
    free_device_memory()

    run = VGGStep(enc, sd, cuda)
    for i, loss in enumerate(run.serial_steps(batches)):
        serial = snapshot(run.net, run.fused, run.fused.opt, loss)
        bad = snapshot_mismatches(layout, graphed[i], serial)
        print("%s step %d: loss %.7f, captured == serial: %s" % (enc, i + 1, float(serial["loss"]), not bad))
        assert not bad, "%s step %d (%s): %s" % (enc, i + 1, "eager" if i == 0 else "graph replay", "; ".join(bad))
    assert run.fused.opt.t == 3
    assert len({float(g["loss"]) for g in graphed}) == 3, "distinct batches must give distinct losses"
    del run, graphed
    free_device_memory()


# ---------------------------------------------------------------------------------------------------------------------
# B. Adam of the step's own gradients
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("enc", VGG)
def test_fused_adam_is_adam_of_the_steps_own_gradients(mcb, cuda, enc):
    from mcb200 import ops
    run = VGGStep(enc, vgg_sd(enc), cuda)
    net, opt = run.net, run.fused.opt
    layout = arena_layout(net)
    for i in range(3):
        X, T = (t.to(cuda) for t in batch(SEED + 10 + i))
        p, m, v = net._p32.clone(), opt.m.clone(), opt.v.clone()
        run.step(X, T)
        assert opt.t == i + 1
        assert bool(net._g32.any()) and not same_bits(p, net._p32), "the step must compute gradients and move weights"
        w16 = torch.zeros_like(net._w16)
        ops.adam_step(p, net._g32, m, v, w16, opt.t, run.lr, run.betas, run.eps, run.wd, 1.0)
        bad = ["%s: first differing tensor %s" % (k, d) for k, d in
               (("p32", arena_mismatch(layout, net._p32, p)), ("m", arena_mismatch(layout, opt.m, m)),
                ("v", arena_mismatch(layout, opt.v, v)), ("w16", arena_mismatch(layout, net._w16, w16)),
                ("w16 against bf16(p32)", arena_mismatch(layout, net._w16, net._p32.to(torch.bfloat16)))) if d]
        print("%s step %d: fused Adam == whole-arena Adam of the step's gradients: %s" % (enc, i + 1, not bad))
        assert not bad, "%s step %d (%s): %s" % (enc, i + 1, "eager" if i == 0 else "graph replay", "; ".join(bad))
        del p, m, v, w16
    del run, net, opt
    free_device_memory()


# ---------------------------------------------------------------------------------------------------------------------
# U. every unit against float64 on the step's own buffers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("enc", VGG)
def test_every_unit_against_float64(mcb, cuda, enc):
    """one eager step, then every unit of the plan re-computed in float64 from the step's own buffers"""
    sd = vgg_sd(enc)
    run = VGGStep(enc, sd, cuda)
    X, T = (t.to(cuda) for t in batch(SEED))
    run.step(X, T)
    torch.cuda.synchronize()
    net, plan = run.net, run.fused.plan
    w16 = {k: f64(v.to(cuda, torch.bfloat16)) for k, v in sd.items() if k.endswith(".weight")}
    b32 = {k: f64(v.to(cuda)) for k, v in sd.items() if k.endswith(".bias")}
    stage_outputs = set()
    first_of_stage = {}
    for kind, prefix, ins, out in plan.units:
        if kind == "conv":
            idx = int(prefix.split(".")[1])
            for si, st in enumerate(net._stages):
                if idx == st[-1]:
                    stage_outputs.add(id(out))
                if idx == st[0] and ins:
                    first_of_stage[si] = ins[0]       # the pooled output of the stage before
    bd = Bounds()
    for kind, prefix, ins, out in plan.units:
        g = plan.grad[id(out)]
        if kind == "conv":
            # the input conv reads the image, rounded to bf16 by the im2col
            x = nchw(ins[0]) if ins else plan.x_in.to(torch.bfloat16)
            src = "pool-skip kernel" if id(out) in stage_outputs else "dgrad epilogue"
            check_conv_half(bd, net, w16, b32, prefix, prefix + ".weight", prefix + ".bias", x, out, g, src)
        elif prefix == "dec1":
            x = torch.cat([nchw(a) for a in ins], 1)
            check_conv_half(bd, net, w16, b32, prefix, "dec1.conv.weight", "dec1.conv.bias", x, out, g, "channel_sum")
            # both data-gradient segments of dec1's input: dec2's gradient is dec1's alone, conv1's also holds the
            # pooled path (the first maximum of each 2x2 window)
            d2, c1 = ins
            c2 = d2.shape[3]
            w = w16["dec1.conv.weight"]
            gs = f64(nchw(g)[list(SAMPLE)])
            shape = (len(SAMPLE),) + tuple(x.shape[1:])
            dx = torch.nn.grad.conv2d_input(shape, w, gs, padding=1)
            adx = torch.nn.grad.conv2d_input(shape, w.abs(), gs.abs(), padding=1)
            del gs
            m2 = (f64(nchw(d2)[list(SAMPLE)]) > 0).double()
            bd.check("data gradient (dec1 -> dec2)", "dec2 output", nchw(plan.grad[id(d2)])[list(SAMPLE)],
                     dx[:, :c2] * m2, adx[:, :c2] * m2, rel=2.0 ** -8)
            c1s = f64(nchw(c1)[list(SAMPLE)])
            m1 = (c1s > 0).double()
            _, where = F.max_pool2d(c1s, 2, 2, return_indices=True)
            gp = f64(nchw(plan.grad[id(first_of_stage[1])])[list(SAMPLE)])
            pooled = F.max_unpool2d(gp, where, 2, 2, output_size=c1s.shape[2:])
            skip = dx[:, c2:]
            # two roundings: the skip segment is stored in bf16 before the pool backward adds the pooled path (2^-7:
            # the first rounding's 2^-8 and its share of the second)
            bd.check("data gradient (dec1 -> conv1)", "conv1 output", nchw(plan.grad[id(c1)])[list(SAMPLE)],
                     (skip + pooled) * m1, adx[:, c2:] * m1, rel=2.0 ** -8, extra=2.0 ** -7 * skip.abs() * m1)
            del dx, adx, m2, c1s, m1, where, gp, pooled, skip
        else:
            # decoder block: relu(conv3x3(cat ins) + b) -> relu(convT(.) + b), half by half
            mid = plan.dec_mid[id(out)]
            x = torch.cat([nchw(a) for a in ins], 1) if len(ins) > 1 else nchw(ins[0])
            check_conv_half(bd, net, w16, b32, prefix + ".block.0", prefix + ".block.0.conv.weight",
                            prefix + ".block.0.conv.bias", x, mid, plan.grad[id(mid)], "convT dgrad epilogue")
            src = "dgrad epilogue" if id(out) in plan.bias_fused else "channel_sum"
            check_conv_half(bd, net, w16, b32, prefix + ".block.1", prefix + ".block.1.weight",
                            prefix + ".block.1.bias", nchw(mid), out, g, src, transposed=True)
        del x
    print("%s: %d checks" % (enc, bd.count))
    bd.report()
    n_enc = sum(len(st) for st in net._stages)
    assert len(plan.units) == n_enc + 6
    assert bd.count == 4 * (n_enc + 1 + 2 * 5) + 2, bd.count     # 4 per conv half, dec1's two data-gradient checks
    assert not bd.fails, "\n".join(bd.fails[:20])
    del run, net, plan, w16, b32
    free_device_memory()


# ---------------------------------------------------------------------------------------------------------------------
# D. step 1 against the fp32 reference
# ---------------------------------------------------------------------------------------------------------------------
def vgg_reference_step(sd, enc, X, T, emulate_bf16):
    """one forward, the configured loss and its gradients with oracle.vgg_oracle on X's device: fp32, or with the CUDA
    path's bf16 storage points emulated.  -> host copies of loss, logits, gradients (by parameter name)"""
    work = {k: v.to(X.device, copy=True) for k, v in V.strip_module_prefix(sd).items()}
    keys = V.trainable_keys(work, enc)
    leaves = [work[k].requires_grad_(True) for k in keys]
    logits = V.VGGUNetOracle(work, enc, emulate_bf16=emulate_bf16).forward(X, training=True)
    loss = V.mixed_loss(logits, T, imsize=(256, 256))
    grads = torch.autograd.grad(loss, leaves)
    out = dict(loss=float(loss.detach()), logits=host(logits), grads={k: host(g) for k, g in zip(keys, grads)})
    del work, leaves, logits, loss, grads
    free_device_memory()
    return out


def deviation(got, ref):
    """(relative L2, cosine) in float64"""
    a, b = got.double().reshape(-1), ref.double().reshape(-1)
    return float((a - b).norm() / (b.norm() + 1e-300)), float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


@pytest.mark.parametrize("enc", VGG)
def test_first_step_against_fp32_reference(mcb, cuda, no_tf32, enc):
    """bounds of test_encoders_vgg_gpu.py: loss to 1e-4 relative, logits to max(1e-3, 2 x the emulation's deviation),
    gradients to 1.15 x the emulation's relative L2 deviation + 0.01 wherever the emulation shows bf16 storage leaves
    them reproducible (<= 5 %); the others finite and rel < 1"""
    sd = vgg_sd(enc)
    X, T = (t.to(cuda) for t in batch(SEED))
    ref = vgg_reference_step(sd, enc, X, T, emulate_bf16=False)
    emu = vgg_reference_step(sd, enc, X, T, emulate_bf16=True)
    run = VGGStep(enc, sd, cuda)
    loss = float(run.step(X, T)[0])
    net = run.net
    got = dict(loss=loss, logits=host(run.fused.plan.logits),
               grads={name: host(grad_view(net, name)) for name, _, _ in net._arena_params()})
    del run, net
    free_device_memory()

    fails = []

    def check(ok, line):
        print(("  " if ok else "! ") + line)
        if not ok:
            fails.append(line)

    loss_rel = abs(got["loss"] - ref["loss"]) / abs(ref["loss"])
    check(loss_rel < 1e-4, "loss %.7f, fp32 %.7f: rel %.2e < 1e-4 (emulation rel %.2e)" % (
        got["loss"], ref["loss"], loss_rel, abs(emu["loss"] - ref["loss"]) / abs(ref["loss"])))
    lg = float((got["logits"] - ref["logits"]).abs().max())
    le = float((emu["logits"] - ref["logits"]).abs().max())
    check(lg <= max(LOGIT_TOL, 2.0 * le), "training logits max-abs %.3e <= max(%.0e, 2 x emulation %.3e)" % (
        lg, LOGIT_TOL, le))
    assert set(got["grads"]) == set(ref["grads"]), set(got["grads"]) ^ set(ref["grads"])
    print("  gradient deviation from fp32 (relative L2 / cosine), CUDA path against its bound from the emulation:")
    bounded = 0
    for k in ref["grads"]:
        rel, cos = deviation(got["grads"][k], ref["grads"][k])
        erel, _ = deviation(emu["grads"][k], ref["grads"][k])
        finite = bool(torch.isfinite(got["grads"][k]).all())
        if erel <= REPRODUCIBLE_REL:
            bounded += 1
            check(finite and rel <= 1.15 * erel + 0.01, "%-28s rel %.3e <= 1.15 x %.3e + 0.01 = %.3e   (cos %.6f)" % (
                k, rel, erel, 1.15 * erel + 0.01, cos))
        else:
            check(finite and rel < 1.0, "%-28s rel %.3e < 1 (emulation %.3e: bottleneck, held to finiteness)   "
                  "(cos %.6f)" % (k, rel, erel, cos))
    print("  %d of %d gradient tensors bounded by the emulation" % (bounded, len(ref["grads"])))
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------------------------------------
# ResNet34 (the AlbuNet plan): part A through PyTorchUNetWeighted._fit_loop
# ---------------------------------------------------------------------------------------------------------------------
RESNET34 = "ResNet34"


def resnet34_model(sd):
    from mcb200.models import PyTorchUNetWeighted
    model = PyTorchUNetWeighted(**bench.unet_config(RESNET34))
    model.model.load_state_dict(sd)
    model._to_device()
    return model


def adam_settings(model):
    """what Model._fit_loop hands FusedTrainStep.step"""
    g = model.optimizer.param_groups[0]
    return g["lr"], tuple(g.get("betas", (0.9, 0.999))), g.get("eps", 1e-8), g.get("weight_decay", 0.0)


def serial_steps(model, batches):
    """the fused step's own segments, run eagerly in program order on the current stream: the side stream is the main
    stream, so the weight-gradient GEMMs and the per-segment Adam hooks run exactly where they are issued.  Program order
    is a valid topological order of the step, so this is the schedule-free result of the same launches.  Yields the
    loss of every step."""
    from mcb200 import ops
    net = model._net()
    net.train()
    lr, betas, eps, wd = adam_settings(model)
    fused = model._fused = model._fused_step(net, batches[0][0].shape, batches[0][1].shape, model._loss_spec())
    fused.plan._side = torch.cuda.current_stream()
    for X, T in batches:
        fused.opt.t += 1
        fused._adam_cfg = (betas, eps, wd)
        fused._hyper.copy_(torch.tensor(ops.adam_hyper(lr, betas, fused.opt.t), dtype=torch.float32))
        fused.plan.x_in.copy_(X)
        fused.target.copy_(T)
        fused._seg_forward()
        fused._loss_partials()
        fused._seg_backward()
        yield fused.loss.reshape(1).clone()     # what FusedTrainStep.step returns


def test_resnet34_captured_step_equals_serial_launch_order(mcb, cuda):
    with torch.random.fork_rng(devices=[]):
        sd = O.make_reference_like_state_dict(34, seed=SEED)
    batches = [tuple(t.to(cuda) for t in batch(SEED + i)) for i in range(3)]

    model = resnet34_model(sd)
    layout = arena_layout(model._net())
    graphed = []
    for i, (X, T) in enumerate(batches):
        loss = model._fit_loop([X, T])["sum"]
        graphed.append(snapshot(model._net(), model._fused, model._fused.opt, loss))
        assert (model._fused.graphs is not None) and model._opt_state.t == i + 1
    del model
    free_device_memory()

    model = resnet34_model(sd)
    for i, loss in enumerate(serial_steps(model, batches)):
        serial = snapshot(model._net(), model._fused, model._fused.opt, loss)
        bad = snapshot_mismatches(layout, graphed[i], serial)
        print("ResNet34 step %d: loss %.7f, captured == serial: %s" % (i + 1, float(serial["loss"]), not bad))
        assert not bad, "step %d (%s): %s" % (i + 1, "eager" if i == 0 else "graph replay", "; ".join(bad))
    assert model._opt_state.t == 3
    del model, graphed
    free_device_memory()
