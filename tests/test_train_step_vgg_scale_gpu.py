"""The VGG-encoder U-Nets' train step at the size bench_encoders.py publishes it: UNet11 (VGG11) and UNetVGG16 (VGG16)
at batch 32 and 320x320, built as bench_encoders.vgg_fused_step builds them (oracle.step_checks.BenchStep:
FusedTrainStep with bench.unet_config's loss and Adam settings).  The captured step against program order (A) and
Adam of the step's own gradients (B) run for these nets in test_train_step_scale_gpu.py.

At this size the VGG nets hold the largest tensors of the project: the 64-channel full-resolution activations have
2.1e8 elements, dec1's 96-channel concat input 3.1e8, and the implicit im2col of dec1's 3x3 conv spans 2.8e9 elements,
past 2^31; each per-channel bias sum runs over 3.3 M pixels.  Checked, per net:
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

At most one batch-32 plan is alive at a time.

Measured on an H100 80GB HBM3 at its 700 W power limit: the file takes about 25 s and at most 26.3 GiB of device memory
(test D); U takes 6 s per net.  U's worst |got - ref| / bound: forward 0.99 (the bf16 rounding of the output itself),
weight gradients 0.27 (VGG16's dec1), bias gradients 0.003 whichever kernel sums them, dec1's data-gradient segments
0.99.  Step 1 against fp32: loss relative error 5.4e-6 (VGG11) and 3.4e-5 (VGG16), as the emulation's; training logits
max-abs 1.1e-3 and 1.2e-3 against the emulation's 1.1e-3 and 1.3e-3.  37 of UNet11's 40 gradient tensors and all 50 of
UNetVGG16's are bounded by the emulation; UNet11's centre block (emulated 0.058 .. 0.065) is held to finiteness."""
import pytest
import torch
import torch.nn.functional as F

from oracle.step_checks import (SEED, VGG, BenchStep, batch, deviation, free_device_memory, reference_step, seeded_sd,
                                step_outputs)
from oracle.step_checks import no_tf32, rng_and_peak_memory  # noqa: F401  (fixtures)
from oracle.unit_checks import SAMPLE, Bounds, check_conv_half, f64, nchw

pytestmark = pytest.mark.gpu

LOGIT_TOL = 1e-3
REPRODUCIBLE_REL = 0.05   # test_encoders_vgg_gpu.py: emulated deviation up to which a gradient is bounded tightly


# ---------------------------------------------------------------------------------------------------------------------
# U. every unit against float64 on the step's own buffers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("enc", VGG)
def test_every_unit_against_float64(mcb, cuda, enc):
    """one eager step, then every unit of the plan re-computed in float64 from the step's own buffers"""
    sd = seeded_sd(enc)
    run = BenchStep(enc, sd, cuda)
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
@pytest.mark.parametrize("enc", VGG)
def test_first_step_against_fp32_reference(mcb, cuda, no_tf32, enc):
    """bounds of test_encoders_vgg_gpu.py: loss to 1e-4 relative, logits to max(1e-3, 2 x the emulation's deviation),
    gradients to 1.15 x the emulation's relative L2 deviation + 0.01 wherever the emulation shows bf16 storage leaves
    them reproducible (<= 5 %); the others finite and rel < 1"""
    sd = seeded_sd(enc)
    X, T = (t.to(cuda) for t in batch(SEED))
    ref = reference_step(enc, sd, X, T, emulate_bf16=False)
    emu = reference_step(enc, sd, X, T, emulate_bf16=True)
    run = BenchStep(enc, sd, cuda)
    got = step_outputs(run, run.step(X, T))
    del run
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
