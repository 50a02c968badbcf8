"""The benchmarks' train step end to end at batch 32 and 320x320: PyTorchUNetWeighted._fit_loop on the ResNet101 U-Net
built exactly as bench.py builds it, and the eval forward of its `infer` workload at batch 64; A and B also run on every
other encoder family the benchmarks train at this size (oracle.step_checks.BenchStep): the AlbuNet-wired ResNet34 plan
through _fit_loop, UNet11 (VGG11) and UNetVGG16 (VGG16) through FusedTrainStep as bench_encoders.py builds them.

The kernels are tested one at a time elsewhere; what only the composed step does is checked here, at the size where its
streams really overlap:
  A. the captured step (side-stream weight gradients, Adam hooks inside the backward graph, graph replays) equals the
     same launches run eagerly in program order on one stream, bit for bit, for three distinct batches.  In program
     order a segment's Adam hook runs exactly where it is issued, so a segment bound of the plan that takes in a
     parameter whose gradient is finished later fails here deterministically.  ResNet101, ResNet34, VGG11, VGG16;
  B. every step's weights and Adam moments are exactly Adam of that step's own final gradients over the whole arena,
     and the bf16 operand copy is exactly the new fp32 weights: a segment hook that fired before its gradients were
     complete, segments that do not tile the arena, or a skipped bf16 refresh all break this.  ResNet101, VGG11, VGG16;
  C. pinned host batches through the double-buffered staging ring, graph replays and the partial last batch of an epoch
     (a second captured step sharing Adam's state) train exactly like the same batches handed over on the device;
  D. step 1 against the fp32 reference (oracle.unet_oracle on the GPU, TF32 off) with the bounds of
     test_unet_configs_gpu.py, the CUDA path measured against a bf16-storage emulation of the same step;
  E. the eval forward (BatchNorm folded into the conv epilogues) on two different batches of 64, eager then graph
     replay, against the fp32 eval reference.
C, D and E are ResNet101's.

Exact equality is the bar of A, B and C: every cross-CTA sum of the step is added in a fixed order
(test_train_step_gpu.py::test_fused_train_steps_are_bitwise_reproducible).  At most one batch-32 plan is alive at a
time; what is compared across runs is kept on the host.

Measured on an H100 80GB HBM3 at its 700 W power limit: the file takes about 90 s and at most 24.5 GiB of device memory
(test D); A takes 24 s on ResNet101 and 8-12 s on each other net.  Step 1 against fp32: loss relative error 8.3e-6,
training logits max-abs 1.5e-4 (the emulation's: 1.6e-4).  The CUDA path is closer to fp32 than the emulation on 174 of
the 340 gradient tensors, and the cosine differences between the two spread about +-0.05 both ways: that is the storage
format's own spread at this size, and the tightest tensor (encoder.layer3.11.bn1.weight, cosine 0.7752 against a bound
of 0.7746) sits at its edge.  Eval logits at batch 64: max-abs 1.5e-4."""
import pytest
import torch

import bench
import bench_data
from oracle import unet_oracle as O
from oracle.step_checks import (N, S, SEED, BenchStep, arena_layout, arena_mismatch, batch, check_adam_of_own_gradients,
                                check_captured_equals_serial, deviation, free_device_memory, host, reference_step,
                                running_stats, same_bits, seeded_sd, step_outputs)
from oracle.step_checks import no_tf32, rng_and_peak_memory  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

ENCODER = "ResNet101"
DEPTH = 101
N_PARTIAL = 20            # the last batch of an epoch (the reference's DataLoader has no drop_last)
N_INFER = 64              # bench.py --workload infer
LOGIT_TOL = 1e-3          # BASELINE.json north star
DECODER_TAIL = ("dec1.block.1.weight", "dec0.conv.weight", "final.weight", "final.bias")


@pytest.fixture(scope="module")
def conditioned_sd():
    """the conditioned checkpoint (raw-init deep gradients are chaotic, see test_unet_configs_gpu.py); the conditioning
    pass only sets the running statistics, so four tiles on the CPU are enough"""
    x, _ = bench_data.train_batch(N, S, seed=SEED)
    with torch.random.fork_rng(devices=[]):
        return O.conditioned_state_dict(DEPTH, torch.from_numpy(x[:4]), seed=SEED)


# ---------------------------------------------------------------------------------------------------------------------
# A. the captured step against the same launches in program order
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("enc", ["ResNet101", "ResNet34", "VGG11", "VGG16"])
def test_captured_step_equals_serial_launch_order(mcb, cuda, enc):
    check_captured_equals_serial(enc, cuda)


# ---------------------------------------------------------------------------------------------------------------------
# B. Adam of the step's own gradients
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("enc", ["ResNet101", "VGG11", "VGG16"])
def test_fused_adam_is_adam_of_the_steps_own_gradients(mcb, cuda, enc):
    check_adam_of_own_gradients(enc, cuda)


# ---------------------------------------------------------------------------------------------------------------------
# C. host staging, replays and the partial batch
# ---------------------------------------------------------------------------------------------------------------------
def test_host_staged_batches_and_partial_batch_train_like_device_batches(mcb, cuda):
    """A, B, C, P, A with P the 20-tile last batch of an epoch.  The host run does not synchronise between steps, like
    bench.py's e2e arm, so the staging ring's slots really are in flight while the previous step computes."""
    sd = seeded_sd(ENCODER)
    a, b, c, p = batch(SEED + 20), batch(SEED + 21), batch(SEED + 22), batch(SEED + 23, N_PARTIAL)
    seq = [a, b, c, p, a]
    runs = {}
    for where in ("device", "host"):
        if where == "device":
            data = [tuple(t.to(cuda) for t in xt) for xt in seq]
        else:
            data = [tuple(t.pin_memory() for t in xt) for xt in seq]
        run = BenchStep(ENCODER, sd, cuda)
        losses = [run.step(*xt) for xt in data]
        torch.cuda.synchronize()
        net, st = run.net, run.fused.opt
        assert len(run.model._fused_cache) == 2 and st.t == 5, (where, len(run.model._fused_cache), st.t)
        runs[where] = dict(losses=[host(l) for l in losses], p32=host(net._p32), m=host(st.m), v=host(st.v),
                           stats=running_stats(net), layout=arena_layout(net))
        del run, net, st, losses, data
        free_device_memory()
    d, h = runs["device"], runs["host"]
    print("losses, device batches: %s" % [float(l) for l in d["losses"]])
    print("losses, host batches:   %s" % [float(l) for l in h["losses"]])
    assert len({float(l) for l in d["losses"]}) == 5, "distinct batches must give distinct losses"
    for i, (x, y) in enumerate(zip(d["losses"], h["losses"])):
        assert same_bits(x, y), "step %d: loss %r from host batches, %r from device batches" % (i + 1, float(y), float(x))
    bad = ["%s: first differing tensor %s" % (k, e) for k in ("p32", "m", "v")
           for e in [arena_mismatch(d["layout"], d[k], h[k])] if e]
    bad += [k for k in d["stats"] if not same_bits(d["stats"][k], h["stats"][k])]
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------
# D. step 1 against the fp32 reference
# ---------------------------------------------------------------------------------------------------------------------
def test_first_step_against_fp32_reference(mcb, cuda, conditioned_sd, no_tf32):
    """bounds of test_unet_configs_gpu.py: the CUDA path may not be farther from fp32 than the bf16 storage format alone
    puts the emulation, tensor by tensor"""
    X, T = (t.to(cuda) for t in batch(SEED))
    ref = reference_step(ENCODER, conditioned_sd, X, T, emulate_bf16=False)
    emu = reference_step(ENCODER, conditioned_sd, X, T, emulate_bf16=True)
    run = BenchStep(ENCODER, conditioned_sd, cuda)
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
    check(lg <= LOGIT_TOL, "training logits max-abs %.3e <= %.0e" % (lg, LOGIT_TOL))
    check(lg <= 1.15 * le + 1e-4, "training logits max-abs %.3e <= 1.15 x emulation %.3e + 1e-4 = %.3e" % (
        lg, le, 1.15 * le + 1e-4))
    assert set(got["grads"]) == set(ref["grads"]), set(got["grads"]) ^ set(ref["grads"])
    print("  gradient deviation from fp32 (relative L2 / cosine), CUDA path against its bound from the emulation:")
    closer = 0
    for k in ref["grads"]:
        rel, cos = deviation(got["grads"][k], ref["grads"][k])
        erel, ecos = deviation(emu["grads"][k], ref["grads"][k])
        closer += rel < erel
        check(rel <= 1.15 * erel + 0.01 and cos >= ecos - 0.05,
              "%-44s rel %.3e <= %.3e   cos %.6f >= %.6f" % (k, rel, 1.15 * erel + 0.01, cos, ecos - 0.05))
        if k in DECODER_TAIL:
            check(rel < 2e-2, "%-44s rel %.3e < 2e-2 (decoder tail)" % (k, rel))
    print("  the CUDA path is closer to fp32 than the emulation on %d of %d gradient tensors" % (closer, len(ref["grads"])))
    worst = (-1.0, "")
    for k, r in ref["stats"].items():
        g = got["stats"][k]
        if not torch.allclose(g, r, rtol=2e-2, atol=1e-3):
            fails.append("running statistic %s: max-abs %.3e" % (k, float((g - r).abs().max())))
        e = float(((g - r).abs() / (1e-3 + 2e-2 * r.abs())).max())
        worst = max(worst, (e, k))
    check(not any(f.startswith("running") for f in fails),
          "running statistics: largest |got - fp32| / (1e-3 + 2e-2 |fp32|) = %.3f <= 1 (%s)" % worst)
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------------------------------------
# E. the infer workload's eval forward
# ---------------------------------------------------------------------------------------------------------------------
def test_infer_eval_forward_against_fp32_reference(mcb, cuda, conditioned_sd, no_tf32):
    """bench.py --workload infer: net.eval() under no_grad at batch 64; the first batch runs eagerly (and is captured),
    the second, different batch is a graph replay"""
    from mcb200 import ops
    from mcb200.models import PyTorchUNet
    model = PyTorchUNet(**bench.unet_config(ENCODER))
    model.model.load_state_dict(conditioned_sd)
    model._to_device()
    net = model.model
    net.eval()
    plan = net.plan(N_INFER, S, S, False)
    work = {k: v.to(cuda) for k, v in O.strip_module_prefix(conditioned_sd).items()}
    for i, seed in enumerate((SEED + 30, SEED + 31)):
        X = batch(seed, N_INFER)[0].to(cuda)
        assert (plan.graph_fwd is not None) == (i == 1)
        with torch.no_grad():
            ref = O.UNetOracle(work, DEPTH).forward(X, training=False)
            logits = net(X)
            probs = ops.softmax2(logits)
            e_logits = float((logits - ref).abs().max())
            e_probs = float((probs - torch.softmax(ref, 1)).abs().max())
        print("batch %d (%s): logits max-abs %.3e <= %.0e, softmax max-abs %.3e <= %.0e" % (
            i + 1, "graph replay" if i else "eager", e_logits, LOGIT_TOL, e_probs, LOGIT_TOL))
        assert e_logits <= LOGIT_TOL and e_probs <= LOGIT_TOL, (i, e_logits, e_probs)
        del X, ref, logits, probs
    del model, net, plan, work
    free_device_memory()
