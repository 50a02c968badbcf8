"""The benchmark's train step end to end: PyTorchUNetWeighted._fit_loop on the ResNet101 U-Net at batch 32 and 320x320,
built exactly as bench.py builds it, and the eval forward of its `infer` workload at batch 64.

The kernels are tested one at a time elsewhere; what only the composed step does is checked here, at the size where its
streams really overlap:
  A. the captured step (side-stream weight gradients, Adam hooks inside the backward graph, graph replays) equals the
     same launches run eagerly in program order on one stream, bit for bit, for three distinct batches;
  B. every step's weights and Adam moments are exactly Adam of that step's own final gradients over the whole arena,
     and the bf16 operand copy is exactly the new fp32 weights: a segment hook that fired before its gradients were
     complete, segments that do not tile the arena, or a skipped bf16 refresh all break this;
  C. pinned host batches through the double-buffered staging ring, graph replays and the partial last batch of an epoch
     (a second captured step sharing Adam's state) train exactly like the same batches handed over on the device;
  D. step 1 against the fp32 reference (oracle.unet_oracle on the GPU, TF32 off) with the bounds of
     test_unet_configs_gpu.py, the CUDA path measured against a bf16-storage emulation of the same step;
  E. the eval forward (BatchNorm folded into the conv epilogues) on two different batches of 64, eager then graph
     replay, against the fp32 eval reference.

Exact equality is the bar of A, B and C: every cross-CTA sum of the step is added in a fixed order
(test_train_step_gpu.py::test_fused_train_steps_are_bitwise_reproducible).  At most one ResNet101 plan at batch 32 is
alive at a time; what is compared across runs is kept on the host.

Measured on an H100 80GB HBM3 at its 700 W power limit: the file takes about 70 s and at most 28.6 GiB of device memory
(test C).  Step 1 against fp32: loss relative error 8.3e-6, training logits max-abs 1.5e-4 (the emulation's: 1.6e-4).
The CUDA path is closer to fp32 than the emulation on 174 of the 340 gradient tensors, and the cosine differences
between the two spread about +-0.05 both ways: that is the storage format's own spread at this size, and the tightest
tensor (encoder.layer3.11.bn1.weight, cosine 0.7752 against a bound of 0.7746) sits at its edge.  Eval logits at
batch 64: max-abs 1.5e-4."""
import gc
import time

import pytest
import torch

import bench
import bench_data
from oracle import unet_oracle as O

pytestmark = pytest.mark.gpu

ENCODER = "ResNet101"
DEPTH = 101
N, S = 32, 320            # bench.py's train batch and net input
N_PARTIAL = 20            # the last batch of an epoch (the reference's DataLoader has no drop_last)
N_INFER = 64              # bench.py --workload infer
SEED = 1234
LOGIT_TOL = 1e-3          # BASELINE.json north star
DECODER_TAIL = ("dec1.block.1.weight", "dec0.conv.weight", "final.weight", "final.bias")
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
    keep the reference's own rounding the same from run to run: the deep gradients compared here are sensitive to it."""
    b = torch.backends
    saved = b.cudnn.allow_tf32, b.cuda.matmul.allow_tf32, b.cudnn.deterministic
    b.cudnn.allow_tf32 = b.cuda.matmul.allow_tf32 = False
    b.cudnn.deterministic = True
    yield
    b.cudnn.allow_tf32, b.cuda.matmul.allow_tf32, b.cudnn.deterministic = saved


@pytest.fixture(scope="module")
def conditioned_sd():
    """the conditioned checkpoint (raw-init deep gradients are chaotic, see test_unet_configs_gpu.py); the conditioning
    pass only sets the running statistics, so four tiles on the CPU are enough"""
    x, _ = bench_data.train_batch(N, S, seed=SEED)
    with torch.random.fork_rng(devices=[]):
        return O.conditioned_state_dict(DEPTH, torch.from_numpy(x[:4]), seed=SEED)


def raw_sd():
    with torch.random.fork_rng(devices=[]):
        return O.make_reference_like_state_dict(DEPTH, seed=SEED)


def new_model(sd, cls=None):
    from mcb200.models import PyTorchUNetWeighted
    model = (cls or PyTorchUNetWeighted)(**bench.unet_config(ENCODER))
    model.model.load_state_dict(sd)
    model._to_device()
    return model


def free_device_memory():
    gc.collect()               # launch plans hold their closures in reference cycles
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def batch(seed, n=N):
    x, t = bench_data.train_batch(n, S, seed=seed)
    return torch.from_numpy(x), torch.from_numpy(t)


def adam_settings(model):
    """what Model._fit_loop hands FusedTrainStep.step"""
    g = model.optimizer.param_groups[0]
    return g["lr"], tuple(g.get("betas", (0.9, 0.999))), g.get("eps", 1e-8), g.get("weight_decay", 0.0)


def bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float64: torch.int64}[t.dtype])


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(bits(a), bits(b))


def host(t):
    return t.detach().cpu().clone()


def arena_layout(net):
    """[(offset, numel, name)] of the parameter arena, top of the arena first.  The arena follows the forward order of
    the layers (stem at 0, classifier on top), so this is the order in which the backward pass completes them."""
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


def snapshot(model, loss):
    """what one train step left behind, on the host"""
    net, fused = model._net(), model._fused
    torch.cuda.synchronize()
    return dict(loss=host(loss), logits=host(fused.plan.logits), g32=host(net._g32), p32=host(net._p32),
                m=host(fused.opt.m), v=host(fused.opt.v), w16=host(net._w16), stats=running_stats(net))


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


def reference_step(sd, X, T, emulate_bf16):
    """one train-mode forward, the configured loss and its gradients with oracle.unet_oracle on X's device: fp32, or with
    the CUDA path's bf16 storage points emulated.  -> host copies of loss, logits, gradients (by parameter name) and the
    running statistics after the step"""
    work = {k: v.to(X.device, copy=True) for k, v in O.strip_module_prefix(sd).items()}
    keys = O.trainable_keys(work)
    leaves = [work[k].requires_grad_(True) for k in keys]
    logits = O.UNetOracle(work, DEPTH, emulate_bf16=emulate_bf16).forward(X, training=True)
    loss = O.mixed_loss(logits, T, imsize=(256, 256))
    grads = torch.autograd.grad(loss, leaves)
    out = dict(loss=float(loss.detach()), logits=host(logits), grads={k: host(g) for k, g in zip(keys, grads)},
               stats={k: host(v) for k, v in work.items() if k.startswith("encoder.") and k.endswith(STATS)})
    del work, leaves, logits, loss, grads
    free_device_memory()
    return out


def deviation(got, ref):
    """(relative L2, cosine) in float64"""
    a, b = got.double().reshape(-1), ref.double().reshape(-1)
    return float((a - b).norm() / (b.norm() + 1e-300)), float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


def cuda_step_outputs(model, loss):
    net = model._net()
    grads = {name: host(net._view(net._g32, net._slots[id(p)])) for name, p, _ in net._arena_params()}
    return dict(loss=float(loss), logits=host(model._fused.plan.logits), grads=grads, stats=running_stats(net))


# ---------------------------------------------------------------------------------------------------------------------
# A. the captured step against the same launches in program order
# ---------------------------------------------------------------------------------------------------------------------
def test_captured_step_equals_serial_launch_order(mcb, cuda):
    sd = raw_sd()
    batches = [tuple(t.to(cuda) for t in batch(SEED + i)) for i in range(3)]

    model = new_model(sd)
    layout = arena_layout(model._net())
    graphed = []
    for i, (X, T) in enumerate(batches):
        graphed.append(snapshot(model, model._fit_loop([X, T])["sum"]))
        assert (model._fused.graphs is not None) and model._opt_state.t == i + 1
    del model
    free_device_memory()

    model = new_model(sd)
    for i, loss in enumerate(serial_steps(model, batches)):
        serial = snapshot(model, loss)
        bad = snapshot_mismatches(layout, graphed[i], serial)
        print("step %d: loss %.7f, captured == serial: %s" % (i + 1, float(serial["loss"]), not bad))
        assert not bad, "step %d (%s): %s" % (i + 1, "eager" if i == 0 else "graph replay", "; ".join(bad))
    assert model._opt_state.t == 3
    del model, graphed
    free_device_memory()


# ---------------------------------------------------------------------------------------------------------------------
# B. Adam of the step's own gradients
# ---------------------------------------------------------------------------------------------------------------------
def test_fused_adam_is_adam_of_the_steps_own_gradients(mcb, cuda):
    from mcb200 import ops
    model = new_model(raw_sd())
    net = model._net()
    layout = arena_layout(net)
    lr, betas, eps, wd = adam_settings(model)
    for i in range(3):
        X, T = (t.to(cuda) for t in batch(SEED + 10 + i))
        st = model._opt_state
        p = net._p32.clone()
        m, v = (st.m.clone(), st.v.clone()) if st is not None else (torch.zeros_like(p), torch.zeros_like(p))
        model._fit_loop([X, T])
        st = model._opt_state
        assert st.t == i + 1
        assert bool(net._g32.any()) and not same_bits(p, net._p32), "the step must compute gradients and move weights"
        w16 = torch.zeros_like(net._w16)
        ops.adam_step(p, net._g32, m, v, w16, st.t, lr, betas, eps, wd, 1.0)
        bad = ["%s: first differing tensor %s" % (k, d) for k, d in
               (("p32", arena_mismatch(layout, net._p32, p)), ("m", arena_mismatch(layout, st.m, m)),
                ("v", arena_mismatch(layout, st.v, v)), ("w16", arena_mismatch(layout, net._w16, w16)),
                ("w16 against bf16(p32)", arena_mismatch(layout, net._w16, net._p32.to(torch.bfloat16)))) if d]
        print("step %d: fused Adam == whole-arena Adam of the step's gradients: %s" % (i + 1, not bad))
        assert not bad, "step %d (%s): %s" % (i + 1, "eager" if i == 0 else "graph replay", "; ".join(bad))
        del p, m, v, w16
    del model
    free_device_memory()


# ---------------------------------------------------------------------------------------------------------------------
# C. host staging, replays and the partial batch
# ---------------------------------------------------------------------------------------------------------------------
def test_host_staged_batches_and_partial_batch_train_like_device_batches(mcb, cuda):
    """A, B, C, P, A with P the 20-tile last batch of an epoch.  The host run does not synchronise between steps, like
    bench.py's e2e arm, so the staging ring's slots really are in flight while the previous step computes."""
    sd = raw_sd()
    a, b, c, p = batch(SEED + 20), batch(SEED + 21), batch(SEED + 22), batch(SEED + 23, N_PARTIAL)
    seq = [a, b, c, p, a]
    runs = {}
    for where in ("device", "host"):
        if where == "device":
            data = [tuple(t.to(cuda) for t in xt) for xt in seq]
        else:
            data = [tuple(t.pin_memory() for t in xt) for xt in seq]
        model = new_model(sd)
        losses = [model._fit_loop(list(xt))["sum"] for xt in data]
        torch.cuda.synchronize()
        net, st = model._net(), model._opt_state
        assert len(model._fused_cache) == 2 and st.t == 5, (where, len(model._fused_cache), st.t)
        runs[where] = dict(losses=[host(l) for l in losses], p32=host(net._p32), m=host(st.m), v=host(st.v),
                           stats=running_stats(net), layout=arena_layout(net))
        del model, net, st, losses, data
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
    ref = reference_step(conditioned_sd, X, T, emulate_bf16=False)
    emu = reference_step(conditioned_sd, X, T, emulate_bf16=True)
    model = new_model(conditioned_sd)
    got = cuda_step_outputs(model, model._fit_loop([X, T])["sum"])
    del model
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
    model = new_model(conditioned_sd, PyTorchUNet)
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
