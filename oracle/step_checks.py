"""TEST INFRASTRUCTURE -- the harness of the train-step tests at the benchmarks' sizes
(tests/test_train_step_scale_gpu.py, tests/test_train_step_vgg_scale_gpu.py, tests/test_train_step_resnet_units_gpu.py
at batch 32 and 320x320, tests/test_train_step_config5_gpu.py at BASELINE.json config 5's batch 16 and 512x512,
tests/test_train_step_ragged_batch_gpu.py at batch 20 and partial batches, tests/test_train_run_lifecycle_gpu.py across
a training run's callbacks), and the helpers the golden-fixture encoder tests share.  Never imported by the product path.

BenchStep is the train step the benchmarks time, for every encoder family they run, at batch n and sxs (N and S, the
default, are bench.py's): the ResNets through PyTorchUNetWeighted._fit_loop as bench.py builds it, VGG11 and VGG16
through FusedTrainStep as bench_encoders.py builds them.  Its serial_steps is the only code of the tests that reaches
into FusedTrainStep's private state.

What the tests compare across runs is kept on the host: snapshot / snapshot_mismatches compare two train steps bit for
bit, and name a difference by the parameter it falls in, in backward order.

A test module imports the fixtures rng_and_peak_memory (autouse: it applies to every test of the module that imports
it) and no_tf32 by name; pytest collects fixtures from a module's globals."""
import gc
import time

import numpy as np
import pytest
import torch

import bench
import bench_data
import bench_encoders
from oracle import unet_oracle as O
from oracle import vgg_oracle as V
from oracle.make_golden_encoders import golden_path
from oracle.unit_checks import nchw

N, S = 32, 320            # bench.py's and bench_encoders.py's train batch and net input
SEED = 1234
RESNET_DEPTH = {"ResNet101": 101, "ResNet34": 34}     # the ResNets trained at batch N and SxS
CONFIG5 = "ResNet152"                                  # BASELINE.json config 5: bench.py --encoder 152 --batch 16
N5, S5 = 16, 512                                       # --size 512
DEPTH = dict(RESNET_DEPTH, **{CONFIG5: 152})           # every ResNet encoder the harness builds
VGG = ("VGG11", "VGG16")
STATS = ("running_mean", "running_var")


# ---------------------------------------------------------------------------------------------------------------------
# fixtures
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def rng_and_peak_memory(cuda):
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


# ---------------------------------------------------------------------------------------------------------------------
# the train step of each encoder family
# ---------------------------------------------------------------------------------------------------------------------
def seeded_sd(enc):
    """the reference-like raw initialisation of `enc`'s U-Net at SEED"""
    with torch.random.fork_rng(devices=[]):
        if enc in VGG:
            return V.make_reference_like_state_dict(enc, seed=SEED)
        return O.make_reference_like_state_dict(DEPTH[enc], seed=SEED)


class BenchStep:
    """the train step the benchmarks time for `enc`, on a net loaded with sd, at batch n and sxs.  fused is that
    FusedTrainStep (for the ResNets the one PyTorchUNetWeighted._fit_loop caches for this shape); adam is what the step
    hands it: (lr, betas, eps, weight_decay)"""

    def __init__(self, enc, sd, dev, n=N, s=S):
        from mcb200.models import FusedTrainStep, PyTorchUNetWeighted
        shape = (n, 3, s, s)
        if enc in VGG:
            cfg, lr, wd = bench_encoders.vgg_step_settings(enc)
            self.adam = (lr, (0.9, 0.999), 1e-8, wd)        # FusedTrainStep.step's defaults, as the benchmark calls it
            net = bench_encoders.vgg_net(enc)
            net.load_state_dict(sd)
            self.model, self.net = None, net.to(dev)
            self.fused = FusedTrainStep(self.net, shape, shape, 0, cfg)
        else:
            model = PyTorchUNetWeighted(**bench.unet_config(enc))
            model.model.load_state_dict(sd)
            model._to_device()
            g = model.optimizer.param_groups[0]             # what Model._fit_loop hands FusedTrainStep.step
            self.adam = (g["lr"], tuple(g.get("betas", (0.9, 0.999))), g.get("eps", 1e-8), g.get("weight_decay", 0.0))
            self.model, self.net = model, model._net()
            self.net.train()
            self.fused = model._fused_step(self.net, shape, shape, model._loss_spec())

    def step(self, X, T):
        """one train step as the benchmark runs it -> the loss, shape (1,).  For the ResNets, fused follows the batch
        shape: it is the captured step _fit_loop ran"""
        if self.model is not None:
            loss = self.model._fit_loop([X, T])["sum"]
            self.fused = self.model._fused
            return loss
        lr, betas, eps, wd = self.adam
        return self.fused.step(X, T, lr=lr, betas=betas, eps=eps, weight_decay=wd)

    def is_replay(self, X, T):
        """whether the next step on (X, T) replays captured graphs (the first step of a shape runs eagerly)"""
        f = self.fused if self.model is None else self.model._fused_cache.get((tuple(X.shape), tuple(T.shape)))
        return f is not None and f.graphs is not None

    def lr(self):
        """the learning rate the next step hands Adam: the optimizer's, which a scheduler may change between steps"""
        return self.adam[0] if self.model is None else self.model.optimizer.param_groups[0]["lr"]

    def serial_steps(self, batches):
        """the fused step's own segments, run eagerly in program order on the current stream, with the Adam scalars
        FusedTrainStep.step sets: the side stream is the main stream, so the weight-gradient GEMMs and the per-segment
        Adam hooks run exactly where they are issued.  Program order is a valid topological order of the step, so this
        is the schedule-free result of the same launches.  For the ResNets a batch of another shape runs the captured
        step _fit_loop keeps for that shape, sharing the one Adam state.  Yields the loss of every step."""
        from mcb200 import ops
        lr, betas, eps, wd = self.adam
        for X, T in batches:
            if self.model is not None:
                self.fused = self.model._fused_step(self.net, X.shape, T.shape, self.model._loss_spec())
            fused = self.fused
            fused.plan._side = torch.cuda.current_stream()
            fused.opt.t += 1
            fused._adam_cfg = (betas, eps, wd)
            fused._hyper.copy_(torch.tensor(ops.adam_hyper(lr, betas, fused.opt.t), dtype=torch.float32))
            fused.plan.x_in.copy_(X)
            fused.target.copy_(T)
            fused._seg_forward()
            fused._loss_partials()
            fused._seg_backward()
            yield fused.loss.reshape(1).clone()     # what FusedTrainStep.step returns


def free_device_memory():
    gc.collect()               # launch plans hold their closures in reference cycles
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def batch(seed, n=N, s=S):
    x, t = bench_data.train_batch(n, s, seed=seed)
    return torch.from_numpy(x), torch.from_numpy(t)


# ---------------------------------------------------------------------------------------------------------------------
# bitwise comparison of train steps
# ---------------------------------------------------------------------------------------------------------------------
def bits(t):
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float64: torch.int64}[t.dtype])


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(bits(a), bits(b))


def host(t):
    return t.detach().cpu().clone()


def arena_layout(net):
    """[(offset, numel, name)] of the parameter arena, top of the arena first.  The arena follows the forward order of
    the layers (stem or input conv at 0, classifier on top), so this is the order in which the backward pass completes
    them."""
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


def snapshot(run, loss):
    """what one train step of the BenchStep run left behind, on the host"""
    net, fused = run.net, run.fused
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


# ---------------------------------------------------------------------------------------------------------------------
# the composed step: the captured step against program order (A), Adam against the step's own gradients (B)
# ---------------------------------------------------------------------------------------------------------------------
def check_captured_equals_serial(enc, cuda, n=N, s=S):
    """three distinct batches through the captured step (eager, then graph replays) and through the same launches in
    program order (BenchStep.serial_steps) on a fresh net: every snapshot bitwise equal.  One plan alive at a time"""
    sd = seeded_sd(enc)
    batches = [tuple(t.to(cuda) for t in batch(SEED + i, n, s)) for i in range(3)]

    run = BenchStep(enc, sd, cuda, n, s)
    layout = arena_layout(run.net)
    graphed = []
    for i, (X, T) in enumerate(batches):
        graphed.append(snapshot(run, run.step(X, T)))
        assert run.fused.graphs is not None and run.fused.opt.t == i + 1
    del run
    free_device_memory()

    run = BenchStep(enc, sd, cuda, n, s)
    for i, loss in enumerate(run.serial_steps(batches)):
        serial = snapshot(run, loss)
        bad = snapshot_mismatches(layout, graphed[i], serial)
        print("%s step %d: loss %.7f, captured == serial: %s" % (enc, i + 1, float(serial["loss"]), not bad))
        assert not bad, "%s step %d (%s): %s" % (enc, i + 1, "eager" if i == 0 else "graph replay", "; ".join(bad))
    assert run.fused.opt.t == 3
    assert len({float(g["loss"]) for g in graphed}) == 3, "distinct batches must give distinct losses"
    del run, graphed
    free_device_memory()


def adam_mismatches(run, layout, X, T):
    """one run.step on (X, T), then every difference between what it left and whole-arena Adam (ops.adam_step) of the
    step's own final gradients from the pre-step p32, m and v, with the learning rate the optimizer held when the step
    ran and the step count t it ran at: p32, m, v, the bf16 operand copy, and the operand copy against bf16(p32).
    -> (loss, list of differences)"""
    from mcb200 import ops
    net = run.net
    opt = run.fused.opt
    _, betas, eps, wd = run.adam
    lr, t = run.lr(), opt.t + 1
    p, m, v = net._p32.clone(), opt.m.clone(), opt.v.clone()
    loss = run.step(X, T)
    opt = run.fused.opt
    assert opt.t == t, "the step must count once: t %d, expected %d" % (opt.t, t)
    assert bool(net._g32.any()) and not same_bits(p, net._p32), "the step must compute gradients and move weights"
    w16 = torch.zeros_like(net._w16)
    ops.adam_step(p, net._g32, m, v, w16, t, lr, betas, eps, wd, 1.0)
    bad = ["%s: first differing tensor %s" % (k, d) for k, d in
           (("p32", arena_mismatch(layout, net._p32, p)), ("m", arena_mismatch(layout, opt.m, m)),
            ("v", arena_mismatch(layout, opt.v, v)), ("w16", arena_mismatch(layout, net._w16, w16)),
            ("w16 against bf16(p32)", arena_mismatch(layout, net._w16, net._p32.to(torch.bfloat16)))) if d]
    del p, m, v, w16
    return loss, bad


def check_adam_of_own_gradients(enc, cuda, n=N, s=S, sizes=None):
    """steps of batch sizes `sizes` (default three of n; eager, then graph replays): each step's fp32 weights and Adam
    moments exactly whole-arena Adam of that step's own final gradients at the t it ran at, and the bf16 operand copy
    exactly the new fp32 weights.

    When `sizes` switches between batch shapes (the ResNets only: a full batch and an epoch's partial last batch through
    _fit_loop), two captured steps are alive and share one Adam state, and every step also equals, bit for bit, the same
    sequence of batches run in program order (BenchStep.serial_steps) on a fresh net: a replay of the full-batch step
    after a tail step equals a serial run of the same sequence, so neither captured step keeps state of its own that the
    other one's steps make stale."""
    sizes = [n] * 3 if sizes is None else list(sizes)
    switch = len(set(sizes)) > 1
    sd = seeded_sd(enc)
    batches = [tuple(t.to(cuda) for t in batch(SEED + 10 + i, k, s)) for i, k in enumerate(sizes)]
    run = BenchStep(enc, sd, cuda, sizes[0], s)
    layout = arena_layout(run.net)
    seen, snaps = set(), []
    for i, (X, T) in enumerate(batches):
        replay = run.is_replay(X, T)
        loss, bad = adam_mismatches(run, layout, X, T)
        assert run.fused.opt.t == i + 1, "step %d ran at t %d" % (i + 1, run.fused.opt.t)
        seen.add(id(run.fused))
        print("%s step %d (batch %d, %s): fused Adam == whole-arena Adam of the step's gradients: %s" % (
            enc, i + 1, sizes[i], "graph replay" if replay else "eager", not bad))
        assert not bad, "%s step %d (batch %d, %s): %s" % (enc, i + 1, sizes[i], "graph replay" if replay else "eager",
                                                          "; ".join(bad))
        if switch:
            snaps.append(snapshot(run, loss))
    if switch:
        assert len(seen) == len(set(sizes)) and len(run.model._fused_cache) == len(set(sizes))
        assert all(f.opt is run.model._opt_state for f in run.model._fused_cache.values()), "one Adam state"
    del run
    free_device_memory()
    if not switch:
        return
    run = BenchStep(enc, sd, cuda, sizes[0], s)
    for i, loss in enumerate(run.serial_steps(batches)):
        bad = snapshot_mismatches(layout, snaps[i], snapshot(run, loss))
        print("%s step %d (batch %d): captured == serial: %s" % (enc, i + 1, sizes[i], not bad))
        assert not bad, "%s step %d (batch %d): %s" % (enc, i + 1, sizes[i], "; ".join(bad))
    assert run.fused.opt.t == len(sizes)
    del run, snaps
    free_device_memory()


# ---------------------------------------------------------------------------------------------------------------------
# step 1 against the fp32 reference
# ---------------------------------------------------------------------------------------------------------------------
def reference_step(enc, sd, X, T, emulate_bf16):
    """one train-mode forward, the configured loss and its gradients with enc's oracle (oracle.unet_oracle or
    oracle.vgg_oracle) on X's device: fp32, or with the CUDA path's bf16 storage points emulated.  -> host copies of
    loss, logits, gradients (by parameter name) and the running statistics after the step"""
    work = {k: v.to(X.device, copy=True) for k, v in O.strip_module_prefix(sd).items()}
    keys = V.trainable_keys(work, enc) if enc in VGG else O.trainable_keys(work)
    leaves = [work[k].requires_grad_(True) for k in keys]
    if enc in VGG:
        logits = V.VGGUNetOracle(work, enc, emulate_bf16=emulate_bf16).forward(X, training=True)
    else:
        logits = O.UNetOracle(work, RESNET_DEPTH[enc], emulate_bf16=emulate_bf16).forward(X, training=True)
    loss = O.mixed_loss(logits, T, imsize=(256, 256))
    grads = torch.autograd.grad(loss, leaves)
    out = dict(loss=float(loss.detach()), logits=host(logits), grads={k: host(g) for k, g in zip(keys, grads)},
               stats={k: host(v) for k, v in work.items() if k.startswith("encoder.") and k.endswith(STATS)})
    del work, leaves, logits, loss, grads
    free_device_memory()
    return out


def step_outputs(run, loss):
    """what reference_step returns, from the step the BenchStep run just took"""
    net = run.net
    grads = {name: host(net._view(net._g32, net._slots[id(p)])) for name, p, _ in net._arena_params()}
    return dict(loss=float(loss), logits=host(run.fused.plan.logits), grads=grads, stats=running_stats(net))


def deviation(got, ref):
    """(relative L2, cosine) in float64"""
    a, b = got.double().reshape(-1), ref.double().reshape(-1)
    return float((a - b).norm() / (b.norm() + 1e-300)), float((a * b).sum() / (a.norm() * b.norm() + 1e-300))


# ---------------------------------------------------------------------------------------------------------------------
# the golden-fixture encoder tests
# ---------------------------------------------------------------------------------------------------------------------
def gold(tag):
    """the arrays of tests/golden/encoders_<tag>.npz"""
    with np.load(golden_path(tag)) as g:
        return {k: g[k] for k in g.files}


def rel_l2(a, b):
    """relative L2 deviation of a from b, in float64 on the host"""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def host_nchw(t):
    """float32 NCHW host copy of a stored NHWC tensor"""
    return nchw(t).float().cpu()
