"""Every unit of the ResNet U-Net inference forward against float64, at the size of bench.py's infer workload: 320x320,
batch 64 (and 37, a partial last batch: a ragged M tail at every stage), for ResNet101 (Bottleneck blocks) and ResNet34
(BasicBlock, the AlbuNet plan).  The model is built as bench.py builds it (oracle.step_checks.BenchStep) from the
conditioned checkpoint, whose running statistics make the BatchNorm fold non-trivial.

The scenario is what the validation monitor does in the middle of training: one train step at batch 32, an eval
forward (eager, then captured), a second train step (Adam and the train-mode BatchNorm kernels rewrite the weights and
running statistics the eval graph reads), then stressed running statistics and gammas written in place into a few
BatchNorms per stage -- running_var 0 (only eps remains), |running_mean| / sqrt(running_var) = 8, negative and zero
gamma -- and a second eval forward on a different batch, which is a graph replay.  Its own buffers (Plan.stem_parts,
Plan.block_parts, Plan.dec_mid) are checked against float64 on the device, from the current fp32 parameters, the bf16
operand copy and the running statistics, every image, CHUNK at a time.  Each unit is recomputed from its own stored
input, so no error compounds.  A is the same operation on absolute values:
  BN fold scale, shift   sc = gamma / sqrt(rv + eps), sh = beta - rm sc,       scale 2^-21 |sc|, shift 2^-21 (|beta| +
                         every BatchNorm (104 / 36)                            |rm sc|)
  stem output a0,        relu(conv(x) sc + sh [+ r]): the 7x7/s2 conv of the   2^-8 |ref| + 2^-16 A |sc| + 2^-20 (|conv
  every block conv       bf16 image, the inner convs with ReLU, the stride-2   sc| + |beta| + |rm sc| + |r|)
                         downsample without, the last conv with the identity
                         or the downsample's stored output as r
  stem, centre max-pool  max_pool2d of the stored input                        bitwise
  decoder halves, dec0   oracle.unit_checks.check_conv_forward                 2^-8 |ref| + 2^-16 A
  logits                 float64 1x1 of the stored dec0 output with the fp32   (C + 2) 2^-24 (A + |b|), C = 32
                         weight and bias
  ops.softmax2           float64 softmax of the stored logits                  2^-18 |ref|
and the replay's logits equal, bit for bit, an eager forward of a freshly built eval plan on the same model and batch:
a graph that read stale scales / shifts, weights or input fails there.

The bounds.  scale: rsqrtf is within 2 ulp (2^-22 relative), rv + eps and the product with gamma round once each
(2^-24, halved by the square root for the sum): 1.375 x 2^-22 < 2^-21.  shift: that error times |rm sc| plus at most
two fp32 roundings of 2^-24 (|beta| + |rm sc|).  Conv outputs: the epilogue multiplies the fp32 accumulator (2^-16 A, the
bound of test_conv_gemm_persistent_gpu.py) by its scale, adds the shift and the bf16 residual (three fp32 roundings)
and rounds the result to bf16 (2^-8 |ref|); the kernel's scale and shift differ from the float64 ones by the bounds
above, so 2^-20 of the fold's terms covers them and the roundings.  Logits: final_conv_fwd is one sequential fp32 fma
chain of C products per pixel and class, then the bias add.

Measured on an H100 80GB HBM3 at its 700 W power limit: ResNet101 at batch 64 (1176 checks) takes 21-22 s, the
conditioning pass on the CPU included, and at most 23.0 GiB of device memory; at batch 37 (813 checks) 6 s and 18.3 GiB;
ResNet34 at batch 64 (496 checks) 6-8 s and 11.5 GiB.  Worst |got - ref| / bound: the folded conv outputs 0.99 (the bf16
rounding of the output itself), decoder halves 0.99, fold scale 0.35 and shift 0.40, logits 0.16, softmax2 0.05,
max-pools exact.  The stressed BatchNorms reach |running_mean| / sqrt(running_var) = 8 and folded scales up to 3.7."""
import pytest
import torch
import torch.nn.functional as F

import bench_data
from oracle import unet_oracle as O
from oracle.step_checks import RESNET_DEPTH, S, SEED, BenchStep, batch, free_device_memory, host, same_bits
from oracle.step_checks import rng_and_peak_memory  # noqa: F401  (fixture)
from oracle.unit_checks import CHUNK, Bounds, bn_affine, check_conv_forward, conv_ref, f64, nchw

pytestmark = pytest.mark.gpu

REL = 2.0 ** -8           # bf16 rounding of a stored output (and its share of what the reference rounds away)
FOLD_TERMS = 2.0 ** -20   # the fold's fp32 roundings and its scale / shift error, of |conv sc| + |beta| + |rm sc| + |r|
PARAM = 2.0 ** -21        # rsqrtf and the fp32 roundings of the fold parameters (see the module docstring)
SOFTMAX_REL = 2.0 ** -18  # test_elementwise_scale_gpu.py::test_loss
N_BN = {"ResNet101": 104, "ResNet34": 36}
CASES = [("ResNet101", 64), ("ResNet101", 37), ("ResNet34", 64)]


@pytest.fixture(scope="module")
def conditioned():
    """enc -> the conditioned checkpoint (oracle.unet_oracle.conditioned_state_dict), computed once per encoder; the
    conditioning pass only sets the running statistics, so four tiles on the CPU are enough"""
    cache = {}

    def get(enc):
        if enc not in cache:
            x, _ = bench_data.train_batch(4, S, seed=SEED)
            with torch.random.fork_rng(devices=[]):
                cache[enc] = O.conditioned_state_dict(RESNET_DEPTH[enc], torch.from_numpy(x), seed=SEED)
        return cache[enc]
    return get


def stress_fold(net, eps):
    """write extreme running statistics and gammas in place into the stem's BatchNorm and, per stage, the first block's
    bn1, its downsample's BatchNorm and the last block's last BatchNorm (a residual conv).  By channel c mod 8:
    0: running_var 0 with gamma scaled by sqrt(eps / (rv + eps)), which keeps the scale; 1: running_mean = +-8 std;
    2: running_mean uniform in +-8 std; 3: gamma negated; 4: gamma 0.  -> the report lines"""
    enc = net.encoder
    last = "bn3" if hasattr(enc.layer1[0], "conv3") else "bn2"
    mods = [("encoder.bn1", enc.bn1)]
    for li, layer in enumerate((enc.layer1, enc.layer2, enc.layer3, enc.layer4)):
        p = "encoder.layer%d." % (li + 1)
        mods.append((p + "0.bn1", layer[0].bn1))
        if layer[0].downsample is not None:
            mods.append((p + "0.downsample.1", layer[0].downsample[1]))
        mods.append((p + "%d.%s" % (len(layer) - 1, last), getattr(layer[-1], last)))
    gen = torch.Generator(device=net._p32.device).manual_seed(SEED)
    lines = []
    for name, mod in mods:
        rm, rv = mod.running_mean, mod.running_var
        gamma = net._vec(mod.weight, net._p32)
        c = torch.arange(rv.numel(), device=rv.device) % 8
        sd = rv.sqrt()
        u = torch.rand(rv.shape, generator=gen, device=rv.device) * 2 - 1
        sign = torch.where(torch.arange(rv.numel(), device=rv.device) % 16 < 8, 1.0, -1.0)
        gamma.copy_(torch.where(c == 0, gamma * (eps / (rv + eps)).sqrt(), gamma))
        gamma.copy_(torch.where(c == 3, -gamma, torch.where(c == 4, torch.zeros_like(gamma), gamma)))
        rm.copy_(torch.where(c == 1, 8 * sign * sd, torch.where(c == 2, 8 * u * sd, rm)))
        rv.copy_(torch.where(c == 0, torch.zeros_like(rv), rv))
        pos = rv > 0
        ratio = float((rm[pos].double().abs() / rv[pos].double().sqrt()).max())
        scale = f64(gamma) / (f64(rv) + eps).sqrt()
        lines.append("    %-32s C %4d: %3d with running_var 0, max |rm|/sqrt(rv) %.2f, gamma min %+.3f (%d <= 0), "
                     "max |scale| %.1f" % (name, rv.numel(), int((rv == 0).sum()), ratio, float(gamma.min()),
                                           int((gamma <= 0).sum()), float(scale.abs().max())))
    return lines


def check_folded_conv(bd, kind, what, x, y, w, conv, fold, relu, residual=None):
    """y = [relu](conv(x) sc + sh [+ r]) over every image, CHUNK at a time: x the conv's NCHW bf16 input, y and the
    residual r the NHWC stored tensors, w the bf16 weight (float64), fold = (sc, sh, |beta| + |rm sc|) in float64"""
    sc, sh, terms0 = (t.view(1, -1, 1, 1) for t in fold)
    for i in range(0, y.shape[0], CHUNK):
        ref, absref = conv_ref(f64(x[i:i + CHUNK]), w, conv)
        ref = ref * sc
        terms = ref.abs() + terms0
        ref = ref + sh
        if residual is not None:
            r = f64(nchw(residual[i:i + CHUNK]))
            ref, terms = ref + r, terms + r.abs()
            del r
        if relu:
            ref = ref.clamp_min(0)
        bd.check(kind, what, nchw(y[i:i + CHUNK]), ref, absref * sc.abs(), rel=REL, extra=FOLD_TERMS * terms)
        del ref, absref, terms


@pytest.mark.parametrize("enc,n", CASES, ids=["%s-b%d" % c for c in CASES])
def test_every_unit_of_the_replayed_eval_forward(mcb, cuda, conditioned, enc, n):
    from mcb200 import engine, ops
    eps = engine.BN_EPS
    run = BenchStep(enc, conditioned(enc), cuda)
    net = run.net
    run.step(*(t.to(cuda) for t in batch(SEED)))
    net.eval()
    with torch.no_grad():
        net(batch(SEED + 40, n)[0].to(cuda))
    plan = net.plan(n, S, S, False)
    assert plan.graph_fwd is not None, "the first eval forward captures the graph"
    net.train()
    run.step(*(t.to(cuda) for t in batch(SEED + 1)))
    assert run.fused.opt.t == 2
    print("%s, batch %d: stressed BatchNorms" % (enc, n))
    print("\n".join(stress_fold(net, eps)))
    net.eval()
    X = batch(SEED + 41, n)[0].to(cuda)
    graph = plan.graph_fwd
    with torch.no_grad():
        net(X)
    torch.cuda.synchronize()
    assert net.plan(n, S, S, False) is plan and plan.graph_fwd is graph, "the second eval forward is a graph replay"

    w = {name: f64(net._view(net._w16, net._slots[id(p)])) for name, p, _ in net._arena_params()}
    p = {name: f64(net._view(net._p32, net._slots[id(p)])) for name, p, _ in net._arena_params()}
    bn_name = {}
    for name, mod in net.named_modules():
        bn_name.setdefault(id(mod), name)
    bd = Bounds()

    # ---- every BatchNorm's folded scale and shift, computed inside the graph from the running statistics
    fold = {}
    for b in plan._bns:
        name = bn_name[id(b.mod)]
        rm, rv = f64(b.mod.running_mean), f64(b.mod.running_var)
        sc, sh = bn_affine(p, name, rm, 1.0 / (rv + eps).sqrt())
        terms0 = p[name + ".bias"].abs() + (rm * sc).abs()
        bd.check("BN fold scale", name, b.scale, sc, 0.0, rel=PARAM)
        bd.check("BN fold shift", name, b.shift, sh, 0.0, extra=PARAM * terms0)
        fold[name] = (sc, sh, terms0)
    assert len(fold) == len(plan._bns) == N_BN[enc], (len(fold), len(plan._bns))

    # ---- stem: 7x7/s2 conv of the bf16 image (im2col + GEMM) with the folded BatchNorm and ReLU, 2x2 max-pool
    sp = plan.stem_parts
    assert sp["z0"] is sp["a0"]
    check_folded_conv(bd, "conv + fold output", "encoder.conv1", plan.x_in.to(torch.bfloat16), sp["a0"],
                      w["encoder.conv1.weight"], net.get_submodule("encoder.conv1"), fold["encoder.bn1"], True)
    for i in range(0, n, CHUNK):
        bd.check("max-pool (bitwise)", "c1", nchw(sp["c1"][i:i + CHUNK]),
                 F.max_pool2d(f64(nchw(sp["a0"][i:i + CHUNK])), 2, 2), 0.0)

    # ---- encoder blocks, every conv from its own stored input
    blocks = [(prefix, ins[0], out) for kind, prefix, ins, out in plan.units if kind == "block"]
    n_parts = 0
    for prefix, x, out in blocks:
        parts = plan.block_parts[id(out)]
        down = parts[-1] if parts[-1].conv.endswith("downsample.0") else None
        last = parts[-2] if down is not None else parts[-1]
        assert last.y is out and parts[0].x is x
        n_parts += len(parts)
        for part in parts:
            assert part.z is part.y
            conv = net.get_submodule(part.conv)
            if part is last:
                res = down.z if down is not None else x
                check_folded_conv(bd, "block output (conv + fold + residual)", part.conv, nchw(part.x), part.y,
                                  w[part.conv + ".weight"], conv, fold[part.bn], True, res)
            else:
                kind = "downsample (conv + fold)" if part is down else "conv + fold output"
                check_folded_conv(bd, kind, part.conv, nchw(part.x), part.y, w[part.conv + ".weight"], conv,
                                  fold[part.bn], part is not down)
    assert n_parts == N_BN[enc] - 1, n_parts

    # ---- centre max-pool, decoder blocks half by half, dec0
    decoders = [(prefix, ins, out) for kind, prefix, ins, out in plan.units if kind == "decoder"]
    c5, pool = blocks[-1][2], decoders[0][1][0]
    for i in range(0, n, CHUNK):
        bd.check("max-pool (bitwise)", "centre", nchw(pool[i:i + CHUNK]),
                 F.max_pool2d(f64(nchw(c5[i:i + CHUNK])), 2, 2), 0.0)
    halves = []
    for prefix, ins, out in decoders:
        mid = plan.dec_mid[id(out)]
        halves.append((prefix + ".block.0", ins, mid, prefix + ".block.0.conv", False))
        halves.append((prefix + ".block.1", (mid,), out, prefix + ".block.1", True))
    halves.append(("dec0", (decoders[-1][2],), plan.classifier_in, "dec0.conv", False))
    for what, ins, y, key, transposed in halves:
        for i in range(0, n, CHUNK):
            x = torch.cat([nchw(a[i:i + CHUNK]) for a in ins], 1)
            check_conv_forward(bd, what, x, y[i:i + CHUNK], w[key + ".weight"], p[key + ".bias"], transposed,
                               images=range(x.shape[0]))
            del x

    # ---- the fp32 1x1 classifier and softmax2 of the logits
    y0 = plan.classifier_in
    k, cin = plan.logits.shape[1], y0.shape[3]
    wf, bf = p["final.weight"].reshape(k, cin), p["final.bias"].view(1, k, 1, 1)
    probs = ops.softmax2(plan.logits)
    for i in range(0, n, CHUNK):
        yi = f64(y0[i:i + CHUNK])
        ref = torch.einsum("nhwc,kc->nkhw", yi, wf) + bf
        absref = torch.einsum("nhwc,kc->nkhw", yi.abs(), wf.abs()) + bf.abs()
        bd.check("logits (fp32 1x1)", "final", plan.logits[i:i + CHUNK], ref, absref, acc=(cin + 2) * 2.0 ** -24)
        del yi, ref, absref
        pr = torch.softmax(f64(plan.logits[i:i + CHUNK]), 1)
        bd.check("softmax2", "final", probs[i:i + CHUNK], pr, 0.0, rel=SOFTMAX_REL)
        del pr

    n_chunks = -(-n // CHUNK)
    print("%s, batch %d: %d checks" % (enc, n, bd.count))
    bd.report()
    # 2 per BatchNorm; per chunk: the stem, its max-pool, every block conv, the centre max-pool, 2 per decoder block,
    # dec0, the logits and softmax2
    assert bd.count == 2 * N_BN[enc] + n_chunks * (1 + 1 + n_parts + 1 + 2 * len(decoders) + 1 + 2), bd.count
    assert not bd.fails, "\n".join(bd.fails[:20])
    assert bool(torch.isfinite(plan.logits).all()), "the stressed fold must keep the logits finite"
    del w, p, fold, probs

    # ---- the replay against an eager forward of a freshly built plan on the same model and batch
    got = host(plan.logits)
    del plan, graph
    net._plans.pop((n, S, S, False))
    free_device_memory()
    with torch.no_grad():
        fresh = host(net(X))
    assert same_bits(got, fresh), "graph replay and a fresh eager eval forward differ in %d of %d logits" % (
        int((got != fresh).sum()), got.numel())
    print("graph replay == fresh eager eval plan, bit for bit")
    del run, net, X
    free_device_memory()
