"""The sigmoid Dice (`dice_activation: 'sigmoid'`, src/models.py:421-454) on the H100 path: the loss kernels against the
float64 closed form (oracle/make_golden_sigmoid_dice.py), the autograd loss and one fused train step against the
unmodified reference (tests/golden/loss_sigmoid_dice.npz), and a guard that the fused step computes the configured
Dice, not the other one.

Tolerances of the kernels (float32 per pixel, float32 per-thread and per-block partial sums, float64 across blocks):
  * the four sums are sums of non-negative terms, each within a few float32 roundings of its float64 value, so each
    sum is held to 2^-16 relative; T counts pixels and is exact;
  * the loss is formed in float64 from those sums: 2^-16 of the cross-entropy part ce_w S / M, plus 2 x 2^-16 x dice_w
    for the Dice ratio (2I + s) / Dn, whose relative perturbation by relative errors e in I and P is at most 2e,
    plus its float32 rounding;
  * dlogits are held per element to 2^-18 of the element's own scale: w / M for the cross-entropy term (which absorbs
    the cancellation in p - onehot), plus dice_w (2 [t=1] / Dn + (2 I + s) / Dn^2) sigmoid'(z1) on class 1 -- the
    bound of the softmax test at the benchmark's size (tests/test_elementwise_scale_gpu.py::test_loss) with sigmoid' for p1 p0."""
import math

import numpy as np
import pytest
import torch

from oracle import synthetic
from oracle import unet_oracle as O
from oracle.make_golden_sigmoid_dice import (BATCH, DECODER_TAIL_KEYS, GOLDEN, SEED, SIZE, STEP_HEAD,
                                             loss_and_dlogits_closed_form, seeded_logits)

pytestmark = pytest.mark.gpu
F64 = torch.float64
DICE_W, CE_W = 0.2, 1.0
LR = 5e-4


def _gold():
    with np.load(GOLDEN) as g:
        return {k: g[k] for k in g.files}


def _case(name):
    """(logits, target, size_c) on the device"""
    if name == "b32_320":      # the benchmark's batch and tile: every thread of both kernels loops over ~12 pixels
        _, t = synthetic.train_batch(32, 320, seed=320, n_rect=40)
        z = seeded_logits(t, seed=320)
    else:
        _, t = synthetic.train_batch(BATCH, SIZE, seed=SEED)
        z = seeded_logits(t)
        if name == "saturated":    # every logit at |z| >= 30: sigmoid is 0 or 1 in float32, sigmoid' ~ exp(-|z|)
            z = np.sign(z) * (30 + 20 * np.abs(z)).astype(np.float32)
    s = t.shape[-1]
    return torch.from_numpy(z).cuda(), torch.from_numpy(t).cuda(), math.sqrt(s * s) / 2.0


def run_kernels(logits, t, size_c, **cfg):
    from mcb200 import ops
    sums = torch.zeros(4, dtype=F64, device=logits.device)
    ops.loss_partials(logits, t, sums, mode=0, size_c=size_c, **cfg)
    dlog, loss = torch.empty_like(logits), torch.zeros((), device=logits.device)
    ops.loss_grad(logits, t, sums, dlog, loss, mode=0, size_c=size_c, **cfg)
    return sums, loss, dlog


def reference_sums(z, t):
    """float64 [I, P, T, S] of the sigmoid Dice and the weighted cross entropy, and the per-pixel w, q1, [t=1]"""
    s = t.shape[-1]
    z, t = z.double(), t.double()
    q1, t1 = torch.sigmoid(z[:, 1]), (t[:, 0] == 1).double()
    w = O.loss_weights(t, imsize=(s, s))
    ce = torch.logsumexp(z, 1) - torch.where(t[:, 0] != 0, z[:, 1], z[:, 0])
    return torch.stack([(q1 * t1).sum(), q1.sum(), t1.sum(), (w * ce).sum()]), w, q1, t1


def dlogit_scale(sums, w, q1, t1):
    I, P, T = (float(v) for v in sums[:3])
    dn, num = P + T + 1.0 + 1e-7, 2 * I + 1.0
    ce = CE_W * w / t1.numel()
    return torch.stack([ce, ce + DICE_W * (2 * t1 / dn + num / dn ** 2) * q1 * (1 - q1)], 1)


def assert_within(got, ref, tol, what):
    err = (got.double() - ref.double()).abs()
    bad = ~(err <= tol)     # NaN fails
    assert not bool(bad.any()), "%s: %d/%d elements off, worst err/bound %g" % (
        what, int(bad.sum()), bad.numel(), float((err / tol).nan_to_num(float("inf")).max()))


@pytest.mark.parametrize("name", ["b2_256", "b32_320", "saturated"])
def test_kernels_against_closed_form(mcb, cuda, name):
    z, t, size_c = _case(name)
    pixels = t[:, 0].numel()
    if name == "b32_320":
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert pixels // (min(-(-pixels // 256), 8 * sms) * 256) >= 3     # every thread loops
    runs = [run_kernels(z, t, size_c, dice_activation="sigmoid") for _ in range(2)]
    (sums, loss, dlog), (sums2, loss2, dlog2) = runs
    assert torch.equal(sums, sums2) and torch.equal(loss, loss2) and torch.equal(dlog, dlog2)
    ref_sums, w, q1, t1 = reference_sums(z, t)
    assert_within(sums, ref_sums, 2.0 ** -16 * ref_sums, "sums [I, P, T, S]")
    assert float(sums[2]) == float(ref_sums[2])
    ref_loss, ref_d = loss_and_dlogits_closed_form(z.double(), t.double(), DICE_W, CE_W, 1.0,
                                                   imsize=(t.shape[-1],) * 2, activation="sigmoid")
    S = float(ref_sums[3])
    bound = 2.0 ** -16 * (CE_W * S / pixels + 2 * DICE_W) + 2.0 ** -24 * abs(float(ref_loss))
    assert abs(float(loss) - float(ref_loss)) <= bound, (float(loss), float(ref_loss), bound)
    assert bool(torch.isfinite(dlog).all())
    assert_within(dlog, ref_d, 2.0 ** -18 * dlogit_scale(ref_sums, w, q1, t1), "dlogits")
    if name == "saturated":
        # sigmoid is exactly 1 above +30 in float32 and below 1e-13 under -30
        assert bool((z.abs() >= 30).all()) and abs(float(sums[1]) - float((z[:, 1] > 0).sum())) < 1e-6


def test_zeroed_activation_field_is_the_softmax_loss(mcb, cuda):
    """a struct whose dice_activation is left 0 computes the softmax loss bit for bit; the plain cross entropy ignores
    the field; a value other than 0 / 1 is refused before any launch"""
    import ctypes
    from mcb200 import _lib as L
    from mcb200 import ops
    z, t, size_c = _case("b2_256")
    zeroed = run_kernels(z, t, size_c)
    softmax = run_kernels(z, t, size_c, dice_activation="softmax")
    sigmoid = run_kernels(z, t, size_c, dice_activation="sigmoid")
    for a, b in zip(zeroed, softmax):
        assert torch.equal(a, b)
    assert not torch.equal(zeroed[1], sigmoid[1]) and not torch.equal(zeroed[2][:, 0], sigmoid[2][:, 0])
    # CE sums and the class-0 cross-entropy gradient do not depend on the Dice activation
    assert torch.equal(zeroed[0][2:], sigmoid[0][2:])
    ref_loss, ref_d = O.loss_and_dlogits_closed_form(z.double(), t.double(), imsize=(SIZE, SIZE))
    assert abs(float(zeroed[1]) - float(ref_loss)) <= 1e-6 * abs(float(ref_loss))
    ce = []
    for act in ("softmax", "sigmoid"):
        sums, loss, dlog = torch.zeros(4, dtype=F64, device=cuda), torch.zeros((), device=cuda), torch.empty_like(z)
        ops.loss_partials(z, t[:, :1].contiguous(), sums, mode=1, dice_activation=act)
        ops.loss_grad(z, t[:, :1].contiguous(), sums, dlog, loss, mode=1, dice_activation=act)
        ce.append((loss, dlog))
    assert torch.equal(ce[0][0], ce[1][0]) and torch.equal(ce[0][1], ce[1][1])
    a = ops._loss_args(z, t, 0, dict(size_c=size_c))
    assert a.dice_activation == 0
    a.dice_activation = 2
    sums = torch.zeros(4, dtype=F64, device=cuda)
    stream = torch.cuda.current_stream().cuda_stream
    assert L.lib.mcb_loss_partials(ctypes.byref(a), sums.data_ptr(), stream) != 0
    assert b"dice_activation 2" in L.lib.mcb_last_error()
    assert L.lib.mcb_loss_grad(ctypes.byref(a), sums.data_ptr(), 1, 1.0, torch.empty_like(z).data_ptr(), None,
                               stream) != 0
    assert float(sums.abs().sum()) == 0.0


def test_autograd_loss_against_reference(mcb, cuda):
    """the loss the validation callbacks call, `loss_function(outputs, target)`, against the reference's autograd"""
    import bench
    from mcb200 import models
    g = _gold()
    z, t, _ = _case("b2_256")
    zz = z.clone().requires_grad_(True)
    loss = models.mixed_dice_cross_entropy_loss(zz, t, dice_weight=DICE_W, cross_entropy_weight=CE_W, smooth=1,
                                                dice_activation="sigmoid", w0=50, sigma=10, imsize=(SIZE, SIZE))
    loss.backward()
    ref, ref_d = float(g["loss"]), torch.from_numpy(g["dlogits"]).to(cuda)
    ref_sums, w, q1, t1 = reference_sums(z, t)
    # the reference's float32 autograd lies within ~2^-22 of this scale of the float64 closed form (held to 2^-16 by
    # tests/test_loss_sigmoid_dice_cpu.py), the kernels within 2^-18 (test_kernels_against_closed_form): 2^-16 holds both
    assert abs(float(loss.detach()) - ref) <= 2e-6 * ref, (float(loss), ref)
    assert_within(zz.grad, ref_d, 2.0 ** -16 * dlogit_scale(ref_sums, w, q1, t1), "dlogits vs reference")
    cfg = bench.unet_config("ResNet34")
    cfg["architecture_config"]["dice"]["dice_activation"] = "sigmoid"
    with torch.random.fork_rng(devices=[cuda]):
        model = models.PyTorchUNetWeighted(**cfg)
    name, fn, weight = model.loss_function[0]
    assert torch.equal((fn(z, t) * weight).detach(), loss.detach())


def _seeded_sd():
    with torch.random.fork_rng():
        return O.make_reference_like_state_dict(34, seed=SEED)


def _fused_model(sd, activation, cuda):
    import bench
    from mcb200.models import PyTorchUNetWeighted
    cfg = bench.unet_config("ResNet34")
    cfg["architecture_config"]["dice"]["dice_activation"] = activation
    with torch.random.fork_rng(devices=[cuda]):
        model = PyTorchUNetWeighted(**cfg)
    model.model.load_state_dict(sd)
    return model


def _batch():
    x, t = synthetic.train_batch(BATCH, SIZE, seed=SEED)
    return torch.from_numpy(x), torch.from_numpy(t)


def test_fused_fit_loop_step_against_reference(mcb, cuda):
    """one PyTorchUNetWeighted._fit_loop step with the sigmoid Dice (fused CUDA train step + in-graph Adam) against the
    reference's, with the bounds of tests/test_encoders_gpu.py::test_fused_fit_loop_step_against_reference"""
    g = _gold()
    sd = _seeded_sd()
    model = _fused_model(sd, "sigmoid", cuda)
    X, T = _batch()
    loss = float(model._fit_loop([X, T])["sum"])
    assert abs(loss - float(g["fit_loss"])) < 1e-3 * abs(float(g["fit_loss"])), (loss, float(g["fit_loss"]))
    got = model._net().state_dict()
    # Adam's first update is lr * g / (|g| + eps): a sign wherever |g| >> eps.  Elements whose gradient is within
    # rounding of zero may step the other way; they are counted, and every other element must take the reference's step
    for k in DECODER_TAIL_KEYS:
        ref = torch.from_numpy(g["step_" + k]).double()
        init = sd[k].reshape(-1)[:STEP_HEAD].double()
        mine = got[k].cpu().reshape(-1)[:STEP_HEAD].double()
        diff = (mine - ref).abs()
        other = int((diff > 0.01 * LR).sum())
        print("    step %-18s max |diff| %.2e, %d of %d elements stepped differently" %
              (k, float(diff.max()), other, diff.numel()))
        assert float((mine - init).abs().max()) <= LR * (1 + 1e-3) + 1e-6, k
        assert other <= 1 + diff.numel() // 100, (k, other)
    assert all(bool(torch.isfinite(v).all()) for v in got.values() if v.is_floating_point())


def test_fused_step_computes_the_configured_dice(mcb, cuda):
    """no substitution: on the same weights and batch the sigmoid and softmax steps run the same forward, return
    different losses, and each returns its own activation's loss of those logits and matches its own reference step"""
    g = _gold()
    sd = _seeded_sd()
    X, T = _batch()
    out = {}
    for act in ("sigmoid", "softmax"):
        model = _fused_model(sd, act, cuda)
        loss = float(model._fit_loop([X, T])["sum"])
        out[act] = (loss, model._fused.plan.logits.detach().clone())
        ref = float(g["fit_loss" if act == "sigmoid" else "fit_loss_softmax"])
        assert abs(loss - ref) < 1e-3 * abs(ref), (act, loss, ref)
        del model
    (l_sig, z), (l_soft, z2) = out["sigmoid"], out["softmax"]
    assert torch.equal(z, z2)
    T = T.to(cuda)
    for act, got in (("sigmoid", l_sig), ("softmax", l_soft)):
        own = float(loss_and_dlogits_closed_form(z.double(), T.double(), activation=act)[0])
        other = float(loss_and_dlogits_closed_form(z.double(), T.double(),
                                                   activation="softmax" if act == "sigmoid" else "sigmoid")[0])
        assert abs(got - own) <= 1e-6 * own, (act, got, own)
        assert abs(got - other) > 50 * abs(got - own) + 1e-5, (act, got, own, other)
    # the Dice terms of the two activations differ by ~2e-4 here; the CUDA forward moves that difference by far less
    d_ref = float(g["fit_loss"]) - float(g["fit_loss_softmax"])
    assert abs((l_sig - l_soft) - d_ref) <= 0.05 * abs(d_ref), (l_sig - l_soft, d_ref)


def test_fused_sigmoid_steps_are_bitwise_reproducible(mcb, cuda):
    x, t = synthetic.train_batch(4, 128, seed=4, n_rect=6)
    X, T = torch.from_numpy(x).to(cuda), torch.from_numpy(t).to(cuda)
    with torch.random.fork_rng():
        sd = O.make_reference_like_state_dict(34, seed=21)
    runs = []
    for _ in range(2):
        model = _fused_model(sd, "sigmoid", cuda)
        losses = [model._fit_loop([X, T])["sum"].detach().cpu().clone() for _ in range(2)]
        runs.append((losses, {k: v.detach().cpu().clone() for k, v in model.model.state_dict().items()}))
        del model
        torch.cuda.empty_cache()
    (la, sa), (lb, sb) = runs
    assert all(torch.equal(a, b) for a, b in zip(la, lb)), (la, lb)
    assert float(la[1]) < float(la[0])
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
