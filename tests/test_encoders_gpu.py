"""The registry's AlbuNet on the H100 path against the unmodified reference (tests/golden/encoders_*.npz, made by
oracle/make_golden_encoders.py) at the seeded initialisation.

Bounds come from tests/golden/emulated_bf16_deviation_encoders.json, the deviation that bf16 storage alone puts between
a bit-faithful CPU emulation of the CUDA path (oracle.unet_oracle.UNetOracle(emulate_bf16=True)) and the fp32
reference.  Logits are held to the north-star 1e-3 max-abs wherever the emulation stays below it.

Gradients are held to 1.15 x the emulated relative L2 deviation + 0.01, tensor by tensor, where the emulation shows
that bf16 storage leaves them reproducible (deviation <= REPRODUCIBLE_REL: the decoder tail, dec2 .. classifier).
Nearer the encoder the seeded initialisation's un-normalised residual chain amplifies rounding (DESIGN.md section 3):
the emulated deviation there is one draw of a rounding-driven quantity, and a second valid bf16 evaluation draws
another (on an H100: 0.47 at the centre conv where the emulation drew 0.73, 0.22 at dec3's conv where it drew 0.16).
Those tensors are checked to be finite and within rel < 1 of the reference; the sharp check of that part of the
network is the per-unit comparison with the emulation on the CUDA path's own tensors, where nothing compounds."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import synthetic
from oracle import unet_oracle as O
from oracle.make_golden_cases import LOGIT_STRIDE
from oracle.make_golden_encoders import DEVIATION_JSON, ENCODER_CASES, ENCODER_GRAD_HEAD, SEED, STEP_HEAD
from oracle.step_checks import gold, host_nchw, rel_l2

pytestmark = pytest.mark.gpu
LOGIT_TOL = 1e-3   # BASELINE.json north_star
REPRODUCIBLE_REL = 0.05
CASES = [c[0] for c in ENCODER_CASES]


def _case(tag):
    return next(c for c in ENCODER_CASES if c[0] == tag)


def _logit_bound(emulated):
    """north-star where the storage format allows it, else the emulated deviation with the gradients' margin"""
    return LOGIT_TOL if emulated < 0.5 * LOGIT_TOL else 1.15 * emulated + 1e-4


def _seeded(depth):
    with torch.random.fork_rng():
        return O.make_reference_like_state_dict(depth, seed=SEED)


@pytest.mark.parametrize("tag", CASES)
def test_logits_loss_and_gradients_against_reference(mcb, cuda, tag):
    from mcb200 import models
    from mcb200.unet_models import AlbuNet
    _, enc, depth, n, s = _case(tag)
    g = gold(tag)
    emu = json.load(open(DEVIATION_JSON))[tag]
    st = LOGIT_STRIDE
    x, t = synthetic.train_batch(n, s, seed=SEED)
    X, T = torch.from_numpy(x).to(cuda), torch.from_numpy(t).to(cuda)
    sd = _seeded(depth)
    net = AlbuNet(num_classes=2, pretrained=False, is_deconv=True)
    net.load_state_dict(sd)
    net.cuda().eval()
    with torch.no_grad():
        ev = net(X[:1]).cpu().numpy()[:, :, ::st, ::st]
    net.train()
    logits = net(X)
    loss = models.mixed_dice_cross_entropy_loss(logits, T, dice_weight=0.2, cross_entropy_weight=1.0, smooth=1, w0=50,
                                                sigma=10, imsize=(256, 256))
    loss.backward()
    tr = logits.detach().cpu().numpy()[:, :, ::st, ::st]
    ev_err, tr_err = np.abs(ev - g["eval_logits"]).max(), np.abs(tr - g["train_logits"]).max()
    loss_rel = abs(float(loss.detach()) - float(g["loss"])) / abs(float(g["loss"]))
    print("%s: eval max-abs %.2e (emulated %.2e), train max-abs %.2e (emulated %.2e), loss rel %.1e" %
          (tag, ev_err, emu["eval_logits_max_abs"], tr_err, emu["train_logits_max_abs"], loss_rel))
    assert ev.shape == g["eval_logits"].shape and tr.shape == g["train_logits"].shape
    assert ev_err < _logit_bound(emu["eval_logits_max_abs"]), ev_err
    assert tr_err < _logit_bound(emu["train_logits_max_abs"]), tr_err
    assert loss_rel < max(1e-4, 1.15 * emu["loss_rel"]), loss_rel
    params = dict(net.named_parameters())
    assert set(emu["grads"]) == {k[len("grad_"):] for k in g if k.startswith("grad_")}
    bounded = 0
    for k, e in sorted(emu["grads"].items()):
        got = params[k].grad.detach().cpu().contiguous().reshape(-1)[:ENCODER_GRAD_HEAD]
        assert bool(torch.isfinite(got).all()), k
        rel = rel_l2(got, torch.from_numpy(g["grad_" + k]))
        print("    grad %-34s rel %.3e (emulated %.3e)" % (k, rel, e["rel"]))
        if e["rel"] <= REPRODUCIBLE_REL:
            assert rel <= 1.15 * e["rel"] + 0.01, (k, rel, e["rel"])
            bounded += 1
        else:
            assert rel < 1.0, (k, rel, e["rel"])     # still the reference's gradient, not noise
    assert bounded >= 6     # dec2, dec1, dec0 and the classifier


def test_every_unit_against_bf16_emulated_oracle(mcb, cuda):
    """each encoder block and decoder block re-run by the bf16-storage emulation on the CUDA path's OWN input and output
    gradient: the forward output and the unit's parameter gradients must agree (nothing compounds across units)"""
    from mcb200.unet_models import AlbuNet
    tag, _, depth, n, s = ENCODER_CASES[0]
    sd = _seeded(depth)
    net = AlbuNet(num_classes=2, pretrained=False, is_deconv=True)
    net.load_state_dict(sd)
    net.cuda().train()
    x, t = synthetic.train_batch(n, s, seed=SEED)
    logits = net(torch.from_numpy(x).to(cuda))
    O.mixed_loss(logits, torch.from_numpy(t).to(cuda), imsize=(256, 256)).backward()
    plan = net.plan(n, s, s, True)
    params = dict(net.named_parameters())
    first_of_layer = {"encoder.layer%d.0" % i for i in range(1, 5)}
    checked = 0
    for kind, prefix, ins, out in plan.units:
        keys = [k for k in sd if k.startswith(prefix + ".") and sd[k].is_floating_point()
                and not k.endswith(("running_mean", "running_var"))]
        leaves = {k: v.clone() for k, v in sd.items() if k.startswith(prefix + ".")}
        for k in keys:
            leaves[k].requires_grad_(True)
        orc = O.UNetOracle(leaves, depth, update_running_stats=False, emulate_bf16=True)
        xin = [host_nchw(a) for a in ins]
        if kind == "block":
            li = int(prefix.split("layer")[1][0])
            y = orc._block(xin[0], prefix, 2 if (prefix in first_of_layer and li > 1) else 1, True)
        else:
            y = orc._decoder(torch.cat(xin, 1) if len(xin) > 1 else xin[0], prefix)
        assert rel_l2(host_nchw(out), y.detach()) < 1.5e-2, (prefix, "forward")
        g_out = host_nchw(plan.grad[id(out)])
        if kind == "decoder":
            g_out = g_out * (y.detach() > 0)   # decoder gradients are stored already masked by the unit's ReLU
        grads = torch.autograd.grad(y, [leaves[k] for k in keys], g_out)
        for k, gr in zip(keys, grads):
            assert rel_l2(params[k].grad.detach(), gr) < 8e-2, (prefix, k)
            checked += 1
    assert len(plan.units) == 16 + 6 and checked > 2 * len(plan.units)


def test_fused_fit_loop_step_against_reference(mcb, cuda):
    """one PyTorchUNetWeighted._fit_loop step (fused CUDA train step + in-graph Adam) against the reference's own"""
    import bench
    from mcb200.models import PyTorchUNetWeighted
    tag, enc, depth, n, s = ENCODER_CASES[0]
    g = gold(tag)
    sd = _seeded(depth)
    with torch.random.fork_rng():
        model = PyTorchUNetWeighted(**bench.unet_config(enc))
    model.model.load_state_dict(sd)
    x, t = synthetic.train_batch(n, s, seed=SEED)
    loss = float(model._fit_loop([torch.from_numpy(x), torch.from_numpy(t)])["sum"])
    assert abs(loss - float(g["fit_loss"])) < 1e-3 * abs(float(g["fit_loss"])), (loss, float(g["fit_loss"]))
    got = model._net().state_dict()
    # decoder-tail tensors have accurate gradients: Adam moved them like the reference did.  Adam's first update is
    # lr * g / (|g| + eps), a sign wherever |g| >> eps: an element whose gradient is within rounding of zero may step
    # the other way (up to 2 lr apart), or part of the way where |g| is comparable to eps.  Such elements are counted,
    # not normed; every other element must have taken the reference's step
    lr = 5e-4
    for k in ("final.weight", "final.bias", "dec0.conv.weight", "dec0.conv.bias", "dec1.block.1.bias"):
        ref = torch.from_numpy(g["step_" + k]).double()
        init = sd[k].reshape(-1)[:STEP_HEAD].double()
        mine = got[k].cpu().reshape(-1)[:STEP_HEAD].double()
        diff = (mine - ref).abs()
        other = int((diff > 0.01 * lr).sum())
        print("    step %-18s max |diff| %.2e, %d of %d elements stepped differently" %
              (k, float(diff.max()), other, diff.numel()))
        assert float((mine - init).abs().max()) <= lr * (1 + 1e-3) + 1e-6, k
        assert other <= 1 + diff.numel() // 100, (k, other)
    # BatchNorm running statistics follow nn.BatchNorm2d's update.  The stem's are tight; the last encoder block's
    # batch statistics sit at the end of the seeded init's rounding-amplifying chain (module docstring: a second bf16
    # evaluation lands a few per cent away, the emulation 1 %), so like the deep gradients they are held to rel < 1
    for k in ("encoder.bn1.running_mean", "encoder.bn1.running_var"):
        ref = torch.from_numpy(g["step_" + k])
        assert torch.allclose(got[k].cpu().reshape(-1)[:STEP_HEAD], ref, rtol=2e-2, atol=1e-3), k
    for k in ("encoder.layer4.2.bn2.running_mean", "encoder.layer4.2.bn2.running_var"):
        rel = rel_l2(got[k].reshape(-1)[:STEP_HEAD], torch.from_numpy(g["step_" + k]))
        print("    step %-34s rel %.2e" % (k, rel))
        assert rel < 1.0, (k, rel)
    assert all(bool(torch.isfinite(v).all()) for v in got.values() if v.is_floating_point())


def test_fused_train_steps_are_bitwise_reproducible(mcb, cuda):
    import bench
    from mcb200.models import PyTorchUNetWeighted
    x, t = synthetic.train_batch(4, 128, seed=4, n_rect=6)
    X, T = torch.from_numpy(x).to(cuda), torch.from_numpy(t).to(cuda)
    runs = []
    with torch.random.fork_rng(devices=[cuda]):
        sd = O.make_reference_like_state_dict(34, seed=21)
        for _ in range(2):
            model = PyTorchUNetWeighted(**bench.unet_config("AlbuNet"))
            model.model.load_state_dict(sd)
            losses = [model._fit_loop([X, T])["sum"].detach().cpu().clone() for _ in range(2)]
            runs.append((losses, {k: v.detach().cpu().clone() for k, v in model.model.state_dict().items()}))
            del model
            torch.cuda.empty_cache()
    (la, sa), (lb, sb) = runs
    assert all(torch.equal(a, b) for a, b in zip(la, lb)), (la, lb)
    assert float(la[1]) < float(la[0])
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k


def test_save_load_transform_round_trip(mcb, cuda, tmp_path):
    """fit -> save (`module.` keys, the reference's DataParallel checkpoint layout) -> load into a fresh transformer ->
    transform: the same weights and the same probabilities"""
    import bench
    from mcb200.models import PyTorchUNetWeighted
    from mcb200.unet_models import AlbuNet
    x, t = synthetic.train_batch(2, 64, seed=3, n_rect=4)
    with torch.random.fork_rng(devices=[cuda]):
        torch.manual_seed(5)
        m = PyTorchUNetWeighted(**bench.unet_config("AlbuNet"))
        m.fit(([[torch.from_numpy(x), torch.from_numpy(t)]], 1))
        path = str(tmp_path / "transformers" / "unet")
        m.save(path)
        saved = torch.load(path)
        m2 = PyTorchUNetWeighted(**bench.unet_config("AlbuNet"))
    g = gold(ENCODER_CASES[0][0])
    assert sorted(saved) == sorted("module." + str(k) for k in g["init_keys"])
    m2.load(path)
    ref = m._net().state_dict()
    for k, v in m2.model.state_dict().items():
        assert torch.equal(v.cpu(), ref[k].cpu()), k
    p1 = m.transform(([torch.from_numpy(x)], 1))["multichannel_map_prediction"]
    p2 = m2.transform(([torch.from_numpy(x)], 1))["multichannel_map_prediction"]
    assert p1.shape == (2, 2, 64, 64) and np.array_equal(p1, p2)
    assert np.allclose(p1.sum(1), 1.0, atol=1e-6)
    net = m2._net()
    assert isinstance(net, AlbuNet)
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 96, 96, device=cuda))   # H, W must be multiples of 64 (the reference fails in torch.cat)
