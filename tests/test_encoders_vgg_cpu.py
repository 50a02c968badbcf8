"""CPU tests of UNet11 and UNetVGG16 (reference src/unet_models.py:56-106, :224-312) against their reference fixtures
tests/golden/encoders_vgg1*_b2_256.npz (made by oracle/make_golden_vgg.py from the unmodified reference):
  * the mirrors' state_dict keys, order and seeded initialisation are the reference's, bit for bit;
  * the oracle restatement reproduces the reference's logits, loss, gradients and one _fit_loop step;
  * the launch plans' FLOPs add up to the reference's hooked forward FLOPs, op counts match the module counts, and the
    backward segments tile the parameter arena;
  * the ResNet plans are the ones the parent commit built;
  * the constructors reject what the H100 path does not build."""
import collections
import hashlib
import json

import numpy as np
import pytest
import torch

from oracle import synthetic
from oracle import vgg_oracle as V
from oracle.make_golden_cases import LOGIT_STRIDE
from oracle.make_golden_encoders import ENCODER_GRAD_HEAD, FLOP_TILE, SEED, STEP_HEAD, golden_path, state_dict_digest
from oracle.make_golden_vgg import GRAD_KEYS, STEP_KEYS, VGG_CASES

CASES = [c[0] for c in VGG_CASES]
ENC = {c[0]: c[1] for c in VGG_CASES}


def _gold(tag):
    with np.load(golden_path(tag)) as g:
        return {k: g[k] for k in g.files}


def _digest_dict(keys, shapes, sha):
    shapes = json.loads(str(shapes))
    return {str(k): (tuple(shapes[str(k)]), str(h)) for k, h in zip(keys, sha)}


def _net(enc):
    from mcb200.unet_models import UNet11, UNetVGG16
    if enc == "VGG11":
        return UNet11(num_classes=2, pretrained=False)
    return UNetVGG16(num_classes=2, dropout_2d=0.0, pretrained=False, is_deconv=True)


@pytest.mark.parametrize("tag", CASES)
def test_mirror_state_dict_and_seeded_init_are_the_reference(mcb, tag):
    g = _gold(tag)
    with torch.random.fork_rng():
        torch.manual_seed(SEED)
        net = _net(ENC[tag])
    keys, shapes, sha = state_dict_digest(net.state_dict())
    assert list(keys) == list(g["init_keys"])                  # same keys, same order, aliases included
    assert _digest_dict(keys, shapes, sha) == _digest_dict(g["init_keys"], g["init_shapes"], g["init_sha256"])


@pytest.mark.parametrize("tag", CASES)
def test_oracle_seeded_state_dict_is_the_reference_init(tag):
    g = _gold(tag)
    with torch.random.fork_rng():
        sd = V.make_reference_like_state_dict(ENC[tag], seed=SEED)
    keys, shapes, sha = state_dict_digest(sd)
    assert list(keys) == list(g["init_keys"])
    assert _digest_dict(keys, shapes, sha) == _digest_dict(g["init_keys"], g["init_shapes"], g["init_sha256"])


@pytest.mark.parametrize("tag", CASES)
def test_oracle_matches_reference_logits_loss_and_gradients(tag):
    g = _gold(tag)
    _, enc, n, s = VGG_CASES[CASES.index(tag)]
    x, t = synthetic.train_batch(n, s, seed=SEED)
    X, T = torch.from_numpy(x), torch.from_numpy(t)
    st = LOGIT_STRIDE
    with torch.random.fork_rng():
        sd = V.make_reference_like_state_dict(enc, seed=SEED)
    with torch.no_grad():
        ev = V.VGGUNetOracle(sd, enc).forward(X[:1])
    assert np.allclose(ev.numpy()[:, :, ::st, ::st], g["eval_logits"], rtol=0, atol=1e-6)
    leaves = {k: sd[k].clone().requires_grad_(True) for k in V.trainable_keys(sd, enc)}
    work = dict(sd)
    work.update(leaves)
    out = V.VGGUNetOracle(work, enc).forward(X, training=True)
    assert np.allclose(out.detach().numpy()[:, :, ::st, ::st], g["train_logits"], rtol=0, atol=1e-6)
    loss = V.mixed_loss(out, T, imsize=(256, 256))
    assert abs(float(loss.detach()) - float(g["loss"])) < 1e-5 * abs(float(g["loss"]))
    names = [k[len("grad_"):] for k in g if k.startswith("grad_")]
    assert names == list(GRAD_KEYS[enc])
    for k, gr in zip(names, torch.autograd.grad(loss, [leaves[k] for k in names])):
        ref = g["grad_" + k]
        got = gr.numpy().reshape(-1)[:ENCODER_GRAD_HEAD]
        assert got.shape == ref.shape
        assert np.allclose(got, ref, rtol=1e-3, atol=1e-6 * np.abs(ref).max() + 1e-12), k


@pytest.mark.parametrize("tag", CASES)
def test_train_step_oracle_matches_reference_fit_loop(tag):
    g = _gold(tag)
    _, enc, n, s = VGG_CASES[CASES.index(tag)]
    x, t = synthetic.train_batch(n, s, seed=SEED)
    with torch.random.fork_rng():
        sd = V.make_reference_like_state_dict(enc, seed=SEED)
    opt = V.AdamOracle(lr=5e-4, weight_decay=1e-4)
    loss, _, _ = V.train_step(sd, enc, torch.from_numpy(x), torch.from_numpy(t), opt, imsize=(256, 256))
    assert abs(float(loss) - float(g["fit_loss"])) < 1e-5 * abs(float(g["fit_loss"]))
    assert sorted(k for k in g if k.startswith("step_")) == sorted("step_" + k for k in STEP_KEYS)
    for k in STEP_KEYS:
        got = sd[k].numpy().reshape(-1)[:STEP_HEAD]
        assert np.allclose(got, g["step_" + k], rtol=1e-4, atol=1e-6), k


@pytest.fixture(scope="module")
def plans(mcb):
    out = {}
    for tag in CASES:
        with torch.random.fork_rng():
            torch.manual_seed(0)
            net = _net(ENC[tag])
        out[tag] = (net, net.plan(1, FLOP_TILE, FLOP_TILE, True), net.plan(1, FLOP_TILE, FLOP_TILE, False))
    return out


def _bwd_ops(plan):
    return [o for layer in plan.bwd_layers for o in layer]


@pytest.mark.parametrize("tag", CASES)
def test_plan_flops_equal_the_hooked_reference(plans, tag):
    net, pt, pe = plans[tag]
    fwd = sum(o.flops for o in pt.fwd_ops)
    assert fwd == float(_gold(tag)["fwd_flops_%d" % FLOP_TILE])
    assert [(o.kind, o.desc, o.flops) for o in pe.fwd_ops] == [(o.kind, o.desc, o.flops) for o in pt.fwd_ops]
    # the input conv counts its real 27-wide reduction; backward: a data-gradient and a weight-gradient GEMM per conv,
    # each as costly as its forward, except that the input conv (the image) has no data gradient
    first = next(o for o in pt.fwd_ops if o.kind == "conv_fwd")
    assert first.flops == 2.0 * FLOP_TILE * FLOP_TILE * 64 * 27
    assert sum(o.flops for o in _bwd_ops(pt)) == 2 * fwd - first.flops
    assert not _bwd_ops(pe)


@pytest.mark.parametrize("tag", CASES)
def test_plan_op_counts_match_the_modules(plans, tag):
    net, pt, _ = plans[tag]
    n_conv = sum(isinstance(m, torch.nn.Conv2d) for m in net.modules())
    n_convt = sum(isinstance(m, torch.nn.ConvTranspose2d) for m in net.modules())
    n_enc = sum(len(s) for s in net._stages)
    assert (n_conv, n_convt, n_enc) == ({"VGG11": (15, 5, 8), "VGG16": (20, 5, 13)}[ENC[tag]])
    fwd = collections.Counter(o.kind for o in pt.fwd_ops)
    bwd = collections.Counter(o.kind for o in _bwd_ops(pt))
    assert fwd["conv_fwd"] == n_conv - 1 and fwd["convt_fwd"] == n_convt and fwd["final_conv"] == 1
    assert fwd["maxpool"] == 5 and bwd["maxpool"] == 5 and fwd["im2col"] == 1
    # one weight-gradient GEMM per conv but the classifier, +1 per skip concat (dec5..dec2, dec1); no data gradient
    # for the input conv and the classifier, +1 per skip concat
    assert bwd["conv_wgrad"] == n_conv - 1 + 5 and bwd["convt_wgrad"] == n_convt
    assert bwd["conv_dgrad"] == n_conv - 2 + 5 and bwd["convt_dgrad"] == n_convt
    # no BatchNorm: no statistics, no BatchNorm kernels, no BatchNorm gradient slices
    assert pt._stats_arena.numel() == 0 and not pt._bns and pt.bn_grad_slices() == []
    assert not any(o.kind.startswith("bn_") for o in list(pt.fwd_ops) + _bwd_ops(pt))
    # every bias gradient is produced exactly once: the encoder convs' and the transposed convs' in a fused dgrad
    # epilogue or a pool backward (bias_fused), the decoder convs' in the transposed convs' data gradients, dec1's by a
    # channel sum, the classifier's in final_conv_bwd
    assert len(pt.bias_fused) == n_enc + n_convt and bwd["channel_sum"] == 1
    assert len(pt.bias_fused) + n_convt + bwd["channel_sum"] + 1 == n_conv + n_convt


@pytest.mark.parametrize("tag", CASES)
def test_backward_segments_tile_the_arena(plans, tag):
    net, pt, _ = plans[tag]
    segs = pt.bwd_segments()
    total = net._p32.numel()
    assert len(segs) == 4
    assert segs[0][0] == 0 and segs[-1][1] == len(pt.bwd_layers)
    assert all(a[1] == b[0] and a[0] < a[1] for a, b in zip(segs, segs[1:]))
    assert segs[0][3] == total and segs[-1][2] == 0 and all(a[2] == b[3] for a, b in zip(segs, segs[1:]))
    bounds = sorted({s[2] for s in segs} | {total})
    for _, p, _ in net._arena_params():
        lo = net._slots[id(p)].off
        hi = lo + p.numel()
        assert any(b0 <= lo and hi <= b1 for b0, b1 in zip(bounds, bounds[1:])), (lo, hi)
    # the decoder | conv5 stage | conv4 stage | rest order
    tags = pt.bwd_tags
    assert set(tags[segs[0][0]:segs[0][1]]) == {"decoder"}
    assert set(tags[segs[1][0]:segs[1][1]]) == {"conv5"} and set(tags[segs[2][0]:segs[2][1]]) == {"conv4"}
    side = [o for o in _bwd_ops(pt) if o.side]
    assert side and all(o.kind in ("conv_wgrad", "convt_wgrad") and o.flops > 0 for o in side)


# (kind, desc, flops) of every forward op and of every backward layer, and bwd_tags, of the ResNet plans at batch 2,
# 320x320 as the parent commit built them (sha256 of their JSON form, see _plan_signature)
RESNET_PLAN_SHA256 = {
    34: "210abc2e65c91d2a5bfbec89c8d3714b379562303d3facd3c54df94fed1cbf11",
    101: "a7fae69bef57bb276766b6d98a73404bec3ba70431ed904b7f6f014b509b7165",
    152: "4f956bb8203628274f48aa676e6c9206519db1366ff2c6423b416d5021494376",
}


def _plan_signature(plan):
    sig = {"fwd": [(o.kind, o.desc, o.flops) for o in plan.fwd_ops],
           "bwd": [[(o.kind, o.desc, o.flops) for o in layer] for layer in plan.bwd_layers],
           "tags": list(plan.bwd_tags)}
    return hashlib.sha256(json.dumps(sig).encode()).hexdigest()


@pytest.mark.parametrize("depth", [34, 101, 152])
def test_resnet_plans_are_unchanged(mcb, depth):
    from mcb200.unet_models import UNetResNet
    with torch.random.fork_rng():
        net = UNetResNet(depth, 2, 32, 0.0, False, True)
    assert _plan_signature(net.plan(2, 320, 320, True)) == RESNET_PLAN_SHA256[depth]


def test_constructors_reject_unbuilt_variants(mcb):
    from mcb200.unet_models import UNet11, UNetVGG16
    with pytest.raises(NotImplementedError):
        UNet11(pretrained=True)
    with pytest.raises(NotImplementedError):
        UNetVGG16(pretrained=True, is_deconv=True)
    with pytest.raises(NotImplementedError):
        UNetVGG16(is_deconv=False)
    with torch.random.fork_rng():
        net = UNet11(num_classes=2)
    with pytest.raises(RuntimeError):
        net(torch.zeros(1, 3, 64, 64))                   # CPU input: there is no CPU fallback
