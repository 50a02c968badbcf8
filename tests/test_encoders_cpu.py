"""CPU tests of the registry's AlbuNet (reference src/unet_models.py:153-221, src/models.py:22-47) against its reference
fixture tests/golden/encoders_albunet_b2_256.npz (made by oracle/make_golden_encoders.py from the unmodified reference):
  * the mirror's state_dict keys, shapes and seeded initialisation are the reference's, bit for bit, and the reference's
    AlbuNet under a seed equals its UNetResNet(34);
  * the oracle restatement reproduces the reference's logits, loss, gradients and one _fit_loop step;
  * the launch plan is UNetResNet(34)'s, and its FLOPs add up to the reference's hooked forward FLOPs;
  * the registry entry builds through PyTorchUNetWeighted(**config)."""
import collections
import json

import numpy as np
import pytest
import torch

from oracle import synthetic
from oracle import unet_oracle as O
from oracle.make_golden_cases import LOGIT_STRIDE
from oracle.make_golden_encoders import (ENCODER_CASES, ENCODER_GRAD_HEAD, FLOP_TILE, SEED, STEP_HEAD, golden_path,
                                         state_dict_digest)

TAG, ENC, DEPTH, N, S = ENCODER_CASES[0]


@pytest.fixture(scope="module")
def gold():
    with np.load(golden_path(TAG)) as g:
        return {k: g[k] for k in g.files}


def _digest_dict(keys, shapes, sha):
    shapes = json.loads(str(shapes))
    return {str(k): (tuple(shapes[str(k)]), str(h)) for k, h in zip(keys, sha)}


def test_reference_albunet_is_unetresnet34_under_a_seed(gold):
    assert list(gold["init_keys"]) == list(gold["twin_keys"])
    assert np.array_equal(gold["init_sha256"], gold["twin_sha256"])
    assert str(gold["init_shapes"]) == str(gold["twin_shapes"])


def test_mirror_state_dict_and_seeded_init_are_the_reference(mcb, gold):
    from mcb200.unet_models import AlbuNet, UNetResNet
    with torch.random.fork_rng():
        torch.manual_seed(SEED)
        net = AlbuNet(num_classes=2, pretrained=False, is_deconv=True)
    assert isinstance(net, UNetResNet)
    keys, shapes, sha = state_dict_digest(net.state_dict())
    assert list(keys) == list(gold["init_keys"])                  # same keys, same order, aliases included
    assert _digest_dict(keys, shapes, sha) == _digest_dict(gold["init_keys"], gold["init_shapes"], gold["init_sha256"])


def test_oracle_seeded_state_dict_is_the_reference_init(gold):
    with torch.random.fork_rng():
        sd = O.make_reference_like_state_dict(DEPTH, seed=SEED)
    ref = _digest_dict(gold["init_keys"], gold["init_shapes"], gold["init_sha256"])
    keys, shapes, sha = state_dict_digest(sd)
    assert _digest_dict(keys, shapes, sha) == ref


def test_oracle_matches_reference_logits_loss_and_gradients(gold):
    x, t = synthetic.train_batch(N, S, seed=SEED)
    X, T = torch.from_numpy(x), torch.from_numpy(t)
    st = LOGIT_STRIDE
    with torch.random.fork_rng():
        sd = O.make_reference_like_state_dict(DEPTH, seed=SEED)
    with torch.no_grad():
        ev = O.UNetOracle({k: v.clone() for k, v in sd.items()}, DEPTH).forward(X[:1], training=False)
    assert np.allclose(ev.numpy()[:, :, ::st, ::st], gold["eval_logits"], rtol=0, atol=1e-6)
    keys = O.trainable_keys(sd)
    leaves = {k: sd[k].clone().requires_grad_(True) for k in keys}
    work = dict(sd)
    work.update(leaves)
    out = O.UNetOracle(work, DEPTH, update_running_stats=False).forward(X, training=True)
    assert np.allclose(out.detach().numpy()[:, :, ::st, ::st], gold["train_logits"], rtol=0, atol=1e-6)
    loss = O.mixed_loss(out, T, imsize=(256, 256))
    assert abs(float(loss.detach()) - float(gold["loss"])) < 1e-5 * abs(float(gold["loss"]))
    names = [k[len("grad_"):] for k in gold if k.startswith("grad_")]
    assert len(names) == 18
    grads = torch.autograd.grad(loss, [leaves[k] for k in names])
    for k, g in zip(names, grads):
        ref = gold["grad_" + k]
        got = g.numpy().reshape(-1)[:ENCODER_GRAD_HEAD]
        assert got.shape == ref.shape
        assert np.allclose(got, ref, rtol=1e-3, atol=1e-6 * np.abs(ref).max() + 1e-12), k


def test_train_step_oracle_matches_reference_fit_loop(gold):
    x, t = synthetic.train_batch(N, S, seed=SEED)
    with torch.random.fork_rng():
        sd = O.make_reference_like_state_dict(DEPTH, seed=SEED)
    opt = O.AdamOracle(lr=5e-4, weight_decay=1e-4)
    loss, _, _ = O.train_step(sd, DEPTH, torch.from_numpy(x), torch.from_numpy(t), opt, imsize=(256, 256))
    assert abs(float(loss) - float(gold["fit_loss"])) < 1e-5 * abs(float(gold["fit_loss"]))
    steps = [k for k in gold if k.startswith("step_")]
    assert len(steps) == 10
    for name in steps:
        got = sd[name[len("step_"):]].numpy().reshape(-1)[:STEP_HEAD]
        assert np.allclose(got, gold[name], rtol=1e-4, atol=1e-6), name


@pytest.fixture(scope="module")
def plans(mcb):
    from mcb200.unet_models import AlbuNet, UNetResNet
    with torch.random.fork_rng():
        torch.manual_seed(0)
        albu = AlbuNet(num_classes=2, pretrained=False, is_deconv=True)
        r34 = UNetResNet(34, 2, 32, 0.0, False, True)
    return albu, albu.plan(1, FLOP_TILE, FLOP_TILE, True), r34.plan(1, FLOP_TILE, FLOP_TILE, True)


def _bwd_ops(plan):
    return [o for layer in plan.bwd_layers for o in layer]


def test_albunet_plan_is_the_resnet34_plan(plans):
    net, pa, pr = plans
    sig = lambda ops: [(o.kind, o.desc, o.flops) for o in ops]  # noqa: E731
    assert sig(pa.fwd_ops) == sig(pr.fwd_ops)
    assert [sig(layer) for layer in pa.bwd_layers] == [sig(layer) for layer in pr.bwd_layers]
    assert pa.bwd_tags == pr.bwd_tags
    n_conv = sum(isinstance(m, torch.nn.Conv2d) for m in net.modules())
    n_convt = sum(isinstance(m, torch.nn.ConvTranspose2d) for m in net.modules())
    assert (n_conv, n_convt) == (44, 6)
    fwd = collections.Counter(o.kind for o in pa.fwd_ops)
    bwd = collections.Counter(o.kind for o in _bwd_ops(pa))
    assert fwd["conv_fwd"] == n_conv - 1 and fwd["convt_fwd"] == n_convt and fwd["final_conv"] == 1
    # one weight-gradient GEMM per conv but the classifier, +1 per skip concat (dec5..dec2); no data gradient for
    # the stem and the classifier, +1 per skip concat
    assert bwd["conv_wgrad"] == n_conv - 1 + 4 and bwd["convt_wgrad"] == n_convt
    assert bwd["conv_dgrad"] == n_conv - 2 + 4 and bwd["convt_dgrad"] == n_convt


def test_albunet_plan_flops_equal_the_hooked_reference(plans, gold):
    _, pa, _ = plans
    fwd = sum(o.flops for o in pa.fwd_ops)
    assert fwd == float(gold["fwd_flops_%d" % FLOP_TILE])
    assert abs(fwd / 1e9 - 41.59) < 0.005
    # backward: a data-gradient and a weight-gradient GEMM per conv, each as costly as its forward, except that the
    # 7x7 stem (input image) has no data gradient
    stem = next(o.flops for o in pa.fwd_ops if o.kind == "conv_fwd")
    assert sum(o.flops for o in _bwd_ops(pa)) == 2 * fwd - stem


def test_albunet_backward_segments_tile_the_arena(plans):
    net, pa, _ = plans
    segs = pa.bwd_segments()
    total = net._p32.numel()
    assert segs[0][0] == 0 and segs[-1][1] == len(pa.bwd_layers)
    assert all(a[1] == b[0] for a, b in zip(segs, segs[1:]))
    assert segs[0][3] == total and segs[-1][2] == 0 and all(a[2] == b[3] for a, b in zip(segs, segs[1:]))
    bounds = sorted({s[2] for s in segs} | {total})
    for _, p, _ in net._arena_params():
        lo = net._slots[id(p)].off
        hi = lo + p.numel()
        assert any(b0 <= lo and hi <= b1 for b0, b1 in zip(bounds, bounds[1:])), (lo, hi)
    side = [o for o in _bwd_ops(pa) if o.side]
    assert side and all(o.kind in ("conv_wgrad", "convt_wgrad") and o.flops > 0 for o in side)


def test_registry_builds_albunet(mcb):
    import bench
    from mcb200 import models
    from mcb200.unet_models import AlbuNet
    entry = models.PRETRAINED_NETWORKS["AlbuNet"]
    assert entry["model"] is AlbuNet and entry["model_config"] == {"num_classes": 2, "pretrained": False,
                                                                   "is_deconv": True}
    with torch.random.fork_rng():
        m = models.PyTorchUNetWeighted(**bench.unet_config("AlbuNet"))
    assert isinstance(m.model, AlbuNet) and m.model.num_classes == 2
    assert len(m.optimizer.param_groups[0]["params"]) == len(list(m.model.parameters()))
    for enc in ("VGG11", "VGG16", "ResNet50"):
        with pytest.raises(NotImplementedError, match="VGG11"):
            models.PyTorchUNetWeighted(**bench.unet_config(enc))


def test_albunet_constructor_rejects_unbuilt_variants(mcb):
    from mcb200.unet_models import AlbuNet
    with pytest.raises(NotImplementedError):
        AlbuNet(pretrained=True, is_deconv=True)
    with pytest.raises(NotImplementedError):
        AlbuNet(is_deconv=False)
