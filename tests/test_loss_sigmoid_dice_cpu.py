"""The sigmoid Dice (`dice_activation: 'sigmoid'`, src/models.py:421-454) without a GPU:
  * the oracle restatement (oracle/make_golden_sigmoid_dice.py) reproduces the unmodified reference's loss, its
    gradient with respect to the logits and one reference _fit_loop step (tests/golden/loss_sigmoid_dice.npz);
  * the transformers carry the configured activation into both the fused train step and the autograd loss, and reject
    an activation the reference does not implement when they are built."""

import numpy as np
import pytest
import torch

from oracle import synthetic
from oracle import unet_oracle as O
from oracle.make_golden_sigmoid_dice import (BATCH, DECODER_TAIL_KEYS, GOLDEN, SEED, SIZE, STEP_HEAD,
                                             loss_and_dlogits_closed_form, mixed_loss, seeded_logits)

IMSIZE = (256, 256)


@pytest.fixture(scope="module")
def gold():
    with np.load(GOLDEN) as g:
        return {k: g[k] for k in g.files}


@pytest.fixture(scope="module")
def batch():
    x, t = synthetic.train_batch(BATCH, SIZE, seed=SEED)
    return torch.from_numpy(x), torch.from_numpy(t), torch.from_numpy(seeded_logits(t))


def grad_scale(z, t):
    """per-element size of dL/dz: the cross-entropy term's weight w / M, plus (class 1) the Dice term's
    dice_w (2 [t=1] / Dn + (2 I + s) / Dn^2) sigmoid'(z1).  The reference sums in float32, so its gradient sits within
    a small multiple of float32 rounding of this scale"""
    z, t = z.double(), t.double()
    w = O.loss_weights(t, imsize=IMSIZE)
    q1, t1 = torch.sigmoid(z[:, 1]), (t[:, 0] == 1).double()
    dn, num = float(q1.sum() + t1.sum()) + 1.0 + 1e-7, 2 * float((q1 * t1).sum()) + 1.0
    ce = w / t1.numel()
    return torch.stack([ce, ce + 0.2 * (2 * t1 / dn + num / dn ** 2) * q1 * (1 - q1)], 1)


def test_fixture_logits_reach_saturation(batch):
    _, _, z = batch
    assert z.dtype == torch.float32 and z.shape == (BATCH, 2, SIZE, SIZE)
    assert float(z.abs().max()) > 100 and 0.01 < float((z.abs() > 30).float().mean()) < 0.05


def test_closed_form_and_autograd_reproduce_the_reference_loss(gold, batch):
    _, t, z = batch
    scale = grad_scale(z, t)
    loss, d = loss_and_dlogits_closed_form(z.double(), t.double(), imsize=IMSIZE, activation="sigmoid")
    ref, ref_d = float(gold["loss"]), torch.from_numpy(gold["dlogits"]).double()
    assert ref_d.shape == z.shape
    assert abs(float(loss) - ref) <= 1e-6 * ref, (float(loss), ref)
    assert bool(((d - ref_d).abs() <= 2.0 ** -16 * scale).all()), float(((d - ref_d).abs() / scale).max())
    zz = z.double().requires_grad_(True)
    la = mixed_loss(zz, t.double(), imsize=IMSIZE, activation="sigmoid")
    la.backward()
    assert abs(float(la.detach()) - ref) <= 1e-6 * ref
    assert bool(((zz.grad - ref_d).abs() <= 2.0 ** -16 * scale).all())
    # the softmax closed form on the same logits is another function (z0 gets a Dice term there)
    soft, ds = loss_and_dlogits_closed_form(z.double(), t.double(), imsize=IMSIZE, activation="softmax")
    assert abs(float(soft) - ref) > 1e-3 * ref
    assert float((ds[:, 0] - ref_d[:, 0]).abs().max()) > 1e3 * float((d[:, 0] - ref_d[:, 0]).abs().max())


def test_train_step_oracle_matches_reference_fit_loop(gold, batch):
    x, t, _ = batch
    sd = O.make_reference_like_state_dict(34, seed=SEED)
    opt = O.AdamOracle(lr=5e-4, weight_decay=1e-4)
    loss, _, _ = O.train_step(sd, 34, x, t, opt, loss_fn=mixed_loss, imsize=IMSIZE, activation="sigmoid")
    assert abs(float(loss) - float(gold["fit_loss"])) < 1e-5 * float(gold["fit_loss"])
    for k in DECODER_TAIL_KEYS:
        assert np.allclose(sd[k].reshape(-1)[:STEP_HEAD].numpy(), gold["step_" + k], rtol=1e-4, atol=1e-6), k
    # the softmax record differs by the Dice term alone: 0.2 x (sigmoid Dice - softmax Dice) of the same logits
    assert abs(float(gold["fit_loss"]) - float(gold["fit_loss_softmax"])) > 1e-5


def test_oracle_rejects_unknown_activation(batch):
    _, t, z = batch
    with pytest.raises(NotImplementedError, match="only sigmoid and softmax are implemented"):
        mixed_loss(z[:, :, :4, :4], t[:, :, :4, :4], activation="tanh")


def _config(activation):
    import bench
    cfg = bench.unet_config("ResNet34")
    cfg["architecture_config"]["dice"]["dice_activation"] = activation
    return cfg


def test_weighted_transformers_carry_the_activation(mcb):
    from mcb200.models import PyTorchUNetWeighted, PyTorchUNetWeightedStream
    for cls in (PyTorchUNetWeighted, PyTorchUNetWeightedStream):
        for activation in ("sigmoid", "softmax"):
            with torch.random.fork_rng():
                m = cls(**_config(activation))
            mode, cfg = m._fused_loss
            assert mode == 0 and cfg["dice_activation"] == activation, (cls, activation)
            assert m.loss_function[0][1].keywords["dice_activation"] == activation
    # a config without the key keeps the reference's default, softmax (src/models.py:386)
    cfg = _config("softmax")
    del cfg["architecture_config"]["dice"]["dice_activation"]
    with torch.random.fork_rng():
        m = PyTorchUNetWeighted(**cfg)
    assert m._fused_loss[1]["dice_activation"] == "softmax"


def test_unknown_activation_is_rejected_at_construction(mcb):
    from mcb200 import models
    for cls in (models.PyTorchUNetWeighted, models.PyTorchUNetWeightedStream):
        with pytest.raises(NotImplementedError, match="only sigmoid and softmax are implemented"):
            cls(**_config("tanh"))
    with pytest.raises(NotImplementedError, match="only sigmoid and softmax are implemented"):
        models.mixed_dice_cross_entropy_loss(torch.zeros(1, 2, 4, 4), torch.zeros(1, 3, 4, 4), dice_activation="relu")


def test_plain_cross_entropy_ignores_the_activation(mcb):
    """the reference's PyTorchUNet never reads architecture_config['dice'] (src/models.py:104-107)"""
    from mcb200.models import PyTorchUNet, PyTorchUNetStream
    for activation in ("sigmoid", "tanh"):
        for cls in (PyTorchUNet, PyTorchUNetStream):
            with torch.random.fork_rng():
                m = cls(**_config(activation))
            assert m._fused_loss == (1, {})


def test_loss_args_encode_the_activation(mcb):
    """mcb_loss_args.dice_activation: 0 softmax (also what a zeroed struct holds), 1 sigmoid"""
    from mcb200 import _lib as L
    from mcb200 import ops
    assert L.LossArgs._fields_[-1] == ("dice_activation", L.C.c_int)
    assert L.LossArgs().dice_activation == 0
    assert [ops.dice_activation_code(a) for a in ("softmax", "sigmoid")] == [0, 1]
    with pytest.raises(NotImplementedError):
        ops.dice_activation_code("Sigmoid")
