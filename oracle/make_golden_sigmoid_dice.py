"""TEST INFRASTRUCTURE -- tests/golden/loss_sigmoid_dice.npz, the reference's mixed Dice / weighted cross-entropy loss
with `dice_activation: 'sigmoid'` (src/models.py:149-161,384-454):

    MCB_REFERENCE_ROOT=<checkout> python -m oracle.make_golden_sigmoid_dice     (runs the UNMODIFIED reference, CPU)

The reference is configured through its own config dict (oracle/ref_shim.py's `config.unet`, ResNet34 at config 1,
b2 256x256) with architecture_config['dice']['dice_activation'] overridden to 'sigmoid'.  Recorded:
  * `loss`, `dlogits`: the loss of PyTorchUNetWeighted.loss_function on seeded_logits(t) and its full autograd gradient
    with respect to those logits, t = synthetic.train_batch(2, 256, 1234)'s target;
  * `fit_loss` and `step_<key>`: the loss of one reference _fit_loop step of PyTorchUNetWeighted built under
    torch.manual_seed(1234), on that batch, and the leading STEP_HEAD elements of the decoder-tail STEP_KEYS after it
    (the record of oracle/make_golden_encoders.py);
  * `fit_loss_softmax`: the same step's loss with the configured softmax Dice, so that a test can tell the two apart.
Inputs and initial weights are not stored: both sides regenerate them from the seed.

It also holds the CPU restatement of the loss with either activation (dice_loss, mixed_loss,
loss_and_dlogits_closed_form): the softmax case is oracle/unet_oracle.py's, the sigmoid case is added here."""
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import synthetic  # noqa: E402
from oracle import unet_oracle as O  # noqa: E402
from oracle.make_golden_encoders import SEED, STEP_HEAD, STEP_KEYS  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "loss_sigmoid_dice.npz")
ENCODER, BATCH, SIZE = "ResNet34", 2, 256
DECODER_TAIL_KEYS = STEP_KEYS[:5]   # final, dec0, dec1's transposed-conv bias: the tensors with accurate gradients


# --------------------------------------------------------------------------------------------------------------------
# the loss with either Dice activation
# --------------------------------------------------------------------------------------------------------------------
def dice_loss(logits, t, smooth=1.0, eps=1e-7, activation="softmax"):
    """multiclass_dice_loss(excluded_classes=[0]) + DiceLoss (src/models.py:421-454, src/steps/pytorch/validation.py:
    8-16) with the reference's two activations; sigmoid acts per channel, so class 1's Dice reads sigmoid(z1) only"""
    if activation == "softmax":
        return O.dice_loss(logits, t, smooth, eps)
    if activation != "sigmoid":
        raise NotImplementedError("only sigmoid and softmax are implemented")
    q1 = torch.sigmoid(logits[:, 1])
    t1 = (t == 1).float()
    return 1 - (2 * torch.sum(q1 * t1) + smooth) / (torch.sum(q1) + torch.sum(t1) + smooth + eps)


def mixed_loss(logits, target, dice_weight=0.2, ce_weight=1.0, smooth=1.0, w0=50.0, sigma=10.0, imsize=(256, 256),
               activation="softmax"):
    """oracle.unet_oracle.mixed_loss with the Dice activation of architecture_config['dice']['dice_activation']"""
    t = target[:, 0].long()
    return dice_weight * dice_loss(logits, t, smooth, activation=activation) + \
        ce_weight * O.weighted_cross_entropy(logits, target, w0, sigma, imsize)


def loss_and_dlogits_closed_form(logits, target, dice_weight=0.2, ce_weight=1.0, smooth=1.0, w0=50.0, sigma=10.0,
                                 imsize=(256, 256), eps=1e-7, activation="softmax"):
    """what the CUDA loss kernels implement.  Sigmoid: the Dice probability is q1 = sigmoid(z1), the cross entropy
    keeps the softmax p, and the Dice term reaches z1 only, through q1 (1 - q1):
        dL/dz1 = ce_w w / M (p1 - [t=1]) + dice_w g q1 (1 - q1),   dL/dz0 = ce_w w / M (p0 - [t=0]),
        g = -(2 [t=1] Dn - (2 I + s)) / Dn^2,   Dn = sum q1 + sum [t=1] + s + eps,   I = sum q1 [t=1]"""
    if activation == "softmax":
        return O.loss_and_dlogits_closed_form(logits, target, dice_weight, ce_weight, smooth, w0, sigma, imsize, eps)
    if activation != "sigmoid":
        raise NotImplementedError("only sigmoid and softmax are implemented")
    w = O.loss_weights(target, w0, sigma, imsize)
    t = target[:, 0]
    M = t.numel()
    z0, z1 = logits[:, 0], logits[:, 1]
    p = torch.softmax(logits, dim=1)
    ce = torch.sum(w * (torch.logsumexp(logits, dim=1) - torch.where(t > 0.5, z1, z0))) / M
    q1 = torch.sigmoid(z1)
    I, P, T = torch.sum(q1 * t), torch.sum(q1), torch.sum(t)
    Dn = P + T + smooth + eps
    loss = dice_weight * (1 - (2 * I + smooth) / Dn) + ce_weight * ce
    g = -(2 * t * Dn - (2 * I + smooth)) / (Dn * Dn)
    d1 = ce_weight * w / M * (p[:, 1] - t) + dice_weight * g * q1 * (1 - q1)
    d0 = ce_weight * w / M * (p[:, 0] - (1 - t))
    return loss, torch.stack([d0, d1], 1)


# --------------------------------------------------------------------------------------------------------------------
# fixture
# --------------------------------------------------------------------------------------------------------------------

def seeded_logits(t, seed=SEED):
    """(n,2,s,s) float32 logits for the target t (n,3,s,s): a partly trained net's, mostly but not always right, with
    every 7th row and 5th column scaled by 25 so that |z| reaches ~30 .. 200, where sigmoid and softmax saturate"""
    n, _, s, _ = t.shape
    rs = np.random.RandomState(seed + 1)
    z = rs.randn(n, 2, s, s).astype(np.float32) * 2
    z[:, 1] += 1.5 * (2 * t[:, 0] - 1)
    z[:, :, ::7, ::5] *= 25
    return z


def reference_config(activation):
    from oracle import ref_shim
    cfg = ref_shim.reference_unet_config(ENCODER, image_hw=(SIZE, SIZE))
    cfg["architecture_config"]["dice"]["dice_activation"] = activation
    return cfg


def golden_reference(mo):
    x, t = synthetic.train_batch(BATCH, SIZE, seed=SEED)
    X, T = torch.from_numpy(x), torch.from_numpy(t)
    rec = {}
    fit = {}
    for activation in ("sigmoid", "softmax"):
        torch.manual_seed(SEED)
        model = mo.PyTorchUNetWeighted(**reference_config(activation))
        if activation == "sigmoid":
            name, loss_fn, weight = model.loss_function[0]
            z = torch.from_numpy(seeded_logits(t)).requires_grad_(True)
            loss = loss_fn(z, T) * weight
            loss.backward()
            rec["loss"] = np.array(float(loss))
            rec["dlogits"] = z.grad.numpy().copy()
        fit[activation] = float(model._fit_loop([X, T])["sum"])
        if activation == "sigmoid":
            sd = model.model.state_dict()
            for k in DECODER_TAIL_KEYS:
                rec["step_" + k] = sd[k].numpy().reshape(-1)[:STEP_HEAD].copy()
    rec["fit_loss"] = np.array(fit["sigmoid"])
    rec["fit_loss_softmax"] = np.array(fit["softmax"])
    np.savez_compressed(GOLDEN, **rec)
    print("loss", float(rec["loss"]), "fit loss sigmoid", fit["sigmoid"], "softmax", fit["softmax"],
          os.path.getsize(GOLDEN) >> 10, "KiB", flush=True)


if __name__ == "__main__":
    warnings.filterwarnings("ignore")
    from oracle import ref_shim
    _, mo, _, _ = ref_shim.reference_modules()
    golden_reference(mo)
