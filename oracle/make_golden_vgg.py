"""TEST INFRASTRUCTURE -- fixtures for the VGG-encoder U-Nets of the encoder registry (src/models.py:22-28), one file per
case under tests/golden/encoders_<tag>.npz, plus the bf16-storage deviation of each case:

    MCB_REFERENCE_ROOT=<checkout> python -m oracle.make_golden_vgg reference   (runs the UNMODIFIED reference, CPU)
    python -m oracle.make_golden_vgg deviation                                 (CPU oracle only, reads the above)

The record layout is oracle/make_golden_encoders.py's (AlbuNet), without the twin network.  `reference` records, per
case, from the reference's own PyTorchUNetWeighted(**config) built under torch.manual_seed(1234) (oracle/ref_shim.py
forces pretrained=False):
  * the initial state_dict: keys, shapes and a SHA-256 per tensor;
  * the algorithmic forward FLOPs of one 320x320 tile, from forward hooks on every Conv2d / ConvTranspose2d;
  * eval logits (image 0) and train logits at every LOGIT_STRIDE-th pixel, the loss, and the leading ENCODER_GRAD_HEAD
    elements of the gradients of the first, a middle and the last encoder conv, of every decoder conv and of final;
  * the loss of one reference _fit_loop step and the leading STEP_HEAD elements of STEP_KEYS after it.
Inputs and initial weights are not stored: both sides regenerate them from the seed.

`deviation` runs oracle.vgg_oracle.VGGUNetOracle(emulate_bf16=True) on the same weights and inputs and writes
tests/golden/emulated_bf16_deviation_vgg.json: per case the logits' max-abs deviation (train and eval), the loss's
relative deviation and per gradient tensor the relative L2 deviation and cosine against the reference."""
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import synthetic  # noqa: E402
from oracle.make_golden_cases import LOGIT_STRIDE  # noqa: E402
from oracle.make_golden_encoders import (ENCODER_GRAD_HEAD, FLOP_TILE, SEED, STEP_HEAD, golden_path,  # noqa: E402
                                         hooked_forward_flops, state_dict_digest)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
DEVIATION_JSON = os.path.join(GOLDEN_DIR, "emulated_bf16_deviation_vgg.json")
# (tag, registry name, batch, size)
VGG_CASES = (("vgg11_b2_256", "VGG11", 2, 256), ("vgg16_b2_256", "VGG16", 2, 256))
_DECODER_GRADS = tuple("%s.%s" % (blk, p) for blk in ("center", "dec5", "dec4", "dec3", "dec2")
                       for p in ("block.0.conv.weight", "block.1.weight")) + ("dec1.conv.weight", "final.weight",
                                                                              "final.bias")
GRAD_KEYS = {"VGG11": ("encoder.0.weight", "encoder.8.weight", "encoder.18.weight") + _DECODER_GRADS,
             "VGG16": ("encoder.0.weight", "encoder.14.weight", "encoder.28.weight") + _DECODER_GRADS}
STEP_KEYS = ("final.weight", "final.bias", "dec1.conv.weight", "dec1.conv.bias", "dec2.block.1.bias",
             "center.block.1.bias", "encoder.0.weight", "encoder.0.bias")


def golden_reference(mo):
    from oracle import ref_shim
    for tag, enc, n, s in VGG_CASES:
        rec = {}
        cfg = ref_shim.reference_unet_config(enc, image_hw=(256, 256))
        torch.manual_seed(SEED)
        model = mo.PyTorchUNetWeighted(**cfg)
        net = model.model
        rec["init_keys"], rec["init_shapes"], rec["init_sha256"] = state_dict_digest(net.state_dict())
        rec["fwd_flops_%d" % FLOP_TILE] = np.array(hooked_forward_flops(net, FLOP_TILE), dtype=np.int64)
        x, t = synthetic.train_batch(n, s, seed=SEED)
        X, T = torch.from_numpy(x), torch.from_numpy(t)
        net.eval()
        with torch.no_grad():
            rec["eval_logits"] = net(X[:1]).numpy()[:, :, ::LOGIT_STRIDE, ::LOGIT_STRIDE].copy()
        net.train()
        out = net(X)
        name, loss_fn, weight = model.loss_function[0]
        loss = loss_fn(out, T) * weight
        loss.backward()
        rec["train_logits"] = out.detach().numpy()[:, :, ::LOGIT_STRIDE, ::LOGIT_STRIDE].copy()
        rec["loss"] = np.array(float(loss))
        params = dict(net.named_parameters())
        for k in GRAD_KEYS[enc]:
            rec["grad_" + k] = params[k].grad.detach().numpy().reshape(-1)[:ENCODER_GRAD_HEAD].copy()
        # one reference train step from the untouched initialisation
        torch.manual_seed(SEED)
        model = mo.PyTorchUNetWeighted(**cfg)
        rec["fit_loss"] = np.array(float(model._fit_loop([X, T])["sum"]))
        sd = model.model.state_dict()
        for k in STEP_KEYS:
            rec["step_" + k] = sd[k].numpy().reshape(-1)[:STEP_HEAD].copy()
        np.savez_compressed(golden_path(tag), **rec)
        print(tag, "loss", float(loss), "fit loss", float(rec["fit_loss"]), "fwd GFLOP/tile @%d" % FLOP_TILE,
              int(rec["fwd_flops_%d" % FLOP_TILE]) / 1e9, os.path.getsize(golden_path(tag)) >> 10, "KiB", flush=True)


def emulated_deviation(tag, enc, n, s):
    """bf16-storage deviation of one case against its reference fixture (see module docstring)"""
    from oracle import vgg_oracle as V
    g = np.load(golden_path(tag))
    x, t = synthetic.train_batch(n, s, seed=SEED)
    X, T = torch.from_numpy(x), torch.from_numpy(t)
    sd = V.make_reference_like_state_dict(enc, seed=SEED)
    with torch.no_grad():
        ev = V.VGGUNetOracle(sd, enc, emulate_bf16=True).forward(X[:1])
    leaves = {k: sd[k].clone().requires_grad_(True) for k in V.trainable_keys(sd, enc)}
    work = dict(sd)
    work.update(leaves)
    logits = V.VGGUNetOracle(work, enc, emulate_bf16=True).forward(X, training=True)
    loss = V.mixed_loss(logits, T, imsize=(256, 256))
    keys = GRAD_KEYS[enc]
    grads = torch.autograd.grad(loss, [leaves[k] for k in keys])
    st = LOGIT_STRIDE
    rec = {"train_logits_max_abs": float(np.abs(logits.detach().numpy()[:, :, ::st, ::st] - g["train_logits"]).max()),
           "eval_logits_max_abs": float(np.abs(ev.numpy()[:, :, ::st, ::st] - g["eval_logits"]).max()),
           "loss_rel": abs(float(loss) - float(g["loss"])) / abs(float(g["loss"])), "grads": {}}
    for k, gr in zip(keys, grads):
        r = torch.from_numpy(g["grad_" + k]).double()
        a = gr.detach().reshape(-1)[:ENCODER_GRAD_HEAD].double()
        rec["grads"][k] = {"rel": float((a - r).norm() / r.norm()), "cos": float((a * r).sum() / (a.norm() * r.norm()))}
    return rec


def golden_deviation():
    out = {}
    for tag, enc, n, s in VGG_CASES:
        out[tag] = emulated_deviation(tag, enc, n, s)
        print(tag, json.dumps(out[tag]), flush=True)
    with open(DEVIATION_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    warnings.filterwarnings("ignore")
    which = sys.argv[1:] or ["reference", "deviation"]
    if "reference" in which:
        from oracle import ref_shim
        _, mo, _, _ = ref_shim.reference_modules()
        golden_reference(mo)
    if "deviation" in which:
        golden_deviation()
