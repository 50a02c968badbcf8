"""TEST INFRASTRUCTURE -- fixtures for the encoder-registry nets beyond UNetResNet (src/models.py:22-47), one file per
case under tests/golden/encoders_<tag>.npz, plus the bf16-storage deviation of each case:

    MCB_REFERENCE_ROOT=<checkout> python -m oracle.make_golden_encoders reference   (runs the UNMODIFIED reference, CPU)
    python -m oracle.make_golden_encoders deviation                                 (CPU oracle only, reads the above)

`reference` records, per case, from the reference's own PyTorchUNetWeighted(**config) built under torch.manual_seed(1234):
  * the initial state_dict: keys, shapes and a SHA-256 per tensor, and the same for the reference's UNetResNet(34) under
    the same seed (AlbuNet is that network without the classifier dropout);
  * the algorithmic forward FLOPs of one 320x320 tile, from forward hooks on every Conv2d / ConvTranspose2d;
  * eval logits (image 0) and train logits at every LOGIT_STRIDE-th pixel, the loss, and the leading ENCODER_GRAD_HEAD
    elements of the gradients of the first, a middle and the last encoder conv and of every decoder conv;
  * the loss of one reference _fit_loop step and the leading STEP_HEAD elements of STEP_KEYS after it.
Inputs and initial weights are not stored: both sides regenerate them from the seed.

`deviation` runs oracle.unet_oracle.UNetOracle(emulate_bf16=True) -- the CUDA path's storage roundings on the CPU -- on
the same weights and inputs and writes tests/golden/emulated_bf16_deviation_encoders.json: per case the logits' max-abs
deviation (train and eval) and per gradient tensor the relative L2 deviation and cosine against the reference."""
import hashlib
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

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
DEVIATION_JSON = os.path.join(GOLDEN_DIR, "emulated_bf16_deviation_encoders.json")
SEED = 1234
# (tag, registry name, ResNet depth of the oracle restatement, batch, size)
ENCODER_CASES = (("albunet_b2_256", "AlbuNet", 34, 2, 256),)
ENCODER_GRAD_KEYS = ("encoder.conv1.weight", "encoder.layer2.0.conv1.weight", "encoder.layer4.2.conv2.weight") + tuple(
    "%s.%s" % (blk, p) for blk in ("center", "dec5", "dec4", "dec3", "dec2", "dec1")
    for p in ("block.0.conv.weight", "block.1.weight")) + ("dec0.conv.weight", "final.weight", "final.bias")
ENCODER_GRAD_HEAD = 8192
STEP_KEYS = ("final.weight", "final.bias", "dec0.conv.weight", "dec0.conv.bias", "dec1.block.1.bias",
             "center.block.1.bias", "encoder.bn1.running_mean", "encoder.bn1.running_var",
             "encoder.layer4.2.bn2.running_mean", "encoder.layer4.2.bn2.running_var")
STEP_HEAD = 4096
FLOP_TILE = 320


def golden_path(tag):
    return os.path.join(GOLDEN_DIR, "encoders_%s.npz" % tag)


def tensor_sha256(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def state_dict_digest(sd):
    """-> (keys, json {key: shape}, sha256 per key) of a state_dict, in its order"""
    keys = list(sd)
    return (np.array(keys), np.array(json.dumps({k: list(sd[k].shape) for k in keys})),
            np.array([tensor_sha256(sd[k]) for k in keys]))


def hooked_forward_flops(net, size):
    """2 x multiply-adds of every Conv2d / ConvTranspose2d in one eval forward of a (1, 3, size, size) tile"""
    total = [0]

    def hook(m, inp, out):
        kh, kw = m.kernel_size
        if isinstance(m, torch.nn.ConvTranspose2d):
            total[0] += 2 * inp[0].numel() * m.out_channels * kh * kw // m.groups
        else:
            total[0] += 2 * out.numel() * m.in_channels * kh * kw // m.groups
    hs = [m.register_forward_hook(hook) for m in net.modules() if isinstance(m, (torch.nn.Conv2d, torch.nn.ConvTranspose2d))]
    was = net.training
    net.eval()
    with torch.no_grad():
        net(torch.zeros(1, 3, size, size))
    net.train(was)
    for h in hs:
        h.remove()
    return total[0]


def golden_reference(um, mo):
    from oracle import ref_shim
    for tag, enc, depth, n, s in ENCODER_CASES:
        rec = {}
        cfg = ref_shim.reference_unet_config(enc, image_hw=(256, 256))
        torch.manual_seed(SEED)
        model = mo.PyTorchUNetWeighted(**cfg)
        net = model.model
        rec["init_keys"], rec["init_shapes"], rec["init_sha256"] = state_dict_digest(net.state_dict())
        torch.manual_seed(SEED)
        twin = um.UNetResNet(depth, 2, 32, 0.0, False, True)
        rec["twin_keys"], rec["twin_shapes"], rec["twin_sha256"] = state_dict_digest(twin.state_dict())
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
        for k in ENCODER_GRAD_KEYS:
            rec["grad_" + k] = params[k].grad.detach().numpy().reshape(-1)[:ENCODER_GRAD_HEAD].copy()
        # one reference train step from the untouched initialisation (the forward above moved the running statistics)
        torch.manual_seed(SEED)
        model = mo.PyTorchUNetWeighted(**cfg)
        rec["fit_loss"] = np.array(float(model._fit_loop([X, T])["sum"]))
        sd = model.model.state_dict()
        for k in STEP_KEYS:
            rec["step_" + k] = sd[k].numpy().reshape(-1)[:STEP_HEAD].copy()
        np.savez_compressed(golden_path(tag), **rec)
        print(tag, "loss", float(loss), "fit loss", float(rec["fit_loss"]), "fwd GFLOP/tile @%d" % FLOP_TILE,
              int(rec["fwd_flops_%d" % FLOP_TILE]) / 1e9, os.path.getsize(golden_path(tag)) >> 10, "KiB", flush=True)


def emulated_deviation(tag, depth, n, s):
    """bf16-storage deviation of one case against its reference fixture (see module docstring)"""
    from oracle import unet_oracle as O
    g = np.load(golden_path(tag))
    x, t = synthetic.train_batch(n, s, seed=SEED)
    X, T = torch.from_numpy(x), torch.from_numpy(t)
    sd = O.make_reference_like_state_dict(depth, seed=SEED)
    with torch.no_grad():
        ev = O.UNetOracle({k: v.clone() for k, v in sd.items()}, depth, update_running_stats=False,
                          emulate_bf16=True).forward(X[:1], training=False)
    leaves = {k: sd[k].clone().requires_grad_(True) for k in O.trainable_keys(sd)}
    work = dict(sd)
    work.update(leaves)
    logits = O.UNetOracle(work, depth, update_running_stats=False, emulate_bf16=True).forward(X, training=True)
    loss = O.mixed_loss(logits, T, imsize=(256, 256))
    grads = torch.autograd.grad(loss, [leaves[k] for k in ENCODER_GRAD_KEYS])
    st = LOGIT_STRIDE
    rec = {"train_logits_max_abs": float(np.abs(logits.detach().numpy()[:, :, ::st, ::st] - g["train_logits"]).max()),
           "eval_logits_max_abs": float(np.abs(ev.numpy()[:, :, ::st, ::st] - g["eval_logits"]).max()),
           "loss_rel": abs(float(loss) - float(g["loss"])) / abs(float(g["loss"])), "grads": {}}
    for k, gr in zip(ENCODER_GRAD_KEYS, grads):
        r = torch.from_numpy(g["grad_" + k]).double()
        a = gr.detach().reshape(-1)[:ENCODER_GRAD_HEAD].double()
        rec["grads"][k] = {"rel": float((a - r).norm() / r.norm()), "cos": float((a * r).sum() / (a.norm() * r.norm()))}
    return rec


def golden_deviation():
    out = {}
    for tag, enc, depth, n, s in ENCODER_CASES:
        out[tag] = emulated_deviation(tag, depth, n, s)
        print(tag, json.dumps(out[tag]), flush=True)
    with open(DEVIATION_JSON, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    warnings.filterwarnings("ignore")
    which = sys.argv[1:] or ["reference", "deviation"]
    if "reference" in which:
        from oracle import ref_shim
        um, mo, _, _ = ref_shim.reference_modules()
        golden_reference(um, mo)
    if "deviation" in which:
        golden_deviation()
