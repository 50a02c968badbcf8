"""TEST INFRASTRUCTURE -- CPU fp32 oracle for the VGG-encoder U-Nets.  Never imported by the product path.

A functional restatement (torch CPU, float32) of
    UNet11.forward                          src/unet_models.py:56-106 (DecoderBlock, 3x3 transposed conv)
    UNetVGG16.forward                       src/unet_models.py:224-312 (DecoderBlockV2, is_deconv=True, dropout 0)
driven by a reference-compatible state_dict (same keys; a `module.` prefix is accepted).  emulate_bf16=True inserts the
CUDA path's storage roundings (bf16 image, conv operands, conv outputs and activation gradients; fp32 accumulation,
biases, classifier and logits), as oracle/unet_oracle.py does for the ResNets.  The losses and Adam are
oracle/unet_oracle.py's.
"""
import torch
import torch.nn.functional as F

from oracle.unet_oracle import AdamOracle, _RoundBF16, _RoundWeightBF16, mixed_loss, strip_module_prefix  # noqa: F401

# encoder (torchvision vgg.features) indices of each stage's convs, and the reference's alias names for them
STAGES = {"VGG11": ((0,), (3,), (6, 8), (11, 13), (16, 18)),
          "VGG16": ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21), (24, 26, 28))}
ALIASES = {"VGG11": {"conv1": 0, "conv2": 3, "conv3s": 6, "conv3": 8, "conv4s": 11, "conv4": 13, "conv5s": 16,
                     "conv5": 18},
           "VGG16": {"conv%d.%d" % (s + 1, 2 * j): idx for s, st in enumerate(STAGES["VGG16"])
                     for j, idx in enumerate(st)}}


def _decoder_channels(enc, nf=32):
    """(name, in, mid, out) of center, dec5..dec2 and the (in, out) of dec1"""
    if enc == "VGG11":
        blocks = [("center", nf * 16, nf * 16, nf * 8), ("dec5", nf * 24, nf * 16, nf * 8),
                  ("dec4", nf * 24, nf * 16, nf * 4), ("dec3", nf * 12, nf * 8, nf * 2), ("dec2", nf * 6, nf * 4, nf)]
        return blocks, (nf * 3, nf)
    blocks = [("center", 512, nf * 16, nf * 8), ("dec5", 512 + nf * 8, nf * 16, nf * 8),
              ("dec4", 512 + nf * 8, nf * 16, nf * 8), ("dec3", 256 + nf * 8, nf * 8, nf * 2),
              ("dec2", 128 + nf * 2, nf * 4, nf)]
    return blocks, (64 + nf, nf)


def make_reference_like_state_dict(enc, num_classes=2, num_filters=32, seed=1234):
    """Random-init parameters with the reference's keys, key order and init: the whole torchvision VGG is built (its
    classifier consumes the random stream as the reference's does), then the decoder modules in the reference's order.
    Deterministic for a given torch build and seed."""
    import torchvision
    torch.manual_seed(seed)
    features = {"VGG11": torchvision.models.vgg11, "VGG16": torchvision.models.vgg16}[enc](weights=None).features
    kt = 3 if enc == "VGG11" else 4
    blocks, (c1_in, c1_out) = _decoder_channels(enc, num_filters)
    mods = []
    for name, cin, mid, cout in blocks:
        conv = torch.nn.Conv2d(cin, mid, 3, padding=1)
        if kt == 3:
            deconv = torch.nn.ConvTranspose2d(mid, cout, 3, 2, 1, output_padding=1)
        else:
            deconv = torch.nn.ConvTranspose2d(mid, cout, 4, 2, 1)
        mods.append((name, conv, deconv))
    dec1 = torch.nn.Conv2d(c1_in, c1_out, 3, padding=1)
    final = torch.nn.Conv2d(num_filters, num_classes, 1)
    sd = {}
    for k, v in features.state_dict().items():
        sd["encoder." + k] = v
    for alias, idx in ALIASES[enc].items():
        sd[alias + ".weight"] = sd["encoder.%d.weight" % idx]
        sd[alias + ".bias"] = sd["encoder.%d.bias" % idx]
    for name, conv, deconv in mods:
        sd[name + ".block.0.conv.weight"] = conv.weight.detach()
        sd[name + ".block.0.conv.bias"] = conv.bias.detach()
        sd[name + ".block.1.weight"] = deconv.weight.detach()
        sd[name + ".block.1.bias"] = deconv.bias.detach()
    sd["dec1.conv.weight"] = dec1.weight.detach()
    sd["dec1.conv.bias"] = dec1.bias.detach()
    sd["final.weight"] = final.weight.detach()
    sd["final.bias"] = final.bias.detach()
    return sd


def trainable_keys(sd, enc):
    """unique trainable tensors: encoder.* and the decoder (the conv1..conv5 aliases point at encoder tensors)"""
    alias = tuple(a + "." for a in ALIASES[enc])
    return [k for k in sd if not k.startswith(alias)]


class VGGUNetOracle:
    """Functional forward of UNet11 ("VGG11") or UNetVGG16 ("VGG16") over a state_dict (no BatchNorm: train and eval
    mode compute the same)"""

    def __init__(self, sd, enc, emulate_bf16=False):
        self.sd = strip_module_prefix(sd)
        self.enc = enc
        self.emu = emulate_bf16

    def _r(self, x):
        return _RoundBF16.apply(x) if self.emu else x

    def _w(self, key):
        w = self.sd[key]
        return _RoundWeightBF16.apply(w) if self.emu else w

    def _conv_relu(self, x, prefix):
        return self._r(F.relu(F.conv2d(x, self._w(prefix + ".weight"), self.sd[prefix + ".bias"], 1, 1)))

    def _decoder(self, x, name):
        sd = self.sd
        x = self._conv_relu(x, name + ".block.0.conv")
        wt = self._w(name + ".block.1.weight")
        if wt.shape[-1] == 3:
            x = F.conv_transpose2d(x, wt, sd[name + ".block.1.bias"], stride=2, padding=1, output_padding=1)
        else:
            x = F.conv_transpose2d(x, wt, sd[name + ".block.1.bias"], stride=2, padding=1)
        return self._r(F.relu(x))

    def forward(self, x, training=False, return_intermediates=False):
        sd = self.sd
        cur = self._r(x)
        skips = []
        for si, stage in enumerate(STAGES[self.enc]):
            if si > 0:
                cur = F.max_pool2d(cur, 2, 2)
            for idx in stage:
                cur = self._conv_relu(cur, "encoder.%d" % idx)
            skips.append(cur)
        c1, c2, c3, c4, c5 = skips
        center = self._decoder(F.max_pool2d(c5, 2, 2), "center")
        d5 = self._decoder(torch.cat([center, c5], 1), "dec5")
        d4 = self._decoder(torch.cat([d5, c4], 1), "dec4")
        d3 = self._decoder(torch.cat([d4, c3], 1), "dec3")
        d2 = self._decoder(torch.cat([d3, c2], 1), "dec2")
        d1 = self._conv_relu(torch.cat([d2, c1], 1), "dec1.conv")
        logits = F.conv2d(d1, sd["final.weight"], sd["final.bias"])   # dropout2d(p=0) is the identity
        if return_intermediates:
            return logits, dict(conv1=c1, conv2=c2, conv3=c3, conv4=c4, conv5=c5, center=center, dec5=d5, dec4=d4,
                                dec3=d3, dec2=d2, dec1=d1)
        return logits


def train_step(sd, enc, x, target, opt, loss_fn=mixed_loss, emulate_bf16=False, **loss_kw):
    """one Model._fit_loop iteration on CPU: forward, loss, backward, Adam.  Mutates sd in place (aliases are kept in
    sync).  Returns (loss, logits, grads)."""
    sd_ = strip_module_prefix(sd)
    keys = trainable_keys(sd_, enc)
    leaves = {k: sd_[k].detach().clone().requires_grad_(True) for k in keys}
    work = dict(sd_)
    work.update(leaves)
    logits = VGGUNetOracle(work, enc, emulate_bf16).forward(x, training=True)
    loss = loss_fn(logits, target, **loss_kw)
    grads = dict(zip(keys, torch.autograd.grad(loss, [leaves[k] for k in keys])))
    with torch.no_grad():
        params = {k: leaves[k].detach() for k in keys}
        opt.step(params, grads)
        for k in keys:
            sd_[k].copy_(params[k])
        for alias, idx in ALIASES[enc].items():
            for p in ("weight", "bias"):
                sd_["%s.%s" % (alias, p)].copy_(sd_["encoder.%d.%s" % (idx, p)])
    return loss.detach(), logits.detach(), grads
