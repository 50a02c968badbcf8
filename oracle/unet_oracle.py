"""TEST INFRASTRUCTURE — CPU fp32 oracle for the network, the losses and the train step.  Never imported by the
product path.

A functional restatement (torch CPU, float32) of
    UNetResNet.forward                      src/unet_models.py:338-403
    torchvision resnet34/101/152 blocks     torchvision/models/resnet.py (BasicBlock / Bottleneck; the reference
                                            pins torchvision 0.2.0, this image has 0.26 — same block arithmetic:
                                            stride on the 3x3, BN eps 1e-5 momentum 0.1, 1x1-s2 + BN downsample)
    DecoderBlockV2 / ConvRelu               src/unet_models.py:25-34,125-150
    multiclass_weighted_cross_entropy etc.  src/models.py:310-454, src/steps/pytorch/validation.py:8-28
    Model._fit_loop                         src/steps/pytorch/models.py:76-113 (Adam + L2, src/models.py:57,287-292)
driven by a reference-compatible state_dict (same keys; a `module.` prefix is accepted).

It is pinned to the real reference in the build container by tests/test_oracle_pins.py (bit-identical logits / loss
on the same state_dict, through oracle/ref_shim.py) and by the golden fixtures in tests/golden/.
"""
import math

import torch
import torch.nn.functional as F

LAYERS = {34: ("basic", [3, 4, 6, 3]), 101: ("bottleneck", [3, 4, 23, 3]), 152: ("bottleneck", [3, 8, 36, 3])}
BN_EPS = 1e-5
BN_MOMENTUM = 0.1


def strip_module_prefix(sd):
    return {(k[7:] if k.startswith("module.") else k): v for k, v in sd.items()}


def make_reference_like_state_dict(encoder_depth, num_classes=2, num_filters=32, seed=1234):
    """Random-init parameters with the reference's key set and init distributions: builds the same module tree
    the reference builds (torchvision resnet + torch default-initialised decoder) — without importing the
    reference — and returns its state_dict.  Deterministic for a given torch build and seed."""
    import torchvision
    torch.manual_seed(seed)
    enc = {34: torchvision.models.resnet34, 101: torchvision.models.resnet101,
           152: torchvision.models.resnet152}[encoder_depth](weights=None)
    bottom = 512 if encoder_depth == 34 else 2048
    nf = num_filters

    def dec(cin, mid, cout):
        return torch.nn.ModuleDict({"conv": torch.nn.Conv2d(cin, mid, 3, padding=1),
                                    "deconv": torch.nn.ConvTranspose2d(mid, cout, 4, 2, 1)})

    blocks = [("center", dec(bottom, nf * 16, nf * 8)), ("dec5", dec(bottom + nf * 8, nf * 16, nf * 8)),
              ("dec4", dec(bottom // 2 + nf * 8, nf * 16, nf * 8)), ("dec3", dec(bottom // 4 + nf * 8, nf * 8, nf * 2)),
              ("dec2", dec(bottom // 8 + nf * 2, nf * 4, nf * 4)), ("dec1", dec(nf * 4, nf * 4, nf))]
    dec0 = torch.nn.Conv2d(nf, nf, 3, padding=1)
    final = torch.nn.Conv2d(nf, num_classes, 1)
    sd = {}
    for k, v in enc.state_dict().items():
        sd["encoder." + k] = v
    # the reference registers the encoder stages a second time (src/unet_models.py:360-371)
    alias = {"conv1.0.": "conv1.", "conv1.1.": "bn1.", "conv2.": "layer1.", "conv3.": "layer2.", "conv4.": "layer3.",
             "conv5.": "layer4."}
    for new, old in alias.items():
        for k, v in enc.state_dict().items():
            if k.startswith(old):
                sd[new + k[len(old):]] = v
    for name, m in blocks:
        sd[name + ".block.0.conv.weight"] = m["conv"].weight.detach()
        sd[name + ".block.0.conv.bias"] = m["conv"].bias.detach()
        sd[name + ".block.1.weight"] = m["deconv"].weight.detach()
        sd[name + ".block.1.bias"] = m["deconv"].bias.detach()
    sd["dec0.conv.weight"] = dec0.weight.detach()
    sd["dec0.conv.bias"] = dec0.bias.detach()
    sd["final.weight"] = final.weight.detach()
    sd["final.bias"] = final.bias.detach()
    return sd


def conditioned_state_dict(encoder_depth, x, seed=1234, damp=0.25):
    """A well-conditioned stand-in for a TRAINED checkpoint (none can be downloaded here): the seed's random init with
    (1) the last BatchNorm scale of every residual block multiplied by `damp` -- residual branches of trained ResNets
    are small next to the identity path; at the raw init 33-50 undamped blocks amplify any rounding difference until
    deep gradients of two valid fp32 evaluations no longer correlate -- and (2) BatchNorm running statistics set to
    the batch statistics of `x` (one train-mode pass with momentum 1), so eval mode normalises like train mode instead
    of with the untouched (0, 1) buffers that make the raw-init net's eval activations explode."""
    sd = make_reference_like_state_dict(encoder_depth, seed=seed)
    last = "bn2" if encoder_depth == 34 else "bn3"
    seen = set()
    for k, v in sd.items():
        if k.startswith("encoder.layer") and k.endswith("." + last + ".weight") and id(v) not in seen:
            v.mul_(damp)       # the conv2..conv5 alias entries share these tensors
            seen.add(id(v))
    with torch.no_grad():
        UNetOracle(sd, encoder_depth, update_running_stats=True, momentum=1.0).forward(x, training=True)
    return sd


class _RoundBF16(torch.autograd.Function):
    """bf16 storage point: value rounded in forward, gradient rounded in backward (the CUDA path stores both
    activations and activation gradients as bf16)"""

    @staticmethod
    def forward(ctx, x):
        return x.to(torch.bfloat16).to(torch.float32)

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).to(torch.float32)


class _RoundWeightBF16(torch.autograd.Function):
    """bf16 operand copy of an fp32 master weight: rounded in forward, gradient passes through in fp32"""

    @staticmethod
    def forward(ctx, w):
        return w.to(torch.bfloat16).to(torch.float32)

    @staticmethod
    def backward(ctx, g):
        return g


class UNetOracle:
    """Functional forward over a state_dict.  training=True uses batch statistics and (optionally) updates the
    running statistics in `sd` in place, exactly like nn.BatchNorm2d.

    emulate_bf16=True inserts the CUDA path's storage roundings (bf16 conv operands, bf16-stored conv outputs,
    activations and activation gradients; fp32 accumulation, statistics, parameters and logits) so that the
    product can be compared at tight tolerance; emulate_bf16=False is the reference's fp32 arithmetic."""

    def __init__(self, sd, encoder_depth, update_running_stats=True, emulate_bf16=False, momentum=BN_MOMENTUM):
        self.momentum = momentum
        self.sd = strip_module_prefix(sd)
        self.depth = encoder_depth
        self.kind, self.blocks = LAYERS[encoder_depth]
        self.update = update_running_stats
        self.emu = emulate_bf16

    def _r(self, x):
        return _RoundBF16.apply(x) if self.emu else x

    def _w(self, key):
        w = self.sd[key]
        return _RoundWeightBF16.apply(w) if self.emu else w

    def _bn(self, x, prefix, training):
        sd = self.sd
        rm, rv = sd[prefix + ".running_mean"], sd[prefix + ".running_var"]
        if training and not self.update:
            rm, rv = rm.clone(), rv.clone()
        y = F.batch_norm(x, rm, rv, sd[prefix + ".weight"], sd[prefix + ".bias"], training, self.momentum, BN_EPS)
        if training and self.update and (prefix + ".num_batches_tracked") in sd:
            sd[prefix + ".num_batches_tracked"] += 1
        return y

    def _block(self, x, p, stride, training):
        sd = self.sd
        identity = x
        r, w = self._r, self._w
        if self.kind == "basic":
            out = r(F.conv2d(x, w(p + ".conv1.weight"), None, stride, 1))
            out = r(F.relu(self._bn(out, p + ".bn1", training)))
            out = r(F.conv2d(out, w(p + ".conv2.weight"), None, 1, 1))
            out = self._bn(out, p + ".bn2", training)
        else:
            out = r(F.conv2d(x, w(p + ".conv1.weight")))
            out = r(F.relu(self._bn(out, p + ".bn1", training)))
            out = r(F.conv2d(out, w(p + ".conv2.weight"), None, stride, 1))
            out = r(F.relu(self._bn(out, p + ".bn2", training)))
            out = r(F.conv2d(out, w(p + ".conv3.weight")))
            out = self._bn(out, p + ".bn3", training)
        if (p + ".downsample.0.weight") in sd:
            identity = r(F.conv2d(x, w(p + ".downsample.0.weight"), None, stride))
            identity = self._bn(identity, p + ".downsample.1", training)
        return r(F.relu(out + identity))

    def _layer(self, x, idx, training):
        for b in range(self.blocks[idx - 1]):
            stride = 2 if (b == 0 and idx > 1) else 1
            x = self._block(x, "encoder.layer%d.%d" % (idx, b), stride, training)
        return x

    def _decoder(self, x, name):
        sd = self.sd
        r, w = self._r, self._w
        x = r(F.relu(F.conv2d(x, w(name + ".block.0.conv.weight"), sd[name + ".block.0.conv.bias"], 1, 1)))
        x = F.conv_transpose2d(x, w(name + ".block.1.weight"), sd[name + ".block.1.bias"], stride=2, padding=1)
        return r(F.relu(x))

    def forward(self, x, training=False, return_intermediates=False):
        sd = self.sd
        r, w = self._r, self._w
        c1 = r(F.conv2d(r(x), w("encoder.conv1.weight"), None, 2, 3))
        c1 = r(F.relu(self._bn(c1, "encoder.bn1", training)))
        c1 = F.max_pool2d(c1, 2, 2)  # src/unet_models.py:356,363 — NOT torchvision's 3x3/s2 max-pool
        c2 = self._layer(c1, 1, training)
        c3 = self._layer(c2, 2, training)
        c4 = self._layer(c3, 3, training)
        c5 = self._layer(c4, 4, training)
        pool = F.max_pool2d(c5, 2, 2)
        center = self._decoder(pool, "center")
        d5 = self._decoder(torch.cat([center, c5], 1), "dec5")
        d4 = self._decoder(torch.cat([d5, c4], 1), "dec4")
        d3 = self._decoder(torch.cat([d4, c3], 1), "dec3")
        d2 = self._decoder(torch.cat([d3, c2], 1), "dec2")
        d1 = self._decoder(d2, "dec1")
        d0 = r(F.relu(F.conv2d(d1, w("dec0.conv.weight"), sd["dec0.conv.bias"], 1, 1)))
        logits = F.conv2d(d0, sd["final.weight"], sd["final.bias"])  # dropout2d(p=0) is the identity
        if return_intermediates:
            return logits, dict(conv1=c1, conv2=c2, conv3=c3, conv4=c4, conv5=c5, center=center, dec5=d5, dec4=d4,
                                dec3=d3, dec2=d2, dec1=d1, dec0=d0)
        return logits


# --------------------------------------------------------------------------------------------------------------------
# losses
# --------------------------------------------------------------------------------------------------------------------
def loss_weights(target, w0=50.0, sigma=10.0, imsize=(256, 256)):
    """get_weights / _get_distance_weights / _get_size_weights (src/models.py:339-381); target (N,3,H,W)"""
    d = target[:, 1]
    s = target[:, 2]
    C = math.sqrt(imsize[0] * imsize[1]) / 2.0
    wd = 1.0 + w0 * torch.exp(-(d ** 2) / (sigma ** 2))
    wd = torch.where(d == 0, torch.ones_like(wd), wd)
    s_ = torch.where(s == 0, torch.ones_like(s), s)
    ws = C / s_
    ws = torch.where(s_ == 1, torch.ones_like(ws), ws)
    return wd * ws


def weighted_cross_entropy(logits, target, w0=50.0, sigma=10.0, imsize=(256, 256)):
    """multiclass_weighted_cross_entropy (src/models.py:310-336)"""
    w = loss_weights(target, w0, sigma, imsize)
    t = target[:, 0].long()
    per_pixel = F.cross_entropy(logits, t, reduction="none")
    return torch.mean(per_pixel * w)


def dice_loss(logits, t, smooth=1.0, eps=1e-7, excluded_classes=(0,)):
    """multiclass_dice_loss + DiceLoss (src/models.py:421-454, src/steps/pytorch/validation.py:8-16)"""
    p = torch.softmax(logits, dim=1)
    loss = 0
    for c in range(logits.shape[1]):
        if c in excluded_classes:
            continue
        tc = (t == c).float()
        loss = loss + (1 - (2 * torch.sum(p[:, c] * tc) + smooth) / (torch.sum(p[:, c]) + torch.sum(tc) + smooth + eps))
    return loss


def mixed_loss(logits, target, dice_weight=0.2, ce_weight=1.0, smooth=1.0, w0=50.0, sigma=10.0, imsize=(256, 256)):
    """mixed_dice_cross_entropy_loss as configured by PyTorchUNetWeighted (src/models.py:149-161,384-418)"""
    t = target[:, 0].long()
    return dice_weight * dice_loss(logits, t, smooth) + ce_weight * weighted_cross_entropy(logits, target, w0, sigma,
                                                                                          imsize)


def plain_ce_loss(logits, target):
    """multiclass_segmentation_loss (src/steps/pytorch/validation.py:25-28)"""
    return F.cross_entropy(logits, target.squeeze(1).long())


def loss_and_dlogits_closed_form(logits, target, dice_weight=0.2, ce_weight=1.0, smooth=1.0, w0=50.0, sigma=10.0,
                                 imsize=(256, 256), eps=1e-7):
    """SURVEY.md Appendix C closed form (2 classes, class 0 excluded from Dice) — what the CUDA loss kernel
    implements; verified against autograd of mixed_loss in tests."""
    w = loss_weights(target, w0, sigma, imsize)
    t = target[:, 0]
    M = t.numel()
    z0, z1 = logits[:, 0], logits[:, 1]
    m = torch.maximum(z0, z1)
    e0, e1 = torch.exp(z0 - m), torch.exp(z1 - m)
    p1 = e1 / (e0 + e1)
    p0 = 1 - p1
    lse = m + torch.log(e0 + e1)
    zt = torch.where(t > 0.5, z1, z0)
    ce = torch.sum(w * (lse - zt)) / M
    I, P, T = torch.sum(p1 * t), torch.sum(p1), torch.sum(t)
    Dn = P + T + smooth + eps
    loss = dice_weight * (1 - (2 * I + smooth) / Dn) + ce_weight * ce
    g = -(2 * t * Dn - (2 * I + smooth)) / (Dn * Dn)
    d1 = ce_weight * w / M * (p1 - t) + dice_weight * g * p1 * p0
    d0 = ce_weight * w / M * (p0 - (1 - t)) - dice_weight * g * p1 * p0
    return loss, torch.stack([d0, d1], 1)


# --------------------------------------------------------------------------------------------------------------------
# train step
# --------------------------------------------------------------------------------------------------------------------
class AdamOracle:
    """torch.optim.Adam(params, lr, weight_decay=wd) (src/models.py:57,287-292): L2 folded into the gradient"""

    def __init__(self, lr=5e-4, weight_decay=1e-4, betas=(0.9, 0.999), eps=1e-8):
        self.lr, self.wd, self.betas, self.eps = lr, weight_decay, betas, eps
        self.m, self.v, self.t = {}, {}, 0

    def step(self, params, grads):
        self.t += 1
        b1, b2 = self.betas
        for k, p in params.items():
            g = grads.get(k)
            if g is None:
                continue
            g = g + self.wd * p
            m = self.m.setdefault(k, torch.zeros_like(p))
            v = self.v.setdefault(k, torch.zeros_like(p))
            m.mul_(b1).add_(g, alpha=1 - b1)
            v.mul_(b2).addcmul_(g, g, value=1 - b2)
            bc1, bc2 = 1 - b1 ** self.t, 1 - b2 ** self.t
            denom = (v.sqrt() / math.sqrt(bc2)).add_(self.eps)
            p.addcdiv_(m, denom, value=-self.lr / bc1)


def trainable_keys(sd):
    """unique trainable tensors: the `encoder.*` copies (aliases conv1..conv5 point at the same parameters) plus
    the decoder; buffers (running stats) and the unused encoder.fc are excluded from gradients but fc still gets
    weight decay in the reference only through grads (None -> skipped by Adam)."""
    keys = []
    for k in sd:
        if k.startswith(("conv1.", "conv2.", "conv3.", "conv4.", "conv5.")):
            continue
        if k.endswith(("running_mean", "running_var", "num_batches_tracked")):
            continue
        if k.startswith("encoder.fc."):
            continue
        keys.append(k)
    return keys


def train_step(sd, encoder_depth, x, target, opt, loss_fn=mixed_loss, **loss_kw):
    """one Model._fit_loop iteration on CPU: forward (train-mode BN), loss, backward, Adam.  Mutates sd in place
    (parameters and BN running statistics; aliases are kept in sync).  Returns (loss, logits, grads)."""
    sd_ = strip_module_prefix(sd)
    keys = trainable_keys(sd_)
    leaves = {k: sd_[k].detach().clone().requires_grad_(True) for k in keys}
    work = dict(sd_)
    work.update(leaves)
    alias = {"conv1.0.": "encoder.conv1.", "conv1.1.": "encoder.bn1.", "conv2.": "encoder.layer1.",
             "conv3.": "encoder.layer2.", "conv4.": "encoder.layer3.", "conv5.": "encoder.layer4."}
    net = UNetOracle(work, encoder_depth)
    logits = net.forward(x, training=True)
    loss = loss_fn(logits, target, **loss_kw)
    grads_list = torch.autograd.grad(loss, [leaves[k] for k in keys], allow_unused=True)
    grads = {k: g for k, g in zip(keys, grads_list)}
    with torch.no_grad():
        params = {k: leaves[k].detach() for k in keys}
        opt.step(params, grads)
        for k in keys:
            sd_[k].copy_(params[k])
        for k in sd_:
            if k.endswith(("running_mean", "running_var", "num_batches_tracked")) and k.startswith("encoder."):
                sd_[k].copy_(work[k])
        for new, old in alias.items():
            for k in list(sd_.keys()):
                if k.startswith(new) and (old + k[len(new):]) in sd_:
                    sd_[k].copy_(sd_[old + k[len(new):]])
    return loss.detach(), logits.detach(), grads
