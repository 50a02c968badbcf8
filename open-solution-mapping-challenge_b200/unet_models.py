"""Mirror of the reference's src/unet_models.py for the ResNet-encoder U-Net, executed by libmcb200.so.

`UNetResNet` keeps the reference's constructor, attribute tree and state_dict keys
(src/unet_models.py:315-403: encoder.*, conv1..conv5 aliases, center/dec5..dec1 `.block.{0.conv,1}`,
dec0.conv, final) so reference checkpoints load and src/pipelines.py / src/models.py drive it unchanged, but:

  * parameters live in ONE flat fp32 arena in the kernels' tap-major layout ([ky][kx][cout][cin]); every
    nn.Parameter is a (permuted) view of it, gradients are views of a second arena, and a bf16 operand copy of the
    arena feeds the tensor cores;
  * forward / backward are static launch plans over preallocated NHWC bf16 activations: wgmma implicit-GEMM convs
    with fused bias/ReLU/BN-statistics epilogues, fused BN+residual+ReLU passes, concat-free decoder convs, and are
    replayed as CUDA graphs;
  * there is no torch fallback: without the CUDA library or a CUDA input, forward raises.
"""
import math

import torch
import torchvision
from torch import nn

from . import ops

BN_MOMENTUM = 0.1
BN_EPS = 1e-5
_ALIGN = 64  # arena slot alignment in elements (TMA bases need 16 B, red.v4 needs 16 B)


class ConvRelu(nn.Module):
    """parameter container for conv3x3 + ReLU (reference src/unet_models.py:25-34)"""

    def __init__(self, in_, out):
        super().__init__()
        self.conv = nn.Conv2d(in_, out, 3, padding=1)
        self.activation = nn.ReLU(inplace=True)


class DecoderBlockV2(nn.Module):
    """parameter container for ConvRelu -> ConvTranspose2d(4, 2, 1) -> ReLU (reference src/unet_models.py:125-150)"""

    def __init__(self, in_channels, middle_channels, out_channels, is_deconv=True):
        super().__init__()
        self.in_channels = in_channels
        if not is_deconv:
            raise NotImplementedError("the H100 path implements the configured is_deconv=True decoder "
                                      "(src/models.py:32-46); the bilinear-upsample variant is not built")
        self.block = nn.Sequential(ConvRelu(in_channels, middle_channels),
                                   nn.ConvTranspose2d(middle_channels, out_channels, kernel_size=4, stride=2, padding=1),
                                   nn.ReLU(inplace=True))


class _Slot:
    __slots__ = ("off", "numel", "shape", "kind")


class UNetResNet(nn.Module):
    """PyTorch-facing U-Net with a ResNet-34/101/152 encoder; same signature as the reference class."""

    def __init__(self, encoder_depth, num_classes, num_filters=32, dropout_2d=0.2, pretrained=False, is_deconv=False):
        super().__init__()
        self.num_classes = num_classes
        self.dropout_2d = dropout_2d
        self.encoder_depth = encoder_depth
        self.num_filters = num_filters
        if pretrained:
            raise NotImplementedError("pretrained=True downloads ImageNet weights; load a state_dict instead")
        if encoder_depth == 34:
            self.encoder = torchvision.models.resnet34(weights=None)
            bottom = 512
        elif encoder_depth == 101:
            self.encoder = torchvision.models.resnet101(weights=None)
            bottom = 2048
        elif encoder_depth == 152:
            self.encoder = torchvision.models.resnet152(weights=None)
            bottom = 2048
        else:
            raise NotImplementedError('only 34, 101, 152 version of Resnet are implemented')
        self.bottom_channel_nr = bottom
        self.pool = nn.MaxPool2d(2, 2)
        self.relu = nn.ReLU(inplace=True)
        self.conv1 = nn.Sequential(self.encoder.conv1, self.encoder.bn1, self.encoder.relu, self.pool)
        self.conv2 = self.encoder.layer1
        self.conv3 = self.encoder.layer2
        self.conv4 = self.encoder.layer3
        self.conv5 = self.encoder.layer4
        nf = num_filters
        self.center = DecoderBlockV2(bottom, nf * 8 * 2, nf * 8, is_deconv)
        self.dec5 = DecoderBlockV2(bottom + nf * 8, nf * 8 * 2, nf * 8, is_deconv)
        self.dec4 = DecoderBlockV2(bottom // 2 + nf * 8, nf * 8 * 2, nf * 8, is_deconv)
        self.dec3 = DecoderBlockV2(bottom // 4 + nf * 8, nf * 4 * 2, nf * 2, is_deconv)
        self.dec2 = DecoderBlockV2(bottom // 8 + nf * 2, nf * 2 * 2, nf * 2 * 2, is_deconv)
        self.dec1 = DecoderBlockV2(nf * 2 * 2, nf * 2 * 2, nf, is_deconv)
        self.dec0 = ConvRelu(nf, nf)
        self.final = nn.Conv2d(nf, num_classes, kernel_size=1)
        self._slots = {}
        self._plans = {}
        self._p32 = self._g32 = self._w16 = None
        self._generation = 0   # bumped whenever the arenas are re-created (device move): plans, CUDA graphs and fused
        self._build_arenas()   # train steps that baked the old pointers in are stale from then on

    # ------------------------------------------------------------------------------------------------ arenas
    def _arena_params(self):
        """unique trainable tensors that the kernels use (encoder.fc is never used by forward)"""
        convt = {id(m.weight) for m in self.modules() if isinstance(m, nn.ConvTranspose2d)}
        seen, out = set(), []
        for name, p in self.named_parameters():
            if id(p) in seen or name.startswith("encoder.fc."):
                continue
            seen.add(id(p))
            out.append((name, p, "convt" if id(p) in convt else ("conv" if p.dim() == 4 else "vec")))
        return out

    def _build_arenas(self):
        params = self._arena_params()
        dev = params[0][1].device
        total = 0
        slots = {}
        for name, p, kind in params:
            assert p.dtype == torch.float32, "the H100 path keeps fp32 master weights (got %s for %s)" % (p.dtype, name)
            s = _Slot()
            s.off, s.numel, s.shape, s.kind = total, p.numel(), tuple(p.shape), kind
            slots[id(p)] = s
            total += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        p32 = torch.zeros(total, dtype=torch.float32, device=dev)
        g32 = torch.zeros(total, dtype=torch.float32, device=dev)
        for name, p, kind in params:
            s = slots[id(p)]
            view = self._view(p32, s)
            view.copy_(p.data)
            p.data = view
            p.grad = None
        self._slots, self._p32, self._g32 = slots, p32, g32
        self._w16 = torch.zeros(total, dtype=torch.bfloat16, device=dev)
        self._plans = {}
        self._generation += 1

    def _params_alias_arena(self):
        """every arena parameter still is a view of the current master arena (no .to()/.cpu() moved it away)"""
        if self._p32 is None:
            return False
        base, dev = self._p32.data_ptr(), self._p32.device
        for _, p, _ in self._arena_params():
            s = self._slots.get(id(p))
            if s is None or p.device != dev or p.dtype != torch.float32 or p.data_ptr() != base + 4 * s.off:
                return False
        return True

    @staticmethod
    def _view(arena, s):
        flat = arena[s.off:s.off + s.numel]
        if s.kind == "conv":
            co, ci, kh, kw = s.shape
            return flat.view(kh, kw, co, ci).permute(2, 3, 0, 1)
        if s.kind == "convt":
            ci, co, kh, kw = s.shape
            return flat.view(kh, kw, co, ci).permute(3, 2, 0, 1)
        return flat.view(s.shape)

    def _apply(self, fn, *args, **kwargs):
        """.cuda() / .cpu() / .to(): nn.Module moves each parameter's data separately, which tears the views off the
        arena -- re-pack them into fresh arenas on the new device.  A call that moves nothing (`.cuda()` on a model that
        already lives there: the reference's save_model does model.cpu(); save; model.cuda() every checkpoint,
        src/steps/pytorch/utils.py:67-75, and `_to_device` runs every batch) keeps arenas, plans and graphs."""
        super()._apply(fn, *args, **kwargs)
        if not self._params_alias_arena():
            self._build_arenas()
        return self

    def state_dict(self, *args, **kwargs):
        sd = super().state_dict(*args, **kwargs)
        if kwargs.get("keep_vars", False):
            return sd
        for k, v in sd.items():
            if isinstance(v, torch.Tensor) and v.dim() == 4 and not v.is_contiguous():
                sd[k] = v.detach().clone(memory_format=torch.contiguous_format)
        return sd

    def grad_views(self):
        return [(p, self._view(self._g32, self._slots[id(p)])) for _, p, _ in self._arena_params()]

    def _packed(self, p, arena):
        """(taps, cout, cin) view of a conv / convT weight inside `arena`"""
        s = self._slots[id(p)]
        flat = arena[s.off:s.off + s.numel]
        if s.kind == "conv":
            co, ci, kh, kw = s.shape
        else:
            ci, co, kh, kw = s.shape
        return flat.view(kh * kw, co, ci)

    def _vec(self, p, arena):
        s = self._slots[id(p)]
        return arena[s.off:s.off + s.numel]

    def refresh_operands(self):
        """bf16 operand copy of the fp32 master arena (done by the fused Adam kernel on the fused train path)"""
        ops.cast_bf16(self._p32, self._w16)

    # ------------------------------------------------------------------------------------------------ forward
    def _check_input(self, x):
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise RuntimeError("UNetResNet (H100 path) needs a CUDA tensor; there is no CPU fallback")
        if self._p32 is None or not self._p32.is_cuda:
            raise RuntimeError("UNetResNet (H100 path): call .cuda() on the model first; there is no CPU fallback")
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("expected input (N, 3, H, W), got %s" % (tuple(x.shape),))
        if x.shape[2] % 64 != 0 or x.shape[3] % 64 != 0:
            # the reference fails in torch.cat for such sizes (SURVEY.md 0.3)
            raise RuntimeError("UNetResNet needs H and W divisible by 64, got %dx%d" % (x.shape[2], x.shape[3]))
        if self.dropout_2d != 0:
            raise NotImplementedError("dropout_2d must be 0.0 (the configured value, src/models.py:32-46)")

    def plan(self, n, h, w, training):
        key = (n, h, w, bool(training))
        pl = self._plans.get(key)
        if pl is None:
            from .engine import Plan
            pl = Plan(self, n, h, w, bool(training))
            self._plans[key] = pl
        return pl

    def forward(self, x):
        self._check_input(x)
        x = x.contiguous().float()
        pl = self.plan(x.shape[0], x.shape[2], x.shape[3], self.training)
        if torch.is_grad_enabled() and self.training:
            if pl.sync_bn:
                raise NotImplementedError("MCB_SYNC_BN needs the fused train step (mcb200.models.PyTorchUNet*): the "
                                          "autograd bridge leaves gradient reduction to the caller")
            from .engine import UNetFunction
            return UNetFunction.apply(x, self, pl, *[p for _, p, _ in self._arena_params()])
        self.refresh_operands()
        return pl.forward(x).clone()
