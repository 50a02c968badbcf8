"""LIBRARY BASELINE — not part of the product path (nothing under open-solution-mapping-challenge_b200/ imports it).

"The baseline to beat on the same box" (SURVEY.md 2.3): the reference's network
(src/unet_models.py:338-403: torchvision ResNet encoder, DecoderBlockV2 with ConvTranspose2d(4, 2, 1),
ConvRelu, 1x1 classifier) and train step (src/steps/pytorch/models.py:76-113 with
PyTorchUNetWeighted's loss, src/models.py:310-454) written with STOCK PyTorch modules and run the way a
PyTorch user would run it on this GPU today: cuDNN / cuBLAS kernels, channels_last, bf16 autocast, torch.optim.Adam
(fused).  The reference itself is not imported: its torch-0.3 idioms (Variable, reduce=False) add nothing
but deprecation shims, hence the restatement; the module tree and state_dict keys are the reference's."""
import torch
import torch.nn.functional as F
import torchvision
from torch import nn


class ConvRelu(nn.Module):
    def __init__(self, in_, out):
        super().__init__()
        self.conv = nn.Conv2d(in_, out, 3, padding=1)

    def forward(self, x):
        return F.relu(self.conv(x), inplace=True)


class DecoderBlockV2(nn.Module):
    def __init__(self, in_channels, middle_channels, out_channels):
        super().__init__()
        self.block = nn.Sequential(ConvRelu(in_channels, middle_channels),
                                   nn.ConvTranspose2d(middle_channels, out_channels, kernel_size=4, stride=2, padding=1),
                                   nn.ReLU(inplace=True))

    def forward(self, x):
        return self.block(x)


class UNetResNet(nn.Module):
    def __init__(self, encoder_depth, num_classes=2, num_filters=32):
        super().__init__()
        self.encoder = {34: torchvision.models.resnet34, 101: torchvision.models.resnet101,
                        152: torchvision.models.resnet152}[encoder_depth](weights=None)
        bottom = 512 if encoder_depth == 34 else 2048
        nf = num_filters
        self.pool = nn.MaxPool2d(2, 2)
        e = self.encoder
        self.conv1 = nn.Sequential(e.conv1, e.bn1, e.relu, self.pool)
        self.conv2, self.conv3, self.conv4, self.conv5 = e.layer1, e.layer2, e.layer3, e.layer4
        self.center = DecoderBlockV2(bottom, nf * 16, nf * 8)
        self.dec5 = DecoderBlockV2(bottom + nf * 8, nf * 16, nf * 8)
        self.dec4 = DecoderBlockV2(bottom // 2 + nf * 8, nf * 16, nf * 8)
        self.dec3 = DecoderBlockV2(bottom // 4 + nf * 8, nf * 8, nf * 2)
        self.dec2 = DecoderBlockV2(bottom // 8 + nf * 2, nf * 4, nf * 4)
        self.dec1 = DecoderBlockV2(nf * 4, nf * 4, nf)
        self.dec0 = ConvRelu(nf, nf)
        self.final = nn.Conv2d(nf, num_classes, kernel_size=1)

    def forward(self, x):
        conv1 = self.conv1(x)
        conv2 = self.conv2(conv1)
        conv3 = self.conv3(conv2)
        conv4 = self.conv4(conv3)
        conv5 = self.conv5(conv4)
        center = self.center(self.pool(conv5))
        dec5 = self.dec5(torch.cat([center, conv5], 1))
        dec4 = self.dec4(torch.cat([dec5, conv4], 1))
        dec3 = self.dec3(torch.cat([dec4, conv3], 1))
        dec2 = self.dec2(torch.cat([dec3, conv2], 1))
        dec1 = self.dec1(dec2)
        return self.final(self.dec0(dec1))


class DecoderBlock(nn.Module):
    """UNet11's decoder block (src/unet_models.py:42-53): ConvRelu -> ConvTranspose2d(3, 2, 1, output_padding=1) -> ReLU"""

    def __init__(self, in_channels, middle_channels, out_channels):
        super().__init__()
        self.block = nn.Sequential(ConvRelu(in_channels, middle_channels),
                                   nn.ConvTranspose2d(middle_channels, out_channels, kernel_size=3, stride=2, padding=1,
                                                      output_padding=1),
                                   nn.ReLU(inplace=True))

    def forward(self, x):
        return self.block(x)


class UNetVGG(nn.Module):
    """UNet11 (src/unet_models.py:56-106) and UNetVGG16 with is_deconv=True, dropout 0 (src/unet_models.py:224-312):
    torchvision VGG features as the encoder, each stage output pooled and concatenated into the decoder"""
    STAGES = {11: ((0,), (3,), (6, 8), (11, 13), (16, 18)),
              16: ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21), (24, 26, 28))}

    def __init__(self, depth, num_classes=2, num_filters=32):
        super().__init__()
        self.encoder = {11: torchvision.models.vgg11, 16: torchvision.models.vgg16}[depth](weights=None).features
        self.stages = self.STAGES[depth]
        nf = num_filters
        if depth == 11:
            self.center = DecoderBlock(nf * 16, nf * 16, nf * 8)
            self.dec5 = DecoderBlock(nf * 24, nf * 16, nf * 8)
            self.dec4 = DecoderBlock(nf * 24, nf * 16, nf * 4)
            self.dec3 = DecoderBlock(nf * 12, nf * 8, nf * 2)
            self.dec2 = DecoderBlock(nf * 6, nf * 4, nf)
        else:
            self.center = DecoderBlockV2(512, nf * 16, nf * 8)
            self.dec5 = DecoderBlockV2(512 + nf * 8, nf * 16, nf * 8)
            self.dec4 = DecoderBlockV2(512 + nf * 8, nf * 16, nf * 8)
            self.dec3 = DecoderBlockV2(256 + nf * 8, nf * 8, nf * 2)
            self.dec2 = DecoderBlockV2(128 + nf * 2, nf * 4, nf)
        self.dec1 = ConvRelu(64 + nf, nf)
        self.final = nn.Conv2d(nf, num_classes, kernel_size=1)

    def forward(self, x):
        skips = []
        for si, stage in enumerate(self.stages):
            if si:
                x = F.max_pool2d(x, 2, 2)
            for idx in stage:
                x = F.relu(self.encoder[idx](x), inplace=True)
            skips.append(x)
        c1, c2, c3, c4, c5 = skips
        center = self.center(F.max_pool2d(c5, 2, 2))
        dec5 = self.dec5(torch.cat([center, c5], 1))
        dec4 = self.dec4(torch.cat([dec5, c4], 1))
        dec3 = self.dec3(torch.cat([dec4, c3], 1))
        dec2 = self.dec2(torch.cat([dec3, c2], 1))
        return self.final(self.dec1(torch.cat([dec2, c1], 1)))


def mixed_loss(logits, target, dice_weight=0.2, ce_weight=1.0, smooth=1.0, w0=50.0, sigma=10.0, imsize=(256, 256)):
    """PyTorchUNetWeighted's loss (src/models.py:149-161, 310-454) in plain torch ops"""
    logits = logits.float()
    mask, d, s = target[:, 0], target[:, 1], target[:, 2]
    c = (imsize[0] * imsize[1]) ** 0.5 / 2.0
    wd = torch.where(d == 0, torch.ones_like(d), 1.0 + w0 * torch.exp(-(d ** 2) / (sigma ** 2)))   # src/models.py:351-361
    s1 = torch.where(s == 0, torch.ones_like(s), s)
    ws = torch.where(s1 == 1, torch.ones_like(s1), c / s1)                                         # src/models.py:364-381
    w = wd * ws
    ce = F.cross_entropy(logits, mask.long(), reduction="none")
    wce = (ce * w).mean()
    p1 = torch.softmax(logits, 1)[:, 1]
    inter = (p1 * mask).sum()
    dice = 1.0 - (2.0 * inter + smooth) / (p1.sum() + mask.sum() + smooth + 1e-7)
    return dice_weight * dice + ce_weight * wce


class TrainStep:
    """zero_grad -> forward (bf16 autocast, channels_last) -> loss -> backward -> Adam(lr 5e-4, L2 1e-4), like _fit_loop"""

    def __init__(self, encoder_depth, device, lr=5e-4, weight_decay=1e-4, net=None):
        torch.backends.cudnn.benchmark = True
        self.net = (net if net is not None else UNetResNet(encoder_depth)).to(device).to(memory_format=torch.channels_last).train()
        self.opt = torch.optim.Adam(self.net.parameters(), lr=lr, weight_decay=weight_decay, fused=True)

    def step(self, x, target):
        x = x.contiguous(memory_format=torch.channels_last)
        self.opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            logits = self.net(x)
        loss = mixed_loss(logits, target)
        loss.backward()
        self.opt.step()
        return loss.detach()

    @classmethod
    def for_encoder(cls, encoder, device):
        """the train step of a src/models.py registry name.  The reference's AlbuNet (src/unet_models.py:153-221) is
        UNetResNet(34) without the classifier dropout, which this restatement never applies: the same net.  VGG11 / VGG16
        are UNet11 / UNetVGG16 (src/models.py:22-28)"""
        if encoder in ("VGG11", "VGG16"):
            return cls(None, device, net=UNetVGG(int(encoder[3:])))
        depth = {"AlbuNet": 34, "ResNet34": 34, "ResNet101": 101, "ResNet152": 152}[encoder]
        return cls(depth, device)

    @torch.no_grad()
    def infer(self, x):
        self.net.eval()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = torch.softmax(self.net(x.contiguous(memory_format=torch.channels_last)).float(), 1)
        self.net.train()
        return out
