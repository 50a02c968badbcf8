"""TEST INFRASTRUCTURE -- the case list and file layout of the U-Net fixtures tests/golden/unet_{configs,conditioned}_*.npz,
shared by their generator (oracle/make_golden.py) and the tests that read them."""
import glob
import os

import numpy as np

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
# BASELINE.json configs: config 1 verbatim (R34 b2 @256), the headline net at the headline resolution (R101 @320, batch
# cut to 2 so the CPU reference finishes in seconds), config 5's net and resolution (R152 @512, batch 1)
CONFIG_CASES = (("r34_b2_256", "ResNet34", 34, 2, 256), ("r101_b2_320", "ResNet101", 101, 2, 320),
                ("r152_b1_512", "ResNet152", 152, 1, 512))
CONFIG_GRAD_KEYS = ("encoder.conv1.weight", "encoder.layer1.0.conv1.weight", "encoder.layer2.0.conv2.weight",
                    "encoder.layer3.1.conv1.weight", "encoder.layer4.0.downsample.0.weight", "center.block.0.conv.bias",
                    "dec3.block.1.weight", "dec1.block.1.weight", "dec0.conv.weight", "final.weight", "final.bias")


GRAD_HEAD = 16384   # leading elements (flattened, reference layout) kept of each gradient

# both families (raw seed-1234 initialisation, and oracle/unet_oracle.py::conditioned_state_dict): logits stored at every
# LOGIT_STRIDE-th pixel in both directions (3 covers every 2x2 parity class of the transposed convs)
LOGIT_STRIDE = 3


def save_unet_golden(family, rec):
    """one file per configuration (each stays below 1 MB)"""
    for tag, *_ in CONFIG_CASES:
        part = {k: v for k, v in rec.items() if k.endswith("_" + tag) or ("_%s_" % tag) in k}
        np.savez_compressed(os.path.join(GOLDEN_DIR, "unet_%s_%s.npz" % (family, tag)), **part)


def load_unet_golden(family):
    """the fixture of one family as a single dict, keyed like save_unet_golden's input"""
    out = {}
    for path in sorted(glob.glob(os.path.join(GOLDEN_DIR, "unet_%s_*.npz" % family))):
        with np.load(path) as g:
            out.update({k: g[k] for k in g.files})
    return out
