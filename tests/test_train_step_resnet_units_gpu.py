"""Every unit of the ResNet U-Net train step against float64, at the benchmark's size: batch 32 and 320x320, the model
built as bench.py builds it (PyTorchUNetWeighted with bench.unet_config's settings, the reference-like raw init), for
ResNet101 (Bottleneck blocks, bench.py's default encoder) and ResNet34 (BasicBlock).

oracle.resnet_step_units.check_every_unit runs two steps and checks every unit of the second, a graph replay, against
float64; its docstring lists the checks and their bounds.  The element-wise forward and data-gradient checks take
oracle.unit_checks.SAMPLE, four images of the 32, the reductions all 32.

Measured on an H100 80GB HBM3 at its 700 W power limit: ResNet101 (1259 checks) takes 13-20 s and at most 16.7 GiB
of device memory, ResNet34 (463 checks) 3-4 s and 9.6 GiB.  Worst |got - ref| / bound: the stored forward outputs, dz
and the data gradients 0.96 .. 0.996 (the bf16 rounding of the output itself), BN mean 0.011, invstd 0.006, running
statistics 0.005, dbeta / dgamma 0.006, weight gradients 0.30 (dec0), bias and classifier sums 0.005, max-pool exact.
The largest |mean| / std of a pre-BN channel is 4.99 (ResNet101's layer1.0 downsample; ResNet34: 4.02, layer1.0.bn1),
and the worst relative invstd error is 2^-19.5 (ResNet34: 2^-20.1): the one-pass variance is well inside its bound."""
import pytest

from oracle.resnet_step_units import check_every_unit
from oracle.step_checks import RESNET_DEPTH
from oracle.step_checks import rng_and_peak_memory  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

CHECKS = {"ResNet101": 1259, "ResNet34": 463}


@pytest.mark.parametrize("enc", list(RESNET_DEPTH))
def test_every_unit_against_float64(mcb, cuda, enc):
    count, _, _ = check_every_unit(enc, cuda)
    assert count == CHECKS[enc]
