"""BASELINE.json config 5's train step -- the ResNet152 U-Net at batch 16 and 512x512 (bench.py --encoder 152 --batch 16
--size 512), the deep-encoder, large-activation case -- unit by unit against float64 and end to end against itself.

At this size every launch has a shape the batch-32 320x320 tests do not reach: the encoder runs at 256/128/64/32/16,
the decoder ends in a 512x512x16 dec0 and classifier, the stem BatchNorm reduces over M = 1 048 576 pixels, and the
launch rules of csrc/conv_gemm.cu pick their tile boxes, N widths, haloed or per-tap paths, persistent tile counts and
weight-gradient splits from these shapes.  ResNet152's 8 layer2 and 36 layer3 blocks give 154 conv + BN parts, and a
longer side-stream and Adam-segment schedule in the captured backward.

  U. every unit of the second step, a graph replay, against float64 (oracle.resnet_step_units, whose docstring lists
     the checks and their bounds, unchanged from the batch-32 test): the stem conv, BN and max-pool, all 154 conv + BN
     parts, the inner and block-input data gradients, c5, every decoder half, dec0 and the final 1x1.  The element-wise
     forward and data-gradient checks take images 0, 5, 10 and 15 (the batch's first and last among them), the
     reductions all 16.  The check count is asserted: 1854;
  A. the captured step equals the same launches run eagerly in program order on one stream, bit for bit over the whole
     arena, the running statistics and the logits, for three distinct batches (test_train_step_scale_gpu.py's A);
  B. every step's weights and Adam moments are exactly Adam of that step's own final gradients over the whole arena,
     and the bf16 operand copy is exactly the new fp32 weights (test_train_step_scale_gpu.py's B).
At most one config-5 plan is alive at a time; what is compared across runs is kept on the host.

Measured on an H100 80GB HBM3 at its 700 W power limit: the file takes 44 s.  U makes 1854 checks in 17 s and peaks
at 25.0 GiB of device memory, A takes 14 s and 18.4 GiB, B 6 s and 19.7 GiB.  Worst |got - ref| / bound in U: the
stored forward outputs, dz and the data gradients 0.984 .. 0.996 (the bf16 rounding of the output itself), BN mean
0.009, invstd 0.011, running statistics 0.004, dbeta / dgamma 0.007, weight gradients 0.356 (dec0), bias and classifier
sums 0.006, max-pool exact.  The largest |mean| / std of a pre-BN channel is 5.23 (encoder.layer1.0.bn1; 4.99 at batch
32 and 320x320), so the one-pass variance loses about 2^-24 chain x 28 of the variance where it lost 2^-24 chain x 26,
and the worst relative invstd error is 2^-18.6 (encoder.layer1.0.downsample.1) against the bound of 2^-12.  The
stem BatchNorm's M = 1 048 576 (819 200 at batch 32 and 320x320) leaves the argument of oracle.resnet_step_units as
it was.

What U does not see: BatchNorm's eps.  eps = 1e-5 moves invstd by eps / (2 var) relative, at most 2^-13.7 here (the
stem BatchNorm), inside the 2^-12 bound; test_elementwise_scale_gpu.py::test_bn_forward pins it."""
import pytest

from oracle.resnet_step_units import check_every_unit
from oracle.step_checks import CONFIG5, N5, S5, check_adam_of_own_gradients, check_captured_equals_serial
from oracle.step_checks import rng_and_peak_memory  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

IMAGES = (0, 5, 10, 15)   # the element-wise checks' images of the 16
PARTS = 154               # conv + BN parts: 50 Bottleneck blocks of 3 convs, 4 downsamples
CHECKS = 1854             # the check-count formula of oracle.resnet_step_units at 154 parts, 100 inner, 50 blocks, 6
#                           decoders


def test_every_unit_against_float64(mcb, cuda):
    count, parts, _ = check_every_unit(CONFIG5, cuda, N5, S5, IMAGES)
    assert (parts, count) == (PARTS, CHECKS)


def test_captured_step_equals_serial_launch_order(mcb, cuda):
    check_captured_equals_serial(CONFIG5, cuda, N5, S5)


def test_fused_adam_is_adam_of_the_steps_own_gradients(mcb, cuda):
    check_adam_of_own_gradients(CONFIG5, cuda, N5, S5)
