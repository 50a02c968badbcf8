"""The ResNet101 U-Net train step at 320x320 at the batch sizes a real training run takes: the reference trains at
batch 20 (neptune.yaml's batch_size_train), and its DataLoader has no drop_last, so every epoch ends in a partial
batch.  13 and 1 stand for such tails.

At these sizes the launch rules of csrc/conv_gemm.cu meet shapes the batch-32 and batch-16 tests do not reach: pixel
boxes and ragged M tails of the forward, data-gradient and weight-gradient GEMMs (pick_tile's row multiple of 16 on the
10x10 maps leaves a partial tile at N = 13 and N = 1), other persistent tile counts and weight-gradient splits,
BatchNorm reductions over pixel counts that are not multiples of 32 (M = 1300 at layer4 for N = 13, 100 for N = 1),
and the loss's pixel normalisation.
  U. every unit of the second step, a graph replay, against float64 (oracle.resnet_step_units, whose docstring lists
     the checks and their bounds, unchanged), at N = 20, 13 and 1.  The element-wise checks take images 0, N/2 and
     N - 1, the reductions all N.  The check count is the module's formula: 1259 at every N;
  A. the captured step equals the same launches run eagerly in program order, bit for bit, at N = 20 and 13
     (oracle.step_checks.check_captured_equals_serial);
  B. every step is exactly whole-arena Adam of its own gradients, at N = 20 and 13, and across a shape switch 32, 13,
     32, 13 through _fit_loop (oracle.step_checks.check_adam_of_own_gradients).  The switch keeps two captured steps
     alive that share one Adam state; each of them is also compared bit for bit with a serial run of the same
     sequence.  With both steps captured, four capture streams (two per step) hold regions of the weight-gradient
     split workspace (wgrad_region_offset in csrc/conv_gemm.cu keeps four).
At most one ResNet101 model is alive at a time; what is compared across runs is kept on the host.

Measured on an H100 80GB HBM3 at its 700 W power limit: the file takes about 100 s.
  U  N = 20: 1259 checks, 17 s, peak 11.4 GiB; N = 13: 1259 checks, 6 s, 8.3 GiB; N = 1: 1259 checks, 4 s, 3.5 GiB.
     Worst |got - ref| / bound at N = 20 / 13 / 1: stored outputs, dz and data gradients 0.980 .. 0.996 at every N
     (the bf16 rounding of the output itself); BN mean 0.012 / 0.009 / 0.008, invstd 0.006 / 0.008 / 0.006, running
     statistics 0.005 / 0.006 / 0.004, dbeta / dgamma 0.006 / 0.004 / 0.005, weight gradients 0.137 / 0.092 / 0.006
     (dec0), bias and classifier sums 0.004 / 0.005 / 0.004, max-pool exact.  Worst relative invstd error 2^-19.5 /
     2^-18.9 / 2^-19.3 against the bound of 2^-12; largest pre-BN |mean| / std 4.99 / 4.98 / 5.04.  No bound changed.
  A  12 s at N = 20 (7.7 GiB) and at N = 13 (5.5 GiB).  B 3 s each (9.0 and 6.7 GiB).  The shape switch 20 s, 16.8 GiB."""
import pytest

from oracle.resnet_step_units import check_every_unit
from oracle.step_checks import N, check_adam_of_own_gradients, check_captured_equals_serial
from oracle.step_checks import rng_and_peak_memory  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

ENCODER = "ResNet101"
PARTS = 103               # conv + BN parts: 33 Bottleneck blocks of 3 convs, 4 downsamples
CHECKS = 1259             # the check-count formula of oracle.resnet_step_units at 103 parts, 66 inner, 33 blocks, 6
#                           decoders: the same at every batch size
TAIL = 13                 # a partial last batch


def images(n):
    """the element-wise checks' images: the first, the middle and the last"""
    return tuple(sorted({0, n // 2, n - 1}))


@pytest.mark.parametrize("n", [20, TAIL, 1])
def test_every_unit_against_float64(mcb, cuda, n):
    count, parts, _ = check_every_unit(ENCODER, cuda, n, images=images(n))
    assert (parts, count) == (PARTS, CHECKS)


@pytest.mark.parametrize("n", [20, TAIL])
def test_captured_step_equals_serial_launch_order(mcb, cuda, n):
    check_captured_equals_serial(ENCODER, cuda, n)


@pytest.mark.parametrize("n", [20, TAIL])
def test_fused_adam_is_adam_of_the_steps_own_gradients(mcb, cuda, n):
    check_adam_of_own_gradients(ENCODER, cuda, n)


def test_shape_switch_full_batch_and_tail_share_one_adam_state(mcb, cuda):
    check_adam_of_own_gradients(ENCODER, cuda, sizes=(N, TAIL, N, TAIL))
