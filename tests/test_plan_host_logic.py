"""CPU tests of the host-side launch planning (mcb200.engine.Plan): the plan is pure Python over preallocated tensors, so
its structure can be checked without a GPU -- launch inventory, algorithmic FLOPs (SURVEY's 205.71 GFLOP/tile for
UNetResNet-101 @320x320), store/accumulate ordering of the gradient buffers, arena segments for the per-segment
optimizer / all-reduce, and which launches are leaves that may run on the side stream."""
import collections

import pytest
import torch
from torch import nn


@pytest.fixture(scope="module")
def net101(mcb):
    from mcb200.unet_models import UNetResNet
    torch.manual_seed(0)
    return UNetResNet(101, 2, 32, 0.0, False, True)


@pytest.fixture(scope="module")
def plan101(net101):
    return net101.plan(1, 320, 320, True)


def _bwd_ops(plan):
    return [o for layer in plan.bwd_layers for o in layer]


def test_algorithmic_flops_match_the_survey_figure(plan101):
    import bench
    fl = sum(o.flops for o in plan101.fwd_ops) + sum(o.flops for o in _bwd_ops(plan101))
    assert abs(fl - bench.FLOP_PER_TILE[(101, 320)]) < 1e6
    assert abs(fl / 1e9 - 205.71) < 0.01


def test_launch_inventory_resnet101(net101, plan101):
    n_bn = sum(isinstance(m, nn.BatchNorm2d) for m in net101.modules())
    n_conv = sum(isinstance(m, nn.Conv2d) for m in net101.modules())
    n_convt = sum(isinstance(m, nn.ConvTranspose2d) for m in net101.modules())
    assert (n_bn, n_conv, n_convt) == (104, 112, 6)
    fwd = collections.Counter(o.kind for o in plan101.fwd_ops)
    bwd = collections.Counter(o.kind for o in _bwd_ops(plan101))
    # forward: every conv but the 1x1 classifier is a tensor-core GEMM launch; the four downsample BatchNorms ride in
    # the residual BN-apply of their block
    assert fwd["conv_fwd"] == n_conv - 1 and fwd["convt_fwd"] == n_convt and fwd["final_conv"] == 1
    assert fwd["bn_apply"] == n_bn - 4
    # backward: one weight-gradient GEMM per conv (+1 per fused skip concat: dec5..dec2), one dz pass per BatchNorm
    assert bwd["conv_wgrad"] == (n_conv - 1) + 4 and bwd["convt_wgrad"] == n_convt
    assert bwd["bn_bwd_apply"] == n_bn
    # BatchNorm-backward reductions stay separate launches only where dy has several producers: stem, 33 block outputs,
    # 4 downsample branches; the 66 inner units get theirs from the data-gradient epilogue
    assert bwd["bn_bwd_reduce"] == 1 + 33 + 4
    # decoder bias gradients are summed in the dgrad epilogues (6 deconv outputs through bias_sum, 6 conv outputs through
    # convt_dgrad); only dec0's remains a launch
    assert bwd["channel_sum"] == 1 and len(plan101.bias_fused) == 6
    assert bwd["conv_dgrad"] == 114 and bwd["convt_dgrad"] == 6


def test_side_stream_candidates_are_leaves(plan101):
    """launches moved to the side stream must only write weight gradients: they are weight-gradient GEMMs"""
    side = [o for o in _bwd_ops(plan101) if o.side]
    # all but the stem's (post-processed in order by stem_unpack_wgrad) and dec0's (kept on the main stream)
    assert len(side) == 115 + 6 - 2
    assert all(o.kind in ("conv_wgrad", "convt_wgrad") and o.flops > 0 for o in side)


def test_backward_layers_run_in_reverse_forward_order(plan101):
    tags = plan101.bwd_tags
    assert tags[0] == "decoder" and tags[-1] == "stem"
    order = {"decoder": 0, "layer4": 1, "layer3": 2, "layer2": 3, "layer1": 4, "stem": 5}
    ranks = [order[t] for t in tags]
    assert ranks == sorted(ranks)
    assert collections.Counter(tags)["layer3"] == 23 and collections.Counter(tags)["layer4"] == 3


def test_arena_segments_partition_parameters_and_layers(net101, plan101):
    segs = plan101.bwd_segments()
    total = net101._p32.numel()
    assert total >= sum(p.numel() for _, p, _ in net101._arena_params())   # (slots may be padded for alignment)
    # layers: contiguous, complete
    assert segs[0][0] == 0 and segs[-1][1] == len(plan101.bwd_layers)
    assert all(a[1] == b[0] for a, b in zip(segs, segs[1:]))
    # arena ranges: the segment that finishes first owns the top of the arena (decoder), ranges tile [0, total)
    assert segs[0][3] == total and segs[-1][2] == 0
    assert all(a[2] == b[3] for a, b in zip(segs, segs[1:]))
    # every parameter lies entirely inside one segment
    bounds = sorted({s[2] for s in segs} | {total})
    for _, p, _ in net101._arena_params():
        slot = net101._slots[id(p)]
        lo, hi = slot.off, slot.off + p.numel()
        assert any(b0 <= lo and hi <= b1 for b0, b1 in zip(bounds, bounds[1:])), (lo, hi)


def test_gradient_buffers_first_store_then_accumulate(mcb):
    """a small ResNet-34 plan: replay the builders' store/accumulate decisions -- every activation gradient is STORED by
    its first writer in execution order and accumulated by the later ones (no memset of activation gradients exists)"""
    from mcb200.unet_models import UNetResNet
    torch.manual_seed(0)
    net = UNetResNet(34, 2, 32, 0.0, False, True)
    plan = net.plan(1, 64, 64, True)
    # every activation that received a gradient was marked written exactly through gmode()
    assert set(plan.grad.keys()) >= plan.written or plan.written <= set(plan.grad.keys()) | set(map(id, [plan.x_in]))
    kinds = collections.Counter(o.kind for o in _bwd_ops(plan))
    n_bn = sum(isinstance(m, nn.BatchNorm2d) for m in net.modules())
    assert kinds["bn_bwd_apply"] == n_bn
    # BasicBlocks: one inner unit per block gets its reductions from the dgrad epilogue
    n_blocks = sum(len(l) for l in (net.encoder.layer1, net.encoder.layer2, net.encoder.layer3, net.encoder.layer4))
    assert kinds["bn_bwd_reduce"] == n_bn - n_blocks


def test_four_backward_segments_for_the_overlapped_all_reduce(net101, plan101):
    """decoder | layer4 | layer3 | layer2 + layer1 + stem: layer3's 23 blocks (the largest parameter group after the
    decoder) reduce while the shallow layers still run"""
    segs = plan101.bwd_segments()
    assert len(segs) == 4
    tags = plan101.bwd_tags
    assert set(tags[segs[0][0]:segs[0][1]]) == {"decoder"} and set(tags[segs[1][0]:segs[1][1]]) == {"layer4"}
    assert set(tags[segs[2][0]:segs[2][1]]) == {"layer3"} and set(tags[segs[3][0]:segs[3][1]]) == {"layer2", "layer1", "stem"}
    sizes = [s[3] - s[2] for s in segs]
    assert sizes[2] > sizes[3] and sizes[0] > sizes[3]      # the exposed last segment is the smallest
