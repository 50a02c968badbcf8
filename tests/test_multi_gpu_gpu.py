"""Two-GPU tests of the data-parallel train step (skipped on a single-GPU box).  One process per GPU over NCCL:
* default (reference DataParallel semantics: per-replica BatchNorm statistics, global-batch loss): the replicas must stay
  bit-identical after several steps on DIFFERENT data -- that only holds if the gradient exchange happened;
* MCB_SYNC_BN=1: BatchNorm over the global batch, so two ranks with half the batch each reproduce ONE process running
  the whole batch (same loss, same updated parameters up to bf16 reduction-order effects)."""
import os

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from oracle import synthetic

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, sync_bn, out):
    import faulthandler
    import torch.distributed as dist
    faulthandler.dump_traceback_later(150, exit=True)   # a hung collective shows its Python stack and fails fast
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), MCB_SYNC_BN=str(int(sync_bn)))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import bench
    import mcb200  # noqa: F401
    from mcb200.models import PyTorchUNetWeighted
    torch.manual_seed(77)
    model = PyTorchUNetWeighted(**bench.unet_config("ResNet34"))
    model._to_device()
    x, t = synthetic.train_batch(4, 64, seed=21, n_rect=6)
    lo, hi = rank * 2, rank * 2 + 2
    X, T = torch.from_numpy(x[lo:hi]).cuda(), torch.from_numpy(t[lo:hi]).cuda()
    losses = [float(model._fit_loop([X, T])["sum"]) for _ in range(3)]
    net = model._net()
    out[rank] = {"losses": losses, "checksum": float(net._p32.double().sum()),
                 "final_w": net.final.weight.detach().float().cpu().numpy().copy(),
                 "bn1_w": net.encoder.bn1.weight.detach().float().cpu().numpy().copy()}
    faulthandler.cancel_dump_traceback_later()
    from mcb200.models import release_captured_graphs
    release_captured_graphs(model)        # graphs that captured NCCL work must go before the communicator does
    faulthandler.dump_traceback_later(60, exit=True)
    dist.destroy_process_group()
    faulthandler.cancel_dump_traceback_later()


def _run_two_ranks(sync_bn):
    mgr = mp.Manager()
    out = mgr.dict()
    port = 29700 + (os.getpid() % 1000) + 50 * int(sync_bn)
    mp.spawn(_worker, args=(2, port, sync_bn, out), nprocs=2, join=True)
    return out[0], out[1]


@pytest.fixture(scope="module")
def two_gpus(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")


@pytest.mark.timeout(600)
def test_replicas_stay_identical_with_per_replica_batchnorm(mcb, two_gpus):
    r0, r1 = _run_two_ranks(sync_bn=False)
    assert r0["losses"] == r1["losses"]                   # the loss is global-batch on every rank
    assert r0["checksum"] == r1["checksum"]               # identical replicas <=> gradients were all-reduced
    assert np.array_equal(r0["final_w"], r1["final_w"]) and np.array_equal(r0["bn1_w"], r1["bn1_w"])
    assert r0["losses"][-1] < r0["losses"][0]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("mode", [2, 1])
def test_sync_bn_reproduces_the_single_process_global_batch(mcb, two_gpus, mode):
    """mode 1: one NCCL all-reduce per BatchNorm; mode 2: the one-shot exchange over NVLink peer memory (csrc/sync.cu)"""
    import bench
    from mcb200.models import PyTorchUNetWeighted
    torch.manual_seed(77)
    model = PyTorchUNetWeighted(**bench.unet_config("ResNet34"))
    model._to_device()
    x, t = synthetic.train_batch(4, 64, seed=21, n_rect=6)
    X, T = torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()
    ref_losses = [float(model._fit_loop([X, T])["sum"]) for _ in range(3)]
    ref_final = model._net().final.weight.detach().float().cpu().numpy()
    ref_bn1 = model._net().encoder.bn1.weight.detach().float().cpu().numpy()
    r0, r1 = _run_two_ranks(sync_bn=mode)
    assert r0["checksum"] == r1["checksum"]
    for a, b in zip(r0["losses"], ref_losses):
        assert abs(a - b) < 2e-3 * abs(b), (r0["losses"], ref_losses)
    assert np.abs(r0["final_w"] - ref_final).max() < 5e-4   # 3 Adam steps of lr 5e-4 move a weight by <= 1.5e-3
    assert np.abs(r0["bn1_w"] - ref_bn1).max() < 5e-4
