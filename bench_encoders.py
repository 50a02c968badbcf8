"""Train-step throughput of every encoder-registry net the H100 path builds (src/models.py:22-47), next to stock
PyTorch + cuDNN on the same net:

    python bench_encoders.py [--nets AlbuNet,ResNet34,ResNet101,ResNet152] [--batch 32] [--size 320]
                             [--steps 20] [--warmup 5] [--no-baseline]

Per net and arm one JSON line: ms per train step (CUDA events around `steps` back-to-back steps on device-resident
synthetic batches), tiles/s, and achieved TFLOP/s from the launch plan's algorithmic FLOPs (forward + backward of every
conv, counted per tile).  The mcb200 arm is PyTorchUNetWeighted._fit_loop (fused CUDA-graph step with in-graph Adam);
the baseline arm is baseline/torch_cudnn_unet.py (bf16 autocast, channels_last, fused torch Adam).  Writes nothing."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def plan_flops_per_tile(net, batch, size):
    pl = net.plan(batch, size, size, True)
    return (sum(o.flops for o in pl.fwd_ops) + sum(o.flops for layer in pl.bwd_layers for o in layer)) / batch


def time_steps(step, warmup, steps):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        loss = step()
    b.record()
    torch.cuda.synchronize()
    assert bool(torch.isfinite(loss).all())
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nets", default="AlbuNet,ResNet34,ResNet101,ResNet152")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=320)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-baseline", action="store_true")
    args = ap.parse_args()
    import bench
    import mcb200  # noqa: F401  (loads libmcb200.so)
    from bench_data import train_batch
    from mcb200.models import PyTorchUNetWeighted
    dev = torch.device("cuda:0")
    x, t = train_batch(args.batch, args.size, seed=1234)
    X, T = torch.from_numpy(x).to(dev), torch.from_numpy(t).to(dev)
    for enc in args.nets.split(","):
        torch.manual_seed(1234)
        model = PyTorchUNetWeighted(**bench.unet_config(enc))
        model._to_device()
        fpt = plan_flops_per_tile(model._net(), args.batch, args.size)
        arms = [("mcb200", lambda: model._fit_loop([X, T])["sum"])]
        if not args.no_baseline:
            from baseline.torch_cudnn_unet import TrainStep
            base = TrainStep.for_encoder(enc, dev)
            arms.append(("torch_cudnn", lambda: base.step(X, T)))
        for arm, step in arms:
            ms = time_steps(step, args.warmup, args.steps)
            print(json.dumps({"net": enc, "arm": arm, "batch": args.batch, "size": args.size, "steps": args.steps,
                              "ms_per_step": round(ms, 3), "tiles_per_s": round(args.batch * 1e3 / ms, 1),
                              "gflop_per_tile": round(fpt / 1e9, 2),
                              "tflops": round(fpt * args.batch / (ms * 1e-3) / 1e12, 1),
                              "gpu": torch.cuda.get_device_name(dev)}), flush=True)
        del model, arms
        if not args.no_baseline:
            del base
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
