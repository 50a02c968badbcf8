"""Train-step throughput of every encoder-registry net the H100 path builds (src/models.py:22-47), next to stock
PyTorch + cuDNN on the same net:

    python bench_encoders.py [--nets AlbuNet,ResNet34,ResNet101,ResNet152,VGG11,VGG16] [--batch 32] [--size 320]
                             [--steps 20] [--warmup 5] [--no-baseline]

Per net and arm one JSON line: ms per train step (CUDA events around `steps` back-to-back steps on device-resident
synthetic batches), tiles/s, and achieved TFLOP/s from the launch plan's algorithmic FLOPs (forward + backward of every
conv, counted per tile).  The mcb200 arm is PyTorchUNetWeighted._fit_loop (fused CUDA-graph step with in-graph Adam);
VGG11 and VGG16 are not in mcb200's registry yet, so their arm builds UNet11 / UNetVGG16 from mcb200.unet_models and
times FusedTrainStep.step itself (the step _fit_loop runs, with the configured weighted loss and Adam settings, without
_fit_loop's per-call host bookkeeping: optimizer param-group lookup, the step cache and the device check).  The baseline arm is
baseline/torch_cudnn_unet.py (bf16 autocast, channels_last, fused torch Adam).  Writes nothing."""
import argparse
import functools
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def plan_flops_per_tile(net, batch, size):
    pl = net.plan(batch, size, size, True)
    return (sum(o.flops for o in pl.fwd_ops) + sum(o.flops for layer in pl.bwd_layers for o in layer)) / batch


def vgg_step_settings(enc):
    """-> (FusedTrainStep loss config, lr, weight decay) of bench.unet_config(enc), as PyTorchUNetWeighted derives them
    (src/models.py:149-161)"""
    import bench
    from mcb200.models import _size_c
    a = bench.unet_config(enc)["architecture_config"]
    wce, lw, dice = a["weighted_cross_entropy"], a["loss_weights"], a["dice"]
    cfg = dict(w0=float(wce["w0"]), sigma=float(wce["sigma"]), size_c=_size_c(wce["imsize"]),
               dice_weight=float(lw["dice_mask"]), ce_weight=float(lw["bce_mask"]), dice_smooth=float(dice["smooth"]))
    lr = a["optimizer_params"]["lr"]
    wd = a["regularizer_params"]["weight_decay_conv2d"] if a["regularizer_params"]["regularize"] else 0.0
    return cfg, lr, wd


def vgg_net(enc):
    """UNet11 / UNetVGG16 as the registry entry builds them (src/models.py:22-28)"""
    from mcb200.unet_models import UNet11, UNetVGG16
    return UNet11(num_classes=2) if enc == "VGG11" else UNetVGG16(num_classes=2, dropout_2d=0.0, is_deconv=True)


def vgg_fused_step(enc, x_shape, t_shape, dev):
    """-> (net, step()) for VGG11 / VGG16: the fused train step PyTorchUNetWeighted would run for the registry entry
    (src/models.py:22-28, 149-161) with bench.unet_config's loss and optimizer settings"""
    from mcb200.models import FusedTrainStep
    cfg, lr, wd = vgg_step_settings(enc)
    net = vgg_net(enc).to(dev)
    fused = FusedTrainStep(net, x_shape, t_shape, 0, cfg)
    return net, lambda X, T: fused.step(X, T, lr=lr, weight_decay=wd)


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
        if enc in ("VGG11", "VGG16"):
            model, vgg_step = vgg_fused_step(enc, tuple(X.shape), tuple(T.shape), dev)
            fpt = plan_flops_per_tile(model, args.batch, args.size)
            arms = [("mcb200", functools.partial(vgg_step, X, T))]
            del vgg_step            # the arm holds the captured step: it goes with `arms` below
        else:
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
        del model, arms, step
        if not args.no_baseline:
            del base
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
