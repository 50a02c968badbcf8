#!/usr/bin/env python
"""augment_profile.py — what the device-side training augmentation costs.

  python scripts/augment_profile.py [--batches 200] [--steps 30] [--out FILE]

Records, in one run on one card:
  chain_ms       device time (CUDA events around the chain, queued behind a device-side wait so that host launch
                 overhead is not counted; median over --batches batches after warm-up) of the whole train-batch chain
                 for batch 32 of 300x300 tiles: augment (csrc/augment.cu) + [Pillow resize] + normalise + target, for
                 the `resize` mode (fast_seq, resize to 256x256) and the `crop_and_pad` mode (crop_seq to 256x256), with
                 distances and sizes; host_ms is the host time to draw the parameters and queue that chain
  fit_ms_step    PyTorchUNetWeighted._fit_loop wall time per step (UNetResNet-101, batch 32, 256x256), median over
                 --steps steps, fed (a) by mcb200.loaders.DeviceBatches from pinned host batches (copy + augment chain +
                 step) and (b) by pre-staged device batches; the two feeds alternate step by step
  card, power_limit_w   read in the same run
One JSON line on stdout (and in --out).  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def host_batch(n, seed, pinned=True):
    import numpy as np
    import torch
    rs = np.random.RandomState(seed)
    t = [torch.from_numpy(rs.randint(0, 256, (n, 300, 300, 3)).astype(np.uint8)),
         torch.from_numpy((rs.rand(n, 300, 300) > 0.7).astype(np.uint8)),
         torch.from_numpy(rs.randint(0, 900, (n, 300, 300)).astype(np.int16)),
         torch.from_numpy(rs.randint(1, 40, (n, 300, 300)).astype(np.int16))]
    return [x.pin_memory() for x in t] if pinned else t


SLEEP_CYCLES = 20_000_000   # ~10 ms at the H100's clocks: longer than the host takes to queue one chain


def chain_ms(batches, warmup=20):
    import time
    import numpy as np
    import torch
    from mcb200 import augmentation as A
    dev = [x.cuda() for x in host_batch(32, 0)]
    rng = np.random.default_rng(0)
    res = {}
    for mode, seq, kw in (("resize", A.fast_seq, dict(resize=(256, 256))),
                          ("crop_and_pad", A.crop_seq((256, 256)), dict(crop_size=(256, 256)))):
        times, host = [], []
        for i in range(warmup + batches):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(SLEEP_CYCLES)      # the device waits here while the host queues the whole chain
            a.record()
            t0 = time.perf_counter()
            A.batch_chain(*dev, params=seq.draw(rng, 32, 300, 300), **kw)
            t1 = time.perf_counter()
            b.record()
            b.synchronize()
            if i >= warmup:
                times.append(a.elapsed_time(b))
                host.append((t1 - t0) * 1e3)
        res[mode] = {"device_ms": round(float(np.median(times)), 4), "host_ms": round(float(np.median(host)), 4)}
    return res


def fit_ms(steps, warmup=5):
    import time
    import numpy as np
    import torch
    import bench
    from mcb200 import augmentation as A
    from mcb200.loaders import DeviceBatches
    from mcb200.models import PyTorchUNetWeighted
    torch.manual_seed(0)
    model = PyTorchUNetWeighted(**bench.unet_config("ResNet101"))
    hosts = [host_batch(32, s) for s in range(2)]
    flow = DeviceBatches(hosts * (warmup + steps), A.fast_seq, np.random.default_rng(1), (256, 256))
    staged = [A.batch_chain(*[x.cuda() for x in h], params=A.fast_seq.draw(np.random.default_rng(s), 32, 300, 300),
                            resize=(256, 256)) for s, h in enumerate(hosts)]
    t_loader, t_staged = [], []
    it = iter(flow)
    for i in range(warmup + steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model._fit_loop(next(it))
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        model._fit_loop(staged[i % 2])
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        if i >= warmup:
            t_loader.append((t1 - t0) * 1e3)
            t_staged.append((t2 - t1) * 1e3)
    return {"loader_pinned_host": round(float(np.median(t_loader)), 3),
            "pre_staged_device": round(float(np.median(t_staged)), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import mcb200  # noqa: F401
    res = {"card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
           "chain_ms_batch32_300px": chain_ms(args.batches), "fit_ms_step_r101_b32_256": fit_ms(args.steps)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
