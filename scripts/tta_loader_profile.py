#!/usr/bin/env python
"""tta_loader_profile.py — what the TTA inference loaders' device chain costs.

  python scripts/tta_loader_profile.py [--batches 300] [--out FILE]

Records, in one run on one card:
  chain_ms     device time (CUDA events around the chain, queued behind a device-side wait so that host launch overhead
               is not counted; median over --batches batches after warm-up) of one batch of 20 variant rows of 300x300
               tiles (rows 0-19 of the unet_tta spec list: two distinct tiles) through mcb200.loaders.tta_variant_batch:
               variant rows (csrc/instances.cu, geometry + colour) + [Pillow resize to 256x256] + pad + normalise, for
               the `resize` and the `crop_and_pad` (pad 10 -> 320x320) modes, with color_shift_runs 2 and without;
               host_ms is the host time to draw the colours and queue that chain
  variants_kernel_ms   device time of the variant-row kernel alone on the same batch, and the bytes it moves
  decode_ms    host time to decode one 300x300 PNG tile (PIL, the DataLoader workers' share), median
  card, power_limit_w   read in the same run
One JSON line on stdout (and in --out).  Needs a CUDA device."""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

SLEEP_CYCLES = 20_000_000   # ~10 ms at the H100's clocks: longer than the host takes to queue one chain
ROWS = 20


def _timed(fn, batches, warmup=20):
    import numpy as np
    import torch
    times, host = [], []
    for i in range(warmup + batches):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(SLEEP_CYCLES)      # the device waits here while the host queues the whole chain
        a.record()
        t0 = time.perf_counter()
        fn()
        t1 = time.perf_counter()
        b.record()
        b.synchronize()
        if i >= warmup:
            times.append(a.elapsed_time(b))
            host.append((t1 - t0) * 1e3)
    return round(float(np.median(times)), 4), round(float(np.median(host)), 4)


def chain_ms(batches):
    import numpy as np
    import torch
    from mcb200 import _lib as L
    from mcb200 import loaders as lo
    tiles = torch.from_numpy(np.random.RandomState(0).randint(0, 256, (2, 300, 300, 3)).astype(np.uint8)).cuda()
    rng = np.random.default_rng(0)
    res = {}
    for runs in (False, 2):
        specs = lo.tta_specs(color_shift_runs=runs)
        params = (specs * 2)[:ROWS]
        src = np.array([0] * len(specs) + [1] * len(specs))[:ROWS]
        colour = np.array([lo.applies_colour(s) for s in params])
        geo = lo.variant_codes(params)

        def codes():
            branch, value = np.zeros(ROWS, np.int32), np.zeros(ROWS, np.int32)
            branch[colour], value[colour] = lo.draw_colour(rng, int(colour.sum()))
            return geo | (branch << 4) | (value << 8)

        for mode, kw in (("resize", dict(resize=(256, 256))), ("crop_and_pad", dict(pad=(10, 10)))):
            dev, host = _timed(lambda: lo.tta_variant_batch(tiles, src, codes(), **kw), batches)
            res["%s_colour%d" % (mode, bool(runs))] = {"device_ms": dev, "host_ms": host}
        out = torch.empty((ROWS, 300, 300, 3), dtype=torch.uint8, device="cuda")
        src_d = torch.from_numpy(src.astype(np.int32)).cuda()
        codes_d = torch.from_numpy(codes()).cuda()
        dev, _ = _timed(lambda: L.fcall("mcb_tta_variants_u8", tiles.data_ptr(), out.data_ptr(), src_d.data_ptr(),
                                        codes_d.data_ptr(), ROWS, 300, 300), batches)
        res["variants_kernel_colour%d" % bool(runs)] = {"device_ms": dev, "bytes": 2 * ROWS * 300 * 300 * 3}
    return res


def decode_ms(n=50):
    import numpy as np
    from PIL import Image
    from mcb200.loaders import SegmentationFiles
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "tile.png")
        Image.fromarray(np.random.RandomState(1).randint(0, 256, (300, 300, 3)).astype(np.uint8)).save(p)
        ds = SegmentationFiles([p])
        times = []
        for _ in range(n):
            t0 = time.perf_counter()
            ds[0]
            times.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(times)), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import mcb200  # noqa: F401
    from augment_profile import power_limit_w
    res = {"card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
           "chain_ms_batch20_300px": chain_ms(args.batches), "decode_ms_png_300px": decode_ms()}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
