#!/usr/bin/env python
"""decode_profile.py — what decoding the JPEG tiles costs, on the device and on the host.

  python scripts/decode_profile.py [--reps 100] [--out FILE]

Records, in one run on one card, for seeded 300x300 JPEG tiles at quality 75 and 95, 4:2:0 and 4:4:4 sampling, and
flat 4:2:0 tiles (quality "flat"):
  device_ms   device time of one batch of 20 and of 64 tiles through the stages of csrc/jpeg.cu, each stage
              separately (parallel entropy decode, IDCT, upsample + colour) and all three, and the one-thread-per-
              segment entropy decode (`entropy_serial`) beside the parallel one (`entropy_speedup`); CUDA events around
              launches queued behind a device-side wait (host launch time kept out), median over --reps after warm-up;
              `speculation` = the parallel decode's counters (guesses held, corrected, longest correction run, exact
              re-decodes of a segment's end)
  worker_ms   host time per file of the device path's worker share (mcb200.jpeg.read_jpeg: read, parse, unstuff, Huffman
              tables), median
  pillow_ms   host time per file of np.array(Image.open(f).convert('RGB')), the loaders' decode, median
  loader_ms_per_batch   wall time per batch to deliver uint8 (N, 300, 300, 3) device batches from files on disk with 4
              DataLoader workers, over 10 batches after 2 of warm-up: `pillow` = Pillow decode in the workers + pinned
              copy (the loaders' path), `device` = read_jpeg in the workers + decode_jpeg_batch; no network runs
              beside it, so the device path's kernel time is not hidden behind anything and neither path is slowed by
              one
  card, power_limit_w   read in the same run
One JSON line on stdout (and in --out).  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SLEEP_CYCLES = 20_000_000   # ~10 ms at the H100's clocks: longer than the host takes to queue the launches


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def _tiles(n, quality, sampling):
    from oracle import jpeg_oracle as O
    if quality is None:                      # flat tiles: every block "DC diff 0 + EOB" after the first
        return [O.encode_pil(np.full((300, 300, 3), 40 + 3 * i, np.uint8), 75, sampling) for i in range(n)]
    return [O.encode_pil(O.content(300, 300, seed=1000 + i), quality, sampling) for i in range(n)]


def device_ms(blobs, reps):
    import torch
    from mcb200 import _lib as L
    from mcb200 import jpeg as J
    recs = [J.load(b) for b in blobs]
    out, _, planes, st = J.decode_records(recs)             # also warms the module up
    assert not st.any()
    pk = J.pack_batch(recs)
    dev = out.device
    batch = J.DeviceBatch(pk, dev)
    tables = torch.from_numpy(J.ycc_tables()).to(dev)
    n, h, w, nb = len(recs), pk["height"], pk["width"], pk["n_blocks"]
    stages = {
        "entropy": batch.entropy_decode,
        "idct": lambda: L.fcall("mcb_jpeg_idct", batch.coef.data_ptr(), batch.qt.data_ptr(), batch.images.data_ptr(),
                                n, nb, planes.data_ptr()),
        "upsample_rgb": lambda: L.fcall("mcb_jpeg_upsample_rgb", planes.data_ptr(), batch.images.data_ptr(),
                                        tables.data_ptr(), n, h, w, out.data_ptr()),
    }
    stages["all"] = lambda: [f() for k, f in list(stages.items())[:3]]
    stages["entropy_serial"] = batch.entropy_decode_serial
    res = {}
    for name, fn in stages.items():
        times = []
        for i in range(10 + reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(SLEEP_CYCLES)
            a.record()
            fn()
            b.record()
            b.synchronize()
            if i >= 10:
                times.append(a.elapsed_time(b))
        res[name] = round(float(np.median(times)), 4)
    assert not batch.status.cpu().numpy().any()
    batch.entropy_decode()
    res["speculation"] = [int(x) for x in batch.counters()]
    res["entropy_speedup"] = round(res["entropy_serial"] / res["entropy"], 2)
    return res


def host_ms(blobs, reps):
    from PIL import Image
    from mcb200 import jpeg as J
    d = tempfile.mkdtemp()
    paths = []
    for i, b in enumerate(blobs):
        p = os.path.join(d, "%d.jpg" % i)
        with open(p, "wb") as f:
            f.write(b)
        paths.append(p)
    worker, pillow = [], []
    for r in range(reps):
        p = paths[r % len(paths)]
        t0 = time.perf_counter()
        J.read_jpeg(p)
        t1 = time.perf_counter()
        np.array(Image.open(p).convert("RGB"))
        t2 = time.perf_counter()
        worker.append((t1 - t0) * 1e3)
        pillow.append((t2 - t1) * 1e3)
    return round(float(np.median(worker)), 4), round(float(np.median(pillow)), 4)


class _BatchFiles:
    """one item per batch of paths: the stacked Pillow decodes, or the list of parsed JpegRecords"""

    def __init__(self, batches, device):
        self.batches, self.device = batches, device

    def __len__(self):
        return len(self.batches)

    def __getitem__(self, i):
        from PIL import Image
        from mcb200 import jpeg as J
        if self.device:
            return [J.read_jpeg(p) for p in self.batches[i]]
        return np.stack([np.array(Image.open(p).convert("RGB")) for p in self.batches[i]])


def loader_ms(blobs, n, batches=10, warmup=2):
    import torch
    from mcb200 import jpeg as J
    d = tempfile.mkdtemp()
    paths = []
    for i in range((batches + warmup) * n):
        p = os.path.join(d, "%d.jpg" % i)
        with open(p, "wb") as f:
            f.write(blobs[i % len(blobs)])
        paths.append(p)
    groups = [paths[i * n:(i + 1) * n] for i in range(batches + warmup)]
    res = {}
    for name, device in (("pillow", False), ("device", True)):
        dl = torch.utils.data.DataLoader(_BatchFiles(groups, device), batch_size=None, num_workers=4,
                                         collate_fn=lambda x: x, prefetch_factor=2)
        for i, item in enumerate(dl):
            if i == warmup:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
            if device:
                J.decode_jpeg_batch(item)
            else:
                torch.from_numpy(item).pin_memory().to("cuda", non_blocking=True)
        torch.cuda.synchronize()
        res[name] = round((time.perf_counter() - t0) * 1e3 / batches, 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import mcb200  # noqa: F401
    if not torch.cuda.is_available():
        raise SystemExit("decode_profile.py needs a CUDA device")
    res = {"card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "tile": "300x300", "cases": []}
    for quality, sampling in ((75, "420"), (75, "444"), (95, "420"), (95, "444"), (None, "420")):
        blobs = _tiles(64, quality, sampling)
        worker, pillow = host_ms(blobs, args.reps)
        case = {"quality": quality or "flat", "sampling": sampling,
                "bytes_per_file": int(np.mean([len(b) for b in blobs])),
                "worker_ms_per_file": worker, "pillow_ms_per_file": pillow}
        for n in (20, 64):
            case["device_ms_batch%d" % n] = device_ms(blobs[:n], args.reps)
            case["loader_ms_per_batch%d" % n] = loader_ms(blobs, n)
        res["cases"].append(case)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
