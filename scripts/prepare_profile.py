"""Throughput of the target preparation from COCO polygons (mcb200.preparation) on the GPU.

    python scripts/prepare_profile.py [--images 256] [--buildings 10 40] [--erode 0 --dilate 0 --border 0]

Reports, beside the card's name and power limit read in the same run:
  * device images/s of `overlay_batch` on 300 x 300 images of seeded synthetic buildings (density and configuration
    are parameters), CUDA events around warmed-up calls, ending in a synchronise;
  * the same end to end through `overlay_masks` into a temporary directory, and its split into device time
    (`overlay_batch` plus the copies back) and the host's encode / write time that the pool does not hide."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--buildings", type=int, nargs=2, default=(10, 40))
    ap.add_argument("--erode", type=int, default=0)
    ap.add_argument("--dilate", type=int, default=0)
    ap.add_argument("--border", type=int, default=0)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--threads", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prepare_profile.py measures on a CUDA device; none is available")
    import mcb200  # noqa: F401
    from mcb200 import preparation as P
    from oracle import overlay_oracle as O

    rs = np.random.RandomState(0)
    lo, hi = a.buildings
    images = [O.synthetic_image_annotations(rs, 300, 300, rs.randint(lo, hi + 1), i, 1000 * i, a.erode == 0)
              for i in range(a.images)]
    n_polys = sum(len(x["segmentation"]) for im in images for x in im)
    cfg = (None, 100), a.erode, a.dilate, a.border, 14
    print("card:", card())
    print("images %d of 300x300, %d polygons, erode %d dilate %d border %d" % (a.images, n_polys, a.erode, a.dilate,
                                                                             a.border))
    for _ in range(2):
        P.overlay_batch(images, 300, 300, *cfg)
    torch.cuda.synchronize()
    times = []
    for _ in range(a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        P.overlay_batch(images, 300, 300, *cfg)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    dev_s = float(np.median(times))
    print("overlay_batch: %.1f ms per call (median of %d, spread %.1f-%.1f), %.0f images/s"
          % (dev_s * 1e3, a.repeats, min(times) * 1e3, max(times) * 1e3, a.images / dev_s))

    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "data", "train"))
        img_meta = [{"id": i, "file_name": "t%06d.jpg" % i, "height": 300, "width": 300} for i in range(a.images)]
        anns = [x for im in images for x in im]
        with open(os.path.join(tmp, "data", "train", "annotation.json"), "w") as f:
            json.dump({"images": img_meta, "annotations": anns}, f)
        orig = P.overlay_batch
        dev_time = []

        def timed(*args, **kw):
            t = time.perf_counter()
            out = orig(*args, **kw)
            torch.cuda.synchronize()
            dev_time.append(time.perf_counter() - t)
            return out
        P.overlay_batch = timed
        t0 = time.perf_counter()
        P.overlay_masks(os.path.join(tmp, "data"), "train", os.path.join(tmp, "out"), [None, 100], a.erode, a.dilate,
                        False, a.threads, a.border, 14)
        total = time.perf_counter() - t0
        P.overlay_batch = orig
    dev = sum(dev_time)
    print("overlay_masks end to end: %.2f s, %.0f images/s (device batches %.2f s, host json / copies / encode / write "
          "%.2f s, %d host threads)" % (total, a.images / total, dev, total - dev, a.threads))


if __name__ == "__main__":
    main()
