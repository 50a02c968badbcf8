"""Generates tests/golden/tta_loaders.npz from the UNMODIFIED reference (src/loaders.py, imported through
oracle/ref_shim.py with MCB_REFERENCE_ROOT naming the checkout):

* TestTimeAugmentationGenerator.transform on two metadata rows for every flip_ud / flip_lr / rotation combination and
  color_shift_runs in {False, 1, 2}: the spec lists, img_ids and X_tta rows;
* test_time_augmentation_transform on a seeded 10x10 uint8 tile for every spec of the full list (color_shift_runs 2)
  that applies no colour (the colour branch draws from imgaug, which the shim stubs out).

The archive is written with fixed zip timestamps, so regenerating it reproduces the file bit for bit:
    MCB_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_tta
"""
import io
import json
import os
import sys
import warnings
import zipfile
from itertools import product

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "tta_loaders.npz")


def tag(ud, lr, rot, runs):
    return "ud%d_lr%d_rot%d_runs%d" % (ud, lr, rot, int(runs))


def combos():
    return [(ud, lr, rot, runs) for ud, lr, rot in product((True, False), repeat=3) for runs in (False, 1, 2)]


def save_npz(path, arrays):
    """np.savez_compressed with a fixed member timestamp"""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            info.external_attr = 0o644 << 16
            z.writestr(info, buf.getvalue())


def main():
    warnings.filterwarnings("ignore")
    ref_shim.install()
    import src.loaders as lo
    rec = {}
    X = np.array([["tiles/a.png"], ["tiles/b.png"]], dtype=object)
    for ud, lr, rot, runs in combos():
        gen = lo.TestTimeAugmentationGenerator(flip_ud=ud, flip_lr=lr, rotation=rot, color_shift_runs=runs)
        got = gen.transform(X)
        t = tag(ud, lr, rot, runs)
        rec["specs_" + t] = np.array(json.dumps(got["tta_params"]))
        rec["ids_" + t] = np.array(got["img_ids"], np.int64)
        rec["xtta_" + t] = np.array(json.dumps(np.asarray(got["X_tta"].values).reshape(-1).tolist()))
    img = np.random.RandomState(21).randint(0, 256, (10, 10, 3)).astype(np.uint8)
    full = full_spec_list(lo)
    plain = [s for s in full if not (s["color_shift"] and not s["ud_flip"] and not s["lr_flip"])]
    rec["transform_img"] = img
    rec["transform_specs"] = np.array(json.dumps(plain))
    rec["transform_out"] = np.stack([np.asarray(lo.test_time_augmentation_transform(img, s)) for s in plain])
    save_npz(OUT, rec)
    print(OUT, os.path.getsize(OUT), "bytes")


def full_spec_list(lo):
    """the reference's spec list for one image with every option on and two colour runs"""
    gen = lo.TestTimeAugmentationGenerator(flip_ud=True, flip_lr=True, rotation=True, color_shift_runs=2)
    return gen.transform(np.array([["x"]], dtype=object))["tta_params"]


if __name__ == "__main__":
    main()
