"""Time the second-level scoring model's prediction for one inference batch: 20 tiles of 300 x 300 with
CATEGORY_LAYERS [1, 19], the 4 136 instance rows of tests/golden/scoring_features.npz in their 400 (image, layer)
frames, through a RandomForest of the configured shape (500 trees, max_depth 20, min_samples_split / min_samples_leaf
100, max_leaf_nodes 500, squared_error, max_features=1.0), trained on the golden's training rows.

Three ways, each ending with the scores on the host:
  * device: mcb200.models.ScoringRandomForest.transform (one upload, one mcb_forest_predict, one readback; the forest
    is already on the device);
  * host, one call: RandomForestRegressor.predict at n_jobs=1 on all rows at once;
  * host, per (image, layer): the reference's loop of one predict per non-empty frame (src/models.py:267-278), n_jobs=1.
The spread is over --repeats runs after one warm-up.  Card name and power limit are read in the same run.

    python scripts/scoring_model_profile.py [--repeats 10] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
FEATURES = ('threshold', 'area', 'mean_prob', 'max_prob', 'bbox_ar', 'bbox_area', 'bbox_fill', 'min_dist_to_border',
            'max_dist_to_border', 'contour_length')


def spread(ts):
    return {"median": float(np.median(ts)), "min": float(np.min(ts)), "max": float(np.max(ts))}


def timed(fn, repeats):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return ts


def main():
    import pandas as pd
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scoring_model_profile needs a CUDA device")
    import mcb200  # noqa: F401
    from mcb200 import models

    g = np.load(os.path.join(ROOT, "tests", "golden", "scoring_features.npz"))
    x_train = np.stack([g["ann_" + c] for c in FEATURES], 1).astype(np.float64)
    y = g["ann_iou"]
    keep = ~np.isnan(y)
    model = models.ScoringRandomForest(0.7, "iou", dict(n_estimators=500, criterion="squared_error", max_depth=20,
                                                        min_samples_split=100, min_samples_leaf=100,
                                                        max_features=1.0, max_leaf_nodes=500, n_jobs=1,
                                                        random_state=0))
    model.estimator.fit(x_train[keep], y[keep])
    model.feature_names = list(FEATURES)
    x = np.stack([g["none_" + c] for c in FEATURES], 1).astype(np.float64)
    counts = g["none_counts"].reshape(20, -1)
    features, at = [], 0
    for image in counts:
        layers = []
        for k in image:
            layers.append(pd.DataFrame(x[at:at + k], columns=list(FEATURES)))
            at += k
        features.append(layers)

    est = model.estimator
    res = {"rows": int(x.shape[0]), "frames": int(counts.size), "trees": len(est.estimators_)}
    device = timed(lambda: model.transform(features), a.repeats)
    one_call = timed(lambda: est.predict(x), a.repeats)
    per_frame = timed(lambda: [est.predict(l[model.feature_names]) for im in features for l in im if len(l)],
                      a.repeats)
    res["device_transform_s"] = spread(device)
    res["host_predict_one_call_s"] = spread(one_call)
    res["host_predict_per_frame_s"] = spread(per_frame)
    got = np.array([v for im in model.transform(features)["scores"] for l in im for v in l])
    res["device_equals_host"] = bool(np.array_equal(got, est.predict(x)))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    res["gpu"] = q.stdout.strip() or torch.cuda.get_device_name(0)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
