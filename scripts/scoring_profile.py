"""Time the second-level scoring features of one inference batch: mcb200.postprocessing.FeatureExtractor on the device
(20 images of 300 x 300, CATEGORY_LAYERS [1, 19] = 20 layers, label maps and float64 probabilities already on the
device, as the batched chain leaves them) against the host get_features_for_image on the same inputs, with
annotations (the scoring_model train pipeline) and without (the inference pipelines).  The host side is
oracle/scoring_oracle.py, the reference's numpy code restated line for line (pycocotools' IoU through the decoded
stand-in), so its time stands for the reference's order of magnitude, not an exact reference timing.  Each device run
ends in the feature tables on the host (the call returns DataFrames), so a host clock around it measures what a
user waits for; the spread is over --repeats runs after one warm-up.

    python scripts/scoring_profile.py [--repeats 10] [--cpu-images 2] [--out result.json]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--cpu-images", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scoring_profile needs a CUDA device")
    import mcb200  # noqa: F401
    from mcb200 import postprocessing as G
    from oracle import scoring_oracle as S

    G.CATEGORY_LAYERS = list(S.SCORING_LAYERS)     # the scoring workflow's configuration; the reference is absent here
    probs, labels, annotations = S.scoring_case()
    lab, pr = torch.from_numpy(labels).cuda(), torch.from_numpy(probs).cuda()
    fe = G.FeatureExtractor()
    res = {"batch": int(labels.shape[0]), "layers": int(labels.shape[1]), "size": int(labels.shape[2]),
           "instances": int(sum(int(l.max()) for im in labels for l in im))}
    for name, ann in (("train", annotations), ("inference", None)):
        fe.transform(lab, pr, ann)
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            fe.transform(lab, pr, ann)
            ts.append(time.perf_counter() - t0)
        k = a.cpu_images
        t0 = time.perf_counter()
        S.feature_extractor(list(labels[:k]), list(probs[:k]), None if ann is None else ann[:k])
        host = (time.perf_counter() - t0) / k * labels.shape[0]
        res[name] = {"device_s_per_batch": {"median": float(np.median(ts)), "min": float(np.min(ts)),
                                            "max": float(np.max(ts))},
                     "host_s_per_batch_extrapolated_from_%d_images" % k: host}
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
