"""Time one epoch-end mAP validation (mcb200.callbacks.ValidationMonitorSegmentation's chain) of N seeded images:
eval forward (UNetResNet-34 on 320 x 320 inputs, the crop_and_pad size of 300 x 300 tiles; timed on its own, since a
random-init net predicts noise), device post-processing on seeded building-like logits
(softmax, resize to 300 x 300, argmax, label, build_score), DeviceCOCOEvaluator.add_batch and result().  Each phase is
bracketed by CUDA events after a device synchronise, so launch time queued before it is kept out; add_batch and
result() include their own host work and device-to-host copies, which is what a user waits for.  Next to it, the
oracle's CPU chain (post_oracle resize / argmax / label / build_score, instances_oracle.create_annotations and
coco_oracle's COCOeval restatement) on the first --cpu-images images.

    python scripts/eval_profile.py [--images 1000] [--batch 20] [--cpu-images 50] [--out result.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=1000)
    ap.add_argument("--batch", type=int, default=20)
    ap.add_argument("--cpu-images", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_profile needs a CUDA device")
    import mcb200  # noqa: F401
    import bench
    import bench_data
    from mcb200 import ops
    from mcb200.callbacks import ValidationMonitorSegmentation
    from mcb200.models import PyTorchUNet
    from oracle import coco_oracle as CO
    from oracle import instances_oracle as I
    from oracle import post_oracle as P
    from oracle import unet_oracle as O

    dev = torch.device("cuda:0")
    model = PyTorchUNet(**bench.unet_config("ResNet34"))
    model.model.load_state_dict(O.make_reference_like_state_dict(34, seed=21))
    model._to_device()
    net = model.model
    net.eval()
    rs = np.random.RandomState(0)
    nb = a.images // a.batch
    xs = [torch.from_numpy(rs.randn(a.batch, 3, 320, 320).astype(np.float32)) for _ in range(nb)]
    # the random-init net predicts noise, so the post-processing and evaluation run on building-like logits instead:
    # log of seeded soft rectangle maps (softmax gives the maps back), about 20 buildings per tile
    maps = [bench_data.probability_maps(a.batch, 320, seed=1000 + b, n_rect=20) for b in range(nb)]
    ev_logits = [torch.from_numpy(np.log(np.maximum(m, 1e-30)).astype(np.float32)) for m in maps]
    ids = list(range(a.images))
    anns, next_id = [], 1
    for i in ids:               # ground truth: the instances of each map's centre crop, so that the AP means something
        lab = P.label(maps[i // a.batch][i % a.batch, 1, 10:310, 10:310] > 0.5)
        for l in range(1, int(lab.max()) + 1):
            inst = (lab == l).astype(np.uint8)
            seg = CO.encode(inst)
            seg["counts"] = seg["counts"].decode("ascii")
            anns.append({"id": next_id, "image_id": i, "category_id": 100, "iscrowd": 0, "area": int(inst.sum()),
                         "segmentation": seg})
            next_id += 1
    import tempfile
    tmp = tempfile.mkdtemp(prefix="mcb_eval_")
    os.makedirs(os.path.join(tmp, "val"))
    with open(os.path.join(tmp, "val", "annotation.json"), "w") as f:
        json.dump({"images": [{"id": i, "height": 300, "width": 300} for i in ids], "annotations": anns,
                   "categories": [{"id": 100}]}, f)

    mon = ValidationMonitorSegmentation(tmp, 14, validate_with_map=True, epoch_every=1)
    mon.meta_valid = ids
    t_build = time.perf_counter()
    ev = mon.evaluator()
    t_build = time.perf_counter() - t_build

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return out, e0.elapsed_time(e1)

    def epoch():
        ev.reset()
        t = {"forward_ms": 0.0, "postprocess_ms": 0.0, "add_batch_ms": 0.0}
        from mcb200.postprocessing import categorize_batch, label_batch, resize_batch, scores_strided
        for b, x in enumerate(xs):
            xd = x.to(dev)
            torch.cuda.synchronize()
            with torch.no_grad():
                _, ms = timed(lambda: net(xd))
            t["forward_ms"] += ms
            logits = ev_logits[b].to(dev)

            def post():
                pr = resize_batch(ops.softmax2(logits.contiguous()), (300, 300))
                cat = categorize_batch(pr)
                planes = torch.stack([(cat == k) for k in range(2)], dim=1).to(torch.uint8).contiguous()
                labels, counts = label_batch(planes, return_counts=True)
                n = pr.shape[0]
                return labels, counts, scores_strided(labels.view(n * 2, 300, 300), pr.view(n * 2, 300, 300), counts,
                                                      4096)
            (labels, counts, scores), ms = timed(post)
            t["postprocess_ms"] += ms
            _, ms = timed(lambda: ev.add_batch(labels, scores, ids[b * a.batch:(b + 1) * a.batch], counts))
            t["add_batch_ms"] += ms
        res, ms = timed(ev.result)
        t["result_ms"] = ms
        t["ap"] = float(res["stats"][0])
        t["detections"] = ev._next_id - 1
        return t

    epoch()                      # warm-up: module loading, allocator, cuDNN-free but first launches
    runs = [epoch() for _ in range(3)]
    t0 = time.perf_counter()          # the monitor's own loop without the forward, wall clock (host launches included)
    mon.model, mon.validation_loss, mon.epoch_id = lambda x: x, {}, 0      # the logits stand in for the forward
    mon.validation_datagen = (ev_logits, None)
    mon._get_validation_loss()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0

    # oracle CPU chain on the first --cpu-images images
    probs = ops.softmax2(torch.cat(ev_logits[:max(1, -(-a.cpu_images // a.batch))]).to(dev)).cpu().numpy()
    probs = probs[:a.cpu_images]
    t0 = time.perf_counter()
    preds = []
    for p in probs:
        r = P.resize_image(p, (300, 300))
        preds.append(P.build_score(P.label_multiclass_image(P.categorize_image(r)), r))
    t_post = time.perf_counter() - t0
    t0 = time.perf_counter()
    I.rle_encode = CO.rle_encode
    res_cpu = I.create_annotations(ids[:len(probs)], preds, [None, 100], [1, 1])
    c_gt = CO.COCO(os.path.join(tmp, "val", "annotation.json"))
    ev_cpu = CO.COCOevalOracle(c_gt, c_gt.loadRes(res_cpu), ids[:len(probs)], [100], 14)
    ev_cpu.evaluate()
    ev_cpu.accumulate()
    ev_cpu.summarize()
    t_eval = time.perf_counter() - t0

    gpu = torch.cuda.get_device_properties(0).name
    try:
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "unavailable (%s)" % e
    med = {k: float(np.median([r[k] for r in runs])) for k in runs[0] if k.endswith("_ms")}
    out = {"gpu": gpu, "power_limit_and_max_sm_clock": q, "images": a.images, "batch": a.batch,
           "device_ms_median_of_3": med, "device_total_ms": sum(med.values()),
           "monitor_wall_s": wall, "ground_truth_tables_build_s": t_build,
           "ap": runs[-1]["ap"], "detections": runs[-1]["detections"],
           "cpu_oracle": {"images": len(probs), "postprocess_s": t_post, "annotations_and_cocoeval_s": t_eval,
                          "per_image_ms": 1000 * (t_post + t_eval) / len(probs)}}
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
