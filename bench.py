#!/usr/bin/env python
"""bench.py — headline benchmark of the H100 hot path.

  python bench.py --gpus N --steps K --warmup W          our arm: ResNet101-UNet train step, batch 32/GPU, 300x300
                                                          tiles replicate-padded to the 320x320 net input
  python bench.py --impl reference ...                    the reference's CPU path (oracle port) on the host cores
  python bench.py --impl torch_cudnn ...                  LIBRARY baseline: the same net / step in stock PyTorch (cuDNN,
                                                          channels_last, bf16 autocast, fused Adam) on the same GPU
  python bench.py --workload infer ...                    BASELINE.json configs[3]: eval forward + full post-processing
                                                          (dense CRF, threshold, erode, label, dilate, score, watershed),
                                                          batch 64, host images in -> host label maps out

One JSON line on stdout (rank 0).  `value` = tiles/s with inputs resident in HBM; `e2e` = the same metric through the
reference-facing API (PyTorchUNetWeighted._fit_loop on pinned HOST batches, loss read back every step).

  --dump-outputs DIR   (train workload) after the timed steps, write what they computed as DIR/<name>.npy (float32 /
                       float64): the last step's loss and a fixed, seeded sample of the trained fp32 parameters.  Inputs
                       and initial weights are seeded, so two builds run with the same arguments compare output for
                       output."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

FLOP_PER_TILE = {(101, 320): 205.71e9, (101, 256): 131.7e9, (34, 256): 79.54e9, (152, 512): 643.0e9}


def unet_config(encoder, lr=5e-4):
    """the `config.unet` dict of the reference's src/pipeline_config.py:61-120 (values from neptune.yaml)"""
    return {
        'architecture_config': {
            'model_params': {'n_filters': 16, 'conv_kernel': 3, 'pool_kernel': 3, 'pool_stride': 2, 'repeat_blocks': 4,
                             'batch_norm': 1, 'dropout': 0.1, 'in_channels': 3, 'out_channels': 2, 'nr_outputs': 1,
                             'encoder': encoder},
            'optimizer_params': {'lr': lr},
            'regularizer_params': {'regularize': True, 'weight_decay_conv2d': 1e-4},
            'weights_init': {'function': 'he'},
            'loss_weights': {'bce_mask': 1.0, 'dice_mask': 0.2},
            'weighted_cross_entropy': {'w0': 50, 'sigma': 10, 'imsize': (256, 256)},
            'dice': {'smooth': 1, 'dice_activation': 'softmax'},
        },
        'training_config': {'epochs': 1},
        'callbacks_config': {},
    }


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d.get("bf16_tflops_sustained", d.get("bf16_tflops")), d.get("hbm_gbs"), "measured (MEASURED_PEAKS.json, sustained)"
    return 989.0, 3350.0, "data sheet (H100 SXM, dense BF16 / HBM3, at 700 W)"


class ClockSampler:
    def __init__(self, index):
        self.path = tempfile.mktemp(suffix=".csv")
        self.proc = None
        self.index = index

    def start(self):
        q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
            "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=open(self.path, "w"), stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def stop(self):
        out = {"sm_mhz": None, "sm_max_mhz": None, "reasons": []}
        if self.proc is None:
            return out
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        rows = []
        for line in open(self.path):
            f = [x.strip() for x in line.split(",")]
            if len(f) >= 7:
                try:
                    rows.append((float(f[0]), float(f[1]), float(f[2]), f[3], f[4], f[5], f[6]))
                except ValueError:
                    pass
        os.unlink(self.path)
        if not rows:
            return out
        busy = [r for r in rows if r[2] > 300] or rows
        sm = sorted(r[0] for r in busy)
        out["sm_mhz"] = sm[len(sm) // 2]
        out["sm_max_mhz"] = rows[0][1]
        out["power_w_max"] = max(r[2] for r in rows)
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        out["reasons"] = [n for i, n in enumerate(names) if any(r[3 + i].lower().startswith("active") for r in rows)]
        return out


def usable_cores():
    """host cores this process may actually use: affinity mask, cgroup CPU quota, capped at 32 (torch's intra-op
    parallelism stops scaling — and on over-subscribed boxes collapses — beyond that for these layer sizes)"""
    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except Exception:
        pass
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(float(q) / float(p))))
    except Exception:
        pass
    return max(1, min(n, 32))


def cpu_reference_arm(args, sample_batch=None, steps=None, warmup=None):
    """the reference's own CPU implementation of the train step (oracle port of Model._fit_loop, fp32, all host
    threads) on a bounded sample of the workload"""
    import torch
    from oracle import unet_oracle as O
    import bench_data as synthetic
    cores = usable_cores()
    torch.set_num_threads(cores)
    b = sample_batch or max(1, min(args.batch, 4))
    steps = steps or max(1, min(args.steps, 3))
    warmup = 1 if warmup is None else warmup
    sd = O.make_reference_like_state_dict(args.encoder, seed=1234)
    x, t = synthetic.train_batch(b, args.size, seed=1234)
    X, T = torch.from_numpy(x), torch.from_numpy(t)
    opt = O.AdamOracle(lr=5e-4, weight_decay=1e-4)
    tw = time.time()
    for _ in range(warmup):
        O.train_step(sd, args.encoder, X, T, opt, imsize=(256, 256))
    tw = (time.time() - tw) / max(warmup, 1)
    if warmup and tw * steps > 60:  # keep the whole arm bounded
        steps = max(1, int(60 / tw))
    t0 = time.time()
    for _ in range(steps):
        O.train_step(sd, args.encoder, X, T, opt, imsize=(256, 256))
    dt = (time.time() - t0) / steps
    return {"value": b / dt, "unit": "tiles/s", "cores": torch.get_num_threads(), "kind": "port",
            "sample": "oracle port of Model._fit_loop (fp32 torch CPU), UNetResNet-%d, batch %d @%dx%d, %d warm-up + %d timed steps"
                      % (args.encoder, b, args.size, args.size, warmup, steps), "ms_per_step": dt * 1e3,
            "steps_run": steps, "warmup_run": warmup, "batch_run": b}


def breakdown(step, n_iter=2):
    """instrumented eager pass: CUDA events around every launch of the plan, grouped by kernel family"""
    import torch
    plan = step.plan
    ops = [("fwd", o) for o in plan.fwd_ops] + [("bwd", o) for l in plan.bwd_layers for o in l]
    acc = {}
    for it in range(n_iter):
        plan._stats_arena.zero_()
        evs = []
        for phase, o in ops:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            o()
            e1.record()
            evs.append((o, e0, e1))
        torch.cuda.synchronize()
        if it == n_iter - 1:
            for o, e0, e1 in evs:
                a = acc.setdefault(o.kind, [0, 0.0, 0.0, 0.0])
                a[0] += 1
                a[1] += e0.elapsed_time(e1)
                a[2] += o.flops
                a[3] += o.bytes
    total = sum(a[1] for a in acc.values())
    per_op = os.environ.get("MCB_BENCH_PER_OP")
    if per_op:
        rows = sorted(((e0.elapsed_time(e1), o) for o, e0, e1 in evs), key=lambda r: -r[0])
        with open(per_op, "w") as f:
            for ms, o in rows:
                f.write("%8.4f ms  %-14s %-40s %7.1f TFLOP/s %8.1f GB/s\n" % (
                    ms, o.kind, o.desc, o.flops / (ms * 1e-3) / 1e12 if ms > 0 else 0,
                    o.bytes / (ms * 1e-3) / 1e9 if ms > 0 else 0))
    out = {}
    for k, a in sorted(acc.items(), key=lambda kv: -kv[1][1]):
        out[k] = {"launches": a[0], "ms": round(a[1], 3), "share": round(a[1] / total, 4),
                  "tflops": round(a[2] / (a[1] * 1e-3) / 1e12, 1) if a[2] else None,
                  "algo_gbs": round(a[3] / (a[1] * 1e-3) / 1e9, 1) if a[3] else None}
    return out, total


def library_baseline(args, dev, Xd, Td, steps=10, warmup=3):
    """stock PyTorch on the same GPU: baseline/torch_cudnn_unet.py (cuDNN, channels_last, bf16 autocast, fused Adam)"""
    import torch
    from baseline.torch_cudnn_unet import TrainStep
    try:
        ts = TrainStep(args.encoder, dev)
        for _ in range(warmup):
            ts.step(Xd, Td)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            loss = ts.step(Xd, Td)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        out = {"value": round(Xd.shape[0] / (ms * 1e-3), 2), "unit": "tiles/s", "ms_per_step": round(ms, 4),
               "steps": steps, "warmup": warmup, "loss_last_step": float(loss),
               "what": "torch %s eager: torchvision ResNet-%d U-Net, cuDNN %s, channels_last, bf16 autocast, "
                       "torch.optim.Adam(fused=True), same batch / size / loss; inputs resident in HBM"
                       % (torch.__version__, args.encoder, torch.backends.cudnn.version())}
        del ts
        torch.cuda.empty_cache()
        return out
    except Exception as e:  # the baseline must never take the product's bench line down with it
        return {"value": None, "error": "%s: %s" % (type(e).__name__, e)}


def library_baseline_line(args, dev, rank, world, workload):
    """--impl torch_cudnn: the library baseline as its own bench line (same metric / config / timing rules)"""
    import torch
    import torch.distributed as dist
    import bench_data as synthetic
    x, t = synthetic.train_batch(args.batch, args.size, seed=1234 + rank)
    Xd, Td = torch.from_numpy(x).to(dev), torch.from_numpy(t).to(dev)
    sampler = ClockSampler(dev.index or 0) if rank == 0 else None
    if sampler:
        sampler.start()
    lb = library_baseline(args, dev, Xd, Td, steps=args.steps, warmup=args.warmup)
    clocks = sampler.stop() if sampler else None
    if world > 1:   # independent replicas (no gradient exchange): a generous upper bound for DDP
        v = torch.tensor([lb["ms_per_step"] or 0.0], device=dev)
        dist.all_reduce(v, op=dist.ReduceOp.MAX)
        lb["ms_per_step"] = float(v)
        lb["value"] = args.batch / (lb["ms_per_step"] * 1e-3)
    peak_tf, _, peak_src = peaks()
    fpt = FLOP_PER_TILE.get((args.encoder, args.size))
    achieved = (lb["value"] or 0) * (fpt or 0) / 1e12
    return {"impl": "torch_cudnn", "metric": "300x300 tiles/sec fwd+bwd ResNet101-UNet",
            "value": round((lb["value"] or 0) * world, 2), "unit": "tiles/s", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": lb.get("ms_per_step"), "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": workload, "global_batch": args.batch * world,
                       "parallelism": "dp%d (independent replicas, no gradient exchange)" % world, "what": lb.get("what")},
            "clocks": clocks, "gpu_launches": 0,
            "roofline": {"bound": "tensor", "achieved": round(achieved, 1), "peak": peak_tf, "unit": "TFLOP/s",
                         "frac": round(achieved / peak_tf, 4), "traffic": None, "peak_source": peak_src},
            "error": lb.get("error")}


# ------------------------------------------------------------------------------------------------------------------
# --workload infer: BASELINE.json configs[3]
# ------------------------------------------------------------------------------------------------------------------
INFER_METRIC = "300x300 tiles/sec inference + full post-processing ResNet101-UNet"
POST_BYTES_PER_IMAGE = 1.44e6   # SURVEY.md 8d: 2x300x300 fp32 probabilities in, 2x300x300 int32 labels out


def infer_workload_name(args):
    return ("UNetResNet-%d eval forward + softmax, batch %d/GPU, 300x300 tiles replicate-padded to %dx%d, then per image: "
            "centre crop -> dense CRF (5 mean-field iterations) -> resize_image (identity size, fp64) -> threshold -> erode 2 -> label -> dilate 2 -> score, "
            "and a marker watershed split of the refined building probability" % (args.encoder, args.batch, args.size,
                                                                                args.size))


def infer_line(args, dev, rank, world):
    """inference + the full per-pixel chain.  `value`: inputs resident in HBM, results left on the device.  `e2e`:
    pinned HOST images in, HOST label maps / scores / watershed labels out, copies inside the timed region."""
    import numpy as np
    import torch
    import torch.distributed as dist
    import bench_data as synthetic
    from mcb200 import ops, postprocessing as G
    from mcb200.models import PyTorchUNet
    b, s = args.batch, args.size
    torch.manual_seed(1234)
    model = PyTorchUNet(**unet_config("ResNet%d" % args.encoder))
    model._to_device()
    net = model.model
    net.eval()
    x, _ = synthetic.train_batch(b, s, seed=1234 + rank)
    Xh = torch.from_numpy(x).pin_memory()
    Xd = Xh.to(dev)
    # a random-init net predicts noise: the chain is fed building-like probability maps of the same shape / dtype
    # (the forward pass still runs on X every step; its output is blended out with weight 0 so that the dependency stays)
    syn = torch.from_numpy(synthetic.probability_maps(b, s, seed=7 + rank)).to(dev)
    mode = "crop" if s == 320 else "resize"
    pp = G.MaskPostprocessor((300, 300), "resize", erode_selem_size=2, dilate_selem_size=2)
    m0 = (s - 300) // 2 if mode == "crop" else 0
    timing = {}

    def chain(X, record=False):
        evs = []

        def mark(name):
            if record:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                evs.append((name, e))
        mark("start")
        with torch.no_grad():
            probs = ops.softmax2(net(X))
        mark("forward+softmax")
        probs = probs * 0.0 + syn
        if mode == "crop":   # prediction_crop (src/pipelines.py:44-60), then the chain's own identity-sized mask_resize
            pc = probs[:, :, m0:s - m0, m0:s - m0].contiguous()
            img = X[:, :, m0:s - m0, m0:s - m0].contiguous()
        else:
            pc, img = probs, X
        mark("crop")
        refined = G.dense_crf_batch(img, pc)
        mark("dense_crf")
        labels, scores, counts, _pr = pp.run_device_graphed(refined)
        mark("resize+threshold+erode+label+dilate+score")
        ws = G.watershed_split(refined[:, 1].contiguous(), hi=0.8, lo=0.5)
        mark("watershed")
        if record:
            torch.cuda.synchronize()
            for (n0, e0), (n1, e1) in zip(evs[:-1], evs[1:]):
                timing[n1] = timing.get(n1, 0.0) + e0.elapsed_time(e1)
        return labels, scores, counts, ws

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms) / steps

    for _ in range(args.warmup):
        chain(Xd)
    sampler = ClockSampler(dev.index or 0) if rank == 0 else None
    if sampler:
        sampler.start()
    ms_dev = timed(lambda: chain(Xd), args.steps)
    clocks = sampler.stop() if sampler else None
    n_rec = 3
    for _ in range(n_rec):
        chain(Xd, record=True)
    stages = {k: round(v / n_rec, 4) for k, v in timing.items()}

    # end to end: host images in, host results out (pinned, reused buffers)
    out_h = {}

    def step_e2e():
        X = Xh.to(dev, non_blocking=True)
        labels, scores, counts, ws = chain(X)
        for k, t in (("labels", labels), ("scores", scores), ("counts", counts), ("ws", ws)):
            if k not in out_h:
                out_h[k] = torch.empty(t.shape, dtype=t.dtype).pin_memory()
            out_h[k].copy_(t, non_blocking=True)
        torch.cuda.current_stream().synchronize()   # the caller owns the results when the call returns

    for _ in range(args.warmup):
        step_e2e()
    ms_e2e = timed(step_e2e, args.steps)
    d2h = int(sum(t.numel() * t.element_size() for t in out_h.values()))
    if rank != 0:
        return None
    _, peak_hbm, peak_src = peaks()
    post_ms = sum(v for k, v in stages.items() if k not in ("forward+softmax",))
    chain_ms = stages.get("resize+threshold+erode+label+dilate+score", 0.0)
    tiles = b * world
    line = {
        "metric": INFER_METRIC, "value": round(tiles / (ms_dev * 1e-3), 2), "unit": "tiles/s", "n_gpus": world,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": round(ms_dev, 4), "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "bf16 (network) / f32, u8, i32 (post-processing)", "data": "synthetic",
        "config": {"workload": infer_workload_name(args), "global_batch": tiles, "parallelism": "dp%d replicas" % world,
                   "l2": "the batch's maps (92 MB of probabilities + labels, GBs of activations) exceed the 50 MB L2"},
        "e2e": {"value": round(tiles / (ms_e2e * 1e-3), 2), "unit": "tiles/s", "ms_per_step": round(ms_e2e, 4),
                "h2d_bytes_per_step": int(Xh.numel() * 4), "d2h_bytes_per_step": d2h,
                "api": "PyTorchUNet net forward on pinned host images -> MaskPostprocessor + dense_crf_batch + "
                       "watershed_split -> pinned host labels / scores / counts / watershed labels"},
        "gpu_launches": None, "clocks": clocks,
        "stages_ms": stages,
        "postproc": {"ms_all_stages": round(post_ms, 4), "share_of_step_all_stages": round(post_ms / (post_ms + stages["forward+softmax"]), 4),
                     "ms_reference_chain": round(chain_ms, 4),
                     "share_of_step_reference_chain": round(chain_ms / (chain_ms + stages["forward+softmax"]), 4),
                     "note": "reference chain = what src/pipelines.py:248-304 runs (threshold, erode, label, dilate, score); "
                             "dense CRF is unwired in the reference and the watershed is not in it"},
        "roofline": {"bound": "hbm", "achieved": round(b * POST_BYTES_PER_IMAGE / (chain_ms * 1e-3) / 1e9, 1) if chain_ms else None,
                     "peak": peak_hbm, "unit": "GB/s",
                     "frac": round(b * POST_BYTES_PER_IMAGE / (chain_ms * 1e-3) / 1e9 / peak_hbm, 4) if chain_ms else None,
                     "traffic": None, "peak_source": peak_src,
                     "what": "reference post-processing chain of one batch: 1.44 MB/image algorithmic (SURVEY.md 8d) / its "
                             "device time"},
    }
    plan = net.module.plan(b, s, s, False) if hasattr(net, "module") else net.plan(b, s, s, False)
    line["gpu_launches"] = (plan.launches_fwd + 40) * args.steps
    if not args.no_cpu_baseline and world == 1:
        cb = infer_cpu_baseline(args)
        line["cpu_baseline"] = cb
    return line


def infer_cpu_baseline(args, n_fwd=2, n_post=8):
    """the reference's CPU path for configs[3] on a bounded sample: eval forward (oracle port, fp32, all host threads) on
    n_fwd tiles + the serial per-image post-processing chain (src/utils.py:352-355 loop over src/postprocessing.py
    functions, restated in oracle/post_oracle.py) on n_post tiles, single process like the reference runs it; dense CRF and
    watershed are the builder's restatements (parity unpinned) timed on one tile each"""
    import numpy as np
    import torch
    from oracle import post_oracle as P, unet_oracle as O
    import bench_data as synthetic
    cores = usable_cores()
    torch.set_num_threads(cores)
    s = args.size
    sd = O.make_reference_like_state_dict(args.encoder, seed=1234)
    x, _ = synthetic.train_batch(n_fwd, s, seed=1234)
    net = O.UNetOracle(sd, args.encoder)
    with torch.no_grad():
        net.forward(torch.from_numpy(x[:1]))
        t0 = time.time()
        net.forward(torch.from_numpy(x))
        t_fwd = (time.time() - t0) / n_fwd
    probs = synthetic.probability_maps(n_post, s, seed=7)
    t0 = time.time()
    for p_ in probs:
        r = P.resize_image(P.crop_image_center_per_class(p_, 300, 300) if s == 320 else p_, (300, 300))
        m_ = P.categorize_multilayer_image(r)
        m_ = P.erode_image(m_, 2)
        l_ = P.label_multilayer_image(m_)
        l_ = P.dilate_image(l_, 2)
        P.build_score(l_, r)
    t_chain = (time.time() - t0) / n_post
    extra = {}
    try:
        p1 = P.crop_image_center_per_class(probs[0], 300, 300) if s == 320 else P.resize_image(probs[0], (300, 300)).astype(np.float32)
        img = np.random.RandomState(0).randn(3, 300, 300).astype(np.float32)
        t0 = time.time()
        P.dense_crf(img, p1.astype(np.float32))
        extra["dense_crf_s_per_image"] = round(time.time() - t0, 3)
    except Exception as e:
        extra["dense_crf_error"] = str(e)
    per_img = t_fwd + t_chain
    return {"value": round(1.0 / per_img, 3), "unit": "tiles/s", "cores": cores, "kind": "port",
            "sample": "oracle port: eval forward on %d tiles (%.2f s/tile, %d threads) + serial reference post-processing chain "
                      "on %d tiles (%.1f ms/tile, 1 process); CRF / watershed excluded from `value` (unwired / absent in "
                      "the reference)" % (n_fwd, t_fwd, cores, n_post, t_chain * 1e3),
            "forward_s_per_tile": round(t_fwd, 3), "postproc_ms_per_tile": round(t_chain * 1e3, 2), **extra}


def infer_reference_line(args):
    cb = infer_cpu_baseline(args)
    return {"impl": "reference", "metric": INFER_METRIC, "value": cb["value"], "unit": "tiles/s", "n_gpus": args.gpus,
            "steps": 1, "warmup": 1, "requested": {"steps": args.steps, "warmup": args.warmup},
            "ms_per_step": round(1e3 / cb["value"], 2), "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": infer_workload_name(args), "global_batch": args.batch * args.gpus, "parallelism": "cpu"},
            "cpu_baseline": cb, "e2e": {"value": cb["value"], "unit": "tiles/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}


_REAL_STDOUT = None


def finish_distributed():
    """orderly multi-GPU exit: every rank is done computing; captured graphs hold NCCL work, so skip the communicator
    teardown (it can wait forever on them) and leave with status 0"""
    import torch
    import torch.distributed as dist
    sys.stdout.flush()
    sys.stderr.flush()
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    os._exit(0)


def emit(line):
    """the ONE JSON line goes to the real stdout; everything else this process (or NCCL's banner, printed from C) writes
    to fd 1 has been rerouted to stderr by main()"""
    data = (json.dumps(line) + "\n").encode()
    if _REAL_STDOUT is None:
        sys.stdout.write(data.decode()); sys.stdout.flush()
    else:
        os.write(_REAL_STDOUT, data)


DUMP_PARAM_SAMPLE = 1 << 20   # parameters written by --dump-outputs (4 MB of float32)


def dump_train_outputs(out_dir, loss, p32):
    """the timed path's results: the loss of its last step and the fp32 master parameters it trained, sampled at
    seeded positions (the same positions for every run of the same network)"""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), loss.detach().double().cpu().numpy().reshape(-1))
    n = p32.numel()
    g = torch.Generator().manual_seed(1234)
    idx = torch.randperm(n, generator=g)[:DUMP_PARAM_SAMPLE].sort().values if n > DUMP_PARAM_SAMPLE else torch.arange(n)
    np.save(os.path.join(out_dir, "params_sample.npy"), p32.detach().reshape(-1)[idx.to(p32.device)].float().cpu().numpy())
    np.save(os.path.join(out_dir, "params_sample_index.npy"), idx.double().numpy())


def main():
    global _REAL_STDOUT
    sys.stdout.flush()
    _REAL_STDOUT = os.dup(1)
    os.dup2(2, 1)
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "torch_cudnn"])
    ap.add_argument("--workload", default="train", choices=["train", "infer"])
    ap.add_argument("--no-library-baseline", action="store_true")
    ap.add_argument("--encoder", type=int, default=101)
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--size", type=int, default=320)
    ap.add_argument("--no-breakdown", action="store_true")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="train workload: write the last timed step's loss and a seeded parameter sample as DIR/*.npy")
    args = ap.parse_args()
    if args.dump_outputs and (args.workload != "train" or args.impl != "ours"):
        raise SystemExit("--dump-outputs writes the outputs of the train workload of impl ours")
    if args.batch is None:
        args.batch = 64 if args.workload == "infer" else 32
    args.warmup = max(args.warmup, 3) if args.impl != "reference" else args.warmup
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    workload = "UNetResNet-%d train step (fwd + weighted-CE/Dice loss + bwd + Adam), batch %d/GPU, 300x300 tiles " \
               "replicate-padded to the %dx%d net input (reference loader_mode crop_and_pad)" % (
                   args.encoder, args.batch, args.size, args.size)

    if args.impl == "reference":
        if rank != 0:
            return
        if args.workload == "infer":
            emit(infer_reference_line(args))
            return
        cb = cpu_reference_arm(args)
        # `steps` / `warmup` are what this arm RAN (each step = one reference train step on a bounded sample of the
        # workload: batch `batch_run` instead of args.batch, so that the run ends within minutes on host cores);
        # the values asked for on the command line are kept under `requested`
        line = {"impl": "reference", "metric": "300x300 tiles/sec fwd+bwd ResNet101-UNet", "value": cb["value"],
                "unit": "tiles/s", "n_gpus": args.gpus, "steps": cb["steps_run"], "warmup": cb["warmup_run"],
                "requested": {"steps": args.steps, "warmup": args.warmup, "batch": args.batch},
                "ms_per_step": cb["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": "f32", "data": "synthetic",
                "config": {"workload": workload, "global_batch": args.batch * args.gpus, "parallelism": "cpu",
                           "sample_batch": cb["batch_run"]},
                "cpu_baseline": {k: cb[k] for k in ("value", "unit", "cores", "kind", "sample")},
                "e2e": {"value": cb["value"], "unit": "tiles/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
                "gpu_launches": 0}
        emit(line)
        return

    import torch
    import torch.distributed as dist
    if not torch.cuda.is_available():
        raise SystemExit("bench.py (impl ours) needs a CUDA device; there is no CPU fallback")
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    dev = torch.device("cuda", local_rank)
    if args.impl == "torch_cudnn":
        line = library_baseline_line(args, dev, rank, world, workload)
        if rank == 0:
            emit(line)
        if world > 1:
            finish_distributed()
        return
    import mcb200
    from mcb200.models import PyTorchUNetWeighted
    import bench_data as synthetic
    if args.workload == "infer":
        line = infer_line(args, dev, rank, world)
        if rank == 0:
            emit(line)
        if world > 1:
            finish_distributed()
        return

    t_start = time.time()

    def note(msg):
        if os.environ.get("MCB_BENCH_VERBOSE"):
            sys.stderr.write("[bench %7.2fs] %s\n" % (time.time() - t_start, msg))
            sys.stderr.flush()

    torch.manual_seed(1234)
    model = PyTorchUNetWeighted(**unet_config("ResNet%d" % args.encoder))
    model._to_device()
    x, t = synthetic.train_batch(args.batch, args.size, seed=1234 + rank)
    Xh, Th = torch.from_numpy(x).pin_memory(), torch.from_numpy(t).pin_memory()
    Xd, Td = Xh.to(dev), Th.to(dev)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms) / steps

    # ---- device-resident arm
    last = {}

    def step_dev():
        last["loss"] = model._fit_loop([Xd, Td])["sum"]

    note("model + data ready")
    for i in range(args.warmup):
        step_dev()
        torch.cuda.synchronize()
        note("warm-up step %d done" % i)
    sampler = ClockSampler(local_rank) if rank == 0 else None
    if sampler:
        sampler.start()
    ms_dev = timed(step_dev, args.steps)
    clocks = sampler.stop() if sampler else None
    loss_dev = float(last["loss"])
    if args.dump_outputs and rank == 0:
        dump_train_outputs(args.dump_outputs, last["loss"], model._net()._p32)
    note("device arm timed: %.3f ms/step" % ms_dev)

    # ---- end-to-end arm: pinned host batches in, loss read back EVERY step.  One step of pipelining: the D2H copy of
    # step i's loss is enqueued (into pinned memory, followed by an event) right behind step i, and the host consumes it
    # after it has enqueued step i+1 -- so the H2D copy of the next batch and the host-side launch work overlap compute.
    # (A plain loss.cpu() of the previous step would be stream-ordered behind the step just enqueued and stall the host
    # for a whole step.)
    loss_host = [torch.zeros(1, dtype=torch.float32).pin_memory() for _ in range(2)]
    loss_ev = [torch.cuda.Event() for _ in range(2)]
    prev = {"i": 0, "pending": False}

    def step_e2e():
        i = prev["i"]
        cur = model._fit_loop([Xh, Th])["sum"]
        loss_host[i & 1].copy_(cur, non_blocking=True)
        loss_ev[i & 1].record()
        if prev["pending"]:
            loss_ev[(i - 1) & 1].synchronize()
            prev["val"] = float(loss_host[(i - 1) & 1])
        prev["pending"] = True
        prev["i"] = i + 1

    for _ in range(args.warmup):
        step_e2e()
    ms_e2e = timed(step_e2e, args.steps)
    note("e2e arm timed: %.3f ms/step" % ms_e2e)

    # data-parallel sanity: every rank trains on different tiles, so the replicas stay identical only if the gradient
    # all-reduce really happened -- a parameter checksum must agree across ranks (a step without the exchange would be
    # faster and meaningless)
    in_sync = None
    if world > 1:
        chk = model._net()._p32.double().sum().reshape(1)
        allc = [torch.zeros_like(chk) for _ in range(world)]
        dist.all_gather(allc, chk)
        vals = [float(c) for c in allc]
        in_sync = (max(vals) - min(vals)) <= 1e-9 * max(1.0, abs(vals[0]))
        if not in_sync:
            raise RuntimeError("replicas diverged (parameter checksums %r): gradient all-reduce missing?" % (vals,))

    # phase split of the captured step (CUDA events between the graph replays), averaged over 5 extra steps
    phases = {}
    fz = model._fused
    for _ in range(5):
        fz.phase_marks = []
        step_dev()
        torch.cuda.synchronize()
        for (n0, e0), (n1, e1) in zip(fz.phase_marks[:-1], fz.phase_marks[1:]):
            phases[n1] = phases.get(n1, 0.0) + e0.elapsed_time(e1) / 5
    fz.phase_marks = None
    tiles = args.batch * world
    value = tiles / (ms_dev * 1e-3)
    e2e = tiles / (ms_e2e * 1e-3)
    fused = model._fused
    if rank != 0:
        if world > 1:
            finish_distributed()
        return
    peak_tf, peak_hbm, peak_src = peaks()
    fpt = FLOP_PER_TILE.get((args.encoder, args.size))
    if fpt is None:
        fpt = (sum(o.flops for o in fused.plan.fwd_ops) + sum(o.flops for l in fused.plan.bwd_layers for o in l)) / args.batch
    achieved = value / world * fpt / 1e12
    line = {
        "metric": "300x300 tiles/sec fwd+bwd ResNet101-UNet", "value": round(value, 2), "unit": "tiles/s",
        "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": round(ms_dev, 4),
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": {"workload": workload, "global_batch": tiles, "parallelism": "dp%d" % world,
                   "bn": ("synchronised over the global batch (MCB_SYNC_BN=%s)" % os.environ.get("MCB_SYNC_BN") if fused.plan.sync_bn
                          else "per-replica batch statistics (reference DataParallel semantics)") if world > 1 else "batch statistics",
                   "grad_allreduce": ("in-graph, per arena segment, overlapped with the backward pass" if fused.inline_allreduce
                                      else "one call after the backward graph") if world > 1 else None,
                   "replicas_in_sync": in_sync,
                   "l2": "per-step working set (activations + gradients, GBs) far exceeds the 50 MB L2; no flush needed",
                   "loss_last_step": loss_dev},
        "e2e": {"value": round(e2e, 2), "unit": "tiles/s", "ms_per_step": round(ms_e2e, 4),
                "h2d_bytes_per_step": int(Xh.numel() * 4 + Th.numel() * 4), "d2h_bytes_per_step": 4,
                "api": "mcb200.models.PyTorchUNetWeighted._fit_loop([X_host_pinned, target_host_pinned]) + async D2H of the loss into pinned memory, consumed one step later"},
        "gpu_launches": fused.count_launches() * args.steps,
        "phases_ms": {k: round(v, 3) for k, v in phases.items()},
        "clocks": clocks,
        "roofline": {"bound": "tensor", "achieved": round(achieved, 1), "peak": peak_tf, "unit": "TFLOP/s",
                     "frac": round(achieved / peak_tf, 4), "traffic": None, "peak_source": peak_src,
                     "what": "conv/convT fwd+dgrad+wgrad wgmma GEMM family: algorithmic conv FLOPs of the step "
                             "(%.2f GFLOP/tile) / whole-step time per GPU" % (fpt / 1e9)},
    }
    if not args.no_breakdown:
        bd, total = breakdown(fused)
        note("breakdown done")
        line["breakdown"] = bd
        gemm = [v for k, v in bd.items() if k.startswith("conv")]
        gemm_ms = sum(v["ms"] for v in gemm)
        gemm_fl = sum((v["tflops"] or 0) * v["ms"] for v in gemm)
        line["roofline"]["gemm_family_ms"] = round(gemm_ms, 3)
        line["roofline"]["gemm_family_tflops"] = round(gemm_fl / gemm_ms, 1) if gemm_ms else None
        line["roofline"]["gemm_family_share_of_step"] = round(gemm_ms / total, 4)
        line["roofline"]["gemm_family_algorithmic_bytes"] = int(sum((v["algo_gbs"] or 0) * v["ms"] * 1e6 for v in gemm))
    if not args.no_library_baseline and world == 1:
        # the stock-PyTorch (cuDNN) train step of the same net on the same GPU, measured right here: the library
        # baseline this framework has to beat
        del Xh, Th
        lb = library_baseline(args, dev, Xd, Td, steps=min(args.steps, 10), warmup=3)
        line["library_baseline"] = lb
        line["library_baseline"]["ours_over_library"] = round(value / lb["value"], 3) if lb.get("value") else None
        note("library baseline done")
    if not args.no_cpu_baseline and world == 1:
        cb = cpu_reference_arm(args, sample_batch=2, steps=2, warmup=1)
        line["cpu_baseline"] = {k: cb[k] for k in ("value", "unit", "cores", "kind", "sample")}
        note("cpu baseline done")
    emit(line)
    if world > 1:
        finish_distributed()


if __name__ == "__main__":
    main()
