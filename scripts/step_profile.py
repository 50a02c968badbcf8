#!/usr/bin/env python
"""step_profile.py — where the benchmark's train step spends its time between kernels.

  python scripts/step_profile.py --out DIR [--encoder 101] [--batch 32] [--size 320] [--replays 3]

Builds the train step exactly as bench.py does (PyTorchUNetWeighted, seeded weights and batch), warms it up so that
both CUDA graphs are captured, then writes under DIR:
  per_op.txt        the per-launch CUDA-event table of bench.breakdown (an eager pass, one event pair per launch)
  trace.json        a torch.profiler trace of `--replays` captured steps
  summary.json      from the trace: kernel count, kernel-busy time, the gaps between consecutive kernels of the main
                    stream, device idle time (no kernel on any stream), kernels shorter than 5 us, and the launches of
                    the fixed-order finishing kernels (name containing "finish")
The summary is also printed as one JSON line.  Needs a CUDA device; profile in a run of its own, not next to timings."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHORT_US = 5.0


def kernel_events(trace_path):
    with open(trace_path) as f:
        tr = json.load(f)
    ev = [e for e in tr.get("traceEvents", []) if e.get("cat") == "kernel" and e.get("ph") == "X"]
    return [(float(e["ts"]), float(e["dur"]), e.get("args", {}).get("stream", -1), e.get("name", "")) for e in ev]


def summarize(kernels, replays):
    """gap and busy figures of a list of (start_us, dur_us, stream, name)"""
    if not kernels:
        raise SystemExit("the trace holds no kernel events")
    by_stream = {}
    for k in kernels:
        by_stream.setdefault(k[2], []).append(k)
    main = max(by_stream, key=lambda s: len(by_stream[s]))
    seq = sorted(by_stream[main])
    gaps = [max(0.0, b[0] - (a[0] + a[1])) for a, b in zip(seq[:-1], seq[1:])]
    # device-wide: union of kernel intervals over all streams
    iv = sorted((k[0], k[0] + k[1]) for k in kernels)
    busy, cur_s, cur_e = 0.0, iv[0][0], iv[0][1]
    for s, e in iv[1:]:
        if s > cur_e:
            busy += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    busy += cur_e - cur_s
    span = iv[-1][1] - iv[0][0]
    fin = [k for k in kernels if "finish" in k[3]]
    per = 1.0 / replays
    return {
        "replays": replays,
        "kernels_per_step": round(len(kernels) * per, 1),
        "main_stream": main,
        "main_stream_kernels_per_step": round(len(seq) * per, 1),
        "streams": {str(s): len(v) for s, v in by_stream.items()},
        "kernel_busy_ms_per_step": round(sum(k[1] for k in kernels) * per / 1e3, 3),
        "main_stream_busy_ms_per_step": round(sum(k[1] for k in seq) * per / 1e3, 3),
        "main_stream_gap_ms_per_step": round(sum(gaps) * per / 1e3, 3),
        "main_stream_median_gap_us": round(sorted(gaps)[len(gaps) // 2], 2) if gaps else None,
        "device_span_ms_per_step": round(span * per / 1e3, 3),
        "device_idle_ms_per_step": round((span - busy) * per / 1e3, 3),
        "kernels_under_5us_per_step": round(sum(1 for k in kernels if k[1] < SHORT_US) * per, 1),
        "finish_kernels_per_step": round(len(fin) * per, 1),
        "finish_kernel_ms_per_step": round(sum(k[1] for k in fin) * per / 1e3, 3),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--encoder", type=int, default=101)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=320)
    ap.add_argument("--replays", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("step_profile.py needs a CUDA device")
    import bench
    import bench_data
    from mcb200.models import PyTorchUNetWeighted
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(1234)
    model = PyTorchUNetWeighted(**bench.unet_config("ResNet%d" % args.encoder))
    model._to_device()
    x, t = bench_data.train_batch(args.batch, args.size, seed=1234)
    Xd, Td = torch.from_numpy(x).to(dev), torch.from_numpy(t).to(dev)
    for _ in range(max(2, args.warmup)):      # the first step runs eagerly and captures the graphs
        model._fit_loop([Xd, Td])
    torch.cuda.synchronize()

    os.environ["MCB_BENCH_PER_OP"] = os.path.join(args.out, "per_op.txt")
    bench.breakdown(model._fused)
    torch.cuda.synchronize()

    from torch.profiler import profile, ProfilerActivity
    trace = os.path.join(args.out, "trace.json")
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(args.replays):
            model._fit_loop([Xd, Td])
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    s = summarize(kernel_events(trace), args.replays)
    s["device"] = torch.cuda.get_device_name(dev)
    s["launches_per_step_counted_by_plan"] = model._fused.count_launches()
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(s, f, indent=1)
    print(json.dumps(s))


if __name__ == "__main__":
    main()
