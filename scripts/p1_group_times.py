"""Where the headline step's device time goes, kernel by kernel: bench.py's resident workload (128 synthetic FM MP1
channels x 4 L1 frames, cu8 resident in HBM, rewind + process per step) under torch.profiler with CUDA activities.

Prints the step time (CUDA events, profiler off), then the device time per step of every kernel by name and its
share of the step, with the card's name, power limit and the SM clock sampled while timing.  --json FILE also
writes the numbers as one JSON object.

    python scripts/p1_group_times.py [--streams 128] [--frames 4] [--steps 10] [--json FILE]
"""
import argparse
import json
import os
import re
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                               # noqa: E402  (captures, stream views, clock sampler)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        name, plim, smax = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": plim, "max_sm_clock": smax}
    except Exception as ex:                                # the numbers stay valid; only the label is missing
        return {"name": None, "error": str(ex)}


def kernel_name(raw):
    m = re.search(r"(k_\w+)(<[^>]*>)?", raw)
    return (m.group(1) + (m.group(2) or "")) if m else raw


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=128)
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--distinct", type=int, default=4)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", metavar="FILE")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import nrsc5_b200

    if not torch.cuda.is_available():
        raise SystemExit("p1_group_times.py: no CUDA device")
    S = args.streams
    caps = bench.make_captures(args.distinct, args.frames)
    views, nbytes = bench.stream_views(caps, S, 0)
    dev = torch.device("cuda", 0)
    devbuf = torch.empty((S, nbytes + 64), dtype=torch.uint8, device=dev)
    host = torch.empty((S, nbytes), dtype=torch.uint8)
    for s, v in enumerate(views):
        host[s] = torch.from_numpy(v)
    devbuf[:, :nbytes].copy_(host)
    devbuf[:, nbytes:] = 127
    stream = torch.cuda.current_stream()
    log_cap = (args.frames + 1) * (18272 + 64) + 96 * 1024
    e = nrsc5_b200.Engine(nstreams=S, input_capacity=nbytes + 4096, device=0, log_capacity=log_cap)
    e.set_cuda_stream(stream.cuda_stream)
    log_stride = (log_cap + 15) & ~15
    logbuf = torch.zeros((S, log_stride), dtype=torch.uint8, device=dev)
    e.attach_device_log(logbuf.data_ptr(), log_stride)

    def step():
        e.attach_device_input(devbuf.data_ptr(), nbytes + 64, nbytes)
        e.rewind()
        e.process()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()

    # step time with the profiler off
    sampler = bench.ClockSampler(0)
    sampler.start()
    sampler.mark_begin()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(args.steps):
        step()
    ev1.record(stream)
    torch.cuda.synchronize()
    step_ms = ev0.elapsed_time(ev1) / args.steps
    clocks = sampler.stop()
    st = e.stats()

    # per-kernel device time, in a run of its own
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    us = defaultdict(float)
    calls = defaultdict(int)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time > 0:
            k = kernel_name(ev.name)
            us[k] += ev.device_time                # microseconds
            calls[k] += 1
    kernels = {k: {"us_per_step": v / args.steps, "share": v / args.steps / (1e3 * step_ms),
                   "calls_per_step": calls[k] / args.steps} for k, v in sorted(us.items(), key=lambda kv: -kv[1])}
    e.close()

    out = {"card": card(), "sm_clock": clocks, "streams": S, "frames": args.frames, "steps": args.steps,
           "ms_per_step": step_ms, "p1_fast_path_fallbacks": int(getattr(st, "p1_fallbacks", -1)),
           "kernel_us_per_step_sum": sum(v["us_per_step"] for v in kernels.values()), "kernels": kernels}
    c = out["card"]
    print(f"{c.get('name')}  power limit {c.get('power_limit')}  max SM clock {c.get('max_sm_clock')}  "
          f"sampled SM clock {clocks.get('sm_mhz')} MHz")
    print(f"{S} streams x {args.frames} frames: {step_ms:.3f} ms per step (CUDA events, profiler off, {args.steps} steps)")
    print(f"{'kernel':28s} {'us/step':>10s} {'share':>7s} {'calls/step':>11s}")
    for k, v in kernels.items():
        print(f"{k:28s} {v['us_per_step']:10.1f} {100 * v['share']:6.1f}% {v['calls_per_step']:11.1f}")
    print(f"{'(sum of kernels)':28s} {out['kernel_us_per_step_sum']:10.1f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
