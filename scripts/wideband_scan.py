"""The band scan (nrsc5b_scan_*) on the GPU: device time of k_scan + k_scan_finish per second of capture, for the
100 FM station slots of a 23.814 MS/s capture (odd offsets -99..+99) and the 118 AM channels of a 1 488 375 S/s
capture (-58..+59), beside the channeliser (k_channelize, with its cs16 split pass) on the same capture.

Gate, before any number: the scan of the timed channel output equals the numpy restatement (tests/scan_oracle.py) on
four of its channels, every accumulator bit for bit.

Each timing is CUDA events around --reps launches after --warmup, alternating scan and channeliser, --runs times; the
median is reported.  The card's name and power limit are read in the same run.  Prints one JSON line (and writes it
to --out).  There is no CPU path: without a CUDA device it fails.

    python scripts/wideband_scan.py [--runs 5 --reps 10 --warmup 3] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def card_info():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as ex:                                        # noqa: BLE001
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "error": repr(ex)[:200]}


def events_ms(fn, reps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def one_band(band, offs, seconds, args):
    import torch
    import scan_oracle as so
    from nrsc5_b200 import channelizer as ch, scan
    wide = ch.WIDE_RATE if band == "fm" else ch.AM_WIDE_RATE
    n = int(seconds * wide)
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    x = torch.clamp(torch.round(torch.randn(2 * n, generator=g, device="cuda") * 3000.0), -32768, 32767).to(torch.int16)
    nout = ch.outputs(x.numel(), band)
    stride = (2 * nout + 64) & ~31
    d_out = torch.zeros((len(offs), stride), dtype=torch.int16, device="cuda")
    with ch.Channelizer(offs, input_cs16=True, band=band) as c, scan.Scanner(len(offs), band) as s:
        chan = lambda: c.run_device(x.data_ptr(), x.numel(), d_out.data_ptr(), stride)      # noqa: E731

        def scan_once():
            s.reset()
            s.push_device(d_out.data_ptr(), stride, nout)
            s.result()
        chan()
        torch.cuda.synchronize()
        s.reset()
        s.push_device(d_out.data_ptr(), stride, nout)
        _, raw = s.result(raw=True)
        mode = scan.MODES[band]
        taps, kappa = scan.make_tables(band)
        J = so.geometry(mode)[4]
        pick = [0, len(offs) // 3, len(offs) // 2, len(offs) - 1]
        y = d_out[pick, : 2 * nout].cpu().numpy()
        acc, _, _ = so.accumulate(y, mode, taps)
        assert np.array_equal(raw[pick, : 6 * J].reshape(-1, 6, J), acc), f"{band}: the scan differs from the restatement"
        t_scan, t_chan = [], []
        for _ in range(args.runs):
            t_scan.append(events_ms(scan_once, args.reps, args.warmup))
            t_chan.append(events_ms(chan, args.reps, args.warmup))
    # 4 int32 multiply-adds per tap and filter output pair; (S + F) / q outputs per S samples (the halo), per channel
    q = so.geometry(mode)[2]
    macs = 4 * 64 * nout / q * len(offs)
    ms_scan, ms_chan = float(np.median(t_scan)), float(np.median(t_chan))
    return {"channels": len(offs), "capture_s": seconds, "channel_outputs": nout,
            "scan_ms": round(ms_scan, 3), "scan_ms_per_s": round(ms_scan / seconds, 3),
            "channelize_ms": round(ms_chan, 3), "channelize_ms_per_s": round(ms_chan / seconds, 3),
            "scan_int_macs": macs, "scan_tmacs_per_s": round(macs / (ms_scan * 1e-3) / 1e12, 3),
            "scan_runs_ms": [round(t, 3) for t in t_scan], "channelize_runs_ms": [round(t, 3) for t in t_chan]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the scan has no CPU path")
    out = {"card": card_info(),
           "fm": one_band("fm", list(range(-99, 100, 2)), args.seconds, args),
           "am": one_band("am", list(range(-58, 60)), args.seconds, args)}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
