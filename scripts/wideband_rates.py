"""The wideband channeliser's FM plans at 23.814, 11.907 and 5.9535 MS/s (D = 32, 16, 8: nrsc5b_chan_create_fm*) on the
GPU, side by side.

Gate, before any number, at the sizes timed: per D the cu8 kernel's head and tail over the timed capture equal the numpy
restatement (tests/chan_oracle_rates.py), the cs16 kernel on 64 (cu8 - 127) equals the cu8 kernel; per D three synthetic
stations (tests/test_channelizer_rates.py's band, interpolated by D / 2) give generated P1 PDUs through the one-shot
path, and the feed at both push sizes gives that path's records, stream for stream.

Reports, from one run, per D:
  * one-shot device time of about 3 s of signal -> every channel of the plan's range (D = 32: +-118, 237 channels;
    16: +-59, 119; 8: +-29, 59), cu8 and cs16 (split pass included), the D alternating, --runs each; the int8 MACs
    computed from the shapes, their share of the dense int8 tensor peak, and channel outputs per second;
  * x real time of the feed (page-locked host memory -> nrsc5b_chan_feed_cs16 -> nrsc5b_process after every push) of
    the three stations into a 3-stream FM cs16 engine at 2^20- and 2^23-byte pushes;
  * the card's name and power limit, read in the same run.
Prints one JSON line.  There is no CPU path: without a CUDA device it fails.

    python scripts/wideband_rates.py [--runs 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")]

H100_INT8_TOPS = 1979.0                                         # H100 SXM data sheet, dense INT8 at 700 W
DS = (32, 16, 8)
RANGE = {32: 118, 16: 59, 8: 29}
SECONDS = 3.0


def card_info():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as ex:                                        # noqa: BLE001
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "error": repr(ex)[:200]}


def without_positions(recs):
    from nrsc5_b200 import engine as eng
    return [(t, {k: v for k, v in r.items() if not (t == eng.REC_BLOCK and k == "start")}) for t, r in recs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5, help="alternating timed runs per D and format (one-shot) / push size (feed)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("wideband_rates.py measures on a CUDA device and there is none")
    import chan_oracle_rates as rates
    import test_channelizer_rates as T
    import nrsc5_b200
    from nrsc5_b200 import channelizer as ch, engine as eng, synth
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    card = card_info()
    stream = torch.cuda.default_stream()
    runs = max(3, args.runs)

    # ---- gate 1 per D, at the timed size; the captures stay resident for the timing
    g = torch.Generator(device=dev)
    setup = {}
    for D in DS:
        offs = list(range(-RANGE[D], RANGE[D] + 1))
        ns = (int(SECONDS * ch.wide_rate(D)) // 32) * 32
        nout = ch.outputs(2 * ns, decim=D)
        g.manual_seed(D)
        x8 = torch.randint(0, 256, (2 * ns,), dtype=torch.uint8, device=dev, generator=g)
        x16 = ((x8.to(torch.int16) - 127) * 64).contiguous()
        a = torch.zeros((len(offs), 2 * nout), dtype=torch.int16, device=dev)
        b = torch.zeros_like(a)
        c8, c16 = ch.Channelizer(offs, decim=D), ch.Channelizer(offs, input_cs16=True, decim=D)
        taps, ph = c8.tables()
        c8.run_device(x8.data_ptr(), 2 * ns, a.data_ptr(), 2 * nout)
        c16.run_device(x16.data_ptr(), 2 * ns, b.data_ptr(), 2 * nout)
        torch.cuda.synchronize()
        assert torch.equal(a, b), f"D = {D}: cs16 kernel on 64 (cu8 - 127) differs from the cu8 kernel"
        k = 300
        head = x8[: 2 * (D * (k - 1) + 256)].cpu().numpy()
        tail = x8[2 * D * (nout - k):].cpu().numpy()
        assert np.array_equal(a[:, : 2 * k].cpu().numpy(), rates.channelize(head, offs, taps, ph, D)), f"D = {D}: head differs"
        assert np.array_equal(a[:, 2 * (nout - k):].cpu().numpy(), rates.channelize(tail, offs, taps, ph, D, n0=nout - k)), \
            f"D = {D}: tail differs"
        del b
        setup[D] = dict(offs=offs, ns=ns, nout=nout, x8=x8, x16=x16, out=a, c8=c8, c16=c16)
    torch.cuda.synchronize()

    # ---- one-shot device time, the D and formats alternating
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 5

    def fn(D, fmt):
        s = setup[D]
        c, x = (s["c8"], s["x8"]) if fmt == "cu8" else (s["c16"], s["x16"])
        return lambda: c.run_device(x.data_ptr(), 2 * s["ns"], s["out"].data_ptr(), 2 * s["nout"], stream.cuda_stream)
    fns = {(D, fmt): fn(D, fmt) for D in DS for fmt in ("cu8", "cs16")}
    for f in fns.values():
        f()
        f()
    torch.cuda.synchronize()
    times = {key: [] for key in fns}
    for _ in range(runs):
        for key, f in fns.items():
            ev0.record(stream)
            for _ in range(reps):
                f()
            ev1.record(stream)
            torch.cuda.synchronize()
            times[key].append(ev0.elapsed_time(ev1) / reps)
    one_shot = {}
    for (D, fmt), ts in times.items():
        s = setup[D]
        ms = sorted(ts)[len(ts) // 2]
        groups = (len(s["offs"]) + 31) // 32
        macs = s["nout"] * groups * 128 * 512 * (2 if fmt == "cs16" else 1)
        one_shot.setdefault(str(D), {})[fmt] = {
            "ms": ms, "ms_runs": ts, "channels": len(s["offs"]), "samples": s["ns"], "outputs_per_channel": s["nout"],
            "x_realtime": s["ns"] / (ms * 1e-3) / ch.wide_rate(D),
            "channel_outputs_per_s": s["nout"] * len(s["offs"]) / (ms * 1e-3),
            "int8_macs": macs, "tensor_tops": 2 * macs / (ms * 1e-3) / 1e12,
            "int8_peak_frac": 2 * macs / (ms * 1e-3) / 1e12 / H100_INT8_TOPS}
    for s in setup.values():
        s["c8"].close()
        s["c16"].close()
    setup.clear()
    torch.cuda.empty_cache()

    # ---- gate 2 and the feed: three stations per D into a 3-stream FM cs16 engine
    feed, found = {}, {}
    for D in DS:
        offs = [m for m, _, _, _ in T.STATIONS[D]]
        S = len(offs)
        x, caps = T._band_capture(D)
        seconds = (x.size // 2) / ch.wide_rate(D)
        with ch.Channelizer(offs, input_cs16=True, decim=D) as c:
            y = c.run(x)
        with nrsc5_b200.Engine(nstreams=S, input_capacity=2 * y.shape[1] + 4096, log_capacity=4 << 20, input_cs16=True) as e:
            for s in range(S):
                e.push_cs16(s, y[s])
            e.process()
            ref = [without_positions(e.drain(s)) for s in range(S)]
        found[str(D)] = []
        for s, cap in enumerate(caps):
            p1 = [r["bits"] for t_, r in ref[s] if t_ == eng.REC_FRAME and r["lc"] == 0]
            assert any(synth.pack_bits(f) in p1 for f in cap.p1_frames), f"D = {D}, station {s}: no generated P1 PDU"
            found[str(D)].append(len(p1))
        host = torch.from_numpy(x).pin_memory()
        nvalues = x.size
        res = {1 << 20: [], 1 << 23: []}
        with ch.Channelizer(offs, input_cs16=True, decim=D) as c, \
                nrsc5_b200.Engine(nstreams=S, input_capacity=4 * ch.outputs(nvalues, decim=D) + 4096, log_capacity=4 << 20,
                                  input_cs16=True) as e:
            for r in range(runs + 1):                            # run 0 is the gated one (and the warm-up)
                for chunk in res:
                    vals = chunk // 2
                    e.reset()
                    c.reset()
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for pos in range(0, nvalues, vals):
                        c.feed(e, (host.data_ptr() + 2 * pos, min(vals, nvalues - pos)))
                        e.process()
                    torch.cuda.synchronize()
                    w = time.perf_counter() - t0
                    got = [without_positions(e.drain(s)) for s in range(S)]
                    if r == 0:
                        assert got == ref, f"D = {D}, {chunk}-byte pushes: the feed decoded other records than the one-shot path"
                    else:
                        res[chunk].append(w)
        feed[str(D)] = {str(chunk): {"pushes": (2 * nvalues + chunk - 1) // chunk, "wall_s": sorted(ws)[len(ws) // 2],
                                     "wall_s_runs": ws, "x_realtime": seconds / sorted(ws)[len(ws) // 2]}
                        for chunk, ws in res.items()}
        feed[str(D)]["signal_s"] = seconds
        del host, x, y
    print(json.dumps({
        "card": card, "one_shot": one_shot,
        "one_shot_what": "device time of nrsc5b_chan_run_device(_cs16) over %.1f s of signal resident in HBM -> every channel "
                         "of the plan's range, median of %d runs of %d launches each, D and formats alternating; cs16 includes "
                         "its split pass; MACs = outputs x groups x 128 rows x 512 (x 2 planes for cs16); peak share against "
                         "%.0f TOP/s (H100 SXM data sheet, dense INT8 at 700 W)" % (SECONDS, runs, reps, H100_INT8_TOPS),
        "feed": feed,
        "feed_what": "page-locked host memory -> nrsc5b_chan_feed_cs16 -> nrsc5b_process after each push, 3-stream FM cs16 "
                     "engine, wall clock; median of %d runs" % runs,
        "parity_gate": {"ok": True, "head_and_tail_equal_restatement": True, "cs16_equals_cu8_on_device": True,
                        "feed_records_equal_one_shot": True, "p1_pdus_per_station": found},
        "workload": "MP1 stations at %s x 100 kHz, amplitudes %s, interpolated by D / 2 into one cs16 capture per D with a "
                    "2 LSB noise floor" % ([m for m, _, _, _ in T.STATIONS[8]], [s for _, s, _, _ in T.STATIONS[8]])}), flush=True)


if __name__ == "__main__":
    main()
