"""The wideband channeliser's rate stage (nrsc5b_chan_create_rate*) on the GPU: captures at 10, 20 and 2.4 MS/s resampled
to the FM plans at D = 16, 32 and 8.

Gates, before any number, at the sizes timed: per capture the handle's head and tail equal the numpy restatement
(tests/chan_oracle_resample.py), the cu8 handle equals the cs16 handle on 64 (cu8 - 127), and pushes of 2^20 bytes give
the one-shot output; three MP1 stations at 10 MS/s (cs16, D = 16) give their generated P1 PDUs through the one-shot
path, and the feed at both push sizes gives that path's records.

Reports, from one run:
  * device time (CUDA events) of nrsc5b_chan_run_device_cs16 on a rate handle over 3 s of signal -> every channel the
    rate allows, and of nrsc5b_chan_resample_device on the same capture - the same k_resample launches alone -, the
    three captures and the two calls alternating, --runs each; k_channelize's time is the difference, and the ratio;
  * k_resample's bytes (input read and planes written from HBM, phase rows read from L2) and int32 MACs from the shapes,
    and the share of each bound (HBM at 3.35 TB/s, the int32 pipes at 132 SMs x 64 lanes x the card's max SM clock);
  * x real time of the feed (page-locked host memory -> nrsc5b_chan_feed_cs16 -> nrsc5b_process after every push) of
    the three stations into a 3-stream FM cs16 engine at 2^20- and 2^23-byte pushes;
  * the card's name, power limit and max SM clock, read in the same run.
Prints one JSON line.  There is no CPU path: without a CUDA device it fails.

    python scripts/wideband_resample.py [--runs 5]
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

HBM_TBS = 3.35                                                  # H100 SXM data sheet, HBM3
CAPTURES = [(10000000, 16), (20000000, 32), (2400000, 8)]       # (fs, D)
SECONDS = 3.0


def card_info():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:                                        # noqa: BLE001
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "max_sm_clock": None, "error": repr(ex)[:200]}


def without_positions(recs):
    from nrsc5_b200 import engine as eng
    return [(t, {k: v for k, v in r.items() if not (t == eng.REC_BLOCK and k == "start")}) for t, r in recs]


def restated(x, offs, G, L, M, taps, ph, D, n0, n):
    """Outputs n0 .. n0 + n - 1 of the handle, restated from the input samples they need."""
    import chan_oracle_rates as rates
    import chan_oracle_resample as rso
    r0, r1 = D * n0, D * (n0 + n - 1) + 256                         # resampled samples
    b0, b1 = (r0 * M) // L, ((r1 - 1) * M) // L + 64                # input samples
    y = rso.resample(x[2 * b0: 2 * b1], G, L, M, n0=r0, nout=r1 - r0, b0=b0)
    return rates.channelize(y, offs, taps, ph, D, n0=n0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5, help="alternating timed runs per capture (one-shot) / push size (feed)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("wideband_resample.py measures on a CUDA device and there is none")
    import test_channelizer_resample as T
    import nrsc5_b200
    from nrsc5_b200 import channelizer as ch, engine as eng, synth
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    card = card_info()
    stream = torch.cuda.default_stream()
    runs = max(3, args.runs)

    # ---- gate 1 per capture, at the timed size; the captures stay resident for the timing
    g = torch.Generator(device=dev)
    setup = {}
    for fs, D in CAPTURES:
        L, M, mo, G = ch.resampler_tables(fs, D)
        offs = list(range(-mo, mo + 1))
        ns = int(SECONDS * fs)
        nout = ch.outputs(2 * ns, decim=D, rate=fs)
        g.manual_seed(D)
        x8 = torch.randint(0, 256, (2 * ns,), dtype=torch.uint8, device=dev, generator=g)
        x16 = ((x8.to(torch.int16) - 127) * 64).contiguous()
        a = torch.zeros((len(offs), 2 * nout), dtype=torch.int16, device=dev)
        b = torch.zeros_like(a)
        c8 = ch.Channelizer(offs, decim=D, rate=fs)
        c16 = ch.Channelizer(offs, input_cs16=True, decim=D, rate=fs)
        taps, ph = c16.tables()
        c8.run_device(x8.data_ptr(), 2 * ns, a.data_ptr(), 2 * nout)
        c16.run_device(x16.data_ptr(), 2 * ns, b.data_ptr(), 2 * nout)
        torch.cuda.synchronize()
        assert torch.equal(a, b), f"{fs} S/s: the cu8 handle differs from the cs16 handle on 64 (cu8 - 127)"
        k = 300
        h16 = x16.cpu().numpy()
        assert np.array_equal(b[:, : 2 * k].cpu().numpy(), restated(h16, offs, G, L, M, taps, ph, D, 0, k)), f"{fs} S/s: head differs"
        assert np.array_equal(b[:, 2 * (nout - k):].cpu().numpy(), restated(h16, offs, G, L, M, taps, ph, D, nout - k, k)), \
            f"{fs} S/s: tail differs"
        piece = (1 << 20) // 2                                     # int16 values per 2^20-byte push
        col = 0
        a.zero_()
        for pos in range(0, 2 * ns, piece):
            col += 2 * c16.push_device(x16.data_ptr() + 2 * pos, min(piece, 2 * ns - pos), a.data_ptr() + 2 * col, 2 * nout)
        torch.cuda.synchronize()
        assert col == 2 * nout and torch.equal(a, b), f"{fs} S/s: streamed differs from one-shot"
        c8.close()
        del x8, b, h16
        setup[fs] = dict(D=D, L=L, M=M, offs=offs, ns=ns, nout=nout, x16=x16, out=a, c=c16)
    torch.cuda.synchronize()

    # ---- device time of the whole handle and of its rate stage alone, captures and calls alternating
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 3

    def fns_of(fs):
        s = setup[fs]
        return {"handle": lambda: s["c"].run_device(s["x16"].data_ptr(), 2 * s["ns"], s["out"].data_ptr(), 2 * s["nout"], stream.cuda_stream),
                "stage": lambda: s["c"].resample_device(s["x16"].data_ptr(), 2 * s["ns"], stream.cuda_stream)}
    fns = {(fs, what): f for fs in setup for what, f in fns_of(fs).items()}
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

    try:
        clock_hz = float(card["max_sm_clock"].split()[0]) * 1e6
    except Exception:                                               # noqa: BLE001
        clock_hz = None
    one_shot = {}
    for fs in setup:
        s = setup[fs]
        ts = times[(fs, "handle")]
        ms = sorted(ts)[len(ts) // 2]
        rs_ts = times[(fs, "stage")]
        K = ch.resampled(s["ns"], fs, s["D"])
        hbm = 4 * s["ns"] + 4 * K                                 # cs16 in, two byte planes out
        l2_rows = 128 * K
        macs = 128 * K
        rs_ms = sorted(rs_ts)[len(rs_ts) // 2]
        chan_ms = ms - rs_ms
        hbm_frac = hbm / (rs_ms * 1e-3) / (HBM_TBS * 1e12) if rs_ms else None
        int_frac = macs / (rs_ms * 1e-3) / (132 * 64 * clock_hz) if rs_ms and clock_hz else None
        one_shot[str(fs)] = {
            "decim": s["D"], "L": s["L"], "M": s["M"], "channels": len(s["offs"]), "samples": s["ns"], "resampled": K,
            "outputs_per_channel": s["nout"], "handle_ms": ms, "handle_ms_runs": ts, "k_resample_ms_runs": rs_ts, "x_realtime": SECONDS / (ms * 1e-3),
            "k_resample_ms": rs_ms, "k_channelize_ms": chan_ms, "resample_over_channelize": rs_ms / chan_ms if chan_ms else None,
            "k_resample_ms_per_s_of_signal": rs_ms / SECONDS,
            "k_resample_hbm_bytes": hbm, "k_resample_l2_table_bytes": l2_rows, "k_resample_int32_macs": macs,
            "k_resample_hbm_frac": hbm_frac, "k_resample_int32_frac": int_frac,
            "k_resample_l2_table_GBps": l2_rows / (rs_ms * 1e-3) / 1e9 if rs_ms else None}
    for s in setup.values():
        s["c"].close()
    setup.clear()
    torch.cuda.empty_cache()

    # ---- gate 2 and the feed: three stations at 10 MS/s into a 3-stream FM cs16 engine
    fs, D = 10000000, 16
    offs, x, caps = T._fm_band(fs, True)
    seconds = (x.size // 2) / fs
    S = len(offs)
    _, ref = T._one_shot_records(x, offs, fs, D, "fm", True)
    ref = [without_positions(r) for r in ref]
    found = []
    for s, cap in enumerate(caps):
        p1 = [r["bits"] for t_, r in ref[s] if t_ == eng.REC_FRAME and r["lc"] == 0]
        assert any(synth.pack_bits(f) in p1 for f in cap.p1_frames), f"station {s}: no generated P1 PDU"
        found.append(len(p1))
    host = torch.from_numpy(x).pin_memory()
    nvalues = x.size
    res = {1 << 20: [], 1 << 23: []}
    with ch.Channelizer(offs, input_cs16=True, decim=D, rate=fs) as c, \
            nrsc5_b200.Engine(nstreams=S, input_capacity=4 * ch.outputs(nvalues, decim=D, rate=fs) + 4096, log_capacity=4 << 20,
                              input_cs16=True) as e:
        for r in range(runs + 1):                                  # run 0 is the gated one (and the warm-up)
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
                    assert got == ref, f"{chunk}-byte pushes: the feed decoded other records than the one-shot path"
                else:
                    res[chunk].append(w)
    feed = {str(chunk): {"pushes": (2 * nvalues + chunk - 1) // chunk, "wall_s": sorted(ws)[len(ws) // 2], "wall_s_runs": ws,
                         "x_realtime": seconds / sorted(ws)[len(ws) // 2]} for chunk, ws in res.items()}
    feed["signal_s"] = seconds
    print(json.dumps({
        "card": card, "one_shot": one_shot,
        "one_shot_what": "CUDA-event device time over %.1f s of signal resident in HBM, median of %d runs of %d calls, "
                         "captures and calls alternating: handle_ms = nrsc5b_chan_run_device_cs16 on a rate handle -> every "
                         "channel the rate allows, k_resample_ms = nrsc5b_chan_resample_device (the same k_resample launches "
                         "alone), k_channelize_ms = the difference; bytes and MACs from the shapes (HBM: 4 B per input sample + 4 B per resampled sample; L2: "
                         "one 128-byte phase row per resampled sample; 128 int32 MACs per resampled sample)" % (SECONDS, runs, reps),
        "feed": feed,
        "feed_what": "page-locked host memory -> nrsc5b_chan_feed_cs16 -> nrsc5b_process after each push, 10 MS/s -> D = 16, "
                     "3-stream FM cs16 engine, wall clock; median of %d runs" % runs,
        "parity_gate": {"ok": True, "head_and_tail_equal_restatement": True, "cu8_equals_cs16_on_device": True,
                        "streamed_equals_one_shot": True, "feed_records_equal_one_shot": True, "p1_pdus_per_station": found}}),
        flush=True)


if __name__ == "__main__":
    main()
