"""The wideband channeliser's AM band plan (nrsc5b_chan_create_am*) on the GPU: one 1 488 375 S/s capture -> the 118
channels of the medium-wave band (10 kHz grid, -58 .. +59) through the 512-tap bank.

Gate, before any number, at the sizes timed: on the device the cs16 kernel on 64 (cu8 - 127) equals the cu8 kernel over
2^24 samples, head and tail of that output equal the numpy restatement (tests/chan_oracle_am.py), the streamed kernel
equals the one-shot one; six synthetic MA1 / MA3 stations 40 dB apart in one cs16 band capture (tests/
test_channelizer_am.py's band) all give generated P1 PDUs through the one-shot channeliser + nrsc5b_push_cs16 path; the
feed into a 118-stream AM engine at both push sizes gives that path's records, stream for stream.

Reports, from one run:
  * one-shot device time of 2^24 samples -> 118 channels, cu8 and cs16 (split pass included), alternating, --runs each;
    the int8 MACs computed from the shapes and the share of the dense int8 tensor peak they amount to;
  * x real time of the feed (page-locked host memory -> nrsc5b_chan_feed_cs16 -> nrsc5b_process after every push) at
    2^15- and 2^20-byte pushes, and how the device time between events recorded around each call on the engine's
    stream divides between the channeliser (the feed) and the receiver (nrsc5b_process: k_am and what follows it);
  * the card's name and power limit, read in the same run.
Prints one JSON line.  There is no CPU path: without a CUDA device it fails.

    python scripts/wideband_am.py [--runs 5]
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
BAND = list(range(-58, 60))                                     # 530 .. 1700 kHz around 1110 kHz
TAPS = 512


def card_info():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as ex:                                        # noqa: BLE001
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "error": repr(ex)[:200]}


def normalised(recs):
    """A stream's records as (L1 records in order, L2 records in order): where a REC_L2 lands among the L1 records, and
    the log offset it carries, depend on how the input was cut into nrsc5b_process calls; nothing else does."""
    from nrsc5_b200 import engine as eng
    l1 = [(t, r) for t, r in recs if t != eng.REC_L2]
    l2 = [{k: v for k, v in r.items() if not k.startswith("frame_")} for t, r in recs if t == eng.REC_L2]
    return l1, l2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5, help="alternating timed runs per format (one-shot) / per push size (feed)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("wideband_am.py measures on a CUDA device and there is none")
    import chan_oracle_am as am
    import test_channelizer_am as T
    from nrsc5_b200 import channelizer as ch, engine as eng
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    card = card_info()
    stream = torch.cuda.default_stream()                         # the engine's stream
    S = len(BAND)
    runs = max(3, args.runs)
    ns = 1 << 24
    nout = ch.outputs(2 * ns, band="am")

    # ---- gate 1: the kernels at the timed size
    g = torch.Generator(device=dev)
    g.manual_seed(3)
    big8 = torch.randint(0, 256, (2 * ns,), dtype=torch.uint8, device=dev, generator=g)
    big16 = ((big8.to(torch.int16) - 127) * 64).contiguous()
    a = torch.zeros((S, 2 * nout), dtype=torch.int16, device=dev)
    b, st = torch.zeros_like(a), torch.zeros_like(a)
    with ch.Channelizer(BAND, band="am") as c8, ch.Channelizer(BAND, input_cs16=True, band="am") as c16:
        taps, ph = c8.tables()
        c8.run_device(big8.data_ptr(), 2 * ns, a.data_ptr(), 2 * nout)
        c16.run_device(big16.data_ptr(), 2 * ns, b.data_ptr(), 2 * nout)
        col = 0
        for pos in range(0, 2 * ns, 3000002):
            col += 2 * c16.push_device(big16.data_ptr() + 2 * pos, min(3000002, 2 * ns - pos), st.data_ptr() + 2 * col, 2 * nout)
        torch.cuda.synchronize()
    assert col == 2 * nout
    assert torch.equal(a, b), "cs16 kernel on 64 (cu8 - 127) differs from the cu8 kernel"
    assert torch.equal(a, st), "streamed cs16 kernel differs from the one-shot kernel"
    h8 = big8.cpu().numpy()
    k = 400
    assert np.array_equal(a[:, : 2 * k].cpu().numpy(), am.channelize(h8[: 2 * (32 * (k - 1) + TAPS)], BAND, taps, ph)), "head differs from the restatement"
    assert np.array_equal(a[:, 2 * (nout - k):].cpu().numpy(), am.channelize(h8[64 * (nout - k):], BAND, taps, ph, n0=nout - k)), \
        "tail differs from the restatement"
    del b, st, h8

    # ---- one-shot device time: 2^24 samples -> 118 channels, cu8 next to cs16, alternating
    g.manual_seed(7)
    big16 = torch.randint(-32768, 32768, (2 * ns,), dtype=torch.int16, device=dev, generator=g)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    times = {"cu8": [], "cs16": []}
    with ch.Channelizer(BAND, band="am") as c8, ch.Channelizer(BAND, input_cs16=True, band="am") as c16:
        fns = {"cu8": lambda: c8.run_device(big8.data_ptr(), 2 * ns, a.data_ptr(), 2 * nout, stream.cuda_stream),
               "cs16": lambda: c16.run_device(big16.data_ptr(), 2 * ns, a.data_ptr(), 2 * nout, stream.cuda_stream)}
        for f in fns.values():
            for _ in range(2):
                f()
        torch.cuda.synchronize()
        for _ in range(runs):
            for name, f in fns.items():
                ev0.record(stream)
                for _ in range(reps):
                    f()
                ev1.record(stream)
                torch.cuda.synchronize()
                times[name].append(ev0.elapsed_time(ev1) / reps)
    groups = (S + 31) // 32
    macs8 = nout * groups * 128 * 2 * TAPS                       # int8 MACs of one cu8 launch (rows of B incl. padding)
    one_shot = {}
    for name, ts in times.items():
        ms = sorted(ts)[len(ts) // 2]
        macs = macs8 * (2 if name == "cs16" else 1)
        one_shot[name] = {"ms": ms, "ms_runs": ts, "int8_macs": macs, "msamples_per_s": ns / (ms * 1e-3) / 1e6,
                          "x_realtime": ns / (ms * 1e-3) / ch.AM_WIDE_RATE, "tensor_tops": 2 * macs / (ms * 1e-3) / 1e12,
                          "int8_peak_frac": 2 * macs / (ms * 1e-3) / 1e12 / H100_INT8_TOPS}
    del big8, big16, a
    torch.cuda.empty_cache()

    # ---- gate 2 and the feed: the band of stations into a 118-stream AM engine
    x, caps = T._band_capture()
    seconds = (x.size // 2) / ch.AM_WIDE_RATE
    with ch.Channelizer(BAND, input_cs16=True, band="am") as c:
        y = c.run(x)
    with T._am_engine(S, 2 * y.shape[1] + 4096) as e:           # the one-shot path: nrsc5b_push_cs16 of every channel, one process
        for s in range(S):
            e.push_cs16(s, y[s])
        e.process()
        ref = [normalised(e.drain(s)) for s in range(S)]
    del y
    found = []
    for (m, _, ma3), cap in zip(T.STATIONS, caps):
        p1 = [r["bits"] for t_, r in ref[BAND.index(m)][0] if t_ == eng.REC_FRAME and r["lc"] == 0]
        gen = {T._pack(bits) for fr in cap.p1_frames.values() for bits in fr}
        assert len(p1) >= 8 and all(f in gen for f in p1), f"station at {m}: P1 PDUs are not the generated ones"
        found.append(len(p1))
    host = torch.from_numpy(x).pin_memory()
    nvalues = x.size
    feed = {}
    with ch.Channelizer(BAND, input_cs16=True, band="am") as c, T._am_engine(S, 4 * ch.outputs(nvalues, band="am") + 4096) as e:
        res = {1 << 15: [], 1 << 20: []}
        for r in range(runs + 1):                                # run 0 is the gated one (and the warm-up)
            for chunk in res:
                vals = chunk // 2
                e.reset()
                c.reset()
                t_feed = t_proc = 0.0
                evs = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for pos in range(0, nvalues, vals):
                    if r:
                        evs[0].record(stream)
                    c.feed(e, (host.data_ptr() + 2 * pos, min(vals, nvalues - pos)))
                    if r:
                        evs[1].record(stream)
                    e.process()
                    if r:
                        evs[2].record(stream)
                        evs[2].synchronize()
                        t_feed += evs[0].elapsed_time(evs[1])
                        t_proc += evs[1].elapsed_time(evs[2])
                torch.cuda.synchronize()
                w = time.perf_counter() - t0
                if r == 0:
                    bad = [s for s in range(S) if normalised(e.drain(s)) != ref[s]]
                    assert not bad, f"{chunk}-byte pushes: streams {bad[:8]} decoded other records than the one-shot path"
                else:
                    e.drain_all_raw()
                    res[chunk].append((w, t_feed, t_proc))
        for chunk, rs in res.items():
            w, tf, tp = sorted(rs)[len(rs) // 2]
            feed[str(chunk)] = {"chunk_bytes": chunk, "pushes": (2 * nvalues + chunk - 1) // chunk, "wall_s": w,
                                "wall_s_runs": [q[0] for q in rs], "x_realtime": seconds / w,
                                "device_ms_channeliser": tf, "device_ms_receiver": tp,
                                "channeliser_share_of_device_time": tf / (tf + tp)}
    print(json.dumps({
        "value": one_shot["cs16"]["x_realtime"], "unit": "x real time (cs16 one-shot, 2^24 samples -> 118 channels)",
        "card": card, "one_shot": one_shot,
        "one_shot_what": "device time of nrsc5b_chan_run_device(_cs16) on an AM-plan handle over 2^24 complex samples resident "
                         "in HBM -> 118 channels, median of %d alternating runs of %d launches each; cs16 includes its split pass; "
                         "MACs = outputs x 4 groups x 128 rows x 1024 (x 2 planes for cs16); peak share against %.0f TOP/s "
                         "(H100 SXM data sheet, dense INT8 at 700 W)" % (runs, reps, H100_INT8_TOPS),
        "feed": feed,
        "feed_what": "page-locked host memory -> nrsc5b_chan_feed_cs16 -> nrsc5b_process after each push, 118-stream AM cs16 "
                     "engine with L2 on; x real time of %.3f s of signal, median of %d runs; device_ms_*: time between events "
                     "recorded on the engine's stream around the feed and around nrsc5b_process, summed over the pushes" % (seconds, runs),
        "parity_gate": {"ok": True, "cs16_equals_cu8_on_device": True, "streamed_equals_one_shot": True,
                        "head_and_tail_equal_restatement": True, "feed_records_equal_one_shot": True,
                        "p1_pdus_per_station": found},
        "workload": "6 synthetic MA1 / MA3 stations at offsets %s x 10 kHz, levels %s dB, in one 1 488 375 S/s cs16 capture with a "
                    "3 LSB noise floor; 118 channels -58 .. +59" % ([m for m, _, _ in T.STATIONS], [d for _, d, _ in T.STATIONS])}), flush=True)


if __name__ == "__main__":
    main()
