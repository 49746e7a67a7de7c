"""The wideband channeliser on cs16 input (nrsc5b_chan_*_cs16) on the GPU: what the 16-bit path costs and what it buys.

Gate, before any number: on the device the cs16 kernel on 64 (cu8 - 127) equals the cu8 kernel on cu8 (one-shot and
streamed); three synthetic MP1 stations 48 dB / 24 dB apart in one 23.814 MS/s cs16 capture (100 channels of
range(-99, 100, 2), the others noise only) all give their generated P1 PDUs through the one-shot channeliser + engine
path; the streamed feed into a 100-stream engine gives that path's records, stream for stream.

Reports, from one run:
  * one-shot device time of a 2^26-sample capture into 100 channels, cs16 (split pass included) next to cu8 on the same
    number of samples, alternating, --runs each; Gsamples/s and the share of the dense int8 tensor peak computed from
    the shapes (the cs16 path issues twice the cu8 kernel's MACs);
  * x real time of the streamed feed (page-locked host memory -> nrsc5b_chan_feed_cs16 -> nrsc5b_process after each
    push) at 2^20- and 2^23-byte pushes;
  * the MER the engine reports for the weakest station from the cs16 capture and from the same band quantised to cu8
    (reported, not gated);
  * the card's name and power limit, read in the same run.
Prints one JSON line.

    python scripts/wideband_cs16.py [--runs 5]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H100_INT8_TOPS = 1979.0                                         # H100 SXM data sheet, dense INT8 at 700 W
OFFS = list(range(-99, 100, 2))                                 # 100 channels, 200 kHz apart
STATIONS = [(11, 250.0), (-23, 1.0), (39, 16.0)]                # (channel offset, scale of (cu8 - 127)): 0, -48, -24 dB
WEAK = 1


def card_info():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as ex:                                        # noqa: BLE001
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "error": repr(ex)[:200]}


def make_band(frames, dev):
    """The stations (kept for their P1 frames) and the band as float I/Q [N][2] on the device (int16 scale)."""
    import torch
    from nrsc5_b200 import channelizer as ch, synth
    caps = [synth.make_fm_mp1(nframes=frames, seed=90 + i, lead_in=700 * i + 40, tail_blocks=2) for i in range(len(STATIONS))]
    n = min(c.cu8.size for c in caps) // 2
    up = 16
    N = n * up
    wide = torch.zeros(N, dtype=torch.complex64, device=dev)
    t = torch.arange(N, dtype=torch.float64, device=dev)
    for c, (m, s) in zip(caps, STATIONS):
        xi = torch.from_numpy(c.cu8[: 2 * n].astype(np.float32) - 127.0).to(dev).view(-1, 2)
        X = torch.fft.fft(torch.complex(xi[:, 0].contiguous(), xi[:, 1].contiguous()))
        Y = torch.zeros(N, dtype=torch.complex64, device=dev)   # band-limited interpolation by 16
        Y[: n // 2] = X[: n // 2]
        Y[-(n - n // 2):] = X[n // 2:]
        y = torch.fft.ifft(Y) * (up * s)
        ph = torch.remainder(t * (m * 100e3 / ch.WIDE_RATE), 1.0) * (2 * math.pi)
        wide += y * torch.complex(torch.cos(ph).float(), torch.sin(ph).float())
        del X, Y, y, ph
    del t
    g = torch.Generator(device=dev)
    g.manual_seed(12)
    iq = torch.stack([wide.real, wide.imag], -1) + torch.randn((N, 2), generator=g, device=dev) * 2.0
    N &= ~31
    return caps, iq[:N].contiguous()


def one_shot_records(c, cap, nvalues, dev):
    """The one-shot path: the whole capture -> [100][stride] -> an engine attached to it, one process."""
    import torch
    import nrsc5_b200
    from nrsc5_b200 import channelizer as ch
    nout = ch.outputs(nvalues)
    stride = (2 * nout + 64) & ~31
    out = torch.zeros((len(OFFS), stride), dtype=torch.int16, device=dev)
    c.run_device(cap.data_ptr(), nvalues, out.data_ptr(), stride)
    torch.cuda.synchronize()
    with nrsc5_b200.Engine(nstreams=len(OFFS), input_capacity=4096, log_capacity=1 << 20, input_cs16=True) as e:
        e.attach_device_input(out.data_ptr(), 2 * stride, 4 * nout)
        e.process()
        recs = e.drain_all()
    del out
    return recs


def mer(recs):
    from nrsc5_b200 import engine as eng
    m = [(r["lower"] + r["upper"]) / 2 for t_, r in recs if t_ == eng.REC_MER]
    return {"mean_db": float(np.mean(m)) if m else None, "reports": len(m)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5, help="alternating timed runs per format (one-shot) / per chunk size (feed)")
    ap.add_argument("--frames", type=int, default=2, help="L1 frames per station")
    args = ap.parse_args()
    import torch
    import nrsc5_b200
    from nrsc5_b200 import channelizer as ch, synth
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    card = card_info()
    stream = torch.cuda.current_stream()
    S = len(OFFS)
    runs = max(3, args.runs)

    # ---- gate 1: identity with cu8 on the device, one-shot and streamed
    g = torch.Generator(device=dev)
    g.manual_seed(3)
    cu8 = torch.randint(0, 256, (64 * 40000,), dtype=torch.uint8, device=dev, generator=g)
    x16 = ((cu8.to(torch.int16) - 127) * 64).contiguous()
    nout = ch.outputs(cu8.numel())
    a = torch.zeros((S, 2 * nout), dtype=torch.int16, device=dev)
    b, s16 = torch.zeros_like(a), torch.zeros_like(a)
    with ch.Channelizer(OFFS) as c8, ch.Channelizer(OFFS, input_cs16=True) as c16:
        c8.run_device(cu8.data_ptr(), cu8.numel(), a.data_ptr(), 2 * nout)
        c16.run_device(x16.data_ptr(), x16.numel(), b.data_ptr(), 2 * nout)
        col = 0
        for pos in range(0, x16.numel(), 300002):
            col += 2 * c16.push_device(x16.data_ptr() + 2 * pos, min(300002, x16.numel() - pos), s16.data_ptr() + 2 * col, 2 * nout)
        torch.cuda.synchronize()
    assert torch.equal(a, b), "cs16 kernel on 64 (cu8 - 127) differs from the cu8 kernel"
    assert torch.equal(a, s16), "streamed cs16 kernel on 64 (cu8 - 127) differs from the cu8 kernel"
    del cu8, x16, a, b, s16

    # ---- gate 2: the stations decode from the one-shot path; the feed equals it
    caps, iq = make_band(args.frames, dev)
    cap = torch.clamp(torch.round(iq), -32768, 32767).to(torch.int16).reshape(-1)
    cap8 = torch.clamp(torch.round(iq / 256.0) + 127.0, 0, 255).to(torch.uint8).reshape(-1)   # the same band in 8 bits
    del iq
    nvalues = cap.numel()
    seconds = (nvalues // 2) / ch.WIDE_RATE
    idx = [OFFS.index(m) for m, _ in STATIONS]
    with ch.Channelizer(OFFS, input_cs16=True) as c:
        ref = one_shot_records(c, cap, nvalues, dev)
    with ch.Channelizer(OFFS) as c8:
        ref8 = one_shot_records(c8, cap8, cap8.numel(), dev)
    del cap8
    found = []
    for i, k in enumerate(idx):
        p1 = [r["bits"] for t_, r in ref[k] if t_ == 1 and r["lc"] == 0]
        found.append(sum(1 for f in caps[i].p1_frames if synth.pack_bits(f) in p1))
        assert found[-1] >= 1, f"station {i} (channel {OFFS[k]}): none of its generated P1 frames came out"
    host = torch.empty(nvalues, dtype=torch.int16).pin_memory()
    host.copy_(cap)
    nout = ch.outputs(nvalues)
    feed = {}
    with ch.Channelizer(OFFS, input_cs16=True) as c, \
            nrsc5_b200.Engine(nstreams=S, input_capacity=4 * nout + 4096, log_capacity=1 << 20, input_cs16=True) as e:
        walls = {1 << 20: [], 1 << 23: []}
        for r in range(runs + 1):                                # run 0 is the gated one (and the warm-up)
            for chunk in walls:
                vals = chunk // 2
                e.reset()
                c.reset()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for pos in range(0, nvalues, vals):
                    c.feed(e, (host.data_ptr() + 2 * pos, min(vals, nvalues - pos)))
                    e.process()
                recs = e.drain_all()
                torch.cuda.synchronize()
                w = time.perf_counter() - t0
                if r == 0:
                    bad = [s for s in range(S) if recs[s] != ref[s]]
                    assert not bad, f"{chunk}-byte pushes: streams {bad[:8]} decoded other records than the one-shot path"
                else:
                    walls[chunk].append(w)
        for chunk, ws in walls.items():
            w = sorted(ws)[len(ws) // 2]
            feed[str(chunk)] = {"chunk_bytes": chunk, "pushes": (2 * nvalues + chunk - 1) // chunk, "wall_s": w, "wall_s_runs": ws,
                                "x_realtime": seconds / w}
    del host, cap
    torch.cuda.empty_cache()

    # ---- one-shot device time: 2^26 samples -> 100 channels, cs16 next to cu8, alternating
    ns = 1 << 26
    g.manual_seed(7)
    big16 = torch.randint(-32768, 32768, (2 * ns,), dtype=torch.int16, device=dev, generator=g)
    big8 = torch.randint(0, 256, (2 * ns,), dtype=torch.uint8, device=dev, generator=g)
    nout = ch.outputs(2 * ns)
    out = torch.zeros((S, 2 * nout), dtype=torch.int16, device=dev)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 5
    times = {"cs16": [], "cu8": []}
    with ch.Channelizer(OFFS) as c8, ch.Channelizer(OFFS, input_cs16=True) as c16:
        fns = {"cs16": lambda: c16.run_device(big16.data_ptr(), 2 * ns, out.data_ptr(), 2 * nout, stream.cuda_stream),
               "cu8": lambda: c8.run_device(big8.data_ptr(), 2 * ns, out.data_ptr(), 2 * nout, stream.cuda_stream)}
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
    macs8 = nout * groups * 128 * 512                            # int8 MACs of one cu8 launch (rows of B incl. padding)
    one_shot = {}
    for name, ts in times.items():
        ms = sorted(ts)[len(ts) // 2]
        macs = macs8 * (2 if name == "cs16" else 1)
        one_shot[name] = {"ms": ms, "ms_runs": ts, "gsamples_per_s": ns / (ms * 1e-3) / 1e9,
                          "x_realtime": ns / (ms * 1e-3) / ch.WIDE_RATE,
                          "tensor_tops": 2 * macs / (ms * 1e-3) / 1e12,
                          "int8_peak_frac": 2 * macs / (ms * 1e-3) / 1e12 / H100_INT8_TOPS}
    one_shot["cs16_over_cu8_rate"] = one_shot["cs16"]["gsamples_per_s"] / one_shot["cu8"]["gsamples_per_s"]
    weak = idx[WEAK]
    print(json.dumps({
        "value": one_shot["cs16"]["gsamples_per_s"], "unit": "Gsamples/s (cs16 one-shot, 2^26 samples -> 100 channels)",
        "card": card, "one_shot": one_shot,
        "one_shot_what": "device time of nrsc5b_chan_run_device(_cs16) over 2^26 complex samples resident in HBM -> 100 "
                         "channels, median of %d alternating runs of %d launches each; cs16 includes its split pass; peak "
                         "share against %.0f TOP/s (H100 SXM data sheet, dense INT8 at 700 W)" % (runs, reps, H100_INT8_TOPS),
        "feed": feed, "feed_what": "page-locked host memory -> nrsc5b_chan_feed_cs16 -> nrsc5b_process after each push, "
                                   "100-stream cs16 engine; x real time of %.3f s of signal, median of %d runs" % (seconds, runs),
        "weak_station_mer": {"channel_offset_100khz": OFFS[weak], "below_strongest_db": 20 * math.log10(STATIONS[0][1] / STATIONS[WEAK][1]),
                             "cs16": mer(ref[weak]), "cu8_quantised": mer(ref8[weak]),
                             "cu8_p1_frames": len([1 for t_, r in ref8[weak] if t_ == 1 and r["lc"] == 0])},
        "parity_gate": {"ok": True, "identity_with_cu8_on_device": True, "feed_records_equal_one_shot": True,
                        "generated_p1_frames_found": found, "generated_p1_frames_per_station": args.frames},
        "workload": "3 synthetic MP1 stations (scales %s of (cu8 - 127)) x16 band-limited into one 23.814 MS/s cs16 capture "
                    "with noise, 100 channels range(-99, 100, 2)" % [s for _, s in STATIONS]}), flush=True)


if __name__ == "__main__":
    main()
