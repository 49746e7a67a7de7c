"""Streaming wideband ingest on the GPU (nrsc5b_chan_feed): a live 23.814 MS/s capture arriving in pieces, channelised
straight into a running 100-stream cs16 engine.

The capture: 16 synthetic MP1 stations made like bench.py's headline captures, interpolated by 16 (band-limited, torch
FFT on the GPU), mixed to 16 of the 100 channels of range(-99, 100, 2) and summed with noise into cu8; the other 84
channels carry only noise.  It is pushed from page-locked host memory in chunks of 2^20 and 2^23 bytes, with an
nrsc5b_process after each.

Gate, before any number: every stream's records equal the one-shot path's (nrsc5b_chan_run_device on the whole
capture, the engine attached to its output, one nrsc5b_process) byte for byte; every station's P1 PDUs include a
generated frame; the channeliser alone, streamed device to device, equals its one-shot output (torch.equal on the device).

Reports x real time of the whole streamed pipeline per chunk size, the streamed channeliser's device time next to the
one-shot kernel's on the same capture, and the card's name and power limit, read in the same run.  Prints one JSON line.

    python scripts/wideband_stream.py [--reps 3]
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


def card_info():
    """The card's name and power limit, read now (they are part of every number this run reports)."""
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as ex:                                        # noqa: BLE001
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "error": repr(ex)[:200]}


def make_capture(offs, st_idx, frames, dev):
    """The stations (kept whole for their P1 frames) and the wideband capture on the device (uint8, a multiple of 64)."""
    import torch
    from nrsc5_b200 import channelizer as ch, synth
    caps = []
    for i in range(len(st_idx)):                                # the headline's station variants (bench.py make_captures)
        kw = dict(nframes=frames, seed=1234 + i, lead_in=0, tail_blocks=2, noise_seed=5 + i)
        if i % 4 == 1:
            kw.update(cfo_hz=120.0)
        elif i % 4 == 2:
            kw.update(cfo_hz=-300.0, noise_lsb=12.0)
        elif i % 4 == 3:
            kw.update(cfo_hz=60.0, noise_lsb=6.0)
        caps.append(synth.make_fm_mp1(**kw))
    n = min(c.cu8.size for c in caps) // 2
    up = 16
    N = n * up
    wide = torch.zeros(N, dtype=torch.complex64, device=dev)
    t = torch.arange(N, dtype=torch.float64, device=dev)
    for c, k in zip(caps, st_idx):
        xi = torch.from_numpy(c.cu8[: 2 * n].astype(np.float32) - 127.0).to(dev).view(-1, 2)
        X = torch.fft.fft(torch.complex(xi[:, 0].contiguous(), xi[:, 1].contiguous()))
        Y = torch.zeros(N, dtype=torch.complex64, device=dev)   # band-limited interpolation by 16
        Y[: n // 2] = X[: n // 2]
        Y[-(n - n // 2):] = X[n // 2:]
        y = torch.fft.ifft(Y) * (up * 0.25)                     # a quarter of the amplitude: 16 stations sum within 8 bits
        ph = torch.remainder(t * (offs[k] * 100e3 / ch.WIDE_RATE), 1.0) * (2 * math.pi)
        wide += y * torch.complex(torch.cos(ph).float(), torch.sin(ph).float())
        del X, Y, y, ph
    del t
    g = torch.Generator(device=dev)
    g.manual_seed(11)
    noise = torch.randn((N, 2), generator=g, device=dev) * 2.0
    cap = torch.clamp(torch.round(torch.stack([wide.real, wide.imag], -1) + noise + 127.0), 0, 255).to(torch.uint8).reshape(-1)
    del wide, noise
    nbytes = cap.numel() & ~63
    return caps, cap[:nbytes].contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="timed runs per measurement (after a gated first run)")
    args = ap.parse_args()
    import torch
    import nrsc5_b200
    from nrsc5_b200 import channelizer as ch, synth
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    card = card_info()
    offs = list(range(-99, 100, 2))                             # 100 channels, 200 kHz apart
    nst, frames = 16, 2
    st_idx = [3 + 6 * i for i in range(nst)]                    # stations 1.2 MHz apart, the channels between them noise only
    caps, cap = make_capture(offs, st_idx, frames, dev)
    nbytes = cap.numel()
    host = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    host.copy_(cap)
    nout = ch.outputs(nbytes)
    stride = (2 * nout + 64) & ~31                              # int16 values between channels: 64-byte aligned rows for the engine
    seconds = (nbytes // 2) / ch.WIDE_RATE
    stream = torch.cuda.current_stream()
    S = len(offs)
    reps = max(1, args.reps)
    sizes = [1 << 20, 1 << 23]
    with ch.Channelizer(offs) as c:
        # ---- the one-shot path: the whole capture resident in HBM -> [100][stride] -> an engine attached to it
        one = torch.zeros((S, stride), dtype=torch.int16, device=dev)
        c.run_device(cap.data_ptr(), nbytes, one.data_ptr(), stride, stream.cuda_stream)
        torch.cuda.synchronize()
        with nrsc5_b200.Engine(nstreams=S, input_capacity=4096, log_capacity=1 << 20, input_cs16=True) as e:
            e.attach_device_input(one.data_ptr(), 2 * stride, 4 * nout)
            e.process()
            ref = e.drain_all()
        # ---- the channeliser alone, streamed device to device, against its one-shot output
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def timed_dev(fn):
            fn()
            torch.cuda.synchronize()
            ev0.record(stream)
            for _ in range(reps):
                fn()
            ev1.record(stream)
            torch.cuda.synchronize()
            return ev0.elapsed_time(ev1) / reps

        one_ms = timed_dev(lambda: c.run_device(cap.data_ptr(), nbytes, one.data_ptr(), stride, stream.cuda_stream))
        streamed = torch.zeros_like(one)
        chan_ms = {}

        def push_all(chunk):
            c.reset()
            col = 0
            for pos in range(0, nbytes, chunk):
                col += 2 * c.push_device(cap.data_ptr() + pos, min(chunk, nbytes - pos), streamed.data_ptr() + 2 * col, stride,
                                         stream.cuda_stream)
            assert col == 2 * nout

        for chunk in sizes:
            streamed.zero_()
            push_all(chunk)
            torch.cuda.synchronize()
            assert torch.equal(streamed[:, : 2 * nout], one[:, : 2 * nout]), \
                f"streamed channeliser output ({chunk}-byte pushes) differs from the one-shot output"
            chan_ms[str(chunk)] = timed_dev(lambda: push_all(chunk))
        del one, streamed
        torch.cuda.empty_cache()
        # ---- the whole streamed pipeline: page-locked chunks -> nrsc5b_chan_feed -> nrsc5b_process after each
        pipe = {}
        with nrsc5_b200.Engine(nstreams=S, input_capacity=4 * nout + 4096, log_capacity=1 << 20, input_cs16=True) as e:
            for chunk in sizes:
                walls = []
                for r in range(reps + 1):                       # the first run is the gated one (and the warm-up)
                    e.reset()
                    c.reset()
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for pos in range(0, nbytes, chunk):
                        c.feed(e, (host.data_ptr() + pos, min(chunk, nbytes - pos)))
                        e.process()
                    recs = e.drain_all()
                    torch.cuda.synchronize()
                    walls.append(time.perf_counter() - t0)
                    if r == 0:
                        bad = [s for s in range(S) if recs[s] != ref[s]]
                        assert not bad, f"{chunk}-byte pushes: streams {bad[:8]} decoded other records than the one-shot path"
                w = sorted(walls[1:])[len(walls[1:]) // 2]
                pipe[str(chunk)] = {"chunk_bytes": chunk, "chunk_ms_of_signal": chunk / 2 / ch.WIDE_RATE * 1e3,
                                    "pushes": (nbytes + chunk - 1) // chunk, "wall_s": w, "wall_s_runs": walls[1:],
                                    "x_realtime": seconds / w}
    found = []
    for i, k in enumerate(st_idx):
        p1 = [r["bits"] for t_, r in ref[k] if t_ == 1 and r["lc"] == 0]
        found.append(sum(1 for f in caps[i].p1_frames if synth.pack_bits(f) in p1))
        assert found[-1] >= 1, f"station {i} (channel {offs[k]}): none of its generated P1 frames came out"
    print(json.dumps({
        "value": pipe[str(1 << 23)]["x_realtime"], "unit": "x real time (2^23-byte pushes, 100 channels, whole pipeline)",
        "card": card, "channels": S, "stations": nst, "capture_bytes": int(nbytes), "capture_seconds": seconds,
        "outputs_per_channel": int(nout), "pipeline": pipe,
        "channeliser_device_ms": {"one_shot": one_ms, "streamed": chan_ms,
                                  "what": "device time over the whole capture: one k_channelize launch vs pushes of that many "
                                          "bytes from device memory (staging, carry and per-push launches)"},
        "parity_gate": {"ok": True, "records_equal_one_shot": True, "channeliser_equal_one_shot": True,
                        "generated_p1_frames_found": found, "generated_p1_frames_per_station": frames},
        "workload": "16 synthetic MP1 stations x16 band-limited into one 23.814 MS/s cu8 capture with noise, 100 channels "
                    "range(-99, 100, 2), pushed from page-locked host memory into one 100-stream cs16 engine"}), flush=True)


if __name__ == "__main__":
    main()
