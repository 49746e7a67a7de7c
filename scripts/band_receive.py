"""The band receiver (nrsc5b_band_*) on the GPU: a wideband capture in pieces -> every HD Radio station in it decoded.
Prints the sessions it opened, seconds of capture per second of wall time, the device time per stage (channelise, scan,
route, engines; CUDA events inside the handle) and k_band_route's achieved bytes/s (bytes read and written over its
device time).  The card's name and power limit are read in the same run.

Without a file: a synthetic FM band at D = 32 (23.814 MS/s cs16), every 100 kHz grid point (235 channels), with a few
MP1 / MP3 / MP11 stations, a carrier and noise; a short warm-up receiver runs first.  With a file: a raw cu8 or cs16
capture at --rate Hz (default: the plan's own rate).  Prints one JSON line (and writes it to --out).  There is no CPU
path: without a CUDA device it fails.

    python scripts/band_receive.py [--seconds 6] [--piece 4194304] [--out result.json]
    python scripts/band_receive.py capture.cs16 --format cs16 --band fm --decim 16 --rate 10000000
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

STATIONS = [(-83, 1, 1.0, 11), (-41, 3, 0.3, 12), (7, 11, 0.5, 13), (52, 1, 0.1, 14), (96, 1, 0.8, 15)]   # offset, psmi, gain, seed


def card_info():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as ex:                                        # noqa: BLE001
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "error": repr(ex)[:200]}


def synthetic_band(seconds):
    """STATIONS at 23.814 MS/s cs16: each 1 488 375 S/s station interpolated by 16 in the frequency domain and moved to
    its offset, with a carrier and a white noise floor."""
    import torch
    from nrsc5_b200 import synth
    fs = 23814000.0
    n = int(seconds * 1488375)
    N = 16 * n
    t = torch.arange(N, dtype=torch.float64, device="cuda")
    wide = torch.zeros(N, dtype=torch.complex64, device="cuda")
    nframes = int(math.ceil(seconds / 1.486)) + 1
    for m, psmi, gain, seed in STATIONS:
        cap = synth.make_fm(psmi=psmi, nframes=nframes, seed=seed, lead_in=500 + 97 * seed, tail_blocks=0)
        x = torch.from_numpy(cap.cu8[: 2 * n].astype(np.float32) - 127.0).cuda().view(-1, 2)
        X = torch.fft.fft(torch.complex(x[:, 0].contiguous(), x[:, 1].contiguous()))
        Y = torch.zeros(N, dtype=torch.complex64, device="cuda")
        Y[: n // 2] = X[: n // 2]
        Y[-(n - n // 2):] = X[n // 2:]
        ph = torch.remainder(t * (m * 100e3 / fs), 1.0) * (2 * math.pi)
        wide += torch.fft.ifft(Y) * (16 * 40.0 * gain) * torch.complex(torch.cos(ph), torch.sin(ph)).to(torch.complex64)
        del X, Y, ph
    ph = torch.remainder(t * (-60 * 100e3 / fs), 1.0) * (2 * math.pi)
    wide += 3000.0 * torch.complex(torch.cos(ph), torch.sin(ph)).to(torch.complex64)
    del t, ph
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    iq = torch.stack([wide.real, wide.imag], -1) + torch.randn((N, 2), generator=g, device="cuda") * 30.0
    return torch.clamp(torch.round(iq), -32768, 32767).to(torch.int16).reshape(-1).cpu().numpy()


def run(x, piece, **kw):
    from nrsc5_b200 import band
    import torch
    host = torch.from_numpy(x).pin_memory()
    t0 = time.perf_counter()
    with band.BandReceiver(**kw) as r:
        for a in range(0, x.size, piece):
            b = min(x.size, a + piece)
            r.push((host.data_ptr() + x.itemsize * a, b - a))
        r.flush()
        wall = time.perf_counter() - t0
        ms, route_bytes = r.times()
        sessions = r.sessions()
        nrec = {s["id"]: len(r.records(s["id"])) for s in sessions}
        nwin = len(r.windows())
    return wall, ms, route_bytes, sessions, nrec, nwin


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("file", nargs="?")
    ap.add_argument("--format", choices=["cu8", "cs16"], default="cs16")
    ap.add_argument("--band", choices=["fm", "am"], default="fm")
    ap.add_argument("--decim", type=int, default=32)
    ap.add_argument("--rate", type=int, default=None)
    ap.add_argument("--seconds", type=float, default=6.0)
    ap.add_argument("--piece", type=int, default=1 << 22, help="values per push")
    ap.add_argument("--window-symbols", type=int, default=128)
    ap.add_argument("--max-stations", type=int, default=32)
    ap.add_argument("--l2", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("band_receive: no CUDA device (the band receiver has no CPU path)")
    kw = dict(band=a.band, decim=a.decim, rate=a.rate, window_symbols=a.window_symbols, max_stations=a.max_stations, l2=a.l2)
    if a.file:
        x = np.fromfile(a.file, dtype=np.int16 if a.format == "cs16" else np.uint8)
        x = x[: x.size & ~1]
        kw["input_cs16"] = a.format == "cs16"
        fs = a.rate or (1488375.0 if a.band == "am" else a.decim * 744187.5)
    else:
        x = synthetic_band(a.seconds)
        kw.update(band="fm", decim=32, rate=None, input_cs16=True)
        fs = 23814000.0
        run(x[: 2 * int(0.5 * fs)], a.piece, **kw)                  # warm-up: module loads, allocations
    seconds = x.size / 2 / fs
    wall, ms, route_bytes, sessions, nrec, nwin = run(x, a.piece, **kw)
    res = {
        "card": card_info(), "band": kw["band"], "decim": kw["decim"], "rate": kw["rate"], "seconds": round(seconds, 3),
        "windows": nwin, "window_symbols": a.window_symbols,
        "capture_seconds_per_second": round(seconds / wall, 2), "wall_s": round(wall, 3),
        "stage_ms": {k: round(v, 2) for k, v in ms.items()},
        "stage_ms_per_capture_second": {k: round(v / seconds, 3) for k, v in ms.items()},
        "route_bytes": route_bytes, "route_GBps": round(route_bytes / (ms["route"] * 1e-3) / 1e9, 1) if ms["route"] else None,
        "sessions": [{"id": s["id"], "offset": s["offset"], "n0": s["n0"], "n1": s["n1"], "records": nrec[s["id"]],
                      "score": round(s["verdict"]["score"], 4)} for s in sessions],
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
