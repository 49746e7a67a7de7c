"""ctypes binding of the band receiver (include/nrsc5_b200.h: nrsc5b_band_*, csrc/band.cu): a live wideband capture in
pieces of any size -> every HD Radio station in it decoded, an engine stream attached when the per-window scan finds a
station and detached when it has lost it.  No CPU fallback: a BandReceiver needs a CUDA device."""
from __future__ import annotations

import ctypes

import numpy as np

from . import channelizer as ch
from .engine import _check, load_library, parse_records
from .scan import ScanResult, _mode

DETECTED, LEAKAGE, ATTACHED, NO_SLOT = 1, 2, 4, 8       # NRSC5B_BAND_* row flags
SYMBOL = {"fm": 2160, "am": 270}                         # S: samples per OFDM symbol at the channel rate


class Config(ctypes.Structure):
    _fields_ = [("device", ctypes.c_int), ("mode", ctypes.c_int), ("decim", ctypes.c_int), ("rate_hz", ctypes.c_uint32),
                ("input_cs16", ctypes.c_int), ("offsets", ctypes.c_void_p), ("nch", ctypes.c_int),
                ("window_symbols", ctypes.c_int), ("hold_windows", ctypes.c_int), ("max_stations", ctypes.c_int),
                ("l2", ctypes.c_int)]


class Session(ctypes.Structure):
    _fields_ = [("id", ctypes.c_int32), ("channel", ctypes.c_int32), ("offset", ctypes.c_int32), ("slot", ctypes.c_int32),
                ("n0", ctypes.c_int64), ("n1", ctypes.c_int64), ("window", ctypes.c_int64), ("verdict", ScanResult)]

    def as_dict(self):
        d = {name: getattr(self, name) for name, _ in self._fields_ if name != "verdict"}
        d["verdict"] = self.verdict.as_dict()
        return d


def _lib():
    L = load_library()
    if not getattr(L, "_band_ready", False):
        vp, sz, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        L.nrsc5b_band_create.argtypes = [ctypes.POINTER(vp), ctypes.POINTER(Config)]
        L.nrsc5b_band_destroy.argtypes = [vp]
        L.nrsc5b_band_destroy.restype = None
        L.nrsc5b_band_push.argtypes = [vp, vp, sz]
        L.nrsc5b_band_flush.argtypes = [vp]
        L.nrsc5b_band_windows.argtypes = [vp, vp, vp, vp, ci, ctypes.POINTER(ci)]
        L.nrsc5b_band_sessions.argtypes = [vp, vp, ci, ctypes.POINTER(ci)]
        L.nrsc5b_band_records.argtypes = [vp, ci, vp, sz, ctypes.POINTER(sz)]
        L.nrsc5b_band_records.restype = ctypes.c_long
        L.nrsc5b_band_channels.argtypes = [vp, vp, ctypes.POINTER(ci)]
        L.nrsc5b_band_times.argtypes = [vp, vp, ctypes.POINTER(ctypes.c_ulonglong)]
        L._band_ready = True
    return L


def make_config(band="fm", decim=ch.DECIM, rate=None, input_cs16=False, offsets=None, window_symbols=128, hold_windows=3,
                max_stations=32, l2=False, device=0):
    """The nrsc5b_band_config_t of these arguments, and the offsets array it points to (keep it alive with the config)."""
    offs = None if offsets is None else np.ascontiguousarray([int(m) for m in offsets], dtype=np.int32)
    cfg = Config(device, _mode(band), int(decim), int(rate or 0), int(bool(input_cs16)),
                 None if offs is None else offs.ctypes.data, 0 if offs is None else offs.size, int(window_symbols),
                 int(hold_windows), int(max_stations), int(bool(l2)))
    return cfg, offs


class BandReceiver:
    """band "fm" (offsets in 100 kHz steps, decim 8 | 16 | 32) or "am" (10 kHz steps); rate: the capture's own rate in
    Hz through the rate stage (None: the plan's rate); input_cs16: int16 capture (False: uint8 cu8); offsets None:
    every grid point (scan.grid_offsets).  push() is synchronous: the windows it completes have been scanned, routed and
    decoded when it returns."""

    def __init__(self, band="fm", decim=32, rate=None, input_cs16=False, offsets=None, window_symbols=128, hold_windows=3,
                 max_stations=32, l2=False, device=0):
        self._L = _lib()
        self.band = band
        self.input_cs16 = bool(input_cs16)
        self._dtype = np.int16 if self.input_cs16 else np.uint8
        cfg, self._offs = make_config(band, decim, rate, input_cs16, offsets, window_symbols, hold_windows, max_stations, l2,
                                      device)
        self._h = ctypes.c_void_p()
        _check(self._L.nrsc5b_band_create(ctypes.byref(self._h), ctypes.byref(cfg)), "nrsc5b_band_create")
        n = ctypes.c_int()
        _check(self._L.nrsc5b_band_channels(self._h, None, ctypes.byref(n)), "nrsc5b_band_channels")
        self.nch = n.value
        offs = np.empty(self.nch, dtype=np.int32)
        _check(self._L.nrsc5b_band_channels(self._h, offs.ctypes.data, ctypes.byref(n)), "nrsc5b_band_channels")
        self.offsets = [int(m) for m in offs]
        self.window_samples = int(window_symbols) * SYMBOL[band]     # W

    def close(self):
        if self._h:
            self._L.nrsc5b_band_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def push(self, data):
        """The next piece of the capture: a uint8 (input_cs16: int16) numpy array, a CUDA tensor of that dtype, or
        (pointer, nvalues) to host or device memory."""
        if isinstance(data, tuple):
            ptr, n = int(data[0]), int(data[1])
        elif hasattr(data, "data_ptr"):
            ptr, n = data.data_ptr(), data.numel()
        else:
            keep = np.ascontiguousarray(data, dtype=self._dtype).reshape(-1)
            ptr, n = (keep.ctypes.data if keep.size else 0), keep.size
        _check(self._L.nrsc5b_band_push(self._h, ctypes.c_void_p(ptr), n), "nrsc5b_band_push")

    def flush(self):
        _check(self._L.nrsc5b_band_flush(self._h), "nrsc5b_band_flush")

    def windows(self):
        """The completed windows not taken yet: [{index, rows: [nrsc5b_scan_t as dict] * nch, flags: int array}]."""
        pending = ctypes.c_int()
        _check(self._L.nrsc5b_band_windows(self._h, None, None, None, 0, ctypes.byref(pending)), "nrsc5b_band_windows")
        n = pending.value
        index = np.empty(max(n, 1), dtype=np.int64)
        rows = (ScanResult * max(n * self.nch, 1))()
        flags = np.empty((max(n, 1), self.nch), dtype=np.uint32)
        got = _check(self._L.nrsc5b_band_windows(self._h, index.ctypes.data, rows, flags.ctypes.data, n, ctypes.byref(pending)),
                     "nrsc5b_band_windows")
        return [{"index": int(index[i]), "rows": [rows[i * self.nch + k].as_dict() for k in range(self.nch)],
                 "flags": flags[i].copy()} for i in range(got)]

    def sessions(self):
        n = ctypes.c_int()
        _check(self._L.nrsc5b_band_sessions(self._h, None, 0, ctypes.byref(n)), "nrsc5b_band_sessions")
        out = (Session * max(n.value, 1))()
        got = _check(self._L.nrsc5b_band_sessions(self._h, out, n.value, ctypes.byref(n)), "nrsc5b_band_sessions")
        return [out[i].as_dict() for i in range(got)]

    def records_raw(self, sid: int) -> bytes:
        need = ctypes.c_size_t()
        rc = self._L.nrsc5b_band_records(self._h, sid, None, 0, ctypes.byref(need))
        if rc != -5:                                              # EFULL: records are waiting, *needed says how many
            _check(rc, "nrsc5b_band_records")
        buf = ctypes.create_string_buffer(max(need.value, 1))
        n = _check(self._L.nrsc5b_band_records(self._h, sid, buf, need.value, ctypes.byref(need)), "nrsc5b_band_records")
        return buf.raw[:n]

    def records(self, sid: int):
        """Session sid's records since the last call, parsed (engine.parse_records)."""
        return parse_records(self.records_raw(sid))

    def times(self):
        """Device milliseconds per stage since create, and the bytes k_band_route read and wrote."""
        ms = (ctypes.c_double * 4)()
        nb = ctypes.c_ulonglong()
        _check(self._L.nrsc5b_band_times(self._h, ms, ctypes.byref(nb)), "nrsc5b_band_times")
        return {"channelise": ms[0], "scan": ms[1], "route": ms[2], "engine": ms[3]}, int(nb.value)


