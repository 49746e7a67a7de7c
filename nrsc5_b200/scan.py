"""ctypes binding of the band scan (include/nrsc5_b200.h: nrsc5b_scan_*, nrsc5b_chan_scan; csrc/scan.cu): which
channels of a channelised band carry an NRSC-5 signal, with each one's symbol timing, fractional CFO and per-sideband
SNR.  scan_band() takes a wideband capture straight to one row per channel.  No CPU fallback: a Scanner needs a CUDA
device."""
from __future__ import annotations

import ctypes

import numpy as np

from . import channelizer as ch
from .engine import _check, load_library

MODES = {"fm": 0, "am": 1}
GEOMETRY = {"fm": dict(F=2048, P=112, q=4, fs=744187.5), "am": dict(F=256, P=14, q=2, fs=46511.71875)}
NTAPS = 64


def _j(band):
    g = GEOMETRY[band]
    return (g["F"] + g["P"]) // g["q"]


def raw_size(band):
    """int64 values per channel of Scanner.result(raw=True) (NRSC5B_SCAN_RAW)."""
    return 12 * _j(band) + 2


class ScanResult(ctypes.Structure):
    _fields_ = [("score", ctypes.c_double), ("threshold", ctypes.c_double), ("symbols", ctypes.c_double),
                ("cfo_hz", ctypes.c_double), ("score_lower", ctypes.c_double), ("score_upper", ctypes.c_double),
                ("threshold_sideband", ctypes.c_double), ("snr_db_lower", ctypes.c_double), ("snr_db_upper", ctypes.c_double),
                ("power_dbfs", ctypes.c_double), ("power_dbfs_lower", ctypes.c_double),
                ("power_dbfs_upper", ctypes.c_double), ("detected", ctypes.c_int32), ("timing", ctypes.c_int32)]

    def as_dict(self):
        return {name: getattr(self, name) for name, _ in self._fields_}


def _lib():
    L = load_library()
    if not getattr(L, "_scan_ready", False):
        vp, sz, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        L.nrsc5b_scan_create.argtypes = [ctypes.POINTER(vp), ci, ci, ci]
        L.nrsc5b_scan_destroy.argtypes = [vp]
        L.nrsc5b_scan_destroy.restype = None
        L.nrsc5b_scan_reset.argtypes = [vp]
        L.nrsc5b_scan_push_device.argtypes = [vp, vp, sz, sz, vp]
        L.nrsc5b_scan_push.argtypes = [vp, vp, sz]
        L.nrsc5b_scan_result.argtypes = [vp, vp, vp]
        L.nrsc5b_chan_scan.argtypes = [vp, vp, vp, sz]
        L.nrsc5b_scan_make_tables.argtypes = [ci, vp, ctypes.POINTER(ctypes.c_double)]
        L._scan_ready = True
    return L


def _mode(band):
    if band not in MODES:
        raise ValueError(f"band: {band!r} is neither 'fm' nor 'am'")
    return MODES[band]


def make_tables(band: str = "fm"):
    """The upper sideband's taps int16 [64][2] (g_L = conj(g_U)) and kappa, without a device."""
    taps = np.empty((NTAPS, 2), dtype=np.int16)
    kappa = ctypes.c_double()
    _check(_lib().nrsc5b_scan_make_tables(_mode(band), taps.ctypes.data, ctypes.byref(kappa)), "nrsc5b_scan_make_tables")
    return taps, kappa.value


class Scanner:
    """A scan of `nch` channels of band "fm" (744 187.5 S/s) or "am" (46 511.72 S/s), cs16 channel output."""
    def __init__(self, nch: int, band: str = "fm", device: int = 0):
        self._L = _lib()
        self.band = band
        self.nch = int(nch)
        self.device = device
        self._h = ctypes.c_void_p()
        _check(self._L.nrsc5b_scan_create(ctypes.byref(self._h), device, _mode(band), self.nch), "nrsc5b_scan_create")

    def close(self):
        if self._h:
            self._L.nrsc5b_scan_destroy(self._h)
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

    def reset(self):
        _check(self._L.nrsc5b_scan_reset(self._h), "nrsc5b_scan_reset")

    def push(self, cs16: np.ndarray):
        """The next samples of every channel: int16 [nch][2 n] (I/Q interleaved).  Synchronous."""
        a = np.ascontiguousarray(cs16, dtype=np.int16).reshape(self.nch, -1)
        if a.shape[1] % 2:
            raise ValueError("cs16: an odd number of int16 values per channel")
        _check(self._L.nrsc5b_scan_push(self._h, a.ctypes.data if a.size else None, a.shape[1] // 2), "nrsc5b_scan_push")

    def push_device(self, d_ch: int, stride: int, nsamples: int, stream: int = 0):
        """nsamples of every channel from device memory [nch][stride] int16 values; asynchronous on `stream`."""
        _check(self._L.nrsc5b_scan_push_device(self._h, ctypes.c_void_p(d_ch), stride, nsamples, ctypes.c_void_p(stream)),
               "nrsc5b_scan_push_device")

    def scan_capture(self, chan: ch.Channelizer, data):
        """Channelise and scan (nrsc5b_chan_scan): data a uint8 (cs16 handles: int16) numpy array or (pointer,
        nvalues) to host or device memory."""
        if isinstance(data, tuple):
            ptr, n = int(data[0]), int(data[1])
        else:
            keep = np.ascontiguousarray(data, dtype=chan._dtype).reshape(-1)
            ptr, n = (keep.ctypes.data if keep.size else 0), keep.size
        _check(self._L.nrsc5b_chan_scan(chan._h, self._h, ctypes.c_void_p(ptr), n), "nrsc5b_chan_scan")
        chan.pushed += n // 2

    def result(self, raw: bool = False):
        """One dict per channel (the nrsc5b_scan_t fields); raw=True: also the exact sums int64 [nch][raw_size]."""
        out = (ScanResult * self.nch)()
        r = np.empty((self.nch, raw_size(self.band)), dtype=np.int64) if raw else None
        _check(self._L.nrsc5b_scan_result(self._h, out, None if r is None else r.ctypes.data), "nrsc5b_scan_result")
        rows = [o.as_dict() for o in out]
        return (rows, r) if raw else rows


def grid_offsets(band: str = "fm", rate=None, decim: int = ch.DECIM):
    """Every grid point whose channel lies inside the capture: the plan's own range (FM: |m| <= 117 at decim 32, 59 at
    16, 29 at 8; AM: 74), or the rate stage's limit where it is tighter."""
    _mode(band)
    lim = 74 if band == "am" else {32: 117, 16: 59, 8: 29}[decim]
    if rate is not None:
        lim = ch.resampler_tables(rate, decim, band)[2] or lim      # 0: a capture at the plan's own rate, no stage
    return list(range(-lim, lim + 1))


def scan_band(capture: np.ndarray, band: str = "fm", rate=None, decim: int = ch.DECIM, offsets=None, device: int = 0):
    """Scan a wideband capture (uint8 cu8 or int16 cs16, I/Q interleaved) at the plan's rate, or at `rate` Hz through
    the rate stage: one row per channel with its offset (100 kHz steps for FM, 10 kHz for AM).  offsets=None:
    grid_offsets(band, rate, decim)."""
    a = np.ascontiguousarray(capture).reshape(-1)
    if a.dtype not in (np.uint8, np.int16):
        raise ValueError("capture: uint8 (cu8) or int16 (cs16)")
    if offsets is None:
        offsets = grid_offsets(band, rate, decim)
    offsets = [int(m) for m in offsets]
    with ch.Channelizer(offsets, device=device, input_cs16=a.dtype == np.int16, band=band, decim=decim, rate=rate) as c, \
            Scanner(len(offsets), band, device) as s:
        s.scan_capture(c, a)
        rows = s.result()
    return [dict(offset=m, **r) for m, r in zip(offsets, rows)]
