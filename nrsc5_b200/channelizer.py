"""ctypes binding of the wideband channeliser (include/nrsc5_b200.h, csrc/channelizer.cu): one cu8 or cs16 capture at
23 814 000 S/s -> FM channels at 744 187.5 S/s cs16, the format nrsc5b_push_cs16 / input_push_cs16 take; with
decim=16 or 8, the same from a capture at 11 907 000 or 5 953 500 S/s (wide_rate(decim)); or, with band="am", one
capture at 1 488 375 S/s -> AM channels (10 kHz grid) at 46 511.71875 S/s cs16 through a 512-tap bank.  rate=fs: a
capture at the radio's own rate (integer Hz) goes through an exact polyphase resampler to the chosen plan's rate first.
No CPU fallback: constructing a Channelizer without a CUDA device raises."""
from __future__ import annotations

import ctypes

import numpy as np

from .engine import EngineError, _check, load_library

WIDE_RATE = 23814000.0          # 32 x 744 187.5
AM_WIDE_RATE = 1488375.0        # 32 x 46 511.71875
TAPS, PERIOD, DECIM = 256, 11907, 32
TAPS_AM = 512
FM_RATE = 744187.5              # every FM plan's output rate
DECIMS = (8, 16, 32)            # the FM plans' decimations: captures at D x 744 187.5 S/s
# band plan -> (taps per channel, suffix of the plan's own entry points)
_BANDS = {"fm": (TAPS, ""), "am": (TAPS_AM, "_am")}
_MODES = {"fm": 0, "am": 1}     # NRSC5B_MODE_FM, NRSC5B_MODE_AM
RS_TAPS = 64                    # taps per phase of the rate stage


def _band(band, decim=DECIM):
    if band not in _BANDS:
        raise ValueError(f"band: {band!r} is neither 'fm' nor 'am'")
    if decim not in DECIMS:
        raise ValueError(f"decim: {decim!r} is not one of {DECIMS}")
    if band == "am" and decim != DECIM:
        raise ValueError(f"decim: the AM plan decimates by {DECIM}, not {decim}")
    return _BANDS[band]


def wide_rate(decim: int = DECIM) -> float:
    """The capture rate of the FM plan that decimates by `decim`: decim x 744 187.5 S/s."""
    _band("fm", decim)
    return decim * FM_RATE


def _lib():
    L = load_library()
    if not getattr(L, "_chan_ready", False):
        vp, sz, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        L.nrsc5b_chan_create.argtypes = [ctypes.POINTER(vp), ci, vp, ci]
        L.nrsc5b_chan_destroy.argtypes = [vp]
        L.nrsc5b_chan_destroy.restype = None
        L.nrsc5b_chan_tables.argtypes = [vp, vp, vp]
        L.nrsc5b_chan_make_tables.argtypes = [vp, ci, vp, vp]
        L.nrsc5b_chan_outputs.argtypes = [sz]
        L.nrsc5b_chan_outputs.restype = ctypes.c_longlong
        L.nrsc5b_chan_run_device.argtypes = [vp, vp, sz, vp, sz, vp]
        L.nrsc5b_chan_run.argtypes = [vp, vp, sz, vp]
        L.nrsc5b_chan_reset.argtypes = [vp]
        L.nrsc5b_chan_push.argtypes = [vp, vp, sz, vp, sz, vp, ctypes.POINTER(ctypes.c_longlong)]
        L.nrsc5b_chan_feed.argtypes = [vp, vp, vp, vp, sz]
        L.nrsc5b_chan_create_cs16.argtypes = [ctypes.POINTER(vp), ci, vp, ci]
        L.nrsc5b_chan_run_device_cs16.argtypes = [vp, vp, sz, vp, sz, vp]
        L.nrsc5b_chan_run_cs16.argtypes = [vp, vp, sz, vp]
        L.nrsc5b_chan_push_cs16.argtypes = [vp, vp, sz, vp, sz, vp, ctypes.POINTER(ctypes.c_longlong)]
        L.nrsc5b_chan_feed_cs16.argtypes = [vp, vp, vp, vp, sz]
        L.nrsc5b_chan_create_am.argtypes = [ctypes.POINTER(vp), ci, vp, ci]
        L.nrsc5b_chan_create_am_cs16.argtypes = [ctypes.POINTER(vp), ci, vp, ci]
        L.nrsc5b_chan_make_tables_am.argtypes = [vp, ci, vp, vp]
        L.nrsc5b_chan_outputs_am.argtypes = [sz]
        L.nrsc5b_chan_outputs_am.restype = ctypes.c_longlong
        L.nrsc5b_chan_create_fm.argtypes = [ctypes.POINTER(vp), ci, ci, vp, ci]
        L.nrsc5b_chan_create_fm_cs16.argtypes = [ctypes.POINTER(vp), ci, ci, vp, ci]
        L.nrsc5b_chan_make_tables_fm.argtypes = [ci, vp, ci, vp, vp]
        L.nrsc5b_chan_outputs_fm.argtypes = [ci, sz]
        L.nrsc5b_chan_outputs_fm.restype = ctypes.c_longlong
        u32, ll = ctypes.c_uint32, ctypes.c_longlong
        L.nrsc5b_chan_create_rate.argtypes = [ctypes.POINTER(vp), ci, ci, ci, u32, vp, ci]
        L.nrsc5b_chan_create_rate_cs16.argtypes = [ctypes.POINTER(vp), ci, ci, ci, u32, vp, ci]
        L.nrsc5b_chan_resampler_tables.argtypes = [ci, ci, u32, vp, vp, vp, vp]
        L.nrsc5b_chan_outputs_rate.argtypes = [ci, ci, u32, ll]
        L.nrsc5b_chan_outputs_rate.restype = ll
        L.nrsc5b_resample.argtypes = [ci, ci, ci, u32, ci, vp, sz, vp]
        L.nrsc5b_chan_resample_device.argtypes = [vp, vp, sz, vp]
        L._chan_ready = True
    return L


def _rate(rate, band, decim):
    """rate (integer Hz) -> the mode / decim / rate the rate-stage entry points take; ValueError for a rate they refuse."""
    _band(band, decim)
    fs = int(rate)
    if fs != rate or not 0 < fs < 1 << 32:
        raise ValueError(f"rate: {rate!r} is not a positive integer number of Hz")
    if _lib().nrsc5b_chan_outputs_rate(_MODES[band], decim, fs, 0) < 0:
        raise ValueError(f"rate: {fs} Hz cannot be resampled to the {band} plan at decim={decim}")
    return _MODES[band], decim, fs


def _counts(rate, decim, band, G=None):
    """(L, M, max_offset) of the rate stage; G: an int16 [L][64] array to receive its table as well."""
    mode, decim, fs = _rate(rate, band, decim)
    L, M, mo = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _check(_lib().nrsc5b_chan_resampler_tables(mode, decim, fs, ctypes.byref(L), ctypes.byref(M), ctypes.byref(mo),
                                               None if G is None else G.ctypes.data), "nrsc5b_chan_resampler_tables")
    return L.value, M.value, mo.value


def resampler_tables(rate, decim: int = DECIM, band: str = "fm"):
    """The rate stage from a capture at `rate` Hz to the plan's rate, without a device: (L, M, max_offset, G) with
    R / fs = L / M and G int16 [L][64] (fs == R: L = M = 1 and the identity row)."""
    L = _counts(rate, decim, band)[0]
    G = np.empty((L, RS_TAPS), dtype=np.int16)
    L, M, mo = _counts(rate, decim, band, G)
    return L, M, mo, G


def resampled(samples: int, rate, decim: int = DECIM, band: str = "fm") -> int:
    """K(T): resampled samples from T input samples at `rate`, by the header's formula (the library exports N_plan(K(T)),
    nrsc5b_chan_outputs_rate, not K itself; this sizes resample()'s output, as stream_outputs sizes a push's)."""
    L, M, _ = _counts(rate, decim, band)
    if L == 1:
        return samples
    return ((samples - RS_TAPS + 1) * L - 1) // M + 1 if samples >= RS_TAPS else 0


def resample(x: np.ndarray, rate, decim: int = DECIM, band: str = "fm", device: int = 0) -> np.ndarray:
    """The rate stage alone on the device (nrsc5b_resample): a uint8 (cu8) or int16 (cs16) capture at `rate` -> int16
    [2 K(T)], y I/Q interleaved."""
    mode, decim, fs = _rate(rate, band, decim)
    a = np.ascontiguousarray(x).reshape(-1)
    assert a.dtype in (np.uint8, np.int16)
    k = resampled(a.size // 2, rate, decim, band)
    out = np.empty(2 * max(k, 1), dtype=np.int16)
    _check(_lib().nrsc5b_resample(device, mode, decim, fs, int(a.dtype == np.int16), a.ctypes.data if a.size else None, a.size,
                                  out.ctypes.data), "nrsc5b_resample")
    return out[: 2 * k]


def stream_outputs(pushed: int, nbytes: int, band: str = "fm", decim: int = DECIM, rate=None) -> int:
    """Outputs per channel a push of nbytes (cu8; cs16: int16 values) emits after `pushed` complex samples
    (include/nrsc5_b200.h): N(T') - N(T), N(T) = (T - 256) // D + 1 for T >= 256, else 0, D = decim (band "am": 512
    for 256); with rate, N_plan(K(T)) of a capture at `rate`."""
    if rate is not None:
        mode, decim, fs = _rate(rate, band, decim)
        f = _lib().nrsc5b_chan_outputs_rate
        return int(f(mode, decim, fs, pushed + nbytes // 2) - f(mode, decim, fs, pushed))
    ntaps = _band(band, decim)[0]

    def n(t):
        return (t - ntaps) // decim + 1 if t >= ntaps else 0
    return n(pushed + nbytes // 2) - n(pushed)


def make_tables(offsets_100khz, band: str = "fm", decim: int = DECIM):
    """The integer tables of the definition, computed on the host (no device): taps[nch][256][2], phasor[11907][2]
    (band "am": offsets in 10 kHz steps, taps[nch][512][2]; decim: the FM plan of a decim x 744 187.5 S/s capture)."""
    ntaps, sfx = _band(band, decim)
    off = np.ascontiguousarray(offsets_100khz, dtype=np.int32)
    taps = np.empty((off.size, ntaps, 2), dtype=np.int16)
    ph = np.empty((PERIOD, 2), dtype=np.int16)
    if decim != DECIM:
        name = "nrsc5b_chan_make_tables_fm"
        _check(_lib().nrsc5b_chan_make_tables_fm(decim, off.ctypes.data, off.size, taps.ctypes.data, ph.ctypes.data), name)
        return taps, ph
    name = "nrsc5b_chan_make_tables" + sfx
    _check(getattr(_lib(), name)(off.ctypes.data, off.size, taps.ctypes.data, ph.ctypes.data), name)
    return taps, ph


def outputs(nbytes: int, band: str = "fm", decim: int = DECIM, rate=None) -> int:
    """Outputs per channel of a capture of nbytes cu8 bytes (or as many int16 values of cs16); with rate, of a capture
    at `rate` through the rate stage (every complex sample counts)."""
    if rate is not None:
        return stream_outputs(0, nbytes, band, decim, rate)
    sfx = _band(band, decim)[1]
    if decim != DECIM:
        return int(_lib().nrsc5b_chan_outputs_fm(decim, nbytes & ~63))
    return int(getattr(_lib(), "nrsc5b_chan_outputs" + sfx)(nbytes & ~63))


class Channelizer:
    """input_cs16=False: the capture is cu8 (uint8, lengths in bytes); True: cs16 (int16, lengths in int16 values,
    the _cs16 entry points).  Either way two input units make one complex sample.  band="am": the AM plan (offsets in
    10 kHz steps of a 1 488 375 S/s capture, 512 taps); decim=16 or 8: the FM plan of a capture at wide_rate(decim)
    (offsets within +-59 or +-29); rate=fs: a capture at fs Hz, resampled to that plan's rate first (rate=None: the capture
    is at the plan's rate; offsets within resampler_tables(rate, decim, band)[2]).  Only create differs, every other call
    is the handle's."""
    def __init__(self, offsets_100khz, device: int = 0, input_cs16: bool = False, band: str = "fm", decim: int = DECIM,
                 rate=None):
        self._L = _lib()
        self.band = band
        self.decim = int(decim)
        self.taps = _band(band, self.decim)[0]
        self.offsets = np.ascontiguousarray(offsets_100khz, dtype=np.int32)
        self.nch = int(self.offsets.size)
        self.input_cs16 = bool(input_cs16)
        self._dtype = np.int16 if self.input_cs16 else np.uint8
        self._sfx = "_cs16" if self.input_cs16 else ""
        self._h = ctypes.c_void_p()
        # a capture at the plan's own rate is the plan itself (the library returns the plan's handle)
        self.rate = None if rate is None or _counts(rate, self.decim, band)[0] == 1 else int(rate)
        if rate is not None:
            name = "nrsc5b_chan_create_rate" + self._sfx
            mode, _, fs = _rate(rate, band, self.decim)
            _check(getattr(self._L, name)(ctypes.byref(self._h), device, mode, self.decim, fs, self.offsets.ctypes.data, self.nch), name)
        elif self.decim != DECIM:
            name = "nrsc5b_chan_create_fm" + self._sfx
            _check(getattr(self._L, name)(ctypes.byref(self._h), device, self.decim, self.offsets.ctypes.data, self.nch), name)
        else:
            name = "nrsc5b_chan_create" + _band(band)[1] + self._sfx
            _check(getattr(self._L, name)(ctypes.byref(self._h), device, self.offsets.ctypes.data, self.nch), name)
        self.device = device
        self.pushed = 0                 # T: complex samples pushed since create / reset (mirrors the handle's count)

    def close(self):
        if self._h:
            self._L.nrsc5b_chan_destroy(self._h)
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

    def tables(self):
        taps = np.empty((self.nch, self.taps, 2), dtype=np.int16)
        ph = np.empty((PERIOD, 2), dtype=np.int16)
        _check(self._L.nrsc5b_chan_tables(self._h, taps.ctypes.data, ph.ctypes.data), "nrsc5b_chan_tables")
        return taps, ph

    def _call(self, name, *args):
        name = name + self._sfx
        return _check(getattr(self._L, name)(*args), name)

    def run(self, cu8: np.ndarray) -> np.ndarray:
        """Host capture (uint8, or int16 with input_cs16; I/Q interleaved) -> int16 array [nch][2 * outputs] (I, Q
        interleaved)."""
        a = np.ascontiguousarray(cu8, dtype=self._dtype).reshape(-1)
        # what the entry point writes: cu8 whole 64-byte rows, cs16 every complex sample
        if self.rate is not None:                  # every complex sample (an odd length is refused by the entry point)
            n = stream_outputs(0, a.size, self.band, self.decim, self.rate)
        else:
            n = stream_outputs(0, a.size, self.band, self.decim) if self.input_cs16 else outputs(a.size, self.band, self.decim)
        out = np.empty((self.nch, 2 * max(n, 0)), dtype=np.int16)
        if n > 0:
            self._call("nrsc5b_chan_run", self._h, a.ctypes.data, a.size, out.ctypes.data)
        return out

    def run_device(self, d_cu8: int, nbytes: int, d_out: int, out_stride: int, stream: int = 0):
        """Device capture (nbytes bytes of cu8, or nbytes int16 values of cs16) -> d_out[nch][out_stride]."""
        self._call("nrsc5b_chan_run_device", self._h, ctypes.c_void_p(d_cu8), nbytes, ctypes.c_void_p(d_out), out_stride,
                   ctypes.c_void_p(stream))

    def resample_device(self, d_in: int, nvalues: int, stream: int = 0):
        """The rate stage of run_device() alone (nrsc5b_chan_resample_device): the same k_resample launches into the
        handle's scratch, no channel output; for timing the stage apart from the channel bank."""
        _check(self._L.nrsc5b_chan_resample_device(self._h, ctypes.c_void_p(d_in), nvalues, ctypes.c_void_p(stream)),
               "nrsc5b_chan_resample_device")

    # ---- streaming: a capture pushed in pieces; the outputs concatenate to run() of the whole capture ----
    def reset(self):
        _check(self._L.nrsc5b_chan_reset(self._h), "nrsc5b_chan_reset")
        self.pushed = 0

    def push_device(self, ptr: int, nbytes: int, d_out: int, out_stride: int, stream: int = 0) -> int:
        """The next nbytes (cs16: int16 values) of the capture at ptr (host or device memory) -> the outputs they
        complete, written to the device buffer d_out[nch][out_stride] (int16 values); asynchronous on `stream`.  Returns
        the outputs per channel."""
        n = ctypes.c_longlong(0)
        self._call("nrsc5b_chan_push", self._h, ctypes.c_void_p(ptr), nbytes, ctypes.c_void_p(d_out), out_stride,
                   ctypes.c_void_p(stream), ctypes.byref(n))
        self.pushed += nbytes // 2
        return int(n.value)

    def push(self, cu8: np.ndarray) -> np.ndarray:
        """The next piece of the capture (uint8, or int16 with input_cs16; I/Q interleaved, even length) -> int16
        [nch][2 * n]: the outputs it completes.  Synchronous."""
        import torch
        a = np.ascontiguousarray(cu8, dtype=self._dtype).reshape(-1)
        n = stream_outputs(self.pushed, a.size, self.band, self.decim, self.rate)
        dev = torch.device("cuda", self.device)
        out = torch.empty((self.nch, 2 * max(n, 1)), dtype=torch.int16, device=dev)
        stream = torch.cuda.current_stream(dev)
        got = self.push_device(a.ctypes.data if a.size else 0, a.size, out.data_ptr(), out.shape[1], stream.cuda_stream)
        assert got == n
        stream.synchronize()
        return out[:, : 2 * n].cpu().numpy()

    def feed(self, engine, data, streams=None):
        """The next piece of the capture -> channel k appended to cs16 stream streams[k] of `engine` (an Engine made
        with input_cs16=True and the band's mode; streams None: stream k).  data: a uint8 (input_cs16: int16) numpy array or (pointer, nbytes
        or int16 values) to host or device memory.  Raises EngineError on NRSC5B_EFULL (nothing taken: process() and feed the same data again)."""
        if isinstance(data, tuple):
            ptr, nbytes = int(data[0]), int(data[1])
            keep = None
        else:
            keep = np.ascontiguousarray(data, dtype=self._dtype).reshape(-1)
            ptr, nbytes = (keep.ctypes.data if keep.size else 0), keep.size
        st = None
        if streams is not None:
            st = np.ascontiguousarray(streams, dtype=np.int32)
            if st.size != self.nch:
                raise ValueError(f"streams: {st.size} entries for {self.nch} channels")
        self._call("nrsc5b_chan_feed", self._h, engine._h, None if st is None else st.ctypes.data, ctypes.c_void_p(ptr), nbytes)
        self.pushed += nbytes // 2
