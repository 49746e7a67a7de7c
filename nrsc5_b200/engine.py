"""ctypes binding of libnrsc5_b200.so (include/nrsc5_b200.h).

Mirrors the reference's own Python binding style (reference support/nrsc5.py:
a ctypes CDLL with thin methods); there is deliberately no CPU fallback: if
the CUDA library is missing or no GPU is present, constructing an Engine raises.
"""
from __future__ import annotations

import ctypes
import os
import struct

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

REC_FRAME, REC_PIDS, REC_SYNC, REC_LOST_SYNC, REC_MER, REC_BER = 1, 2, 3, 4, 5, 6
REC_SOFT_PM, REC_BLOCK = 8, 9
REC_PAD = 12                                                  # an unused slot: no call, parse_records skips it
REC_L2 = 20                                                   # L2 framing of one frame (include/nrsc5_b200.h)
EV_SERVICE, EV_ALIGN, EV_AAS, EV_PACKET = 16, 17, 18, 19      # its events: the reference's L2 -> L3 calls
L2F_LOST, L2F_EV_OVERFLOW = 1, 2


class EngineError(RuntimeError):
    pass


class _Config(ctypes.Structure):
    _fields_ = [("device", ctypes.c_int), ("nstreams", ctypes.c_int), ("mode", ctypes.c_int),
                ("input_capacity", ctypes.c_size_t), ("log_capacity", ctypes.c_size_t),
                ("emit_soft", ctypes.c_int), ("input_cs16", ctypes.c_int)]


class Stats(ctypes.Structure):
    _fields_ = [("blocks", ctypes.c_uint64), ("samples", ctypes.c_uint64),
                ("p1_frames", ctypes.c_uint64), ("kernel_launches", ctypes.c_uint64),
                ("p1_fallbacks", ctypes.c_uint64), ("log_overflows", ctypes.c_uint64)]


def lib_path() -> str:
    return os.path.join(_HERE, "libnrsc5_b200.so")


_lib = None


def load_library():
    """Load libnrsc5_b200.so; raises EngineError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not os.path.exists(p):
        raise EngineError(f"{p} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)")
    L = ctypes.CDLL(p)
    vp, sz, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    L.nrsc5b_version.restype = ctypes.c_char_p
    L.nrsc5b_create.argtypes = [ctypes.POINTER(vp), ctypes.POINTER(_Config)]
    L.nrsc5b_destroy.argtypes = [vp]
    L.nrsc5b_destroy.restype = None
    L.nrsc5b_reset.argtypes = [vp, ci]
    L.nrsc5b_rewind.argtypes = [vp]
    L.nrsc5b_set_profiling.argtypes = [vp, ci]
    L.nrsc5b_get_kernel_times.argtypes = [vp, vp, vp]
    L.nrsc5b_get_phase_cycles.argtypes = [vp, vp, vp]
    L.nrsc5b_get_am_phase_cycles.argtypes = [vp, vp]
    L.nrsc5b_set_cuda_stream.argtypes = [vp, vp]
    L.nrsc5b_push_cu8.argtypes = [vp, ci, vp, sz]
    L.nrsc5b_push_cs16.argtypes = [vp, ci, vp, sz]
    L.nrsc5b_push_cu8_device.argtypes = [vp, ci, vp, sz]
    L.nrsc5b_push_cu8_all.argtypes = [vp, vp, sz, sz]
    L.nrsc5b_attach_device_input.argtypes = [vp, vp, sz, sz]
    L.nrsc5b_attach_device_log.argtypes = [vp, vp, sz]
    L.nrsc5b_process.argtypes = [vp]
    L.nrsc5b_process_available.argtypes = [vp]
    L.nrsc5b_push_fence.argtypes = [vp]
    L.nrsc5b_process_fence.argtypes = [vp, ci]
    L.nrsc5b_synchronize.argtypes = [vp]
    L.nrsc5b_prepare_async.argtypes = [vp]
    L.nrsc5b_stage_cu8.argtypes = [vp, ci, vp, sz]
    L.nrsc5b_stage_cs16.argtypes = [vp, ci, vp, sz]
    L.nrsc5b_submit.argtypes = [vp, ci]
    L.nrsc5b_poll.argtypes = [vp, ci]
    L.nrsc5b_batch_records.argtypes = [vp, ci, ctypes.POINTER(sz)]
    L.nrsc5b_batch_records.restype = vp
    L.nrsc5b_drain.argtypes = [vp, ci, vp, sz, ctypes.POINTER(sz)]
    L.nrsc5b_drain.restype = ctypes.c_long
    L.nrsc5b_drain_all.argtypes = [vp, vp, sz, vp]
    L.nrsc5b_set_sync_state.argtypes = [vp, ci, ci]
    L.nrsc5b_take_overflow.argtypes = [vp, ci]
    L.nrsc5b_get_stats.argtypes = [vp, ctypes.POINTER(Stats)]
    L.nrsc5b_enable_l2.argtypes = [vp, ci]
    L.nrsc5b_l2_frames.argtypes = [ci, ctypes.c_char_p, sz, vp, sz, ctypes.POINTER(sz)]
    L.nrsc5b_l2_frames.restype = ctypes.c_long
    L.nrsc5b_halfband_fm.argtypes = [ci, vp, sz, vp]
    L.nrsc5b_viterbi_k7.argtypes = [ci, vp, vp, ci, ci]
    L.nrsc5b_viterbi_k7_ex.argtypes = [ci, vp, vp, ci, ci, ctypes.POINTER(ci)]
    L.nrsc5b_viterbi_k7_fast.argtypes = [ci, vp, ci, ci, ci, vp, vp]
    L.nrsc5b_rs_decode.argtypes = [ci, vp, vp, ci]
    L.nrsc5b_fft2048.argtypes = [ci, vp, vp, ci]
    _lib = L
    return L


def _check(rc, what):
    if rc < 0:
        names = {-1: "ENODEV (no CUDA device; no CPU path exists)", -2: "EINVAL", -3: "ENOMEM", -4: "ECUDA", -5: "EFULL",
                 -6: "EOVERFLOW (a stream's record log overflowed: raise log_capacity)"}
        raise EngineError(f"{what} failed: {names.get(rc, rc)}")
    return rc


def parse_l2(pay: bytes) -> dict:
    """Payload of a REC_L2 record -> its header fields, the PDU bytes and the events in call order.  A packet
    event's `data` is cut out of the PDU bytes, so that events compare directly with the oracle's L2 records."""
    frame_off, lc, nbits, pci, flags, pdu_len, ev_len, ordinal = struct.unpack_from("<8I", pay, 0)
    ev = pay[32:32 + ev_len]
    pdu = bytes(pay[32 + ev_len:32 + ev_len + pdu_len])
    events, off = [], 0
    while off < len(ev):
        ty, plen = struct.unpack_from("<II", ev, off)
        p = ev[off + 8: off + 8 + plen]
        off += 8 + ((plen + 3) & ~3)
        if ty == EV_SERVICE:
            k = ("program", "access", "type", "codec_mode", "blend_control", "gain", "common_delay", "latency")
            r = dict(zip(k, struct.unpack("<8i", p[:32])))
        elif ty == EV_ALIGN:
            r = dict(zip(("program", "stream_id", "offset"), struct.unpack("<3I", p[:12])))
        elif ty == EV_AAS:
            r = {"data": bytes(p)}
        elif ty == EV_PACKET:
            prog, sid, seq, shape, fl, size, at = struct.unpack("<7I", p[:28])
            r = {"program": prog, "stream_id": sid, "seq": seq, "shape": shape, "flags": fl, "size": size,
                 "data": pdu[at:at + size]}
        else:
            raise EngineError(f"corrupt L2 event stream (type {ty})")
        events.append((ty, r))
    return {"frame_off": frame_off, "lc": lc, "nbits": nbits, "pci": pci, "flags": flags, "ordinal": ordinal,
            "pdu": pdu, "events": events}


def with_l2_in_call_order(raw: bytes):
    """A drained record stream with every REC_L2 moved right behind the REC_FRAME it belongs to and expanded into
    its events - the order in which the reference makes the calls (frame_push -> frame_process)."""
    offs = []
    records = parse_records(raw, offs)
    l2_of = {r["frame_rec_off"]: r for ty, r in records if ty == REC_L2}
    out = []
    for (ty, r), at in zip(records, offs):
        if ty == REC_L2:
            continue
        out.append((ty, r))
        if ty == REC_FRAME and at in l2_of:
            out.extend(l2_of[at]["events"])
    return out


def parse_records(raw: bytes, offsets: list = None):
    """Decode the engine's record stream into (type, dict) tuples (offsets: gets each record's byte offset).
    REC_PAD records stand for no call and are left out."""
    out = []
    off, n = 0, len(raw)
    while off < n:
        ty, plen = struct.unpack_from("<II", raw, off)
        if ty == REC_PAD:
            off += 8 + ((plen + 3) & ~3)
            continue
        if offsets is not None:
            offsets.append(off)
        pay = raw[off + 8: off + 8 + plen]
        off += 8 + ((plen + 3) & ~3)
        if ty == REC_FRAME:
            lc, nbits = struct.unpack_from("<II", pay, 0)
            rec = {"lc": lc, "nbits": nbits, "bits": bytes(pay[8:])}
        elif ty == REC_PIDS:
            rec = {"bits": bytes(pay[:10]), "crc_ok": (pay[10] if len(pay) > 10 else None)}   # CRC-12 verdict (pids.c:52-86)
        elif ty == REC_SYNC:
            f, psmi = struct.unpack_from("<fi", pay)
            flags = struct.unpack_from("<4i", pay, 8) if len(pay) >= 24 else (-1, -1, -1, -1)   # AM: pli, hppi, aabi, rdbi
            rec = {"freq_offset": f, "psmi": psmi, "flags": list(flags)}
        elif ty == REC_LOST_SYNC:
            rec = {}
        elif ty == REC_MER:
            lo, up = struct.unpack("<ff", pay)
            rec = {"lower": lo, "upper": up}
        elif ty == REC_BER:
            rec = {"cber": struct.unpack("<f", pay)[0]}
        elif ty == REC_SOFT_PM:
            rec = {"bc": struct.unpack_from("<I", pay, 0)[0], "soft": np.frombuffer(pay[4:], dtype=np.int8).copy()}
        elif ty == REC_BLOCK:
            st, se, ang, pr, pi, cfo, start = struct.unpack("<iifffiq", pay[:32])
            rec = {"state": st, "samperr": se, "angle": ang, "phase": complex(pr, pi), "cfo": cfo, "start": start}
        elif ty == REC_L2:
            rec = parse_l2(pay)
            rec["frame_rec_off"] = rec["frame_off"] - 16      # where that frame's record starts in this drain
        elif ty in (10, 11):
            rec = {"dbg": struct.unpack("<%di" % (plen // 4), pay)}
        else:
            raise EngineError(f"corrupt record stream (type {ty} at {off})")
        out.append((ty, rec))
    return out


class Engine:
    """Many independent FM channels decoded on one GPU.

    push_cu8()/process()/drain() mirror input_push_cu8() and the downstream
    frame_push / pids_frame_push / nrsc5_report_* calls of the reference
    (see include/nrsc5_b200.h for the file:line map).
    """

    def __init__(self, nstreams: int, input_capacity: int, device: int = 0, log_capacity: int = 1 << 20,
                 emit_soft: bool = False, input_cs16=None, mode: str = "fm"):
        self._L = load_library()
        self._h = ctypes.c_void_p()
        if mode not in ("fm", "am"):
            raise EngineError("mode must be 'fm' or 'am'")
        am = mode == "am"
        # input format: FM defaults to cu8 at 1 488 375 S/s (input_cs16=True: cs16 at 744 187.5 S/s); AM defaults to
        # cs16 at 46 511.72 S/s (input_cs16=False: cu8 at 1 488 375 S/s, decimated by 32 on the device).
        # input_capacity is in bytes of what the receive chain keeps per stream: cu8 bytes (FM), cs16 bytes (FM cs16
        # and AM, whatever AM's input format)
        if input_cs16 is None:
            input_cs16 = am
        cfg = _Config(device, nstreams, int(am), input_capacity, log_capacity, int(emit_soft), int(bool(input_cs16)))
        _check(self._L.nrsc5b_create(ctypes.byref(self._h), ctypes.byref(cfg)), "nrsc5b_create")
        self.nstreams = nstreams
        self._log_cap = log_capacity + 64
        self._keep = []
        self.allow_overflow = False        # True: a truncated record log is not an error (tests of that very case)

    def close(self):
        if self._h:
            self._L.nrsc5b_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def set_cuda_stream(self, stream_ptr: int):
        _check(self._L.nrsc5b_set_cuda_stream(self._h, ctypes.c_void_p(stream_ptr)), "set_cuda_stream")

    def reset(self, stream: int = -1):
        _check(self._L.nrsc5b_reset(self._h, stream), "nrsc5b_reset")

    def rewind(self):
        _check(self._L.nrsc5b_rewind(self._h), "nrsc5b_rewind")

    def set_profiling(self, on: bool):
        _check(self._L.nrsc5b_set_profiling(self._h, int(on)), "nrsc5b_set_profiling")

    def kernel_times(self):
        ms = (ctypes.c_double * 4)()
        n = (ctypes.c_ulonglong * 4)()
        _check(self._L.nrsc5b_get_kernel_times(self._h, ms, n), "nrsc5b_get_kernel_times")
        # slot 1 = the stream-resident front-end kernel (k_stream), slot 3 = the P1 decode kernel group
        out = {"front": {"ms": ms[1], "launches": int(n[1])}, "p1": {"ms": ms[3], "launches": int(n[3])}}
        if n[2]:
            out["l2"] = {"ms": ms[2], "launches": int(n[2])}      # k_l2, only when L2 runs on the device
        return out

    def phase_cycles(self):
        """SM cycles per phase of k_stream summed over streams: {name: (cycles, count)}."""
        c = (ctypes.c_ulonglong * 12)()
        n = (ctypes.c_ulonglong * 12)()
        _check(self._L.nrsc5b_get_phase_cycles(self._h, c, n), "nrsc5b_get_phase_cycles")
        names = ["pids_flush", "prep_acquire", "prep_fine", "demod", "sync_fine", "sync_acquire",
                 "sync_fine.gather", "sync_fine.costas", "sync_fine.tables_feedback", "sync_fine.stage",
                 "sync_fine.equalise", "sync_fine.demap_tail"]
        return {k: (int(c[i]), int(n[i])) for i, k in enumerate(names)}

    def am_phase_cycles(self):
        c = (ctypes.c_ulonglong * 12)()
        _check(self._L.nrsc5b_get_am_phase_cycles(self._h, c), "nrsc5b_get_am_phase_cycles")
        names = ["window_acquire", "pass1_carrier", "pass2_bins", "sync_slicing", "pids", "p1_p3_interleaver", "of_which_p3_post",
                 "of_which_interleaver", "all_decodes_k9_recursion", "all_decodes_traceback", "window_load_fine_blocks", "traceback_repair_rounds"]
        return {k: int(c[i]) for i, k in enumerate(names)}

    def push_cu8(self, stream: int, samples):
        """samples: uint8 numpy array / bytes (host) — length counts uint8 values, multiple of 4."""
        a = np.ascontiguousarray(np.frombuffer(samples, dtype=np.uint8) if isinstance(samples, (bytes, bytearray)) else samples,
                                 dtype=np.uint8)
        _check(self._L.nrsc5b_push_cu8(self._h, stream, a.ctypes.data, a.size), "nrsc5b_push_cu8")

    def push_cu8_device(self, stream: int, dev_ptr: int, nbytes: int):
        _check(self._L.nrsc5b_push_cu8_device(self._h, stream, ctypes.c_void_p(dev_ptr), nbytes), "nrsc5b_push_cu8_device")

    def attach_device_input(self, dev_ptr: int, stride: int, nbytes: int):
        _check(self._L.nrsc5b_attach_device_input(self._h, ctypes.c_void_p(dev_ptr), stride, nbytes), "attach_device_input")

    def attach_device_log(self, dev_ptr: int, stride: int):
        _check(self._L.nrsc5b_attach_device_log(self._h, ctypes.c_void_p(dev_ptr), stride), "attach_device_log")
        self._log_cap = stride + 64

    def process(self):
        _check(self._L.nrsc5b_process(self._h), "nrsc5b_process")

    def process_available(self):
        _check(self._L.nrsc5b_process_available(self._h), "nrsc5b_process_available")

    def push_cs16(self, stream: int, samples):
        """samples: int16 numpy array (I, Q interleaved, 744 187.5 S/s); an engine made with input_cs16=True."""
        a = np.ascontiguousarray(samples, dtype=np.int16)
        _check(self._L.nrsc5b_push_cs16(self._h, stream, a.ctypes.data, a.size), "nrsc5b_push_cs16")

    def push_cu8_all(self, host_ptr: int, host_stride: int, nbytes: int):
        """nbytes for every stream from one page-locked slab (stream s at host_ptr + s*host_stride)."""
        _check(self._L.nrsc5b_push_cu8_all(self._h, ctypes.c_void_p(host_ptr), host_stride, nbytes), "nrsc5b_push_cu8_all")

    def push_fence(self) -> int:
        return _check(self._L.nrsc5b_push_fence(self._h), "nrsc5b_push_fence")

    def process_fence(self, token: int):
        _check(self._L.nrsc5b_process_fence(self._h, token), "nrsc5b_process_fence")

    # ---- asynchronous use (include/nrsc5_b200.h): staged input, one batch in flight, records exported to host memory
    def stage_cu8(self, stream: int, samples) -> int:
        """Returns 0, or -5 (EFULL: the device buffer is full of unused samples; the engine kept the rest - poll /
        submit and call stage_cu8(stream, b"") until it returns 0)."""
        a = np.ascontiguousarray(np.frombuffer(samples, dtype=np.uint8) if isinstance(samples, (bytes, bytearray)) else samples,
                                 dtype=np.uint8)
        rc = self._L.nrsc5b_stage_cu8(self._h, stream, a.ctypes.data if a.size else None, a.size)
        if rc != -5:
            _check(rc, "nrsc5b_stage_cu8")
        return rc

    def submit(self, flush: bool = False) -> int:
        return _check(self._L.nrsc5b_submit(self._h, int(flush)), "nrsc5b_submit")

    def poll(self, wait: bool = False) -> int:
        return _check(self._L.nrsc5b_poll(self._h, int(wait)), "nrsc5b_poll")

    def batch_records(self, stream: int):
        n = ctypes.c_size_t(0)
        ptr = self._L.nrsc5b_batch_records(self._h, stream, ctypes.byref(n))
        if self._L.nrsc5b_take_overflow(self._h, stream) and not self.allow_overflow:
            raise EngineError(f"stream {stream}: record log overflowed (log_capacity too small)")
        return parse_records(ctypes.string_at(ptr, n.value)) if ptr and n.value else []

    def synchronize(self):
        _check(self._L.nrsc5b_synchronize(self._h), "nrsc5b_synchronize")

    def drain_raw(self, stream: int) -> bytes:
        need = ctypes.c_size_t(0)
        buf = ctypes.create_string_buffer(self._log_cap)
        n = self._L.nrsc5b_drain(self._h, stream, buf, self._log_cap, ctypes.byref(need))
        _check(n, "nrsc5b_drain")
        if self._L.nrsc5b_take_overflow(self._h, stream) and not self.allow_overflow:
            raise EngineError(f"stream {stream}: record log overflowed (log_capacity too small); the drained records are a prefix")
        return buf.raw[:n]

    def drain(self, stream: int):
        return parse_records(self.drain_raw(stream))

    def drain_all_raw(self, out: np.ndarray = None):
        """Records of every stream in one call; `out` = optional (pinned) uint8 array [nstreams, stride]."""
        if out is None:
            out = np.empty((self.nstreams, self._log_cap), dtype=np.uint8)
        sizes = (ctypes.c_size_t * self.nstreams)()
        rc = self._L.nrsc5b_drain_all(self._h, out.ctypes.data, out.strides[0], sizes)
        if not (rc == -6 and self.allow_overflow):
            _check(rc, "nrsc5b_drain_all")
        return [out[s, :sizes[s]] for s in range(self.nstreams)]

    def drain_all(self):
        return [parse_records(r.tobytes()) for r in self.drain_all_raw()]

    def enable_l2(self, on: bool = True):
        """L2 framing on the device: every frame's REC_FRAME is followed (at the end of its pass) by a REC_L2."""
        _check(self._L.nrsc5b_enable_l2(self._h, int(on)), "nrsc5b_enable_l2")

    def set_sync_state(self, stream: int, state: int):
        _check(self._L.nrsc5b_set_sync_state(self._h, stream, state), "nrsc5b_set_sync_state")

    def stats(self) -> Stats:
        st = Stats()
        _check(self._L.nrsc5b_get_stats(self._h, ctypes.byref(st)), "nrsc5b_get_stats")
        return st


# ---- single-stage helpers (parity tests) ----
def halfband_fm(cu8: np.ndarray, device: int = 0) -> np.ndarray:
    a = np.ascontiguousarray(cu8, dtype=np.uint8)
    n = a.size // 4
    out = np.empty(2 * n, dtype=np.int16)
    _check(load_library().nrsc5b_halfband_fm(device, a.ctypes.data, n, out.ctypes.data), "nrsc5b_halfband_fm")
    return out


def viterbi_k7(soft: np.ndarray, length: int, device: int = 0, want_fallbacks: bool = False):
    """Batch of tail-biting K=7 decodes.  With want_fallbacks also returns how many frames the fast
    register-resident path handed to the exact fallback kernels."""
    s = np.ascontiguousarray(soft, dtype=np.int8)
    nframes = s.size // (3 * length)
    out = np.empty(nframes * length, dtype=np.uint8)
    fb = ctypes.c_int(0)
    _check(load_library().nrsc5b_viterbi_k7_ex(device, s.ctypes.data, out.ctypes.data, length, nframes, ctypes.byref(fb)),
           "nrsc5b_viterbi_k7_ex")
    out = out.reshape(nframes, length)
    return (out, fb.value) if want_fallbacks else out


def viterbi_k7_fast(soft: np.ndarray, length: int, chunk: int, device: int = 0):
    """The K=7 decoder's register-resident fast path alone, with chunks of `chunk` steps: its decision words
    [nframes][length + 64][2] (uint32) and its per-frame retry verdicts (True: it would hand the frame to the exact
    fallback)."""
    s = np.ascontiguousarray(soft, dtype=np.int8)
    nframes = s.size // (3 * length)
    dec = np.empty((nframes, length + 64, 2), dtype=np.uint32)
    retry = np.empty(nframes, dtype=np.int32)
    _check(load_library().nrsc5b_viterbi_k7_fast(device, s.ctypes.data, length, nframes, chunk, dec.ctypes.data,
                                                 retry.ctypes.data), "nrsc5b_viterbi_k7_fast")
    return dec, retry != 0


def l2_frames(frames, device: int = 0, cap: int = 64 << 20):
    """L2 alone: frames = [(lc, nbits, packed bits) | None (= frame_reset)] -> the REC_L2 records, one per frame."""
    blob = bytearray()
    for f in frames:
        if f is None:
            blob += struct.pack("<II", 0, 0)
        else:
            lc, nbits, bits = f
            nb = (nbits + 7) // 8
            blob += struct.pack("<II", lc, nbits) + bytes(bits[:nb]) + bytes((-nb) % 4)
    out = ctypes.create_string_buffer(cap)
    need = ctypes.c_size_t(0)
    n = load_library().nrsc5b_l2_frames(device, bytes(blob), len(blob), out, cap, ctypes.byref(need))
    _check(n, "nrsc5b_l2_frames")
    return [r for t, r in parse_records(out.raw[:n]) if t == REC_L2]


def rs_decode(blocks: np.ndarray, device: int = 0):
    b = np.ascontiguousarray(blocks, dtype=np.uint8).reshape(-1, 255).copy()
    rc = np.empty(b.shape[0], dtype=np.int32)
    _check(load_library().nrsc5b_rs_decode(device, b.ctypes.data, rc.ctypes.data, b.shape[0]), "nrsc5b_rs_decode")
    return rc, b


def viterbi_k9(sym: np.ndarray, gens=(0o561, 0o657, 0o711), warmup: int = 0, chunk_warmup: int = 0, device: int = 0):
    """The AM chain's K=9 decoder on a batch of frames: sym int8 [njobs, 3 * len] of -1 / 0 / +1; returns (bits uint8
    [njobs, len], repair rounds of the segmented traceback int32 [njobs], chunks of the recursion run again int32 [njobs])."""
    a = np.ascontiguousarray(sym, dtype=np.int8)
    a = a.reshape(1, -1) if a.ndim == 1 else a
    njobs, n = a.shape[0], a.shape[1] // 3
    out = np.empty((njobs, n), dtype=np.uint8)
    rounds = np.empty(njobs, dtype=np.int32)
    L = load_library()
    L.nrsc5b_viterbi_k9.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_uint,
                                    ctypes.c_uint, ctypes.c_uint, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    _check(L.nrsc5b_viterbi_k9(device, a.ctypes.data, out.ctypes.data, n, njobs, *gens, warmup, chunk_warmup, rounds.ctypes.data),
           "nrsc5b_viterbi_k9")
    return out, rounds & 0xffff, rounds >> 16


def fft2048(x: np.ndarray, device: int = 0) -> np.ndarray:
    a = np.ascontiguousarray(x, dtype=np.complex64).reshape(-1, 2048)
    out = np.empty_like(a)
    _check(load_library().nrsc5b_fft2048(device, a.ctypes.data, out.ctypes.data, a.shape[0]), "nrsc5b_fft2048")
    return out
