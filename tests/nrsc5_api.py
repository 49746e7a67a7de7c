"""Minimal ctypes driver of the reference's PUBLIC API (reference include/nrsc5.h: nrsc5_open_pipe,
nrsc5_set_callback, nrsc5_pipe_samples_cu8, nrsc5_close) - test infrastructure.  It is pointed either at
the unmodified reference (oracle/_ref/libnrsc5_ref.so) or at the drop-in built on the CUDA engine
(nrsc5_b200/dropin/_build/libnrsc5.so) and digests the events both deliver through the same callback.

Event layout (nrsc5.h:369-613): `unsigned int event` followed by a union aligned to 8 bytes.
"""
import ctypes
import struct

EV = {0: "LOST_DEVICE", 1: "IQ", 2: "SYNC", 3: "LOST_SYNC", 4: "MER", 5: "BER", 6: "HDC", 7: "AUDIO", 8: "ID3",
      9: "SIG", 10: "LOT", 11: "SIS", 12: "STREAM", 13: "PACKET", 14: "AUDIO_SERVICE", 15: "STATION_ID",
      16: "STATION_NAME", 17: "STATION_SLOGAN", 18: "STATION_MESSAGE", 19: "STATION_LOCATION", 20: "ASD",
      21: "DSD", 22: "EMERGENCY_ALERT", 23: "HERE_IMAGE", 24: "LOT_HEADER", 25: "LOT_FRAGMENT", 26: "AGC",
      27: "EXCITER_INFO", 28: "IMPORTER_INFO", 29: "LEAP_SECOND_OFFSET", 30: "LOCAL_TIME"}

CALLBACK = ctypes.CFUNCTYPE(None, ctypes.c_void_p, ctypes.c_void_p)


def fnv1a32(b: bytes) -> int:
    h = 0x811C9DC5
    for x in b:
        h = ((h ^ x) * 0x01000193) & 0xFFFFFFFF
    return h


def run(lib_path: str, cu8: bytes, chunk: int = 32768, cs16: bool = False, am: bool = False):
    """Decode `cu8` through the public API in `chunk`-byte pushes (main.c:1097-1119 uses 32768);
    returns the event digest list, IQ events left out.  With cs16=True the bytes are int16 I/Q at the
    decimated rate and go through nrsc5_pipe_samples_cs16 (whose length counts int16 values).  am=True selects
    NRSC5_MODE_AM (nrsc5_set_mode, nrsc5.h:84-85) before the first push."""
    L = ctypes.CDLL(lib_path)
    L.nrsc5_open_pipe.argtypes = [ctypes.POINTER(ctypes.c_void_p)]
    L.nrsc5_set_callback.argtypes = [ctypes.c_void_p, CALLBACK, ctypes.c_void_p]
    L.nrsc5_pipe_samples_cu8.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint]
    L.nrsc5_pipe_samples_cs16.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint]
    L.nrsc5_close.argtypes = [ctypes.c_void_p]
    events = []

    def on_event(evt, _opaque):
        ty = ctypes.c_uint.from_address(evt).value
        if ty == 1:
            return
        name = EV.get(ty, str(ty))
        u = evt + 8
        if name == "SYNC":
            fo, psmi, pli, hppi, aabi, rdbi = struct.unpack("<fiiiii", ctypes.string_at(u, 24))
            events.append([name, round(fo, 2), psmi, pli, hppi, aabi, rdbi])
        elif name == "MER":
            lo, up = struct.unpack("<ff", ctypes.string_at(u, 8))
            events.append([name, round(lo, 3), round(up, 3)])
        elif name == "BER":
            events.append([name, round(struct.unpack("<f", ctypes.string_at(u, 4))[0], 6)])
        elif name == "HDC":
            program, = struct.unpack("<I", ctypes.string_at(u, 4))
            data, count = struct.unpack("<QQ", ctypes.string_at(u + 8, 16))
            events.append([name, program, count, fnv1a32(ctypes.string_at(data, count))])
        else:
            events.append([name])

    cb = CALLBACK(on_event)
    h = ctypes.c_void_p()
    rc = L.nrsc5_open_pipe(ctypes.byref(h))
    assert rc == 0, "nrsc5_open_pipe failed"
    L.nrsc5_set_callback(h, cb, None)
    if am:
        L.nrsc5_set_mode.argtypes = [ctypes.c_void_p, ctypes.c_int]
        assert L.nrsc5_set_mode(h, 1) == 0
    buf = ctypes.create_string_buffer(bytes(cu8), len(cu8))
    base = ctypes.addressof(buf)
    for off in range(0, len(cu8), chunk):
        n = min(chunk, len(cu8) - off)
        if cs16:
            L.nrsc5_pipe_samples_cs16(h, base + off, n // 2)
        else:
            L.nrsc5_pipe_samples_cu8(h, base + off, n)
    L.nrsc5_close(h)
    return events
