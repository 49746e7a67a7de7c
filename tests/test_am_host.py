"""The AM engine's code (nrsc5_b200/csrc/am.cuh, AM_HD functions) compiled for the CPU and run with one lane
(tests/am_host.cu) against the oracle and the golden vectors, and with the 32 lanes of the GPU warp emulated by fibres:
the same source the GPU runs."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import common
import port
import reftap
from nrsc5_b200 import synth_am

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "_build", "libam_host.so")

pytestmark = pytest.mark.skipif(not port.available(), reason="oracle/_ref/liboracle.so not built")


def _lib():
    src = [os.path.join(HERE, "am_host.cu"), os.path.join(common.ROOT, "nrsc5_b200", "csrc", "am.cuh"),
           os.path.join(common.ROOT, "nrsc5_b200", "csrc", "am_tables.h")]
    if not os.path.exists(SO) or any(os.path.getmtime(p) > os.path.getmtime(SO) for p in src):
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "--expt-extended-lambda", "--expt-relaxed-constexpr", "-O2", "-shared", "-Xcompiler", "-fPIC", "-o", SO,
                        src[0], "-L" + os.path.join(common.ROOT, "oracle", "_ref"), "-loracle",
                        "-Xlinker", "-rpath", "-Xlinker", os.path.join(common.ROOT, "oracle", "_ref")], check=True)
    L = ctypes.CDLL(SO)
    L.am_host_decode.restype = ctypes.c_long
    L.am_host_decode.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t]
    L.am_host_decode_lanes.restype = ctypes.c_long
    L.am_host_decode_lanes.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int,
                                       ctypes.c_int]
    L.am_host_decimate.restype = ctypes.c_long
    L.am_host_decimate.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_uint, ctypes.c_size_t, ctypes.c_int,
                                   ctypes.c_int]
    return L


def host_decimate(cu8, ring_bytes=1 << 16, chunk=1 << 15, lanes=1, order=1):
    a = np.ascontiguousarray(cu8, dtype=np.uint8)
    out = np.zeros(2 * (a.size // 64), dtype=np.int16)
    n = _lib().am_host_decimate(a.ctypes.data, a.size, out.ctypes.data, ring_bytes, chunk, lanes, order)
    assert n != -3, "lanes met at different barriers"
    assert n == a.size // 64
    return out


def host_decode(cs16, lanes=1, order=1):
    a = np.ascontiguousarray(cs16, dtype=np.int16)
    buf = ctypes.create_string_buffer(8 << 20)
    if lanes == 1:
        n = _lib().am_host_decode(a.ctypes.data, a.size & ~1, buf, len(buf))
    else:
        n = _lib().am_host_decode_lanes(a.ctypes.data, a.size & ~1, buf, len(buf), lanes, order)
    assert n != -2, "lanes ended with different private AmState copies"
    assert n != -3, "lanes met at different AM_SYNC() sites"
    assert n >= 0
    return reftap._parse(buf.raw[:n])


@pytest.mark.parametrize("name", list(common.AM_CASES))
def test_am_engine_code_on_host_matches_oracle(name):
    cap = synth_am.make_am_ma1(**common.AM_CASES[name])
    got = host_decode(cap.cs16)
    ref = port.decode_am(cap.cs16)
    assert common.summarize(got) == common.summarize(ref)


@pytest.mark.parametrize("name,order", [("ma1_noisy", 1), ("ma3_noisy", -1)])
def test_am_engine_code_with_32_emulated_lanes(name, order):
    """k_am's warp emulated by 32 fibres (tests/am_host.cu): the lane-strided work split and the placement of the
    AM_SYNC() barriers, with the lanes scheduled in ascending and in descending order."""
    cap = synth_am.make_am_ma1(**common.AM_CASES[name])
    got = host_decode(cap.cs16, lanes=32, order=order)
    ref = port.decode_am(cap.cs16)
    assert common.summarize(got) == common.summarize(ref)


@pytest.mark.parametrize("lanes,order,chunk", [(1, 1, 1 << 15), (256, 1, 40004), (256, -1, 4), (96, 1, 60000)])
def test_am_cu8_front_end_on_host(lanes, order, chunk):
    """decim_tile (five cascaded halfband stages, cu8 -> cs16 / 32) with the engine's ring and tiling arithmetic
    against the oracle's restatement of input_push_cu8 (reference src/input.c:52-117), on random bytes - which
    drive the int16 accumulators into wrap-around - and on a real AM capture."""
    rng = np.random.default_rng(21)
    noise = rng.integers(0, 256, 64 * 3000 + 36, dtype=np.uint8)
    cap = synth_am.make_am_ma1(nframes=1, seed=2, lead_in=100, carrier=8000.0, unit=40.0)
    sig = synth_am.am_to_cu8(cap.cs16[: 2 * 4000])
    for x in (noise, sig):
        want = port.decimate_am(x)
        got = host_decimate(x, ring_bytes=1 << 16, chunk=chunk, lanes=lanes, order=order)
        assert np.array_equal(got, want[: got.size]) and got.size == want.size
