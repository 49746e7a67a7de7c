"""The K=7 fast path's decision words, step by step, against a sequential 64-state add-compare-select in numpy.

k_v64_fwd keeps the 64 path metrics in registers in a layout that changes from step to step and packs each step's
64 decisions into the fixed word format that k_v64_emit and the exact fallback read.  Decoded bits alone could hide
a misplaced decision that no survivor path happens to use; here every stored word of every accepted frame must
equal the sequential pass's.  The tests run on the GPU and, through the CPU emulation of the kernels
(tests/emu), on machines without one.
"""
import os
import sys

import numpy as np
import pytest

from nrsc5_b200 import engine as eng
from nrsc5_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
BIAS = 384                      # any common bias leaves the decisions unchanged; the fast path's is kept for clarity


def _parity(v):
    v = np.asarray(v)
    p = np.zeros_like(v)
    for k in range(7):
        p ^= (v >> k) & 1
    return p


def _branch_signs():
    """sign (+1/-1) with which soft value i enters the metric of the branch (state 2b, input 0), b = 0..31 (the
    expected code bits of src/conv_dec.c:139-154 with the polynomials 0133, 0171, 0165)"""
    reg = np.arange(32) << 1
    return np.stack([2 * _parity(reg & g) - 1 for g in (0o133, 0o171, 0o165)], axis=1)


def sequential_decisions(soft, length):
    """[nframes][3*length] int8 -> [nframes][length+64][2] uint32: one pass over length+64 steps from all-zero
    metrics, step g reading the soft triple of bit (g - 32) mod length; new state n = b + 32*x from predecessors
    2b (even) and 2b+1 (odd); the odd predecessor wins ties (src/conv_gen.h:47,55)."""
    soft = np.asarray(soft, dtype=np.int64).reshape(len(soft), length, 3)
    nf, total = soft.shape[0], length + 64
    sg = _branch_signs()                                         # [32][3]
    pm = np.zeros((nf, 64), dtype=np.int64)
    n = np.arange(64)
    word = (n >> 3) & 1
    bit = (8 * (n >> 4) + (n & 7)).astype(np.uint64)
    dec = np.zeros((nf, total, 2), dtype=np.uint32)
    for g in range(total):
        s = soft[:, (g - 32) % length, :]                        # [nf][3]
        mp = BIAS + s @ sg.T                                     # [nf][32]: branch (2b, input 0)
        mm = 2 * BIAS - mp                                       # the complementary code bits
        ev, od = pm[:, 0::2], pm[:, 1::2]
        x = np.concatenate([ev + mp, ev + mm], axis=1)           # even predecessor into new states b, b+32
        y = np.concatenate([od + mm, od + mp], axis=1)           # odd predecessor
        d = y >= x
        pm = np.where(d, y, x)
        pm -= pm.min(axis=1, keepdims=True)
        for w in (0, 1):
            sel = word == w
            dec[:, g, w] = (d[:, sel].astype(np.uint64) << bit[sel]).sum(axis=1).astype(np.uint32)
    return dec


@pytest.fixture(params=[pytest.param("gpu", marks=pytest.mark.gpu), "emu"])
def library(request):
    if request.param == "gpu":
        yield
        return
    sys.path.insert(0, os.path.join(HERE, "emu"))
    import build_emu
    so = build_emu.build()
    saved = (eng.lib_path, eng._lib)
    eng.lib_path = lambda: so
    eng._lib = None
    yield
    eng.lib_path, eng._lib = saved


def _encoded(rng, length, amp, sigma):
    u = rng.integers(0, 2, length, dtype=np.uint8)
    c = synth.conv_encode_tb(u).reshape(-1).astype(np.float64)
    s = np.clip((2 * c - 1) * amp + (rng.normal(0, sigma, c.size) if sigma else 0), -127, 127).astype(np.int8)
    s[5::6] = 0                                                  # punctured positions, as the P1 depuncturer leaves them
    return s


def _check(soft, length, chunks):
    ref = sequential_decisions(soft, length)
    for ch in chunks:
        dec, retry = eng.viterbi_k7_fast(soft, length, ch)
        assert not retry.any(), (ch, retry)
        for f in range(len(soft)):
            bad = np.nonzero((dec[f] != ref[f]).any(axis=1))[0]
            assert bad.size == 0, f"chunk {ch}, frame {f}: first differing step {bad[:1]} of {bad.size}"


def test_p1_frames_clean_and_noisy(library):
    rng = np.random.default_rng(11)
    length = 146176
    soft = np.stack([_encoded(rng, length, 60, 0), _encoded(rng, length, 40, 40)])
    # 1152: the chunk length 128 streams get on an H100; 1376: a last chunk of 128 steps
    _check(soft, length, (1152, 1376))


def test_p3_frame(library):
    rng = np.random.default_rng(12)
    length = 4608
    soft = np.stack([_encoded(rng, length, 40, 40), _encoded(rng, length, 30, 35)])
    # 256: the extended-partition groups' chunk; 352 and 800 leave partial last chunks of 96 and 672 steps
    _check(soft, length, (256, 352, 800))


def test_retry_verdicts(library):
    """Metrics that could saturate the reference's int16 arithmetic are handed to the exact fallback.  Pure noise
    is handed over where the chunks' metric vectors or survivors did not converge - the verdicts below are the
    ones the kernels gave before the metric layouts changed - and where it is not, its decisions are exact too."""
    length = 4608
    u = np.random.default_rng(13).integers(0, 2, length, dtype=np.uint8)
    full = ((2 * synth.conv_encode_tb(u).reshape(-1).astype(np.int16) - 1) * 127).astype(np.int8)
    noise = [np.random.default_rng(seed).integers(-127, 128, 3 * length).astype(np.int8) for seed in range(100, 105)]
    soft = np.stack([full] + noise)
    ref = sequential_decisions(soft, length)
    expect = {256: [True, True, True, False, False, True], 1024: [True, True, True, False, False, False]}
    for ch, verdicts in expect.items():
        dec, retry = eng.viterbi_k7_fast(soft, length, ch)
        assert retry.tolist() == verdicts, ch
        for f in np.nonzero(~retry)[0]:
            assert np.array_equal(dec[f], ref[f]), (ch, f)
