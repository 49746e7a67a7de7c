"""The K=7 fast path's saturation guard at its limit, against the reference's int16 arithmetic restated in numpy.

The reference adds path metrics in saturating int16 and subtracts their minimum after every step whose index is
0 mod 79 (src/conv_dec.c:419, conv_sse.h:56-66).  k_v64_fwd never saturates, so its decisions are the reference's
only while no metric can reach 32767 between two of those normalisations: right after one the spread is at most
12*381, so a window of steps whose soft magnitudes sum to at most 32767 - 12*381 = 28195 is safe, and a frame with
a window above that must be flagged `retry` and go to the exact fallback.  Here single windows are driven to 28195
and 28196 at every phase of the normalisation inside the fast path's 8-step groups, across the tail-biting seam,
inside and across chunk starts, and at the end of the frame.  Accepted frames must give exactly the saturating
pass's decision words, and every frame's decoded bits must equal the oracle's.  The tests run on the GPU and,
through the CPU emulation of the kernels (tests/emu), on machines without one.
"""
import os
import sys

import numpy as np
import pytest

import port
from nrsc5_b200 import engine as eng
from nrsc5_b200 import synth
from test_viterbi_decisions import _branch_signs, sequential_decisions

HERE = os.path.dirname(os.path.abspath(__file__))
NORM = 79                       # the reference normalises after every step whose index is 0 mod NORM
LIMIT = 32767 - 12 * 381        # largest window sum that cannot saturate: 28195
TARGETS = (LIMIT, LIMIT + 1)


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


def window_sums(soft, length):
    """Sum of |s0|+|s1|+|s2| over the steps of each normalisation window of one frame.  Window k holds the steps
    79(k-1)+1 .. 79k, the ones after a normalisation up to and including the next, cut to the frame's steps
    0 .. length+63; step g reads the triple of bit (g - 32) mod length.  These are the windows k_vitc_fwd checks."""
    a = np.abs(np.asarray(soft, dtype=np.int64).reshape(length, 3)).sum(axis=1)
    g = np.arange(length + 64)
    return np.bincount((g + NORM - 1) // NORM, weights=a[(g - 32) % length]).astype(np.int64)


def could_saturate(soft, length):
    return bool((window_sums(soft, length) > LIMIT).any())


def decision_words(d):
    """[..., 64] bool (set = the survivor of new state n comes from the odd predecessor) -> [..., 2] uint32 in the
    fast path's format, the one sequential_decisions writes: the bit of state n is bit 8*(n>>4) + (n&7) of word
    (n>>3)&1."""
    n = np.arange(64)
    weight = np.zeros((64, 2), dtype=np.uint64)
    weight[n, (n >> 3) & 1] = np.uint64(1) << (8 * (n >> 4) + (n & 7)).astype(np.uint64)
    return (d.astype(np.uint64) @ weight).astype(np.uint32)


def saturating_pass(soft, length):
    """[nframes][3*length] int8 -> (decision words [nframes][length+64][2] uint32, path metrics after the last step
    [nframes][64], whether any add saturated [nframes]): the reference's pass in its own arithmetic.  Every add
    saturates to int16, the minimum is subtracted (saturating) after every step whose index is 0 mod 79, and the
    decisions follow sequential_decisions: the odd predecessor wins ties, in the same word format."""
    soft = np.asarray(soft, dtype=np.int64).reshape(-1, length, 3)
    nf, total = soft.shape[0], length + 64
    steps = np.arange(total)
    m = soft[:, (steps - 32) % length, :] @ _branch_signs().T   # [nf][total][32]: branch (2b, input 0)
    pm = np.zeros((nf, 64), dtype=np.int64)
    d = np.empty((nf, total, 64), dtype=bool)
    saturated = np.zeros(nf, dtype=bool)

    def sat(v):
        c = np.clip(v, -32768, 32767)
        saturated[:] |= (c != v).any(axis=1)
        return c

    for g in range(total):
        ev, od, mg = pm[:, 0::2], pm[:, 1::2], m[:, g]
        x = sat(np.concatenate([ev + mg, ev - mg], axis=1))    # even predecessor into new states b, b+32
        y = sat(np.concatenate([od - mg, od + mg], axis=1))    # odd predecessor
        d[:, g] = y >= x
        pm = np.maximum(x, y)
        if g % NORM == 0:
            pm = sat(pm - pm.min(axis=1, keepdims=True))
    return decision_words(d), pm, saturated


def traceback(dec, pm, length):
    """Decoded bits from decision words and the last step's metrics: from the first maximum, as the reference."""
    nf, total = dec.shape[0], length + 64
    state = np.argmax(pm, axis=1)
    out = np.zeros((nf, length), dtype=np.uint8)
    rows = np.arange(nf)
    for g in range(total - 1, -1, -1):
        if 32 <= g < 32 + length:
            out[:, g - 32] = (state >> 5) & 1
        word = dec[rows, g, (state >> 3) & 1].astype(np.int64)
        state = ((state << 1) & 62) | ((word >> (8 * (state >> 4) + (state & 7))) & 1)
    return out


def frame(length, k, target, seed, amp=40, margin=300):
    """A clean tail-biting codeword at amplitude `amp` with the punctured positions (5::6) zero, except that the
    triples read by the steps of window k get magnitudes summing to exactly `target`.  Every other window stays at
    least `margin` under the limit."""
    rng = np.random.default_rng(seed)
    u = rng.integers(0, 2, length, dtype=np.uint8)
    sign = 2 * synth.conv_encode_tb(u).reshape(-1).astype(np.int64) - 1
    soft = sign * amp
    soft[5::6] = 0
    steps = np.arange(max(0, NORM * (k - 1) + 1), min(length + 64, NORM * k + 1))
    bits = (steps - 32) % length
    assert np.unique(bits).size == bits.size
    idx = (3 * bits[:, None] + np.arange(3)).reshape(-1)
    mag = np.full(idx.size, target // idx.size)
    mag[:target % idx.size] += 1
    assert mag.max() <= 127, "the window is too short for this target"
    soft[idx] = sign[idx] * mag
    soft = soft.astype(np.int8)
    ws = window_sums(soft, length)
    assert ws[k] == target, (k, ws[k], target)
    assert np.delete(ws, k).max() <= LIMIT - margin, (k, np.delete(ws, k).max())
    return soft


def last_window(length):
    """index k of a frame's last window, the one no normalisation closes"""
    return (length + 63 + NORM - 1) // NORM


def check(soft, length, chunks, want_retry):
    """The fast path's verdicts at every chunk length, its decision words on every accepted frame, and the whole
    decoder's bits on every frame"""
    soft = np.stack(soft)
    want_retry = np.asarray(want_retry)
    assert [could_saturate(s, length) for s in soft] == want_retry.tolist()
    dec_ref, _, _ = saturating_pass(soft, length)
    for ch in chunks:
        dec, retry = eng.viterbi_k7_fast(soft, length, ch)
        assert retry.tolist() == want_retry.tolist(), ch
        for f in np.nonzero(~retry)[0]:
            bad = np.nonzero((dec[f] != dec_ref[f]).any(axis=1))[0]
            assert bad.size == 0, f"chunk {ch}, frame {f}: first differing step {bad[:1]} of {bad.size}"
    got, fallbacks = eng.viterbi_k7(soft, length, want_fallbacks=True)
    for f in range(len(soft)):
        assert np.array_equal(got[f], port.viterbi(soft[f])), f
    if length >= 2048:                                         # shorter frames do not use the fast path
        assert fallbacks == want_retry.sum()


def test_saturating_pass_matches_oracle():
    """The restatement decodes the oracle's bits on frames that saturate and on frames that do not, and where nothing
    saturates its decision words are the plain sequential pass's."""
    length = 2304
    rng = np.random.default_rng(21)
    u = rng.integers(0, 2, length, dtype=np.uint8)
    code = 2 * synth.conv_encode_tb(u).reshape(-1).astype(np.int64) - 1
    noisy = np.clip(code * 50 + rng.normal(0, 45, code.size), -127, 127).astype(np.int8)
    noisy[5::6] = 0
    full = (code * 127).astype(np.int8)
    flipped = np.where(rng.random(code.size) < 0.01, -full, full)   # full scale, 1% of the signs wrong
    rand = rng.integers(-127, 128, 3 * length).astype(np.int8)
    soft = np.stack([noisy, full, flipped, rand])
    dec, pm, saturated = saturating_pass(soft, length)
    assert saturated.tolist() == [False, True, True, False]
    bits = traceback(dec, pm, length)
    for f in range(len(soft)):
        assert np.array_equal(bits[f], port.viterbi(soft[f])), f
    plain = sequential_decisions(soft, length)
    assert np.array_equal(dec[~saturated], plain[~saturated])
    for f in np.nonzero(saturated)[0]:                         # and where it does, it changes decisions
        assert not np.array_equal(dec[f], plain[f]), f


def test_window_at_every_group_phase(library):
    """The window that goes over closes with a normalisation at each of the 8 positions of an 8-step group"""
    length = 4608
    ks = range(8, 16)                                          # 79k mod 8 takes every value 0..7
    assert sorted(NORM * k % 8 for k in ks) == list(range(8))
    soft = [frame(length, k, t, seed=k) for k in ks for t in TARGETS]
    check(soft, length, (256, 1152), [t > LIMIT for k in ks for t in TARGETS])


def test_window_across_tail_biting_seam(library):
    """Window 1 (steps 1..79) reads bits len-31..len-1 and 0..47, most of which the frame's last steps read again"""
    for length in (2304, 4608):
        soft = [frame(length, 1, t, seed=length) for t in TARGETS]
        check(soft, length, (256, 1152), [False, True])


@pytest.mark.parametrize("ch", [256, 1152])
def test_window_at_chunk_start(library, ch):
    """A window inside the warm-up of the next chunk, and one that straddles the chunk's first step"""
    length = 4608
    start = ch                                                  # the first step of chunk 1
    straddle = (start + NORM - 1) // NORM                       # holds steps start - 1 and start
    inside = straddle - 1
    assert NORM * (straddle - 1) < start - 1 and NORM * inside - NORM + 1 >= start - 256
    soft = [frame(length, k, t, seed=k) for k in (inside, straddle) for t in TARGETS]
    check(soft, length, (ch,), [False, True, False, True])


def test_last_window_can_go_over(library):
    """MP2's short P3 (2304 bits): the last window has 76 steps (2292..2367), up to 76*381 = 28956"""
    length = 2304
    k = last_window(length)
    assert NORM * (k - 1) + 1 == 2292
    targets = (LIMIT, LIMIT + 1, 28500, 76 * 381)
    soft = [frame(length, k, t, seed=k + t) for t in targets]
    check(soft, length, (32, 256, 1152), [t > LIMIT for t in targets])


@pytest.mark.parametrize("length, chunks", [(80, ()), (4608, (32, 256)), (146176, (1024, 1152))])
def test_last_window_full_scale_is_safe(library, length, chunks):
    """PIDS (80 bits, a 64-step last window), the 4608-bit partitions and P1 (10 steps each) cannot go over in their
    last window: full scale there must not be flagged.  PIDS frames are not a multiple of 32 bits and never take the
    fast path; they are decoded end to end only."""
    k = last_window(length)
    nsteps = length + 64 - NORM * (k - 1) - 1
    assert nsteps == (64 if length == 80 else 10)
    check([frame(length, k, 381 * nsteps, seed=length)], length, chunks, [False])
