"""TEST INFRASTRUCTURE ONLY.  The channeliser's definition for either band plan and either sample format
(include/nrsc5_b200.h) restated in numpy, one-shot and streamed: exact integer arithmetic on the tables the library
publishes.  The filter length is the tap table's (256: FM plan, 512: AM plan); the mixer step is the plan's (1600 m_k
for FM, 2560 m_k for AM).  With the FM parameters it is oracle/chan_oracle.py and tests/chan_oracle_cs16.py."""
import numpy as np

PERIOD, DECIM = 11907, 32
MIX_AM = 2560
BLOCK = 4096                                                                       # outputs gathered at a time


def outputs_of(samples: int, ntaps: int) -> int:
    """N(T): outputs whose ntaps-sample windows lie within the first T complex samples."""
    return (samples - ntaps) // DECIM + 1 if samples >= ntaps else 0


def channelize(x: np.ndarray, offsets, taps: np.ndarray, phasor: np.ndarray, mix_step: int = MIX_AM, n0: int = 0) -> np.ndarray:
    """x: uint8 (cu8) or int16 (cs16), I/Q interleaved, whole complex samples -> int16 [nch][2 * nout].  n0: index of
    the first output when x is a slice of a longer capture starting at its sample 32 * n0 (the mixer runs on)."""
    a = np.asarray(x).reshape(-1)
    assert a.dtype in (np.uint8, np.int16) and a.size % 2 == 0
    cu8 = a.dtype == np.uint8
    ntaps = taps.shape[1]
    nout = outputs_of(a.size // 2, ntaps)
    xr = a[0::2].astype(np.int64) - (127 if cu8 else 0)
    xi = a[1::2].astype(np.int64) - (127 if cu8 else 0)
    out = np.zeros((len(offsets), 2 * max(nout, 0)), dtype=np.int16)
    # float64 holds these sums exactly (products below 2^30, 512 of them below 2^39 < 2^53) and multiplies much faster
    wr = taps[:, :, 0].astype(np.float64).T                                        # [ntaps][nch]
    wi = taps[:, :, 1].astype(np.float64).T
    step = np.array([(mix_step * int(m)) % PERIOD for m in offsets], dtype=np.int64)
    for b0 in range(0, nout, BLOCK):
        nb = min(BLOCK, nout - b0)
        idx = (np.arange(b0, b0 + nb)[:, None] * DECIM + np.arange(ntaps)[None, :])
        XR, XI = xr[idx].astype(np.float64), xi[idx].astype(np.float64)
        ar = (XR @ wr - XI @ wi).astype(np.int64)                                  # |acc| < 2^36
        ai = (XI @ wr + XR @ wi).astype(np.int64)
        if cu8:
            vr, vi = (ar + (1 << 12)) >> 13, (ai + (1 << 12)) >> 13
        else:
            vr = np.clip((ar + (1 << 18)) >> 19, -32768, 32767)
            vi = np.clip((ai + (1 << 18)) >> 19, -32768, 32767)
        n = np.arange(b0, b0 + nb, dtype=np.int64) + int(n0)
        q = (step[None, :] * (n % PERIOD)[:, None]) % PERIOD                       # [nb][nch]
        pr = phasor[q, 0].astype(np.int64)
        pi = phasor[q, 1].astype(np.int64)
        zr = (vr * pr + vi * pi + (1 << 14)) >> 15                                # v * conj(P)
        zi = (vi * pr - vr * pi + (1 << 14)) >> 15
        out[:, 2 * b0: 2 * (b0 + nb): 2] = np.clip(zr, -32768, 32767).astype(np.int16).T
        out[:, 2 * b0 + 1: 2 * (b0 + nb): 2] = np.clip(zi, -32768, 32767).astype(np.int16).T
    return out


def channelize_stream(chunks, offsets, taps: np.ndarray, phasor: np.ndarray, mix_step: int = MIX_AM):
    """The streaming form (nrsc5b_chan_push*): the capture arrives as `chunks` (each of even length, any of them
    empty).  A handle keeps T, the samples pushed so far, and the carry, the samples from 32 N(T) on; a push taking T
    to T' emits outputs N(T) .. N(T') - 1, computed from carry + chunk with the mixer at the absolute index N(T), and
    keeps the samples from 32 N(T') on (at most ntaps - 1).  Returns one int16 [nch][2 * n] array per push."""
    ntaps = taps.shape[1]
    carry, pushed, outs = None, 0, []
    for chunk in chunks:
        c = np.asarray(chunk).reshape(-1)
        assert c.size % 2 == 0, "pushes are whole complex samples"
        first, last = outputs_of(pushed, ntaps), outputs_of(pushed + c.size // 2, ntaps)
        held = c if carry is None else np.concatenate([carry, c])                 # starts at sample 32 N(T)
        n = last - first
        outs.append(channelize(held[: 2 * (DECIM * n + ntaps - DECIM)] if n > 0 else held[:0], offsets, taps, phasor, mix_step, n0=first))
        pushed += c.size // 2
        carry = held[2 * DECIM * n:]
        assert carry.size == 2 * (pushed - DECIM * last) <= 2 * (ntaps - 1)
    return outs
