"""TEST INFRASTRUCTURE ONLY.  The channeliser's cs16 definition (include/nrsc5_b200.h, nrsc5b_chan_create_cs16)
restated in numpy, one-shot and streamed: exact integer arithmetic on the tables the library publishes
(nrsc5b_chan_make_tables), the same tables, rotation and output rounding as the cu8 restatement in
oracle/chan_oracle.py."""
import numpy as np

from chan_oracle import DECIM, PERIOD, TAPS


def channelize_cs16(cs16: np.ndarray, offsets, taps: np.ndarray, phasor: np.ndarray, n0: int = 0) -> np.ndarray:
    """The cs16 definition (include/nrsc5_b200.h, nrsc5b_chan_create_cs16): int16 I/Q interleaved (even length) ->
    int16 [nch][2 * nout]; acc = sum W x (no offset), v = sat16((acc + 2^18) >> 19), then the cu8 rotation.  n0 as in
    channelize."""
    a = np.asarray(cs16, dtype=np.int16).reshape(-1)
    assert a.size % 2 == 0, "whole complex samples"
    ns = a.size // 2
    nout = (ns - TAPS) // DECIM + 1 if ns >= TAPS else 0
    xr = a[0::2].astype(np.int64)
    xi = a[1::2].astype(np.int64)
    out = np.zeros((len(offsets), 2 * max(nout, 0)), dtype=np.int16)
    if nout <= 0:
        return out
    idx = (np.arange(nout)[:, None] * DECIM + np.arange(TAPS)[None, :])
    XR, XI = xr[idx], xi[idx]
    n = np.arange(nout, dtype=np.int64) + int(n0)
    for k, m in enumerate(offsets):
        wr = taps[k, :, 0].astype(np.int64)
        wi = taps[k, :, 1].astype(np.int64)
        ar = XR @ wr - XI @ wi                                                     # |acc| < 2^36: exact in int64
        ai = XI @ wr + XR @ wi
        vr = np.clip((ar + (1 << 18)) >> 19, -32768, 32767)
        vi = np.clip((ai + (1 << 18)) >> 19, -32768, 32767)
        step = (1600 * int(m)) % PERIOD
        q = (step * (n % PERIOD)) % PERIOD
        pr = phasor[q, 0].astype(np.int64)
        pi = phasor[q, 1].astype(np.int64)
        zr = (vr * pr + vi * pi + (1 << 14)) >> 15                                # v * conj(P)
        zi = (vi * pr - vr * pi + (1 << 14)) >> 15
        out[k, 0::2] = np.clip(zr, -32768, 32767).astype(np.int16)
        out[k, 1::2] = np.clip(zi, -32768, 32767).astype(np.int16)
    return out


def channelize_cs16_stream(chunks, offsets, taps: np.ndarray, phasor: np.ndarray):
    """The streaming form of channelize_cs16 (nrsc5b_chan_push_cs16): the capture arrives as `chunks` (int16, each of
    even length, any of them empty).  A handle keeps T, the samples pushed so far, and the carry, the samples from
    32 N(T) on; a push taking T to T' emits outputs N(T) .. N(T') - 1, computed from carry + chunk with the mixer at the
    absolute index N(T), and keeps the samples from 32 N(T') on.  Returns one int16 [nch][2 * n] array per push."""
    def outputs_of(t):
        return (t - TAPS) // DECIM + 1 if t >= TAPS else 0
    carry = np.zeros(0, dtype=np.int16)
    pushed = 0
    outs = []
    for chunk in chunks:
        c = np.asarray(chunk, dtype=np.int16).reshape(-1)
        assert c.size % 2 == 0, "pushes are whole complex samples"
        first, last = outputs_of(pushed), outputs_of(pushed + c.size // 2)
        held = np.concatenate([carry, c])                                          # starts at sample 32 N(T)
        n = last - first
        outs.append(channelize_cs16(held[: 2 * (DECIM * n + TAPS - DECIM)] if n > 0 else held[:0], offsets, taps, phasor, n0=first))
        pushed += c.size // 2
        carry = held[2 * DECIM * n:]
        assert carry.size == 2 * (pushed - DECIM * last) <= 510
    return outs
