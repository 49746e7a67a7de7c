"""TEST INFRASTRUCTURE ONLY.  The channeliser's rate stage (include/nrsc5_b200.h: nrsc5b_chan_create_rate) restated in
numpy, one-shot and streamed: y from G, L and M in exact int64, then the plan's own restatement on y
(tests/chan_oracle_rates.py for FM, tests/chan_oracle_am.py for AM), the plan running its cs16 definition.

    b_n = floor(n M / L),  p_n = n M mod L
    y[n] = sat16((sum_{j<64} G[p_n][j] x[b_n + j] + 2^13) >> 14)      (cu8: x = 64 (x8 - 127))
    K(T) = T >= 64 ? ((T - 63) L - 1) // M + 1 : 0"""
import numpy as np

import chan_oracle_am
import chan_oracle_rates

J = 64
BLOCK = 8192                                                                       # outputs gathered at a time


def resampled_of(samples: int, L: int, M: int) -> int:
    """K(T): resampled samples whose 64-sample windows lie within the first T input samples."""
    return ((samples - J + 1) * L - 1) // M + 1 if samples >= J else 0


def _as_cs16(x):
    a = np.asarray(x).reshape(-1)
    assert a.dtype in (np.uint8, np.int16) and a.size % 2 == 0
    return a.astype(np.int64) if a.dtype == np.int16 else 64 * (a.astype(np.int64) - 127)


def resample(x, G: np.ndarray, L: int, M: int, n0: int = 0, nout=None, b0: int = 0) -> np.ndarray:
    """x: uint8 (cu8) or int16 (cs16), I/Q interleaved -> int16 y[2 nout], I/Q interleaved.  The outputs are n0 ..
    n0 + nout - 1 of a capture whose sample b0 is x's sample 0 (nout None: every output x completes, from n0 on)."""
    a = _as_cs16(x)
    xr, xi = a[0::2], a[1::2]
    if nout is None:
        nout = resampled_of(xr.size + b0, L, M) - n0
    g = G.astype(np.int64)
    y = np.empty(2 * max(nout, 0), dtype=np.int16)
    for c0 in range(0, nout, BLOCK):
        n = np.arange(n0 + c0, n0 + min(nout, c0 + BLOCK), dtype=np.int64)
        q = n * M
        b, p = q // L - b0, q % L
        idx = b[:, None] + np.arange(J)[None, :]
        gp = g[p]
        for part, v in ((0, xr), (1, xi)):
            acc = (gp * v[idx]).sum(axis=1)
            y[2 * c0 + part: 2 * (c0 + n.size): 2] = np.clip((acc + (1 << 13)) >> 14, -32768, 32767)
    return y


def resample_stream(chunks, G: np.ndarray, L: int, M: int):
    """The rate stage of a stream: one int16 array of new resampled samples per push.  A push taking T to T' makes
    y[K(T)] .. y[K(T') - 1] from the input carry (the samples from b_{K(T)} on) and the push."""
    carry, base, pushed, outs = None, 0, 0, []
    for chunk in chunks:
        c = np.asarray(chunk).reshape(-1)
        assert c.size % 2 == 0
        held = c if carry is None else np.concatenate([carry, c])                # starts at input sample `base`
        k0, k1 = resampled_of(pushed, L, M), resampled_of(pushed + c.size // 2, L, M)
        outs.append(resample(held, G, L, M, n0=k0, nout=k1 - k0, b0=base))
        pushed += c.size // 2
        nb = (k1 * M) // L                                                         # b_{K(T')}
        carry, base = held[2 * (nb - base):], nb
        assert carry.size == 2 * (pushed - nb) <= 2 * (J - 1)
    return outs


def channelize(x, offsets, G, L, M, taps, phasor, band: str = "fm", decim: int = 32) -> np.ndarray:
    """The whole handle one-shot: int16 [nch][2 N_plan(K(T))]."""
    y = resample(x, G, L, M)
    if band == "am":
        return chan_oracle_am.channelize(y, offsets, taps, phasor)
    return chan_oracle_rates.channelize(y, offsets, taps, phasor, decim)


def channelize_stream(chunks, offsets, G, L, M, taps, phasor, band: str = "fm", decim: int = 32):
    """The whole handle streamed: one int16 [nch][2 n] array per push."""
    ys = resample_stream(chunks, G, L, M)
    if band == "am":
        return chan_oracle_am.channelize_stream(ys, offsets, taps, phasor)
    return chan_oracle_rates.channelize_stream(ys, offsets, taps, phasor, decim)
