"""numpy restatement of the band scan (include/nrsc5_b200.h, csrc/scan.cu): every accumulator in exact int64 and the
metrics in double, rounded as the kernel rounds them."""
import math

import numpy as np

MODES = {0: dict(F=2048, P=112, q=4, fs=744187.5), 1: dict(F=256, P=14, q=2, fs=46511.71875)}
HALO = 63


def geometry(mode):
    m = MODES[mode]
    S = m["F"] + m["P"]
    return m["F"], m["P"], m["q"], S, S // m["q"], m["fs"]


def _sat16(v):
    return np.clip(v, -32768, 32767)


def sidebands(y, taps):
    """y: int16 [2 T] I/Q interleaved -> (z_L, z_U) at every n = 0..T-1 with n >= 63 (z[n] at index n; earlier
    positions 0), as int64 [T, 2]."""
    c = y[0::2].astype(np.int64)
    d = y[1::2].astype(np.int64)
    T = c.size
    a = taps[:, 0].astype(np.int64)
    b = taps[:, 1].astype(np.int64)
    zl = np.zeros((T, 2), dtype=np.int64)
    zu = np.zeros((T, 2), dtype=np.int64)
    if T < 64:
        return zl, zu
    # correlation form: sum_u g[u] y[n - 63 + u]
    A = np.correlate(c, a, "valid")
    B = np.correlate(d, b, "valid")
    Cs = np.correlate(d, a, "valid")
    D = np.correlate(c, b, "valid")
    r = 1 << 14
    zu[63:, 0] = _sat16((A - B + r) >> 15)
    zu[63:, 1] = _sat16((Cs + D + r) >> 15)
    zl[63:, 0] = _sat16((A + B + r) >> 15)
    zl[63:, 1] = _sat16((Cs - D + r) >> 15)
    return zl, zu


def accumulate(ys, mode, taps):
    """ys: int16 [nch][2 T] -> (acc int64 [nch][6][J], power sums (python ints) [nch], T)."""
    F, P, q, S, J, _ = geometry(mode)
    ys = np.atleast_2d(ys)
    nch, T = ys.shape[0], ys.shape[1] // 2
    acc = np.zeros((nch, 6, J), dtype=np.int64)
    pw = []
    n = np.arange(64, T - F, q)                    # n = 0 (mod q), 63 <= n, n + F <= T - 1
    for k in range(nch):
        y = ys[k]
        pw.append(int(np.sum(y.astype(np.int64) ** 2)))
        if n.size == 0:
            continue
        zs = sidebands(y, taps)
        j = (n % S) // q
        for s in range(2):
            z0, z1 = zs[s][n], zs[s][n + F]
            pr = z0[:, 0] * z1[:, 0] + z0[:, 1] * z1[:, 1]
            pi = z0[:, 1] * z1[:, 0] - z0[:, 0] * z1[:, 1]
            e = (z0 ** 2).sum(1) + (z1 ** 2).sum(1)
            for c, v in enumerate((pr, pi, e)):
                acc[k, 3 * s + c] = _bincount64(j, v, J)
    return acc, pw, T


def _bincount64(j, v, J):
    out = np.zeros(J, dtype=np.int64)
    np.add.at(out, j, v)
    return out


def products(mode, T):
    F, _, q, _, _, _ = geometry(mode)
    last = T - 1 - F
    first = (HALO + q - 1) // q
    return 0 if last < first * q else last // q - first + 1


def windows(acc, mode):
    """C_s, E_s: int64 [nch][6][J] (the same layout as the folds)."""
    _, P, q, _, J, _ = geometry(mode)
    W = P // q
    out = np.zeros_like(acc)
    for i in range(W):
        out += np.roll(acc, -i, axis=2)
    return out


def _i2d(v):
    return float(v)


def metrics(acc, pw, T, mode, c, kappa, c1):
    """The nrsc5b_scan_t fields per channel, as dicts."""
    F, P, q, S, J, fs = geometry(mode)
    W = P // q
    cw = windows(acc, mode)
    npr = products(mode, T)
    symbols = npr * q / S
    thr = c / math.sqrt(npr * P / S) if npr > 0 else math.inf
    thr1 = c1 / math.sqrt(npr * P / S) if npr > 0 else math.inf
    res = []
    for k in range(acc.shape[0]):
        tot = [int(acc[k, i].astype(object).sum()) * W for i in range(6)]
        Cr = [int(x) for x in cw[k, 0]]
        Ci = [int(x) for x in cw[k, 1]]
        Ur = [int(x) for x in cw[k, 3]]
        Ui = [int(x) for x in cw[k, 4]]
        dr = np.array([_i2d(J * (Cr[j] + Ur[j]) - (tot[0] + tot[3])) / J for j in range(J)])
        di = np.array([_i2d(J * (Ci[j] + Ui[j]) - (tot[1] + tot[4])) / J for j in range(J)])
        v = dr * dr + di * di
        j = int(np.argmax(v))
        mag = math.sqrt(v[j])
        e = 0.5 * float(int(cw[k, 2, j]) + int(cw[k, 5, j]))
        r = dict(score=mag / e if e > 0 else 0.0, threshold=thr, threshold_sideband=thr1, symbols=symbols)
        r["timing"] = (q * j - 32) % S
        r["cfo_hz"] = -math.atan2(di[j], dr[j]) * fs / (2 * math.pi * F) if mag > 0 else 0.0
        r["j"] = j
        for s, name in ((0, "lower"), (1, "upper")):
            sr = _i2d(J * int(cw[k, 3 * s, j]) - tot[3 * s]) / J
            si = _i2d(J * int(cw[k, 3 * s + 1, j]) - tot[3 * s + 1]) / J
            emean = _i2d(tot[3 * s + 2]) / J
            ms = math.sqrt(sr * sr + si * si)
            es = 0.5 * float(int(cw[k, 3 * s + 2, j]))
            r["score_" + name] = ms / es if es > 0 else 0.0
            r["d_" + name] = (sr, si)
            rho = ms / (0.5 * emean) if emean > 0 else 0.0
            r["rho_" + name] = rho
            r["snr_db_" + name] = -math.inf if rho <= 0 else math.inf if rho >= kappa else 10 * math.log10(rho / (kappa - rho))
            en = float(tot[3 * s + 2] // W)
            r["power_dbfs_" + name] = 10 * math.log10(en / (2.0 * npr) / 2 ** 30) if npr > 0 and en > 0 else -math.inf
        (lr, li), (ur, ui) = r.pop("d_lower"), r.pop("d_upper")
        dot = lr * ur + li * ui
        m2 = math.sqrt((lr * lr + li * li) * (ur * ur + ui * ui))
        r["detected"] = int(symbols >= 32 and r["score"] >= thr and min(r["score_lower"], r["score_upper"]) >= thr1
                            and dot >= math.sqrt(0.5) * m2)
        r["power_dbfs"] = 10 * math.log10(pw[k] / T / 2 ** 30) if T > 0 and pw[k] > 0 else -math.inf
        res.append(r)
    return res


def scan(ys, mode, taps, c, kappa, c1):
    acc, pw, T = accumulate(ys, mode, taps)
    return acc, metrics(acc, pw, T, mode, c, kappa, c1)


def gamma(taps, q):
    """sum_k |r(k q)|^2, r the normalised autocorrelation of the taps: the correlation of neighbouring products."""
    g = taps[:, 0].astype(np.float64) + 1j * taps[:, 1]
    r = np.correlate(g, g, "full") / np.sum(np.abs(g) ** 2)
    lags = np.arange(-63, 64)
    return float(np.sum(np.abs(r[lags % q == 0]) ** 2))


def response_db(taps, f, fs):
    """|H(f)| in dB of z = sum_u g[u] y[n - 63 + u] for y = e^{j 2 pi f n / fs}."""
    g = taps[:, 0].astype(np.float64) + 1j * taps[:, 1]
    u = np.arange(64) - 63
    H = np.exp(2j * np.pi * np.outer(np.asarray(f, dtype=np.float64) / fs, u)) @ g / 32768.0
    return 20 * np.log10(np.maximum(np.abs(H), 1e-300))
