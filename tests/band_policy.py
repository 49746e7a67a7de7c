"""The band receiver's policy (include/nrsc5_b200.h, nrsc5b_band_*: suppression, detach, attach) restated in Python, on
the rows of each window's verdict: what flags every window gets and which sessions open and close."""

DETECTED, LEAKAGE, ATTACHED, NO_SLOT = 1, 2, 4, 8
GEOM = {"fm": dict(S=2160, r=1, tol=56), "am": dict(S=270, r=2, tol=7)}     # tol: P / 2


def leakage(offsets, rows, k, band):
    g = GEOM[band]
    for j, rj in enumerate(rows):
        if j == k or not rj["detected"] or abs(offsets[j] - offsets[k]) > g["r"]:
            continue
        stronger = rj["score"] > rows[k]["score"] or (rj["score"] == rows[k]["score"] and offsets[j] < offsets[k])
        dt = abs(rj["timing"] - rows[k]["timing"]) % g["S"]
        if stronger and min(dt, g["S"] - dt) <= g["tol"]:
            return True
    return False


def run(offsets, band, windows, W, hold, max_stations, end=None):
    """windows: per window the rows (dicts with detected, score, timing) of every channel.  end: the last channel
    sample at a flush (None: no flush).  Returns (flags per window, sessions as dicts)."""
    nch = len(offsets)
    sessions, open_, absent, owner, all_flags = [], {}, {}, [None] * max_stations, []
    for w, rows in enumerate(windows):
        flags, present = [0] * nch, [False] * nch
        for k, rk in enumerate(rows):
            if rk["detected"]:
                flags[k] |= DETECTED
                if leakage(offsets, rows, k, band):
                    flags[k] |= LEAKAGE
                else:
                    present[k] = True
        for k in sorted(open_):
            absent[k] = 0 if present[k] else absent[k] + 1
        for k in [k for k in sorted(open_) if absent[k] >= hold]:
            s = sessions[open_.pop(k)]
            s["n1"] = w * W
            owner[s["slot"]] = None
            s["slot"] = -1
        for k in range(nch):
            if not present[k] or k in open_:
                continue
            if None not in owner:
                flags[k] |= NO_SLOT
                continue
            slot = owner.index(None)
            sid = len(sessions)
            sessions.append(dict(id=sid, channel=k, offset=offsets[k], slot=slot, n0=w * W, n1=-1, window=w))
            owner[slot] = sid
            open_[k] = sid
            absent[k] = 0
        for k in open_:
            flags[k] |= ATTACHED
        all_flags.append(flags)
    if end is not None:
        for k, sid in open_.items():
            sessions[sid]["n1"] = end
            sessions[sid]["slot"] = -1
    return all_flags, sessions
