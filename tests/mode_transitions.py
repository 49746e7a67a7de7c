"""Captures in which one stream changes service mode or loses sync while P3 / P4 frames are being produced (test
infrastructure for tests/test_gpu_mode_transitions.py and tests/test_oracle_mode_transitions.py).

A sync loss is forced the way a receiver meets it on air, but from clean signal: one P1 frame carries an audio PCI
and a header the RS(255,247) check cannot correct, so the header predicate of the reference's frame_push
(src/frame.c:535-540) drops sync when that frame is decoded at block 15.  Every frame of the block of the loss is
decoded from signal and compares exactly.  The next capture is appended directly (a link of a chain)."""
import numpy as np

from nrsc5_b200 import synth, synth_am, synth_l2

GAP_BYTES = 2 * 600000                 # 0.4 s of noise at 1 488 375 S/s (cu8)


def bad_p1(seed, nbits=synth.P1_BITS):
    """A packed P1 frame with an audio PCI whose audio header the receiver cannot correct: sync is lost on it."""
    rng = np.random.default_rng(seed)
    if nbits == synth.P1_BITS:
        return synth.pack_bits(synth.build_p1_frame_bits(rng, valid_header=False))
    pdu = rng.integers(0, 256, synth_l2.pdu_len(nbits), dtype=np.uint8).tobytes()
    return synth_l2.frame_from_pdu(pdu, nbits, synth_l2.PCI_AUDIO)


def fm_link(psmi, nframes, seed, bad_at=None, lead_in=0, cfo_hz=0.0, noise_lsb=2.0):
    """One FM capture of `nframes` L1 frames (+ 2 blocks); P1 frame `bad_at` (None: none) loses sync."""
    p1 = [None] * nframes
    if bad_at is not None:
        p1[bad_at] = bad_p1(seed + 1000)
    return synth.make_fm(psmi=psmi, nframes=nframes, seed=seed, lead_in=lead_in, tail_blocks=2, cfo_hz=cfo_hz,
                         noise_lsb=noise_lsb, p1_frames=p1)


def noise_gap(seed, nbytes=GAP_BYTES):
    rng = np.random.default_rng(seed)
    return np.clip(np.rint(rng.standard_normal(nbytes) * 6 + 127), 0, 255).astype(np.uint8)


def cu8_of(caps):
    cu8 = np.concatenate([c if isinstance(c, np.ndarray) else c.cu8 for c in caps])
    return cu8[: cu8.size & ~3]


# (a) a sync loss in the block that also ends a P3 (and, MP11, a P4) frame: P1 frame 3 of 5, P3 flowing since frame 2
LOSS_CASES = {"mp3": 3, "mp11": 11, "mp2": 2}


def loss_capture(name):
    psmi = LOSS_CASES[name]
    return fm_link(psmi, 5, seed=700 + psmi, bad_at=3, lead_in=300, cfo_hz=40.0)


# (b) one stream through MP11 -> MP1 -> MP3 -> MP2 -> MP11: (psmi, frames, lead-in, carrier offset) per link
CHAIN = [(11, 5, 300, 0.0), (1, 3, 0, 50.0), (3, 5, 77, -30.0), (2, 5, 0, 20.0), (11, 3, 150, 0.0)]


def chain_links(gaps=False):
    """The links of the chain; each ends in a P1 frame that loses sync (gaps=False) or is followed by 0.4 s of
    noise (gaps=True, all headers valid)."""
    out = []
    for i, (psmi, n, lead, cfo) in enumerate(CHAIN):
        last = i == len(CHAIN) - 1
        out.append(fm_link(psmi, n, seed=800 + 10 * i, bad_at=None if (gaps or last) else n - 1, lead_in=lead,
                           cfo_hz=cfo))
        if gaps and not last:
            out.append(noise_gap(900 + i))
    return out


def chain_capture(gaps=False):
    return cu8_of(chain_links(gaps))


def transmitted(links):
    """Packed bits of every P1, P3 and P4 frame and every PIDS frame the links carry."""
    frames, pids = set(), set()
    for c in links:
        if isinstance(c, np.ndarray):
            continue
        for f in list(c.p1_frames) + list(c.p3_frames) + list(c.p4_frames):
            frames.add(synth.pack_bits(f))
        for f in c.pids_frames:
            pids.add(synth.pack_bits(f))
    return frames, pids


# (c) three streams in one engine: MP1 throughout; MP1 -> MP11 (groups 0 and 2 enabled mid-run); MP3 -> MP1
def lazy_streams():
    s0 = fm_link(1, 9, seed=1101, lead_in=500, cfo_hz=-60.0)
    s1 = [fm_link(1, 4, seed=1111, bad_at=3, lead_in=100), fm_link(11, 5, seed=1112)]
    s2 = [fm_link(3, 5, seed=1121, bad_at=4, lead_in=200, cfo_hz=30.0), fm_link(1, 4, seed=1122)]
    return [cu8_of(s) for s in ([s0], s1, s2)], [transmitted(s) for s in ([s0], s1, s2)]


# (f) AM: one stream MA1 -> MA3 -> MA1, the first two links end in a P1 frame that loses sync
def am_chain():
    links = []
    for i, psmi in enumerate((1, 2, 1)):
        p1 = None
        if i < 2:
            p1 = [None] * (8 * 13)
            p1[8 * 7] = bad_p1(1300 + i, nbits=3750)       # logical frame 7, the first of its 8 P1 frames
        links.append(synth_am.make_am_ma1(nframes=10, seed=1310 + i, lead_in=(500, 40, 0)[i], psmi=psmi,
                                          p1_frames=p1).cs16)
    return np.concatenate(links)


def am_rdbi(psmi):
    """MA1 (psmi 1) / MA3 (psmi 2) with rdbi = 1: no P3, PIDS1 zeroed in MA1 (reference src/decode.c:494,523)."""
    return synth_am.make_am_ma1(nframes=10, seed=1400 + psmi, lead_in=321, psmi=psmi, flags=(0, 0, 0, 1)).cs16


# (g) PSMI aliases: compatibility_mode maps the 64 values onto six modes (reference src/sync.c:30-35); the coarse
# vote only takes 0..15 (sync.c:396), so a value >= 16 never acquires
ALIASES = [4, 7, 10, 12, 15]
NEVER = 19                              # compatibility mode 3


def alias_capture(psmi):
    return fm_link(psmi, 3, seed=1500 + psmi, lead_in=211, cfo_hz=25.0).cu8
