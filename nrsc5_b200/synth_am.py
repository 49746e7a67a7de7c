"""Synthetic NRSC-5 AM (hybrid MA1, all-digital MA3) captures, cs16 I/Q at 46 511.72 S/s, with known L1 PDUs.

The reference ships no modulator; like synth.py for FM this inverts the receive chain stage by stage
(recipe: SURVEY.md §8(d) "AM MA1 recipe", every step derived from the decoder):

  P1 (8 x 3750 bit / frame): scramble (reference src/decode.c:279-294) -> K=9 tail-biting encoder E1
  (0561,0657,0711) -> puncture 1,0,1,1,0,1,1,0,1,1,1,1,1,1,1 (decode.c:186-195) -> split over the backup
  (bl,bu: this frame) and main (ml,mu: sent three frames EARLIER, decode.h:7, decode.c:175-176) bit sets with
  the delay tables of decode.c:27-32 -> bit_map into the 64-QAM primary sidebands (decode.c:67-95)
  P3 (24 000 bit / frame): E2 (0561,0753,0711), puncture 1,0,1,1,0,0 -> el (QPSK tertiary), eu (16-QAM secondary)
  PIDS (80 bit / block): E3 unpunctured -> il / iu -> the two 16-QAM PIDS carriers (decode.c:474-500)
  -> constellations of sync.c:37-88, training symbols of sync.c:673-710, reference carrier of sync.c:208-236,
  complementary lower sideband (sync.c:616-633) -> 256-point OFDM with 14-sample prefix and the receiver's
  pulse shape, circularly advanced by 121 samples (acquire.c:239-248), on top of a strong carrier.

MA3 (make_am_ma3): the primary sidebands move to the inner partitions, P3 (30 000 bit, E1, punctured like P1)
is split like P1 into backup/main sets carried by 64-QAM secondary (upper) and tertiary (lower) partitions, the
PIDS carriers sit at -27/+27 and nothing is complementary (sync.c:624,670-671,694-696; decode.c:117-141).

Test infrastructure for the AM rows of the scope table (SURVEY §8 a21); pure numpy.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from functools import lru_cache

import numpy as np

from .synth import PCI_FIXED, conv_encode_tb, pn_sequence

FFT = 256
CP = 14
SYM = FFT + CP                      # 270 samples per OFDM symbol
BLKSZ = 32
BLOCK_SAMPLES = SYM * BLKSZ         # 8640 cs16 complex samples per block
BLOCKS_PER_FRAME = 8
CENTER = 128
P1_BITS = 3750
P3_BITS = 24000
P3_BITS_MA3 = 30000
PIDS_BITS = 80
GENS_E1 = (0o561, 0o657, 0o711)
GENS_E2 = (0o561, 0o753, 0o711)     # also E3 (PIDS)
BL_DELAY, ML_DELAY, BU_DELAY, MU_DELAY = (2, 1, 5), (11, 6, 7), (10, 8, 9), (4, 3, 0)
EL_DELAY, EU_DELAY = (0, 1), (2, 3, 5, 4)
PIDS_IL_DELAY = (0, 1, 12, 13, 6, 5, 18, 17, 11, 7, 23, 19)
PIDS_IU_DELAY = (2, 4, 14, 16, 3, 8, 15, 20, 9, 10, 21, 22)
QAM64_LEVEL = {0: -3.5, 4: -2.5, 6: -1.5, 2: -0.5, 3: 0.5, 7: 1.5, 5: 2.5, 1: 3.5}      # inverse of gray8, sync.c:49-66
QAM16_LEVEL = {0: -1.5, 2: -0.5, 3: 0.5, 1: 1.5}                                          # inverse of gray4, sync.c:37-47


def _bit_map_pos(k):
    """(row, col) of interleaver cell k (bit_map, reference src/decode.c:67-72)."""
    col = (9 * k) % 25
    row = (11 * col + 16 * (k // 25) + 11 * (k // 50)) % 32
    return row, col


@lru_cache(maxsize=None)
def _ma1_index_sets():
    """For every decoder bit set, the (block, row, col, bit plane) its n-th bit is read from
    (interleaver_ma1, reference src/decode.c:74-116)."""
    def table(nn, b_of, k_of, p_of):
        n = np.arange(nn)
        b, k, p = b_of(n), k_of(n), p_of(n)
        row, col = _bit_map_pos(k)
        return b, row, col, p
    return {
        "bl": table(18000, lambda n: n // 2250, lambda n: (n + n // 750 + 1) % 750, lambda n: n % 3),
        "ml": table(18000, lambda n: (3 * n + 3) % 8, lambda n: (n + n // 3000 + 3) % 750, lambda n: 3 + n % 3),
        "bu": table(18000, lambda n: n // 2250, lambda n: (n + n // 750) % 750, lambda n: n % 3),
        "mu": table(18000, lambda n: (3 * n) % 8, lambda n: (n + n // 3000 + 2) % 750, lambda n: 3 + n % 3),
        "el": table(12000, lambda n: (3 * n + n // 3000) % 8, lambda n: (n + n // 6000) % 750, lambda n: n % 2),
        "eu": table(24000, lambda n: (3 * n + n // 3000 + 2 * (n // 12000)) % 8, lambda n: (n + n // 6000) % 750,
                    lambda n: n % 4),
        # MA3 (decode.c:117-141): P3's backup/main sets in the tertiary (ebl, eml) and secondary (ebu, emu) matrices
        "ebl": table(18000, lambda n: (3 * n + 3) % 8, lambda n: (n + n // 3000 + 3) % 750, lambda n: n % 3),
        "eml": table(18000, lambda n: (3 * n + 3) % 8, lambda n: (n + n // 3000 + 3) % 750, lambda n: 3 + n % 3),
        "ebu": table(18000, lambda n: (3 * n) % 8, lambda n: (n + n // 3000 + 2) % 750, lambda n: n % 3),
        "emu": table(18000, lambda n: (3 * n) % 8, lambda n: (n + n // 3000 + 2) % 750, lambda n: 3 + n % 3),
    }


def _split_p1(c1):
    """72000 punctured P1 code bits of a frame -> (bl, ml, bu, mu), 18000 bits each (decode.c:141-151)."""
    c = c1.reshape(6000, 12)
    return tuple(c[:, list(d)].reshape(-1) for d in (BL_DELAY, ML_DELAY, BU_DELAY, MU_DELAY))


def _split_p3(c3):
    c = c3.reshape(6000, 6)
    return c[:, list(EL_DELAY)].reshape(-1), c[:, list(EU_DELAY)].reshape(-1)


def _frame_bits(rng, nbits, pci_bits, pci_start, pci_step):
    """Descrambled frame bits as handed to frame_push() (reference src/frame.c:645-714): per-byte bit reversal
    (the last group may be shorter than a byte), PCI bits at logical positions pci_start + pci_step * h, the rest
    packed MSB-first into the PDU.  PCI = fixed data only; the PDU's last byte rules out a fixed-data sync."""
    logical = np.zeros(nbits, dtype=np.uint8)
    pos = pci_start + pci_step * np.arange(pci_bits)
    is_pci = np.zeros(nbits, dtype=bool)
    is_pci[pos] = True
    logical[pos] = [(PCI_FIXED >> (23 - h)) & 1 for h in range(pci_bits)]
    npay = nbits - pci_bits
    pdu = rng.integers(0, 256, (npay + 7) // 8, dtype=np.uint8)
    pdu[npay // 8 - 1] = 0x12
    logical[~is_pci] = np.unpackbits(pdu)[:npay]
    i = np.arange(nbits)
    start = (i >> 3) << 3
    blen = np.minimum(8, nbits - start)
    phys = start + blen - 1 - (i & 7)
    ok = (i & 7) < blen
    bits = np.zeros(nbits, dtype=np.uint8)
    bits[phys[ok]] = logical[ok]
    return bits


def _encode(bits, gens, keep):
    pn = pn_sequence(bits.size)
    coded = conv_encode_tb(bits ^ pn, gens=gens, k=9).reshape(-1)
    mask = np.tile(np.array(keep, dtype=bool), coded.size // len(keep))
    return coded[mask]


def ref_bits_am(bc: int, psmi: int = 1, pli: int = 0, hppi: int = 0, aabi: int = 0, rdbi: int = 0) -> np.ndarray:
    """32 bits of the AM reference subcarrier for block `bc` (find_block_am, reference src/sync.c:208-236):
    fixed pattern, even-parity groups, block count at 17..19, service mode at 26..30."""
    d = np.zeros(32, dtype=np.uint8)
    for i in (1, 2, 5, 9, 21, 22):
        d[i] = 1
    d[7], d[11], d[12], d[15] = pli, hppi, aabi, rdbi
    d[8] = d[7]
    d[13] = d[10] ^ d[11] ^ d[12]
    d[17], d[18], d[19] = (bc >> 2) & 1, (bc >> 1) & 1, bc & 1
    d[20] = d[15] ^ d[16] ^ d[17] ^ d[18] ^ d[19]
    for k, sh in zip(range(26, 31), (4, 3, 2, 1, 0)):
        d[k] = (psmi >> sh) & 1
    d[31] = np.bitwise_xor.reduce(d[23:31])
    return d


@dataclass
class AmCapture:
    cs16: np.ndarray                                     # int16 [2 * nsamples], I/Q interleaved
    p1_frames: dict = field(default_factory=dict)        # logical frame -> list of 8 uint8[3750]
    p3_frames: dict = field(default_factory=dict)        # logical frame -> uint8[24000]
    pids_frames: list = field(default_factory=list)      # uint8[80] per transmitted block


def make_am_ma3(**kw) -> AmCapture:
    """AM all-digital MA3 capture (see make_am_ma1 for the arguments)."""
    return make_am_ma1(psmi=2, **kw)


def make_am_ma1(nframes: int = 10, seed: int = 1234, lead_in: int = 500, carrier: float = 10000.0, unit: float = 50.0,
                noise_lsb: float = 0.0, noise_seed: int = 5, cfo_hz: float = 0.0, psmi: int = 1,
                flags: tuple = (0, 0, 0, 0), p1_frames=None) -> AmCapture:
    """AM hybrid MA1 (psmi 1) or all-digital MA3 (psmi 2) capture of `nframes` transmitted L1 frames (8 blocks each).  The receiver needs the 0x5670
    block-count run to lock, then four frames before it decodes (decode.c:512,569), and the main bits of a
    frame travel three frames ahead of its backup bits: frame F comes out when frames F-3 .. F+1 were received."""
    rng = np.random.default_rng(seed)
    idx = _ma1_index_sets()
    cap = AmCapture(cs16=None)
    nlog = nframes + 3
    frng = np.random.default_rng(seed + 77)                          # MA3 outer-partition filler
    p1 = [[_frame_bits(rng, P1_BITS, 22, 120, 160) for _ in range(8)] for _ in range(nlog)]
    if p1_frames is not None:               # caller's P1 PDUs (packed MSB first, 3750 bits each: synth_l2.py), in order
        src = iter(p1_frames)
        for f in range(nlog):
            for k in range(8):
                pk = next(src, None)
                if pk is not None:
                    p1[f][k] = np.unpackbits(np.frombuffer(pk, dtype=np.uint8))[:P1_BITS]
    ma3 = psmi == 2
    assert psmi in (1, 2)
    if ma3:
        p3 = [_frame_bits(rng, P3_BITS_MA3, 24, 120, 1240) for _ in range(nlog)]     # frame.c:676-680
    else:
        p3 = [_frame_bits(rng, P3_BITS, 24, 120, 992) for _ in range(nlog)]
    keep_e1 = (1, 0, 1, 1, 0, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1)
    sets = []
    for f in range(nlog):
        c1 = np.concatenate([_encode(b, GENS_E1, keep_e1) for b in p1[f]])          # 72000
        bl, ml, bu, mu = _split_p1(c1)
        if ma3:
            c3 = _encode(p3[f], GENS_E1, keep_e1)                                    # 72000 (decode.c:214-229)
            ebl, eml, ebu, emu = _split_p1(c3)
            sets.append(dict(bl=bl, ml=ml, bu=bu, mu=mu, ebl=ebl, eml=eml, ebu=ebu, emu=emu))
        else:
            c3 = _encode(p3[f], GENS_E2, (1, 0, 1, 1, 0, 0))                         # 36000
            el, eu = _split_p3(c3)
            sets.append(dict(bl=bl, ml=ml, bu=bu, mu=mu, el=el, eu=eu))
        cap.p1_frames[f] = p1[f]
        cap.p3_frames[f] = p3[f]

    shape = np.ones(SYM)
    shape[:CP] = np.sin(np.pi / 2 * np.arange(CP) / CP)
    shape[FFT:] = np.cos(np.pi / 2 * np.arange(CP) / CP)
    k_of_bin = np.arange(FFT) - CENTER
    adv = np.exp(2j * np.pi * k_of_bin * 121 / FFT)                   # the receiver stores samples shifted by 121
    sig = np.zeros(nframes * BLOCKS_PER_FRAME * BLOCK_SAMPLES, dtype=np.complex128)
    lev64 = np.array([QAM64_LEVEL[c] for c in range(8)])
    lev16 = np.array([QAM16_LEVEL[c] for c in range(4)])

    for x in range(nframes):
        def fill(names_frames, shape3):
            m = np.zeros(shape3, dtype=np.uint8)
            for name, fr in names_frames:
                b, row, col, p = idx[name]
                np.bitwise_or.at(m, (b, row, col), (sets[fr][name].astype(np.uint8) << p).astype(np.uint8))
            return m
        pl = fill([("bl", x), ("ml", x + 3)], (8, 32, 25))
        pu = fill([("bu", x), ("mu", x + 3)], (8, 32, 25))
        if ma3:
            tt = fill([("ebl", x), ("eml", x + 3)], (8, 32, 25))
            ss = fill([("ebu", x), ("emu", x + 3)], (8, 32, 25))
        else:
            tt = fill([("el", x)], (8, 32, 25))
            ss = fill([("eu", x)], (8, 32, 25))
        for bc in range(8):
            # PIDS (decode.c:474-500)
            pb = rng.integers(0, 2, PIDS_BITS, dtype=np.uint8)
            cap.pids_frames.append(pb)
            cp = _encode(pb, GENS_E2, (1,)).reshape(10, 24)
            il = cp[:, list(PIDS_IL_DELAY)].reshape(-1)
            iu = cp[:, list(PIDS_IU_DELAY)].reshape(-1)
            sb = np.zeros((32, 2), dtype=np.uint8)
            n = np.arange(120)
            for arr, which, koff in ((il, 0, 11), (iu, 1, 0)):
                k = (n + n // 60 + koff) % 30
                row = (11 * (k + k // 15) + 3) % 32
                np.bitwise_or.at(sb, (row, which), (arr.astype(np.uint8) << (n % 4)).astype(np.uint8))
            S = np.zeros((BLKSZ, FFT), dtype=np.complex128)           # receiver bin order (after fftshift)
            S[:, CENTER] = carrier / unit
            q64 = lambda c: lev64[c & 7] + 1j * lev64[c >> 3]
            q16 = lambda c: lev16[c & 3] + 1j * lev16[c >> 2]
            qpsk = lambda c: ((c & 1) - 0.5) + 1j * ((c >> 1) - 0.5)
            up = np.zeros((BLKSZ, 82), dtype=np.complex128)            # wanted value of upper carrier CENTER + i
            lo = np.zeros((BLKSZ, 82), dtype=np.complex128)            # wanted (mirrored) value of CENTER - i
            d = ref_bits_am(bc, psmi, *flags)
            up[:, 1] = 1.5j * (2.0 * d - 1.0)
            cols = np.arange(25)
            i = np.arange(1, 82)
            if not ma3:
                up[:, 27] = q16(sb[:, 0])
                up[:, 53] = q16(sb[:, 1])
                up[[8, 24], 27] = 1.5 - 0.5j                            # PIDS training (sync.c:673-674)
                up[[8, 24], 53] = 1.5 - 0.5j
                up[:, 57:82] = q64(pu[bc])
                lo[:, 57:82] = q64(pl[bc])
                up[:, 28:53] = q16(ss[bc])
                up[:, 2:27] = qpsk(tt[bc])
                for col in cols:                                        # training rows (sync.c:699-710)
                    for tr in ((5 + 11 * col) % 32, (21 + 11 * col) % 32):
                        up[tr, 57 + col] = 2.5 - 2.5j
                        lo[tr, 57 + col] = 2.5 - 2.5j
                        up[tr, 28 + col] = 1.5 - 0.5j
                        up[tr, 2 + col] = -0.5 + 0.5j
                S[:, CENTER + i] = up[:, 1:]
                # lower sideband: the receiver takes -conj of it and, up to index 53, adds it to the upper one
                S[:, CENTER - i[:53]] = -np.conj(up[:, 1:54])
                S[:, CENTER - i[56:]] = -np.conj(lo[:, 57:])
            else:
                # MA3: PIDS at -27 / +27, primary at the inner partitions, secondary = upper middle, tertiary =
                # lower middle, all 64-QAM with 2.5-2.5j training; the outer partitions are not received
                lo[:, 27] = q16(sb[:, 0])
                up[:, 27] = q16(sb[:, 1])
                lo[[8, 24], 27] = 1.5 - 0.5j
                up[[8, 24], 27] = 1.5 - 0.5j
                up[:, 2:27] = q64(pu[bc])
                lo[:, 2:27] = q64(pl[bc])
                up[:, 28:53] = q64(ss[bc])
                lo[:, 28:53] = q64(tt[bc])
                for col in cols:
                    for tr in ((5 + 11 * col) % 32, (21 + 11 * col) % 32):
                        for a in (up, lo):
                            a[tr, 2 + col] = 2.5 - 2.5j
                            a[tr, 28 + col] = 2.5 - 2.5j
                lo[:, 1] = up[:, 1]                                     # until the mode is known the receiver adds the sidebands
                # the receiver's coarse timing search listens only at |index| 56..85 (band-pass of acquire.c:63-96,
                # made for the hybrid primary sidebands) and never demodulates those carriers in MA3: unrelated
                # 64-QAM filler there lets it lock as quickly as on a hybrid signal
                up[:, 57:82] = q64(frng.integers(0, 64, (BLKSZ, 25)))
                lo[:, 57:82] = q64(frng.integers(0, 64, (BLKSZ, 25)))
                S[:, CENTER + i] = up[:, 1:]
                S[:, CENTER - i] = -np.conj(lo[:, 1:])
            X = np.zeros((BLKSZ, FFT), dtype=np.complex128)
            X[:, k_of_bin % FFT] = S * adv[None, :]
            y = np.fft.ifft(X, axis=1) * FFT * unit
            ysym = y[:, np.arange(SYM) % FFT] * shape[None, :]
            o = (x * BLOCKS_PER_FRAME + bc) * BLOCK_SAMPLES
            sig[o:o + BLOCK_SAMPLES] = ysym.reshape(-1)

    nrng = np.random.default_rng(noise_seed)
    lead = carrier + nrng.standard_normal(lead_in) * 3 + 1j * nrng.standard_normal(lead_in) * 3     # never exact zeros
    full = np.concatenate([lead, sig])
    if cfo_hz:
        full = full * np.exp(2j * np.pi * cfo_hz * np.arange(full.size) / 46511.71875)
    if noise_lsb > 0:
        full = full + noise_lsb * (nrng.standard_normal(full.size) + 1j * nrng.standard_normal(full.size))
    iq = np.empty(2 * full.size)
    iq[0::2] = full.real
    iq[1::2] = full.imag
    q = np.clip(np.rint(iq), -32767, 32767).astype(np.int16)
    # the reference's NCO turns NaN for good on an exact-zero sample (acquire.c:199-201): keep clear of it
    z = (q[0::2] == 0) & (q[1::2] == 0)
    q[0::2][z] = 1
    cap.cs16 = q
    return cap


def am_to_cu8(cs16: np.ndarray, gain: float = 1.0) -> np.ndarray:
    """cs16 at 46 511.72 S/s -> cu8 at 1 488 375 S/s, the other input format of the AM receiver
    (input_push_cu8 -> decimate_samples, reference src/input.c:52-117: (u8 - 127) * 4, then five halfband
    decimators of gain 2 each, so one cu8 LSB is worth 128 cs16 LSB).  Polyphase interpolation by 32."""
    from scipy.signal import resample_poly
    z = cs16[0::2].astype(np.float64) + 1j * cs16[1::2].astype(np.float64)
    up = resample_poly(z, 32, 1) * (gain / 128.0)
    out = np.empty(2 * up.size, dtype=np.float64)
    out[0::2] = up.real
    out[1::2] = up.imag
    return np.clip(np.rint(out + 127.0), 0, 255).astype(np.uint8)


def make_am_band(stations, cs16: bool = True, noise_lsb: float = 3.0, seed: int = 9) -> np.ndarray:
    """A band capture at 1 488 375 S/s for the wideband channeliser's AM plan (include/nrsc5_b200.h,
    nrsc5b_chan_create_am): `stations` = (narrowband cs16 capture at 46 511.72 S/s, offset m in 10 kHz steps from the
    capture centre, gain) each, interpolated by 32 as am_to_cu8 does, moved to its offset (10 kHz / 1 488 375 Hz =
    80 / 11907 cycles per sample), scaled and summed over the length of the shortest one, with a noise floor of
    `noise_lsb` LSB per component (channels without a station must not be exact zeros: see the header), and quantised.
    Returns int16 I/Q interleaved (cs16=True; gain 1 keeps a station's cs16 level) or uint8 (cu8, where gain 1 / 64
    keeps it at the channeliser's output)."""
    from scipy.signal import resample_poly
    n = min(c.size for c, _, _ in stations) // 2
    t = np.arange(32 * n, dtype=np.float64)
    wide = np.zeros(32 * n, dtype=np.complex128)
    for c, m, gain in stations:
        z = c[0:2 * n:2].astype(np.float64) + 1j * c[1:2 * n:2].astype(np.float64)
        wide += resample_poly(z, 32, 1) * gain * np.exp(2j * np.pi * ((80 * m) % 11907) / 11907.0 * t)
    rng = np.random.default_rng(seed)
    wide += noise_lsb * (rng.standard_normal(wide.size) + 1j * rng.standard_normal(wide.size))
    iq = np.empty(2 * wide.size)
    iq[0::2] = wide.real
    iq[1::2] = wide.imag
    if cs16:
        return np.clip(np.rint(iq), -32768, 32767).astype(np.int16)
    return np.clip(np.rint(iq + 127.0), 0, 255).astype(np.uint8)
