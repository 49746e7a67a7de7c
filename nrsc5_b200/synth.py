"""Synthetic NRSC-5 FM captures (cu8 I/Q at 1 488 375 S/s) with known L1 PDUs.

The reference ships no modulator.  This generator inverts the receive chain
stage by stage, so that a correct receiver returns exactly the frame bits
generated here (recipe: SURVEY.md §8(d), each step derived from the decoder):

  payload -> scramble (reference src/decode.c:279-294) -> rate-1/3 K=7
  tail-biting encode, g=(0133,0171,0165) (decode.c:238-255, conv_dec.c:139-154)
  -> puncture 1,1,1,1,1,0 (decode.c:263) -> inverse of interleaver I / II
  (decode.c:296-342); for MP3 also P3: puncture 1,0,1,1,0,1 and the inverse of
  the convolutional interleaver IV (decode.c:344-376) onto the PX1 partitions
  (sync.c:552-573) -> QPSK map onto partitions (sync.c:509-536) + DBPSK
  reference subcarriers (sync.c:96-99,169-186) -> 2x-oversampled OFDM with the
  receiver's raised-sine pulse shape (acquire.c:322-331) -> cu8 (defines.h:93).

Used by bench.py for its synthetic workload and by the tests; pure numpy.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from functools import lru_cache

import numpy as np

FFT = 2048
CP = 112
FFTCP = FFT + CP
BLKSZ = 32
LB_START = 1024 - 546
UB_END = 1024 + 546
P1_BITS = 146176
PIDS_BITS = 80
PM_BLOCK = 23040
BLOCKS_PER_FRAME = 16
SAMPLES_PER_BLOCK_CU8 = FFTCP * BLKSZ * 2  # complex cu8 samples per L1 block
PCI_AUDIO = 0x38D8D3
PCI_FIXED = 0x3634CE
PM_V = np.array([10, 2, 18, 6, 14, 8, 16, 0, 12, 4, 11, 3, 19, 7, 15, 9, 17, 1, 13, 5])
GENS_K7 = (0o133, 0o171, 0o165)


# ----------------------------------------------------------------------------
# bit-level pieces
# ----------------------------------------------------------------------------
@lru_cache(maxsize=None)
def pn_sequence(n: int) -> np.ndarray:
    """The descrambler's bit sequence (reference src/decode.c:279-294)."""
    out = np.empty((n + 7) // 8 * 8, dtype=np.uint8)
    val = 0x3FF
    for i in range(out.size):
        bit = ((val >> 9) ^ val) & 1
        val |= bit << 11
        val >>= 1
        out[i] = bit
    return out[:n]


def conv_encode_tb(u: np.ndarray, gens=GENS_K7, k: int = 7) -> np.ndarray:
    """Tail-biting rate-1/3 encoder; returns coded[len(u), 3] in {0,1}.
    Register convention of reference src/decode.c:243-249: newest bit at bit k-1."""
    u = np.asarray(u, dtype=np.uint8)
    out = np.zeros((u.size, len(gens)), dtype=np.uint8)
    for gi, g in enumerate(gens):
        acc = np.zeros(u.size, dtype=np.uint8)
        for b in range(k):
            if (g >> b) & 1:
                acc ^= np.roll(u, (k - 1) - b)
        out[:, gi] = acc
    return out


@lru_cache(maxsize=None)
def interleaver_i_index() -> np.ndarray:
    """Matrix index read by interleaver I for each of the 365 440 punctured P1
    bits (reference src/decode.c:296-322 with J=20,B=16,C=36,M=1)."""
    i = np.arange(P1_BITS * 5 // 2, dtype=np.int64)
    J, B, C = 20, 16, 36
    part = PM_V[i % 20]
    block = ((i // J) + part * 7) % B
    k = i // (J * B)
    row = (k * 11) % 32
    col = (k * 11 + k // (32 * 9)) % C
    return (block * 32 + row) * (J * C) + part * C + col


@lru_cache(maxsize=None)
def interleaver_ii_index() -> np.ndarray:
    """[16, 200] matrix indices for the PIDS bits of each block
    (reference src/decode.c:324-342 with b=200, I0=365 440)."""
    J, B, C, b, I0 = 20, 16, 36, 200, 365440
    i = np.arange(16 * b, dtype=np.int64)
    part = PM_V[i % 20]
    block = i // b
    k = ((i // J) % (b // J)) + (I0 // (J * B))
    row = (k * 11) % 32
    col = (k * 11 + k // (32 * 9)) % C
    return ((block * 32 + row) * (J * C) + part * C + col).reshape(16, b)


# ----------------------------------------------------------------------------
# GF(256) Reed-Solomon (255,247) systematic encoder, poly 0x11d, fcr=1, prim=1
# (decoder side: reference src/rs_decode.c, src/rs_init.c:31-133 as configured
#  by src/frame.c:747).  The reference only declares an encoder (rs_char.h:48).
# ----------------------------------------------------------------------------
@lru_cache(maxsize=None)
def _gf_tables():
    exp = np.zeros(512, dtype=np.int32)
    log = np.zeros(256, dtype=np.int32)
    sr = 1
    for i in range(255):
        exp[i] = sr
        log[sr] = i
        sr <<= 1
        if sr & 0x100:
            sr ^= 0x11D
    exp[255:510] = exp[0:255]
    return exp, log


def _gf_mul(a: int, b: int) -> int:
    if a == 0 or b == 0:
        return 0
    exp, log = _gf_tables()
    return int(exp[log[a] + log[b]])


@lru_cache(maxsize=None)
def _rs_genpoly():
    exp, _ = _gf_tables()
    g = [1]
    for i in range(8):
        root = int(exp[1 + i])
        ng = [0] * (len(g) + 1)
        for j, c in enumerate(g):  # multiply by (x + root); g[j] is coeff of x^j
            ng[j + 1] ^= c
            ng[j] ^= _gf_mul(c, root)
        g = ng
    return g  # degree 8, g[8] == 1


def rs_parity(msg247: bytes) -> bytes:
    """Parity of the systematic (255,247) code; msg247[0] is the highest-degree
    symbol.  Returns 8 bytes, highest degree first (codeword = msg + parity)."""
    g = _rs_genpoly()
    rem = [0] * 8  # rem[0] = coefficient of x^7
    for m in msg247:
        fb = m ^ rem[0]
        rem = rem[1:] + [0]
        if fb:
            for j in range(8):
                rem[j] ^= _gf_mul(fb, g[7 - j])
    return bytes(rem)


def audio_pdu_header(fields: bytes | None = None, rng=None) -> bytes:
    """A valid 96-byte RS-protected L2 audio-PDU header as laid out by reference
    src/frame.c:158-196: buf[0..7] parity, buf[8..13] header fields, rest payload.
    Default fields: codec 0, stream 0, nop=0, hef=0, la_location=13, so the
    reference's frame_process() consumes the header, finds no packets and stops."""
    buf = bytearray(96)
    if rng is not None:
        buf[14:96] = rng.integers(0, 256, 82, dtype=np.uint8).tobytes()
    if fields is None:
        fields = bytes([0x00, 0x00, 0x00, 0x00, 0x00, 13])
    buf[8:14] = fields
    # reference block: hdr[254 - i] = buf[i]; positions 0..158 are zero padding
    msg = bytes(159) + bytes(buf[95 - k] for k in range(88))
    par = rs_parity(msg)  # block[247..254] = buf[7..0]
    for k in range(8):
        buf[7 - k] = par[k]
    return bytes(buf)


def build_p1_frame_bits(rng, pci: int = PCI_AUDIO, valid_header: bool = True) -> np.ndarray:
    """146 176 descrambled frame bits exactly as handed to frame_push()
    (reference src/frame.c:645-714): per-byte bit reversal, 24 PCI bits at
    logical positions 116176 + 1248 h, the rest packed MSB-first into the PDU."""
    logical = np.zeros(P1_BITS, dtype=np.uint8)
    pci_pos = 116176 + 1248 * np.arange(24)
    is_pci = np.zeros(P1_BITS, dtype=bool)
    is_pci[pci_pos] = True
    logical[pci_pos] = [(pci >> (23 - h)) & 1 for h in range(24)]
    npdu = P1_BITS - 24
    pdu = rng.integers(0, 256, npdu // 8, dtype=np.uint8)
    if valid_header:
        pdu[:96] = np.frombuffer(audio_pdu_header(rng=rng), dtype=np.uint8)
    else:
        # last PDU byte with unequal nibbles (no fixed-data sync, frame.c:448-456)
        pdu[-1] = 0x12
    logical[~is_pci] = np.unpackbits(pdu)  # MSB first
    i = np.arange(P1_BITS)
    phys = (i & ~7) + 7 - (i & 7)
    bits = np.zeros(P1_BITS, dtype=np.uint8)
    bits[phys] = logical
    return bits


def pids_crc12(pids: np.ndarray) -> int:
    """CRC-12 over bits 0..67 of a PIDS frame in pids_frame_push's bit order (reference src/pids.c:52-72)."""
    reg = 0
    for i in range(67, -1, -1):
        low = reg & 1
        reg = (reg >> 1) ^ (int(pids[i]) << 15)
        if low:
            reg ^= 0xD010
    for _ in range(16):
        low = reg & 1
        reg >>= 1
        if low:
            reg ^= 0xD010
    return (reg ^ 0x955) & 0xFFF


def pids_with_crc(frame_bits: np.ndarray) -> np.ndarray:
    """The same 80 frame bits with bits 68..79 (in pids_frame_push's per-byte reversed order, src/pids.c:1036-1040)
    replaced by the CRC-12 of the first 68, so that the reference's L2 accepts the frame."""
    i = np.arange(80)
    order = ((i >> 3) << 3) + 7 - (i & 7)            # pids[i] = frame_bits[order[i]]
    pids = frame_bits[order].copy()
    crc = pids_crc12(pids)
    pids[68:80] = [(crc >> (11 - k)) & 1 for k in range(12)]
    out = frame_bits.copy()
    out[order] = pids
    return out


# ----------------------------------------------------------------------------
# reference subcarriers
# ----------------------------------------------------------------------------
def ref_raw_bits(bc: int, psmi: int, rsid: int) -> np.ndarray:
    """32 raw BPSK bits of one reference subcarrier for one block, such that
    decode_ref_fm() (reference src/sync.c:169-186) accepts it and decodes
    block count `bc` and service mode `psmi` after DBPSK decoding."""
    r = np.zeros(32, dtype=np.uint8)
    fixed = {0: 0, 1: 1, 2: 0, 3: 0, 4: 0, 5: 1, 6: 1, 8: 1, 9: 0, 10: rsid >> 1,
             11: (rsid >> 1) ^ (rsid & 1), 13: 0, 14: 0, 20: 0, 21: 1, 22: 0, 31: 0}
    for k, v in fixed.items():
        r[k] = v
    r[15] = 0
    for n, sh in zip(range(16, 20), (3, 2, 1, 0)):
        r[n] = r[n - 1] ^ ((bc >> sh) & 1)
    r[23] = r[24] = 0
    for n, sh in zip(range(25, 31), (5, 4, 3, 2, 1, 0)):
        r[n] = r[n - 1] ^ ((psmi >> sh) & 1)
    return r


# ----------------------------------------------------------------------------
# capture
# ----------------------------------------------------------------------------
@dataclass
class FmCapture:
    cu8: np.ndarray                      # uint8 [2 * nsamples], I/Q interleaved
    p1_frames: list = field(default_factory=list)    # list of uint8[146176] frame bits
    pids_frames: list = field(default_factory=list)  # list of uint8[80], block order
    p3_frames: list = field(default_factory=list)    # MP2/MP3/MP11: list of uint8[2304 or 4608] the receiver will output
    p4_frames: list = field(default_factory=list)    # MP11: list of uint8[4608] (PX2)
    psmi: int = 1
    lead_in: int = 0


# ----------------------------------------------------------------------------
# P3 (MP3): convolutional interleaver IV
# ----------------------------------------------------------------------------
P3_BITS = 4608
PX1_BLOCK = 4608                      # PX1 soft bits per block in MP3 (2 partitions per sideband)
IV_N = 147456                         # interleaver IV span: 16 P3 frames = 32 blocks


@lru_cache(maxsize=None)
def interleaver_iv_delay(frame_len: int = P3_BITS) -> np.ndarray:
    """D[m]: the deinterleaver's output m (mod N) is the input it received D[m] positions earlier, 1 <= D <= N
    (reference src/decode.c:344-376; MP3/MP11: J=4, M=2, N=147456; MP2, frame_len 2304: J=2, M=4, N=73728):
    it reads internal[A(m)] before it stores input m at internal[m]."""
    if frame_len == P3_BITS:
        J, M, N = 4, 2, IV_N
    else:
        J, M, N = 2, 4, IV_N // 2
    B, C = 32, 36
    bk_bits, bk_adj = 32 * C, 32 * C - 1
    m = np.arange(N, dtype=np.int64)
    part = ((m + 2 * (M // 4)) // M) % J
    pti = np.empty(N, dtype=np.int64)
    for pp in range(J):
        sel = part == pp
        pti[sel] = np.arange(int(sel.sum()))
    block = (pti + part * 7 - bk_adj * (pti // bk_bits)) % B
    row = ((11 * pti) % bk_bits) // C
    col = (pti * 11) % C
    A = (block * 32 + row) * (J * C) + part * C + col
    return np.where(A < m, m - A, m - A + N)


def build_p3_frame_bits(rng, nbits: int = P3_BITS) -> np.ndarray:
    """4608 (MP2: 2304) descrambled P3 / P4 frame bits as handed to frame_push() (frame.c:658-668: PCI at logical
    bits 120 + 184 h, MP2: 120 + 88 h); PCI says fixed data only and the last byte rules out a fixed-data sync
    (frame.c:448-456)."""
    step = 184 if nbits == P3_BITS else 88
    logical = np.zeros(nbits, dtype=np.uint8)
    pci_pos = 120 + step * np.arange(24)
    is_pci = np.zeros(nbits, dtype=bool)
    is_pci[pci_pos] = True
    logical[pci_pos] = [(PCI_FIXED >> (23 - h)) & 1 for h in range(24)]
    pdu = rng.integers(0, 256, (nbits - 24) // 8, dtype=np.uint8)
    pdu[-1] = 0x12
    logical[~is_pci] = np.unpackbits(pdu)
    i = np.arange(nbits)
    phys = (i & ~7) + 7 - (i & 7)
    bits = np.zeros(nbits, dtype=np.uint8)
    bits[phys] = logical
    return bits


def _px_stream(prng, nblocks: int, first_even: int, frame_len: int, supplied=None):
    """The bit stream of one extended-partition group (PX1 or PX2) over `nblocks` blocks of `frame_len` soft bits
    each, and the frames a receiver hands out: the deinterleaver starts with the first even block it sees and
    returns frame c (inputs of blocks 2c, 2c+1 counted from there) once 16 frames have gone in; transmit stream
    position j carries the punctured coded bit of output position k = j + D[k mod N]."""
    ncalls = (nblocks - first_even) // 2
    D = interleaver_iv_delay(frame_len)
    N = D.size
    px = prng.integers(0, 2, nblocks * frame_len, dtype=np.uint8)
    tx = px[first_even * frame_len:]
    pn = pn_sequence(frame_len)
    keep3 = np.tile(np.array([1, 0, 1, 1, 0, 1], dtype=bool), frame_len * 3 // 6)
    frames = []
    for c in range(ncalls):
        fb = build_p3_frame_bits(prng, frame_len)
        if supplied is not None and c < len(supplied) and supplied[c] is not None:      # caller's PDUs (packed, synth_l2.py)
            fb = np.unpackbits(np.frombuffer(supplied[c], dtype=np.uint8))[:frame_len]
        u = conv_encode_tb(fb ^ pn).reshape(-1)[keep3]                 # 2 * frame_len transmitted bits
        k = c * 2 * frame_len + np.arange(2 * frame_len, dtype=np.int64)
        j = k - D[k % N]
        ok = j >= 0
        tx[j[ok]] = u[ok]
        if c >= N // (2 * frame_len):
            frames.append(fb)
    return px, frames


@lru_cache(maxsize=None)
def _shape2x() -> np.ndarray:
    """Receiver pulse shape (reference src/acquire.c:322-331) sampled at 2x."""
    j = np.arange(2 * FFTCP, dtype=np.float64)
    s = np.ones(2 * FFTCP)
    s[: 2 * CP] = np.sin(np.pi / 2 * j[: 2 * CP] / (2 * CP))
    s[2 * FFT:] = np.cos(np.pi / 2 * (j[2 * FFT:] - 2 * FFT) / (2 * CP))
    return s


def _block_matrix_to_bins(mat_block: np.ndarray, refs: dict) -> np.ndarray:
    """mat_block: [32 rows][20 partitions][36 cols] bits -> complex S[32, 2048]
    in the receiver's fftshift-ed bin order (sync.c:509-536)."""
    S = np.zeros((BLKSZ, FFT), dtype=np.complex128)
    sym = (2.0 * mat_block.astype(np.float64) - 1.0)
    iq = sym[:, :, 0::2] + 1j * sym[:, :, 1::2]  # [32, 20, 18]
    for p in range(20):
        base = LB_START + 19 * p + 1 if p < 10 else (UB_END - 190) + 19 * (p - 10) + 1
        S[:, base:base + 18] = iq[:, p, :]
    for b, raw in refs.items():
        S[:, b] = (2.0 * raw.astype(np.float64) - 1.0) * (1 + 1j)
    return S


def make_fm_mp1(**kw) -> FmCapture:
    """FM hybrid MP1 (PSMI 1), see make_fm."""
    return make_fm(psmi=1, **kw)


def compat_mode(psmi: int) -> int:
    """compatibility_mode[psmi] of the reference (src/sync.c:30-35)."""
    return (0, 1, 2, 3, 1, 5, 6, 5, 6, 1, 2, 11, 1, 5, 6, 5)[psmi & 15] if psmi & 15 else (0 if psmi == 0 else 6)


def make_fm_mp3(**kw) -> FmCapture:
    """FM extended hybrid MP3 (PSMI 3): 13 reference subcarriers and 12 partitions per sideband, P3 on the
    two PX1 partitions per sideband.  P3 frames only come out after the interleaver has filled
    (16 P3 frames = 2 L1 frames), so use nframes >= 3."""
    return make_fm(psmi=3, **kw)


def make_fm(psmi: int = 1, nframes: int = 2, seed: int = 1234, lead_in: int = 1000, cfo_hz: float = 0.0,
            noise_lsb: float = 0.0, noise_seed: int = 5, rms_lsb: float = 20.0,
            tail_blocks: int = 2, valid_header: bool = True, pci: int = PCI_AUDIO,
            start_bc: int = 0, pids_crc: bool = False, p1_frames=None, p3_frames=None) -> FmCapture:
    """FM capture of service mode `psmi` holding `nframes` complete L1 frames
    followed by `tail_blocks` further blocks so the last frame flushes
    (the reference has no flush call, SURVEY §3.5).

    What the reference does with the service modes (src/sync.c:343-357,537-595): MP2 = one more partition per
    sideband carrying P3 frames of 2304 bits (PX1); MP3 = two more, P3 frames of 4608 bits; MP11 = four more,
    PX1 as in MP3 plus PX2 with P4 frames of 4608 bits; MP5 / MP6 = fourteen partitions per sideband tracked,
    equalised and counted in the MER, only the twenty main ones decoded (filled with unrelated QPSK here).
    Any of the 64 PSMI values: the capture is laid out by its compatibility mode (compat_mode: 1, 2, 3, 5, 6 or 11)
    and the reference subcarriers carry the raw value, which is what the receiver reports in its SYNC."""
    cm = compat_mode(psmi)
    assert 0 <= psmi < 64 and cm in (1, 2, 3, 5, 6, 11)
    rng = np.random.default_rng(seed)
    nref = {1: 11, 2: 12, 3: 13, 5: 15, 6: 15, 11: 15}[cm]
    nblocks = nframes * BLOCKS_PER_FRAME + tail_blocks
    idx_i = interleaver_i_index()
    idx_ii = interleaver_ii_index()
    pn_p1 = pn_sequence(P1_BITS)
    pn_pids = pn_sequence(PIDS_BITS)
    cap = FmCapture(cu8=None, psmi=psmi, lead_in=lead_in)

    nfr_total = (nblocks + start_bc + BLOCKS_PER_FRAME - 1) // BLOCKS_PER_FRAME
    mats = []
    for f in range(nfr_total):
        if p1_frames is not None and f < len(p1_frames) and p1_frames[f] is not None:   # caller's P1 PDUs (packed, synth_l2.py)
            bits = np.unpackbits(np.frombuffer(p1_frames[f], dtype=np.uint8))[:P1_BITS]
        else:
            bits = build_p1_frame_bits(rng, pci=pci, valid_header=valid_header)
        coded = conv_encode_tb(bits ^ pn_p1).reshape(-1)          # 438528
        keep = np.ones(coded.size, dtype=bool)
        keep[5::6] = False
        mat = np.zeros(16 * PM_BLOCK, dtype=np.uint8)
        mat[idx_i] = coded[keep]
        pids_this = []
        for bc in range(16):
            pb = rng.integers(0, 2, PIDS_BITS, dtype=np.uint8)
            if pids_crc:
                pb = pids_with_crc(pb)
            pc = conv_encode_tb(pb ^ pn_pids).reshape(-1)         # 240
            k2 = np.ones(pc.size, dtype=bool)
            k2[5::6] = False
            mat[idx_ii[bc]] = pc[k2]
            pids_this.append(pb)
        mats.append((bits, pids_this, mat.reshape(16, 32, 20, 36)))

    # extended partitions: (first bin of the 18 data carriers, ...) per group in the receiver's demap order
    # (sync.c:537-595) and the bits they carry, [block][symbol][group][carrier][re, im]
    first_even = start_bc % 2                         # PX blocks before the first even block are read by nobody
    ext = []                                          # (bases, bits)
    if cm == 3:
        px1, cap.p3_frames = _px_stream(np.random.default_rng(seed + 7919), nblocks, first_even, PX1_BLOCK, p3_frames)
        ext.append(((LB_START + 190 + 1, LB_START + 209 + 1, UB_END - 228 + 1, UB_END - 209 + 1),
                    px1.reshape(nblocks, BLKSZ, 4, 18, 2)))
    elif cm == 2:
        px1, cap.p3_frames = _px_stream(np.random.default_rng(seed + 7919), nblocks, first_even, PX1_BLOCK // 2)
        ext.append(((LB_START + 190 + 1, UB_END - 209 + 1), px1.reshape(nblocks, BLKSZ, 2, 18, 2)))
    elif cm == 11:
        px1, cap.p3_frames = _px_stream(np.random.default_rng(seed + 7919), nblocks, first_even, PX1_BLOCK, p3_frames)
        px2, cap.p4_frames = _px_stream(np.random.default_rng(seed + 7920), nblocks, first_even, PX1_BLOCK)
        ext.append(((LB_START + 190 + 1, LB_START + 209 + 1, UB_END - 228 + 1, UB_END - 209 + 1),
                    px1.reshape(nblocks, BLKSZ, 4, 18, 2)))
        ext.append(((LB_START + 228 + 1, LB_START + 247 + 1, UB_END - 266 + 1, UB_END - 247 + 1),
                    px2.reshape(nblocks, BLKSZ, 4, 18, 2)))
    elif cm in (5, 6):
        fill = np.random.default_rng(seed + 7921).integers(0, 2, (nblocks, BLKSZ, 8, 18, 2), dtype=np.uint8)
        ext.append((tuple(LB_START + 19 * q + 1 for q in range(10, 14)) + tuple(UB_END - 19 * (q + 1) + 1 for q in range(13, 9, -1)),
                    fill))

    sh = _shape2x()
    sig = np.zeros(nblocks * BLKSZ * 2 * FFTCP, dtype=np.complex128)
    first_full = None
    for blk in range(nblocks):
        g = blk + start_bc
        f, bc = divmod(g, 16)
        bits, pids_this, mat = mats[f]
        refs = {}
        for i in range(nref):
            raw = ref_raw_bits(bc, psmi, (30 - i) & 3)
            refs[LB_START + 19 * i] = raw
            refs[UB_END - 19 * i] = raw
        S = _block_matrix_to_bins(mat[bc], refs)
        for bases, bits_x in ext:                     # PX1 / PX2 / filler partitions (sync.c:537-595)
            symx = 2.0 * bits_x[blk].astype(np.float64) - 1.0
            iqx = symx[..., 0] + 1j * symx[..., 1]    # [32, groups, 18]
            for q, base in enumerate(bases):
                S[:, base:base + 18] = iqx[:, q, :]
        # receiver computes fftshift(FFT(conj(x)));  build y = conj(x) at 2x rate
        S2 = np.zeros((BLKSZ, 2 * FFT), dtype=np.complex128)
        fidx = (np.arange(FFT) - FFT // 2) % (2 * FFT)
        S2[:, fidx] = S
        y = np.fft.ifft(S2, axis=1) * (2 * FFT)
        ysym = y[:, np.arange(2 * FFTCP) % (2 * FFT)] * sh[None, :]
        sig[blk * BLKSZ * 2 * FFTCP:(blk + 1) * BLKSZ * 2 * FFTCP] = np.conj(ysym).reshape(-1)
    # bookkeeping of what a receiver will output
    for f in range(nfr_total):
        g0 = f * 16 - start_bc
        if g0 >= 0 and g0 + 16 <= nblocks:
            cap.p1_frames.append(mats[f][0])
    for blk in range(nblocks):
        f, bc = divmod(blk + start_bc, 16)
        cap.pids_frames.append(mats[f][1][bc])

    sig *= rms_lsb / np.sqrt(np.mean(np.abs(sig) ** 2) / 2.0)
    nlead = lead_in
    full = np.concatenate([np.zeros(nlead, dtype=np.complex128), sig])
    if cfo_hz != 0.0:
        t = np.arange(full.size)
        full *= np.exp(2j * np.pi * cfo_hz * t / 1488375.0)
    nrng = np.random.default_rng(noise_seed)
    sigma = noise_lsb if noise_lsb > 0 else 0.0
    # the lead-in always carries a little noise so it is not a constant run
    lead_sigma = max(sigma, 1.0)
    noise = np.empty(full.size, dtype=np.complex128)
    noise.real = nrng.standard_normal(full.size)
    noise.imag = nrng.standard_normal(full.size)
    scale = np.full(full.size, sigma)
    scale[:nlead] = lead_sigma
    full += noise * scale
    iq = np.empty(2 * full.size, dtype=np.float64)
    iq[0::2] = full.real
    iq[1::2] = full.imag
    cap.cu8 = np.clip(np.rint(iq + 127.0), 0, 255).astype(np.uint8)
    return cap


def pack_bits(bits: np.ndarray) -> bytes:
    """MSB-first packing, the format of the engine's and reftap's PDU records."""
    return np.packbits(np.asarray(bits, dtype=np.uint8)).tobytes()
