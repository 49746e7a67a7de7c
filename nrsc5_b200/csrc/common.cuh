// Shared definitions for the nrsc5_b200 CUDA engine (sm_90a).
//
// Vocabulary follows the reference domain: a *stream* is one independent
// radio channel (one nrsc5_t in the reference); a *block* is 32 OFDM symbols
// (reference src/defines.h:20); an L1 *frame* is 16 blocks.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nb {

constexpr int NFFT = 2048;
constexpr int NCP = 112;
constexpr int NSYM = NFFT + NCP;            // 2160 decimated samples per OFDM symbol
constexpr int BLK = 32;                     // symbols per block
constexpr int NACQ = NSYM * (BLK + 1);      // 71280: acquisition window (reference src/acquire.h:12)
constexpr int LB0 = NFFT / 2 - 546;         // 478
constexpr int UB1 = NFFT / 2 + 546;         // 1570
constexpr int PW = 19;
constexpr int MAXPART = 14;
constexpr int SIDE = MAXPART * PW + 1;      // 267 bins kept per sideband (reference src/sync.c:785-789)
constexpr int NBINS = 2 * SIDE;             // 534
constexpr int PM_BLOCK = 23040;
constexpr int P1_LEN = 146176;
constexpr int P1_ENC = P1_LEN * 5 / 2;      // 365440
constexpr int P1_VIT = P1_LEN * 3;          // 438528
constexpr int P1_STEPS = P1_LEN + 64;       // tail-biting: 32 pre-roll + 32 post-roll
constexpr int PIDS_LEN = 80;
constexpr int P3_LEN = 4608;                // P3 frame bits in MP3/MP11 (reference src/defines.h:53)
constexpr int IV_N = 147456;                // span of interleaver IV (reference src/decode.c:350)
constexpr int PX_RING = 2 * IV_N;
constexpr int P3_SLOTS = 8;                 // P3 frames per stream and pass (one per two blocks)
constexpr int P3_DEC_STRIDE = 5120;         // decisions per frame: 5 fallback chunks of 1024 >= 4608 + 64
constexpr int P3S_LEN = 2304, IV_NS = IV_N / 2;    // MP2: P3 frame bits, interleaver IV span (decode.c:346-350)

// The extended-partition decode groups, in launch order - the reference's call order, P3 before P4:
//   0 = MP3 / MP11's P3, 1 = MP2's short P3, 2 = MP11's P4.
// len: frame bits, which are also the group's soft bits per block; its interleaver IV spans 32 frames (IV_N, IV_NS)
// and reads the delay table iv_delay (len == P3_LEN) or iv_delay_s.  ring: 0 = PX1, 1 = PX2.  lc: logical channel.
// modes: bit m set = compatibility mode m feeds the group (a mode feeds at most one group per ring).
// The host launches a group once a stream has asked for it: bit g of px_need_of(mode).
struct PxGroup { int len, ring, lc, modes; };
constexpr int PX_GROUPS = 3;
__host__ __device__ constexpr PxGroup px_group(int g)
{
    return g == 0 ? PxGroup{ P3_LEN, 0, 1, 1 << 3 | 1 << 11 }
         : g == 1 ? PxGroup{ P3S_LEN, 0, 1, 1 << 2 }
                  : PxGroup{ P3_LEN, 1, 2, 1 << 11 };
}
static_assert(32 * P3_LEN == IV_N && 32 * P3S_LEN == IV_NS, "a group's interleaver IV spans 32 frames");
__host__ __device__ constexpr int px_need_of(int cm)
{
    int need = 0;
    for (int g = 0; g < PX_GROUPS; g++) need |= (px_group(g).modes >> cm & 1) << g;
    return need;
}
constexpr int ST_NONE = 0, ST_COARSE = 1, ST_FINE = 2;

// record types (include/nrsc5_b200.h)
constexpr uint32_t REC_FRAME = 1, REC_PIDS = 2, REC_SYNC = 3, REC_LOST_SYNC = 4, REC_MER = 5,
                   REC_BER = 6, REC_SOFT_PM = 8, REC_BLOCK = 9, REC_PAD = 12;

// bin index inside the compact 534-bin spectrum kept per symbol
__host__ __device__ inline int compact_of_bin(int b)   // b in fftshift-ed coordinates
{
    if (b >= LB0 && b < LB0 + SIDE) return b - LB0;
    if (b > UB1 - SIDE && b <= UB1) return SIDE + (b - (UB1 - SIDE + 1));
    return -1;
}

constexpr int L2_QUEUE = 40;                // frames + resets one pass can hand to L2 (16 blocks: 1 P1, 8 P3, 8 P4)

// Per-stream persistent state.  One instance per stream in device memory.
struct StreamState {
    // input cursor
    long long in_avail;        // cu8 complex samples available from absolute index 0
    long long start;           // decimated index of the acquisition window's first sample
    // acquisition (reference src/acquire.h:24-28)
    float prev_angle;
    float2 phase;
    int keep_extra;
    int cfo;
    int state;
    // feedback from sync (reference src/sync.h:21-22)
    int samperr;
    float angle;
    // sync (reference src/sync.h:13-31)
    int psmi, cfo_wait, bc, mer_cnt;
    float err_lb, err_ub;
    // decode
    int started_pm;
    // per-block hand-off prep -> demod -> sync
    int active;                // this step has a full window for the stream
    int blk_samperr;
    int blk_state_in;
    int blk_go;                // cluster per stream: the owner CTA's word to its helpers - 1 demodulate this block, 0 leave
    float theta;               // NCO step, radians per decimated sample
    float2 phase0;             // NCO phase at the first sample of the block
    // P1 hand-off sync -> p1 kernel
    int p1_ready;
    int p1_slow;               // this frame needs saturating Viterbi arithmetic
    int p1_retry;              // the register-resident fast path could not prove its result: use the exact fallback kernels
    unsigned p1_rec;           // log offset of the reserved BER payload (FRAME record follows)
    unsigned p1_lost_rec;      // log offset of the REC_PAD slot kept for the frame's sync loss, 0xffffffff = none
    int p1_errs;               // channel bit errors counted so far
    int p1_done;               // k_p1_fin CTAs finished
    int pids_pending;          // PIDS frames (of blocks pids_bc[]) waiting to be decoded into the log slots pids_rec[];
    int pids_bc[16];           // k_stream decodes them together, one warp each, before it exits
    unsigned pids_rec[16];
    // extended partitions: convolutional interleaver IV bookkeeping per ring, [0] = PX1, [1] = PX2 (reference
    // src/decode.c:344-437) ...
    long long px_total[2];     // soft bits taken in since the interleaver (re)started
    int px_started[2];
    // ... and per decode group (px_group) the frames waiting for the decode kernels that follow k_stream
    int xq_pending[PX_GROUPS];
    long long xq_k0[PX_GROUPS][P3_SLOTS];  // interleaver position of each frame's first soft bit
    unsigned xq_rec[PX_GROUPS][P3_SLOTS];  // log offset of each frame's reserved FRAME record
    int force_state;           // host override (nrsc5b_set_sync_state), -1 = none
    // L2 on the device (l2.cuh): what the pass handed to L2 so far, in the reference's call order - frames by the log
    // offset of their packed bits (0xffffffff: the log was full), nbits == 0 for a frame_reset (entering fine sync)
    int l2_n;
    unsigned l2_off[L2_QUEUE], l2_lc[L2_QUEUE], l2_nbits[L2_QUEUE];
    // output log cursor
    unsigned log_len;
    unsigned log_overflow;
    unsigned long long blocks_done;
    unsigned long long frames_done;
    unsigned long long p1_fallbacks;    // P1 frames decoded by the exact fallback Viterbi
    // SM cycles spent per phase of k_stream (thread 0's clock): pids flush, prep with acquisition, prep in FINE,
    // demod, sync of a block that started in FINE, sync of any other block (vote / CFO search)
    unsigned long long ph_cyc[6];
    unsigned long long ph_n[6];
    // sub-phases of a FINE block's sync: reference gather, Costas loops, amplitude/phase tables + feedback,
    // staging, equalise + error sums, demap + bookkeeping
    unsigned long long sy_cyc[6];
    // history of the coarse band-pass FIR: the last 31 samples it was fed
    short bp_hist[31][2];
    short bp_hist_next[31][2];     // ... of the window being acquired (front_acq_tiles), taken over once all its tiles are done
};

struct EngineDims {
    int nstreams;
    size_t in_stride;          // bytes between streams in the cu8 buffer
    size_t log_cap;            // bytes of log per stream
    int emit_soft;
    int cs16;                  // input is cs16 at the decimated rate: 4 bytes per sample, no halfband
    int px_enabled;            // bit g: the host launches extended-partition decode group g after k_stream
    int l2;                    // frames also go through L2 on the device (nrsc5b_enable_l2)
    int cluster;               // CTAs per stream in k_stream (thread-block cluster): 1, 2 or 4
};

// buffers of one extended-partition decode group, [S][P3_SLOTS]... (null until the host enables the group)
struct PxBufs {
    int8_t *vin;               // [3 * len] deinterleaved + depunctured soft bits
    uint2 *dec;                // [P3_DEC_STRIDE] survivor decisions
    uint32_t *spec, *end;      // [19][32] fast Viterbi chunk boundary metrics
    int *endstate;             // [1]
    uint2 *fspec, *fend;       // [5][16] fallback Viterbi
    int *fhstate, *ftbend;     // [5]
    uint32_t *bits;            // [len / 32] decoded (still scrambled) bits
    int *flags;                // [4] ready, slow, retry, -
};

// Per-engine control words in device memory (one engine = one instance: engines on one device share nothing).
struct EngineCtl {
    unsigned long long progress;   // bumped by every stream that processed a block
    unsigned px_need;              // bit g: a stream waits for decode group g, which the host has not enabled
    unsigned more;                 // streams that could go on after the last pass of a batch (a full window is buffered)
};

// What the host needs to know about a stream to plan the next batch of passes (written when k_stream / k_am exit).
struct StreamBrief {
    long long start;               // decimated index of the window's first sample
    int state, bc, p1_ready, pad_;
};

// Pointers to all device arrays, passed by value to kernels.
struct DevPtrs {
    EngineCtl *ctl;            // [1]
    StreamBrief *brief;        // [S]
    const uint8_t *iq;         // [S][in_stride] cu8
    StreamState *st;           // [S]
    float *cfreq;              // [S][2048]
    float *cphase;             // [S][2048]
    float2 *nco;               // [S][2160]  window * exp(j*theta*j)
    float2 *bins;              // [S][32][534]
    int8_t *pm;                // [S][16][23040]
    short2 *ydec;              // [S][71280]   decimated window (coarse acquisition scratch)
    float2 *acq_sums;          // [S][2160]    cyclic-prefix correlation per sample offset (coarse acquisition)
    float2 *tbuf;              // [S][71280]   band-passed window (coarse acquisition scratch)
    int8_t *vit_in;            // [S][438528]
    uint2 *vit_dec;            // [S][146240]
    uint32_t *p1_bits;         // [S][146176/32] decoded (still scrambled) bits, bit k of word w = frame bit 32w+k
    uint2 *vspec, *vend;       // [S][143][16] chunk boundary metrics of the fallback P1 Viterbi
    int *hstate, *tbend;       // [S][143]
    uint32_t *v64_spec, *v64_end;   // [S][V64 chunks][32] chunk boundary metrics of the fast P1 Viterbi
    int *v64_endstate;         // [S]
    int8_t *px_ring[2];        // [S][2 * IV_N] PX1 / PX2 (MP11) soft bits in arrival order (the last two interleaver spans)
    const uint32_t *iv_delay;  // [IV_N] interleaver IV: output m comes from the input iv_delay[m] positions earlier
    const uint32_t *iv_delay_s;     // [IV_NS] interleaver IV of MP2 (J=2, M=4)
    PxBufs xb[PX_GROUPS];      // per decode group (px_group)
    uint8_t *log;              // [S][log_cap]
    const float *shape;        // [2160]
    const float2 *twid;        // [FFT_TW] twiddle tables of fft2048_block (fft.cuh)
    const uint32_t *p1_lut;    // [365440] interleaver I gather index
    const uint8_t *pn;         // [146176] descrambler sequence, one bit per byte
    const uint32_t *pnw;       // [146176/32] the same, packed (bit i of word i/32)
};

// ---- log writer: one CTA owns a stream's log at any time ----
__device__ inline uint8_t *log_reserve(const DevPtrs &p, const EngineDims &d, int s, uint32_t type, uint32_t plen)
{
    StreamState &st = p.st[s];
    uint32_t need = 8 + ((plen + 3) & ~3u);
    if ((size_t)st.log_len + need > d.log_cap) {
        st.log_overflow = 1;
        return nullptr;
    }
    uint8_t *w = p.log + (size_t)s * d.log_cap + st.log_len;
    reinterpret_cast<uint32_t *>(w)[0] = type;
    reinterpret_cast<uint32_t *>(w)[1] = plen;
    st.log_len += need;
    return w + 8;
}

// hands a frame (off = log offset of its packed bits, 0xffffffff when the log was full) or, with nbits == 0, a
// frame_reset to the L2 kernel that ends the pass
__device__ __forceinline__ void l2_enqueue(StreamState &st, int l2_on, unsigned off, unsigned lc, unsigned nbits)
{
    if (!l2_on) return;
    if (st.l2_n >= L2_QUEUE) {                 // cannot happen with 16 blocks per pass; the host is told if it does
        st.log_overflow = 1;
        return;
    }
    const int e = st.l2_n++;
    st.l2_off[e] = off;
    st.l2_lc[e] = lc;
    st.l2_nbits[e] = nbits;
}

// The halfband decimator /2 of the cu8 front end (reference src/firdecim_q15.c:137-151, input.c:52-94; taps
// int16{-134,1078,-4417,19864}) over a run of R consecutive outputs: y[r] from the cu8 words w[r] .. w[r+7], where
// word q holds input samples 2q (low half) and 2q+1 (high half) - before the stream's first sample the words are
// 0x7f7f7f7f, the decimator's zero history (firdecim_q15.c:33).
//   y = x[2d-7] + sum_k ((x[2d-14+2k] + x[2d-2k]) * tap_k) >> 15,   x = (u8 - 127) * 64
// i.e. per term (s * tap_k) >> 9 with s = u8 + u8 - 254, floored term by term as the reference does, plus 64 times the
// centre sample.  |y| <= 256 * 25493 / 512 + 8192 < 32767: int accumulators are exact and never wrap.
// The window slides one word per output, so each word is loaded once, not once per output that uses it.  The bytes
// are never extracted: one byte permute puts the real and imaginary bytes of a tap pair side by side, and a
// two-way dot product with the tap in both 16-bit halves of `a` forms (u8 + u8) * tap - 254 * tap in one instruction
// per component (the bias is its addend); the centre term is a dot product with 64 as well.  Every product is the
// exact integer of the form above.  w[] and y[] may be shared or global memory.
//
// dp2a: c + a.h0 * b.b0 + a.h1 * b.b1 (HI = false) or b.b2, b.b3 (HI = true), a's halves signed, b's bytes unsigned
template <bool HI>
__device__ __forceinline__ int dp2a_su(int a, uint32_t b, int c)
{
#if defined(NB_EMU)
    const int s = HI ? 16 : 0;
    return c + (int)(short)(a & 0xffff) * (int)((b >> s) & 0xffu) + (int)(short)(a >> 16) * (int)((b >> (s + 8)) & 0xffu);
#else
    int d;
    if (HI) asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    else    asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
#endif
}

template <int R>
__device__ __forceinline__ void halfband_run(const uint32_t *w, short2 *y)
{
    const int tap[4] = { -134, 1078, -4417, 19864 };
    uint32_t v[R + 7];
#pragma unroll
    for (int q = 0; q < R + 7; q++) v[q] = w[q];
#pragma unroll
    for (int r = 0; r < R; r++) {
        // 64 x[2r+7] - 127 * 64, from the high half of word r + 3
        int ar = dp2a_su<true>(64, v[r + 3], -127 * 64), ai = dp2a_su<true>(64 << 16, v[r + 3], -127 * 64);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t pr = __byte_perm(v[r + k], v[r + 7 - k], 0x5140);   // re(2(r+k)), re(2(r+7-k)), im, im
            const int tt = (tap[k] & 0xffff) | (tap[k] << 16);
            ar += dp2a_su<false>(tt, pr, -254 * tap[k]) >> 9;
            ai += dp2a_su<true>(tt, pr, -254 * tap[k]) >> 9;
        }
        y[r] = make_short2((short)ar, (short)ai);
    }
}

}  // namespace nb
