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
constexpr int P3_VIT = P3_LEN * 3;          // 13824
constexpr int PX1_BLOCK = 4608;             // PX1 soft bits per block (2 partitions per sideband)
constexpr int IV_N = 147456;                // span of interleaver IV (reference src/decode.c:350)
constexpr int PX_RING = 2 * IV_N;
constexpr int P3_SLOTS = 8;                 // P3 frames per stream and pass (one per two blocks)
constexpr int P3_DEC_STRIDE = 5120;         // decisions per frame: 5 fallback chunks of 1024 >= 4608 + 64
constexpr int ST_NONE = 0, ST_COARSE = 1, ST_FINE = 2;

// record types (include/nrsc5_b200.h)
constexpr uint32_t REC_FRAME = 1, REC_PIDS = 2, REC_SYNC = 3, REC_LOST_SYNC = 4, REC_MER = 5,
                   REC_BER = 6, REC_SOFT_PM = 8, REC_BLOCK = 9;

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
    int p1_errs;               // channel bit errors counted so far
    int p1_done;               // k_p1_fin CTAs finished
    int pids_pending;          // PIDS frames (of blocks pids_bc[]) waiting to be decoded into the log slots pids_rec[];
    int pids_bc[16];           // k_stream decodes them together, one warp each, before it exits
    unsigned pids_rec[16];
    // P3 (MP3/MP11 PX1 partitions): convolutional interleaver IV bookkeeping (reference src/decode.c:344-414)
    long long px_total;        // PX1 soft bits taken in since the interleaver (re)started
    int px_started;
    int p3_pending;            // P3 frames waiting for the decode kernels that follow k_stream
    long long p3_k0[8];        // interleaver position of each frame's first soft bit
    unsigned p3_rec[8];        // log offset of each frame's reserved FRAME record
    // the other extended-partition channels, decoded by kernel groups the host only launches once a stream has
    // asked for them (g_px_need): [0] = MP2's 2304-bit P3 frames (PX1 ring, one partition per sideband),
    // [1] = MP11's P4 frames (PX2 ring)
    long long px2_total;       // PX2 soft bits taken in since the interleaver (re)started
    int px2_started;
    int xq_pending[2];
    long long xq_k0[2][8];
    unsigned xq_rec[2][8];
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
    int px_enabled;            // PX_NEED_* bits: the extended-partition decode groups the host launches after k_stream
    int l2;                    // frames also go through L2 on the device (nrsc5b_enable_l2)
    int cluster;               // CTAs per stream in k_stream (thread-block cluster): 1, 2 or 4
};

// buffers of one extra extended-partition decode group (same roles as the p3_* arrays)
struct PxBufs {
    int8_t *vin;
    uint2 *dec;
    uint32_t *spec, *end;
    int *endstate;
    uint2 *fspec, *fend;
    int *fhstate, *ftbend;
    uint32_t *bits;
    int *flags;
};
constexpr int PX_NEED_SHORT = 1, PX_NEED_PX2 = 2, PX_NEED_P3 = 4;   // MP2 | MP11 (P4) | MP3 and MP11 (4608-bit P3)
constexpr int P3S_LEN = 2304, IV_NS = IV_N / 2;    // MP2: P3 frame bits, interleaver IV span (decode.c:346-350)

// Per-engine control words in device memory (one engine = one instance: engines on one device share nothing).
struct EngineCtl {
    unsigned long long progress;   // bumped by every stream that processed a block
    unsigned px_need;              // PX_NEED_* bits: a stream waits for a decode group the host has not enabled
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
    int8_t *px_ring;           // [S][2 * IV_N] PX1 soft bits in arrival order (the last two interleaver spans)
    const uint32_t *iv_delay;  // [IV_N] interleaver IV: output m comes from the input iv_delay[m] positions earlier
    int8_t *p3_vin;            // [S][8][13824] deinterleaved + depunctured P3 soft bits
    uint2 *p3_dec;             // [S][8][P3_DEC_STRIDE] survivor decisions
    uint32_t *p3_spec, *p3_end;     // [S][8][P3 chunks][32] fast Viterbi chunk boundary metrics
    int *p3_endstate;          // [S][8]
    uint2 *p3_fspec, *p3_fend; // [S][8][5][16] fallback Viterbi
    int *p3_fhstate, *p3_ftbend;    // [S][8][5]
    uint32_t *p3_bits;         // [S][8][144] decoded (still scrambled) bits
    int *p3_flags;             // [S][8][4] ready, slow, retry, -
    int8_t *px2_ring;          // [S][2 * IV_N] PX2 soft bits (MP11)
    const uint32_t *iv_delay_s;     // [IV_NS] interleaver IV of MP2 (J=2, M=4)
    PxBufs xb[2];              // extra groups (null until the host enables them)
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

// cu8 byte of absolute input sample n (component c); before the stream start
// the decimator window holds zeros, i.e. byte 127 (reference src/firdecim_q15.c:33)
__device__ __forceinline__ int q15_of_u8(int v) { return (v - 127) * 64; }

// halfband decimator output y[d] for one stream (reference src/firdecim_q15.c:137-151,
// taps int16{-134,1078,-4417,19864}): exact integer arithmetic.
__device__ __forceinline__ short2 halfband_at(const uint8_t *iq, long long d)
{
    // y[d] = x[2d-7] + sum_k ((x[2d-14+2k] + x[2d-2k]) * tap_k) >> 15
    const int tap[4] = { -134, 1078, -4417, 19864 };
    long long n0 = 2 * d - 14;
    int accr = 0, acci = 0;
    if (n0 >= 0) {
        // input samples may land (asynchronous copies) while a kernel runs: read them through L2 only
        const uint8_t *b = iq + 2 * n0;
        auto ld = [&](int i) -> int { return q15_of_u8(__ldcg(b + i)); };
#pragma unroll
        for (int k = 0; k < 4; k++) {
            int ar = ld(4 * k) + ld(2 * (14 - 2 * k));
            int ai = ld(4 * k + 1) + ld(2 * (14 - 2 * k) + 1);
            accr = (short)(accr + ((ar * tap[k]) >> 15));
            acci = (short)(acci + ((ai * tap[k]) >> 15));
        }
        accr = (short)(accr + ld(14));
        acci = (short)(acci + ld(15));
    } else {
        auto rd = [&](long long n, int c) -> int { return n < 0 ? 0 : q15_of_u8(__ldcg(iq + 2 * n + c)); };
#pragma unroll
        for (int k = 0; k < 4; k++) {
            int ar = rd(n0 + 2 * k, 0) + rd(n0 + 14 - 2 * k, 0);
            int ai = rd(n0 + 2 * k, 1) + rd(n0 + 14 - 2 * k, 1);
            accr = (short)(accr + ((ar * tap[k]) >> 15));
            acci = (short)(acci + ((ai * tap[k]) >> 15));
        }
        accr = (short)(accr + rd(n0 + 7, 0));
        acci = (short)(acci + rd(n0 + 7, 1));
    }
    return make_short2((short)accr, (short)acci);
}

}  // namespace nb
