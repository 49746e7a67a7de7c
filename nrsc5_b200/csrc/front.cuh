// The stream-resident front end: ONE persistent CTA per stream (k_stream) runs, block after block,
//
//   pids   the previous block's PIDS frame                                            (decode.c:463-471)
//   prep   window check, coarse acquisition when not in FINE sync, feedback, NCO      (acquire.c:98-168)
//   demod  cu8 -> halfband -> NCO/window/fold -> 2048-pt FFT -> 534 bins, 32 symbols  (input.c:52-94,
//                                                   firdecim_q15.c:137-165, acquire.c:237-257, sync.c:779-790)
//   sync   Costas, COARSE->FINE vote / CFO search, equalise, feedback, MER, soft demap (sync.c:90-610)
//
// until the stream runs out of buffered samples, completes an L1 frame (the P1 decode kernels must run
// before the next block: their RS header check feeds back into the sync state, frame.c:538) or has done
// `max_blocks` blocks.  The block-to-block feedback (timing error, phase) never leaves the SM; streams
// share nothing, so there are no inter-CTA flags, fences or queues.  The 1024 threads form 8 teams of
// 128; a team demodulates one OFDM symbol at a time (4 passes per 32-symbol block).
//
// This translation unit is compiled with -fmad=false: float expressions keep the reference's
// evaluation order wherever a discrete decision depends on them.
#pragma once
#include "pids_crc.cuh"
#include "common.cuh"
#include "fft.cuh"
#include "viterbi_pack.cuh"

namespace nb {

constexpr int FRONT_THREADS = 1024;
constexpr int TEAMS = FRONT_THREADS / 128;         // symbol teams of 128 threads
constexpr int MAXREF = 15;                         // reference subcarriers per sideband (14 partitions + 1)
constexpr int IN_BYTES = 4 * NSYM + 28 + 16 + 16;  // staged cu8 bytes per symbol (+ alignment slack) = 8700
constexpr int IN_STRIDE = 8704;
constexpr int ACQ_TILE = 4096;                     // decimated samples per acquisition tile

__device__ int g_dbg;                              // experiment switches (nrsc5b_debug_set), 0 in production

__constant__ int c_compat_mode[64];
__constant__ unsigned c_pn80[3];                   // first 80 bits of the descrambler sequence (bit i of word i/32)
__constant__ short c_bp_tap[32];                   // coarse band-pass taps, tap[i] pairs w[i] and w[32-i]

// complex helpers with the reference's (gcc, no FMA) evaluation order
__device__ __forceinline__ float2 cmulf(float2 a, float2 b)
{
    return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ float2 cexp_j(float a)       // cexpf(I*a)
{
    float s, c;
    sincosf(a, &s, &c);
    return make_float2(c, s);
}

__device__ __forceinline__ int partitions_per_band(int psmi)
{
    switch (c_compat_mode[psmi & 63]) {
    case 2: return 11;
    case 3: return 12;
    case 5: case 6: case 11: return 14;
    default: return 10;
    }
}

// input_set_sync_state (reference src/input.c:172-188)
__device__ void set_state(const DevPtrs &p, const EngineDims &d, int s, int ns)
{
    StreamState &st = p.st[s];
    if (st.state == ns) return;
    if (st.state == ST_FINE) log_reserve(p, d, s, REC_LOST_SYNC, 0);
    if (ns == ST_FINE) {
        float fo = (float)(((double)st.prev_angle - 2 * M_PI * st.cfo) * 744187.5 / (2 * M_PI * NFFT));
        uint8_t *w = log_reserve(p, d, s, REC_SYNC, 8);
        if (w) {
            reinterpret_cast<float *>(w)[0] = fo;
            reinterpret_cast<int *>(w)[1] = st.psmi;
        }
    }
    st.state = ns;
}

// ---------------------------------------------------------------------------
// shared memory: one buffer, reinterpreted per task phase
// ---------------------------------------------------------------------------
constexpr int DEMOD_RUN = 17;                      // decimated samples per thread and symbol: consecutive, a stride coprime with the 32 banks
constexpr int TEAM_SMEM = IN_STRIDE + NSYM * (int)sizeof(short2);   // 17 344 bytes
struct DemodSmem {
    // per team: the symbol's staged cu8 (IN_STRIDE bytes), then its NSYM decimated samples (short2); the FFT exchange
    // buffer aliases the start of both
    float2 buf[TEAMS][TEAM_SMEM / sizeof(float2)];
};
static_assert(FFT_SMEM_ELEMS * sizeof(float2) <= TEAM_SMEM && TEAM_SMEM % 16 == 0, "a team's FFT buffer");
static_assert(DEMOD_RUN * FFT_THREADS >= NSYM && DEMOD_RUN % 2 == 1, "a symbol's runs");
struct PrepSmem {
    uint32_t words[ACQ_TILE + 40];                 // cu8 of one acquisition tile (+ 7 words of halfband, 31 of FIR history)
    short2 ytile[ACQ_TILE + 32];                   // its halfband outputs, preceded by the 31 the band-pass looks back on
    float2 sums[NSYM];
    float red_mag[FRONT_THREADS];
    int red_idx[FRONT_THREADS];
    float2 red_v[FRONT_THREADS];
};
// coarse acquisition by one CTA (front_prep_single): the window in tiles of one symbol period, so that term j of every
// offset's cyclic-prefix correlation needs tiles j and j+1 only - the band-passed window never leaves the SM
constexpr int ACQ1_RUN = 3;                        // odd: conflict-free; 731 runs cover NSYM + 31 outputs
constexpr int ACQ1_WORDS = (NSYM + 38 + 3 + 3) / 4 * 4;   // a tile's cu8 words from a 16-byte boundary (word phase <= 3)
static_assert(ACQ1_RUN * FRONT_THREADS >= NSYM + 31 && ACQ1_RUN % 2 == 1, "a tile's runs");
struct Acq1Smem {
    uint32_t words[2][ACQ1_WORDS];                 // cu8 of tiles j and j+1 (asynchronous copies, double-buffered)
    short2 ytile[NSYM + 32];                       // tile j's halfband outputs, preceded by the 31 the band-pass looks back on
    float2 ring[2][NSYM];                          // band-passed tiles j-1 and j: what the correlation reads
    float2 sums[NSYM];
    float2 shape[NCP];                             // (shape[j], shape[j + NFFT]) for the pulse-shaped sliding sum
    float red_mag[FRONT_THREADS];
    int red_idx[FRONT_THREADS];
    float2 red_v[FRONT_THREADS];
};
struct PidsSmem {
    int8_t vit[PIDS_LEN * 3];
    uint2 dec[PIDS_LEN + 64];
};
constexpr int ZS = 32;                              // row stride of the per-reference arrays (>= 2 * MAXREF)
static_assert(2 * MAXREF <= 32, "a reference slot fits the 5 bits of FrontSmem::ref_plan");
constexpr int EQ_LD = BLK + 1;                      // padded row of the equalisation buffer (bank-conflict free)
constexpr int EQ_MAXPART = 12;                      // partitions per sideband the equaliser stages in shared memory (MP1..MP3);
                                                    // the two more of MP5/MP6/MP11 are equalised in place in global memory
constexpr int EQ_ROWS = 2 * EQ_MAXPART * (PW - 1);  // data carriers of both sidebands
struct SyncSmem {
    float phs[BLK][ZS];                            // the Costas loop's phase, laid out like FrontSmem::zref
    float2 eph[2 * MAXREF][BLK];                   // exp(j*phs)
    float smag[2 * MAXREF];
    float cfq[2 * MAXREF];                         // Costas frequency of every reference after the block
    union {
        float2 eq[EQ_ROWS][EQ_LD];                 // data carriers [sideband*rows + partition*18 + k-1][symbol]
        struct {                                   // CFO search (never at the same time as the equaliser)
            int offs[76][22];                      // block offset found by every (trial, carrier), -1 = none
            int verdict[76];                       // winning block offset of a trial, -1 = trial failed
            int winner;
        } srch;
    };
    float wred[FRONT_THREADS / 32][2];             // per-warp error sums (lower, upper sideband)
    float fb_w[2][MAXREF], fb_xy[2][MAXREF + 1];   // feedback terms (phase differences, bin * frequency)
    float4 rowc[EQ_ROWS];                          // per carrier row: k*|upper ref|, (19-k)*|lower ref|, slots
    int ref_ok[2 * MAXREF], ref_bc[2 * MAXREF], ref_psmi[2 * MAXREF];
    bool px_on[2];                                 // the block feeds PX1 / PX2, from interleaver position px_T
    long long px_T[2];
    uint8_t *soft_w;                               // REC_SOFT_PM payload
    int do_search;
};
// A block's set-up: what its demod reads, and what a FINE block's prep commits to the stream's state.  k_stream<false>
// computes it for the next block in front_sync (warp 1, beside the demap) and uses it if that block runs in FINE sync.
struct BlockSet {
    int samperr;                                   // window offset
    int ok;                                        // set up by the last block's sync, not yet committed or discarded
    float prev_angle, angle;                       // the NCO angle before and after the CFO correction
    float theta;
    float2 phase0, phase;                          // NCO phase at the block's first sample and after its 32 symbols
};
struct FrontSmem {
    float2 tw[FFT_TW];                             // FFT twiddle tables (fft.cuh)
    float2 nco[NSYM];                              // window[j] * exp(j*theta*j) of the current block
    float2 symphase[BLK];                          // phase0 * exp(j*theta*NSYM*sym) of the current block's symbols
    BlockSet blk;                                  // (k_stream<false>) the current block's set-up, or the next one's
    // reference carriers [symbol][reference slot], stored by the demodulating teams beside the kept bins (outside the
    // union: the sync phase reads them without a round trip through global memory), then rotated by the Costas loops.
    // The threads of a warp each walk one reference, symbol by symbol, so the slot index is the contiguous one.
    float2 zref[BLK][ZS];
    uint8_t ref_plan[128];                         // per demod thread: which of its kept-bin stores is a reference carrier, and its slot
    union {
        DemodSmem demod;
        PrepSmem prep;
        Acq1Smem acq1;
        SyncSmem sync;
        PidsSmem pidsq[16];
    } u;
};

// ---------------------------------------------------------------------------
// pids: interleaver II + depuncture (decode.c:324-342), K=7 Viterbi, descramble (decode.c:279-294)
// ---------------------------------------------------------------------------
// One warp decodes pending PIDS frame `e` of the stream into its reserved log slot.
__device__ void pids_decode_warp(const DevPtrs &p, const EngineDims &d, int s, int e, PidsSmem &sm, int lane)
{
    const StreamState &st = p.st[s];
    const int bc = st.pids_bc[e];
    const int8_t *pmall = p.pm + (size_t)s * 16 * PM_BLOCK;
    const int8_t PMV[20] = { 10, 2, 18, 6, 14, 8, 16, 0, 12, 4, 11, 3, 19, 7, 15, 9, 17, 1, 13, 5 };
    for (int o = lane; o < PIDS_LEN * 3; o += 32) {
        int8_t v = 0;
        if (o % 6 != 5) {
            unsigned i = (unsigned)bc * 200 + (unsigned)(o - o / 6);
            unsigned part = (unsigned)PMV[i % 20];
            unsigned block = i / 200;
            unsigned k = (i / 20) % 10 + P1_ENC / 320;
            unsigned row = (k * 11) % 32, col = (k * 11 + k / 288) % 36;
            v = pmall[(block * 32 + row) * 720 + part * 36 + col];
        }
        sm.vit[o] = v;
    }
    __syncwarp();
    // both half-warps decode the same frame (the packed kernel works on two chunks per warp); FM PIDS
    // soft bits are punctured 1,1,1,1,1,0, so the int16 metrics cannot saturate
    const int l = lane & 15;
    VitHalf<false> vh;
    vh.init(l);
    vitc_run<false>(vh, sm.vit, PIDS_LEN, PIDS_LEN + 64, 0, PIDS_LEN + 64, 0, sm.dec, lane < 16, l);
    __syncwarp();
    // first maximum in state order; lane l holds states 2l, 2l+32 (E) and 2l+1, 2l+33 (O)
    int v = (short)(vh.E & 0xffff), state = 2 * l;
    const int w1 = (short)(vh.O & 0xffff);
    if (w1 > v) { v = w1; state = 2 * l + 1; }
    int v2 = (short)(vh.E >> 16), idx2 = 2 * l + 32;
    const int w3 = (short)(vh.O >> 16);
    if (w3 > v2) { v2 = w3; idx2 = 2 * l + 33; }
    if (v2 > v) { v = v2; state = idx2; }
#pragma unroll
    for (int o = 8; o; o >>= 1) {
        const int ov = __shfl_xor_sync(0xffffffffu, v, o, 16), oi = __shfl_xor_sync(0xffffffffu, state, o, 16);
        if (ov > v || (ov == v && oi < state)) { v = ov; state = oi; }
    }
    if (lane == 0) {
        uint8_t pk[10];
        for (int i = 0; i < 10; i++) pk[i] = 0;
        for (int q = PIDS_LEN + 63; q >= 0; q--) {
            if (q >= 32 && q < 32 + PIDS_LEN) {
                const int i = q - 32;
                const int bit = ((state >> 5) & 1) ^ (int)((c_pn80[i >> 5] >> (i & 31)) & 1u);
                pk[i >> 3] |= (uint8_t)(bit << (7 - (i & 7)));
            }
            state = vitc_prev_head(state, sm.dec, q);
        }
        if (st.pids_rec[e] != 0xffffffffu) {
            uint8_t *w = p.log + (size_t)s * d.log_cap + st.pids_rec[e];
            for (int i = 0; i < 10; i++) w[i] = pk[i];
            w[10] = (uint8_t)pids_crc12_ok(pk);          // pids.c:1042: what pids_frame_push will find
        }
    }
}

// decode every pending PIDS frame of the stream (at most 16), one warp each
__device__ void front_pids_flush(const DevPtrs &p, const EngineDims &d, int s, PidsSmem *sm, int t)
{
    StreamState &st = p.st[s];
    const int n = st.pids_pending, warp = t >> 5;
    if (warp < n) pids_decode_warp(p, d, s, warp, sm[warp], t & 31);
    __syncthreads();
    if (t == 0) st.pids_pending = 0;
}

// ---------------------------------------------------------------------------
// prep (reference src/acquire.c:98-168, src/sync.c:769-777, src/firdecim_q15.c:95-109,154-158)
// ---------------------------------------------------------------------------
// The decimated input of one acquisition tile: ytile[k] = y[i0 - 31 + k], k < L + 31, from the tile's words
// (word v holds input samples 2 (start + i0 - 38 + v) and the next).  The window's first tile starts with the previous
// window's last 31 outputs (bp_hist).  cu8: halfband_run over runs of RUN outputs per thread; the last run is moved
// back to end at the tile's end and overlaps its neighbour's, writing the same values.
constexpr int ACQ_RUN = 5;                         // odd: conflict-free; 1024 runs cover ACQ_TILE + 31 outputs
static_assert(ACQ_RUN * FRONT_THREADS >= ACQ_TILE + 31, "a tile's runs");
template <int RUN>
__device__ __forceinline__ void acq_tile_input(const EngineDims &d, const uint32_t *words, short2 *ytile, const StreamState &st,
                                               int i0, int L, int t)
{
    const int kb = i0 == 0 ? 31 : 0;
    if (t < kb) ytile[t] = make_short2(st.bp_hist[t][0], st.bp_hist[t][1]);
    const int n = L + 31 - kb;
    if (d.cs16) {                                  // already decimated: the sample itself
        for (int k = kb + t; k < L + 31; k += FRONT_THREADS) {
            const uint32_t w = words[k + 7];
            ytile[k] = make_short2((short)(w & 0xffff), (short)(w >> 16));
        }
    } else if (RUN * t < n) {
        const int k = kb + min(RUN * t, n - RUN);
        halfband_run<RUN>(words + k, ytile + k);
    }
}

// 32-tap symmetric Q15 band-pass (acquire.c:120-127, firdecim_q15.c:95-109) of output j of a tile: yy[k] = y[j - 31 + k]
__device__ __forceinline__ float2 acq_bandpass(const short2 *yy)
{
    short accr = 0, acci = 0;
#pragma unroll 5
    for (int k = 1; k < 16; k++) {
        const short2 a = yy[k], b = yy[32 - k];
        accr = (short)(accr + ((((int)a.x + (int)b.x) * c_bp_tap[k]) >> 15));
        acci = (short)(acci + ((((int)a.y + (int)b.y) * c_bp_tap[k]) >> 15));
    }
    const short2 c = yy[16];
    accr = (short)(accr + (((int)c.x * c_bp_tap[16]) >> 15));
    acci = (short)(acci + (((int)c.y * c_bp_tap[16]) >> 15));
    return make_float2(__fdiv_rn((float)accr, 32767.0f), __fdiv_rn((float)acci, -32767.0f));
}

// NCO of a block in closed form, with the pulse shape folded in (acquire.c:243-252): nco[j] = shape[j] * exp(j*theta*j)
__device__ __forceinline__ void fill_nco(const DevPtrs &p, float2 *nco, float theta, int t, int nthreads = FRONT_THREADS)
{
    for (int j = t; j < NSYM; j += nthreads) {
        float2 e = cexp_j(theta * (float)j);
        if (j < NCP || j >= NFFT) {
            const float w = __ldg(&p.shape[j]);
            e = make_float2(e.x * w, e.y * w);
        }
        nco[j] = e;
    }
}

// phase of symbol `sym`'s kept bins (closed form of the NCO phase at the symbol's start): phase0 * exp(j*theta*NSYM*sym)
__device__ __forceinline__ void fill_symphase(float2 *symphase, float theta, float2 phase0, int sym)
{
    double sn, cs;
    sincos((double)theta * (double)(NSYM * sym), &sn, &cs);
    symphase[sym] = cmul(phase0, make_float2((float)cs, (float)sn));
}

// A block's NCO from its window offset b.samperr and angle b.prev_angle (before the CFO correction) and the stream's
// phase after the previous block (acquire.c:243-252)
__device__ __forceinline__ void block_setup(BlockSet &b, const StreamState &st)
{
    const int adj = NSYM / 2 - b.samperr;
    float angle = b.prev_angle;
    angle = (float)((double)angle - 2 * M_PI * st.cfo);
    const float pre = (float)(-adj) * angle / (float)NFFT;
    const float2 ph = cmulf(st.phase, cexp_j(pre));
    const float theta = angle / (float)NFFT;
    // NCO phase after the 32 symbols of this block (acquire.c:250-252, closed form)
    double sn, cs;
    sincos((double)theta * (double)(NSYM * BLK), &sn, &cs);
    const float2 pe = cmulf(ph, make_float2((float)cs, (float)sn));
    const float nrm = sqrtf(pe.x * pe.x + pe.y * pe.y);
    b.angle = angle;
    b.theta = theta;
    b.phase0 = ph;
    b.phase = make_float2(pe.x / nrm, pe.y / nrm);
}

// sync_adjust (sync.c:769-777): the Costas phases of the kept bins follow the window's move by adj samples
__device__ __forceinline__ void sync_adjust(const DevPtrs &p, int s, int adj, int t)
{
    if (adj == 0) return;
    float *cp = p.cphase + (size_t)s * NFFT;
    for (int i = t; i < SIDE; i += FRONT_THREADS) {
        const int bl = LB0 + i, bu = UB1 - i;
        cp[bl] = (float)((double)cp[bl] - (double)(adj * (bl - NFFT / 2) * 2) * M_PI / NFFT);
        cp[bu] = (float)((double)cp[bu] - (double)(adj * (bu - NFFT / 2) * 2) * M_PI / NFFT);
    }
}

// the block's parameters into the stream's state, and its REC_BLOCK record (thread 0)
__device__ __forceinline__ void block_commit(const DevPtrs &p, const EngineDims &d, int s, const BlockSet &b, int state_in)
{
    StreamState &st = p.st[s];
    st.phase0 = b.phase0;
    st.theta = b.theta;
    st.blk_samperr = b.samperr;
    st.blk_state_in = state_in;
    st.phase = b.phase;
    uint8_t *w = log_reserve(p, d, s, REC_BLOCK, 32);
    if (w) {
        int *wi = reinterpret_cast<int *>(w);
        float *wf = reinterpret_cast<float *>(w);
        wi[0] = state_in; wi[1] = b.samperr; wf[2] = b.angle; wf[3] = b.phase0.x; wf[4] = b.phase0.y; wi[5] = st.cfo;
        wi[6] = (int)(unsigned)(st.start & 0xffffffffLL);
        wi[7] = (int)(st.start >> 32);
    }
}

// Returns false (uniformly) when the stream has no complete 33-symbol window buffered.
// prep, first part (the stream's owner CTA): does the stream have a whole window, and in which state does the block start?
// Returns 0 = nothing to do, 1 = a block in fine sync, 2 = a block that starts with coarse acquisition.
__device__ int front_prep_begin(const DevPtrs &p, const EngineDims &d, int s, int t)
{
    StreamState &st = p.st[s];
    __shared__ int sh_active;
    if (t == 0) {
        if (st.force_state >= 0) {
            set_state(p, d, s, st.force_state);
            st.force_state = -1;
        }
        // in_avail is advanced by asynchronous copies while this kernel runs
        const long long avail = *reinterpret_cast<volatile long long *>(&st.in_avail);
        int act = avail >= 2 * (st.start + NACQ);
        if (act && st.state == ST_FINE) {
            // P3 / P4 frames (MP2, MP3, MP11) are decoded by kernel groups the host adds to the pass only when a
            // stream asks: wait at the block boundary until it has (nrsc5b_process looks at the flag).  Streams
            // in MP1 / MP5 / MP6 never pay for those launches.
            const int need = px_need_of(c_compat_mode[st.psmi & 63]);
            if (need & ~d.px_enabled) {
                atomicOr(&p.ctl->px_need, (unsigned)need);
                act = 0;
            }
        }
        st.active = act;
        sh_active = act ? (st.state == ST_FINE ? 1 : 2) : 0;
        if (act) atomicAdd(&p.ctl->progress, 1ull);
    }
    __syncthreads();
    const int mode = sh_active;
    __syncthreads();
    return mode;
}

// Coarse acquisition, the part that is spread over the stream's CTAs (one, or the `nranks` of its cluster):
// the 71280-sample window in tiles - cu8 words -> shared memory (coalesced), halfband /2 (input.c:52-94), 32-tap
// symmetric Q15 band-pass (acquire.c:120-127, firdecim_q15.c:95-109) -> float window in `tb`; CTA `rank` takes every
// nranks-th tile.  (The window's last 31 band-pass inputs become the next window's history: parked in bp_hist_next,
// because the CTA with the first tile may not have read the old history yet.)
__device__ void front_acq_tiles(const DevPtrs &p, const EngineDims &d, int s, PrepSmem &sm, int t, int rank, int nranks)
{
    StreamState &st = p.st[s];
    const uint8_t *iq = p.iq + (size_t)s * d.in_stride;
    float2 *tb = p.tbuf + (size_t)s * NACQ;
    const long long start = nranks > 1 ? __ldcg(&st.start) : st.start;
    const uint32_t *iqw = reinterpret_cast<const uint32_t *>(iq);
    for (int i0 = rank * ACQ_TILE; i0 < NACQ; i0 += nranks * ACQ_TILE) {
        const int L = min(ACQ_TILE, NACQ - i0);
        const long long w0 = start + i0 - 38;                 // word of halfband output i0-31's first input
        for (int v = t; v < L + 38; v += FRONT_THREADS) {
            const long long a = w0 + v;
            // before the stream starts the decimator sees zeros = byte 127; through L2 only (asynchronous pushes)
            sm.words[v] = a >= 0 ? __ldcg(iqw + a) : (d.cs16 ? 0u : 0x7f7f7f7fu);
        }
        __syncthreads();
        acq_tile_input<ACQ_RUN>(d, sm.words, sm.ytile, st, i0, L, t);
        __syncthreads();
        for (int j = t; j < L; j += FRONT_THREADS) tb[i0 + j] = acq_bandpass(sm.ytile + j);
        if (i0 + L == NACQ && t < 31) {                       // the window's last 31 outputs: the next window's history
            const short2 v = sm.ytile[L + t];
            st.bp_hist_next[t][0] = v.x;
            st.bp_hist_next[t][1] = v.y;
        }
        __syncthreads();
    }
}

// cyclic-prefix correlation per sample offset (acquire.c:129-134): CTA `rank` takes its share of the 2160 offsets (each
// offset's sum is one thread's, in the reference's order) and leaves them in global memory for the owner
__device__ void front_acq_corr(const DevPtrs &p, int s, int t, int rank, int nranks)
{
    const float2 *tb = p.tbuf + (size_t)s * NACQ;
    float2 *sums = p.acq_sums + (size_t)s * NSYM;
    const int lo = rank * NSYM / nranks, hi = (rank + 1) * NSYM / nranks;
    for (int i = lo + t; i < hi; i += FRONT_THREADS) {
        float2 acc = make_float2(0.f, 0.f);
        for (int j = 0; j < BLK; j++) {
            const float2 a = __ldcg(&tb[i + j * NSYM]), b = __ldcg(&tb[i + j * NSYM + NFFT]);   // (written by other SMs too)
            float2 pr = cmulf(a, make_float2(b.x, -b.y));
            acc.x += pr.x;
            acc.y += pr.y;
        }
        sums[i] = acc;
    }
}

// prep, last part (owner CTA): timing and angle of the block - from the correlation sums when acquiring (mode 2) -,
// sync_adjust, the block's NCO table and REC_BLOCK record
__device__ void front_prep_finish(const DevPtrs &p, const EngineDims &d, int s, PrepSmem &sm, float2 *nco, float2 *symphase,
                                  BlockSet &b, int t, int mode)
{
    StreamState &st = p.st[s];
    const int state_in = st.state;
    if (mode == 2) {
        const float2 *gs = p.acq_sums + (size_t)s * NSYM;
        for (int i = t; i < NSYM; i += FRONT_THREADS) sm.sums[i] = __ldcg(&gs[i]);
        if (t < 31) {
            st.bp_hist[t][0] = __ldcg(&st.bp_hist_next[t][0]);
            st.bp_hist[t][1] = __ldcg(&st.bp_hist_next[t][1]);
        }
        __syncthreads();
        // pulse-shaped sliding sum and arg-max (acquire.c:136-151)
        float best = -1.0f;
        int besti = 0;
        float2 bestv = make_float2(0.f, 0.f);
        for (int i = t; i < NSYM; i += FRONT_THREADS) {
            float2 v = make_float2(0.f, 0.f);
            for (int j = 0; j < NCP; j++) {
                int q = i + j;
                if (q >= NSYM) q -= NSYM;
                const float2 sv = sm.sums[q];
                const float a = __ldg(&p.shape[j]), b = __ldg(&p.shape[j + NFFT]);
                v.x += (sv.x * a) * b;
                v.y += (sv.y * a) * b;
            }
            const float mag = v.x * v.x + v.y * v.y;
            if (mag > best) { best = mag; besti = i; bestv = v; }
        }
        sm.red_mag[t] = best; sm.red_idx[t] = besti; sm.red_v[t] = bestv;
        __syncthreads();
        for (int o = FRONT_THREADS / 2; o; o >>= 1) {
            if (t < o) {
                const float m2 = sm.red_mag[t + o];
                const int i2 = sm.red_idx[t + o];
                if (m2 > sm.red_mag[t] || (m2 == sm.red_mag[t] && i2 < sm.red_idx[t])) {
                    sm.red_mag[t] = m2; sm.red_idx[t] = i2; sm.red_v[t] = sm.red_v[t + o];
                }
            }
            __syncthreads();
        }
        if (t == 0) {
            const float2 w = cmulf(sm.red_v[0], cexp_j(-st.prev_angle));
            const float angle_diff = atan2f(w.y, w.x);
            const float factor = (st.prev_angle != 0.0f) ? 0.25f : 1.0f;
            const float angle = st.prev_angle + (angle_diff * factor);
            st.prev_angle = angle;
            b.prev_angle = angle;
            b.samperr = (sm.red_idx[0] + NSYM - 15) % NSYM;
            if (st.state == ST_NONE) st.state = ST_COARSE;
        }
    } else if (t == 0) {
        b.samperr = NSYM / 2 + st.samperr;
        st.samperr = 0;
        const float angle = st.prev_angle + (-st.angle);
        st.angle = 0;
        st.prev_angle = angle;
        b.prev_angle = angle;
    }
    __syncthreads();
    sync_adjust(p, s, NSYM / 2 - b.samperr, t);
    if (t == 0) {
        block_setup(b, st);
        block_commit(p, d, s, b, state_in);
    }
    __syncthreads();
    // NCO of this block in closed form, with the pulse shape folded in (acquire.c:243-252):
    // nco[j] = shape[j] * exp(j*theta*j); the per-symbol phase is applied to the kept bins
    fill_nco(p, nco, b.theta, t);
    if (t >= FRONT_THREADS - BLK) fill_symphase(symphase, b.theta, b.phase0, t - (FRONT_THREADS - BLK));
    __syncthreads();
}

// prep of a block by ONE CTA (k_stream<false>, a stream per CTA): everything front_prep_begin / front_acq_tiles /
// front_acq_corr / front_prep_finish do, in one piece - kept as one function because the 128-stream kernel is at its
// 64-register ceiling and the split version costs it spills.
// A block in FINE sync whose set-up the previous block's front_sync computed (b.ok) only commits it: the state that
// set-up was computed from has not changed since (in FINE sync only this prep and the sync's feedback write samperr,
// angle, prev_angle, cfo and phase).  Its NCO table and symbol phases are filled by threads 1..1023 while thread 0
// decides whether the block runs; a block that takes the other path fills them again below.
__device__ bool front_prep_single(const DevPtrs &p, const EngineDims &d, int s, Acq1Smem &sm, float2 *nco, float2 *symphase,
                                  BlockSet &b, int t)
{
    StreamState &st = p.st[s];
    __shared__ int sh_active;
    if (t == 0) {
        // the decision's loads first, all in flight together (the other threads wait for it); in_avail is advanced by
        // asynchronous copies while this kernel runs
        const int fs = st.force_state;
        const long long avail = *reinterpret_cast<volatile long long *>(&st.in_avail);
        const long long start = st.start;
        const int psmi = st.psmi;
        int state = st.state;
        if (fs >= 0) {
            set_state(p, d, s, fs);
            st.force_state = -1;
            state = fs;
        }
        int act = avail >= 2 * (start + NACQ);
        if (act && state == ST_FINE) {
            // P3 / P4 frames (MP2, MP3, MP11) are decoded by kernel groups the host adds to the pass only when a
            // stream asks: wait at the block boundary until it has (nrsc5b_process looks at the flag).  Streams
            // in MP1 / MP5 / MP6 never pay for those launches.
            const int need = px_need_of(c_compat_mode[psmi & 63]);
            if (need & ~d.px_enabled) {
                atomicOr(&p.ctl->px_need, (unsigned)need);
                act = 0;
            }
        }
        st.active = act;
        sh_active = act ? (state == ST_FINE && b.ok ? 2 : 1) : 0;
        b.ok = 0;
        if (act) atomicAdd(&p.ctl->progress, 1ull);
    } else {
        fill_nco(p, nco, b.theta, t - 1, FRONT_THREADS - 1);
        if (t >= FRONT_THREADS - BLK) fill_symphase(symphase, b.theta, b.phase0, t - (FRONT_THREADS - BLK));
    }
    __syncthreads();
    if (!sh_active) return false;
    if (sh_active == 2) {
        sync_adjust(p, s, NSYM / 2 - b.samperr, t);
        if (t == 0) {
            st.samperr = 0;
            st.angle = 0;
            st.prev_angle = b.prev_angle;
            block_commit(p, d, s, b, ST_FINE);
        }
        return true;                                   // (k_stream reads the block's parameters from b)
    }

    const uint8_t *iq = p.iq + (size_t)s * d.in_stride;
    const int state_in = st.state;
    if (state_in != ST_FINE) {
        const long long start = st.start;
        // the 71280-sample window in 33 tiles of one symbol period: cu8 words -> shared memory (asynchronous copies,
        // tile j+1's in flight while tile j is filtered), halfband /2 (input.c:52-94), band-pass -> float tile in the
        // ring.  Once tile j+1 is in the ring, term j of every offset's cyclic-prefix correlation (acquire.c:129-134)
        // is added: y[j*NSYM + i] and y[j*NSYM + i + NFFT] lie in tiles j and j+1.  The thread of offset i adds its
        // terms in j order, so every sum has the reference's order.
        constexpr int NT = BLK + 1;
        static_assert(NACQ == NT * NSYM, "the window is whole tiles");
        const int woff = (int)((start - 38) & 3);                  // the same for every tile: NSYM is a multiple of 4
        static_assert(NSYM % 4 == 0, "tiles start at the same word phase");
        const int nvec = (woff + NSYM + 38 + 3) / 4;               // the 16-byte pieces that hold a needed word
        auto fetch = [&](int T) {                                  // tile T's words, from the 16-byte boundary below
            const long long w0 = start + (long long)T * NSYM - 38; // word of halfband output T*NSYM-31's first input
            const long long w0a = w0 & ~3LL;
            uint4 *dst = reinterpret_cast<uint4 *>(sm.words[T & 1]);
            for (int v = t; v < nvec; v += FRONT_THREADS) {
                const long long a = w0a + 4 * v;
                if (a >= 0) {                                      // through L2 only: the input is advanced by asynchronous pushes
#if defined(NB_EMU)
                    dst[v] = *reinterpret_cast<const uint4 *>(iq + 4 * a);
#else
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst + v)), "l"(iq + 4 * a) : "memory");
#endif
                } else {                                           // before the stream starts the decimator sees zeros = byte 127
                    const uint32_t z = d.cs16 ? 0u : 0x7f7f7f7fu;
                    dst[v] = make_uint4(z, z, z, z);
                }
            }
#if !defined(NB_EMU)
            asm volatile("cp.async.commit_group;" ::: "memory");
#endif
        };
        for (int i = t; i < NSYM; i += FRONT_THREADS) sm.sums[i] = make_float2(0.f, 0.f);
        if (t < NCP) sm.shape[t] = make_float2(__ldg(&p.shape[t]), __ldg(&p.shape[t + NFFT]));
        fetch(0);
#pragma unroll 1
        for (int T = 0; T <= NT; T++) {                            // pass NT only adds the last term
            if (T + 1 < NT) fetch(T + 1);                          // (its buffer was last read before the previous barrier)
#if !defined(NB_EMU)
            if (T + 1 < NT) asm volatile("cp.async.wait_group 1;" ::: "memory");
            else asm volatile("cp.async.wait_group 0;" ::: "memory");
#endif
            __syncthreads();
            if (T < NT) acq_tile_input<ACQ1_RUN>(d, sm.words[T & 1] + woff, sm.ytile, st, T * NSYM, NSYM, t);
            if (T >= 2) {                                          // term j = T-2: tiles j and j+1, both in the ring
                const float2 *ya = sm.ring[T & 1], *yb = sm.ring[(T - 1) & 1];
                for (int i = t; i < NSYM; i += FRONT_THREADS) {
                    const float2 a = ya[i], b = i + NFFT < NSYM ? ya[i + NFFT] : yb[i + NFFT - NSYM];
                    const float2 pr = cmulf(a, make_float2(b.x, -b.y));
                    sm.sums[i].x += pr.x;
                    sm.sums[i].y += pr.y;
                }
            }
            __syncthreads();
            if (T < NT) {
                float2 *y = sm.ring[T & 1];
                for (int j = t; j < NSYM; j += FRONT_THREADS) y[j] = acq_bandpass(sm.ytile + j);
                if (T == NT - 1 && t < 31) {                       // keep the window's last 31 outputs as history
                    const short2 v = sm.ytile[NSYM + t];
                    st.bp_hist[t][0] = v.x;
                    st.bp_hist[t][1] = v.y;
                }
            }
        }
        __syncthreads();
        // pulse-shaped sliding sum and arg-max (acquire.c:136-151)
        float best = -1.0f;
        int besti = 0;
        float2 bestv = make_float2(0.f, 0.f);
        for (int i = t; i < NSYM; i += FRONT_THREADS) {
            float2 v = make_float2(0.f, 0.f);
            for (int j = 0; j < NCP; j++) {
                int q = i + j;
                if (q >= NSYM) q -= NSYM;
                const float2 sv = sm.sums[q];
                const float2 ab = sm.shape[j];
                v.x += (sv.x * ab.x) * ab.y;
                v.y += (sv.y * ab.x) * ab.y;
            }
            const float mag = v.x * v.x + v.y * v.y;
            if (mag > best) { best = mag; besti = i; bestv = v; }
        }
        sm.red_mag[t] = best; sm.red_idx[t] = besti; sm.red_v[t] = bestv;
        __syncthreads();
        for (int o = FRONT_THREADS / 2; o; o >>= 1) {
            if (t < o) {
                const float m2 = sm.red_mag[t + o];
                const int i2 = sm.red_idx[t + o];
                if (m2 > sm.red_mag[t] || (m2 == sm.red_mag[t] && i2 < sm.red_idx[t])) {
                    sm.red_mag[t] = m2; sm.red_idx[t] = i2; sm.red_v[t] = sm.red_v[t + o];
                }
            }
            __syncthreads();
        }
        if (t == 0) {
            const float2 w = cmulf(sm.red_v[0], cexp_j(-st.prev_angle));
            const float angle_diff = atan2f(w.y, w.x);
            const float factor = (st.prev_angle != 0.0f) ? 0.25f : 1.0f;
            const float angle = st.prev_angle + (angle_diff * factor);
            st.prev_angle = angle;
            b.prev_angle = angle;
            b.samperr = (sm.red_idx[0] + NSYM - 15) % NSYM;
            if (st.state == ST_NONE) st.state = ST_COARSE;
        }
    } else if (t == 0) {
        b.samperr = NSYM / 2 + st.samperr;
        st.samperr = 0;
        const float angle = st.prev_angle + (-st.angle);
        st.angle = 0;
        st.prev_angle = angle;
        b.prev_angle = angle;
    }
    __syncthreads();
    sync_adjust(p, s, NSYM / 2 - b.samperr, t);
    if (t == 0) {
        block_setup(b, st);
        block_commit(p, d, s, b, state_in);
    }
    __syncthreads();
    // NCO of this block in closed form, with the pulse shape folded in (acquire.c:243-252):
    // nco[j] = shape[j] * exp(j*theta*j); the per-symbol phase is applied to the kept bins
    fill_nco(p, nco, b.theta, t);
    if (t >= FRONT_THREADS - BLK) fill_symphase(symphase, b.theta, b.phase0, t - (FRONT_THREADS - BLK));
    __syncthreads();
    return true;
}

// ---------------------------------------------------------------------------
// demod: one OFDM symbol per 128-thread half of the CTA
// ---------------------------------------------------------------------------
__device__ __forceinline__ float2 sample_q15(short2 h)
{
    const float sc = 1.0f / 32767.0f;
    return make_float2((float)h.x * sc, (float)h.y * -sc);    // conj(x)/32767, acquire.c:160-161
}

__device__ void front_demod(const DevPtrs &p, const EngineDims &d, int s, int sym, DemodSmem &sm, const float2 *nco,
                            const float2 *symphase, const float2 *tw, float2 (*zref)[ZS], const uint8_t *ref_plan,
                            int half, int tl, long long start, int samperr)
{
    float2 *buf = sm.buf[half];
    uint8_t *in = reinterpret_cast<uint8_t *>(buf);
    const int bar = 1 + half;                            // named barrier of this 128-thread team
    const long long base = start + samperr + (long long)NSYM * sym;
    const long long b0 = 4 * base - 28;                  // first needed cu8 byte (may be < 0 at stream start)
    const long long b0a = b0 & ~15LL;
    const int off = (int)(b0 - b0a);
    const uint8_t *iq = p.iq + (size_t)s * d.in_stride;
    bar_sync(bar);                                       // the team has read the previous symbol's FFT buffer
    {
        // the symbol's cu8 bytes go to shared memory by asynchronous 16-byte copies (cp.async.cg: through L2 only - samples
        // may have landed after an earlier, partial read of the same line - and past the register file)
        // Vector v = tl + 128 i of the thread: four of them, and a fifth below nvec (542 or 543) - unrolled, with the
        // addresses at constant offsets.  Only the stream's first symbols (b0a < 0) test each vector for the history.
        const int nvec = (off + 4 * NSYM + 28 + 15) / 16;
        static_assert(4 * 128 < (4 * NSYM + 28 + 15) / 16 && (12 + 4 * NSYM + 28 + 15) / 16 <= 5 * 128, "a symbol's copies");
        uint4 *dst = reinterpret_cast<uint4 *>(in) + tl;
        const uint8_t *src = iq + b0a + 16 * tl;
        const bool head = b0a < 0;
#pragma unroll
        for (int i = 0; i < 5; i++) {
            if (i == 4 && tl + 4 * 128 >= nvec) break;
            if (!head || b0a + 16 * (tl + 128 * i) >= 0) {
#if defined(NB_EMU)
                dst[128 * i] = *reinterpret_cast<const uint4 *>(src + 2048 * i);
#else
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst + 128 * i)), "l"(src + 2048 * i) : "memory");
#endif
            } else {
                dst[128 * i] = make_uint4(0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu);   // before the stream's first sample
            }
        }
#if !defined(NB_EMU)
        asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
#endif
    }
    bar_sync(bar);

    // sw points at the 32-bit word holding input samples (2*base-14, 2*base-13): decimated sample j uses words j..j+7
    const uint32_t *sw = reinterpret_cast<const uint32_t *>(in + off);
    const short2 *y;
    if (d.cs16) {                                         // cs16 input: word j+7 is sample j of the symbol
        y = reinterpret_cast<const short2 *>(sw + 7);
    } else {
        // the halfband, DEMOD_RUN consecutive samples per thread into the team's sample array (the last run is moved
        // back to end at the symbol's last sample: it overlaps its neighbour's and writes the same values)
        short2 *yw = reinterpret_cast<short2 *>(in + IN_STRIDE);
        const int j0 = min(DEMOD_RUN * tl, NSYM - DEMOD_RUN);
        halfband_run<DEMOD_RUN>(sw + j0, yw + j0);
        y = yw;
        bar_sync(bar);
    }
    // rotate by the block's NCO table (window folded in); j = n1*128 + tl.  (Point 0 and its fold first: with all 16
    // points' loads in flight before the fold, the 64 registers do not suffice and the FFT spills.)
    float2 v[16];
    v[0] = cmul(sample_q15(y[tl]), nco[tl]);
    if (tl < NCP) {                                       // fold the windowed tail onto the head (acquire.c:247-248)
        const int j = NFFT + tl;
        v[0] = cadd(v[0], cmul(sample_q15(y[j]), nco[j]));
    }
#pragma unroll
    for (int n1 = 1; n1 < 16; n1++) {
        const int j = n1 * 128 + tl;
        v[n1] = cmul(sample_q15(y[j]), nco[j]);
    }
    bar_sync(bar);                                        // every thread is done with the staged input and the samples
    float2 out[2][8];
    fft2048_block<true>(v, out, buf, tw, tl, bar);
    const float2 sp = symphase[sym];

    // kept bins (sync.c:785-789, fftshift defines.h:123-138): with q = tl + 128 h and natural bin k = q + 256 k3,
    //   k3 = 5 (q >= 222) -> compact q - 222,  k3 = 6 (q <= 232) -> q + 34      (lower sideband, bins 478..744)
    //   k3 = 1 (q >= 24)  -> compact q + 243,  k3 = 2 (q <= 34)  -> q + 499     (upper sideband, bins 1304..1570)
    // The reference carriers also go to zref[sym].  A thread makes at most one such store: ref_plan[tl] holds its index
    // 4 h + k (the k-th store of round h) in bits 5-7 and its slot in bits 0-4, or 0xff for none (store 7 never
    // happens: q = tl + 128 > 34).  So each store costs one compare and a predicated shared store.  (A table rather
    // than arithmetic on q: per-thread constants would be hoisted out of the symbol loop and spilled.)
    float2 *dst = p.bins + ((size_t)s * BLK + sym) * NBINS;
    const unsigned plan = ref_plan[tl];
    float2 *zp = zref[sym] + (plan & 31u);
    const unsigned pk = plan >> 5;
    auto put = [&](int c, float2 v, unsigned k) {
        dst[c] = v;
        if (pk == k) *zp = v;
    };
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int q = tl + 128 * h;
        if (q >= 222) put(q - 222, cmul(out[h][5], sp), 4 * h);
        if (q <= 232) put(q + 34, cmul(out[h][6], sp), 4 * h + 1);
        if (q >= 24) put(q + 243, cmul(out[h][1], sp), 4 * h + 2);
        if (q <= 34) put(q + 499, cmul(out[h][2], sp), 4 * h + 3);
    }
}

// ---------------------------------------------------------------------------
// sync (reference src/sync.c)
// ---------------------------------------------------------------------------
__device__ __forceinline__ int ref_bin(int slot)                // slot < MAXREF: lower sideband, else upper
{
    return slot < MAXREF ? LB0 + PW * slot : UB1 - PW * (slot - MAXREF);
}

// The Costas loop below is 32 DEPENDENT steps per reference carrier on one warp - its cost is the latency of one
// step's chain phase -> exp(-j phase) -> rotate -> arg -> filter -> phase.  Two short-chain replacements for the
// library calls on that chain (selected by FAST): the rotation by the SFU's sin / cos (|phase| <= pi; absolute error
// 2^-21.4, the size of a float's last bit at 1.0), and the loop error - the argument of u^2, i.e. of a point in the
// right half plane while the loop tracks - by one reciprocal and a degree-8 polynomial in t^2 (fitted on [0, 1], max
// error 1.2e-7 rad).  Both errors are of the size by which CUDA's sincosf / atan2f differ from the reference's libm;
// the parity tests bound the consequence (soft bits within one step, PDUs exact).
__device__ __forceinline__ float atan2_short(float y, float x)
{
    const float ax = fabsf(x), ay = fabsf(y);
    const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
    const float t = mx > 0.f ? __fdividef(mn, mx) : 0.f;
    const float z = t * t;
    float p = 0.0028340641874819994f;
    p = __fmaf_rn(p, z, -0.016005029901862144f);
    p = __fmaf_rn(p, z, 0.042587608098983765f);
    p = __fmaf_rn(p, z, -0.07495445758104324f);
    p = __fmaf_rn(p, z, 0.10636754333972931f);
    p = __fmaf_rn(p, z, -0.14202570915222168f);
    p = __fmaf_rn(p, z, 0.19992484152317047f);
    p = __fmaf_rn(p, z, -0.3333306610584259f);
    p = __fmaf_rn(p, z, 1.0f);
    float r = p * t;
    if (ay > ax) r = 1.57079637f - r;
    if (x < 0.f) r = 3.14159274f - r;
    return copysignf(r, y);
}

// adjust_ref (sync.c:90-130) on one row of 32 symbols
__device__ __forceinline__ void costas_row(float2 *z, float *phs, int zs, float &cfreq, float &cphase, int cfo, float alpha, float beta, bool FAST)
{
    // sync pattern -1, 1, -1, -1, -1, 1, 1, 0, 1, -1, 0, 0, 0, -1, -1, 0, 0, 0, 0, 0, -1, 1, -1, 0 x8, -1 as bit masks
    const unsigned pat_pos = (1u << 1) | (1u << 5) | (1u << 6) | (1u << 8) | (1u << 21);
    const unsigned pat_neg = (1u << 0) | (1u << 2) | (1u << 3) | (1u << 4) | (1u << 9) | (1u << 13) | (1u << 14) | (1u << 20) |
                             (1u << 22) | (1u << 31);
    const float cfo_freq = (float)(2 * M_PI * cfo * NCP / NFFT);
    const float PI_F = 3.14159274101257324f;                  // smallest float above pi: (ph > M_PI) <=> (ph >= PI_F)
    const float TWO_PI_HI = 6.28318548202514648f, TWO_PI_LO = -1.74845553e-07f;
    float f = cfreq, ph = cphase;
    // (kept rolled: one warp runs this alone, straight-line code would be bound by instruction fetch)
#pragma unroll 1
    for (int n = 0; n < BLK; n++) {
        const float2 v = z[n * zs];
        // u = v * exp(-j*ph); the loop error arg(v^2 * exp(-2j*ph)) / 2 equals arg(u^2) / 2
        float2 rot;
        if (FAST) {
            float sn, cs;
            __sincosf(-ph, &sn, &cs);
            rot = make_float2(cs, sn);
        } else {
            rot = cexp_j(-ph);
        }
        const float2 u = cmulf(v, rot);
        const float error = (FAST ? atan2_short((u.x * u.y) * 2.0f, u.x * u.x - u.y * u.y)
                                  : atan2f((u.x * u.y) * 2.0f, u.x * u.x - u.y * u.y)) * 0.5f;
        phs[n * zs] = ph;
        z[n * zs] = u;
        f += beta * error;
        if (f > 0.5f) f = 0.5f;
        if (f < -0.5f) f = -0.5f;
        ph += (f + cfo_freq) + (alpha * error);
        // (float)((double)ph -+ 2*pi) without double arithmetic on the serial path: 2*pi = HI + LO, the first
        // step is exact (Sterbenz), the second rounds once
        if (ph >= PI_F) ph = (ph - TWO_PI_HI) - TWO_PI_LO;
        if (ph <= -PI_F) ph = (ph + TWO_PI_HI) + TWO_PI_LO;
    }
    float x = 0;
#pragma unroll 4
    for (int n = 0; n < BLK; n++) x += z[n * zs].x * (float)((int)((pat_pos >> n) & 1u) - (int)((pat_neg >> n) & 1u));
    if (x < 0) {
#pragma unroll 4
        for (int n = 0; n < BLK; n++) {
            phs[n * zs] = (float)((double)phs[n * zs] + M_PI);
            z[n * zs] = make_float2(z[n * zs].x * -1.0f, z[n * zs].y * -1.0f);
        }
        ph = (float)((double)ph + M_PI);
    }
    cfreq = f;
    cphase = ph;
}

__device__ __forceinline__ int needle_bit(int n, unsigned rsid)       // -1 = don't care (sync.c:171-174)
{
    const signed char base[BLK] = { 0, 1, 0, 0, 0, 1, 1, -1, 1, 0, 0, 0, -1, 0, 0, -1,
                                    -1, -1, -1, -1, 0, 1, 0, -1, -1, -1, -1, -1, -1, -1, -1, 0 };
    if (n == 10) return (int)(rsid >> 1);
    if (n == 11) return (int)((rsid >> 1) ^ (rsid & 1));
    return base[n];
}

// find_ref_fm (sync.c:188-207): cyclic offset of the sync pattern, also trying the inverted bits
__device__ int ref_find(const float2 *z, int zs, unsigned rsid)
{
    unsigned raw = 0;
    for (int n = 0; n < BLK; n++)
        if (!(z[n * zs].x <= 0)) raw |= 1u << n;
    for (int pass = 0; pass < 2; pass++) {
        for (int n = 0; n < BLK; n++) {
            int i;
            for (i = 0; i < BLK; i++) {
                const int nb_ = needle_bit(i, rsid);
                if (nb_ < 0) continue;
                if (nb_ != (int)((raw >> ((n + i) & 31)) & 1)) break;
            }
            if (i == BLK) return n;
        }
        raw = ~raw;
    }
    return -1;
}

__device__ __forceinline__ float half_pi_wrap(float a, float b)        // sync.c:284-290
{
    float dd = a - b;
    while ((double)dd > M_PI / 2) dd = (float)((double)dd - M_PI);
    while ((double)dd < -M_PI / 2) dd = (float)((double)dd + M_PI);
    return dd;
}

__device__ __forceinline__ int8_t soft_demap(float x, float mult)      // sync.c:69-73
{
    // lroundf semantics (round half away from zero) without the libm call: |v| <= 127 so v - trunc(v) is exact
    const float v = fmaxf(fminf(x, 1.0f), -1.0f) * mult;
    int r = __float2int_rz(v);
    const float f = v - (float)r;
    if (f >= 0.5f) r++;
    else if (f <= -0.5f) r--;
    return (int8_t)r;
}

template <bool CL>
__device__ void front_sync(const DevPtrs &p, const EngineDims &d, int s, SyncSmem &sm, float2 (*zref)[ZS], BlockSet &b, int t)
{
    StreamState &st = p.st[s];
    float *cfreq = p.cfreq + (size_t)s * NFFT;
    float *cphase = p.cphase + (size_t)s * NFFT;
    // [symbol][534]; written by the demodulating teams - with a cluster per stream (CL), on other SMs: every read then
    // goes to L2 (__ldcg), never to this SM's L1
    float2 *bins = p.bins + (size_t)s * BLK * NBINS;
    auto ldbin = [](const float2 *q) -> float2 { return CL ? __ldcg(q) : *q; };
    const float loop_bw = 0.05f, damping = 0.70710678f;
    const float denom = 1 + (2 * damping * loop_bw) + (loop_bw * loop_bw);
    const float alpha = (4 * damping * loop_bw) / denom, beta = (4 * loop_bw * loop_bw) / denom;

    int ppb = partitions_per_band(st.psmi);
    int nref = ppb + 1;
    long long sy0 = clock64();
    const bool sy_on = st.state == ST_FINE;
    auto sylap = [&](int k) {
        if (t == 0 && sy_on) {
            const long long c1 = clock64();
            st.sy_cyc[k] += (unsigned long long)(c1 - sy0);
            sy0 = c1;
        }
    };
    // data carriers of both sidebands -> shared memory as [carrier][symbol] (coalesced reads along the carriers).
    // Element idx = n * rows2 + r is walked incrementally, without a division per element: the staging warps share
    // their schedulers with the Costas warp, whose chain is the phase's critical path.
    auto stage_eq = [&](int first, int stride) {
        const int rows = min(ppb, EQ_MAXPART) * (PW - 1), rows2 = 2 * rows;
        const int dn = stride / rows2, dr = stride - dn * rows2;
        int n = first / rows2, r = first - n * rows2;
#pragma unroll 4
        for (; n < BLK;) {
            const int sb = r >= rows, rr = sb ? r - rows : r;
            const int i = rr / (PW - 1);
            // lower: PW * i + k, upper: (NBINS - 1 - PW) - PW * i + k, with k = rr - (PW - 1) * i + 1
            const int ci = sb == 0 ? rr + i + 1 : (NBINS - PW) + rr - (2 * PW - 1) * i;
            sm.eq[r][n] = ldbin(&bins[(size_t)n * NBINS + ci]);
            r += dr;
            n += dn;
            if (r >= rows2) { r -= rows2; n++; }
        }
    };
    const bool pre_staged = st.state == ST_FINE && !(g_dbg & 1);   // partitions known: stage while warp 0 runs the Costas loops
    // reference carriers: stored in zref by the demodulating teams; with a cluster per stream the helpers' symbols
    // are only in global memory, so the owner gathers them all from there
    if (CL) {
        for (int i = t; i < ZS * BLK; i += FRONT_THREADS) {
            const int slot = i & (ZS - 1), n = i / ZS;
            const int ii = slot < MAXREF ? slot : slot - MAXREF;
            if (slot < 2 * MAXREF && ii < nref) zref[n][slot] = ldbin(&bins[(size_t)n * NBINS + compact_of_bin(ref_bin(slot))]);
        }
        __syncthreads();
    }
    sylap(0);
    // one Costas loop per reference carrier (sync.c:359-363), then its mean amplitude (calc_smag, sync.c:254-261:
    // the FINE equaliser's, taken here from the same rotated row)
    if (t < 2 * MAXREF) {
        const int i = t < MAXREF ? t : t - MAXREF;
        if (i < nref) {
            const int b = ref_bin(t);
            float f = cfreq[b], ph = cphase[b];
            costas_row(&zref[0][t], &sm.phs[0][t], ZS, f, ph, 0, alpha, beta, !(g_dbg & 2));
            cfreq[b] = f;
            cphase[b] = ph;
            sm.cfq[t] = f;
            float sum = 0;
            for (int n = 0; n < BLK; n++) sum += fabsf(zref[n][t].x);
            sm.smag[t] = sum / BLK;
        }
    } else if (t >= 32 && pre_staged) {
        stage_eq(t - 32, FRONT_THREADS - 32);
    }
    __syncthreads();
    sylap(1);

    if (st.state == ST_COARSE) {                 // sync.c:366-421
        if (t < 2 * MAXREF) {
            const int i = t < MAXREF ? t : t - MAXREF;
            sm.ref_ok[t] = 0;
            if (i < nref) {
                const float2 *z = &zref[0][t];
                const unsigned rsid = (unsigned)(30 - i) & 3;
                bool ok = true;
                unsigned raw = 0;
                for (int n = 0; n < BLK; n++) {
                    const int nbit = needle_bit(n, rsid);
                    const int pos = z[n * ZS].x > 0 ? 1 : 0;
                    if (nbit >= 0 && nbit != pos) ok = false;
                    if (!(z[n * ZS].x <= 0)) raw |= 1u << n;
                }
                const unsigned dd = raw ^ (raw << 1);        // DBPSK decode, prev = 0 (sync.c:138-148)
                auto bit = [&](int n) { return (dd >> n) & 1u; };
                sm.ref_ok[t] = ok;
                sm.ref_bc[t] = (int)(bit(16) << 3 | bit(17) << 2 | bit(18) << 1 | bit(19));
                sm.ref_psmi[t] = (int)(bit(25) << 5 | bit(26) << 4 | bit(27) << 3 | bit(28) << 2 | bit(29) << 1 | bit(30));
            }
        }
        __syncthreads();
        if (t == 0) {
            unsigned good = 0;
            for (int r = 0; r < 2 * MAXREF; r++)
                if (sm.ref_ok[r]) good++;
            sm.do_search = 0;
            if (good >= 4) {
                // strict majorities; the PSMI majority is only looked for among 0..15 (sync.c:396)
                int mbc = -1, mps = -1;
                for (int v = 0; v < 16; v++) {
                    unsigned nbc = 0, nps = 0;
                    for (int r = 0; r < 2 * MAXREF; r++) {
                        if (!sm.ref_ok[r]) continue;
                        nbc += sm.ref_bc[r] == v;
                        nps += sm.ref_psmi[r] == v;
                    }
                    if (nbc > good / 2) mbc = v;
                    if (nps > good / 2) mps = v;
                }
                if (mbc >= 0 && mps >= 0) {
                    st.bc = mbc;
                    st.psmi = mps;
                    set_state(p, d, s, ST_FINE);
                    l2_enqueue(st, d.l2, 0u, 0, 0);            // frame_reset (sync.c:405-409)
                    st.started_pm = 0;                   // decode_reset (decode.c:556-565)
                    st.px_total[0] = st.px_total[1] = 0;
                    st.px_started[0] = st.px_started[1] = 0;
                }
            } else if (st.cfo_wait == 0) {
                sm.do_search = 1;
            } else {
                st.cfo_wait--;
            }
        }
        __syncthreads();
        if (sm.do_search) {                      // detect_cfo (sync.c:292-337)
            // The reference tries the 76 integer offsets one after the other; each trial runs the Costas loop on
            // 22 carriers (cfo + the reference positions), looks for the sync pattern and puts the carriers back,
            // and the first offset with three agreeing block positions wins.  A trial only touches the state of
            // its own 22 bins, and two trials share a bin only if they are 19 apart - so every BIN has its own
            // short chain of trials (at most 4), and the chains of different bins are independent.  One thread
            // per bin walks its chain on a private copy (snapshots in the acquisition scratch), the winner is
            // picked exactly as the reference does, and only the snapshots up to the winner are committed.
            // First give the search the Costas-rotated references (adjust_ref has already run on them).
            for (int i = t; i < ZS * BLK; i += FRONT_THREADS) {
                const int slot = i & (ZS - 1), n = i / ZS;
                const int ii = slot < MAXREF ? slot : slot - MAXREF;
                if (slot < 2 * MAXREF && ii < nref) bins[(size_t)n * NBINS + compact_of_bin(ref_bin(slot))] = zref[n][slot];
            }
            for (int i = t; i < 76 * 22; i += FRONT_THREADS) sm.srch.offs[i / 22][i % 22] = -1;
            __syncthreads();
            constexpr int SB_BINS = 2 * PW * 2 + 10 * PW;                  // 266 bins a sideband's trials can touch
            constexpr int NSB = 2 * SB_BINS;
            float2 *snap = p.tbuf + (size_t)s * NACQ;                     // [4][32][NSB] row snapshots
            float *sphs = reinterpret_cast<float *>(p.ydec + (size_t)s * NACQ);   // [32][NSB] Costas phases
            float fs[4], phsn[4];
            int cfo_of[4], nq = 0, ci = -1, b = 0;
            if (t < NSB) {
                const int upper = t >= SB_BINS;
                b = upper ? (UB1 - 10 * PW - 2 * PW) + (t - SB_BINS) : (LB0 - 2 * PW) + t;
                ci = compact_of_bin(b);
                float f = cfreq[b], ph = cphase[b];
                // trials touching this bin, in increasing cfo: lower cfo = b - LB0 - 19 i, upper cfo = b - UB1 + 19 i
                int ref_i[4];
                for (int step = 0; step <= 10; step++) {
                    const int i = upper ? step : 10 - step;
                    const int cfo = upper ? b - UB1 + PW * i : b - LB0 - PW * i;
                    if (cfo >= -2 * PW && cfo < 2 * PW && nq < 4) {
                        ref_i[nq] = i;
                        cfo_of[nq] = cfo;
                        nq++;
                    }
                }
                // (the lanes of a warp walk their chains in step: trial q of every bin together)
                for (int q = 0; q < nq; q++) {
                    const int i = ref_i[q], cfo = cfo_of[q];
                    float2 *row = snap + (size_t)q * BLK * NSB + t;
                    const float2 *src = q ? snap + (size_t)(q - 1) * BLK * NSB + t : nullptr;
                    for (int n = 0; n < BLK; n++)
                        row[(size_t)n * NSB] = q ? src[(size_t)n * NSB]
                                                 : (ci >= 0 ? ldbin(&bins[(size_t)n * NBINS + ci]) : make_float2(0.f, 0.f));
                    costas_row(row, sphs + t, NSB, f, ph, cfo, alpha, beta, false);
                    sm.srch.offs[cfo + 2 * PW][2 * i + upper] = ref_find(row, NSB, (unsigned)(30 - i) & 3);
                    for (int n = 0; n < BLK; n++)            // reset_ref (sync.c:132-136)
                        row[(size_t)n * NSB] = cmulf(row[(size_t)n * NSB], cexp_j(sphs[(size_t)n * NSB + t]));
                    fs[q] = f;
                    phsn[q] = ph;
                }
            }
            __syncthreads();
            // every trial's verdict (sync.c:320-336), then the first successful trial
            if (t < 76) {
                int best = -1;
                unsigned bestn = 0;
                for (int k = 0; k < BLK; k++) {
                    unsigned nv = 0;
                    for (int r = 0; r < 22; r++) nv += sm.srch.offs[t][r] == k;
                    if (nv > bestn) { best = k; bestn = nv; }
                }
                sm.srch.verdict[t] = (best >= 0 && bestn >= 3) ? best : -1;
            }
            __syncthreads();
            if (t == 0) {
                int win = 1 << 20;                            // no winner: every trial ran
                for (int c = 0; c < 76; c++)
                    if (sm.srch.verdict[c] >= 0) { win = c - 2 * PW; break; }
                sm.srch.winner = win;
                if (win < (1 << 20)) {
                    st.keep_extra = ((BLK - sm.srch.verdict[win + 2 * PW]) % BLK) * NSYM;
                    st.cfo += win;
                    st.cfo_wait = 8;
                }
            }
            __syncthreads();
            if (t < NSB) {
                // commit what the sequential search would have left behind: the last trial <= the winner
                const int win = sm.srch.winner;
                int q = -1;
                for (int k = 0; k < nq; k++)
                    if (cfo_of[k] <= win) q = k;
                if (q >= 0) {
                    cfreq[b] = fs[q];
                    cphase[b] = phsn[q];
                    if (ci >= 0) {
                        const float2 *row = snap + (size_t)q * BLK * NSB + t;
                        for (int n = 0; n < BLK; n++) bins[(size_t)n * NBINS + ci] = row[(size_t)n * NSB];
                    }
                }
            }
        }
        __syncthreads();
        // (partitions_per_band stays what it was at entry even if the vote changed psmi, sync.c:343-357)
    }

    if (st.state == ST_FINE) {
        // exp(j*phase) per (reference, symbol), the equaliser's per-row constants, and the staging if it did not run
        // beside the Costas loops
        for (int i = t; i < 2 * MAXREF * BLK; i += FRONT_THREADS) {
            const int slot = i >> 5, n = i & 31;
            const int ii = slot < MAXREF ? slot : slot - MAXREF;
            if (ii < nref) sm.eph[slot][n] = cexp_j(sm.phs[n][slot]);
        }
        const int bc = st.bc;
        int8_t *pm = p.pm + ((size_t)s * 16 + bc) * PM_BLOCK;
        const int rows = min(ppb, EQ_MAXPART) * (PW - 1), rows2 = 2 * rows;
        // per carrier row: the two interpolation weights and the reference slots on either side
        for (int r = t; r < rows2; r += FRONT_THREADS) {
            const int sb = r >= rows, rr = sb ? r - rows : r;
            const int i = rr / (PW - 1), k = rr - i * (PW - 1) + 1;
            int slot_lo, slot_hi;
            if (sb == 0) { slot_lo = i; slot_hi = i + 1; }
            else { slot_lo = MAXREF + i + 1; slot_hi = MAXREF + i; }
            sm.rowc[r] = make_float4((float)k * sm.smag[slot_hi], (float)(PW - k) * sm.smag[slot_lo],
                                     __int_as_float(slot_hi), __int_as_float(slot_lo));
        }
        sylap(2);
        if (!pre_staged) stage_eq(t, FRONT_THREADS);
        // the extended partitions' interleaver positions, read before thread 0 advances them below
        const int cm = c_compat_mode[st.psmi & 63];
        const bool has_px1 = cm == 2 || cm == 3 || cm == 11;
        if (t == 0) {
            sm.px_on[0] = has_px1 && (st.px_started[0] || (bc & 1) == 0);      // decode_push_px1, decode.c:393-399
            sm.px_on[1] = cm == 11 && (st.px_started[1] || (bc & 1) == 0);     // decode_push_px2, decode.c:416-422
            sm.px_T[0] = st.px_total[0];
            sm.px_T[1] = st.px_total[1];
        }
        __syncthreads();
        sylap(3);
        // equalise (adjust_data, sync.c:263-282) and squared error to the nearest QPSK point (sync.c:465-488)
        float e_lb = 0.f, e_ub = 0.f;
        if (ppb > EQ_MAXPART) {
            // MP5 / MP6 / MP11 (14 partitions per sideband): partitions 12 and 13 do not fit the shared-memory
            // stage; they are equalised where they lie (2 x 2 x 18 carriers x 32 symbols) - they count in the MER
            // and MP11's PX2 demap reads them back from there
            const int xrows = (ppb - EQ_MAXPART) * (PW - 1);
            for (int idx = t; idx < 2 * xrows * BLK; idx += FRONT_THREADS) {
                const int r = idx >> 5, n = idx & (BLK - 1);
                const int sb = r >= xrows, rr = sb ? r - xrows : r;
                const int i = EQ_MAXPART + rr / (PW - 1), k = rr % (PW - 1) + 1;
                const int ci = sb == 0 ? PW * i + k : (NBINS - 1 - PW) - PW * i + k;
                const int slot_lo = sb == 0 ? i : MAXREF + i + 1, slot_hi = sb == 0 ? i + 1 : MAXREF + i;
                const float fa = (float)k * sm.smag[slot_hi], fb = (float)(PW - k) * sm.smag[slot_lo];
                const float2 up = sm.eph[slot_hi][n], lp = sm.eph[slot_lo][n];
                const float c = fa * up.x + fb * lp.x, dd = fa * up.y + fb * lp.y;
                const float rden = __fdividef(19.0f, c * c + dd * dd);
                const float2 C = make_float2((c + dd) * rden, (c - dd) * rden);
                const float2 v = cmulf(ldbin(&bins[(size_t)n * NBINS + ci]), C);
                bins[(size_t)n * NBINS + ci] = v;
                const float dx = (v.x >= 0 ? 1.0f : -1.0f) - v.x, dy = (v.y >= 0 ? 1.0f : -1.0f) - v.y;
                const float e = dx * dx + dy * dy;
                if (sb) e_ub += e;
                else e_lb += e;
            }
        }
        for (int idx = t; idx < rows2 * BLK; idx += FRONT_THREADS) {
            const int r = idx >> 5, n = idx & (BLK - 1);
            const float4 rc = sm.rowc[r];
            const float fa = rc.x, fb = rc.y;
            const float2 up = sm.eph[__float_as_int(rc.z)][n], lp = sm.eph[__float_as_int(rc.w)][n];
            const float c = fa * up.x + fb * lp.x, dd = fa * up.y + fb * lp.y;
            const float rden = __fdividef(19.0f, c * c + dd * dd);
            // (19 + 19j) / (c + j dd)
            const float2 C = make_float2((c + dd) * rden, (c - dd) * rden);
            const float2 v = cmulf(sm.eq[r][n], C);
            sm.eq[r][n] = v;
            const float dx = (v.x >= 0 ? 1.0f : -1.0f) - v.x, dy = (v.y >= 0 ? 1.0f : -1.0f) - v.y;
            const float e = dx * dx + dy * dy;
            if (r >= rows) e_ub += e;
            else e_lb += e;
        }
        // modulation error per sideband: a fixed-shape tree (thread, warp shuffle, then warp 0's lane 0 over the warps'
        // sums - which every warp repeats for itself and takes from its lane 0, instead of a barrier behind warp 0)
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            e_lb += __shfl_xor_sync(0xffffffffu, e_lb, o);
            e_ub += __shfl_xor_sync(0xffffffffu, e_ub, o);
        }
        if ((t & 31) == 0) { sm.wred[t >> 5][0] = e_lb; sm.wred[t >> 5][1] = e_ub; }
        __syncthreads();
        float mult[2], e_sb[2];
        {
            const int lane = t & 31;
            float a = sm.wred[lane][0], b = sm.wred[lane][1];
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                a += __shfl_xor_sync(0xffffffffu, a, o);
                b += __shfl_xor_sync(0xffffffffu, b, o);
            }
            e_sb[0] = __shfl_sync(0xffffffffu, a, 0);
            e_sb[1] = __shfl_sync(0xffffffffu, b, 0);
            const float mer_lb = 2.0f * BLK * (float)(ppb * 18) / e_sb[0], mer_ub = 2.0f * BLK * (float)(ppb * 18) / e_sb[1];
            mult[0] = fmaxf(fminf(mer_lb * 10, 127.0f), 1.0f);
            mult[1] = fmaxf(fminf(mer_ub * 10, 127.0f), 1.0f);
        }
        sylap(4);
        // Warps 2..31 demap; meanwhile warp 0's thread 0 does the block's record bookkeeping and warp 1 the timing /
        // phase feedback: neither touches what the demap reads, and both only feed the next block.
        constexpr int DEMAP_T0 = 64;
        if (t >= DEMAP_T0) {
            const int td = t - DEMAP_T0;
            constexpr int DSTRIDE = FRONT_THREADS - DEMAP_T0;
            // soft demap (sync.c:509-536) of the 10 primary-main partitions of each sideband into the interleaver
            // matrix, four soft bits (two carriers) per thread
            for (int item = td; item < BLK * 20 * 9; item += DSTRIDE) {
                const int n = item / 180, rem = item - n * 180;
                const int part = rem / 9, c4 = rem - part * 9;             // part 0..19 in demap order
                const int sb = part >= 10;
                // lower sideband: partition index; upper: the reference walks them upwards, storage is downwards
                const int r = (sb ? rows + (19 - part) * (PW - 1) : part * (PW - 1)) + 2 * c4;
                const float ml = mult[sb];
                const float2 a = sm.eq[r][n], b = sm.eq[r + 1][n];
                const unsigned w = (unsigned)(uint8_t)soft_demap(a.x, ml) | ((unsigned)(uint8_t)soft_demap(a.y, ml) << 8) |
                                   ((unsigned)(uint8_t)soft_demap(b.x, ml) << 16) | ((unsigned)(uint8_t)soft_demap(b.y, ml) << 24);
                *reinterpret_cast<uint32_t *>(pm + n * 720 + part * 36 + 4 * c4) = w;
            }
            // Extended partitions (sync.c:537-595): MP2 = one more partition per sideband (PX1, 2304 soft bits per
            // block), MP3 / MP11 = two more (PX1, 4608), MP11 = another two (PX2, 4608, both sidebands scaled with the
            // LOWER sideband's factor, sync.c:591-592).  They go to the convolutional interleaver's store in arrival
            // order.  The mode is looked up afresh here, so the block that reaches FINE sync demaps them although it
            // did not equalise them (its partition count was fixed at entry): partitions the equaliser staged come
            // from shared memory, the others from global memory (equalised in place above, or raw).
            const int eqparts = rows / (PW - 1);
            auto px_demap = [&](int8_t *ring, long long T, int nq, int base, bool lower_scale_only) {
                const int per_sym = nq * 36;
                for (int item = td; item < BLK * nq * 9; item += DSTRIDE) {
                    const int n = item / (nq * 9), rem = item - n * (nq * 9);
                    const int q = rem / 9, c4 = rem - q * 9;
                    // nq == 4: lower base, lower base+1, upper base+1, upper base (counted from the band edge); nq == 2: lower, upper
                    const int sb = q >= nq / 2;
                    const int i = nq == 2 ? base : ((q == 0 || q == 3) ? base : base + 1);
                    float2 a, b;
                    if (i < eqparts) {
                        const int r = (sb ? rows : 0) + i * (PW - 1) + 2 * c4;
                        a = sm.eq[r][n];
                        b = sm.eq[r + 1][n];
                    } else {
                        const int ci = (sb == 0 ? PW * i : (NBINS - 1 - PW) - PW * i) + 1 + 2 * c4;
                        a = ldbin(&bins[(size_t)n * NBINS + ci]);
                        b = ldbin(&bins[(size_t)n * NBINS + ci + 1]);
                    }
                    const float ml = mult[lower_scale_only ? 0 : sb];
                    const unsigned w = (unsigned)(uint8_t)soft_demap(a.x, ml) | ((unsigned)(uint8_t)soft_demap(a.y, ml) << 8) |
                                       ((unsigned)(uint8_t)soft_demap(b.x, ml) << 16) | ((unsigned)(uint8_t)soft_demap(b.y, ml) << 24);
                    const long long pos = (T + n * per_sym + q * 36 + 4 * c4) % PX_RING;
                    *reinterpret_cast<uint32_t *>(ring + pos) = w;
                }
            };
            if (sm.px_on[0]) px_demap(p.px_ring[0] + (size_t)s * PX_RING, sm.px_T[0], cm == 2 ? 2 : 4, 10, false);
            if (sm.px_on[1]) px_demap(p.px_ring[1] + (size_t)s * PX_RING, sm.px_T[1], 4, 12, true);
        } else if (t >= 32) {
            // timing / phase feedback (sync.c:426-463): the terms are computed in parallel, then summed by one lane in
            // the reference's order (same values, same rounding as the sequential loop)
            const int lane = t & 31;
            if (lane < ppb) {
                sm.fb_w[0][lane] = half_pi_wrap(sm.phs[0][lane], sm.phs[0][lane + 1]);
                sm.fb_w[1][lane] = half_pi_wrap(sm.phs[0][MAXREF + lane + 1], sm.phs[0][MAXREF + lane]);
            }
            if (lane <= ppb) {
                sm.fb_xy[0][lane] = (float)(LB0 + PW * lane - NFFT / 2) * sm.cfq[lane];
                sm.fb_xy[1][lane] = (float)(UB1 - PW * lane - NFFT / 2) * sm.cfq[MAXREF + lane];
            }
            __syncwarp();
            float fb_angle = 0;
            if (lane == 31) {
                float samperr = 0, angle = 0, sum_xy = 0, sum_x2 = 0;
                for (int i = 0; i < ppb; i++) {
                    samperr += sm.fb_w[0][i];
                    samperr += sm.fb_w[1][i];
                }
                // x / (2 pi) as a multiplication by the double reciprocal: the result is rounded to float anyway
                const double inv_2pi = 1.0 / (2 * M_PI);
                samperr = (float)((double)(samperr / (float)(ppb * 2) * (float)NFFT / (float)PW) * inv_2pi);
                for (int i = 0; i <= ppb; i++) {
                    float x;
                    x = (float)(LB0 + PW * i - NFFT / 2);
                    angle += sm.cfq[i]; sum_xy += sm.fb_xy[0][i]; sum_x2 += x * x;
                    x = (float)(UB1 - PW * i - NFFT / 2);
                    angle += sm.cfq[MAXREF + i]; sum_xy += sm.fb_xy[1][i]; sum_x2 += x * x;
                }
                samperr = (float)((double)samperr - (double)((sum_xy / sum_x2) * (float)NFFT) * inv_2pi * BLK);
                const int se = (int)roundf(samperr);
                st.samperr = se;
                angle /= (float)((ppb + 1) * 2);
                st.angle = angle;
                fb_angle = angle;
                if (!CL) {                       // the next block's set-up, as its FINE prep would compute it
                    b.samperr = NSYM / 2 + se;
                    b.prev_angle = st.prev_angle + (-angle);
                    block_setup(b, st);
                    b.ok = 1;
                }
            }
            fb_angle = __shfl_sync(0xffffffffu, fb_angle, 31);
            const int i = lane < MAXREF ? lane : lane - MAXREF;
            if (lane < 2 * MAXREF && i < nref) cfreq[ref_bin(lane)] = sm.cfq[lane] - fb_angle;
        } else if (t == 0) {
            st.err_lb += e_sb[0];
            st.err_ub += e_sb[1];
            if (++st.mer_cnt == 16) {
                const float signal = (float)(2 * BLK * (ppb * 18) * st.mer_cnt);
                uint8_t *w = log_reserve(p, d, s, REC_MER, 8);
                if (w) {
                    reinterpret_cast<float *>(w)[0] = 10 * log10f(signal / st.err_lb);
                    reinterpret_cast<float *>(w)[1] = 10 * log10f(signal / st.err_ub);
                }
                st.mer_cnt = 0;
                st.err_lb = 0;
                st.err_ub = 0;
            }
            if (d.emit_soft) {                  // filled below, once the demap is done
                sm.soft_w = log_reserve(p, d, s, REC_SOFT_PM, 4 + PM_BLOCK);
                if (sm.soft_w) *reinterpret_cast<uint32_t *>(sm.soft_w) = (uint32_t)bc;
            }
            // PIDS (decode.c:463-471): the frames of a pass are decoded together when k_stream exits; the record
            // slot is reserved here to keep the stream's record order
            uint8_t *w = log_reserve(p, d, s, REC_PIDS, 11);             // 80 bits + CRC verdict
            const int e = st.pids_pending;
            st.pids_rec[e] = w ? (unsigned)(w - (p.log + (size_t)s * d.log_cap)) : 0xffffffffu;
            st.pids_bc[e] = bc;
            st.pids_pending = e + 1;
            // P1 bookkeeping (decode.c:383-390); the BER and FRAME records are reserved now so that they keep
            // their place in the stream's record order (decode.c:458-460)
            if (bc == 0) st.started_pm = 1;
            unsigned lost_slot = 0xffffffffu;
            if (st.started_pm && bc == 15) {
                // both or neither: a BER record whose frame did not fit is taken back (its payload would never be filled)
                const unsigned len0 = st.log_len;
                uint8_t *bw = log_reserve(p, d, s, REC_BER, 4);
                uint8_t *fw = bw ? log_reserve(p, d, s, REC_FRAME, 8 + P1_LEN / 8) : nullptr;
                if (!fw) { st.log_len = len0; bw = nullptr; }
                st.p1_rec = (bw && fw) ? (unsigned)(bw - (p.log + (size_t)s * d.log_cap)) : 0xffffffffu;
                if (fw) {
                    reinterpret_cast<uint32_t *>(fw)[0] = 0;            // P1 logical channel
                    reinterpret_cast<uint32_t *>(fw)[1] = P1_LEN;
                    // the sync loss the frame's header check may report (k_p1_fin) comes before this block's P3 / P4
                    // frames: the reference's frame_push reports it inside decode_push_pm, which runs before
                    // decode_push_px1 / _px2.  Keep a slot for it here; it is taken back below if no such frame follows.
                    uint8_t *lw = log_reserve(p, d, s, REC_PAD, 0);
                    if (lw) lost_slot = (unsigned)(lw - 8 - (p.log + (size_t)s * d.log_cap));
                }
                st.p1_lost_rec = lost_slot;
                l2_enqueue(st, d.l2, st.p1_rec != 0xffffffffu ? st.p1_rec + 4 + 8 + 8 : 0xffffffffu, 0, P1_LEN);   // BER payload | FRAME header | lc, nbits | bits
                st.p1_ready = 1;
            }
            // P3 / P4 bookkeeping (decode_push_px1 / _px2, decode.c:393-437): every second block closes a span of the
            // interleaver (2 * len soft bits); once a whole cycle (32 * len) has gone through, it yields a frame.  A
            // mode feeds at most one group per ring, so each ring advances once.  The records are reserved now, in
            // group order: P3 before P4, like the reference's calls.  Unrolled, so that each group's constants fold:
            // thread 0 runs this while the CTA waits, and a rolled loop costs MP3 streams measurably more.
#pragma unroll
            for (int g = 0; g < PX_GROUPS; g++) {
                const PxGroup x = px_group(g);
                if (!(x.modes >> cm & 1)) continue;
                if ((bc & 1) == 0) st.px_started[x.ring] = 1;
                if (!st.px_started[x.ring]) continue;
                st.px_total[x.ring] += x.len;
                const long long k0 = st.px_total[x.ring] - 2 * x.len;
                if ((bc & 1) && k0 >= 32 * x.len && st.xq_pending[g] < P3_SLOTS) {
                    uint8_t *fw = log_reserve(p, d, s, REC_FRAME, 8 + x.len / 8);
                    const int e = st.xq_pending[g];
                    st.xq_k0[g][e] = k0;
                    st.xq_rec[g][e] = fw ? (unsigned)(fw - (p.log + (size_t)s * d.log_cap)) : 0xffffffffu;
                    if (fw) {
                        reinterpret_cast<uint32_t *>(fw)[0] = x.lc;
                        reinterpret_cast<uint32_t *>(fw)[1] = x.len;
                    }
                    l2_enqueue(st, d.l2, fw ? st.xq_rec[g][e] + 8 : 0xffffffffu, x.lc, x.len);
                    st.xq_pending[g] = e + 1;
                }
            }
            if (lost_slot != 0xffffffffu && st.log_len == lost_slot + 8) {      // no P3 / P4 frame after it (MP1 logs
                st.log_len = lost_slot;                                          // never hold the slot)
                st.p1_lost_rec = 0xffffffffu;
            }
            st.bc = (bc + 1) % 16;
        }
        __syncthreads();
        if (d.emit_soft && sm.soft_w)
            for (int o = t; o < PM_BLOCK; o += FRONT_THREADS) sm.soft_w[4 + o] = (uint8_t)pm[o];
    }
    if (t == 0) {                                // window overlap carry (acquire.c:259-262)
        const int keep = NSYM + (NSYM / 2 - st.blk_samperr) + st.keep_extra;
        st.keep_extra = 0;
        st.start += NACQ - keep;
        st.blocks_done++;
    }
    sylap(5);
}

// ---------------------------------------------------------------------------
// the stream-resident kernel: one CTA per stream - or, when the engine has fewer streams than the GPU has SMs, a
// thread-block CLUSTER of d.cluster CTAs per stream (engine.cu picks 1, 2 or 4): the cluster's first CTA owns the
// stream (prep, sync, feedback, bookkeeping), all of them demodulate - 8 teams each, so a block's 32 symbols take
// 4 / 2 / 1 rounds - and hand the kept bins over through L2.  The hand-offs are two hardware cluster barriers per
// block (barrier.cluster, release / acquire); the block's parameters travel through the stream's state in global
// memory, every CTA builds its own copy of the NCO table.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void cluster_barrier()
{
#if defined(NB_EMU)
    // (the emulator runs one CTA at a time: engines are created with cluster = 1 there)
#else
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
#endif
}

template <bool CL>
__global__ void __launch_bounds__(FRONT_THREADS, 1) k_stream(DevPtrs p, EngineDims d, int max_blocks, int last_pass)
{
#if defined(NB_EMU)
    unsigned char *front_smem_raw = emu::dyn_smem();
#else
    extern __shared__ __align__(16) unsigned char front_smem_raw[];
#endif
    FrontSmem &sm = *reinterpret_cast<FrontSmem *>(front_smem_raw);
    const int t = threadIdx.x, team = t >> 7, tl = t & 127;
    const int C = CL ? d.cluster : 1;                 // (CL: launched as clusters of d.cluster = 2 or 4 CTAs)
    const int s = (int)blockIdx.x / C, rank = (int)blockIdx.x % C;
    StreamState &st = p.st[s];
    for (int i = t; i < FFT_TW; i += FRONT_THREADS) sm.tw[i] = __ldg(&p.twid[i]);
    if (t < 128) {                                     // front_demod's stores of thread t: compact q-222, q+34, q+243, q+499
        unsigned m = 0xffu;                            // lower slot i: compact 19 i; upper slot MAXREF + i: 533 - 19 i
        for (int h = 0; h < 2; h++) {
            const int q = t + 128 * h;
            const int c[4] = { q >= 222 ? q - 222 : -1, q <= 232 ? q + 34 : -1, q >= 24 ? q + 243 : -1, q <= 34 ? q + 499 : -1 };
            for (int k = 0; k < 4; k++) {
                if (c[k] < 0) continue;
                const int slot = c[k] < SIDE ? (c[k] % PW == 0 ? c[k] / PW : -1)
                                             : ((NBINS - 1 - c[k]) % PW == 0 ? MAXREF + (NBINS - 1 - c[k]) / PW : -1);
                if (slot >= 0) m = (unsigned)(4 * h + k) << 5 | (unsigned)slot;   // (at most one per thread)
            }
        }
        sm.ref_plan[t] = (uint8_t)m;
    }
    if (t == 0) {                                     // (the first block's prep fills its NCO tables from these)
        sm.blk.ok = 0;
        sm.blk.theta = 0.f;
        sm.blk.phase0 = make_float2(0.f, 0.f);
    }
    __syncthreads();

    const bool owner = !CL || rank == 0;
    if (max_blocks > 16) max_blocks = 16;             // the PIDS queue (and its interleaver matrix rows) hold 16 blocks
    if (owner && t == 0) {                            // decoded by the kernels that followed the previous pass
        for (int g = 0; g < PX_GROUPS; g++) st.xq_pending[g] = 0;
    }
    __syncthreads();
    for (int nb = 0;; nb++) {
        long long c0 = clock64();
        auto lap = [&](int ph) {
            if (owner && t == 0) {
                const long long c1 = clock64();
                st.ph_cyc[ph] += (unsigned long long)(c1 - c0);
                st.ph_n[ph]++;
                c0 = c1;
            }
        };
        // a completed interleaver matrix is decoded (and its header checked) before the next block
        // blk_go: 0 = the pass is over, 1 = demodulate the block (its parameters are in place), 2 = coarse acquisition
        // first - which the stream's CTAs share
        int mode = 0;
        if (!CL) {
            if (nb < max_blocks && !st.p1_ready) mode = front_prep_single(p, d, s, sm.u.acq1, sm.nco, sm.symphase, sm.blk, t) ? 1 : 0;
            if (mode == 0) break;
        } else {
            if (owner) {
                if (nb < max_blocks && !st.p1_ready) mode = front_prep_begin(p, d, s, t);
                if (mode == 1) front_prep_finish(p, d, s, sm.u.prep, sm.nco, sm.symphase, sm.blk, t, 1);
            }
            if (owner && t == 0) {
                st.blk_go = mode;
                __threadfence();
            }
            cluster_barrier();                        // the helpers read the block's parameters behind this barrier
            if (!owner) mode = __ldcg(&st.blk_go);
            if (mode == 0) break;
            if (mode == 2) {
                front_acq_tiles(p, d, s, sm.u.prep, t, rank, C);
                __threadfence();
                cluster_barrier();                    // the whole window is in L2
                front_acq_corr(p, s, t, rank, C);
                __threadfence();
                cluster_barrier();
                if (owner) {
                    front_prep_finish(p, d, s, sm.u.prep, sm.nco, sm.symphase, sm.blk, t, 2);
                    __threadfence();
                }
                cluster_barrier();                    // the block's parameters are in place
            }
        }
        lap(st.blk_state_in == ST_FINE ? 2 : 1);
        const long long start = CL ? __ldcg(&st.start) : st.start;
        // (k_stream<false>: thread 0 may still be committing the block's parameters to the stream's state)
        const int samperr = CL ? __ldcg(&st.blk_samperr) : sm.blk.samperr;
        if (CL && !owner) {                                 // a helper CTA builds its own copy of the block's NCO tables
            const float theta = __ldcg(&st.theta);
            fill_nco(p, sm.nco, theta, t);
            if (t >= FRONT_THREADS - BLK) fill_symphase(sm.symphase, theta, __ldcg(&st.phase0), t - (FRONT_THREADS - BLK));
            __syncthreads();
        }
#pragma unroll 1
        for (int pass = 0; pass < BLK / (TEAMS * C); pass++)
            front_demod(p, d, s, (pass * C + rank) * TEAMS + team, sm.u.demod, sm.nco, sm.symphase, sm.tw, sm.zref, sm.ref_plan,
                            team, tl, start, samperr);
        if (CL) {
            __threadfence();
            cluster_barrier();                        // every CTA's bins are in L2
        }
        if (CL && !owner) continue;
        __syncthreads();
        lap(3);
        front_sync<CL>(p, d, s, sm.u.sync, sm.zref, sm.blk, t);
        __syncthreads();
        lap(st.blk_state_in == ST_FINE ? 4 : 5);
    }
    if (CL && !owner) return;
    __syncthreads();
    if (st.pids_pending) {
        const long long c0 = clock64();
        front_pids_flush(p, d, s, sm.u.pidsq, t);
        if (t == 0) {
            st.ph_cyc[0] += (unsigned long long)(clock64() - c0);
            st.ph_n[0]++;
        }
    }
    if (t == 0) {
        // for the host's planning of the next batch: where the stream stands, and - after a batch's last pass -
        // whether it could go on at once (a frame it just completed is decoded by the kernels that follow this one)
        StreamBrief b;
        b.start = st.start;
        b.state = st.state;
        b.bc = st.bc;
        b.p1_ready = st.p1_ready;
        b.pad_ = 0;
        p.brief[s] = b;
        const long long avail = *reinterpret_cast<volatile long long *>(&st.in_avail);
        if (last_pass && avail >= 2 * (st.start + NACQ)) atomicAdd(&p.ctl->more, 1u);
    }
}

}  // namespace nb
