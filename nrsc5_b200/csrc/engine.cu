// nrsc5_b200 engine: per-block control, acquisition, sync/equalise/demap,
// L1 decode kernels and the host-side C ABI (include/nrsc5_b200.h).
//
// This translation unit is compiled with -fmad=false: the acquisition and
// sync arithmetic keeps the reference's float operation order so that every
// discrete decision (timing arg-max, reference-subcarrier votes, rounded
// timing error) is taken on the same values as the reference computes, up to
// the GPU's libm.  The FFT-heavy demodulator lives in frontend.cu.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <new>
#include <vector>

#include "../../include/nrsc5_b200.h"
#include "chan_feed.h"
#include "common.cuh"
// NVTX ranges around the host-side phases (header-only NVTX 3: no library to link; a no-op unless a tool is attached -
// `ncu --nvtx`, Nsight Systems): process / submit / poll, and per pass the front end and the decode groups
#if defined(NB_EMU)
struct NvtxRange { explicit NvtxRange(const char *) {} };
#else
#include <nvtx3/nvToolsExt.h>
struct NvtxRange {
    explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};
#endif
#include "rs.cuh"
#include "viterbi.cuh"
#include "viterbi_chunk.cuh"
#include "viterbi64.cuh"
#include "front.cuh"
#include "am.cuh"
#include "am_tables.h"
#include "l2.cuh"

namespace nb {

void launch_fft_test(const float2 *in, float2 *out, const float2 *twid, int nffts, cudaStream_t stream);
void launch_halfband_test(const uint8_t *cu8, long long npairs, short2 *out, cudaStream_t stream);

// ===========================================================================
// P1 decode: for every stream whose interleaver matrix is complete —
//   k_p1_gather : interleaver I + depuncture 1,1,1,1,1,0  (decode.c:296-322)
//   k_vitc_fwd / k_vitc_ends / k_vitc_emit : K=7 tail-biting Viterbi (viterbi_chunk.cuh)
//   k_p1_fin    : channel BER (decode.c:234-265), descramble (:279-294), packing,
//                 and the L2 header predicate that feeds back into the sync state
//                 (frame.c:645-714,527-541,158-179; rs_decode.c)
// ===========================================================================
constexpr int P1_THREADS = 256;
constexpr int P1_NCH = (P1_STEPS + CH_LEN - 1) / CH_LEN;             // 143

// Interleaver I as a row-wise pass: all P1 soft bits that come from matrix row r of the 16 blocks
// (decode.c:296-322: row = 11k % 32, k = i / 320) are the 320-bit groups k = 3r % 32 + 32m.  A CTA stages
// those 16 x 720 bytes with coalesced loads and writes each group's 384 depunctured bytes contiguously;
// inside a group the source offset (block, partition) depends on the position only, the column on k only.
__constant__ uint16_t c_p1_src[320];                                   // (block * 720 + partition * 36) of position w

__global__ void __launch_bounds__(256) k_p1_gather(DevPtrs p, EngineDims d)
{
    const int s = blockIdx.y, r = blockIdx.x, t = threadIdx.x;
    StreamState &st = p.st[s];
    if (!st.p1_ready) return;
    __shared__ __align__(16) int8_t rows[16 * 720];
    __shared__ uint16_t src[320];
    for (int i = t; i < 320; i += 256) src[i] = c_p1_src[i];
    if (r == 0 && t == 0) {
        // (the BER and FRAME records were reserved by the block's sync, in record order)
        st.p1_errs = 0;
        st.p1_done = 0;
        st.p1_retry = 0;
    }
    const int8_t *pm = p.pm + (size_t)s * 16 * PM_BLOCK;
    for (int v = t; v < 16 * 45; v += 256) {
        const int blk = v / 45, q = v - blk * 45;
        reinterpret_cast<uint4 *>(rows)[v] = *reinterpret_cast<const uint4 *>(pm + (size_t)(blk * 32 + r) * 720 + 16 * q);
    }
    __syncthreads();
    uint32_t *vout = reinterpret_cast<uint32_t *>(p.vit_in + (size_t)s * P1_VIT);
    const int k0 = (3 * r) & 31;                                        // 11 * 3 = 1 (mod 32)
    for (int item = t; item < 36 * 96; item += 256) {
        const int m = item / 96, wq = item - m * 96;
        const int k = k0 + 32 * m;
        if (k >= P1_ENC / 320) break;
        const int col = (11 * k + k / 288) % 36;
        uint32_t word = 0;
#pragma unroll
        for (int bb = 0; bb < 4; bb++) {
            const int o = 4 * wq + bb, q = o / 6, r6 = o - 6 * q;
            if (r6 != 5) word |= (uint32_t)(uint8_t)rows[src[5 * q + r6] + col] << (8 * bb);
        }
        vout[96 * k + wq] = word;
    }
}

constexpr int FIN_BYTES = 1024;                                      // packed PDU bytes per CTA
constexpr int FIN_CTAS = (P1_LEN / 8 + FIN_BYTES - 1) / FIN_BYTES;   // 18

__device__ __forceinline__ unsigned p1_bit(const uint32_t *bw, int i)
{
    return (bw[i >> 5] >> (i & 31)) & 1u;
}

__constant__ uint32_t c_spread3[256];                                 // bit k of the index -> bit 3k

__global__ void __launch_bounds__(P1_THREADS) k_p1_fin(DevPtrs p, EngineDims d)
{
    const int s = blockIdx.y, t = threadIdx.x;
    StreamState &st = p.st[s];
    if (!st.p1_ready) return;
    __shared__ int red[P1_THREADS];
    __shared__ int sh_last;
    __shared__ uint8_t hdr[96];
    __shared__ GfTab gf;
    __shared__ uint32_t spread[256];
    spread[t] = c_spread3[t];
    __syncthreads();
    const int8_t *vin = p.vit_in + (size_t)s * P1_VIT;
    const uint32_t *bw = p.p1_bits + (size_t)s * (P1_LEN / 32);
    uint8_t *rec = st.p1_rec == 0xffffffffu ? nullptr : p.log + (size_t)s * d.log_cap + st.p1_rec;
    uint8_t *frame = rec ? rec + 4 + 8 + 8 : nullptr;                // BER payload (4) | FRAME header (8) | lc,nbits (8) | bytes
    const int byte0 = blockIdx.x * FIN_BYTES, byte1 = min(P1_LEN / 8, byte0 + FIN_BYTES);
    int errs = 0;
    static_assert(FIN_BYTES % P1_THREADS == 0, "whole iterations");
#pragma unroll
    for (int it = 0; it < FIN_BYTES / P1_THREADS; it++) {          // independent iterations: their loads overlap
        const int bi = byte0 + t + it * P1_THREADS;
        if (bi >= byte1) break;
        // 14 decoded bits around this byte: frame bits 8*bi-6 .. 8*bi+7 (tail-biting wrap at the frame start)
        unsigned win;
        {
            const int i0 = 8 * bi - 6;
            if (i0 >= 0) {
                const int w0 = i0 >> 5;
                const uint32_t lo = bw[w0], hi = (w0 + 1 < P1_LEN / 32) ? bw[w0 + 1] : 0u;
                win = __funnelshift_r(lo, hi, i0 & 31) & 0x3fffu;
            } else {
                win = (bw[P1_LEN / 32 - 1] >> 26) | ((bw[0] & 0xffu) << 6);
            }
        }
        // re-encode (decode.c:243-249): the register of bit i holds bits i-6..i, newest at bit 6; code bit of
        // polynomial g for the byte's 8 bits at once = XOR over the taps of g of (win >> tap)
        const unsigned e0 = (win ^ (win >> 1) ^ (win >> 3) ^ (win >> 4) ^ (win >> 6)) & 0xffu;      // 0133
        const unsigned e1 = (win ^ (win >> 3) ^ (win >> 4) ^ (win >> 5) ^ (win >> 6)) & 0xffu;      // 0171
        const unsigned e2 = (win ^ (win >> 2) ^ (win >> 4) ^ (win >> 5) ^ (win >> 6)) & 0xffu;      // 0165
        const unsigned enc24 = spread[e0] | (spread[e1] << 1) | (spread[e2] << 2);
        // signs of the 24 soft values of these 8 bits: bit m = (soft[24*bi + m] > 0)
        unsigned pos24 = 0;
        const uint2 *q = reinterpret_cast<const uint2 *>(vin + 24 * (size_t)bi);
#pragma unroll
        for (int h = 0; h < 3; h++) {
            const uint2 v = q[h];
#pragma unroll
            for (int g = 0; g < 2; g++) {
                const unsigned x = g ? v.y : v.x;
                const unsigned nz = ((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x;          // bit 7 of a byte: byte != 0
                const unsigned ps = ((nz & ~x) >> 7) & 0x01010101u;                 // byte > 0
                pos24 |= ((ps * 0x01020408u) >> 24) << (8 * h + 4 * g);
            }
        }
        // channel bit errors on the unpunctured positions (decode.c:234-259); every 6th soft value is a puncture
        errs += __popc((enc24 ^ pos24) & 0x7df7dfu);
        // descramble (decode.c:279-294) and pack MSB first
        const unsigned bits8 = ((win >> 6) & 0xffu) ^ ((p.pnw[bi >> 2] >> (8 * (bi & 3))) & 0xffu);
        if (frame) frame[bi] = (uint8_t)(__brev(bits8) >> 24);
    }
    red[t] = errs;
    __syncthreads();
    for (int o = P1_THREADS / 2; o; o >>= 1) {
        if (t < o) red[t] += red[t + o];
        __syncthreads();
    }
    if (t == 0) {
        atomicAdd(&st.p1_errs, red[0]);
        __threadfence();
        sh_last = atomicAdd(&st.p1_done, 1) == FIN_CTAS - 1;
    }
    __syncthreads();
    if (!sh_last) return;
    // last CTA of this stream: BER record, and the L2 feedback predicate
    // (frame.c:645-714 PCI, :146-156 has_audio, :527-541 header RS check)
    __threadfence();
    gf_tab_load(gf, t, P1_THREADS);
    if (t < 96) {
        // PDU byte n of frame_push() is the bit-reversed packed byte n (the reference swaps the bit order per byte)
        unsigned v = frame ? __ldcg(frame + t) : 0;
        hdr[t] = (uint8_t)(__brev(v) >> 24);
    }
    __syncthreads();
    if (t < 32) {                                        // warp 0: the 24 PCI bits a lane each, the header by the warp's RS decoder
        unsigned bit = 0;
        if (t < 24) {
            const unsigned i = 116176u + 1248u * t;
            const unsigned phys = (i & ~7u) + 7 - (i & 7);
            bit = ((p1_bit(bw, (int)phys) ^ (p.pnw[phys >> 5] >> (phys & 31))) & 1u) << (23 - t);
        }
        const unsigned pci = warp_xor(bit);
        const bool has_audio = (pci & 0xFFFFFC) != (0x3634CE & 0xFFFFFC);
        const int ok = has_audio ? rs8_fix_header_warp(gf, hdr, t) : 1;
        if (t == 0) {
            if (rec) *reinterpret_cast<float *>(rec) = (float)atomicAdd(&st.p1_errs, 0) / (float)P1_ENC;
            if (!ok) {
                if (st.state == ST_FINE && st.p1_lost_rec != 0xffffffffu) {     // the slot k_stream kept between this
                    *reinterpret_cast<uint32_t *>(p.log + (size_t)s * d.log_cap + st.p1_lost_rec) = REC_LOST_SYNC;
                    st.state = ST_NONE;                                          // frame and its block's P3 / P4 frames
                } else {
                    set_state(p, d, s, ST_NONE);
                }
            }
            if (st.p1_retry) st.p1_fallbacks++;
            st.p1_ready = 0;
            st.p1_slow = 0;
            st.p1_retry = 0;
            st.frames_done++;
        }
    }
}

__host__ __device__ inline VitcArgs p1_vitc_args(const DevPtrs &dp)
{
    VitcArgs a;
    a.vin = dp.vit_in;
    a.dec = dp.vit_dec;
    a.vspec = dp.vspec;
    a.vend = dp.vend;
    a.hstate = dp.hstate;
    a.tbend = dp.tbend;
    a.bitsw = dp.p1_bits;
    a.ready = &dp.st[0].p1_retry;      // the fallback only decodes what the fast path gave up on
    a.slow = &dp.st[0].p1_slow;
    a.ready_stride = (int)(sizeof(StreamState) / sizeof(int));
    a.len = P1_LEN;
    a.nch = P1_NCH;
    a.dec_stride = (size_t)P1_NCH * CH_LEN;
    return a;
}

__host__ __device__ inline V64Args p1_v64_args(const DevPtrs &dp, int ch)
{
    V64Args a;
    a.vin = dp.vit_in;
    a.dec = dp.vit_dec;
    a.vspec = dp.v64_spec;
    a.vend = dp.v64_end;
    a.endstate = dp.v64_endstate;
    a.bitsw = dp.p1_bits;
    a.ready = &dp.st[0].p1_ready;
    a.retry = &dp.st[0].p1_retry;
    a.stride = (int)(sizeof(StreamState) / sizeof(int));
    a.len = P1_LEN;
    a.ch = ch;
    a.nch = (P1_STEPS + ch - 1) / ch;
    a.dec_stride = (size_t)P1_NCH * CH_LEN;
    return a;
}

// ===========================================================================
// Extended-partition decode (MP2, MP3, MP11): for every frame of decode group G (px_group) the pass queued
// (decode_push_px1 / _px2, reference src/decode.c:393-437) -
//   k_px_gather<G> : interleaver IV as a gather through its delay table + depuncture 1,0,1,1,0,1 (decode.c:344-376)
//   the same Viterbi kernels as P1 (fast path with 256-step chunks, exact fallback)
//   k_px_fin<G>    : descramble (decode.c:279-294) and pack into the frame's reserved record
// These frames feed nothing back into the receiver (frame.c:535-540 only acts on P1), so they can wait for the end
// of the pass.  G is a template argument so that the interleaver span is a compile-time divisor.
// ===========================================================================
template <int G>
__global__ void __launch_bounds__(256) k_px_gather(DevPtrs p, EngineDims d)
{
    constexpr int len = px_group(G).len, span = 32 * len;
    const int s = blockIdx.y, slot = blockIdx.x, t = threadIdx.x;
    const StreamState &st = p.st[s];
    const PxBufs &xb = p.xb[G];
    int *fl = xb.flags + ((size_t)s * P3_SLOTS + slot) * 4;
    const bool on = slot < st.xq_pending[G];
    if (t == 0) { fl[0] = on; fl[1] = 0; fl[2] = 0; }
    if (!on) return;
    const long long k0 = st.xq_k0[G][slot];
    const uint32_t *delay = len == P3_LEN ? p.iv_delay : p.iv_delay_s;
    const int8_t *ring = p.px_ring[px_group(G).ring] + (size_t)s * PX_RING;
    uint32_t *vout = reinterpret_cast<uint32_t *>(xb.vin + ((size_t)s * P3_SLOTS + slot) * (3 * len));
    // 12 outputs = 8 transmitted soft bits: positions 0 2 3 5 | 6 8 9 11 of each dozen, zeros in between
    for (int g = t; g < 3 * len / 12; g += 256) {
        int8_t v[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const long long k = k0 + 8 * g + i;
            const long long j = k - (long long)__ldg(&delay[k % span]);
            v[i] = ring[j % PX_RING];
        }
        auto b = [&](int i) { return (uint32_t)(uint8_t)v[i]; };
        vout[3 * g + 0] = b(0) | (b(1) << 16) | (b(2) << 24);
        vout[3 * g + 1] = (b(3) << 8) | (b(4) << 16);
        vout[3 * g + 2] = b(5) | (b(6) << 8) | (b(7) << 24);
    }
}

template <int G>
__global__ void __launch_bounds__(128) k_px_fin(DevPtrs p, EngineDims d)
{
    constexpr int len = px_group(G).len;
    const int s = blockIdx.y, slot = blockIdx.x, t = threadIdx.x;
    const StreamState &st = p.st[s];
    if (slot >= st.xq_pending[G]) return;
    const unsigned rec = st.xq_rec[G][slot];
    if (rec == 0xffffffffu) return;
    uint8_t *frame = p.log + (size_t)s * d.log_cap + rec + 8;          // past lc, nbits
    const uint32_t *bw = p.xb[G].bits + ((size_t)s * P3_SLOTS + slot) * (len / 32);
    for (int w = t; w < len / 32; w += 128) {
        const uint32_t x = bw[w] ^ p.pnw[w];                            // the descrambler restarts with every frame
        // MSB-first bytes
        reinterpret_cast<uint32_t *>(frame)[w] = __brev(__byte_perm(x, 0, 0x0123));
    }
}

__host__ __device__ inline V64Args px_v64_args(const DevPtrs &dp, int g)
{
    const PxBufs &xb = dp.xb[g];
    const int len = px_group(g).len;
    V64Args a;
    a.vin = xb.vin;
    a.dec = xb.dec;
    a.vspec = xb.spec;
    a.vend = xb.end;
    a.endstate = xb.endstate;
    a.bitsw = xb.bits;
    a.ready = xb.flags;
    a.retry = xb.flags + 2;
    a.stride = 4;
    a.len = len;
    a.ch = 256;
    a.nch = (len + 64 + 255) / 256;
    a.dec_stride = P3_DEC_STRIDE;
    return a;
}

__host__ __device__ inline VitcArgs px_vitc_args(const DevPtrs &dp, int g)
{
    const PxBufs &xb = dp.xb[g];
    const int len = px_group(g).len;
    VitcArgs a;
    a.vin = xb.vin;
    a.dec = xb.dec;
    a.vspec = xb.fspec;
    a.vend = xb.fend;
    a.hstate = xb.fhstate;
    a.tbend = xb.ftbend;
    a.bitsw = xb.bits;
    a.ready = xb.flags + 2;            // the fallback only decodes what the fast path gave up on
    a.slow = xb.flags + 1;
    a.ready_stride = 4;
    a.len = len;
    a.nch = (len + 64 + CH_LEN - 1) / CH_LEN;
    a.dec_stride = P3_DEC_STRIDE;
    return a;
}

constexpr size_t VITC_EMIT_SMEM = (size_t)VITC_EMIT_WARPS * VITC_EMIT_STEPS * sizeof(uint2);

// input_reset for a range of streams (reference src/input.c:126-138)
__global__ void k_reset(DevPtrs p, EngineDims d, int only)
{
    const int s = blockIdx.x, t = threadIdx.x;
    if (only >= 0 && s != only) return;
    for (int i = t; i < NFFT; i += blockDim.x) {
        p.cfreq[(size_t)s * NFFT + i] = 0.f;
        p.cphase[(size_t)s * NFFT + i] = 0.f;
    }
    if (t == 0) {
        StreamState &st = p.st[s];
        const long long avail = st.in_avail;
        StreamState z;
        memset(&z, 0, sizeof(z));
        z.phase = make_float2(1.0f, 0.0f);
        z.psmi = 1;
        z.state = ST_NONE;
        z.force_state = -1;
        z.in_avail = only == -2 ? avail : 0;     // -2: keep the attached input (rewind)
        st = z;
    }
}

// ---------------------------------------------------------------------------
// stage kernels for the parity tests
// ---------------------------------------------------------------------------
__global__ void k_viterbi_test(const int8_t *in, uint8_t *out, uint2 *dec, int len)
{
    const int f = blockIdx.x, t = threadIdx.x;
    const int8_t *vin = in + (size_t)f * 3 * len;
    uint2 *dd = dec + (size_t)f * (len + 64);
    int state = viterbi_forward(vin, len, dd, t);
    __syncwarp();
    if (t == 0) {
        uint8_t *o = out + (size_t)f * len;
        for (int q = len + 63; q >= 0; q--) {
            if (q >= 32 && q < 32 + len) o[q - 32] = (uint8_t)((state >> 5) & 1);
            state = vit_prev(state, dd[q]);
        }
    }
}

// ===========================================================================
// AM (hybrid MA1): one warp per stream runs the chain of am.cuh over every complete 33-symbol window
// ===========================================================================
// every lane of k_am's warp holds the same 96 header bytes (am.cuh computes them redundantly) and all call this together
struct AmFixHeader {
    const GfTab *gf;
    __host__ __device__ int operator()(uint8_t *pdu) const
    {
#if defined(__CUDA_ARCH__) || defined(NB_EMU)
        return rs8_fix_header_warp(*gf, pdu, (int)(threadIdx.x & 31));
#else
        (void)pdu;
        return 1;
#endif
    }
};

__global__ void __launch_bounds__(nbam::AM_THREADS) k_am(DevPtrs p, EngineDims d, nbam::AmState *ast, nbam::AmWork *aw,
                                                         const nbam::AmTables *tb, int max_blocks, int last_pass)
{
    const int s = blockIdx.x;
#if defined(NB_EMU)
    unsigned char *am_smem_raw = emu::dyn_smem();
#else
    extern __shared__ __align__(16) unsigned char am_smem_raw[];     // sizeof(nbam::AmSmem) bytes (above the 48 KB a static array may have)
#endif
    nbam::AmSmem &sm = *reinterpret_cast<nbam::AmSmem *>(am_smem_raw);
    __shared__ GfTab gf;
    const nbam::Lanes L = { (int)threadIdx.x, nbam::AM_THREADS, &sm, g_dbg };
    gf_tab_load(gf, (int)threadIdx.x, nbam::AM_THREADS);
    __syncthreads();
    StreamState &fs = p.st[s];
    nbam::AmState st = ast[s];                             // every thread's own copy of the receiver's scalars
    st.log_len = fs.log_len;                               // the host rewinds the log when it drains it ...
    st.log_overflow = fs.log_overflow;                     // ... and takes the overflow flag with it
    st.l2_on = d.l2;
    st.l2_n = 0;
    static_assert(nbam::AM_L2_QUEUE <= L2_QUEUE, "the L2 kernel reads the queue from StreamState");
    const nbam::AmIo io = { reinterpret_cast<const int16_t *>(p.iq + (size_t)s * d.in_stride), p.log + (size_t)s * d.log_cap,
                            (unsigned)d.log_cap };
    int nb_done = 0;
    __shared__ long long sh_avail;
    for (; nb_done < max_blocks; nb_done++) {
        // the sample count can grow while the kernel runs (asynchronous pushes): one thread reads it for the whole CTA
        if (threadIdx.x == 0) sh_avail = *reinterpret_cast<volatile long long *>(&fs.in_avail) / 2;    // cs16 complex samples
        __syncthreads();
        const long long avail = sh_avail;
        if (avail < st.start + nbam::NACQ) break;
        nbam::process_window(st, aw[s], *tb, io, L, AmFixHeader{ &gf });
        __syncthreads();
    }
    __syncthreads();
    if (L.lane == 0) {
        ast[s] = st;
        fs.log_len = st.log_len;
        if (st.log_overflow) fs.log_overflow = 1;
        fs.blocks_done = st.blocks_done;
        fs.start = st.start;
        fs.state = st.state;
        fs.l2_n = st.l2_n;                                 // k_l2 follows this launch (launch_pass)
        for (int i = 0; i < st.l2_n; i++) {
            fs.l2_off[i] = aw[s].l2_off[i];
            fs.l2_lc[i] = aw[s].l2_lc[i];
            fs.l2_nbits[i] = aw[s].l2_nbits[i];
        }
        if (nb_done) atomicAdd(&p.ctl->progress, (unsigned long long)nb_done);
        StreamBrief b;
        b.start = st.start;
        b.state = st.state;
        b.bc = 0;
        b.p1_ready = 0;
        b.pad_ = 0;
        p.brief[s] = b;
        const long long avail = *reinterpret_cast<volatile long long *>(&fs.in_avail) / 2;
        if (last_pass && avail >= st.start + nbam::NACQ) atomicAdd(&p.ctl->more, 1u);
    }
}

// AM cu8 input (input_push_cu8 in AM mode, reference src/input.c:52-117): one tile of nbam::DEC_T cs16 outputs per
// CTA, computed from the stream's raw cu8 ring (am.cuh: decim_tile).  Launched on the copy stream behind the
// copy that delivered the raw samples; the new sample count is published after it.
__global__ void __launch_bounds__(256) k_am_decim(const uint8_t *ring, unsigned ring_bytes, long long raw_avail, long long k0,
                                                  int nout, short2 *out)
{
    __shared__ nbam::DecimScratch sc;
    const int first = (int)blockIdx.x * nbam::DEC_T;
    const int n = min(nbam::DEC_T, nout - first);
    nbam::decim_tile(ring, ring_bytes, raw_avail, k0 + first, n, out + first, sc, nbam::Lanes{ (int)threadIdx.x, (int)blockDim.x });
}

__global__ void k_rs_test(uint8_t *blocks, int *rc, int n)        // one warp per codeword
{
    __shared__ GfTab gf;
    gf_tab_load(gf, (int)threadIdx.x, (int)blockDim.x);
    __syncthreads();
    const int i = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= n) return;
    const int r = rs8_decode_warp(gf, blocks + (size_t)i * 255, lane);
    if (lane == 0) rc[i] = r;
}

// stage entry point: the AM decoder (am.cuh: viterbi_k9_warp + viterbi_k9_traceback) on `njobs` independent tail-biting
// frames of `len` bits, one CTA each; rounds[j] = repair rounds the segmented traceback needed
__global__ void __launch_bounds__(nbam::AM_THREADS) k_am_vit_test(const int8_t *in, uint8_t *out, uint32_t *dec, size_t dec_words, int len,
                                                                  unsigned g0, unsigned g1, unsigned g2, int warmup, int chunk_warmup, int *rounds)
{
#if defined(__CUDA_ARCH__)                                                    // (the decoder's device branch does not exist in the host pass)
#if defined(NB_EMU)
    unsigned char *vit_test_smem = emu::dyn_smem();
#else
    extern __shared__ __align__(16) unsigned char vit_test_smem[];    // AmVitSlot + AmVitRows
#endif
    nbam::AmVitSlot *vit = reinterpret_cast<nbam::AmVitSlot *>(vit_test_smem);
    nbam::AmVitRows &rows = *reinterpret_cast<nbam::AmVitRows *>(vit_test_smem + nbam::VIT_TEST_SLOTS_BYTES);
    const int j = blockIdx.x, t = threadIdx.x;
    uint32_t *decw = dec + (size_t)j * dec_words;
    const long long c0 = clock64();
    const int redone = nbam::viterbi_k9_forward(vit, decw, t, in + (size_t)j * 3 * len, len, g0, g1, g2, chunk_warmup);
    const long long c1 = clock64();
    const int r = nbam::viterbi_k9_traceback(vit[0], rows, decw, t, out + (size_t)j * len, len, warmup);
    if (t == 0) {
        rounds[j] = r | (redone << 16);
        if (g_dbg & 8) printf("k9 job %d: recursion %lld cycles (%d chunks again), traceback %lld cycles, %d repair rounds\n", j, c1 - c0, redone, clock64() - c1, r);
    }
#endif
}

// ===========================================================================
// L2 framing (l2.cuh): the last kernel of a pass.  One CTA per stream walks the frames (and frame_resets) k_stream
// queued, in the reference's call order, and appends one REC_L2 record per frame to the stream's log.
// ===========================================================================
__global__ void __launch_bounds__(nbl2::L2_THREADS) k_l2(DevPtrs p, EngineDims d, nbl2::L2State *l2)
{
    const int s = blockIdx.x;
    StreamState &st = p.st[s];
    const int n = st.l2_n;
    if (n == 0) return;
    uint8_t *base = p.log + (size_t)s * d.log_cap;
    const nbl2::L2Sink sink = { base, d.log_cap, &st.log_len, &st.log_overflow };
    for (int e = 0; e < n; e++) {
        const unsigned off = st.l2_off[e], nbits = st.l2_nbits[e];
        if (nbits == 0) {
            if (threadIdx.x == 0) nbl2::l2_reset(l2[s]);
            __syncthreads();
        } else if (off != 0xffffffffu) {
            nbl2::l2_frame(l2[s], base + off, nbits, st.l2_lc[e], off, sink);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) st.l2_n = 0;
}

// state of a stream's L2 as the reference has it after calloc + frame_init (frame.c:744-749)
__global__ void k_l2_init(nbl2::L2State *l2, int only)
{
    const int s = blockIdx.x;
    if (only >= 0 && s != only) return;
    uint32_t *w = reinterpret_cast<uint32_t *>(l2 + s);
    static_assert(sizeof(nbl2::L2State) % 4 == 0, "word-wise clear");
    for (size_t i = threadIdx.x; i < sizeof(nbl2::L2State) / 4; i += blockDim.x) w[i] = 0;
    __syncthreads();
    if (threadIdx.x == 0) nbl2::l2_reset(l2[s]);
}

// End of an asynchronous batch (nrsc5b_submit): every stream's records go to page-locked host memory the device
// writes directly (16 bytes per store), with a header saying how many; the device log is rewound.  The host reads
// them when the batch's event has fired - no sized device->host copy, no round trip for the sizes.
struct ExportHdr {
    unsigned log_len, log_overflow;
};

__global__ void __launch_bounds__(256) k_export(DevPtrs p, EngineDims d, uint8_t *host_log, size_t host_stride, ExportHdr *hdr)
{
    const int s = blockIdx.x, t = threadIdx.x;
    StreamState &st = p.st[s];
    const unsigned n = st.log_len;
    const uint4 *src = reinterpret_cast<const uint4 *>(p.log + (size_t)s * d.log_cap);
    uint4 *dst = reinterpret_cast<uint4 *>(host_log + (size_t)s * host_stride);
    for (unsigned i = t; i < (n + 15) / 16; i += blockDim.x) dst[i] = src[i];
    __syncthreads();
    if (t == 0) {
        hdr[s].log_len = n;
        // (a frame whose record is reserved but not decoded yet would leave as a hole: the host plans a decode group
        // into every pass that can complete a frame, so this cannot happen - if it does, say so instead of shipping it)
        hdr[s].log_overflow = st.log_overflow | (st.p1_ready ? 2u : 0u);
        st.log_len = 0;
        st.log_overflow = 0;
        __threadfence_system();
    }
}

// stage entry point: a list of frames (desc: offset into `frames`, lc, nbits; nbits == 0 = frame_reset) through one
// stream's L2, records into out[cap]
__global__ void __launch_bounds__(nbl2::L2_THREADS) k_l2_test(nbl2::L2State *l2, const uint8_t *frames, const uint32_t *desc,
                                                               int ndesc, uint8_t *out, size_t cap, unsigned *len_ovf)
{
    const nbl2::L2Sink sink = { out, cap, len_ovf, len_ovf + 1 };
    for (int e = 0; e < ndesc; e++) {
        const unsigned off = desc[3 * e], lc = desc[3 * e + 1], nbits = desc[3 * e + 2];
        if (nbits == 0) {
            if (threadIdx.x == 0) nbl2::l2_reset(*l2);
            __syncthreads();
        } else {
            nbl2::l2_frame(*l2, frames + off, nbits, lc, (unsigned)e, sink);
        }
    }
}

}  // namespace nb

// ===========================================================================
// host side
// ===========================================================================
using namespace nb;

static size_t vitc_emit_smem() { return VITC_EMIT_SMEM; }

#define CK(x)                                                                                      \
    do {                                                                                           \
        cudaError_t e_ = (x);                                                                      \
        if (e_ != cudaSuccess) {                                                                   \
            fprintf(stderr, "nrsc5_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
            return NRSC5B_ECUDA;                                                                   \
        }                                                                                          \
    } while (0)


// Page-locked host buffers come from a small process-wide pool: cudaMallocHost / cudaFreeHost cost about a millisecond
// each, and a handle that is opened and closed per capture (the drop-in: nrsc5_open_pipe ... nrsc5_close) would pay for a
// dozen of them inside its close.  Buffers go back to the pool when an engine is destroyed and are handed to the next
// engine that asks for the same size.
#include <map>
#include <mutex>
static std::mutex g_pin_mu;
static std::multimap<size_t, void *> g_pin_free;
static std::map<void *, size_t> g_pin_size;

static cudaError_t pinned_alloc(void **out, size_t n)
{
    {
        std::lock_guard<std::mutex> lk(g_pin_mu);
        auto it = g_pin_free.find(n);
        if (it != g_pin_free.end()) {
            *out = it->second;
            g_pin_free.erase(it);
            return cudaSuccess;
        }
    }
    const cudaError_t rc = cudaMallocHost(out, n);
    if (rc == cudaSuccess) {
        std::lock_guard<std::mutex> lk(g_pin_mu);
        g_pin_size[*out] = n;
    }
    return rc;
}

static void pinned_release(void *p)
{
    if (!p) return;
    std::lock_guard<std::mutex> lk(g_pin_mu);
    auto it = g_pin_size.find(p);
    if (it != g_pin_size.end()) g_pin_free.insert({ it->second, p });
}

struct nrsc5b_engine {
    nrsc5b_config_t cfg;
    EngineDims dims;
    DevPtrs dp;
    cudaStream_t stream;
    cudaStream_t copy_stream;          // host->device input copies overlap with compute on `stream`
    uint8_t *iq_owned;                 // engine-owned cu8 buffer (null when attached)
    std::vector<long long> pushed;     // complex cu8 samples pushed per stream
    std::vector<unsigned> drained;     // log bytes already handed out per stream
    std::vector<uint8_t> overflowed;   // a drain found this stream's log truncated (until nrsc5b_take_overflow)
    uint8_t *trim_scratch;             // bounce buffer of trim_stream (allocated on first use)
    uint8_t *pinned;                   // staging for pushes
    size_t pinned_cap;
    cudaEvent_t pinned_free;
    long long *avail_rows;             // pinned, 16 x S entries (nrsc5b_push_cu8_all), allocated on first use
    unsigned avail_rows_pos;
    long long *avail_ring;             // pinned, 4096 entries
    unsigned avail_pos;
    cudaEvent_t reset_done;            // copy stream waits for resets issued on the compute stream
    cudaEvent_t fence[64];             // push fences (nrsc5b_push_fence), created on first use
    unsigned fence_next;
    StreamState *h_state;              // pinned mirror for read-back
    nrsc5b_stats_t stats;
    unsigned long long last_progress;
    // host-side planning of the passes (plan_passes): the device's control words and per-stream briefs, read back
    // into page-locked memory behind every batch
    EngineCtl *h_ctl;
    StreamBrief *h_brief;
    // asynchronous batches (nrsc5b_submit / nrsc5b_poll): records exported into page-locked host memory
    uint8_t *xlog;                     // [S][xlog_stride], page-locked, written by k_export
    size_t xlog_stride;
    ExportHdr *xhdr;                   // [S], page-locked
    cudaEvent_t batch_done;
    bool in_flight, batch_decoded;
    bool stalled;                      // the last batch moved no stream although the host's count said it could: no new
    long long stalled_units;           // batch until more samples have arrived (guards the caller's flush loop)
    // staged input (nrsc5b_stage_cu8 / _cs16): pushes land in page-locked memory and go to the device in one copy
    // per stream when a batch is submitted
    struct Staged { int stream; size_t off, n; };
    uint8_t *stage[2];
    size_t stage_cap, stage_fill;
    int stage_cur;
    cudaEvent_t stage_free[2];
    std::vector<Staged> staged;
    std::vector<uint8_t> carry;            // samples of a staging call that found the device buffer full (NRSC5B_EFULL)
    int carry_stream;
    std::vector<long long> staged_units;   // per stream: staged 2-byte units not yet counted in `pushed`
    std::vector<uint8_t> unpublished;      // per stream: samples copied to the device whose count the kernels have not been told
    bool direct_push;                      // a push outside the staging area since the last batch (its count is published at once)
    // NRSC5_B200_TRACE=1: where the host side of the asynchronous path spends its time (printed by nrsc5b_destroy)
    struct Trace {
        unsigned long long batches, passes, decode_passes, flushes, trims, polls_ready, submits_idle;
        double s_flush, s_trim, s_stage_wait, s_submit, s_poll_wait;
    } tr;
    bool trace_on;
    std::vector<void *> allocs;
    int v64_ch;                        // chunk length of the fast P1 Viterbi (chosen from the stream count)
    nbam::AmState *am_st;              // AM mode: per-stream state, work arrays, tables
    nbam::AmWork *am_work;
    nbam::AmTables *am_tb;
    uint8_t *am_ring;                  // AM with cu8 input: per-stream ring of raw samples ahead of the /32 decimator
    unsigned am_ring_bytes;            // bytes per stream, a power of two
    std::vector<long long> am_raw_bytes, am_dec_out;   // raw bytes received / cs16 samples produced per stream
    nbl2::L2State *l2;                 // L2 on the device (nrsc5b_enable_l2): per-stream state, null until enabled
    int profiling;
    cudaEvent_t pev[5];
    double kernel_ms[4];
    unsigned long long kernel_n[4];
};

static const float k_bp_coeff[32] = {
    -0.000685643230099231f, 0.005636964458972216f, 0.009015781804919243f, -0.015486305579543114f,
    -0.035108357667922974f, 0.017446253448724747f, 0.08155813068151474f, 0.007995186373591423f,
    -0.13311293721199036f, -0.0727422907948494f, 0.15914097428321838f, 0.16498781740665436f,
    -0.1324498951435089f, -0.2484012246131897f, 0.051773931831121445f, 0.2821577787399292f,
    0.051773931831121445f, -0.2484012246131897f, -0.1324498951435089f, 0.16498781740665436f,
    0.15914097428321838f, -0.0727422907948494f, -0.13311293721199036f, 0.007995186373591423f,
    0.08155813068151474f, 0.017446253448724747f, -0.035108357667922974f, -0.015486305579543114f,
    0.009015781804919243f, 0.005636964458972216f, -0.000685643230099231f, 0.0f
};

static int upload_tables(int device)
{
    static int done_for = -1;
    if (done_for == device) return 0;
    uint8_t ex[256], lg[256];
    unsigned v = 1;
    lg[0] = 255;
    ex[255] = 0;
    for (int i = 0; i < 255; i++) {
        ex[i] = (uint8_t)v;
        lg[v] = (uint8_t)i;
        v <<= 1;
        if (v & 0x100) v ^= 0x11d;
    }
    CK(cudaMemcpyToSymbol(c_gf_exp, ex, 256));
    CK(cudaMemcpyToSymbol(c_gf_log, lg, 256));
    static const int compat[64] = {
        0, 1, 2, 3, 1, 5, 6, 5, 6, 1, 2, 11, 1, 5, 6, 5, 6, 1, 2, 3, 1, 5, 6, 5, 6, 1, 2, 11, 1, 5, 6, 5,
        6, 1, 2, 3, 1, 5, 6, 5, 6, 1, 2, 11, 1, 5, 6, 5, 6, 1, 2, 3, 1, 5, 6, 5, 6, 1, 2, 11, 1, 5, 6, 5
    };
    CK(cudaMemcpyToSymbol(c_compat_mode, compat, sizeof(compat)));
    short taps[32];
    for (int i = 0; i < 32; i++) taps[i] = (short)(k_bp_coeff[31 - i] * 32767.0f);
    CK(cudaMemcpyToSymbol(c_bp_tap, taps, sizeof(taps)));
    unsigned pn80[3] = { 0, 0, 0 }, reg = 0x3ff;       // descrambler LFSR (reference src/decode.c:279-294)
    for (int i = 0; i < 80; i++) {
        const unsigned b = ((reg >> 9) ^ reg) & 1;
        reg |= b << 11;
        reg >>= 1;
        pn80[i >> 5] |= b << (i & 31);
    }
    CK(cudaMemcpyToSymbol(c_pn80, pn80, sizeof(pn80)));
    done_for = device;
    return 0;
}

template <typename T>
static int dev_alloc(nrsc5b_engine *e, T **ptr, size_t count, bool zero = true)
{
    void *q = nullptr;
    if (cudaMalloc(&q, count * sizeof(T)) != cudaSuccess) return NRSC5B_ENOMEM;
    if (zero && cudaMemset(q, 0, count * sizeof(T)) != cudaSuccess) return NRSC5B_ECUDA;
    e->allocs.push_back(q);
    *ptr = reinterpret_cast<T *>(q);
    return 0;
}

static std::vector<float2> make_twiddles()
{
    // fft.cuh layout: tw1[k1*128 + t] = W^(t*k1), then tw2[k2*8 + n3] = W^(16*n3*k2)
    std::vector<float2> tw(FFT_TW);
    auto w = [](int m) {
        double a = -2.0 * M_PI * (double)(m % NFFT) / (double)NFFT;
        return make_float2((float)cos(a), (float)sin(a));
    };
    for (int k1 = 0; k1 < 16; k1++)
        for (int t = 0; t < 128; t++) tw[k1 * 128 + t] = w(t * k1);
    for (int k2 = 0; k2 < 16; k2++)
        for (int n3 = 0; n3 < 8; n3++) tw[FFT_TW1 + k2 * 8 + n3] = w(16 * n3 * k2);
    return tw;
}

static void init_state_host(StreamState &st)
{
    memset(&st, 0, sizeof(st));
    st.phase = make_float2(1.0f, 0.0f);
    st.psmi = 1;
    st.state = ST_NONE;
    st.force_state = -1;
}

static void launch_k_stream(nrsc5b_engine *e, int last_pass);

extern "C" int nrsc5b_debug_set(int flags);

extern "C" const char *nrsc5b_version(void) { return "nrsc5_b200 0.1 (sm_90a)"; }

extern "C" int nrsc5b_create(nrsc5b_engine_t **out, const nrsc5b_config_t *cfg)
{
    if (!out || !cfg || cfg->nstreams <= 0 || (cfg->mode != NRSC5B_MODE_FM && cfg->mode != NRSC5B_MODE_AM)) return NRSC5B_EINVAL;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || cfg->device >= ndev) {
        fprintf(stderr, "nrsc5_b200: no usable CUDA device (the engine has no CPU path)\n");
        return NRSC5B_ENODEV;
    }
    if (cudaSetDevice(cfg->device) != cudaSuccess) return NRSC5B_ENODEV;
    nrsc5b_engine *e = new (std::nothrow) nrsc5b_engine();
    if (!e) return NRSC5B_ENOMEM;
    e->cfg = *cfg;
    e->stream = 0;
    e->copy_stream = nullptr;
    e->iq_owned = nullptr;
    e->trim_scratch = nullptr;
    e->am_st = nullptr;
    e->am_work = nullptr;
    e->am_tb = nullptr;
    e->am_ring = nullptr;
    e->am_ring_bytes = 0;
    e->avail_rows = nullptr;
    e->avail_rows_pos = 0;
    for (int i = 0; i < 64; i++) e->fence[i] = nullptr;
    e->fence_next = 0;
    e->stats = nrsc5b_stats_t{};
    e->last_progress = 0;
    e->h_ctl = nullptr; e->h_brief = nullptr;
    e->xlog = nullptr; e->xlog_stride = 0; e->xhdr = nullptr; e->batch_done = nullptr; e->in_flight = false; e->batch_decoded = false; e->stalled = false; e->stalled_units = 0;
    e->stage[0] = e->stage[1] = nullptr; e->stage_cap = 0; e->stage_fill = 0; e->stage_cur = 0;
    e->stage_free[0] = e->stage_free[1] = nullptr;
    e->profiling = 0;
    for (int i = 0; i < 5; i++) e->pev[i] = nullptr;
    for (int i = 0; i < 4; i++) { e->kernel_ms[i] = 0; e->kernel_n[i] = 0; }
    e->pinned = nullptr; e->h_state = nullptr; e->pinned_free = nullptr; e->avail_ring = nullptr; e->avail_pos = 0; e->reset_done = nullptr;
    const int S = cfg->nstreams;
    if (const char *dbg = getenv("NRSC5_B200_DBG")) nrsc5b_debug_set(atoi(dbg));      // kernel experiment switches (A/B runs)
    e->dims.nstreams = S;
    e->dims.in_stride = (cfg->input_capacity + 63) & ~(size_t)63;
    e->dims.log_cap = cfg->log_capacity ? ((cfg->log_capacity + 15) & ~(size_t)15) : (1u << 20);
    e->dims.emit_soft = cfg->emit_soft;
    e->dims.cs16 = cfg->input_cs16 ? 1 : 0;
    e->dims.px_enabled = 0;
    e->pushed.assign(S, 0);
    e->staged_units.assign(S, 0);
    e->unpublished.assign(S, 0);
    e->direct_push = false;
    e->tr = {};
    e->trace_on = getenv("NRSC5_B200_TRACE") != nullptr;
    e->drained.assign(S, 0);
    e->overflowed.assign(S, 0);
    int rc = upload_tables(cfg->device);
    if (rc) { delete e; return rc; }

    DevPtrs &dp = e->dp;
    memset(&dp, 0, sizeof(dp));
#define DA(field, type, count)                                              \
    do {                                                                    \
        type *tmp_ = nullptr;                                               \
        rc = dev_alloc(e, &tmp_, (count));                                  \
        if (rc) { nrsc5b_destroy(e); return rc; }                           \
        dp.field = tmp_;                                                    \
    } while (0)
    if (e->dims.in_stride) {
        uint8_t *tmp = nullptr;
        rc = dev_alloc(e, &tmp, (size_t)S * e->dims.in_stride + 64, false);
        if (rc) { nrsc5b_destroy(e); return rc; }
        cudaMemset(tmp, 0x7f, (size_t)S * e->dims.in_stride + 64);
        e->iq_owned = tmp;
        dp.iq = tmp;
    }
    DA(ctl, EngineCtl, 1);
    DA(brief, StreamBrief, S);
    DA(st, StreamState, S);
    DA(cfreq, float, (size_t)S * NFFT);
    DA(cphase, float, (size_t)S * NFFT);
    DA(nco, float2, (size_t)S * NSYM);
    DA(bins, float2, (size_t)S * BLK * NBINS);
    DA(pm, int8_t, (size_t)S * 16 * PM_BLOCK);
    DA(ydec, short2, (size_t)S * NACQ);
    DA(acq_sums, float2, (size_t)S * NSYM);
    DA(tbuf, float2, (size_t)S * NACQ);
    DA(vit_in, int8_t, (size_t)S * P1_VIT);
    DA(vit_dec, uint2, (size_t)S * P1_NCH * CH_LEN);
    DA(vspec, uint2, (size_t)S * P1_NCH * 16);
    DA(vend, uint2, (size_t)S * P1_NCH * 16);
    DA(tbend, int, (size_t)S * P1_NCH);
    DA(hstate, int, (size_t)S * P1_NCH);
    DA(p1_bits, uint32_t, (size_t)S * (P1_LEN / 32));
    {
        // fast Viterbi: one thread per chunk; pick the chunk length so that the warps of all streams' frames
        // make one wave over the GPU's warp schedulers (4 per SM)
        int sms = 132;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg->device);
        int wpf = (4 * sms) / S;
        if (wpf < 1) wpf = 1;
        if (wpf > 18) wpf = 18;
        int ch = (P1_STEPS + 32 * wpf - 1) / (32 * wpf);
        ch = (ch + 31) & ~31;
        if (ch < 256) ch = 256;
        e->v64_ch = ch;
        const size_t nch = (size_t)(P1_STEPS + ch - 1) / ch;
        DA(v64_spec, uint32_t, (size_t)S * nch * 32);
        DA(v64_end, uint32_t, (size_t)S * nch * 32);
        DA(v64_endstate, int, (size_t)S);
    }
    DA(px_ring[0], int8_t, (size_t)S * PX_RING);
    DA(px_ring[1], int8_t, (size_t)S * PX_RING);
    DA(log, uint8_t, (size_t)S * e->dims.log_cap);
    if (cfg->mode == NRSC5B_MODE_AM) {
        rc = dev_alloc(e, &e->am_st, (size_t)S);
        if (!rc) rc = dev_alloc(e, &e->am_work, (size_t)S);
        if (!rc) rc = dev_alloc(e, &e->am_tb, 1);
        if (rc) { nrsc5b_destroy(e); return rc; }
        nbam::AmTables *tb = new nbam::AmTables;
        if (!rc && !cfg->input_cs16) {                      // cu8 at 1 488 375 S/s: decimated by 32 on arrival
            e->am_ring_bytes = 1u << 20;
            rc = dev_alloc(e, &e->am_ring, (size_t)S * e->am_ring_bytes);
            if (rc) { delete tb; nrsc5b_destroy(e); return rc; }
            e->am_raw_bytes.assign(S, 0);
            e->am_dec_out.assign(S, 0);
        }
        nbam::am_fill_tables(*tb);
        cudaMemcpy(e->am_tb, tb, sizeof(*tb), cudaMemcpyHostToDevice);
        delete tb;
    }
    {
        // tables
        std::vector<float> shape(NSYM);
        for (int i = 0; i < NSYM; i++) {
            if (i < NCP) shape[i] = sinf(M_PI / 2 * i / NCP);
            else if (i < NFFT) shape[i] = 1;
            else shape[i] = cosf(M_PI / 2 * (i - NFFT) / NCP);
        }
        float *dshape = nullptr;
        rc = dev_alloc(e, &dshape, NSYM);
        if (rc) { nrsc5b_destroy(e); return rc; }
        cudaMemcpy(dshape, shape.data(), NSYM * sizeof(float), cudaMemcpyHostToDevice);
        dp.shape = dshape;
        std::vector<float2> tw = make_twiddles();
        float2 *dtw = nullptr;
        rc = dev_alloc(e, &dtw, FFT_TW);
        if (rc) { nrsc5b_destroy(e); return rc; }
        cudaMemcpy(dtw, tw.data(), FFT_TW * sizeof(float2), cudaMemcpyHostToDevice);
        dp.twid = dtw;
        static const int PMV[20] = { 10, 2, 18, 6, 14, 8, 16, 0, 12, 4, 11, 3, 19, 7, 15, 9, 17, 1, 13, 5 };
        std::vector<uint32_t> lut(P1_ENC);
        for (unsigned i = 0; i < (unsigned)P1_ENC; i++) {
            unsigned part = (unsigned)PMV[i % 20];
            unsigned block = (i / 20 + part * 7) % 16;
            unsigned k = i / 320;
            unsigned row = (k * 11) % 32, col = (k * 11 + k / 288) % 36;
            lut[i] = (block * 32 + row) * 720 + part * 36 + col;
        }
        {
            uint16_t src[320];
            for (int w = 0; w < 320; w++) {
                const int part = PMV[w % 20], blk = (w / 20 + 7 * part) % 16;
                src[w] = (uint16_t)(blk * 720 + part * 36);
            }
            cudaMemcpyToSymbol(c_p1_src, src, sizeof(src));
        }
        {
            // interleaver IV (decode.c:344-376, MP3/MP11: J=4, B=32, C=36, M=2): output m reads internal[A(m)]
            // before input m is stored at internal[m]; as a delay: m - A(m) if A(m) < m, else one span more
            std::vector<uint32_t> dl(IV_N);
            unsigned pt[4] = { 0, 0, 0, 0 };
            for (unsigned m = 0; m < (unsigned)IV_N; m++) {
                const unsigned part = (m / 2) % 4, pti = pt[part]++;
                const unsigned block = (pti + part * 7 - 1151 * (pti / 1152)) % 32;
                const unsigned row = ((11 * pti) % 1152) / 36, col = (pti * 11) % 36;
                const unsigned A = (block * 32 + row) * 144 + part * 36 + col;
                dl[m] = A < m ? m - A : m - A + IV_N;
            }
            uint32_t *ddl = nullptr;
            rc = dev_alloc(e, &ddl, IV_N);
            if (rc) { nrsc5b_destroy(e); return rc; }
            cudaMemcpy(ddl, dl.data(), dl.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
            dp.iv_delay = ddl;
            // MP2 (frame length 2304): J=2, M=4, span 73728, partition = ((m + 2) / 4) % 2
            std::vector<uint32_t> ds(IV_NS);
            unsigned pts[2] = { 0, 0 };
            for (unsigned m = 0; m < (unsigned)IV_NS; m++) {
                const unsigned part = ((m + 2) / 4) % 2, pti = pts[part]++;
                const unsigned block = (pti + part * 7 - 1151 * (pti / 1152)) % 32;
                const unsigned row = ((11 * pti) % 1152) / 36, col = (pti * 11) % 36;
                const unsigned A = (block * 32 + row) * 72 + part * 36 + col;
                ds[m] = A < m ? m - A : m - A + IV_NS;
            }
            uint32_t *dds = nullptr;
            rc = dev_alloc(e, &dds, IV_NS);
            if (rc) { nrsc5b_destroy(e); return rc; }
            cudaMemcpy(dds, ds.data(), ds.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
            dp.iv_delay_s = dds;
        }
        uint32_t *dlut = nullptr;
        rc = dev_alloc(e, &dlut, P1_ENC);
        if (rc) { nrsc5b_destroy(e); return rc; }
        cudaMemcpy(dlut, lut.data(), P1_ENC * sizeof(uint32_t), cudaMemcpyHostToDevice);
        dp.p1_lut = dlut;
        std::vector<uint8_t> pn(P1_LEN);
        unsigned reg = 0x3ff;
        for (int i = 0; i < P1_LEN; i++) {
            unsigned b = ((reg >> 9) ^ reg) & 1;
            reg |= b << 11;
            reg >>= 1;
            pn[i] = (uint8_t)b;
        }
        uint8_t *dpn = nullptr;
        rc = dev_alloc(e, &dpn, P1_LEN);
        if (rc) { nrsc5b_destroy(e); return rc; }
        cudaMemcpy(dpn, pn.data(), P1_LEN, cudaMemcpyHostToDevice);
        dp.pn = dpn;
        std::vector<uint32_t> pnw(P1_LEN / 32, 0u);
        for (int i = 0; i < P1_LEN; i++) pnw[i >> 5] |= (uint32_t)pn[i] << (i & 31);
        uint32_t *dpnw = nullptr;
        rc = dev_alloc(e, &dpnw, P1_LEN / 32);
        if (rc) { nrsc5b_destroy(e); return rc; }
        cudaMemcpy(dpnw, pnw.data(), pnw.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
        dp.pnw = dpnw;
        {
            uint32_t sp[256];
            for (int v = 0; v < 256; v++) {
                sp[v] = 0;
                for (int k = 0; k < 8; k++) sp[v] |= (uint32_t)((v >> k) & 1) << (3 * k);
            }
            cudaMemcpyToSymbol(c_spread3, sp, sizeof(sp));
        }
    }
#undef DA
    e->pinned_cap = 8u << 20;
    if (cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking) != cudaSuccess) { nrsc5b_destroy(e); return NRSC5B_ECUDA; }
    if (pinned_alloc((void **)&e->pinned, e->pinned_cap) != cudaSuccess ||
        pinned_alloc((void **)&e->h_state, sizeof(StreamState) * S) != cudaSuccess ||
        pinned_alloc((void **)&e->avail_ring, sizeof(long long) * 4096) != cudaSuccess ||
        pinned_alloc((void **)&e->h_ctl, sizeof(EngineCtl)) != cudaSuccess ||
        pinned_alloc((void **)&e->h_brief, sizeof(StreamBrief) * S) != cudaSuccess ||
        cudaEventCreateWithFlags(&e->batch_done, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&e->reset_done, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&e->pinned_free, cudaEventDisableTiming) != cudaSuccess) {
        nrsc5b_destroy(e);
        return NRSC5B_ENOMEM;
    }
    if (cudaFuncSetAttribute(k_stream<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FrontSmem)) != cudaSuccess ||
        cudaFuncSetAttribute(k_stream<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FrontSmem)) != cudaSuccess ||
        cudaFuncSetAttribute(k_am, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(nbam::AmSmem)) != cudaSuccess ||
        cudaFuncSetAttribute(k_vitc_emit, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vitc_emit_smem()) != cudaSuccess ||
        cudaFuncSetAttribute(k_v64_emit, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)V64_EMIT_SMEM) != cudaSuccess) {
        nrsc5b_destroy(e);
        return NRSC5B_ECUDA;
    }
    e->dims.cluster = 1;
#if !defined(NB_EMU)
    if (cfg->mode == NRSC5B_MODE_FM) {
        // fewer streams than SMs: a cluster of 4 or 2 CTAs per stream shares the demodulation of every block
        int sms = 132;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg->device);
        const char *force = getenv("NRSC5_B200_CLUSTER");
        for (int c = 4; c >= 2; c >>= 1) {
            if (force ? atoi(force) != c : S * c > sms) continue;
            cudaLaunchConfig_t lc = {};
            lc.gridDim = dim3((unsigned)(S * c));
            lc.blockDim = dim3(FRONT_THREADS);
            lc.dynamicSmemBytes = sizeof(FrontSmem);
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeClusterDimension;
            at[0].val.clusterDim.x = (unsigned)c;
            at[0].val.clusterDim.y = 1;
            at[0].val.clusterDim.z = 1;
            lc.attrs = at;
            lc.numAttrs = 1;
            int nclusters = 0;
            if (cudaOccupancyMaxActiveClusters(&nclusters, k_stream<true>, &lc) == cudaSuccess && (force || nclusters >= S)) {
                e->dims.cluster = c;
                break;
            }
            cudaGetLastError();
        }
    }
#endif
    *out = e;
    rc = nrsc5b_reset(e, -1);
    if (rc == 0 && cudaDeviceSynchronize() != cudaSuccess) rc = NRSC5B_ECUDA;
#if !defined(NB_EMU)
    if (rc == 0 && e->dims.cluster > 1) {
        // trial launch (no input yet: every stream returns at once): a cluster shape the device refuses falls back to
        // one CTA per stream instead of failing later
        launch_k_stream(e, 0);
        if (cudaDeviceSynchronize() != cudaSuccess || cudaGetLastError() != cudaSuccess) {
            cudaGetLastError();
            fprintf(stderr, "nrsc5_b200: clusters of %d CTAs per stream not available here, using one CTA per stream\n", e->dims.cluster);
            e->dims.cluster = 1;
        }
    }
#endif
    if (rc) { nrsc5b_destroy(e); *out = nullptr; return rc; }
    return NRSC5B_OK;
}

extern "C" void nrsc5b_destroy(nrsc5b_engine_t *e)
{
    if (!e) return;
    cudaDeviceSynchronize();
    if (e->trace_on && e->h_state) {
        // SM cycles stream 0's k_stream spent per phase (device clock): what the GPU side of the wall time is made of
        if (cudaMemcpy(e->h_state, e->dp.st, sizeof(StreamState), cudaMemcpyDeviceToHost) == cudaSuccess) {
            const StreamState &z = e->h_state[0];
            fprintf(stderr, "nrsc5_b200 trace: stream 0 k_stream Mcycles {pids %.2f, prep_acq %.2f (%llu), prep_fine %.2f (%llu), demod %.2f (%llu), "
                            "sync_fine %.2f, sync_acq %.2f}, blocks %llu, frames %llu\n",
                    z.ph_cyc[0] * 1e-6, z.ph_cyc[1] * 1e-6, z.ph_n[1], z.ph_cyc[2] * 1e-6, z.ph_n[2], z.ph_cyc[3] * 1e-6, z.ph_n[3],
                    z.ph_cyc[4] * 1e-6, z.ph_cyc[5] * 1e-6, z.blocks_done, z.frames_done);
        }
    }
    if (e->trace_on)
        fprintf(stderr, "nrsc5_b200 trace: {\"batches\": %llu, \"passes\": %llu, \"decode_passes\": %llu, \"launches\": %llu, \"flushes\": %llu, "
                        "\"trims\": %llu, \"polls_ready\": %llu, \"submits_idle\": %llu, \"s_submit\": %.6f, \"s_flush\": %.6f, \"s_stage_wait\": %.6f, "
                        "\"s_trim\": %.6f, \"s_poll_wait\": %.6f, \"cluster\": %d}\n",
                e->tr.batches, e->tr.passes, e->tr.decode_passes, (unsigned long long)e->stats.kernel_launches, e->tr.flushes, e->tr.trims,
                e->tr.polls_ready, e->tr.submits_idle, e->tr.s_submit, e->tr.s_flush, e->tr.s_stage_wait, e->tr.s_trim, e->tr.s_poll_wait,
                e->dims.cluster);
    for (void *q : e->allocs) cudaFree(q);
    if (e->pinned) pinned_release(e->pinned);
    if (e->h_state) pinned_release(e->h_state);
    if (e->avail_ring) pinned_release(e->avail_ring);
    if (e->avail_rows) pinned_release(e->avail_rows);
    if (e->h_ctl) pinned_release(e->h_ctl);
    if (e->h_brief) pinned_release(e->h_brief);
    if (e->xlog) pinned_release(e->xlog);
    if (e->xhdr) pinned_release(e->xhdr);
    if (e->batch_done) cudaEventDestroy(e->batch_done);
    for (int i = 0; i < 2; i++) {
        if (e->stage[i]) pinned_release(e->stage[i]);
        if (e->stage_free[i]) cudaEventDestroy(e->stage_free[i]);
    }
    if (e->reset_done) cudaEventDestroy(e->reset_done);
    for (int i = 0; i < 64; i++) if (e->fence[i]) cudaEventDestroy(e->fence[i]);
    if (e->pinned_free) cudaEventDestroy(e->pinned_free);
    if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
    for (int i = 0; i < 5; i++) if (e->pev[i]) cudaEventDestroy(e->pev[i]);
    delete e;
}

extern "C" int nrsc5b_set_cuda_stream(nrsc5b_engine_t *e, void *cuda_stream)
{
    if (!e) return NRSC5B_EINVAL;
    e->stream = reinterpret_cast<cudaStream_t>(cuda_stream);
    return NRSC5B_OK;
}

extern "C" int nrsc5b_reset(nrsc5b_engine_t *e, int stream)
{
    if (!e || stream >= e->dims.nstreams) return NRSC5B_EINVAL;
    const int S = e->dims.nstreams;
    CK(cudaStreamSynchronize(e->copy_stream));       // no input copy of the old contents may still be in flight
    if (e->in_flight) {                              // an asynchronous batch: let it finish; its records are void
        CK(cudaEventSynchronize(e->batch_done));
        e->in_flight = false;
    }
    {
        std::vector<nrsc5b_engine::Staged> keep;
        for (const auto &g : e->staged)
            if (stream >= 0 && g.stream != stream) keep.push_back(g);
        e->staged.swap(keep);
    }
    k_reset<<<S, 256, 0, e->stream>>>(e->dp, e->dims, stream < 0 ? -1 : stream);
    if (e->l2) k_l2_init<<<S, 256, 0, e->stream>>>(e->l2, stream < 0 ? -1 : stream);
    CK(cudaEventRecord(e->reset_done, e->stream));
    CK(cudaStreamWaitEvent(e->copy_stream, e->reset_done, 0));
    e->stats.kernel_launches += 1;
    if (e->am_st) {
        nbam::AmState z;
        memset(&z, 0, sizeof(z));
        nbam::am_reset_state(z);
        for (int s = 0; s < S; s++) {
            if (stream >= 0 && s != stream) continue;
            CK(cudaMemcpyAsync(e->am_st + s, &z, sizeof(z), cudaMemcpyHostToDevice, e->stream));
            CK(cudaMemsetAsync(e->am_work + s, 0, sizeof(nbam::AmWork), e->stream));
        }
        CK(cudaStreamSynchronize(e->stream));              // `z` lives on this stack frame
    }
    for (int s = 0; s < S; s++) {
        if (stream >= 0 && s != stream) continue;
        e->pushed[s] = 0;
        e->staged_units[s] = 0;
        e->h_brief[s] = StreamBrief{ 0, ST_NONE, 0, 0, 0 };
        e->drained[s] = 0;
        if (e->am_ring) e->am_raw_bytes[s] = e->am_dec_out[s] = 0;
    }
    CK(cudaGetLastError());
    return NRSC5B_OK;
}

/* Restart every stream from sample 0 of the input it already holds (benchmark loops). */
extern "C" int nrsc5b_rewind(nrsc5b_engine_t *e)
{
    if (!e) return NRSC5B_EINVAL;
    k_reset<<<e->dims.nstreams, 256, 0, e->stream>>>(e->dp, e->dims, -2);
    if (e->l2) k_l2_init<<<e->dims.nstreams, 256, 0, e->stream>>>(e->l2, -1);
    e->stats.kernel_launches += 1;
    if (e->am_st) {                                        // AM: the receiver state lives in AmState / AmWork
        nbam::AmState z;
        memset(&z, 0, sizeof(z));
        nbam::am_reset_state(z);
        for (int s = 0; s < e->dims.nstreams; s++) {
            CK(cudaMemcpyAsync(e->am_st + s, &z, sizeof(z), cudaMemcpyHostToDevice, e->stream));
            CK(cudaMemsetAsync(e->am_work + s, 0, sizeof(nbam::AmWork), e->stream));
        }
        CK(cudaStreamSynchronize(e->stream));              // `z` lives on this stack frame
    }
    for (int s = 0; s < e->dims.nstreams; s++) {
        e->drained[s] = 0;
        e->h_brief[s] = StreamBrief{ 0, ST_NONE, 0, 0, 0 };
    }
    CK(cudaGetLastError());
    return NRSC5B_OK;
}

static double wall_s()
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

static int publish_avail(nrsc5b_engine *e, int s, cudaStream_t on);

// tells the kernels (on stream `on`) about the staged samples copied since the last time
static int publish_pending(nrsc5b_engine *e, cudaStream_t on)
{
    for (int s = 0; s < e->dims.nstreams; s++)
        if (e->unpublished[s]) {
            int rc = publish_avail(e, s, on);
            if (rc) return rc;
            e->unpublished[s] = 0;
        }
    return 0;
}

static int publish_avail(nrsc5b_engine *e, int s, cudaStream_t on)
{
    // staged through a small pinned ring so that the asynchronous copy has a stable source
    if (e->avail_pos && (e->avail_pos & 4095) == 0) CK(cudaStreamSynchronize(on));   // ring wrap: let pending copies drain
    long long *slot = e->avail_ring + (e->avail_pos++ & 4095);
    *slot = e->pushed[s];
    CK(cudaMemcpyAsync(reinterpret_cast<uint8_t *>(e->dp.st + s) + offsetof(StreamState, in_avail), slot, sizeof(*slot),
                       cudaMemcpyHostToDevice, on));
    return 0;
}

__global__ void k_trim_state(DevPtrs p, int s, long long drop, nbam::AmState *ast)
{
    p.st[s].start -= drop;
    p.st[s].in_avail -= 2 * drop;
    if (ast) ast[s].start -= drop;
}

// Discards the samples a stream's window has moved past (everything more than 64 decimated samples before
// the window start), so that an endless stream fits a fixed input buffer.  Synchronous; only called when a
// push would not fit.
static int trim_stream(nrsc5b_engine *e, int s)
{
    CK(cudaStreamSynchronize(e->copy_stream));
    CK(cudaStreamSynchronize(e->stream));
    StreamState st;
    CK(cudaMemcpy(&st, e->dp.st + s, sizeof(st), cudaMemcpyDeviceToHost));
    long long drop = (st.start - 64) & ~7LL;                  // decimated samples; 32-byte granularity in cu8
    if (st.start < 72 || drop <= 0) return 0;
    const size_t off = 4 * (size_t)drop, have = 2 * (size_t)e->pushed[s];
    if (off >= have) return 0;
    const size_t rem = have - off;
    uint8_t *base = e->iq_owned + (size_t)s * e->dims.in_stride;
    if (!e->trim_scratch) {
        void *q = nullptr;
        if (cudaMalloc(&q, e->dims.in_stride) != cudaSuccess) return NRSC5B_ENOMEM;
        e->allocs.push_back(q);
        e->trim_scratch = reinterpret_cast<uint8_t *>(q);
    }
    CK(cudaMemcpyAsync(e->trim_scratch, base + off, rem, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(base, e->trim_scratch, rem, cudaMemcpyDeviceToDevice, e->stream));
    k_trim_state<<<1, 1, 0, e->stream>>>(e->dp, s, drop, e->am_st);
    e->pushed[s] -= 2 * drop;
    e->h_brief[s].start = st.start - drop;
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

static int push_bytes(nrsc5b_engine_t *e, int stream, const uint8_t *buf, size_t nbytes);
static int push_am_cu8(nrsc5b_engine_t *e, int stream, const uint8_t *buf, size_t nbytes);

extern "C" int nrsc5b_push_cu8(nrsc5b_engine_t *e, int stream, const uint8_t *buf, size_t nbytes)
{
    if (!e || e->dims.cs16) return NRSC5B_EINVAL;
    if (e->am_ring) return push_am_cu8(e, stream, buf, nbytes);
    return push_bytes(e, stream, buf, nbytes);
}

// host -> device copy of input on the copy stream: page-locked caller memory is DMA'd directly, pageable memory
// goes through the engine's pinned staging buffer
static int copy_in(nrsc5b_engine_t *e, uint8_t *dst, const uint8_t *buf, size_t nbytes)
{
    cudaPointerAttributes attr;
    bool pinned_src = cudaPointerGetAttributes(&attr, buf) == cudaSuccess && attr.type == cudaMemoryTypeHost;
    cudaGetLastError();
    if (pinned_src) {
        CK(cudaMemcpyAsync(dst, buf, nbytes, cudaMemcpyHostToDevice, e->copy_stream));
    } else {
        size_t done = 0;
        while (done < nbytes) {
            size_t n = nbytes - done < e->pinned_cap ? nbytes - done : e->pinned_cap;
            CK(cudaEventSynchronize(e->pinned_free));
            memcpy(e->pinned, buf + done, n);
            CK(cudaMemcpyAsync(dst + done, e->pinned, n, cudaMemcpyHostToDevice, e->copy_stream));
            CK(cudaEventRecord(e->pinned_free, e->copy_stream));
            done += n;
        }
    }
    return NRSC5B_OK;
}

/* AM, cu8 at 1 488 375 S/s (input_push_cu8 in AM mode, reference src/input.c:96-117): the raw samples go into the
 * stream's ring, k_am_decim turns every complete group of 32 into one cs16 sample appended to the stream's
 * sample buffer, and only that count is published to the receive chain (k_am reads cs16 either way). */
static int push_am_cu8(nrsc5b_engine_t *e, int stream, const uint8_t *buf, size_t nbytes)
{
    if (stream < 0 || stream >= e->dims.nstreams || (nbytes & 3) || !e->iq_owned) return NRSC5B_EINVAL;
    const unsigned R = e->am_ring_bytes;
    uint8_t *ring = e->am_ring + (size_t)stream * R;
    while (nbytes) {
        const size_t n = nbytes < (size_t)R - 4096 ? nbytes : (size_t)R - 4096;     // keeps the 434 samples of history intact
        const long long raw_after = e->am_raw_bytes[stream] + (long long)n;
        const long long can = raw_after / 64;
        const int nout = (int)(can - e->am_dec_out[stream]);
        size_t off = (size_t)e->pushed[stream] * 2;
        if (off + 4 * (size_t)nout > e->dims.in_stride) {
            int rc = trim_stream(e, stream);
            if (rc) return rc;
            off = (size_t)e->pushed[stream] * 2;
            if (off + 4 * (size_t)nout > e->dims.in_stride) return NRSC5B_EFULL;
        }
        const size_t pos = (size_t)(e->am_raw_bytes[stream] & (long long)(R - 1));
        const size_t first = n < R - pos ? n : R - pos;
        int rc = copy_in(e, ring + pos, buf, first);
        if (!rc && n > first) rc = copy_in(e, ring, buf + first, n - first);
        if (rc) return rc;
        e->am_raw_bytes[stream] = raw_after;
        if (nout > 0) {
            short2 *out = reinterpret_cast<short2 *>(e->iq_owned + (size_t)stream * e->dims.in_stride + off);
            k_am_decim<<<(nout + nbam::DEC_T - 1) / nbam::DEC_T, 256, 0, e->copy_stream>>>(ring, R, raw_after / 2, e->am_dec_out[stream],
                                                                                          nout, out);
            e->stats.kernel_launches += 1;
            e->am_dec_out[stream] = can;
            e->pushed[stream] += 2LL * nout;
            e->direct_push = true;
            rc = publish_avail(e, stream, e->copy_stream);
            if (rc) return rc;
        }
        buf += n;
        nbytes -= n;
    }
    CK(cudaGetLastError());
    return NRSC5B_OK;
}

/* cs16: 4 bytes per (already decimated) complex sample; the engine counts input in 2-byte units either way, so
 * a cs16 sample counts like the two cu8 samples it stands for */
extern "C" int nrsc5b_push_cs16(nrsc5b_engine_t *e, int stream, const int16_t *buf, size_t nvalues)
{
    if (!e || !e->dims.cs16 || (nvalues & 1)) return NRSC5B_EINVAL;
    return push_bytes(e, stream, reinterpret_cast<const uint8_t *>(buf), 2 * nvalues);
}

static int push_bytes(nrsc5b_engine_t *e, int stream, const uint8_t *buf, size_t nbytes)
{
    if (!e || stream < 0 || stream >= e->dims.nstreams || (nbytes & 3) || !e->iq_owned) return NRSC5B_EINVAL;
    size_t off = (size_t)e->pushed[stream] * 2;
    if (off + nbytes > e->dims.in_stride) {
        int rc = trim_stream(e, stream);                       // make room: drop what the window has passed
        if (rc) return rc;
        off = (size_t)e->pushed[stream] * 2;
    }
    if (off + nbytes > e->dims.in_stride) return NRSC5B_EFULL;
    uint8_t *dst = e->iq_owned + (size_t)stream * e->dims.in_stride + off;
    {
        int rc = copy_in(e, dst, buf, nbytes);
        if (rc) return rc;
    }
    e->pushed[stream] += (long long)(nbytes / 2);
    e->direct_push = true;
    // published on the copy stream, i.e. after the samples themselves have landed
    return publish_avail(e, stream, e->copy_stream);
}

/* The same number of bytes for every stream from one page-locked host slab (stream s at host + s*host_stride):
 * a single strided copy and a single publication of the new sample counts instead of one pair per stream. */
extern "C" int nrsc5b_push_cu8_all(nrsc5b_engine_t *e, const uint8_t *host, size_t host_stride, size_t nbytes)
{
    if (!e || !host || (nbytes & 3) || !e->iq_owned || nbytes > host_stride || e->am_ring) return NRSC5B_EINVAL;
    const int S = e->dims.nstreams;
    for (int s = 1; s < S; s++)
        if (e->pushed[s] != e->pushed[0]) return NRSC5B_EINVAL;          // streams must be in step
    size_t off = (size_t)e->pushed[0] * 2;
    if (off + nbytes > e->dims.in_stride) return NRSC5B_EFULL;
    CK(cudaMemcpy2DAsync(e->iq_owned + off, e->dims.in_stride, host, host_stride, nbytes, S, cudaMemcpyHostToDevice,
                         e->copy_stream));
    // publish: one strided copy of the new count into every stream's state, after the samples
    if (!e->avail_rows && pinned_alloc((void **)&e->avail_rows, sizeof(long long) * 16 * S) != cudaSuccess) return NRSC5B_ENOMEM;
    if (e->avail_rows_pos && (e->avail_rows_pos & 15) == 0) CK(cudaStreamSynchronize(e->copy_stream));   // rows recycled
    long long *row = e->avail_rows + (size_t)(e->avail_rows_pos++ & 15) * S;
    for (int s = 0; s < S; s++) row[s] = e->pushed[0] + (long long)(nbytes / 2);
    CK(cudaMemcpy2DAsync(reinterpret_cast<uint8_t *>(e->dp.st) + offsetof(StreamState, in_avail), sizeof(StreamState), row,
                         sizeof(long long), sizeof(long long), S, cudaMemcpyHostToDevice, e->copy_stream));
    for (int s = 0; s < S; s++) e->pushed[s] += (long long)(nbytes / 2);
    e->direct_push = true;
    return NRSC5B_OK;
}

extern "C" int nrsc5b_push_cu8_device(nrsc5b_engine_t *e, int stream, const void *dev_buf, size_t nbytes)
{
    if (!e || stream < 0 || stream >= e->dims.nstreams || (nbytes & 3) || !e->iq_owned || e->am_ring) return NRSC5B_EINVAL;
    size_t off = (size_t)e->pushed[stream] * 2;
    if (off + nbytes > e->dims.in_stride) return NRSC5B_EFULL;
    CK(cudaMemcpyAsync(e->iq_owned + (size_t)stream * e->dims.in_stride + off, dev_buf, nbytes,
                       cudaMemcpyDeviceToDevice, e->stream));
    e->pushed[stream] += (long long)(nbytes / 2);
    e->direct_push = true;
    return publish_avail(e, stream, e->stream);
}

extern "C" int nrsc5b_attach_device_input(nrsc5b_engine_t *e, const void *dev_buf, size_t stride, size_t nbytes)
{
    if (!e || !dev_buf || (nbytes & 3) || nbytes > stride || e->am_ring) return NRSC5B_EINVAL;   // AM cu8 is decimated on arrival
    e->dp.iq = reinterpret_cast<const uint8_t *>(dev_buf);
    e->dims.in_stride = stride;
    e->direct_push = true;
    for (int s = 0; s < e->dims.nstreams; s++) {
        e->pushed[s] = (long long)(nbytes / 2);
        int rc = publish_avail(e, s, e->stream);
        if (rc) return rc;
    }
    return NRSC5B_OK;
}

// The engine's side of nrsc5b_chan_feed (chan_feed.h): the channeliser writes cs16 samples straight behind each
// target stream's data in the engine's own input buffers, on the engine's CUDA stream.
int nbfeed_reserve(nrsc5b_engine_t *e, int device, int mode, const int *streams, int nch, long long nout, FeedTarget *t, long long *dst)
{
    if (!e || !t || !dst || nch <= 0 || nout < 0) return NRSC5B_EINVAL;
    if (e->cfg.mode != mode || !e->dims.cs16 || !e->iq_owned || e->dp.iq != e->iq_owned || device != e->cfg.device ||
        e->in_flight)
        return NRSC5B_EINVAL;
    const int S = e->dims.nstreams;
    if (!streams && nch > S) return NRSC5B_EINVAL;
    std::vector<uint8_t> seen(S, 0);
    for (int k = 0; k < nch; k++) {
        const int s = streams ? streams[k] : k;
        if (s < 0 || s >= S || seen[s]) return NRSC5B_EINVAL;
        seen[s] = 1;
    }
    // all or nothing: every target stream must take the whole push (trim the full ones, then look again)
    const size_t need = 4 * (size_t)nout;
    bool full = false;
    for (int k = 0; k < nch; k++) {
        const int s = streams ? streams[k] : k;
        if ((size_t)e->pushed[s] * 2 + need <= e->dims.in_stride) continue;
        int rc = trim_stream(e, s);
        if (rc) return rc;
        if ((size_t)e->pushed[s] * 2 + need > e->dims.in_stride) full = true;
    }
    if (full) return NRSC5B_EFULL;
    t->stream = e->stream;
    t->base = reinterpret_cast<int16_t *>(e->iq_owned);
    for (int k = 0; k < nch; k++) {
        const int s = streams ? streams[k] : k;
        dst[k] = (long long)(((size_t)s * e->dims.in_stride + (size_t)e->pushed[s] * 2) / sizeof(int16_t));
    }
    return NRSC5B_OK;
}

int nbfeed_commit(nrsc5b_engine_t *e, const int *streams, int nch, long long nout)
{
    if (nout <= 0) return NRSC5B_OK;
    for (int k = 0; k < nch; k++) {
        const int s = streams ? streams[k] : k;
        e->pushed[s] += 2 * nout;                              // 2-byte units: a cs16 sample counts as two
        int rc = publish_avail(e, s, e->stream);               // on the feed's stream, i.e. after the samples
        if (rc) return rc;
    }
    e->direct_push = true;
    return NRSC5B_OK;
}

extern "C" int nrsc5b_attach_device_log(nrsc5b_engine_t *e, void *dev_buf, size_t stride)
{
    if (!e || !dev_buf || stride < 4096 || (stride & 15)) return NRSC5B_EINVAL;
    CK(cudaStreamSynchronize(e->stream));
    e->dp.log = reinterpret_cast<uint8_t *>(dev_buf);
    e->dims.log_cap = stride;
    return NRSC5B_OK;
}

static void launch_vitc(const VitcArgs &a, int nframes, cudaStream_t stream)
{
    dim3 gf((a.nch + 2 * VITC_FWD_WARPS - 1) / (2 * VITC_FWD_WARPS), nframes);
    k_vitc_fwd<<<gf, VITC_FWD_WARPS * 32, 0, stream>>>(a);
    k_vitc_ends<<<nframes, 32, 0, stream>>>(a);
    dim3 ge((a.nch + VITC_EMIT_WARPS - 1) / VITC_EMIT_WARPS, nframes);
    k_vitc_emit<<<ge, VITC_EMIT_WARPS * 32, vitc_emit_smem(), stream>>>(a);
}

static void launch_v64(const V64Args &a, int nframes, cudaStream_t stream)
{
    k_v64_fwd<<<dim3((a.nch + V64_FWD_THREADS - 1) / V64_FWD_THREADS, nframes), V64_FWD_THREADS, 0, stream>>>(a);
    k_v64_check<<<nframes, V64_CHECK_THREADS, 0, stream>>>(a);
    const int nwin = (a.len + 64 + V64_WIN - 1) / V64_WIN;
    k_v64_emit<<<dim3((nwin + V64_EMIT_WARPS - 1) / V64_EMIT_WARPS, nframes), V64_EMIT_WARPS * 32, V64_EMIT_SMEM, stream>>>(a);
}

// Extended-partition decode group G, once a stream has asked for it (enable_px_groups).
template <int G>
static void launch_px_group(nrsc5b_engine *e)
{
    if (!(e->dims.px_enabled & (1 << G))) return;
    const int S = e->dims.nstreams;
    k_px_gather<G><<<dim3(P3_SLOTS, S), 256, 0, e->stream>>>(e->dp, e->dims);
    launch_v64(px_v64_args(e->dp, G), S * P3_SLOTS, e->stream);
    launch_vitc(px_vitc_args(e->dp, G), S * P3_SLOTS, e->stream);
    k_px_fin<G><<<dim3(P3_SLOTS, S), 128, 0, e->stream>>>(e->dp, e->dims);
    e->stats.kernel_launches += 8;
}

static void launch_p1(nrsc5b_engine *e)
{
    NvtxRange nvtx_("nrsc5b: P1/P3 decode groups");
    const int S = e->dims.nstreams;
    k_p1_gather<<<dim3(32, S), 256, 0, e->stream>>>(e->dp, e->dims);
    launch_v64(p1_v64_args(e->dp, e->v64_ch), S, e->stream);      // fast path ...
    launch_vitc(p1_vitc_args(e->dp), S, e->stream);               // ... exact fallback for the frames it flagged
    k_p1_fin<<<dim3(FIN_CTAS, S), P1_THREADS, 0, e->stream>>>(e->dp, e->dims);
    e->stats.kernel_launches += 8;
    static_assert(PX_GROUPS == 3, "one launch per decode group, in group order");
    launch_px_group<0>(e);
    launch_px_group<1>(e);
    launch_px_group<2>(e);
}

// Allocates the buffers of the decode groups named in `need` (bit g = group g) and adds them to the passes.
static int enable_px_groups(nrsc5b_engine *e, unsigned need)
{
    const size_t F = (size_t)e->dims.nstreams * P3_SLOTS;
    for (int g = 0; g < PX_GROUPS; g++) {
        if (!(need & (1u << g)) || (e->dims.px_enabled & (1 << g))) continue;
        const int len = px_group(g).len;
        PxBufs &xb = e->dp.xb[g];
        int rc = dev_alloc(e, &xb.vin, F * 3 * len);
        if (!rc) rc = dev_alloc(e, &xb.dec, F * P3_DEC_STRIDE);
        if (!rc) rc = dev_alloc(e, &xb.spec, F * 19 * 32);
        if (!rc) rc = dev_alloc(e, &xb.end, F * 19 * 32);
        if (!rc) rc = dev_alloc(e, &xb.endstate, F);
        if (!rc) rc = dev_alloc(e, &xb.fspec, F * 5 * 16);
        if (!rc) rc = dev_alloc(e, &xb.fend, F * 5 * 16);
        if (!rc) rc = dev_alloc(e, &xb.fhstate, F * 5);
        if (!rc) rc = dev_alloc(e, &xb.ftbend, F * 5);
        if (!rc) rc = dev_alloc(e, &xb.bits, F * (len / 32));
        if (!rc) rc = dev_alloc(e, &xb.flags, F * 4);
        if (rc) return rc;
        e->dims.px_enabled |= 1 << g;
    }
    return NRSC5B_OK;
}

// One pass: every stream runs its front end up to its next frame boundary (at most BLOCKS_PER_PASS blocks,
// one persistent CTA per stream), then the P1 decode of the streams that completed an interleaver matrix.
// last_pass: the batch ends here - streams that could go on at once say so in EngineCtl::more.
// with_decode = false: the host knows that no stream can complete a frame in this pass (plan_passes), the decode
// groups and k_l2 would find nothing.
constexpr int BLOCKS_PER_PASS = 16;

// k_stream with one CTA per stream, or - engines with few streams - a thread-block cluster of dims.cluster CTAs per
// stream (the cluster dimension is a launch attribute)
static void launch_k_stream(nrsc5b_engine *e, int last_pass)
{
    const int S = e->dims.nstreams, C = e->dims.cluster > 1 ? e->dims.cluster : 1;
#if !defined(NB_EMU)
    if (C > 1) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)(S * C));
        cfg.blockDim = dim3(FRONT_THREADS);
        cfg.dynamicSmemBytes = sizeof(FrontSmem);
        cfg.stream = e->stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = (unsigned)C;
        at[0].val.clusterDim.y = 1;
        at[0].val.clusterDim.z = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        if (cudaLaunchKernelEx(&cfg, k_stream<true>, e->dp, e->dims, (int)BLOCKS_PER_PASS, last_pass) != cudaSuccess) {
            // (checked once at creation with a trial launch; a failure here is reported by the caller's cudaGetLastError)
            fprintf(stderr, "nrsc5_b200: cluster launch of k_stream failed: %s\n", cudaGetErrorString(cudaPeekAtLastError()));
        }
        return;
    }
#endif
    k_stream<false><<<S, FRONT_THREADS, sizeof(FrontSmem), e->stream>>>(e->dp, e->dims, BLOCKS_PER_PASS, last_pass);
}

static int launch_pass(nrsc5b_engine *e, bool last_pass, bool with_decode = true)
{
    NvtxRange nvtx_("nrsc5b: pass");
    if (last_pass) cudaMemsetAsync(reinterpret_cast<uint8_t *>(e->dp.ctl) + offsetof(EngineCtl, more), 0, sizeof(unsigned), e->stream);
    if (e->am_st) {                                        // AM: one kernel does the whole chain, window after window
        const bool l2 = e->l2 && e->dims.l2;              // with L2 on, a launch stops after 16 blocks: its frames fit the queue
        k_am<<<e->dims.nstreams, nbam::AM_THREADS, sizeof(nbam::AmSmem), e->stream>>>(e->dp, e->dims, e->am_st, e->am_work, e->am_tb, l2 ? nbam::AM_L2_BLOCKS : 1 << 20,
                                                     last_pass ? 1 : 0);
        e->stats.kernel_launches += 1;
        if (l2) {
            k_l2<<<e->dims.nstreams, nbl2::L2_THREADS, 0, e->stream>>>(e->dp, e->dims, e->l2);
            e->stats.kernel_launches += 1;
        }
        return 0;
    }
    const bool prof = e->profiling != 0;
    if (prof) cudaEventRecord(e->pev[0], e->stream);
    launch_k_stream(e, last_pass ? 1 : 0);
    e->stats.kernel_launches += 1;
    if (prof) cudaEventRecord(e->pev[1], e->stream);
    if (with_decode) launch_p1(e);
    if (prof) cudaEventRecord(e->pev[2], e->stream);
    // L2 framing of everything the pass decoded (only when enabled, nrsc5b_enable_l2); a pass without decode groups
    // can still have queued a frame_reset (fine sync entered), which the next k_l2 takes
    if (with_decode && e->l2 && e->dims.l2) {
        k_l2<<<e->dims.nstreams, nbl2::L2_THREADS, 0, e->stream>>>(e->dp, e->dims, e->l2);
        e->stats.kernel_launches += 1;
    }
    if (prof) {
        cudaEventRecord(e->pev[3], e->stream);
        cudaEventSynchronize(e->pev[3]);
        float ms = 0;
        cudaEventElapsedTime(&ms, e->pev[0], e->pev[1]);
        e->kernel_ms[1] += ms; e->kernel_n[1] += 1;
        cudaEventElapsedTime(&ms, e->pev[1], e->pev[2]);
        e->kernel_ms[3] += ms; e->kernel_n[3] += 1;
        if (e->l2 && e->dims.l2) {
            cudaEventElapsedTime(&ms, e->pev[2], e->pev[3]);
            e->kernel_ms[2] += ms; e->kernel_n[2] += 1;
        }
    }
    return 0;
}

// How many passes the samples buffered on the host's count can need, from what the host knows of every stream
// (StreamBrief: window position, sync state, block count - read back behind every batch): a block needs a whole
// 33-symbol window and moves it on by 32 symbols +- the timing correction; a pass ends at a frame boundary.  The
// count errs on the high side (a surplus pass finds nothing to do); 0 = no stream can complete a block, nothing is
// launched at all.  *first_needs_decode: whether a stream can complete a frame in the first pass.
static int plan_passes(const nrsc5b_engine *e, bool count_staged, bool *first_needs_decode)
{
    const bool am = e->am_st != nullptr;
    const long long win = am ? nbam::NACQ : NACQ, adv = am ? nbam::SYM * nbam::BLK : NSYM * BLK;
    const long long slack = am ? 40 : 160;                 // the window can advance by less than `adv` (timing correction)
    int passes = 0;
    bool decode = am || e->dims.px_enabled != 0;           // (extended-partition frames complete every second block)
    for (int s = 0; s < e->dims.nstreams; s++) {
        const StreamBrief &b = e->h_brief[s];
        if (b.p1_ready) decode = true;
        const long long have = (e->pushed[s] + (count_staged ? e->staged_units[s] : 0)) / 2;
        if (have < b.start + win) { if (b.p1_ready && passes < 1) passes = 1; continue; }
        const long long blocks = 1 + (have - b.start - win) / (adv - slack);
        long long segs;
        if (am) {
            segs = (e->l2 && e->dims.l2) ? (blocks + nbam::AM_L2_BLOCKS - 1) / nbam::AM_L2_BLOCKS : 1;
        } else if (b.state == ST_FINE) {
            const long long first = BLOCKS_PER_PASS - b.bc;         // blocks up to and including the frame's last one
            segs = blocks <= first ? 1 : 1 + (blocks - first + BLOCKS_PER_PASS - 1) / BLOCKS_PER_PASS;
            if (blocks >= first) decode = true;
        } else {
            segs = (blocks + BLOCKS_PER_PASS - 1) / BLOCKS_PER_PASS + 1;   // acquisition re-aligns the frame boundaries
            decode = true;
        }
        if (segs > passes) passes = (int)(segs > 12 ? 12 : segs);
    }
    if (first_needs_decode) *first_needs_decode = decode;
    return passes;
}

// Reads the control words and briefs of the batch just enqueued into page-locked memory (asynchronously).
static int enqueue_readback(nrsc5b_engine *e)
{
    CK(cudaMemcpyAsync(e->h_ctl, e->dp.ctl, sizeof(EngineCtl), cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(e->h_brief, e->dp.brief, sizeof(StreamBrief) * e->dims.nstreams, cudaMemcpyDeviceToHost, e->stream));
    return 0;
}

/* Per-kernel device time (CUDA events around every launch; slows the run down, use a separate pass).
 * Slots: [1] = the stream-resident front-end kernel k_stream, [3] = the P1 decode group, [2] = k_l2; [0] unused. */
extern "C" int nrsc5b_set_profiling(nrsc5b_engine_t *e, int on)
{
    if (!e) return NRSC5B_EINVAL;
    if (on && !e->pev[0])
        for (int i = 0; i < 5; i++) CK(cudaEventCreate(&e->pev[i]));
    e->profiling = on;
    for (int i = 0; i < 4; i++) { e->kernel_ms[i] = 0; e->kernel_n[i] = 0; }
    return NRSC5B_OK;
}

extern "C" int nrsc5b_debug_set(int flags)
{
    CK(cudaMemcpyToSymbol(g_dbg, &flags, sizeof(flags)));
    return NRSC5B_OK;
}

extern "C" int nrsc5b_get_phase_cycles(nrsc5b_engine_t *e, unsigned long long *cyc5, unsigned long long *n5)
{
    // twelve slots (see StreamState::ph_cyc, sy_cyc)
    if (!e || !cyc5 || !n5) return NRSC5B_EINVAL;
    CK(cudaStreamSynchronize(e->stream));
    const int S = e->dims.nstreams;
    CK(cudaMemcpy(e->h_state, e->dp.st, sizeof(StreamState) * S, cudaMemcpyDeviceToHost));
    for (int i = 0; i < 12; i++) { cyc5[i] = 0; n5[i] = 0; }
    for (int s = 0; s < S; s++) {
        for (int i = 0; i < 6; i++) { cyc5[i] += e->h_state[s].ph_cyc[i]; n5[i] += e->h_state[s].ph_n[i]; }
        // slots 6..11: sub-phases of the FINE sync (same call count as slot 4, approximately)
        for (int i = 0; i < 6; i++) { cyc5[6 + i] += e->h_state[s].sy_cyc[i]; n5[6 + i] += e->h_state[s].ph_n[4]; }
    }
    return NRSC5B_OK;
}

/* AM: SM cycles k_am spent per phase, summed over streams since the last reset / rewind (thread 0's clock): window +
 * coarse acquisition, first demodulation pass (carrier), second pass (bins), sync + slicing, PIDS, P1/P3 group incl. the two
 * following, P3 post-processing, interleaver; then, across all decodes: K=9 recursion, traceback; window load of a block in
 * fine sync; spare. */
extern "C" int nrsc5b_get_am_phase_cycles(nrsc5b_engine_t *e, unsigned long long *cyc12)
{
    if (!e || !cyc12 || !e->am_work) return NRSC5B_EINVAL;
    CK(cudaStreamSynchronize(e->stream));
    for (int i = 0; i < 12; i++) cyc12[i] = 0;
    for (int s = 0; s < e->dims.nstreams; s++) {
        unsigned long long v[16];
        CK(cudaMemcpy(v, reinterpret_cast<uint8_t *>(e->am_work + s) + offsetof(nbam::AmWork, ph_cyc), sizeof(v), cudaMemcpyDeviceToHost));
        for (int i = 0; i < 12; i++) cyc12[i] += v[i];
        if (getenv("NRSC5_B200_TRACE") && s == 0) fprintf(stderr, "nrsc5_b200 trace: AM stream 0 traceback Mcycles {warm-up %.2f, walks %.2f, checks %.2f}, until return %.2f, slot 8 %.2f slot 9 %.2f\n", v[12] * 1e-6, v[13] * 1e-6, v[14] * 1e-6, v[15] * 1e-6, v[8] * 1e-6, v[9] * 1e-6);
    }
    return NRSC5B_OK;
}

extern "C" int nrsc5b_get_kernel_times(nrsc5b_engine_t *e, double *ms4, unsigned long long *n4)
{
    if (!e || !ms4 || !n4) return NRSC5B_EINVAL;
    for (int i = 0; i < 4; i++) { ms4[i] = e->kernel_ms[i]; n4[i] = e->kernel_n[i]; }
    return NRSC5B_OK;
}

static int flush_staged(nrsc5b_engine *e);
extern "C" int nrsc5b_prepare_async(nrsc5b_engine_t *e);

static int process_impl(nrsc5b_engine_t *e, bool wait_for_copies)
{
    NvtxRange nvtx_("nrsc5b_process");
    if (!e) return NRSC5B_EINVAL;
    if (e->in_flight) return NRSC5B_EINVAL;                // an asynchronous batch is open: nrsc5b_poll first
    {
        int rc = flush_staged(e);
        if (!rc) rc = publish_pending(e, e->copy_stream);
        if (rc) return rc;
    }
    if (wait_for_copies) {
        // everything pushed before this call: the compute stream waits (on the device) for the copy stream
        const unsigned slot = e->fence_next++ & 63;
        if (!e->fence[slot]) CK(cudaEventCreateWithFlags(&e->fence[slot], cudaEventDisableTiming));
        CK(cudaEventRecord(e->fence[slot], e->copy_stream));
        CK(cudaStreamWaitEvent(e->stream, e->fence[slot], 0));
    }
    // Batches of passes sized by plan_passes() from the host's sample counts and the streams' last known positions;
    // behind every batch one small read-back (control words + briefs) and one synchronisation.  A caller that pushes
    // less than a block at a time therefore launches nothing on most calls.
    for (int guard = 0; guard < 1 << 20; guard++) {
        bool decode = true;
        const int passes = plan_passes(e, false, &decode);
        if (passes == 0) break;
        for (int i = 0; i < passes; i++) {
            int rc = launch_pass(e, i == passes - 1, i > 0 || decode);
            if (rc) return rc;
        }
        int rc = enqueue_readback(e);
        if (rc) return rc;
        CK(cudaStreamSynchronize(e->stream));
        CK(cudaGetLastError());
        const unsigned long long delta = e->h_ctl->progress - e->last_progress;
        e->last_progress = e->h_ctl->progress;
        if (passes > 1 || decode)                          // (a brief is written before its pass's decode groups run)
            for (int s = 0; s < e->dims.nstreams; s++) e->h_brief[s].p1_ready = 0;
        if (e->h_ctl->px_need & ~(unsigned)e->dims.px_enabled) {
            // a stream in MP2 / MP3 / MP11 waits at a block boundary for its decode group: add it and go on
            rc = enable_px_groups(e, e->h_ctl->px_need);
            if (rc) return rc;
            continue;
        }
        if (e->h_ctl->more == 0) break;                    // no stream has another whole window
        if (delta == 0) {
            // streams report more input than they could use: samples still in flight on the copy stream
            if (!wait_for_copies || cudaStreamQuery(e->copy_stream) == cudaSuccess) break;
            CK(cudaStreamSynchronize(e->copy_stream));
        }
    }
    return NRSC5B_OK;
}

/* A fence behind everything pushed so far (pushes are asynchronous copies on the engine's copy stream).
 * Returns a token >= 0 for nrsc5b_process_fence; tokens are recycled after 64 newer fences. */
extern "C" int nrsc5b_push_fence(nrsc5b_engine_t *e)
{
    if (!e) return NRSC5B_EINVAL;
    const unsigned slot = e->fence_next++ & 63;
    if (!e->fence[slot]) CK(cudaEventCreateWithFlags(&e->fence[slot], cudaEventDisableTiming));
    CK(cudaEventRecord(e->fence[slot], e->copy_stream));
    return (int)slot;
}

/* Processes what had been pushed when the fence was taken, as soon as it has landed - later pushes keep
 * copying meanwhile (the way to overlap host->device transfer with compute). */
extern "C" int nrsc5b_process_fence(nrsc5b_engine_t *e, int token)
{
    if (!e || token < 0 || token >= 64 || !e->fence[token]) return NRSC5B_EINVAL;
    CK(cudaStreamWaitEvent(e->stream, e->fence[token], 0));
    return process_impl(e, false);
}

extern "C" int nrsc5b_process(nrsc5b_engine_t *e) { return process_impl(e, true); }
extern "C" int nrsc5b_process_available(nrsc5b_engine_t *e) { return process_impl(e, false); }

// ===========================================================================
// Asynchronous use (one stream or many): staged input, one batch of passes in flight, records exported to host memory
// ===========================================================================
static int stage_bytes(nrsc5b_engine *e, int stream, const uint8_t *buf, size_t nbytes)
{
    if (stream < 0 || stream >= e->dims.nstreams || (nbytes & 3) || !e->iq_owned || e->am_ring) return NRSC5B_EINVAL;
    if (!e->stage[0]) {
        int rc = nrsc5b_prepare_async(e);
        if (rc) return rc;
    }
    // a call that came back with NRSC5B_EFULL left the rest of its samples here (the caller's buffer may be gone by
    // the time it retries): they go first; the retry passes (NULL, 0)
    if (!e->carry.empty()) {
        std::vector<uint8_t> rest;
        rest.swap(e->carry);
        const int cs = e->carry_stream;
        int rc = stage_bytes(e, cs, rest.data(), rest.size());
        if (rc) {
            if (rc == NRSC5B_EFULL && nbytes) {                 // still no room: the new samples queue up behind
                e->carry.insert(e->carry.end(), buf, buf + nbytes);
            }
            return rc;
        }
    }
    while (nbytes) {
        if (e->stage_fill == e->stage_cap) {               // this half is full: send it, go on in the other one
            int rc = flush_staged(e);
            if (rc == NRSC5B_EFULL) {
                e->carry.assign(buf, buf + nbytes);
                e->carry_stream = stream;
            }
            if (rc) return rc;
        }
        const size_t n = nbytes < e->stage_cap - e->stage_fill ? nbytes : e->stage_cap - e->stage_fill;
        memcpy(e->stage[e->stage_cur] + e->stage_fill, buf, n);
        if (!e->staged.empty() && e->staged.back().stream == stream && e->staged.back().off + e->staged.back().n == e->stage_fill)
            e->staged.back().n += n;                        // the usual case: one stream, contiguous pushes
        else
            e->staged.push_back({ stream, e->stage_fill, n });
        e->stage_fill += n;
        e->staged_units[stream] += (long long)(n / 2);
        buf += n;
        nbytes -= n;
    }
    return NRSC5B_OK;
}

/* input_push_cu8 / input_push_cs16 without a CUDA call: the samples are copied into page-locked memory and reach the
 * device - one copy per stream - when the next batch is submitted (nrsc5b_submit), when the staging area (4 MiB) is
 * full, or when nrsc5b_process runs. */
extern "C" int nrsc5b_stage_cu8(nrsc5b_engine_t *e, int stream, const uint8_t *buf, size_t nbytes)
{
    if (!e || e->dims.cs16) return NRSC5B_EINVAL;
    return stage_bytes(e, stream, buf, nbytes);
}

extern "C" int nrsc5b_stage_cs16(nrsc5b_engine_t *e, int stream, const int16_t *buf, size_t nvalues)
{
    if (!e || !e->dims.cs16 || (nvalues & 1)) return NRSC5B_EINVAL;
    return stage_bytes(e, stream, reinterpret_cast<const uint8_t *>(buf), 2 * nvalues);
}

static int flush_staged(nrsc5b_engine *e)
{
    // The samples travel now; the kernels are told about them by the next batch (publish_pending on the compute
    // stream, nrsc5b_submit) - never in the middle of one: a batch sees exactly the sample counts it was planned with.
    if (e->staged.empty()) return NRSC5B_OK;
    const double t0 = e->trace_on ? wall_s() : 0;
    const uint8_t *src = e->stage[e->stage_cur];
    while (!e->staged.empty()) {
        nrsc5b_engine::Staged &g = e->staged.front();
        size_t off = (size_t)e->pushed[g.stream] * 2;
        if (off + g.n > e->dims.in_stride) {
            const double t1 = e->trace_on ? wall_s() : 0;
            int rc = trim_stream(e, g.stream);                  // make room: drop what the window has passed
            if (e->trace_on) { e->tr.trims++; e->tr.s_trim += wall_s() - t1; }
            if (rc) return rc;
            off = (size_t)e->pushed[g.stream] * 2;
        }
        // as much of the entry as the device buffer takes (an entry can be larger than a small buffer)
        const size_t room = e->dims.in_stride > off ? (e->dims.in_stride - off) & ~(size_t)3 : 0;
        const size_t n = g.n < room ? g.n : room;
        if (n) {
            CK(cudaMemcpyAsync(e->iq_owned + (size_t)g.stream * e->dims.in_stride + off, src + g.off, n, cudaMemcpyHostToDevice,
                               e->copy_stream));
            e->pushed[g.stream] += (long long)(n / 2);
            e->staged_units[g.stream] -= (long long)(n / 2);
            e->unpublished[g.stream] = 1;
            g.off += n;
            g.n -= n;
        }
        if (g.n) return NRSC5B_EFULL;                           // the rest stays on the list (and in this staging half)
        e->staged.erase(e->staged.begin());
    }
    CK(cudaEventRecord(e->stage_free[e->stage_cur], e->copy_stream));
    e->stage_cur ^= 1;
    e->stage_fill = 0;
    const double t2 = e->trace_on ? wall_s() : 0;
    CK(cudaEventSynchronize(e->stage_free[e->stage_cur]));      // the other half: its copy was issued a whole half ago
    if (e->trace_on) { e->tr.flushes++; e->tr.s_stage_wait += wall_s() - t2; e->tr.s_flush += wall_s() - t0; }
    return NRSC5B_OK;
}

/* Allocates what the asynchronous path needs (page-locked staging halves and export buffers) now instead of at the
 * first nrsc5b_stage_* / nrsc5b_submit call - a few milliseconds of cudaMallocHost that a caller may not want inside
 * its first push. */
extern "C" int nrsc5b_prepare_async(nrsc5b_engine_t *e)
{
    if (!e) return NRSC5B_EINVAL;
    if (!e->stage[0]) {
        e->stage_cap = 4u << 20;
        for (int i = 0; i < 2; i++) {
            if (pinned_alloc((void **)&e->stage[i], e->stage_cap) != cudaSuccess) return NRSC5B_ENOMEM;
            CK(cudaEventCreateWithFlags(&e->stage_free[i], cudaEventDisableTiming));
        }
    }
    if (!e->xlog) {
        const int S = e->dims.nstreams;
        e->xlog_stride = (e->dims.log_cap + 15) & ~(size_t)15;
        if (pinned_alloc((void **)&e->xlog, (size_t)S * e->xlog_stride) != cudaSuccess ||
            pinned_alloc((void **)&e->xhdr, sizeof(ExportHdr) * S) != cudaSuccess) return NRSC5B_ENOMEM;
    }
    return NRSC5B_OK;
}

/* Enqueues - without waiting for anything - the passes that the samples staged / pushed so far can need, followed by
 * the export of every stream's records to host memory.  Returns 1 if a batch was enqueued, 0 if there is nothing to
 * do (no stream has a whole block buffered: nothing is launched, no CUDA call is made) or a batch is still in flight,
 * < 0 on error.  flush != 0: also send staged input that does not complete a block yet (end of stream). */
extern "C" int nrsc5b_submit(nrsc5b_engine_t *e, int flush)
{
    NvtxRange nvtx_("nrsc5b_submit");
    if (!e) return NRSC5B_EINVAL;
    if (e->in_flight) return 0;
    bool decode = true;
    const int passes = plan_passes(e, true, &decode);
    if (passes == 0 && !flush) {
        if (e->trace_on) e->tr.submits_idle++;
        return 0;                                              // the usual case of a small push: no CUDA call at all
    }
    int rc = flush_staged(e);
    if (rc == NRSC5B_EFULL) rc = NRSC5B_OK;                // no room yet: the batch runs on what the device holds and frees some
    if (rc) return rc;
    if (passes == 0) return 0;
    if (e->stalled) {
        // the last batch moved no stream: nothing to gain from another one until the device holds more samples
        long long units = 0;
        for (int s = 0; s < e->dims.nstreams; s++) units += e->pushed[s];
        if (units == e->stalled_units) return 0;
        e->stalled = false;
    }
    const double t0 = e->trace_on ? wall_s() : 0;
    if (e->direct_push) decode = true;                     // counts published outside a batch: plan nothing on them
    e->direct_push = false;
    const int S = e->dims.nstreams;
    if (!e->xlog) {
        rc = nrsc5b_prepare_async(e);
        if (rc) return rc;
    }
    {
        const unsigned slot = e->fence_next++ & 63;
        if (!e->fence[slot]) CK(cudaEventCreateWithFlags(&e->fence[slot], cudaEventDisableTiming));
        CK(cudaEventRecord(e->fence[slot], e->copy_stream));
        CK(cudaStreamWaitEvent(e->stream, e->fence[slot], 0));
    }
    rc = publish_pending(e, e->stream);                    // behind the copies, in front of the passes
    if (rc) return rc;
    for (int i = 0; i < passes; i++) {
        rc = launch_pass(e, i == passes - 1, i > 0 || decode);
        if (rc) return rc;
    }
    if (e->trace_on) { e->tr.batches++; e->tr.passes += passes; e->tr.decode_passes += passes - 1 + (decode ? 1 : 0); }
    k_export<<<S, 256, 0, e->stream>>>(e->dp, e->dims, e->xlog, e->xlog_stride, e->xhdr);
    e->stats.kernel_launches += 1;
    rc = enqueue_readback(e);
    if (rc) return rc;
    CK(cudaEventRecord(e->batch_done, e->stream));
    CK(cudaGetLastError());
    e->in_flight = true;
    e->batch_decoded = passes > 1 || decode;
    if (e->trace_on) e->tr.s_submit += wall_s() - t0;
    return 1;
}

/* 1: the batch in flight has finished - its records are in host memory (nrsc5b_batch_records) until the next
 * nrsc5b_submit; 0: no batch in flight, or (wait == 0) it is still running; < 0 on error. */
extern "C" int nrsc5b_poll(nrsc5b_engine_t *e, int wait)
{
    NvtxRange nvtx_("nrsc5b_poll");
    if (!e) return NRSC5B_EINVAL;
    if (!e->in_flight) return 0;
    if (wait) {
        const double t0 = e->trace_on ? wall_s() : 0;
        CK(cudaEventSynchronize(e->batch_done));
        if (e->trace_on) e->tr.s_poll_wait += wall_s() - t0;
    } else {
        const cudaError_t q = cudaEventQuery(e->batch_done);
        if (q == cudaErrorNotReady) return 0;
        CK(q);
    }
    e->in_flight = false;
    if (e->trace_on) e->tr.polls_ready++;
    if (e->h_ctl->progress == e->last_progress && !(e->h_ctl->px_need & ~(unsigned)e->dims.px_enabled)) {
        e->stalled = true;
        e->stalled_units = 0;
        for (int s = 0; s < e->dims.nstreams; s++) e->stalled_units += e->pushed[s];
    }
    e->last_progress = e->h_ctl->progress;
    if (e->batch_decoded)
        for (int s = 0; s < e->dims.nstreams; s++) e->h_brief[s].p1_ready = 0;
    for (int s = 0; s < e->dims.nstreams; s++)
        if (e->xhdr[s].log_overflow) {
            e->overflowed[s] = 1;
            e->stats.log_overflows++;
        }
    if (e->h_ctl->px_need & ~(unsigned)e->dims.px_enabled) {
        int rc = enable_px_groups(e, e->h_ctl->px_need);        // the waiting streams go on with the next batch
        if (rc) return rc;
    }
    return 1;
}

/* Records of `stream` from the batch nrsc5b_poll last reported (same format as nrsc5b_drain); valid until the next
 * nrsc5b_submit. */
extern "C" const uint8_t *nrsc5b_batch_records(nrsc5b_engine_t *e, int stream, size_t *nbytes)
{
    if (!e || !e->xlog || stream < 0 || stream >= e->dims.nstreams || e->in_flight) {
        if (nbytes) *nbytes = 0;
        return nullptr;
    }
    if (nbytes) *nbytes = e->xhdr[stream].log_len;
    return e->xlog + (size_t)stream * e->xlog_stride;
}

extern "C" int nrsc5b_synchronize(nrsc5b_engine_t *e)
{
    if (!e) return NRSC5B_EINVAL;
    CK(cudaStreamSynchronize(e->stream));
    return NRSC5B_OK;
}

extern "C" long nrsc5b_drain(nrsc5b_engine_t *e, int stream, uint8_t *out, size_t cap, size_t *needed)
{
    if (!e || stream < 0 || stream >= e->dims.nstreams) return NRSC5B_EINVAL;
    CK(cudaStreamSynchronize(e->stream));
    StreamState st;
    CK(cudaMemcpy(&st, e->dp.st + stream, sizeof(st), cudaMemcpyDeviceToHost));
    size_t avail = st.log_len - e->drained[stream];
    if (needed) *needed = avail;
    if (!out || cap < avail) return avail == 0 ? 0 : NRSC5B_EFULL;
    if (avail) {
        CK(cudaMemcpy(out, e->dp.log + (size_t)stream * e->dims.log_cap + e->drained[stream], avail,
                      cudaMemcpyDeviceToHost));
    }
    // the log is rewound once fully drained, and the overflow flag goes with it (log_len, log_overflow are adjacent)
    static_assert(offsetof(StreamState, log_overflow) == offsetof(StreamState, log_len) + sizeof(unsigned), "cleared together");
    const unsigned zero[2] = { 0, 0 };
    CK(cudaMemcpy(reinterpret_cast<uint8_t *>(e->dp.st + stream) + offsetof(StreamState, log_len), zero, sizeof(zero),
                  cudaMemcpyHostToDevice));
    e->drained[stream] = 0;
    if (st.log_overflow) {
        // the records handed out are a prefix of what the stream produced: told to the caller (nrsc5b_take_overflow,
        // stats.log_overflows), once per truncated drain
        e->overflowed[stream] = 1;
        e->stats.log_overflows++;
        fprintf(stderr, "nrsc5_b200: stream %d output log overflowed (raise log_capacity)\n", stream);
    }
    return (long)avail;
}

/* All streams at once: records of stream s go to out + s*out_stride, their byte count to sizes[s].  One
 * device->host copy of the stream states, then one asynchronous copy per stream and a single wait. */
extern "C" int nrsc5b_drain_all(nrsc5b_engine_t *e, uint8_t *out, size_t out_stride, size_t *sizes)
{
    NvtxRange nvtx_("nrsc5b_drain_all");
    if (!e || !out || !sizes) return NRSC5B_EINVAL;
    const int S = e->dims.nstreams;
    CK(cudaMemcpyAsync(e->h_state, e->dp.st, sizeof(StreamState) * S, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    int rc = NRSC5B_OK;
    for (int s = 0; s < S; s++) {
        const size_t avail = e->h_state[s].log_len - e->drained[s];
        sizes[s] = avail;
        if (avail > out_stride) { rc = NRSC5B_EFULL; sizes[s] = 0; continue; }
        if (avail)
            CK(cudaMemcpyAsync(out + (size_t)s * out_stride, e->dp.log + (size_t)s * e->dims.log_cap + e->drained[s], avail,
                               cudaMemcpyDeviceToHost, e->stream));
    }
    bool truncated = false;
    if (rc == NRSC5B_OK) {
        // rewind every log and clear its overflow flag (strided 8-byte writes of zero into the states)
        CK(cudaMemset2DAsync(reinterpret_cast<uint8_t *>(e->dp.st) + offsetof(StreamState, log_len), sizeof(StreamState), 0,
                             2 * sizeof(unsigned), S, e->stream));
        for (int s = 0; s < S; s++) {
            e->drained[s] = 0;
            if (e->h_state[s].log_overflow) {
                e->overflowed[s] = 1;
                e->stats.log_overflows++;
                truncated = true;
                fprintf(stderr, "nrsc5_b200: stream %d output log overflowed (raise log_capacity)\n", s);
            }
        }
    }
    CK(cudaStreamSynchronize(e->stream));
    return rc ? rc : (truncated ? NRSC5B_EOVERFLOW : NRSC5B_OK);
}

extern "C" int nrsc5b_take_overflow(nrsc5b_engine_t *e, int stream)
{
    if (!e || stream < 0 || stream >= e->dims.nstreams) return NRSC5B_EINVAL;
    const int v = e->overflowed[stream];
    e->overflowed[stream] = 0;
    return v;
}

extern "C" int nrsc5b_set_sync_state(nrsc5b_engine_t *e, int stream, int state)
{
    if (!e || stream < 0 || stream >= e->dims.nstreams || state < 0 || state > 2) return NRSC5B_EINVAL;
    CK(cudaMemcpyAsync(reinterpret_cast<uint8_t *>(e->dp.st + stream) + offsetof(StreamState, force_state), &state,
                       sizeof(int), cudaMemcpyHostToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return NRSC5B_OK;
}

extern "C" int nrsc5b_get_stats(nrsc5b_engine_t *e, nrsc5b_stats_t *out)
{
    if (!e || !out) return NRSC5B_EINVAL;
    CK(cudaStreamSynchronize(e->stream));
    const int S = e->dims.nstreams;
    CK(cudaMemcpy(e->h_state, e->dp.st, sizeof(StreamState) * S, cudaMemcpyDeviceToHost));
    unsigned long long frames = 0, samples = 0, blocks = 0, fb = 0;
    for (int s = 0; s < S; s++) {
        fb += e->h_state[s].p1_fallbacks;
        frames += e->h_state[s].frames_done;
        blocks += e->h_state[s].blocks_done;
        samples += (unsigned long long)(2 * e->h_state[s].start);
    }
    e->stats.p1_frames = frames;
    e->stats.p1_fallbacks = fb;
    e->stats.blocks = blocks;
    e->stats.samples = samples;
    *out = e->stats;
    return NRSC5B_OK;
}

// ---- stage entry points ---------------------------------------------------
static int use_device(int device)
{
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device >= ndev) {
        fprintf(stderr, "nrsc5_b200: no usable CUDA device (the engine has no CPU path)\n");
        return NRSC5B_ENODEV;
    }
    if (cudaSetDevice(device) != cudaSuccess) return NRSC5B_ENODEV;
    return upload_tables(device);
}

extern "C" int nrsc5b_halfband_fm(int device, const uint8_t *cu8, size_t npairs, int16_t *out)
{
    int rc = use_device(device);
    if (rc) return rc;
    uint8_t *din = nullptr;
    short2 *dout = nullptr;
    CK(cudaMalloc(&din, 4 * npairs + 64));
    CK(cudaMalloc(&dout, npairs * sizeof(short2)));
    CK(cudaMemcpy(din, cu8, 4 * npairs, cudaMemcpyHostToDevice));
    launch_halfband_test(din, (long long)npairs, dout, 0);
    CK(cudaMemcpy(out, dout, npairs * sizeof(short2), cudaMemcpyDeviceToHost));
    cudaFree(din);
    cudaFree(dout);
    return NRSC5B_OK;
}

static int viterbi_k7_impl(int device, const int8_t *in, uint8_t *out, int len, int nframes, int *fallbacks);

extern "C" int nrsc5b_viterbi_k7(int device, const int8_t *in, uint8_t *out, int len, int nframes)
{
    return viterbi_k7_impl(device, in, out, len, nframes, nullptr);
}

/* Same, and reports how many frames the register-resident fast path handed to the exact fallback kernels. */
extern "C" int nrsc5b_viterbi_k7_ex(int device, const int8_t *in, uint8_t *out, int len, int nframes, int *fallbacks)
{
    return viterbi_k7_impl(device, in, out, len, nframes, fallbacks);
}

/* The register-resident fast path alone, with chunks of `ch` steps: its decision words (every one of the len + 64
 * steps) and its per-frame retry verdict - what the exact fallback would be asked to redo. */
extern "C" int nrsc5b_viterbi_k7_fast(int device, const int8_t *in, int len, int nframes, int ch, uint32_t *dec, int *retry)
{
    int rc = use_device(device);
    if (rc) return rc;
    if (len < 32 || (len % 32) || nframes <= 0 || ch < 32 || (ch % 32)) return NRSC5B_EINVAL;
    const int total = len + 64;
    V64Args b;
    b.stride = 1;
    b.len = len;
    b.ch = ch;
    b.nch = (total + ch - 1) / ch;
    b.dec_stride = (size_t)total;
    int8_t *din = nullptr;
    int *dflags = nullptr;                           // [ready | retry] x nframes
    CK(cudaMalloc(&din, (size_t)nframes * 3 * len));
    CK(cudaMemcpy(din, in, (size_t)nframes * 3 * len, cudaMemcpyHostToDevice));
    std::vector<int> fl(2 * (size_t)nframes, 0);
    for (int i = 0; i < nframes; i++) fl[i] = 1;
    CK(cudaMalloc(&dflags, fl.size() * sizeof(int)));
    CK(cudaMemcpy(dflags, fl.data(), fl.size() * sizeof(int), cudaMemcpyHostToDevice));
    b.vin = din;
    b.ready = dflags;
    b.retry = dflags + nframes;
    CK(cudaMalloc(&b.dec, (size_t)nframes * total * sizeof(uint2)));
    CK(cudaMalloc(&b.bitsw, (size_t)nframes * (len / 32) * sizeof(uint32_t)));
    CK(cudaMalloc(&b.vspec, (size_t)nframes * b.nch * 32 * sizeof(uint32_t)));
    CK(cudaMalloc(&b.vend, (size_t)nframes * b.nch * 32 * sizeof(uint32_t)));
    CK(cudaMalloc(&b.endstate, (size_t)nframes * sizeof(int)));
    CK(cudaFuncSetAttribute(k_v64_emit, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)V64_EMIT_SMEM));
    launch_v64(b, nframes, 0);
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(dec, b.dec, (size_t)nframes * total * sizeof(uint2), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(retry, b.retry, (size_t)nframes * sizeof(int), cudaMemcpyDeviceToHost));
    cudaFree(din); cudaFree(dflags); cudaFree(b.dec); cudaFree(b.bitsw);
    cudaFree(b.vspec); cudaFree(b.vend); cudaFree(b.endstate);
    return NRSC5B_OK;
}

static int viterbi_k7_impl(int device, const int8_t *in, uint8_t *out, int len, int nframes, int *fallbacks)
{
    int rc = use_device(device);
    if (rc) return rc;
    if (len < 32 || nframes <= 0) return NRSC5B_EINVAL;
    int8_t *din = nullptr;
    uint8_t *dout = nullptr;
    size_t nin = (size_t)nframes * 3 * len;
    CK(cudaMalloc(&din, nin));
    CK(cudaMalloc(&dout, (size_t)nframes * len));
    CK(cudaMemcpy(din, in, nin, cudaMemcpyHostToDevice));
    if (len >= 2048 && (len % 32) == 0) {
        // the engine's P1 path: register-resident fast decoder, then the exact fallback for flagged frames
        const int total = len + 64;
        int *dflags = nullptr;                       // [ready | slow | retry] x nframes
        CK(cudaMalloc(&dflags, (size_t)nframes * 3 * sizeof(int)));
        std::vector<int> fl(3 * (size_t)nframes, 0);
        for (int i = 0; i < nframes; i++) fl[i] = 1;
        CK(cudaMemcpy(dflags, fl.data(), fl.size() * sizeof(int), cudaMemcpyHostToDevice));
        uint32_t *dbw = nullptr;
        CK(cudaMalloc(&dbw, (size_t)nframes * (len / 32) * sizeof(uint32_t)));
        VitcArgs a;
        a.len = len;
        a.nch = (total + CH_LEN - 1) / CH_LEN;
        a.dec_stride = (size_t)a.nch * CH_LEN;
        a.ready_stride = 1;
        CK(cudaMalloc(&a.dec, (size_t)nframes * a.dec_stride * sizeof(uint2)));
        CK(cudaMalloc(&a.vspec, (size_t)nframes * a.nch * 16 * sizeof(uint2)));
        CK(cudaMalloc(&a.vend, (size_t)nframes * a.nch * 16 * sizeof(uint2)));
        CK(cudaMalloc(&a.tbend, (size_t)nframes * a.nch * sizeof(int)));
        CK(cudaMalloc(&a.hstate, (size_t)nframes * a.nch * sizeof(int)));
        a.vin = din;
        a.bitsw = dbw;
        a.ready = dflags + 2 * nframes;              // the fallback decodes the frames flagged `retry`
        a.slow = dflags + nframes;
        V64Args b;
        b.vin = din;
        b.dec = a.dec;
        b.bitsw = dbw;
        b.ready = dflags;
        b.retry = dflags + 2 * nframes;
        b.stride = 1;
        b.len = len;
        b.ch = len >= 16384 ? 1024 : 256;
        b.nch = (total + b.ch - 1) / b.ch;
        b.dec_stride = a.dec_stride;
        CK(cudaMalloc(&b.vspec, (size_t)nframes * b.nch * 32 * sizeof(uint32_t)));
        CK(cudaMalloc(&b.vend, (size_t)nframes * b.nch * 32 * sizeof(uint32_t)));
        CK(cudaMalloc(&b.endstate, (size_t)nframes * sizeof(int)));
        CK(cudaFuncSetAttribute(k_vitc_emit, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vitc_emit_smem()));
        CK(cudaFuncSetAttribute(k_v64_emit, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)V64_EMIT_SMEM));
        launch_v64(b, nframes, 0);
        launch_vitc(a, nframes, 0);
        {
            size_t nb = (size_t)nframes * len;
            k_vitc_unpack<<<(unsigned)((nb + 255) / 256), 256>>>(dbw, dout, nb);
        }
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(fl.data(), dflags, fl.size() * sizeof(int), cudaMemcpyDeviceToHost));
        if (fallbacks) {
            *fallbacks = 0;
            for (int i = 0; i < nframes; i++) *fallbacks += fl[2 * (size_t)nframes + i] != 0;
        }
        cudaFree(a.dec); cudaFree(a.vspec); cudaFree(a.vend); cudaFree(a.tbend); cudaFree(a.hstate); cudaFree(dflags); cudaFree(dbw);
        cudaFree(b.vspec); cudaFree(b.vend); cudaFree(b.endstate);
    } else {
        uint2 *ddec = nullptr;
        CK(cudaMalloc(&ddec, (size_t)nframes * (len + 64) * sizeof(uint2)));
        k_viterbi_test<<<nframes, 32>>>(din, dout, ddec, len);
        CK(cudaDeviceSynchronize());
        cudaFree(ddec);
    }
    CK(cudaMemcpy(out, dout, (size_t)nframes * len, cudaMemcpyDeviceToHost));
    cudaFree(din);
    cudaFree(dout);
    return NRSC5B_OK;
}

extern "C" int nrsc5b_rs_decode(int device, uint8_t *blocks, int *rcs, int n)
{
    int rc = use_device(device);
    if (rc) return rc;
    uint8_t *db = nullptr;
    int *dr = nullptr;
    CK(cudaMalloc(&db, (size_t)n * 255));
    CK(cudaMalloc(&dr, (size_t)n * sizeof(int)));
    CK(cudaMemcpy(db, blocks, (size_t)n * 255, cudaMemcpyHostToDevice));
    k_rs_test<<<(n + 3) / 4, 128>>>(db, dr, n);
    CK(cudaMemcpy(blocks, db, (size_t)n * 255, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(rcs, dr, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
    cudaFree(db);
    cudaFree(dr);
    return NRSC5B_OK;
}

/* The AM chain's K=9 rate-1/3 tail-biting decoder alone (reference src/conv_dec.c with K = 9, as decode.c:487,515-539
 * calls it): njobs frames of len bits, in = 3 * len hard symbols each (-1, 0 = punctured, +1), out = len bits each.
 * warmup <= 0: the production warm-up of the segmented traceback; rounds (optional, [njobs]) = repair rounds it took. */
extern "C" int nrsc5b_viterbi_k9(int device, const int8_t *in, uint8_t *out, int len, int njobs, unsigned g0, unsigned g1, unsigned g2,
                                 int warmup, int chunk_warmup, int *rounds)
{
    if (!in || !out || len < 32 || njobs < 1) return NRSC5B_EINVAL;
    for (size_t i = 0; i < (size_t)njobs * 3 * len; i++)
        if (in[i] < -1 || in[i] > 1) return NRSC5B_EINVAL;                 // the AM chain slices hard
    int rc = use_device(device);
    if (rc) return rc;
    const size_t dec_words = (size_t)((len + 64 + 2) / 3) * 32;
    int8_t *di = nullptr;
    uint8_t *dout = nullptr;
    uint32_t *dd = nullptr;
    int *dr = nullptr;
    CK(cudaMalloc(&di, (size_t)njobs * 3 * len));
    CK(cudaMalloc(&dout, (size_t)njobs * len));
    CK(cudaMalloc(&dd, (size_t)njobs * dec_words * 4));
    CK(cudaMalloc(&dr, (size_t)njobs * sizeof(int)));
    CK(cudaMemcpy(di, in, (size_t)njobs * 3 * len, cudaMemcpyHostToDevice));
    const size_t smem = nbam::VIT_TEST_SLOTS_BYTES + 4 * (size_t)nbam::VIT_TB_WORDS;
    CK(cudaFuncSetAttribute(k_am_vit_test, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_am_vit_test<<<njobs, nbam::AM_THREADS, smem>>>(di, dout, dd, dec_words, len, g0, g1, g2, warmup > 0 ? warmup : nbam::VIT_WARMUP,
                                                 chunk_warmup > 0 ? chunk_warmup : nbam::VIT_CHUNK_WARMUP, dr);
    CK(cudaGetLastError());
    CK(cudaMemcpy(out, dout, (size_t)njobs * len, cudaMemcpyDeviceToHost));
    if (rounds) CK(cudaMemcpy(rounds, dr, (size_t)njobs * sizeof(int), cudaMemcpyDeviceToHost));
    cudaFree(di);
    cudaFree(dout);
    cudaFree(dd);
    cudaFree(dr);
    return NRSC5B_OK;
}

/* L2 framing on the device for every frame the engine decodes from now on (FM and AM engines). */
extern "C" int nrsc5b_enable_l2(nrsc5b_engine_t *e, int on)
{
    if (!e) return NRSC5B_EINVAL;
    CK(cudaStreamSynchronize(e->stream));
    if (on && !e->l2) {
        int rc = dev_alloc(e, &e->l2, (size_t)e->dims.nstreams, false);
        if (rc) return rc;
        k_l2_init<<<e->dims.nstreams, 256, 0, e->stream>>>(e->l2, -1);
        CK(cudaGetLastError());
    }
    e->dims.l2 = on ? 1 : 0;
    return NRSC5B_OK;
}

/* L2 alone: frames = {u32 lc, u32 nbits, packed bits padded to 4 bytes} back to back, nbits == 0 = frame_reset
 * (reference src/frame.c:645 frame_push, :716 frame_reset); one REC_L2 record per frame into out. */
extern "C" long nrsc5b_l2_frames(int device, const uint8_t *frames, size_t nbytes, uint8_t *out, size_t cap, size_t *needed)
{
    int rc = use_device(device);
    if (rc) return rc;
    if (!frames || !out) return NRSC5B_EINVAL;
    std::vector<uint32_t> desc;
    size_t off = 0;
    while (off + 8 <= nbytes) {
        uint32_t h[2];
        memcpy(h, frames + off, 8);
        off += 8;
        desc.push_back((uint32_t)off);
        desc.push_back(h[0]);
        desc.push_back(h[1]);
        if (h[1] == 0) continue;
        if (h[0] > 2) return NRSC5B_EINVAL;                       // logical channel: P1, P3, P4 (L2State::ccc[3])
        const size_t nb = (h[1] + 7) / 8;
        if (off + nb > nbytes) return NRSC5B_EINVAL;
        off += (nb + 3) & ~(size_t)3;
    }
    const int nd = (int)(desc.size() / 3);
    if (nd == 0) { if (needed) *needed = 0; return 0; }
    nbl2::L2State *st = nullptr;
    uint8_t *df = nullptr, *dout = nullptr;
    uint32_t *dd = nullptr;
    unsigned *dlen = nullptr;
    unsigned lo[2] = { 0, 0 };
    auto run = [&]() -> int {
        CK(cudaMalloc(&st, sizeof(nbl2::L2State)));
        CK(cudaMalloc(&df, nbytes + 16));
        CK(cudaMalloc(&dd, desc.size() * sizeof(uint32_t)));
        CK(cudaMalloc(&dout, cap));
        CK(cudaMalloc(&dlen, 2 * sizeof(unsigned)));
        CK(cudaMemset(dlen, 0, 2 * sizeof(unsigned)));
        CK(cudaMemcpy(df, frames, nbytes, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(dd, desc.data(), desc.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
        k_l2_init<<<1, 256>>>(st, -1);
        k_l2_test<<<1, nbl2::L2_THREADS>>>(st, df, dd, nd, dout, cap, dlen);
        CK(cudaGetLastError());
        CK(cudaMemcpy(lo, dlen, sizeof(lo), cudaMemcpyDeviceToHost));
        if (lo[0]) CK(cudaMemcpy(out, dout, lo[0], cudaMemcpyDeviceToHost));
        return NRSC5B_OK;
    };
    rc = run();
    cudaFree(st); cudaFree(df); cudaFree(dd); cudaFree(dout); cudaFree(dlen);      // also on the error paths
    if (rc) return rc;
    if (needed) *needed = lo[0];
    return lo[1] ? (long)NRSC5B_EFULL : (long)lo[0];
}

extern "C" int nrsc5b_fft2048(int device, const float *in, float *out, int nffts)
{
    int rc = use_device(device);
    if (rc) return rc;
    float2 *di = nullptr, *dout = nullptr, *dtw = nullptr;
    size_t n = (size_t)nffts * NFFT;
    CK(cudaMalloc(&di, n * sizeof(float2)));
    CK(cudaMalloc(&dout, n * sizeof(float2)));
    CK(cudaMalloc(&dtw, FFT_TW * sizeof(float2)));
    std::vector<float2> tw = make_twiddles();
    CK(cudaMemcpy(dtw, tw.data(), FFT_TW * sizeof(float2), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(di, in, n * sizeof(float2), cudaMemcpyHostToDevice));
    launch_fft_test(di, dout, dtw, nffts, 0);
    CK(cudaMemcpy(out, dout, n * sizeof(float2), cudaMemcpyDeviceToHost));
    cudaFree(di);
    cudaFree(dout);
    cudaFree(dtw);
    return NRSC5B_OK;
}
