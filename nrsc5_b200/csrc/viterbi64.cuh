// Register-resident chunk-parallel Viterbi (K=7, rate 1/3, tail-biting): the fast path of the P1 decode.
//
// The reference decodes a frame with one sequential pass of len+64 add-compare-select steps (reference
// src/conv_dec.c:402-427, SSE kernel src/conv_sse.h:56-66,233-315).  Here
//
//   k_v64_fwd    one THREAD per chunk of `ch` steps: all 64 path metrics live in 32 registers as packed
//                u16x2, a step is 16 fully unrolled butterfly pairs with no cross-lane traffic at all, most
//                of them updating their registers in place; every chunk first replays V64_WARM warm-up
//                steps from all-zero metrics
//   k_v64_check  accepts the frame only if every chunk's warmed-up metric vector equals - up to one common
//                constant - the vector its predecessor ended with (equal vectors => equal decisions from
//                there on, so accepted decisions are exactly the sequential pass's); picks the end state
//   k_v64_emit   one warp per 1024-step window: the survivor state at the window's end is the one all 64
//                survivors of the following 128 steps merge into (checked, not assumed); 32 lanes then
//                emit 32 bits each from guessed segment end states that are verified against their
//                neighbours from the known window end downwards
//
// Anything that cannot be proven on this path (a chunk that did not converge, survivors that did not
// merge, metrics that could saturate in the reference's int16 arithmetic) flags the frame `retry`; it is
// then decoded by the exact half-warp kernels of viterbi_chunk.cuh.  Speculation only ever costs time.
//
// Arithmetic.  Add-compare-select decisions depend only on metric differences, so - as long as nothing
// saturates in the reference and nothing wraps here - they are unchanged by (a) adding the same bias to
// all branch metrics of a step and (b) subtracting a common constant from all path metrics.  With the
// bias V64_BIAS = 384 >= 3*127 every branch metric is positive, path metrics are unsigned, halves never
// carry into each other and plain 32-bit integer adds do two states at a time.  The minimum is subtracted
// every V64_NORM = 32 steps (a whole number of layout cycles, see V64State): right after that every metric is
// at most the spread 12*381 = 4572, and a branch metric adds at most 765, so the candidates X (even
// predecessor) and Y (odd) formed in the 32 steps up to the next subtraction stay below
// 4572 + 32*765 = 29052 < 2^15 (any interval up to 36 steps would).  In that range one DPX instruction
// (VIADDMNMX.U16x2) gives N = max(X, Y) per half, and  (Y + 0x8000 - N) >> 15  is the comparison  Y >= X
// (0 <= N - Y < 2^15: no borrow between the halves; ties: the odd predecessor wins, as in
// src/conv_gen.h:47,55).
//
// Decision word of a step (uint2 w): the bit of new state n is bit 8*(n>>4) + (n&7) of w.x (n&8 == 0) or
// w.y (n&8 != 0); set = the survivor comes from the odd predecessor 2*(n&31)+1.
#pragma once
#include <type_traits>
#include <utility>
#include "common.cuh"
#include "viterbi_chunk.cuh"

namespace nb {

constexpr int V64_WARM = 256;
constexpr int V64_NORM = 32;
constexpr int V64_GROUP = 8;                           // forward steps per loop iteration: two layout cycles
constexpr int V64_BIAS = 384;
constexpr int V64_WIN = 1024;                           // traceback window (steps per emit warp)
constexpr int V64_HEAD = 128;                           // look-ahead in which all survivors must merge
constexpr int V64_GUESS = 64;                           // look-ahead of a segment's (verified) end-state guess

struct V64Args {
    const int8_t *vin;      // [frames][3*len]
    uint2 *dec;             // [frames][dec_stride] decision words, one per step
    uint32_t *vspec;        // [frames][nch][32] metrics at each chunk start (after warm-up)
    uint32_t *vend;         // [frames][nch][32] metrics at each chunk end
    int *endstate;          // [frames] survivor state after the last step
    uint32_t *bitsw;        // [frames][len/32] decoded bits
    const int *ready;       // ready[f*stride] != 0 selects the frames to decode
    int *retry;             // retry[f*stride] = 1: decode this frame with the exact fallback kernels
    int stride;             // in ints
    int len;                // frame length in bits (multiple of 32)
    int ch;                 // chunk length in steps (multiple of 32)
    int nch;                // chunks per frame
    size_t dec_stride;      // uint2 per frame
};

__device__ __forceinline__ unsigned v64_umin(unsigned a, unsigned b)
{
    unsigned r;
#if defined(NB_EMU)
    r = emu_min_u16x2(a, b);
#else
    asm("min.u16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
#endif
    return r;
}
__device__ __forceinline__ unsigned v64_prmt(unsigned a, unsigned b, unsigned sel)
{
    unsigned r;
#if defined(NB_EMU)
    r = emu_prmt(a, b, sel);
#else
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
#endif
    return r;
}
// per halfword max(a + b, c), unsigned, the add wrapping modulo 2^16: one DPX VIADDMNMX.U16x2 on sm_90
__device__ __forceinline__ unsigned v64_addmax(unsigned a, unsigned b, unsigned c)
{
#if defined(NB_EMU)
    return emu_max_u16x2(emu_add_s16x2(a, b), c);
#else
    return __viaddmax_u16x2(a, b, c);
#endif
}
// |x| of each signed byte of x (|-128| = 128)
__device__ __forceinline__ unsigned v64_absb4(unsigned x)
{
#if defined(NB_EMU)
    unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        const int v = (int8_t)(x >> (8 * i));
        r |= (unsigned)(v < 0 ? -v : v) << (8 * i);
    }
    return r;
#else
    return __vabsdiffs4(x, 0u);
#endif
}

// sign pattern of butterfly b: expected code bits of the branch (state 2b, input 0), src/conv_dec.c:139-154
__host__ __device__ constexpr int v64_parity(unsigned v)
{
    return (int)((v ^ (v >> 1) ^ (v >> 2) ^ (v >> 3) ^ (v >> 4) ^ (v >> 5) ^ (v >> 6)) & 1u);
}
// the 3 code bits of butterfly b as a negation mask: bit 2-i set = the branch (state 2b, input 0) expects soft
// value i to be negative.  Its metric is BIAS + sum of +-s_i; the other branch into the same new state has mask ^ 7.
__host__ __device__ constexpr int v64_neg(int b)
{
    const unsigned reg = (unsigned)b << 1;
    return (v64_parity(reg & 0133u) ? 0 : 4) | (v64_parity(reg & 0171u) ? 0 : 2) | (v64_parity(reg & 0165u) ? 0 : 1);
}

// Metric layouts.  A step pairs the registers whose states differ in state bit 0.  Writing the two results back
// into the registers of their inputs moves every state bit k of the old layout to bit k-1 of the new states and
// bit 0 to the new bit 5: at phase J of the 4-step cycle, state bit k sits at bit (k + J) % 6 of the 6-bit
// location register | half << 5 (`v64_state`).  Phase 0 is the canonical P[i] = (pm[i], pm[i+32]).  Phases
// 0..2 update in place (a register renaming, no instructions); phase 3 re-packs into phase 0 with two PRMTs per
// pair.  In place, at most 4 steps could follow phase 0 before state bit 0 reached the half (where a step's two
// registers would be one); the cycle is 4 so that it divides the loop's step groups (4 steps = 12 bytes = 3
// aligned soft words), the chunk boundaries, the warm-up and V64_NORM, and every published vector is canonical.
__host__ __device__ constexpr int v64_state(int J, int reg, int half)     // state at (reg, half) in phase J
{
    const int x = reg | (half << 5);
    int n = 0;
    for (int k = 0; k < 6; k++) n |= ((x >> ((k + J) % 6)) & 1) << k;
    return n;
}

// 64-state path metrics of one chunk; phase 0 layout P[i] = (pm[i], pm[i+32]) as u16x2
struct V64State {
    unsigned P[32];

    // step at cycle phase J (layout J in, layout (J + 1) % 4 out); s0,s1,s2 = soft values; returns the decision word
    template <int J>
    __device__ __forceinline__ uint2 step(int s0, int s1, int s2)
    {
        // the two butterflies of a register differ in state bit H of their even predecessors, i.e. in bit H of
        // the encoder register: the soft values whose generator taps that bit change sign between the halves
        constexpr int H = 5 - J;
        constexpr int flip = (((0133 >> H) & 1) << 2) | (((0171 >> H) & 1) << 1) | ((0165 >> H) & 1);
        // 8 packed biased branch metrics M[m] = (BIAS + sum(+-s, m), BIAS + sum(+-s, m ^ flip)), as
        // (common part) * 0x10001 + (part that changes sign) * 0xFFFF0001 - exact, the low half never borrows
        unsigned M[8];
#pragma unroll
        for (int m = 0; m < 8; m++) {
            const int v0 = (m & 4) ? -s0 : s0, v1 = (m & 2) ? -s1 : s1, v2 = (m & 1) ? -s2 : s2;
            const int com = V64_BIAS + ((flip & 4) ? 0 : v0) + ((flip & 2) ? 0 : v1) + ((flip & 1) ? 0 : v2);
            const int dif = ((flip & 4) ? v0 : 0) + ((flip & 2) ? v1 : 0) + ((flip & 1) ? v2 : 0);
            M[m] = (unsigned)com * 0x10001u + (unsigned)dif * 0xFFFF0001u;
        }
        // Decision bits are gathered into accumulators A[] whose bytes each hold states of one byte of the
        // output word (bit n & 7) and are then moved into place: by byte permutes, and for J >= 2 - where the two
        // halves of a register are states of the same output byte and so go to two bytes of A - after
        // merging byte pairs with one multiply by 0x101 (the two bytes hold disjoint bits: no carries).
        auto acc_of = [](int n) -> int {
            return J == 0 ? (n >> 3) & 1 : J == 1 ? (n >> 4) & 1 : ((n >> 3) & 1) | (((n >> 4) & 1) << 1);
        };
        auto byte_of = [](int n) -> int {
            return J == 0 ? n >> 4 : J == 1 ? ((n >> 5) & 1) | (((n >> 3) & 1) << 1)
                                            : (((n >> 5) & 1) << 1) | ((n >> (4 - J)) & 1);
        };
        unsigned A[4] = { 0, 0, 0, 0 };
        unsigned N[32];
#pragma unroll
        for (int l = 0; l < 16; l++) {
            const int rE = ((l >> J) << (J + 1)) | (l & ((1 << J) - 1)), rO = rE | (1 << J);
            const unsigned E = P[rE], O = P[rO];
            const int b = v64_state(J, rE, 0) >> 1, bh = v64_state(J, rE, 1) >> 1;     // butterflies lo, hi
            const unsigned Mp = M[v64_neg(b)], Mm = M[v64_neg(b) ^ 7];
            const unsigned Y1 = O + Mm, Y2 = O + Mp;
            const unsigned N0 = v64_addmax(E, Mp, Y1), N1 = v64_addmax(E, Mm, Y2);     // new b, bh | +32
            const unsigned T1 = Y1 + 0x80008000u - N0, T2 = Y2 + 0x80008000u - N1;     // bit 15/31: Y >= X
            // new states of T1 lo, T1 hi, T2 lo, T2 hi; PRMT selector nibbles 9,B,D,F = sign of T byte 1,3,5,7
            const int st[4] = { b, bh, b | 32, bh | 32 };
            unsigned sel = 0, mask = 0;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                sel |= (unsigned)(9 + 2 * i) << (4 * byte_of(st[i]));
                mask |= 1u << (8 * byte_of(st[i]) + (st[i] & 7));
            }
            A[acc_of(b)] |= v64_prmt(T1, T2, sel) & mask;
            if constexpr (J < 3) {
                N[rE] = N0;
                N[rO] = N1;
            } else {
                N[b] = v64_prmt(N0, N1, 0x5410);
                N[bh] = v64_prmt(N0, N1, 0x7632);
            }
        }
#pragma unroll
        for (int i = 0; i < 32; i++) P[i] = N[i];
        if constexpr (J == 0) {
            return make_uint2(A[0], A[1]);
        } else if constexpr (J == 1) {
            return make_uint2(v64_prmt(A[0], A[1], 0x5140), v64_prmt(A[0], A[1], 0x7362));
        } else {
#pragma unroll
            for (int i = 0; i < 4; i++) A[i] *= 0x101u;
            return make_uint2(v64_prmt(A[0], A[2], 0x7351), v64_prmt(A[1], A[3], 0x7351));
        }
    }

    __device__ __forceinline__ void normalise()
    {
        unsigned m = P[0];
#pragma unroll
        for (int i = 1; i < 32; i++) m = v64_umin(m, P[i]);
        m = v64_umin(m, v64_prmt(m, 0, 0x1032));
#pragma unroll
        for (int i = 0; i < 32; i++) P[i] -= m;
    }
};

__device__ __forceinline__ int v64_prev(int state, uint2 w)
{
    const unsigned word = (state & 8) ? w.y : w.x;
    return ((state << 1) & 62) | (int)((word >> (8 * (state >> 4) + (state & 7))) & 1u);
}

// f(integral_constant<int, K>) for K = 0, 1, ...: loop bodies whose layout phase is a template argument
template <class F, int... K>
__device__ __forceinline__ void v64_unroll(F &f, std::integer_sequence<int, K...>)
{
    (f(std::integral_constant<int, K>{}), ...);
}

// ---------------------------------------------------------------------------
// forward pass: one thread per chunk
// ---------------------------------------------------------------------------
constexpr int V64_FWD_THREADS = 128;                   // 4 warps: one per warp scheduler of an SM

__global__ void __launch_bounds__(V64_FWD_THREADS) k_v64_fwd(V64Args a)
{
    const int f = blockIdx.y;
    if (!a.ready[(size_t)f * a.stride]) return;
    const int c = blockIdx.x * V64_FWD_THREADS + threadIdx.x;
    if (c >= a.nch) return;
    const int total = a.len + 64;
    const int8_t *vin = a.vin + (size_t)f * 3 * a.len;
    uint2 *dec = a.dec + (size_t)f * a.dec_stride;
    const int s_begin = c * a.ch, s_end = min(total, s_begin + a.ch);
    // saturation guard (see viterbi_chunk.cuh): between two of the reference's normalisations (every 79
    // steps) the metrics grow by at most the sum of |s0|+|s1|+|s2|; with a spread of at most 12*381 after
    // a normalisation, sums <= 32767 - 12*381 cannot saturate.  Every 79-step window lies inside the
    // range (warm-up included) of at least one chunk, which compares it when it reaches the window's
    // closing normalisation; the frame's last window has none, so the chunk that ends the frame compares
    // it after its last step.
    const int sat_limit = 32767 - 12 * 381;
    int wsum = 0;
    bool bad = false;

    V64State vs;
#pragma unroll
    for (int i = 0; i < 32; i++) vs.P[i] = 0;

    // V64_GROUP steps (3 soft bytes each) per iteration, whole cycles of metric layouts: the unrolled body must
    // stay inside the 32 KB instruction cache, one warp per scheduler cannot hide instruction fetches.  The
    // next iteration's words are loaded one iteration ahead.  Each iteration starts and ends in the canonical
    // layout, so the published vectors and the normalisation see P[i] = (pm[i], pm[i+32]).
    static_assert(V64_GROUP % 4 == 0 && 32 % V64_GROUP == 0 && V64_WARM % V64_GROUP == 0 && V64_NORM % V64_GROUP == 0,
                  "groups are whole layout cycles and tile chunks (multiples of 32 steps), the warm-up and V64_NORM");
    constexpr int GW = 3 * V64_GROUP / 4;               // soft words per group
    const uint32_t *vw = reinterpret_cast<const uint32_t *>(vin);
    const int fw = 3 * a.len / 4;                       // soft words per frame
    // step g reads bit (g - 32) mod len: jw = its first soft word, advanced group by group
    auto fetch = [&](int g, int &jw, uint32_t (&x)[GW]) {
        if (g >= 0 && g < s_end) {
#pragma unroll
            for (int i = 0; i < GW; i++) x[i] = vw[jw + i];
        } else {
#pragma unroll
            for (int i = 0; i < GW; i++) x[i] = 0;
        }
        jw = jw + GW >= fw ? jw + GW - fw : jw + GW;
    };
    const int g_first = s_begin - V64_WARM;
    int wc = ((g_first % 79) + 79) % 79;               // index modulo 79 of the group's first step
    int jw = 3 * (((g_first - 32) % a.len + a.len) % a.len) / 4;
    uint32_t nw[GW];
    fetch(g_first, jw, nw);
#pragma unroll 1
    for (int g0 = g_first; g0 < s_end; g0 += V64_GROUP) {
        uint32_t sw[GW];
#pragma unroll
        for (int i = 0; i < GW; i++) sw[i] = nw[i];
        fetch(g0 + V64_GROUP, jw, nw);
        const bool store = g0 >= s_begin;
        // saturation guard per group: |s| of the group's soft bytes, bytewise; at most one of the reference's
        // normalisations (after the step with index = 0 mod 79, src/conv_dec.c:419) falls into it
        uint32_t u[GW];
        int gsum = 0;
#pragma unroll
        for (int i = 0; i < GW; i++) {
            u[i] = v64_absb4(sw[i]);
            gsum = (int)__dp4a(u[i], 0x01010101u, (unsigned)gsum);
        }
        if (wc == 0 || wc > 79 - V64_GROUP) {
            const int nb = 3 * (wc == 0 ? 1 : 80 - wc);    // soft bytes up to and including that step
            int head = 0;
#pragma unroll
            for (int i = 0; i < GW; i++) {                 // dp4a weights: word i's bytes among the first nb
                const int k = min(max(nb - 4 * i, 0), 4);
                head = (int)__dp4a(u[i], k ? 0x01010101u >> (8 * (4 - k)) : 0u, (unsigned)head);
            }
            bad |= wsum + head > sat_limit;
            wsum = gsum - head;
        } else {
            wsum += gsum;
        }
        wc = wc + V64_GROUP >= 79 ? wc + V64_GROUP - 79 : wc + V64_GROUP;
        uint2 held = make_uint2(0, 0);
        auto one = [&](auto kc) {
            constexpr int k = decltype(kc)::value;
            auto sb = [&](int pos) -> int {               // sign-extended byte `pos` of the group
                const unsigned sel = (unsigned)(pos & 3) * 0x1111u | 0x8880u;
                return (int)v64_prmt(sw[pos >> 2], 0, sel);
            };
            const int s0 = sb(3 * k), s1 = sb(3 * k + 1), s2 = sb(3 * k + 2);
            const uint2 w = vs.template step<k % 4>(s0, s1, s2);
            if (k & 1) {
                if (store) *reinterpret_cast<uint4 *>(dec + g0 + k - 1) = make_uint4(held.x, held.y, w.x, w.y);
            } else {
                held = w;
            }
        };
        v64_unroll(one, std::make_integer_sequence<int, V64_GROUP>{});
        if (((g0 + V64_GROUP) & (V64_NORM - 1)) == 0) vs.normalise();
        if (g0 + V64_GROUP == s_begin) {                   // warm-up done: publish the speculative start vector
            uint32_t *o = a.vspec + ((size_t)f * a.nch + c) * 32;
#pragma unroll
            for (int i = 0; i < 32; i++) o[i] = vs.P[i];
        }
    }
    if (s_end == total) bad |= wsum > sat_limit;
    {
        uint32_t *o = a.vend + ((size_t)f * a.nch + c) * 32;
#pragma unroll
        for (int i = 0; i < 32; i++) o[i] = vs.P[i];
    }
    if (bad) atomicExch(&a.retry[(size_t)f * a.stride], 1);
}

// ---------------------------------------------------------------------------
// check: one CTA per frame; warp w verifies chunks w, w+nwarps, ...; warp 0 also picks the end state
// ---------------------------------------------------------------------------
constexpr int V64_CHECK_THREADS = 256;

__global__ void __launch_bounds__(V64_CHECK_THREADS) k_v64_check(V64Args a)
{
    const int f = blockIdx.x;
    if (!a.ready[(size_t)f * a.stride]) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = V64_CHECK_THREADS / 32;
    const uint32_t *vspec = a.vspec + (size_t)f * a.nch * 32, *vend = a.vend + (size_t)f * a.nch * 32;
    bool ok = true;
    for (int c = 1 + warp; c < a.nch; c += nwarps) {
        const unsigned x = vend[(size_t)(c - 1) * 32 + lane], y = vspec[(size_t)c * 32 + lane];
        // equal up to one constant added to all 64 metrics (reference point: state 0)
        const int xr = (int)(__shfl_sync(0xffffffffu, x, 0) & 0xffff), yr = (int)(__shfl_sync(0xffffffffu, y, 0) & 0xffff);
        ok &= ((int)(x & 0xffff) - xr == (int)(y & 0xffff) - yr) && ((int)(x >> 16) - xr == (int)(y >> 16) - yr);
    }
    if (!__all_sync(0xffffffffu, ok) && lane == 0) atomicExch(&a.retry[(size_t)f * a.stride], 1);
    if (warp == 0) {
        // first maximum in state order (reference src/conv_dec.c:310-317); lane i holds states i and i+32
        const unsigned x = vend[(size_t)(a.nch - 1) * 32 + lane];
        int v = (int)(x & 0xffff), idx = lane;
        const int v2 = (int)(x >> 16);
        if (v2 > v) { v = v2; idx = lane + 32; }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const int ov = __shfl_xor_sync(0xffffffffu, v, o), oi = __shfl_xor_sync(0xffffffffu, idx, o);
            if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
        }
        if (lane == 0) a.endstate[f] = idx;
    }
}

// ---------------------------------------------------------------------------
// emit: one warp per 1024-step window
// ---------------------------------------------------------------------------
constexpr int V64_EMIT_WARPS = 4;
constexpr int V64_EMIT_STEPS = V64_WIN + V64_HEAD;
// staged decisions are padded by one word per 32 steps: the lanes walk segments 32 steps apart at the same time
constexpr int V64_EMIT_LD = V64_EMIT_STEPS + V64_EMIT_STEPS / 32 + 1;
constexpr size_t V64_EMIT_SMEM = (size_t)V64_EMIT_WARPS * V64_EMIT_LD * sizeof(uint2);
__device__ __forceinline__ int v64_pad(int q) { return q + (q >> 5); }

__global__ void __launch_bounds__(V64_EMIT_WARPS * 32) k_v64_emit(V64Args a)
{
#if defined(NB_EMU)
    unsigned char *v64_smem = emu::dyn_smem();
#else
    extern __shared__ __align__(16) unsigned char v64_smem[];
#endif
    const int f = blockIdx.y;
    if (!a.ready[(size_t)f * a.stride]) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int total = a.len + 64;
    const int w = blockIdx.x * V64_EMIT_WARPS + warp;
    const int lo = w * V64_WIN;
    if (lo >= total) return;
    uint2 *sd = reinterpret_cast<uint2 *>(v64_smem) + (size_t)warp * V64_EMIT_LD;
    const uint2 *dec = a.dec + (size_t)f * a.dec_stride + lo;
    const int n = min(total - lo, V64_WIN);             // steps of this window
    const int nst = min(total - lo, V64_EMIT_STEPS);    // staged steps (incl. look-ahead)
    for (int i = lane; i < nst; i += 32) sd[v64_pad(i)] = dec[i];
    __syncwarp();
    auto walk = [&](int state, int from, int to) {      // state after local step `from` -> state after local step `to`
        for (int q = from; q > to; q--) state = v64_prev(state, sd[v64_pad(q)]);
        return state;
    };
    // the window's end state: the frame's end state for the last window, otherwise the state all survivors
    // of the look-ahead merge into
    int true_end;
    if (nst == n) {
        true_end = a.endstate[f];
    } else {
        // all 64 survivors (two per lane) of a look-ahead of 64 steps, else of the whole staged look-ahead
        bool merged = false;
        int ref = 0;
        for (int look = min(V64_HEAD / 2, nst - n); ; look = nst - n) {
            int e0 = lane, e1 = lane + 32;
            for (int q = n + look - 1; q > n - 1; q--) {
                const uint2 w = sd[v64_pad(q)];
                e0 = v64_prev(e0, w);
                e1 = v64_prev(e1, w);
            }
            ref = __shfl_sync(0xffffffffu, e0, 0);
            merged = __all_sync(0xffffffffu, e0 == ref && e1 == ref);
            if (merged || look == nst - n) break;
        }
        if (!merged) {
            if (lane == 0) atomicExch(&a.retry[(size_t)f * a.stride], 1);
            return;
        }
        true_end = ref;
    }
    const int seg_end = 32 * lane + 31;                 // local index of this lane's last step
    const bool have = 32 * lane < n;
    int g;                                              // state after local step seg_end
    if (!have) g = 0;
    else if (seg_end >= n - 1) g = true_end;
    else if (seg_end + V64_GUESS >= nst) g = walk(true_end, n - 1, seg_end);         // near the frame end
    else g = walk(0, seg_end + V64_GUESS, seg_end);                                 // guess
    unsigned word = 0;
    int b = 0;                                          // state before the segment's first step
    auto emit = [&](int gstate) {
        int state = gstate;
        unsigned ww = 0;
        for (int k = 31; k >= 0; k--) {
            ww |= (unsigned)((state >> 5) & 1) << k;
            state = v64_prev(state, sd[33 * lane + k]);
        }
        word = ww;
        b = state;
    };
    if (have) emit(g);
    // verification from the window end downwards
    const int nseg = (n + 31) / 32;
    for (;;) {
        const int bnext = __shfl_down_sync(0xffffffffu, b, 1);
        const bool wrong = have && lane < nseg - 1 && g != bnext;
        const unsigned m = __ballot_sync(0xffffffffu, wrong);
        if (!m) break;
        const int jj = 31 - __clz(m);                   // highest wrong segment: its right neighbour is already final
        if (lane == jj) { g = bnext; emit(g); }
    }
    const int widx = (lo >> 5) + lane - 1;              // frame bit 32*widx = step lo + 32*lane - 32
    if (have && widx >= 0 && widx < a.len / 32) a.bitsw[(size_t)f * (a.len / 32) + widx] = word;
}

}  // namespace nb
