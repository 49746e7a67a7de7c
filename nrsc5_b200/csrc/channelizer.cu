// Wideband channeliser (SURVEY §8 f3): one cu8 capture at 32 x 744 187.5 = 23 814 000 S/s -> up to hundreds of
// FM channels at 744 187.5 S/s cs16, written straight into the receive engine's cs16 input buffers.  The reference has
// no such stage (its ingest is one narrowband device per handle, reference src/nrsc5.c:130-207, src/rtltcp.c); this is
// the step in front of input_push_cs16 (src/input.c:119-124) that makes "many channels per GPU" a physical workload.
//
// It is the one dense contraction of the whole system, and the one kernel here that runs on the tensor cores:  for
// channel k and output sample n
//
//     acc[k][n] = sum_{u < 256} W_k[u] * (x[32 n + u] - (127 + 127j))        W_k[u] = round(2^19 h[255-u] e^{-j 2 pi 50 m_k u / 11907})
//     y[k][n]   = sat16( ((acc + 2^12) >> 13) * conj(P[(1600 m_k n) mod 11907]) + 2^14 >> 15 )
//
// (m_k = the channel's offset from the capture centre in units of 100 kHz; 100 kHz / 23.814 MHz = 50 / 11907, so
// every phasor comes from ONE table P[i] = round(32767 e^{+j 2 pi i / 11907}); all arithmetic is integer, the rounding
// shifts are arithmetic - the definition is exact and tests/test_channelizer.py restates it in numpy.)
//
// As a GEMM:  D[n][r] = sum_kappa A[n][kappa] * B[r][kappa],  kappa = 2u + {0: real, 1: imaginary part of x}
//   A[n][.]  = the 512 raw capture bytes starting at byte 64 n           (unsigned 8-bit, straight from the capture:
//              the rows overlap - row n+1 starts 64 bytes after row n - so the capture is addressed as a [rows][64 B]
//              matrix and K chunk c of row n is matrix row n + c: eight TMA boxes per tile, no im2col pass)
//   B[r][.]  = per channel four rows: {real, imaginary} x {high, low byte} of the 16-bit taps (signed 8-bit; the
//              real row holds Wr, -Wi alternating, the imaginary row Wi, Wr).  Channel cl = 4 p + q of the group owns
//              rows 16 p + 2 q + {0: real, 1: imaginary} (high bytes) and the same + 8 (low bytes): in the wgmma
//              accumulator layout, where lane q = lane % 4 holds columns 8 j + 2 q, +1 of every 8-column block j,
//              one thread then holds all four sums of its channels and the epilogue needs no shuffles.
//   D        = int32 in registers; acc = 256 * D_high + D_low - 127 * (sum of the row), the last term a per-channel constant
// Hopper wgmma (u8 x s8 -> s32), M = 64 output samples x N = 128 rows (32 channels) x K = 512 per tile, both operands
// K-major in shared memory with the 64-byte swizzle.  One persistent CTA per (channel group, tile slot), three
// warpgroups: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers that take the CTA's tiles in
// turn, each issuing its tile's 16 wgmmas and then running the epilogue from its own registers (rounding, rotation,
// saturation -> cs16 stores) while the other consumer's wgmmas run.  The 32 channels' taps (64 KB) stay in shared
// memory for the CTA's lifetime; capture tiles go through a ring of four 32 KB stages.
//
// cs16 input (nrsc5b_chan_*_cs16): the same taps, phasor table, mixer index and output rounding, but no offset and
// unit gain (1 output LSB per input LSB):
//
//     acc[k][n] = sum_{u < 256} W_k[u] * x[32 n + u]                              (exact: |acc| < 2^36)
//     v         = sat16((acc + 2^18) >> 19)
//     y[k][n]   = sat16((v * conj(P[(1600 m_k n) mod 11907]) + 2^14) >> 15)
//
// For x16 = 64 (x8 - 127) this is the cu8 definition bit for bit: (64 a + 2^18) >> 19 == (a + 2^12) >> 13, and the cu8
// filter output stays below 2^28 (the table check below), so |v| < 2^15 there and sat16 does nothing.  On cs16 input
// near full scale |v| reaches about 2^16 (sum |h| = 1.40); the saturation keeps the rotation's products in 32 bits.
// The kernel splits every sample as x = 256 x_hi + x_lo (x_hi signed, x_lo unsigned bytes) into two planes laid out
// like a cu8 capture (k_split_cs16, into handle-owned staging: TMA cannot address the bytes of an int16), reduces the
// x_hi plane (wgmma s8 x s8) to A1 = sum W x_hi (|A1| < 2^28) in 32 registers, then the x_lo plane (wgmma u8 x s8)
// to A2 = sum W x_lo (|A2| < 2^29) in the 64 accumulators, and combines acc = 256 A1 + A2 in exact 32-bit pieces
// before the shared epilogue.  A tile's two planes take two consecutive stages of the ring.
//
// AM band plan (nrsc5b_chan_create_am*): one capture at 32 x 46 511.71875 = 1 488 375 S/s, the rate the reference asks
// of an AM device, spans +-744 kHz - the whole medium-wave band - and goes to 10 kHz channels at 46 511.71875 S/s cs16,
// what an AM engine reads.  10 kHz / 1 488 375 Hz = 80 / 11907: the same phasor table P.  m_k = the offset in 10 kHz
// steps, |m_k| <= 74:
//
//     W_k[u]  = round(2^19 h_am[511-u] conj(P[(80 m_k u) mod 11907]) / 32767)            u < 512
//     cu8:   acc = sum_{u<512} W_k[u] (x[32 n + u] - (127+127j));  v = (acc + 2^12) >> 13
//     cs16:  acc = sum_{u<512} W_k[u]  x[32 n + u];                v = sat16((acc + 2^18) >> 19)
//     y[k][n] = sat16((v conj(P[(2560 m_k n) mod 11907]) + 2^14) >> 15)
//     N_am(T) = T >= 512 ? (T - 512) / 32 + 1 : 0;   carry = the samples from 32 N_am(T) on (<= 511 samples)
//
// h_am: 512-tap Kaiser-windowed sinc (-6 dB at 23 kHz, beta 8.8), unit DC gain.  Measured on the integer taps of
// channel 0: within +-0.001 dB up to 15 kHz, 87.1 dB down from 31.5 kHz on (tests/test_channelizer_am.py holds them to
// +-0.25 dB and 80 dB).  FM's 256 taps would give about 48 dB there, and in a hybrid AM signal the digital carriers sit
// 30 - 50 dB under an analog carrier, the aliases of the stations k x 46.5 kHz away a few kHz off centre, on top of them.
// The tap scale stays 2^19 (the bounds are re-derived at make_tables), the cu8 gain 64 output LSB per input LSB.
// In the kernel the second 256 taps are the same GEMM on capture-matrix rows 8 further on: KPASS = 2 passes of K = 512
// into the same accumulators (16 TMA boxes and 32 wgmmas per tile and plane).  Shared memory: both tap halves resident
// (131 072 B) + two 32 KB stages (65 536 B), one per consumer warpgroup, which a tile's passes and planes go through
// one after the other + alignment, barriers and epilogue tables (25 744 B) = 222 352 B, the same total as the FM
// instantiation's 64 KB of taps + four stages.  A consumer's loads and wgmmas therefore alternate; what overlaps is
// the other consumer's loads, wgmmas and epilogue.  The input is 1/16 of the FM rate: residency, not speed, is the limit.
//
// FM plans at 11 907 000 and 5 953 500 S/s (nrsc5b_chan_create_fm*, D = 16 and 8; D = 32 is the FM plan above): the
// same output rate, output mixer and epilogue, 256 taps at scale 2^14 D (the prototype's peak doubles each time D halves),
//
//     W_k[u] = round(2^14 D h_D[255-u] conj(P[((1600/D) m_k u) mod 11907]) / 32767)
//     cu8:   v = (acc + 2^(s-1)) >> s,  s = 13 - log2(32/D);   cs16:  v = sat16((acc + 2^(t-1)) >> t),  t = 19 - log2(32/D)
//     N_D(T) = T >= 256 ? (T - 256) / D + 1 : 0
//
// with the window of output n at x[D n ..].  In the kernel Q = 32 / D outputs share a capture-matrix row; Q tensor maps
// over the same memory, 2 D bytes apart, feed the phase-major boxes of a tile (k_channelize's Q).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <vector>

#include "../../include/nrsc5_b200.h"
#include "chan_feed.h"
#include "chan_scan.h"

namespace nbch {

constexpr int DECIM = 32, PASS_TAPS = 256, KBYTES = 2 * PASS_TAPS; // one pass: 256 taps, 512 bytes of K per output row (FM: one pass, AM: two)
constexpr int CHUNK = 64, NCHUNK = KBYTES / CHUNK;               // K chunks of 64 bytes (one capture-matrix row each) per pass
constexpr int TILE_M = 64;                                        // output samples per tile (one warpgroup's wgmma M)
constexpr int GROUP = 32, TILE_N = 4 * GROUP;                    // channels per CTA, rows of B
constexpr int PERIOD = 11907;                                     // phasor table length (100 kHz / 23.814 MHz = 50 / 11907)
constexpr int SHIFT1 = 13, TAP_SCALE_LOG2 = 19;                   // unit DC gain -> 64 LSB per input LSB (the cu8 -> Q15 convention);
                                                                  // taps stay below 127 * 256 + 127: both bytes of the split are int8
constexpr int THREADS = 384;                                      // producer warpgroup + two consumer warpgroups
constexpr int STAGES = 4;                                         // most capture stages a ring has (the barriers are laid out for it)
constexpr uint32_t A_STAGE_BYTES = NCHUNK * TILE_M * CHUNK;      // 32768: one pass of one plane of a tile
constexpr uint32_t W_BYTES = NCHUNK * TILE_N * CHUNK;            // 65536: one pass of a group's taps
constexpr int HALF = PERIOD / 2 + 1;                              // phasor table entries 0 .. 5953; the rest are their conjugates
// half table, rotation steps, offset corrections, destination offsets
constexpr uint32_t EPI_BYTES = ((HALF * 4 + 15) & ~15) + GROUP * 4 + 2 * GROUP * 4 + GROUP * 8;
// KPASS = 1 (256 taps): 64 KB of taps + four stages = 222 352 B.  KPASS = 2 (512 taps): both tap halves stay resident
// (128 KB), which leaves room for a ring of two stages - again 222 352 B - that a tile's passes and planes go through
// one after the other.
constexpr int stages_of(int kpass) { return kpass == 1 ? STAGES : 2; }
constexpr uint32_t smem_bytes(int kpass)
{
    return kpass * W_BYTES + stages_of(kpass) * A_STAGE_BYTES + 1024 /* alignment */ + 256 /* barriers */ + EPI_BYTES;
}
static_assert(smem_bytes(1) <= 227 * 1024 && smem_bytes(2) <= 227 * 1024, "more shared memory than an H100 block may have");
// cs16: the byte planes of up to PLANE_SAMPLES samples, x_hi rows first, then x_lo rows (one TMA map over both)
constexpr long long PLANE_SAMPLES = (1ll << 22) + 256;
constexpr int PLANE_ROWS = (int)(2 * PLANE_SAMPLES / CHUNK);
// outputs per launch of the one-shot cs16 entry: D n + taps - D <= PLANE_SAMPLES (2^22 / D with 256 taps, 2^17 - 7 with
// 512 taps at D = 32)
constexpr long long piece_out(int taps, int decim)
{
    return (PLANE_SAMPLES - taps) / decim + 1 < (1ll << 22) / decim ? (PLANE_SAMPLES - taps) / decim + 1 : (1ll << 22) / decim;
}
static_assert(piece_out(256, 32) == 1ll << 17 && DECIM * piece_out(512, 32) + 512 - DECIM <= PLANE_SAMPLES, "a one-shot piece must fit the planes");
static_assert(8 * piece_out(256, 8) + 256 - 8 <= PLANE_SAMPLES && 16 * piece_out(256, 16) + 256 - 16 <= PLANE_SAMPLES, "a one-shot piece must fit the planes");

struct Params {
    int nch;                   // channels
    int ngroups;
    int n0mod;                 // (absolute index of this launch's output 0) mod 11907: the mixer runs on across launches
    long long nout;            // output samples per channel
    long long tiles;           // ceil(nout / TILE_M)
    int16_t *out;              // cs16 (I, Q interleaved): output n of channel k goes to out + dst[k] + 2 n
    const long long *dst;      // [nch] int16 offsets of each channel's output 0; null: dst[k] = k * out_stride
    size_t out_stride;
    const int *rot_step;       // [nch] (1600 m_k) mod 11907 (AM plan: 2560 m_k)
    const long long *corr;     // [nch][2] 127 * (sum Wr - sum Wi), 127 * (sum Wi + sum Wr)   (already in acc units)
    const short2 *phasor;      // [PERIOD]
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity)
{
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                     smem_u32(dst)),
                 "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
// K-major operand tile in shared memory, 64-byte rows, SWIZZLE_64B: 8-row groups 512 bytes apart
__device__ __forceinline__ uint64_t wgmma_desc_sw64(const void *tile, uint32_t byte_offset)
{
    const uint32_t addr = smem_u32(tile) + byte_offset;
    uint64_t d = 0;
    d |= (uint64_t)((addr & 0x3FFFFu) >> 4);                 // start address
    d |= (uint64_t)1 << 16;                                    // leading byte offset (unused for swizzled K-major): 1
    d |= (uint64_t)(512u >> 4) << 32;                          // stride byte offset: 8 rows x 64 B
    d |= (uint64_t)2 << 62;                                    // layout type SWIZZLE_64B
    return d;
}
// D (64 x 128 int32, this thread's 64 of them) += A (64 x 32 capture bytes, unsigned) * B (128 x 32 tap bytes, signed)^T;
// accumulate = 0 overwrites D
__device__ __forceinline__ void wgmma_u8s8(uint32_t (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
        "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(da), "l"(db), "r"(accumulate)
        : "memory");
}
// the same with a signed A (the x_hi plane of a cs16 capture)
__device__ __forceinline__ void wgmma_s8s8(uint32_t (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
        "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "
        "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(da), "l"(db), "r"(accumulate)
        : "memory");
}

struct Barriers {
    uint64_t w_full, a_full[STAGES], a_empty[STAGES];
};

// The ring: unit `it` of a CTA's sequence (a tile's U = PLANES * KPASS stages in a row, the tiles going to the two
// consumers in turn) lands in stage ring_stage(it), which has been filled ring_use(it) times before.  A thread may only
// wait for a barrier phase if it has seen the one before (a wait for the parity of a phase that has not begun passes at
// once), so a stage is only ever read by one consumer.  KPASS = 1: four stages taken round robin - U divides 2, so
// consumer w gets stages w, w + 2 (cu8) or 2 w, 2 w + 1 (cs16).  KPASS = 2: two stages, stage w is consumer w's, and
// its units pass through it one at a time.
template <int U, int KPASS>
__device__ __forceinline__ int ring_stage(unsigned it) { return KPASS == 1 ? it % STAGES : (it / U) & 1; }
template <int U, int KPASS>
__device__ __forceinline__ unsigned ring_use(unsigned it) { return KPASS == 1 ? it / STAGES : (it / (2 * U)) * U + it % U; }

// The capture matrix as Q = 32 / D tensor maps over the same memory: map p starts at byte 2 D p (0 | 0, 32 | 0, 16,
// 32, 48: all 16-byte aligned, as TMA requires), so output n = Q j + p reads rows j .. j + 7 of map p.
template <int Q>
struct XMaps {
    CUtensorMap m[Q];
};

// CS16: the maps address the two byte planes of a cs16 capture, the x_lo plane PLANE_ROWS rows after the x_hi plane.
// KPASS: K = 512 passes per output row (256 taps each).  Pass ps of output n reads capture-matrix rows n + 8 ps ..
// n + 8 ps + 7 against tap chunks 8 ps .. 8 ps + 7 and adds into the same accumulators, so a 512-tap tile is two
// stages of the ring per plane; with cs16 the x_hi plane is folded into A1 after all its passes, then the x_lo plane runs.
// Q = 32 / D: consecutive outputs 2 D bytes apart, Q per capture-matrix row.  A tile is still 64 consecutive outputs;
// its stage is filled phase-major, every K chunk as Q boxes of 64 / Q rows (a multiple of the 8-row swizzle atom),
// box p holding outputs 64 tile + Q i + p, i < 64 / Q, from map p.  Tile row r is therefore output
// 64 tile + Q (r mod 64 / Q) + r / (64 / Q).  The shifts follow the tap scale 2^14 D: s = 13 - log2 Q (cu8) and
// t = 19 - log2 Q (cs16) keep unit DC gain.
template <bool CS16, int KPASS, int Q>
__global__ void __launch_bounds__(THREADS, 1) k_channelize(const __grid_constant__ XMaps<Q> maps, const __grid_constant__ CUtensorMap map_w,
                                                           Params p)
{
    static_assert(Q == 1 || Q == 2 || Q == 4, "D = 32, 16 or 8");
    static_assert(KPASS == 1 || Q == 1, "512-tap plans decimate by 32");
    constexpr int LQ = Q == 1 ? 0 : (Q == 2 ? 1 : 2);
    constexpr int SH_CU8 = SHIFT1 - LQ, SH_CS16 = TAP_SCALE_LOG2 - LQ;   // s, t
    constexpr int BOX = TILE_M / Q;                                // rows per box, outputs per phase of a tile
    constexpr int PLANES = CS16 ? 2 : 1;                           // a tile takes PLANES * KPASS capture stages
    constexpr int NST = stages_of(KPASS), WB = KPASS * (int)W_BYTES, U = PLANES * KPASS;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t *smem_w = smem;                                        // [KPASS * 8 chunks][128 rows][64 B]
    uint8_t *smem_a = smem + WB;                                   // [NST][8 chunks][64 rows][64 B]
    Barriers &bar = *reinterpret_cast<Barriers *>(smem + WB + NST * A_STAGE_BYTES);
    // the epilogue's tables in shared memory: the first half of the phasor table (P[11907 - i] = conj(P[i]), made so on
    // the host), and this group's rotation steps, offset corrections and output destinations
    short2 *ph_half = reinterpret_cast<short2 *>(smem + WB + NST * A_STAGE_BYTES + 256);
    int *s_rot = reinterpret_cast<int *>(reinterpret_cast<uint8_t *>(ph_half) + ((HALF * 4 + 15) & ~15));
    uint32_t *s_corr = reinterpret_cast<uint32_t *>(s_rot + GROUP);
    long long *s_dst = reinterpret_cast<long long *>(s_corr + 2 * GROUP);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int group = (int)blockIdx.x % p.ngroups, slot = (int)blockIdx.x / p.ngroups, nslots = (int)gridDim.x / p.ngroups;

    for (int i = threadIdx.x; i < HALF; i += THREADS) ph_half[i] = p.phasor[i];
    for (int i = threadIdx.x; i < GROUP; i += THREADS) {
        const int ch = min(group * GROUP + i, p.nch - 1);
        s_rot[i] = p.rot_step[ch];
        s_corr[2 * i] = (uint32_t)p.corr[2 * ch];
        s_corr[2 * i + 1] = (uint32_t)p.corr[2 * ch + 1];
        s_dst[i] = p.dst ? p.dst[ch] : (long long)ch * (long long)p.out_stride;
    }
    if (threadIdx.x == 0) {
        mbar_init(&bar.w_full, 1);
        for (int i = 0; i < NST; i++) {
            mbar_init(&bar.a_full[i], 1);
            mbar_init(&bar.a_empty[i], 4);                         // one arrival per warp of the consuming warpgroup
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int wgi = __shfl_sync(0xffffffffu, threadIdx.x / 128, 0);   // warpgroup index, known to be warp-uniform
    if (wgi == 0) {
        // ===== TMA producer (one thread) =====
        if (threadIdx.x == 0) {
            mbar_expect_tx(&bar.w_full, WB);
            for (int c = 0; c < KPASS * NCHUNK; c++)
                tma_load_2d(smem_w + (size_t)c * TILE_N * CHUNK, &map_w, &bar.w_full, 0, (group * KPASS * NCHUNK + c) * TILE_N);
            unsigned it = 0;
            for (long long tile = slot; tile < p.tiles; tile += nslots)
                for (int pp = 0; pp < PLANES * KPASS; pp++, it++) {   // cs16: the x_hi plane's passes, then the x_lo plane's
                    const int pl = pp / KPASS, ps = pp % KPASS;
                    const int s = ring_stage<U, KPASS>(it);
                    if (KPASS == 1 ? it >= STAGES : ring_use<U, KPASS>(it) > 0) mbar_wait(&bar.a_empty[s], (ring_use<U, KPASS>(it) - 1) & 1);
                    mbar_expect_tx(&bar.a_full[s], A_STAGE_BYTES);
                    for (int c = 0; c < NCHUNK; c++)             // K chunk c of pass ps of output row j = capture-matrix row j + 8 ps + c
#pragma unroll
                        for (int ph = 0; ph < Q; ph++)
                            tma_load_2d(smem_a + (size_t)s * A_STAGE_BYTES + (size_t)c * TILE_M * CHUNK + (size_t)ph * BOX * CHUNK, &maps.m[ph],
                                        &bar.a_full[s], 0, (int)(tile * BOX) + ps * NCHUNK + c + pl * PLANE_ROWS);
                }
        }
        return;
    }
    // ===== consumers: warpgroup 1 takes the CTA's even tiles, warpgroup 2 the odd ones =====
    const int wg = wgi - 1, wwarp = warp & 3;
    const int q = lane & 3;                                        // this thread's channels: cl = 4 i + q, i = 0 .. 7
    int16_t *row[8];                                               // where their output 0 goes
#pragma unroll
    for (int i = 0; i < 8; i++) row[i] = p.out + s_dst[4 * i + q];
    mbar_wait(&bar.w_full, 0);
    unsigned it = (unsigned)wg * PLANES * KPASS;
    for (long long tile = slot + (long long)wg * nslots; tile < p.tiles; tile += 2ll * nslots, it += 2 * PLANES * KPASS) {
        uint32_t d[64];                                            // (the first wgmma overwrites it: accumulate = 0)
        int a1[32];                                                // cs16: A1 = sum W x_hi, [channel i][row h][re, im]
        if constexpr (CS16) {
#pragma unroll 1
            for (int ps = 0; ps < KPASS; ps++) {
                const int s = ring_stage<U, KPASS>(it + ps);
                mbar_wait(&bar.a_full[s], ring_use<U, KPASS>(it + ps) & 1);
                asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
                for (int c = 0; c < NCHUNK; c++)
#pragma unroll
                    for (int k = 0; k < CHUNK / 32; k++) {
                        const uint64_t da = wgmma_desc_sw64(smem_a + (size_t)s * A_STAGE_BYTES + (size_t)c * TILE_M * CHUNK, 32u * k);
                        const uint64_t db = wgmma_desc_sw64(smem_w + (size_t)(ps * NCHUNK + c) * TILE_N * CHUNK, 32u * k);
                        wgmma_s8s8(d, da, db, (ps | c | k) ? 1u : 0u);
                    }
                asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
                asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
                __syncwarp();
                if (lane == 0) mbar_arrive(&bar.a_empty[s]);
            }
            // |A1| <= 128 sum(|Wr| + |Wi|) < 2^28: the wrapped 32-bit 256 hi + lo is the value
#pragma unroll
            for (int i = 0; i < 8; i++)
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    a1[4 * i + 2 * h] = (int)(256u * d[8 * i + 2 * h] + d[8 * i + 4 + 2 * h]);
                    a1[4 * i + 2 * h + 1] = (int)(256u * d[8 * i + 2 * h + 1] + d[8 * i + 5 + 2 * h]);
                }
        }
#pragma unroll 1
        for (int ps = 0; ps < KPASS; ps++) {
            const unsigned il = it + (PLANES - 1) * KPASS + ps;    // the stage of the unsigned operand (cu8: the capture; cs16: x_lo)
            const int s = ring_stage<U, KPASS>(il);
            mbar_wait(&bar.a_full[s], ring_use<U, KPASS>(il) & 1);
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int c = 0; c < NCHUNK; c++)
#pragma unroll
                for (int k = 0; k < CHUNK / 32; k++) {             // wgmma K = 32 bytes
                    const uint64_t da = wgmma_desc_sw64(smem_a + (size_t)s * A_STAGE_BYTES + (size_t)c * TILE_M * CHUNK, 32u * k);
                    const uint64_t db = wgmma_desc_sw64(smem_w + (size_t)(ps * NCHUNK + c) * TILE_N * CHUNK, 32u * k);
                    wgmma_u8s8(d, da, db, (ps | c | k) ? 1u : 0u);
                }
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar.a_empty[s]);           // the stage's bytes are no longer needed
        }

        // ===== epilogue: rows 16 wwarp + lane / 4 (h = 0) and + 8 (h = 1) of the tile =====
        // 32-bit arithmetic throughout: 256 * hi + lo wraps, the filter output itself is bounded by
        // 128 * sum(|Wr| + |Wi|) < 2^28 (checked when the tables are made), so the wrapped sum is the value; after
        // the shift a component is below 2^15 and the rotation's two products stay below 2^31.  The phasor index
        // (1600 m_k (n0 + n)) mod 11907 is taken from nmod = (n0 mod 11907 + n) mod 11907 < 11907, so its product
        // with the rotation step stays below 11907^2 < 2^32.
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int r = 16 * wwarp + (lane >> 2) + 8 * h;       // tile row -> output: 64 tile + r when Q = 1
            const long long n = Q == 1 ? tile * TILE_M + 16 * wwarp + (lane >> 2) + 8 * h : tile * TILE_M + (Q * (r % BOX) + r / BOX);
            const int nmod = (int)((p.n0mod + n) % PERIOD);
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int cl = 4 * i + q, ch = group * GROUP + cl;
                const unsigned qi = ((unsigned)s_rot[cl] * (unsigned)nmod) % (unsigned)PERIOD;   // < 11907^2 < 2^32
                const bool up = qi >= (unsigned)HALF;
                const short2 v2 = ph_half[up ? (unsigned)PERIOD - qi : qi];
                const int phx = v2.x, phy = up ? -v2.y : v2.y;
                int vr, vi;
                if constexpr (CS16) {
                    // acc = 256 A1 + A2 < 2^36; with A1 = 2^(t-8) (A1 >> (t-8)) + (A1 & (2^(t-8) - 1)), t = 19 (D = 32):
                    // (acc + 2^(t-1)) >> t = (A1 >> (t-8)) + ((256 (A1 & (2^(t-8) - 1)) + A2 + 2^(t-1)) >> t), all terms below 2^30
                    constexpr int SPLIT = SH_CS16 - 8;
                    const int a2r = (int)(256u * d[8 * i + 2 * h] + d[8 * i + 4 + 2 * h]);           // |A2| < 2^29
                    const int a2i = (int)(256u * d[8 * i + 2 * h + 1] + d[8 * i + 5 + 2 * h]);
                    const int br = a1[4 * i + 2 * h], bi = a1[4 * i + 2 * h + 1];
                    vr = (br >> SPLIT) + ((((br & ((1 << SPLIT) - 1)) << 8) + a2r + (1 << (SH_CS16 - 1))) >> SH_CS16);
                    vi = (bi >> SPLIT) + ((((bi & ((1 << SPLIT) - 1)) << 8) + a2i + (1 << (SH_CS16 - 1))) >> SH_CS16);
                    vr = vr > 32767 ? 32767 : (vr < -32768 ? -32768 : vr);                            // sat16: the rotation stays in 32 bits
                    vi = vi > 32767 ? 32767 : (vi < -32768 ? -32768 : vi);
                } else {
                    const int ar = (int)(256u * d[8 * i + 2 * h] + d[8 * i + 4 + 2 * h] - s_corr[2 * cl]);
                    const int ai = (int)(256u * d[8 * i + 2 * h + 1] + d[8 * i + 5 + 2 * h] - s_corr[2 * cl + 1]);
                    vr = (ar + (1 << (SH_CU8 - 1))) >> SH_CU8;
                    vi = (ai + (1 << (SH_CU8 - 1))) >> SH_CU8;
                }
                int zr = vr * phx + vi * phy, zi = vi * phx - vr * phy;        // v * conj(P)
                zr = (zr + (1 << 14)) >> 15;
                zi = (zi + (1 << 14)) >> 15;
                zr = zr > 32767 ? 32767 : (zr < -32768 ? -32768 : zr);
                zi = zi > 32767 ? 32767 : (zi < -32768 ? -32768 : zi);
                const uint32_t packed = (uint32_t)(uint16_t)(int16_t)zr | ((uint32_t)(uint16_t)(int16_t)zi << 16);
                if (ch < p.nch && n < p.nout) *reinterpret_cast<uint32_t *>(row[i] + 2 * n) = packed;
            }
        }
    }
}

// cs16 -> the two byte planes the kernel reads: x = 256 hi + lo, hi[v] = x[v] >> 8 (signed), lo[v] = x[v] & 255, v
// counting int16 values (so each plane is laid out like a cu8 capture).  Four complex samples per thread; src 16-byte
// aligned.
__global__ void k_split_cs16(const int16_t *__restrict__ src, long long nvalues, uint8_t *__restrict__ hi, uint8_t *__restrict__ lo)
{
    const long long v0 = 8 * ((long long)blockIdx.x * blockDim.x + threadIdx.x);
    if (v0 + 8 <= nvalues) {
        const uint4 w = *reinterpret_cast<const uint4 *>(src + v0);
        // little-endian: value 2j of a word is its bytes 0 (low), 1 (high); value 2j + 1 its bytes 2, 3
        *reinterpret_cast<uint2 *>(hi + v0) = make_uint2(__byte_perm(w.x, w.y, 0x7531), __byte_perm(w.z, w.w, 0x7531));
        *reinterpret_cast<uint2 *>(lo + v0) = make_uint2(__byte_perm(w.x, w.y, 0x6420), __byte_perm(w.z, w.w, 0x6420));
    } else {
        for (long long v = v0; v < nvalues; v++) {
            hi[v] = (uint8_t)(src[v] >> 8);
            lo[v] = (uint8_t)src[v];
        }
    }
}

// Streaming: after a launch over the staging buffer has used the outputs it could, the samples from 32 x (outputs) on -
// at most taps - 1 samples: 510 bytes of cu8 or 1020 of cs16 with 256 taps, 1022 or 2044 with 512 - move to the front
// of the buffer, where the next push's bytes are appended to them.  Source and destination can overlap: one block (of nbytes / 2 threads or more) reads everything
// before it writes.
__global__ void k_move_carry(uint8_t *buf, size_t from, int nbytes)
{
    const int i = 2 * (int)threadIdx.x;
    uint16_t v = 0;
    if (i < nbytes) v = *reinterpret_cast<const uint16_t *>(buf + from + i);
    __syncthreads();
    if (i < nbytes) *reinterpret_cast<uint16_t *>(buf + i) = v;
}

// Rate stage (nrsc5b_chan_create_rate*): a capture at fs -> the plan's capture rate R, R / fs = L / M in lowest terms,
//     y[n] = sat16((sum_{j<64} G[p_n][j] x[b_n + j] + 2^13) >> 14),   b_n = floor(n M / L),  p_n = n M mod L
// (cu8: x = 64 (x8 - 127)), written straight into the byte planes the cs16 instantiations of k_channelize read.
// A CTA takes RS_TILE consecutive outputs n0 + i: it stages their input span - at most (RS_TILE - 1) M / L + 65 samples,
// M / L <= 4 (fs <= 4 R) - from the 16-byte boundary below it into shared memory with cp.async, then each thread reads
// its phase row (64 taps, 128 B, L2-resident: L <= 11907 rows) and forms one output in exact int32 arithmetic
// (sum_j |G[p][j]| < 2^16 is checked when the table is made, so |acc| + 2^13 < 2^31).
constexpr int RS_TAPS = 64;                                       // J: taps per phase
constexpr int RS_TILE = 256;                                      // outputs per CTA (one per thread)
constexpr int RS_MAX_L = 11907;                                   // phases: the table stays within 1.5 MB
constexpr int RS_CARRY = 512;                                     // resampled samples a streamed carry can hold (< the plan's taps)
static_assert(RS_CARRY >= 2 * PASS_TAPS, "the carry holds fewer samples than the longest plan's taps");
// staged samples: a span at M / L <= 4 and up to 7 below the 16-byte boundary, in whole 16-byte words of either format
constexpr int RS_SPAN = ((RS_TILE - 1) * 4 + 1 + RS_TAPS + 7 + 7) / 8 * 8;

__device__ __forceinline__ void cp_async16(void *dst, const void *src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}

// Outputs n = 0 .. nout - 1 of the stage, n at phase (p0 + n M) mod L and window start b0 + floor((p0 + n M) / L) of
// the samples at `in` (16-byte aligned, in_len samples of 2 (cu8) or 4 (cs16) bytes; every window lies inside them);
// output n goes to hi[2 n], hi[2 n + 1] (the signed high bytes of I, Q) and lo[...] (the low bytes).  The one 64-bit
// product per CTA is its first output's q = p0 + n M, bounded by the launch, not by the capture.
template <bool CU8>
__global__ void __launch_bounds__(RS_TILE) k_resample(const uint8_t *__restrict__ in, long long in_len, long long b0, int p0, int L, int M,
                                                      long long nout, const int16_t *__restrict__ G, uint8_t *__restrict__ hi,
                                                      uint8_t *__restrict__ lo)
{
    constexpr int BPS = CU8 ? 2 : 4;                               // bytes per complex sample
    __shared__ alignas(16) uint8_t raw[RS_SPAN * BPS];
    __shared__ alignas(16) uint32_t conv[CU8 ? RS_SPAN : 1];       // cu8: the span as 16-bit (I, Q) = 64 (x8 - 127)
    const long long nt0 = (long long)blockIdx.x * RS_TILE;
    const int nt = (int)(nout - nt0 < RS_TILE ? nout - nt0 : RS_TILE);
    const long long q0 = (long long)p0 + nt0 * M;
    const long long bt = b0 + q0 / L;                              // the tile's first window start (absolute sample)
    const int pt = (int)(q0 % L);
    const int span = (int)(((long long)pt + (long long)(nt - 1) * M) / L) + RS_TAPS;   // samples the tile reads
    const long long a0 = (bt * BPS) & ~15ll;                       // staging starts at the 16-byte boundary below bt
    const int skip = (int)(bt * BPS - a0) / BPS;                   // samples before bt in the staging buffer
    const int nbytes = (skip + span) * BPS;
    const long long avail = in_len * BPS - a0;                     // bytes of the input from a0 on
    for (int c = threadIdx.x; 16 * c < nbytes; c += RS_TILE) {
        if (16ll * c + 16 <= avail)
            cp_async16(raw + 16 * c, in + a0 + 16 * c);
        else
            for (int k = 0; k < 16; k++) raw[16 * c + k] = 16ll * c + k < avail ? in[a0 + 16 * c + k] : 0;
    }
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    const uint32_t *xs;
    if constexpr (CU8) {
        for (int s = threadIdx.x; s < skip + span; s += RS_TILE) {
            const uint32_t v = *reinterpret_cast<const uint16_t *>(raw + 2 * s);
            const int xr = 64 * ((int)(v & 255) - 127), xi = 64 * ((int)(v >> 8) - 127);
            conv[s] = (uint32_t)(uint16_t)(int16_t)xr | ((uint32_t)(uint16_t)(int16_t)xi << 16);
        }
        __syncthreads();
        xs = conv + skip;
    } else {
        xs = reinterpret_cast<const uint32_t *>(raw) + skip;
    }
    const int i = threadIdx.x;
    if (i >= nt) return;
    const int qi = pt + i * M;                                     // < 11907 + 255 x 47628 < 2^24
    const int b = qi / L, p = qi - b * L;
    const uint4 *row = reinterpret_cast<const uint4 *>(G + (size_t)p * RS_TAPS);
    const uint32_t *x = xs + b;
    int ar = 0, ai = 0;
#pragma unroll
    for (int c = 0; c < RS_TAPS / 8; c++) {
        const uint4 w = __ldg(row + c);
        const uint32_t ws[4] = { w.x, w.y, w.z, w.w };
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int g0 = (int)(ws[k] << 16) >> 16, g1 = (int)ws[k] >> 16;
            const uint32_t x0 = x[8 * c + 2 * k], x1 = x[8 * c + 2 * k + 1];
            ar += g0 * ((int)(x0 << 16) >> 16) + g1 * ((int)(x1 << 16) >> 16);
            ai += g0 * ((int)x0 >> 16) + g1 * ((int)x1 >> 16);
        }
    }
    int yr = (ar + (1 << 13)) >> 14, yi = (ai + (1 << 13)) >> 14;
    yr = yr > 32767 ? 32767 : (yr < -32768 ? -32768 : yr);
    yi = yi > 32767 ? 32767 : (yi < -32768 ? -32768 : yi);
    const uint32_t packed = (uint32_t)(uint16_t)(int16_t)yr | ((uint32_t)(uint16_t)(int16_t)yi << 16);
    const long long n = nt0 + i;
    reinterpret_cast<uint16_t *>(hi)[n] = (uint16_t)__byte_perm(packed, 0, 0x0031);   // high bytes of I, Q
    reinterpret_cast<uint16_t *>(lo)[n] = (uint16_t)__byte_perm(packed, 0, 0x0020);   // low bytes
}

constexpr size_t stage_cap_cu8(int taps) { return (4u << 20) + 2 * (size_t)taps; }   // cu8 staging: the carry (< 2 taps bytes) + 4 MiB of new capture
constexpr size_t STAGE_CAP_CS16 = 4 * PLANE_SAMPLES;              // cs16 staging: as many samples as the planes hold (16 MiB + 1 KiB)
constexpr int DST_RING = 8;                                       // destination tables in flight (nrsc5b_chan_feed)

}  // namespace nbch

// ===========================================================================
// host side
// ===========================================================================
using namespace nbch;

// A band plan: everything that differs between the FM grids (100 kHz channels of a D x 744 187.5 S/s capture, D = 32,
// 16 or 8) and the AM grid (10 kHz channels of a 1 488 375 S/s capture).  All share the 11907-entry phasor table:
// 100 kHz / (D x 744 187.5 Hz) = (1600 / D) / 11907, 10 kHz / 1 488 375 Hz = 80 / 11907; the mixer steps are D x those.
struct Plan {
    int taps;                             // per channel: KPASS = taps / 256 passes of the kernel
    int decim;                            // D: input samples per output; the tap scale is 2^14 D, the kernel's Q = 32 / D
    int tap_step, mix_step;               // phasor steps per input sample in W_k, per output sample in the mixer
    double fc, beta;                      // prototype: Kaiser-windowed sinc, -6 dB at fc (cycles per input sample)
    int max_offset;                       // |m_k| the capture holds (0: not limited)
    int engine_mode;                      // the engine nrsc5b_chan_feed may write into
};
static int log2_of(int v) { return v == 8 ? 3 : v == 16 ? 4 : 5; }   // D
static int shift_cu8(const Plan &pl) { return SHIFT1 - (5 - log2_of(pl.decim)); }   // s: 13 at D = 32
// FM: -6 dB at 372 kHz: flat over a hybrid FM channel (+-200 kHz), >= 55 dB down from 544 kHz on (what folds onto the
// channel after the decimation to 744 187.5 S/s)
static const Plan PLAN_FM = { 256, 32, 50, 1600, 372000.0 / 23814000.0, 5.65, 0, NRSC5B_MODE_FM };
// The same analogue spec at 11 907 000 and 5 953 500 S/s: the 256 taps span 2 and 4 times the time, so the transition
// from 200 to 544 kHz is 2 and 4 times as many bins wide and a wider window (beta 9) fits in it.  Measured on the
// integer taps of channel 0: D = 16 within 0.001 dB over +-200 kHz and 85.4 dB down from 544 kHz on, D = 8 within
// 0.001 dB and 80.2 dB down (the rounding of taps at the 2^14 D scale is the floor there).  The captures span
// +-5.95 and +-2.98 MHz: offsets beyond +-59 and +-29 are not in them.
static const Plan PLAN_FM16 = { 256, 16, 100, 1600, 372000.0 / 11907000.0, 9.0, 59, NRSC5B_MODE_FM };
static const Plan PLAN_FM8 = { 256, 8, 200, 1600, 372000.0 / 5953500.0, 9.0, 29, NRSC5B_MODE_FM };
// AM: -6 dB at 23 kHz.  The integer taps of channel 0 are within +-0.001 dB up to 15 kHz (a hybrid AM channel) and
// 87.1 dB down from 31.5 kHz on: what folds onto a channel after /32 are the stations k x 46.5 kHz away, which on the
// 10 kHz grid land a few kHz off centre, on carriers 30 - 50 dB below an analog host.  The capture spans +-744 kHz:
// offsets beyond +-74 are not in it.
static const Plan PLAN_AM = { 512, 32, 80, 2560, 23000.0 / 1488375.0, 8.8, 74, NRSC5B_MODE_AM };

// decim -> the FM plan (32: PLAN_FM itself); null for anything else
static const Plan *fm_plan(int decim) { return decim == 32 ? &PLAN_FM : decim == 16 ? &PLAN_FM16 : decim == 8 ? &PLAN_FM8 : nullptr; }

struct nrsc5b_channelizer {
    int device, nch, ngroups;
    const Plan *plan;                     // the band plan, fixed at create
    bool cs16;                            // the input format, fixed at create
    std::vector<int> offsets;             // m_k: channel offset from the capture centre in channel steps (100 kHz | 10 kHz)
    std::vector<int16_t> taps;            // [nch][plan->taps][2] (Wr, Wi) of W_k[u]
    std::vector<short2> phasor;           // [PERIOD]
    int8_t *d_w;                          // [ngroups][8 KPASS][128][64]
    int *d_rot;
    long long *d_corr;
    short2 *d_phasor;
    CUtensorMap map_w;
    PFN_cuTensorMapEncodeTiled_v12000 encode;
    // streaming (nrsc5b_chan_push / nrsc5b_chan_feed)
    long long pushed;                     // T: complex samples pushed since create / reset
    uint8_t *d_stage;                     // [stage_cap_cu8 or STAGE_CAP_CS16]: carry (samples from D N(T) on) | the bytes being pushed
    uint8_t *d_planes;                    // cs16: [2][PLANE_SAMPLES * 2] the x_hi and x_lo planes a launch reads
    CUtensorMap map_stage[4];             // what a streamed launch reads: d_stage (cu8) or d_planes (cs16), one map per phase
    cudaEvent_t stage_done;               // the last work that used d_stage / d_planes (calls may come on different CUDA streams)
    long long *h_dst, *d_dst;             // [DST_RING][nch] page-locked / device: per-channel destinations of a feed
    cudaEvent_t dst_copied[DST_RING];
    unsigned dst_pos;
    // rate stage (nrsc5b_chan_create_rate*; rs_L = 0: none): the capture at fs goes through k_resample into d_planes,
    // and the plan runs its cs16 definition on the result.  d_stage then holds the raw input from b_{K(T)} on.
    int rs_L, rs_M;                       // R / fs = L / M
    int16_t *d_G;                         // [rs_L][64] the phase table
    uint8_t *d_rcarry;                    // [2 planes][2 RS_CARRY] the streamed resampled carry (the planes are shared)
    long long rs_k;                       // K(T): resampled samples made since create / reset
    long long rs_b;                       // b_{K(T)}: the input sample at row 0 of d_stage
    int rs_p;                             // p_{K(T)} = K(T) M mod L
};

// the kernel reads the byte planes of a cs16 capture (a cs16 handle, or any handle with a rate stage)
static bool reads_planes(const nrsc5b_channelizer *c) { return c->cs16 || c->rs_L; }

static double bessel_i0(double x)
{
    double s = 1, t = 1;
    for (int k = 1; k < 50; k++) {
        t *= (x / (2 * k)) * (x / (2 * k));
        s += t;
    }
    return s;
}

// The integer tables of the definition, on the host (no device needed): phasor[11907], taps[nch][plan taps] = W_k[u]
// and, for the kernel, the B operand bytes, the rotation steps and the per-channel offset corrections.
//
// The bounds the kernel relies on, for every plan (S = sum_u |Wr| + |Wi| <= sqrt(2) 2^14 D sum|h| + taps):
//   tap bytes     |W| <= 2^14 D max h, about 2^14 D x 2 fc: 16 374 (FM, every D), 16 197 (AM) < 127 x 256 + 127, so
//                 both bytes are int8.  The -6 dB point stays at 372 kHz, so 2 fc doubles each time D halves; at a
//                 fixed 2^19 the peak would be 32 760 (D = 16) and 65 520 (D = 8), hence the scale 2^14 D;
//   wgmma sums    a pass adds 512 products below 255 x 128: < 2^24, two passes < 2^25, far inside int32;
//   cu8           |acc| <= 128 S < 2^(15 + s) <= 2^28 (checked below), so |v| < 2^15 after the shift by s = 13 - log2(32 / D)
//                 and the rotation's products stay in 32 bits: sum|h| = 1.40 (FM D = 32), 1.59 (D = 16: beta 9), 1.88
//                 (D = 8), 1.59 (AM, twice the taps but the same relative cut-off, so only the window's longer tails
//                 add) bound 128 S / 2^s by 2^14.0, 2^14.2, 2^14.4 and 2^14.2; over all offsets the tables reach 2^26.85
//                 (FM, +-118) and 2^27.11 (AM, +-74) at D = 32;
//   cs16          |A1| <= 128 S < 2^28 and |A2| <= 255 S < 2^29 by the same check, |acc| <= 2^15 S < 2^36.
// So 512 taps hold at scale 2^19 and the AM plan keeps it.
static bool offsets_ok(const Plan &pl, const int *offsets, int nch)
{
    for (int k = 0; pl.max_offset && k < nch; k++)
        if (offsets[k] < -pl.max_offset || offsets[k] > pl.max_offset) return false;
    return true;
}

static void make_tables(const Plan &pl, const int *offsets, int nch, std::vector<short2> &phasor, std::vector<int16_t> &taps, std::vector<int8_t> *w,
                        std::vector<int> *rot, std::vector<long long> *corr)
{
    phasor.resize(PERIOD);
    for (int i = 0; i <= PERIOD / 2; i++) {
        const double a = 2.0 * M_PI * i / PERIOD;
        phasor[i] = make_short2((short)lrint(32767.0 * cos(a)), (short)lrint(32767.0 * sin(a)));
    }
    for (int i = PERIOD / 2 + 1; i < PERIOD; i++)                          // exactly conjugate-symmetric: the kernel keeps half of it
        phasor[i] = make_short2(phasor[PERIOD - i].x, (short)-phasor[PERIOD - i].y);
    // prototype low-pass: Kaiser-windowed sinc, unit DC gain
    const int TAPS = pl.taps, KPASS = TAPS / PASS_TAPS;
    const int scale_log2 = TAP_SCALE_LOG2 - (5 - log2_of(pl.decim));   // 2^14 D
    std::vector<double> h(TAPS);
    {
        const double fc = pl.fc, beta = pl.beta;
        double sum = 0;
        for (int t = 0; t < TAPS; t++) {
            const double x = t - (TAPS - 1) / 2.0;
            const double sinc = fabs(x) < 1e-12 ? 2 * fc : sin(2 * M_PI * fc * x) / (M_PI * x);
            const double r = 2.0 * t / (TAPS - 1) - 1.0;
            h[t] = sinc * bessel_i0(beta * sqrt(1 - r * r)) / bessel_i0(beta);
            sum += h[t];
        }
        for (int t = 0; t < TAPS; t++) h[t] /= sum;
    }
    const int ngroups = (nch + GROUP - 1) / GROUP;
    taps.assign((size_t)nch * TAPS * 2, 0);
    if (w) w->assign((size_t)ngroups * KPASS * W_BYTES, 0);
    if (rot) rot->assign(nch, 0);
    if (corr) corr->assign((size_t)nch * 2, 0);
    for (int k = 0; k < nch; k++) {
        const int m = offsets[k];
        const long long step = (((long long)pl.tap_step * m) % PERIOD + PERIOD) % PERIOD;
        if (rot) (*rot)[k] = (int)((((long long)pl.mix_step * m) % PERIOD + PERIOD) % PERIOD);
        long long swr = 0, swi = 0, sabs = 0;
        const int g = k / GROUP, cl = k % GROUP;
        const int brow = 16 * (cl / 4) + 2 * (cl % 4);                   // B rows of the channel: brow + part (+ 8: low bytes)
        for (int u = 0; u < TAPS; u++) {
            // W_k[u] = 2^14 D h[TAPS-1-u] e^{-j 2 pi tap_step m u / 11907}, from the integer phasor table
            const short2 ph = phasor[(size_t)((step * u) % PERIOD)];
            const double g0 = ldexp(h[TAPS - 1 - u], scale_log2) / 32767.0;
            const int wr = (int)lrint(g0 * ph.x), wi = (int)lrint(-g0 * ph.y);
            taps[((size_t)k * TAPS + u) * 2 + 0] = (int16_t)wr;
            taps[((size_t)k * TAPS + u) * 2 + 1] = (int16_t)wi;
            swr += wr;
            swi += wi;
            sabs += (wr < 0 ? -wr : wr) + (wi < 0 ? -wi : wi);
            if (!w) continue;
            // rows of B: real = (Wr, -Wi) against (xr, xi); imaginary = (Wi, Wr); each 16-bit value as signed high and low bytes
            const int vals[2][2] = { { wr, -wi }, { wi, wr } };
            for (int part = 0; part < 2; part++)
                for (int comp = 0; comp < 2; comp++) {
                    const int v = vals[part][comp];
                    const int hi = (v + 128) >> 8, lo = v - 256 * hi;           // v = 256 hi + lo, both in [-128, 127]
                    if (hi < -128 || hi > 127) { fprintf(stderr, "nrsc5_b200: channeliser tap out of range\n"); abort(); }
                    const int kappa = 2 * u + comp, ck = kappa / CHUNK, b = kappa % CHUNK;
                    const size_t base = ((size_t)(g * KPASS * NCHUNK + ck) * TILE_N) * CHUNK;
                    (*w)[base + (size_t)(brow + part) * CHUNK + b] = (int8_t)hi;
                    (*w)[base + (size_t)(brow + 8 + part) * CHUNK + b] = (int8_t)lo;
                }
        }
        // the kernel's epilogue computes in 32 bits (k_channelize): the filter output must stay below 2^(15 + s) <= 2^28
        if (128 * sabs >= (1ll << (15 + shift_cu8(pl)))) { fprintf(stderr, "nrsc5_b200: channeliser taps too large for the 32-bit epilogue\n"); abort(); }
        if (corr) {
            (*corr)[2 * k + 0] = 127ll * (swr - swi);
            (*corr)[2 * k + 1] = 127ll * (swi + swr);
        }
    }
}

static int tables_of(const Plan &pl, const int *offsets, int nch, int16_t *taps, int16_t *phasor)
{
    if (!offsets || nch <= 0 || nch > 4096 || !offsets_ok(pl, offsets, nch)) return NRSC5B_EINVAL;
    std::vector<short2> ph;
    std::vector<int16_t> tp;
    make_tables(pl, offsets, nch, ph, tp, nullptr, nullptr, nullptr);
    if (taps) memcpy(taps, tp.data(), tp.size() * sizeof(int16_t));
    if (phasor) memcpy(phasor, ph.data(), PERIOD * sizeof(short2));
    return NRSC5B_OK;
}

/* The definition's tables without a device: taps[nch][256][2], phasor[11907][2] (either may be NULL). */
extern "C" int nrsc5b_chan_make_tables(const int *offsets_100khz, int nch, int16_t *taps, int16_t *phasor)
{
    return tables_of(PLAN_FM, offsets_100khz, nch, taps, phasor);
}

/* The AM plan's: taps[nch][512][2], and the same phasor table. */
extern "C" int nrsc5b_chan_make_tables_am(const int *offsets_10khz, int nch, int16_t *taps, int16_t *phasor)
{
    return tables_of(PLAN_AM, offsets_10khz, nch, taps, phasor);
}

/* The FM plan at D x 744 187.5 S/s: taps[nch][256][2], the same phasor table. */
extern "C" int nrsc5b_chan_make_tables_fm(int decim, const int *offsets_100khz, int nch, int16_t *taps, int16_t *phasor)
{
    const Plan *pl = fm_plan(decim);
    return pl ? tables_of(*pl, offsets_100khz, nch, taps, phasor) : NRSC5B_EINVAL;
}

// ---- rate stage: a capture at any integer rate fs -> the plan's capture rate R through a polyphase resampler ----
//
// R / fs = L / M in lowest terms (2R and 2 fs are integers).  G[L][64]: a Kaiser-windowed sinc (beta 8.41, 85 dB) of
// 64 L taps designed at L fs, -6 dB at min(fs, R) / 2, phase p holding taps p + (63 - j) L, j < 64.  Each phase is
// scaled to sum 2^14 and rounded by largest remainder, so that it sums to exactly 2^14 (DC gain exactly 1).  The usable
// band is |f| <= f_p = (min(fs, R) - 11 fs / 128) / 2 (11 fs / 128: the Kaiser transition width of 85 dB over 64 taps
// per phase, 5.37 fs / 64, rounded up), in integers 512 f_p = 128 min(2 fs, 2 R) - 22 fs; a channel must lie inside
// it: |m| step + half width <= f_p (FM: 100 kHz steps, 200 kHz; AM: 10 kHz, 15 kHz).
constexpr double RS_BETA = 8.41;
struct RateStage {
    const Plan *plan;
    int L, M;                             // R / fs = L / M
    int max_offset;                       // largest usable |m| (fs == R: the plan's own limit, 0 = none)
    uint32_t rate;                        // fs
};

// 2R: twice the plan's capture rate, an integer for every plan (D x 1 488 375 for FM, 2 976 750 for AM)
static long long twice_rate(const Plan &pl) { return pl.engine_mode == NRSC5B_MODE_AM ? 2976750ll : (long long)pl.decim * 1488375ll; }

// mode / decim / fs -> the stage's counts; false for anything the library does not take
static bool rate_stage(int mode, int decim, uint32_t rate_hz, RateStage *rs)
{
    const Plan *pl = mode == NRSC5B_MODE_FM ? fm_plan(decim) : mode == NRSC5B_MODE_AM && decim == DECIM ? &PLAN_AM : nullptr;
    if (!pl || rate_hz == 0) return false;
    const long long r2 = twice_rate(*pl), f2 = 2ll * rate_hz;
    if (64ll * rate_hz < r2 || f2 > 4 * r2) return false;          // R / 32 <= fs <= 4 R
    const long long g = std::gcd(r2, f2);
    if (r2 / g > RS_MAX_L) return false;
    rs->plan = pl;
    rs->L = (int)(r2 / g);
    rs->M = (int)(f2 / g);
    rs->rate = rate_hz;
    if (rs->L == 1 && rs->M == 1) {                                // fs == R: the plan itself
        rs->max_offset = pl->max_offset;
        return true;
    }
    const bool am = pl->engine_mode == NRSC5B_MODE_AM;
    const long long step = am ? 10000 : 100000, half = am ? 15000 : 200000;
    const long long fp512 = 128 * std::min(f2, r2) - 22ll * rate_hz;
    if (fp512 < 512 * half) return false;                          // not even channel 0 fits
    long long mo = (fp512 - 512 * half) / (512 * step);
    if (pl->max_offset && mo > pl->max_offset) mo = pl->max_offset;
    rs->max_offset = (int)mo;
    return true;
}

static bool rate_offsets_ok(const RateStage &rs, const int *offsets, int nch)
{
    if (rs.L == 1) return offsets_ok(*rs.plan, offsets, nch);
    for (int k = 0; k < nch; k++)
        if (offsets[k] < -rs.max_offset || offsets[k] > rs.max_offset) return false;
    return true;
}

// K(T): resampled samples whose 64-sample windows lie within the first T input samples
static long long resampled_of(int L, int M, long long samples) { return samples < RS_TAPS ? 0 : ((samples - RS_TAPS + 1) * L - 1) / M + 1; }

// G[L][64] of a stage (L > 1).  Checks that every tap fits int16 and every phase's sum |G| < 2^16, which keeps the
// kernel's int32 accumulation exact for any cs16 input: |acc| + 2^13 <= 2^15 (2^16 - 1) + 2^13 < 2^31.
static void design_resampler(const RateStage &rs, std::vector<int16_t> &G)
{
    const int L = rs.L, N = RS_TAPS * L;
    const double fc = std::min(2.0 * rs.rate, (double)twice_rate(*rs.plan)) / 4.0 / ((double)L * rs.rate);   // cycles per sample at L fs
    const double i0b = bessel_i0(RS_BETA);
    std::vector<double> h(N);
    for (int t = 0; t < N; t++) {
        const double x = t - (N - 1) / 2.0;
        const double sinc = fabs(x) < 1e-12 ? 2 * fc : sin(2 * M_PI * fc * x) / (M_PI * x);
        const double r = 2.0 * t / (N - 1) - 1.0;
        h[t] = sinc * bessel_i0(RS_BETA * sqrt(std::max(0.0, 1 - r * r))) / i0b;
    }
    G.assign((size_t)L * RS_TAPS, 0);
    for (int p = 0; p < L; p++) {
        double v[RS_TAPS], sum = 0;
        for (int j = 0; j < RS_TAPS; j++) sum += (v[j] = h[p + (size_t)(RS_TAPS - 1 - j) * L]);
        long long fl[RS_TAPS], total = 0;
        int order[RS_TAPS];
        for (int j = 0; j < RS_TAPS; j++) {
            v[j] *= 16384.0 / sum;
            fl[j] = (long long)floor(v[j]);
            total += fl[j];
            order[j] = j;
        }
        // the 2^14 - sum(floor) units go to the taps with the largest remainders (ties: the lower j)
        std::stable_sort(order, order + RS_TAPS, [&](int a, int b) { return v[a] - fl[a] > v[b] - fl[b]; });
        const long long extra = 16384 - total;
        long long sabs = 0;
        for (int j = 0; j < RS_TAPS; j++) {
            const long long g = fl[order[j]] + (j < extra ? 1 : 0);
            if (g < -32768 || g > 32767) { fprintf(stderr, "nrsc5_b200: resampler tap out of range\n"); abort(); }
            G[(size_t)p * RS_TAPS + order[j]] = (int16_t)g;
            sabs += g < 0 ? -g : g;
        }
        if (extra < 0 || extra > RS_TAPS || sabs >= 65536) { fprintf(stderr, "nrsc5_b200: resampler phase out of bounds\n"); abort(); }
    }
}

// nout resampled samples into the planes from sample `at` on: phase p0 and window start b0 (input samples counted from
// `in`, 16-byte aligned, in_len samples of 2 (cu8) or 4 (cs16) bytes)
static int launch_resample(bool cu8, const void *in, long long in_len, long long b0, int p0, int L, int M, long long nout, const int16_t *d_G,
                           uint8_t *planes, long long at, cudaStream_t stream)
{
    if (nout <= 0) return NRSC5B_OK;
    const unsigned grid = (unsigned)((nout + RS_TILE - 1) / RS_TILE);
    const uint8_t *src = reinterpret_cast<const uint8_t *>(in);
    uint8_t *hi = planes + 2 * at, *lo = planes + 2 * PLANE_SAMPLES + 2 * at;
    if (cu8) k_resample<true><<<grid, RS_TILE, 0, stream>>>(src, in_len, b0, p0, L, M, nout, d_G, hi, lo);
    else k_resample<false><<<grid, RS_TILE, 0, stream>>>(src, in_len, b0, p0, L, M, nout, d_G, hi, lo);
    return cudaGetLastError() == cudaSuccess ? NRSC5B_OK : NRSC5B_ECUDA;
}

static bool attach_rate(nrsc5b_channelizer *c, const RateStage &rs)
{
    std::vector<int16_t> G;
    design_resampler(rs, G);
    c->rs_L = rs.L;
    c->rs_M = rs.M;
    return cudaMalloc(&c->d_rcarry, 4 * RS_CARRY) == cudaSuccess && cudaMalloc(&c->d_G, G.size() * sizeof(int16_t)) == cudaSuccess &&
           cudaMemcpy(c->d_G, G.data(), G.size() * sizeof(int16_t), cudaMemcpyHostToDevice) == cudaSuccess;
}

/* L, M, the largest usable |offset| and G[L][64] of a rate stage, without a device (fs == R: L = M = 1 and G the
 * identity row). */
extern "C" int nrsc5b_chan_resampler_tables(int mode, int decim, uint32_t rate_hz, int *L, int *M, int *max_offset, int16_t *G)
{
    RateStage rs;
    if (!rate_stage(mode, decim, rate_hz, &rs)) return NRSC5B_EINVAL;
    if (L) *L = rs.L;
    if (M) *M = rs.M;
    if (max_offset) *max_offset = rs.max_offset;
    if (G) {
        std::vector<int16_t> g;
        if (rs.L == 1) g.assign(RS_TAPS, 0), g[0] = 16384;
        else design_resampler(rs, g);
        memcpy(G, g.data(), g.size() * sizeof(int16_t));
    }
    return NRSC5B_OK;
}

// The kernel instantiation of a handle: 512 taps (AM) only at D = 32
static const void *kernel_of(const nrsc5b_channelizer *c)
{
    const bool cs = reads_planes(c);
    if (c->plan->taps != PASS_TAPS) return cs ? (const void *)k_channelize<true, 2, 1> : (const void *)k_channelize<false, 2, 1>;
    switch (c->plan->decim) {
    case 16: return cs ? (const void *)k_channelize<true, 1, 2> : (const void *)k_channelize<false, 1, 2>;
    case 8: return cs ? (const void *)k_channelize<true, 1, 4> : (const void *)k_channelize<false, 1, 4>;
    default: return cs ? (const void *)k_channelize<true, 1, 1> : (const void *)k_channelize<false, 1, 1>;
    }
}

// Q = 32 / D maps of a capture matrix: map p over the nbytes bytes at base + 2 D p, [rows][64 B], boxes of 64 / Q rows,
// 64-byte swizzle.  Rows past the end read as zero; only outputs the launch does not write touch them (an output's
// window ends inside its map's whole rows).
static bool encode_maps(nrsc5b_channelizer *c, CUtensorMap *maps, const void *base, size_t nbytes)
{
    const int D = c->plan->decim, Q = DECIM / D;
    for (int ph = 0; ph < Q; ph++) {
        const size_t off = (size_t)(2 * D * ph);
        const cuuint64_t dims[2] = { CHUNK, (cuuint64_t)((nbytes - off) / CHUNK) };
        const cuuint64_t strides[1] = { CHUNK };
        const cuuint32_t box[2] = { CHUNK, (cuuint32_t)(TILE_M / Q) }, es[2] = { 1, 1 };
        if (c->encode(&maps[ph], CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t *>(reinterpret_cast<const uint8_t *>(base) + off), dims,
                      strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return false;
    }
    return true;
}

static int create(const Plan &pl, nrsc5b_channelizer_t **out, int device, const int *offsets_100khz, int nch, bool cs16,
                  const RateStage *rs = nullptr)
{
    if (!out || !offsets_100khz || nch <= 0 || nch > 4096 || !offsets_ok(pl, offsets_100khz, nch)) return NRSC5B_EINVAL;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device >= ndev) {
        fprintf(stderr, "nrsc5_b200: no usable CUDA device (the channeliser has no CPU path)\n");
        return NRSC5B_ENODEV;
    }
    if (cudaSetDevice(device) != cudaSuccess) return NRSC5B_ENODEV;
    nrsc5b_channelizer *c = new nrsc5b_channelizer();
    c->device = device;
    c->nch = nch;
    c->ngroups = (nch + GROUP - 1) / GROUP;
    c->plan = &pl;
    c->cs16 = cs16;
    c->offsets.assign(offsets_100khz, offsets_100khz + nch);
    c->d_w = nullptr; c->d_rot = nullptr; c->d_corr = nullptr; c->d_phasor = nullptr;
    c->pushed = 0; c->d_stage = nullptr; c->d_planes = nullptr; c->stage_done = nullptr;
    c->h_dst = nullptr; c->d_dst = nullptr; c->dst_pos = 0;
    for (int i = 0; i < DST_RING; i++) c->dst_copied[i] = nullptr;
    c->rs_L = 0; c->rs_M = 0; c->d_G = nullptr; c->d_rcarry = nullptr; c->rs_k = 0; c->rs_b = 0; c->rs_p = 0;
    // driver entry point for the tensor-map encoder (no link-time dependency on libcuda)
    {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) { delete c; return NRSC5B_ECUDA; }
        c->encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
    }
    std::vector<int8_t> w;
    std::vector<int> rot;
    std::vector<long long> corr;
    make_tables(pl, offsets_100khz, nch, c->phasor, c->taps, &w, &rot, &corr);
    const int kpass = pl.taps / PASS_TAPS;
    bool ok = cudaMalloc(&c->d_w, w.size()) == cudaSuccess && cudaMalloc(&c->d_rot, nch * sizeof(int)) == cudaSuccess &&
              cudaMalloc(&c->d_corr, corr.size() * sizeof(long long)) == cudaSuccess &&
              cudaMalloc(&c->d_phasor, PERIOD * sizeof(short2)) == cudaSuccess;
    ok = ok && cudaMemcpy(c->d_w, w.data(), w.size(), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(c->d_rot, rot.data(), nch * sizeof(int), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(c->d_corr, corr.data(), corr.size() * sizeof(long long), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(c->d_phasor, c->phasor.data(), PERIOD * sizeof(short2), cudaMemcpyHostToDevice) == cudaSuccess;
    if (ok) {
        // taps as a [ngroups * 8 KPASS * 128 rows][64 B] matrix, boxes of 128 rows, 64-byte swizzle
        const cuuint64_t dims[2] = { CHUNK, (cuuint64_t)c->ngroups * kpass * NCHUNK * TILE_N };
        const cuuint64_t strides[1] = { CHUNK };
        const cuuint32_t box[2] = { CHUNK, TILE_N }, es[2] = { 1, 1 };
        ok = c->encode(&c->map_w, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, c->d_w, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    }
    // the streaming staging buffer (cu8) or the cs16 byte planes as a [rows][64 B] capture matrix (rows past a launch's
    // valid bytes only feed outputs the launch does not write)
    // (a rate stage: the raw input staging - STAGE_CAP_CS16 bytes in either format - and the planes it writes)
    if (ok && rs) ok = attach_rate(c, *rs);
    const bool pl16 = reads_planes(c);
    const size_t stage_cap = pl16 ? STAGE_CAP_CS16 : stage_cap_cu8(pl.taps), planes = pl16 ? 4 * PLANE_SAMPLES : 0;
    ok = ok && cudaMalloc(&c->d_stage, stage_cap) == cudaSuccess && cudaMemset(c->d_stage, 0, stage_cap) == cudaSuccess &&
         cudaEventCreateWithFlags(&c->stage_done, cudaEventDisableTiming) == cudaSuccess;
    if (ok && pl16) ok = cudaMalloc(&c->d_planes, planes) == cudaSuccess && cudaMemset(c->d_planes, 0, planes) == cudaSuccess;
    if (ok) ok = encode_maps(c, c->map_stage, pl16 ? c->d_planes : c->d_stage, pl16 ? planes : stage_cap);
    if (ok)
        ok = cudaFuncSetAttribute(kernel_of(c), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes(kpass)) == cudaSuccess;
    if (!ok) {
        nrsc5b_chan_destroy(c);
        return NRSC5B_ECUDA;
    }
    *out = c;
    return NRSC5B_OK;
}

extern "C" int nrsc5b_chan_create(nrsc5b_channelizer_t **out, int device, const int *offsets_100khz, int nch)
{
    return create(PLAN_FM, out, device, offsets_100khz, nch, false);
}

extern "C" int nrsc5b_chan_create_cs16(nrsc5b_channelizer_t **out, int device, const int *offsets_100khz, int nch)
{
    return create(PLAN_FM, out, device, offsets_100khz, nch, true);
}

extern "C" int nrsc5b_chan_create_am(nrsc5b_channelizer_t **out, int device, const int *offsets_10khz, int nch)
{
    return create(PLAN_AM, out, device, offsets_10khz, nch, false);
}

extern "C" int nrsc5b_chan_create_am_cs16(nrsc5b_channelizer_t **out, int device, const int *offsets_10khz, int nch)
{
    return create(PLAN_AM, out, device, offsets_10khz, nch, true);
}

// FM plans at D x 744 187.5 S/s, D = 32 (the plan of nrsc5b_chan_create itself), 16 or 8
extern "C" int nrsc5b_chan_create_fm(nrsc5b_channelizer_t **out, int device, int decim, const int *offsets_100khz, int nch)
{
    const Plan *pl = fm_plan(decim);
    return pl ? create(*pl, out, device, offsets_100khz, nch, false) : NRSC5B_EINVAL;
}

extern "C" int nrsc5b_chan_create_fm_cs16(nrsc5b_channelizer_t **out, int device, int decim, const int *offsets_100khz, int nch)
{
    const Plan *pl = fm_plan(decim);
    return pl ? create(*pl, out, device, offsets_100khz, nch, true) : NRSC5B_EINVAL;
}

// A capture at any rate fs (integer Hz) -> the plan of (mode, decim) through the rate stage; fs == R: the plan itself
static int create_rate(nrsc5b_channelizer_t **out, int device, int mode, int decim, uint32_t rate_hz, const int *offsets, int nch, bool cs16)
{
    RateStage rs;
    if (!out || !offsets || nch <= 0 || nch > 4096 || !rate_stage(mode, decim, rate_hz, &rs) || !rate_offsets_ok(rs, offsets, nch))
        return NRSC5B_EINVAL;
    return create(*rs.plan, out, device, offsets, nch, cs16, rs.L == 1 ? nullptr : &rs);
}

extern "C" int nrsc5b_chan_create_rate(nrsc5b_channelizer_t **out, int device, int mode, int decim, uint32_t rate_hz, const int *offsets,
                                       int nch)
{
    return create_rate(out, device, mode, decim, rate_hz, offsets, nch, false);
}

extern "C" int nrsc5b_chan_create_rate_cs16(nrsc5b_channelizer_t **out, int device, int mode, int decim, uint32_t rate_hz,
                                            const int *offsets, int nch)
{
    return create_rate(out, device, mode, decim, rate_hz, offsets, nch, true);
}

extern "C" void nrsc5b_chan_destroy(nrsc5b_channelizer_t *c)
{
    if (!c) return;
    cudaFree(c->d_w);
    cudaFree(c->d_rot);
    cudaFree(c->d_corr);
    cudaFree(c->d_phasor);
    cudaFree(c->d_stage);
    cudaFree(c->d_planes);
    cudaFree(c->d_G);
    cudaFree(c->d_rcarry);
    cudaFree(c->d_dst);
    if (c->h_dst) cudaFreeHost(c->h_dst);
    if (c->stage_done) cudaEventDestroy(c->stage_done);
    for (int i = 0; i < DST_RING; i++)
        if (c->dst_copied[i]) cudaEventDestroy(c->dst_copied[i]);
    delete c;
}

/* The integer tables the definition is made of (for the numpy restatement in the tests): taps[nch][256 | 512][2] =
 * (Wr, Wi) of W_k[u], phasor[11907][2]. */
extern "C" int nrsc5b_chan_tables(nrsc5b_channelizer_t *c, int16_t *taps, int16_t *phasor)
{
    if (!c) return NRSC5B_EINVAL;
    if (taps) memcpy(taps, c->taps.data(), c->taps.size() * sizeof(int16_t));
    if (phasor) memcpy(phasor, c->phasor.data(), PERIOD * sizeof(short2));
    return NRSC5B_OK;
}

// N(T): outputs whose windows (one per D samples, as long as the plan's filter) lie within the first T samples of a capture
static long long outputs_of(const Plan &pl, long long samples) { return samples < pl.taps ? 0 : (samples - pl.taps) / pl.decim + 1; }

/* How many output samples a capture of `nbytes` gives per channel: every output needs 256 input samples (AM: 512). */
extern "C" long long nrsc5b_chan_outputs(size_t nbytes) { return outputs_of(PLAN_FM, (long long)(nbytes / 2)); }
extern "C" long long nrsc5b_chan_outputs_am(size_t nbytes) { return outputs_of(PLAN_AM, (long long)(nbytes / 2)); }
extern "C" long long nrsc5b_chan_outputs_fm(int decim, size_t nbytes)
{
    const Plan *pl = fm_plan(decim);
    return pl ? outputs_of(*pl, (long long)(nbytes / 2)) : NRSC5B_EINVAL;
}
/* N_plan(K(T)) for T input samples at fs */
extern "C" long long nrsc5b_chan_outputs_rate(int mode, int decim, uint32_t rate_hz, long long samples)
{
    RateStage rs;
    if (!rate_stage(mode, decim, rate_hz, &rs) || samples < 0) return NRSC5B_EINVAL;
    return outputs_of(*rs.plan, rs.L == 1 ? samples : resampled_of(rs.L, rs.M, samples));
}

// the handle's outputs per channel from the first T input samples
static long long outputs_in(const nrsc5b_channelizer *c, long long samples)
{
    return outputs_of(*c->plan, c->rs_L ? resampled_of(c->rs_L, c->rs_M, samples) : samples);
}

template <bool CS16, int KPASS, int Q>
static void launch_k(const CUtensorMap *maps, const CUtensorMap &map_w, const Params &p, unsigned grid, cudaStream_t stream)
{
    XMaps<Q> m;
    memcpy(m.m, maps, sizeof(m.m));
    k_channelize<CS16, KPASS, Q><<<grid, THREADS, smem_bytes(KPASS), stream>>>(m, map_w, p);
}

// outputs n0 .. n0 + nout - 1 of the capture whose sample D n0 is row 0 of maps[0] (cs16: of both planes in the maps;
// the plan's Q maps): output n0 + j of channel k goes to out + dst[k] + 2 j (dst null: k * out_stride)
static int launch(nrsc5b_channelizer *c, const CUtensorMap *maps, long long n0, long long nout, int16_t *out, const long long *dst,
                  size_t out_stride, cudaStream_t stream)
{
    Params p;
    p.nch = c->nch;
    p.ngroups = c->ngroups;
    p.n0mod = (int)(n0 % PERIOD);
    p.nout = nout;
    p.tiles = (nout + TILE_M - 1) / TILE_M;
    p.out = out;
    p.dst = dst;
    p.out_stride = out_stride;
    p.rot_step = c->d_rot;
    p.corr = c->d_corr;
    p.phasor = c->d_phasor;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
    long long slots = sms / c->ngroups;
    if (slots < 1) slots = 1;
    if (slots > p.tiles) slots = p.tiles;
    const unsigned grid = (unsigned)(slots * c->ngroups);
    const bool cs = reads_planes(c);
    if (c->plan->taps != PASS_TAPS) (cs ? launch_k<true, 2, 1> : launch_k<false, 2, 1>)(maps, c->map_w, p, grid, stream);
    else if (c->plan->decim == 16) (cs ? launch_k<true, 1, 2> : launch_k<false, 1, 2>)(maps, c->map_w, p, grid, stream);
    else if (c->plan->decim == 8) (cs ? launch_k<true, 1, 4> : launch_k<false, 1, 4>)(maps, c->map_w, p, grid, stream);
    else (cs ? launch_k<true, 1, 1> : launch_k<false, 1, 1>)(maps, c->map_w, p, grid, stream);
    return cudaGetLastError() == cudaSuccess ? NRSC5B_OK : NRSC5B_ECUDA;
}

// cs16: the first nsamples (<= PLANE_SAMPLES) of the device capture at src (16-byte aligned) -> the handle's planes,
// then outputs n0 .. n0 + nout - 1 of them as launch() writes them
static int split_launch(nrsc5b_channelizer *c, const int16_t *src, long long nsamples, long long n0, long long nout, int16_t *out,
                        const long long *dst, size_t out_stride, cudaStream_t stream)
{
    const long long nvalues = 2 * nsamples, threads = (nvalues + 7) / 8;
    k_split_cs16<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(src, nvalues, c->d_planes, c->d_planes + 2 * PLANE_SAMPLES);
    if (cudaGetLastError() != cudaSuccess) return NRSC5B_ECUDA;
    return launch(c, c->map_stage, n0, nout, out, dst, out_stride, stream);
}

// Streaming through a rate stage.  Two carries: the input samples from b_{K(T)} on (at most 63) stay at the front of
// d_stage, and the resampled samples from D N(K(T)) on (fewer than the plan's taps) are kept, as their two plane bytes,
// in d_rcarry.  The planes are shared with the one-shot entry points, which write them from row 0, so a piece puts the
// carry back at the front of the planes before it resamples behind it, and takes the new carry out again after the
// channel bank has run.  A piece is bounded by both buffers: the raw staging holds STAGE_CAP_CS16 bytes, and the
// piece's K(T') - K(T) <= piece L / M + 1 new resampled samples must fit the planes after the carry.
static int stream_in_rate(nrsc5b_channelizer *c, const void *src, size_t nsamples, int16_t *out, const long long *dst, size_t out_stride,
                          cudaMemcpyKind kind, cudaStream_t stream)
{
    const Plan &pl = *c->plan;
    const int D = pl.decim, L = c->rs_L, M = c->rs_M;
    const size_t bps = c->cs16 ? 4 : 2, cap = STAGE_CAP_CS16 / bps;
    long long written = 0;
    for (size_t done = 0; done < nsamples;) {
        const size_t icarry = (size_t)(c->pushed - c->rs_b);
        const long long first = outputs_of(pl, c->rs_k), rcarry = c->rs_k - D * first;
        const long long room = (PLANE_SAMPLES - rcarry - 1) * M / L;
        size_t piece = nsamples - done < cap - icarry ? nsamples - done : cap - icarry;
        if ((long long)piece > room) piece = (size_t)room;
        if (cudaMemcpyAsync(c->d_stage + bps * icarry, reinterpret_cast<const uint8_t *>(src) + bps * done, bps * piece, kind, stream) !=
            cudaSuccess)
            return NRSC5B_ECUDA;
        const long long t1 = c->pushed + (long long)piece, k1 = resampled_of(L, M, t1), nk = k1 - c->rs_k;
        const long long held = rcarry + nk, nl = outputs_of(pl, held);   // (nk = 0: nothing new, the planes are not read)
        if (nk > 0) {
            for (int pn = 0; rcarry > 0 && pn < 2; pn++)       // the resampled carry back to the front of both planes
                if (cudaMemcpyAsync(c->d_planes + pn * 2 * PLANE_SAMPLES, c->d_rcarry + pn * 2 * RS_CARRY, 2 * (size_t)rcarry,
                                    cudaMemcpyDeviceToDevice, stream) != cudaSuccess)
                    return NRSC5B_ECUDA;
            int rc = launch_resample(!c->cs16, c->d_stage, (long long)(icarry + piece), 0, c->rs_p, L, M, nk, c->d_G, c->d_planes, rcarry, stream);
            if (rc) return rc;
            const long long q = c->rs_p + nk * M, b1 = c->rs_b + q / L;   // nk M < 2^39: bounded by the piece
            k_move_carry<<<1, (unsigned)(RS_TAPS * bps / 2), 0, stream>>>(c->d_stage, bps * (size_t)(b1 - c->rs_b), (int)(bps * (t1 - b1)));
            if (cudaGetLastError() != cudaSuccess) return NRSC5B_ECUDA;
            c->rs_p = (int)(q % L);
            c->rs_b = b1;
            c->rs_k = k1;
            if (nl > 0 && (rc = launch(c, c->map_stage, first, nl, out + 2 * written, dst, out_stride, stream))) return rc;
            const long long keep = held - D * nl;                // the new resampled carry, out of the planes
            for (int pn = 0; keep > 0 && pn < 2; pn++)
                if (cudaMemcpyAsync(c->d_rcarry + pn * 2 * RS_CARRY, c->d_planes + pn * 2 * PLANE_SAMPLES + 2 * D * nl, 2 * (size_t)keep,
                                    cudaMemcpyDeviceToDevice, stream) != cudaSuccess)
                    return NRSC5B_ECUDA;
        }
        c->pushed = t1;
        written += nl;
        done += piece;
    }
    return NRSC5B_OK;
}

// The streaming core of nrsc5b_chan_push* and nrsc5b_chan_feed*: appends nsamples complex samples (cu8 or cs16, the
// handle's format) at `src` to the handle's stream and writes the outputs they complete, N(T) .. N(T') - 1, output
// N(T) + j of channel k to out + dst[k] + 2 j (dst: a device table; null: k * out_stride).  Pushes larger than the
// staging buffer go through it in pieces.  Asynchronous on `stream`; the source is read by a copy on that stream.
static int stream_in(nrsc5b_channelizer *c, const void *src, size_t nsamples, int16_t *out, const long long *dst, size_t out_stride,
                     cudaStream_t stream)
{
    if (!nsamples) return NRSC5B_OK;
    const Plan &pl = *c->plan;
    const size_t bps = c->cs16 ? 4 : 2, cap = (c->cs16 ? STAGE_CAP_CS16 : stage_cap_cu8(pl.taps)) / bps;   // bytes per sample, samples staged
    const int D = pl.decim;
    // device memory: a device-to-device copy; page-locked host memory: DMA straight from it; pageable host memory: the
    // driver stages it (the copy returns once it has read the caller's bytes)
    cudaPointerAttributes attr;
    const bool on_device = cudaPointerGetAttributes(&attr, src) == cudaSuccess &&
                           (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged);
    cudaGetLastError();
    const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    if (cudaStreamWaitEvent(stream, c->stage_done, 0) != cudaSuccess) return NRSC5B_ECUDA;
    if (c->rs_L) {
        const int rc = stream_in_rate(c, src, nsamples, out, dst, out_stride, kind, stream);
        if (rc) return rc;
        return cudaEventRecord(c->stage_done, stream) == cudaSuccess ? NRSC5B_OK : NRSC5B_ECUDA;
    }
    long long written = 0;
    for (size_t done = 0; done < nsamples;) {
        const long long first = outputs_of(pl, c->pushed);        // absolute index of staging row 0's output
        const size_t carry = (size_t)(c->pushed - D * first);
        const size_t piece = nsamples - done < cap - carry ? nsamples - done : cap - carry;
        if (cudaMemcpyAsync(c->d_stage + bps * carry, reinterpret_cast<const uint8_t *>(src) + bps * done, bps * piece, kind, stream) !=
            cudaSuccess)
            return NRSC5B_ECUDA;
        const long long held = (long long)(carry + piece), nl = outputs_of(pl, held);
        if (nl > 0) {
            int rc = c->cs16 ? split_launch(c, reinterpret_cast<const int16_t *>(c->d_stage), held, first, nl, out + 2 * written, dst,
                                            out_stride, stream)
                             : launch(c, c->map_stage, first, nl, out + 2 * written, dst, out_stride, stream);
            if (rc) return rc;
            k_move_carry<<<1, (unsigned)(pl.taps * bps / 2), 0, stream>>>(c->d_stage, bps * D * nl, (int)(bps * (held - D * nl)));
            if (cudaGetLastError() != cudaSuccess) return NRSC5B_ECUDA;
        }
        c->pushed += (long long)piece;
        written += nl;
        done += piece;
    }
    return cudaEventRecord(c->stage_done, stream) == cudaSuccess ? NRSC5B_OK : NRSC5B_ECUDA;
}

extern "C" int nrsc5b_chan_reset(nrsc5b_channelizer_t *c)
{
    if (!c) return NRSC5B_EINVAL;
    c->pushed = 0;                                            // the carry is what lies beyond D N(T): nothing now
    c->rs_k = c->rs_b = 0;                                    // (a rate stage's two carries likewise)
    c->rs_p = 0;
    return NRSC5B_OK;
}

// nsamples complex samples of the handle's format at src (checked by the caller)
static int push(nrsc5b_channelizer *c, const void *src, size_t nsamples, void *d_out, size_t out_stride, void *cuda_stream, long long *nout)
{
    const long long n = outputs_in(c, c->pushed + (long long)nsamples) - outputs_in(c, c->pushed);
    if (n > 0 && (!d_out || ((uintptr_t)d_out & 3) || (out_stride & 1) || (size_t)(2 * n) > out_stride)) return NRSC5B_EINVAL;
    if (cudaSetDevice(c->device) != cudaSuccess) return NRSC5B_ENODEV;
    const int rc = stream_in(c, src, nsamples, reinterpret_cast<int16_t *>(d_out), nullptr, out_stride,
                             reinterpret_cast<cudaStream_t>(cuda_stream));
    if (rc == NRSC5B_OK && nout) *nout = n;
    return rc;
}

int nbchan_info(const nrsc5b_channelizer_t *c, int *device, int *mode, int *cs16, int *nch)
{
    if (!c) return NRSC5B_EINVAL;
    *device = c->device;
    *mode = c->plan->engine_mode;
    *cs16 = c->cs16;
    *nch = c->nch;
    return NRSC5B_OK;
}

long long nbchan_outputs_after(const nrsc5b_channelizer_t *c, long long samples)
{
    return outputs_in(c, c->pushed + samples) - outputs_in(c, c->pushed);
}

extern "C" int nrsc5b_chan_push(nrsc5b_channelizer_t *c, const uint8_t *cu8, size_t nbytes, void *d_out, size_t out_stride,
                                void *cuda_stream, long long *nout)
{
    if (nout) *nout = 0;
    if (!c || c->cs16 || (nbytes & 1) || (nbytes && !cu8)) return NRSC5B_EINVAL;
    return push(c, cu8, nbytes / 2, d_out, out_stride, cuda_stream, nout);
}

extern "C" int nrsc5b_chan_push_cs16(nrsc5b_channelizer_t *c, const int16_t *cs16, size_t nvalues, void *d_out, size_t out_stride,
                                     void *cuda_stream, long long *nout)
{
    if (nout) *nout = 0;
    if (!c || !c->cs16 || (nvalues & 1) || (nvalues && !cs16)) return NRSC5B_EINVAL;
    return push(c, cs16, nvalues / 2, d_out, out_stride, cuda_stream, nout);
}

// nsamples complex samples of the handle's format at src (checked by the caller)
static int feed(nrsc5b_channelizer *c, nrsc5b_engine_t *e, const int *streams, const void *src, size_t nsamples)
{
    const long long n = outputs_in(c, c->pushed + (long long)nsamples) - outputs_in(c, c->pushed);
    if (cudaSetDevice(c->device) != cudaSuccess) return NRSC5B_ENODEV;
    const size_t nch = (size_t)c->nch;
    if (!c->h_dst) {
        bool ok = cudaHostAlloc(reinterpret_cast<void **>(&c->h_dst), DST_RING * nch * sizeof(long long), cudaHostAllocDefault) == cudaSuccess;
        if (!ok) c->h_dst = nullptr;
        ok = ok && cudaMalloc(&c->d_dst, DST_RING * nch * sizeof(long long)) == cudaSuccess;
        for (int i = 0; ok && i < DST_RING; i++) ok = cudaEventCreateWithFlags(&c->dst_copied[i], cudaEventDisableTiming) == cudaSuccess;
        if (!ok) {
            if (c->h_dst) cudaFreeHost(c->h_dst);
            cudaFree(c->d_dst);
            for (int i = 0; i < DST_RING; i++)
                if (c->dst_copied[i]) cudaEventDestroy(c->dst_copied[i]);
            c->h_dst = c->d_dst = nullptr;
            for (int i = 0; i < DST_RING; i++) c->dst_copied[i] = nullptr;
            return NRSC5B_ENOMEM;
        }
    }
    // a slot of the destination ring is rewritten DST_RING feeds after its copy was queued: by then it has long run
    const unsigned slot = c->dst_pos % DST_RING;
    if (cudaEventSynchronize(c->dst_copied[slot]) != cudaSuccess) return NRSC5B_ECUDA;
    long long *h_dst = c->h_dst + slot * nch, *d_dst = c->d_dst + slot * nch;
    FeedTarget t;
    int rc = nbfeed_reserve(e, c->device, c->plan->engine_mode, streams, c->nch, n, &t, h_dst);
    if (rc) return rc;
    if (n > 0) {
        if (cudaMemcpyAsync(d_dst, h_dst, nch * sizeof(long long), cudaMemcpyHostToDevice, t.stream) != cudaSuccess ||
            cudaEventRecord(c->dst_copied[slot], t.stream) != cudaSuccess)
            return NRSC5B_ECUDA;
        c->dst_pos++;
    }
    rc = stream_in(c, src, nsamples, t.base, d_dst, 0, t.stream);
    if (rc) return rc;
    return nbfeed_commit(e, streams, c->nch, n);
}

extern "C" int nrsc5b_chan_feed(nrsc5b_channelizer_t *c, nrsc5b_engine_t *e, const int *streams, const uint8_t *cu8, size_t nbytes)
{
    if (!c || c->cs16 || !e || (nbytes & 1) || (nbytes && !cu8)) return NRSC5B_EINVAL;
    return feed(c, e, streams, cu8, nbytes / 2);
}

extern "C" int nrsc5b_chan_feed_cs16(nrsc5b_channelizer_t *c, nrsc5b_engine_t *e, const int *streams, const int16_t *cs16, size_t nvalues)
{
    if (!c || !c->cs16 || !e || (nvalues & 1) || (nvalues && !cs16)) return NRSC5B_EINVAL;
    return feed(c, e, streams, cs16, nvalues / 2);
}

// One-shot through a rate stage: the device capture at src (16-byte aligned, nin samples of the handle's format) ->
// out[nch][out_stride], PIECE_OUT plan outputs at a time: their resampled samples D n0 .. D (n0 + nl - 1) + taps - 1
// (all below K(nin)) go from the caller's capture into the planes, and the plan runs on them.
// (bank = false: the rate stage alone, the same launches of k_resample into the planes without the channel bank)
static int run_rate(nrsc5b_channelizer *c, const void *src, long long nin, int16_t *out, size_t out_stride, cudaStream_t stream,
                    bool bank = true)
{
    const int TAPS = c->plan->taps, D = c->plan->decim, L = c->rs_L, M = c->rs_M;
    const long long PIECE_OUT = piece_out(TAPS, D);
    const long long nout = outputs_in(c, nin);
    if (cudaStreamWaitEvent(stream, c->stage_done, 0) != cudaSuccess) return NRSC5B_ECUDA;   // the planes are shared with the stream
    for (long long n0 = 0; n0 < nout; n0 += PIECE_OUT) {
        const long long nl = nout - n0 < PIECE_OUT ? nout - n0 : PIECE_OUT, r0 = D * n0, q = r0 * M;
        int rc = launch_resample(!c->cs16, src, nin, q / L, (int)(q % L), L, M, D * nl + TAPS - D, c->d_G, c->d_planes, 0, stream);
        if (!rc && bank) rc = launch(c, c->map_stage, n0, nl, out + 2 * n0, nullptr, out_stride, stream);
        if (rc) return rc;
    }
    return cudaEventRecord(c->stage_done, stream) == cudaSuccess ? NRSC5B_OK : NRSC5B_ECUDA;
}

/* The rate stage of a rate handle's one-shot device path on its own (for timing it apart from the channel bank): the
 * same k_resample launches into the handle's planes as nrsc5b_chan_run_device* makes for this capture (nvalues cu8
 * bytes or cs16 int16 values, the handle's format, 16-byte aligned), and nothing else.  Asynchronous on cuda_stream. */
extern "C" int nrsc5b_chan_resample_device(nrsc5b_channelizer_t *c, const void *d_in, size_t nvalues, void *cuda_stream)
{
    if (!c || !c->rs_L || !d_in || ((uintptr_t)d_in & 15) || (nvalues & 1)) return NRSC5B_EINVAL;
    if (cudaSetDevice(c->device) != cudaSuccess) return NRSC5B_ENODEV;
    return run_rate(c, d_in, (long long)(nvalues / 2), nullptr, 0, reinterpret_cast<cudaStream_t>(cuda_stream), false);
}

/* Device-resident capture (cu8, I/Q interleaved, 23 814 000 S/s; 64-byte aligned, nbytes of it valid) -> out[nch][out_stride]
 * cs16 on the device (out_stride in int16 values, >= 2 * outputs; 4-byte aligned rows).  Asynchronous on `cuda_stream`. */
extern "C" int nrsc5b_chan_run_device(nrsc5b_channelizer_t *c, const void *d_cu8, size_t nbytes, void *d_out, size_t out_stride,
                                      void *cuda_stream)
{
    if (!c || c->cs16 || !d_cu8 || !d_out || ((uintptr_t)d_out & 3) || (out_stride & 1)) return NRSC5B_EINVAL;
    if (c->rs_L ? ((uintptr_t)d_cu8 & 15) || (nbytes & 1) : ((uintptr_t)d_cu8 & 63) || (nbytes & 63)) return NRSC5B_EINVAL;
    const long long nout = outputs_in(c, (long long)(nbytes / 2));
    if (nout <= 0) return NRSC5B_OK;
    if ((size_t)(2 * nout) > out_stride) return NRSC5B_EINVAL;
    if (cudaSetDevice(c->device) != cudaSuccess) return NRSC5B_ENODEV;
    if (c->rs_L) return run_rate(c, d_cu8, (long long)(nbytes / 2), reinterpret_cast<int16_t *>(d_out), out_stride, reinterpret_cast<cudaStream_t>(cuda_stream));
    // the capture as a [rows][64 B] matrix, one map per phase; rows past the end read as zero (only rows of outputs >= nout touch them)
    CUtensorMap map_x[4];
    if (!encode_maps(c, map_x, d_cu8, nbytes)) return NRSC5B_ECUDA;
    return launch(c, map_x, 0, nout, reinterpret_cast<int16_t *>(d_out), nullptr, out_stride, reinterpret_cast<cudaStream_t>(cuda_stream));
}

/* Device-resident cs16 capture (16-byte aligned, nvalues even) -> out[nch][out_stride] as nrsc5b_chan_run_device writes it.
 * Goes through the handle's planes PIECE_OUT outputs at a time; the caller's buffer is only read. */
extern "C" int nrsc5b_chan_run_device_cs16(nrsc5b_channelizer_t *c, const void *d_cs16, size_t nvalues, void *d_out, size_t out_stride,
                                           void *cuda_stream)
{
    if (!c || !c->cs16 || !d_cs16 || !d_out || ((uintptr_t)d_cs16 & 15) || (nvalues & 1) || ((uintptr_t)d_out & 3) || (out_stride & 1))
        return NRSC5B_EINVAL;
    const int TAPS = c->plan->taps, D = c->plan->decim;
    const long long PIECE_OUT = piece_out(TAPS, D);
    const long long nout = outputs_in(c, (long long)(nvalues / 2));
    if (nout <= 0) return NRSC5B_OK;
    if ((size_t)(2 * nout) > out_stride) return NRSC5B_EINVAL;
    if (cudaSetDevice(c->device) != cudaSuccess) return NRSC5B_ENODEV;
    const cudaStream_t stream = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (c->rs_L) return run_rate(c, d_cs16, (long long)(nvalues / 2), reinterpret_cast<int16_t *>(d_out), out_stride, stream);
    const int16_t *src = reinterpret_cast<const int16_t *>(d_cs16);
    int16_t *out = reinterpret_cast<int16_t *>(d_out);
    if (cudaStreamWaitEvent(stream, c->stage_done, 0) != cudaSuccess) return NRSC5B_ECUDA;   // the planes are shared with the stream
    for (long long n0 = 0; n0 < nout; n0 += PIECE_OUT) {
        const long long nl = nout - n0 < PIECE_OUT ? nout - n0 : PIECE_OUT;
        const int rc = split_launch(c, src + 2 * D * n0, D * nl + TAPS - D, n0, nl, out + 2 * n0, nullptr, out_stride, stream);
        if (rc) return rc;
    }
    return cudaEventRecord(c->stage_done, stream) == cudaSuccess ? NRSC5B_OK : NRSC5B_ECUDA;
}

// host capture of `bytes` bytes -> device (padded to whole 64-byte rows) -> the format's device entry -> host out
static int run_host(nrsc5b_channelizer *c, const void *in, size_t bytes, size_t count, long long nout, int16_t *out)
{
    if (cudaSetDevice(c->device) != cudaSuccess) return NRSC5B_ENODEV;
    uint8_t *d_in = nullptr;
    int16_t *d_out = nullptr;
    const size_t padded = (bytes + 63) & ~(size_t)63, stride = (size_t)(2 * nout);
    int rc = NRSC5B_ECUDA;
    if (cudaMalloc(&d_in, padded + 64) == cudaSuccess && cudaMalloc(&d_out, (size_t)c->nch * stride * sizeof(int16_t)) == cudaSuccess &&
        cudaMemset(d_in, 0, padded + 64) == cudaSuccess && cudaMemcpy(d_in, in, bytes, cudaMemcpyHostToDevice) == cudaSuccess) {
        rc = c->cs16 ? nrsc5b_chan_run_device_cs16(c, d_in, count, d_out, stride, nullptr) : nrsc5b_chan_run_device(c, d_in, count, d_out, stride, nullptr);
        if (rc == NRSC5B_OK && cudaDeviceSynchronize() != cudaSuccess) {
            fprintf(stderr, "nrsc5_b200: channeliser kernel failed: %s\n", cudaGetErrorString(cudaGetLastError()));
            rc = NRSC5B_ECUDA;
        }
        if (rc == NRSC5B_OK && cudaMemcpy(out, d_out, (size_t)c->nch * stride * sizeof(int16_t), cudaMemcpyDeviceToHost) != cudaSuccess)
            rc = NRSC5B_ECUDA;
    }
    cudaFree(d_in);
    cudaFree(d_out);
    return rc;
}

/* Host convenience (tests): host capture in, host cs16 out[nch][2 * outputs]. */
extern "C" int nrsc5b_chan_run(nrsc5b_channelizer_t *c, const uint8_t *cu8, size_t nbytes, int16_t *out)
{
    if (!c || c->cs16 || !cu8 || !out || (c->rs_L && (nbytes & 1))) return NRSC5B_EINVAL;
    if (!c->rs_L) nbytes &= ~(size_t)63;                    // whole 64-byte rows (32 complex samples); a rate stage takes every sample
    const long long nout = outputs_in(c, (long long)(nbytes / 2));
    if (nout <= 0) return NRSC5B_OK;
    return run_host(c, cu8, nbytes, nbytes, nout, out);
}

extern "C" int nrsc5b_chan_run_cs16(nrsc5b_channelizer_t *c, const int16_t *cs16, size_t nvalues, int16_t *out)
{
    if (!c || !c->cs16 || !cs16 || !out || (nvalues & 1)) return NRSC5B_EINVAL;
    const long long nout = outputs_in(c, (long long)(nvalues / 2));
    if (nout <= 0) return NRSC5B_OK;
    return run_host(c, cs16, 2 * nvalues, nvalues, nout, out);
}

/* The rate stage alone, for kernel-level parity: host capture (cu8 bytes or cs16 int16 values, nvalues of them, even)
 * at fs -> host out[2 K(T)] = y[0 .. K(T) - 1] (I, Q interleaved); synchronous.  fs == R has no stage: NRSC5B_EINVAL. */
extern "C" int nrsc5b_resample(int device, int mode, int decim, uint32_t rate_hz, int cs16, const void *in, size_t nvalues, int16_t *out)
{
    RateStage rs;
    if (!rate_stage(mode, decim, rate_hz, &rs) || rs.L == 1 || (nvalues & 1) || (nvalues && (!in || !out))) return NRSC5B_EINVAL;
    const long long T = (long long)(nvalues / 2), K = resampled_of(rs.L, rs.M, T);
    if (K <= 0) return NRSC5B_OK;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device >= ndev || cudaSetDevice(device) != cudaSuccess) return NRSC5B_ENODEV;
    std::vector<int16_t> G;
    design_resampler(rs, G);
    const size_t bytes = nvalues * (cs16 ? 2 : 1);
    const long long PIECE = 1ll << 22;
    uint8_t *d_in = nullptr, *d_planes = nullptr;
    int16_t *d_G = nullptr;
    std::vector<uint8_t> hi(2 * (size_t)PIECE), lo(2 * (size_t)PIECE);
    bool ok = cudaMalloc(&d_in, (bytes + 15) & ~(size_t)15) == cudaSuccess && cudaMalloc(&d_planes, 4 * PLANE_SAMPLES) == cudaSuccess &&
              cudaMalloc(&d_G, G.size() * sizeof(int16_t)) == cudaSuccess && cudaMemcpy(d_in, in, bytes, cudaMemcpyHostToDevice) == cudaSuccess &&
              cudaMemcpy(d_G, G.data(), G.size() * sizeof(int16_t), cudaMemcpyHostToDevice) == cudaSuccess;
    for (long long r0 = 0; ok && r0 < K; r0 += PIECE) {
        const long long nr = K - r0 < PIECE ? K - r0 : PIECE, q = r0 * rs.M;
        ok = launch_resample(!cs16, d_in, T, q / rs.L, (int)(q % rs.L), rs.L, rs.M, nr, d_G, d_planes, 0, nullptr) == NRSC5B_OK &&
             cudaMemcpy(hi.data(), d_planes, 2 * nr, cudaMemcpyDeviceToHost) == cudaSuccess &&
             cudaMemcpy(lo.data(), d_planes + 2 * PLANE_SAMPLES, 2 * nr, cudaMemcpyDeviceToHost) == cudaSuccess;
        for (long long v = 0; ok && v < 2 * nr; v++) out[2 * r0 + v] = (int16_t)(256 * (int8_t)hi[v] + lo[v]);
    }
    if (!ok) fprintf(stderr, "nrsc5_b200: resampler failed: %s\n", cudaGetErrorString(cudaGetLastError()));
    cudaFree(d_in);
    cudaFree(d_planes);
    cudaFree(d_G);
    return ok ? NRSC5B_OK : NRSC5B_ECUDA;
}
