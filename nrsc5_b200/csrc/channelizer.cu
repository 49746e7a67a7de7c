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
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/nrsc5_b200.h"

namespace nbch {

constexpr int DECIM = 32, TAPS = 256, KBYTES = 2 * TAPS;          // 512 bytes of K per output row
constexpr int CHUNK = 64, NCHUNK = KBYTES / CHUNK;               // K chunks of 64 bytes (one capture-matrix row each)
constexpr int TILE_M = 64;                                        // output samples per tile (one warpgroup's wgmma M)
constexpr int GROUP = 32, TILE_N = 4 * GROUP;                    // channels per CTA, rows of B
constexpr int PERIOD = 11907;                                     // phasor table length (100 kHz / 23.814 MHz = 50 / 11907)
constexpr int SHIFT1 = 13, TAP_SCALE_LOG2 = 19;                   // unit DC gain -> 64 LSB per input LSB (the cu8 -> Q15 convention);
                                                                  // taps stay below 127 * 256 + 127: both bytes of the split are int8
constexpr int THREADS = 384;                                      // producer warpgroup + two consumer warpgroups
constexpr int STAGES = 4;
constexpr uint32_t A_STAGE_BYTES = NCHUNK * TILE_M * CHUNK;      // 32768
constexpr uint32_t W_BYTES = NCHUNK * TILE_N * CHUNK;            // 65536
constexpr int HALF = PERIOD / 2 + 1;                              // phasor table entries 0 .. 5953; the rest are their conjugates
constexpr uint32_t EPI_BYTES = ((HALF * 4 + 15) & ~15) + GROUP * 4 + 2 * GROUP * 4;   // half table, rotation steps, offset corrections
constexpr uint32_t SMEM_BYTES = W_BYTES + STAGES * A_STAGE_BYTES + 1024 /* alignment */ + 256 /* barriers */ + EPI_BYTES;
static_assert(SMEM_BYTES <= 227 * 1024, "more shared memory than an H100 block may have");

struct Params {
    int nch;                   // channels
    int ngroups;
    long long nout;            // output samples per channel
    long long tiles;           // ceil(nout / TILE_M)
    int16_t *out;              // [nch][out_stride] cs16 (I, Q interleaved): int16 pairs
    size_t out_stride;         // int16 values between channels
    const int *rot_step;       // [nch] (1600 m_k) mod 11907
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

struct Barriers {
    uint64_t w_full, a_full[STAGES], a_empty[STAGES];
};

__global__ void __launch_bounds__(THREADS, 1) k_channelize(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w,
                                                           Params p)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t *smem_w = smem;                                        // [8 chunks][128 rows][64 B]
    uint8_t *smem_a = smem + W_BYTES;                              // [STAGES][8 chunks][64 rows][64 B]
    Barriers &bar = *reinterpret_cast<Barriers *>(smem + W_BYTES + STAGES * A_STAGE_BYTES);
    // the epilogue's tables in shared memory: the first half of the phasor table (P[11907 - i] = conj(P[i]), made so on
    // the host), and this group's rotation steps and offset corrections
    short2 *ph_half = reinterpret_cast<short2 *>(smem + W_BYTES + STAGES * A_STAGE_BYTES + 256);
    int *s_rot = reinterpret_cast<int *>(reinterpret_cast<uint8_t *>(ph_half) + ((HALF * 4 + 15) & ~15));
    uint32_t *s_corr = reinterpret_cast<uint32_t *>(s_rot + GROUP);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int group = (int)blockIdx.x % p.ngroups, slot = (int)blockIdx.x / p.ngroups, nslots = (int)gridDim.x / p.ngroups;

    for (int i = threadIdx.x; i < HALF; i += THREADS) ph_half[i] = p.phasor[i];
    for (int i = threadIdx.x; i < GROUP; i += THREADS) {
        const int ch = min(group * GROUP + i, p.nch - 1);
        s_rot[i] = p.rot_step[ch];
        s_corr[2 * i] = (uint32_t)p.corr[2 * ch];
        s_corr[2 * i + 1] = (uint32_t)p.corr[2 * ch + 1];
    }
    if (threadIdx.x == 0) {
        mbar_init(&bar.w_full, 1);
        for (int i = 0; i < STAGES; i++) {
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
            mbar_expect_tx(&bar.w_full, W_BYTES);
            for (int c = 0; c < NCHUNK; c++)
                tma_load_2d(smem_w + (size_t)c * TILE_N * CHUNK, &map_w, &bar.w_full, 0, (group * NCHUNK + c) * TILE_N);
            unsigned it = 0;
            for (long long tile = slot; tile < p.tiles; tile += nslots, it++) {
                const int s = it % STAGES;
                if (it >= STAGES) mbar_wait(&bar.a_empty[s], (it / STAGES - 1) & 1);
                mbar_expect_tx(&bar.a_full[s], A_STAGE_BYTES);
                for (int c = 0; c < NCHUNK; c++)                 // K chunk c of output row n = capture-matrix row n + c
                    tma_load_2d(smem_a + (size_t)s * A_STAGE_BYTES + (size_t)c * TILE_M * CHUNK, &map_x, &bar.a_full[s], 0,
                                (int)(tile * TILE_M) + c);
            }
        }
        return;
    }
    // ===== consumers: warpgroup 1 takes the CTA's even tiles, warpgroup 2 the odd ones =====
    const int wg = wgi - 1, wwarp = warp & 3;
    const int q = lane & 3;                                        // this thread's channels: cl = 4 i + q, i = 0 .. 7
    mbar_wait(&bar.w_full, 0);
    unsigned it = (unsigned)wg;
    for (long long tile = slot + (long long)wg * nslots; tile < p.tiles; tile += 2ll * nslots, it += 2) {
        const int s = it % STAGES;
        mbar_wait(&bar.a_full[s], (it / STAGES) & 1);
        uint32_t d[64];                                            // (the first wgmma overwrites it: accumulate = 0)
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
        for (int c = 0; c < NCHUNK; c++)
#pragma unroll
            for (int k = 0; k < CHUNK / 32; k++) {                 // wgmma K = 32 bytes
                const uint64_t da = wgmma_desc_sw64(smem_a + (size_t)s * A_STAGE_BYTES + (size_t)c * TILE_M * CHUNK, 32u * k);
                const uint64_t db = wgmma_desc_sw64(smem_w + (size_t)c * TILE_N * CHUNK, 32u * k);
                wgmma_u8s8(d, da, db, (c | k) ? 1u : 0u);
            }
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        __syncwarp();
        if (lane == 0) mbar_arrive(&bar.a_empty[s]);               // the stage's bytes are no longer needed

        // ===== epilogue: rows 16 wwarp + lane / 4 (h = 0) and + 8 (h = 1) of the tile =====
        // 32-bit arithmetic throughout: 256 * hi + lo wraps, the filter output itself is bounded by
        // 128 * sum(|Wr| + |Wi|) < 2^28 (checked when the tables are made), so the wrapped sum is the value; after
        // the shift a component is below 2^15 and the rotation's two products stay below 2^31.
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const long long n = tile * TILE_M + 16 * wwarp + (lane >> 2) + 8 * h;
            const int nmod = (int)(n % PERIOD);
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const int cl = 4 * i + q, ch = group * GROUP + cl;
                const unsigned qi = ((unsigned)s_rot[cl] * (unsigned)nmod) % (unsigned)PERIOD;   // < 11907^2 < 2^32
                const bool up = qi >= (unsigned)HALF;
                const short2 v2 = ph_half[up ? (unsigned)PERIOD - qi : qi];
                const int phx = v2.x, phy = up ? -v2.y : v2.y;
                const int ar = (int)(256u * d[8 * i + 2 * h] + d[8 * i + 4 + 2 * h] - s_corr[2 * cl]);
                const int ai = (int)(256u * d[8 * i + 2 * h + 1] + d[8 * i + 5 + 2 * h] - s_corr[2 * cl + 1]);
                const int vr = (ar + (1 << (SHIFT1 - 1))) >> SHIFT1, vi = (ai + (1 << (SHIFT1 - 1))) >> SHIFT1;
                int zr = vr * phx + vi * phy, zi = vi * phx - vr * phy;        // v * conj(P)
                zr = (zr + (1 << 14)) >> 15;
                zi = (zi + (1 << 14)) >> 15;
                zr = zr > 32767 ? 32767 : (zr < -32768 ? -32768 : zr);
                zi = zi > 32767 ? 32767 : (zi < -32768 ? -32768 : zi);
                const uint32_t packed = (uint32_t)(uint16_t)(int16_t)zr | ((uint32_t)(uint16_t)(int16_t)zi << 16);
                if (ch < p.nch && n < p.nout) *reinterpret_cast<uint32_t *>(p.out + (size_t)ch * p.out_stride + 2 * n) = packed;
            }
        }
    }
}

}  // namespace nbch

// ===========================================================================
// host side
// ===========================================================================
using namespace nbch;

struct nrsc5b_channelizer {
    int device, nch, ngroups;
    std::vector<int> offsets;             // m_k: channel offset from the capture centre in 100 kHz steps
    std::vector<int16_t> taps;            // [nch][TAPS][2] (Wr, Wi) of W_k[u]
    std::vector<short2> phasor;           // [PERIOD]
    int8_t *d_w;                          // [ngroups][8][128][64]
    int *d_rot;
    long long *d_corr;
    short2 *d_phasor;
    CUtensorMap map_w;
    PFN_cuTensorMapEncodeTiled_v12000 encode;
};

static double bessel_i0(double x)
{
    double s = 1, t = 1;
    for (int k = 1; k < 50; k++) {
        t *= (x / (2 * k)) * (x / (2 * k));
        s += t;
    }
    return s;
}

// The integer tables of the definition, on the host (no device needed): phasor[11907], taps[nch][256] = W_k[u] and, for
// the kernel, the B operand bytes, the rotation steps and the per-channel offset corrections.
static void make_tables(const int *offsets, int nch, std::vector<short2> &phasor, std::vector<int16_t> &taps, std::vector<int8_t> *w,
                        std::vector<int> *rot, std::vector<long long> *corr)
{
    phasor.resize(PERIOD);
    for (int i = 0; i <= PERIOD / 2; i++) {
        const double a = 2.0 * M_PI * i / PERIOD;
        phasor[i] = make_short2((short)lrint(32767.0 * cos(a)), (short)lrint(32767.0 * sin(a)));
    }
    for (int i = PERIOD / 2 + 1; i < PERIOD; i++)                          // exactly conjugate-symmetric: the kernel keeps half of it
        phasor[i] = make_short2(phasor[PERIOD - i].x, (short)-phasor[PERIOD - i].y);
    // prototype low-pass: Kaiser-windowed sinc, -6 dB at 372 kHz: flat over a hybrid FM channel (+-200 kHz), >= 55 dB down from 544 kHz on (what folds onto the channel after /32), unit DC gain
    std::vector<double> h(TAPS);
    {
        const double fc = 372000.0 / 23814000.0, beta = 5.65;
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
    if (w) w->assign((size_t)ngroups * W_BYTES, 0);
    if (rot) rot->assign(nch, 0);
    if (corr) corr->assign((size_t)nch * 2, 0);
    for (int k = 0; k < nch; k++) {
        const int m = offsets[k];
        const long long step = (((long long)50 * m) % PERIOD + PERIOD) % PERIOD;
        if (rot) (*rot)[k] = (int)((((long long)1600 * m) % PERIOD + PERIOD) % PERIOD);
        long long swr = 0, swi = 0, sabs = 0;
        const int g = k / GROUP, cl = k % GROUP;
        const int brow = 16 * (cl / 4) + 2 * (cl % 4);                   // B rows of the channel: brow + part (+ 8: low bytes)
        for (int u = 0; u < TAPS; u++) {
            // W_k[u] = 2^19 h[255-u] e^{-j 2 pi 50 m u / 11907}, from the integer phasor table
            const short2 ph = phasor[(size_t)((step * u) % PERIOD)];
            const double g0 = ldexp(h[TAPS - 1 - u], TAP_SCALE_LOG2) / 32767.0;
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
                    const size_t base = ((size_t)(g * NCHUNK + ck) * TILE_N) * CHUNK;
                    (*w)[base + (size_t)(brow + part) * CHUNK + b] = (int8_t)hi;
                    (*w)[base + (size_t)(brow + 8 + part) * CHUNK + b] = (int8_t)lo;
                }
        }
        // the kernel's epilogue computes in 32 bits (k_channelize): the filter output must stay below 2^28
        if (128 * sabs >= (1ll << 28)) { fprintf(stderr, "nrsc5_b200: channeliser taps too large for the 32-bit epilogue\n"); abort(); }
        if (corr) {
            (*corr)[2 * k + 0] = 127ll * (swr - swi);
            (*corr)[2 * k + 1] = 127ll * (swi + swr);
        }
    }
}

/* The definition's tables without a device: taps[nch][256][2], phasor[11907][2] (either may be NULL). */
extern "C" int nrsc5b_chan_make_tables(const int *offsets_100khz, int nch, int16_t *taps, int16_t *phasor)
{
    if (!offsets_100khz || nch <= 0 || nch > 4096) return NRSC5B_EINVAL;
    std::vector<short2> ph;
    std::vector<int16_t> tp;
    make_tables(offsets_100khz, nch, ph, tp, nullptr, nullptr, nullptr);
    if (taps) memcpy(taps, tp.data(), tp.size() * sizeof(int16_t));
    if (phasor) memcpy(phasor, ph.data(), PERIOD * sizeof(short2));
    return NRSC5B_OK;
}

extern "C" int nrsc5b_chan_create(nrsc5b_channelizer_t **out, int device, const int *offsets_100khz, int nch)
{
    if (!out || !offsets_100khz || nch <= 0 || nch > 4096) return NRSC5B_EINVAL;
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
    c->offsets.assign(offsets_100khz, offsets_100khz + nch);
    c->d_w = nullptr; c->d_rot = nullptr; c->d_corr = nullptr; c->d_phasor = nullptr;
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
    make_tables(offsets_100khz, nch, c->phasor, c->taps, &w, &rot, &corr);
    bool ok = cudaMalloc(&c->d_w, w.size()) == cudaSuccess && cudaMalloc(&c->d_rot, nch * sizeof(int)) == cudaSuccess &&
              cudaMalloc(&c->d_corr, corr.size() * sizeof(long long)) == cudaSuccess &&
              cudaMalloc(&c->d_phasor, PERIOD * sizeof(short2)) == cudaSuccess;
    ok = ok && cudaMemcpy(c->d_w, w.data(), w.size(), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(c->d_rot, rot.data(), nch * sizeof(int), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(c->d_corr, corr.data(), corr.size() * sizeof(long long), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(c->d_phasor, c->phasor.data(), PERIOD * sizeof(short2), cudaMemcpyHostToDevice) == cudaSuccess;
    if (ok) {
        // taps as a [ngroups * 8 * 128 rows][64 B] matrix, boxes of 128 rows, 64-byte swizzle
        const cuuint64_t dims[2] = { CHUNK, (cuuint64_t)c->ngroups * NCHUNK * TILE_N };
        const cuuint64_t strides[1] = { CHUNK };
        const cuuint32_t box[2] = { CHUNK, TILE_N }, es[2] = { 1, 1 };
        ok = c->encode(&c->map_w, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, c->d_w, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    }
    if (ok) ok = cudaFuncSetAttribute(k_channelize, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES) == cudaSuccess;
    if (!ok) {
        nrsc5b_chan_destroy(c);
        return NRSC5B_ECUDA;
    }
    *out = c;
    return NRSC5B_OK;
}

extern "C" void nrsc5b_chan_destroy(nrsc5b_channelizer_t *c)
{
    if (!c) return;
    cudaFree(c->d_w);
    cudaFree(c->d_rot);
    cudaFree(c->d_corr);
    cudaFree(c->d_phasor);
    delete c;
}

/* The integer tables the definition is made of (for the numpy restatement in the tests): taps[nch][256][2] = (Wr, Wi)
 * of W_k[u], phasor[11907][2]. */
extern "C" int nrsc5b_chan_tables(nrsc5b_channelizer_t *c, int16_t *taps, int16_t *phasor)
{
    if (!c) return NRSC5B_EINVAL;
    if (taps) memcpy(taps, c->taps.data(), c->taps.size() * sizeof(int16_t));
    if (phasor) memcpy(phasor, c->phasor.data(), PERIOD * sizeof(short2));
    return NRSC5B_OK;
}

/* How many output samples a capture of `nbytes` gives per channel: every output needs 256 input samples. */
extern "C" long long nrsc5b_chan_outputs(size_t nbytes)
{
    const long long samples = (long long)(nbytes / 2);
    return samples < TAPS ? 0 : (samples - TAPS) / DECIM + 1;
}

/* Device-resident capture (cu8, I/Q interleaved, 23 814 000 S/s; 64-byte aligned, nbytes of it valid) -> out[nch][out_stride]
 * cs16 on the device (out_stride in int16 values, >= 2 * outputs; 4-byte aligned rows).  Asynchronous on `cuda_stream`. */
extern "C" int nrsc5b_chan_run_device(nrsc5b_channelizer_t *c, const void *d_cu8, size_t nbytes, void *d_out, size_t out_stride,
                                      void *cuda_stream)
{
    if (!c || !d_cu8 || !d_out || ((uintptr_t)d_cu8 & 63) || (nbytes & 63) || ((uintptr_t)d_out & 3) || (out_stride & 1)) return NRSC5B_EINVAL;
    const long long nout = nrsc5b_chan_outputs(nbytes);
    if (nout <= 0) return NRSC5B_OK;
    if ((size_t)(2 * nout) > out_stride) return NRSC5B_EINVAL;
    if (cudaSetDevice(c->device) != cudaSuccess) return NRSC5B_ENODEV;
    // the capture as a [rows][64 B] matrix; rows past the end read as zero (only rows of outputs >= nout touch them)
    CUtensorMap map_x;
    const cuuint64_t dims[2] = { CHUNK, (cuuint64_t)(nbytes / CHUNK) };
    const cuuint64_t strides[1] = { CHUNK };
    const cuuint32_t box[2] = { CHUNK, TILE_M }, es[2] = { 1, 1 };
    if (c->encode(&map_x, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void *>(d_cu8), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return NRSC5B_ECUDA;
    Params p;
    p.nch = c->nch;
    p.ngroups = c->ngroups;
    p.nout = nout;
    p.tiles = (nout + TILE_M - 1) / TILE_M;
    p.out = reinterpret_cast<int16_t *>(d_out);
    p.out_stride = out_stride;
    p.rot_step = c->d_rot;
    p.corr = c->d_corr;
    p.phasor = c->d_phasor;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device);
    long long slots = sms / c->ngroups;
    if (slots < 1) slots = 1;
    if (slots > p.tiles) slots = p.tiles;
    k_channelize<<<(unsigned)(slots * c->ngroups), THREADS, SMEM_BYTES, reinterpret_cast<cudaStream_t>(cuda_stream)>>>(map_x, c->map_w, p);
    return cudaGetLastError() == cudaSuccess ? NRSC5B_OK : NRSC5B_ECUDA;
}

/* Host convenience (tests): host capture in, host cs16 out[nch][2 * outputs]. */
extern "C" int nrsc5b_chan_run(nrsc5b_channelizer_t *c, const uint8_t *cu8, size_t nbytes, int16_t *out)
{
    if (!c || !cu8 || !out) return NRSC5B_EINVAL;
    nbytes &= ~(size_t)63;                                  // whole 64-byte rows (32 complex samples)
    const long long nout = nrsc5b_chan_outputs(nbytes);
    if (nout <= 0) return NRSC5B_OK;
    if (cudaSetDevice(c->device) != cudaSuccess) return NRSC5B_ENODEV;
    uint8_t *d_in = nullptr;
    int16_t *d_out = nullptr;
    const size_t padded = (nbytes + 63) & ~(size_t)63, stride = (size_t)(2 * nout);
    int rc = NRSC5B_ECUDA;
    if (cudaMalloc(&d_in, padded + 64) == cudaSuccess && cudaMalloc(&d_out, (size_t)c->nch * stride * sizeof(int16_t)) == cudaSuccess &&
        cudaMemset(d_in, 0, padded + 64) == cudaSuccess && cudaMemcpy(d_in, cu8, nbytes, cudaMemcpyHostToDevice) == cudaSuccess) {
        rc = nrsc5b_chan_run_device(c, d_in, nbytes, d_out, stride, nullptr);
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
