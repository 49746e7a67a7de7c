// Band scan: which channels of a channelised band carry an NRSC-5 signal, and each one's symbol timing, fractional CFO
// and per-sideband SNR.  The reference has no counterpart (its ingest is one narrowband device per handle, reference
// src/nrsc5.c:130-207); the nearest thing is the coarse acquisition of one stream (src/acquire.c:120-158), which folds
// the cyclic-prefix correlation over 32 symbols and takes the arg-max.  The scan does that for every channel at once,
// exactly in integers, over as many symbols as it is given.  Definition (include/nrsc5_b200.h restates it):
//
//     z_s[n]    = sat16((sum_{u<64} g_s[u] y[n - 63 + u] + 2^14) >> 15)      per component, n = 0 (mod q), n >= 63
//     p_s[n]    = z_s[n] conj(z_s[n + F]),  e_s[n] = |z_s[n]|^2 + |z_s[n + F]|^2              (int64; n + F < T)
//     Fold_s[j] = sum_m p_s[q j + m S],     En_s[j] likewise                                  j < J = S / q
//     C_s[j]    = sum_{i < P/q} Fold_s[(j + i) mod J],  E_s[j] likewise
//
// FM: F = 2048, P = 112, q = 4; AM: F = 256, P = 14, q = 2; S = F + P.  g_U is a Kaiser-windowed complex band-pass
// over the upper sideband's carriers and g_L = conj(g_U) the mirror image, so both filters come from four real sums:
// with g_U = a + jb and y = c + jd, A = sum ac, B = sum bd, Cs = sum ad, D = sum bc give z_U = (A - B, Cs + D) and
// z_L = (A + B, Cs - D).  make_taps keeps sum|a| and sum|b| below 2^16, so each of the four sums is exact in int32.
//
// k_scan: one CTA per (channel, span of chunks).  A chunk is CH product positions (a whole number of symbols): its
// CH + F + 63 input samples are staged into shared memory by cp.async, split into q phase planes so that the threads of
// a warp read consecutive words for every tap; then (CH + F) / q filter outputs of both sidebands, then the products.
// A thread owns fold positions j and keeps their six sums in registers over all the CTA's chunks, then adds them into
// the handle's int64 accumulators with atomicAdd: integer addition is associative, so the accumulators equal the
// definition bit for bit whatever the grid and the split into pushes.  Streaming keeps the last F + 63 samples of
// every channel (the history) and T, the samples pushed: a push counts exactly the products whose later sample is new.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/nrsc5_b200.h"
#include "chan_scan.h"

namespace nbscan {

constexpr int NTAPS = 64, HALO = NTAPS - 1;
constexpr int THREADS = 256;
constexpr long long MAX_SYMBOLS = 1ll << 24;      // |Re p|, |Im p| <= 2^31 and e <= 2^32: Fold, En fit int64 up to 2^24 symbols

struct Mode {
    int F, P, q;
    double fs;
    double c;        // tau(M) = c / sqrt(M P / q)
    double c1;       // tau_1(M) = c1 / sqrt(M P / q), each sideband at the timing found
    double kappa;    // ceiling of rho_s for a noise-free station
};
// c and kappa: see include/nrsc5_b200.h (nrsc5b_scan_make_tables) for where they come from
static const Mode MODES[2] = {
    { 2048, 112, 4, 744187.5, NRSC5B_SCAN_C_FM, NRSC5B_SCAN_C1_FM, NRSC5B_SCAN_KAPPA_FM },
    { 256, 14, 2, 46511.71875, NRSC5B_SCAN_C_AM, NRSC5B_SCAN_C1_AM, NRSC5B_SCAN_KAPPA_AM },
};

struct Taps {
    int2 g[NTAPS];                                // (Re, Im) of g_U[u]
};

struct ScanParams {
    const uint32_t *in;                           // the push's samples, channel k at in + k * in_stride (cs16 pairs)
    long long in_stride;                          // in 32-bit words
    const uint32_t *hist;                         // [nch][hist_cap]: samples T0 - hist_len .. T0 - 1 of every channel
    int hist_cap, hist_len;
    long long t0, t1;                             // samples pushed before / after this push
    long long n_a, n_b;                           // the push's product positions: n_a <= n < n_b, n = 0 (mod q)
    int chunks, chunks_per_cta;
    unsigned long long *acc;                      // [nch][2 sidebands][3: Fold re, Fold im, En][J]
};

__device__ __forceinline__ int sat16(long long v) { return v > 32767 ? 32767 : v < -32768 ? -32768 : (int)v; }

template <int F, int P, int Q, int CH>
struct Geometry {
    static constexpr int S = F + P, J = S / Q, W = CH + F + HALO, ZN = (CH + F) / Q;
    // plane length = 32 / Q (mod 32): lane i of a staging warp writes bank (32 / Q) (i % Q) + i / Q, all distinct
    static constexpr int PL = ((W + Q - 1) / Q + 31) / 32 * 32 + 32 / Q;
    static constexpr int JPT = (J + THREADS - 1) / THREADS;    // fold positions per thread
    static constexpr size_t SMEM = (size_t)(Q * PL + 2 * ZN) * sizeof(uint32_t);
    static_assert(CH % S == 0 && S % Q == 0 && F % Q == 0 && P % Q == 0, "chunk / symbol / subsampling mismatch");
};

template <int F, int P, int Q, int CH>
__global__ void __launch_bounds__(THREADS) k_scan(const __grid_constant__ ScanParams p, const __grid_constant__ Taps taps)
{
    using G = Geometry<F, P, Q, CH>;
    extern __shared__ __align__(16) uint32_t smem[];
    uint32_t *planes = smem;                      // [Q][PL]: sample i of the chunk window at planes[i % Q][i / Q]
    uint32_t *zu = smem + Q * G::PL, *zl = zu + G::ZN;
    const int ch = blockIdx.y, tid = threadIdx.x;
    const uint32_t *in = p.in + ch * p.in_stride;
    const uint32_t *hist = p.hist + (size_t)ch * p.hist_cap;
    const long long h0 = p.t0 - p.hist_len;       // absolute index of hist[0]

    long long acc[G::JPT][6];
#pragma unroll
    for (int r = 0; r < G::JPT; r++)
#pragma unroll
        for (int c = 0; c < 6; c++) acc[r][c] = 0;

    const int c_first = blockIdx.x * p.chunks_per_cta;
    const int c_last = min(p.chunks, c_first + p.chunks_per_cta);
    for (int ck = c_first; ck < c_last; ck++) {
        const long long c0 = p.n_a + (long long)ck * CH;          // first product position of the chunk (= 0 mod q)
        // stage samples c0 - 63 .. c0 + CH + F - 1: the history, the push's own samples, zero where neither holds them
        for (int i = tid; i < G::W; i += THREADS) {
            const long long a = c0 - HALO + i;
            const uint32_t *src = in;
            int bytes = 0;
            if (a >= h0 && a < p.t0) { src = hist + (a - h0); bytes = 4; }
            else if (a >= p.t0 && a < p.t1) { src = in + (a - p.t0); bytes = 4; }
            const unsigned dst = (unsigned)__cvta_generic_to_shared(planes + (i % Q) * G::PL + i / Q);
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(dst), "l"(src), "r"(bytes));
        }
        asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;\n" ::: "memory");
        __syncthreads();
        // both sidebands' filter outputs at c0 + q k, k < ZN
        for (int k = tid; k < G::ZN; k += THREADS) {
            int A = 0, B = 0, Cs = 0, D = 0;
#pragma unroll
            for (int u = 0; u < NTAPS; u++) {
                const uint32_t w = planes[(u % Q) * G::PL + k + u / Q];
                const int c = (int)(short)(w & 0xffffu), d = (int)w >> 16;
                const int ga = taps.g[u].x, gb = taps.g[u].y;
                A += ga * c;
                B += gb * d;
                Cs += ga * d;
                D += gb * c;
            }
            const int ur = sat16(((long long)A - B + (1 << 14)) >> 15), ui = sat16(((long long)Cs + D + (1 << 14)) >> 15);
            const int lr = sat16(((long long)A + B + (1 << 14)) >> 15), li = sat16(((long long)Cs - D + (1 << 14)) >> 15);
            zu[k] = (uint32_t)(ur & 0xffff) | ((uint32_t)ui << 16);
            zl[k] = (uint32_t)(lr & 0xffff) | ((uint32_t)li << 16);
        }
        __syncthreads();
        // products: fold position j takes n = c0 + off + m S, m < CH / S
        const int c0mod = (int)(c0 % G::S);
#pragma unroll
        for (int r = 0; r < G::JPT; r++) {
            const int j = tid + r * THREADS;
            if (j >= G::J) break;
            int off = Q * j - c0mod;
            if (off < 0) off += G::S;
            for (int m = 0; m < CH / G::S; m++) {
                const long long n = c0 + off + (long long)m * G::S;
                if (n >= p.n_b) break;
                const int k = (off + m * G::S) / Q;
#pragma unroll
                for (int s = 0; s < 2; s++) {
                    const uint32_t *z = s ? zu : zl;
                    const uint32_t w0 = z[k], w1 = z[k + F / Q];
                    const long long ar = (short)(w0 & 0xffffu), ai = (int)w0 >> 16, br = (short)(w1 & 0xffffu), bi = (int)w1 >> 16;
                    acc[r][3 * s + 0] += ar * br + ai * bi;
                    acc[r][3 * s + 1] += ai * br - ar * bi;
                    acc[r][3 * s + 2] += ar * ar + ai * ai + br * br + bi * bi;
                }
            }
        }
        __syncthreads();                           // the planes and z are rewritten by the next chunk
    }
    unsigned long long *out = p.acc + (size_t)ch * 6 * G::J;
#pragma unroll
    for (int r = 0; r < G::JPT; r++) {
        const int j = tid + r * THREADS;
        if (j >= G::J) break;
#pragma unroll
        for (int c = 0; c < 6; c++)
            if (acc[r][c]) atomicAdd(out + c * G::J + j, (unsigned long long)acc[r][c]);
    }
}

// sum |y|^2 of the push's samples into a 128-bit counter per channel (lo, hi): a carry out of lo goes into hi, so the
// total is exact and independent of the order of the additions
__global__ void __launch_bounds__(THREADS) k_scan_power(const uint32_t *in, long long in_stride, long long n, unsigned long long *pow)
{
    const uint32_t *x = in + blockIdx.y * in_stride;
    long long s = 0;
    for (long long i = blockIdx.x * (long long)THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * THREADS) {
        const uint32_t w = x[i];
        const long long a = (short)(w & 0xffffu), b = (int)w >> 16;
        s += a * a + b * b;
    }
    __shared__ long long red[THREADS / 32];
    for (int o = 16; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < THREADS / 32; w++) t += (unsigned long long)red[w];
        if (t) {
            unsigned long long *c = pow + 2 * blockIdx.y;
            const unsigned long long old = atomicAdd(c, t);
            if (old + t < old) atomicAdd(c + 1, 1ull);
        }
    }
}

__device__ double i128_to_double(__int128 x)
{
    const bool neg = x < 0;
    const unsigned __int128 m = neg ? (unsigned __int128)(-x) : (unsigned __int128)x;
    const double v = __dadd_rn(__dmul_rn((double)(unsigned long long)(m >> 64), 18446744073709551616.0), (double)(unsigned long long)m);
    return neg ? -v : v;
}

struct FinishParams {
    const unsigned long long *acc;                 // [nch][6][J]
    const unsigned long long *pow;                 // [nch][2]
    long long *raw;                                // [nch][NRSC5B_SCAN_RAW(J)] or null
    nrsc5b_scan_t *res;                            // [nch]
    long long samples, products;                   // T and N_p(T)
    double fs, kappa, threshold, threshold_sideband, symbols;
    int detect;                                    // M >= 32
};

// One CTA per channel: the window sums C_s, E_s, the arg-max of |C - mean C| (ties: the smallest j) and the metrics,
// every double operation rounded as written (no contraction) so that the numpy restatement reproduces them.
template <int F, int P, int Q>
__global__ void __launch_bounds__(THREADS) k_scan_finish(const __grid_constant__ FinishParams p)
{
    constexpr int S = F + P, J = S / Q, W = P / Q;
    __shared__ long long cw[6][J];                 // C_L re, im, E_L, C_U re, im, E_U
    __shared__ __int128 tot[6];
    __shared__ double best_v[THREADS];
    __shared__ int best_j[THREADS];
    const int ch = blockIdx.x, tid = threadIdx.x;
    const unsigned long long *a = p.acc + (size_t)ch * 6 * J;
    for (int i = tid; i < 6 * J; i += THREADS) {
        const int c = i / J, j = i % J;
        long long s = 0;
        for (int k = 0; k < W; k++) s += (long long)a[c * J + (j + k) % J];
        cw[c][j] = s;
    }
    if (tid < 6) {
        __int128 s = 0;
        for (int j = 0; j < J; j++) s += (long long)a[tid * J + j];
        tot[tid] = s * W;                          // sum_j C_s[j] = (P / q) sum_j Fold_s[j]
    }
    __syncthreads();
    if (p.raw) {
        long long *r = p.raw + (size_t)ch * NRSC5B_SCAN_RAW(J);
        for (int i = tid; i < 6 * J; i += THREADS) {
            r[i] = (long long)a[i];
            r[6 * J + i] = cw[i / J][i % J];
        }
        if (tid == 0) {
            r[12 * J] = (long long)p.pow[2 * ch];
            r[12 * J + 1] = (long long)p.pow[2 * ch + 1];
        }
    }
    // |C[j] - mean C|^2 with C = C_L + C_U; D = (J C[j] - sum C) / J exactly in 128 bits before the one rounding
    double bv = -1.0;
    int bj = 0;
    for (int j = tid; j < J; j += THREADS) {
        const double dr = i128_to_double((__int128)J * ((__int128)cw[0][j] + cw[3][j]) - (tot[0] + tot[3])) / J;
        const double di = i128_to_double((__int128)J * ((__int128)cw[1][j] + cw[4][j]) - (tot[1] + tot[4])) / J;
        const double v = __dadd_rn(__dmul_rn(dr, dr), __dmul_rn(di, di));
        if (v > bv) { bv = v; bj = j; }
    }
    best_v[tid] = bv;
    best_j[tid] = bj;
    __syncthreads();
    for (int o = THREADS / 2; o; o >>= 1) {
        if (tid < o) {
            const double v2 = best_v[tid + o];
            const int j2 = best_j[tid + o];
            if (v2 > best_v[tid] || (v2 == best_v[tid] && j2 < best_j[tid])) { best_v[tid] = v2; best_j[tid] = j2; }
        }
        __syncthreads();
    }
    if (tid) return;
    const int j = best_j[0];
    nrsc5b_scan_t r;
    const double dr = i128_to_double((__int128)J * ((__int128)cw[0][j] + cw[3][j]) - (tot[0] + tot[3])) / J;
    const double di = i128_to_double((__int128)J * ((__int128)cw[1][j] + cw[4][j]) - (tot[1] + tot[4])) / J;
    const double mag = sqrt(best_v[0]);
    const double e = 0.5 * (double)(cw[2][j] + cw[5][j]);
    r.score = e > 0 ? mag / e : 0.0;
    r.threshold = p.threshold;
    r.threshold_sideband = p.threshold_sideband;
    r.symbols = p.symbols;
    r.timing = ((Q * j - 32) % S + S) % S;
    r.cfo_hz = mag > 0 ? -atan2(di, dr) * p.fs / (2.0 * M_PI * F) : 0.0;
    double snr[2], pw[2], sc[2], dre[2], dim[2];
    for (int s = 0; s < 2; s++) {
        const double sr = i128_to_double((__int128)J * cw[3 * s][j] - tot[3 * s]) / J;
        const double si = i128_to_double((__int128)J * cw[3 * s + 1][j] - tot[3 * s + 1]) / J;
        const double emean = i128_to_double(tot[3 * s + 2]) / J;
        const double ms = sqrt(__dadd_rn(__dmul_rn(sr, sr), __dmul_rn(si, si)));
        dre[s] = sr;
        dim[s] = si;
        const double es = 0.5 * (double)cw[3 * s + 2][j];
        sc[s] = es > 0 ? ms / es : 0.0;
        const double rho = emean > 0 ? ms / (0.5 * emean) : 0.0;
        snr[s] = rho <= 0 ? -INFINITY : rho >= p.kappa ? INFINITY : 10.0 * log10(rho / (p.kappa - rho));
        // mean |z_s|^2 over the products' samples: sum_j En_s[j] counts 2 N_p of them
        const double en = i128_to_double(tot[3 * s + 2] / W);
        pw[s] = p.products > 0 && en > 0 ? 10.0 * log10(en / (2.0 * (double)p.products) / 1073741824.0) : -INFINITY;
    }
    r.score_lower = sc[0];
    r.score_upper = sc[1];
    // the two sidebands of one station share its carrier: their CP correlations agree in phase (within 45 degrees)
    const double dot = __dadd_rn(__dmul_rn(dre[0], dre[1]), __dmul_rn(dim[0], dim[1]));
    const double m2 = sqrt(__dmul_rn(__dadd_rn(__dmul_rn(dre[0], dre[0]), __dmul_rn(dim[0], dim[0])),
                                     __dadd_rn(__dmul_rn(dre[1], dre[1]), __dmul_rn(dim[1], dim[1]))));
    r.detected = p.detect && r.score >= p.threshold && sc[0] >= p.threshold_sideband && sc[1] >= p.threshold_sideband &&
                 dot >= M_SQRT1_2 * m2;
    r.snr_db_lower = snr[0];
    r.snr_db_upper = snr[1];
    r.power_dbfs_lower = pw[0];
    r.power_dbfs_upper = pw[1];
    const double py = i128_to_double(((__int128)p.pow[2 * ch + 1] << 64) | (__int128)p.pow[2 * ch]);
    r.power_dbfs = p.samples > 0 && py > 0 ? 10.0 * log10(py / (double)p.samples / 1073741824.0) : -INFINITY;
    p.res[ch] = r;
}

// FM: 4 symbols a chunk; AM: 32 (the same 8640 positions)
constexpr int CH_FM = 4 * 2160, CH_AM = 32 * 270;
using GFM = Geometry<2048, 112, 4, CH_FM>;
using GAM = Geometry<256, 14, 2, CH_AM>;

}  // namespace nbscan

// ===========================================================================
// host side
// ===========================================================================
using namespace nbscan;

struct nrsc5b_scanner {
    int device, mode, nch;
    const Mode *m;
    Taps taps;
    long long pushed;                              // T
    int hist_cap, hist_len;                        // F + 63; min(T, F + 63)
    uint32_t *d_hist[2];                           // [nch][hist_cap], the current one is d_hist[cur]
    int cur;
    unsigned long long *d_acc, *d_pow;             // [nch][6][J], [nch][2]
    long long *d_raw;                              // [nch][raw] (finish)
    nrsc5b_scan_t *d_res;
    uint32_t *d_in;                                // nrsc5b_scan_push's staging, in_cap samples per channel
    size_t in_cap;
    int16_t *d_chout;                              // nrsc5b_chan_scan's channel output, [nch][2 CHAN_OUT]
    cudaEvent_t done;                              // the last push (the next one, reset and result follow it)
};

namespace {

constexpr long long CHAN_OUT = 1 << 16;            // channel outputs per piece of nrsc5b_chan_scan

int J_of(const Mode &m) { return (m.F + m.P) / m.q; }
int raw_of(const Mode &m) { return NRSC5B_SCAN_RAW(J_of(m)); }

double bessel_i0(double x)
{
    double s = 1, t = 1;
    for (int k = 1; k < 50; k++) {
        t *= (x / (2 * k)) * (x / (2 * k));
        s += t;
    }
    return s;
}

double kaiser_beta(double A) { return 0.5842 * pow(A - 21, 0.4) + 0.07886 * (A - 21); }

// g_U[u], Q15: a Kaiser-windowed sinc low-pass (-6 dB at fc, unit DC gain) moved to the upper sideband's centre f0
//   FM: f0 = 151 kHz, fc = 37 kHz, window for 42 dB: the two transitions lie between 100 kHz and carrier 356
//       (129.4 kHz) and between carrier 478 (173.7 kHz) and 202 kHz; measured >= 41.3 dB down at |f| <= 100 kHz and
//       at f >= 202 kHz, within 0.13 dB over carriers 356..478
//   AM: f0 = 10.4 kHz, fc = 5 kHz, window for 37 dB, minus the window scaled to cancel the sum (a null at DC); the
//       rounding residual goes to tap 31, so sum g_U = 0 exactly.  Measured within 0.11 dB over 6.5 - 14 kHz, 15.6 dB
//       down at 5 kHz and 49 dB at 3 kHz: the passband is carriers 33..81 (see include/nrsc5_b200.h for why).
// (the phase reference is the filter's centre, so h symmetric makes g_L = conj(g_U) the mirror image)
void make_taps(int mode, Taps &t)
{
    const bool am = mode == NRSC5B_MODE_AM;
    const Mode &m = MODES[am];
    const double f0 = am ? 10400.0 : 151e3;
    const double fc = am ? 5000.0 : 37e3;
    const double beta = kaiser_beta(am ? 37.0 : 42.0), i0b = bessel_i0(beta);
    double h[NTAPS], w[NTAPS], hs = 0, ws = 0;
    for (int u = 0; u < NTAPS; u++) {
        const double x = u - 31.5, r = 2.0 * u / (NTAPS - 1) - 1.0;
        w[u] = bessel_i0(beta * sqrt(1.0 - r * r)) / i0b;
        const double a = 2 * fc / m.fs * x;
        h[u] = 2 * fc / m.fs * (a == 0 ? 1.0 : sin(M_PI * a) / (M_PI * a)) * w[u];
        hs += h[u];
        ws += w[u];
    }
    double gr[NTAPS], gi[NTAPS], sr = 0, si = 0;
    for (int u = 0; u < NTAPS; u++) {
        const double ph = -2 * M_PI * f0 / m.fs * (u - 31.5);
        gr[u] = h[u] / hs * cos(ph);
        gi[u] = h[u] / hs * sin(ph);
        sr += gr[u];
        si += gi[u];
    }
    int ar = 0, ai = 0;
    for (int u = 0; u < NTAPS; u++) {
        if (am) {
            gr[u] -= sr / ws * w[u];
            gi[u] -= si / ws * w[u];
        }
        t.g[u] = make_int2((int)lrint(32768.0 * gr[u]), (int)lrint(32768.0 * gi[u]));
        ar += t.g[u].x;
        ai += t.g[u].y;
    }
    if (am) {
        t.g[31].x -= ar;
        t.g[31].y -= ai;
    }
}

// products a capture of T samples holds per sideband: n = 0 (mod q), 63 <= n <= T - 1 - F
long long products_of(const Mode &m, long long T)
{
    const long long first = (HALO + m.q - 1) / m.q, last = T - 1 - m.F;
    return last < first * m.q ? 0 : last / m.q - first + 1;
}

int valid_mode(int mode) { return mode == NRSC5B_MODE_FM || mode == NRSC5B_MODE_AM; }

}  // namespace

extern "C" int nrsc5b_scan_make_tables(int mode, int16_t *taps, double *kappa)
{
    if (!valid_mode(mode)) return NRSC5B_EINVAL;
    Taps t;
    make_taps(mode, t);
    if (taps)
        for (int u = 0; u < NTAPS; u++) {
            taps[2 * u] = (int16_t)t.g[u].x;
            taps[2 * u + 1] = (int16_t)t.g[u].y;
        }
    if (kappa) *kappa = MODES[mode == NRSC5B_MODE_AM].kappa;
    return NRSC5B_OK;
}

extern "C" void nrsc5b_scan_destroy(nrsc5b_scanner_t *s)
{
    if (!s) return;
    cudaFree(s->d_hist[0]);
    cudaFree(s->d_hist[1]);
    cudaFree(s->d_acc);
    cudaFree(s->d_pow);
    cudaFree(s->d_raw);
    cudaFree(s->d_res);
    cudaFree(s->d_in);
    cudaFree(s->d_chout);
    if (s->done) cudaEventDestroy(s->done);
    delete s;
}

extern "C" int nrsc5b_scan_reset(nrsc5b_scanner_t *s)
{
    if (!s) return NRSC5B_EINVAL;
    if (cudaSetDevice(s->device) != cudaSuccess) return NRSC5B_ENODEV;
    if (cudaEventSynchronize(s->done) != cudaSuccess) return NRSC5B_ECUDA;
    s->pushed = 0;
    s->hist_len = 0;
    const bool ok = cudaMemsetAsync(s->d_acc, 0, (size_t)s->nch * 6 * J_of(*s->m) * sizeof(long long), nullptr) == cudaSuccess &&
                    cudaMemsetAsync(s->d_pow, 0, (size_t)s->nch * 2 * sizeof(long long), nullptr) == cudaSuccess &&
                    cudaStreamSynchronize(nullptr) == cudaSuccess;
    return ok ? NRSC5B_OK : NRSC5B_ECUDA;
}

extern "C" int nrsc5b_scan_create(nrsc5b_scanner_t **out, int device, int mode, int nch)
{
    if (!out || !valid_mode(mode) || nch <= 0 || nch > 4096) return NRSC5B_EINVAL;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
        fprintf(stderr, "nrsc5_b200: no usable CUDA device (the band scan has no CPU path)\n");
        return NRSC5B_ENODEV;
    }
    if (cudaSetDevice(device) != cudaSuccess) return NRSC5B_ENODEV;
    nrsc5b_scanner *s = new nrsc5b_scanner();
    s->device = device;
    s->mode = mode;
    s->nch = nch;
    s->m = &MODES[mode == NRSC5B_MODE_AM];
    make_taps(mode, s->taps);
    s->hist_cap = s->m->F + HALO;
    s->cur = 0;
    const size_t J = (size_t)J_of(*s->m), n = (size_t)nch;
    bool ok = cudaMalloc(&s->d_hist[0], n * s->hist_cap * 4) == cudaSuccess && cudaMalloc(&s->d_hist[1], n * s->hist_cap * 4) == cudaSuccess &&
              cudaMalloc(&s->d_acc, n * 6 * J * 8) == cudaSuccess && cudaMalloc(&s->d_pow, n * 2 * 8) == cudaSuccess &&
              cudaMalloc(&s->d_raw, n * raw_of(*s->m) * 8) == cudaSuccess && cudaMalloc(&s->d_res, n * sizeof(nrsc5b_scan_t)) == cudaSuccess &&
              cudaEventCreateWithFlags(&s->done, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(k_scan<2048, 112, 4, CH_FM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GFM::SMEM) == cudaSuccess &&
         cudaFuncSetAttribute(k_scan<256, 14, 2, CH_AM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GAM::SMEM) == cudaSuccess;
    if (!ok || nrsc5b_scan_reset(s) != NRSC5B_OK) {
        nrsc5b_scan_destroy(s);
        return NRSC5B_ECUDA;
    }
    *out = s;
    return NRSC5B_OK;
}

// work already queued on another CUDA stream that the next call must follow (pushes may come on different streams)
static int follow(nrsc5b_scanner_t *s, cudaStream_t st) { return cudaStreamWaitEvent(st, s->done, 0) == cudaSuccess ? NRSC5B_OK : NRSC5B_ECUDA; }

extern "C" int nrsc5b_scan_push_device(nrsc5b_scanner_t *s, const void *d_ch, size_t stride, size_t nsamples, void *cuda_stream)
{
    if (!s || (nsamples && (!d_ch || ((uintptr_t)d_ch & 3) || (stride & 1) || stride < 2 * nsamples))) return NRSC5B_EINVAL;
    const Mode &m = *s->m;
    const long long t0 = s->pushed, t1 = t0 + (long long)nsamples;
    if (t1 / (m.F + m.P) > MAX_SYMBOLS) return NRSC5B_EINVAL;
    if (!nsamples) return NRSC5B_OK;
    if (cudaSetDevice(s->device) != cudaSuccess) return NRSC5B_ENODEV;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(cuda_stream);
    if (follow(s, st)) return NRSC5B_ECUDA;
    const uint32_t *in = reinterpret_cast<const uint32_t *>(d_ch);
    const long long in_stride = (long long)(stride / 2);
    // products whose later sample is new: max(T0 - F, 63) <= n < T1 - F, n = 0 (mod q)
    long long n_a = t0 - m.F > HALO ? t0 - m.F : HALO;
    n_a = (n_a + m.q - 1) / m.q * m.q;
    const long long n_b = t1 - m.F;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, s->device);
    const bool am = s->mode == NRSC5B_MODE_AM;
    if (n_b > n_a) {
        const int CH = am ? CH_AM : CH_FM;
        ScanParams p;
        p.in = in;
        p.in_stride = in_stride;
        p.hist = s->d_hist[s->cur];
        p.hist_cap = s->hist_cap;
        p.hist_len = s->hist_len;
        p.t0 = t0;
        p.t1 = t1;
        p.n_a = n_a;
        p.n_b = n_b;
        p.chunks = (int)((n_b - n_a + CH - 1) / CH);
        // about eight CTAs per SM in all: enough to fill the machine, few enough that the atomics stay a small cost
        const long long want = (long long)sms * 8;
        long long per = ((long long)p.chunks * s->nch + want - 1) / want;
        if (per < 1) per = 1;
        p.chunks_per_cta = (int)per;
        p.acc = s->d_acc;
        const dim3 grid((unsigned)((p.chunks + per - 1) / per), (unsigned)s->nch);
        if (am) k_scan<256, 14, 2, CH_AM><<<grid, THREADS, GAM::SMEM, st>>>(p, s->taps);
        else k_scan<2048, 112, 4, CH_FM><<<grid, THREADS, GFM::SMEM, st>>>(p, s->taps);
        if (cudaGetLastError() != cudaSuccess) return NRSC5B_ECUDA;
    }
    long long pb = ((long long)nsamples + THREADS * 16 - 1) / (THREADS * 16), pmax = (long long)sms * 8 / s->nch;
    if (pb > pmax) pb = pmax;
    if (pb < 1) pb = 1;
    k_scan_power<<<dim3((unsigned)pb, (unsigned)s->nch), THREADS, 0, st>>>(in, in_stride, (long long)nsamples, s->d_pow);
    if (cudaGetLastError() != cudaSuccess) return NRSC5B_ECUDA;
    // the new history: the last min(T1, F + 63) samples of (history, push)
    const long long hn = t1 < s->hist_cap ? t1 : s->hist_cap;
    uint32_t *dst = s->d_hist[1 - s->cur];
    const size_t hp = (size_t)s->hist_cap * 4, ip = (size_t)in_stride * 4;
    bool ok;
    if ((long long)nsamples >= hn) {
        ok = cudaMemcpy2DAsync(dst, hp, in + (nsamples - hn), ip, (size_t)hn * 4, s->nch, cudaMemcpyDeviceToDevice, st) == cudaSuccess;
    } else {
        const long long keep = hn - (long long)nsamples;
        ok = cudaMemcpy2DAsync(dst, hp, s->d_hist[s->cur] + (s->hist_len - keep), hp, (size_t)keep * 4, s->nch, cudaMemcpyDeviceToDevice,
                               st) == cudaSuccess &&
             cudaMemcpy2DAsync(dst + keep, hp, in, ip, nsamples * 4, s->nch, cudaMemcpyDeviceToDevice, st) == cudaSuccess;
    }
    if (!ok || cudaEventRecord(s->done, st) != cudaSuccess) return NRSC5B_ECUDA;
    s->cur = 1 - s->cur;
    s->hist_len = (int)hn;
    s->pushed = t1;
    return NRSC5B_OK;
}

extern "C" int nrsc5b_scan_push(nrsc5b_scanner_t *s, const int16_t *cs16, size_t nsamples)
{
    if (!s || (nsamples && !cs16)) return NRSC5B_EINVAL;
    if (!nsamples) return nrsc5b_scan_push_device(s, nullptr, 0, 0, nullptr);
    if (cudaSetDevice(s->device) != cudaSuccess) return NRSC5B_ENODEV;
    if (nsamples > s->in_cap) {
        cudaFree(s->d_in);
        s->d_in = nullptr;
        s->in_cap = 0;
        if (cudaMalloc(&s->d_in, (size_t)s->nch * nsamples * 4) != cudaSuccess) return NRSC5B_ENOMEM;
        s->in_cap = nsamples;
    }
    if (cudaEventSynchronize(s->done) != cudaSuccess ||
        cudaMemcpy(s->d_in, cs16, (size_t)s->nch * nsamples * 4, cudaMemcpyHostToDevice) != cudaSuccess)
        return NRSC5B_ECUDA;
    const int rc = nrsc5b_scan_push_device(s, s->d_in, 2 * nsamples, nsamples, nullptr);
    if (rc) return rc;
    return cudaEventSynchronize(s->done) == cudaSuccess ? NRSC5B_OK : NRSC5B_ECUDA;
}

extern "C" int nrsc5b_scan_result(nrsc5b_scanner_t *s, nrsc5b_scan_t *out, int64_t *raw)
{
    if (!s || !out) return NRSC5B_EINVAL;
    if (cudaSetDevice(s->device) != cudaSuccess) return NRSC5B_ENODEV;
    const Mode &m = *s->m;
    const long long np = products_of(m, s->pushed);
    FinishParams p;
    p.acc = s->d_acc;
    p.pow = s->d_pow;
    p.raw = raw ? s->d_raw : nullptr;
    p.res = s->d_res;
    p.samples = s->pushed;
    p.products = np;
    p.fs = m.fs;
    p.kappa = m.kappa;
    p.symbols = (double)np * m.q / (m.F + m.P);
    p.threshold = np > 0 ? m.c / sqrt((double)np * m.P / (m.F + m.P)) : INFINITY;   // c / sqrt(M P / q)
    p.threshold_sideband = np > 0 ? m.c1 / sqrt((double)np * m.P / (m.F + m.P)) : INFINITY;
    p.detect = p.symbols >= 32.0;
    cudaStream_t st = nullptr;
    if (follow(s, st)) return NRSC5B_ECUDA;
    if (s->mode == NRSC5B_MODE_AM) k_scan_finish<256, 14, 2><<<s->nch, THREADS, 0, st>>>(p);
    else k_scan_finish<2048, 112, 4><<<s->nch, THREADS, 0, st>>>(p);
    if (cudaGetLastError() != cudaSuccess) return NRSC5B_ECUDA;
    bool ok = cudaMemcpyAsync(out, s->d_res, (size_t)s->nch * sizeof(nrsc5b_scan_t), cudaMemcpyDeviceToHost, st) == cudaSuccess;
    if (raw) ok = ok && cudaMemcpyAsync(raw, s->d_raw, (size_t)s->nch * raw_of(m) * 8, cudaMemcpyDeviceToHost, st) == cudaSuccess;
    return ok && cudaStreamSynchronize(st) == cudaSuccess ? NRSC5B_OK : NRSC5B_ECUDA;
}

// nrsc5b_chan_scan: the channeliser's streaming push into the scanner's own buffer, then the scan of it, piece by piece
// (at most CHAN_OUT outputs per channel at a time), all on the legacy default stream
extern "C" int nrsc5b_chan_scan(nrsc5b_channelizer_t *c, nrsc5b_scanner_t *s, const void *capture, size_t nvalues)
{
    int device, mode, cs16, nch;
    if (!c || !s || (nvalues & 1) || (nvalues && !capture) || nbchan_info(c, &device, &mode, &cs16, &nch) ||
        device != s->device || mode != s->mode || nch != s->nch)
        return NRSC5B_EINVAL;
    const long long total = (long long)(nvalues / 2);
    // the symbol bound first, so that a refused call changes neither handle
    const long long more = nbchan_outputs_after(c, total);
    if ((s->pushed + more) / (s->m->F + s->m->P) > MAX_SYMBOLS) return NRSC5B_EINVAL;
    if (!total) return NRSC5B_OK;
    if (cudaSetDevice(s->device) != cudaSuccess) return NRSC5B_ENODEV;
    if (!s->d_chout && cudaMalloc(&s->d_chout, (size_t)nch * 4 * CHAN_OUT) != cudaSuccess) {
        s->d_chout = nullptr;
        return NRSC5B_ENOMEM;
    }
    const size_t bps = cs16 ? 4 : 2;
    for (long long done = 0; done < total;) {
        // the longest piece whose outputs fit the buffer (outputs grow with the piece, by about one per D samples)
        long long lo = 1, hi = total - done;
        while (lo < hi) {
            const long long mid = lo + (hi - lo + 1) / 2;
            if (nbchan_outputs_after(c, mid) <= CHAN_OUT) lo = mid;
            else hi = mid - 1;
        }
        const void *src = reinterpret_cast<const uint8_t *>(capture) + bps * done;
        long long nout = 0;
        int rc = cs16 ? nrsc5b_chan_push_cs16(c, reinterpret_cast<const int16_t *>(src), 2 * (size_t)lo, s->d_chout, 2 * CHAN_OUT, nullptr, &nout)
                      : nrsc5b_chan_push(c, reinterpret_cast<const uint8_t *>(src), 2 * (size_t)lo, s->d_chout, 2 * CHAN_OUT, nullptr, &nout);
        if (rc) return rc;
        if (nout > 0 && (rc = nrsc5b_scan_push_device(s, s->d_chout, 2 * CHAN_OUT, (size_t)nout, nullptr))) return rc;
        done += lo;
    }
    return NRSC5B_OK;
}
