// Stand-alone stage kernels (FFT, halfband) behind the C ABI's single-stage entry points; the product
// kernels live in front.cuh / viterbi_chunk.cuh / engine.cu.
#include "common.cuh"
#include "fft.cuh"

namespace nb {

// ---------------------------------------------------------------------------
// stand-alone stage kernels for the numerics / parity tests
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(FFT_THREADS) k_fft_test(const float2 *in, float2 *outp, const float2 *twid)
{
    __shared__ float2 buf[FFT_SMEM_ELEMS];
    const int t = threadIdx.x;
    const float2 *x = in + (size_t)blockIdx.x * NFFT;
    float2 v[16], out[2][8];
#pragma unroll
    for (int n1 = 0; n1 < 16; n1++) v[n1] = x[n1 * 128 + t];
    fft2048_block(v, out, buf, twid, t);
    float2 *y = outp + (size_t)blockIdx.x * NFFT;
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
        for (int k3 = 0; k3 < 8; k3++) y[t + 128 * h + 256 * k3] = out[h][k3];
}

void launch_fft_test(const float2 *in, float2 *out, const float2 *twid, int nffts, cudaStream_t stream)
{
    k_fft_test<<<nffts, FFT_THREADS, 0, stream>>>(in, out, twid);
}

// the cu8 decimator alone, from a zero history: the demodulator's halfband_run (runs of 17 per thread, input words
// staged in shared memory) over npairs outputs, i.e. 4 * npairs input bytes
constexpr int HB_RUN = 17, HB_THREADS = 128, HB_OUT = HB_RUN * HB_THREADS;

__global__ void __launch_bounds__(HB_THREADS) k_halfband_test(const uint8_t *cu8, long long npairs, short2 *out)
{
    __shared__ uint32_t words[HB_OUT + 7];
    __shared__ short2 y[HB_OUT];
    const int t = threadIdx.x;
    const long long d0 = (long long)blockIdx.x * HB_OUT;
    const uint32_t *cw = reinterpret_cast<const uint32_t *>(cu8);
    for (int v = t; v < HB_OUT + 7; v += HB_THREADS) {
        const long long q = d0 - 7 + v;                  // output d reads words d-7 .. d
        words[v] = q >= 0 && q < npairs ? cw[q] : 0x7f7f7f7fu;
    }
    __syncthreads();
    halfband_run<HB_RUN>(words + HB_RUN * t, y + HB_RUN * t);
    __syncthreads();
    for (int v = t; v < HB_OUT && d0 + v < npairs; v += HB_THREADS) out[d0 + v] = y[v];
}

void launch_halfband_test(const uint8_t *cu8, long long npairs, short2 *out, cudaStream_t stream)
{
    const long long bl = (npairs + HB_OUT - 1) / HB_OUT;
    if (bl > 0) k_halfband_test<<<(unsigned)bl, HB_THREADS, 0, stream>>>(cu8, npairs, out);
}

}  // namespace nb
