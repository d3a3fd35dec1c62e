// The device FFT of the audio kernels (k_stream_audio.cu: the streaming slot call; k_audio.cu: the offline audio call).  A real FFT
// of n_fft points runs as a complex FFT of H = n_fft / 2 points (radix 2, fp32, in shared memory) with the even / odd split folded in
// before (inverse) or after (forward) it.  The tables (window, twiddles, envelopes) are computed in double on the host (audio_tables).
#pragma once
#include <cuda_runtime.h>

namespace fsn {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ float2 cmul_conj(float2 a, float2 b) { return make_float2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y); }   // a conj(b)

// In-place radix-2 decimation-in-time FFTs of H points each, nb of them H apart in z (input in bit-reversed order within each
// transform, output in natural order).  tw[k] = exp(-2 pi i k / N), N = 2 H; INV: exp(+...), unscaled.  Butterfly t of a stage lies in
// transform t / (H / 2): H / 2 is a multiple of every half-span h, so the index arithmetic of one transform carries over unchanged.
template <bool INV>
__device__ __forceinline__ void fft_dit(float2* z, const float2* __restrict__ tw, int H, int nb = 1) {
    for (int h = 1; h < H; h <<= 1) {
        const int step = H / h;                                  // W_{2h}^p = W_N^{p N / (2h)} = tw[p * H / h]
        for (int t = threadIdx.x; t < nb * (H / 2); t += blockDim.x) {
            const int p = t & (h - 1), i0 = ((t - p) << 1) + p, i1 = i0 + h;
            const float2 w = __ldg(tw + p * step);
            const float2 u = z[i0], v = INV ? cmul_conj(z[i1], w) : cmul(z[i1], w);
            z[i0] = make_float2(u.x + v.x, u.y + v.y);
            z[i1] = make_float2(u.x - v.x, u.y - v.y);
        }
        __syncthreads();
    }
}

__device__ __forceinline__ int bitrev(int n, int lg) { return (int)(__brev((unsigned)n) >> (32 - lg)); }

// Forward split: bin f (0 <= f <= H) of the real FFT of x from Z = FFT_H(x[2n] + i x[2n + 1]), p = Z[f mod H], q = Z[(H - f) mod H],
// w = tw[f]:  X[f] = Xe[f] + W_N^f Xo[f], Xe = (p + conj q) / 2, Xo = (p - conj q) / 2i
__device__ __forceinline__ float2 rfft_split(float2 p, float2 q, float2 w) {
    const float2 xe = make_float2(0.5f * (p.x + q.x), 0.5f * (p.y - q.y));
    const float2 xo = make_float2(0.5f * (p.y + q.y), -0.5f * (p.x - q.x));
    const float2 t = cmul(w, xo);
    return make_float2(xe.x + t.x, xe.y + t.y);
}

// Inverse split: Z[k] (0 <= k < H) from the half spectrum E, p = E[k], q = E[H - k], w = tw[k]:  Z[k] = Xe[k] + i Xo[k],
// Xe = (p + conj q) / 2, Xo = (p - conj q) conj(W_N^k) / 2.  z = IFFT_H(Z) / H interleaves the inverse real transform:
// y[2n] = Re z[n], y[2n + 1] = Im z[n]
__device__ __forceinline__ float2 irfft_split(float2 p, float2 q, float2 w) {
    const float2 xe = make_float2(0.5f * (p.x + q.x), 0.5f * (p.y - q.y));
    const float2 xo = cmul_conj(make_float2(0.5f * (p.x - q.x), 0.5f * (p.y + q.y)), w);
    return make_float2(xe.x - xo.y, xe.y + xo.x);
}

}  // namespace fsn
