// Audio in and out of the streaming slot call (fsn_stream_step_audio_slots, DESIGN.md §3.10): per slot and tick, the analysis kernel
// turns one hop of samples into one frame of torch.stft(center=True, reflect, periodic Hann), and the synthesis kernel turns the mask
// the model step produced into one hop of torch.istft output (decompress_cIRM x noisy spectrum, inverse real FFT, window, overlap-add,
// division by the window envelope).  One CTA per slot; the real FFTs of n_fft points run as complex FFTs of n_fft / 2 points
// (radix 2, fp32, in shared memory) with the even / odd split folded in.  The tables (window, twiddles, 1 / envelope) are computed in
// double on the host once per handle.
#include <cmath>

#include "fsn_common.cuh"
#include "fsn_kernels.h"

namespace fsn {

constexpr int AUDIO_THREADS = 128;
constexpr int AUDIO_MAX_HOP = 512;                              // n_fft <= 1024

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ float2 cmul_conj(float2 a, float2 b) { return make_float2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y); }   // a conj(b)

// In-place radix-2 decimation-in-time FFT of H points (input in bit-reversed order, output in natural order).  tw[k] = exp(-2 pi i k / N),
// N = 2 H; INV: exp(+...), unscaled.
template <bool INV>
__device__ __forceinline__ void fft_dit(float2* z, const float2* __restrict__ tw, int H) {
    for (int h = 1; h < H; h <<= 1) {
        const int step = H / h;                                  // W_{2h}^p = W_N^{p N / (2h)} = tw[p * H / h]
        for (int t = threadIdx.x; t < H / 2; t += blockDim.x) {
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

// grid B: analysis of one tick.  STORE: the slot's hop goes to its history ring (hop q at q % 3).  FRAME: frame j = tick - 1 of the
// session, original samples [hop (j - 1), hop (j + 1)) reflected at 0 and, once the session's length is known, at L - 1; its spectrum
// goes to the ring (frame j at j % (la + 1)) and its magnitude to the model's input row.  ZERO: the same two rows are zero (the
// right padding of the look-ahead).  A slot without an op touches nothing.
__global__ void __launch_bounds__(AUDIO_THREADS) stream_stft_kernel(StreamAudioLaunch a) {
    __shared__ float2 z[AUDIO_MAX_HOP];
    const int b = blockIdx.x, op = a.op[b];
    if (!(op & (AUDIO_STORE | AUDIO_FRAME | AUDIO_ZERO))) return;
    const int H = a.n_fft >> 1, F = H + 1, k = a.tick[b], lg = 31 - __clz(H);
    float* hist = a.hist + (size_t)b * 3 * H;
    if (op & AUDIO_STORE) {
        const float* x = a.samples + (size_t)b * H;
        for (int i = threadIdx.x; i < H; i += blockDim.x) hist[(k % 3) * H + i] = x[i];
        __syncthreads();                                         // frame 0 reads the first sample of the hop stored now
    }
    if (!(op & (AUDIO_FRAME | AUDIO_ZERO))) return;
    const int j = k - 1;
    float2* spec = a.spec + ((size_t)b * (a.la + 1) + j % (a.la + 1)) * F;
    float* mag = a.mag + (size_t)b * F;
    if (op & AUDIO_ZERO) {
        for (int f = threadIdx.x; f < F; f += blockDim.x) { spec[f] = make_float2(0.f, 0.f); mag[f] = 0.f; }
        return;
    }
    const int L = a.hops[b] * H;                                 // 0 while the session's length is unknown
    for (int n = threadIdx.x; n < H; n += blockDim.x) {          // z[n] = x[2n] + i x[2n + 1], windowed, stored bit-reversed
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            int p = H * (j - 1) + 2 * n + e;
            if (p < 0) p = -p;
            if (L && p >= L) p = 2 * (L - 1) - p;
            v[e] = hist[((p / H) % 3) * H + p % H] * __ldg(a.window + 2 * n + e);
        }
        z[bitrev(n, lg)] = make_float2(v[0], v[1]);
    }
    __syncthreads();
    fft_dit<false>(z, a.twiddle, H);
    // X[f] = Xe[f] + W_N^f Xo[f], Xe = (Z[f] + conj Z[H - f]) / 2, Xo = (Z[f] - conj Z[H - f]) / 2i  (indices mod H)
    for (int f = threadIdx.x; f < F; f += blockDim.x) {
        const float2 p = z[f & (H - 1)], q = z[(H - f) & (H - 1)];
        const float2 xe = make_float2(0.5f * (p.x + q.x), 0.5f * (p.y - q.y));
        const float2 xo = make_float2(0.5f * (p.y + q.y), -0.5f * (p.x - q.x));
        const float2 t = cmul(__ldg(a.twiddle + f), xo);
        const float2 X = make_float2(xe.x + t.x, xe.y + t.y);
        spec[f] = X;
        mag[f] = hypotf(X.x, X.y);
    }
}

// grid B: synthesis of one tick.  SYNTH: frame m = tick - 1 - la from the mask row the model step wrote this tick and the spectrum
// ring; the second half of the windowed frame becomes the slot's tail.  EMIT (m >= 1): out = (tail of frame m - 1 + first half) / env,
// which is hop m - 1 of the session.  Every row without EMIT is written as zero.
__global__ void __launch_bounds__(AUDIO_THREADS) stream_istft_kernel(StreamAudioLaunch a) {
    __shared__ float2 z[AUDIO_MAX_HOP];
    __shared__ float2 e[AUDIO_MAX_HOP + 1];
    const int b = blockIdx.x, op = a.op[b];
    const int H = a.n_fft >> 1, F = H + 1, lg = 31 - __clz(H);
    float* out = a.out + (size_t)b * H;
    if (!(op & AUDIO_SYNTH)) {
        for (int i = threadIdx.x; i < H; i += blockDim.x) out[i] = 0.f;
        return;
    }
    const int m = a.tick[b] - 1 - a.la;
    const float2* spec = a.spec + ((size_t)b * (a.la + 1) + m % (a.la + 1)) * F;
    const float* mask = a.mask + (size_t)b * 2 * F;
    for (int f = threadIdx.x; f < F; f += blockDim.x) {          // decompress_cIRM x noisy spectrum (inferencer.py:152-157)
        const float m0 = decompress_cirm(mask[f]), m1 = decompress_cirm(mask[F + f]);
        const float2 x = spec[f];
        float2 E = make_float2(m0 * x.x - m1 * x.y, m1 * x.x + m0 * x.y);
        if (f == 0 || f == H) E.y = 0.f;                         // a real inverse transform ignores the DC and Nyquist imaginary parts
        e[f] = E;
    }
    __syncthreads();
    // Z[k] = Xe[k] + i Xo[k], Xe = (E[k] + conj E[H - k]) / 2, Xo = (E[k] - conj E[H - k]) conj(W_N^k) / 2; z = IFFT_H(Z) / H
    // interleaves the inverse real transform: y[2n] = Re z[n], y[2n + 1] = Im z[n]
    for (int k = threadIdx.x; k < H; k += blockDim.x) {
        const float2 p = e[k], q = e[H - k];
        const float2 xe = make_float2(0.5f * (p.x + q.x), 0.5f * (p.y - q.y));
        const float2 xo = cmul_conj(make_float2(0.5f * (p.x - q.x), 0.5f * (p.y + q.y)), __ldg(a.twiddle + k));
        z[bitrev(k, lg)] = make_float2(xe.x - xo.y, xe.y + xo.x);
    }
    __syncthreads();
    fft_dit<true>(z, a.twiddle, H);
    const float* y = reinterpret_cast<const float*>(z);
    const float s = 1.0f / (float)H;
    float* tail = a.tail + (size_t)b * H;
    const bool emit = op & AUDIO_EMIT;
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
        const float lo = y[i] * s * __ldg(a.window + i), hi = y[H + i] * s * __ldg(a.window + H + i);
        if (emit) out[i] = (tail[i] + lo) * __ldg(a.inv_env + i);
        else out[i] = 0.f;
        tail[i] = hi;
    }
}

void launch_stream_stft(const StreamAudioLaunch& a, cudaStream_t s) { stream_stft_kernel<<<a.B, AUDIO_THREADS, 0, s>>>(a); }
void launch_stream_istft(const StreamAudioLaunch& a, cudaStream_t s) { stream_istft_kernel<<<a.B, AUDIO_THREADS, 0, s>>>(a); }

// Tables of one n_fft, computed in double: periodic Hann window [n_fft], twiddles exp(-2 pi i k / n_fft) for k = 0 .. n_fft / 2
// (n_fft / 2 + 1 of them), 1 / (w^2(i) + w^2(i + hop)) for i < hop.
void stream_audio_tables(int n_fft, std::vector<float>& window, std::vector<float>& twiddle, std::vector<float>& inv_env) {
    const int H = n_fft / 2;
    const double PI = 3.14159265358979323846;
    std::vector<double> w(n_fft);
    for (int i = 0; i < n_fft; ++i) w[i] = 0.5 - 0.5 * cos(2.0 * PI * i / n_fft);
    window.assign(w.begin(), w.end());
    twiddle.resize(2 * (H + 1));
    for (int k = 0; k <= H; ++k) {
        twiddle[2 * k] = (float)cos(2.0 * PI * k / n_fft);
        twiddle[2 * k + 1] = (float)-sin(2.0 * PI * k / n_fft);
    }
    inv_env.resize(H);
    for (int i = 0; i < H; ++i) inv_env[i] = (float)(1.0 / (w[i] * w[i] + w[i + H] * w[i + H]));
}

}  // namespace fsn
