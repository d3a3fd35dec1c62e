// Audio in and out of the streaming slot call (fsn_stream_step_audio_slots, DESIGN.md §3.10): per slot and tick, the analysis kernel
// turns one hop of samples into one frame of torch.stft(center=True, reflect, periodic Hann), and the synthesis kernel turns the mask
// the model step produced into one hop of torch.istft output (decompress_cIRM x noisy spectrum, inverse real FFT, window, overlap-add,
// division by the window envelope).  One CTA per slot; the real FFTs of n_fft points run as complex FFTs of n_fft / 2 points
// (radix 2, fp32, in shared memory, fsn_fft.cuh) with the even / odd split folded in.  The tables (window, twiddles, 1 / envelope) are
// computed in double on the host once per handle (audio_tables).
#include "fsn_common.cuh"
#include "fsn_fft.cuh"
#include "fsn_kernels.h"

namespace fsn {

constexpr int AUDIO_THREADS = 128;
constexpr int AUDIO_MAX_HOP = 512;                              // n_fft <= 1024

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
    for (int f = threadIdx.x; f < F; f += blockDim.x) {
        const float2 X = rfft_split(z[f & (H - 1)], z[(H - f) & (H - 1)], __ldg(a.twiddle + f));
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
    for (int k = threadIdx.x; k < H; k += blockDim.x) z[bitrev(k, lg)] = irfft_split(e[k], e[H - k], __ldg(a.twiddle + k));
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

}  // namespace fsn
