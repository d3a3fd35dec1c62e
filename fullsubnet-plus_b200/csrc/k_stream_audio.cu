// Audio in and out of the streaming slot calls (DESIGN.md §3.10, §3.14): per slot and tick, the analysis turns one hop of samples into
// one frame of torch.stft(center=True, reflect, periodic Hann), and the synthesis turns the mask the model step produced into one hop
// of torch.istft output (decompress_cIRM x noisy spectrum, inverse real FFT, window, overlap-add, division by the window envelope).
// One CTA per slot; the real FFTs of n_fft points run as complex FFTs of n_fft / 2 points (radix 2, fp32, in shared memory,
// fsn_fft.cuh) with the even / odd split folded in.  The tables (window, twiddles, 1 / envelope) are computed in double on the host
// once per handle (audio_tables).  Every audio call runs this one pair: each slot's ticks of the call run in order inside its CTA, one
// for the per-hop call (fsn_stream_step_audio_slots), up to K for the chunk call (fsn_stream_step_audio_chunk) and the sample call
// (fsn_stream_step_audio_samples).  The sample call adds sample-granular rows, partial hops and the exact end; the hop calls pass none.
#include "fsn_common.cuh"
#include "fsn_fft.cuh"
#include "fsn_kernels.h"

namespace fsn {

constexpr int AUDIO_THREADS = 128;
constexpr int AUDIO_MAX_HOP = 512;                              // n_fft <= 1024

// Frame j of a session from its history ring hist [3, H] (hop q at q % 3): original samples [H (j - 1), H (j + 1)) reflected at 0 and,
// with L > 0 (the session's length), at L - 1.  Spectrum to spec[f], magnitude to mag[f ms].  z: shared scratch of H points.
__device__ __forceinline__ void analyse_frame(const float* hist, int j, int L, int H, int lg, const float* __restrict__ window,
                                              const float2* __restrict__ twiddle, float2* z, float2* spec, float* mag, int ms) {
    for (int n = threadIdx.x; n < H; n += blockDim.x) {          // z[n] = x[2n] + i x[2n + 1], windowed, stored bit-reversed
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            int p = H * (j - 1) + 2 * n + e;
            if (p < 0) p = -p;
            if (L && p >= L) p = 2 * (L - 1) - p;
            v[e] = hist[((p / H) % 3) * H + p % H] * __ldg(window + 2 * n + e);
        }
        z[bitrev(n, lg)] = make_float2(v[0], v[1]);
    }
    __syncthreads();
    fft_dit<false>(z, twiddle, H);
    for (int f = threadIdx.x; f <= H; f += blockDim.x) {
        const float2 X = rfft_split(z[f & (H - 1)], z[(H - f) & (H - 1)], __ldg(twiddle + f));
        spec[f] = X;
        mag[f * ms] = hypotf(X.x, X.y);
    }
}

// Synthesis of one frame from its mask rows mask[f ms], mask[(F + f) ms] and noisy spectrum spec: the second half of the windowed
// inverse transform becomes the tail; with emit, out[i] = (tail + first half) / env (the session's next hop), else out[i] = 0.
// z, e: shared scratch of H and H + 1 points.  LIM: the mask gets the slot's attenuation floor lam (limit_mask, DESIGN.md §3.18).
template <bool LIM>
__device__ __forceinline__ void synth_frame(const float* mask, int ms, const float2* spec, float* tail, float* out, bool emit, int H,
                                            int lg, const float* __restrict__ window, const float2* __restrict__ twiddle,
                                            const float* __restrict__ inv_env, float2* z, float2* e, float lam) {
    const int F = H + 1;
    for (int f = threadIdx.x; f < F; f += blockDim.x) {          // decompress_cIRM x noisy spectrum (inferencer.py:152-157)
        float m0 = decompress_cirm(mask[f * ms]), m1 = decompress_cirm(mask[(F + f) * ms]);
        if (LIM) limit_mask(m0, m1, lam);
        const float2 x = spec[f];
        float2 E = make_float2(m0 * x.x - m1 * x.y, m1 * x.x + m0 * x.y);
        if (f == 0 || f == H) E.y = 0.f;                         // a real inverse transform ignores the DC and Nyquist imaginary parts
        e[f] = E;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < H; k += blockDim.x) z[bitrev(k, lg)] = irfft_split(e[k], e[H - k], __ldg(twiddle + k));
    __syncthreads();
    fft_dit<true>(z, twiddle, H);
    const float* y = reinterpret_cast<const float*>(z);
    const float s = 1.0f / (float)H;
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
        const float lo = y[i] * s * __ldg(window + i), hi = y[H + i] * s * __ldg(window + H + i);
        if (emit) out[i] = (tail[i] + lo) * __ldg(inv_env + i);
        else out[i] = 0.f;
        tail[i] = hi;
    }
}

// The model planes' address of slot b's column c (row 0 of its rows rows): [B, rows, Km]
__device__ __forceinline__ size_t chunk_col(const StreamAudioLaunch& a, int b, int c, int rows) {
    return ((size_t)b * rows) * a.Km + c;
}

// Hop-chunk i of a slot's call into the history ring (hop k at k % 3): session samples P = i hop + t (t < n) counted from the start
// of the slot's first pending hop; those at P >= r0 come from the call's row, x[P - r0] (the r0 below are already in the ring)
__device__ __forceinline__ void store_samples(float* hist, int k, const float* x, int i, int n, int r0, int H) {
    for (int t = threadIdx.x; t < n; t += blockDim.x) {
        const int P = i * H + t;
        if (P >= r0) hist[(k % 3) * H + t] = x[P - r0];
    }
}

// grid B: the analysis of a slot's active ticks, in order, from its row of S samples, whose first hop completes the r0 pending ones.
// Stored hops go to the history ring (hop q at q % 3); the spectrum of model column c goes to the scratch sspec (the ring still holds
// the frames the synthesis of this call reads), its magnitude to the model's input.  The trailing r samples (the next pending hop, or
// at a FLUSH the partial end) go to ring slot (k0 + nstore) % 3 at iteration nstore: after the analysis of frame k0 + nstore - 2, the
// last reader of the hop that slot held, and before that of frame k0 + nstore, the first reader of the new one.  A session that has
// ended is reflected at L = K hop + r, and its frames past the end (j > K) are zero.  With zero_out the output rows are zeroed (no
// synthesis runs in the call).
__global__ void __launch_bounds__(AUDIO_THREADS) stream_stft_kernel(StreamAudioLaunch a) {
    __shared__ float2 z[AUDIO_MAX_HOP];
    const int b = blockIdx.x, na = a.na[b];
    const int H = a.n_fft >> 1, F = H + 1, lg = 31 - __clz(H), k0 = a.k0[b], st = a.start[b], ns = a.nstore[b], K = a.hops[b];
    const int r0 = a.r0 ? a.r0[b] : 0, r = a.r ? a.r[b] : 0;
    float* hist = a.hist + (size_t)b * 3 * H;
    const float* x = a.samples + (size_t)b * a.S;
    for (int i = 0; i < na; ++i) {
        const int k = k0 + i;
        __syncthreads();                                         // the last tick's reads of hist and z are done
        if (i <= ns) {
            store_samples(hist, k, x, i, i < ns ? H : r, r0, H);
            __syncthreads();
        }
        if (i < st) continue;                                    // a START stores hop 0 and analyses no frame
        const int c = i - st, j = k - 1;
        float2* spec = a.sspec + ((size_t)b * a.K + c) * F;
        float* mag = a.mag + chunk_col(a, b, c, F);
        const int ms = a.Km;
        if (K && j > K) {
            for (int f = threadIdx.x; f < F; f += blockDim.x) { spec[f] = make_float2(0.f, 0.f); mag[f * ms] = 0.f; }
        } else {
            analyse_frame(hist, j, K ? K * H + r : 0, H, lg, a.window, a.twiddle, z, spec, mag, ms);
        }
    }
    if (na <= ns) {                                              // no tick reads the trailing hop's ring slot in this call
        __syncthreads();
        store_samples(hist, k0 + ns, x, ns, r, r0, H);
    }
    if (a.zero_out) {
        float* out = a.out + (size_t)b * a.So;
        for (int t = threadIdx.x; t < a.So; t += blockDim.x) out[t] = 0.f;
    }
}

// grid B: the synthesis of a slot's model columns, in order, into its output row of So samples.  Column c synthesises frame
// m = j - la (if m >= 0) from its mask and the spectrum of frame m: from the scratch if this call analysed it, else from the ring.
// Emitted hops fill the front of the output row.  A session that ends at L = K hop + r with r > 0 emits, after frame K, its last r
// samples: frame K's tail times 1 / w^2(i + hop), as the offline synthesis does.  The rest of the row is zero.  Then the caller's
// masks by tick (zero on the START tick and past the active ticks) and the ring's last la + 1 frames, written only after every read
// of the ring.  LIM: with the slots' attenuation floors a.lam (the instantiation without them is the synthesis as it was before
// limits existed).
template <bool LIM>
__global__ void __launch_bounds__(AUDIO_THREADS) stream_istft_kernel(StreamAudioLaunch a) {
    __shared__ float2 z[AUDIO_MAX_HOP];
    __shared__ float2 e[AUDIO_MAX_HOP + 1];
    const int b = blockIdx.x, na = a.na[b], st = a.start[b], K = a.K, R = a.la + 1;
    const int H = a.n_fft >> 1, F = H + 1, lg = 31 - __clz(H);
    const int kf = na > st ? na - st : 0, j0 = a.k0[b] + st - 1;  // model columns, the frame of column 0
    const int Kend = a.hops[b], rend = Kend && a.r ? a.r[b] : 0;
    float* out = a.out + (size_t)b * a.So;
    float* tail = a.tail + (size_t)b * H;
    float2* ring = a.spec + (size_t)b * R * F;
    const float2* sspec = a.sspec + (size_t)b * K * F;
    const float lam = LIM ? __ldg(a.lam + b) : 0.f;
    int nout = 0, nlast = 0;                                     // hops emitted, then the r samples of the end
    for (int c = 0; c < kf; ++c) {
        const int m = j0 + c - a.la;
        if (m < 0) continue;
        __syncthreads();                                         // the last frame's reads of z and e are done
        const float2* spec = m >= j0 ? sspec + (size_t)(m - j0) * F : ring + (m % R) * F;
        synth_frame<LIM>(a.mask + chunk_col(a, b, c, 2 * F), a.Km, spec, tail, out + (size_t)nout * H, m >= 1, H, lg, a.window,
                         a.twiddle, a.inv_env, z, e, lam);
        nout += m >= 1;
        if (m == Kend && rend) {                                 // each thread reads the tail entries it has just written
            for (int i = threadIdx.x; i < rend; i += blockDim.x) out[(size_t)nout * H + i] = tail[i] * __ldg(a.inv_last + i);
            nlast = rend;
        }
    }
    const int n = nout * H + nlast;
    for (int t = n + threadIdx.x; t < a.So; t += blockDim.x) out[t] = 0.f;
    if (a.umask) {
        float* um = a.umask + (size_t)b * 2 * F * K;
        for (size_t t = threadIdx.x; t < (size_t)2 * F * K; t += blockDim.x) {
            const int r = (int)(t / K), i = (int)(t % K), c = i - st;
            um[t] = (i >= st && i < na) ? a.mask[chunk_col(a, b, c, 2 * F) + (size_t)r * a.Km] : 0.f;
        }
    }
    __syncthreads();                                             // every read of the ring is done
    for (int t = threadIdx.x; t < R * F; t += blockDim.x) {
        const int c = kf - R + t / F, f = t % F;
        if (c >= 0) ring[((j0 + c) % R) * F + f] = sspec[(size_t)c * F + f];
    }
}

void launch_stream_stft(const StreamAudioLaunch& a, cudaStream_t s) { stream_stft_kernel<<<a.B, AUDIO_THREADS, 0, s>>>(a); }
void launch_stream_istft(const StreamAudioLaunch& a, cudaStream_t s) {
    if (a.lam) stream_istft_kernel<true><<<a.B, AUDIO_THREADS, 0, s>>>(a);
    else stream_istft_kernel<false><<<a.B, AUDIO_THREADS, 0, s>>>(a);
}

}  // namespace fsn
