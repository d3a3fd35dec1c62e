// Audio in and out of the offline forward (fsn_model_enhance_audio, DESIGN.md §3.12): per sub-batch, the analysis kernel turns each
// clip's samples into the mag / real / imag planes of torch.stft(center=True, reflect, periodic Hann) that the forward reads, and the
// synthesis kernel turns the enhanced spectrum the forward's epilogue wrote into torch.istft(length = L_b) of each clip.  Every clip is
// reflected at its own end and synthesised over its own T_b = L_b / hop + 1 frames.  The FFTs are those of the streaming audio call
// (fsn_fft.cuh), several frames per CTA.  Also the host tables both audio paths share (audio_tables).
#include <cmath>

#include "fsn_common.cuh"
#include "fsn_fft.cuh"
#include "fsn_kernels.h"

namespace fsn {

constexpr int AUDIO_OFF_THREADS = 256;
constexpr int AUDIO_RUN_POINTS = 2048;                           // frames (analysis) / hops (synthesis) per CTA: 2048 / hop
constexpr int AUDIO_OFF_MAX_HOP = 512;                           // n_fft <= 1024
constexpr int AUDIO_OFF_MIN_HOP = 32;                            // n_fft >= 64
constexpr int AUDIO_MAX_RUN = AUDIO_RUN_POINTS / AUDIO_OFF_MIN_HOP;
// (R + 1) (H + 1) float2 over every hop H = 2048 / R: largest at H = 512 (5 x 513)
constexpr int AUDIO_TILE = (AUDIO_RUN_POINTS / AUDIO_OFF_MAX_HOP + 1) * (AUDIO_OFF_MAX_HOP + 1);
static_assert((AUDIO_MAX_RUN + 1) * (AUDIO_OFF_MIN_HOP + 1) <= AUDIO_TILE, "the tile bound holds at the smallest hop too");

__device__ __forceinline__ int clip_len(const AudioLaunch& a, int b) { return a.len ? a.len[b] : a.Lall; }

// grid (ceil(T / R), B), R = 2048 / hop: frames t0 .. t0 + R - 1 of clip b.  The run's original samples [hop (t0 - 1), hop (t0 + R))
// are staged once, reflected at 0 and at L_b - 1 (torch.stft's center padding), then windowed into R half-size complex FFTs.  The
// spectra go through a [F][R] shared tile so that the planes (t innermost) are stored along t.  Frames at or past T_b are zero.
__global__ void __launch_bounds__(AUDIO_OFF_THREADS) audio_stft_kernel(AudioLaunch a) {
    __shared__ float xs[AUDIO_RUN_POINTS + AUDIO_OFF_MAX_HOP];
    __shared__ float2 z[AUDIO_RUN_POINTS];
    __shared__ float2 X[AUDIO_TILE];
    const int b = blockIdx.y, H = a.n_fft >> 1, F = H + 1, lg = 31 - __clz(H), R = AUDIO_RUN_POINTS / H, ld = R + 1;
    const int t0 = blockIdx.x * R, Lb = clip_len(a, b), Tb = Lb / H + 1;
    const int nv = Tb - t0 < R ? Tb - t0 : R;                    // frames of the run that exist (block-uniform; <= 0: none)
    if (nv > 0) {
        const float* x = a.wave + (size_t)b * a.L;
        for (int j = threadIdx.x; j < (nv + 1) * H; j += blockDim.x) {
            int p = H * (t0 - 1) + j;
            if (p < 0) p = -p;
            if (p >= Lb) p = 2 * (Lb - 1) - p;                  // L_b > hop: every reflected index lies in [0, L_b)
            xs[j] = __ldg(x + p);
        }
        __syncthreads();
        for (int i = threadIdx.x; i < nv * H; i += blockDim.x) {  // frame r: z[n] = x[2n] + i x[2n + 1], windowed, stored bit-reversed
            const int r = i / H, n = i - r * H;
            const float* xr = xs + r * H + 2 * n;
            z[r * H + bitrev(n, lg)] = make_float2(xr[0] * __ldg(a.window + 2 * n), xr[1] * __ldg(a.window + 2 * n + 1));
        }
        __syncthreads();
        fft_dit<false>(z, a.twiddle, H, nv);
        for (int i = threadIdx.x; i < nv * F; i += blockDim.x) {
            const int r = i / F, f = i - r * F;
            const float2* zr = z + r * H;
            X[f * ld + r] = rfft_split(zr[f & (H - 1)], zr[(H - f) & (H - 1)], __ldg(a.twiddle + f));
        }
        __syncthreads();
    }
    const size_t plane = (size_t)a.B * F * a.T;
    for (int i = threadIdx.x; i < F * R; i += blockDim.x) {
        const int f = i / R, r = i - f * R, t = t0 + r;
        if (t >= a.T) continue;
        const float2 v = r < nv ? X[f * ld + r] : make_float2(0.f, 0.f);
        float* o = a.planes + ((size_t)b * F + f) * a.T + t;
        o[0] = hypotf(v.x, v.y);
        o[plane] = v.x;
        o[2 * plane] = v.y;
    }
}

// grid (ceil(ceil(L / hop) / R), B), R = 2048 / hop: output hops q0 .. q0 + R - 1 of clip b from frames q0 .. q0 + R (those < T_b).
// Sample n = q hop + i is w(i + hop) y_q(i + hop) + w(i) y_{q+1}(i) over w^2(i + hop) + w^2(i); past frame T_b - 2's window (the last
// L_b mod hop samples) frame q + 1 does not exist and the envelope is w^2(i + hop) alone, as in torch.istft.  Each sample is written
// once; samples in [L_b, L) are zero.
__global__ void __launch_bounds__(AUDIO_OFF_THREADS) audio_istft_kernel(AudioLaunch a) {
    __shared__ float2 E[AUDIO_TILE];
    __shared__ float2 z[AUDIO_RUN_POINTS + AUDIO_OFF_MAX_HOP];
    const int b = blockIdx.y, H = a.n_fft >> 1, F = H + 1, lg = 31 - __clz(H), R = AUDIO_RUN_POINTS / H;
    const int q0 = blockIdx.x * R, Lb = clip_len(a, b), Tb = Lb / H + 1;
    const int nf = Tb - q0 < R + 1 ? Tb - q0 : R + 1;            // frames to synthesise (block-uniform; <= 0: none)
    if (nf > 0) {
        const float2* e = a.enh + (size_t)b * F * a.T + q0;
        for (int i = threadIdx.x; i < nf * F; i += blockDim.x) {  // along t: nf consecutive frames of each bin
            const int f = i / nf, r = i - f * nf;
            float2 v = e[(size_t)f * a.T + r];
            if (f == 0 || f == H) v.y = 0.f;                     // a real inverse transform ignores the DC and Nyquist imaginary parts
            E[r * F + f] = v;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < nf * H; i += blockDim.x) {
            const int r = i / H, k = i - r * H;
            z[r * H + bitrev(k, lg)] = irfft_split(E[r * F + k], E[r * F + H - k], __ldg(a.twiddle + k));
        }
        __syncthreads();
        fft_dit<true>(z, a.twiddle, H, nf);
    }
    const float* y = reinterpret_cast<const float*>(z);          // frame r: y[r n_fft .. (r + 1) n_fft)
    const float s = 1.0f / (float)H;
    float* out = a.out + (size_t)b * a.L;
    for (int i = threadIdx.x; i < R * H; i += blockDim.x) {
        const long long n = (long long)q0 * H + i;
        if (n >= a.L) break;
        float v = 0.f;
        if (n < Lb) {
            const int r = i / H, k = i - r * H;
            const float hi = y[r * a.n_fft + H + k] * s * __ldg(a.window + H + k);
            if (q0 + r + 1 < Tb) v = (hi + y[(r + 1) * a.n_fft + k] * s * __ldg(a.window + k)) * __ldg(a.inv_env + k);
            else v = hi * __ldg(a.inv_last + k);
        }
        out[n] = v;
    }
}

static int run_tiles(long long n, int R) { return (int)((n + R - 1) / R); }

cudaError_t launch_audio_stft(const AudioLaunch& a, cudaStream_t s) {
    const int R = AUDIO_RUN_POINTS / (a.n_fft / 2);
    audio_stft_kernel<<<dim3(run_tiles(a.T, R), a.B), AUDIO_OFF_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}
cudaError_t launch_audio_istft(const AudioLaunch& a, cudaStream_t s) {
    const int H = a.n_fft / 2, R = AUDIO_RUN_POINTS / H;
    audio_istft_kernel<<<dim3(run_tiles((a.L + H - 1) / H, R), a.B), AUDIO_OFF_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}

void audio_tables(int n_fft, std::vector<float>& tab) {
    const int H = n_fft / 2;
    const double PI = 3.14159265358979323846;
    std::vector<double> w(n_fft);
    for (int i = 0; i < n_fft; ++i) w[i] = 0.5 - 0.5 * cos(2.0 * PI * i / n_fft);
    tab.assign(w.begin(), w.end());
    for (int k = 0; k <= H; ++k) {
        tab.push_back((float)cos(2.0 * PI * k / n_fft));
        tab.push_back((float)-sin(2.0 * PI * k / n_fft));
    }
    for (int i = 0; i < H; ++i) tab.push_back((float)(1.0 / (w[i] * w[i] + w[i + H] * w[i + H])));
    for (int i = 0; i < H; ++i) tab.push_back((float)(1.0 / (w[i + H] * w[i + H])));
}

}  // namespace fsn
