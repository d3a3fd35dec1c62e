// Objective scores of enhanced speech against its clean reference (fsn_metric_si_sdr, fsn_metric_stoi, DESIGN.md §3.20;
// fsn_metric_sdr, §3.21), one score per clip of a ragged [B, L] batch.  Every reduction that feeds a decision or a score is fp64,
// over a fixed per-clip tiling and in a fixed order, with no atomics: a clip's score depends on its own samples only, bit for bit,
// whatever else is in the batch.
//
// SI-SDR: two passes over the samples (the noise energy |e - a r|^2 is summed directly: the closed form |e|^2 - 2 a <r, e> + a^2 |r|^2
// cancels catastrophically at high SI-SDR), each a per-chunk partial kernel and a per-clip finalize kernel.
//
// STOI (classic, as pystoi 0.3.3): resampling to 10 kHz (an Octave-compatible Kaiser sinc, scipy's resample_poly alignment) is
// recomputed wherever a 10 kHz sample is needed, never stored.  Four kernels: frame energies of x; a per-clip max and keep-mask
// compaction; the band envelopes of the compacted x and y, gathered straight from the kept frames' original positions; the
// per-segment correlations with per-CTA partials; and the per-clip mean.
//
// SDR (BSS Eval v3 for one source, mir_eval's 512-tap distortion filter), fp64 throughout: the 512-lag auto- and cross-correlations
// as per-tile partials and their per-clip sum; a Levinson solve of the 512 x 512 Toeplitz system per clip; the projection P = c * r
// computed explicitly with per-tile sums of P^2 and (e' - P)^2 (the closed form |e|^2 - c.D cancels at high SDR); the per-clip score.
#include <cmath>
#include <vector>

#include "fsn_common.cuh"
#include "fsn_fft.cuh"
#include "fsn_kernels.h"

namespace fsn {

constexpr int MET_THREADS = 256;
constexpr int SISDR_CHUNK = 16384;           // samples per partial: 64 per thread
constexpr int STOI_FS = 10000, STOI_FRAME = 256, STOI_HOP = 128, STOI_BANDS = 15, STOI_SEG = 30;
constexpr int STOI_ENERGY_FRAMES = 16;       // frames per CTA of the energy kernel
constexpr int STOI_ENV_FRAMES = 8;           // envelope frames per CTA (x and y: 16 half-size FFTs)
constexpr int STOI_SEGS = 16;                // segments per CTA of the correlation kernel (x 16 band lanes)
constexpr int STOI_SCAN_THREADS = 1024;
constexpr double STOI_EPS = 2.220446049250313e-16;   // float64 machine epsilon
constexpr double STOI_SHORT = 1e-5;                  // fewer than 30 envelope frames
constexpr int SDR_F = 512;                   // distortion filter taps = correlation lags
constexpr int SDR_KB = 16;                   // lags per register block of the correlation kernel (x 2: R and D)
constexpr int SDR_RUN = 112;                 // samples per lane of the correlation kernel
constexpr int SDR_CORR_TILE = 32 * SDR_RUN;  // 3584 samples per correlation CTA
constexpr int SDR_PROJ_TILE = 4096;          // outputs per projection CTA: 16 per thread

__constant__ int c_band_lo[STOI_BANDS] = {7, 9, 11, 14, 17, 22, 27, 34, 43, 55, 69, 87, 109, 138, 174};
__constant__ int c_band_hi[STOI_BANDS] = {9, 11, 14, 17, 22, 27, 34, 43, 55, 69, 87, 109, 138, 174, 219};

// Sum of v over the CTA in a fixed order (butterfly within each warp, then warp 0 over the warps in index order); every thread gets it.
__device__ double block_sum(double v, double* sh) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[w] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < nw; ++i) s += sh[i];
        sh[32] = s;
    }
    __syncthreads();
    return sh[32];
}

// ---- SI-SDR ---------------------------------------------------------------------------------------------------------------------

// grid (nchunk, B): chunk blockIdx.x of clip b.  PASS 0: (<r, e>, <r, r>); PASS 1: (|a r|^2, |e - a r|^2) with a = alpha[b].
template <int PASS>
__global__ void __launch_bounds__(MET_THREADS) si_sdr_partial_kernel(SiSdrLaunch a) {
    __shared__ double sh[33];
    const int b = blockIdx.y;
    const long long Lb = a.len[b], i0 = (long long)blockIdx.x * SISDR_CHUNK;
    if (i0 >= Lb) return;                                         // block-uniform
    const long long i1 = Lb - i0 < SISDR_CHUNK ? Lb : i0 + SISDR_CHUNK;
    const float* r = a.ref + (size_t)b * a.L;
    const float* e = a.est + (size_t)b * a.L;
    const double al = PASS ? a.alpha[b] : 0.0;
    double s0 = 0.0, s1 = 0.0;
    for (long long i = i0 + threadIdx.x; i < i1; i += MET_THREADS) {
        const double rv = __ldg(r + i), ev = __ldg(e + i);
        if (PASS == 0) { s0 += rv * ev; s1 += rv * rv; }
        else { const double p = al * rv, n = ev - p; s0 += p * p; s1 += n * n; }
    }
    s0 = block_sum(s0, sh);
    s1 = block_sum(s1, sh);
    if (threadIdx.x == 0) a.part[(size_t)b * a.nchunk + blockIdx.x] = make_double2(s0, s1);
}

// grid B: clip b's partials in chunk order.  PASS 0: alpha[b]; PASS 1: the score.
template <int PASS>
__global__ void __launch_bounds__(MET_THREADS) si_sdr_final_kernel(SiSdrLaunch a) {
    __shared__ double sh[33];
    const int b = blockIdx.x;
    const int n = (int)((a.len[b] + SISDR_CHUNK - 1) / SISDR_CHUNK);
    const double2* p = a.part + (size_t)b * a.nchunk;
    double s0 = 0.0, s1 = 0.0;
    for (int i = threadIdx.x; i < n; i += MET_THREADS) { s0 += p[i].x; s1 += p[i].y; }
    s0 = block_sum(s0, sh);
    s1 = block_sum(s1, sh);
    if (threadIdx.x == 0) {
        if (PASS == 0) a.alpha[b] = s0 / s1;
        else a.out[b] = 10.0 * log10(s0 / s1);
    }
}

cudaError_t launch_si_sdr(const SiSdrLaunch& a, cudaStream_t s) {
    const dim3 grid(a.nchunk, a.B);
    si_sdr_partial_kernel<0><<<grid, MET_THREADS, 0, s>>>(a);
    si_sdr_final_kernel<0><<<a.B, MET_THREADS, 0, s>>>(a);
    si_sdr_partial_kernel<1><<<grid, MET_THREADS, 0, s>>>(a);
    si_sdr_final_kernel<1><<<a.B, MET_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}

// ---- STOI -----------------------------------------------------------------------------------------------------------------------

__device__ __forceinline__ long long stoi_n10k(const StoiLaunch& a, long long Lb) {   // resampled length: ceil(L_b up / down)
    return (Lb * a.up + a.down - 1) / a.down;
}
__device__ __forceinline__ long long stoi_frames(long long n) {                       // range(0, n - 256, 128)
    return n > STOI_FRAME ? (n - STOI_FRAME + STOI_HOP - 1) / STOI_HOP : 0;
}

// 10 kHz sample m of the clip x (L_b samples): y[m] = sum_j x[j] up h[half + m down - j up], taken from the polyphase table as
// sum_k x[jhi - k] poly[ph][k] with jhi = floor((half + m down) / up), ph its remainder; x is zero outside [0, L_b).  fp32.
__device__ float resample_at(const StoiLaunch& a, const float* __restrict__ x, long long Lb, long long m) {
    if (a.up == a.down) return __ldg(x + m);
    const long long c = a.half + m * a.down, jhi = c / a.up;
    const float* hp = a.poly + (size_t)(c - jhi * a.up) * a.ntap;
    const long long k0 = jhi >= Lb ? jhi - Lb + 1 : 0;
    const long long k1 = jhi + 1 < a.ntap ? jhi + 1 : a.ntap;
    float s = 0.f;
    for (long long k = k0; k < k1; ++k) s = fmaf(__ldg(x + jhi - k), __ldg(hp + k), s);
    return s;
}

// grid (ceil(F / 16), B): frames f0 .. f0 + 15 of clip b's x.  The 10 kHz samples [128 f0, 128 (f0 + nf + 1)) are computed once into
// shared memory; warp w sums frames w and w + 8 (each |w(u) x(128 f + u)|^2 over u, fp64) and stores 20 log10(|frame| + EPS).
__global__ void __launch_bounds__(MET_THREADS) stoi_energy_kernel(StoiLaunch a) {
    __shared__ float xs[(STOI_ENERGY_FRAMES + 1) * STOI_HOP];
    const int b = blockIdx.y;
    const long long Lb = a.len[b], Fb = stoi_frames(stoi_n10k(a, Lb)), f0 = (long long)blockIdx.x * STOI_ENERGY_FRAMES;
    if (f0 >= Fb) return;
    const int nf = Fb - f0 < STOI_ENERGY_FRAMES ? (int)(Fb - f0) : STOI_ENERGY_FRAMES;
    const float* x = a.x + (size_t)b * a.L;
    for (int i = threadIdx.x; i < (nf + 1) * STOI_HOP; i += MET_THREADS) xs[i] = resample_at(a, x, Lb, f0 * STOI_HOP + i);
    __syncthreads();
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int r = w; r < nf; r += MET_THREADS / 32) {
        double s = 0.0;
        for (int u = lane; u < STOI_FRAME; u += 32) {
            const double v = __ldg(a.win + u) * xs[r * STOI_HOP + u];
            s += v * v;
        }
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) a.energy[(size_t)b * a.F + f0 + r] = 20.0 * log10(sqrt(s) + STOI_EPS);
    }
}

// grid B, 1024 threads: clip b's max energy, then the kept frames (max - 40 - energy < 0) in frame order into kept[b][0 .. K_b).
__global__ void __launch_bounds__(STOI_SCAN_THREADS) stoi_keep_kernel(StoiLaunch a) {
    __shared__ double smax[STOI_SCAN_THREADS / 32];
    __shared__ int wcount[STOI_SCAN_THREADS / 32];
    const int b = blockIdx.x, w = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = STOI_SCAN_THREADS / 32;
    const long long Fb = stoi_frames(stoi_n10k(a, a.len[b]));
    const double* e = a.energy + (size_t)b * a.F;
    double mx = -INFINITY;
    for (long long i = threadIdx.x; i < Fb; i += STOI_SCAN_THREADS) mx = fmax(mx, e[i]);
    for (int o = 16; o; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) smax[w] = mx;
    __syncthreads();
    mx = smax[0];
    for (int i = 1; i < nw; ++i) mx = fmax(mx, smax[i]);
    int* kept = a.kept + (size_t)b * a.F;
    long long base = 0;
    for (long long i0 = 0; i0 < Fb; i0 += STOI_SCAN_THREADS) {
        const long long i = i0 + threadIdx.x;
        const bool keep = i < Fb && (mx - 40.0 - e[i]) < 0.0;
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        __syncthreads();                                          // the previous round's wcount has been read
        if (lane == 0) wcount[w] = __popc(bal);
        __syncthreads();
        long long off = base;
        int tot = 0;
        for (int k = 0; k < nw; ++k) { if (k < w) off += wcount[k]; tot += wcount[k]; }
        if (keep) kept[off + __popc(bal & ((1u << lane) - 1u))] = (int)i;
        base += tot;
    }
    if (threadIdx.x == 0) a.nkept[b] = (int)base;
}

// grid (ceil((F - 1) / 8), B): envelope frames j0 .. j0 + 7 of clip b.  The compacted signal's 128-sample block m is the second
// half of kept frame m - 1 plus the first half of kept frame m, so STFT frame j (blocks j, j + 1) is gathered from the original 10 kHz
// positions.  The frames are windowed, zero-padded to 512 points and transformed as 256-point complex FFTs (fsn_fft.cuh); thread
// (t, band) sums its band's |X|^2 in fp64 and stores the square root.
__global__ void __launch_bounds__(MET_THREADS) stoi_envelope_kernel(StoiLaunch a) {
    constexpr int H = STOI_FRAME, NB = STOI_ENV_FRAMES + 1;
    __shared__ float cs[2][NB * STOI_HOP];
    __shared__ float2 z[2 * STOI_ENV_FRAMES * H];
    const int b = blockIdx.y;
    const long long Lb = a.len[b];
    const int J = a.nkept[b] - 1, j0 = blockIdx.x * STOI_ENV_FRAMES;
    if (j0 >= J) return;
    const int ne = J - j0 < STOI_ENV_FRAMES ? J - j0 : STOI_ENV_FRAMES;
    const int* kept = a.kept + (size_t)b * a.F;
    for (int i = threadIdx.x; i < 2 * (ne + 1) * STOI_HOP; i += MET_THREADS) {
        const int sig = i / ((ne + 1) * STOI_HOP), r = i - sig * (ne + 1) * STOI_HOP, m = j0 + r / STOI_HOP, t = r % STOI_HOP;
        const float* x = (sig ? a.y : a.x) + (size_t)b * a.L;
        float v = 0.f;
        if (m >= 1) v = __ldg(a.win + STOI_HOP + t) * resample_at(a, x, Lb, (long long)kept[m - 1] * STOI_HOP + STOI_HOP + t);
        v += __ldg(a.win + t) * resample_at(a, x, Lb, (long long)kept[m] * STOI_HOP + t);     // m <= J = K - 1
        cs[sig][r] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * ne * H; i += MET_THREADS) {   // transform q = sig ne + e: z[n] = f[2n] + i f[2n + 1], bit-reversed
        const int q = i / H, n = i - q * H, sig = q / ne, e = q - sig * ne;
        float2 v = make_float2(0.f, 0.f);
        if (n < STOI_HOP) {
            const float* f = cs[sig] + e * STOI_HOP + 2 * n;
            v = make_float2(__ldg(a.win + 2 * n) * f[0], __ldg(a.win + 2 * n + 1) * f[1]);
        }
        z[q * H + bitrev(n, 8)] = v;
    }
    __syncthreads();
    fft_dit<false>(z, a.tw, H, 2 * ne);
    const int q = threadIdx.x / 16, band = threadIdx.x % 16;
    if (q < 2 * ne && band < STOI_BANDS) {
        const float2* zq = z + q * H;
        double s = 0.0;
        for (int f = c_band_lo[band]; f < c_band_hi[band]; ++f) {
            const float2 X = rfft_split(zq[f], zq[H - f], __ldg(a.tw + f));
            s += (double)X.x * X.x + (double)X.y * X.y;
        }
        const int sig = q / ne, e = q - sig * ne;
        a.env[(((size_t)sig * a.B + b) * a.F + j0 + e) * 16 + band] = sqrt(s);
    }
}

// grid (ceil((F - 30) / 16), B): thread (segment s0 + t / 16, band t % 16) computes its segment's correlation (pystoi: scale y to x's
// norm, clip at x (1 + 10^(15/20)), remove the means, normalise, correlate); the CTA's sum, in thread order, is partial blockIdx.x.
__global__ void __launch_bounds__(MET_THREADS) stoi_segment_kernel(StoiLaunch a) {
    __shared__ double sh[33];
    const int b = blockIdx.y, S = a.nkept[b] - 1 - (STOI_SEG - 1), s0 = blockIdx.x * STOI_SEGS;
    if (s0 >= S) return;
    const int s = s0 + threadIdx.x / 16, band = threadIdx.x % 16;
    double corr = 0.0;
    if (s < S && band < STOI_BANDS) {
        const double* X = a.env + ((size_t)b * a.F + s) * 16 + band;
        const double* Y = X + (size_t)a.B * a.F * 16;
        double sxx = 0.0, syy = 0.0;
        for (int k = 0; k < STOI_SEG; ++k) { sxx += X[16 * k] * X[16 * k]; syy += Y[16 * k] * Y[16 * k]; }
        const double nc = sqrt(sxx) / (sqrt(syy) + STOI_EPS), clip = 1.0 + 5.623413251903491;   // 10^(15 / 20)
        double my = 0.0, mx = 0.0;
        for (int k = 0; k < STOI_SEG; ++k) { my += fmin(Y[16 * k] * nc, X[16 * k] * clip); mx += X[16 * k]; }
        my /= STOI_SEG;
        mx /= STOI_SEG;
        double syp = 0.0, sxc = 0.0, sxy = 0.0;
        for (int k = 0; k < STOI_SEG; ++k) {
            const double u = fmin(Y[16 * k] * nc, X[16 * k] * clip) - my, v = X[16 * k] - mx;
            syp += u * u; sxc += v * v; sxy += u * v;
        }
        corr = sxy / ((sqrt(syp) + STOI_EPS) * (sqrt(sxc) + STOI_EPS));
    }
    corr = block_sum(corr, sh);
    if (threadIdx.x == 0) a.part[(size_t)b * a.P + blockIdx.x] = corr;
}

// grid B: the mean correlation over clip b's segments and bands, or 1e-5 below 30 envelope frames.
__global__ void __launch_bounds__(MET_THREADS) stoi_final_kernel(StoiLaunch a) {
    __shared__ double sh[33];
    const int b = blockIdx.x, S = a.nkept[b] - 1 - (STOI_SEG - 1);
    if (S < 1) { if (threadIdx.x == 0) a.out[b] = STOI_SHORT; return; }
    const int n = (S + STOI_SEGS - 1) / STOI_SEGS;
    double v = 0.0;
    for (int i = threadIdx.x; i < n; i += MET_THREADS) v += a.part[(size_t)b * a.P + i];
    v = block_sum(v, sh);
    if (threadIdx.x == 0) a.out[b] = v / ((double)S * STOI_BANDS);
}

static double bessel_i0(double x) {
    double s = 1.0, t = 1.0;
    for (int k = 1; k < 500 && t > 1e-18 * s; ++k) { t *= (x / (2 * k)) * (x / (2 * k)); s += t; }
    return s;
}

static long long gcd_ll(long long p, long long q) { while (q) { const long long r = p % q; p = q; q = r; } return p; }

void stoi_geometry(int sr, StoiLaunch& a) {
    const long long g = gcd_ll(STOI_FS, sr);
    a.up = (int)(STOI_FS / g);
    a.down = (int)(sr / g);
    if (a.up == a.down) { a.half = 0; a.ntap = 0; return; }
    const double cutoff = 1.0 / (2 * (a.up > a.down ? a.up : a.down)), roll_off = cutoff / 10;
    a.half = (int)std::ceil((60.0 - 8) / (28.714 * roll_off));
    a.ntap = (2 * a.half + 1 + a.up - 1) / a.up;
}

size_t stoi_table_floats(const StoiLaunch& a) { return (size_t)a.up * a.ntap + 3 * STOI_FRAME; }

// [twiddles: 256 float2][window: 256][poly: up x ntap], as floats (the twiddles first: float2 loads need 8-byte alignment).  h: pystoi's resample_oct filter (Kaiser beta = 0.1102 (60 - 8.7),
// sinc cut off at 1 / (2 max(up, down))), normalised to unit sum, times up as resample_poly scales it; poly[ph][k] = h[ph + k up].
void stoi_tables(const StoiLaunch& a, std::vector<float>& tab) {
    const double PI = 3.14159265358979323846;
    const int nh = 2 * a.half + 1;
    std::vector<double> h(nh > 1 ? nh : 0);
    if (a.up != a.down) {
        const double cutoff = 1.0 / (2 * (a.up > a.down ? a.up : a.down)), beta = 0.1102 * (60.0 - 8.7), i0b = bessel_i0(beta);
        double sum = 0.0;
        for (int i = 0; i < nh; ++i) {
            const double t = i - a.half, u = 2 * cutoff * t;
            const double sinc = t == 0 ? 1.0 : std::sin(PI * u) / (PI * u);
            const double r = 2.0 * i / (nh - 1) - 1.0;
            h[i] = bessel_i0(beta * std::sqrt(1.0 - r * r)) / i0b * (2 * a.up * cutoff * sinc);
            sum += h[i];
        }
        for (double& v : h) v = v / sum * a.up;
    }
    tab.clear();
    for (int k = 0; k < STOI_FRAME; ++k) {
        tab.push_back((float)std::cos(2.0 * PI * k / (2 * STOI_FRAME)));
        tab.push_back((float)-std::sin(2.0 * PI * k / (2 * STOI_FRAME)));
    }
    for (int u = 0; u < STOI_FRAME; ++u) tab.push_back((float)(0.5 - 0.5 * std::cos(2.0 * PI * (u + 1) / (STOI_FRAME + 1))));
    const size_t p0 = tab.size();
    tab.resize(p0 + (size_t)a.up * a.ntap, 0.f);
    for (int i = 0; i < nh && a.up != a.down; ++i) tab[p0 + (size_t)(i % a.up) * a.ntap + i / a.up] = (float)h[i];
}

static size_t carve(size_t& off, size_t bytes) { const size_t o = off; off += (bytes + 255) / 256 * 256; return o; }
template <typename T> static T* at(void* ws, size_t o) { return ws ? reinterpret_cast<T*>(static_cast<char*>(ws) + o) : nullptr; }

// [lengths: B int64][partials: B x nchunk double2][alpha: B double]
size_t si_sdr_layout(SiSdrLaunch& a, void* ws, int B, long long Lmax) {
    size_t off = 0;
    a.B = B;
    a.nchunk = (int)((Lmax + SISDR_CHUNK - 1) / SISDR_CHUNK);
    a.len = at<long long>(ws, carve(off, (size_t)B * sizeof(long long)));
    a.part = at<double2>(ws, carve(off, (size_t)B * a.nchunk * sizeof(double2)));
    a.alpha = at<double>(ws, carve(off, (size_t)B * sizeof(double)));
    return off;
}

// [lengths: B int64][tables (stoi_tables)][energy: B x F double][kept: B x F int][K: B int][env: 2 x B x F x 16 double][partials:
// B x P double], F = the longest clip's frame count, P = ceil(F / 16).  stoi_geometry(a) first.
size_t stoi_layout(StoiLaunch& a, void* ws, int B, long long Lmax) {
    const long long n = (Lmax * a.up + a.down - 1) / a.down;
    const long long F = n > STOI_FRAME ? (n - STOI_FRAME + STOI_HOP - 1) / STOI_HOP : 0, Fs = F > 0 ? F : 1;
    size_t off = 0;
    a.B = B;
    a.F = F;
    a.P = (Fs + STOI_SEGS - 1) / STOI_SEGS;
    a.len = at<long long>(ws, carve(off, (size_t)B * sizeof(long long)));
    const size_t tab = carve(off, stoi_table_floats(a) * sizeof(float));
    a.tw = at<float2>(ws, tab);
    a.win = at<float>(ws, tab + 2 * STOI_FRAME * sizeof(float));
    a.poly = at<float>(ws, tab + 3 * STOI_FRAME * sizeof(float));
    a.energy = at<double>(ws, carve(off, (size_t)B * Fs * sizeof(double)));
    a.kept = at<int>(ws, carve(off, (size_t)B * Fs * sizeof(int)));
    a.nkept = at<int>(ws, carve(off, (size_t)B * sizeof(int)));
    a.env = at<double>(ws, carve(off, (size_t)2 * B * Fs * 16 * sizeof(double)));
    a.part = at<double>(ws, carve(off, (size_t)B * a.P * sizeof(double)));
    return off;
}

static unsigned grid_x(long long n, int per) { return (unsigned)(n > 0 ? (n + per - 1) / per : 1); }

cudaError_t launch_stoi(const StoiLaunch& a, cudaStream_t s) {
    stoi_energy_kernel<<<dim3(grid_x(a.F, STOI_ENERGY_FRAMES), a.B), MET_THREADS, 0, s>>>(a);
    stoi_keep_kernel<<<a.B, STOI_SCAN_THREADS, 0, s>>>(a);
    stoi_envelope_kernel<<<dim3(grid_x(a.F - 1, STOI_ENV_FRAMES), a.B), MET_THREADS, 0, s>>>(a);
    stoi_segment_kernel<<<dim3(grid_x(a.F - STOI_SEG, STOI_SEGS), a.B), MET_THREADS, 0, s>>>(a);
    stoi_final_kernel<<<a.B, MET_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}

// ---- SDR (BSS Eval v3, one source, 512-tap distortion filter) --------------------------------------------------------------------

// Shared-memory index of staged sample m: one pad double per 16, so runs that start 16 q samples apart (q odd, or q = 1 plus its pad)
// sit an odd number of doubles apart and a half-warp's 64-bit loads hit 16 different bank pairs.
__device__ __forceinline__ int sdr_pad(int m) { return m + (m >> 4); }

constexpr int SDR_CS = SDR_CORR_TILE + SDR_F + (SDR_CORR_TILE + SDR_F) / 16;   // padded staged length per signal, correlations
constexpr int SDR_PS = SDR_PROJ_TILE + SDR_F + (SDR_PROJ_TILE + SDR_F) / 16;   // the same, projection
static_assert(SDR_RUN % SDR_KB == 0 && (SDR_RUN / 16) % 2 == 1 && SDR_PROJ_TILE == MET_THREADS * 16, "sdr tiling");

// Sums each of the 2 H accumulators over the warp and leaves the sum of accumulator l in lane l's acc[0]: at each halving step the
// lanes with bit h set keep the upper half of the live accumulators and their partners the lower half (fixed pairs, fixed order).
template <int H>
__device__ __forceinline__ void reduce_scatter(double* acc, int lane) {
    const bool up = lane & H;
#pragma unroll
    for (int j = 0; j < H; ++j) {
        const double send = up ? acc[j] : acc[j + H], keep = up ? acc[j + H] : acc[j];
        acc[j] = keep + __shfl_xor_sync(0xffffffffu, send, H);
    }
    if constexpr (H > 1) reduce_scatter<H / 2>(acc, lane);
}

// grid (ceil(max L_b / 3584), B): samples n0 .. n0 + 3583 of clip b.  r and e are staged as fp64 with a 512-sample halo (zero past
// L_b); an fp32 x fp32 product is exact in fp64, so only the sums round.  Warp w takes lag blocks k0 = 16 kb, kb = w, w + 8, ..; lane l
// sums its 112-sample run n0 + 112 l + s for all 16 lags of R and of D, with the 16 values r[n + k0 + j] and e[n + k0 + j] in a
// circular register window that takes one new sample per step.  A reduce-scatter over the lanes (fixed pairs, so fixed order) leaves
// lane l with the warp's sum of accumulator l: R[k0 + l] for l < 16, D[k0 + l - 16] above.  Partial [b][tile][R 0..511, D 0..511].
__global__ void __launch_bounds__(MET_THREADS) sdr_corr_kernel(SdrLaunch a) {
    extern __shared__ __align__(8) double sdr_sm[];
    double* rs = sdr_sm;
    double* es = sdr_sm + SDR_CS;
    const int b = blockIdx.y;
    const long long Lb = a.len[b], n0 = (long long)blockIdx.x * SDR_CORR_TILE;
    if (n0 >= Lb) return;                                         // block-uniform
    const float* r = a.ref + (size_t)b * a.L;
    const float* e = a.est + (size_t)b * a.L;
    for (int m = threadIdx.x; m < SDR_CORR_TILE + SDR_F; m += MET_THREADS) {
        const long long n = n0 + m;
        rs[sdr_pad(m)] = n < Lb ? (double)__ldg(r + n) : 0.0;
        es[sdr_pad(m)] = n < Lb ? (double)__ldg(e + n) : 0.0;
    }
    __syncthreads();
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, m0 = lane * SDR_RUN;
    double* out = a.corr + ((size_t)b * a.nct + blockIdx.x) * (2 * SDR_F);
    for (int kb = w; kb < SDR_F / SDR_KB; kb += MET_THREADS / 32) {
        const int k0 = kb * SDR_KB;
        double acc[2 * SDR_KB], wr[SDR_KB], we[SDR_KB];
#pragma unroll
        for (int j = 0; j < SDR_KB; ++j) {
            acc[j] = 0.0; acc[SDR_KB + j] = 0.0;
            wr[j] = rs[sdr_pad(m0 + k0 + j)]; we[j] = es[sdr_pad(m0 + k0 + j)];
        }
        for (int s = 0; s < SDR_RUN; s += SDR_KB) {                  // m0 + s and m0 + s + k0 + 16 are multiples of 16
            const double* xr = rs + sdr_pad(m0 + s);
            const double* nr = rs + sdr_pad(m0 + s + k0 + SDR_KB);
            const double* ne = es + sdr_pad(m0 + s + k0 + SDR_KB);
#pragma unroll
            for (int u = 0; u < SDR_KB; ++u) {                       // slot (u + j) % 16 holds sample m0 + s + u + k0 + j
                const double x = xr[u];
#pragma unroll
                for (int j = 0; j < SDR_KB; ++j) {
                    acc[j] = fma(x, wr[(u + j) % SDR_KB], acc[j]);
                    acc[SDR_KB + j] = fma(x, we[(u + j) % SDR_KB], acc[SDR_KB + j]);
                }
                wr[u] = nr[u];
                we[u] = ne[u];
            }
        }
        reduce_scatter<16>(acc, lane);
        out[lane < SDR_KB ? k0 + lane : SDR_F + k0 + lane - SDR_KB] = acc[0];
    }
}

// grid (32, B): correlations 32 x .. 32 x + 31 of clip b summed over its tiles.  Warp g sums tiles g, g + 8, .. in order; lane 0 .. 31
// of warp 0 then adds the eight warp sums in warp order.
__global__ void __launch_bounds__(MET_THREADS) sdr_corr_sum_kernel(SdrLaunch a) {
    __shared__ double sh[MET_THREADS / 32][32];
    const int b = blockIdx.y, w = threadIdx.x >> 5, lane = threadIdx.x & 31, i = blockIdx.x * 32 + lane;
    const long long nt = (a.len[b] + SDR_CORR_TILE - 1) / SDR_CORR_TILE;
    const double* p = a.corr + (size_t)b * a.nct * (2 * SDR_F) + i;
    double s = 0.0;
    for (long long t = w; t < nt; t += MET_THREADS / 32) s += p[t * (2 * SDR_F)];
    sh[w][lane] = s;
    __syncthreads();
    if (w == 0) {
        s = sh[0][lane];
        for (int k = 1; k < MET_THREADS / 32; ++k) s += sh[k][lane];
        a.rd[(size_t)b * 2 * SDR_F + i] = s;
    }
}

// grid B, one warp: G c = D by Levinson's recursion (Durbin's prediction-error filter f, G_m f = E_m e_0, grown one order per step,
// and the solution x of the leading m x m system corrected by (D_m - <x, R[m - .]>) / E_{m+1} times the reversed new filter), fp64.
// R[0] = 0 (a silent reference) or a prediction error that is not a positive finite number stops it, and c is NaN.
__global__ void __launch_bounds__(32) sdr_solve_kernel(SdrLaunch a) {
    __shared__ double R[SDR_F], D[SDR_F], f[2][SDR_F], x[SDR_F];
    const int b = blockIdx.x, lane = threadIdx.x;
    const double* rd = a.rd + (size_t)b * 2 * SDR_F;
    for (int i = lane; i < SDR_F; i += 32) { R[i] = rd[i]; D[i] = rd[SDR_F + i]; f[0][i] = f[1][i] = x[i] = 0.0; }
    __syncwarp();
    double E = R[0];
    bool ok = E > 0.0;
    if (lane == 0) { f[0][0] = 1.0; x[0] = D[0] / E; }
    __syncwarp();
    for (int m = 1, cur = 0; m < SDR_F && ok; ++m, cur ^= 1) {      // f[cur] holds the order-m filter, zero from index m on
        const double* A = f[cur];
        double* An = f[cur ^ 1];
        double dl = 0.0, ep = 0.0;
        for (int j = lane; j < m; j += 32) { const double rr = R[m - j]; dl = fma(A[j], rr, dl); ep = fma(x[j], rr, ep); }
        for (int o = 16; o; o >>= 1) { dl += __shfl_xor_sync(0xffffffffu, dl, o); ep += __shfl_xor_sync(0xffffffffu, ep, o); }
        const double kappa = -dl / E;
        E = fma(kappa, dl, E);                                        // E_m (1 - kappa^2)
        ok = E > 0.0 && isfinite(E);                                  // the same on every lane: the butterfly sums are
        for (int j = lane; j <= m; j += 32) An[j] = fma(kappa, A[m - j], A[j]);
        __syncwarp();
        const double g = (D[m] - ep) / E;
        for (int j = lane; j <= m; j += 32) x[j] = fma(g, An[m - j], x[j]);
        __syncwarp();
    }
    for (int i = lane; i < SDR_F; i += 32) a.coef[(size_t)b * SDR_F + i] = ok ? x[i] : __longlong_as_double(0x7ff8000000000000LL);
}

// grid (ceil((max L_b + 511) / 4096), B): outputs p0 .. p0 + 4095 of clip b.  r[p0 - 512 ..] is staged as fp64 (zero outside the clip);
// thread t computes P[n] = sum_k c[k] r[n - k] for its 16 outputs q0 = 16 t .., the values r[n - k] in a circular window that takes one
// new sample per lag, then sums P^2 and (e' - P)^2 in output order; the CTA's sums (block_sum) are partial blockIdx.x.  Past
// n = L_b + 510 both P and e' are zero, so a tile's tail adds nothing.
__global__ void __launch_bounds__(MET_THREADS) sdr_proj_kernel(SdrLaunch a) {
    __shared__ double rs[SDR_PS];
    __shared__ double cs[SDR_F];
    __shared__ double sh[33];
    const int b = blockIdx.y;
    const long long Lb = a.len[b], p0 = (long long)blockIdx.x * SDR_PROJ_TILE;
    if (p0 >= Lb + SDR_F - 1) return;                             // block-uniform
    const float* r = a.ref + (size_t)b * a.L;
    const float* e = a.est + (size_t)b * a.L;
    for (int m = threadIdx.x; m < SDR_PROJ_TILE + SDR_F; m += MET_THREADS) {
        const long long n = p0 - SDR_F + m;
        rs[sdr_pad(m)] = n >= 0 && n < Lb ? (double)__ldg(r + n) : 0.0;
    }
    for (int k = threadIdx.x; k < SDR_F; k += MET_THREADS) cs[k] = a.coef[(size_t)b * SDR_F + k];
    __syncthreads();
    const int q0 = threadIdx.x * 16;
    double acc[16], win[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) { acc[j] = 0.0; win[j] = rs[sdr_pad(q0 + SDR_F + j)]; }   // lag 0: slot j holds r[p0 + q0 + j]
    for (int k0 = 0; k0 < SDR_F; k0 += 16) {
        const double* nr = rs + sdr_pad(q0 + SDR_F - 16 - k0);       // next sample at lag k0 + u: nr[15 - u] (r[p0 + q0 - k0 - u - 1])
#pragma unroll
        for (int u = 0; u < 16; ++u) {                               // slot (j - u) % 16 holds r[p0 + q0 + j - k0 - u]
            const double c = cs[k0 + u];
#pragma unroll
            for (int j = 0; j < 16; ++j) acc[j] = fma(c, win[(j - u + 16) % 16], acc[j]);
            win[15 - u] = nr[15 - u];
        }
    }
    double sp = 0.0, sn = 0.0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const long long n = p0 + q0 + j;
        const double ev = n < Lb ? (double)__ldg(e + n) : 0.0, d = ev - acc[j];
        sp = fma(acc[j], acc[j], sp);
        sn = fma(d, d, sn);
    }
    sp = block_sum(sp, sh);
    sn = block_sum(sn, sh);
    if (threadIdx.x == 0) a.part[(size_t)b * a.npt + blockIdx.x] = make_double2(sp, sn);
}

// grid B: clip b's projection partials in tile order, then 10 log10(sum P^2 / sum (e' - P)^2).
__global__ void __launch_bounds__(MET_THREADS) sdr_final_kernel(SdrLaunch a) {
    __shared__ double sh[33];
    const int b = blockIdx.x;
    const int n = (int)((a.len[b] + SDR_F - 1 + SDR_PROJ_TILE - 1) / SDR_PROJ_TILE);
    const double2* p = a.part + (size_t)b * a.npt;
    double s0 = 0.0, s1 = 0.0;
    for (int i = threadIdx.x; i < n; i += MET_THREADS) { s0 += p[i].x; s1 += p[i].y; }
    s0 = block_sum(s0, sh);
    s1 = block_sum(s1, sh);
    if (threadIdx.x == 0) a.out[b] = 10.0 * log10(s0 / s1);
}

// [lengths: B int64][correlation partials: B x nct x 1024 double][R, D: B x 1024 double][c: B x 512 double][projection partials:
// B x npt double2], nct = ceil(max L_b / 3584), npt = ceil((max L_b + 511) / 4096).
size_t sdr_layout(SdrLaunch& a, void* ws, int B, long long Lmax) {
    size_t off = 0;
    a.B = B;
    a.nct = (Lmax + SDR_CORR_TILE - 1) / SDR_CORR_TILE;
    a.npt = (Lmax + SDR_F - 1 + SDR_PROJ_TILE - 1) / SDR_PROJ_TILE;
    a.len = at<long long>(ws, carve(off, (size_t)B * sizeof(long long)));
    a.corr = at<double>(ws, carve(off, (size_t)B * a.nct * 2 * SDR_F * sizeof(double)));
    a.rd = at<double>(ws, carve(off, (size_t)B * 2 * SDR_F * sizeof(double)));
    a.coef = at<double>(ws, carve(off, (size_t)B * SDR_F * sizeof(double)));
    a.part = at<double2>(ws, carve(off, (size_t)B * a.npt * sizeof(double2)));
    return off;
}

cudaError_t launch_sdr(const SdrLaunch& a, cudaStream_t s) {
    const size_t smem = 2 * SDR_CS * sizeof(double);
    cudaError_t e = cudaFuncSetAttribute(sdr_corr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    sdr_corr_kernel<<<dim3((unsigned)a.nct, a.B), MET_THREADS, smem, s>>>(a);
    sdr_corr_sum_kernel<<<dim3(2 * SDR_F / 32, a.B), MET_THREADS, 0, s>>>(a);
    sdr_solve_kernel<<<a.B, 32, 0, s>>>(a);
    sdr_proj_kernel<<<dim3((unsigned)a.npt, a.B), MET_THREADS, 0, s>>>(a);
    sdr_final_kernel<<<a.B, MET_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}

}  // namespace fsn
