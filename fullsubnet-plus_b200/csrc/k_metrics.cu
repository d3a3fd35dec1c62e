// Objective scores of enhanced speech against its clean reference (fsn_metric_si_sdr, fsn_metric_stoi; DESIGN.md §3.20), one
// score per clip of a ragged [B, L] batch.  Every reduction that feeds a decision or a score is fp64, over a fixed per-clip tiling
// and in a fixed order, with no atomics: a clip's score depends on its own samples only, bit for bit, whatever else is in the batch.
//
// SI-SDR: two passes over the samples (the noise energy |e - a r|^2 is summed directly: the closed form |e|^2 - 2 a <r, e> + a^2 |r|^2
// cancels catastrophically at high SI-SDR), each a per-chunk partial kernel and a per-clip finalize kernel.
//
// STOI (classic, as pystoi 0.3.3): resampling to 10 kHz (an Octave-compatible Kaiser sinc, scipy's resample_poly alignment) is
// recomputed wherever a 10 kHz sample is needed, never stored.  Four kernels: frame energies of x; a per-clip max and keep-mask
// compaction; the band envelopes of the compacted x and y, gathered straight from the kept frames' original positions; the
// per-segment correlations with per-CTA partials; and the per-clip mean.
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

}  // namespace fsn
