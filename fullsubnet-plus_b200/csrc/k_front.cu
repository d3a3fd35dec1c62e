// Full-band front end of the FullSubNet+/FullSubNet forward on sm_90a:
//   * utterance Laplace norm + TSSE ("MulCA") channel attention     (K1 + K2 of SURVEY.md 2a)
//   * the output Linear of fullsubnet.Model's full-band LSTM (the TCN of FullSubNet+ is in k_gemm_tc5.cu)  (K3)
//   * utterance mean of the (never materialised) unfolded sub-band input and the fp16 packing of the
//     per-step LSTM input tiles                                                                  (K4)
#include "fsn_common.cuh"
#include "fsn_kernels.h"
#include "../../include/fsnplus_b200.h"

namespace fsn {

static thread_local bool g_chain_launch = false;       // set by the forward of the calling thread right before it enqueues the chain
bool fsn_chain_launch_enabled() { return g_chain_launch; }
void fsn_chain_launch_set(bool on) { g_chain_launch = on; }

// =============================================================================================
// K1 + K2: x / (mean(x) + 1e-5), then the TSSE gate.
// reference: audio_zen/model/base_model.py:210-225, audio_zen/model/module/attention_model.py:78-98
// conv(no padding) -> average pool is linear, so each pooled feature is
//   b_k[c] + sum_j w_k[c,j] * mean_t x[c, j : T'-k+1+j]
// i.e. 18 windowed means per channel, all derived from the row sum and the first / last 15 samples.
// Three kernels: row statistics over the whole GPU (one warp per (sample, branch, bin) row: the only pass that is bound by reading the
// input), the gate per (sample, branch) from those 35 numbers per row, and the scaling pass (tsse_apply_kernel; its read hits L2).
// =============================================================================================
constexpr int TSSE_KMAX = 16;
constexpr int TSSE_ROWW = 3 + 2 * TSSE_KMAX;         // per row: sum, max, min, KMAX exclusive prefix sums, KMAX exclusive suffix sums

__global__ void __launch_bounds__(256) tsse_rowstats_kernel(TsseLaunch a) {
    pdl_trigger();
    pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int F = a.F;
    const int r = blockIdx.x * 8 + warp;                          // (branch, sample, bin)
    if (r >= a.nbranch * a.B * F) return;
    const int z = r / F, f = r % F, br = z / a.B, b = z % a.B;
    const float* row = a.x[br] + ((size_t)b * F + f) * a.T;       // row pitch a.T; the sample's own extent T (input), Tp (padded)
    const int Tp = a.tlen ? a.tlen[z] : a.Tp, T = Tp - (a.Tp - a.T);
    float acc = 0.f, mx = -INFINITY, mn = INFINITY;
    for (int t0 = 0; t0 < T; t0 += 256) {                         // eight independent loads per lane in flight
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) { const int t = t0 + u * 32 + lane; v[u] = (t < T) ? __ldg(row + t) : 0.f; }
#pragma unroll
        for (int u = 0; u < 8; ++u)
            if (t0 + u * 32 + lane < T) { acc += v[u]; mx = fmaxf(mx, v[u]); mn = fminf(mn, v[u]); }
    }
    acc = warp_sum(acc);
#pragma unroll
    for (int o = 16; o; o >>= 1) { mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); }
    // exclusive prefix sums over the first / last KMAX samples of the padded row: lane j holds sample j (head) and
    // sample Tp-1-j (tail; t >= T is the zero look-ahead pad), one shuffle scan each
    float hv = (lane < TSSE_KMAX && lane < T) ? row[lane] : 0.f;
    const int tt = Tp - 1 - lane;
    float tv = (lane < TSSE_KMAX && tt >= 0 && tt < T) ? row[tt] : 0.f;
    float hs = hv, ts = tv;
#pragma unroll
    for (int o = 1; o < TSSE_KMAX; o <<= 1) {
        const float uh = __shfl_up_sync(0xffffffffu, hs, o), ut = __shfl_up_sync(0xffffffffu, ts, o);
        if (lane >= o) { hs += uh; ts += ut; }
    }
    float* out = a.rows + (size_t)r * TSSE_ROWW;
    if (lane == 0) { out[0] = acc; out[1] = mx; out[2] = mn; }
    if (lane < TSSE_KMAX) { out[3 + lane] = hs - hv; out[3 + TSSE_KMAX + lane] = ts - tv; }
}

__global__ void __launch_bounds__(1024) tsse_norm_kernel(TsseLaunch a) {
    extern __shared__ float sm[];
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.x, br = blockIdx.y;
    const int F = a.F, Tp = a.tlen ? a.tlen[br * a.B + b] : a.Tp, T = Tp - (a.Tp - a.T);   // this sample's extent
    // shared memory: 5 F + F / 2 + 1 floats (tsse_norm_smem).  The exclusive prefix / suffix sums of the first / last KMAX samples stay in
    // the row statistics (global memory, just written by tsse_rowstats_kernel), read only by the thread of their channel.
    float* S = sm;                                  // [F] row sums
    float* sq = S + F;                              // [F]
    float* gate = sq + F;                           // [F]
    float* f1 = gate + F;                           // [F/2]
    float* Mx = f1 + (F / 2 + 1);                   // [F] row max / [F] row min (CBAM squeeze)
    float* Mn = Mx + F;
    __shared__ float s_inv;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
    const float* rows = a.rows + ((size_t)br * a.B + b) * F * TSSE_ROWW;   // [F][TSSE_ROWW]: sum, max, min, prefix sums, suffix sums
    for (int f = threadIdx.x; f < F; f += blockDim.x) {
        S[f] = rows[(size_t)f * TSSE_ROWW];
        Mx[f] = rows[(size_t)f * TSSE_ROWW + 1];
        Mn[f] = rows[(size_t)f * TSSE_ROWW + 2];
    }
    __syncthreads();
    if (warp == 0) {
        double tot = 0.0;
        for (int f = lane; f < F; f += 32) tot += (double)S[f];
        tot = warp_sum_d(tot);
        if (lane == 0) s_inv = a.prenorm ? 1.0f : (float)(1.0 / (tot / ((double)F * (double)Tp) + 1e-5));
    }
    __syncthreads();
    const float inv = s_inv;

    if (a.attention) {
        const TsseParams& p = a.p[br];
        const int kind = a.attention - 1;
        const float rT = 1.0f / (float)Tp;
        if (kind == FSN_ATTN_TSSE) {                 // attention_model.py:78-104: three depthwise convs, time-averaged, mixed by a 3 -> 1 linear
            for (int c = threadIdx.x; c < F; c += blockDim.x) {
                const float* Pfx = rows + (size_t)c * TSSE_ROWW + 3;              // Pfx[j] = sum_{t<j} x[c][t]
                const float* Sfx = Pfx + TSSE_KMAX;                               // Sfx[m] = sum_{t>=Tp-m} x[c][t]
                float s = p.cat_b[0];
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                    const int k = a.ksz[i];
                    const float rlen = 1.0f / (float)(Tp - k + 1);
                    float acc = 0.f;
                    for (int j = 0; j < k; ++j) {
                        float wsum = S[c] - Pfx[j] - Sfx[k - 1 - j];
                        acc = fmaf(p.conv_w[i][c * k + j], wsum, acc);
                    }
                    float feat = fmaxf(fmaf(acc, inv * rlen, p.conv_b[i][c]), 0.f);
                    s = fmaf(p.cat_w[i], feat, s);
                }
                sq[c] = s;
            }
        } else {                                     // SE / CBAM / ECA squeeze: mean over the padded frames (attention_model.py:29,320,353)
            for (int c = threadIdx.x; c < F; c += blockDim.x) {
                sq[c] = S[c] * inv * rT;
                // CBAM max squeeze (:321) of x * inv: the sign of inv picks max or min; the zero look-ahead pad takes part
                float m = (inv >= 0.f) ? Mx[c] * inv : Mn[c] * inv;
                if (Tp > T) m = fmaxf(m, 0.f);
                Mx[c] = m;
            }
        }
        __syncthreads();
        if (kind == FSN_ATTN_ECA && a.sub > 1 && br == 0) {
            // subband_num > 1 (fullsubnet_plus.py:146-153, mag branch): the F bins are reflect-padded to (F / sub + 1) * sub and
            // every `sub` consecutive bins form one attention channel whose "time" axis is sub * Tp long
            const int sub = a.sub, Cg = F / sub + 1;
            const float w0 = p.eca_w[0], w1 = p.eca_w[1], w2 = p.eca_w[2];
            float* sg = Mx;                           // [Cg] group squeeze, f1: [Cg] group gate (Cg <= F / 2 + 1)
            for (int c = threadIdx.x; c < Cg; c += blockDim.x) {
                float acc = 0.f;
                for (int j = 0; j < sub; ++j) { int f = c * sub + j; if (f >= F) f = 2 * F - 2 - f; acc += S[f]; }
                sg[c] = acc * inv / ((float)Tp * (float)sub);
            }
            __syncthreads();
            for (int c = threadIdx.x; c < Cg; c += blockDim.x) {
                const float y = w0 * (c > 0 ? sg[c - 1] : 0.f) + w1 * sg[c] + w2 * (c + 1 < Cg ? sg[c + 1] : 0.f);
                f1[c] = 1.0f / (1.0f + __expf(-y));
            }
            __syncthreads();
            for (int c = threadIdx.x; c < F; c += blockDim.x) gate[c] = f1[c / sub];
        } else if (kind == FSN_ATTN_ECA) {           // attention_model.py:355-357: conv1d over the channel axis, k = 3, zero padding, no bias
            const float w0 = p.eca_w[0], w1 = p.eca_w[1], w2 = p.eca_w[2];
            for (int c = threadIdx.x; c < F; c += blockDim.x) {
                const float y = w0 * (c > 0 ? sq[c - 1] : 0.f) + w1 * sq[c] + w2 * (c + 1 < F ? sq[c + 1] : 0.f);
                gate[c] = 1.0f / (1.0f + __expf(-y));
            }
        } else {
            // two small dense layers (F -> F/2 -> F): four output rows per warp at a time so that 4 x ceil(F/32) independent weight loads are
            // in flight per lane (with one row per warp and 8 warps this phase was 50 dependent L2 round trips = 55 us of the 69 us kernel)
            const int Cr = F / 2;
            for (int o0 = warp * 4; o0 < Cr; o0 += nwarp * 4) {
                float acc[4] = {0.f, 0.f, 0.f, 0.f}, acm[4] = {0.f, 0.f, 0.f, 0.f};
                for (int c = lane; c < F; c += 32) {
                    const float sv = sq[c], mv = Mx[c];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float w = (o0 + j < Cr) ? __ldg(p.fc1_w + (size_t)(o0 + j) * F + c) : 0.f;
                        acc[j] = fmaf(w, sv, acc[j]);
                        acm[j] = fmaf(w, mv, acm[j]);
                    }
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float a1 = warp_sum(acc[j]);
                    float v = 0.f;
                    if (o0 + j < Cr) v = fmaxf(a1 + p.fc1_b[o0 + j], 0.f);
                    if (kind == FSN_ATTN_CBAM) { const float a2 = warp_sum(acm[j]); if (o0 + j < Cr) v += fmaxf(a2 + p.fc1_b[o0 + j], 0.f); }   // shared fc1 on both squeezes (:324-329)
                    if (lane == 0 && o0 + j < Cr) f1[o0 + j] = v;
                }
            }
            __syncthreads();
            for (int o0 = warp * 4; o0 < F; o0 += nwarp * 4) {
                float acc[4] = {0.f, 0.f, 0.f, 0.f};
                for (int c = lane; c < Cr; c += 32) {
                    const float fv = f1[c];
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[j] = fmaf((o0 + j < F) ? __ldg(p.fc2_w + (size_t)(o0 + j) * Cr + c) : 0.f, fv, acc[j]);
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float a1 = warp_sum(acc[j]);
                    if (lane == 0 && o0 + j < F) gate[o0 + j] = 1.0f / (1.0f + __expf(-(a1 + p.fc2_b[o0 + j])));
                }
            }
        }
        __syncthreads();
    }
    // per-row scale (gate * 1/(mean + 1e-5)); the bulk multiply + time-major transpose runs in tsse_apply_kernel on the whole GPU
    float amax = 0.f;
    for (int f = threadIdx.x; f < F; f += blockDim.x) {
        const float sc = a.attention ? gate[f] * inv : inv;
        a.scale[((size_t)br * a.B + b) * F + f] = sc;
        const float* rw = a.rows + (((size_t)br * a.B + b) * F + f) * TSSE_ROWW;       // row max / min (Mx / Mn may hold the CBAM squeeze by now)
        amax = fmaxf(amax, fmaxf(fabsf(rw[1]), fabsf(rw[2])) * fabsf(sc));
    }
    if (a.amax) {                                                                      // max |x0| of this (sample, branch): scale of the fp16 hidden activation
        __shared__ float s_amax[32];
#pragma unroll
        for (int o = 16; o; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        if (lane == 0) s_amax[warp] = amax;
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int i = 1; i < nwarp; ++i) amax = fmaxf(amax, s_amax[i]);
            a.amax[(size_t)br * a.B + b] = amax;
        }
    }
}

// out[z][f][t] = x[z][f][t] * scale[z][f] (zero in the look-ahead pad) in both layouts; one CTA per 32 x 32 tile.
__global__ void __launch_bounds__(256) tsse_apply_kernel(TsseLaunch a) {
    __shared__ float tr[32][33];
    pdl_trigger();
    pdl_wait();
    const int z = blockIdx.z, br = z / a.B, b = z % a.B, F = a.F, Tp = a.Tp;
    const int T = a.tlen ? a.tlen[z] - (a.Tp - a.T) : a.T;        // frames of this sample's input: zero from here on in both layouts
    const int f0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* x = a.x[br] + (size_t)b * F * a.T;
    float* out = a.out + (size_t)z * F * a.P;
    float* otm = a.out_tm ? a.out_tm + (size_t)z * Tp * a.Cp : nullptr;
    for (int rr = warp; rr < 32; rr += 8) {
        const int f = f0 + rr, t = t0 + lane;
        float v = 0.f;
        if (f < F && t < a.P) {
            v = (t < T) ? x[(size_t)f * a.T + t] * a.scale[(size_t)z * F + f] : 0.f;
            out[(size_t)f * a.P + t] = v;
        }
        tr[rr][lane] = v;
    }
    __syncthreads();
    if (otm)
        for (int rr = warp; rr < 32; rr += 8) {
            const int t = t0 + rr, f = f0 + lane;
            if (t < Tp && f < F) otm[(size_t)t * a.Cp + f] = tr[lane][rr];
        }
}

size_t tsse_norm_smem(int F) { return sizeof(float) * ((size_t)F * 5 + F / 2 + 8); }

const char* launch_tsse_norm(const TsseLaunch& a, cudaStream_t s, cudaError_t* err) {
    const size_t smem = tsse_norm_smem(a.F);
    if ((*err = cudaFuncSetAttribute(tsse_norm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem))) return "tsse_norm_kernel";
    if ((*err = launch_chain(tsse_rowstats_kernel, dim3((a.nbranch * a.B * a.F + 7) / 8), dim3(256), 0, s, a))) return "tsse_rowstats_kernel";
    if ((*err = launch_chain(tsse_norm_kernel, dim3(a.B, a.nbranch), dim3(1024), smem, s, a))) return "tsse_norm_kernel";
    if ((*err = launch_chain(tsse_apply_kernel, dim3((a.P + 31) / 32, (a.F + 31) / 32, a.B * a.nbranch), dim3(256), 0, s, a)))
        return "tsse_apply_kernel";
    return nullptr;
}


// =============================================================================================
// Input normalisations other than offline_laplace_norm.  reference: base_model.py:227-258 (cumulative_laplace_norm),
// :260-275 (offline_gaussian_norm), :277-316 (cumulative_layer_norm); all applied AFTER the look-ahead zero padding
// (fullsubnet_plus.py:137-144), so the padded frames take part and come out non-zero for the centred norms.
// One CTA per (sample, branch): per-frame sums over F, a serial fp64 scan over the frames, y = x * a[t] + b[t].
// =============================================================================================
__global__ void __launch_bounds__(256) input_norm_kernel(NormLaunch a) {
    const int b = blockIdx.x, br = blockIdx.y, F = a.F, T = a.T, Tp = a.Tp;
    const int Tpe = a.tlen ? a.tlen[br * a.B + b] : Tp, Te = Tpe - (Tp - T);   // this sample's extent: padded, input
    float* cs = a.frames + ((size_t)br * a.B + b) * 4 * Tp;   // [Tp] column sums (global scratch: any clip length fits)
    float* cq = cs + Tp;        // [Tp] column sums of squares
    float* sa = cq + Tp;        // [Tp] scale
    float* sb = sa + Tp;        // [Tp] shift
    const float* x = a.x[br] + (size_t)b * F * T;
    for (int t = threadIdx.x; t < Tp; t += blockDim.x) {
        float s = 0.f, q = 0.f;
        if (t < Te)
            for (int f = 0; f < F; ++f) { const float v = x[(size_t)f * T + t]; s += v; q = fmaf(v, v, q); }
        cs[t] = s; cq[t] = q;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const double EPS = 1.1920928955078125e-07;            // np.finfo(np.float32).eps (audio_zen/constant.py:8)
        if (a.type == FSN_NORM_OFFLINE_GAUSSIAN) {
            double s = 0, q = 0;
            for (int t = 0; t < Tpe; ++t) { s += cs[t]; q += cq[t]; }
            const double n = (double)F * Tpe, mu = s / n;
            const double var = (q - n * mu * mu) / (n - 1.0);  // torch.std: unbiased
            const double inv = 1.0 / (sqrt(var > 0 ? var : 0) + 1e-5);
            for (int t = 0; t < Tpe; ++t) { sa[t] = (float)inv; sb[t] = (float)(-mu * inv); }
        } else {
            double s = 0, q = 0;
            for (int t = 0; t < Tpe; ++t) {
                s += cs[t]; q += cq[t];
                const double cnt = (double)F * (t + 1), cm = s / cnt;
                if (a.type == FSN_NORM_CUMULATIVE_LAPLACE) { sa[t] = (float)(1.0 / (cm + EPS)); sb[t] = 0.f; }
                else {
                    const double cv = (q - 2.0 * cm * s) / cnt + cm * cm;
                    const double inv = 1.0 / sqrt(cv + EPS);
                    sa[t] = (float)inv; sb[t] = (float)(-cm * inv);
                }
            }
        }
        for (int t = Tpe; t < Tp; ++t) { sa[t] = 0.f; sb[t] = 0.f; }      // past this sample's end: y = 0
    }
    __syncthreads();
    float* y = a.y + ((size_t)br * a.B + b) * F * Tp;
    for (int e = threadIdx.x; e < F * Tp; e += blockDim.x) {
        const int f = e / Tp, t = e % Tp;
        const float v = (t < Te) ? x[(size_t)f * T + t] : 0.f;
        y[e] = fmaf(v, sa[t], sb[t]);
    }
}

cudaError_t launch_input_norm(const NormLaunch& a, cudaStream_t s) {
    input_norm_kernel<<<dim3(a.B, a.nbranch), 256, 0, s>>>(a);
    return cudaGetLastError();
}

// =============================================================================================
// Output Linear of the full-band LSTM of fullsubnet.Model (fullsubnet.py:86, sequence_model.py:118-121):
// Y[z] = act(W * X[z] + b) on the [Z, K, P] layout as a TF32 tensor-core GEMM (mma.sync m16n8k8), 64x64x32 tiles, 4 warps.
// (The TCN's 1x1 convolutions run on wgmma, k_gemm_tc5.cu; this small GEMM is latency-bound: Z <= 64, K = 512, M = 257.)
// =============================================================================================
__global__ void __launch_bounds__(128) conv1x1_tf32_kernel(ConvLaunch a) {
    __shared__ uint32_t Ws[64][36];
    __shared__ uint32_t Xs[32][72];
    const int z = blockIdx.z;
    const int m0 = blockIdx.y * 64, t0 = blockIdx.x * 64;
    const int M = a.M, K = a.K, Tp = a.Tp, P = a.P;
    const float* W = a.W;
    const float* X = a.X + (size_t)z * K * P;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wm = warp >> 1, wn = warp & 1;

    float acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

    for (int k0 = 0; k0 < K; k0 += 32) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            int e = tid + 128 * j, r = e >> 5, c = e & 31;
            float v = (m0 + r < M && k0 + c < K) ? W[(size_t)(m0 + r) * K + k0 + c] : 0.f;
            Ws[r][c] = f2tf32(v);
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            int e = tid + 128 * j, kk = e >> 6, tt = e & 63;
            float v = (k0 + kk < K && t0 + tt < Tp) ? X[(size_t)(k0 + kk) * P + t0 + tt] : 0.f;
            Xs[kk][tt] = f2tf32(v);
        }
        __syncthreads();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            uint32_t af[2][4], bf[4][2];
            const int r = lane >> 2, c = ks * 8 + (lane & 3);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                int rr = wm * 32 + mt * 16 + r;
                af[mt][0] = Ws[rr][c]; af[mt][1] = Ws[rr + 8][c]; af[mt][2] = Ws[rr][c + 4]; af[mt][3] = Ws[rr + 8][c + 4];
            }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                int nn = wn * 32 + nt * 8 + (lane >> 2);
                bf[nt][0] = Xs[ks * 8 + (lane & 3)][nn];
                bf[nt][1] = Xs[ks * 8 + (lane & 3) + 4][nn];
            }
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) mma_tf32_1688(acc[mt][nt], af[mt], bf[nt][0], bf[nt][1]);
        }
        __syncthreads();
    }

    float* Y = a.Y + (size_t)z * M * P;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                int row = m0 + wm * 32 + mt * 16 + (lane >> 2) + ((q & 2) ? 8 : 0);
                int col = t0 + wn * 32 + nt * 8 + 2 * (lane & 3) + (q & 1);
                if (row < M && col < Tp) Y[(size_t)row * P + col] = apply_act(acc[mt][nt][q] + a.bias[row], a.act);
            }
}

void launch_conv1x1(const ConvLaunch& a, cudaStream_t s) {
    conv1x1_tf32_kernel<<<dim3((a.Tp + 63) / 64, (a.M + 63) / 64, a.Z), 128, 0, s>>>(a);
}

// =============================================================================================
// K4: sub-band input.  reference: fullsubnet_plus.py:167-202 / fullsubnet.py:90-111 + base_model.py:15-47.
// The [B, F, I, T'] unfolded tensor is never materialised in fp32: its utterance mean follows from
// row sums (each reflected row counted as often as it appears in some window), and the normalised
// values are written once, in fp16, directly in the per-step 128-row tile images the LSTM kernels
// stream (K-major, SWIZZLE_128B, 64 halves per row; columns >= I and rows >= B*F are zero).  A wide input (64 < I <= 128, DESIGN.md
// §3.3) is written as plain fp16 rows of 128 halves instead (Fp16Wide): the A operand of layer 0's input-projection GEMM, or the
// generic kernel's time-major input.
// =============================================================================================
// row sums (and sums of squares) of the window source and the full-band outputs: one warp per row, the whole GPU
__global__ void __launch_bounds__(256) sb_rowsum_kernel(SbPackLaunch a) {
    pdl_trigger();
    pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int F = a.F, nsrc = 1 + a.nfb;
    const int r = blockIdx.x * 8 + warp;                       // (b, which, f)
    if (r >= a.B * nsrc * F) return;
    const int b = r / (nsrc * F), which = (r / F) % nsrc, f = r % F;
    const int Tp = a.tlen ? a.tlen[b] : a.Tp;
    const float* row = (which == 0) ? a.win + ((size_t)b * F + f) * a.Pw
                                    : ((which == 1) ? a.fb[0] : (which == 2) ? a.fb[1] : a.fb[2]) + ((size_t)b * F + f) * a.P;
    float acc = 0.f, acq = 0.f;
    for (int t = lane; t < Tp; t += 32) { const float v = row[t]; acc += v; acq = fmaf(v, v, acq); }
    acc = warp_sum(acc); acq = warp_sum(acq);
    if (lane == 0) { a.rowsum[2 * (size_t)r] = acc; a.rowsum[2 * (size_t)r + 1] = acq; }
}

__global__ void __launch_bounds__(256) sb_stats_kernel(SbPackLaunch a) {
    pdl_trigger();
    pdl_wait();
    const int b = blockIdx.x, F = a.F, Tp = a.tlen ? a.tlen[b] : a.Tp, nsrc = 1 + a.nfb;
    __shared__ double red[16];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
    const float* S = a.rowsum + (size_t)b * nsrc * F * 2;        // [which][f][2]
    double tot = 0.0, tq = 0.0;
    const int nw = 2 * a.Ns + 1, nf = 2 * a.Nf + 1;
    for (int e = threadIdx.x; e < F * nw; e += blockDim.x) {
        const int i = reflect_idx(e / nw + e % nw - a.Ns, F);
        tot += (double)S[2 * i]; tq += (double)S[2 * i + 1];
    }
    for (int k = 0; k < a.nfb; ++k)
        for (int e = threadIdx.x; e < F * nf; e += blockDim.x) {
            const int i = (k + 1) * F + reflect_idx(e / nf + e % nf - a.Nf, F);
            tot += (double)S[2 * i]; tq += (double)S[2 * i + 1];
        }
    tot = warp_sum_d(tot); tq = warp_sum_d(tq);
    if (lane == 0) { red[warp] = tot; red[8 + warp] = tq; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0, q = 0;
        for (int i = 0; i < nwarp; ++i) { s += red[i]; q += red[8 + i]; }
        const double n = (double)F * (double)(nw + a.nfb * nf) * (double)Tp, mu = s / n;
        a.mu[b] = (float)mu;
        if (a.sigma) { const double var = (q - n * mu * mu) / (n - 1.0); a.sigma[b] = (float)sqrt(var > 0 ? var : 0); }
    }
}

const char* launch_sb_stats(const SbPackLaunch& a, cudaStream_t s, cudaError_t* err) {
    if ((*err = launch_chain(sb_rowsum_kernel, dim3((a.B * (1 + a.nfb) * a.F + 7) / 8), dim3(256), 0, s, a))) return "sb_rowsum_kernel";
    if ((*err = launch_chain(sb_stats_kernel, dim3(a.B), dim3(256), 0, s, a))) return "sb_stats_kernel";
    return nullptr;
}

// Stores of the normalised sub-band input.  Fp16Img: the SWIZZLE_128B images of the LSTM kernels (values clamped to the fp16
// range).  Fp32Tm: the sub-band TCN's time-major fp32 rows of 64 channels, plus max |x| per sequence (block 0's fp16 store scale).
// Both packers compute every value once and hand 8 consecutive channels k0 .. k0 + 7 of (sequence row, frame t) to store().
// kChunk: the store takes the bin range a.f0 .. a.f0 + a.Fc - 1 (rows b * Fc + f - f0); without it every bin, rows b * F + f.
struct Fp16Img {
    static constexpr bool kChunk = false;
    static constexpr int kWidth = 64;                  // channels per row
    static constexpr bool kTimeMajor = false;
    static __device__ __forceinline__ void store(const SbPackLaunch& a, int row, int t, int k0, const float (&v)[8]) {
        float w[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) w[i] = fminf(fmaxf(v[i], -65504.f), 65504.f);
        char* img = reinterpret_cast<char*>(a.ximg) + ((size_t)(row >> 7) * a.Tw + (t - a.t0)) * (128 * 128);
        *reinterpret_cast<uint4*>(img + sw128_offset(row & 127, k0)) =
            make_uint4(pack_half2(w[0], w[1]), pack_half2(w[2], w[3]), pack_half2(w[4], w[5]), pack_half2(w[6], w[7]));
    }
    static __device__ __forceinline__ void finish(const SbPackLaunch&, int, float, unsigned) {}
};
struct Fp32Tm {
    static constexpr bool kChunk = true;
    static constexpr int kWidth = 64;
    static __device__ __forceinline__ void store(const SbPackLaunch& a, int row, int t, int k0, const float (&v)[8]) {
        float4* dst = reinterpret_cast<float4*>(a.xtm + ((size_t)row * a.Tp + t) * 64 + k0);
        dst[0] = make_float4(v[0], v[1], v[2], v[3]);
        dst[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
    // max over the lanes of `group` (lanes that share the sequence row), one atomic per group (values >= 0: int order = float order)
    static __device__ __forceinline__ void finish(const SbPackLaunch& a, int row, float m, unsigned width) {
        for (unsigned o = 1; o < width; o <<= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if ((threadIdx.x & (width - 1)) == 0 && row >= 0) atomicMax(reinterpret_cast<int*>(a.amax + row), __float_as_int(m));
    }
};
// Fp16Wide: rows of 128 halves, unswizzled (values clamped like Fp16Img).  TM = false: the rows of layer 0's input-projection GEMM,
// (tile * Tw + t - t0) * 128 + r in the order of the recurrence's hseq; TM = true: the generic kernel's time-major input
// [Tw, ntiles * 128, 128], row (t - t0) * ntiles * 128 + row.
__device__ __forceinline__ size_t wide_row(bool tm, int row, int t, int t0, int Tw, int ntiles) {
    return tm ? (size_t)(t - t0) * ntiles * 128 + row : ((size_t)(row >> 7) * Tw + (t - t0)) * 128 + (row & 127);
}
__device__ __forceinline__ uint4 pack_half8(const float (&v)[8]) {
    float w[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) w[i] = fminf(fmaxf(v[i], -65504.f), 65504.f);
    return make_uint4(pack_half2(w[0], w[1]), pack_half2(w[2], w[3]), pack_half2(w[4], w[5]), pack_half2(w[6], w[7]));
}
template <bool TM>
struct Fp16Wide {
    static constexpr bool kChunk = false;
    static constexpr int kWidth = 128;
    static constexpr bool kTimeMajor = TM;
    static __device__ __forceinline__ void store(const SbPackLaunch& a, int row, int t, int k0, const float (&v)[8]) {
        *reinterpret_cast<uint4*>(a.ximg + wide_row(TM, row, t, a.t0, a.Tw, a.ntiles) * 128 + k0) = pack_half8(v);
    }
    static __device__ __forceinline__ void finish(const SbPackLaunch&, int, float, unsigned) {}
};
__device__ __forceinline__ float vmax8(float m, const float (&v)[8]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) m = fmaxf(m, fabsf(v[i]));
    return m;
}

// One CTA = (sample, 32 consecutive bins of the range, 32 frames).  The window source rows [f0 - Ns, f0 + 31 + Ns] (reflected) and the
// full-band rows of the 32 bins are staged once in shared memory; work item = (bin, frame, 8 channels), so 8 consecutive lanes
// write one whole row of 64 channels (one 128-byte line of the SWIZZLE_128B image).  Rows of 128 channels (Fp16Wide): 16 lanes per
// row, the CTA's bins in two passes of 16.
constexpr int SBP_F = 32, SBP_T = 32;
template <class Store>
__global__ void __launch_bounds__(256) sb_pack_kernel(SbPackLaunch a) {
    extern __shared__ float sm[];
    const int fb = Store::kChunk ? a.f0 : 0, Fn = Store::kChunk ? a.Fc : a.F;   // bins fb .. fb + Fn - 1
    const int F = a.F, Tp = a.t0 + a.Tw, b = blockIdx.z, f0 = fb + blockIdx.y * SBP_F, t0 = a.t0 + blockIdx.x * SBP_T;   // Tp: the window's end
    const int Tpe = a.tlen ? a.tlen[b] : Tp;                       // frames t >= Tpe are past this sample's end: written as zero
    const int nw = 2 * a.Ns + 1, nf = 2 * a.Nf + 1, I = nw + a.nfb * nf;
    const int wrows = SBP_F + 2 * a.Ns, frows = SBP_F + 2 * a.Nf;
    float* wsm = sm;                                   // [wrows][SBP_T + 1]
    float* fsm = sm + wrows * (SBP_T + 1);             // [nfb][frows][SBP_T + 1]
    const bool gauss = (a.norm_type == FSN_NORM_OFFLINE_GAUSSIAN);
    const float inv = gauss ? 1.0f / (a.sigma[b] + 1e-5f) : 1.0f / (a.mu[b] + 1e-5f);
    const float sub = gauss ? a.mu[b] : 0.f;
    for (int e = threadIdx.x; e < wrows * SBP_T; e += blockDim.x) {
        const int rr = e / SBP_T, tt = e % SBP_T, t = t0 + tt;
        const int f = reflect_idx(min(f0 + rr - a.Ns, F - 1 + a.Ns), F);
        wsm[rr * (SBP_T + 1) + tt] = (t < Tpe) ? a.win[((size_t)b * F + f) * a.Pw + t] : 0.f;
    }
    for (int q = 0; q < a.nfb; ++q) {
        const float* src = (q == 0) ? a.fb[0] : (q == 1) ? a.fb[1] : a.fb[2];
        for (int e = threadIdx.x; e < frows * SBP_T; e += blockDim.x) {
            const int rr = e / SBP_T, tt = e % SBP_T, t = t0 + tt;
            const int f = reflect_idx(min(f0 + rr - a.Nf, F - 1 + a.Nf), F);
            fsm[(q * frows + rr) * (SBP_T + 1) + tt] = (t < Tpe) ? src[((size_t)b * F + f) * a.P + t] : 0.f;
        }
    }
    __syncthreads();
    // work item (bin fr of the tile, chunk c of 8 channels)
    auto pack_bin = [&](int fr, int c) {
        const int f = f0 + fr;
        const bool live = f < fb + Fn;
        const int row = b * Fn + (f - fb);
        auto val = [&](int k, int tt) -> float {
            float v = 0.f;
            if (k < nw) v = wsm[(fr + k) * (SBP_T + 1) + tt];
            else if (k < I) { const int kk = k - nw, q = kk / nf, j = kk % nf; v = fsm[(q * frows + fr + j) * (SBP_T + 1) + tt]; }
            return (k < I && t0 + tt < Tpe) ? (v - sub) * inv : 0.f;
        };
        float m = 0.f;
        for (int tt = 0; live && tt < SBP_T && t0 + tt < Tp; ++tt) {
            float v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = val(c * 8 + i, tt);
            m = vmax8(m, v);
            Store::store(a, row, t0 + tt, c * 8, v);
        }
        Store::finish(a, live ? row : -1, m, 8);
    };
    if (Store::kWidth == 64) {
        pack_bin(threadIdx.x >> 3, threadIdx.x & 7);
    } else {                                                        // 16 chunks per row: two passes of 16 bins
        pack_bin(threadIdx.x >> 4, threadIdx.x & 15);
        pack_bin((threadIdx.x >> 4) + 16, threadIdx.x & 15);
    }
}

// Cumulative norms of the 4-D sub-band input (base_model.py:227-258 / :277-316 with dim 1 = F folded into the batch): every
// sequence (b, f) is normalised by the running mean (and std) over its I channels.  One warp per sequence, lanes over
// frames, warp scan with carry.  Rows of 128 channels (Fp16Wide) hold 64 values per thread as the 64-wide rows do: the first half's
// values enter the sums, the second half's are kept, and the first half is read again for its stores.
template <class Store>
__global__ void __launch_bounds__(128) sb_pack_cum_kernel(SbPackLaunch a) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int fb = Store::kChunk ? a.f0 : 0, Fn = Store::kChunk ? a.Fc : a.F;   // bins fb .. fb + Fn - 1
    const int row = blockIdx.x * 4 + warp, F = a.F, Tp = a.t0 + a.Tw;   // Tp: the window's end
    if (row >= a.B * Fn) return;
    // f < F always: the unsigned modulo changes no value, it tells the compiler f's range (without it, it keeps 64 neighbour addresses
    // live across the frame loop and spills)
    const int b = row / Fn, f = (int)((unsigned)(fb + row % Fn) % (unsigned)F);
    const int Tpe = a.tlen ? a.tlen[b] : a.Tp;                     // frames t >= Tpe are past this sample's end: written as zero
    const int nw = 2 * a.Ns + 1, nf = 2 * a.Nf + 1, I = nw + a.nfb * nf;
    const double EPS = 1.1920928955078125e-07;
    double cs = 0.0, cq = 0.0;                                   // running sums carried across 32-frame chunks (and windows: a.cum)
    if (a.cum && a.t0 > 0) { cs = a.cum[2 * (size_t)row]; cq = a.cum[2 * (size_t)row + 1]; }
    float mx = 0.f;
    constexpr int K0 = Store::kWidth - 64;                        // the first channel held in v
    for (int t0 = a.t0; t0 < Tp; t0 += 32) {
        const int t = t0 + lane;
        auto load = [&](int k) -> float {                         // channel k of (sequence, frame t)
            float x = 0.f;
            if (t < Tpe && k < I) {
                if (k < nw) x = a.win[((size_t)b * F + reflect_idx(f + k - a.Ns, F)) * a.Pw + t];
                else {
                    const int kk = k - nw, qq = kk / nf, j = kk % nf;
                    const float* src = (qq == 0) ? a.fb[0] : (qq == 1) ? a.fb[1] : a.fb[2];
                    x = src[((size_t)b * F + reflect_idx(f + j - a.Nf, F)) * a.P + t];
                }
            }
            return x;
        };
        float v[64];
        float s = 0.f, q = 0.f;
        if (K0) {
#pragma unroll
            for (int k = 0; k < K0; ++k) { const float x = load(k); s += x; q = fmaf(x, x, q); }
        }
#pragma unroll
        for (int k = 0; k < 64; ++k) {
            const float x = load(K0 + k);
            v[k] = x; s += x; q = fmaf(x, x, q);
        }
        double ds = s, dq = q;                                   // inclusive scan over the 32 frames of this chunk
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double us = __shfl_up_sync(0xffffffffu, ds, o), uq = __shfl_up_sync(0xffffffffu, dq, o);
            if (lane >= o) { ds += us; dq += uq; }
        }
        ds += cs; dq += cq;
        const double cnt = (double)I * (t + 1), cm = ds / cnt;
        float sc, sh;
        if (a.norm_type == FSN_NORM_CUMULATIVE_LAPLACE) { sc = (float)(1.0 / (cm + EPS)); sh = 0.f; }
        else { const double cv = (dq - 2.0 * cm * ds) / cnt + cm * cm; const double inv = 1.0 / sqrt(cv + EPS); sc = (float)inv; sh = (float)(-cm * inv); }
        cs = __shfl_sync(0xffffffffu, ds, 31); cq = __shfl_sync(0xffffffffu, dq, 31);
        if (t < Tp) {
            if (K0) {
#pragma unroll 1
                for (int c = 0; c < K0 / 8; ++c) {
                    float w[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) w[i] = (c * 8 + i < I && t < Tpe) ? fmaf(load(c * 8 + i), sc, sh) : 0.f;
                    mx = vmax8(mx, w);
                    Store::store(a, row, t, c * 8, w);
                }
            }
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                float w[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) w[i] = (K0 + c * 8 + i < I && t < Tpe) ? fmaf(v[c * 8 + i], sc, sh) : 0.f;
                mx = vmax8(mx, w);
                Store::store(a, row, t, K0 + c * 8, w);
            }
        }
    }
    if (a.cum && lane == 0) { a.cum[2 * (size_t)row] = cs; a.cum[2 * (size_t)row + 1] = cq; }
    Store::finish(a, row, mx, 32);
}

// The launchers of the packers return the name of the kernel whose launch failed (and its error in *err), or null
template <class Store>
static const char* sb_pack_go(const SbPackLaunch& a, cudaStream_t s, cudaError_t* err) {
    const int Fn = Store::kChunk ? a.Fc : a.F;
    if (a.norm_type == FSN_NORM_CUMULATIVE_LAPLACE || a.norm_type == FSN_NORM_CUMULATIVE_LAYER) {
        sb_pack_cum_kernel<Store><<<(a.B * Fn + 3) / 4, 128, 0, s>>>(a);
        return (*err = cudaGetLastError()) ? "sb_pack_cum_kernel" : nullptr;
    }
    const size_t smem = sizeof(float) * (SBP_T + 1) * ((SBP_F + 2 * a.Ns) + a.nfb * (SBP_F + 2 * a.Nf));
    if ((*err = cudaFuncSetAttribute(sb_pack_kernel<Store>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem))) return "sb_pack_kernel";
    sb_pack_kernel<Store><<<dim3((a.Tw + SBP_T - 1) / SBP_T, (Fn + SBP_F - 1) / SBP_F, a.B), 256, smem, s>>>(a);
    return (*err = cudaGetLastError()) ? "sb_pack_kernel" : nullptr;
}
// The raw form (SbPackLaunch::raw): one thread per (row, frame, 8 channels), 8 consecutive threads write one row of a step's image
// (Store = Fp16Img; 16 threads per row of Fp16Wide)
template <class Store>
__global__ void __launch_bounds__(256) sb_pack_raw_kernel(SbPackLaunch a) {
    constexpr int NC = Store::kWidth / 8, LNC = NC == 8 ? 3 : 4;
    const int I = 2 * a.Ns + 1 + a.nfb * (2 * a.Nf + 1), rows = a.B * a.F;
    const long long n = (long long)((rows + 255) / 256 * 2) * a.Tw * 128 * NC;    // every row of the padded tile pairs
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i & (NC - 1)), r = (int)((i >> LNC) & 127);
        const long long q = i >> (LNC + 7);
        const int row = (int)(q / a.Tw) * 128 + r, t = a.t0 + (int)(q % a.Tw);
        float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (row < rows && t < (a.tlen ? a.tlen[row / a.F] : a.Tp))
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (c * 8 + e < I) v[e] = a.raw[((size_t)row * I + c * 8 + e) * a.Tp + t];
        // the time-major rows stop at ntiles * 128: the pad tile of a pair is not part of the generic kernel's input
        if (!Store::kTimeMajor || row < a.ntiles * 128) Store::store(a, row, t, c * 8, v);
    }
}

template <class Store>
static const char* sb_pack_any(const SbPackLaunch& a, cudaStream_t s, cudaError_t* err) {
    if (!a.raw) return sb_pack_go<Store>(a, s, err);
    sb_pack_raw_kernel<Store><<<1024, 256, 0, s>>>(a);
    return (*err = cudaGetLastError()) ? "sb_pack_raw_kernel" : nullptr;
}
const char* launch_sb_pack(const SbPackLaunch& a, cudaStream_t s, cudaError_t* err) { return sb_pack_any<Fp16Img>(a, s, err); }
const char* launch_sb_pack_wide(const SbPackLaunch& a, bool time_major, cudaStream_t s, cudaError_t* err) {
    return time_major ? sb_pack_any<Fp16Wide<true>>(a, s, err) : sb_pack_any<Fp16Wide<false>>(a, s, err);
}
const char* launch_sb_pack_tm(const SbPackLaunch& a, cudaStream_t s, cudaError_t* err) {
    if ((*err = cudaMemsetAsync(a.amax, 0, (size_t)a.B * a.Fc * sizeof(float), s))) return "cudaMemsetAsync of the sub-band TCN's maxima";
    return sb_pack_go<Fp32Tm>(a, s, err);
}

__global__ void tm_to_fm_kernel(const float* x, int ld, float* y, int Z, int C, int Tp) {
    const size_t n = (size_t)Z * C * Tp;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t t = i % Tp, c = (i / Tp) % C, z = i / ((size_t)Tp * C);
        y[i] = x[(z * Tp + t) * ld + c];
    }
}
void launch_tm_to_fm(const float* x, int ld, float* y, int Z, int C, int Tp, cudaStream_t s) {
    tm_to_fm_kernel<<<1024, 256, 0, s>>>(x, ld, y, Z, C, Tp);
}



// =============================================================================================
// Streaming forms of the cumulative norms: the running sums live in global memory (fp64) and one launch handles K frames of every
// slot, frame after frame, with the same reduction order and running sums for each frame -- so one launch over K frames writes the
// bits K launches of one frame write.  reference: base_model.py:227-258 / :277-316 evaluated one column at a time.
// Frame k of slot b is its frame n0 + k, n0 = slot[b] (or n when slot is null).
// =============================================================================================
__global__ void __launch_bounds__(256) stream_norm_kernel(StreamNormLaunch a) {
    __shared__ double red[16];
    __shared__ float s_a, s_b;
    const int b = blockIdx.x, F = a.F, n0 = a.slot ? a.slot[b] : a.n;
    if (n0 < 0) {                                                   // held: frames unread, sums untouched, zero rows
        for (int i = threadIdx.x; i < F * a.K; i += blockDim.x) a.y[((size_t)b * F + i / a.K) * a.P + i % a.K] = 0.f;
        return;
    }
    const float* x = a.x + (size_t)b * F * a.K;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, kb = a.kf ? a.kf[b] : a.K;
    for (int i = threadIdx.x; i < F * (a.K - kb); i += blockDim.x)  // frames past the slot's count: zero
        a.y[((size_t)b * F + i / (a.K - kb)) * a.P + kb + i % (a.K - kb)] = 0.f;
    double cs = n0 == 0 ? 0.0 : a.cum[2 * b], cq = n0 == 0 ? 0.0 : a.cum[2 * b + 1];   // thread 0's running sums
#pragma unroll 1
    for (int k = 0; k < kb; ++k) {
        const int n = n0 + k;
        double s = 0, q = 0;
        for (int f = threadIdx.x; f < F; f += blockDim.x) { const double v = x[(size_t)f * a.K + k]; s += v; q += v * v; }
        s = warp_sum_d(s); q = warp_sum_d(q);
        if (lane == 0) { red[warp] = s; red[8 + warp] = q; }
        __syncthreads();
        if (threadIdx.x == 0) {
            double ts = 0, tq = 0;
            for (int i = 0; i < 8; ++i) { ts += red[i]; tq += red[8 + i]; }
            const double EPS = 1.1920928955078125e-07;
            cs += ts; cq += tq;
            const double cnt = (double)F * (n + 1), cm = cs / cnt;
            if (a.type == FSN_NORM_CUMULATIVE_LAPLACE) { s_a = (float)(1.0 / (cm + EPS)); s_b = 0.f; }
            else { const double cv = (cq - 2.0 * cm * cs) / cnt + cm * cm, inv = 1.0 / sqrt(cv + EPS); s_a = (float)inv; s_b = (float)(-cm * inv); }
        }
        __syncthreads();
        for (int f = threadIdx.x; f < F; f += blockDim.x) a.y[((size_t)b * F + f) * a.P + k] = fmaf(x[(size_t)f * a.K + k], s_a, s_b);
        __syncthreads();                                            // red, s_a and s_b are reused by the next frame
    }
    if (threadIdx.x == 0) { a.cum[2 * b] = cs; a.cum[2 * b + 1] = cq; }
}
void launch_stream_norm(const StreamNormLaunch& a, cudaStream_t s) { stream_norm_kernel<<<a.B, 256, 0, s>>>(a); }

// thread = sequence (b, f); frames k0 .. k0 + Kw - 1 of the chunk into the window-local images [tile, Kw, 128, 64]
__global__ void __launch_bounds__(128) stream_pack_kernel(StreamPackLaunch a) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x, F = a.F;
    if (row >= a.B * F) return;
    const int b = row / F, f = row % F;
    const int nw = 2 * a.Ns + 1, nf = 2 * a.Nf + 1, I = nw + nf;
    const int n0 = a.slot ? a.slot[b] : a.n;
    int crow = row;                                                 // the row of the images
    if (a.idx) {                                                    // compact rows: session idx[b] - j0 of this sub-batch, or not packed
        const int j = n0 < 0 ? -1 : a.idx[b] - a.j0;
        if (j < 0 || j >= a.nsess) return;
        crow = j * F + f;
    }
    const int tile = crow >> 7, r = crow & 127;
    char* img = reinterpret_cast<char*>(a.ximg) + (size_t)tile * a.Kw * (128 * 128);
    if (n0 < 0) {                                                   // held: frames unread, sums untouched, zero input rows
        for (int k = 0; k < a.Kw; ++k)
#pragma unroll
            for (int c = 0; c < 8; ++c) *reinterpret_cast<uint4*>(img + (size_t)k * (128 * 128) + sw128_offset(r, c * 8)) = make_uint4(0u, 0u, 0u, 0u);
        return;
    }
    const float* mag = a.mag + (size_t)b * F * a.K;
    const float* fb = a.fb + (size_t)b * F * a.Pfb;
    double cs = n0 + a.k0 == 0 ? 0.0 : a.cum[2 * row], cq = n0 + a.k0 == 0 ? 0.0 : a.cum[2 * row + 1];
    const int kb = a.kf ? a.kf[b] : a.K;
#pragma unroll 1
    for (int kk = 0; kk < a.Kw; ++kk) {
        const int k = a.k0 + kk, n = n0 + k;
        if (k >= kb) {                                              // past the slot's frames: zero input rows, sums untouched
#pragma unroll
            for (int c = 0; c < 8; ++c) *reinterpret_cast<uint4*>(img + (size_t)kk * (128 * 128) + sw128_offset(r, c * 8)) = make_uint4(0u, 0u, 0u, 0u);
            continue;
        }
        int fo = f;                                                 // opaque per frame: the 64 neighbour offsets are recomputed, not
        asm volatile("" : "+r"(fo));                                // hoisted out of the frame loop (which spills them)
        float v[64];
        double s = 0, q = 0;
#pragma unroll
        for (int i = 0; i < 64; ++i) {
            float x = 0.f;
            if (i < nw) x = mag[(size_t)reflect_idx(fo + i - a.Ns, F) * a.K + k];
            else if (i < I) x = fb[(size_t)reflect_idx(fo + (i - nw) - a.Nf, F) * a.Pfb + k];
            v[i] = x; s += x; q += (double)x * x;
        }
        const double EPS = 1.1920928955078125e-07;
        cs += s; cq += q;
        const double cnt = (double)I * (n + 1), cm = cs / cnt;
        float sc, sh;
        if (a.type == FSN_NORM_CUMULATIVE_LAPLACE) { sc = (float)(1.0 / (cm + EPS)); sh = 0.f; }
        else { const double cv = (cq - 2.0 * cm * cs) / cnt + cm * cm, inv = 1.0 / sqrt(cv + EPS); sc = (float)inv; sh = (float)(-cm * inv); }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float w[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) w[i] = (c * 8 + i < I) ? fminf(fmaxf(fmaf(v[c * 8 + i], sc, sh), -65504.f), 65504.f) : 0.f;
            *reinterpret_cast<uint4*>(img + (size_t)kk * (128 * 128) + sw128_offset(r, c * 8)) =
                make_uint4(pack_half2(w[0], w[1]), pack_half2(w[2], w[3]), pack_half2(w[4], w[5]), pack_half2(w[6], w[7]));
        }
    }
    a.cum[2 * row] = cs; a.cum[2 * row + 1] = cq;
}
// The same for one frame (K = 1, no compact rows): the arithmetic above without the frame loop, in 96 registers instead of 120; at
// 1024 slots it runs 49 us per tick where the K-frame kernel at K = 1 takes 55 us (H100 80GB HBM3, 700 W; DESIGN.md §4)
__global__ void __launch_bounds__(128) stream_pack_frame_kernel(StreamPackLaunch a) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x, F = a.F;
    if (row >= a.B * F) return;
    const int b = row / F, f = row % F, tile = row >> 7, r = row & 127;
    const int nw = 2 * a.Ns + 1, nf = 2 * a.Nf + 1, I = nw + nf;
    char* img = reinterpret_cast<char*>(a.ximg) + (size_t)tile * (128 * 128);
    const int n = a.slot ? a.slot[b] : a.n;                         // the frame count of this row's slot
    if (n < 0) {                                                    // held: frame unread, sums untouched, zero input row
#pragma unroll
        for (int c = 0; c < 8; ++c) *reinterpret_cast<uint4*>(img + sw128_offset(r, c * 8)) = make_uint4(0u, 0u, 0u, 0u);
        return;
    }
    float v[64];
    double s = 0, q = 0;
#pragma unroll
    for (int k = 0; k < 64; ++k) {
        float x = 0.f;
        if (k < nw) x = a.mag[(size_t)b * F + reflect_idx(f + k - a.Ns, F)];
        else if (k < I) x = a.fb[((size_t)b * F + reflect_idx(f + (k - nw) - a.Nf, F)) * a.Pfb];
        v[k] = x; s += x; q += (double)x * x;
    }
    const double EPS = 1.1920928955078125e-07;
    const double cs = (n == 0 ? 0.0 : a.cum[2 * row]) + s, cq = (n == 0 ? 0.0 : a.cum[2 * row + 1]) + q;
    a.cum[2 * row] = cs; a.cum[2 * row + 1] = cq;
    const double cnt = (double)I * (n + 1), cm = cs / cnt;
    float sc, sh;
    if (a.type == FSN_NORM_CUMULATIVE_LAPLACE) { sc = (float)(1.0 / (cm + EPS)); sh = 0.f; }
    else { const double cv = (cq - 2.0 * cm * cs) / cnt + cm * cm, inv = 1.0 / sqrt(cv + EPS); sc = (float)inv; sh = (float)(-cm * inv); }
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        float w[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) w[i] = (c * 8 + i < I) ? fminf(fmaxf(fmaf(v[c * 8 + i], sc, sh), -65504.f), 65504.f) : 0.f;
        *reinterpret_cast<uint4*>(img + sw128_offset(r, c * 8)) =
            make_uint4(pack_half2(w[0], w[1]), pack_half2(w[2], w[3]), pack_half2(w[4], w[5]), pack_half2(w[6], w[7]));
    }
}

// The wide form (64 < I <= 128) of both kernels above, one launch for K frames: plain rows of 128 halves, in the order of layer 0's
// input-projection GEMM with compact rows (idx: row (tile * Kw + kk) * 128 + r), else time-major [Kw, ntiles * 128, 128] for the
// generic kernel.  A thread holds 64 values at a time: the first half's enter the sums, the second half's are kept, and the first
// half is read again for its stores (same sums, same order as one pass over 128).
__global__ void __launch_bounds__(128) stream_pack_wide_kernel(StreamPackLaunch a) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x, F = a.F;
    if (row >= a.B * F) return;
    const int b = row / F, f = row % F;
    const int nw = 2 * a.Ns + 1, nf = 2 * a.Nf + 1, I = nw + nf;
    const int n0 = a.slot ? a.slot[b] : a.n;
    int crow = row;                                                 // the row of the images
    if (a.idx) {                                                    // compact rows: session idx[b] - j0 of this sub-batch, or not packed
        const int j = n0 < 0 ? -1 : a.idx[b] - a.j0;
        if (j < 0 || j >= a.nsess) return;
        crow = j * F + f;
    }
    const int ntiles = (a.B * F + 127) / 128;
    auto dst = [&](int kk) { return a.ximg + wide_row(a.idx == nullptr, crow, kk, 0, a.Kw, ntiles) * 128; };
    auto zero_row = [&](int kk) {
        uint4* d = reinterpret_cast<uint4*>(dst(kk));
#pragma unroll
        for (int c = 0; c < 16; ++c) d[c] = make_uint4(0u, 0u, 0u, 0u);
    };
    if (n0 < 0) {                                                   // held: frames unread, sums untouched, zero input rows
        for (int k = 0; k < a.Kw; ++k) zero_row(k);
        return;
    }
    const float* mag = a.mag + (size_t)b * F * a.K;
    const float* fb = a.fb + (size_t)b * F * a.Pfb;
    double cs = n0 + a.k0 == 0 ? 0.0 : a.cum[2 * row], cq = n0 + a.k0 == 0 ? 0.0 : a.cum[2 * row + 1];
    const int kb = a.kf ? a.kf[b] : a.K;
#pragma unroll 1
    for (int kk = 0; kk < a.Kw; ++kk) {
        const int k = a.k0 + kk, n = n0 + k;
        if (k >= kb) { zero_row(kk); continue; }                    // past the slot's frames: zero input rows, sums untouched
        int fo = f;                                                 // opaque per frame: the neighbour offsets are recomputed, not
        asm volatile("" : "+r"(fo));                                // hoisted out of the frame loop
        auto load = [&](int i) -> float {
            float x = 0.f;
            if (i < nw) x = mag[(size_t)reflect_idx(fo + i - a.Ns, F) * a.K + k];
            else if (i < I) x = fb[(size_t)reflect_idx(fo + (i - nw) - a.Nf, F) * a.Pfb + k];
            return x;
        };
        float v[64];
        double s = 0, q = 0;
#pragma unroll
        for (int i = 0; i < 64; ++i) { const float x = load(i); s += x; q += (double)x * x; }
#pragma unroll
        for (int i = 0; i < 64; ++i) { const float x = load(64 + i); v[i] = x; s += x; q += (double)x * x; }
        const double EPS = 1.1920928955078125e-07;
        cs += s; cq += q;
        const double cnt = (double)I * (n + 1), cm = cs / cnt;
        float sc, sh;
        if (a.type == FSN_NORM_CUMULATIVE_LAPLACE) { sc = (float)(1.0 / (cm + EPS)); sh = 0.f; }
        else { const double cv = (cq - 2.0 * cm * cs) / cnt + cm * cm, inv = 1.0 / sqrt(cv + EPS); sc = (float)inv; sh = (float)(-cm * inv); }
        uint4* d = reinterpret_cast<uint4*>(dst(kk));
        auto store64 = [&](int k0) {                                // channels k0 .. k0 + 63 from v
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                float w[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) w[i] = (k0 + c * 8 + i < I) ? fmaf(v[c * 8 + i], sc, sh) : 0.f;
                d[k0 / 8 + c] = pack_half8(w);
            }
        };
        store64(64);
        asm volatile("" : "+r"(fo));
#pragma unroll
        for (int i = 0; i < 64; ++i) v[i] = load(i);
        store64(0);
    }
    a.cum[2 * row] = cs; a.cum[2 * row + 1] = cq;
}

void launch_stream_pack(const StreamPackLaunch& a, cudaStream_t s) {
    if (a.K == 1 && !a.idx) stream_pack_frame_kernel<<<(a.B * a.F + 127) / 128, 128, 0, s>>>(a);
    else stream_pack_kernel<<<(a.B * a.F + 127) / 128, 128, 0, s>>>(a);
}
void launch_stream_pack_wide(const StreamPackLaunch& a, cudaStream_t s) {
    stream_pack_wide_kernel<<<(a.B * a.F + 127) / 128, 128, 0, s>>>(a);
}

// The compact masks of one sub-batch [nsess, 2, F, K] into the slots' rows of d_mask [B, 2, F, K]: column k of slot b is the mask of
// its frame slot[b] + k - la, zero while that index is negative.  zero_held: also write the rows of held slots as zeros.
__global__ void stream_chunk_scatter_kernel(StreamChunkScatterLaunch a) {
    const size_t plane = (size_t)2 * a.F * a.K, n = (size_t)a.B * plane;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / plane), k = (int)(i % a.K), n0 = a.slot[b];
        if (n0 < 0) {
            if (a.zero_held) a.dst[i] = 0.f;
            continue;
        }
        const int j = a.idx[b] - a.j0;
        if (j < 0 || j >= a.nsess) continue;
        const size_t e = i % plane;                                 // (o, f, k) of the dst plane
        a.dst[i] = (n0 + k < a.la || k >= a.Ks) ? 0.f : a.src[(size_t)j * 2 * a.F * a.Ks + e / a.K * a.Ks + k];
    }
}
void launch_stream_chunk_scatter(const StreamChunkScatterLaunch& a, cudaStream_t s) {
    const size_t n = (size_t)a.B * 2 * a.F * a.K;
    size_t blocks = (n + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    stream_chunk_scatter_kernel<<<(unsigned)blocks, 256, 0, s>>>(a);
}

// decompress_cIRM + complex multiply (inferencer.py:152-157, mask.py:60-63) in one pass.
__global__ void apply_cirm_kernel(const float* crm, const float2* noisy, float2* enh, int FT, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t b = i / FT, e = i % FT;
    float m[2];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        float v = crm[(b * 2 + c) * FT + e];
        v = (v >= 9.9f) ? 9.9f : ((v <= -9.9f) ? -9.9f : v);           // limit * (m >= limit) - limit * (m <= -limit) + m * (|m| < limit)
        m[c] = -10.f * logf((10.f - v) / (10.f + v));
    }
    const float2 x = noisy[i];
    enh[i] = make_float2(m[0] * x.x - m[1] * x.y, m[1] * x.x + m[0] * x.y);
}
// LIM: each clip's attenuation floor lam[b] (limit_mask); the instantiation without it is the pass as it was before limits existed
template <bool LIM>
__global__ void apply_cirm_planar_kernel(const float* crm, const float* nreal, const float* nimag, float2* enh, int T, int FT, size_t n,
                                         const int* tlen, int la, const float* lam) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t b = i / FT, e = i % FT;
    if (tlen && (int)(e % T) >= tlen[b] - la) { enh[i] = make_float2(0.f, 0.f); return; }   // past the clip: the planes are not read
    float m0 = decompress_cirm(crm[(b * 2 + 0) * FT + e]), m1 = decompress_cirm(crm[(b * 2 + 1) * FT + e]);
    if (LIM) limit_mask(m0, m1, __ldg(lam + b));
    const float xr = nreal[i], xi = nimag[i];
    enh[i] = make_float2(m0 * xr - m1 * xi, m1 * xr + m0 * xi);
}
void launch_apply_cirm_planar(const float* crm, const float* nreal, const float* nimag, float2* enh, int B, int F, int T, const int* tlen,
                              int la, cudaStream_t s, const float* lam) {
    const size_t n = (size_t)B * F * T;
    if (lam) apply_cirm_planar_kernel<true><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(crm, nreal, nimag, enh, T, F * T, n, tlen, la, lam);
    else apply_cirm_planar_kernel<false><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(crm, nreal, nimag, enh, T, F * T, n, tlen, la, lam);
}
void launch_apply_cirm(const float* crm, const float2* noisy, float2* enh, int B, int F, int T, cudaStream_t s) {
    const size_t n = (size_t)B * F * T;
    apply_cirm_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(crm, noisy, enh, F * T, n);
}

__global__ void pad_copy_kernel(const float* x, float* y, int rows, int F, int T, int P, const int* tlen, int la) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)rows * P) return;
    int t = (int)(i % P);
    size_t r = i / P;
    const int Te = tlen ? tlen[r / F] - la : T;                   // frames of this sample's input
    y[i] = (t < Te) ? x[r * T + t] : 0.f;
}
void launch_pad_copy(const float* x, float* y, int B, int F, int T, int P, const int* tlen, int la, cudaStream_t s) {
    size_t n = (size_t)B * F * P;
    pad_copy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(x, y, B * F, F, T, P, tlen, la);
}

__global__ void fb_pack_kernel(const float* x, __half* y, int B, int F, int Tp, int P, int rows_pad, int Ipad) {
    // y[t][b][k] = x[b][k][t]
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)Tp * rows_pad * Ipad) return;
    int k = (int)(i % Ipad);
    int b = (int)((i / Ipad) % rows_pad);
    int t = (int)(i / ((size_t)Ipad * rows_pad));
    float v = (b < B && k < F) ? x[((size_t)b * F + k) * P + t] : 0.f;
    y[i] = __float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f));
}
void launch_fb_pack(const float* x, __half* y, int B, int F, int Tp, int P, int rows_pad, int Ipad, cudaStream_t s) {
    size_t n = (size_t)Tp * rows_pad * Ipad;
    fb_pack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(x, y, B, F, Tp, P, rows_pad, Ipad);
}

}  // namespace fsn
