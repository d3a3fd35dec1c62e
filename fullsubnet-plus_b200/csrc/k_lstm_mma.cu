// Generic persistent stacked-LSTM kernel (legacy tensor path, mma.sync m16n8k16 fp16 -> fp32).
//
// One CTA owns R sequences (rows) for ALL time steps and ALL layers: hidden state stays in shared
// memory (fp16, double buffered per layer), cell state in an fp32 scratch that only this CTA touches
// (L2 resident), weights are streamed from L2 in mma-fragment order.  Any hidden size that is a
// multiple of 16 and up to 4 layers are supported, which makes this the kernel behind
//   * the full-band LSTM of fullsubnet.Model           (reference fullsubnet.py:39-47,86-87)
//   * sub-band LSTMs outside the layer-wise wgmma kernel's envelope (hidden not a multiple of 64 or > 512, output_size != 2),
//     lstm_impl = "mma" and the streaming sub-band step
// LSTM cell definition: nn.LSTM as used at audio_zen/model/module/sequence_model.py:32-38,118
// (gate rows i,f,g,o; c = s(f)c + s(i)tanh(g); h = s(o)tanh(c); zero initial state).
#include "fsn_common.cuh"
#include "fsn_kernels.h"
#include "../../include/fsnplus_b200.h"

namespace fsn {

struct MmaSmemPlan { int HS, XS; size_t hb_bytes, xs_bytes, fc_bytes, total; };

static inline MmaSmemPlan mma_plan(int L, int H, int Ipad, int R, int O) {
    MmaSmemPlan p;
    p.HS = H + 8; p.XS = Ipad + 8;
    p.hb_bytes = (size_t)L * 2 * R * p.HS * 2;
    p.xs_bytes = (size_t)R * p.XS * 2;
    p.fc_bytes = (size_t)O * H * 4;
    p.total = p.hb_bytes + p.xs_bytes + p.fc_bytes;
    return p;
}

template <int R, bool FAST>
__global__ void __launch_bounds__(256, 1) lstm_mma_kernel(LstmMmaLaunch a) {
    constexpr int MT = R / 16;
    extern __shared__ __align__(16) unsigned char smraw[];
    const int L = a.L, H = a.H, Ipad = a.Ipad, Tp = a.Tp;
    const int HS = H + 8, XS = Ipad + 8;
    __half* hb = reinterpret_cast<__half*>(smraw);                       // [L][2][R][HS]
    __half* xs = hb + (size_t)L * 2 * R * HS;                            // [R][XS]
    float* fcw = reinterpret_cast<float*>(xs + (size_t)R * XS);          // [O][H]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int row0 = blockIdx.x * R;
    const int ngroups = H / 8;

    for (int i = tid; i < (int)((size_t)L * 2 * R * HS / 2); i += blockDim.x) reinterpret_cast<uint32_t*>(hb)[i] = 0u;
    if (a.hstate && a.resume) {                          // streaming: h_{-1} of every layer goes into the "previous" buffer (index 1 at t = 0)
        __syncthreads();
        for (int e = tid; e < L * R * (H / 2); e += blockDim.x) {
            const int l = e / (R * (H / 2)), r = (e / (H / 2)) % R, u2 = e % (H / 2);
            reinterpret_cast<uint32_t*>(hb + ((size_t)l * 2 + 1) * R * HS + (size_t)r * HS)[u2] =
                reinterpret_cast<const uint32_t*>(a.hstate + ((size_t)l * a.rows_alloc + row0 + r) * H)[u2];
        }
    }
    if (a.out) for (int i = tid; i < a.O * H; i += blockDim.x) fcw[i] = a.w.fc_w[i];
    __syncthreads();

    for (int t = 0; t < Tp; ++t) {
        const int p = t & 1;
        // ---- stage x_t rows ------------------------------------------------------------------
        {
            const int cpr = Ipad / 8;                                    // 16-byte chunks per row
            for (int e = tid; e < R * cpr; e += blockDim.x) {
                const int r = e / cpr, c = e % cpr;
                uint4 v;
                if (a.img) {
                    const int grow = row0 + r, tile = grow >> 7, rr = grow & 127;
                    const char* src = reinterpret_cast<const char*>(a.img) + ((size_t)tile * Tp + t) * 16384 + sw128_offset(rr, c * 8);
                    v = __ldg(reinterpret_cast<const uint4*>(src));
                } else {
                    v = __ldg(reinterpret_cast<const uint4*>(a.xplain + ((size_t)t * a.rows_pad + row0 + r) * Ipad + c * 8));
                }
                *reinterpret_cast<uint4*>(xs + (size_t)r * XS + c * 8) = v;
            }
        }
        __syncthreads();

        for (int l = 0; l < L; ++l) {
            const __half* seg0 = (l == 0) ? xs : hb + ((size_t)(l - 1) * 2 + p) * R * HS;
            const int st0 = (l == 0) ? XS : HS, ks0 = ((l == 0) ? Ipad : H) / 16;
            const __half* seg1 = hb + ((size_t)l * 2 + (p ^ 1)) * R * HS;
            const int ks1 = H / 16, ksteps = ks0 + ks1;
            __half* hout = hb + ((size_t)l * 2 + p) * R * HS;
            const uint4* wf = a.w.wfrag[l];
            const float* bias = a.w.bias[l];
            float* cst = a.cstate + (size_t)l * a.rows_alloc * H;
            const bool top = (l == L - 1);

            for (int g = warp; g < ngroups; g += 8) {
                float acc[MT][4][4];
#pragma unroll
                for (int i = 0; i < MT; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j)
#pragma unroll
                        for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;
                const uint4* wg = wf + ((size_t)g * ksteps) * 64 + lane * 2;
#pragma unroll 2
                for (int ks = 0; ks < ksteps; ++ks) {
                    const uint4 w0 = __ldg(wg + (size_t)ks * 64), w1 = __ldg(wg + (size_t)ks * 64 + 1);
                    const __half* seg = (ks < ks0) ? seg0 : seg1;
                    const int st = (ks < ks0) ? st0 : HS, kk = ((ks < ks0) ? ks : ks - ks0) * 16;
#pragma unroll
                    for (int mt = 0; mt < MT; ++mt) {
                        uint32_t af[4];
                        ldmatrix_x4(af, smem_u32(seg + (size_t)(mt * 16 + (lane & 15)) * st + kk + (lane >> 4) * 8));
                        mma_f16_16816(acc[mt][0], af, w0.x, w0.y);
                        mma_f16_16816(acc[mt][1], af, w0.z, w0.w);
                        mma_f16_16816(acc[mt][2], af, w1.x, w1.y);
                        mma_f16_16816(acc[mt][3], af, w1.z, w1.w);
                    }
                }
                // ---- cell update for this group of 8 hidden units -----------------------------
#pragma unroll
                for (int mt = 0; mt < MT; ++mt)
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int r = mt * 16 + (lane >> 2) + ((q & 2) ? 8 : 0);
                        const int u = g * 8 + 2 * (lane & 3) + (q & 1);
                        const size_t ci = (size_t)(row0 + r) * H + u;
                        const float gi = acc[mt][0][q] + bias[u], gf = acc[mt][1][q] + bias[H + u];
                        const float gg = acc[mt][2][q] + bias[2 * H + u], go = acc[mt][3][q] + bias[3 * H + u];
                        const float cprev = (t == 0 && !a.resume) ? 0.f : cst[ci];
                        float c, h;
                        if (a.gru) { h = gru_cell_plain<FAST>(gi, gf, gg, go, cprev); c = h; }
                        else { c = sigm<FAST>(gf) * cprev + sigm<FAST>(gi) * tanh_<FAST>(gg); h = sigm<FAST>(go) * tanh_<FAST>(c); }
                        cst[ci] = c;
                        hout[(size_t)r * HS + u] = __float2half_rn(h);
                        if (top && a.hseq && row0 + r < a.rows) a.hseq[((size_t)(row0 + r) * H + u) * a.P + t] = h;
                    }
            }
            __syncthreads();
        }
        // ---- fused output layer (sequence_model.py:119-121) and [B, O, F, T] layout (fullsubnet_plus.py:206-208)
        if (a.out && t >= a.la) {
            const __half* htop = hb + ((size_t)(L - 1) * 2 + p) * R * HS;
            for (int e = tid; e < R * a.O; e += blockDim.x) {
                const int r = e / a.O, o = e % a.O, grow = row0 + r;
                if (grow >= a.rows) continue;
                const int b = grow / a.F, f = grow % a.F;
                if (a.tlen && t >= a.tlen[b]) { a.out[(((size_t)b * a.O + o) * a.F + f) * (Tp - a.la) + (t - a.la)] = 0.f; continue; }   // past the clip's end
                float acc = a.w.fc_b[o];
                const __half2* hr = reinterpret_cast<const __half2*>(htop + (size_t)r * HS);
                const float* w = fcw + (size_t)o * H;
                for (int u = 0; u < H / 2; ++u) {
                    const float2 hv = __half22float2(hr[u]);
                    acc = fmaf(hv.x, w[2 * u], acc);
                    acc = fmaf(hv.y, w[2 * u + 1], acc);
                }
                if (a.act == FSN_ACT_RELU) acc = fmaxf(acc, 0.f);
                else if (a.act == FSN_ACT_TANH) acc = tanhf(acc);
                else if (a.act == FSN_ACT_RELU6) acc = fminf(fmaxf(acc, 0.f), 6.f);
                a.out[(((size_t)b * a.O + o) * a.F + f) * (Tp - a.la) + (t - a.la)] = acc;
            }
        }
        // (the next iteration's x staging is separated from these reads by the barrier after it)
    }
    if (a.hstate) {                                      // streaming: carry the last hidden state of every layer
        __syncthreads();
        const int pl = (Tp - 1) & 1;
        for (int e = tid; e < L * R * (H / 2); e += blockDim.x) {
            const int l = e / (R * (H / 2)), r = (e / (H / 2)) % R, u2 = e % (H / 2);
            reinterpret_cast<uint32_t*>(a.hstate + ((size_t)l * a.rows_alloc + row0 + r) * H)[u2] =
                reinterpret_cast<const uint32_t*>(hb + ((size_t)l * 2 + pl) * R * HS + (size_t)r * HS)[u2];
        }
    }
}

static int pick_rows(int L, int H, int Ipad, int O) {
    for (int R : {64, 32, 16})
        if (mma_plan(L, H, Ipad, R, O).total <= 227 * 1024) return R;
    return 0;
}

size_t lstm_mma_cstate_bytes(int L, int rows, int H, int* rows_alloc) {
    int ra = ((rows + 63) / 64) * 64;
    if (rows_alloc) *rows_alloc = ra;
    return (size_t)L * ra * H * sizeof(float);
}

template <int R>
static int launch_r(const LstmMmaLaunch& a, cudaStream_t s) {
    MmaSmemPlan p = mma_plan(a.L, a.H, a.Ipad, R, a.out ? a.O : 0);
    dim3 grid((a.rows + R - 1) / R);
    cudaError_t e;
    if (a.fast) {
        e = cudaFuncSetAttribute(lstm_mma_kernel<R, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.total);
        if (e != cudaSuccess) return (int)e;
        lstm_mma_kernel<R, true><<<grid, 256, p.total, s>>>(a);
    } else {
        e = cudaFuncSetAttribute(lstm_mma_kernel<R, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.total);
        if (e != cudaSuccess) return (int)e;
        lstm_mma_kernel<R, false><<<grid, 256, p.total, s>>>(a);
    }
    return (int)cudaGetLastError();
}

int launch_lstm_mma(const LstmMmaLaunch& a, cudaStream_t s) {
    if (a.H % 16 || a.Ipad % 16 || a.L < 1 || a.L > 4) return (int)cudaErrorInvalidValue;
    const int R = pick_rows(a.L, a.H, a.Ipad, a.out ? a.O : 0);
    if (R == 64) return launch_r<64>(a, s);
    if (R == 32) return launch_r<32>(a, s);
    if (R == 16) return launch_r<16>(a, s);
    return (int)cudaErrorInvalidValue;
}

}  // namespace fsn
