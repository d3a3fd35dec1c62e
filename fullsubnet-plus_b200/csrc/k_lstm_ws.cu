// Weight-stationary persistent stacked LSTM for FEW sequences (rows <= 64): the full-band LSTM of fullsubnet.Model
// (reference fullsubnet.py:39-47,86-87 -> sequence_model.py:113-122: nn.LSTM(F, H, L, batch_first)), where the "batch" is just
// the B utterances.  With so few rows the recurrence is latency-bound and the weights (7.4 MB fp16 for F=257, H=512, L=2) are
// the big operand, so the roles flip compared to the sub-band kernel: every CTA PINS a slice of the weights in shared memory
// for the whole sequence (4 hidden units x i,f,g,o x all K, both layers: 57 KB), all CTAs work on the SAME rows, exchange the
// tiny hidden state (64 x H fp16) through L2 and meet at a grid-wide barrier after every layer-step.
//   * grid = H / 4 CTAs (128 for H = 512), launched cooperatively (co-residency is required by the barrier);
//   * per layer-step: cp.async the A operand [64 x K] (x_t | h_prev, or h_{l-1} | h_prev) into shared memory, 8 warps = 4 row
//     tiles x 2 column tiles of mma.sync.m16n8k16, gates of one (row, unit) meet in a thread pair via one shuffle, cell state
//     stays in registers, h written as fp16 to the exchange buffer (double buffered by step parity);
//   * barrier = one atomicAdd + acquire-spin per CTA (with a clock watchdog).
// Streaming: the exchange buffer and a cell-state buffer persist across launches (resume + absolute step offset).
#include "fsn_common.cuh"
#include "fsn_kernels.h"
#include "../../include/fsnplus_b200.h"

namespace fsn {

constexpr int WS_ROWS = 64;
constexpr int WS_UNITS = 4;          // hidden units per CTA -> 16 gate columns (two n8 tiles)
constexpr int WS_THREADS = 256;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(counter, 1u);
        const long long t0 = clock64();
        unsigned int v;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
            if (clock64() - t0 > FSN_MBAR_TIMEOUT_CYCLES) __trap();
        } while (v < target);
    }
    __syncthreads();
}

// SLOTS: the streaming slot call (a.slot != null); the other instantiations compile without its per-row tests
template <bool FAST, bool SLOTS>
__global__ void __launch_bounds__(WS_THREADS, 1) lstm_ws_kernel(LstmWsLaunch a) {
    extern __shared__ __align__(16) unsigned char smraw[];
    const int L = a.L, H = a.H, Ipad = a.Ipad, Tp = a.Tp;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int u0 = blockIdx.x * WS_UNITS;
    const int KA = (Ipad > H ? Ipad : H) + H + 8;                    // padded row stride of the A tile (halves)
    // shared memory: per-layer weight slices [16][K_l + 8], then the A tile [64][KA]
    __half* wsm = reinterpret_cast<__half*>(smraw);
    size_t woff[4];
    size_t off = 0;
    for (int l = 0; l < L; ++l) { woff[l] = off; off += (size_t)16 * (((l == 0) ? Ipad : H) + H + 8); }
    __half* asm_ = wsm + off;

    // ---- pin my weight slice: column n of my 16 = gate (n & 3) of unit u0 + (n >> 2) -> weight row gate*H + unit
    for (int l = 0; l < L; ++l) {
        const int Kin = (l == 0) ? a.I : H, Kin_pad = (l == 0) ? Ipad : H, K = Kin_pad + H, WS = K + 8;
        const float* wih = a.w_ih[l];
        const float* whh = a.w_hh[l];
        for (int e = tid; e < 16 * K; e += WS_THREADS) {
            const int n = e / K, k = e % K;
            const int row = (n & 3) * H + u0 + (n >> 2);
            float v;
            if (k < Kin_pad) v = (k < Kin) ? wih[(size_t)row * Kin + k] : 0.f;
            else v = whh[(size_t)row * H + (k - Kin_pad)];
            wsm[woff[l] + (size_t)n * WS + k] = __float2half_rn(v);
        }
    }
    // biases of my gate columns and cell state: warp w = (row tile mt = w >> 1, column tile nt = w & 1); thread holds C-fragment
    // positions (rows r, r + 8) x (cols 2q, 2q + 1) of the n8 tile -> unit u0 + 2 nt + (q >> 1), gates (2 (q & 1), 2 (q & 1) + 1)
    const int mt = warp >> 1, nt = warp & 1, q = lane & 3, r0 = mt * 16 + (lane >> 2);
    const int unit = u0 + 2 * nt + (q >> 1);
    const bool owner = (q & 1) == 0;                                // even q: holds i,f and (after the shuffle) g,o -> does the cell update
    float bias[4][4];                                                // [layer][gate]
    float cst[4][2];                                                 // [layer][row r0 / r0 + 8]
#pragma unroll
    for (int l = 0; l < 4; ++l) {
        if (l < L) {
#pragma unroll
            for (int g = 0; g < 4; ++g) bias[l][g] = a.b_ih[l][g * H + unit] + a.b_hh[l][g * H + unit];
            cst[l][0] = (a.resume && a.cbuf) ? a.cbuf[((size_t)l * WS_ROWS + r0) * H + unit] : 0.f;
            cst[l][1] = (a.resume && a.cbuf) ? a.cbuf[((size_t)l * WS_ROWS + r0 + 8) * H + unit] : 0.f;
        }
    }
    // streaming slot call: rows r0 / r0 + 8 held (they keep cst and carry their previous h forward)
    // (and kf: from step hf[rr] on)
    bool held[2] = {false, false};
    int hf[2] = {Tp, Tp};
    if (SLOTS)
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            held[rr] = r0 + rr * 8 < a.rows && a.slot[r0 + rr * 8] < 0;
            if (a.kf && r0 + rr * 8 < a.rows) hf[rr] = a.kf[r0 + rr * 8];
        }
    __syncthreads();

    unsigned int bar_target = 0;
    const unsigned int G = gridDim.x;
    for (int t = 0; t < Tp; ++t) {
        const int par = (a.t0 + t) & 1;
#pragma unroll
        for (int l = 0; l < 4; ++l) {
            if (l >= L) break;
            const int K0 = (l == 0) ? Ipad : H, K = K0 + H, WS = K + 8;
            // ---- A tile: [64 rows][K0 | H] ---------------------------------------------------------------
            const __half* s0 = (l == 0) ? a.x + (size_t)t * a.rows_pad * Ipad : a.hbuf + ((size_t)(l - 1) * 2 + par) * WS_ROWS * H;
            const int ld0 = (l == 0) ? Ipad : H;
            const __half* s1 = a.hbuf + ((size_t)l * 2 + (par ^ 1)) * WS_ROWS * H;
            const int c0 = K0 / 8, c1 = H / 8;
            for (int e = tid; e < WS_ROWS * (c0 + c1); e += WS_THREADS) {
                const int r = e / (c0 + c1), c = e % (c0 + c1);
                if (c < c0) cp_async16(asm_ + (size_t)r * KA + c * 8, s0 + (size_t)r * ld0 + c * 8);
                else cp_async16(asm_ + (size_t)r * KA + K0 + (c - c0) * 8, s1 + (size_t)r * H + (c - c0) * 8);
            }
            cp_async_wait_all();
            __syncthreads();
            // ---- gates[16 rows x 8 cols] for my (mt, nt) --------------------------------------------------
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            const __half* wl = wsm + woff[l] + (size_t)(nt * 8 + (lane >> 2)) * WS + q * 2;
            const uint32_t abase = smem_u32(asm_ + (size_t)(mt * 16 + (lane & 15)) * KA + (lane >> 4) * 8);
#pragma unroll 4
            for (int ks = 0; ks < K / 16; ++ks) {
                uint32_t af[4];
                ldmatrix_x4(af, abase + ks * 32);
                const uint32_t b0 = *reinterpret_cast<const uint32_t*>(wl + ks * 16);
                const uint32_t b1 = *reinterpret_cast<const uint32_t*>(wl + ks * 16 + 8);
                mma_f16_16816(acc, af, b0, b1);
            }
            // acc[0], acc[1]: row r0, gates (2(q&1), 2(q&1)+1); acc[2], acc[3]: row r0 + 8.  Pair exchange: even q gets g,o.
            const float o0 = __shfl_xor_sync(0xffffffffu, acc[0], 1), o1 = __shfl_xor_sync(0xffffffffu, acc[1], 1);
            const float o2 = __shfl_xor_sync(0xffffffffu, acc[2], 1), o3 = __shfl_xor_sync(0xffffffffu, acc[3], 1);
            if (owner) {
                __half* hout = a.hbuf + ((size_t)l * 2 + par) * WS_ROWS * H;
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    if (SLOTS && (held[rr] || t >= hf[rr])) {                                  // h_prev (A tile column K0 + unit) into this step's parity
                        const int row = r0 + rr * 8;
                        hout[(size_t)row * H + unit] = asm_[(size_t)row * KA + K0 + unit];
                        continue;
                    }
                    const float gi = (rr ? acc[2] : acc[0]) + bias[l][0], gf = (rr ? acc[3] : acc[1]) + bias[l][1];
                    const float gg = (rr ? o2 : o0) + bias[l][2], go = (rr ? o3 : o1) + bias[l][3];
                    float c, h;
                    if (a.gru) { h = gru_cell_plain<FAST>(gi, gf, gg, go, cst[l][rr]); c = h; }
                    else { c = sigm<FAST>(gf) * cst[l][rr] + sigm<FAST>(gi) * tanh_<FAST>(gg); h = sigm<FAST>(go) * tanh_<FAST>(c); }
                    cst[l][rr] = c;
                    const int row = r0 + rr * 8;
                    hout[(size_t)row * H + unit] = __float2half_rn(h);
                    if (l == L - 1 && a.hseq && row < a.rows) a.hseq[((size_t)row * H + unit) * a.P + t] = h;
                }
            }
            bar_target += G;
            grid_barrier(a.barrier, bar_target);                    // h of this layer-step is visible to every CTA
        }
    }
    if (a.cbuf && owner) {
#pragma unroll
        for (int l = 0; l < 4; ++l)
            if (l < L) {
                a.cbuf[((size_t)l * WS_ROWS + r0) * H + unit] = cst[l][0];
                a.cbuf[((size_t)l * WS_ROWS + r0 + 8) * H + unit] = cst[l][1];
            }
    }
}

static size_t ws_smem(int L, int H, int Ipad) {
    size_t halves = 0;
    for (int l = 0; l < L; ++l) halves += (size_t)16 * (((l == 0) ? Ipad : H) + H + 8);
    halves += (size_t)WS_ROWS * ((Ipad > H ? Ipad : H) + H + 8);
    return halves * 2;
}

bool lstm_ws_supported(int L, int H, int Ipad, int rows, int num_sms) {
    return L >= 1 && L <= 4 && rows <= WS_ROWS && H % 16 == 0 && Ipad % 16 == 0 && H / WS_UNITS <= num_sms && ws_smem(L, H, Ipad) <= 227 * 1024;
}

int launch_lstm_ws(const LstmWsLaunch& a, cudaStream_t s) {
    const size_t smem = ws_smem(a.L, a.H, a.Ipad);
    const int grid = a.H / WS_UNITS;
    cudaError_t e = cudaMemsetAsync(a.barrier, 0, sizeof(unsigned int), s);
    if (e != cudaSuccess) return (int)e;
    LstmWsLaunch arg = a;
    void* params[] = {&arg};
    void (*k)(LstmWsLaunch) = a.fast ? (a.slot ? lstm_ws_kernel<true, true> : lstm_ws_kernel<true, false>)
                                     : (a.slot ? lstm_ws_kernel<false, true> : lstm_ws_kernel<false, false>);
    e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    e = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(k), dim3(grid), dim3(WS_THREADS), params, smem, s);
    return (int)e;
}

}  // namespace fsn
