// TCN full-band model (K3 of SURVEY.md 2a) on the Hopper tensor cores: the 1x1 convolutions of the eight TCNBlocks and the
// output Linear as persistent wgmma GEMMs over time-major activations, plus the depth-wise convolution between them.  The same
// kernels run the optional sub-band TCN (sequence_model = "TCN": one branch, the B*F sequences as the gLN groups, EPI5_GLN_HEAD
// last).  The input projection of the layer-wise LSTM path runs on gemm_f16_pair_kernel below (128 x 256 tiles on CTA pairs), or on
// this GEMM kernel (EPI5_F16OUT) for shapes without tile pairs and under FSN_GIN_GEMM=128.
//
// reference: TCNBlock.forward (audio_zen/model/module/causal_conv.py:96-108) and SequenceModel.forward, TCN branch
// (audio_zen/model/module/sequence_model.py:106-112).
//
// Formulation.  Activations are stored time-major, rows = (branch, sample, frame), columns = channels (padded to a
// multiple of 32 floats = one 128-byte swizzle atom), so every 1x1 convolution is  D[rows, C_out] = X[rows, C_in] *
// W[C_out, C_in]^T  with BOTH operands K-major -- the layout PyTorch already stores W in.  Tiles of 128 rows x 128 bytes of k
// (A) and NT x 128 bytes of k (B) are fetched by TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B) into a shared-memory ring by one
// producer warp; two consumer warpgroups (64 rows each) multiply them with wgmma (tf32 on the fp32 residual stream, f16 on the
// fp16 hidden activations) into register accumulators and run the epilogue on those registers while the producer already
// fetches the next tile:
//   EPI_PRELU_STATS : + bias, PReLU, per-sample sum / sum-of-squares for the following gLN, store as fp16 times a per-sample power of
//                     two (fp16_store_scale: the hidden, 512-channel activations of a block live in fp16 -- the same 10 mantissa
//                     bits the tf32 product consumed, half the bytes; the normalised real / imag streams reach 1e6 and beyond)
//   EPI_GLN_RES     : gLN folded analytically -- conv(W, gLN(y)) = rstd * (W diag(gamma)) y - mean rstd s1 + s2 --
//                     so the GEMM runs on the raw activation and the per-sample affine is applied here, + residual (fp32 stream),
//                     + the running max |x| per sample of the new stream (the next block's store scale).
//                     Its operands (hidden activation, folded weights) are fp16: 64-element k-blocks.
//   EPI_OUT         : + bias, output activation, transposed into [branch, B, F, T'].
//   EPI_F16OUT      : fp16 result, row-major (Gin of the layer-wise LSTM, k_lstm_tc5r.cu).
//   EPI_GLN_HEAD    : last block of the sub-band TCN (one 64-column N tile, so a row's channels live in one lane quad): GLN_RES's
//                     new stream, then ReLU, Linear(I -> O) reduced over the quad, the output activation, and the mask (or the
//                     enhanced spectrum) of frames t >= look_ahead.  The final stream never goes to memory.
#include <cuda.h>

#include "fsn_common.cuh"
#include "fsn_kernels.h"
#include "../../include/fsnplus_b200.h"

namespace fsn {

constexpr int G5_CONS = 2;                                // consumer warpgroups, rows 64 wg .. 64 wg + 63 of a 128-row tile
constexpr int G5_THREADS = (4 * G5_CONS + 1) * 32;        // + one TMA producer warp (warp 8)
constexpr int G5_A_BYTES = 128 * 128;

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
                 : "memory");
}
// the same box written into the shared memory of every CTA in `mask` (same offset in each), completion on the mbarrier at the same
// offset in each
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar, uint16_t mask) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%2, %3}], [%4], %5;" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "h"(mask)
                 : "memory");
}

// one 32-byte k-step of the 64 x NT warpgroup tile: 16 fp16 or 8 tf32 elements
template <int NT, bool AH>
__device__ __forceinline__ void g5_mma(float (&acc)[NT / 2], uint64_t ad, uint64_t bd, uint32_t accumulate) {
    if constexpr (NT == 128) { if constexpr (AH) wgmma_f16_n128(acc, ad, bd, accumulate); else wgmma_tf32_n128(acc, ad, bd, accumulate); }
    else { static_assert(NT == 64, "NT is 64 or 128"); if constexpr (AH) wgmma_f16_n64(acc, ad, bd, accumulate); else wgmma_tf32_n64(acc, ad, bd, accumulate); }
}

// fp16 results (PRELU_STATS, F16OUT) leave through a per-warp staging tile: the accumulator fragment gives a lane 4 bytes of 8 rows
// per store, so direct stores wrote 16-byte pieces of 8 lines per instruction; staged, a warp writes whole 512-byte row runs.
// Tile = the warp's 16 rows x NT halves, 16-byte units XOR-swizzled by (row & 7) so both the fragment writes and the row reads are
// free of bank conflicts.  frag(j, h) = the packed pair (columns 8 j + 2 (lane % 4), + 1) of row (lane / 4) + 8 h.
template <int NT, typename Frag>
__device__ __forceinline__ void g5_store_f16_from(uint8_t* stg, int lane, Frag frag, __half* gbase, size_t ld, int nvalid) {
    constexpr int U = NT / 8;                                   // 16-byte units per row
#pragma unroll
    for (int j = 0; j < U; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = (lane >> 2) + 8 * h;
            *reinterpret_cast<uint32_t*>(stg + r * NT * 2 + ((j ^ (r & 7)) << 4) + (lane & 3) * 4) = frag(j, h);
        }
    __syncwarp();
    constexpr int RPI = 32 / U;                                 // rows per store instruction
#pragma unroll
    for (int i = 0; i < 16 / RPI; ++i) {
        const int r = i * RPI + lane / U, u = lane % U;
        const uint4 v = *reinterpret_cast<const uint4*>(stg + r * NT * 2 + ((u ^ (r & 7)) << 4));
        if (r < nvalid) *reinterpret_cast<uint4*>(gbase + (size_t)r * ld + u * 8) = v;
    }
    __syncwarp();
}
template <int NT>
__device__ __forceinline__ void g5_store_f16(uint8_t* stg, int lane, const uint32_t (&hp)[NT / 8][2], __half* gbase, size_t ld, int nvalid) {
    g5_store_f16_from<NT>(stg, lane, [&](int j, int h) { return hp[j][h]; }, gbase, ld, nvalid);
}

// sum (PRELU_STATS) or max (GLN_RES) of one value per lane into a per-sample slot: rows of a warp almost always belong to one
// sample -- reduce in the warp, one atomic per warp; lanes whose row is invalid pass key -1
__device__ __forceinline__ void g5_stats_add(int key, double s, double q, double* out) {
    if (__match_any_sync(0xffffffffu, key) == 0xffffffffu) {
        s = warp_sum_d(s); q = warp_sum_d(q);
        if ((threadIdx.x & 31) == 0 && key >= 0) { atomicAdd(&out[2 * key], s); atomicAdd(&out[2 * key + 1], q); }
    } else if (key >= 0) {
        atomicAdd(&out[2 * key], s);
        atomicAdd(&out[2 * key + 1], q);
    }
}
__device__ __forceinline__ void g5_max_add(int key, float v, float* out) {
    if (__match_any_sync(0xffffffffu, key) == 0xffffffffu) {
#pragma unroll
        for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
        if ((threadIdx.x & 31) == 0 && key >= 0) atomicMax(reinterpret_cast<int*>(out + key), __float_as_int(v));
    } else if (key >= 0) {
        atomicMax(reinterpret_cast<int*>(out + key), __float_as_int(v));
    }
}

// gLN of group z from its sum and sum of squares over `count` elements (stats[2z], stats[2z+1]): mean and 1 / sqrt(var + 1e-8)
__device__ __forceinline__ void gln_mean_rstd(const double* stats, int z, double count, float& mean, float& rstd) {
    const double mu = stats[2 * z] / count, var = stats[2 * z + 1] / count - mu * mu;
    mean = (float)mu;
    rstd = (float)(1.0 / sqrt((var > 0 ? var : 0) + 1e-8));
}

// one channel of the folded gLN + residual (EPI_GLN_RES): x + rstd * acc - mean * rstd * s1 + b
__device__ __forceinline__ float gln_res(float x, float acc, float mean, float rstd, float s1, float b) {
    return x + fmaf(rstd, acc, fmaf(-mean * rstd, s1, b));
}

template <int EPI, int NT>
__global__ void __launch_bounds__(G5_THREADS, 1)
gemm_tc5_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, GemmTc5Launch a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int nstage = a.nstage;
    constexpr int stage_bytes = G5_A_BYTES + NT * 128;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    uint8_t* stg = smem + (size_t)nstage * stage_bytes + (warp & 7) * 16 * NT * 2;    // this consumer warp's fp16 staging tile
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)nstage * stage_bytes + 8 * 16 * NT * 2);
    uint64_t* empty = full + nstage;

    if (tid == 0) {
        for (int i = 0; i < nstage; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 4 * G5_CONS); }
        fence_barrier_init();
    }
    __syncthreads();
    // chained launch: the barriers are set up while the previous kernel of the chain drains; nothing it wrote is read (and nothing it
    // reads is overwritten) before this point
    pdl_trigger();
    pdl_wait();
    constexpr bool HEAD = (EPI == EPI5_GLN_HEAD || EPI == EPI5_GLN_HEAD_LIM);
    constexpr bool AH = (EPI == EPI5_GLN_RES || EPI == EPI5_F16OUT || HEAD);   // fp16 operands: a 128-byte swizzle atom holds 64 k-elements instead of 32
    constexpr int KBW = AH ? 64 : 32;
    const int nkb = a.Kp / KBW;
    const int tiles_per_branch = a.tiles_m * a.ntiles_n;
    const int total = a.nbranch * tiles_per_branch;

    if (warp == 4 * G5_CONS) {
        if (lane == 0) {
            int slot = 0; uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
                const int br = tile / tiles_per_branch, rem = tile % tiles_per_branch;
                const int mt = rem / a.ntiles_n, nt = rem % a.ntiles_n;
                const int arow = br * a.rows_per_branch + mt * 128, brow = br * a.Npad + nt * NT;
                for (int kb = 0; kb < nkb; ++kb) {
                    mbar_wait(&empty[slot], ph ^ 1);
                    uint8_t* st = smem + (size_t)slot * stage_bytes;
                    mbar_arrive_expect_tx(&full[slot], stage_bytes);
                    tma_load_2d(st, &mapA, kb * KBW, arow, &full[slot]);
                    tma_load_2d(st + G5_A_BYTES, &mapB, kb * KBW, brow, &full[slot]);
                    if (++slot == nstage) { slot = 0; ph ^= 1; }
                }
            }
        }
        return;
    }

    const int wg = warp >> 2, wi = warp & 3;
    float acc[NT / 2];
    int slot = 0; uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int br = tile / tiles_per_branch, rem = tile % tiles_per_branch;
        const int mt = rem / a.ntiles_n, nt = rem % a.ntiles_n;
        // ---- main loop: one 128-byte k-block per ring slot, the slot is handed back as soon as its MMAs have retired ----
        int prev = -1;
        for (int kb = 0; kb < nkb; ++kb) {
            mbar_wait(&full[slot], ph);
            wgmma_fence();
            const uint32_t sa = smem_u32(smem + (size_t)slot * stage_bytes);
            const uint64_t adesc = wgmma_desc_sw128(sa + wg * 64 * 128), bdesc = wgmma_desc_sw128(sa + G5_A_BYTES);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) g5_mma<NT, AH>(acc, adesc + 2 * kk, bdesc + 2 * kk, (kb | kk) != 0);
            wgmma_commit();
            if (prev >= 0) {
                wgmma_wait<1>();
                if (lane == 0) mbar_arrive(&empty[prev]);
            }
            prev = slot;
            if (++slot == nstage) { slot = 0; ph ^= 1; }
        }
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(&empty[prev]);
        wgmma_fence_regs(acc);

        // ---- epilogue on the accumulator fragment: rows rl[h] of the tile, column pairs n0 + 8 j + 2 (lane % 4) ----
        const int n0 = nt * NT, cq = 2 * (lane & 3);
        int rib[2], z[2], tt[2], tz[2];
        bool valid[2], live[2];
        size_t grow[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            rib[h] = mt * 128 + wg * 64 + wi * 16 + (lane >> 2) + 8 * h;         // row inside the branch
            valid[h] = rib[h] < a.rows_per_branch;
            z[h] = br * a.B + rib[h] / a.Tp;
            tt[h] = rib[h] % a.Tp;
            grow[h] = (size_t)br * a.rows_per_branch + rib[h];
            tz[h] = (a.tlen && valid[h]) ? __ldg(a.tlen + z[h] / a.zdiv) : a.Tp;   // the frames of group z[h]
            live[h] = valid[h] && tt[h] < tz[h];                                  // a row of the clip (not past its end)
        }
        // rows of this warp: rib0 .. rib0 + 15 of the branch, nvalid of them exist
        const int rib0 = mt * 128 + wg * 64 + wi * 16;
        const int nvalid = a.rows_per_branch - rib0;
        __half* gbase = a.Y16 + ((size_t)br * a.rows_per_branch + rib0) * a.ldY + n0;
        if constexpr (EPI == EPI5_F16OUT) {
            uint32_t hp[NT / 8][2];
#pragma unroll
            for (int j = 0; j < NT / 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h) hp[j][h] = pack_half2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            g5_store_f16<NT>(stg, lane, hp, gbase, a.ldY, nvalid);
        } else if constexpr (EPI == EPI5_PRELU_STATS) {
            const float slope = __ldg(a.prelu[br]);
            const float* bias = a.bias[br];
            // fp16 store scale of the hidden activation: a power of two from the absolute maximum of this sample's input stream (the
            // normalised real / imaginary branches reach 1e5 and beyond -- 1 / mean(real) is unbounded); undone exactly by the gLN that follows
            float ysc[2], ls[2] = {0.f, 0.f}, lq[2] = {0.f, 0.f};
            uint32_t hp[NT / 8][2];
#pragma unroll
            for (int h = 0; h < 2; ++h) ysc[h] = valid[h] ? fp16_store_scale(__ldg(a.amax_in + z[h])) : 1.f;
#pragma unroll
            for (int j = 0; j < NT / 8; ++j) {
                const int n = n0 + 8 * j + cq;
                const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + n));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float y[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float t = acc[4 * j + 2 * h + e] + (e ? b2.y : b2.x);
                        t = (t >= 0.f) ? t : slope * t;
                        t = live[h] ? t : 0.f;                    // past the clip's end: zero, and nothing added to the statistics
                        ls[h] += t; lq[h] = fmaf(t, t, lq[h]);
                        y[e] = fminf(fmaxf(t * ysc[h], -65504.f), 65504.f);
                    }
                    hp[j][h] = pack_half2(y[0], y[1]);
                }
            }
            g5_store_f16<NT>(stg, lane, hp, gbase, a.ldY, nvalid);
#pragma unroll
            for (int h = 0; h < 2; ++h) g5_stats_add(valid[h] ? z[h] : -1, (double)ls[h], (double)lq[h], a.stats_out);
        } else if constexpr (EPI == EPI5_GLN_RES) {
            const float* bias = a.bias[br];
            const float* s1 = a.s1[br];
            float mean[2] = {0.f, 0.f}, rstd[2] = {1.f, 1.f}, rowmax[2] = {0.f, 0.f};
#pragma unroll
            for (int h = 0; h < 2; ++h)
                if (valid[h]) gln_mean_rstd(a.stats_in, z[h], a.count_row * tz[h], mean[h], rstd[h]);
#pragma unroll
            for (int j = 0; j < NT / 8; ++j) {
                const int n = n0 + 8 * j + cq;
                if (n >= a.Npad) continue;                            // past the channels of this branch (the tile overhangs)
                const float2 s12 = __ldg(reinterpret_cast<const float2*>(s1 + n)), b2 = __ldg(reinterpret_cast<const float2*>(bias + n));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!valid[h]) continue;
                    const float2 x = *reinterpret_cast<const float2*>(a.Xold + grow[h] * a.ldY + n);
                    float2 o;
                    o.x = gln_res(x.x, acc[4 * j + 2 * h], mean[h], rstd[h], s12.x, b2.x);
                    o.y = gln_res(x.y, acc[4 * j + 2 * h + 1], mean[h], rstd[h], s12.y, b2.y);
                    if (!live[h]) o = make_float2(0.f, 0.f);
                    rowmax[h] = fmaxf(rowmax[h], fmaxf(fabsf(o.x), fabsf(o.y)));
                    *reinterpret_cast<float2*>(a.Y + grow[h] * a.ldY + n) = o;
                    if (a.Xrelu) *reinterpret_cast<float2*>(a.Xrelu + grow[h] * a.ldY + n) = make_float2(fmaxf(o.x, 0.f), fmaxf(o.y, 0.f));
                }
            }
            if (a.amax_out) {                                 // max |x| of the new stream per sample (max is order-independent: deterministic)
#pragma unroll
                for (int h = 0; h < 2; ++h) g5_max_add(valid[h] ? z[h] : -1, rowmax[h], a.amax_out);
            }
        } else if constexpr (HEAD) {
            static_assert(NT == 64, "the head needs all channels of a row in one lane quad");
            const float* bias = a.bias[br];
            const float* s1 = a.s1[br];
            float mean[2] = {0.f, 0.f}, rstd[2] = {1.f, 1.f}, fc[2][8];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
#pragma unroll
                for (int q = 0; q < 8; ++q) fc[h][q] = 0.f;
                if (valid[h]) gln_mean_rstd(a.stats_in, z[h], a.count_row * tz[h], mean[h], rstd[h]);
            }
#pragma unroll
            for (int j = 0; j < NT / 8; ++j) {
                const int n = 8 * j + cq;
                const float2 s12 = __ldg(reinterpret_cast<const float2*>(s1 + n)), b2 = __ldg(reinterpret_cast<const float2*>(bias + n));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!live[h]) continue;
                    const float2 x = *reinterpret_cast<const float2*>(a.Xold + grow[h] * a.ldY + n);
                    const float o0 = fmaxf(gln_res(x.x, acc[4 * j + 2 * h], mean[h], rstd[h], s12.x, b2.x), 0.f);
                    const float o1 = fmaxf(gln_res(x.y, acc[4 * j + 2 * h + 1], mean[h], rstd[h], s12.y, b2.y), 0.f);
#pragma unroll
                    for (int q = 0; q < 8; ++q)
                        if (q < a.O) {
                            const float2 w = __ldg(reinterpret_cast<const float2*>(a.fc_w + q * 64 + n));
                            fc[h][q] = fmaf(o0, w.x, fmaf(o1, w.y, fc[h][q]));
                        }
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int q = 0; q < 8; ++q)
#pragma unroll
                    for (int o = 1; o < 4; o <<= 1) fc[h][q] += __shfl_xor_sync(0xffffffffu, fc[h][q], o);
            const int Tout = a.Tp - a.la;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!valid[h] || (lane & 3) != 0 || tt[h] < a.la) continue;
                const int ob = z[h] / a.Fg, of = a.f0 + z[h] % a.Fg;
                const size_t ni = ((size_t)ob * a.F + of) * Tout + (tt[h] - a.la);
                if (!live[h]) {                                // past the clip's end: zeros, the noisy planes are not read
                    if (a.enh) a.enh[ni] = make_float2(0.f, 0.f);
                    else
                        for (int q = 0; q < a.O; ++q) a.out[(((size_t)ob * a.O + q) * a.F + of) * Tout + (tt[h] - a.la)] = 0.f;
                } else if (a.enh) {                            // fused decompress_cIRM x noisy spectrum (inferencer.py:152-157), O = 2
                    float m0 = decompress_cirm(apply_act(fc[h][0] + __ldg(a.fc_b), a.act));
                    float m1 = decompress_cirm(apply_act(fc[h][1] + __ldg(a.fc_b + 1), a.act));
                    if constexpr (EPI == EPI5_GLN_HEAD_LIM) limit_mask(m0, m1, __ldg(a.lam + ob));   // the clip's attenuation floor
                    const float nr = __ldg(a.nreal + ni), nim = __ldg(a.nimag + ni);
                    a.enh[ni] = make_float2(m0 * nr - m1 * nim, m1 * nr + m0 * nim);
                } else {
#pragma unroll
                    for (int q = 0; q < 8; ++q)
                        if (q < a.O) a.out[(((size_t)ob * a.O + q) * a.F + of) * Tout + (tt[h] - a.la)] = apply_act(fc[h][q] + __ldg(a.fc_b + q), a.act);
                }
            }
        } else {
            const float* bias = a.bias[br];
#pragma unroll
            for (int j = 0; j < NT / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = n0 + 8 * j + cq + e;
                    if (n >= a.F) continue;
                    const float bv = __ldg(bias + n);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        if (valid[h]) a.out[((size_t)z[h] * a.F + n) * a.P + tt[h]] = apply_act(acc[4 * j + 2 * h + e] + bv, a.act);
                }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// row-major [rows, cols] matrix, boxes of box_rows x 128 bytes (32 floats / 64 halves), SWIZZLE_128B
static int make_tmap_2d(void* out_map, CUtensorMapDataType type, size_t esize, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) return -1;
        fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    const cuuint64_t gdim[2] = {cols, rows};
    const cuuint64_t gstride[1] = {cols * esize};
    const cuuint32_t box[2] = {(cuuint32_t)(128 / esize), box_rows};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(reinterpret_cast<CUtensorMap*>(out_map), type, 2, const_cast<void*>(base), gdim, gstride,
                    box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -(int)r;
}
int make_tmap_f32_2d(void* out_map, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    return make_tmap_2d(out_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, sizeof(float), base, rows, cols, box_rows);
}
int make_tmap_f16_2d(void* out_map, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    return make_tmap_2d(out_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, sizeof(__half), base, rows, cols, box_rows);
}

template <int E, int NT>
static int g5_launch(const CUtensorMap& mA, const CUtensorMap& mB, GemmTc5Launch a, int num_sms, cudaStream_t s) {
    const int stage_bytes = G5_A_BYTES + NT * 128;
    const int stg_bytes = 8 * 16 * NT * 2;                       // fp16 staging tiles of the eight consumer warps
    a.nstage = (227 * 1024 - 1024 - 256 - stg_bytes) / stage_bytes;
    if (a.nstage > 8) a.nstage = 8;
    const size_t smem = (size_t)a.nstage * stage_bytes + stg_bytes + 1024 + 256;
    const int total = a.nbranch * a.tiles_m * a.ntiles_n;
    const int grid = total < num_sms ? total : num_sms;
    cudaError_t e = cudaFuncSetAttribute(gemm_tc5_kernel<E, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    e = launch_chain(gemm_tc5_kernel<E, NT>, dim3(grid), dim3(G5_THREADS), smem, s, mA, mB, a);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

int launch_gemm_tc5(const void* mapA, const void* mapB, GemmTc5Launch a, int num_sms, cudaStream_t s) {
    const bool head = a.epi == EPI5_GLN_HEAD || a.epi == EPI5_GLN_HEAD_LIM;
    const bool f16k = a.epi == EPI5_GLN_RES || head;
    if ((a.NT != 64 && a.NT != 128) || a.Kp % (f16k ? 64 : 32) || a.Npad % 2) return (int)cudaErrorInvalidValue;
    if (head && (a.NT != 64 || a.Npad != 64 || a.ntiles_n != 1 || a.nbranch != 1 || a.O < 1 || a.O > 8 || (a.enh && a.O != 2)))
        return (int)cudaErrorInvalidValue;
    if (a.epi == EPI5_GLN_HEAD_LIM && (!a.enh || !a.lam)) return (int)cudaErrorInvalidValue;
    const CUtensorMap& mA = *reinterpret_cast<const CUtensorMap*>(mapA);
    const CUtensorMap& mB = *reinterpret_cast<const CUtensorMap*>(mapB);
    if (a.NT == 64) {
        if (a.epi == EPI5_GLN_HEAD) return g5_launch<EPI5_GLN_HEAD, 64>(mA, mB, a, num_sms, s);
        if (a.epi == EPI5_GLN_HEAD_LIM) return g5_launch<EPI5_GLN_HEAD_LIM, 64>(mA, mB, a, num_sms, s);
        if (a.epi == EPI5_PRELU_STATS) return g5_launch<EPI5_PRELU_STATS, 64>(mA, mB, a, num_sms, s);
        if (a.epi == EPI5_GLN_RES) return g5_launch<EPI5_GLN_RES, 64>(mA, mB, a, num_sms, s);
        return g5_launch<EPI5_OUT, 64>(mA, mB, a, num_sms, s);
    }
    if (a.epi == EPI5_PRELU_STATS) return g5_launch<EPI5_PRELU_STATS, 128>(mA, mB, a, num_sms, s);
    if (a.epi == EPI5_GLN_RES) return g5_launch<EPI5_GLN_RES, 128>(mA, mB, a, num_sms, s);
    return g5_launch<EPI5_OUT, 128>(mA, mB, a, num_sms, s);
}

// ---------------------------------------------------------------------------------------------
// Input projection of the layer-wise LSTM path on 128 x 256 tiles, the weight tile shared by a CTA pair (EPI5_F16OUT only).
// On 128 x 128 tiles every byte brought from L2 into shared memory feeds 64 FLOP, and at K = 384 the kernel moves 58 GB per
// flagship step that way -- bound by what the L2 delivers, not by HBM or the tensor cores.  Here the two CTAs of a cluster take
// M tiles 2p and 2p + 1 of the same 256-column N tile: each TMA-loads its own 128-row A box and one 128-row half of the 256-row
// B block, multicast to both, so per k-block a CTA pulls 16 KB of A and 16 KB of B for twice the MMAs (128 FLOP per byte).  Each
// consumer warpgroup runs m64n256k16 into 128 accumulator registers; the 256 columns leave in two 128-column passes through the
// staging tiles.  The k order (64-wide k-blocks, four 16-wide steps, fp32 accumulation) is the 128 x 128 kernel's: same bits.
// An `empty` slot counts the consumer warps of BOTH CTAs (the peer's half of B lands in this CTA's slot too), and no CTA exits
// while its peer may still arrive on its barriers.  The producer is a whole warpgroup (one thread issues the copies) so that the
// register file can be moved to the consumers with setmaxnreg: 128 accumulators plus the epilogue do not fit the 168 registers
// per thread that an even split of 288 or 384 threads leaves.
// ---------------------------------------------------------------------------------------------
constexpr int GP_CL = 2;                                  // CTAs per cluster: M tiles 2p, 2p + 1
constexpr int GP_NT = 256;                                // N tile
constexpr int GP_STAGE = G5_A_BYTES + GP_NT * 128;        // 16 KB of A + 32 KB of B per k-block
constexpr int GP_STG = 8 * 16 * 128 * 2;                  // fp16 staging tiles of the eight consumer warps, one 128-column pass
constexpr int GP_THREADS = 4 * (G5_CONS + 1) * 32;        // two consumer warpgroups + the producer warpgroup (warps 8-11)
constexpr int GP_REG_CONS = 232, GP_REG_PROD = 40;        // 2 x 128 x 232 + 128 x 40 <= 64 K registers

__global__ void __cluster_dims__(GP_CL, 1, 1) __launch_bounds__(GP_THREADS, 1)
gemm_f16_pair_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, GemmTc5Launch a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int nstage = a.nstage;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t rank = cluster_ctarank();
    uint8_t* stg = smem + (size_t)nstage * GP_STAGE + (warp & 7) * 16 * 128 * 2;   // this consumer warp's staging tile
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)nstage * GP_STAGE + GP_STG);
    uint64_t* empty = full + nstage;

    if (tid == 0) {
        for (int i = 0; i < nstage; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 4 * G5_CONS * GP_CL); }
        fence_barrier_init();
    }
    __syncthreads();
    cluster_sync_all();                                   // the barriers of both CTAs are initialised before any multicast or remote arrive
    pdl_trigger();
    pdl_wait();
    const int nkb = a.Kp / 64;
    const int pairs = a.tiles_m / GP_CL * a.ntiles_n;     // (M tile pair, N tile), N inner: clusters in flight share their A rows in L2
    const int cluster = blockIdx.x / GP_CL, nclusters = gridDim.x / GP_CL;

    if (warp >= 4 * G5_CONS) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(GP_REG_PROD));
        if (warp == 4 * G5_CONS && lane == 0) {
            int slot = 0; uint32_t ph = 0;
            for (int pt = cluster; pt < pairs; pt += nclusters) {
                const int mt = pt / a.ntiles_n * GP_CL + (int)rank, nt = pt % a.ntiles_n;
                for (int kb = 0; kb < nkb; ++kb) {
                    mbar_wait(&empty[slot], ph ^ 1);
                    uint8_t* st = smem + (size_t)slot * GP_STAGE;
                    mbar_arrive_expect_tx(&full[slot], GP_STAGE);   // my A box + both halves of B (mine and the peer's)
                    tma_load_2d(st, &mapA, kb * 64, mt * 128, &full[slot]);
                    tma_load_2d_multicast(st + G5_A_BYTES + rank * 128 * 128, &mapB, kb * 64, nt * GP_NT + (int)rank * 128, &full[slot],
                                          (uint16_t)((1u << GP_CL) - 1));
                    if (++slot == nstage) { slot = 0; ph ^= 1; }
                }
            }
        }
        __syncwarp();
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(GP_REG_CONS));
        const int wg = warp >> 2, wi = warp & 3;
        float acc[GP_NT / 2];
        int slot = 0; uint32_t ph = 0;
        for (int pt = cluster; pt < pairs; pt += nclusters) {
            const int mt = pt / a.ntiles_n * GP_CL + (int)rank, nt = pt % a.ntiles_n;
            int prev = -1;
            for (int kb = 0; kb < nkb; ++kb) {
                mbar_wait(&full[slot], ph);
                wgmma_fence();
                const uint32_t sa = smem_u32(smem + (size_t)slot * GP_STAGE);
                const uint64_t adesc = wgmma_desc_sw128(sa + wg * 64 * 128), bdesc = wgmma_desc_sw128(sa + G5_A_BYTES);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) wgmma_f16_n256(acc, adesc + 2 * kk, bdesc + 2 * kk, (kb | kk) != 0);
                wgmma_commit();
                if (prev >= 0) {
                    wgmma_wait<1>();
                    if (lane == 0)
                        for (uint32_t r = 0; r < GP_CL; ++r) mbar_arrive_cluster(mapa_u32(smem_u32(&empty[prev]), r));
                }
                prev = slot;
                if (++slot == nstage) { slot = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            if (lane == 0)
                for (uint32_t r = 0; r < GP_CL; ++r) mbar_arrive_cluster(mapa_u32(smem_u32(&empty[prev]), r));
            wgmma_fence_regs(acc);

            // rows rib0 .. rib0 + 15 of this warp, columns nt * 256 + 128 p .. + 127 in pass p (accumulator columns 8 j + 2 (lane % 4) of
            // the 256 are acc[4 j + 2 h + e], j = 16 p .. 16 p + 15).  Pairs are packed as they are staged: next to 128 accumulators
            // there is no room for a packed copy of a pass.
            const int rib0 = mt * 128 + wg * 64 + wi * 16;
            __half* gbase = a.Y16 + (size_t)rib0 * a.ldY + nt * GP_NT;
#pragma unroll
            for (int p = 0; p < 2; ++p)
                g5_store_f16_from<128>(stg, lane, [&](int j, int h) { return pack_half2(acc[64 * p + 4 * j + 2 * h], acc[64 * p + 4 * j + 2 * h + 1]); },
                                       gbase + p * 128, a.ldY, a.rows_per_branch - rib0);
        }
    }
    cluster_sync_all();                                   // no CTA leaves while its peer may still arrive on its barriers
}

static int gp_launch(const CUtensorMap& mA, const CUtensorMap& mB, GemmTc5Launch a, cudaStream_t s) {
    a.nstage = (227 * 1024 - 1024 - 256 - GP_STG) / GP_STAGE;      // 4 stages of 48 KB + 32 KB of staging tiles
    const size_t smem = (size_t)a.nstage * GP_STAGE + GP_STG + 1024 + 256;
    cudaError_t e = cudaFuncSetAttribute(gemm_f16_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    // persistent: as many clusters as can be resident at once, never more than the tile pairs
    cudaLaunchConfig_t q{};
    q.gridDim = dim3(GP_CL); q.blockDim = dim3(GP_THREADS); q.dynamicSmemBytes = smem;
    int ncl = 0;
    e = cudaOccupancyMaxActiveClusters(&ncl, gemm_f16_pair_kernel, &q);
    if (e != cudaSuccess) return (int)e;
    if (ncl < 1) return (int)cudaErrorInvalidConfiguration;
    const int pairs = a.tiles_m / GP_CL * a.ntiles_n;
    if (ncl > pairs) ncl = pairs;
    e = launch_chain(gemm_f16_pair_kernel, dim3(GP_CL * ncl), dim3(GP_THREADS), smem, s, mA, mB, a);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

// Input projection of the layer-wise LSTM path: C[M, N] = A[M, K] B[N, K]^T, fp16 operands, fp32 accumulation, fp16 result.
// reference: the W_ih x_t half of nn.LSTM / nn.GRU (audio_zen/model/module/sequence_model.py:31-46,113-119), batched over all
// rows and time steps because it has no recurrence.  M = row tiles x frames x 128, N = 4H (a multiple of 256), K = 64 or H.
bool gemm_f16_supported(long long M, int N, int K) { return M > 0 && M % 128 == 0 && M / 128 < (1LL << 31) / 128 && N % 128 == 0 && K % 64 == 0 && K >= 64; }

// 128 x 256 pair tiles (gemm_f16_pair_kernel) when N is a multiple of 256 and the 128-row M tiles pair up -- every call of the
// layer-wise path: M = ntp x frames x 128 with ntp even -- unless g.tile_n = 128 asks for the 128 x 128 kernel
bool gemm_f16_pair_tiles(const GemmF16Launch& g) { return g.tile_n != 128 && g.N % GP_NT == 0 && (g.M / 128) % GP_CL == 0; }

int launch_gemm_f16(const void* A, const void* B, const GemmF16Launch& g, int num_sms, cudaStream_t s) {
    if (!gemm_f16_supported(g.M, g.N, g.K) || g.ldc != g.N || (g.tile_n != 0 && g.tile_n != 128 && g.tile_n != GP_NT))
        return (int)cudaErrorInvalidValue;
    alignas(64) CUtensorMap mA, mB;
    if (make_tmap_f16_2d(&mA, A, (uint64_t)g.M, (uint64_t)g.K, 128) || make_tmap_f16_2d(&mB, B, (uint64_t)g.N, (uint64_t)g.K, 128))
        return (int)cudaErrorInvalidValue;
    GemmTc5Launch a{};
    a.Kp = g.K; a.NT = 128; a.ntiles_n = g.N / 128; a.Npad = g.N;
    a.rows_per_branch = (int)g.M; a.tiles_m = (int)(g.M / 128); a.nbranch = 1; a.Tp = 1; a.B = 1;
    a.epi = EPI5_F16OUT; a.Y16 = g.C; a.ldY = g.N;
    if (gemm_f16_pair_tiles(g)) {
        a.NT = GP_NT; a.ntiles_n = g.N / GP_NT;
        return gp_launch(mA, mB, a, s);
    }
    return g5_launch<EPI5_F16OUT, 128>(mA, mB, a, num_sms, s);
}

// gLN1 apply -> depth-wise conv (k=3, dilation d, zero padding in the normalised domain; causal or symmetric taps) -> PReLU2 + gLN2 statistics,
// on the time-major [rows, C] fp16 layout.  reference: causal_conv.py:100-106.  One CTA = one sample x 64 channels x DW_TCH frames
// (+ a halo of 2d frames either side): the slab is staged once in shared memory in fp32 with the gLN already applied, so every input
// element is read once from HBM/L2 (halo rows twice) and the three taps come from shared memory.  All arithmetic in fp32; the
// statistics are taken before the result is rounded to fp16.  Clips of any length: the frame axis is chunked.
constexpr int DW_CH = 64, DW_TCH = 256, DW_HALO = 18;    // 2 * max dilation (9) frames: covers both tap geometries
__global__ void __launch_bounds__(256) dwconv_tm_kernel(DwTmLaunch a) {
    extern __shared__ float slab[];                       // [rows <= DW_TCH + 2 DW_HALO][DW_CH]
    __shared__ double red[16];
    pdl_trigger();
    pdl_wait();
    // grid.x = Z * (C / 64): the group count (B * F sequences for the sub-band TCN) exceeds gridDim.z's 65535
    const int ncb = a.C / DW_CH, z = blockIdx.x / ncb, g = z / a.B, c0 = (blockIdx.x % ncb) * DW_CH;
    const int C = a.C, Tp = a.Tp, d = a.dilation;
    const int Tz = a.tlen ? __ldg(a.tlen + z / a.zdiv) : Tp;          // frames of group z: taps past them read zero, rows past them are zero
    const int t0 = blockIdx.y * DW_TCH, t1 = min(t0 + DW_TCH, Tp);
    const int lo = max(t0 - 2 * d, 0), hi = min(t1 + 2 * d, Tz);    // staged frames [lo, hi)
    float mean, rstd;
    gln_mean_rstd(a.stats_in, z, (double)C * (double)Tz, mean, rstd);
    const float slope = __ldg(a.prelu[g]);
    const float unscale = 1.0f / fp16_store_scale(__ldg(a.amax + z));     // exact: a power of two
    const size_t base = (size_t)z * Tp * C + c0;
    const int cq = threadIdx.x & 15, tr = threadIdx.x >> 4;           // 16 columns of 4 channels x 16 frame rows per pass
    // per-channel constants: staged once per CTA (64 channels x 6 values) instead of scalar loads per thread; four channels per thread
    // keep the register count low enough for several CTAs per SM.
    __shared__ __align__(16) float cst[6][DW_CH];                     // gamma, beta, w0, w1, w2, bias
    if (threadIdx.x < DW_CH) {
        const int ch = c0 + threadIdx.x;
        cst[0][threadIdx.x] = __ldg(a.gamma[g] + ch);
        cst[1][threadIdx.x] = __ldg(a.beta[g] + ch);
        const float* wp = a.w[g] + (size_t)ch * 3;
        cst[2][threadIdx.x] = __ldg(wp); cst[3][threadIdx.x] = __ldg(wp + 1); cst[4][threadIdx.x] = __ldg(wp + 2);
        cst[5][threadIdx.x] = __ldg(a.b[g] + ch);
    }
    __syncthreads();
    float ga[4], be[4], w0[4], w1[4], w2[4], bb[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int ch = cq * 4 + e;
        const float gr = cst[0][ch] * rstd;
        ga[e] = gr * unscale;                                  // X holds y * 2^-k: (y - mean) rstd gamma + beta = X (2^k rstd gamma) + (beta - mean rstd gamma)
        be[e] = cst[1][ch] - mean * gr;
        w0[e] = cst[2][ch]; w1[e] = cst[3][ch]; w2[e] = cst[4][ch]; bb[e] = cst[5][ch];
    }
    for (int t = lo + tr; t < hi; t += 16) {
        const uint2 v = __ldg(reinterpret_cast<const uint2*>(a.X + base + (size_t)t * C + cq * 4));
        const float2 p0 = __half22float2(*reinterpret_cast<const __half2*>(&v.x)), p1 = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
        *reinterpret_cast<float4*>(slab + (size_t)(t - lo) * DW_CH + cq * 4) =
            make_float4(fmaf(p0.x, ga[0], be[0]), fmaf(p0.y, ga[1], be[1]), fmaf(p1.x, ga[2], be[2]), fmaf(p1.y, ga[3], be[3]));
    }
    __syncthreads();
    float ls = 0.f, lq = 0.f;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int t = t0 + tr; t < t1; t += 16) {
        if (t >= Tz) { *reinterpret_cast<uint2*>(a.Y + base + (size_t)t * C + cq * 4) = make_uint2(0u, 0u); continue; }
        // taps (w0, w1, w2): non-causal (t-d, t, t+d); causal (t-2d, t-d, t) -- padding 2d + chomp, causal_conv.py:74-75,104-105
        const int tl = a.causal ? t - 2 * d : t - d, tm = a.causal ? t - d : t, tr2 = a.causal ? t : t + d;
        const float4 m = (tm >= 0) ? *reinterpret_cast<const float4*>(slab + (size_t)(tm - lo) * DW_CH + cq * 4) : zero;
        const float4 l = (tl >= 0) ? *reinterpret_cast<const float4*>(slab + (size_t)(tl - lo) * DW_CH + cq * 4) : zero;
        const float4 r = (tr2 < Tz) ? *reinterpret_cast<const float4*>(slab + (size_t)(tr2 - lo) * DW_CH + cq * 4) : zero;
        const float lv[4] = {l.x, l.y, l.z, l.w}, mv[4] = {m.x, m.y, m.z, m.w}, rv[4] = {r.x, r.y, r.z, r.w};
        float o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            float y = fmaf(w0[e], lv[e], fmaf(w1[e], mv[e], fmaf(w2[e], rv[e], bb[e])));
            y = (y >= 0.f) ? y : slope * y;
            ls += y; lq = fmaf(y, y, lq);
            o[e] = fminf(fmaxf(y, -65504.f), 65504.f);
        }
        *reinterpret_cast<uint2*>(a.Y + base + (size_t)t * C + cq * 4) = make_uint2(pack_half2(o[0], o[1]), pack_half2(o[2], o[3]));
    }
    double s1 = warp_sum_d((double)ls), s2 = warp_sum_d((double)lq);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { red[warp] = s1; red[8 + warp] = s2; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double x1 = 0, x2 = 0;
        for (int i = 0; i < 8; ++i) { x1 += red[i]; x2 += red[8 + i]; }
        atomicAdd(&a.stats_out[2 * z], x1);
        atomicAdd(&a.stats_out[2 * z + 1], x2);
    }
}

int launch_dwconv_tm(const DwTmLaunch& a, cudaStream_t s) {
    if (a.C % DW_CH || 2 * a.dilation > DW_HALO || (long long)a.Z * (a.C / DW_CH) > 0x7fffffffLL || (a.Tp + DW_TCH - 1) / DW_TCH > 65535)
        return (int)cudaErrorInvalidValue;
    const int rows = (a.Tp < DW_TCH ? a.Tp : DW_TCH + 2 * DW_HALO);
    const size_t smem = (size_t)rows * DW_CH * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(dwconv_tm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    e = launch_chain(dwconv_tm_kernel, dim3(a.Z * (a.C / DW_CH), (a.Tp + DW_TCH - 1) / DW_TCH, 1), dim3(256), smem, s, a);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

}  // namespace fsn
