// Single-layer recurrent LSTM / GRU kernel on the Hopper tensor cores (wgmma): the sub-band model of every stack the project
// runs (reference sequence_model.py:31-46,113-122; BASELINE configs #1 and #5).
//
// Decomposition (the classic time-batched split, one layer at a time):
//   gates_l(t) = W_ih_l x_l(t) + W_hh_l h_l(t-1) + b
//   * the first layer's input is 64 wide: its projection is part of the recurrence -- every step the 64 x 64 input tile (the swizzled
//     image of k_front.cu's packer) is one more k-block of the A operand, W_ih one more k-block in front of every gate chunk of the
//     stream (lstm_tc5_pack_first_layer);
//   * deeper layers' input projection has no recurrence: Gin_l = X_l W_ih_l^T is ONE GEMM over all rows and all time steps
//     (launch_gemm_f16, k_gemm_tc5.cu: fp16 in / fp32 accumulate / fp16 out), its gate columns pre-permuted to the order this
//     kernel's threads read them in (lstm_tc5r_gin_order);
//   * this kernel runs the recurrence of one layer for all time steps.  A CTA owns 64 sequences: h(t-1) lives in shared memory
//     (fp16, the swizzled K-major A operand of wgmma, double-buffered by step parity), W_hh streams from L2 through a ring of
//     16 KB k-blocks (128 gate columns x 64 k).  The two CTAs of a cluster share the stream: each fetches half of every k-block
//     and multicasts it to both, so the L2 reads W_hh once per 128 sequences.  Two consumer warpgroups take the 128-column
//     gate chunks in turn (m64n128k16, accumulator in registers): while one runs its cell update the other's MMAs are in
//     flight.  Each warpgroup has a ring of its own, consumed strictly in order (a shared ring would let one warpgroup wait on a
//     slot two phases ahead, which an mbarrier parity wait cannot tell from the phase before), and each ring a producer warp of its
//     own, so that one warpgroup's slow slot never holds back the other's stream.  The epilogue adds Gin_l(t), does
//     the cell update and writes h_l(t) both into the next step's A buffer and, for all but the last layer, as the next layer's
//     GEMM input (fp16, row-major); the last layer applies the output Linear(H -> 2) and writes the mask (or the enhanced spectrum).
// Long clips run one launch per time window (LstmTc5rLaunch::t0 / Tw, DESIGN.md §3.7): h enters from and leaves to a per-layer fp16
// state, c stays in the per-layer cstate, so a windowed layer computes exactly what one launch over all frames computes.
// Gate chunk j, column n = cg * 32 + q * 8 + u: gate q (i, f, g, o / GRU pseudo-gates r, z, n_x, n_h) of hidden unit
// 32 j + 8 cg + u (fsn_tc5_gate_row), so every thread's accumulator fragment holds all four gates of its units.
#include "fsn_common.cuh"
#include "fsn_kernels.h"
#include "../../include/fsnplus_b200.h"

#include <cstring>
#include <vector>

namespace fsn {

constexpr int R5_STAGE = 16384;                 // one k-block of one chunk of the packed stream: 128 gate columns x 64 k x fp16
constexpr int R5_CL = 2;                        // CTAs per cluster sharing the weight stream
constexpr int R5_ROWS = 64;                     // sequences per CTA
constexpr int R5_THREADS = 10 * 32;             // warps 0-7: two consumer warpgroups; warps 8, 9: the bulk-copy producers of rings 0, 1
constexpr int R5_MAX_SMEM = 227 * 1024;
constexpr int R5_XTILE = R5_ROWS * 128;         // one step's input tile of a CTA: 64 rows x 64 halves, SWIZZLE_128B
constexpr int R5_FCPART = 2 * R5_ROWS * 2 * 4;  // last layer: [2 step parities][64 rows][2] fp32 Linear partials of warpgroup 1

// Shared memory of one layer: [stages][h: 2 parities][input tiles: first layer][fc partials: last layer][barriers].  Whatever the
// fixed part leaves goes to the weight rings; ring 0 gets (nstage + 1) / 2 slots, ring 1 nstage / 2.
struct R5Plan { int nstage; size_t total; };
static inline R5Plan r5_plan(int H, bool kx, bool last) {
    R5Plan p;
    const size_t fixed = (size_t)2 * R5_ROWS * H * 2 + (kx ? 2 * R5_XTILE : 0) + (last ? R5_FCPART : 0) + 1024 /*align*/ + 4 * 8 /*xfull, xempty*/;
    const long avail = R5_MAX_SMEM - (long)fixed;
    p.nstage = (int)(avail / (R5_STAGE + 2 * 8));                  // a slot and its full / empty barriers
    if (p.nstage > 8) p.nstage = 8;
    if (p.nstage < 0) p.nstage = 0;
    p.total = fixed + (size_t)p.nstage * (R5_STAGE + 2 * 8);
    return p;
}
// first slot and slot count of ring r (the ring of consumer warpgroup r) out of nstage
__device__ __forceinline__ int r5_ring_base(int nstage, int r) { return r ? (nstage + 1) / 2 : 0; }
__device__ __forceinline__ int r5_ring_slots(int nstage, int r) { return r ? nstage / 2 : (nstage + 1) / 2; }

bool lstm_tc5r_supported(int H, int O) { return H % 64 == 0 && H >= 64 && H <= 512 && O == 2; }
size_t lstm_tc5r_cstate_bytes(int ntiles, int H) { return (size_t)((ntiles + 1) / 2 * 2) * H * 128 * sizeof(float); }
int64_t lstm_tc5r_weight_stream_bytes(int H) { return (int64_t)(H / 32) * (H / 64) * R5_STAGE; }

// LIM (last layer with enh only): each clip's mask gets its attenuation floor a.lam[clip] before the product (limit_mask); a sibling
// instantiation, so the kernels without a limit are the same code as before it existed
template <int H, bool FAST, bool GRU, bool LAST, bool LIM = false>
__global__ void __cluster_dims__(R5_CL, 1, 1) __launch_bounds__(R5_THREADS, 1) lstm_tc5r_kernel(LstmTc5rLaunch a, int nstage) {
    extern __shared__ uint8_t smem_raw[];
    constexpr int NCH = H / 32, KBH = H / 64, HBUF = KBH * R5_ROWS * 128;
    // steps t0 .. tend - 1 of the clip (the window); t is the absolute step throughout: the window-local buffers (images, Gin, hseq) are
    // indexed with t - t0, and since t0 % 4 == 0 the step parities and the phases of the input-tile barriers match a launch from t = 0
    const int t0 = a.t0, tend = a.t0 + a.Tw;
    const int cta = blockIdx.x;
    const uint32_t rank = cluster_ctarank();
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* stages = smem;
    uint8_t* hbuf = stages + (size_t)nstage * R5_STAGE;                     // [2][KBH][64 rows][128 B], SWIZZLE_128B
    const int KX = a.ximg ? 1 : 0, KT = KX + KBH;                          // k-blocks per gate chunk: [input][hidden]
    uint8_t* xbuf = hbuf + 2 * HBUF;                                       // [2 step parities][R5_XTILE] input tiles (first layer only)
    float* fcpart = reinterpret_cast<float*>(xbuf + KX * 2 * R5_XTILE);    // [2 step parities][64 rows][2] (last layer only)
    uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(fcpart) + (LAST ? R5_FCPART : 0));   // [nstage]: ring 0, ring 1
    uint64_t* empty = full + nstage;
    uint64_t* xfull = empty + nstage;                                      // [2]: input tile of the step parity landed
    uint64_t* xempty = xfull + 2;                                          // [2]: every MMA of the step that read it has retired

    if (tid == 0) {
        for (int i = 0; i < nstage; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 4 * R5_CL); }
        for (int i = 0; i < 2; ++i) { mbar_init(&xfull[i], 1); mbar_init(&xempty[i], 1); }
        fence_barrier_init();
    }
    if (a.hstate && t0 > 0) {                                              // h(t0 - 1) of the previous window into parity t0 & 1 = 0
        for (int i = tid; i < R5_ROWS * H / 8; i += R5_THREADS) {
            const int r = i / (H / 8), u = (i % (H / 8)) * 8;
            *reinterpret_cast<uint4*>(hbuf + (u >> 6) * R5_ROWS * 128 + sw128_offset(r, u & 63)) =
                __ldcg(reinterpret_cast<const uint4*>(a.hstate + (size_t)(cta * R5_ROWS + r) * H + u));
        }
    } else {
        for (int i = tid; i < HBUF / 16; i += R5_THREADS) reinterpret_cast<uint4*>(hbuf)[i] = make_uint4(0, 0, 0, 0);   // h(-1) = 0
    }
    fence_proxy_async();
    __syncthreads();
    cluster_sync_all();                                                    // barriers of both CTAs are initialised

    if (warp >= 8) {
        // ======================= producer of ring r: my half of every k-block of the chunks j = r, r + 2, ..., multicast to both CTAs
        // (one producer per ring, so neither ring waits for the other warpgroup to free a slot; weights do not depend on h, so each
        // producer runs ahead into the next step as far as its ring allows)
        if (lane == 0) {
            constexpr uint32_t PART = R5_STAGE / R5_CL;
            const int r = warp - 8, base = r5_ring_base(nstage, r), NS = r5_ring_slots(nstage, r);
            const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(a.wstream) + rank * PART;
            const uint64_t pol_w = l2_policy_evict_last();          // the weights, re-read every step by every cluster: must survive the Gin stream
            int slot = 0; uint32_t ph = 0;
            for (int t = t0; t < tend; ++t) {
                if (KX && r == 0) {                                 // my 64 rows of the step's input image
                    mbar_wait(&xempty[t & 1], ((t >> 1) & 1) ^ 1);
                    mbar_arrive_expect_tx(&xfull[t & 1], R5_XTILE);
                    bulk_g2s(xbuf + (t & 1) * R5_XTILE, reinterpret_cast<const uint8_t*>(a.ximg) + (((size_t)(cta >> 1) * a.Tw + (t - t0)) * 128 + (cta & 1) * R5_ROWS) * 128,
                             R5_XTILE, &xfull[t & 1]);
                }
                for (int j = r; j < NCH; j += 2)
                    for (int q = 0; q < KT; ++q) {
                        const int i = base + slot;
                        mbar_wait(&empty[i], ph ^ 1);
                        mbar_arrive_expect_tx(&full[i], R5_STAGE);
                        bulk_g2s_multicast(stages + (size_t)i * R5_STAGE + rank * PART, wsrc + (size_t)(j * KT + q) * R5_STAGE, PART, &full[i],
                                           (uint16_t)((1u << R5_CL) - 1), pol_w);
                        if (++slot == NS) { slot = 0; ph ^= 1; }
                    }
            }
        }
    } else {
        // ======================= consumers: warpgroup wg takes the chunks j = wg, wg + 2, ... =================
        const int wg = warp >> 2, wi = warp & 3, wt = tid & 127, cq = 2 * (lane & 3);
        int rl[2], grow[2];
        size_t mrow0[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            rl[h] = wi * 16 + (lane >> 2) + 8 * h;
            grow[h] = cta * R5_ROWS + rl[h];
            // + t * 128: row of the (tile, t - t0) block of Gin / hseq (mod 2^64: the sum is the window-local row)
            mrow0[h] = ((size_t)(cta >> 1) * a.Tw - t0) * 128 + (cta & 1) * R5_ROWS + rl[h];
        }
        const int Tout = a.Tp - a.la;
        const float L2E = 1.4426950408889634f;
        float* cbase = a.cstate + (size_t)cta * NCH * 4 * 128 * 4;
        float acc[64];
        const bool has_gin = a.gin != nullptr;
        const int rbase = r5_ring_base(nstage, wg), NS = r5_ring_slots(nstage, wg);
        int rslot = 0; uint32_t rph = 0;                            // position in this warpgroup's ring (slots rbase ..)
        for (int t = t0; t < tend; ++t) {
            const uint8_t* hA = hbuf + (size_t)(t & 1) * HBUF;
            uint8_t* hN = hbuf + (size_t)((t + 1) & 1) * HBUF;
            float fc0[2] = {0.f, 0.f}, fc1[2] = {0.f, 0.f};
            for (int j = wg; j < NCH; j += 2) {
                // input projection, cell state and biases of this chunk: in flight while the MMAs run
                // (Gin columns of a chunk are in lane-quad order, lstm_tc5r_gin_order: the 32 values of my row are 64 contiguous bytes;
                // word cg * 4 + q holds gate q of units cq, cq + 1 of column group cg)
                uint32_t gw[2][16] = {};
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!has_gin) break;
                    const uint4* gp = reinterpret_cast<const uint4*>(a.gin + (mrow0[h] + (size_t)t * 128) * (size_t)(4 * H) + j * 128 + (lane & 3) * 32);
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const uint4 v = __ldcs(gp + i);
                        gw[h][4 * i] = v.x; gw[h][4 * i + 1] = v.y; gw[h][4 * i + 2] = v.z; gw[h][4 * i + 3] = v.w;
                    }
                }
                float4 c4[4];
                float4* cp = reinterpret_cast<float4*>(cbase + (size_t)j * 4 * 128 * 4) + wt;
#pragma unroll
                for (int v = 0; v < 4; ++v) c4[v] = (t == 0) ? make_float4(0.f, 0.f, 0.f, 0.f) : __ldcg(cp + v * 128);

                if (KX && j == wg) mbar_wait(&xfull[t & 1], (uint32_t)(t >> 1) & 1u);    // the step's input tile
                int prev = -1;
#pragma unroll 1
                for (int kb = 0; kb < KT; ++kb) {
                    const int slot = rbase + rslot;
                    mbar_wait(&full[slot], rph);
                    if (++rslot == NS) { rslot = 0; rph ^= 1; }
                    wgmma_fence();
                    const uint8_t* ablk = (kb < KX) ? xbuf + (t & 1) * R5_XTILE : hA + (kb - KX) * R5_ROWS * 128;
                    const uint64_t adesc = wgmma_desc_sw128(smem_u32(ablk));
                    const uint64_t bdesc = wgmma_desc_sw128(smem_u32(stages + (size_t)slot * R5_STAGE));
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) wgmma_f16_n128(acc, adesc + 2 * kk, bdesc + 2 * kk, (kb | kk) != 0);
                    wgmma_commit();
                    if (prev >= 0) {
                        wgmma_wait<1>();
                        if (lane == 0)
                            for (uint32_t r = 0; r < R5_CL; ++r) mbar_arrive_cluster(mapa_u32(smem_u32(&empty[prev]), r));
                    }
                    prev = slot;
                }
                wgmma_wait<0>();
                if (lane == 0)
                    for (uint32_t r = 0; r < R5_CL; ++r) mbar_arrive_cluster(mapa_u32(smem_u32(&empty[prev]), r));
                wgmma_fence_regs(acc);

                // cell update: thread holds rows rl[h], units 32 j + 8 cg + cq + e, all four gates (accumulator column block 4 cg + q)
                float cn[16];
#pragma unroll
                for (int cg = 0; cg < 4; ++cg) {
                    float bq[4][2];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const float2 b2 = __ldg(reinterpret_cast<const float2*>(a.bias + j * 128 + cg * 32 + q * 8 + cq));
                        bq[q][0] = b2.x; bq[q][1] = b2.y;
                    }
                    const int u0 = j * 32 + cg * 8 + cq;
                    float hv[2][2];
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            auto pre = [&](int q) {
                                const __half2 g2 = *reinterpret_cast<const __half2*>(&gw[h][cg * 4 + q]);
                                return acc[4 * (4 * cg + q) + 2 * h + e] + (has_gin ? (e ? __high2float(g2) : __low2float(g2)) : 0.f);
                            };
                            const int v = h * 8 + cg * 2 + e;
                            const float cprev = reinterpret_cast<const float*>(c4)[v];
                            if (GRU) {
                                gru_cell<FAST>(fmaf(pre(0), -L2E, bq[0][e]), fmaf(pre(1), -L2E, bq[1][e]), fmaf(pre(2), -2.f * L2E, bq[2][e]),
                                               fmaf(pre(3), -2.f * L2E, bq[3][e]), cprev, hv[h][e]);
                                cn[v] = hv[h][e];
                            } else {
                                lstm_cell<FAST>(fmaf(pre(0), -L2E, bq[0][e]), fmaf(pre(1), -L2E, bq[1][e]), fmaf(pre(2), -2.f * L2E, bq[2][e]),
                                                fmaf(pre(3), -L2E, bq[3][e]), cprev, cn[v], hv[h][e]);
                            }
                        }
                    float2 w0 = make_float2(0.f, 0.f), w1 = w0;
                    if (LAST) {
                        w0 = __ldg(reinterpret_cast<const float2*>(a.fc_w + u0));
                        w1 = __ldg(reinterpret_cast<const float2*>(a.fc_w + H + u0));
                    }
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint32_t hp = pack_half2(hv[h][0], hv[h][1]);
                        *reinterpret_cast<uint32_t*>(hN + (u0 >> 6) * R5_ROWS * 128 + sw128_offset(rl[h], u0 & 63)) = hp;
                        if (!LAST) *reinterpret_cast<uint32_t*>(a.hseq + (mrow0[h] + (size_t)t * 128) * H + u0) = hp;   // next layer's GEMM input
                        if (LAST) {
                            fc0[h] = fmaf(hv[h][0], w0.x, fmaf(hv[h][1], w0.y, fc0[h]));
                            fc1[h] = fmaf(hv[h][0], w1.x, fmaf(hv[h][1], w1.y, fc1[h]));
                        }
                    }
                }
#pragma unroll
                for (int v = 0; v < 4; ++v) __stcg(cp + v * 128, make_float4(cn[4 * v], cn[4 * v + 1], cn[4 * v + 2], cn[4 * v + 3]));
            }
            if (LAST) {                                             // the four lanes of a row hold disjoint units: reduce, then across the warpgroups
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int o = 1; o < 4; o <<= 1) {
                        fc0[h] += __shfl_xor_sync(0xffffffffu, fc0[h], o);
                        fc1[h] += __shfl_xor_sync(0xffffffffu, fc1[h], o);
                    }
                if (wg == 1 && (lane & 3) == 0)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        fcpart[((t & 1) * R5_ROWS + rl[h]) * 2] = fc0[h];
                        fcpart[((t & 1) * R5_ROWS + rl[h]) * 2 + 1] = fc1[h];
                    }
            }
            fence_proxy_async();                                    // h(t) (generic stores) -> the next step's wgmma (async proxy)
            asm volatile("bar.sync 1, 256;" ::: "memory");
            if (KX && tid == 0) mbar_arrive(&xempty[t & 1]);        // every MMA of step t has retired: the input tile may be replaced
            if (LAST && wg == 0 && (lane & 3) == 0 && t >= a.la) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (grow[h] >= a.rows) continue;
                    const int ob = grow[h] / a.F, of = grow[h] % a.F;
                    if (a.tlen && t >= __ldg(a.tlen + ob)) {       // past the clip's end: zeros, the noisy planes are not read
                        const size_t ni = ((size_t)ob * a.F + of) * Tout + (t - a.la);
                        if (a.enh) a.enh[ni] = make_float2(0.f, 0.f);
                        else { a.out[(((size_t)ob * 2 + 0) * a.F + of) * Tout + (t - a.la)] = 0.f; a.out[(((size_t)ob * 2 + 1) * a.F + of) * Tout + (t - a.la)] = 0.f; }
                        continue;
                    }
                    const float o0 = apply_act(fc0[h] + fcpart[((t & 1) * R5_ROWS + rl[h]) * 2] + __ldg(a.fc_b), a.act);
                    const float o1 = apply_act(fc1[h] + fcpart[((t & 1) * R5_ROWS + rl[h]) * 2 + 1] + __ldg(a.fc_b + 1), a.act);
                    const size_t ni = ((size_t)ob * a.F + of) * Tout + (t - a.la);
                    if (a.enh) {                                       // fused decompress_cIRM x noisy spectrum (inferencer.py:152-157)
                        float m0 = decompress_cirm(o0), m1 = decompress_cirm(o1);
                        if (LIM) limit_mask(m0, m1, __ldg(a.lam + ob));
                        const float nr = __ldg(a.nreal + ni), nim = __ldg(a.nimag + ni);
                        a.enh[ni] = make_float2(m0 * nr - m1 * nim, m1 * nr + m0 * nim);
                    } else {
                        a.out[(((size_t)ob * 2 + 0) * a.F + of) * Tout + (t - a.la)] = o0;
                        a.out[(((size_t)ob * 2 + 1) * a.F + of) * Tout + (t - a.la)] = o1;
                    }
                }
            }
        }
    }
    __syncthreads();
    if (a.hstate) {                                                        // h(t0 + Tw - 1): the A buffer of step parity Tw
        const uint8_t* hL = hbuf + (size_t)(tend & 1) * HBUF;
        for (int i = tid; i < R5_ROWS * H / 8; i += R5_THREADS) {
            const int r = i / (H / 8), u = (i % (H / 8)) * 8;
            __stcg(reinterpret_cast<uint4*>(a.hstate + (size_t)(cta * R5_ROWS + r) * H + u),
                   *reinterpret_cast<const uint4*>(hL + (u >> 6) * R5_ROWS * 128 + sw128_offset(r, u & 63)));
        }
    }
    cluster_sync_all();                                            // no CTA leaves while its peer may still arrive on its barriers
}

template <int HH, bool FF, bool GG, bool LL, bool LIM = false>
static int r5_go(const LstmTc5rLaunch& a, int grid, const R5Plan& p, cudaStream_t s) {
    cudaError_t e = cudaFuncSetAttribute(lstm_tc5r_kernel<HH, FF, GG, LL, LIM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.total);
    if (e != cudaSuccess) return (int)e;
    lstm_tc5r_kernel<HH, FF, GG, LL, LIM><<<grid, R5_THREADS, p.total, s>>>(a, p.nstage);
    return (int)cudaGetLastError();
}
template <int HH>
static int r5_dispatch(const LstmTc5rLaunch& a, int grid, const R5Plan& p, cudaStream_t s) {
    const int key = (a.fast ? 4 : 0) | (a.gru ? 2 : 0) | (a.last ? 1 : 0);
    if (a.last && a.enh && a.lam) {                                 // the last layer with an attenuation limit
        switch (key) {
            case 1: return r5_go<HH, false, false, true, true>(a, grid, p, s);
            case 3: return r5_go<HH, false, true, true, true>(a, grid, p, s);
            case 5: return r5_go<HH, true, false, true, true>(a, grid, p, s);
            default: return r5_go<HH, true, true, true, true>(a, grid, p, s);
        }
    }
    switch (key) {
        case 0: return r5_go<HH, false, false, false>(a, grid, p, s);
        case 1: return r5_go<HH, false, false, true>(a, grid, p, s);
        case 2: return r5_go<HH, false, true, false>(a, grid, p, s);
        case 3: return r5_go<HH, false, true, true>(a, grid, p, s);
        case 4: return r5_go<HH, true, false, false>(a, grid, p, s);
        case 5: return r5_go<HH, true, false, true>(a, grid, p, s);
        case 6: return r5_go<HH, true, true, false>(a, grid, p, s);
        default: return r5_go<HH, true, true, true>(a, grid, p, s);
    }
}

int launch_lstm_tc5r(const LstmTc5rLaunch& a, cudaStream_t s) {
    if (!lstm_tc5r_supported(a.H, 2) || a.Tw < 1 || a.t0 < 0 || a.t0 % 4 || a.t0 + a.Tw > a.Tp) return (int)cudaErrorInvalidValue;
    const R5Plan p = r5_plan(a.H, a.ximg != nullptr, a.last != 0);
    if (p.nstage < 2) return (int)cudaErrorInvalidValue;
    const int grid = (a.ntiles + 1) / 2 * 2 * (128 / R5_ROWS);    // whole clusters; the buffers cover the padded tile pair
    switch (a.H) {
        case 64: return r5_dispatch<64>(a, grid, p, s);
        case 128: return r5_dispatch<128>(a, grid, p, s);
        case 192: return r5_dispatch<192>(a, grid, p, s);
        case 256: return r5_dispatch<256>(a, grid, p, s);
        case 320: return r5_dispatch<320>(a, grid, p, s);
        case 384: return r5_dispatch<384>(a, grid, p, s);
        case 448: return r5_dispatch<448>(a, grid, p, s);
        case 512: return r5_dispatch<512>(a, grid, p, s);
    }
    return (int)cudaErrorInvalidValue;
}

// ---------------------------------------------------------------------------------------------
// Host-side packing for one layer.
//   * recurrent stream: per chunk j, KBH stages of 16 KB = [128 gate columns (fsn_tc5_gate_row) x 64 k] of W_hh, K-major,
//     SWIZZLE_128B -- the layer-0 "hidden block" format of fsn_tc5_pack_weights;
//   * input-projection matrix for the GEMM: fp16 [4H, Kpad] row-major, row j * 128 + n = W_ih row fsn_tc5_gate_row(H, j, n),
//     so that column j * 128 + cg * 32 + q * 8 + u of Gin is gate q of hidden unit 32 j + 8 cg + u;
//   * biases: [4H] in the same column order, pre-scaled: the epilogue evaluates exp2(-log2(e) (acc + b)) as one FMA (tanh gates: -2 log2(e)).
// ---------------------------------------------------------------------------------------------
static inline uint16_t r5_h_bits(float f) { __half h = __float2half_rn(f); uint16_t b; std::memcpy(&b, &h, 2); return b; }

void lstm_tc5r_pack_layer(int H, int Kin, int Kpad, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, bool gru,
                          std::vector<uint16_t>& stream, std::vector<uint16_t>& wih_perm, std::vector<float>& bias) {
    const int NCH = H / 32, KBH = H / 64;
    stream.assign((size_t)NCH * KBH * (R5_STAGE / 2), 0);
    wih_perm.assign((size_t)4 * H * Kpad, 0);
    bias.assign((size_t)4 * H, 0.f);
    for (int j = 0; j < NCH; ++j)
        for (int n = 0; n < 128; ++n) {
            const int row = fsn_tc5_gate_row(H, j, n);
            for (int kb = 0; kb < KBH; ++kb) {
                uint8_t* img = reinterpret_cast<uint8_t*>(stream.data()) + ((size_t)j * KBH + kb) * R5_STAGE;
                for (int k = 0; k < 64; ++k) {
                    const uint16_t b = r5_h_bits(w_hh[(size_t)row * H + kb * 64 + k]);
                    std::memcpy(img + sw128_offset(n, k), &b, 2);
                }
            }
            for (int k = 0; k < Kin; ++k) wih_perm[((size_t)j * 128 + n) * Kpad + k] = r5_h_bits(w_ih[(size_t)row * Kin + k]);
            const int qg = (n % 32) / 8;
            const float sc = (qg == 2 || (qg == 3 && gru)) ? -2.8853900817779268f : -1.4426950408889634f;
            bias[(size_t)j * 128 + n] = sc * (b_ih[row] + b_hh[row]);
        }
}

// Row order of the input-projection matrix the GEMM multiplies with, so that the Gin columns of chunk j come out in the order the
// recurrent kernel reads them: column j * 128 + p * 32 + cg * 8 + q * 2 + e  <-  packed row j * 128 + (cg * 32 + q * 8 + 2 p + e).
void lstm_tc5r_gin_order(int H, int Kpad, std::vector<uint16_t>& wih_perm) {
    const std::vector<uint16_t> src(wih_perm);
    for (int j = 0; j < H / 32; ++j)
        for (int m = 0; m < 128; ++m) {
            const int p = m / 32, cg = (m / 8) % 4, q = (m / 2) % 4, e = m % 2;
            const int n = cg * 32 + q * 8 + 2 * p + e;
            std::memcpy(&wih_perm[((size_t)j * 128 + m) * Kpad], &src[((size_t)j * 128 + n) * Kpad], (size_t)Kpad * 2);
        }
}

}  // namespace fsn

extern "C" int64_t fsn_tc5r_weight_stream_bytes(int32_t H) { return (H % 64 || H < 64 || H > 512) ? -1 : fsn::lstm_tc5r_weight_stream_bytes(H); }

extern "C" int fsn_tc5r_pack_layer(int32_t H, int32_t Kin, int32_t Kpad, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                   int32_t gru, uint16_t* h_stream, uint16_t* h_wih, float* h_bias) {
    if (H % 64 || H < 64 || H > 512 || Kin < 1 || Kin > Kpad || !w_ih || !w_hh || !b_ih || !b_hh || !h_stream || !h_wih || !h_bias) return FSN_EINVAL;
    std::vector<uint16_t> st, wp;
    std::vector<float> bp;
    fsn::lstm_tc5r_pack_layer(H, Kin, Kpad, w_ih, w_hh, b_ih, b_hh, gru != 0, st, wp, bp);
    std::memcpy(h_stream, st.data(), st.size() * 2);
    std::memcpy(h_wih, wp.data(), wp.size() * 2);
    std::memcpy(h_bias, bp.data(), bp.size() * 4);
    return FSN_OK;
}

extern "C" int fsn_tc5r_gin_weights(int32_t H, int32_t Kin, int32_t Kpad, const float* w_ih, uint16_t* h_wih) {
    if (H % 64 || H < 64 || H > 512 || Kin < 1 || Kin > Kpad || !w_ih || !h_wih) return FSN_EINVAL;
    const std::vector<float> zero((size_t)4 * H * H, 0.f);             // W_hh and the biases do not enter the input-projection matrix
    std::vector<uint16_t> st, wp;
    std::vector<float> bp;
    fsn::lstm_tc5r_pack_layer(H, Kin, Kpad, w_ih, zero.data(), zero.data(), zero.data(), false, st, wp, bp);
    fsn::lstm_tc5r_gin_order(H, Kpad, wp);
    std::memcpy(h_wih, wp.data(), wp.size() * 2);
    return FSN_OK;
}

extern "C" int32_t fsn_tc5r_ring_stages(int32_t H, int32_t first, int32_t last) {
    return (H % 64 || H < 64 || H > 512) ? FSN_EINVAL : fsn::r5_plan(H, first != 0, last != 0).nstage;
}
