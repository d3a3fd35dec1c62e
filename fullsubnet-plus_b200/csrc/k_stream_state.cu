// Save, load and START reset of streaming sessions (DESIGN.md §3.11): one launch moves the state of n slots between the handle's
// per-slot rows and the canonical payload, [n, stride] bytes, or zeroes those rows.  grid (n, items): block (i, j) handles work item j
// of session i -- a piece of at most `chunk` bytes of one layer of one segment (StreamStateLaunch).  Memory-bound by design: each
// thread keeps four 16-byte loads in flight before it stores them.
#include "fsn_common.cuh"
#include "fsn_kernels.h"

namespace fsn {

template <typename V>
__device__ __forceinline__ void copy_vec(const char* __restrict__ src, char* __restrict__ dst, uint32_t bytes) {
    const V* s = reinterpret_cast<const V*>(src);
    V* d = reinterpret_cast<V*>(dst);
    const uint32_t n = bytes / sizeof(V), step = blockDim.x;
    uint32_t i = threadIdx.x;
    for (; i + 3 * step < n; i += 4 * step) {
        const V a = s[i], b = s[i + step], c = s[i + 2 * step], e = s[i + 3 * step];
        d[i] = a; d[i + step] = b; d[i + 2 * step] = c; d[i + 3 * step] = e;
    }
    for (; i < n; i += step) d[i] = s[i];
}

template <typename V>
__device__ __forceinline__ void zero_vec(char* __restrict__ dst, uint32_t bytes) {
    V* d = reinterpret_cast<V*>(dst);
    for (uint32_t i = threadIdx.x; i < bytes / sizeof(V); i += blockDim.x) d[i] = V{};
}

__global__ void __launch_bounds__(256) stream_state_copy_kernel(StreamStateLaunch a) {
    const int i = blockIdx.x;
    const StreamStateItem it = a.item[blockIdx.y];
    const StreamStateSeg& g = a.seg[it.seg];
    const int slot = a.slots[i];
    char* h = g.base + it.layer * g.layer_stride + (size_t)slot * g.slot_bytes + it.begin;
    if (a.dir == STREAM_STATE_ZERO) {
        if (g.vec == 16) zero_vec<uint4>(h, it.end - it.begin);
        else zero_vec<uint2>(h, it.end - it.begin);
        return;
    }
    char* p = a.payload + (size_t)i * a.stride + g.pay_off + (size_t)it.layer * g.slot_bytes + it.begin;
    const char* src = a.dir == STREAM_STATE_SAVE ? h : p;
    char* dst = a.dir == STREAM_STATE_SAVE ? p : h;
    if (g.vec == 16) copy_vec<uint4>(src, dst, it.end - it.begin);
    else copy_vec<uint2>(src, dst, it.end - it.begin);
}

int launch_stream_state(const StreamStateLaunch& a, cudaStream_t s) {
    stream_state_copy_kernel<<<dim3(a.n, a.nitem), 256, 0, s>>>(a);
    return (int)cudaGetLastError();
}

// The sub-band h and c of the sessions of a chunk's sub-batch between the handle and the layer-wise recurrence's carry
// (fsn_stream_step_chunk, DESIGN.md §3.13).  Thread = (layer, compact row j F + f, 8 hidden units).  h: fp16 rows, 16 bytes at a time.
// c (GRU: its fp32 h): the handle's row-major [rows_alloc, H] against lstm_tc5r_kernel's CTA-private order -- CTA cta = row / 64,
// chunk j = u / 32, thread wt and fragment element v of the float4 at cstate + (cta NCH + j) 2048 + (v / 4 * 128 + wt) * 4 + v % 4.
__global__ void __launch_bounds__(256) stream_sb_carry_kernel(StreamSbCarryLaunch a) {
    const int H = a.H, NCH = H / 32, F = a.F;
    const size_t per_layer = (size_t)a.n * F * (H / 8), n = per_layer * a.L;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int l = (int)(i / per_layer);
        const size_t e = i % per_layer;
        const int jr = (int)(e / (H / 8)), u0 = (int)(e % (H / 8)) * 8;
        const int hrow = a.sess[jr / F] * F + jr % F;              // the handle's row of this sequence
        uint4* hh = reinterpret_cast<uint4*>(a.h_handle + (l * (size_t)a.rows_alloc + hrow) * H + u0);
        uint4* hc = reinterpret_cast<uint4*>(a.h_carry + l * a.h_layer + (size_t)jr * H + u0);
        float* ch = a.c_handle + (l * (size_t)a.rows_alloc + hrow) * H + u0;
        float* cc = a.c_carry + l * a.c_layer + (size_t)(jr / 64) * NCH * 2048;
        const int rl = jr % 64, wi = rl / 16, hr = (rl % 16) / 8, lr = rl % 8;
#pragma unroll
        for (int w = 0; w < 8; ++w) {
            const int u = u0 + w, j = u / 32, cg = (u % 32) / 8, q = (u % 8) / 2, ev = u % 2;
            const int wt = wi * 32 + lr * 4 + q, v = hr * 8 + cg * 2 + ev;
            float* c = cc + (size_t)j * 2048 + ((v / 4) * 128 + wt) * 4 + v % 4;
            if (a.out) ch[w] = *c;
            else *c = ch[w];
        }
        if (a.out) *hh = *hc;
        else *hc = *hh;
    }
}

void launch_stream_sb_carry(const StreamSbCarryLaunch& a, cudaStream_t s) {
    const size_t n = (size_t)a.L * a.n * a.F * (a.H / 8);
    size_t blocks = (n + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    stream_sb_carry_kernel<<<(unsigned)blocks, 256, 0, s>>>(a);
}

}  // namespace fsn
