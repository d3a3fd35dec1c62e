// Overlapped-chunk sessions (fsn_chunk_stream_step, DESIGN.md §3.16): around one batched offline audio forward of every chunk the call
// completed, the gather of the chunks' input rows from each slot's sample ring and the call's samples, and the cross-fade of the
// enhanced rows into each slot's output.  One CTA per slot for both; no FFT of their own (the forward is fsn_model_enhance_audio's).
// Positions are relative to the slot's next chunk start a0 = k0 H (64-bit on the host only): sample a0 + r of the session lies in the
// ring at (phase + r) mod R, R = C + P, when r < rel0, in the call's row at r - rel0 when rel0 <= r < rel1, and is zero below lo
// (the zero pre-context of chunk 0) and from rel1 on (past the session's end at FLUSH; no completed chunk reads there otherwise).
#include "fsn_common.cuh"
#include "fsn_kernels.h"

namespace fsn {

constexpr int CHUNK_THREADS = 256;

// grid B: the rows of slot b's completed chunks (chunk k0 + i at batch row row0 + i), then the call's samples appended to the ring.
// The ring keeps the last R written positions, which cover everything the slot's next chunk reads (< 2H + P samples), and is written
// only after every row of the slot has been gathered.
__global__ void __launch_bounds__(CHUNK_THREADS) chunk_gather_kernel(ChunkStreamLaunch a) {
    const int b = blockIdx.x;
    const int* p = a.plan + (size_t)b * CHUNK_PLAN_FIELDS;
    const int nc = p[CP_NC], row0 = p[CP_ROW0], rel0 = p[CP_REL0], rel1 = p[CP_REL1], lo = p[CP_LO], ph = p[CP_PHASE];
    const int H = a.C >> 1, W = a.C + a.P, R = W;
    const float* x = a.samples + (size_t)b * a.S;
    float* ring = a.ring + (size_t)b * R;
    for (int i = 0; i < nc; ++i) {
        float* row = a.rows + (size_t)(row0 + i) * W;
        for (int j = threadIdx.x; j < W; j += blockDim.x) {
            const int r = i * H - a.P + j;
            float v = 0.f;
            if (r >= lo && r < rel1) v = r >= rel0 ? x[r - rel0] : ring[(ph + r + R) % R];
            row[j] = v;
        }
    }
    __syncthreads();                                             // every read of the ring is done
    const int r0 = rel1 - R > rel0 ? rel1 - R : rel0;
    for (int r = r0 + (int)threadIdx.x; r < rel1; r += blockDim.x) ring[(ph + r) % R] = x[r - rel0];
}

// grid B: slot b's enhanced rows in chunk order.  Chunk k's row minus its first P samples is e_k; region k of the output is e_k's
// first half (k = 0: unwindowed) or e_k[0, H) w[0, H) + tail, and the tail becomes e_k[H, C) w[H, C).  The regions go to the front of
// the slot's output row, cut at nout (the session's end at FLUSH), zeros after them.  Thread t owns position t of every region and
// of the tail, so the chunks chain without barriers.
__global__ void __launch_bounds__(CHUNK_THREADS) chunk_crossfade_kernel(ChunkStreamLaunch a) {
    const int b = blockIdx.x;
    const int* p = a.plan + (size_t)b * CHUNK_PLAN_FIELDS;
    const int nc = p[CP_NC], row0 = p[CP_ROW0], first = p[CP_LO] == 0, nout = p[CP_NOUT];   // first: chunk k0 is chunk 0
    const int H = a.C >> 1, W = a.C + a.P;
    const size_t ow = (size_t)a.S + a.C;
    float* out = a.out + (size_t)b * ow;
    float* tail = a.tail + (size_t)b * chunk_tail_stride(a.C);
    for (int t = threadIdx.x; t < H; t += blockDim.x) {
        const float w0 = __ldg(a.window + t), w1 = __ldg(a.window + H + t);
        float tl = tail[t];
        for (int i = 0; i < nc; ++i) {
            const float* e = a.enh + (size_t)(row0 + i) * W + a.P;
            const float v = (first && i == 0) ? e[t] : e[t] * w0 + tl;
            const int o = i * H + t;
            if (o < nout) out[o] = v;
            tl = e[H + t] * w1;
        }
        if (nc) tail[t] = tl;
    }
    for (size_t o = (size_t)nout + threadIdx.x; o < ow; o += blockDim.x) out[o] = 0.f;
}

void launch_chunk_gather(const ChunkStreamLaunch& a, cudaStream_t s) { chunk_gather_kernel<<<a.B, CHUNK_THREADS, 0, s>>>(a); }
void launch_chunk_crossfade(const ChunkStreamLaunch& a, cudaStream_t s) { chunk_crossfade_kernel<<<a.B, CHUNK_THREADS, 0, s>>>(a); }

}  // namespace fsn
