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

}  // namespace fsn
