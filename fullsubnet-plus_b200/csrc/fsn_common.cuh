// Common device helpers for the fsnplus_b200 kernels (sm_90a only: wgmma, TMA, mbarrier, clusters).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#ifdef FSN_MBAR_DEBUG
#include <cstdio>
#endif

#if defined(__CUDA_ARCH__) && !defined(__CUDA_ARCH_FEAT_SM90_ALL)
#error "fsnplus_b200 kernels must be compiled with -gencode arch=compute_90a,code=sm_90a"
#endif

namespace fsn {

// ----------------------------------------------------------------------------------------------
// small math
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2f(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcpf(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float tanh_approx(float x) { float y; asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// sigmoid / tanh from ex2 + rcp (about 2 ulp each): the accurate path.
__device__ __forceinline__ float sigmoid_acc(float x) {
    // 1 / (1 + 2^(-x*log2e)); ex2 saturates to +inf / 0 cleanly, rcp(inf) = 0.
    return rcpf(1.0f + ex2f(-1.4426950408889634f * x));
}
__device__ __forceinline__ float tanh_acc(float x) {
    // 1 - 2 / (1 + 2^(2x*log2e))
    return 1.0f - 2.0f * rcpf(1.0f + ex2f(2.8853900817779268f * x));
}
// MUFU.TANH based variants (max rel. err 2^-11): the fast path, selectable per kernel.
__device__ __forceinline__ float sigmoid_fast(float x) { return fmaf(0.5f, tanh_approx(0.5f * x), 0.5f); }

template <bool FAST> __device__ __forceinline__ float sigm(float x) { return FAST ? sigmoid_fast(x) : sigmoid_acc(x); }
template <bool FAST> __device__ __forceinline__ float tanh_(float x) { return FAST ? tanh_approx(x) : tanh_acc(x); }

// output activation of SequenceModel (sequence_model.py:84-93, 120-121); codes = FSN_ACT_* of include/fsnplus_b200.h
__device__ __forceinline__ float apply_act(float y, int act) {
    if (act == 1) return fmaxf(y, 0.f);
    if (act == 2) return tanhf(y);
    if (act == 3) return fminf(fmaxf(y, 0.f), 6.f);
    return y;
}

// decompress_cIRM (audio_zen/acoustics/mask.py:60-63, K = 10, limit = 9.9): limit*(m >= limit) - limit*(m <= -limit) + m*(|m| < limit)
// is a clamp; then -K log((K - m) / (K + m)).
__device__ __forceinline__ float decompress_cirm(float v) {
    v = (v >= 9.9f) ? 9.9f : ((v <= -9.9f) ? -9.9f : v);
    return -10.f * logf((10.f - v) / (10.f + v));
}

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// Programmatic dependent launch (front-end chain, ~30 short kernels per forward): a kernel launched with launch_chain() may start
// while its predecessor in the stream is still draining -- its CTAs are placed as SMs free up and run their prologue (barrier
// init) -- and MUST execute pdl_wait() before it touches anything the predecessor reads or writes; pdl_wait returns
// when the predecessor grid has completed and its memory is visible (a no-op for a normally launched kernel).  pdl_trigger() lets
// the successor begin launching once every CTA of this grid has executed it.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Power-of-two down-scale for storing an activation in fp16 whose input stream has absolute maximum `amax` (per sample): exact
// (no rounding), never amplifies (a bias term must not overflow when the stream is tiny), 1 for amax < 1.
__device__ __forceinline__ float fp16_store_scale(float amax) {
    int e = 0;
    frexpf(fminf(amax, 3.0e38f), &e);                  // amax = m 2^e, m in [0.5, 1)
    e = e < 0 ? 0 : (e > 126 ? 126 : e);
    return __int_as_float((127 - e) << 23);            // 2^-e
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Reflect index used by BaseModel.unfold (F.pad mode="reflect", no edge repeat):
// reference audio_zen/model/base_model.py:38.
__host__ __device__ __forceinline__ int reflect_idx(int p, int F) {
    if (p < 0) p = -p;
    if (p > F - 1) p = 2 * (F - 1) - p;
    return p;
}

// Byte offset of element (row r, half k) inside a K-major tile of 64 halves (128 bytes) per row stored with the
// 128-byte swizzle the wgmma shared-memory descriptor (SWIZZLE_128B) and TMA expect: rows at 128 B pitch,
// 16-byte chunk index XORed with (row & 7).  Tile base must be 1024-byte aligned.
__host__ __device__ __forceinline__ uint32_t sw128_offset(uint32_t r, uint32_t k) {
    return r * 128u + ((((k >> 3) ^ (r & 7u)) & 7u) << 4) + ((k & 7u) << 1);
}

// ----------------------------------------------------------------------------------------------
// shared-memory / mbarrier / bulk-copy / wgmma PTX wrappers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must trap (-> launch error reported to the host), never hang the box.
#ifndef FSN_MBAR_TIMEOUT_CYCLES
#define FSN_MBAR_TIMEOUT_CYCLES 3000000000ll   // ~1.6 s at H100 boost clock; no legitimate wait is longer than ms
#endif
#ifdef FSN_MBAR_DEBUG
// debug builds (-DFSN_MBAR_DEBUG): a watchdog expiry reports WHICH wait of which role hung before trapping
#define mbar_wait(bar, parity) mbar_wait_dbg(bar, parity, __LINE__)
__device__ __noinline__ void mbar_report(int line, uint32_t parity) {
    printf("mbar timeout: line %d block %d thread %d (warp %d) parity %u\n", line, (int)blockIdx.x, (int)threadIdx.x, (int)(threadIdx.x >> 5), parity);
}
__device__ __forceinline__ void mbar_wait_dbg(uint64_t* bar, uint32_t parity, int line) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > FSN_MBAR_TIMEOUT_CYCLES) { mbar_report(line, parity); __nanosleep(2000000); __trap(); }
    }
}
#else
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > FSN_MBAR_TIMEOUT_CYCLES) { __trap(); }
    }
}
#endif

// 1-D bulk async copy global -> shared (TMA engine, SASS UBLKCP), completion on an mbarrier.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// L2 eviction-priority hint for data every CTA re-reads (the weight streams of the recurrent kernel)
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}

// ---- wgmma (sm_90a warpgroup MMA) ---------------------------------------------------------
// Shared-memory matrix descriptor, K-major, SWIZZLE_128B, 128-byte rows, 8-row groups 1024 B apart (the layout sw128_offset
// describes and TMA writes with CU_TENSOR_MAP_SWIZZLE_128B).  Advancing K by 32 bytes inside the swizzle atom = start address + 2.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);          // start address      [0,14)
    d |= (uint64_t)1u << 16;                              // leading byte off.  [16,30) (ignored for swizzled K-major)
    d |= (uint64_t)(1024u >> 4) << 32;                    // stride byte offset [32,46)
    d |= (uint64_t)1u << 62;                              // SWIZZLE_128B       [62,64)
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across an asynchronous wgmma
template <int R> __device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x N] (+)= A[64 x K-step] * B[N x K-step]^T, both operands K-major in shared memory.  Accumulator fragment of thread
// (warp w of the warpgroup, lane l): d[4 j + 2 h + e] = D[16 w + l / 4 + 8 h][8 j + 2 (l % 4) + e].
__device__ __forceinline__ void wgmma_f16_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate));
}
// the 64 x 256 warpgroup tile of the input-projection GEMM (k_gemm_tc5.cu, gemm_f16_pair_kernel): fragment as above, j = 0 .. 31
__device__ __forceinline__ void wgmma_f16_n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate));
}

// ---- clusters ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of `smem_addr` (a shared::cta address valid in every CTA) inside CTA `rank`
__device__ __forceinline__ uint32_t mapa_u32(uint32_t smem_addr, uint32_t rank) {
    uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank)); return r;
}
// Arrive on an mbarrier of any CTA of the cluster.  CTA-scope release: it only has to order this thread's completed reads of a
// ring slot (wgmma, retired by wgmma.wait_group) before the producer refills it; a cluster-scope release would also wait for every
// outstanding global store of the thread.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
// 1-D bulk copy global -> shared of every CTA in `mask` (same offset in each), completion on the mbarrier at the same offset in each
__device__ __forceinline__ void bulk_g2s_multicast(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar, uint16_t mask, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint [%0], [%1], %2, [%3], %4, %5;" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "h"(mask), "l"(policy)
                 : "memory");
}

// One LSTM cell.  ai/af/ao = -log2(e) * (gate pre-activation), ag = -2 log2(e) * (g pre-activation): the scale and
// the bias are folded into one FMA on the accumulator (biases are stored pre-scaled).
// Accurate path: 5 ex2 + 3 rcp (i*tanh(g) and o*tanh(c) share one reciprocal each); fast path: 5 tanh.approx.
template <bool FAST>
__device__ __forceinline__ void lstm_cell(float ai, float af, float ag, float ao, float cprev, float& c, float& h) {
    if (FAST) {
        const float K = -0.34657359027997264f;                                // -0.5 / log2(e)
        const float si = fmaf(0.5f, tanh_approx(ai * K), 0.5f), sf = fmaf(0.5f, tanh_approx(af * K), 0.5f);
        c = fmaf(sf, cprev, si * tanh_approx(ag * K));
        h = fmaf(0.5f, tanh_approx(ao * K), 0.5f) * tanh_approx(c);
    } else {
        const float ei = ex2f(ai), ef = ex2f(af);
        const float eg = ex2f(fminf(fmaxf(ag, -43.f), 43.f));                  // tanh saturates: |g| <= 15
        const float ig = (1.f - eg) * rcpf((1.f + ei) * (1.f + eg));          // sigmoid(i) * tanh(g)
        c = fmaf(rcpf(1.f + ef), cprev, ig);
        const float eo = ex2f(ao);
        const float ec = ex2f(fminf(fmaxf(c * -2.8853900817779268f, -43.f), 43.f));
        h = (1.f - ec) * rcpf((1.f + eo) * (1.f + ec));                       // sigmoid(o) * tanh(c)
    }
}

// One GRU cell on the same four accumulators: the GRU weights are packed as pseudo-gates (r, z, n_x, n_h) -- n_x holds
// W_in x + b_in (zero recurrent block), n_h holds W_hn h + b_hn (zero input block) -- so every LSTM kernel computes it
// unchanged up to this function.  nn.GRU (sequence_model.py:39-46): n = tanh(n_x + r n_h); h = (1 - z) n + z h_prev.
// ar/az = -log2(e) * pre-activation; anx/anh = -2 log2(e) * pre-activation.  The "cell state" slot carries h in fp32.
template <bool FAST>
__device__ __forceinline__ void gru_cell(float ar, float az, float anx, float anh, float hprev, float& h) {
    float r, z, n;
    if (FAST) {
        const float K = -0.34657359027997264f;                                // -0.5 / log2(e)
        r = fmaf(0.5f, tanh_approx(ar * K), 0.5f);
        z = fmaf(0.5f, tanh_approx(az * K), 0.5f);
        n = tanh_approx(fmaf(r, anh, anx) * K);
    } else {
        r = rcpf(1.f + ex2f(ar));
        z = rcpf(1.f + ex2f(az));
        const float en = ex2f(fminf(fmaxf(fmaf(r, anh, anx), -43.f), 43.f));
        n = (1.f - en) * rcpf(1.f + en);
    }
    h = fmaf(z, hprev - n, n);
}
// plain-argument form for the generic kernels
template <bool FAST>
__device__ __forceinline__ float gru_cell_plain(float gr, float gz, float gnx, float gnh, float hprev) {
    const float r = sigm<FAST>(gr), z = sigm<FAST>(gz);
    const float n = tanh_<FAST>(fmaf(r, gnh, gnx));
    return fmaf(z, hprev - n, n);
}

// ---- warp-level tensor path (mma.sync) used by the generic kernels ------------------------------
__device__ __forceinline__ void mma_f16_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_tf32_1688(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t f2tf32(float x) { uint32_t r; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x)); return r; }
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t smem_addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_addr));
}

}  // namespace fsn
