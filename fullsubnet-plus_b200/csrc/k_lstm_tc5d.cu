// Host-side packing of the sub-band weight stream (128 gate columns x 64 k SWIZZLE_128B stages in consumption order) and the shared
// swizzle helper, exposed through the C ABI (include/fsnplus_b200.h) so the packed layouts can be checked on a machine without a GPU.
#include "fsn_common.cuh"
#include "fsn_kernels.h"
#include "../../include/fsnplus_b200.h"

#include <cstring>

static constexpr int kStage = 16384;      // one stage: 128 gate columns x 64 k x fp16

// ---------------------------------------------------------------------------------------------
// Stream order per time step: layer 0, chunk j = 0..H/32-1: [x block][H/64 hidden blocks];
//                             layer 1, chunk j:              [H/64 blocks of W_ih1][H/64 blocks of W_hh1].
// Stage = 128 gate columns (fsn_tc5_gate_row) x 64 k, K-major, SWIZZLE_128B.
// ---------------------------------------------------------------------------------------------
static inline uint16_t d5_h_bits(float f) {
    __half h = __float2half_rn(f);
    uint16_t b;
    std::memcpy(&b, &h, 2);
    return b;
}

extern "C" int64_t fsn_tc5_weight_stream_bytes(int32_t I, int32_t H) {
    if (H % 64 || I > 64) return -1;
    const int NCH = H / 32, KBH = H / 64;
    return (int64_t)(NCH * (1 + KBH) + NCH * 2 * KBH) * kStage;
}

// Gate column n (0..127) of chunk j <-> weight row: n = cg*32 + q*8 + u, q in (i,f,g,o), hidden unit 32 j + 8 cg + u.
extern "C" int32_t fsn_tc5_gate_row(int32_t H, int32_t j, int32_t n) { return ((n % 32) / 8) * H + 32 * j + 8 * (n / 32) + (n % 8); }

// one stage: 128 gate columns of chunk j x 64 k, getw(n, k)
template <class G> static void pack_stage(uint16_t* dst, size_t s, G&& getw) {
    uint8_t* img = reinterpret_cast<uint8_t*>(dst) + s * kStage;
    for (int n = 0; n < 128; ++n)
        for (int k = 0; k < 64; ++k) {
            uint16_t b = d5_h_bits(getw(n, k));
            std::memcpy(img + fsn::sw128_offset(n, k), &b, 2);
        }
}

// Layer-0 section of the stream, [x block][H/64 hidden blocks] per chunk: also the weight stream of the layer-wise kernel's first
// layer, whose input projection is part of the recurrence (k_lstm_tc5r.cu).
void fsn::lstm_tc5_pack_first_layer(int I, int H, const float* w_ih0, const float* w_hh0, uint16_t* dst) {
    const int NCH = H / 32, KBH = H / 64;
    size_t s = 0;
    for (int j = 0; j < NCH; ++j) {
        auto row = [&](int n) { return fsn_tc5_gate_row(H, j, n); };
        pack_stage(dst, s++, [&](int n, int k) { return k < I ? w_ih0[(size_t)row(n) * I + k] : 0.f; });
        for (int kb = 0; kb < KBH; ++kb) pack_stage(dst, s++, [&](int n, int k) { return w_hh0[(size_t)row(n) * H + kb * 64 + k]; });
    }
}

extern "C" int fsn_tc5_pack_weights(int32_t I, int32_t H, const float* w_ih0, const float* w_hh0, const float* w_ih1,
                                    const float* w_hh1, uint16_t* dst) {
    if (H % 64 || I > 64) return FSN_EINVAL;
    const int NCH = H / 32, KBH = H / 64;
    fsn::lstm_tc5_pack_first_layer(I, H, w_ih0, w_hh0, dst);
    size_t s = (size_t)NCH * (1 + KBH);
    for (int j = 0; j < NCH; ++j) {
        auto row = [&](int n) { return fsn_tc5_gate_row(H, j, n); };
        for (int kb = 0; kb < KBH; ++kb) pack_stage(dst, s++, [&](int n, int k) { return w_ih1[(size_t)row(n) * H + kb * 64 + k]; });
        for (int kb = 0; kb < KBH; ++kb) pack_stage(dst, s++, [&](int n, int k) { return w_hh1[(size_t)row(n) * H + kb * 64 + k]; });
    }
    return FSN_OK;
}

extern "C" uint32_t fsn_sw128_offset(uint32_t row, uint32_t k) { return fsn::sw128_offset(row, k); }
