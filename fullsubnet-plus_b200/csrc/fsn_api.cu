// C ABI of fsnplus_b200 (include/fsnplus_b200.h): model object, parameter store keyed by the reference's
// state_dict names, packing into kernel layouts, and the forward orchestration.
#include "../../include/fsnplus_b200.h"
#include "fsn_common.cuh"
#include "fsn_kernels.h"

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

using namespace fsn;

static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CK(x)                                                                                               \
    do {                                                                                                    \
        cudaError_t e_ = (x);                                                                               \
        if (e_ != cudaSuccess) return fail(FSN_ECUDA, "%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    // grow-only; a fresh allocation is zero-filled ON THE STREAM THAT WILL USE IT (a legacy-stream cudaMemset is not ordered
    // against kernels on a non-blocking stream)
    int ensure(size_t n, bool zero, cudaStream_t s = nullptr) {
        if (n <= bytes) return 0;
        if (p) cudaFree(p);
        p = nullptr; bytes = 0;
        cudaError_t e = cudaMalloc(&p, n);
        if (e != cudaSuccess) return (int)e;
        bytes = n;
        if (zero) e = cudaMemsetAsync(p, 0, n, s);
        return (int)e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
};

struct ParamSpec { std::string key; int64_t numel; };

// The packed block weights of one TCN (pack_tcn_blocks): nbr branches (key prefixes pre[b] = "<module>.sequence_model.") of C channels
// padded to Cp, gLN2 folded into the second 1x1 convolution; NT / ntiles = N tile and N tiles of its Cp-wide GEMMs.
struct TcnWeights {
    const char* name = "";                             // in error messages
    std::vector<std::string> pre;
    int nbr = 0, C = 0, Cp = 0, NT = 0, ntiles = 0;
    DevBuf W1, W2, S1, S2b;                            // [8][nbr][512][Cp] tf32, [8][nbr][Cp][512] fp16, [8][nbr][Cp] x2
    alignas(64) unsigned char mapW1[8][128], mapW2[8][128];
    void release() { W1.release(); W2.release(); S1.release(); S2b.release(); }
};

// The scratch of the eight blocks of one TCN over `rows` time-major rows: two fp32 streams [rows, Cp] (ping-pong), the fp16 hidden
// activations [rows, 512] before and after the depth-wise convolution, and the statistics (tcn_stats_bytes).
struct TcnScratch {
    DevBuf xa, xb, y1, y2, stats;
    alignas(64) unsigned char mapXa[128], mapXb[128], mapY2[128];
};

// The geometry a lane's workspaces were last sized for: B clips of T frames, window Tw, bin chunk Fc (0: whole clip / all bins); B = 0: none
struct WsGeo {
    int B = 0, T = 0, Tw = 0, Fc = 0;
    bool operator!=(const WsGeo& o) const { return B != o.B || T != o.T || Tw != o.Tw || Fc != o.Fc; }
};

// The plan of a plain forward: sub-batch Bs, window Tw, bin chunk Fc (0: whole clip / all bins), workspace bytes (ws_sizes)
struct Plan { int Bs = 0, Tw = 0, Fc = 0; int64_t bytes = 0; };

// Statistics of a TCN with Z gLN groups: [8 blocks][gLN1, gLN2][Z][sum, sum of squares] doubles, then [8 blocks][Z] floats, the max |x|
// per group of the stream entering each block (the fp16 store scale of its hidden activation).
static size_t tcn_stats_bytes(size_t Z) { return 8 * 2 * Z * 2 * sizeof(double) + 8 * Z * sizeof(float); }
static double* tcn_gln_sums(void* stats, size_t Z, int blk, int k) { return static_cast<double*>(stats) + (2 * blk + k) * Z * 2; }   // k = 0: gLN1, 1: gLN2
static float* tcn_amax(void* stats, size_t Z, int blk) { return reinterpret_cast<float*>(static_cast<double*>(stats) + 8 * 2 * Z * 2) + blk * Z; }

struct fsn_model {
    fsn_config cfg;
    std::vector<ParamSpec> specs;
    std::map<std::string, std::vector<float>> host;   // raw fp32 parameters (reference layout)
    std::map<std::string, float*> dev;                // same, on device
    DevBuf arena;
    bool finalized = false;
    int Isb = 0;                                      // sub-band LSTM input size
    // packed LSTM weights
    DevBuf sb_frag[4], sb_bias[4];
    DevBuf fb_frag[4], fb_bias[4];
    // layer-wise wgmma path (k_lstm_tc5r.cu): per-layer recurrent streams, permuted input-projection matrices, biases
    DevBuf r_stream[4], r_wih[4], r_bias[4], r_gin, r_hseq;    // r_wih: input-projection matrices of the layers > 0
    DevBuf r_hstate, sb_cum;                           // windowed forwards: per-layer h at the window's end, the packer's cumulative sums
    // Front-end workspaces (everything the full-band stage writes and the sub-band LSTM reads), grow-only, keyed by the last
    // geometry.  TWO lanes: the pipelined entry points (fsn_model_submit / fsn_model_forward_host_async) run the front end of
    // batch i+1 in lane (i+1)&1 on the front stream while the sub-band LSTM of batch i still reads lane i&1 on the LSTM stream.
    struct Lane {
        WsGeo geo;
        DevBuf fbin, fbout, mu, ximg, magpad, fbx, hseq;
        DevBuf x0, xr;                                 // time-major fb input / relu'd last residual
        TcnScratch tcn;                                // the full-band TCN's blocks (written on the front stream)
        DevBuf tsse_scale, sb_rowsum;
        DevBuf xn, sigma;                              // pre-normalised inputs / sub-band std for the non-default norm types
        DevBuf sbx;                                    // sub-band TCN: input [B*Fc*T', 64] fp32 time-major | max |x| per sequence [B*Fc] (Fc = F unchunked)
        DevBuf tlen;                                   // ragged forwards: per-sample extent frames[b] + look_ahead as int32 [3][B] (clip_len)
        alignas(64) unsigned char mapX0[128], mapXr[128], mapSbx[128];
        cudaEvent_t ev_front = nullptr, ev_lstm = nullptr;   // front end written / LSTM finished reading this lane
        bool used = false;                             // ev_lstm has been recorded (a pipelined batch ran / may still run in this lane)
    } lane[2];
    int last_lane = 0;
    DevBuf cstate, mask_tmp, stage_in[3], stage_out;   // LSTM-side scratch (one LSTM runs at a time), host-entry staging
    // wgmma TCN (FullSubNet+): the three full-band TCNs (branches of F channels) and their output Linear [3][Cp][Cp] tf32 + bias [3][Cp]
    bool tcn5 = false;
    int num_sms = 132;
    TcnWeights tcn_fb;
    DevBuf fb_fc, fb_fc_b;
    alignas(64) unsigned char map_fb_fc[128];
    DevBuf ws_h, ws_bar;                               // weight-stationary full-band LSTM: h exchange buffer, grid barrier
    // sub-band TCN (cfg.sb_tcn): one branch of Isb channels, the Linear head [O][64], and the scratch of the eight blocks -- shared by
    // both lanes and ordered on the sub-band stream (like r_gin); block 0's stream maxima are written with the lane's input (sbx)
    TcnWeights tcn_sb;
    DevBuf sb_fc;
    TcnScratch sb_scratch;
    int64_t launches = 0;
    int last_impl = 0;
    // tuning knobs, read ONCE at fsn_model_create (never on the forward path): FSN_LSTM_IMPL overrides cfg.lstm_impl,
    // FSN_NO_WS=1 keeps the full-band LSTM of fullsubnet.Model off the weight-stationary kernel
    int env_impl = 0;
    // FSN_FRONT_OVERLAP=1: the pipelined entry points run the front end of batch i+1 concurrently with the sub-band LSTM of batch i
    // (two lanes, two streams).  Off by default: no gain at the flagship size on the H100 (DESIGN.md §4), the LSTM occupies every SM.
    bool env_front_overlap = false;
    int env_pdl = -1;                                  // FSN_PDL: 0 / 1 / -1 (auto: small batches only)
    double ws_cap_bytes = 24e9;                        // FSN_WS_CAP_GB: larger batches are run as sub-batches (plain forward entry points)
    int env_sb_window = 0;                             // FSN_SB_WINDOW: force a sub-band time window of this many frames (multiple of 32)
    int env_sb_chunk = 0;                              // FSN_SB_CHUNK: run the sub-band TCN in chunks of this many bins (>= num_freqs: unchunked)
    Plan plan;                                         // plan of the last plain forward
    bool env_no_ws = false;
    int env_gin_tile_n = 0;                            // FSN_GIN_GEMM=128: the input-projection GEMM on 128 x 128 tiles (GemmF16Launch::tile_n)
    // pipelined execution: front-end stream, LSTM stream (higher priority), copy-in / copy-out streams, per-slot events
    cudaStream_t s_front = nullptr, s_lstm = nullptr, s_in = nullptr, s_out = nullptr;
    cudaEvent_t ev_in = nullptr, ev_plain = nullptr;   // caller's inputs ready / last plain forward finished
    bool plain_pending = false;
    cudaEvent_t ev_h2d[2] = {}, ev_d2h[2] = {}, ev_done[2] = {};   // per staging slot: inputs copied / mask copied out / forward finished
    bool d2h_used[2] = {false, false};
    DevBuf a_in[2][3], a_out[2];
    int64_t nsub = 0;
    static const int NEV = 32;
    cudaEvent_t ev0[NEV] = {}, ev1[NEV] = {};               // sub-band LSTM start / end
    cudaEvent_t evf0[NEV] = {}, evf1[NEV] = {};             // front end start / end (same ring index)
    int64_t nfwd = 0;                                 // forwards whose LSTM events were recorded
    // ragged forwards: pinned staging slots of the per-sample extents.  A slot is refilled only after the event recorded behind its
    // H2D copy has fired, so the caller's frames array is free when the call returns and no stream has to be synchronised.
    static const int NLEN = 4;
    struct LenSlot { int32_t* h = nullptr; size_t cap = 0; cudaEvent_t ev = nullptr; bool used = false; } len_slot[NLEN];
    int64_t nlen = 0;
};

// ---------------------------------------------------------------------------------------------
// parameter registry: exactly the reference's state_dict (SURVEY.md 8b)
// ---------------------------------------------------------------------------------------------
static void add(std::vector<ParamSpec>& v, const std::string& k, int64_t n) { v.push_back({k, n}); }

static void lstm_specs(std::vector<ParamSpec>& v, const std::string& pre, int I, int H, int L, int O, int G) {
    for (int l = 0; l < L; ++l) {                                   // G = 4 gate blocks for nn.LSTM, 3 for nn.GRU
        const std::string s = std::to_string(l);
        add(v, pre + ".sequence_model.weight_ih_l" + s, (int64_t)G * H * (l == 0 ? I : H));
        add(v, pre + ".sequence_model.weight_hh_l" + s, (int64_t)G * H * H);
        add(v, pre + ".sequence_model.bias_ih_l" + s, G * H);
        add(v, pre + ".sequence_model.bias_hh_l" + s, G * H);
    }
    add(v, pre + ".fc_output_layer.weight", (int64_t)O * H);
    add(v, pre + ".fc_output_layer.bias", O);
}

// SequenceModel(C, O, sequence_model="TCN"): 8 TCNBlock(C -> 512 -> C) + Linear(C -> O) (sequence_model.py:47-58,80-81)
static void tcn_specs(std::vector<ParamSpec>& v, const std::string& pre, int C, int O) {
    for (int i = 0; i < 8; ++i) {
        const std::string q = pre + ".sequence_model." + std::to_string(i);
        add(v, q + ".conv1x1.weight", (int64_t)512 * C);
        add(v, q + ".conv1x1.bias", 512);
        add(v, q + ".prelu1.weight", 1);
        add(v, q + ".norm1.weight", 512);
        add(v, q + ".norm1.bias", 512);
        add(v, q + ".depthwise_conv.weight", 512 * 3);
        add(v, q + ".depthwise_conv.bias", 512);
        add(v, q + ".prelu2.weight", 1);
        add(v, q + ".norm2.weight", 512);
        add(v, q + ".norm2.bias", 512);
        add(v, q + ".sconv.weight", (int64_t)C * 512);
        add(v, q + ".sconv.bias", C);
    }
    add(v, pre + ".fc_output_layer.weight", (int64_t)O * C);
    add(v, pre + ".fc_output_layer.bias", O);
}

// Channels of the sub-band input: a bin with 2 Ns neighbours of the magnitude, and with 2 Nf of each full-band output (3 in FullSubNet+)
static int sb_input_size(const fsn_config& c) {
    return (2 * c.sb_num_neighbors + 1) + (c.model_kind == FSN_KIND_PLUS ? 3 : 1) * (2 * c.fb_num_neighbors + 1);
}

// The layer-wise kernels (k_lstm_tc5r.cu) take this geometry (hidden % 64 == 0 and <= 512, output_size 2, input <= 64): their weights are packed
static bool tc5r_ok(const fsn_config& c) {
    return !c.sb_tcn && lstm_tc5r_supported(c.sb_hidden, c.output_size) && sb_input_size(c) <= 64;
}

// The sub-band LSTM runs layer-wise (else on the generic mma.sync kernel): lstm_impl = auto or tcgen05 (FSN_LSTM_TCGEN05, the historical
// name of the tensor-core path) on a geometry those kernels take.  env_impl: FSN_LSTM_IMPL or 0.
static bool runs_layerwise(const fsn_config& c, int env_impl) {
    const int impl = env_impl ? env_impl : c.lstm_impl;
    return tc5r_ok(c) && (impl == FSN_LSTM_AUTO || impl == FSN_LSTM_TCGEN05);
}

static void build_specs(fsn_model* m) {
    const fsn_config& c = m->cfg;
    const int F = c.num_freqs;
    auto& v = m->specs;
    m->Isb = sb_input_size(c);
    if (c.model_kind == FSN_KIND_PLUS) {
        const char* sfx[3] = {"", "_real", "_imag"};
        const char* cn[3] = {"smallConv1d", "middleConv1d", "largeConv1d"};
        for (int b = 0; b < 3; ++b) {
            const std::string p = std::string("channel_attention") + sfx[b];
            if (c.channel_attention == FSN_ATTN_ECA) { add(v, p + ".conv.weight", 3); continue; }
            if (c.channel_attention == FSN_ATTN_TSSE) {
                for (int i = 0; i < 3; ++i) {
                    add(v, p + "." + cn[i] + ".0.weight", (int64_t)F * c.kersize[i]);
                    add(v, p + "." + cn[i] + ".0.bias", F);
                }
                add(v, p + ".feature_concate_fc.weight", 3);
                add(v, p + ".feature_concate_fc.bias", 1);
            }
            add(v, p + ".fc1.weight", (int64_t)(F / 2) * F);
            add(v, p + ".fc1.bias", F / 2);
            add(v, p + ".fc2.weight", (int64_t)F * (F / 2));
            add(v, p + ".fc2.bias", F);
        }
        for (int b = 0; b < 3; ++b) tcn_specs(v, std::string("fb_model") + sfx[b], F, F);
    } else {
        lstm_specs(v, "fb_model", F, c.fb_hidden, c.num_layers, F, c.rnn_type == FSN_RNN_GRU ? 3 : 4);
    }
    if (c.sb_tcn) tcn_specs(v, "sb_model", m->Isb, c.output_size);       // hidden width 512: sb_hidden and num_layers are unused
    else lstm_specs(v, "sb_model", m->Isb, c.sb_hidden, c.num_layers, c.output_size, c.rnn_type == FSN_RNN_GRU ? 3 : 4);
}

// ---------------------------------------------------------------------------------------------
// packing
// ---------------------------------------------------------------------------------------------
static uint16_t h_bits(float f) { __half h = __float2half_rn(f); uint16_t b; std::memcpy(&b, &h, 2); return b; }

// mma.sync fragment order (k_lstm_mma.cu): [group of 8 units][k16 step][lane][i.b0 i.b1 f.b0 f.b1 | g.b0 g.b1 o.b0 o.b1]
static void pack_mma_layer(const float* w_ih, const float* w_hh, int Kin, int Kin_pad, int H, std::vector<uint32_t>& out) {
    const int K = Kin_pad + H, ksteps = K / 16, groups = H / 8;
    out.assign((size_t)groups * ksteps * 32 * 8, 0u);
    auto wcat = [&](int row, int k) -> float {
        if (k < Kin_pad) return k < Kin ? w_ih[(size_t)row * Kin + k] : 0.f;
        return w_hh[(size_t)row * H + (k - Kin_pad)];
    };
    for (int g = 0; g < groups; ++g)
        for (int ks = 0; ks < ksteps; ++ks)
            for (int lane = 0; lane < 32; ++lane) {
                uint32_t* dst = &out[(((size_t)g * ksteps + ks) * 32 + lane) * 8];
                const int n = g * 8 + lane / 4, k0 = ks * 16 + (lane % 4) * 2;
                for (int q = 0; q < 4; ++q) {
                    const int row = q * H + n;
                    dst[2 * q] = (uint32_t)h_bits(wcat(row, k0)) | ((uint32_t)h_bits(wcat(row, k0 + 1)) << 16);
                    dst[2 * q + 1] = (uint32_t)h_bits(wcat(row, k0 + 8)) | ((uint32_t)h_bits(wcat(row, k0 + 9)) << 16);
                }
            }
}

static int upload(DevBuf& b, const void* src, size_t bytes) {
    int e = b.ensure(bytes, false);
    if (e) return e;
    return (int)cudaMemcpy(b.p, src, bytes, cudaMemcpyHostToDevice);
}

// nn.GRU (sequence_model.py:39-46) on the LSTM kernels: rewrite the (r, z, n) parameters as four pseudo-gate blocks
//   r: [W_ir | W_hr], z: [W_iz | W_hz], n_x: [W_in | 0], n_h: [0 | W_hn]   (biases alike)
// in the nn.LSTM layout; the expanded arrays replace the originals in m->host, so every packer downstream is unchanged.
static void expand_gru(fsn_model* m, const std::string& pre, int I, int H, int L) {
    for (int l = 0; l < L; ++l) {
        const std::string s = std::to_string(l);
        const int K = (l == 0) ? I : H;
        auto& wi = m->host[pre + ".sequence_model.weight_ih_l" + s];
        auto& wh = m->host[pre + ".sequence_model.weight_hh_l" + s];
        auto& bi = m->host[pre + ".sequence_model.bias_ih_l" + s];
        auto& bh = m->host[pre + ".sequence_model.bias_hh_l" + s];
        // each array is expanded on its own size, so a later fsn_model_set_param of a single key re-expands just that key
        if (wi.size() == (size_t)3 * H * K) {                       // r, z, n_x input blocks; the n_h input block stays zero
            std::vector<float> w4((size_t)4 * H * K, 0.f);
            std::copy(wi.begin(), wi.end(), w4.begin());
            wi.swap(w4);
        }
        if (wh.size() == (size_t)3 * H * H) {                       // r, z recurrent blocks; n_x recurrent block zero; n_h <- W_hn
            std::vector<float> w4((size_t)4 * H * H, 0.f);
            std::copy(wh.begin(), wh.begin() + (size_t)2 * H * H, w4.begin());
            std::copy(wh.begin() + (size_t)2 * H * H, wh.end(), w4.begin() + (size_t)3 * H * H);
            wh.swap(w4);
        }
        if (bi.size() == (size_t)3 * H) { bi.resize((size_t)4 * H, 0.f); }
        if (bh.size() == (size_t)3 * H) {
            std::vector<float> b4((size_t)4 * H, 0.f);
            std::copy(bh.begin(), bh.begin() + 2 * H, b4.begin());
            std::copy(bh.begin() + 2 * H, bh.end(), b4.begin() + 3 * H);
            bh.swap(b4);
        }
    }
}

static int pack_lstm(fsn_model* m, const std::string& pre, int I, int Ipad, int H, int L, DevBuf* frag, DevBuf* bias) {
    for (int l = 0; l < L; ++l) {
        const std::string s = std::to_string(l);
        const auto& wi = m->host[pre + ".sequence_model.weight_ih_l" + s];
        const auto& wh = m->host[pre + ".sequence_model.weight_hh_l" + s];
        const auto& bi = m->host[pre + ".sequence_model.bias_ih_l" + s];
        const auto& bh = m->host[pre + ".sequence_model.bias_hh_l" + s];
        std::vector<uint32_t> f;
        pack_mma_layer(wi.data(), wh.data(), l == 0 ? I : H, l == 0 ? Ipad : H, H, f);
        int e = upload(frag[l], f.data(), f.size() * 4);
        if (e) return e;
        std::vector<float> b(4 * H);
        for (int i = 0; i < 4 * H; ++i) b[i] = bi[i] + bh[i];
        e = upload(bias[l], b.data(), b.size() * 4);
        if (e) return e;
    }
    return 0;
}


// tf32 rounding (round-to-nearest on the 13 dropped mantissa bits) so the tensor core's truncation is exact
static float to_tf32(float x) {
    uint32_t u; std::memcpy(&u, &x, 4);
    if ((u & 0x7f800000u) == 0x7f800000u) return x;
    u += 0x00000fffu + ((u >> 13) & 1u);
    u &= 0xffffe000u;
    float y; std::memcpy(&y, &u, 4);
    return y;
}

// TCN block weights for the wgmma GEMMs (k_gemm_tc5.cu): channel dim C padded to Cp (multiple of 32), the branches (key prefixes
// pre[b] = "<module>.sequence_model.") stacked, gLN2 folded into the second 1x1 convolution:
//   conv(W2, gLN(y)) = rstd * (W2 diag(gamma2)) y - mean * rstd * s1 + s2,  s1[n] = sum_c W2'[n,c],  s2[n] = sum_c W2[n,c] beta2[c]
// W1 [8][nbr][512][Cp] tf32, W2' [8][nbr][Cp][512] fp16, s1 / s2 + conv bias [8][nbr][Cp]; tensor maps per block: W1 in 128-row
// boxes, W2' in NT-row boxes.
static int pack_tcn_blocks(fsn_model* m, TcnWeights& w, const char* name, const std::vector<std::string>& pre, int C, int Cp) {
    const int nbr = (int)pre.size(), Hd = 512;
    w.name = name; w.pre = pre; w.nbr = nbr; w.C = C; w.Cp = Cp;
    // N tile of the Cp-wide GEMMs: 64 or 128 columns (the last tile of a branch may overhang; those columns are not stored)
    w.NT = Cp <= 64 ? 64 : 128;
    w.ntiles = (Cp + w.NT - 1) / w.NT;
    std::vector<float> W1((size_t)8 * nbr * Hd * Cp, 0.f);
    std::vector<__half> W2((size_t)8 * nbr * Cp * Hd, __float2half_rn(0.f));     // second 1x1 conv: fp16 operands (hidden activations are fp16)
    std::vector<float> S1((size_t)8 * nbr * Cp, 0.f), S2b((size_t)8 * nbr * Cp, 0.f);
    for (int blk = 0; blk < 8; ++blk)
        for (int b = 0; b < nbr; ++b) {
            const std::string q = pre[b] + std::to_string(blk) + ".";
            const auto& w1 = m->host[q + "conv1x1.weight"];
            const auto& w2 = m->host[q + "sconv.weight"];
            const auto& b2 = m->host[q + "sconv.bias"];
            const auto& g2 = m->host[q + "norm2.weight"];
            const auto& be2 = m->host[q + "norm2.bias"];
            float* d1 = &W1[((size_t)blk * nbr + b) * Hd * Cp];
            for (int o = 0; o < Hd; ++o)
                for (int k = 0; k < C; ++k) d1[(size_t)o * Cp + k] = to_tf32(w1[(size_t)o * C + k]);
            __half* d2 = &W2[((size_t)blk * nbr + b) * Cp * Hd];
            for (int n = 0; n < C; ++n) {
                double s1 = 0, s2 = 0;
                for (int k = 0; k < Hd; ++k) {
                    const __half wh = __float2half_rn(w2[(size_t)n * Hd + k] * g2[k]);
                    const float wf = __half2float(wh);
                    d2[(size_t)n * Hd + k] = wh;
                    s1 += (double)wf;
                    s2 += (double)w2[(size_t)n * Hd + k] * (double)be2[k];
                }
                S1[((size_t)blk * nbr + b) * Cp + n] = (float)s1;
                S2b[((size_t)blk * nbr + b) * Cp + n] = (float)(s2 + (double)b2[n]);
            }
        }
    if (upload(w.W1, W1.data(), W1.size() * 4) || upload(w.W2, W2.data(), W2.size() * sizeof(__half)) ||
        upload(w.S1, S1.data(), S1.size() * 4) || upload(w.S2b, S2b.data(), S2b.size() * 4))
        return fail(FSN_ECUDA, "upload of the %s weights failed", name);
    for (int blk = 0; blk < 8; ++blk) {
        if (make_tmap_f32_2d(w.mapW1[blk], static_cast<float*>(w.W1.p) + (size_t)blk * nbr * Hd * Cp, nbr * Hd, Cp, 128) ||
            make_tmap_f16_2d(w.mapW2[blk], static_cast<__half*>(w.W2.p) + (size_t)blk * nbr * Cp * Hd, nbr * Cp, Hd, w.NT))
            return fail(FSN_ECUDA, "cuTensorMapEncodeTiled failed for the %s weights", name);
    }
    return FSN_OK;
}

// the three full-band TCNs of FullSubNet+ (F channels each) and their output Linear
static int pack_tcn5(fsn_model* m) {
    const fsn_config& c = m->cfg;
    const int F = c.num_freqs, Cp = (F + 31) / 32 * 32;
    const char* sfx[3] = {"", "_real", "_imag"};
    std::vector<std::string> pre;
    for (int b = 0; b < 3; ++b) pre.push_back(std::string("fb_model") + sfx[b] + ".sequence_model.");
    int rc = pack_tcn_blocks(m, m->tcn_fb, "full-band TCN", pre, F, Cp);
    if (rc) return rc;
    std::vector<float> Wfc((size_t)3 * Cp * Cp, 0.f), Bfc((size_t)3 * Cp, 0.f);
    for (int b = 0; b < 3; ++b) {
        const auto& w = m->host[std::string("fb_model") + sfx[b] + ".fc_output_layer.weight"];
        const auto& bb = m->host[std::string("fb_model") + sfx[b] + ".fc_output_layer.bias"];
        for (int n = 0; n < F; ++n) {
            for (int k = 0; k < F; ++k) Wfc[((size_t)b * Cp + n) * Cp + k] = to_tf32(w[(size_t)n * F + k]);
            Bfc[(size_t)b * Cp + n] = bb[n];
        }
    }
    if (upload(m->fb_fc, Wfc.data(), Wfc.size() * 4) || upload(m->fb_fc_b, Bfc.data(), Bfc.size() * 4))
        return fail(FSN_ECUDA, "upload of the TCN weights failed");
    if (make_tmap_f32_2d(m->map_fb_fc, m->fb_fc.p, 3 * Cp, Cp, m->tcn_fb.NT)) return fail(FSN_ECUDA, "cuTensorMapEncodeTiled failed (fc)");
    m->tcn5 = true;
    return FSN_OK;
}

// the sub-band TCN (sequence_model = "TCN"): one branch of Isb <= 64 channels padded to 64 -- the GLN_HEAD epilogue needs a row's
// channels in one 64-column N tile -- and its Linear(Isb -> O) as [O][64] fp32 (read by that epilogue)
static int pack_sb_tcn(fsn_model* m) {
    const int I = m->Isb, O = m->cfg.output_size;
    int rc = pack_tcn_blocks(m, m->tcn_sb, "sub-band TCN", {"sb_model.sequence_model."}, I, 64);
    if (rc) return rc;
    std::vector<float> fc((size_t)O * 64, 0.f);
    const auto& w = m->host["sb_model.fc_output_layer.weight"];
    for (int o = 0; o < O; ++o)
        for (int k = 0; k < I; ++k) fc[(size_t)o * 64 + k] = w[(size_t)o * I + k];
    if (upload(m->sb_fc, fc.data(), fc.size() * 4)) return fail(FSN_ECUDA, "upload of the sub-band TCN head failed");
    return FSN_OK;
}

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" int fsn_version(void) { return 100; }
extern "C" const char* fsn_last_error(void) { return g_err; }

extern "C" int fsn_model_create(const fsn_config* cfg, fsn_model** out) {
    if (!cfg || !out) return fail(FSN_EINVAL, "null argument");
    const fsn_config& c = *cfg;
    if (c.model_kind != FSN_KIND_PLUS && c.model_kind != FSN_KIND_FSN) return fail(FSN_EINVAL, "unknown model_kind %d", c.model_kind);
    if (c.num_freqs > 2048) return fail(FSN_EINVAL, "num_freqs > 2048 is not supported");
    if (c.num_freqs < 4 || c.look_ahead < 0 || c.sb_num_neighbors < 0 || c.fb_num_neighbors < 0) return fail(FSN_EINVAL, "bad geometry");
    if (c.sb_num_neighbors >= c.num_freqs || c.fb_num_neighbors >= c.num_freqs) return fail(FSN_EINVAL, "reflect padding needs neighbors < num_freqs");
    if (c.sb_tcn != 0 && c.sb_tcn != 1) return fail(FSN_EINVAL, "sb_tcn must be 0 or 1");
    if (c.sb_tcn && c.model_kind != FSN_KIND_PLUS) return fail(FSN_EINVAL, "a TCN sub-band model needs FullSubNet_Plus (fullsubnet.Model asserts GRU / LSTM)");
    if (c.num_layers < 1 || c.num_layers > 4) return fail(FSN_EINVAL, "num_layers must be 1..4");
    if (!c.sb_tcn && (c.sb_hidden % 16 || c.sb_hidden < 16)) return fail(FSN_EINVAL, "sb_model_hidden_size must be a multiple of 16");
    if (c.model_kind == FSN_KIND_FSN && (c.fb_hidden % 16 || c.fb_hidden < 16)) return fail(FSN_EINVAL, "fb_model_hidden_size must be a multiple of 16");
    if (c.output_size < 1 || c.output_size > 8) return fail(FSN_EINVAL, "output_size must be 1..8");
    if (c.rnn_type != FSN_RNN_LSTM && c.rnn_type != FSN_RNN_GRU) return fail(FSN_EINVAL, "unknown rnn_type %d", c.rnn_type);
    if (c.norm_type < FSN_NORM_OFFLINE_LAPLACE || c.norm_type > FSN_NORM_CUMULATIVE_LAYER) return fail(FSN_EINVAL, "unknown norm_type %d", c.norm_type);
    if (c.model_kind == FSN_KIND_PLUS) {
        if (c.channel_attention < FSN_ATTN_TSSE || c.channel_attention > FSN_ATTN_ECA) return fail(FSN_EINVAL, "unknown channel_attention %d", c.channel_attention);
        if (c.subband_num > 1 && c.channel_attention != FSN_ATTN_ECA)
            return fail(FSN_EINVAL, "subband_num > 1 needs the ECA attention (the reference forward raises for the others)");
        if (c.subband_num < 0 || c.subband_num > c.num_freqs / 2) return fail(FSN_EINVAL, "bad subband_num %d", c.subband_num);
        for (int i = 0; i < 3; ++i)
            if (c.channel_attention == FSN_ATTN_TSSE && (c.kersize[i] < 1 || c.kersize[i] > 16)) return fail(FSN_EINVAL, "kersize must be in 1..16");
    }
    const int isb = sb_input_size(c);
    if (isb > 64) return fail(FSN_EINVAL, "sub-band input size %d > 64 not supported", isb);
    int sb_window = 0;
    if (const char* e = getenv("FSN_SB_WINDOW"); e && *e) {
        char* end = nullptr;
        const long w = strtol(e, &end, 10);
        if (*end || w < 32 || w % 32 || w > (1L << 30)) return fail(FSN_EINVAL, "FSN_SB_WINDOW=%s: the window must be a positive multiple of 32 frames", e);
        sb_window = (int)w;
    }
    int sb_chunk = 0;
    if (const char* e = getenv("FSN_SB_CHUNK"); e && *e) {
        char* end = nullptr;
        const long w = strtol(e, &end, 10);
        if (*end || w < 1) return fail(FSN_EINVAL, "FSN_SB_CHUNK=%s: the chunk must be a positive number of bins", e);
        sb_chunk = w < c.num_freqs ? (int)w : c.num_freqs;
    }
    // FSN_GIN_GEMM: N tile of the deeper layers' input-projection GEMM.  Unset or 256: 128 x 256 tiles on CTA pairs wherever the shape
    // allows; 128: the 128 x 128 kernel everywhere (A/B runs in one process; both compute the same bits)
    int gin_tile_n = 0;
    if (const char* e = getenv("FSN_GIN_GEMM"); e && *e) {
        if (strcmp(e, "128") && strcmp(e, "256")) return fail(FSN_EINVAL, "FSN_GIN_GEMM=%s: the N tile must be 128 or 256", e);
        gin_tile_n = atoi(e);
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(FSN_ECUDA, "no CUDA device: fsnplus_b200 has no CPU fallback");
    fsn_model* m = new fsn_model();
    m->cfg = c;
    m->env_gin_tile_n = gin_tile_n;
    m->env_sb_window = sb_window;
    m->env_sb_chunk = sb_chunk;
    { const char* e = getenv("FSN_LSTM_IMPL"); if (e && *e) m->env_impl = atoi(e); }
    { const char* e = getenv("FSN_NO_WS"); m->env_no_ws = e && atoi(e) != 0; }
    { const char* e = getenv("FSN_FRONT_OVERLAP"); m->env_front_overlap = e && atoi(e) != 0; }
    // FSN_PDL: programmatic dependent launch of the ~30 kernels of the front-end chain.  0 = never, 1 = always, unset = only for small
    // batches, where the forward is launch-latency-bound; for large batches a denser front end leaves no gaps for the side stream's
    // iSTFT kernels of the pipelined entry points.
    { const char* e = getenv("FSN_PDL"); m->env_pdl = e ? (atoi(e) != 0 ? 1 : 0) : -1; }
    { const char* e = getenv("FSN_WS_CAP_GB"); if (e && atof(e) > 0) m->ws_cap_bytes = atof(e) * 1e9; }
    build_specs(m);
    for (int i = 0; i < fsn_model::NEV; ++i) { cudaEventCreate(&m->ev0[i]); cudaEventCreate(&m->ev1[i]); cudaEventCreate(&m->evf0[i]); cudaEventCreate(&m->evf1[i]); }
    { cudaDeviceProp prop; int dev = 0; cudaGetDevice(&dev); if (cudaGetDeviceProperties(&prop, dev) == cudaSuccess) m->num_sms = prop.multiProcessorCount; }
    *out = m;
    return FSN_OK;
}

static void release_ws(fsn_model& m);

extern "C" void fsn_model_destroy(fsn_model* m) {
    if (!m) return;
    cudaDeviceSynchronize();
    release_ws(*m);
    DevBuf* all[] = {&m->arena, &m->stage_in[0], &m->stage_in[1], &m->stage_in[2], &m->stage_out, &m->fb_fc, &m->fb_fc_b, &m->sb_fc};
    for (auto* b : all) b->release();
    m->tcn_fb.release(); m->tcn_sb.release();
    for (auto& ln : m->lane) {
        if (ln.ev_front) cudaEventDestroy(ln.ev_front);
        if (ln.ev_lstm) cudaEventDestroy(ln.ev_lstm);
    }
    for (int i = 0; i < 4; ++i) { m->r_stream[i].release(); m->r_wih[i].release(); m->r_bias[i].release(); }
    if (m->s_front) { cudaStreamDestroy(m->s_front); cudaStreamDestroy(m->s_lstm); cudaEventDestroy(m->ev_in); }
    if (m->ev_plain) cudaEventDestroy(m->ev_plain);
    if (m->s_in) { cudaStreamDestroy(m->s_in); cudaStreamDestroy(m->s_out); for (int i = 0; i < 2; ++i) { cudaEventDestroy(m->ev_h2d[i]); cudaEventDestroy(m->ev_d2h[i]); cudaEventDestroy(m->ev_done[i]); } }
    for (int i = 0; i < 2; ++i) { m->a_out[i].release(); for (int j = 0; j < 3; ++j) m->a_in[i][j].release(); }
    for (int i = 0; i < fsn_model::NEV; ++i) {
        if (m->ev0[i]) cudaEventDestroy(m->ev0[i]);
        if (m->ev1[i]) cudaEventDestroy(m->ev1[i]);
        if (m->evf0[i]) cudaEventDestroy(m->evf0[i]);
        if (m->evf1[i]) cudaEventDestroy(m->evf1[i]);
    }
    for (int i = 0; i < 4; ++i) { m->sb_frag[i].release(); m->sb_bias[i].release(); m->fb_frag[i].release(); m->fb_bias[i].release(); }
    for (auto& ls : m->len_slot) {
        if (ls.h) cudaFreeHost(ls.h);
        if (ls.ev) cudaEventDestroy(ls.ev);
    }
    delete m;
}

extern "C" int fsn_model_num_params(const fsn_model* m) { return m ? (int)m->specs.size() : 0; }
extern "C" int fsn_model_param_info(const fsn_model* m, int i, const char** key, int64_t* numel) {
    if (!m || i < 0 || i >= (int)m->specs.size()) return fail(FSN_EINVAL, "bad index");
    if (key) *key = m->specs[i].key.c_str();
    if (numel) *numel = m->specs[i].numel;
    return FSN_OK;
}

extern "C" int fsn_model_set_param(fsn_model* m, const char* key, const float* h, int64_t numel) {
    if (!m || !key || !h) return fail(FSN_EINVAL, "null argument");
    for (const auto& s : m->specs)
        if (s.key == key) {
            if (s.numel != numel) return fail(FSN_EINVAL, "size mismatch for %s: expected %lld, got %lld", key, (long long)s.numel, (long long)numel);
            m->host[key].assign(h, h + numel);
            m->finalized = false;
            return FSN_OK;
        }
    return fail(FSN_EINVAL, "unexpected key %s", key);
}

extern "C" int fsn_model_finalize(fsn_model* m) {
    if (!m) return fail(FSN_EINVAL, "null model");
    const fsn_config& c = m->cfg;
    for (const auto& s : m->specs)
        if (!m->host.count(s.key)) return fail(FSN_ESTATE, "missing parameter %s", s.key.c_str());
    if (c.rnn_type == FSN_RNN_GRU) {
        if (!c.sb_tcn) expand_gru(m, "sb_model", m->Isb, c.sb_hidden, c.num_layers);
        if (c.model_kind == FSN_KIND_FSN) expand_gru(m, "fb_model", c.num_freqs, c.fb_hidden, c.num_layers);
    }
    size_t total = 0;
    for (const auto& s : m->specs) total += (m->host[s.key].size() * 4 + 255) & ~(size_t)255;
    if (m->arena.ensure(total, false)) return fail(FSN_ECUDA, "cudaMalloc of %zu bytes failed", total);
    size_t off = 0;
    for (const auto& s : m->specs) {
        const auto& hv = m->host[s.key];
        float* d = reinterpret_cast<float*>(static_cast<char*>(m->arena.p) + off);
        CK(cudaMemcpy(d, hv.data(), hv.size() * 4, cudaMemcpyHostToDevice));
        m->dev[s.key] = d;
        off += (hv.size() * 4 + 255) & ~(size_t)255;
    }
    if (!c.sb_tcn && pack_lstm(m, "sb_model", m->Isb, 64, c.sb_hidden, c.num_layers, m->sb_frag, m->sb_bias)) return fail(FSN_ECUDA, "packing sb_model failed");
    if (c.model_kind == FSN_KIND_FSN) {
        const int Ipad = (c.num_freqs + 15) / 16 * 16;
        if (pack_lstm(m, "fb_model", c.num_freqs, Ipad, c.fb_hidden, c.num_layers, m->fb_frag, m->fb_bias)) return fail(FSN_ECUDA, "packing fb_model failed");
    }
    if (tc5r_ok(c)) {
        const int H = c.sb_hidden;
        for (int l = 0; l < c.num_layers; ++l) {
            const std::string q = "sb_model.sequence_model.", sl = std::to_string(l);
            const int Kin = (l == 0) ? m->Isb : H, Kpad = (l == 0) ? 64 : H;
            std::vector<uint16_t> st, wp;
            std::vector<float> bp;
            lstm_tc5r_pack_layer(H, Kin, Kpad, m->host[q + "weight_ih_l" + sl].data(), m->host[q + "weight_hh_l" + sl].data(),
                                 m->host[q + "bias_ih_l" + sl].data(), m->host[q + "bias_hh_l" + sl].data(), c.rnn_type == FSN_RNN_GRU, st, wp, bp);
            if (l == 0) {                                                   // first layer: [W_ih | W_hh] blocks, the input projection is in the recurrence
                st.assign((size_t)(H / 32) * (1 + H / 64) * 8192, 0);
                lstm_tc5_pack_first_layer(Kin, H, m->host[q + "weight_ih_l0"].data(), m->host[q + "weight_hh_l0"].data(), st.data());
            } else {                                                        // deeper layers: W_hh blocks + the input-projection GEMM's matrix
                lstm_tc5r_gin_order(H, Kpad, wp);
                if (upload(m->r_wih[l], wp.data(), wp.size() * 2)) return fail(FSN_ECUDA, "upload of the layer-wise LSTM weights failed");
            }
            if (upload(m->r_stream[l], st.data(), st.size() * 2) || upload(m->r_bias[l], bp.data(), bp.size() * 4))
                return fail(FSN_ECUDA, "upload of the layer-wise LSTM weights failed");
        }
    }
    if (c.model_kind == FSN_KIND_PLUS) {
        int rc = pack_tcn5(m);
        if (rc) return rc;
    }
    if (c.sb_tcn) {
        int rc = pack_sb_tcn(m);
        if (rc) return rc;
    }
    m->finalized = true;
    return FSN_OK;
}

static const float* P(fsn_model* m, const std::string& k) { return m->dev.at(k); }


static void fill_ws(fsn_model* m, LstmWsLaunch& w) {
    const fsn_config& c = m->cfg;
    for (int l = 0; l < c.num_layers; ++l) {
        const std::string s = std::to_string(l);
        w.w_ih[l] = P(m, "fb_model.sequence_model.weight_ih_l" + s); w.w_hh[l] = P(m, "fb_model.sequence_model.weight_hh_l" + s);
        w.b_ih[l] = P(m, "fb_model.sequence_model.bias_ih_l" + s); w.b_hh[l] = P(m, "fb_model.sequence_model.bias_hh_l" + s);
    }
    w.L = c.num_layers; w.H = c.fb_hidden; w.I = c.num_freqs; w.Ipad = (c.num_freqs + 15) / 16 * 16; w.fast = c.fast_math; w.gru = c.rnn_type == FSN_RNN_GRU;
}

// The implementation the sub-band LSTM reports (last_impl), and the one a forced lstm_impl names in its error
static int pick_impl(const fsn_model* m) {
    const int impl = m->env_impl ? m->env_impl : m->cfg.lstm_impl;
    return runs_layerwise(m->cfg, m->env_impl) ? FSN_LSTM_TCGEN05 : impl == FSN_LSTM_AUTO ? FSN_LSTM_MMA : impl;
}

// Encode the tensor maps of TCN w's scratch over `rows` rows
static int map_tcn_scratch(TcnScratch& sc, const TcnWeights& w, long long rows) {
    if (make_tmap_f32_2d(sc.mapXa, sc.xa.p, rows, w.Cp, 128) || make_tmap_f32_2d(sc.mapXb, sc.xb.p, rows, w.Cp, 128) ||
        make_tmap_f16_2d(sc.mapY2, sc.y2.p, rows, 512, 128))
        return fail(FSN_ECUDA, "cuTensorMapEncodeTiled failed for the %s", w.name);
    return FSN_OK;
}

// Bytes of every forward workspace buffer for a batch of B clips of T frames, the sub-band images and the layer-wise path's Gin / layer
// output sized by the window Tw (0: the whole clip), the sub-band TCN's input and scratch by the bin chunk Fc (0: all bins).  One field
// per entry of the table WS; ensure_ws allocates exactly these sizes, so the plan's count is what a forward holds.
struct WsSizes {
    size_t fbin = 0, fbout = 0, mu = 0, sigma = 0, tsse_scale = 0, sb_rowsum = 0, xn = 0, tlen = 0;       // lane: front end, ragged extents
    size_t sbx = 0, ximg = 0;                                                   // lane: sub-band TCN input, or the sub-band images
    size_t x0 = 0, xr = 0, tcn_xa = 0, tcn_xb = 0, tcn_y1 = 0, tcn_y2 = 0, tcn_stats = 0;   // lane, FullSubNet+: the full-band TCN
    size_t magpad = 0, fbx = 0, hseq = 0;                                       // lane, fullsubnet.Model
    size_t cstate = 0, r_gin = 0, r_hseq = 0, r_hstate = 0, sb_cum = 0;         // sub-band LSTM scratch
    size_t sb_xa = 0, sb_xb = 0, sb_y1 = 0, sb_y2 = 0, sb_stats = 0;            // sub-band TCN scratch
    size_t ws_h = 0, ws_bar = 0;                                                // fullsubnet.Model's weight-stationary h exchange, barrier
    size_t mask_tmp = 0;                                                        // the generic kernel's scratch mask: not counted
    size_t total() const;
};
static WsSizes ws_sizes(const fsn_config& c, bool layerwise, int B, int T, int Tw, int Fc = 0) {
    WsSizes z;
    const int F = c.num_freqs, Tp = T + c.look_ahead, Pp = (Tp + 3) & ~3, Ts = Tw ? Tw : Tp;
    const int nbr = (c.model_kind == FSN_KIND_PLUS) ? 3 : 1;
    const size_t rows = (size_t)B * F, ntiles = ((rows + 127) / 128 + 1) / 2 * 2;   // whole pairs of 128-row tiles (clusters of k_lstm_tc5r.cu)
    z.fbin = z.fbout = (size_t)nbr * B * F * Pp * 4;
    z.mu = z.sigma = (size_t)B * 4;
    z.tsse_scale = (size_t)nbr * B * F * 4 * (1 + tsse_row_floats());          // per-row scale | row statistics
    z.sb_rowsum = (size_t)B * 4 * F * 2 * 4;
    z.tlen = (size_t)3 * B * sizeof(int32_t);                                   // counted whether the forward is ragged or not
    if (c.norm_type != FSN_NORM_OFFLINE_LAPLACE) z.xn = (size_t)nbr * B * F * Tp * 4;
    if (c.sb_tcn) {
        const size_t seqs = (size_t)B * (Fc ? Fc : F), srows = seqs * Tp;      // the sequences of one chunk run
        z.sbx = srows * 64 * 4 + seqs * 4;                                      // input | block 0's stream maxima
        z.sb_xa = z.sb_xb = srows * 64 * 4; z.sb_y1 = z.sb_y2 = srows * 512 * sizeof(__half); z.sb_stats = tcn_stats_bytes(seqs);
    } else {
        z.ximg = ntiles * Ts * 16384;
    }
    int ra = 0;
    size_t cs = c.sb_tcn ? 0 : lstm_mma_cstate_bytes(c.num_layers, (int)rows, c.sb_hidden, &ra), cs5 = 0;
    if (layerwise) {
        const size_t M = ntiles * Ts * 128;
        cs5 = lstm_tc5r_cstate_bytes((int)ntiles, c.sb_hidden);
        if (c.num_layers > 1) { z.r_gin = M * 4 * c.sb_hidden * 2; z.r_hseq = M * c.sb_hidden * 2; }
        if (Tw) {                                                               // windowed: c / h of every layer carried to the next window
            cs5 *= c.num_layers;
            z.r_hstate = (size_t)c.num_layers * ntiles * 128 * c.sb_hidden * 2;
            if (c.norm_type == FSN_NORM_CUMULATIVE_LAPLACE || c.norm_type == FSN_NORM_CUMULATIVE_LAYER) z.sb_cum = rows * 2 * sizeof(double);
        }
    }
    if (c.model_kind == FSN_KIND_FSN) {
        int ra2 = 0;
        const size_t csf = lstm_mma_cstate_bytes(c.num_layers, B, c.fb_hidden, &ra2);
        if (csf > cs) cs = csf;
    }
    z.cstate = cs > cs5 ? cs : cs5;
    if (c.model_kind == FSN_KIND_PLUS) {
        const size_t trows = (size_t)3 * B * Tp, Cp = (size_t)(F + 31) / 32 * 32;   // pack_tcn5's Cp
        z.x0 = z.xr = trows * Cp * 4;
        z.tcn_xa = z.tcn_xb = trows * Cp * 4; z.tcn_y1 = z.tcn_y2 = trows * 512 * sizeof(__half); z.tcn_stats = tcn_stats_bytes((size_t)3 * B);
    } else {
        const size_t Ipad = (F + 15) / 16 * 16, rows_pad = (B + 63) / 64 * 64;
        z.magpad = (size_t)B * F * Pp * 4;
        z.fbx = (size_t)Tp * rows_pad * Ipad * 2;
        z.hseq = (size_t)B * c.fb_hidden * Pp * 4;
        z.ws_h = (size_t)c.num_layers * 2 * 64 * c.fb_hidden * 2; z.ws_bar = 64;   // counted whether that kernel runs or not
    }
    return z;
}

// The forward workspace: every buffer is one entry of WS.  ensure_ws sizes them (grows to the plan, gives back what exceeds it),
// release_ws frees them, fsn_model_workspace_bytes and the plan (WsSizes::total) count them, all from this table.  ensure_ws
// allocates in table order.
using Lane = fsn_model::Lane;
enum : unsigned {
    WS_LANE = 1,        // one per lane (else one for the model, shared by both lanes: the sub-band stage runs one batch at a time)
    WS_ZERO = 2,        // a fresh allocation is zero-filled, on the buffer's stream
    WS_SL = 4,          // ordered on the sub-band stream sl (else the front stream s)
    WS_REGEO = 8,       // a new geometry frees it first: the fresh zero-filled allocation keeps pad rows and columns zero
    WS_ON_USE = 16,     // allocated where it is used, not by ensure_ws: ragged extents, weight-stationary LSTM, the scratch mask
};
struct WsBuf {
    DevBuf& (*buf)(fsn_model&, Lane&);   // the buffer (a model's buffer ignores the lane)
    size_t WsSizes::*need;               // its bytes in the plan
    unsigned flags;
};
#define LANE_BUF(f) [](fsn_model&, Lane& ln) -> DevBuf& { return ln.f; }
#define MODEL_BUF(f) [](fsn_model& m, Lane&) -> DevBuf& { return m.f; }
static const WsBuf WS[] = {
    {LANE_BUF(fbin), &WsSizes::fbin, WS_LANE | WS_ZERO},
    {LANE_BUF(fbout), &WsSizes::fbout, WS_LANE | WS_ZERO},
    {LANE_BUF(mu), &WsSizes::mu, WS_LANE | WS_ZERO},
    {LANE_BUF(sigma), &WsSizes::sigma, WS_LANE | WS_ZERO},
    {LANE_BUF(tsse_scale), &WsSizes::tsse_scale, WS_LANE | WS_ZERO},
    {LANE_BUF(sb_rowsum), &WsSizes::sb_rowsum, WS_LANE | WS_ZERO},
    {LANE_BUF(xn), &WsSizes::xn, WS_LANE | WS_ZERO},
    {LANE_BUF(sbx), &WsSizes::sbx, WS_LANE | WS_REGEO},                            // fully written by the packer
    // the sub-band TCN's scratch: every buffer is fully written before it is read (the pad columns by the packer / the epilogue)
    {MODEL_BUF(sb_scratch.xa), &WsSizes::sb_xa, WS_SL},
    {MODEL_BUF(sb_scratch.xb), &WsSizes::sb_xb, WS_SL},
    {MODEL_BUF(sb_scratch.y1), &WsSizes::sb_y1, WS_SL},
    {MODEL_BUF(sb_scratch.y2), &WsSizes::sb_y2, WS_SL},
    {MODEL_BUF(sb_scratch.stats), &WsSizes::sb_stats, WS_SL},
    {LANE_BUF(ximg), &WsSizes::ximg, WS_LANE | WS_ZERO | WS_REGEO},                // rows beyond B*F and k >= I stay zero
    {MODEL_BUF(r_hstate), &WsSizes::r_hstate, WS_SL},
    {MODEL_BUF(sb_cum), &WsSizes::sb_cum, WS_SL},
    {MODEL_BUF(r_gin), &WsSizes::r_gin, WS_SL},
    {MODEL_BUF(r_hseq), &WsSizes::r_hseq, WS_SL},
    {MODEL_BUF(cstate), &WsSizes::cstate, WS_ZERO | WS_SL},
    {LANE_BUF(x0), &WsSizes::x0, WS_LANE | WS_ZERO | WS_REGEO},                    // pad columns of x0 (and of every stream) stay zero
    {LANE_BUF(xr), &WsSizes::xr, WS_LANE | WS_ZERO | WS_REGEO},
    {LANE_BUF(tcn.xa), &WsSizes::tcn_xa, WS_LANE | WS_ZERO | WS_REGEO},
    {LANE_BUF(tcn.xb), &WsSizes::tcn_xb, WS_LANE | WS_ZERO | WS_REGEO},
    {LANE_BUF(tcn.y1), &WsSizes::tcn_y1, WS_LANE | WS_ZERO | WS_REGEO},
    {LANE_BUF(tcn.y2), &WsSizes::tcn_y2, WS_LANE | WS_ZERO | WS_REGEO},
    {LANE_BUF(tcn.stats), &WsSizes::tcn_stats, WS_LANE | WS_ZERO | WS_REGEO},
    {LANE_BUF(magpad), &WsSizes::magpad, WS_LANE | WS_ZERO},
    {LANE_BUF(fbx), &WsSizes::fbx, WS_LANE | WS_ZERO},
    {LANE_BUF(hseq), &WsSizes::hseq, WS_LANE | WS_ZERO},
    {LANE_BUF(tlen), &WsSizes::tlen, WS_LANE | WS_ON_USE},                         // stage_lengths
    {MODEL_BUF(ws_h), &WsSizes::ws_h, WS_ON_USE},                                  // forward_impl
    {MODEL_BUF(ws_bar), &WsSizes::ws_bar, WS_ON_USE},
    {MODEL_BUF(mask_tmp), &WsSizes::mask_tmp, WS_ON_USE},                          // run_sb_lstm
};

size_t WsSizes::total() const {
    size_t n = 0;
    for (const WsBuf& e : WS) n += this->*e.need;
    return n;
}

static void release_lane(fsn_model& m, Lane& ln) {
    for (const WsBuf& e : WS) if (e.flags & WS_LANE) e.buf(m, ln).release();
    ln.geo = WsGeo{};
}
static void release_ws(fsn_model& m) {
    for (Lane& ln : m.lane) release_lane(m, ln);
    for (const WsBuf& e : WS) if (!(e.flags & WS_LANE)) e.buf(m, m.lane[0]).release();
}

// Length limits of one forward (B clips of T frames), from the 32-bit quantities of the kernels on every path: the depth-wise TCN
// convolution's grid covers T' in blocks of 256 frames along gridDim.y (<= 65535); the cIRM passes index one clip's F x T' plane with
// an int; the full-band TCN GEMMs address their 3 B T' time-major rows (+ one 128-row tile) with int row indices and int32 tensor-map
// coordinates.  Every element offset beyond these is 64-bit.  The sub-band TCN's B Fc T' row limit per chunk run (SB_MAX_ROWS) is kept by
// the planner and checked with its workspace.
static const long long SB_MAX_ROWS = 0x7fffffffLL - 128;
static const long long FSN_MAX_TP = 65535LL * 256;
static long long max_clips_for_rows(const fsn_config& c, int T) {
    return c.model_kind == FSN_KIND_PLUS ? (0x7fffffffLL - 128) / (3LL * (T + c.look_ahead)) : 0x7fffffffLL;
}
static int check_length(const fsn_config& c, int B, int T) {
    const long long Tp = (long long)T + c.look_ahead;
    if (Tp > FSN_MAX_TP) return fail(FSN_EINVAL, "T + look_ahead = %lld frames exceeds the limit of %lld (65535 x 256, the TCN convolution grid)", Tp, FSN_MAX_TP);
    if ((long long)c.num_freqs * Tp > 0x7fffffffLL)
        return fail(FSN_EINVAL, "num_freqs x (T + look_ahead) = %lld exceeds 2^31 - 1, the per-clip plane index limit", (long long)c.num_freqs * Tp);
    if (B > max_clips_for_rows(c, T))
        return fail(FSN_EINVAL, "3 x B x (T + look_ahead) = %lld rows exceeds the full-band TCN's 2^31 row limit", 3LL * B * Tp);
    return FSN_OK;
}

// Size lane ln and the model's buffers for a forward of B clips of T frames with window Tw and bin chunk Fc (ws_sizes), each fresh
// allocation zero-filled on its own stream (s: front end, sl: sub-band stage), and encode their tensor maps.
static int ensure_ws(fsn_model* m, Lane& ln, int B, int T, int Tw, int Fc, cudaStream_t s, cudaStream_t sl) {
    const fsn_config& c = m->cfg;
    const int F = c.num_freqs, Tp = T + c.look_ahead;
    const long long srows = (long long)B * (Fc ? Fc : F) * Tp;          // sub-band TCN: the rows of one chunk run
    if (c.sb_tcn && srows > SB_MAX_ROWS)
        return fail(FSN_EINVAL, "B * %s * (T + look_ahead) = %lld rows exceeds the sub-band TCN's 2^31 limit", Fc ? "bins per chunk" : "num_freqs", srows);
    if (c.model_kind == FSN_KIND_PLUS && !m->tcn5) return fail(FSN_ESTATE, "the TCN weights were not packed");
    const WsSizes z = ws_sizes(c, runs_layerwise(c, m->env_impl), B, T, Tw, Fc);
    const WsGeo geo{B, T, Tw, Fc};
    const bool regeo = ln.geo != geo;
    if (Tw || Fc) {
        // A windowed or bin-chunked forward exists to bound the workspace: first give back every buffer earlier forwards left larger than
        // it needs, and the pipelined entry points' second lane, so that the model then holds at most the plan's bytes.
        for (const WsBuf& e : WS) if (e.buf(*m, ln).bytes > z.*e.need) e.buf(*m, ln).release();
        release_lane(*m, m->lane[&ln == &m->lane[0] ? 1 : 0]);
    }
    for (const WsBuf& e : WS) {
        DevBuf& b = e.buf(*m, ln);
        if (e.flags & WS_ON_USE) continue;
        if (regeo && (e.flags & WS_REGEO)) b.release();
        if (b.ensure(z.*e.need, e.flags & WS_ZERO, (e.flags & WS_SL) ? sl : s)) return fail(FSN_ECUDA, "workspace allocation failed for B=%d T=%d", B, T);
    }
    // every forward encodes the tensor maps on the buffers as they now are: none outlives the allocation it was encoded for
    if (c.sb_tcn) {
        if (make_tmap_f32_2d(ln.mapSbx, ln.sbx.p, srows, 64, 128)) return fail(FSN_ECUDA, "cuTensorMapEncodeTiled failed for the sub-band input");
        if (int rc = map_tcn_scratch(m->sb_scratch, m->tcn_sb, srows)) return rc;
    }
    if (c.model_kind == FSN_KIND_PLUS) {
        const long long trows = 3LL * B * Tp;
        if (make_tmap_f32_2d(ln.mapX0, ln.x0.p, trows, m->tcn_fb.Cp, 128) || make_tmap_f32_2d(ln.mapXr, ln.xr.p, trows, m->tcn_fb.Cp, 128))
            return fail(FSN_ECUDA, "cuTensorMapEncodeTiled failed for the activations");
        if (int rc = map_tcn_scratch(ln.tcn, m->tcn_fb, trows)) return rc;
    }
    ln.geo = geo;
    return FSN_OK;
}

// d_enh != null: write the enhanced spectrum (decompress_cIRM x noisy) instead of the mask -- fused into the epilogue of the
// layer-wise kernel's last layer, a separate pass over a scratch mask for the generic kernel
// Tw > 0: the sub-band stage runs in time windows of Tw frames (the last one shorter); for each window the images are packed (`sp`, the
// front end's packer arguments) and every layer resumes from the h / c its previous window left (DESIGN.md §3.7).  Tw = 0: the images of
// the whole clip are already packed and every layer runs once over all frames.
static int run_sb_lstm(fsn_model* m, Lane& ln, int B, int T, int Tw, SbPackLaunch sp, float* d_out, const float* d_real,
                       const float* d_imag, float* d_enh, const int* tlen, cudaStream_t s) {
    const fsn_config& c = m->cfg;
    const int F = c.num_freqs, Tp = T + c.look_ahead, rows = B * F, ntiles = (rows + 127) / 128;
    const int impl = pick_impl(m);
    m->last_impl = impl;
    if (runs_layerwise(c, m->env_impl)) {
        // one recurrent launch per layer; the first one also projects its input (the packed images), each deeper one is preceded by
        // one GEMM: the input projection of every row and time step of the window (k_gemm_tc5.cu)
        const int H = c.sb_hidden, ntp = (ntiles + 1) / 2 * 2;
        const size_t cs_layer = lstm_tc5r_cstate_bytes(ntiles, H) / sizeof(float), hs_layer = (size_t)ntp * 128 * H;
        for (int w0 = 0; w0 < Tp; w0 += (Tw ? Tw : Tp)) {
            const int tw = Tw ? (Tp - w0 < Tw ? Tp - w0 : Tw) : Tp;
            if (Tw) {
                sp.t0 = w0; sp.Tw = tw;
                launch_sb_pack(sp, s);
                m->launches++;
            }
            const long long M = (long long)ntp * tw * 128;
            for (int l = 0; l < c.num_layers; ++l) {
                if (l > 0) {
                    // row-major Gin[M, 4H] = X[M, H] * Wp[4H, H]^T, both operands K-major
                    GemmF16Launch g{M, 4 * H, H, static_cast<__half*>(m->r_gin.p), 4LL * H, m->env_gin_tile_n};
                    int ge = launch_gemm_f16(m->r_hseq.p, m->r_wih[l].p, g, m->num_sms, s);
                    if (ge) return fail(FSN_ECUDA, "input-projection GEMM launch failed (layer %d): %s", l, cudaGetErrorString((cudaError_t)ge));
                    m->launches++;
                }
                LstmTc5rLaunch a{};
                a.wstream = static_cast<const __half*>(m->r_stream[l].p);
                a.bias = static_cast<const float*>(m->r_bias[l].p);
                a.fc_w = P(m, "sb_model.fc_output_layer.weight");
                a.fc_b = P(m, "sb_model.fc_output_layer.bias");
                a.H = H; a.rows = rows; a.Tp = Tp; a.ntiles = ntiles;
                a.t0 = w0; a.Tw = tw;
                if (l == 0) a.ximg = static_cast<const __half*>(ln.ximg.p);
                else a.gin = static_cast<const __half*>(m->r_gin.p);
                a.hseq = static_cast<__half*>(m->r_hseq.p);
                a.cstate = static_cast<float*>(m->cstate.p) + (Tw ? l * cs_layer : 0);
                if (Tw) a.hstate = static_cast<__half*>(m->r_hstate.p) + l * hs_layer;
                a.out = d_out; a.F = F; a.la = c.look_ahead;
                a.act = c.sb_act; a.fast = c.fast_math; a.gru = c.rnn_type == FSN_RNN_GRU; a.last = (l == c.num_layers - 1);
                a.nreal = d_real; a.nimag = d_imag; a.enh = reinterpret_cast<float2*>(d_enh); a.tlen = tlen;
                int e = launch_lstm_tc5r(a, s);
                if (e) return fail(FSN_ECUDA, "layer-wise LSTM launch failed (layer %d): %s", l, cudaGetErrorString((cudaError_t)e));
                m->launches++;
            }
        }
    } else if (Tw) {
        return fail(FSN_EINVAL, "time windows of the sub-band stage need the layer-wise LSTM path");
    } else if (impl == FSN_LSTM_TCGEN05) {
        return fail(FSN_EINVAL, "the tensor-core LSTM needs hidden %% 64 == 0 and <= 512, input <= 64, output_size 2");
    } else {
        LstmMmaLaunch a{};
        for (int l = 0; l < c.num_layers; ++l) {
            a.w.wfrag[l] = static_cast<const uint4*>(m->sb_frag[l].p);
            a.w.bias[l] = static_cast<const float*>(m->sb_bias[l].p);
        }
        a.w.fc_w = P(m, "sb_model.fc_output_layer.weight");
        a.w.fc_b = P(m, "sb_model.fc_output_layer.bias");
        a.L = c.num_layers; a.H = c.sb_hidden; a.I = m->Isb; a.Ipad = 64;
        a.rows = rows; a.Tp = Tp;
        a.img = static_cast<const __half*>(ln.ximg.p); a.ntiles = ntiles;
        a.cstate = static_cast<float*>(m->cstate.p);
        lstm_mma_cstate_bytes(c.num_layers, rows, c.sb_hidden, &a.rows_alloc);
        a.out = d_out; a.O = c.output_size; a.F = F; a.la = c.look_ahead; a.act = c.sb_act;
        a.fast = c.fast_math; a.gru = c.rnn_type == FSN_RNN_GRU; a.tlen = tlen;
        if (d_enh) {                                                    // generic kernel: mask into a scratch buffer, then one fused post-processing pass
            if (m->mask_tmp.ensure((size_t)B * 2 * F * T * 4, false, s)) return fail(FSN_ECUDA, "allocation failed");
            a.out = static_cast<float*>(m->mask_tmp.p);
        }
        int e = launch_lstm_mma(a, s);
        if (e) return fail(FSN_ECUDA, "mma LSTM launch failed: %s", cudaGetErrorString((cudaError_t)e));
        if (d_enh) { launch_apply_cirm_planar(a.out, d_real, d_imag, reinterpret_cast<float2*>(d_enh), B, F, T, tlen, c.look_ahead, s); m->launches++; }
    }
    m->launches++;
    return FSN_OK;
}

// the M side of a GEMM over the time-major rows (branch, group, frame) of TCN w: G gLN groups per branch of Tp frames each
static void set_tcn_rows(GemmTc5Launch& g, const TcnWeights& w, int G, int Tp) {
    g.rows_per_branch = G * Tp; g.tiles_m = (G * Tp + 127) / 128; g.nbranch = w.nbr; g.Tp = Tp; g.B = G;
}

// The eight blocks of TCN w (SequenceModel TCN branch, sequence_model.py:47-58; TCNBlock, causal_conv.py:96-108) on stream s: per block
// GEMM1 (1x1 conv + PReLU + gLN1 statistics), the depth-wise convolution, GEMM2 (folded gLN2 + residual), the stream ping-ponging between
// sc.xa and sc.xb from the input x (tensor map xmap).  amax0: block 0's stream maxima [nbr * G], written with the input.  The last
// GEMM2 ends as `last` says: its epilogue (EPI5_GLN_RES or EPI5_GLN_HEAD) and that epilogue's own outputs (Xrelu, or the head fields).
// tlen / zdiv: the per-sample extents of a ragged forward (GemmTc5Launch::tlen), or null.
static int run_tcn_blocks(fsn_model* m, const TcnWeights& w, TcnScratch& sc, const float* x, const unsigned char* xmap, const float* amax0,
                          int G, int Tp, bool causal, const GemmTc5Launch& last, const int* tlen, int zdiv, cudaStream_t s) {
    static const int dil[8] = {1, 2, 5, 9, 1, 2, 5, 9};
    const size_t Z = (size_t)w.nbr * G;
    const float* curp = x;
    const unsigned char* curmap = xmap;
    for (int blk = 0; blk < 8; ++blk) {
        double* st1 = tcn_gln_sums(sc.stats.p, Z, blk, 0);
        double* st2 = tcn_gln_sums(sc.stats.p, Z, blk, 1);
        const float* amax_in = blk ? tcn_amax(sc.stats.p, Z, blk) : amax0;
        auto key = [&](int b, const char* leaf) { return w.pre[b] + std::to_string(blk) + "." + leaf; };
        GemmTc5Launch g1{};
        set_tcn_rows(g1, w, G, Tp);
        g1.epi = EPI5_PRELU_STATS; g1.Kp = w.Cp; g1.NT = 128; g1.ntiles_n = 4; g1.Npad = 512;
        for (int b = 0; b < w.nbr; ++b) { g1.bias[b] = P(m, key(b, "conv1x1.bias")); g1.prelu[b] = P(m, key(b, "prelu1.weight")); }
        g1.stats_out = st1; g1.Y16 = static_cast<__half*>(sc.y1.p); g1.ldY = 512; g1.amax_in = amax_in; g1.tlen = tlen; g1.zdiv = zdiv;
        int e = launch_gemm_tc5(curmap, w.mapW1[blk], g1, m->num_sms, s);
        if (e) return fail(FSN_ECUDA, "%s GEMM1 launch failed: %s", w.name, cudaGetErrorString((cudaError_t)e));
        m->launches++;

        DwTmLaunch dw{};
        dw.X = static_cast<const __half*>(sc.y1.p); dw.Y = static_cast<__half*>(sc.y2.p);
        dw.Z = (int)Z; dw.B = G; dw.C = 512; dw.Tp = Tp; dw.dilation = dil[blk]; dw.causal = causal ? 1 : 0;
        dw.stats_in = st1; dw.stats_out = st2; dw.amax = amax_in; dw.tlen = tlen; dw.zdiv = zdiv;
        for (int b = 0; b < w.nbr; ++b) {
            dw.gamma[b] = P(m, key(b, "norm1.weight")); dw.beta[b] = P(m, key(b, "norm1.bias"));
            dw.w[b] = P(m, key(b, "depthwise_conv.weight")); dw.b[b] = P(m, key(b, "depthwise_conv.bias"));
            dw.prelu[b] = P(m, key(b, "prelu2.weight"));
        }
        e = launch_dwconv_tm(dw, s);
        if (e) return fail(FSN_ECUDA, "%s depth-wise conv launch failed: %s", w.name, cudaGetErrorString((cudaError_t)e));
        m->launches++;

        float* nxtp = static_cast<float*>((blk & 1) ? sc.xb.p : sc.xa.p);
        GemmTc5Launch g2 = blk < 7 ? GemmTc5Launch{} : last;
        if (blk < 7) { g2.epi = EPI5_GLN_RES; g2.amax_out = tcn_amax(sc.stats.p, Z, blk + 1); }
        set_tcn_rows(g2, w, G, Tp);
        g2.Kp = 512; g2.NT = w.NT; g2.ntiles_n = w.ntiles; g2.Npad = w.Cp;
        for (int b = 0; b < w.nbr; ++b) {
            g2.bias[b] = static_cast<const float*>(w.S2b.p) + ((size_t)blk * w.nbr + b) * w.Cp;
            g2.s1[b] = static_cast<const float*>(w.S1.p) + ((size_t)blk * w.nbr + b) * w.Cp;
        }
        g2.stats_in = st2; g2.count_row = 512; g2.tlen = tlen; g2.zdiv = zdiv;
        g2.Xold = curp; g2.ldY = w.Cp;
        if (g2.epi == EPI5_GLN_RES) g2.Y = nxtp;
        e = launch_gemm_tc5(sc.mapY2, w.mapW2[blk], g2, m->num_sms, s);
        if (e) return fail(FSN_ECUDA, "%s GEMM2 launch failed: %s", w.name, cudaGetErrorString((cudaError_t)e));
        m->launches++;
        curp = nxtp;
        curmap = (blk & 1) ? sc.mapXb : sc.mapXa;
    }
    return FSN_OK;
}

// The sub-band TCN (sequence_model = "TCN", fullsubnet_plus.py:102-110): the TCN blocks with one branch, the B*F sequences of the sub-band
// input as the gLN groups and Isb (<= 64) channels in one 64-column N tile; the last block's second 1x1 convolution ends in ReLU + Linear +
// activation (EPI5_GLN_HEAD) and writes the mask -- or, with d_enh, the enhanced spectrum.
// Fc > 0: the sequences run in chunks of Fc bins (the last one narrower), each packed here from the front end's whole-clip outputs (`sp`,
// the front end's packer arguments) into the same buffers; every sequence is its own gLN group, so nothing carries from one chunk to the
// next (DESIGN.md §3.8).  Fc = 0: the input of all bins is already packed and the blocks run once.
static int run_sb_tcn(fsn_model* m, Lane& ln, int B, int T, int Fc, SbPackLaunch sp, float* d_out, const float* d_real,
                      const float* d_imag, float* d_enh, const int* tlen, cudaStream_t s) {
    const fsn_config& c = m->cfg;
    const int F = c.num_freqs, Tp = T + c.look_ahead, W = Fc ? Fc : F;
    m->last_impl = FSN_LSTM_TCN;
    GemmTc5Launch head{};
    head.epi = EPI5_GLN_HEAD;
    head.fc_w = static_cast<const float*>(m->sb_fc.p); head.fc_b = P(m, "sb_model.fc_output_layer.bias");
    head.O = c.output_size; head.la = c.look_ahead; head.F = F; head.act = c.sb_act;
    head.out = d_out; head.nreal = d_real; head.nimag = d_imag; head.enh = reinterpret_cast<float2*>(d_enh);
    float* x = static_cast<float*>(ln.sbx.p);
    float* amax0 = x + (size_t)B * W * Tp * 64;
    for (int f0 = 0; f0 < F; f0 += W) {
        const int fc = F - f0 < W ? F - f0 : W, Z = B * fc;
        if (Fc) {
            sp.xtm = x; sp.amax = amax0; sp.f0 = f0; sp.Fc = fc;
            launch_sb_pack_tm(sp, s);
            m->launches++;
        }
        CK(cudaMemsetAsync(m->sb_scratch.stats.p, 0, tcn_stats_bytes(Z), s));
        head.Fg = fc; head.f0 = f0;
        int rc = run_tcn_blocks(m, m->tcn_sb, m->sb_scratch, x, ln.mapSbx, amax0, Z, Tp, false, head, tlen, fc, s);
        if (rc) return rc;
    }
    return FSN_OK;
}

// The whole forward.  Front end (norm, attention, full-band model, sub-band statistics + packing) on stream `s` into lane `ln`;
// the sub-band LSTM on stream `sl` (== s for the plain entry point; the pipelined entry points pass the LSTM stream, ordered
// after the front end by the lane's ev_front).
// Copy the per-sample extents frames[b] + look_ahead of a ragged forward into the lane's device buffer ln.tlen ([3][B]: one row per
// full-band branch, so a full-band gLN group z = branch * B + b indexes it directly) through the next pinned staging slot.
static int stage_lengths(fsn_model* m, Lane& ln, const int32_t* h_frames, int B, cudaStream_t s) {
    fsn_model::LenSlot& ls = m->len_slot[m->nlen++ % fsn_model::NLEN];
    const size_t n = (size_t)3 * B;
    if (!ls.ev) CK(cudaEventCreateWithFlags(&ls.ev, cudaEventDisableTiming));
    if (ls.used) CK(cudaEventSynchronize(ls.ev));                        // the copy that last read this slot has completed
    if (ls.cap < n) {
        if (ls.h) CK(cudaFreeHost(ls.h));
        ls.h = nullptr; ls.cap = 0;
        CK(cudaHostAlloc(reinterpret_cast<void**>(&ls.h), n * sizeof(int32_t), cudaHostAllocDefault));
        ls.cap = n;
    }
    for (int br = 0; br < 3; ++br)
        for (int b = 0; b < B; ++b) ls.h[(size_t)br * B + b] = h_frames[b] + m->cfg.look_ahead;
    if (ln.tlen.ensure(n * sizeof(int32_t), false, s)) return fail(FSN_ECUDA, "workspace allocation failed for the clip lengths");
    CK(cudaMemcpyAsync(ln.tlen.p, ls.h, n * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CK(cudaEventRecord(ls.ev, s));
    ls.used = true;
    return FSN_OK;
}

// h_frames: the frame count of every sample of a ragged batch (validated by the caller), or null when every sample spans T frames
// Tw: time window of the sub-band stage (0: the whole clip; > 0 needs s == sl, the plain entry points)
// Fc: bin chunk of the sub-band TCN (0: all bins at once; > 0 needs s == sl, the plain entry points)
static int forward_impl(fsn_model* m, Lane& ln, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                        const int32_t* h_frames, float* d_out, float* d_enh, cudaStream_t s, cudaStream_t sl, int Tw = 0, int Fc = 0) {
    if (!m || !d_mag || (!d_out && !d_enh)) return fail(FSN_EINVAL, "null argument");
    if (d_enh && (!d_real || !d_imag)) return fail(FSN_EINVAL, "the enhanced-spectrum output needs the noisy real and imaginary planes");
    if (d_enh && m->cfg.output_size != 2) return fail(FSN_EINVAL, "the enhanced-spectrum output needs output_size 2 (a complex mask)");
    if (!m->finalized) return fail(FSN_ESTATE, "fsn_model_finalize has not been called");
    const fsn_config& c = m->cfg;
    if (B < 1 || T < 1) return fail(FSN_EINVAL, "bad batch/frames");
    if (c.model_kind == FSN_KIND_PLUS && (!d_real || !d_imag)) return fail(FSN_EINVAL, "FullSubNet_Plus.forward needs mag, real and imag");
    const int F = c.num_freqs, Tp = T + c.look_ahead, Pp = (Tp + 3) & ~3;
    // chained (programmatic dependent) launches of this thread's front-end kernels: see env_pdl; "small" = at most 16 row-tile pairs,
    // where the forward is launch-latency-bound
    fsn_chain_launch_set(m->env_pdl == 1 || (m->env_pdl < 0 && ((long long)B * F + 255) / 256 <= 16));
    if (c.model_kind == FSN_KIND_PLUS && c.channel_attention == FSN_ATTN_TSSE)
        for (int i = 0; i < 3; ++i)
            if (Tp < c.kersize[i]) return fail(FSN_EINVAL, "sequence shorter than the TSSE kernel size");
    int rc = check_length(c, B, T);
    if (rc) return rc;
    rc = ensure_ws(m, ln, B, T, Tw, Fc, s, sl);
    if (rc) return rc;
    const int* tl = nullptr;                                            // per-sample extents on the device (null: all Tp)
    if (h_frames) {
        rc = stage_lengths(m, ln, h_frames, B, s);
        if (rc) return rc;
        tl = static_cast<const int*>(ln.tlen.p);
    }
    m->launches = 0;
    m->last_lane = (int)(&ln - m->lane);
    const int evi = (int)(m->nfwd % fsn_model::NEV);
    cudaEventRecord(m->evf0[evi], s);

    SbPackLaunch sp{};
    sp.B = B; sp.F = F; sp.Tp = Tp; sp.Ns = c.sb_num_neighbors; sp.Nf = c.fb_num_neighbors; sp.P = Pp;
    sp.mu = static_cast<float*>(ln.mu.p);
    sp.sigma = static_cast<float*>(ln.sigma.p);
    sp.rowsum = static_cast<float*>(ln.sb_rowsum.p);
    sp.norm_type = c.norm_type;
    sp.ximg = static_cast<__half*>(ln.ximg.p);
    sp.ntiles = (B * F + 127) / 128;
    sp.t0 = 0; sp.Tw = Tp;
    sp.cum = Tw ? static_cast<double*>(m->sb_cum.p) : nullptr;
    sp.tlen = tl;
    sp.f0 = 0; sp.Fc = F;

    if (c.model_kind == FSN_KIND_PLUS) {
        const char* sfx[3] = {"", "_real", "_imag"};
        const char* cn[3] = {"smallConv1d", "middleConv1d", "largeConv1d"};
        TsseLaunch ta{};
        ta.x[0] = d_mag; ta.x[1] = d_real; ta.x[2] = d_imag;
        ta.nbranch = 3; ta.B = B; ta.F = F; ta.T = T; ta.Tp = Tp; ta.P = Pp; ta.attention = 1 + c.channel_attention; ta.sub = c.subband_num;
        for (int i = 0; i < 3; ++i) ta.ksz[i] = c.kersize[i];
        for (int b = 0; b < 3; ++b) {
            const std::string p = std::string("channel_attention") + sfx[b];
            if (c.channel_attention == FSN_ATTN_ECA) { ta.p[b].eca_w = P(m, p + ".conv.weight"); continue; }
            if (c.channel_attention == FSN_ATTN_TSSE) {
                for (int i = 0; i < 3; ++i) {
                    ta.p[b].conv_w[i] = P(m, p + "." + cn[i] + ".0.weight");
                    ta.p[b].conv_b[i] = P(m, p + "." + cn[i] + ".0.bias");
                }
                ta.p[b].cat_w = P(m, p + ".feature_concate_fc.weight"); ta.p[b].cat_b = P(m, p + ".feature_concate_fc.bias");
            }
            ta.p[b].fc1_w = P(m, p + ".fc1.weight"); ta.p[b].fc1_b = P(m, p + ".fc1.bias");
            ta.p[b].fc2_w = P(m, p + ".fc2.weight"); ta.p[b].fc2_b = P(m, p + ".fc2.bias");
        }
        ta.out = static_cast<float*>(ln.fbin.p);
        ta.scale = static_cast<float*>(ln.tsse_scale.p);
        ta.rows = ta.scale + (size_t)ta.nbranch * B * F;
        ta.out_tm = static_cast<float*>(ln.x0.p); ta.Cp = m->tcn_fb.Cp;
        ta.tlen = tl;
        if (c.norm_type != FSN_NORM_OFFLINE_LAPLACE) {
            NormLaunch na{};
            na.x[0] = d_mag; na.x[1] = d_real; na.x[2] = d_imag; na.y = static_cast<float*>(ln.xn.p);
            na.nbranch = 3; na.B = B; na.F = F; na.T = T; na.Tp = Tp; na.type = c.norm_type; na.tlen = tl;
            launch_input_norm(na, s); m->launches++;
            for (int b = 0; b < 3; ++b) ta.x[b] = static_cast<const float*>(ln.xn.p) + (size_t)b * B * F * Tp;
            ta.T = Tp; ta.prenorm = 1;                                  // padded frames are part of the normalised signal
        }
        const TcnWeights& w = m->tcn_fb;
        CK(cudaMemsetAsync(ln.tcn.stats.p, 0, tcn_stats_bytes(3 * B), s));
        ta.amax = tcn_amax(ln.tcn.stats.p, 3 * B, 0);                  // block 0: written by the gate kernel
        launch_tsse_norm(ta, s); m->launches += 3;

        GemmTc5Launch last{};                                           // the last block also writes relu(x) for the output Linear
        last.epi = EPI5_GLN_RES; last.Xrelu = static_cast<float*>(ln.xr.p);
        rc = run_tcn_blocks(m, w, ln.tcn, static_cast<const float*>(ln.x0.p), ln.mapX0, ta.amax, B, Tp, c.tcn_causal, last, tl, 1, s);
        if (rc) return rc;
        GemmTc5Launch g3{};
        set_tcn_rows(g3, w, B, Tp);
        g3.epi = EPI5_OUT; g3.Kp = w.Cp; g3.NT = w.NT; g3.ntiles_n = w.ntiles; g3.Npad = w.Cp;
        for (int b = 0; b < 3; ++b) g3.bias[b] = static_cast<const float*>(m->fb_fc_b.p) + (size_t)b * w.Cp;
        g3.out = static_cast<float*>(ln.fbout.p); g3.F = F; g3.P = Pp; g3.act = c.fb_act;    // finite past each clip's end; the sub-band stages mask it
        int e = launch_gemm_tc5(ln.mapXr, m->map_fb_fc, g3, m->num_sms, s);
        if (e) return fail(FSN_ECUDA, "TCN output GEMM launch failed: %s", cudaGetErrorString((cudaError_t)e));
        m->launches++;

        sp.win = static_cast<const float*>(ln.fbin.p); sp.Pw = Pp;      // post-attention mag branch (fullsubnet_plus.py:182)
        sp.nfb = 3;
        for (int b = 0; b < 3; ++b) sp.fb[b] = static_cast<const float*>(ln.fbout.p) + (size_t)b * B * F * Pp;
    } else {
        TsseLaunch ta{};
        ta.x[0] = d_mag; ta.nbranch = 1; ta.B = B; ta.F = F; ta.T = T; ta.Tp = Tp; ta.P = Pp; ta.attention = 0;
        ta.out = static_cast<float*>(ln.fbin.p);
        ta.scale = static_cast<float*>(ln.tsse_scale.p);
        ta.rows = ta.scale + (size_t)ta.nbranch * B * F;
        ta.tlen = tl;
        if (c.norm_type != FSN_NORM_OFFLINE_LAPLACE) {
            NormLaunch na{};
            na.x[0] = d_mag; na.y = static_cast<float*>(ln.xn.p);
            na.nbranch = 1; na.B = B; na.F = F; na.T = T; na.Tp = Tp; na.type = c.norm_type; na.tlen = tl;
            launch_input_norm(na, s); m->launches++;
            ta.x[0] = static_cast<const float*>(ln.xn.p); ta.T = Tp; ta.prenorm = 1;
        }
        launch_tsse_norm(ta, s); m->launches += 3;
        launch_pad_copy(d_mag, static_cast<float*>(ln.magpad.p), B, F, T, Pp, tl, c.look_ahead, s); m->launches++;
        // the full-band LSTM is causal, and its input (fb_in) is already zero past each clip's end: its outputs there are masked by the
        // sub-band stages
        const int Ipad = (F + 15) / 16 * 16, rows_pad = (B + 63) / 64 * 64;
        launch_fb_pack(static_cast<const float*>(ln.fbin.p), static_cast<__half*>(ln.fbx.p), B, F, Tp, Pp, rows_pad, Ipad, s); m->launches++;
        if (lstm_ws_supported(c.num_layers, c.fb_hidden, Ipad, B, m->num_sms) && !m->env_no_ws) {
            const size_t hb = (size_t)c.num_layers * 2 * 64 * c.fb_hidden * 2;
            if (m->ws_h.ensure(hb, false, s) || m->ws_bar.ensure(64, true, s)) return fail(FSN_ECUDA, "allocation failed");
            CK(cudaMemsetAsync(m->ws_h.p, 0, hb, s));
            LstmWsLaunch w{};
            fill_ws(m, w);
            w.rows = B; w.rows_pad = rows_pad; w.Tp = Tp;
            w.x = static_cast<const __half*>(ln.fbx.p); w.hbuf = static_cast<__half*>(m->ws_h.p); w.cbuf = nullptr;
            w.barrier = static_cast<unsigned int*>(m->ws_bar.p);
            w.hseq = static_cast<float*>(ln.hseq.p); w.P = Pp; w.resume = 0; w.t0 = 0;
            int e = launch_lstm_ws(w, s);
            if (e) return fail(FSN_ECUDA, "weight-stationary full-band LSTM launch failed: %s", cudaGetErrorString((cudaError_t)e));
            m->launches++;
        } else {
        LstmMmaLaunch a{};
        for (int l = 0; l < c.num_layers; ++l) {
            a.w.wfrag[l] = static_cast<const uint4*>(m->fb_frag[l].p);
            a.w.bias[l] = static_cast<const float*>(m->fb_bias[l].p);
        }
        a.L = c.num_layers; a.H = c.fb_hidden; a.I = F; a.Ipad = Ipad; a.rows = B; a.Tp = Tp;
        a.xplain = static_cast<const __half*>(ln.fbx.p); a.rows_pad = rows_pad;
        a.cstate = static_cast<float*>(m->cstate.p);
        lstm_mma_cstate_bytes(c.num_layers, B, c.fb_hidden, &a.rows_alloc);
        a.hseq = static_cast<float*>(ln.hseq.p); a.P = Pp; a.fast = c.fast_math; a.gru = c.rnn_type == FSN_RNN_GRU;
        int e = launch_lstm_mma(a, s);
        if (e) return fail(FSN_ECUDA, "full-band LSTM launch failed: %s", cudaGetErrorString((cudaError_t)e));
        m->launches++;
        }
        ConvLaunch cf{};
        cf.X = static_cast<const float*>(ln.hseq.p); cf.Y = static_cast<float*>(ln.fbout.p);
        cf.Z = B; cf.M = F; cf.K = c.fb_hidden; cf.Tp = Tp; cf.P = Pp; cf.act = c.fb_act;
        cf.W = P(m, "fb_model.fc_output_layer.weight"); cf.bias = P(m, "fb_model.fc_output_layer.bias");
        launch_conv1x1(cf, s); m->launches++;

        sp.win = static_cast<const float*>(ln.magpad.p); sp.Pw = Pp;    // raw padded magnitude (fullsubnet.py:94)
        sp.nfb = 1;
        sp.fb[0] = static_cast<const float*>(ln.fbout.p);
    }
    launch_sb_stats(sp, s); m->launches += 2;
    if (c.sb_tcn) {
        if (!Fc) {                                                      // chunked: run_sb_tcn packs each chunk
            sp.xtm = static_cast<float*>(ln.sbx.p);
            sp.amax = sp.xtm + (size_t)B * F * Tp * 64;
            launch_sb_pack_tm(sp, s);
            m->launches++;
        }
    } else if (!Tw) {                                                   // windowed: run_sb_lstm packs each window
        launch_sb_pack(sp, s);
        m->launches++;
    }
    cudaEventRecord(m->evf1[evi], s);
    if (sl != s) {                                                      // pipelined: the LSTM stream picks the lane up when the front end is done
        CK(cudaEventRecord(ln.ev_front, s));
        CK(cudaStreamWaitEvent(sl, ln.ev_front, 0));
    }
    cudaEventRecord(m->ev0[evi], sl);
    rc = c.sb_tcn ? run_sb_tcn(m, ln, B, T, Fc, sp, d_out, d_real, d_imag, d_enh, tl, sl)
                  : run_sb_lstm(m, ln, B, T, Tw, sp, d_out, d_real, d_imag, d_enh, tl, sl);
    cudaEventRecord(m->ev1[evi], sl);
    if (rc) return rc;
    m->nfwd++;
    CK(cudaGetLastError());
    return FSN_OK;
}

// ---------------------------------------------------------------------------------------------
// pipelined execution: internal streams, lanes
// ---------------------------------------------------------------------------------------------
static int ensure_pipeline(fsn_model* m) {
    if (m->s_front) return FSN_OK;
    int lo = 0, hi = 0;
    CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));                     // hi = numerically lowest = highest priority
    CK(cudaStreamCreateWithPriority(&m->s_front, cudaStreamNonBlocking, lo));
    CK(cudaStreamCreateWithPriority(&m->s_lstm, cudaStreamNonBlocking, hi));   // the LSTM's clusters win the SMs when both are pending
    CK(cudaEventCreateWithFlags(&m->ev_in, cudaEventDisableTiming));
    for (auto& ln : m->lane) {
        CK(cudaEventCreateWithFlags(&ln.ev_front, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&ln.ev_lstm, cudaEventDisableTiming));
    }
    return FSN_OK;
}

// one pipelined batch: inputs are ready once `ready` (an event, may be null) has fired; returns the lane used
static int submit_impl(fsn_model* m, cudaEvent_t ready, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                       float* d_out, float* d_enh, int* lane_out) {
    int rc = ensure_pipeline(m);
    if (rc) return rc;
    // overlap needs the opt-in (see env_front_overlap) and FullSubNet+ (fullsubnet.Model's full-band LSTM is a cooperative launch and
    // shares the LSTM scratch): otherwise one lane, one stream -- the pipeline still overlaps copies and the caller's post-processing
    const bool overlap = m->env_front_overlap && (m->cfg.model_kind == FSN_KIND_PLUS);
    const int slot = overlap ? (int)(m->nsub & 1) : 0;
    Lane& ln = m->lane[slot];
    cudaStream_t sf = overlap ? m->s_front : m->s_lstm;
    if (ready) CK(cudaStreamWaitEvent(sf, ready, 0));
    if (m->plain_pending) { CK(cudaStreamWaitEvent(sf, m->ev_plain, 0)); CK(cudaStreamWaitEvent(m->s_lstm, m->ev_plain, 0)); }
    if (ln.used) CK(cudaStreamWaitEvent(sf, ln.ev_lstm, 0));              // the LSTM that read this lane has finished
    rc = forward_impl(m, ln, d_mag, d_real, d_imag, B, T, nullptr, d_out, d_enh, sf, m->s_lstm);
    if (rc) return rc;
    CK(cudaEventRecord(ln.ev_lstm, m->s_lstm));
    ln.used = true;
    m->nsub++;
    if (lane_out) *lane_out = slot;
    return FSN_OK;
}

// Workspace per sample (bytes) of a forward with T frames: the per-sample slices of every grow-only buffer of ensure_ws.  The
// layer-wise path dominates: its time-batched input projection Gin takes 257 x T' x 4H x 2 bytes per sample (0.2 GB at config #5).
// This estimate picks the sub-batch of a batch that fits unwindowed (plan_forward); it counts F rows per sample where the layer-wise
// buffers hold whole pairs of 128-row tiles, so plan_forward checks its choice against the exact count of ws_sizes.
static double ws_bytes_per_sample(const fsn_config& c, bool layerwise, int T) {
    const double F = c.num_freqs, Tp = T + c.look_ahead, rows = F;              // sequences per sample
    double b = 0;
    if (c.model_kind == FSN_KIND_PLUS) b += 3 * F * Tp * 4 * 2 + 3 * Tp * (4.0 * ((c.num_freqs + 31) / 32 * 32) + 512) * 4;   // fb_in/out, X0/Xa/Xb/Xr (fp32), Y1/Y2 (fp16)
    else b += F * Tp * 4 * 4 + Tp * (F + c.fb_hidden) * 4;
    if (c.sb_tcn) {                                                             // input + two fp32 streams of 64 channels, two fp16 hidden
        b += rows * Tp * (3 * 64 * 4 + 2 * 512 * 2) + rows * (tcn_stats_bytes(1) + 4);   // buffers of 512; statistics, the input's max |x|
        return b;
    }
    b += rows * Tp * 128;                                                       // packed sub-band images (when used)
    b += rows * c.num_layers * c.sb_hidden * 4;                                  // cell state
    if (layerwise && c.num_layers > 1) b += rows * Tp * (4.0 * c.sb_hidden + c.sb_hidden) * 2;   // Gin + layer output sequence
    return b;
}

// The largest v in [lo, hi] with ok(v), or lo if there is none; ok(lo) is not asked.  ok must hold up to some v and fail after it.
template <class Ok> static int largest(int lo, int hi, Ok ok) {
    while (lo < hi) { const int mid = (lo + hi + 1) / 2; if (ok(mid)) lo = mid; else hi = mid - 1; }
    return lo;
}

// The plan of a plain forward (fsn_plan_forward_bins): sub-batch Bs, sub-band window Tw (0: whole clip) and, for the sub-band TCN, bin
// chunk Fc (0: all bins) so that the exact workspace (ws_sizes) stays within cap.
//   * the sub-batch of the per-sample estimate, if it fits unwindowed: the forward of every release before windows existed;
//   * else (layer-wise path only) the largest sub-batch that fits with a window of 256 frames (32 if none does), then the longest window
//     (a multiple of 32) that fits, evened out over the same number of windows; more sequences in flight keep more SMs busy;
//   * nothing fits: one clip at a time with a 256-frame window, allocated anyway.
// force > 0 (FSN_SB_WINDOW) windows every layer-wise forward with exactly that window.  Sub-batches are equal splits of B.
// The sub-band TCN is never windowed (every gLN spans a whole sequence) but runs in bin chunks (DESIGN.md §3.8):
//   * the sub-batch of the per-sample estimate, if it fits unchunked: the forward before chunks existed;
//   * else, over every equal split Bs, the widest chunk that fits, evened out over the same number of chunks; the plan with the fewest
//     chunk runs ceil(B / Bs) * ceil(F / Fc) wins, ties to the larger Bs (Fc = F, unchunked, is a candidate);
//   * nothing fits: one clip at a time in one-bin chunks, allocated anyway.
// Every chunk run keeps Bs * Fc * T' <= SB_MAX_ROWS.  force_bins > 0 (FSN_SB_CHUNK) chunks every TCN forward with exactly that many bins
// (>= F: unchunked) and the largest equal split that fits with them.
static Plan plan_forward(const fsn_config& c, bool layerwise, int B, int T, double cap, int force, int force_bins) {
    const int Tp = T + c.look_ahead, wmax = (Tp + 31) / 32 * 32;
    const long long blim = max_clips_for_rows(c, T);             // sub-batches never exceed the full-band TCN's row limit
    auto split = [&](int bmax) { if (bmax > blim) bmax = (int)blim; if (bmax < 1) bmax = 1; if (B <= bmax) return B; const int n = (B + bmax - 1) / bmax; return (B + n - 1) / n; };
    auto bytes = [&](int bs, int tw) { return (double)ws_sizes(c, layerwise, bs, T, tw).total(); };
    // largest equal split bs with fits(bs) (0 if even one clip does not fit)
    auto max_split = [&](auto fits) { const int b = largest(0, B, [&](int v) { return fits(split(v)); }); return b ? split(b) : 0; };
    const double per = ws_bytes_per_sample(c, layerwise, T);
    const double bmax = cap / (per > 1 ? per : 1);
    Plan p{split(bmax < B ? (int)bmax : B)};
    if (c.sb_tcn) {
        const int F = c.num_freqs;
        auto fits = [&](int bs, int fc) { return (long long)bs * fc * Tp <= SB_MAX_ROWS && ws_sizes(c, false, bs, T, 0, fc < F ? fc : 0).total() <= cap; };
        const int fforce = force_bins > 0 ? (force_bins < F ? force_bins : F) : 0;
        if (fforce) {                                                   // chunks of fforce bins (F: unchunked), the largest equal split that fits
            if (fforce < F || !fits(p.Bs, F)) {
                const int b = max_split([&](int bs) { return fits(bs, fforce); });
                p.Bs = b ? b : 1;
            }
            p.Fc = fforce < F ? fforce : 0;
        } else if (!fits(p.Bs, F)) {
            long long best = -1;
            p.Bs = 1; p.Fc = 1;
            for (int n = 1, prev = 0; n <= B; ++n) {                    // the equal splits, largest first
                const int bs = (B + n - 1) / n;
                if (bs == prev || bs > blim) continue;
                prev = bs;
                const int fc = largest(0, F, [&](int v) { return fits(bs, v); });   // widest chunk that fits
                if (!fc) continue;
                const int nch = (F + fc - 1) / fc;
                const long long runs = (long long)((B + bs - 1) / bs) * nch;
                if (best < 0 || runs < best) { best = runs; p.Bs = bs; p.Fc = (F + nch - 1) / nch; }
            }
            if (p.Fc >= F) p.Fc = 0;
        }
    } else if (layerwise && force > 0) {
        p.Tw = force;
        const int b = max_split([&](int bs) { return bytes(bs, force) <= cap; });
        p.Bs = b ? b : 1;
    } else if (layerwise && bytes(p.Bs, 0) > cap) {
        int b = 0, wmin = 0;
        for (int w : {256, 32}) {
            wmin = w < wmax ? w : wmax;
            if ((b = max_split([&](int bs) { return bytes(bs, wmin) <= cap; }))) break;
        }
        if (!b) {
            p.Bs = 1; p.Tw = 256 < wmax ? 256 : wmax;
        } else if (bytes(b, 0) <= cap) {
            p.Bs = b;                                                   // the smaller sub-batch fits unwindowed
        } else {
            p.Bs = b;
            const int u = largest(wmin / 32, wmax / 32, [&](int v) { return bytes(b, 32 * v) <= cap; });   // longest window, in 32-frame units
            const int nwin = (Tp + 32 * u - 1) / (32 * u);
            p.Tw = ((Tp + nwin - 1) / nwin + 31) / 32 * 32;
        }
    }
    p.bytes = (int64_t)ws_sizes(c, layerwise, p.Bs, T, p.Tw, p.Fc).total();
    return p;
}

static int forward_plain(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                         const int32_t* h_frames, float* d_out, float* d_enh, void* stream) {
    if (!m) return fail(FSN_EINVAL, "null argument");
    if (!m->finalized) return fail(FSN_ESTATE, "fsn_model_finalize has not been called");
    if (B < 1 || T < 1) return fail(FSN_EINVAL, "bad batch/frames");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    for (auto& ln : m->lane)                                             // batches still in flight in the pipeline share the scratch buffers
        if (ln.used) CK(cudaStreamWaitEvent(s, ln.ev_lstm, 0));
    // Samples are independent, so a batch whose workspace would exceed the cap (FSN_WS_CAP_GB, default 24 of the 80 GB) is run as
    // equal sub-batches one after the other on the same stream -- same results, bounded memory (e.g. 256 clips on the layer-wise path);
    // a clip too long for the cap runs its sub-band stage in time windows (plan_forward) -- same bits, O(window) sub-band memory --
    // or, with the sub-band TCN, in bin chunks -- O(chunk) sub-band memory.
    if (int rc = check_length(m->cfg, 1, T)) return rc;
    m->plan = plan_forward(m->cfg, runs_layerwise(m->cfg, m->env_impl), B, T, m->ws_cap_bytes, m->env_sb_window, m->env_sb_chunk);
    const int Bs = m->plan.Bs, Tw = m->plan.Tw, Fc = m->plan.Fc;
    int rc = FSN_OK;
    if (Bs >= B) {
        rc = forward_impl(m, m->lane[0], d_mag, d_real, d_imag, B, T, h_frames, d_out, d_enh, s, s, Tw, Fc);
    } else {
        const size_t in_stride = (size_t)m->cfg.num_freqs * T, out_stride = (size_t)m->cfg.output_size * m->cfg.num_freqs * T;
        int64_t launches = 0;
        for (int b0 = 0; b0 < B && rc == FSN_OK; b0 += Bs) {
            const int nb = (B - b0 < Bs) ? B - b0 : Bs;
            rc = forward_impl(m, m->lane[0], d_mag + b0 * in_stride, d_real ? d_real + b0 * in_stride : nullptr, d_imag ? d_imag + b0 * in_stride : nullptr,
                              nb, T, h_frames ? h_frames + b0 : nullptr, d_out ? d_out + b0 * out_stride : nullptr,
                              d_enh ? d_enh + b0 * in_stride * 2 : nullptr, s, s, Tw, Fc);
            launches += m->launches;
        }
        m->launches = launches;
    }
    if (rc) return rc;
    if (!m->ev_plain) CK(cudaEventCreateWithFlags(&m->ev_plain, cudaEventDisableTiming));
    CK(cudaEventRecord(m->ev_plain, s));
    m->plain_pending = true;
    return FSN_OK;
}

static int submit_plain(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                        float* d_out, float* d_enh, void* stream) {
    if (!m) return fail(FSN_EINVAL, "null argument");
    int rc = ensure_pipeline(m);
    if (rc) return rc;
    CK(cudaEventRecord(m->ev_in, static_cast<cudaStream_t>(stream)));    // everything enqueued on the caller's stream so far (the inputs)
    return submit_impl(m, m->ev_in, d_mag, d_real, d_imag, B, T, d_out, d_enh, nullptr);
}

extern "C" int fsn_model_forward(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                 float* d_out, void* stream) {
    if (!d_out) return fail(FSN_EINVAL, "null argument");
    return forward_plain(m, d_mag, d_real, d_imag, B, T, nullptr, d_out, nullptr, stream);
}
extern "C" int fsn_model_forward_enhance(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                         float* d_enh, void* stream) {
    if (!d_enh) return fail(FSN_EINVAL, "null argument");
    return forward_plain(m, d_mag, d_real, d_imag, B, T, nullptr, nullptr, d_enh, stream);
}

// The frame counts of a ragged batch: each in 1..T, and long enough for the TSSE convolutions.  Returns the array to pass on: null
// when every clip spans all T frames, so that case runs exactly the unmasked forward.
static int check_frames(const fsn_model* m, const int32_t* h_frames, int32_t B, int32_t T, const int32_t** use) {
    *use = nullptr;
    if (!h_frames) return FSN_OK;
    if (!m) return fail(FSN_EINVAL, "null argument");
    const fsn_config& c = m->cfg;
    int kmax = 1;
    if (c.model_kind == FSN_KIND_PLUS && c.channel_attention == FSN_ATTN_TSSE)
        for (int i = 0; i < 3; ++i) kmax = c.kersize[i] > kmax ? c.kersize[i] : kmax;
    bool all = true;
    for (int b = 0; b < B; ++b) {
        const int n = h_frames[b];
        if (n < 1 || n > T) return fail(FSN_EINVAL, "frames[%d] = %d is outside 1..T = %d", b, n, T);
        if (n + c.look_ahead < kmax)
            return fail(FSN_EINVAL, "frames[%d] = %d: frames + look_ahead = %d is shorter than the TSSE kernel size %d", b, n, n + c.look_ahead, kmax);
        all = all && n == T;
    }
    if (!all) *use = h_frames;
    return FSN_OK;
}

extern "C" int fsn_model_forward_ragged(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                        const int32_t* h_frames, float* d_out, void* stream) {
    if (!d_out) return fail(FSN_EINVAL, "null argument");
    if (B < 1 || T < 1) return fail(FSN_EINVAL, "bad batch/frames");
    const int32_t* fr = nullptr;
    int rc = check_frames(m, h_frames, B, T, &fr);
    return rc ? rc : forward_plain(m, d_mag, d_real, d_imag, B, T, fr, d_out, nullptr, stream);
}
extern "C" int fsn_model_forward_enhance_ragged(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                                const int32_t* h_frames, float* d_enh, void* stream) {
    if (!d_enh) return fail(FSN_EINVAL, "null argument");
    if (B < 1 || T < 1) return fail(FSN_EINVAL, "bad batch/frames");
    const int32_t* fr = nullptr;
    int rc = check_frames(m, h_frames, B, T, &fr);
    return rc ? rc : forward_plain(m, d_mag, d_real, d_imag, B, T, fr, nullptr, d_enh, stream);
}
extern "C" int fsn_model_submit(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                float* d_out, void* stream) {
    if (!d_out) return fail(FSN_EINVAL, "null argument");
    return submit_plain(m, d_mag, d_real, d_imag, B, T, d_out, nullptr, stream);
}
extern "C" int fsn_model_submit_enhance(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                        float* d_enh, void* stream) {
    if (!d_enh) return fail(FSN_EINVAL, "null argument");
    return submit_plain(m, d_mag, d_real, d_imag, B, T, nullptr, d_enh, stream);
}

extern "C" int fsn_model_last_lane(const fsn_model* m) { return m ? m->last_lane : 0; }

extern "C" int fsn_model_wait_lane(fsn_model* m, int32_t lane, void* stream) {
    if (!m || lane < 0 || lane > 1) return fail(FSN_EINVAL, "bad argument");
    if (m->lane[lane].used) CK(cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), m->lane[lane].ev_lstm, 0));
    return FSN_OK;
}

extern "C" int fsn_model_wait(fsn_model* m, void* stream) {
    if (!m) return fail(FSN_EINVAL, "null model");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    for (auto& ln : m->lane)
        if (ln.used) CK(cudaStreamWaitEvent(s, ln.ev_lstm, 0));
    return FSN_OK;
}

extern "C" int fsn_model_forward_host(fsn_model* m, const float* h_mag, const float* h_real, const float* h_imag, int32_t B, int32_t T,
                                      float* h_out, void* stream) {
    if (!m || !h_mag || !h_out) return fail(FSN_EINVAL, "null argument");
    const fsn_config& c = m->cfg;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t in_bytes = (size_t)B * c.num_freqs * T * 4, out_bytes = (size_t)B * c.output_size * c.num_freqs * T * 4;
    const float* hin[3] = {h_mag, h_real, h_imag};
    const int nin = (c.model_kind == FSN_KIND_PLUS) ? 3 : 1;
    for (int i = 0; i < nin; ++i) {
        if (!hin[i]) return fail(FSN_EINVAL, "missing input %d", i);
        if (m->stage_in[i].ensure(in_bytes, false)) return fail(FSN_ECUDA, "staging allocation failed");
        CK(cudaMemcpyAsync(m->stage_in[i].p, hin[i], in_bytes, cudaMemcpyHostToDevice, s));
    }
    if (m->stage_out.ensure(out_bytes, false)) return fail(FSN_ECUDA, "staging allocation failed");
    int rc = fsn_model_forward(m, static_cast<const float*>(m->stage_in[0].p), static_cast<const float*>(m->stage_in[1].p),
                               static_cast<const float*>(m->stage_in[2].p), B, T, static_cast<float*>(m->stage_out.p), stream);
    if (rc) return rc;
    CK(cudaMemcpyAsync(h_out, m->stage_out.p, out_bytes, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return FSN_OK;
}

extern "C" int fsn_model_forward_host_async(fsn_model* m, const float* h_mag, const float* h_real, const float* h_imag, int32_t B, int32_t T,
                                            float* h_out, void* stream) {
    if (!m || !h_mag || !h_out) return fail(FSN_EINVAL, "null argument");
    (void)stream;                                                        // host buffers carry no stream order; the work runs on internal streams
    const fsn_config& c = m->cfg;
    int rc = ensure_pipeline(m);
    if (rc) return rc;
    if (!m->s_in) {
        CK(cudaStreamCreateWithFlags(&m->s_in, cudaStreamNonBlocking));
        CK(cudaStreamCreateWithFlags(&m->s_out, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            CK(cudaEventCreateWithFlags(&m->ev_h2d[i], cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&m->ev_d2h[i], cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&m->ev_done[i], cudaEventDisableTiming));
        }
    }
    const int slot = (int)(m->nsub & 1);                                 // staging slot (the workspace lane is chosen by submit_impl)
    const size_t in_bytes = (size_t)B * c.num_freqs * T * 4, out_bytes = (size_t)B * c.output_size * c.num_freqs * T * 4;
    const float* hin[3] = {h_mag, h_real, h_imag};
    const int nin = (c.model_kind == FSN_KIND_PLUS) ? 3 : 1;
    // the forward that read this input slot (front end: mag / real / imag; fused epilogue: real / imag) has finished
    if (m->d2h_used[slot]) CK(cudaStreamWaitEvent(m->s_in, m->ev_done[slot], 0));
    for (int i = 0; i < nin; ++i) {
        if (!hin[i]) return fail(FSN_EINVAL, "missing input %d", i);
        if (m->a_in[slot][i].bytes < in_bytes) {
            CK(cudaDeviceSynchronize());                                       // (re)allocation only on the first calls / size changes
            if (m->a_in[slot][i].ensure(in_bytes, false)) return fail(FSN_ECUDA, "staging allocation failed");
        }
        CK(cudaMemcpyAsync(m->a_in[slot][i].p, hin[i], in_bytes, cudaMemcpyHostToDevice, m->s_in));
    }
    CK(cudaEventRecord(m->ev_h2d[slot], m->s_in));
    if (m->a_out[slot].bytes < out_bytes) {
        CK(cudaDeviceSynchronize());
        if (m->a_out[slot].ensure(out_bytes, false)) return fail(FSN_ECUDA, "staging allocation failed");
    }
    if (m->d2h_used[slot]) CK(cudaStreamWaitEvent(m->s_lstm, m->ev_d2h[slot], 0));   // the copy-out that read this output slot is done
    int used = 0;
    rc = submit_impl(m, m->ev_h2d[slot], static_cast<const float*>(m->a_in[slot][0].p), static_cast<const float*>(m->a_in[slot][1].p),
                     static_cast<const float*>(m->a_in[slot][2].p), B, T, static_cast<float*>(m->a_out[slot].p), nullptr, &used);
    if (rc) return rc;
    CK(cudaEventRecord(m->ev_done[slot], m->s_lstm));
    CK(cudaStreamWaitEvent(m->s_out, m->ev_done[slot], 0));
    CK(cudaMemcpyAsync(h_out, m->a_out[slot].p, out_bytes, cudaMemcpyDeviceToHost, m->s_out));
    CK(cudaEventRecord(m->ev_d2h[slot], m->s_out));
    m->d2h_used[slot] = true;
    return FSN_OK;
}

extern "C" int fsn_model_sync_host(fsn_model* m) {
    if (!m) return fail(FSN_EINVAL, "null model");
    if (m->s_in) { CK(cudaStreamSynchronize(m->s_in)); }
    if (m->s_lstm) { CK(cudaStreamSynchronize(m->s_front)); CK(cudaStreamSynchronize(m->s_lstm)); }
    if (m->s_out) { CK(cudaStreamSynchronize(m->s_out)); }
    return FSN_OK;
}

extern "C" int fsn_model_get_stage(fsn_model* m, const char* name, float* d_dst, int64_t numel, void* stream) {
    if (!m || !name || !d_dst) return fail(FSN_EINVAL, "null argument");
    Lane& ln = m->lane[m->last_lane];
    if (!ln.geo.B) return fail(FSN_ESTATE, "no forward has run yet");
    const fsn_config& c = m->cfg;
    const int F = c.num_freqs, Tp = ln.geo.T + c.look_ahead, Pp = (Tp + 3) & ~3, B = ln.geo.B;
    const int nbr = (c.model_kind == FSN_KIND_PLUS) ? 3 : 1;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const std::string n(name);
    if (n == "fb_in" || n == "fb_out") {
        if (numel != (int64_t)nbr * B * F * Tp) return fail(FSN_EINVAL, "%s needs %lld elements", name, (long long)nbr * B * F * Tp);
        const void* src = (n == "fb_in") ? ln.fbin.p : ln.fbout.p;
        CK(cudaMemcpy2DAsync(d_dst, (size_t)Tp * 4, src, (size_t)Pp * 4, (size_t)Tp * 4, (size_t)nbr * B * F, cudaMemcpyDeviceToDevice, s));
        return FSN_OK;
    }
    if (n == "sb_in") {
        if (!c.sb_tcn) return fail(FSN_EINVAL, "sb_in is kept only by the sub-band TCN (sequence_model = \"TCN\")");
        if (ln.geo.Fc) return fail(FSN_ESTATE, "sb_in is not kept: the last forward was chunked over bins (%d per chunk), its buffer holds the last chunk only", ln.geo.Fc);
        if (numel != (int64_t)B * F * m->Isb * Tp) return fail(FSN_EINVAL, "sb_in needs %lld elements", (long long)B * F * m->Isb * Tp);
        launch_tm_to_fm(static_cast<const float*>(ln.sbx.p), 64, d_dst, B * F, m->Isb, Tp, s);
        CK(cudaGetLastError());
        return FSN_OK;
    }
    if (n == "sb_mu") {
        if (numel != B) return fail(FSN_EINVAL, "sb_mu needs %d elements", B);
        CK(cudaMemcpyAsync(d_dst, ln.mu.p, (size_t)B * 4, cudaMemcpyDeviceToDevice, s));
        return FSN_OK;
    }
    return fail(FSN_EINVAL, "unknown stage %s", name);
}


// ---------------------------------------------------------------------------------------------
// streaming step API (causal fullsubnet.Model)
// ---------------------------------------------------------------------------------------------
struct fsn_stream {
    fsn_model* m;
    int B, n = 0;
    DevBuf cum_in, cum_sb, fbin, fbx, hseq, fbout, ximg, c_fb, c_sb, h_fb, h_sb, ws_h, ws_c, ws_bar;
    bool use_ws = false;
    int ra_fb = 0, ra_sb = 0, rows_pad = 0, Ipad = 0;
};

extern "C" int fsn_stream_create(fsn_model* m, int32_t B, fsn_stream** out) {
    if (!m || !out || B < 1) return fail(FSN_EINVAL, "bad argument");
    if (!m->finalized) return fail(FSN_ESTATE, "fsn_model_finalize has not been called");
    const fsn_config& c = m->cfg;
    if (c.model_kind != FSN_KIND_FSN) return fail(FSN_EINVAL, "streaming needs fullsubnet.Model (FullSubNet+ is not causal: TSSE pools over all time)");
    if (c.norm_type != FSN_NORM_CUMULATIVE_LAPLACE && c.norm_type != FSN_NORM_CUMULATIVE_LAYER)
        return fail(FSN_EINVAL, "streaming needs a cumulative norm_type");
    fsn_stream* st = new fsn_stream();
    st->m = m; st->B = B;
    const int F = c.num_freqs, rows = B * F, ntiles = (rows + 127) / 128;
    st->Ipad = (F + 15) / 16 * 16; st->rows_pad = (B + 63) / 64 * 64;
    int e = 0;
    e |= st->cum_in.ensure((size_t)B * 2 * sizeof(double), true);
    e |= st->cum_sb.ensure((size_t)rows * 2 * sizeof(double), true);
    e |= st->fbin.ensure((size_t)B * F * 4 * 4, true);
    e |= st->fbx.ensure((size_t)st->rows_pad * st->Ipad * 2, true);
    e |= st->hseq.ensure((size_t)B * c.fb_hidden * 4 * 4, true);
    e |= st->fbout.ensure((size_t)B * F * 4 * 4, true);
    e |= st->ximg.ensure((size_t)ntiles * 16384, true);
    e |= st->c_fb.ensure(lstm_mma_cstate_bytes(c.num_layers, B, c.fb_hidden, &st->ra_fb), true);
    e |= st->c_sb.ensure(lstm_mma_cstate_bytes(c.num_layers, rows, c.sb_hidden, &st->ra_sb), true);
    e |= st->h_fb.ensure((size_t)c.num_layers * st->ra_fb * c.fb_hidden * 2, true);
    e |= st->h_sb.ensure((size_t)c.num_layers * st->ra_sb * c.sb_hidden * 2, true);
    st->use_ws = lstm_ws_supported(c.num_layers, c.fb_hidden, st->Ipad, B, m->num_sms) && !m->env_no_ws;
    if (st->use_ws) {
        e |= st->ws_h.ensure((size_t)c.num_layers * 2 * 64 * c.fb_hidden * 2, true);
        e |= st->ws_c.ensure((size_t)c.num_layers * 64 * c.fb_hidden * 4, true);
        e |= st->ws_bar.ensure(64, true);
    }
    if (e) { delete st; return fail(FSN_ECUDA, "stream state allocation failed"); }
    *out = st;
    return FSN_OK;
}

extern "C" void fsn_stream_destroy(fsn_stream* st) {
    if (!st) return;
    DevBuf* all[] = {&st->cum_in, &st->cum_sb, &st->fbin, &st->fbx, &st->hseq, &st->fbout, &st->ximg, &st->c_fb, &st->c_sb, &st->h_fb, &st->h_sb, &st->ws_h, &st->ws_c, &st->ws_bar};
    for (auto* b : all) b->release();
    delete st;
}

extern "C" int fsn_stream_step(fsn_stream* st, const float* d_mag, float* d_mask, int32_t* h_valid, void* stream) {
    if (!st || !d_mag || !d_mask) return fail(FSN_EINVAL, "null argument");
    fsn_model* m = st->m;
    const fsn_config& c = m->cfg;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int B = st->B, F = c.num_freqs, n = st->n, resume = n > 0;
    StreamNormLaunch na{d_mag, static_cast<float*>(st->fbin.p), static_cast<double*>(st->cum_in.p), B, F, 4, n, c.norm_type};
    launch_stream_norm(na, s);
    launch_fb_pack(static_cast<const float*>(st->fbin.p), static_cast<__half*>(st->fbx.p), B, F, 1, 4, st->rows_pad, st->Ipad, s);
    int e = 0;
    if (st->use_ws) {
        LstmWsLaunch w{};
        fill_ws(m, w);
        w.rows = B; w.rows_pad = st->rows_pad; w.Tp = 1;
        w.x = static_cast<const __half*>(st->fbx.p); w.hbuf = static_cast<__half*>(st->ws_h.p); w.cbuf = static_cast<float*>(st->ws_c.p);
        w.barrier = static_cast<unsigned int*>(st->ws_bar.p);
        w.hseq = static_cast<float*>(st->hseq.p); w.P = 4; w.resume = resume; w.t0 = n;
        e = launch_lstm_ws(w, s);
    } else {
        LstmMmaLaunch a{};
        for (int l = 0; l < c.num_layers; ++l) { a.w.wfrag[l] = static_cast<const uint4*>(m->fb_frag[l].p); a.w.bias[l] = static_cast<const float*>(m->fb_bias[l].p); }
        a.L = c.num_layers; a.H = c.fb_hidden; a.I = F; a.Ipad = st->Ipad; a.rows = B; a.Tp = 1;
        a.xplain = static_cast<const __half*>(st->fbx.p); a.rows_pad = st->rows_pad;
        a.cstate = static_cast<float*>(st->c_fb.p); a.rows_alloc = st->ra_fb;
        a.hseq = static_cast<float*>(st->hseq.p); a.P = 4; a.fast = c.fast_math; a.gru = c.rnn_type == FSN_RNN_GRU;
        a.hstate = static_cast<__half*>(st->h_fb.p); a.resume = resume;
        e = launch_lstm_mma(a, s);
    }
    if (e) return fail(FSN_ECUDA, "full-band LSTM step failed: %s", cudaGetErrorString((cudaError_t)e));
    ConvLaunch cf{};
    cf.X = static_cast<const float*>(st->hseq.p); cf.Y = static_cast<float*>(st->fbout.p);
    cf.Z = B; cf.M = F; cf.K = c.fb_hidden; cf.Tp = 1; cf.P = 4; cf.act = c.fb_act;
    cf.W = P(m, "fb_model.fc_output_layer.weight"); cf.bias = P(m, "fb_model.fc_output_layer.bias");
    launch_conv1x1(cf, s);
    StreamPackLaunch pa{d_mag, static_cast<const float*>(st->fbout.p), 4, static_cast<double*>(st->cum_sb.p), static_cast<__half*>(st->ximg.p),
                        B, F, c.sb_num_neighbors, c.fb_num_neighbors, n, c.norm_type};
    launch_stream_pack(pa, s);
    LstmMmaLaunch b{};
    for (int l = 0; l < c.num_layers; ++l) { b.w.wfrag[l] = static_cast<const uint4*>(m->sb_frag[l].p); b.w.bias[l] = static_cast<const float*>(m->sb_bias[l].p); }
    b.w.fc_w = P(m, "sb_model.fc_output_layer.weight"); b.w.fc_b = P(m, "sb_model.fc_output_layer.bias");
    b.L = c.num_layers; b.H = c.sb_hidden; b.I = m->Isb; b.Ipad = 64; b.rows = B * F; b.Tp = 1;
    b.img = static_cast<const __half*>(st->ximg.p); b.ntiles = (B * F + 127) / 128;
    b.cstate = static_cast<float*>(st->c_sb.p); b.rows_alloc = st->ra_sb;
    b.out = d_mask; b.O = c.output_size; b.F = F; b.la = 0; b.act = c.sb_act; b.fast = c.fast_math; b.gru = c.rnn_type == FSN_RNN_GRU;
    b.hstate = static_cast<__half*>(st->h_sb.p); b.resume = resume;
    e = launch_lstm_mma(b, s);
    if (e) return fail(FSN_ECUDA, "sub-band LSTM step failed: %s", cudaGetErrorString((cudaError_t)e));
    CK(cudaGetLastError());
    if (h_valid) *h_valid = (n >= c.look_ahead) ? 1 : 0;
    st->n++;
    return FSN_OK;
}

extern "C" int fsn_apply_cirm(const float* d_crm, const float* d_noisy, float* d_enh, int32_t B, int32_t F, int32_t T, void* stream) {
    if (!d_crm || !d_noisy || !d_enh || B < 1 || F < 1 || T < 1) return fail(FSN_EINVAL, "bad argument");
    launch_apply_cirm(d_crm, reinterpret_cast<const float2*>(d_noisy), reinterpret_cast<float2*>(d_enh), B, F, T, static_cast<cudaStream_t>(stream));
    CK(cudaGetLastError());
    return FSN_OK;
}

extern "C" int fsn_gemm_f16(const void* d_a, const void* d_b, void* d_c, int64_t M, int32_t N, int32_t K, int32_t tile_n, void* stream) {
    if (!d_a || !d_b || !d_c || !gemm_f16_supported(M, N, K) || (tile_n != 0 && tile_n != 128 && tile_n != 256))
        return fail(FSN_EINVAL, "fsn_gemm_f16: M = %lld, N = %d, K = %d, tile_n = %d: needs M %% 128 == 0, N %% 128 == 0, K %% 64 == 0, tile_n 0 / 128 / 256",
                    (long long)M, N, K, tile_n);
    int dev = 0, sms = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    GemmF16Launch g{M, N, K, static_cast<__half*>(d_c), N, tile_n};
    const int e = launch_gemm_f16(d_a, d_b, g, sms, static_cast<cudaStream_t>(stream));
    if (e) return fail(FSN_ECUDA, "fsn_gemm_f16 launch failed: %s", cudaGetErrorString((cudaError_t)e));
    return FSN_OK;
}
extern "C" int32_t fsn_gemm_f16_tile_n(int64_t M, int32_t N, int32_t K, int32_t tile_n) {
    if (!gemm_f16_supported(M, N, K)) return fail(FSN_EINVAL, "fsn_gemm_f16_tile_n: unsupported shape");
    GemmF16Launch g{M, N, K, nullptr, N, tile_n};
    return gemm_f16_pair_tiles(g) ? 256 : 128;
}

extern "C" int64_t fsn_model_last_launch_count(const fsn_model* m) { return m ? m->launches : 0; }
extern "C" int fsn_model_lstm_ms_history(fsn_model* m, float* h_ms, int32_t n) {
    if (!m || !h_ms || n < 1) return 0;
    int64_t avail = m->nfwd < fsn_model::NEV ? m->nfwd : fsn_model::NEV;
    if (n > avail) n = (int32_t)avail;
    for (int i = 0; i < n; ++i) {
        const int evi = (int)((m->nfwd - n + i) % fsn_model::NEV);
        float ms = -1.f;
        if (cudaEventSynchronize(m->ev1[evi]) != cudaSuccess || cudaEventElapsedTime(&ms, m->ev0[evi], m->ev1[evi]) != cudaSuccess) ms = -1.f;
        h_ms[i] = ms;
    }
    return n;
}
// [front start, front end, LSTM start, LSTM end] in ms relative to the front start of the oldest reported forward
extern "C" int fsn_model_timeline(fsn_model* m, float* h_ms4, int32_t n) {
    if (!m || !h_ms4 || n < 1) return 0;
    int64_t avail = m->nfwd < fsn_model::NEV ? m->nfwd : fsn_model::NEV;
    if (n > avail) n = (int32_t)avail;
    if (n < 1) return 0;
    const int base = (int)((m->nfwd - n) % fsn_model::NEV);
    for (int i = 0; i < n; ++i) {
        const int evi = (int)((m->nfwd - n + i) % fsn_model::NEV);
        cudaEvent_t ev[4] = {m->evf0[evi], m->evf1[evi], m->ev0[evi], m->ev1[evi]};
        for (int k = 0; k < 4; ++k) {
            float ms = -1.f;
            if (cudaEventSynchronize(ev[k]) != cudaSuccess || cudaEventElapsedTime(&ms, m->evf0[base], ev[k]) != cudaSuccess) ms = -1.f;
            h_ms4[4 * i + k] = ms;
        }
    }
    return n;
}
extern "C" float fsn_model_last_lstm_ms(fsn_model* m) {
    float ms = -1.f;
    return fsn_model_lstm_ms_history(m, &ms, 1) == 1 ? ms : -1.f;
}
extern "C" int fsn_model_last_lstm_impl(const fsn_model* m) { return m ? m->last_impl : 0; }

static int put_plan(const Plan& p, int32_t* Bs, int32_t* Tw, int32_t* Fc, int64_t* bytes) {
    *Bs = p.Bs; *Tw = p.Tw; *Fc = p.Fc;
    if (bytes) *bytes = p.bytes;
    return FSN_OK;
}

extern "C" int fsn_plan_forward_bins(const fsn_config* cfg, int32_t B, int32_t T, double cap_bytes, int32_t force_window, int32_t force_bins,
                                     int32_t* Bs, int32_t* Tw, int32_t* Fc, int64_t* bytes) {
    if (!cfg || !Bs || !Tw || !Fc || B < 1 || T < 1 || !(cap_bytes > 0)) return fail(FSN_EINVAL, "bad argument");
    if (force_window < 0 || force_window % 32) return fail(FSN_EINVAL, "force_window must be 0 or a positive multiple of 32");
    if (force_bins < 0) return fail(FSN_EINVAL, "force_bins must be 0 or a positive number of bins");
    if (cfg->num_freqs < 4 || cfg->num_layers < 1 || cfg->num_layers > 4 || cfg->look_ahead < 0) return fail(FSN_EINVAL, "bad configuration");
    if (int rc = check_length(*cfg, 1, T)) return rc;
    return put_plan(plan_forward(*cfg, runs_layerwise(*cfg, 0), B, T, cap_bytes, force_window, force_bins), Bs, Tw, Fc, bytes);
}

extern "C" int fsn_plan_forward(const fsn_config* cfg, int32_t B, int32_t T, double cap_bytes, int32_t force_window, int32_t* Bs, int32_t* Tw,
                                int64_t* bytes) {
    int32_t fc = 0;
    return fsn_plan_forward_bins(cfg, B, T, cap_bytes, force_window, 0, Bs, Tw, &fc, bytes);
}

extern "C" int fsn_model_plan_bins(const fsn_model* m, int32_t B, int32_t T, int32_t* Bs, int32_t* Tw, int32_t* Fc, int64_t* bytes) {
    if (!m || !Bs || !Tw || !Fc || B < 1 || T < 1) return fail(FSN_EINVAL, "bad argument");
    if (int rc = check_length(m->cfg, 1, T)) return rc;
    return put_plan(plan_forward(m->cfg, runs_layerwise(m->cfg, m->env_impl), B, T, m->ws_cap_bytes, m->env_sb_window, m->env_sb_chunk),
                    Bs, Tw, Fc, bytes);
}

extern "C" int fsn_model_plan(const fsn_model* m, int32_t B, int32_t T, int32_t* Bs, int32_t* Tw, int64_t* bytes) {
    int32_t fc = 0;
    return fsn_model_plan_bins(m, B, T, Bs, Tw, &fc, bytes);
}

extern "C" int fsn_model_release_workspace(fsn_model* m) {
    if (!m) return fail(FSN_EINVAL, "null model");
    CK(cudaDeviceSynchronize());                                         // nothing in flight may still read the buffers
    release_ws(*m);
    return FSN_OK;
}

extern "C" int64_t fsn_model_workspace_bytes(const fsn_model* m) {
    if (!m) return 0;
    fsn_model& mm = const_cast<fsn_model&>(*m);                          // the table's accessors are not const; nothing is changed
    size_t n = 0;
    for (const WsBuf& e : WS)
        for (int i = 0; i < ((e.flags & WS_LANE) ? 2 : 1); ++i) n += e.buf(mm, mm.lane[i]).bytes;
    return (int64_t)n;
}

extern "C" int fsn_model_last_plan(const fsn_model* m, int32_t* Bs, int32_t* Tw) {
    if (!m || !Bs || !Tw) return fail(FSN_EINVAL, "null argument");
    *Bs = m->plan.Bs; *Tw = m->plan.Tw;
    return FSN_OK;
}

extern "C" int fsn_model_last_plan_bins(const fsn_model* m, int32_t* Bs, int32_t* Tw, int32_t* Fc) {
    if (!m || !Bs || !Tw || !Fc) return fail(FSN_EINVAL, "null argument");
    return put_plan(m->plan, Bs, Tw, Fc, nullptr);
}
