// C ABI of fsnplus_b200 (include/fsnplus_b200.h): model object, parameter store keyed by the reference's
// state_dict names, packing into kernel layouts, and the forward orchestration.
#include "../../include/fsnplus_b200.h"
#include "fsn_common.cuh"
#include "fsn_kernels.h"

#include <algorithm>
#include <cerrno>
#include <cmath>
#include <cstdarg>
#include <cstddef>
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
    // against kernels on a non-blocking stream).  poison (FSN_POISON, fsn_model::env_poison): a buffer not promised zero is filled
    // whole with 0xFF bytes on the same stream at every call that ensures it -- NaN in fp16 / fp32 / fp64, -1 in int32 -- so that
    // a read of anything the call did not write shows in its outputs.  Without it nothing is enqueued unless the buffer grows.
    int ensure(size_t n, bool zero, cudaStream_t s = nullptr, bool poison = false) {
        if (n > bytes) {
            if (p) cudaFree(p);
            p = nullptr; bytes = 0;
            cudaError_t e = cudaMalloc(&p, n);
            if (e != cudaSuccess) return (int)e;
            bytes = n;
            if (zero && (e = cudaMemsetAsync(p, 0, n, s)) != cudaSuccess) return (int)e;
        }
        if (poison && !zero && p) return (int)cudaMemsetAsync(p, 0xFF, bytes, s);
        return 0;
    }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
};

// Pinned host staging of small int32 arrays on their way to the device: a ring of slots, each refilled only after the event recorded
// behind its last H2D copy has fired.  So the caller's host array is free when a call returns and no stream has to be synchronised.
struct PinnedStage {
    static const int NSLOT = 4;
    struct Slot { int32_t* h = nullptr; size_t cap = 0; cudaEvent_t ev = nullptr; bool used = false; } slot[NSLOT];
    int64_t next = 0;
    Slot* cur = nullptr;
    // The next slot, holding at least n int32, once the copy that last read it has completed
    int take(size_t n, int32_t** h) {
        Slot& g = *(cur = &slot[next++ % NSLOT]);
        if (!g.ev) CK(cudaEventCreateWithFlags(&g.ev, cudaEventDisableTiming));
        if (g.used) CK(cudaEventSynchronize(g.ev));
        if (g.cap < n) {
            // every slot grows at once: cudaFreeHost synchronises the device, so a call that stages more values than any before it
            // synchronises once, and the calls after it up to that size never do
            for (Slot& o : slot) {
                if (o.used) CK(cudaEventSynchronize(o.ev));
                if (o.h) CK(cudaFreeHost(o.h));
                o.h = nullptr; o.cap = 0;
                CK(cudaHostAlloc(reinterpret_cast<void**>(&o.h), n * sizeof(int32_t), cudaHostAllocDefault));
                o.cap = n;
            }
        }
        *h = g.h;
        return FSN_OK;
    }
    // Copy the first n int32 of the slot last taken to d on stream s
    int send(void* d, size_t n, cudaStream_t s) {
        CK(cudaMemcpyAsync(d, cur->h, n * sizeof(int32_t), cudaMemcpyHostToDevice, s));
        CK(cudaEventRecord(cur->ev, s));
        cur->used = true;
        return FSN_OK;
    }
    ~PinnedStage() {
        for (Slot& g : slot) {
            if (g.h) cudaFreeHost(g.h);
            if (g.ev) cudaEventDestroy(g.ev);
        }
    }
};

// The calls of one handle run in call order whatever streams they are issued on: each waits for the event recorded behind the
// previous one, then records its own.  The handle's state and scratch are shared by all its calls.
struct CallOrder {
    cudaEvent_t ev = nullptr;
    bool used = false;
    int wait(cudaStream_t s) {
        if (used) CK(cudaStreamWaitEvent(s, ev, 0));
        return FSN_OK;
    }
    int record(cudaStream_t s) {
        if (!ev) CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        CK(cudaEventRecord(ev, s));
        used = true;
        return FSN_OK;
    }
    // call f() between the two; the event is recorded even when f fails part-way, behind whatever it enqueued
    template <class Fn> int run(void* stream, Fn f) {
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        if (int rc = wait(s)) return rc;
        const int rc = f(), rr = record(s);
        return rc ? rc : rr;
    }
    ~CallOrder() { if (ev) cudaEventDestroy(ev); }
};

// weights_id: folds n bytes into h 8 bytes at a time (the last word zero-padded).  Each step is a bijection of h (xor, odd multiply,
// xorshift), so two byte strings of the same length that differ in any word give different results.
static uint64_t hash_words(uint64_t h, const void* p, size_t n) {
    const unsigned char* b = static_cast<const unsigned char*>(p);
    for (size_t i = 0; i < n; i += 8) {
        uint64_t w = 0;
        memcpy(&w, b + i, n - i < 8 ? n - i : 8);
        h = (h ^ w) * 0x100000001b3ull;
        h ^= h >> 29;
    }
    return h;
}

struct ParamSpec { std::string key; int64_t numel; };

// Every fsn_config field by name, in declaration order: the saved-session check (cfg_diff) and the model file's config section
// (fsn_model_file_write, read_model_file) name the fields from this one list
static const struct CfgField { const char* name; size_t off; } kCfgFields[] = {
    {"model_kind", offsetof(fsn_config, model_kind)}, {"num_freqs", offsetof(fsn_config, num_freqs)},
    {"look_ahead", offsetof(fsn_config, look_ahead)}, {"sb_num_neighbors", offsetof(fsn_config, sb_num_neighbors)},
    {"fb_num_neighbors", offsetof(fsn_config, fb_num_neighbors)}, {"fb_hidden", offsetof(fsn_config, fb_hidden)},
    {"sb_hidden", offsetof(fsn_config, sb_hidden)}, {"num_layers", offsetof(fsn_config, num_layers)},
    {"output_size", offsetof(fsn_config, output_size)}, {"fb_act", offsetof(fsn_config, fb_act)}, {"sb_act", offsetof(fsn_config, sb_act)},
    {"norm_type", offsetof(fsn_config, norm_type)}, {"kersize[0]", offsetof(fsn_config, kersize)},
    {"kersize[1]", offsetof(fsn_config, kersize) + 4}, {"kersize[2]", offsetof(fsn_config, kersize) + 8},
    {"lstm_impl", offsetof(fsn_config, lstm_impl)},
    {"fast_math", offsetof(fsn_config, fast_math)}, {"channel_attention", offsetof(fsn_config, channel_attention)},
    {"rnn_type", offsetof(fsn_config, rnn_type)}, {"subband_num", offsetof(fsn_config, subband_num)},
    {"tcn_causal", offsetof(fsn_config, tcn_causal)}, {"sb_tcn", offsetof(fsn_config, sb_tcn)}};
static_assert(sizeof(fsn_config) == sizeof(kCfgFields) / sizeof(kCfgFields[0]) * sizeof(int32_t), "kCfgFields names every fsn_config field");

// The packed block weights of one TCN (pack_tcn_blocks): nbr branches of C channels padded to Cp, gLN2 folded into the second 1x1
// convolution; NT / ntiles = N tile and N tiles of its Cp-wide GEMMs.
struct TcnWeights {
    const char* name = "";                             // in error messages
    int nbr = 0, C = 0, Cp = 0, NT = 0, ntiles = 0;
    DevBuf W1, W2, S1, S2b;                            // [8][nbr][512][Cp] tf32, [8][nbr][Cp][512] fp16, [8][nbr][Cp] x2
    struct Block { const float *conv1x1_b, *prelu1, *norm1_w, *norm1_b, *dw_w, *dw_b, *prelu2; } p[8][3];   // [block][branch], unpacked
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
    std::map<std::string, std::vector<float>> host;   // raw fp32 parameters (reference layout), copied to `arena` at finalize
    std::map<std::string, uint64_t> param_hash;       // per key: hash of the key and its fp32 bytes as set (fsn_model_set_param)
    uint64_t weights_id = 0;                          // the per-key hashes combined in key order at fsn_model_finalize; 0 before
    DevBuf arena;
    bool finalized = false;
    int Isb = 0;                                      // sub-band LSTM input size
    // packed LSTM weights
    DevBuf sb_frag[4], sb_bias[4];
    DevBuf fb_frag[4], fb_bias[4];
    // launch templates, bound at every fsn_model_finalize (bind_weights): weights and model constants only; each launch adds its geometry,
    // buffers and state, so none names a state_dict key.  The offline forward and the streaming step share them.
    TsseParams tsse[3] = {};                          // FullSubNet+: the channel attention of each branch
    LstmWsLaunch fb_ws{};                             // fullsubnet.Model: the full-band LSTM, weight-stationary kernel
    LstmMmaLaunch fb_mma{};                           // fullsubnet.Model: the full-band LSTM, generic kernel
    ConvLaunch fb_out{};                              // fullsubnet.Model: the full band's output Linear
    LstmMmaLaunch sb_mma{};                           // the sub-band LSTM, generic kernel
    const float *sb_fc_w = nullptr, *sb_fc_b = nullptr;   // the sub band's output Linear: layer-wise kernels, TCN head (bias only)
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
    int last_fb_ws = 0;                 // the last forward's full-band LSTM ran on the weight-stationary kernel (fsn_model_last_fb_ws)
    // tuning knobs, read ONCE at fsn_model_create (never on the forward path): FSN_LSTM_IMPL overrides cfg.lstm_impl,
    // FSN_NO_WS=1 keeps the full-band LSTM of fullsubnet.Model off the weight-stationary kernel
    int env_impl = 0;
    bool layerwise = false;                            // the sub-band route, fixed with config and knobs at create: runs_layerwise
    // FSN_FRONT_OVERLAP=1: the pipelined entry points run the front end of batch i+1 concurrently with the sub-band LSTM of batch i
    // (two lanes, two streams).  Off by default: no gain at the flagship size on the H100 (DESIGN.md §4), the LSTM occupies every SM.
    bool env_front_overlap = false;
    int env_pdl = -1;                                  // FSN_PDL: 0 / 1 / -1 (auto: small batches only)
    double ws_cap_bytes = 24e9;                        // FSN_WS_CAP_GB: larger batches are run as sub-batches (plain forward entry points)
    int env_sb_window = 0;                             // FSN_SB_WINDOW: force a sub-band time window of this many frames (multiple of 32)
    int env_sb_chunk = 0;                              // FSN_SB_CHUNK: run the sub-band TCN in chunks of this many bins (>= num_freqs: unchunked)
    Plan plan;                                         // plan of the last plain forward
    bool env_no_ws = false;
    // FSN_POISON=1 (tests): every call fills the scratch it uses that is not promised zero with NaN first (DevBuf::ensure's poison):
    // the forward workspace entries of WS without WS_ZERO, and the streaming and chunk-session scratch; handles made from the model
    // take it from here.  State, weights, tables and staging are never filled.
    bool env_poison = false;
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
    PinnedStage len_stage;                            // ragged forwards: the per-sample extents
    // audio call (fsn_model_enhance_audio): its workspace (the analysis planes, the enhanced spectrum) is in the table WS; the tables of
    // its n_fft are uploaded at finalize.  au_valid: the workspace holds the whole batch of the last forward, an audio call
    DevBuf au_planes, au_enh, au_tab;
    bool au_valid = false;
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

// A wide sub-band input (64 < Isb <= 128, DESIGN.md §3.3): packed as plain fp16 rows of 128 halves (the fused first-layer tile and the
// swizzled images hold 64); the layer-wise path projects it with one GEMM per window, the generic kernel reads it with Ipad = 128
static bool sb_wide(const fsn_config& c) { return sb_input_size(c) > 64; }
// bytes of one packed sub-band input row (one sequence, one frame)
static size_t sb_row_bytes(const fsn_config& c) { return sb_wide(c) ? 256 : 128; }

// The layer-wise kernels (k_lstm_tc5r.cu) take this geometry (hidden % 64 == 0 and <= 512, output_size 2, input <= 128): their weights are packed
static bool tc5r_ok(const fsn_config& c) {
    return !c.sb_tcn && lstm_tc5r_supported(c.sb_hidden, c.output_size) && sb_input_size(c) <= 128;
}

// The sub-band LSTM runs layer-wise (else on the generic mma.sync kernel): lstm_impl = auto or tcgen05 (FSN_LSTM_TCGEN05, the historical
// name of the tensor-core path) on a geometry those kernels take.  env_impl: FSN_LSTM_IMPL or 0.
static bool runs_layerwise(const fsn_config& c, int env_impl) {
    const int impl = env_impl ? env_impl : c.lstm_impl;
    return tc5r_ok(c) && (impl == FSN_LSTM_AUTO || impl == FSN_LSTM_TCGEN05);
}

// The state_dict keys and sizes a valid configuration expects, in the reference's order (fsn_model_param_info, the model file)
static std::vector<ParamSpec> param_specs(const fsn_config& c) {
    const int F = c.num_freqs;
    std::vector<ParamSpec> v;
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
    const int isb = sb_input_size(c);
    if (c.sb_tcn) tcn_specs(v, "sb_model", isb, c.output_size);           // hidden width 512: sb_hidden and num_layers are unused
    else lstm_specs(v, "sb_model", isb, c.sb_hidden, c.num_layers, c.output_size, c.rnn_type == FSN_RNN_GRU ? 3 : 4);
    return v;
}

// ---------------------------------------------------------------------------------------------
// packing
// ---------------------------------------------------------------------------------------------
using DevPtrs = std::map<std::string, const float*>;   // every parameter's copy in the arena, by key (fsn_model_finalize)
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
// boxes, W2' in NT-row boxes.  The parameters the kernels read unpacked are bound from dev into w.p.
static int pack_tcn_blocks(fsn_model* m, const DevPtrs& dev, TcnWeights& w, const char* name, const std::vector<std::string>& pre, int C,
                           int Cp) {
    const int nbr = (int)pre.size(), Hd = 512;
    w.name = name; w.nbr = nbr; w.C = C; w.Cp = Cp;
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
            w.p[blk][b] = {dev.at(q + "conv1x1.bias"), dev.at(q + "prelu1.weight"), dev.at(q + "norm1.weight"), dev.at(q + "norm1.bias"),
                           dev.at(q + "depthwise_conv.weight"), dev.at(q + "depthwise_conv.bias"), dev.at(q + "prelu2.weight")};
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
static int pack_tcn5(fsn_model* m, const DevPtrs& dev) {
    const fsn_config& c = m->cfg;
    const int F = c.num_freqs, Cp = (F + 31) / 32 * 32;
    const char* sfx[3] = {"", "_real", "_imag"};
    std::vector<std::string> pre;
    for (int b = 0; b < 3; ++b) pre.push_back(std::string("fb_model") + sfx[b] + ".sequence_model.");
    int rc = pack_tcn_blocks(m, dev, m->tcn_fb, "full-band TCN", pre, F, Cp);
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
static int pack_sb_tcn(fsn_model* m, const DevPtrs& dev) {
    const int I = m->Isb, O = m->cfg.output_size;
    int rc = pack_tcn_blocks(m, dev, m->tcn_sb, "sub-band TCN", {"sb_model.sequence_model."}, I, 64);
    if (rc) return rc;
    std::vector<float> fc((size_t)O * 64, 0.f);
    const auto& w = m->host["sb_model.fc_output_layer.weight"];
    for (int o = 0; o < O; ++o)
        for (int k = 0; k < I; ++k) fc[(size_t)o * 64 + k] = w[(size_t)o * I + k];
    if (upload(m->sb_fc, fc.data(), fc.size() * 4)) return fail(FSN_ECUDA, "upload of the sub-band TCN head failed");
    return FSN_OK;
}

// The launch templates of fsn_model (after the packers), each where its model part exists: the attention for FullSubNet+, the full band
// for fullsubnet.Model, the generic sub-band LSTM unless the sub band is a TCN
static void bind_weights(fsn_model* m, const DevPtrs& dev) {
    const fsn_config& c = m->cfg;
    const int L = c.num_layers, gru = c.rnn_type == FSN_RNN_GRU;
    if (c.model_kind == FSN_KIND_PLUS) {
        const char* sfx[3] = {"", "_real", "_imag"};
        const char* cn[3] = {"smallConv1d", "middleConv1d", "largeConv1d"};
        for (int b = 0; b < 3; ++b) {
            TsseParams& t = m->tsse[b];
            const std::string p = std::string("channel_attention") + sfx[b];
            if (c.channel_attention == FSN_ATTN_ECA) { t.eca_w = dev.at(p + ".conv.weight"); continue; }
            if (c.channel_attention == FSN_ATTN_TSSE) {
                for (int i = 0; i < 3; ++i) {
                    t.conv_w[i] = dev.at(p + "." + cn[i] + ".0.weight");
                    t.conv_b[i] = dev.at(p + "." + cn[i] + ".0.bias");
                }
                t.cat_w = dev.at(p + ".feature_concate_fc.weight"); t.cat_b = dev.at(p + ".feature_concate_fc.bias");
            }
            t.fc1_w = dev.at(p + ".fc1.weight"); t.fc1_b = dev.at(p + ".fc1.bias");
            t.fc2_w = dev.at(p + ".fc2.weight"); t.fc2_b = dev.at(p + ".fc2.bias");
        }
    } else {
        const int F = c.num_freqs, Ipad = (F + 15) / 16 * 16;
        LstmWsLaunch& w = m->fb_ws;
        LstmMmaLaunch& a = m->fb_mma;
        for (int l = 0; l < L; ++l) {
            const std::string q = "fb_model.sequence_model.", s = std::to_string(l);
            w.w_ih[l] = dev.at(q + "weight_ih_l" + s); w.w_hh[l] = dev.at(q + "weight_hh_l" + s);
            w.b_ih[l] = dev.at(q + "bias_ih_l" + s); w.b_hh[l] = dev.at(q + "bias_hh_l" + s);
            a.w.wfrag[l] = static_cast<const uint4*>(m->fb_frag[l].p);
            a.w.bias[l] = static_cast<const float*>(m->fb_bias[l].p);
        }
        w.L = L; w.H = c.fb_hidden; w.I = F; w.Ipad = Ipad; w.fast = c.fast_math; w.gru = gru;
        a.L = L; a.H = c.fb_hidden; a.I = F; a.Ipad = Ipad; a.fast = c.fast_math; a.gru = gru;
        ConvLaunch& cf = m->fb_out;
        cf.W = dev.at("fb_model.fc_output_layer.weight"); cf.bias = dev.at("fb_model.fc_output_layer.bias");
        cf.M = F; cf.K = c.fb_hidden; cf.act = c.fb_act;
    }
    m->sb_fc_b = dev.at("sb_model.fc_output_layer.bias");
    if (!c.sb_tcn) {
        m->sb_fc_w = dev.at("sb_model.fc_output_layer.weight");
        LstmMmaLaunch& a = m->sb_mma;
        for (int l = 0; l < L; ++l) {
            a.w.wfrag[l] = static_cast<const uint4*>(m->sb_frag[l].p);
            a.w.bias[l] = static_cast<const float*>(m->sb_bias[l].p);
        }
        a.w.fc_w = m->sb_fc_w; a.w.fc_b = m->sb_fc_b;
        a.L = L; a.H = c.sb_hidden; a.I = m->Isb; a.Ipad = sb_wide(c) ? 128 : 64;
        a.O = c.output_size; a.F = c.num_freqs; a.act = c.sb_act; a.fast = c.fast_math; a.gru = gru;
    }
}

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" int fsn_version(void) { return 101; }
extern "C" const char* fsn_last_error(void) { return g_err; }

// The configuration checks of fsn_model_create, host only: fsn_model_file_write and the model file reader refuse what create refuses,
// with the same code and message
static int config_check(const fsn_config& c) {
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
    if (c.sb_tcn && isb > 64)
        return fail(FSN_EINVAL, "sub-band input size %d > 64 not supported by the sub-band TCN (its output head holds a row's channels in one 64-column tile)", isb);
    if (isb > 128) return fail(FSN_EINVAL, "sub-band input size %d > 128 not supported", isb);
    return FSN_OK;
}

extern "C" int fsn_model_create(const fsn_config* cfg, fsn_model** out) {
    if (!cfg || !out) return fail(FSN_EINVAL, "null argument");
    const fsn_config& c = *cfg;
    if (int rc = config_check(c)) return rc;
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
    m->layerwise = runs_layerwise(c, m->env_impl);
    { const char* e = getenv("FSN_NO_WS"); m->env_no_ws = e && atoi(e) != 0; }
    { const char* e = getenv("FSN_POISON"); m->env_poison = e && atoi(e) != 0; }
    { const char* e = getenv("FSN_FRONT_OVERLAP"); m->env_front_overlap = e && atoi(e) != 0; }
    // FSN_PDL: programmatic dependent launch of the ~30 kernels of the front-end chain.  0 = never, 1 = always, unset = only for small
    // batches, where the forward is launch-latency-bound; for large batches a denser front end leaves no gaps for the side stream's
    // iSTFT kernels of the pipelined entry points.
    { const char* e = getenv("FSN_PDL"); m->env_pdl = e ? (atoi(e) != 0 ? 1 : 0) : -1; }
    { const char* e = getenv("FSN_WS_CAP_GB"); if (e && atof(e) > 0) m->ws_cap_bytes = atof(e) * 1e9; }
    m->Isb = sb_input_size(c);
    m->specs = param_specs(c);
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
    DevBuf* all[] = {&m->arena, &m->stage_in[0], &m->stage_in[1], &m->stage_in[2], &m->stage_out, &m->fb_fc, &m->fb_fc_b, &m->sb_fc, &m->au_tab};
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
            uint64_t x = hash_words(0xcbf29ce484222325ull, key, strlen(key));
            x = hash_words(x, &numel, sizeof(numel));
            m->param_hash[key] = hash_words(x, h, (size_t)numel * sizeof(float));
            m->finalized = false;
            m->weights_id = 0;
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
    DevPtrs dev;
    for (const auto& s : m->specs) {
        const auto& hv = m->host[s.key];
        float* d = reinterpret_cast<float*>(static_cast<char*>(m->arena.p) + off);
        CK(cudaMemcpy(d, hv.data(), hv.size() * 4, cudaMemcpyHostToDevice));
        dev[s.key] = d;
        off += (hv.size() * 4 + 255) & ~(size_t)255;
    }
    if (!c.sb_tcn && pack_lstm(m, "sb_model", m->Isb, sb_wide(c) ? 128 : 64, c.sb_hidden, c.num_layers, m->sb_frag, m->sb_bias))
        return fail(FSN_ECUDA, "packing sb_model failed");
    if (c.model_kind == FSN_KIND_FSN) {
        const int Ipad = (c.num_freqs + 15) / 16 * 16;
        if (pack_lstm(m, "fb_model", c.num_freqs, Ipad, c.fb_hidden, c.num_layers, m->fb_frag, m->fb_bias)) return fail(FSN_ECUDA, "packing fb_model failed");
    }
    if (tc5r_ok(c)) {
        const int H = c.sb_hidden;
        for (int l = 0; l < c.num_layers; ++l) {
            const std::string q = "sb_model.sequence_model.", sl = std::to_string(l);
            const bool fused = l == 0 && !sb_wide(c);                       // the input projection is part of the recurrence
            const int Kin = (l == 0) ? m->Isb : H, Kpad = (l == 0) ? (fused ? 64 : 128) : H;
            std::vector<uint16_t> st, wp;
            std::vector<float> bp;
            lstm_tc5r_pack_layer(H, Kin, Kpad, m->host[q + "weight_ih_l" + sl].data(), m->host[q + "weight_hh_l" + sl].data(),
                                 m->host[q + "bias_ih_l" + sl].data(), m->host[q + "bias_hh_l" + sl].data(), c.rnn_type == FSN_RNN_GRU, st, wp, bp);
            if (fused) {                                                    // first layer: [W_ih | W_hh] blocks, the input projection is in the recurrence
                st.assign((size_t)(H / 32) * (1 + H / 64) * 8192, 0);
                lstm_tc5_pack_first_layer(Kin, H, m->host[q + "weight_ih_l0"].data(), m->host[q + "weight_hh_l0"].data(), st.data());
            } else {                                                        // deeper layers, and a wide first layer: W_hh blocks + the input-projection GEMM's matrix
                lstm_tc5r_gin_order(H, Kpad, wp);
                if (upload(m->r_wih[l], wp.data(), wp.size() * 2)) return fail(FSN_ECUDA, "upload of the layer-wise LSTM weights failed");
            }
            if (upload(m->r_stream[l], st.data(), st.size() * 2) || upload(m->r_bias[l], bp.data(), bp.size() * 4))
                return fail(FSN_ECUDA, "upload of the layer-wise LSTM weights failed");
        }
    }
    if (c.model_kind == FSN_KIND_PLUS) {
        int rc = pack_tcn5(m, dev);
        if (rc) return rc;
    }
    if (c.sb_tcn) {
        int rc = pack_sb_tcn(m, dev);
        if (rc) return rc;
    }
    bind_weights(m, dev);
    const int nfft = 2 * (c.num_freqs - 1);
    if (nfft >= 64 && nfft <= 1024 && !(nfft & (nfft - 1))) {             // the audio call's tables, for the n_fft it takes (audio_fft_ok)
        std::vector<float> tab;
        audio_tables(nfft, tab);
        if (upload(m->au_tab, tab.data(), tab.size() * sizeof(float))) return fail(FSN_ECUDA, "upload of the audio tables failed");
    }
    // The uploads above are legacy-stream copies from pageable memory, which may return before their DMA lands, and the packers may
    // launch there: a forward on a non-blocking stream is not ordered after them, so the weights are in place when finalize returns
    CK(cudaDeviceSynchronize());
    uint64_t id = 0xcbf29ce484222325ull;
    for (const auto& kv : m->param_hash) id = hash_words(id, &kv.second, sizeof(kv.second));   // std::map: key order
    id ^= id >> 33; id *= 0xff51afd7ed558ccdull; id ^= id >> 33;                              // final avalanche
    m->weights_id = id ? id : 1;                                                               // 0 means "not finalized"
    m->finalized = true;
    return FSN_OK;
}

// ---------------------------------------------------------------------------------------------
// model file (DESIGN.md §3.15): the configuration by field name and the reference state_dict in one little-endian, versioned,
// checksummed file.  Host only.
// ---------------------------------------------------------------------------------------------
static_assert(__BYTE_ORDER__ == __ORDER_LITTLE_ENDIAN__, "the model file's integers and floats are copied in host byte order");
static const char kFileMagic[8] = {'F', 'S', 'N', 'M', 'O', 'D', 'E', 'L'};
static const uint32_t kFileVersion = 1;
static const uint64_t kFileHashBasis = 0xcbf29ce484222325ull;   // hash_words over every byte before the checksum, from the FNV-1a basis

static void put_bytes(std::vector<unsigned char>& b, const void* p, size_t n) {
    const unsigned char* c = static_cast<const unsigned char*>(p);
    b.insert(b.end(), c, c + n);
}
template <class T> static void put(std::vector<unsigned char>& b, T v) { put_bytes(b, &v, sizeof(T)); }

// Matches records (keys[i], numel[i]) with the configuration's spec list: (*rec)[s] is the record of spec s.  FSN_EINVAL with the
// messages of fsn_model_set_param (an unexpected key, a size mismatch) and fsn_model_finalize (a missing parameter), or a duplicate key.
static int match_params(const std::vector<ParamSpec>& specs, const std::vector<std::string>& keys, const std::vector<int64_t>& numel,
                        std::vector<int>* rec) {
    std::map<std::string, int> idx;
    for (size_t s = 0; s < specs.size(); ++s) idx[specs[s].key] = (int)s;
    rec->assign(specs.size(), -1);
    for (size_t i = 0; i < keys.size(); ++i) {
        const auto it = idx.find(keys[i]);
        if (it == idx.end()) return fail(FSN_EINVAL, "unexpected key %s", keys[i].c_str());
        const ParamSpec& s = specs[it->second];
        if (numel[i] != s.numel)
            return fail(FSN_EINVAL, "size mismatch for %s: expected %lld, got %lld", s.key.c_str(), (long long)s.numel, (long long)numel[i]);
        int& r = (*rec)[it->second];
        if (r >= 0) return fail(FSN_EINVAL, "duplicate key %s", s.key.c_str());
        r = (int)i;
    }
    for (size_t s = 0; s < specs.size(); ++s)
        if ((*rec)[s] < 0) return fail(FSN_EINVAL, "missing parameter %s", specs[s].key.c_str());
    return FSN_OK;
}

// Writes b to path through path + ".tmp" and a rename: a failed write leaves no file at path and removes its temporary
static int write_file(const char* path, const std::vector<unsigned char>& b) {
    const std::string tmp = std::string(path) + ".tmp";
    FILE* f = fopen(tmp.c_str(), "wb");
    if (!f) return fail(FSN_EINVAL, "cannot create %s: %s", tmp.c_str(), strerror(errno));
    int err = 0;
    if (fwrite(b.data(), 1, b.size(), f) != b.size()) err = errno ? errno : EIO;
    if (fflush(f) && !err) err = errno;
    if (fclose(f) && !err) err = errno;
    if (err) {
        remove(tmp.c_str());
        return fail(FSN_EINVAL, "writing %s failed: %s", tmp.c_str(), strerror(err));
    }
    if (rename(tmp.c_str(), path)) {
        err = errno;
        remove(tmp.c_str());
        return fail(FSN_EINVAL, "cannot rename %s to %s: %s", tmp.c_str(), path, strerror(err));
    }
    return FSN_OK;
}

extern "C" int fsn_model_file_write(const char* path, const fsn_config* cfg, int32_t n, const char* const* keys, const float* const* h_data,
                                    const int64_t* numel) {
    if (!path || !cfg) return fail(FSN_EINVAL, "null argument");
    if (n < 0) return fail(FSN_EINVAL, "n = %d: the parameter count is negative", n);
    if (n > 0 && (!keys || !h_data || !numel)) return fail(FSN_EINVAL, "null argument");
    if (int rc = config_check(*cfg)) return rc;
    std::vector<std::string> k(n);
    for (int i = 0; i < n; ++i) {
        if (!keys[i] || !h_data[i]) return fail(FSN_EINVAL, "null argument: keys[%d] or h_data[%d]", i, i);
        k[i] = keys[i];
    }
    const std::vector<ParamSpec> specs = param_specs(*cfg);
    std::vector<int> rec;
    if (int rc = match_params(specs, k, std::vector<int64_t>(numel, numel + n), &rec)) return rc;
    size_t bytes = sizeof(kFileMagic) + 4 + 4 + 4 + 8;
    for (const auto& f : kCfgFields) bytes += 2 + strlen(f.name) + 4;
    for (const auto& s : specs) bytes += 2 + s.key.size() + 8 + (size_t)s.numel * 4;
    std::vector<unsigned char> b;
    b.reserve(bytes);
    put_bytes(b, kFileMagic, sizeof(kFileMagic));
    put<uint32_t>(b, kFileVersion);
    put<uint32_t>(b, (uint32_t)(sizeof(kCfgFields) / sizeof(kCfgFields[0])));
    for (const auto& f : kCfgFields) {
        int32_t v;
        memcpy(&v, reinterpret_cast<const char*>(cfg) + f.off, 4);
        put<uint16_t>(b, (uint16_t)strlen(f.name));
        put_bytes(b, f.name, strlen(f.name));
        put<int32_t>(b, v);
    }
    put<uint32_t>(b, (uint32_t)specs.size());
    for (size_t s = 0; s < specs.size(); ++s) {
        put<uint16_t>(b, (uint16_t)specs[s].key.size());
        put_bytes(b, specs[s].key.data(), specs[s].key.size());
        put<int64_t>(b, specs[s].numel);
        put_bytes(b, h_data[rec[s]], (size_t)specs[s].numel * 4);
    }
    put<uint64_t>(b, hash_words(kFileHashBasis, b.data(), b.size()));
    return write_file(path, b);
}

// One parameter record of a model file: its key, size and the byte offset of its float32 data
struct FileRecord { std::string key; int64_t numel; size_t off; };

// Reads and verifies a whole model file: magic, version, bounds, trailing bytes, checksum, config field names, the configuration
// (config_check) and the key set (match_params).  On success *cfg is the configuration, *bytes the file and *recs its records in
// spec order.  Every error is FSN_EINVAL; a structural one names the file and, for a truncation, the byte offset.
static int read_model_file(const char* path, fsn_config* cfg, std::vector<unsigned char>* bytes, std::vector<FileRecord>* recs) {
    FILE* f = fopen(path, "rb");
    if (!f) return fail(FSN_EINVAL, "cannot open %s: %s", path, strerror(errno));
    std::vector<unsigned char>& b = *bytes;
    size_t n = 0;
    b.resize(1 << 20);
    for (;;) {
        n += fread(b.data() + n, 1, b.size() - n, f);
        if (n < b.size()) break;
        b.resize(2 * b.size());
    }
    b.resize(n);
    const bool rerr = ferror(f);
    fclose(f);
    if (rerr) return fail(FSN_EINVAL, "reading %s failed", path);

    size_t pos = 0;
    auto get = [&](void* dst, uint64_t k, const std::string& what) -> int {
        if (n - pos < k)
            return fail(FSN_EINVAL, "model file %s: truncated: %s at byte %zu needs %llu bytes, the file ends at byte %zu", path, what.c_str(),
                        pos, (unsigned long long)k, n);
        if (dst) memcpy(dst, b.data() + pos, k);
        pos += k;
        return FSN_OK;
    };
    char magic[8];
    if (int rc = get(magic, 8, "the magic")) return rc;
    if (memcmp(magic, kFileMagic, 8)) return fail(FSN_EINVAL, "model file %s: bad magic (not an FSNMODEL file)", path);
    uint32_t version = 0, nfield = 0, nparam = 0;
    if (int rc = get(&version, 4, "the format version")) return rc;
    if (version != kFileVersion) return fail(FSN_EINVAL, "model file %s: format version %u, this library reads version %u", path, version, kFileVersion);
    if (int rc = get(&nfield, 4, "the config field count")) return rc;
    std::vector<std::pair<std::string, int32_t>> fields;
    for (uint32_t i = 0; i < nfield; ++i) {
        const std::string at = "config field " + std::to_string(i);
        uint16_t len = 0;
        int32_t v = 0;
        if (int rc = get(&len, 2, "the name length of " + at)) return rc;
        std::string name(len, '\0');
        if (int rc = get(&name[0], len, "the name of " + at)) return rc;
        if (int rc = get(&v, 4, "the value of config field " + name)) return rc;
        fields.emplace_back(name, v);
    }
    if (int rc = get(&nparam, 4, "the parameter count")) return rc;
    std::vector<FileRecord> r;
    for (uint32_t i = 0; i < nparam; ++i) {
        const std::string at = "parameter " + std::to_string(i);
        uint16_t len = 0;
        if (int rc = get(&len, 2, "the key length of " + at)) return rc;
        if (len == 0 || len > 255)
            return fail(FSN_EINVAL, "model file %s: %s: key length %u at byte %zu (a key is 1..255 bytes)", path, at.c_str(), len, pos - 2);
        FileRecord q;
        q.key.assign(len, '\0');
        if (int rc = get(&q.key[0], len, "the key of " + at)) return rc;
        if (int rc = get(&q.numel, 8, "the size of parameter " + q.key)) return rc;
        if (q.numel < 0) return fail(FSN_EINVAL, "model file %s: parameter %s: negative size %lld at byte %zu", path, q.key.c_str(), (long long)q.numel, pos - 8);
        q.off = pos;
        const uint64_t data = (uint64_t)q.numel <= UINT64_MAX / 4 ? (uint64_t)q.numel * 4 : UINT64_MAX;
        if (int rc = get(nullptr, data, "the data of parameter " + q.key)) return rc;
        r.push_back(std::move(q));
    }
    if (n - pos < 8) return get(nullptr, 8, "the checksum");
    if (n - pos > 8) return fail(FSN_EINVAL, "model file %s: %zu trailing bytes after the checksum at byte %zu", path, n - pos - 8, pos);
    uint64_t stored;
    memcpy(&stored, b.data() + pos, 8);
    const uint64_t sum = hash_words(kFileHashBasis, b.data(), pos);
    if (stored != sum)
        return fail(FSN_EINVAL, "model file %s: checksum mismatch (stored %016llx, computed %016llx): the file is corrupt", path,
                    (unsigned long long)stored, (unsigned long long)sum);

    fsn_config c;
    memset(&c, 0, sizeof(c));                                         // a field the file does not name takes 0, the documented default
    std::vector<bool> seen(sizeof(kCfgFields) / sizeof(kCfgFields[0]), false);
    for (const auto& fv : fields) {
        size_t j = 0;
        while (j < seen.size() && fv.first != kCfgFields[j].name) ++j;
        if (j == seen.size()) return fail(FSN_EINVAL, "model file %s: unknown config field \"%s\"", path, fv.first.c_str());
        if (seen[j]) return fail(FSN_EINVAL, "model file %s: config field %s appears twice", path, kCfgFields[j].name);
        seen[j] = true;
        memcpy(reinterpret_cast<char*>(&c) + kCfgFields[j].off, &fv.second, 4);
    }
    if (int rc = config_check(c)) return rc;
    std::vector<std::string> keys;
    std::vector<int64_t> numel;
    for (const auto& q : r) { keys.push_back(q.key); numel.push_back(q.numel); }
    std::vector<int> rec;
    const std::vector<ParamSpec> specs = param_specs(c);
    if (int rc = match_params(specs, keys, numel, &rec)) return rc;
    recs->clear();
    for (int i : rec) recs->push_back(r[i]);
    *cfg = c;
    return FSN_OK;
}

extern "C" int fsn_model_file_config(const char* path, fsn_config* cfg) {
    if (!path || !cfg) return fail(FSN_EINVAL, "null argument");
    fsn_config c;
    std::vector<unsigned char> b;
    std::vector<FileRecord> recs;
    if (int rc = read_model_file(path, &c, &b, &recs)) return rc;
    *cfg = c;
    return FSN_OK;
}

extern "C" int fsn_model_load(const char* path, fsn_model** out) {
    if (!out) return fail(FSN_EINVAL, "null argument");
    *out = nullptr;
    if (!path) return fail(FSN_EINVAL, "null argument");
    fsn_config c;
    std::vector<unsigned char> b;
    std::vector<FileRecord> recs;
    if (int rc = read_model_file(path, &c, &b, &recs)) return rc;
    fsn_model* m = nullptr;
    if (int rc = fsn_model_create(&c, &m)) return rc;
    std::vector<float> v;                                             // the records' data is not 4-byte aligned in the file
    for (const auto& q : recs) {
        v.resize((size_t)q.numel);
        memcpy(v.data(), b.data() + q.off, (size_t)q.numel * 4);
        if (int rc = fsn_model_set_param(m, q.key.c_str(), v.data(), q.numel)) { fsn_model_destroy(m); return rc; }
    }
    if (int rc = fsn_model_finalize(m)) { fsn_model_destroy(m); return rc; }
    *out = m;
    return FSN_OK;
}

// The implementation the sub-band LSTM reports (last_impl), and the one a forced lstm_impl names in its error
static int pick_impl(const fsn_model* m) {
    const int impl = m->env_impl ? m->env_impl : m->cfg.lstm_impl;
    return m->layerwise ? FSN_LSTM_TCGEN05 : impl == FSN_LSTM_AUTO ? FSN_LSTM_MMA : impl;
}

// Encode the tensor maps of TCN w's scratch over `rows` rows
static int map_tcn_scratch(TcnScratch& sc, const TcnWeights& w, long long rows) {
    if (make_tmap_f32_2d(sc.mapXa, sc.xa.p, rows, w.Cp, 128) || make_tmap_f32_2d(sc.mapXb, sc.xb.p, rows, w.Cp, 128) ||
        make_tmap_f16_2d(sc.mapY2, sc.y2.p, rows, 512, 128))
        return fail(FSN_ECUDA, "cuTensorMapEncodeTiled failed for the %s", w.name);
    return FSN_OK;
}

// Bytes of every forward workspace buffer for a batch of B clips of T frames, the sub-band images and the layer-wise path's Gin / layer
// output sized by the window Tw (0: the whole clip), the sub-band TCN's input and scratch by the bin chunk Fc (0: all bins); with
// audio (fsn_model_enhance_audio) also its analysis planes and enhanced spectrum, and the clips' sample counts.  One field per entry of
// the table WS; ensure_ws allocates exactly these sizes, so the plan's count is what a forward holds.
struct WsSizes {
    size_t fbin = 0, fbout = 0, mu = 0, sigma = 0, tsse_scale = 0, sb_rowsum = 0, xn = 0, tlen = 0;       // lane: front end, ragged extents
    size_t sbx = 0, ximg = 0;                                                   // lane: sub-band TCN input, or the sub-band images
    size_t x0 = 0, xr = 0, tcn_xa = 0, tcn_xb = 0, tcn_y1 = 0, tcn_y2 = 0, tcn_stats = 0;   // lane, FullSubNet+: the full-band TCN
    size_t magpad = 0, fbx = 0, hseq = 0;                                       // lane, fullsubnet.Model
    size_t cstate = 0, r_gin = 0, r_hseq = 0, r_hstate = 0, sb_cum = 0;         // sub-band LSTM scratch
    size_t sb_xa = 0, sb_xb = 0, sb_y1 = 0, sb_y2 = 0, sb_stats = 0;            // sub-band TCN scratch
    size_t ws_h = 0, ws_bar = 0;                                                // fullsubnet.Model's weight-stationary h exchange, barrier
    size_t mask_tmp = 0;                                                        // the generic kernel's scratch mask: not counted
    size_t au_planes = 0, au_enh = 0;                                           // audio call: mag / real / imag planes, enhanced spectrum
    size_t total() const;
};
static WsSizes ws_sizes(const fsn_config& c, bool layerwise, int B, int T, int Tw, int Fc = 0, bool audio = false, bool lim = false) {
    WsSizes z;
    const int F = c.num_freqs, Tp = T + c.look_ahead, Pp = (Tp + 3) & ~3, Ts = Tw ? Tw : Tp;
    const int nbr = (c.model_kind == FSN_KIND_PLUS) ? 3 : 1;
    const size_t rows = (size_t)B * F, ntiles = ((rows + 127) / 128 + 1) / 2 * 2;   // whole pairs of 128-row tiles (clusters of k_lstm_tc5r.cu)
    z.fbin = z.fbout = (size_t)nbr * B * F * Pp * 4;
    // fbout is also input_norm_kernel's per-frame scratch: it runs before anything writes or reads the full-band outputs (front_end).
    // num_freqs >= 4 makes the scratch (16 bytes per frame) fit within fbout's F * Pp * 4 bytes; the max keeps that explicit.
    if (c.norm_type != FSN_NORM_OFFLINE_LAPLACE) z.fbout = std::max(z.fbout, input_norm_frames_bytes(nbr, B, Tp));
    z.mu = z.sigma = (size_t)B * 4;
    z.tsse_scale = (size_t)nbr * B * F * 4 * (1 + tsse_row_floats());          // per-row scale | row statistics
    z.sb_rowsum = (size_t)B * 4 * F * 2 * 4;
    z.tlen = (size_t)(3 + audio + lim) * B * sizeof(int32_t);                   // counted whether the forward is ragged or not; lim: the
                                                                                // clips' attenuation floors (stage_lengths)
    if (audio) { z.au_planes = (size_t)3 * B * F * T * 4; z.au_enh = (size_t)B * F * T * 8; }
    if (c.norm_type != FSN_NORM_OFFLINE_LAPLACE) z.xn = (size_t)nbr * B * F * Tp * 4;
    if (c.sb_tcn) {
        const size_t seqs = (size_t)B * (Fc ? Fc : F), srows = seqs * Tp;      // the sequences of one chunk run
        z.sbx = srows * 64 * 4 + seqs * 4;                                      // input | block 0's stream maxima
        z.sb_xa = z.sb_xb = srows * 64 * 4; z.sb_y1 = z.sb_y2 = srows * 512 * sizeof(__half); z.sb_stats = tcn_stats_bytes(seqs);
    } else {
        z.ximg = ntiles * Ts * 128 * sb_row_bytes(c);                          // wide: GEMM rows / time-major rows of 128 halves
    }
    int ra = 0;
    size_t cs = c.sb_tcn ? 0 : lstm_mma_cstate_bytes(c.num_layers, (int)rows, c.sb_hidden, &ra), cs5 = 0;
    if (layerwise) {
        const size_t M = ntiles * Ts * 128;
        cs5 = lstm_tc5r_cstate_bytes((int)ntiles, c.sb_hidden);
        if (c.num_layers > 1 || sb_wide(c)) z.r_gin = M * 4 * c.sb_hidden * 2;   // a wide layer 0 is projected by the GEMM too
        if (c.num_layers > 1) z.r_hseq = M * c.sb_hidden * 2;
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
    WS_ZERO = 2,        // a fresh allocation is zero-filled, on the buffer's stream; without it, FSN_POISON fills it with NaN at every call
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
    {LANE_BUF(fbout), &WsSizes::fbout, WS_LANE | WS_ZERO},                         // first input_norm_kernel's scratch (ws_sizes)
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
    {MODEL_BUF(ws_h), &WsSizes::ws_h, WS_ON_USE},                                  // front_end: zeroed by every forward that uses it
    {MODEL_BUF(ws_bar), &WsSizes::ws_bar, WS_ON_USE},
    {MODEL_BUF(mask_tmp), &WsSizes::mask_tmp, WS_ON_USE},                          // run_sb_lstm
    {MODEL_BUF(au_planes), &WsSizes::au_planes, 0},                                // written whole by the analysis kernel
    {MODEL_BUF(au_enh), &WsSizes::au_enh, 0},                                      // written whole by the sub-band stage's epilogue
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
    m.au_valid = false;
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
// Clips of one forward that the launch grids hold: gridDim.y and gridDim.z take at most 65535 blocks, and the front end's
// tsse_apply_kernel puts its (branch, clip) planes on gridDim.z (3 B in FullSubNet+); the sub-band packer, fullsubnet.Model's
// full-band output convolution and the audio transforms put the clips on gridDim.y or z.
static const long long FSN_MAX_GRID_YZ = 65535;
static long long max_clips_for_grid(const fsn_config& c) { return FSN_MAX_GRID_YZ / (c.model_kind == FSN_KIND_PLUS ? 3 : 1); }
static int check_length(const fsn_config& c, int B, int T, bool front = true) {
    const long long Tp = (long long)T + c.look_ahead;
    if (Tp > FSN_MAX_TP) return fail(FSN_EINVAL, "T + look_ahead = %lld frames exceeds the limit of %lld (65535 x 256, the TCN convolution grid)", Tp, FSN_MAX_TP);
    if ((long long)c.num_freqs * Tp > 0x7fffffffLL)
        return fail(FSN_EINVAL, "num_freqs x (T + look_ahead) = %lld exceeds 2^31 - 1, the per-clip plane index limit", (long long)c.num_freqs * Tp);
    if (B > max_clips_for_rows(c, T))
        return fail(FSN_EINVAL, "3 x B x (T + look_ahead) = %lld rows exceeds the full-band TCN's 2^31 row limit", 3LL * B * Tp);
    const long long glim = front ? max_clips_for_grid(c) : FSN_MAX_GRID_YZ;   // the sub-band hook runs no front end (no TSSE planes)
    if (B > glim)
        return fail(FSN_EINVAL, "B = %d clips exceeds the launch-grid limit of %lld clips per forward (65535 blocks on gridDim.y / z%s)", B,
                    glim, front && c.model_kind == FSN_KIND_PLUS ? ", 3 B for the TSSE planes" : "");
    return FSN_OK;
}

// One offline call, as every offline entry point fills it, checks it once (check_batch) and runs it (run_plain, submit_impl, the test
// hook): B clips of T frames (the audio call: T of its longest clip), their inputs and one output.  The kind of entry point (call)
// decides the checks and the way the batch runs.
enum Call { CALL_FORWARD, CALL_PIPELINED, CALL_AUDIO, CALL_HOOK };
struct Batch {
    Call call = CALL_FORWARD;
    const float *mag = nullptr, *real = nullptr, *imag = nullptr;   // noisy spectra [B, F, T] (the audio call: its STFT planes)
    int B = 0, T = 0;
    const int32_t* frames = nullptr;           // frame count of every clip of a ragged batch; null: every clip spans T frames
    float *mask = nullptr, *enh = nullptr;     // output: the mask [B, O, F, T] or the enhanced spectrum [B, F, T] complex
    // the audio call: waveform rows [B, L] in and out and the clips' sample counts (null: every clip is L samples); once checked, the
    // longest clip Lall and the counts as int32 (null: every clip is Lall samples)
    const float* wave = nullptr; float* wave_out = nullptr; long long L = 0; const int64_t* lengths = nullptr;
    int Lall = 0; const int32_t* samples = nullptr;
    const float* raw = nullptr; int Tw = 0;    // the test hook: the sub-band input [B*F, Isb, T'] and its time window
    // the _lim calls: every clip's attenuation limit in dB (host, null: none); once checked, its floor lam = 10^(-dB / 20) per clip (host,
    // null when every floor is 0: the batch then runs exactly the unlimited forward) and, in the forward, the floors on the device
    const float* atten_db = nullptr; const float* lam = nullptr; const float* dlam = nullptr;
};

// The longest TSSE kernel (1 without the TSSE attention): every clip needs frames + look_ahead >= it
static int tsse_kmax(const fsn_config& c) {
    int k = 1;
    if (c.model_kind == FSN_KIND_PLUS && c.channel_attention == FSN_ATTN_TSSE)
        for (int i = 0; i < 3; ++i) k = c.kersize[i] > k ? c.kersize[i] : k;
    return k;
}

// The frame counts of a ragged batch: each in 1..T, and long enough for the TSSE convolutions.  Drops them (b.frames = null) when every
// clip spans all T frames, so that case runs exactly the unmasked forward.
static int check_frames(const fsn_config& c, Batch& b) {
    if (!b.frames) return FSN_OK;
    const int kmax = tsse_kmax(c);
    bool all = true;
    for (int i = 0; i < b.B; ++i) {
        const int n = b.frames[i];
        if (n < 1 || n > b.T) return fail(FSN_EINVAL, "frames[%d] = %d is outside 1..T = %d", i, n, b.T);
        if (n + c.look_ahead < kmax)
            return fail(FSN_EINVAL, "frames[%d] = %d: frames + look_ahead = %d is shorter than the TSSE kernel size %d", i, n, n + c.look_ahead, kmax);
        all = all && n == b.T;
    }
    if (all) b.frames = nullptr;
    return FSN_OK;
}

// The audio call's geometry: n_fft = 2 (num_freqs - 1) a power of two from 64 to 1024
static int audio_fft_ok(const fsn_config& c) {
    const int N = 2 * (c.num_freqs - 1);
    if (N < 64 || N > 1024 || (N & (N - 1)))
        return fail(FSN_EINVAL, "num_freqs %d: the audio call needs n_fft = 2 (num_freqs - 1) to be a power of two from 64 to 1024 "
                                "(num_freqs 33, 65, 129, 257 or 513)", c.num_freqs);
    return FSN_OK;
}

// The audio call's geometry and clips (check_batch, fsn_plan_audio): n_fft = 2 (num_freqs - 1), every clip longer than n_fft / 2
// (torch.stft's reflect padding) and no longer than L, with enough frames for the TSSE kernels (check_frames, in samples), and the
// forward's length limits on T = max_b L_b / hop + 1.  *Lmax: the longest clip; *all: every clip is Lmax samples long.
static int audio_check(const fsn_config& c, int32_t B, int64_t L, const int64_t* h_lengths, int* T, int* Lmax, bool* all) {
    if (int rc = audio_fft_ok(c)) return rc;
    if (B < 1) return fail(FSN_EINVAL, "B = %d: the batch needs at least one clip", B);
    if (L < 1 || L > 0x7fffffffLL) return fail(FSN_EINVAL, "L = %lld: the row length must be 1 .. 2^31 - 1 samples", (long long)L);
    const int H = c.num_freqs - 1, kmax = tsse_kmax(c);                 // hop = n_fft / 2
    long long mx = 0;
    *all = true;
    for (int b = 0; b < (h_lengths ? B : 1); ++b) {
        const long long n = h_lengths ? h_lengths[b] : L;
        char nm[40];
        if (h_lengths) snprintf(nm, sizeof(nm), "clip %d: h_lengths[%d]", b, b);
        else snprintf(nm, sizeof(nm), "L");
        if (n <= H)
            return fail(FSN_EINVAL, "%s = %lld: a clip needs more than n_fft / 2 = %d samples (torch.stft's reflect padding)", nm, n, H);
        if (n > L) return fail(FSN_EINVAL, "%s = %lld exceeds the row length L = %lld", nm, n, (long long)L);
        if (n / H + 1 + c.look_ahead < kmax)
            return fail(FSN_EINVAL, "%s = %lld samples give %lld frames: frames + look_ahead = %lld is shorter than the TSSE kernel size %d "
                                    "(a clip needs at least %lld samples)", nm, n, n / H + 1, n / H + 1 + c.look_ahead, kmax,
                        (long long)(kmax - c.look_ahead - 1) * H);
        if (b && n != mx) *all = false;
        if (n > mx) mx = n;
    }
    *Lmax = (int)mx;
    *T = (int)(mx / H + 1);
    return check_length(c, 1, *T);
}

// An attenuation limit of L dB (DESIGN.md §3.18), entry i of h_atten_db: L >= 0 or +inf, else FSN_EINVAL naming what it limits (the clip
// or slot `id`) and the value.  Its floor lam = 10^(-L / 20), computed in double and rounded to float (+inf: 0, no limit).
static int atten_floor(double db, const char* what, int id, int i, float* lam) {
    if (!(db >= 0.0))
        return fail(FSN_EINVAL, "%s %d: h_atten_db[%d] = %g: an attenuation limit is a number of dB >= 0 (+inf: no limit)", what, id, i, db);
    *lam = (float)std::pow(10.0, -db / 20.0);
    return FSN_OK;
}

// The floors of b's clips into lam from b.atten_db; b.lam stays null when there is no array or every floor is 0 (no limit on any clip)
static int check_atten(Batch& b, std::vector<float>* lam) {
    if (!b.atten_db) return FSN_OK;
    lam->resize((size_t)b.B);
    bool any = false;
    for (int i = 0; i < b.B; ++i) {
        if (int rc = atten_floor(b.atten_db[i], "clip", i, i, &(*lam)[i])) return rc;
        any = any || (*lam)[i] > 0.f;
    }
    if (any) b.lam = lam->data();
    return FSN_OK;
}

// Every check of an offline call, before it allocates, copies, records or waits on anything.  The audio call also sets b.T and
// b.Lall and, for a ragged batch, b.samples and b.frames (unless every clip has T frames) into lens.  A plain forward is checked for
// the length limits of one clip: plan_forward keeps every sub-batch within them.
static int check_batch(const fsn_model* m, Batch& b, std::vector<int32_t>* lens = nullptr, std::vector<float>* lam = nullptr) {
    if (b.atten_db && (!lam || b.call == CALL_PIPELINED || b.call == CALL_HOOK)) return fail(FSN_EINVAL, "this call takes no attenuation limit");
    if (b.call == CALL_AUDIO) {
        if (!m) return fail(FSN_EINVAL, "m is null");
        if (!b.wave) return fail(FSN_EINVAL, "d_wave is null ([B, L] float32 samples on the device)");
        if (!b.wave_out) return fail(FSN_EINVAL, "d_out is null ([B, L] float32 on the device)");
        if (!m->finalized) return fail(FSN_ESTATE, "fsn_model_finalize has not been called");
        bool all = true;
        if (int rc = audio_check(m->cfg, b.B, b.L, b.lengths, &b.T, &b.Lall, &all)) return rc;
        if (m->cfg.output_size != 2) return fail(FSN_EINVAL, "the audio call needs output_size 2 (a complex mask)");
        if (!all) {                                                     // ragged: every clip's sample count, then its frame count
            lens->resize(2 * (size_t)b.B);
            for (int i = 0; i < b.B; ++i) (*lens)[b.B + i] = ((*lens)[i] = (int32_t)b.lengths[i]) / (m->cfg.num_freqs - 1) + 1;
            b.samples = lens->data(); b.frames = lens->data() + b.B;
        }
        if (int rc = check_frames(m->cfg, b)) return rc;                // drops the frame counts when every clip has T frames
        return check_atten(b, lam);
    }
    const bool hook = b.call == CALL_HOOK;
    if (!m || !(hook ? b.raw : b.mag) || (!b.mask && !b.enh)) return fail(FSN_EINVAL, "null argument");
    if (!m->finalized) return fail(FSN_ESTATE, "fsn_model_finalize has not been called");
    const fsn_config& c = m->cfg;
    if (hook && c.sb_tcn) return fail(FSN_EINVAL, "fsn_model_sb_forward runs the sub-band LSTM / GRU; this model's sub-band model is the TCN");
    if (b.enh && (!b.real || !b.imag)) return fail(FSN_EINVAL, "the enhanced-spectrum output needs the noisy real and imaginary planes");
    if (b.enh && c.output_size != 2) return fail(FSN_EINVAL, "the enhanced-spectrum output needs output_size 2 (a complex mask)");
    if (b.B < 1 || b.T < 1) return fail(FSN_EINVAL, "bad batch/frames");
    if (!hook && c.model_kind == FSN_KIND_PLUS && (!b.real || !b.imag)) return fail(FSN_EINVAL, "FullSubNet_Plus.forward needs mag, real and imag");
    if (hook && (b.Tw < 0 || b.Tw % 32)) return fail(FSN_EINVAL, "Tw = %d: the window must be 0 or a positive multiple of 32 frames", b.Tw);
    if (hook && b.Tw && !m->layerwise) return fail(FSN_EINVAL, "time windows of the sub-band stage need the layer-wise LSTM path");
    if (int rc = check_frames(c, b)) return rc;
    if (!hook && b.T + c.look_ahead < tsse_kmax(c)) return fail(FSN_EINVAL, "sequence shorter than the TSSE kernel size");
    if (b.atten_db && !b.enh) return fail(FSN_EINVAL, "an attenuation limit applies to the enhanced spectrum, not to the mask");
    if (int rc = check_length(c, b.call == CALL_FORWARD ? 1 : b.B, b.T, !hook)) return rc;
    return check_atten(b, lam);
}

// Size lane ln and the model's buffers for a forward of B clips of T frames with window Tw and bin chunk Fc (ws_sizes; audio: the audio
// call's), each fresh allocation zero-filled on its own stream (s: front end, sl: sub-band stage), and encode their tensor maps.
static int ensure_ws(fsn_model* m, Lane& ln, int B, int T, int Tw, int Fc, cudaStream_t s, cudaStream_t sl, bool audio = false,
                     bool lim = false) {
    const fsn_config& c = m->cfg;
    const int F = c.num_freqs, Tp = T + c.look_ahead;
    const long long srows = (long long)B * (Fc ? Fc : F) * Tp;          // sub-band TCN: the rows of one chunk run
    if (c.sb_tcn && srows > SB_MAX_ROWS)
        return fail(FSN_EINVAL, "B * %s * (T + look_ahead) = %lld rows exceeds the sub-band TCN's 2^31 limit", Fc ? "bins per chunk" : "num_freqs", srows);
    if (c.model_kind == FSN_KIND_PLUS && !m->tcn5) return fail(FSN_ESTATE, "the TCN weights were not packed");
    const WsSizes z = ws_sizes(c, m->layerwise, B, T, Tw, Fc, audio, lim);
    const WsGeo geo{B, T, Tw, Fc};
    m->au_valid = false;
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
        if (b.ensure(z.*e.need, e.flags & WS_ZERO, (e.flags & WS_SL) ? sl : s, m->env_poison)) return fail(FSN_ECUDA, "workspace allocation failed for B=%d T=%d", B, T);
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

// One window of the layer-wise sub-band recurrence, layer after layer: for l > 0 the input-projection GEMM of every row and frame of
// the window into gin (k_gemm_tc5.cu), then lstm_tc5r_kernel; layer 0 projects its input (the packed images) itself, or, with a wide
// input, through the same GEMM from a.ximg's rows of 128 halves (K = 128).  a: the window's launch (rows, ntiles, Tp, t0, Tw, ximg, hseq,
// out, la and the epilogue) with layer 0's cstate and hstate (null: none); layer l's lie cs_layer floats and hs_layer halves further.
// Returns the number of launches, or the error code.
static int sb_layers(fsn_model* m, const LstmTc5rLaunch& a, __half* gin, size_t cs_layer, size_t hs_layer, cudaStream_t s) {
    const fsn_config& c = m->cfg;
    const int H = c.sb_hidden;
    int launches = 0;
    for (int l = 0; l < c.num_layers; ++l) {
        LstmTc5rLaunch al = a;
        if (l > 0 || sb_wide(c)) {
            // row-major Gin[M, 4H] = X[M, K] * Wp[4H, K]^T, both operands K-major (K = H; a wide layer 0: 128)
            const int K = l > 0 ? H : 128;
            GemmF16Launch g{(long long)(a.ntiles + 1) / 2 * 2 * a.Tw * 128, 4 * H, K, gin, 4LL * H, m->env_gin_tile_n};
            const int ge = launch_gemm_f16(l > 0 ? static_cast<const void*>(a.hseq) : static_cast<const void*>(a.ximg), m->r_wih[l].p, g, m->num_sms, s);
            if (ge) return fail(FSN_ECUDA, "input-projection GEMM launch failed (layer %d): %s", l, cudaGetErrorString((cudaError_t)ge));
            launches++;
            al.ximg = nullptr; al.gin = gin;
        }
        al.wstream = static_cast<const __half*>(m->r_stream[l].p);
        al.bias = static_cast<const float*>(m->r_bias[l].p);
        al.fc_w = m->sb_fc_w;
        al.fc_b = m->sb_fc_b;
        al.H = H; al.F = c.num_freqs; al.act = c.sb_act; al.fast = c.fast_math; al.gru = c.rnn_type == FSN_RNN_GRU; al.last = (l == c.num_layers - 1);
        al.cstate = a.cstate + l * cs_layer;
        if (a.hstate) al.hstate = a.hstate + l * hs_layer;
        const int e = launch_lstm_tc5r(al, s);
        if (e) return fail(FSN_ECUDA, "layer-wise LSTM launch failed (layer %d): %s", l, cudaGetErrorString((cudaError_t)e));
        launches++;
    }
    return launches;
}

// The sub-band LSTM / GRU's input images of the frames sp names (a wide input: plain rows of 128 halves, time-major for the generic
// kernel): the whole clip's, a window's, or the test hook's raw input
static int pack_images(fsn_model* m, const SbPackLaunch& sp, cudaStream_t s) {
    cudaError_t e = cudaSuccess;
    const char* k = sb_wide(m->cfg) ? launch_sb_pack_wide(sp, !m->layerwise, s, &e) : launch_sb_pack(sp, s, &e);
    if (k) return fail(FSN_ECUDA, "%s launch failed: %s", k, cudaGetErrorString(e));
    m->launches++;
    return FSN_OK;
}

// b.enh != null: write the enhanced spectrum (decompress_cIRM x noisy) instead of the mask -- fused into the epilogue of the
// layer-wise kernel's last layer, a separate pass over a scratch mask for the generic kernel
// Tw > 0: the sub-band stage runs in time windows of Tw frames (the last one shorter); for each window the images are packed (`sp`, the
// front end's packer arguments) and every layer resumes from the h / c its previous window left (DESIGN.md §3.7).  Tw = 0: the images of
// the whole clip are already packed and every layer runs once over all frames.
static int run_sb_lstm(fsn_model* m, Lane& ln, const Batch& b, int Tw, SbPackLaunch sp, const int* tlen, cudaStream_t s) {
    const fsn_config& c = m->cfg;
    const int B = b.B, T = b.T, F = c.num_freqs, Tp = T + c.look_ahead, rows = B * F, ntiles = (rows + 127) / 128;
    const int impl = pick_impl(m);
    m->last_impl = impl;
    if (m->layerwise) {
        // one recurrent launch per layer; the first one also projects its input (the packed images), each deeper one is preceded by
        // one GEMM: the input projection of every row and time step of the window (sb_layers)
        const size_t cs_layer = lstm_tc5r_cstate_bytes(ntiles, c.sb_hidden) / sizeof(float);
        const size_t hs_layer = (size_t)(ntiles + 1) / 2 * 2 * 128 * c.sb_hidden;
        for (int w0 = 0; w0 < Tp; w0 += (Tw ? Tw : Tp)) {
            const int tw = Tw ? (Tp - w0 < Tw ? Tp - w0 : Tw) : Tp;
            if (Tw) {
                sp.t0 = w0; sp.Tw = tw;
                if (int rc = pack_images(m, sp, s)) return rc;
            }
            LstmTc5rLaunch a{};
            a.rows = rows; a.Tp = Tp; a.ntiles = ntiles; a.t0 = w0; a.Tw = tw;
            a.ximg = static_cast<const __half*>(ln.ximg.p);
            a.hseq = static_cast<__half*>(m->r_hseq.p);
            a.cstate = static_cast<float*>(m->cstate.p);
            if (Tw) a.hstate = static_cast<__half*>(m->r_hstate.p);
            a.out = b.mask; a.la = c.look_ahead;
            a.nreal = b.real; a.nimag = b.imag; a.enh = reinterpret_cast<float2*>(b.enh); a.tlen = tlen; a.lam = b.dlam;
            const int nl = sb_layers(m, a, static_cast<__half*>(m->r_gin.p), Tw ? cs_layer : 0, hs_layer, s);
            if (nl < 0) return nl;
            m->launches += nl;
        }
    } else if (Tw) {
        return fail(FSN_EINVAL, "time windows of the sub-band stage need the layer-wise LSTM path");
    } else if (impl == FSN_LSTM_TCGEN05) {
        return fail(FSN_EINVAL, "the tensor-core LSTM needs hidden %% 64 == 0 and <= 512, input <= 128, output_size 2");
    } else {
        LstmMmaLaunch a = m->sb_mma;
        a.rows = rows; a.Tp = Tp;
        if (sb_wide(c)) { a.xplain = static_cast<const __half*>(ln.ximg.p); a.rows_pad = ntiles * 128; }   // time-major rows of 128 halves
        else a.img = static_cast<const __half*>(ln.ximg.p);
        a.ntiles = ntiles;
        a.cstate = static_cast<float*>(m->cstate.p);
        lstm_mma_cstate_bytes(c.num_layers, rows, c.sb_hidden, &a.rows_alloc);
        a.out = b.mask; a.la = c.look_ahead; a.tlen = tlen;
        if (b.enh) {                                                    // generic kernel: mask into a scratch buffer, then one fused post-processing pass
            if (m->mask_tmp.ensure((size_t)B * 2 * F * T * 4, false, s, m->env_poison)) return fail(FSN_ECUDA, "allocation failed");
            a.out = static_cast<float*>(m->mask_tmp.p);
        }
        int e = launch_lstm_mma(a, s);
        if (e) return fail(FSN_ECUDA, "mma LSTM launch failed: %s", cudaGetErrorString((cudaError_t)e));
        if (b.enh) { launch_apply_cirm_planar(a.out, b.real, b.imag, reinterpret_cast<float2*>(b.enh), B, F, T, tlen, c.look_ahead, s, b.dlam); m->launches++; }
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
        const TcnWeights::Block* p = w.p[blk];
        GemmTc5Launch g1{};
        set_tcn_rows(g1, w, G, Tp);
        g1.epi = EPI5_PRELU_STATS; g1.Kp = w.Cp; g1.NT = 128; g1.ntiles_n = 4; g1.Npad = 512;
        for (int b = 0; b < w.nbr; ++b) { g1.bias[b] = p[b].conv1x1_b; g1.prelu[b] = p[b].prelu1; }
        g1.stats_out = st1; g1.Y16 = static_cast<__half*>(sc.y1.p); g1.ldY = 512; g1.amax_in = amax_in; g1.tlen = tlen; g1.zdiv = zdiv;
        int e = launch_gemm_tc5(curmap, w.mapW1[blk], g1, m->num_sms, s);
        if (e) return fail(FSN_ECUDA, "%s GEMM1 launch failed: %s", w.name, cudaGetErrorString((cudaError_t)e));
        m->launches++;

        DwTmLaunch dw{};
        dw.X = static_cast<const __half*>(sc.y1.p); dw.Y = static_cast<__half*>(sc.y2.p);
        dw.Z = (int)Z; dw.B = G; dw.C = 512; dw.Tp = Tp; dw.dilation = dil[blk]; dw.causal = causal ? 1 : 0;
        dw.stats_in = st1; dw.stats_out = st2; dw.amax = amax_in; dw.tlen = tlen; dw.zdiv = zdiv;
        for (int b = 0; b < w.nbr; ++b) {
            dw.gamma[b] = p[b].norm1_w; dw.beta[b] = p[b].norm1_b; dw.w[b] = p[b].dw_w; dw.b[b] = p[b].dw_b; dw.prelu[b] = p[b].prelu2;
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
static int run_sb_tcn(fsn_model* m, Lane& ln, const Batch& b, int Fc, SbPackLaunch sp, const int* tlen, cudaStream_t s) {
    const fsn_config& c = m->cfg;
    const int B = b.B, F = c.num_freqs, Tp = b.T + c.look_ahead, W = Fc ? Fc : F;
    m->last_impl = FSN_LSTM_TCN;
    GemmTc5Launch head{};
    head.epi = b.dlam ? EPI5_GLN_HEAD_LIM : EPI5_GLN_HEAD;
    head.fc_w = static_cast<const float*>(m->sb_fc.p); head.fc_b = m->sb_fc_b;
    head.O = c.output_size; head.la = c.look_ahead; head.F = F; head.act = c.sb_act;
    head.out = b.mask; head.nreal = b.real; head.nimag = b.imag; head.enh = reinterpret_cast<float2*>(b.enh); head.lam = b.dlam;
    float* x = static_cast<float*>(ln.sbx.p);
    float* amax0 = x + (size_t)B * W * Tp * 64;
    for (int f0 = 0; f0 < F; f0 += W) {
        const int fc = F - f0 < W ? F - f0 : W, Z = B * fc;
        if (Fc) {
            sp.xtm = x; sp.amax = amax0; sp.f0 = f0; sp.Fc = fc;
            cudaError_t e = cudaSuccess;
            if (const char* k = launch_sb_pack_tm(sp, s, &e)) return fail(FSN_ECUDA, "%s launch failed: %s", k, cudaGetErrorString(e));
            m->launches++;
        }
        CK(cudaMemsetAsync(m->sb_scratch.stats.p, 0, tcn_stats_bytes(Z), s));
        head.Fg = fc; head.f0 = f0;
        int rc = run_tcn_blocks(m, m->tcn_sb, m->sb_scratch, x, ln.mapSbx, amax0, Z, Tp, false, head, tlen, fc, s);
        if (rc) return rc;
    }
    return FSN_OK;
}

// The state of the full-band LSTM of fullsubnet.Model (run_fb), as LstmWsLaunch / LstmMmaLaunch name it; cbuf and hstate are null in
// the offline forward, which keeps no state.  slot, kf: the streaming slot calls' per-slot counts and frame counts, or null.
struct FbState {
    __half* hbuf; float* cbuf; unsigned int* barrier;  // weight-stationary kernel
    float* cstate; int rows_alloc; __half* hstate;     // generic kernel
    int resume, t0;
    const int *slot, *kf;
};

// The full band of fullsubnet.Model over `rows` clips (or slots) of Tp frames at row pitch P: fb_pack of fbin [rows, F, P] into fbx
// [Tp, rows_pad, Ipad], the LSTM into hseq [rows, H, P] (the weight-stationary kernel if use_ws, else the generic one), then the output
// Linear into fbout [rows, F, P].  Returns the number of launches, or minus the LSTM's launch error (each caller words its report).
static int run_fb(fsn_model* m, const float* fbin, __half* fbx, float* hseq, float* fbout, int rows, int rows_pad, int Tp, int P,
                  bool use_ws, const FbState& fs, cudaStream_t s) {
    launch_fb_pack(fbin, fbx, rows, m->cfg.num_freqs, Tp, P, rows_pad, m->fb_mma.Ipad, s);
    LstmWsLaunch w = m->fb_ws;
    LstmMmaLaunch a = m->fb_mma;
    w.rows = rows; w.rows_pad = rows_pad; w.Tp = Tp; w.x = fbx; w.hseq = hseq; w.P = P;
    w.hbuf = fs.hbuf; w.cbuf = fs.cbuf; w.barrier = fs.barrier; w.resume = fs.resume; w.t0 = fs.t0; w.slot = fs.slot; w.kf = fs.kf;
    a.rows = rows; a.rows_pad = rows_pad; a.Tp = Tp; a.xplain = fbx; a.hseq = hseq; a.P = P;
    a.cstate = fs.cstate; a.rows_alloc = fs.rows_alloc; a.hstate = fs.hstate; a.resume = fs.resume; a.slot = fs.slot; a.kf = fs.kf;
    a.slot_rows = fs.hstate ? 1 : 0;                                    // streaming: row r is slot r
    if (int e = use_ws ? launch_lstm_ws(w, s) : launch_lstm_mma(a, s)) return -e;
    ConvLaunch cf = m->fb_out;
    cf.X = hseq; cf.Y = fbout; cf.Z = rows; cf.Tp = Tp; cf.P = P;
    launch_conv1x1(cf, s);
    return 3;
}

// Copy the per-sample extents frames[b] + look_ahead of a ragged forward into the lane's device buffer ln.tlen ([3][B]: one row per
// full-band branch, so a full-band gLN group z = branch * B + b indexes it directly) through the model's pinned staging.  h_samples:
// the audio call's sample counts, appended as a fourth row in the same copy, or null.  h_frames may be null when h_samples is not
// (clips of one frame count but different sample counts): the three rows are then zero and unread.  h_lam: the clips' attenuation
// floors (float), appended as the last row of the same copy, or null; *d_lam: that row on the device.
static int stage_lengths(fsn_model* m, Lane& ln, const int32_t* h_frames, int B, cudaStream_t s, const int32_t* h_samples = nullptr,
                         const float* h_lam = nullptr, const float** d_lam = nullptr) {
    const size_t rows = 3 + (h_samples ? 1 : 0), n = (rows + (h_lam ? 1 : 0)) * B;
    int32_t* h = nullptr;
    if (int rc = m->len_stage.take(n, &h)) return rc;
    for (int br = 0; br < 3; ++br)
        for (int b = 0; b < B; ++b) h[(size_t)br * B + b] = h_frames ? h_frames[b] + m->cfg.look_ahead : 0;
    if (h_samples) memcpy(h + (size_t)3 * B, h_samples, (size_t)B * sizeof(int32_t));
    if (h_lam) memcpy(h + rows * B, h_lam, (size_t)B * sizeof(float));
    if (ln.tlen.ensure(n * sizeof(int32_t), false, s, m->env_poison)) return fail(FSN_ECUDA, "workspace allocation failed for the clip lengths");
    if (h_lam) *d_lam = reinterpret_cast<const float*>(static_cast<const int32_t*>(ln.tlen.p) + rows * B);
    return m->len_stage.send(ln.tlen.p, n, s);
}

// Set lane ln up for checked batch b (every forward and the test hook): this thread's chained (programmatic dependent) launches, see
// env_pdl -- "small" = at most 16 row-tile pairs, where the forward is launch-latency-bound; the workspace for window Tw and bin
// chunk Fc (ensure_ws); the clips' lengths on the device, *tl (null on entry): their frame extents, unless every clip spans T', and with
// them the clips' attenuation floors, *dlam (null on entry; stays null without b.lam).  Resets the launch count.
static int prepare(fsn_model* m, Lane& ln, const Batch& b, int Tw, int Fc, cudaStream_t s, cudaStream_t sl, const int** tl,
                   const float** dlam = nullptr) {
    fsn_chain_launch_set(m->env_pdl == 1 || (m->env_pdl < 0 && ((long long)b.B * m->cfg.num_freqs + 255) / 256 <= 16));
    if (int rc = ensure_ws(m, ln, b.B, b.T, Tw, Fc, s, sl, b.wave != nullptr, b.lam != nullptr)) return rc;
    if (b.frames || b.samples || b.lam) {
        if (int rc = stage_lengths(m, ln, b.frames, b.B, s, b.samples, b.lam, dlam)) return rc;
        if (b.frames) *tl = static_cast<const int*>(ln.tlen.p);
    }
    m->launches = 0;
    m->last_lane = (int)(&ln - m->lane);
    return FSN_OK;
}

// Audio analysis: the STFT of every clip of b into the audio workspace, whose planes then are b's inputs and whose enhanced spectrum
// its output.  al: the launch, kept for the synthesis after the sub-band stage.
static int audio_analysis(fsn_model* m, Lane& ln, Batch& b, AudioLaunch& al, cudaStream_t s) {
    const int F = m->cfg.num_freqs, N = 2 * (F - 1);
    const AudioTables tab = audio_table_ptrs(static_cast<const float*>(m->au_tab.p), N);
    al.wave = b.wave; al.out = b.wave_out; al.L = b.L;
    al.len = b.samples ? static_cast<const int*>(ln.tlen.p) + 3 * b.B : nullptr; al.Lall = b.Lall;
    al.B = b.B; al.T = b.T; al.n_fft = N;
    al.planes = static_cast<float*>(m->au_planes.p); al.enh = static_cast<const float2*>(m->au_enh.p);
    al.window = tab.window; al.twiddle = tab.twiddle; al.inv_env = tab.inv_env; al.inv_last = tab.inv_last;
    if (cudaError_t e = launch_audio_stft(al, s)) return fail(FSN_ECUDA, "audio_stft_kernel launch failed: %s", cudaGetErrorString(e));
    m->launches++;
    const size_t plane = (size_t)b.B * F * b.T;
    b.mag = al.planes; b.real = al.planes + plane; b.imag = al.planes + 2 * plane;
    b.mask = nullptr; b.enh = static_cast<float*>(m->au_enh.p);
    return FSN_OK;
}

// The sub-band packer's arguments for a batch of B clips of T frames in lane ln, window Tw, extents tl; the front end adds its sources,
// the test hook its raw input (SbPackLaunch::raw)
static SbPackLaunch pack_args(const fsn_model* m, Lane& ln, int B, int T, int Tw, const int* tl) {
    const fsn_config& c = m->cfg;
    SbPackLaunch sp{};
    sp.B = B; sp.F = c.num_freqs; sp.Tp = T + c.look_ahead; sp.Ns = c.sb_num_neighbors; sp.Nf = c.fb_num_neighbors; sp.P = (sp.Tp + 3) & ~3;
    sp.nfb = c.model_kind == FSN_KIND_PLUS ? 3 : 1;
    sp.mu = static_cast<float*>(ln.mu.p); sp.sigma = static_cast<float*>(ln.sigma.p); sp.rowsum = static_cast<float*>(ln.sb_rowsum.p);
    sp.norm_type = c.norm_type;
    sp.ximg = static_cast<__half*>(ln.ximg.p);
    sp.ntiles = (B * sp.F + 127) / 128;
    sp.t0 = 0; sp.Tw = sp.Tp;
    sp.cum = Tw ? static_cast<double*>(m->sb_cum.p) : nullptr;
    sp.tlen = tl;
    sp.f0 = 0; sp.Fc = sp.F;
    return sp;
}

// The front end on stream s into lane ln: the input norm of every branch (3 in FullSubNet+, 1 in fullsubnet.Model), FullSubNet+'s
// channel attention, the full-band model and the sub-band statistics; adds the full-band outputs to the packer's arguments sp
static int front_end(fsn_model* m, Lane& ln, const Batch& bt, const int* tl, SbPackLaunch& sp, cudaStream_t s) {
    const fsn_config& c = m->cfg;
    const int B = bt.B, T = bt.T, F = c.num_freqs, Tp = T + c.look_ahead, Pp = sp.P;
    const bool plus = c.model_kind == FSN_KIND_PLUS;
    const int nbr = plus ? 3 : 1;
    TsseLaunch ta{{bt.mag, plus ? bt.real : nullptr, plus ? bt.imag : nullptr}};
    ta.nbranch = nbr; ta.B = B; ta.F = F; ta.T = T; ta.Tp = Tp; ta.P = Pp;
    ta.out = static_cast<float*>(ln.fbin.p);
    ta.scale = static_cast<float*>(ln.tsse_scale.p);
    ta.rows = ta.scale + (size_t)nbr * B * F;
    ta.tlen = tl;
    if (c.norm_type != FSN_NORM_OFFLINE_LAPLACE) {
        const NormLaunch na{{ta.x[0], ta.x[1], ta.x[2]}, static_cast<float*>(ln.xn.p), nbr, B, F, T, Tp, c.norm_type, tl,
                            static_cast<float*>(ln.fbout.p)};            // scratch: the full-band outputs are written later
        if (cudaError_t e = launch_input_norm(na, s)) return fail(FSN_ECUDA, "input_norm_kernel launch failed: %s", cudaGetErrorString(e));
        m->launches++;
        for (int b = 0; b < nbr; ++b) ta.x[b] = static_cast<const float*>(ln.xn.p) + (size_t)b * B * F * Tp;
        ta.T = Tp; ta.prenorm = 1;                                      // padded frames are part of the normalised signal
    }
    if (plus) {
        ta.attention = 1 + c.channel_attention; ta.sub = c.subband_num;
        for (int i = 0; i < 3; ++i) ta.ksz[i] = c.kersize[i];
        for (int b = 0; b < 3; ++b) ta.p[b] = m->tsse[b];
        ta.out_tm = static_cast<float*>(ln.x0.p); ta.Cp = m->tcn_fb.Cp;
        m->last_fb_ws = 0;
        CK(cudaMemsetAsync(ln.tcn.stats.p, 0, tcn_stats_bytes(3 * B), s));
        ta.amax = tcn_amax(ln.tcn.stats.p, 3 * B, 0);                  // block 0: written by the gate kernel
    }
    cudaError_t e = cudaSuccess;
    if (const char* k = launch_tsse_norm(ta, s, &e)) return fail(FSN_ECUDA, "%s launch failed: %s", k, cudaGetErrorString(e));
    m->launches += 3;

    if (plus) {
        const TcnWeights& w = m->tcn_fb;
        GemmTc5Launch last{};                                           // the last block also writes relu(x) for the output Linear
        last.epi = EPI5_GLN_RES; last.Xrelu = static_cast<float*>(ln.xr.p);
        int rc = run_tcn_blocks(m, w, ln.tcn, static_cast<const float*>(ln.x0.p), ln.mapX0, ta.amax, B, Tp, c.tcn_causal, last, tl, 1, s);
        if (rc) return rc;
        GemmTc5Launch g3{};
        set_tcn_rows(g3, w, B, Tp);
        g3.epi = EPI5_OUT; g3.Kp = w.Cp; g3.NT = w.NT; g3.ntiles_n = w.ntiles; g3.Npad = w.Cp;
        for (int b = 0; b < 3; ++b) g3.bias[b] = static_cast<const float*>(m->fb_fc_b.p) + (size_t)b * w.Cp;
        g3.out = static_cast<float*>(ln.fbout.p); g3.F = F; g3.P = Pp; g3.act = c.fb_act;    // finite past each clip's end; the sub-band stages mask it
        const int eo = launch_gemm_tc5(ln.mapXr, m->map_fb_fc, g3, m->num_sms, s);
        if (eo) return fail(FSN_ECUDA, "TCN output GEMM launch failed: %s", cudaGetErrorString((cudaError_t)eo));
        m->launches++;

        sp.win = static_cast<const float*>(ln.fbin.p); sp.Pw = Pp;      // post-attention mag branch (fullsubnet_plus.py:182)
        for (int b = 0; b < 3; ++b) sp.fb[b] = static_cast<const float*>(ln.fbout.p) + (size_t)b * B * F * Pp;
    } else {
        launch_pad_copy(bt.mag, static_cast<float*>(ln.magpad.p), B, F, T, Pp, tl, c.look_ahead, s); m->launches++;
        // the full-band LSTM is causal, and its input (fb_in) is already zero past each clip's end: its outputs there are masked by the
        // sub-band stages
        m->last_fb_ws = lstm_ws_supported(c.num_layers, c.fb_hidden, m->fb_ws.Ipad, B, m->num_sms) && !m->env_no_ws;
        if (m->last_fb_ws) {
            const size_t hb = (size_t)c.num_layers * 2 * 64 * c.fb_hidden * 2;
            if (m->ws_h.ensure(hb, false, s) || m->ws_bar.ensure(64, true, s)) return fail(FSN_ECUDA, "allocation failed");
            CK(cudaMemsetAsync(m->ws_h.p, 0, hb, s));
        }
        FbState fs{static_cast<__half*>(m->ws_h.p), nullptr, static_cast<unsigned int*>(m->ws_bar.p), static_cast<float*>(m->cstate.p)};
        lstm_mma_cstate_bytes(c.num_layers, B, c.fb_hidden, &fs.rows_alloc);
        const int nl = run_fb(m, static_cast<const float*>(ln.fbin.p), static_cast<__half*>(ln.fbx.p), static_cast<float*>(ln.hseq.p),
                              static_cast<float*>(ln.fbout.p), B, (B + 63) / 64 * 64, Tp, Pp, m->last_fb_ws, fs, s);
        if (nl < 0)
            return fail(FSN_ECUDA, "%sfull-band LSTM launch failed: %s", m->last_fb_ws ? "weight-stationary " : "", cudaGetErrorString((cudaError_t)-nl));
        m->launches += nl;

        sp.win = static_cast<const float*>(ln.magpad.p); sp.Pw = Pp;    // raw padded magnitude (fullsubnet.py:94)
        sp.fb[0] = static_cast<const float*>(ln.fbout.p);
    }
    if (const char* k = launch_sb_stats(sp, s, &e)) return fail(FSN_ECUDA, "%s launch failed: %s", k, cudaGetErrorString(e));
    m->launches += 2;
    return FSN_OK;
}

// The whole clip's sub-band input on stream s, unless the sub-band stage packs it itself: window by window (Tw, run_sb_lstm) or chunk
// by chunk (Fc, run_sb_tcn)
static int pack_clip(fsn_model* m, Lane& ln, SbPackLaunch sp, int Tw, int Fc, cudaStream_t s) {
    if (m->cfg.sb_tcn) {
        if (Fc) return FSN_OK;
        sp.xtm = static_cast<float*>(ln.sbx.p);
        sp.amax = sp.xtm + (size_t)sp.B * sp.F * sp.Tp * 64;
        cudaError_t e = cudaSuccess;
        if (const char* k = launch_sb_pack_tm(sp, s, &e)) return fail(FSN_ECUDA, "%s launch failed: %s", k, cudaGetErrorString(e));
        m->launches++;
    } else if (!Tw) {
        return pack_images(m, sp, s);
    }
    return FSN_OK;
}

// The sub-band stage on stream sl: the LSTM / GRU or the TCN over the packed input (sp: the packer's arguments, for windows and chunks)
static int sub_band(fsn_model* m, Lane& ln, const Batch& b, int Tw, int Fc, const SbPackLaunch& sp, const int* tl, cudaStream_t sl) {
    return m->cfg.sb_tcn ? run_sb_tcn(m, ln, b, Fc, sp, tl, sl) : run_sb_lstm(m, ln, b, Tw, sp, tl, sl);
}

// The forward of checked batch b in lane ln, its stages in order: audio analysis (the audio call), the front end and the whole clip's
// sub-band packing on stream `s`, the sub-band stage and audio synthesis on stream `sl` (== s for the plain driver; the pipeline passes
// the LSTM stream, ordered after the front end by the lane's ev_front).
// Tw: time window of the sub-band stage (0: the whole clip; > 0 needs s == sl, the plain driver)
// Fc: bin chunk of the sub-band TCN (0: all bins at once; > 0 needs s == sl, the plain driver)
static int forward_impl(fsn_model* m, Lane& ln, const Batch& in, cudaStream_t s, cudaStream_t sl, int Tw = 0, int Fc = 0) {
    const int* tl = nullptr;                                            // per-sample extents on the device (null: all Tp)
    const float* dlam = nullptr;                                        // attenuation floors on the device (null: no limit)
    int rc = prepare(m, ln, in, Tw, Fc, s, sl, &tl, &dlam);
    if (rc) return rc;
    const int evi = (int)(m->nfwd % fsn_model::NEV);
    cudaEventRecord(m->evf0[evi], s);
    Batch b = in;
    b.dlam = dlam;
    AudioLaunch al{};
    if (in.wave && (rc = audio_analysis(m, ln, b, al, s))) return rc;
    SbPackLaunch sp = pack_args(m, ln, b.B, b.T, Tw, tl);
    if ((rc = front_end(m, ln, b, tl, sp, s)) || (rc = pack_clip(m, ln, sp, Tw, Fc, s))) return rc;
    cudaEventRecord(m->evf1[evi], s);
    if (sl != s) {                                                      // pipelined: the LSTM stream picks the lane up when the front end is done
        CK(cudaEventRecord(ln.ev_front, s));
        CK(cudaStreamWaitEvent(sl, ln.ev_front, 0));
    }
    cudaEventRecord(m->ev0[evi], sl);
    rc = sub_band(m, ln, b, Tw, Fc, sp, tl, sl);
    cudaEventRecord(m->ev1[evi], sl);
    if (rc) return rc;
    if (in.wave) {                                                      // the iSTFT of every clip over its own frames
        if (cudaError_t e = launch_audio_istft(al, sl)) return fail(FSN_ECUDA, "audio_istft_kernel launch failed: %s", cudaGetErrorString(e));
        m->launches++;
    }
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

// one checked pipelined batch (after ensure_pipeline): inputs are ready once `ready` (an event, may be null) has fired; returns the lane used
static int submit_impl(fsn_model* m, cudaEvent_t ready, const Batch& b, int* lane_out) {
    // overlap needs the opt-in (see env_front_overlap) and FullSubNet+ (fullsubnet.Model's full-band LSTM is a cooperative launch and
    // shares the LSTM scratch): otherwise one lane, one stream -- the pipeline still overlaps copies and the caller's post-processing
    const bool overlap = m->env_front_overlap && (m->cfg.model_kind == FSN_KIND_PLUS);
    const int slot = overlap ? (int)(m->nsub & 1) : 0;
    Lane& ln = m->lane[slot];
    cudaStream_t sf = overlap ? m->s_front : m->s_lstm;
    if (ready) CK(cudaStreamWaitEvent(sf, ready, 0));
    if (m->plain_pending) { CK(cudaStreamWaitEvent(sf, m->ev_plain, 0)); CK(cudaStreamWaitEvent(m->s_lstm, m->ev_plain, 0)); }
    if (ln.used) CK(cudaStreamWaitEvent(sf, ln.ev_lstm, 0));              // the LSTM that read this lane has finished
    if (int rc = forward_impl(m, ln, b, sf, m->s_lstm)) return rc;
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
static double ws_bytes_per_sample(const fsn_config& c, bool layerwise, int T, bool audio) {
    const double F = c.num_freqs, Tp = T + c.look_ahead, rows = F;              // sequences per sample
    double b = audio ? 20 * F * T : 0;                                           // the audio call's planes and enhanced spectrum
    if (c.model_kind == FSN_KIND_PLUS) b += 3 * F * Tp * 4 * 2 + 3 * Tp * (4.0 * ((c.num_freqs + 31) / 32 * 32) + 512) * 4;   // fb_in/out, X0/Xa/Xb/Xr (fp32), Y1/Y2 (fp16)
    else b += F * Tp * 4 * 4 + Tp * (F + c.fb_hidden) * 4;
    if (c.sb_tcn) {                                                             // input + two fp32 streams of 64 channels, two fp16 hidden
        b += rows * Tp * (3 * 64 * 4 + 2 * 512 * 2) + rows * (tcn_stats_bytes(1) + 4);   // buffers of 512; statistics, the input's max |x|
        return b;
    }
    b += rows * Tp * sb_row_bytes(c);                                           // packed sub-band images (when used)
    b += rows * c.num_layers * c.sb_hidden * 4;                                  // cell state
    if (layerwise && c.num_layers > 1) b += rows * Tp * (4.0 * c.sb_hidden + c.sb_hidden) * 2;   // Gin + layer output sequence
    else if (layerwise && sb_wide(c)) b += rows * Tp * 4.0 * c.sb_hidden * 2;     // a wide layer 0's Gin
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
// (>= F: unchunked) and the largest equal split that fits with them.  audio: the audio call's plan, its workspace counted (ws_sizes).
static Plan plan_forward(const fsn_config& c, bool layerwise, int B, int T, double cap, int force, int force_bins, bool audio = false,
                         bool lim = false) {
    const int Tp = T + c.look_ahead, wmax = (Tp + 31) / 32 * 32;
    // sub-batches never exceed the full-band TCN's row limit or the launch grids
    const long long blim = std::min(max_clips_for_rows(c, T), max_clips_for_grid(c));
    auto split = [&](int bmax) { if (bmax > blim) bmax = (int)blim; if (bmax < 1) bmax = 1; if (B <= bmax) return B; const int n = (B + bmax - 1) / bmax; return (B + n - 1) / n; };
    auto bytes = [&](int bs, int tw) { return (double)ws_sizes(c, layerwise, bs, T, tw, 0, audio, lim).total(); };
    // largest equal split bs with fits(bs) (0 if even one clip does not fit)
    auto max_split = [&](auto fits) { const int b = largest(0, B, [&](int v) { return fits(split(v)); }); return b ? split(b) : 0; };
    const double per = ws_bytes_per_sample(c, layerwise, T, audio);
    const double bmax = cap / (per > 1 ? per : 1);
    Plan p{split(bmax < B ? (int)bmax : B)};
    if (c.sb_tcn) {
        const int F = c.num_freqs;
        auto fits = [&](int bs, int fc) { return (long long)bs * fc * Tp <= SB_MAX_ROWS && ws_sizes(c, false, bs, T, 0, fc < F ? fc : 0, audio, lim).total() <= cap; };
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
    p.bytes = (int64_t)ws_sizes(c, layerwise, p.Bs, T, p.Tw, p.Fc, audio, lim).total();
    return p;
}

// Make stream s wait for the pipelined batches still in flight: they share the scratch buffers
static int wait_lanes(fsn_model* m, cudaStream_t s) {
    for (auto& ln : m->lane)
        if (ln.used) CK(cudaStreamWaitEvent(s, ln.ev_lstm, 0));
    return FSN_OK;
}

// A plain call (forward, audio, test hooks) on stream s runs after the pipelined batches and after the last plain call, on whichever
// stream that ran: they all use lane 0's workspace.  mark_plain records the call's end for the next one.
static int wait_plain(fsn_model* m, cudaStream_t s) {
    if (m->plain_pending) CK(cudaStreamWaitEvent(s, m->ev_plain, 0));
    return wait_lanes(m, s);
}
static int mark_plain(fsn_model* m, cudaStream_t s) {
    if (!m->ev_plain) CK(cudaEventCreateWithFlags(&m->ev_plain, cudaEventDisableTiming));
    CK(cudaEventRecord(m->ev_plain, s));
    m->plain_pending = true;
    return FSN_OK;
}

// Clips b0 .. b0 + nb - 1 of batch b (fewer at its end): every pointer advanced by its per-clip stride
static Batch slice(const fsn_config& c, const Batch& b, int b0, int nb) {
    const size_t plane = (size_t)c.num_freqs * b.T;
    auto at = [b0](auto* p, size_t stride) { return p ? p + b0 * stride : p; };
    Batch s = b;
    s.B = b.B - b0 < nb ? b.B - b0 : nb;
    s.mag = at(b.mag, plane); s.real = at(b.real, plane); s.imag = at(b.imag, plane); s.frames = at(b.frames, 1);
    s.mask = at(b.mask, c.output_size * plane); s.enh = at(b.enh, 2 * plane);
    s.wave = at(b.wave, b.L); s.wave_out = at(b.wave_out, b.L); s.samples = at(b.samples, 1); s.lam = at(b.lam, 1);
    return s;
}

// The plain forward of checked batch b on stream s, after the pipelined batches in flight.  Samples are independent, so a batch whose
// workspace would exceed the cap (FSN_WS_CAP_GB, default 24 of the 80 GB) is run as equal sub-batches one after the other on the same
// stream -- same results, bounded memory (e.g. 256 clips on the layer-wise path); a clip too long for the cap runs its sub-band stage
// in time windows (plan_forward) -- same bits, O(window) sub-band memory -- or, with the sub-band TCN, in bin chunks -- O(chunk)
// sub-band memory.
static int run_plain(fsn_model* m, const Batch& b, cudaStream_t s) {
    int rc = wait_plain(m, s);
    if (rc) return rc;
    const bool audio = b.call == CALL_AUDIO;
    m->plan = plan_forward(m->cfg, m->layerwise, b.B, b.T, m->ws_cap_bytes, m->env_sb_window, m->env_sb_chunk, audio, b.lam != nullptr);
    const int Bs = m->plan.Bs;
    int64_t launches = 0;
    for (int b0 = 0; b0 < b.B && rc == FSN_OK; b0 += Bs) {
        rc = forward_impl(m, m->lane[0], slice(m->cfg, b, b0, Bs), s, s, m->plan.Tw, m->plan.Fc);
        launches += m->launches;
    }
    m->launches = launches;
    const int rr = mark_plain(m, s);                                    // also behind a sub-batch that failed part-way
    if (rc) return rc;
    m->au_valid = audio && Bs >= b.B;
    return rr;
}

// A device-buffer spectral call: check batch b, then run it plain or pipelined
static int run_spectra(fsn_model* m, Batch b, void* stream) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    std::vector<float> lam;
    if (int rc = check_batch(m, b, nullptr, &lam)) return rc;
    if (b.call == CALL_FORWARD) return run_plain(m, b, s);
    if (int rc = ensure_pipeline(m)) return rc;
    CK(cudaEventRecord(m->ev_in, s));                                   // everything enqueued on the caller's stream so far (the inputs)
    return submit_impl(m, m->ev_in, b, nullptr);
}

extern "C" int fsn_model_forward(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                 float* d_out, void* stream) {
    return run_spectra(m, Batch{CALL_FORWARD, d_mag, d_real, d_imag, B, T, nullptr, d_out}, stream);
}
extern "C" int fsn_model_forward_enhance(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                         float* d_enh, void* stream) {
    return fsn_model_forward_enhance_lim(m, d_mag, d_real, d_imag, B, T, nullptr, nullptr, d_enh, stream);
}

extern "C" int fsn_model_forward_ragged(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                        const int32_t* h_frames, float* d_out, void* stream) {
    return run_spectra(m, Batch{CALL_FORWARD, d_mag, d_real, d_imag, B, T, h_frames, d_out}, stream);
}
extern "C" int fsn_model_forward_enhance_ragged(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                                const int32_t* h_frames, float* d_enh, void* stream) {
    return fsn_model_forward_enhance_lim(m, d_mag, d_real, d_imag, B, T, h_frames, nullptr, d_enh, stream);
}
extern "C" int fsn_model_forward_enhance_lim(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                             const int32_t* h_frames, const float* h_atten_db, float* d_enh, void* stream) {
    Batch b{CALL_FORWARD, d_mag, d_real, d_imag, B, T, h_frames, nullptr, d_enh};
    b.atten_db = h_atten_db;
    return run_spectra(m, b, stream);
}

extern "C" int fsn_model_enhance_audio(fsn_model* m, const float* d_wave, int32_t B, int64_t L, const int64_t* h_lengths, float* d_out,
                                       void* stream) {
    return fsn_model_enhance_audio_lim(m, d_wave, B, L, h_lengths, nullptr, d_out, stream);
}
extern "C" int fsn_model_enhance_audio_lim(fsn_model* m, const float* d_wave, int32_t B, int64_t L, const int64_t* h_lengths,
                                           const float* h_atten_db, float* d_out, void* stream) {
    Batch b{CALL_AUDIO, nullptr, nullptr, nullptr, B, 0, nullptr, nullptr, nullptr, d_wave, d_out, L, h_lengths};
    b.atten_db = h_atten_db;
    std::vector<int32_t> lens;
    std::vector<float> lam;
    if (int rc = check_batch(m, b, &lens, &lam)) return rc;
    return run_plain(m, b, static_cast<cudaStream_t>(stream));
}

// Test hook: the sub-band stage alone on a given input, through the forward's own setup (prepare) and sub-band stage (its GEMM dispatch,
// per-layer state, windows and epilogues); only the packer's arguments differ (SbPackLaunch::raw: the input as given instead of the
// normalised unfold).  Outside the timing-event ring and the plan of the last plain forward.
extern "C" int fsn_model_sb_forward(fsn_model* m, const float* d_x, int32_t B, int32_t T, int32_t Tw, const int32_t* h_frames,
                                    float* d_out, const float* d_real, const float* d_imag, float* d_enh, void* stream) {
    Batch b{CALL_HOOK, nullptr, d_real, d_imag, B, T, h_frames, d_out, d_enh, nullptr, nullptr, 0, nullptr, 0, nullptr, d_x, Tw};
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int* tl = nullptr;
    int rc = check_batch(m, b);
    if (rc || (rc = wait_plain(m, s))) return rc;
    if (!(rc = prepare(m, m->lane[0], b, Tw, 0, s, s, &tl))) {
        Lane& ln = m->lane[0];
        SbPackLaunch sp = pack_args(m, ln, B, T, Tw, tl);
        sp.raw = d_x;
        if (!(rc = pack_clip(m, ln, sp, Tw, 0, s)) && !(rc = sub_band(m, ln, b, Tw, 0, sp, tl, s)))
            if (cudaError_t e = cudaGetLastError()) rc = fail(FSN_ECUDA, "fsn_model_sb_forward: %s", cudaGetErrorString(e));
    }
    const int rr = mark_plain(m, s);                                    // also behind a call that failed part-way
    return rc ? rc : rr;
}

extern "C" int fsn_model_submit(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                float* d_out, void* stream) {
    return run_spectra(m, Batch{CALL_PIPELINED, d_mag, d_real, d_imag, B, T, nullptr, d_out}, stream);
}
extern "C" int fsn_model_submit_enhance(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                        float* d_enh, void* stream) {
    return run_spectra(m, Batch{CALL_PIPELINED, d_mag, d_real, d_imag, B, T, nullptr, nullptr, d_enh}, stream);
}

extern "C" int fsn_model_last_lane(const fsn_model* m) { return m ? m->last_lane : 0; }

extern "C" int fsn_model_wait_lane(fsn_model* m, int32_t lane, void* stream) {
    if (!m || lane < 0 || lane > 1) return fail(FSN_EINVAL, "bad argument");
    if (m->lane[lane].used) CK(cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), m->lane[lane].ev_lstm, 0));
    return FSN_OK;
}

extern "C" int fsn_model_wait(fsn_model* m, void* stream) {
    if (!m) return fail(FSN_EINVAL, "null model");
    return wait_lanes(m, static_cast<cudaStream_t>(stream));
}

// The host-buffer calls' batch, checked before any staging: the inputs the model reads (mag; FullSubNet+: real and imag too) and the
// output [B, O, F, T] in host memory
static int host_batch(fsn_model* m, Call call, const float* const (&hin)[3], int32_t B, int32_t T, float* h_out, Batch* b) {
    if (!m || !hin[0] || !h_out) return fail(FSN_EINVAL, "null argument");
    for (int i = 1; i < (m->cfg.model_kind == FSN_KIND_PLUS ? 3 : 1); ++i)
        if (!hin[i]) return fail(FSN_EINVAL, "missing input %d", i);
    *b = Batch{call, hin[0], hin[1], hin[2], B, T, nullptr, h_out};
    return check_batch(m, *b);
}

extern "C" int fsn_model_forward_host(fsn_model* m, const float* h_mag, const float* h_real, const float* h_imag, int32_t B, int32_t T,
                                      float* h_out, void* stream) {
    const float* const hin[3] = {h_mag, h_real, h_imag};
    Batch b;
    if (int rc = host_batch(m, CALL_FORWARD, hin, B, T, h_out, &b)) return rc;
    const fsn_config& c = m->cfg;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t in_bytes = (size_t)B * c.num_freqs * T * 4, out_bytes = (size_t)B * c.output_size * c.num_freqs * T * 4;
    const int nin = (c.model_kind == FSN_KIND_PLUS) ? 3 : 1;
    for (int i = 0; i < nin; ++i) {
        if (m->stage_in[i].ensure(in_bytes, false)) return fail(FSN_ECUDA, "staging allocation failed");
        CK(cudaMemcpyAsync(m->stage_in[i].p, hin[i], in_bytes, cudaMemcpyHostToDevice, s));
    }
    if (m->stage_out.ensure(out_bytes, false)) return fail(FSN_ECUDA, "staging allocation failed");
    b.mag = static_cast<const float*>(m->stage_in[0].p); b.real = static_cast<const float*>(m->stage_in[1].p);
    b.imag = static_cast<const float*>(m->stage_in[2].p); b.mask = static_cast<float*>(m->stage_out.p);
    if (int rc = run_plain(m, b, s)) return rc;
    CK(cudaMemcpyAsync(h_out, m->stage_out.p, out_bytes, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return FSN_OK;
}

extern "C" int fsn_model_forward_host_async(fsn_model* m, const float* h_mag, const float* h_real, const float* h_imag, int32_t B, int32_t T,
                                            float* h_out, void* stream) {
    (void)stream;                                                        // host buffers carry no stream order; the work runs on internal streams
    const float* const hin[3] = {h_mag, h_real, h_imag};
    Batch b;
    if (int rc = host_batch(m, CALL_PIPELINED, hin, B, T, h_out, &b)) return rc;
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
    const int nin = (c.model_kind == FSN_KIND_PLUS) ? 3 : 1;
    // the forward that read this input slot (front end: mag / real / imag; fused epilogue: real / imag) has finished
    if (m->d2h_used[slot]) CK(cudaStreamWaitEvent(m->s_in, m->ev_done[slot], 0));
    for (int i = 0; i < nin; ++i) {
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
    b.mag = static_cast<const float*>(m->a_in[slot][0].p); b.real = static_cast<const float*>(m->a_in[slot][1].p);
    b.imag = static_cast<const float*>(m->a_in[slot][2].p); b.mask = static_cast<float*>(m->a_out[slot].p);
    if ((rc = submit_impl(m, m->ev_h2d[slot], b, nullptr))) return rc;
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

static int get_stage(fsn_model* m, const char* name, float* d_dst, int64_t numel, cudaStream_t s) {
    Lane& ln = m->lane[m->last_lane];
    const fsn_config& c = m->cfg;
    const int F = c.num_freqs, Tp = ln.geo.T + c.look_ahead, Pp = (Tp + 3) & ~3, B = ln.geo.B;
    const int nbr = (c.model_kind == FSN_KIND_PLUS) ? 3 : 1;
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
    if (n == "sb_img") {
        if (c.sb_tcn) return fail(FSN_EINVAL, "sb_img is the LSTM / GRU's input: the sub-band TCN keeps sb_in instead");
        if (ln.geo.Tw) return fail(FSN_ESTATE, "sb_img is not kept: the last forward packed the images in windows (%d frames each), its buffer holds the last window only", ln.geo.Tw);
        const size_t bytes = ws_sizes(c, m->layerwise, B, ln.geo.T, 0).ximg;
        if (numel * 4 != (int64_t)bytes) return fail(FSN_EINVAL, "sb_img needs %lld elements", (long long)(bytes / 4));
        CK(cudaMemcpyAsync(d_dst, ln.ximg.p, bytes, cudaMemcpyDeviceToDevice, s));
        return FSN_OK;
    }
    if (n == "stft" || n == "enh") {
        if (!m->au_valid)
            return fail(FSN_ESTATE, "%s is kept only by an audio call (fsn_model_enhance_audio) that ran as one sub-batch, and the last forward was not one", name);
        const int64_t cnt = (int64_t)(n == "stft" ? 3 : 2) * B * F * ln.geo.T;
        if (numel != cnt) return fail(FSN_EINVAL, "%s needs %lld elements", name, (long long)cnt);
        CK(cudaMemcpyAsync(d_dst, n == "stft" ? m->au_planes.p : m->au_enh.p, (size_t)cnt * 4, cudaMemcpyDeviceToDevice, s));
        return FSN_OK;
    }
    if (n == "sb_mu") {
        if (numel != B) return fail(FSN_EINVAL, "sb_mu needs %d elements", B);
        CK(cudaMemcpyAsync(d_dst, ln.mu.p, (size_t)B * 4, cudaMemcpyDeviceToDevice, s));
        return FSN_OK;
    }
    return fail(FSN_EINVAL, "unknown stage %s", name);
}

// Ordered like a plain call: after the forward it reads, whatever stream that ran on, and before the next call rewrites the workspace
extern "C" int fsn_model_get_stage(fsn_model* m, const char* name, float* d_dst, int64_t numel, void* stream) {
    if (!m || !name || !d_dst) return fail(FSN_EINVAL, "null argument");
    if (!m->lane[m->last_lane].geo.B) return fail(FSN_ESTATE, "no forward has run yet");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = wait_plain(m, s)) return rc;
    const int rc = get_stage(m, name, d_dst, numel, s), rr = mark_plain(m, s);
    return rc ? rc : rr;
}


// ---------------------------------------------------------------------------------------------
// streaming step API (causal fullsubnet.Model)
// ---------------------------------------------------------------------------------------------
// The scratch of a step of K frames over all B slots (step_frames), P = K rounded up to 4: the normalised input [B, F, P], its fp16
// form [K, rows_pad, Ipad], the top layer's h [B, H, P], the full-band output [B, F, P] and the sub-band images (img bytes, zeroed)
struct fsn_stream;
struct StepScratch {
    DevBuf fbin, fbx, hseq, fbout, ximg;
    int ensure(const fsn_stream& st, int K, size_t img, bool zero, cudaStream_t s);
    void release() { for (DevBuf* b : {&fbin, &fbx, &hseq, &fbout, &ximg}) b->release(); }
};
// the generic sub-band step's images of `rows` rows over K frames (wide: time-major rows of 128 halves)
static size_t step_img_bytes(const fsn_config& c, long long rows, int K) { return (size_t)((rows + 127) / 128) * K * 128 * sb_row_bytes(c); }

struct fsn_stream {
    fsn_model* m;
    int B, n = 0;                                      // n: ticks of the handle (the weight-stationary exchange-buffer parity)
    DevBuf cum_in, cum_sb, h_fb, c_fb, h_sb, c_sb, ws_h, ws_c;   // session state (the table STATE)
    StepScratch tick;                                  // the per-frame and per-hop calls' scratch (K = 1)
    DevBuf ws_bar;
    bool use_ws = false;
    int ra_fb = 0, ra_sb = 0, rows_pad = 0, Ipad = 0;
    // slot calls (fsn_stream_step_slots, the chunk call): once used, every step runs per slot.  nb: frames each slot has consumed since
    // its START (seeded with n at the first slot call); d_slot [4 B]: this call's per-slot values for the kernels -- the counts (-1 =
    // held), then the chunk call's layer-wise session lists, then the slots a START zeroes.  They reach the device through `stage`.
    bool slots = false;
    std::vector<int32_t> nb, all_step, valid;
    DevBuf d_slot;
    PinnedStage stage;                                 // every tick's d_slot values, and the slot lists of save / load
    CallOrder order;                                   // every call that takes a stream runs after the handle's previous one
    // A handle serves either the mask calls (fsn_stream_step, fsn_stream_step_slots) or the audio call, whichever it meets first:
    // FSN_STATE_MODE_MASK or FSN_STATE_MODE_AUDIO, 0 before
    int mode = 0;
    // audio calls (fsn_stream_step_audio_slots, fsn_stream_step_audio_chunk), allocated at their first use.  Per slot on the host:
    // a_tick = ticks of the session so far, HOLD excluded (-1: no session); a_hops = its hops K, known from its first FLUSH (0 before);
    // a_pend = samples of its partial next hop (fsn_stream_step_audio_samples, 0 .. hop - 1; held in ring slot a_tick % 3).
    // On the device: the history ring, the noisy-spectrum ring, the overlap tail and the tables
    std::vector<int32_t> a_tick, a_hops, a_pend;
    std::vector<float> a_tables;
    DevBuf a_hist, a_spec, a_tail, a_tab;
    // save / load (fsn_stream_save_slots, fsn_stream_load_slots): the slot list of the last call on the device
    DevBuf x_slot;
    // chunk call (fsn_stream_step_chunk, DESIGN.md §3.13): its scratch, allocated at its first use, grow-only, apart from the model's
    // workspace (the model may forward offline on another stream meanwhile).  On the layer-wise path the images are those of one
    // sub-batch, and c_*: its Gin / layer output, the per-layer h / c carry and the compact masks
    StepScratch chunk;
    DevBuf c_gin, c_hsb, c_h, c_c, c_mask;
    // audio calls (DESIGN.md §3.10, §3.14): their scratch, allocated at their first use, grow-only: the spectra of the call's frames
    // [B, K, F], the model's input and output planes (runs of columns, see StreamAudioChunkLaunch) and the staged per-slot plan
    DevBuf x_spec, x_mag, x_mask, x_plan;
    // attenuation floors of the audio calls (fsn_stream_set_atten_lim, DESIGN.md §3.18): [B] on the host, empty until first set; staged
    // with each audio call's plan when any is > 0.  A handle setting, not session state
    std::vector<float> lam;
    // the last call that stepped the model, for fsn_stream_get_stage: its scratch (null before any step and after an audio call that
    // stepped none), its K, whether its sub band ran layer-wise and whether it was an audio call (x_mag then holds its input)
    const StepScratch* last = nullptr;
    int last_K = 0;
    bool last_lw = false, last_audio = false;
    int last_spec_K = 0;                // the last audio call's K: the slot stride (in frames) of its spectrum scratch x_spec
};

int StepScratch::ensure(const fsn_stream& st, int K, size_t img, bool zero, cudaStream_t s) {
    const size_t B = st.B, F = st.m->cfg.num_freqs, P = (K + 3) & ~3;
    const bool poison = st.m->env_poison;                               // the images' pad rows stay zero: never poisoned
    int e = fbin.ensure(B * F * P * 4, zero, s, poison);
    e |= fbx.ensure((size_t)K * st.rows_pad * st.Ipad * 2, zero, s, poison);
    e |= hseq.ensure(B * st.m->cfg.fb_hidden * P * 4, zero, s, poison);
    e |= fbout.ensure(B * F * P * 4, zero, s, poison);
    e |= ximg.ensure(img, true, s);
    return e;
}

// The state of a session: one entry per buffer, in payload order (DESIGN.md §3.11).  The handle's allocation (fsn_stream_create,
// audio_alloc), its release, the payload layout (state_layout), the save / load copy and the START reset all read this table.
enum { SEG_CUM_IN, SEG_CUM_SB, SEG_FB_H, SEG_FB_C, SEG_SB_H, SEG_SB_C, SEG_HIST, SEG_SPEC, SEG_TAIL, NSEG };
static_assert(NSEG <= STREAM_STATE_MAX_SEG, "every segment fits the copy kernel's table");
enum : unsigned {
    ST_LAYERS = 1,      // one set of rows per LSTM layer (else one set)
    ST_BINS = 2,        // F rows per slot, one per bin (else one row)
    ST_START = 4,       // a START zeroes it: the recurrent state (the norm sums restart at count 0, the audio state at slot tick 0)
    ST_AUDIO = 8,       // audio mode only, after every segment of both modes
    ST_PARITY = 16,     // the weight-stationary variant holds two parities of rows per layer
};
struct StateBuf {
    DevBuf fsn_stream::*buf;
    DevBuf fsn_stream::*ws;                            // the weight-stationary full-band step's buffer in its place (64 rows), or null
    size_t (*row_bytes)(const fsn_config&);
    unsigned flags;
};
static const StateBuf STATE[NSEG] = {
    {&fsn_stream::cum_in, nullptr, [](const fsn_config&) -> size_t { return 2 * sizeof(double); }, 0},   // running sum, sum of squares
    {&fsn_stream::cum_sb, nullptr, [](const fsn_config&) -> size_t { return 2 * sizeof(double); }, ST_BINS},
    {&fsn_stream::h_fb, &fsn_stream::ws_h, [](const fsn_config& c) -> size_t { return c.fb_hidden * sizeof(__half); }, ST_LAYERS | ST_START | ST_PARITY},
    {&fsn_stream::c_fb, &fsn_stream::ws_c, [](const fsn_config& c) -> size_t { return c.fb_hidden * sizeof(float); }, ST_LAYERS | ST_START},
    {&fsn_stream::h_sb, nullptr, [](const fsn_config& c) -> size_t { return c.sb_hidden * sizeof(__half); }, ST_LAYERS | ST_BINS | ST_START},
    {&fsn_stream::c_sb, nullptr, [](const fsn_config& c) -> size_t { return c.sb_hidden * sizeof(float); }, ST_LAYERS | ST_BINS | ST_START},
    {&fsn_stream::a_hist, nullptr, [](const fsn_config& c) -> size_t { return 3 * (c.num_freqs - 1) * sizeof(float); }, ST_AUDIO},   // 3 hops
    {&fsn_stream::a_spec, nullptr, [](const fsn_config& c) -> size_t { return (c.look_ahead + 1) * c.num_freqs * sizeof(float2); }, ST_AUDIO},
    {&fsn_stream::a_tail, nullptr, [](const fsn_config& c) -> size_t { return (c.num_freqs - 1) * sizeof(float); }, ST_AUDIO},      // 1 hop
};
static size_t seg_slot_bytes(const fsn_config& c, int i) { return (STATE[i].flags & ST_BINS ? c.num_freqs : 1) * STATE[i].row_bytes(c); }
static int seg_layers(const fsn_config& c, int i) { return STATE[i].flags & ST_LAYERS ? c.num_layers : 1; }

// Where handle st keeps segment i: slot b's rows of layer l at buf + offset + l * layer + b * seg_slot_bytes.  Layers of the generic
// step's buffers are its rows_alloc rows apart.  The weight-stationary step's h is double-buffered by tick parity (tick n reads
// (n - 1) & 1, writes n & 1): the state is the parity the handle's next tick reads.
struct SegPlace { DevBuf* buf; size_t offset, layer; };
static SegPlace seg_place(fsn_stream* st, int i) {
    const StateBuf& e = STATE[i];
    const fsn_config& c = st->m->cfg;
    const size_t row = e.row_bytes(c);
    SegPlace p{&(st->*e.buf), 0, (size_t)st->B * seg_slot_bytes(c, i)};
    if (st->use_ws && e.ws) {
        p.buf = &(st->*e.ws);
        p.layer = (e.flags & ST_PARITY ? 2 : 1) * 64 * row;
        if (e.flags & ST_PARITY) p.offset = ((st->n ^ 1) & 1) * 64 * row;
    } else if (e.flags & ST_LAYERS) {
        p.layer = (size_t)(e.flags & ST_BINS ? st->ra_sb : st->ra_fb) * row;
    }
    return p;
}

// Allocate, zero-filled on stream s, the state segments of both modes (audio = 0) or of the audio mode only (audio = ST_AUDIO)
static int state_alloc(fsn_stream* st, unsigned audio, cudaStream_t s) {
    int e = 0;
    for (int i = 0; i < NSEG; ++i)
        if ((STATE[i].flags & ST_AUDIO) == audio) {
            const SegPlace p = seg_place(st, i);
            e |= p.buf->ensure(seg_layers(st->m->cfg, i) * p.layer, true, s);
        }
    return e;
}

// stream_state_copy_kernel's work items for the a.nseg segments of a: each layer cut into items of at most `chunk` bytes (32 KB, doubled
// until the items fit)
static void state_items(StreamStateLaunch& a) {
    auto cut = [&](size_t chunk) {
        int k = 0;
        for (int i = 0; i < a.nseg; ++i)               // segments left out have L = 0
            for (int l = 0; l < a.seg[i].L; ++l)
                for (size_t b = 0, n = a.seg[i].slot_bytes; b < n; b += chunk) {
                    if (k == STREAM_STATE_MAX_ITEMS) return false;
                    a.item[k++] = StreamStateItem{i, l, (uint32_t)b, (uint32_t)(b + chunk < n ? b + chunk : n)};
                }
        a.nitem = k;
        return true;
    };
    for (size_t chunk = 32768; !cut(chunk); chunk *= 2) {}
}

// stream_state_copy_kernel's tables for the segments i < ns whose flags include `need`: each at its handle place and payload offset
// off[i] (off null: zeroing, no payload), cut into items by state_items
static void state_launch(fsn_stream* st, int ns, unsigned need, const size_t* off, StreamStateLaunch& a) {
    const fsn_config& c = st->m->cfg;
    a.nseg = ns;
    for (int i = 0; i < ns; ++i) {
        if ((STATE[i].flags & need) != need) continue;
        const SegPlace p = seg_place(st, i);
        const size_t n = seg_slot_bytes(c, i);
        a.seg[i] = StreamStateSeg{static_cast<char*>(p.buf->p) + p.offset, p.layer, n, off ? off[i] : 0, seg_layers(c, i),
                                  (n % 16 || p.layer % 16) ? 8 : 16};
    }
    state_items(a);
}

// The configurations that stream: fullsubnet.Model with a cumulative norm
static int streams_ok(const fsn_config& c) {
    if (c.model_kind != FSN_KIND_FSN)
        return fail(FSN_EINVAL, "model_kind %d: streaming needs fullsubnet.Model (FullSubNet+ is not causal: TSSE pools over all time)", c.model_kind);
    if (c.norm_type != FSN_NORM_CUMULATIVE_LAPLACE && c.norm_type != FSN_NORM_CUMULATIVE_LAYER)
        return fail(FSN_EINVAL, "norm_type %d: streaming needs a cumulative norm_type", c.norm_type);
    return FSN_OK;
}

extern "C" int fsn_stream_create(fsn_model* m, int32_t B, fsn_stream** out) {
    if (!m || !out || B < 1) return fail(FSN_EINVAL, "bad argument");
    if (!m->finalized) return fail(FSN_ESTATE, "fsn_model_finalize has not been called");
    const fsn_config& c = m->cfg;
    if (int rc = streams_ok(c)) return rc;
    fsn_stream* st = new fsn_stream();
    st->m = m; st->B = B;
    const int F = c.num_freqs, rows = B * F;
    st->Ipad = (F + 15) / 16 * 16; st->rows_pad = (B + 63) / 64 * 64;
    lstm_mma_cstate_bytes(1, B, 1, &st->ra_fb);
    lstm_mma_cstate_bytes(1, rows, 1, &st->ra_sb);
    st->use_ws = lstm_ws_supported(c.num_layers, c.fb_hidden, st->Ipad, B, m->num_sms) && !m->env_no_ws;
    // scratch, then state, then the barrier: with the state allocated first, steps at 16-64 slots measured ~0.03 ms slower per tick
    int e = st->tick.ensure(*st, 1, step_img_bytes(c, rows, 1), true, nullptr);
    e |= state_alloc(st, 0, nullptr);
    if (st->use_ws) e |= st->ws_bar.ensure(64, true);
    e |= st->d_slot.ensure((size_t)4 * B * sizeof(int32_t), false);
    // the zero-fills above ran on the legacy stream, which a first step on a non-blocking stream is not ordered after
    if (e || cudaDeviceSynchronize() != cudaSuccess) { fsn_stream_destroy(st); return fail(FSN_ECUDA, "stream state allocation failed"); }
    *out = st;
    return FSN_OK;
}

extern "C" void fsn_stream_destroy(fsn_stream* st) {
    if (!st) return;
    cudaDeviceSynchronize();                                             // nothing in flight may still use the buffers
    for (const StateBuf& e : STATE) {
        (st->*e.buf).release();
        if (e.ws) (st->*e.ws).release();
    }
    st->tick.release();
    st->chunk.release();
    for (DevBuf* b : {&st->ws_bar, &st->d_slot, &st->x_slot, &st->a_tab, &st->c_gin, &st->c_hsb, &st->c_h, &st->c_c, &st->c_mask,
                      &st->x_spec, &st->x_mag, &st->x_mask, &st->x_plan})
        b->release();
    delete st;
}

static int claim_mode(fsn_stream* st, int mode) {
    if (st->mode && st->mode != mode)
        return fail(FSN_ESTATE, mode == FSN_STATE_MODE_AUDIO
                                    ? "this handle serves the mask calls (fsn_stream_step, fsn_stream_step_slots): create another for audio"
                                    : "this handle serves the audio call (fsn_stream_step_audio_slots): create another for masks");
    st->mode = mode;
    return FSN_OK;
}

// A handle that has only used fsn_stream_step takes per-slot counts, each slot at the handle's frame count
static void use_slot_counts(fsn_stream* st) {
    if (!st->slots) st->nb.assign(st->B, st->n);
    st->slots = true;
}

// The layer-wise sub band of a chunk step (DESIGN.md §3.13, §3.14): its stepping sessions in groups of one frame count kf each.  Per
// group: the plan of its nact sessions, and on the device each slot's session index in the group (-1 = not in it) and its slots
struct LwGroup { Plan p; int nact, kf; const int *idx, *sess; };

// K frames of every slot on scratch x (DESIGN.md §3.9, §3.13, §3.14): d_mag [B, F, K] -> d_mask [B, 2, F, K].  slot: null (the
// lockstep step: every slot at frame n) or the device per-slot counts (-1 = held); kf: null (every stepping slot runs K frames) or the
// device per-slot frame counts (a stepping slot runs frames 0 .. kf - 1 and holds after them); zero[nzero]: device list of the slots
// whose recurrent state is zeroed first (a START's).  The full band runs in place over every slot; the sub band too (lw null: the
// per-frame step's kernel and state), or on the layer-wise kernels over the stepping sessions only, one pass per frame-count group.
static int step_frames(fsn_stream* st, StepScratch& x, const float* d_mag, int K, const int* slot, const int* kf, const int* zero,
                       int nzero, float* d_mask, const std::vector<LwGroup>* lw, cudaStream_t s) {
    fsn_model* m = st->m;
    const fsn_config& c = m->cfg;
    const int B = st->B, F = c.num_freqs, L = c.num_layers, n = st->n, Pk = (K + 3) & ~3;
    const int resume = slot ? 1 : n > 0;                                // slot calls: a START zeroes instead of resume = 0
    st->last = nullptr;                                                 // until this step completes, fsn_stream_get_stage refuses
    if (nzero) {
        StreamStateLaunch z{};
        state_launch(st, NSEG, ST_START, nullptr, z);
        z.slots = zero; z.n = nzero; z.dir = STREAM_STATE_ZERO;
        if (int e = launch_stream_state(z, s)) return fail(FSN_ECUDA, "session state reset failed: %s", cudaGetErrorString((cudaError_t)e));
    }
    StreamNormLaunch na{d_mag, static_cast<float*>(x.fbin.p), static_cast<double*>(st->cum_in.p), B, F, K, Pk, n, c.norm_type, slot, kf};
    launch_stream_norm(na, s);
    const FbState fs{static_cast<__half*>(st->ws_h.p), static_cast<float*>(st->ws_c.p), static_cast<unsigned int*>(st->ws_bar.p),
                     static_cast<float*>(st->c_fb.p), st->ra_fb, static_cast<__half*>(st->h_fb.p), resume, n, slot, kf};
    const int nl = run_fb(m, static_cast<const float*>(x.fbin.p), static_cast<__half*>(x.fbx.p), static_cast<float*>(x.hseq.p),
                          static_cast<float*>(x.fbout.p), B, st->rows_pad, K, Pk, st->use_ws, fs, s);
    if (nl < 0) return fail(FSN_ECUDA, "full-band LSTM step failed: %s", cudaGetErrorString((cudaError_t)-nl));
    StreamPackLaunch pa{d_mag, static_cast<const float*>(x.fbout.p), Pk, static_cast<double*>(st->cum_sb.p), static_cast<__half*>(x.ximg.p),
                        B, F, K, c.sb_num_neighbors, c.fb_num_neighbors, n, c.norm_type, 0, K, slot, nullptr, 0, 0, kf};
    const bool wide = sb_wide(c);
    if (!lw) {
        if (wide) launch_stream_pack_wide(pa, s);
        else launch_stream_pack(pa, s);
        LstmMmaLaunch b = m->sb_mma;
        b.rows = B * F; b.Tp = K; b.out = d_mask; b.la = 0;
        b.ntiles = (B * F + 127) / 128;
        if (wide) { b.xplain = static_cast<const __half*>(x.ximg.p); b.rows_pad = b.ntiles * 128; }   // time-major rows of 128 halves
        else b.img = static_cast<const __half*>(x.ximg.p);
        b.cstate = static_cast<float*>(st->c_sb.p); b.rows_alloc = st->ra_sb;
        b.hstate = static_cast<__half*>(st->h_sb.p); b.resume = resume; b.slot = slot; b.slot_rows = F; b.slot_la = c.look_ahead; b.kf = kf;
        if (int e = launch_lstm_mma(b, s)) return fail(FSN_ECUDA, "sub-band LSTM step failed: %s", cudaGetErrorString((cudaError_t)e));
    } else {
        // layer-wise sub band, per group of kf frames: its sessions compacted to rows j F + f, in sub-batches of p.Bs sessions and
        // windows of p.Tw frames.  The recurrence runs as window t0 = 4 + w0 of a 4 + kf step sequence with la = 4: it loads h / c from
        // the carry (t0 > 0), its parities are those of a launch from 0 (t0 % 4 == 0), and local frame k is output column k of
        // [bs, 2, F, kf]; the scatter zeroes the slots' columns from kf on
        const int H = c.sb_hidden;
        int zero_held = 1;
        for (const LwGroup& g : *lw) {
            const int Kg = g.kf, bs_max = g.p.Bs, tw_max = g.p.Tw ? g.p.Tw : Kg;
            for (int j0 = 0; j0 < g.nact; j0 += bs_max) {
                const int bs = g.nact - j0 < bs_max ? g.nact - j0 : bs_max, nt = (bs * F + 127) / 128;
                const size_t cs_layer = lstm_tc5r_cstate_bytes(nt, H) / sizeof(float), hs_layer = (size_t)(nt + 1) / 2 * 2 * 128 * H;
                StreamSbCarryLaunch cy{static_cast<__half*>(st->h_sb.p), static_cast<float*>(st->c_sb.p), st->ra_sb,
                                       static_cast<__half*>(st->c_h.p), hs_layer, static_cast<float*>(st->c_c.p), cs_layer, g.sess + j0, bs, F, H, L, 0};
                launch_stream_sb_carry(cy, s);
                for (int w0 = 0; w0 < Kg; w0 += tw_max) {
                    const int tw = Kg - w0 < tw_max ? Kg - w0 : tw_max;
                    pa.k0 = w0; pa.Kw = tw; pa.idx = g.idx; pa.j0 = j0; pa.nsess = bs;
                    if (wide) launch_stream_pack_wide(pa, s);
                    else launch_stream_pack(pa, s);
                    LstmTc5rLaunch a{};
                    a.rows = bs * F; a.Tp = 4 + Kg; a.ntiles = nt; a.t0 = 4 + w0; a.Tw = tw;
                    a.ximg = static_cast<const __half*>(x.ximg.p); a.hseq = static_cast<__half*>(st->c_hsb.p);
                    a.cstate = static_cast<float*>(st->c_c.p); a.hstate = static_cast<__half*>(st->c_h.p);
                    a.out = static_cast<float*>(st->c_mask.p); a.la = 4;
                    if (int nl = sb_layers(m, a, static_cast<__half*>(st->c_gin.p), cs_layer, hs_layer, s); nl < 0) return nl;
                }
                cy.out = 1;
                launch_stream_sb_carry(cy, s);
                StreamChunkScatterLaunch sc{static_cast<const float*>(st->c_mask.p), d_mask, slot, g.idx, j0, bs, B, F, K, Kg, c.look_ahead,
                                            zero_held};
                launch_stream_chunk_scatter(sc, s);
                zero_held = 0;
            }
        }
        if (zero_held) {                                                // no stepping session: every row is held
            StreamChunkScatterLaunch sc{nullptr, d_mask, slot, nullptr, 0, 0, B, F, K, K, c.look_ahead, 1};
            launch_stream_chunk_scatter(sc, s);
        }
    }
    CK(cudaGetLastError());
    st->n += K;
    st->last = &x; st->last_K = K; st->last_lw = lw != nullptr; st->last_audio = false;
    return FSN_OK;
}

extern "C" int fsn_stream_step(fsn_stream* st, const float* d_mag, float* d_mask, int32_t* h_valid, void* stream) {
    if (!st || !d_mag || !d_mask) return fail(FSN_EINVAL, "null argument");
    if (int rc = claim_mode(st, FSN_STATE_MODE_MASK)) return rc;
    if (st->slots) {                                                    // the slot call with every slot stepping
        st->all_step.assign(st->B, FSN_SLOT_STEP);
        st->valid.resize(st->B);
        const int rc = fsn_stream_step_slots(st, d_mag, d_mask, st->all_step.data(), st->valid.data(), stream);
        if (rc) return rc;
        bool all = true;
        for (int v : st->valid) all = all && v;
        if (h_valid) *h_valid = all ? 1 : 0;
        return FSN_OK;
    }
    const int n = st->n;
    const fsn_config& c = st->m->cfg;
    // sized at create: grows nothing, and enqueues only FSN_POISON's fill
    const int rc = st->order.run(stream, [&] {
        if (st->tick.ensure(*st, 1, step_img_bytes(c, (long long)st->B * c.num_freqs, 1), false, static_cast<cudaStream_t>(stream)))
            return fail(FSN_ECUDA, "step scratch allocation failed");
        return step_frames(st, st->tick, d_mag, 1, nullptr, nullptr, nullptr, 0, d_mask, nullptr, static_cast<cudaStream_t>(stream));
    });
    if (rc) return rc;
    if (h_valid) *h_valid = (n >= st->m->cfg.look_ahead) ? 1 : 0;
    return FSN_OK;
}

// ---------------------------------------------------------------------------------------------
// chunk call: K frames per slot and call (DESIGN.md §3.13)
// ---------------------------------------------------------------------------------------------
// The layer-wise sub-band scratch of a chunk call for a sub-batch of bs sessions, K frames, windows of tw frames (tw = K: one window):
// the images, Gin and the layer output (ws_sizes: the offline forward's windowed buffers), the per-layer h carry (r_hstate's size),
// the per-layer c carry and the compact masks [bs, 2, F, K]
static size_t chunk_sb_bytes(const fsn_config& c, int bs, int K, int tw) {
    const WsSizes z = ws_sizes(c, true, bs, K, tw);
    const int ntiles = (int)(((size_t)bs * c.num_freqs + 127) / 128);
    return z.ximg + z.r_gin + z.r_hseq + z.r_hstate + (size_t)c.num_layers * lstm_tc5r_cstate_bytes(ntiles, c.sb_hidden) +
           (size_t)bs * 2 * c.num_freqs * K * sizeof(float);
}

// Length limits of a chunk: the layer-wise recurrence runs K + 4 steps (t0 = 4, see fsn_stream_step_chunk), within a forward's frame
// limit; a session's K frames of one bin plane are indexed with an int
static int chunk_check(const fsn_config& c, int K) {
    if (K < 1) return fail(FSN_EINVAL, "K = %d: a chunk has at least 1 frame", K);
    if ((long long)K + 4 > FSN_MAX_TP)
        return fail(FSN_EINVAL, "K = %d exceeds the chunk limit of %lld frames (65535 x 256 - 4, the frame limit of a forward)", K, FSN_MAX_TP - 4);
    if ((long long)c.num_freqs * K > 0x7fffffffLL)
        return fail(FSN_EINVAL, "num_freqs x K = %lld exceeds 2^31 - 1, the per-session plane index limit", (long long)c.num_freqs * K);
    return FSN_OK;
}

// The plan of a chunk call with n stepping sessions: on the layer-wise path the sessions run in equal sub-batches of Bs so that
// chunk_sb_bytes stays within cap (the largest that fits, evened out); if even one session's K frames do not fit, one session at a
// time in windows of Tw frames (a multiple of 4, the longest that fits, evened out; 4 if none does).  Tw = 0: one window.  The generic
// path runs in place over the handle's slots in one piece (bytes: its images).
static int chunk_plan(const fsn_config& c, bool layerwise, int n, int K, double cap, Plan* p) {
    if (int rc = streams_ok(c)) return rc;
    if (n < 1) return fail(FSN_EINVAL, "n_active = %d: a plan needs at least 1 stepping session", n);
    if (int rc = chunk_check(c, K)) return rc;
    *p = Plan{n};
    if (!layerwise) {
        p->bytes = (int64_t)step_img_bytes(c, (long long)n * c.num_freqs, K);
        return FSN_OK;
    }
    auto fits = [&](int bs, int tw) { return (double)chunk_sb_bytes(c, bs, K, tw) <= cap; };
    if (!fits(n, K)) {
        if (const int b = largest(0, n, [&](int v) { return fits(v, K); })) {
            const int nsub = (n + b - 1) / b;
            p->Bs = (n + nsub - 1) / nsub;
        } else {
            p->Bs = 1;
            const int u = largest(1, K / 4, [&](int v) { return fits(1, 4 * v); });
            const int nwin = (K + 4 * u - 1) / (4 * u);
            p->Tw = ((K + nwin - 1) / nwin + 3) / 4 * 4;
            if (p->Tw >= K) p->Tw = 0;
        }
    }
    p->bytes = (int64_t)chunk_sb_bytes(c, p->Bs, K, p->Tw ? p->Tw : K);
    return FSN_OK;
}

extern "C" int fsn_stream_chunk_plan(const fsn_config* cfg, int32_t n_active, int32_t K, double cap_bytes, int32_t* Bs, int32_t* Tw,
                                     int64_t* bytes) {
    if (!cfg) return fail(FSN_EINVAL, "cfg is null");
    if (!(cap_bytes > 0)) return fail(FSN_EINVAL, "cap_bytes = %g: the cap must be > 0", cap_bytes);
    Plan p;
    if (int rc = chunk_plan(*cfg, runs_layerwise(*cfg, 0), n_active, K, cap_bytes, &p)) return rc;
    if (Bs) *Bs = p.Bs;
    if (Tw) *Tw = p.Tw;
    if (bytes) *bytes = p.bytes;
    return FSN_OK;
}

// The chunk scratch of a layer-wise sub-band step of K frames under plan p: images, Gin, layer output, h / c carry and compact masks
static int chunk_lw_ensure(fsn_stream* st, const Plan& p, int K, cudaStream_t s) {
    const fsn_config& c = st->m->cfg;
    const int F = c.num_freqs, nt = (p.Bs * F + 127) / 128;
    const WsSizes z = ws_sizes(c, true, p.Bs, K, p.Tw ? p.Tw : K);
    const bool poison = st->m->env_poison;
    int e = st->chunk.ensure(*st, K, z.ximg, false, s);
    e |= st->c_gin.ensure(z.r_gin, false, s, poison);
    e |= st->c_hsb.ensure(z.r_hseq, false, s, poison);
    e |= st->c_h.ensure(z.r_hstate, true, s);
    e |= st->c_c.ensure((size_t)c.num_layers * lstm_tc5r_cstate_bytes(nt, c.sb_hidden), true, s);
    e |= st->c_mask.ensure((size_t)p.Bs * 2 * F * K * sizeof(float), false, s, poison);
    return e;
}

// The layer-wise sub band's session groups of a chunk step whose slot b runs kf[b] frames (0: not stepping), one per distinct
// count in increasing order: each planned under the model's cap and the chunk scratch grown to fit it, before any state changes
// (allocation failures go to *e)
static int lw_groups(fsn_stream* st, const std::vector<int>& kf, std::vector<LwGroup>* lw, int* e, cudaStream_t s) {
    std::vector<int> ks;
    for (int v : kf) if (v) ks.push_back(v);
    std::sort(ks.begin(), ks.end());
    for (size_t i = 0, j; i < ks.size(); i = j) {
        for (j = i; j < ks.size() && ks[j] == ks[i]; ++j) {}
        LwGroup g{Plan{}, (int)(j - i), ks[i], nullptr, nullptr};
        if (int rc = chunk_plan(st->m->cfg, true, g.nact, g.kf, st->m->ws_cap_bytes, &g.p)) return rc;
        *e |= chunk_lw_ensure(st, g.p, g.kf, s);
        lw->push_back(g);
    }
    return FSN_OK;
}

// The groups' slot lists, staged at h on their way to d: per group each slot's session index [B] (-1: not in it), then its slots
// [nact].  Returns the number of values.
static size_t lw_stage(const std::vector<int>& kf, std::vector<LwGroup>& lw, int32_t* h, const int32_t* d) {
    const int B = (int)kf.size();
    size_t at = 0;
    for (LwGroup& g : lw) {
        int32_t *idx = h + at, *sess = idx + B;
        g.idx = d + at; g.sess = d + at + B;
        for (int b = 0, j = 0; b < B; ++b) {
            idx[b] = kf[b] == g.kf ? j : -1;
            if (kf[b] == g.kf) sess[j++] = b;
        }
        at += B + g.nact;
    }
    return at;
}

// The slot calls after their argument checks: every slot advances K frames by its flag (fsn_stream_step_slots: K = 1 on the per-tick
// scratch; the chunk call: on its own scratch, with the layer-wise sub band where the offline forward runs it).  Errors change no state.
static int step_slots(fsn_stream* st, const float* d_mag, int K, float* d_mask, const int32_t* h_flags, int32_t* h_valid, bool chunk,
                      cudaStream_t s) {
    fsn_model* m = st->m;
    const fsn_config& c = m->cfg;
    const int B = st->B, F = c.num_freqs, la = c.look_ahead;
    if (int rc = chunk_check(c, K)) return rc;
    bool reset = false;
    for (int b = 0; b < B; ++b) {
        const int f = h_flags[b];
        if (f != FSN_SLOT_HOLD && f != FSN_SLOT_STEP && f != FSN_SLOT_START)
            return fail(FSN_EINVAL, "slot %d: flag %d is not FSN_SLOT_HOLD (0), FSN_SLOT_STEP (1) or FSN_SLOT_START (2)", b, f);
        reset = reset || f == FSN_SLOT_START;
    }
    if (st->mode == FSN_STATE_MODE_AUDIO) return claim_mode(st, FSN_STATE_MODE_MASK);
    // the scratch, before any state changes (DevBuf::ensure only grows); on the layer-wise path every stepping session runs K
    // frames: one group
    const bool layerwise = chunk && m->layerwise;
    StepScratch& x = chunk ? st->chunk : st->tick;
    st->last = nullptr;                                                 // the scratch may be reallocated below
    std::vector<int> kf;
    std::vector<LwGroup> lw;
    int e = 0;
    if (layerwise) {
        for (int b = 0; b < B; ++b) kf.push_back(h_flags[b] == FSN_SLOT_HOLD ? 0 : K);
        if (int rc = lw_groups(st, kf, &lw, &e, s)) return rc;
    }
    if (lw.empty()) e |= x.ensure(*st, K, layerwise ? 0 : step_img_bytes(c, (long long)B * F, K), false, s);
    if (e) return fail(FSN_ECUDA, "chunk scratch allocation failed (B = %d, K = %d)", B, K);
    if (int rc = claim_mode(st, FSN_STATE_MODE_MASK)) return rc;
    use_slot_counts(st);
    // staged per-slot values: counts [B] (-1 = held), the layer-wise group's lists, then the START list
    int32_t* h = nullptr;
    if (int rc = st->stage.take((size_t)4 * B, &h)) return rc;
    const int* d = static_cast<const int*>(st->d_slot.p);
    const size_t nlw = lw_stage(kf, lw, h + B, d + B);
    int32_t *cnt = h, *zero = h + B + nlw;
    int nzero = 0;
    for (int b = 0; b < B; ++b) {
        cnt[b] = h_flags[b] == FSN_SLOT_HOLD ? -1 : h_flags[b] == FSN_SLOT_START ? 0 : st->nb[b];
        if (reset && cnt[b] == 0) zero[nzero++] = b;                    // started, or never stepped
    }
    if (int rc = st->stage.send(st->d_slot.p, B + nlw + nzero, s)) return rc;
    if (int rc = step_frames(st, x, d_mag, K, d, nullptr, d + B + nlw, nzero, d_mask, layerwise ? &lw : nullptr, s)) return rc;
    for (int b = 0; b < B; ++b) {
        h_valid[b] = 0;
        if (cnt[b] < 0) continue;
        st->nb[b] = cnt[b] + K;
        const int v = cnt[b] + K - la;
        h_valid[b] = v < 0 ? 0 : v > K ? K : v;
    }
    return FSN_OK;
}

extern "C" int fsn_stream_step_slots(fsn_stream* st, const float* d_mag, float* d_mask, const int32_t* h_flags, int32_t* h_valid,
                                     void* stream) {
    if (!st || !d_mag || !d_mask) return fail(FSN_EINVAL, "null argument");
    if (!h_flags) return fail(FSN_EINVAL, "h_flags is null (one flag per slot, slots 0..%d)", st->B - 1);
    if (!h_valid) return fail(FSN_EINVAL, "h_valid is null (one result per slot, slots 0..%d)", st->B - 1);
    return st->order.run(stream, [&] { return step_slots(st, d_mag, 1, d_mask, h_flags, h_valid, false, static_cast<cudaStream_t>(stream)); });
}

extern "C" int fsn_stream_step_chunk(fsn_stream* st, const float* d_mag, int32_t K, float* d_mask, const int32_t* h_flags,
                                     int32_t* h_valid, void* stream) {
    if (!st) return fail(FSN_EINVAL, "st is null");
    if (!d_mag) return fail(FSN_EINVAL, "d_mag is null (K magnitude frames per slot, [B, F, K] float32 on the device)");
    if (!d_mask) return fail(FSN_EINVAL, "d_mask is null (K mask columns per slot, [B, 2, F, K] float32 on the device)");
    if (!h_flags) return fail(FSN_EINVAL, "h_flags is null (one flag per slot, slots 0..%d)", st->B - 1);
    if (!h_valid) return fail(FSN_EINVAL, "h_valid is null (one result per slot, slots 0..%d)", st->B - 1);
    return st->order.run(stream, [&] { return step_slots(st, d_mag, K, d_mask, h_flags, h_valid, true, static_cast<cudaStream_t>(stream)); });
}

// Audio state of the handle, zero-filled on the call's stream, and the tables of its n_fft (computed in double).
static int audio_alloc(fsn_stream* st, cudaStream_t s) {
    const size_t B = st->B, F = st->m->cfg.num_freqs;
    int e = state_alloc(st, ST_AUDIO, s);
    audio_tables((int)(2 * (F - 1)), st->a_tables);
    e |= st->a_tab.ensure(st->a_tables.size() * sizeof(float), false, s);
    if (e) return fail(FSN_ECUDA, "audio stream state allocation failed");
    CK(cudaMemcpyAsync(st->a_tab.p, st->a_tables.data(), st->a_tables.size() * sizeof(float), cudaMemcpyHostToDevice, s));
    st->a_tick.assign(B, -1);
    st->a_hops.assign(B, 0);
    st->a_pend.assign(B, 0);
    return FSN_OK;
}

// The rules of slot b's flag f against its session that every audio call checks, in the order they are reported: the flag's range;
// for a START, STEP or FLUSH the call's own count check count(name of the flag); then a STEP or FLUSH needs a session, a STEP one
// whose input has not ended, and a FLUSH after the session's FLUSH a count n of 0.  arg, unit: the count's argument and unit.
template <class CountCheck>
static int audio_session_check(const fsn_stream* st, int b, int f, int n, const char* arg, const char* unit, CountCheck count) {
    if (f < FSN_SLOT_HOLD || f > FSN_SLOT_FLUSH)
        return fail(FSN_EINVAL, "slot %d: flag %d is not FSN_SLOT_HOLD (0), FSN_SLOT_STEP (1), FSN_SLOT_START (2) or FSN_SLOT_FLUSH (3)", b, f);
    if (f == FSN_SLOT_HOLD) return FSN_OK;
    const char* name = f == FSN_SLOT_START ? "START" : f == FSN_SLOT_STEP ? "STEP" : "FLUSH";
    if (int rc = count(name)) return rc;
    if (f == FSN_SLOT_START) return FSN_OK;
    const int t = st->a_tick.empty() ? -1 : st->a_tick[b], Kh = st->a_hops.empty() ? 0 : st->a_hops[b];
    if (t < 0) return fail(FSN_EINVAL, "slot %d: %s on a slot without a session (START one first)", b, name);
    if (f == FSN_SLOT_STEP && Kh)
        return fail(FSN_EINVAL, "slot %d: STEP after the session's FLUSH (its input has ended: START a new session)", b);
    if (f == FSN_SLOT_FLUSH && Kh && n)
        return fail(FSN_EINVAL, "slot %d: FLUSH with %s = %d after the session's FLUSH (its input has ended: pass 0 %s)", b, arg, n, unit);
    return FSN_OK;
}

// One slot's ticks in an audio call of K hops (DESIGN.md §3.10, §3.14).  Flag f with n hops stands for K per-hop ticks: START,
// STEP x (n - 1) / STEP x n / STEP x n then FLUSH, the rest HOLD.  The active ones -- every tick but the HOLDs and the FLUSH ticks past
// the session's end -- come first: na of them, at slot ticks k0 .. k0 + na - 1 (a START's k0 is 0).  The first nstore store the row's
// hops, and every active tick but a START's is a model frame.  hops: the session's K after the call (0 before its FLUSH); nout: the
// hops the call emits (those of slot ticks k >= la + 2).  Checks the flag and hop count against the slot's session.  A session at
// tick 0 (started by the sample call with less than a hop) runs its START tick with its first hop, whatever the flag.  r: the samples
// past the last whole hop of a session the sample call ends (L = (t + n) hop + r), 0 for the hop calls.
struct AudioSlotPlan { int k0, na, start, nstore, hops, nout; };
static int audio_slot_plan(const fsn_stream* st, int b, int f, int n, int K, AudioSlotPlan* p, int r = 0) {
    const int la = st->m->cfg.look_ahead;
    const int t = st->a_tick.empty() ? -1 : st->a_tick[b], Kh = st->a_hops.empty() ? 0 : st->a_hops[b];
    *p = AudioSlotPlan{t, 0, 0, 0, Kh, 0};
    const int lo = f == FSN_SLOT_FLUSH ? 0 : 1;
    if (int rc = audio_session_check(st, b, f, n, "h_hops", "hops", [&](const char* name) {
            return n < lo || n > K ? fail(FSN_EINVAL, "slot %d: h_hops = %d: a %s consumes %d to K = %d hops", b, n, name, lo, K) : FSN_OK;
        }))
        return rc;
    if (f == FSN_SLOT_HOLD) return FSN_OK;
    if (f == FSN_SLOT_START) {
        *p = AudioSlotPlan{0, n, 1, n, 0, 0};
    } else {
        if (f == FSN_SLOT_FLUSH && !Kh && t + n < 2 && !(t + n == 1 && r))
            return fail(FSN_EINVAL, "slot %d: FLUSH after %d hop: a session needs at least 2 hops (the STFT's reflect padding reads "
                                    "n_fft / 2 + 1 samples)", b, t + n);
        p->k0 = t; p->nstore = n; p->start = t == 0;
        if (f == FSN_SLOT_STEP) {
            p->na = n;
        } else {                                                        // active up to slot tick K + la + 1, then a FLUSH is a HOLD
            p->hops = Kh ? Kh : n < K ? t + n : 0;                      // n = K: no FLUSH tick yet, the end is not known
            const int left = p->hops ? p->hops + la + 2 - t : n;
            p->na = left < 0 ? 0 : left < K ? left : K;
        }
    }
    const int e0 = p->k0 > la + 2 ? p->k0 : la + 2, e1 = p->k0 + p->na;
    p->nout = e1 > e0 ? e1 - e0 : 0;
    return FSN_OK;
}

// The sample call's part of an audio call (fsn_stream_step_audio_samples, DESIGN.md §3.19): per slot the samples pending before the
// call and the trailing partial hop after it (StreamAudioLaunch::r0, r), the rows' strides, and whether any slot ticks (else only
// the analysis kernel runs: it stores the partial hops and zeroes the output rows)
struct SampleRows { const int32_t *r0, *r; int S, So; bool tick; };

// The audio calls after their argument checks: every slot advances by its plan (fsn_stream_step_audio_slots: K = 1, one hop per
// START / STEP) through the K-hop kernels around one K-frame model step.  The per-hop call (chunk = false) steps the model on the
// per-tick scratch with the generic sub band; the chunk call on its own scratch, with the layer-wise sub band where the offline
// forward runs it.  smp: the sample call's rows and planes (null for the hop calls: rows of K hops, no partial hops).  Errors
// change no state.
static int run_audio(fsn_stream* st, const std::vector<AudioSlotPlan>& plan, const float* d_samples, int K, bool chunk, float* d_out,
                     float* d_mask, const SampleRows* smp, cudaStream_t s) {
    fsn_model* m = st->m;
    const fsn_config& c = m->cfg;
    const int B = st->B, F = c.num_freqs, la = c.look_ahead, N = 2 * (F - 1);
    // The model's frames: slot b's kf of them, left-aligned in columns 0 .. kf - 1 of [B, F, Km], Km the largest kf.  One K-frame
    // step runs them all, each slot holding after its kf frames; on the layer-wise path its sub band runs one pass per group of
    // sessions with one kf (in steady state a single group).  Km = 0 (every slot holds): no model step.
    std::vector<int> kf(B);
    int Km = 0, nzero = 0;
    for (int b = 0; b < B; ++b) {
        kf[b] = plan[b].na > plan[b].start ? plan[b].na - plan[b].start : 0;
        Km = kf[b] > Km ? kf[b] : Km;
        nzero += kf[b] && plan[b].k0 + plan[b].start == 1;          // model frame 0 in column 0: a START's reset
    }
    const bool layerwise = chunk && m->layerwise;
    StepScratch& x = chunk ? st->chunk : st->tick;
    st->last = nullptr;                                                 // the scratch may be reallocated below
    std::vector<LwGroup> lw;
    int e = 0;
    if (layerwise)
        if (int rc = lw_groups(st, kf, &lw, &e, s)) return rc;
    size_t nstage = (size_t)7 * B + nzero;
    for (const LwGroup& g : lw) nstage += B + g.nact;
    const bool lim = std::any_of(st->lam.begin(), st->lam.end(), [](float v) { return v > 0.f; });
    const size_t lam_at = nstage;                                       // the slots' attenuation floors, last (when any is set)
    if (lim) nstage += B;
    const size_t smp_at = nstage;                                       // the sample call's two planes after everything else
    if (smp) nstage += 2 * (size_t)B;
    if (Km) e |= x.ensure(*st, Km, layerwise ? 0 : step_img_bytes(c, (long long)B * F, Km), false, s);
    e |= st->x_spec.ensure((size_t)B * K * F * sizeof(float2), false, s, m->env_poison);
    e |= st->x_mag.ensure((size_t)B * F * Km * sizeof(float), false, s, m->env_poison);
    e |= st->x_mask.ensure((size_t)B * 2 * F * Km * sizeof(float), false, s, m->env_poison);
    e |= st->x_plan.ensure(nstage * sizeof(int32_t), false, s);
    if (e) return fail(FSN_ECUDA, "audio chunk scratch allocation failed (B = %d, K = %d)", B, K);
    if (int rc = claim_mode(st, FSN_STATE_MODE_AUDIO)) return rc;
    if (st->a_tick.empty())
        if (int rc = audio_alloc(st, s)) return rc;
    // staged: the five per-slot planes of the kernels, the model's frame counts at column 0 (-1 = held) and frame counts, the
    // slots whose model frame 0 is in this call, then the layer-wise groups' lists
    int32_t* h = nullptr;
    if (int rc = st->stage.take(nstage, &h)) return rc;
    const int32_t* d = static_cast<const int32_t*>(st->x_plan.p);
    int32_t *cnt = h + 5 * B, *kfp = h + 6 * B, *zero = h + 7 * B;
    for (int b = 0, z = 0; b < B; ++b) {
        const AudioSlotPlan& p = plan[b];
        h[b] = p.k0; h[B + b] = p.na; h[2 * B + b] = p.start; h[3 * B + b] = p.nstore; h[4 * B + b] = p.hops;
        cnt[b] = kf[b] ? p.k0 + p.start - 1 : -1;
        kfp[b] = kf[b];
        if (kf[b] && cnt[b] == 0) zero[z++] = b;
    }
    lw_stage(kf, lw, zero + nzero, d + 7 * B + nzero);
    if (lim) memcpy(h + lam_at, st->lam.data(), (size_t)B * sizeof(float));
    if (smp) {
        memcpy(h + smp_at, smp->r0, (size_t)B * sizeof(int32_t));
        memcpy(h + smp_at + B, smp->r, (size_t)B * sizeof(int32_t));
    }
    if (int rc = st->stage.send(st->x_plan.p, nstage, s)) return rc;
    StreamAudioLaunch a{};
    a.k0 = d; a.na = d + B; a.start = d + 2 * B; a.nstore = d + 3 * B; a.hops = d + 4 * B;
    a.samples = d_samples; a.out = d_out;
    a.S = a.So = K * (F - 1);
    if (smp) { a.r0 = d + smp_at; a.r = d + smp_at + B; a.S = smp->S; a.So = smp->So; a.zero_out = !smp->tick; }
    a.hist = static_cast<float*>(st->a_hist.p); a.spec = static_cast<float2*>(st->a_spec.p); a.tail = static_cast<float*>(st->a_tail.p);
    a.sspec = static_cast<float2*>(st->x_spec.p); a.mag = static_cast<float*>(st->x_mag.p); a.mask = static_cast<float*>(st->x_mask.p);
    a.umask = d_mask;
    const AudioTables tab = audio_table_ptrs(static_cast<const float*>(st->a_tab.p), N);
    a.window = tab.window; a.twiddle = tab.twiddle; a.inv_env = tab.inv_env; a.inv_last = tab.inv_last;
    a.B = B; a.K = K; a.Km = Km; a.n_fft = N; a.la = la;
    a.lam = lim ? reinterpret_cast<const float*>(d + lam_at) : nullptr;
    launch_stream_stft(a, s);
    if (a.zero_out) {                                                   // no tick: no model step and no synthesis
        st->last = nullptr;
        CK(cudaGetLastError());
        return FSN_OK;
    }
    // at Km = 1 the counts alone say which slots step a frame: no frame counts, so the per-frame step's kernels and arguments
    if (Km)
        if (int rc = step_frames(st, x, a.mag, Km, d + 5 * B, Km > 1 ? d + 6 * B : nullptr, d + 7 * B, nzero,
                                 static_cast<float*>(st->x_mask.p), layerwise ? &lw : nullptr, s))
            return rc;
    if (Km) { st->last_audio = true; st->last_spec_K = K; }
    else st->last = nullptr;
    launch_stream_istft(a, s);
    CK(cudaGetLastError());
    return FSN_OK;
}

// The hop calls (fsn_stream_step_audio_slots: K = 1, h_hops null; fsn_stream_step_audio_chunk): their plans, then run_audio
static int step_audio(fsn_stream* st, const float* d_samples, int K, const int32_t* h_flags, const int32_t* h_hops, float* d_out,
                      int32_t* h_nout, float* d_mask, cudaStream_t s) {
    const fsn_config& c = st->m->cfg;
    const int B = st->B;
    if (int rc = audio_fft_ok(c)) return rc;
    if (int rc = chunk_check(c, K)) return rc;                         // num_freqs x K < 2^31 bounds the rows' K x hop too
    std::vector<AudioSlotPlan> plan(B);
    for (int b = 0; b < B; ++b) {                                       // every slot is checked before any state changes
        const int n = h_hops ? h_hops[b] : h_flags[b] == FSN_SLOT_FLUSH ? 0 : 1;
        if (int rc = audio_slot_plan(st, b, h_flags[b], n, K, &plan[b])) return rc;
        if ((h_flags[b] == FSN_SLOT_STEP || h_flags[b] == FSN_SLOT_FLUSH) && !st->a_pend.empty() && st->a_pend[b])
            return fail(FSN_EINVAL, "slot %d: %s on a session holding a partial hop of %d samples (continue it with "
                                    "fsn_stream_step_audio_samples)", b, h_flags[b] == FSN_SLOT_STEP ? "STEP" : "FLUSH", st->a_pend[b]);
    }
    if (st->mode == FSN_STATE_MODE_MASK) return claim_mode(st, FSN_STATE_MODE_AUDIO);
    if (int rc = run_audio(st, plan, d_samples, K, h_hops != nullptr, d_out, d_mask, nullptr, s)) return rc;
    for (int b = 0; b < B; ++b) {
        const AudioSlotPlan& p = plan[b];
        if (h_flags[b] != FSN_SLOT_HOLD) { st->a_tick[b] = p.k0 + p.na; st->a_hops[b] = p.hops; st->a_pend[b] = 0; }
        h_nout[b] = p.nout;
    }
    return FSN_OK;
}

extern "C" int fsn_stream_step_audio_slots(fsn_stream* st, const float* d_samples, float* d_out, const int32_t* h_flags,
                                           int32_t* h_valid, float* d_mask, void* stream) {
    if (!st) return fail(FSN_EINVAL, "st is null");
    if (!d_samples) return fail(FSN_EINVAL, "d_samples is null (one hop of samples per slot, [B, hop] float32 on the device)");
    if (!d_out) return fail(FSN_EINVAL, "d_out is null (one hop of output per slot, [B, hop] float32 on the device)");
    if (!h_flags) return fail(FSN_EINVAL, "h_flags is null (one flag per slot, slots 0..%d)", st->B - 1);
    if (!h_valid) return fail(FSN_EINVAL, "h_valid is null (one result per slot, slots 0..%d)", st->B - 1);
    return st->order.run(stream, [&] {
        return step_audio(st, d_samples, 1, h_flags, nullptr, d_out, h_valid, d_mask, static_cast<cudaStream_t>(stream));
    });
}

extern "C" int fsn_stream_step_audio_chunk(fsn_stream* st, const float* d_samples, int32_t K, const int32_t* h_flags,
                                           const int32_t* h_hops, float* d_out, int32_t* h_nout, float* d_mask, void* stream) {
    if (!st) return fail(FSN_EINVAL, "st is null");
    if (!d_samples) return fail(FSN_EINVAL, "d_samples is null (K hops of samples per slot, [B, K x hop] float32 on the device)");
    if (!d_out) return fail(FSN_EINVAL, "d_out is null (K hops of output per slot, [B, K x hop] float32 on the device)");
    if (!h_flags) return fail(FSN_EINVAL, "h_flags is null (one flag per slot, slots 0..%d)", st->B - 1);
    if (!h_hops) return fail(FSN_EINVAL, "h_hops is null (one hop count per slot, slots 0..%d)", st->B - 1);
    if (!h_nout) return fail(FSN_EINVAL, "h_nout is null (one result per slot, slots 0..%d)", st->B - 1);
    return st->order.run(stream, [&] {
        return step_audio(st, d_samples, K, h_flags, h_hops, d_out, h_nout, d_mask, static_cast<cudaStream_t>(stream));
    });
}

// Any number of samples per slot and call (DESIGN.md §3.19).  Each slot's completed hops become the ticks of a hop call: START with n
// hops (a START, or any first hop of a session at tick 0), STEP with n, or FLUSH with n and then the ticks that end the session.  A
// call of at most one hop per slot and no FLUSH runs the per-hop call's path; any other the K-hop path, K the most ticks of a slot.
// The partial hops are the kernels' r0 / r planes.  Every check runs before any state changes.
extern "C" int fsn_stream_step_audio_samples(fsn_stream* st, const float* d_samples, int32_t S, const int32_t* h_flags,
                                             const int32_t* h_counts, float* d_out, int32_t* h_nout, void* stream) {
    if (!st) return fail(FSN_EINVAL, "st is null");
    if (!d_samples) return fail(FSN_EINVAL, "d_samples is null (S samples per slot, [B, S] float32 on the device)");
    if (!d_out) return fail(FSN_EINVAL, "d_out is null ([B, S + (look_ahead + 3) hop] float32 on the device)");
    if (!h_flags) return fail(FSN_EINVAL, "h_flags is null (one flag per slot, slots 0..%d)", st->B - 1);
    if (!h_counts) return fail(FSN_EINVAL, "h_counts is null (one sample count per slot, slots 0..%d)", st->B - 1);
    if (!h_nout) return fail(FSN_EINVAL, "h_nout is null (one result per slot, slots 0..%d)", st->B - 1);
    if (S < 1) return fail(FSN_EINVAL, "S = %d: the rows hold at least one sample", S);
    const fsn_config& c = st->m->cfg;
    if (int rc = audio_fft_ok(c)) return rc;
    const int B = st->B, H = c.num_freqs - 1, la = c.look_ahead;
    const long long So = (long long)S + (long long)(la + 3) * H;
    if (So > 0x7fffffffLL) return fail(FSN_EINVAL, "S + (look_ahead + 3) hop = %lld output samples per row: past 2^31 - 1", So);
    const bool fresh = st->a_tick.empty();
    std::vector<int32_t> n(B, 0), need(B, 0), r0(B, 0), r(B, 0);
    int K = 0;
    bool flush = false, consume = false;
    for (int b = 0; b < B; ++b) {                                       // every slot is checked before any state changes
        const int f = h_flags[b], cnt = h_counts[b];
        if (int rc = audio_session_check(st, b, f, cnt, "h_counts", "samples", [&](const char*) {
                return cnt < 0 || cnt > S ? fail(FSN_EINVAL, "slot %d: h_counts = %d is outside [0, S = %d]", b, cnt, S) : FSN_OK;
            }))
            return rc;
        const int t = fresh ? -1 : st->a_tick[b], Kh = fresh ? 0 : st->a_hops[b], p0 = fresh ? 0 : st->a_pend[b];
        r0[b] = r[b] = p0;
        if (f == FSN_SLOT_HOLD) continue;
        consume = consume || cnt > 0;
        if (f == FSN_SLOT_START) r0[b] = 0;
        const long long tot = (long long)r0[b] + cnt;
        n[b] = (int)(tot / H);
        r[b] = (int)(tot % H);
        need[b] = n[b];
        if (f == FSN_SLOT_FLUSH) {
            if (Kh) {
                need[b] = Kh + la + 2 - t > 0 ? Kh + la + 2 - t : 0;
            } else {
                const long long L = (long long)(t + n[b]) * H + r[b];
                if (L <= H)
                    return fail(FSN_EINVAL, "slot %d: FLUSH would end a session of %lld samples: a session needs more than n_fft / 2 = %d "
                                            "(the STFT's reflect padding reads n_fft / 2 + 1 samples)", b, L, H);
                need[b] = n[b] + la + 2;
            }
            flush = flush || need[b] > 0;
        }
        K = need[b] > K ? need[b] : K;
    }
    const bool chunk = flush || K > 1;                                  // else the per-hop call's path
    const int Kc = K ? K : 1;
    if (chunk)
        if (int rc = chunk_check(c, Kc)) return rc;
    std::vector<AudioSlotPlan> plan(B);
    for (int b = 0; b < B; ++b) {
        const int f = h_flags[b];
        AudioSlotPlan& p = plan[b];
        if (f == FSN_SLOT_HOLD || (f != FSN_SLOT_FLUSH && !n[b])) {     // no tick; a START of less than a hop starts at tick 0
            if (int rc = audio_slot_plan(st, b, FSN_SLOT_HOLD, 0, Kc, &p)) return rc;
            if (f == FSN_SLOT_START) { p.k0 = 0; p.hops = 0; }
        } else if (int rc = audio_slot_plan(st, b, f, n[b], Kc, &p, f == FSN_SLOT_FLUSH ? r[b] : 0)) {
            return rc;
        }
    }
    if (st->mode == FSN_STATE_MODE_MASK) return claim_mode(st, FSN_STATE_MODE_AUDIO);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int rc = st->order.run(stream, [&] {
        if (K == 0 && !consume) {                                       // nothing to store or synthesise: the rows are zero
            if (int rc = claim_mode(st, FSN_STATE_MODE_AUDIO)) return rc;
            if (st->a_tick.empty())
                if (int rc = audio_alloc(st, s)) return rc;
            CK(cudaMemsetAsync(d_out, 0, (size_t)B * So * sizeof(float), s));
            return FSN_OK;
        }
        const SampleRows rows{r0.data(), r.data(), S, (int)So, K > 0};
        return run_audio(st, plan, d_samples, Kc, chunk, d_out, nullptr, &rows, s);
    });
    if (rc) return rc;
    for (int b = 0; b < B; ++b) {
        const int f = h_flags[b];
        const AudioSlotPlan& p = plan[b];
        h_nout[b] = p.nout * H;
        if (f == FSN_SLOT_HOLD) continue;
        st->a_tick[b] = p.k0 + p.na;
        st->a_hops[b] = p.hops;
        st->a_pend[b] = f == FSN_SLOT_FLUSH ? 0 : r[b];
        if (f == FSN_SLOT_FLUSH) h_nout[b] += r[b];                     // the partial end (0 for a session a hop call ended)
    }
    return FSN_OK;
}

extern "C" int fsn_stream_fb_ws(const fsn_stream* st) { return st && st->use_ws ? 1 : 0; }

static int stream_get_stage(fsn_stream* st, const char* name, float* d_dst, int64_t numel, void* stream) {
    const std::string n(name);
    if (n != "fb_in" && n != "fb_out" && n != "sb_img" && n != "mag" && n != "mask" && n != "spec")
        return fail(FSN_EINVAL, "unknown stage %s", name);
    if (!st->last) return fail(FSN_ESTATE, "no step call has stepped the model yet, or the last one failed or stepped no frame");
    const fsn_config& c = st->m->cfg;
    const int B = st->B, F = c.num_freqs, K = st->last_K, Pk = (K + 3) & ~3;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (n == "fb_in" || n == "fb_out") {
        if (numel != (int64_t)B * F * K) return fail(FSN_EINVAL, "%s needs %lld elements", name, (long long)B * F * K);
        const void* src = (n == "fb_in") ? st->last->fbin.p : st->last->fbout.p;
        CK(cudaMemcpy2DAsync(d_dst, (size_t)K * 4, src, (size_t)Pk * 4, (size_t)K * 4, (size_t)B * F, cudaMemcpyDeviceToDevice, s));
        return FSN_OK;
    }
    if (n == "sb_img") {
        if (st->last_lw)
            return fail(FSN_ESTATE, "sb_img is not kept: the last step ran the sub band layer-wise, its images are compact rows per group, sub-batch and window");
        const size_t bytes = step_img_bytes(c, (long long)B * F, K);
        if (numel * 4 != (int64_t)bytes) return fail(FSN_EINVAL, "sb_img needs %lld elements", (long long)(bytes / 4));
        CK(cudaMemcpyAsync(d_dst, st->last->ximg.p, bytes, cudaMemcpyDeviceToDevice, s));
        return FSN_OK;
    }
    if (!st->last_audio) return fail(FSN_ESTATE, "%s is kept only by the audio calls, and the last step was a mask call", name);
    if (n == "spec") {                                                  // [B, K, F] complex of the call's scratch [B, K_call, F]
        if (numel != (int64_t)2 * B * K * F) return fail(FSN_EINVAL, "spec needs %lld elements", (long long)2 * B * K * F);
        const size_t row = (size_t)K * F * sizeof(float2);
        CK(cudaMemcpy2DAsync(d_dst, row, st->x_spec.p, (size_t)st->last_spec_K * F * sizeof(float2), row, (size_t)B, cudaMemcpyDeviceToDevice, s));
        return FSN_OK;
    }
    const int rows = n == "mask" ? 2 * F : F;
    if (numel != (int64_t)B * rows * K) return fail(FSN_EINVAL, "%s needs %lld elements", name, (long long)B * rows * K);
    CK(cudaMemcpyAsync(d_dst, n == "mask" ? st->x_mask.p : st->x_mag.p, (size_t)B * rows * K * 4, cudaMemcpyDeviceToDevice, s));
    return FSN_OK;
}

extern "C" int fsn_stream_get_stage(fsn_stream* st, const char* name, float* d_dst, int64_t numel, void* stream) {
    if (!st || !name || !d_dst) return fail(FSN_EINVAL, "null argument");
    return st->order.run(stream, [&] { return stream_get_stage(st, name, d_dst, numel, stream); });
}

// ---------------------------------------------------------------------------------------------
// overlapped-chunk sessions (DESIGN.md §3.16): the reference's overlapped_chunk inferencer (inferencer.py:191-250) per slot, every
// chunk completed in a call enhanced in one offline audio forward
// ---------------------------------------------------------------------------------------------
static const int CHUNK_PRE = 256;                      // P: the reference's pre-context, in samples at every geometry

// Per slot on the host: n = samples of the session so far (-1: no session) and k = its chunks enhanced; chunk k covers session samples
// [k H - P, k H + C), and y[0, k H) has been emitted (all of y[0, L) once the session has ended).  On the device: the sample ring
// [B, C + P], the overlap tail [B, chunk_tail_stride(C)] and the window [C]; the plan and the batch's rows are per call, grow-only;
// x_slot: the slot list of the last save / load (DESIGN.md §3.17), grow-only.
struct fsn_chunk_stream {
    fsn_model* m;
    int B, C;
    std::vector<int64_t> n, k;
    DevBuf ring, tail, window, plan, rows, enh, x_slot;
    PinnedStage stage;
    CallOrder order;                                   // step, save and load run in call order whatever their streams
    std::vector<float> lam_db;                         // attenuation limits in dB (fsn_chunk_stream_set_atten_lim): [B], empty until first set
};

// The chunk lengths a handle can take on its own, whatever the model: even, H >= P, C + P < 2^30
static int chunk_length_ok(int C) {
    if (C < 2 || C % 2) return fail(FSN_EINVAL, "chunk_samples = %d: the chunk length must be even (two halves of 50 %% overlap)", C);
    if (C / 2 < CHUNK_PRE)
        return fail(FSN_EINVAL, "chunk_samples = %d: the half-chunk %d is shorter than the %d-sample pre-context (chunk_samples >= %d)", C,
                    C / 2, CHUNK_PRE, 2 * CHUNK_PRE);
    if ((long long)C > 0x3fffffffLL - CHUNK_PRE)
        return fail(FSN_EINVAL, "chunk_samples = %d exceeds 2^30 - 1 - %d samples", C, CHUNK_PRE);
    return FSN_OK;
}

// The plan of slot b for flag f and count c (CP_* fields into p), and its n and k after the call.  Checks the flag and the count.
static int chunk_slot_plan(const fsn_chunk_stream* cs, int b, int f, int c, int S, int row0, int32_t* p, int64_t* n1, int64_t* k1) {
    const int H = cs->C / 2;
    if (f < FSN_SLOT_HOLD || f > FSN_SLOT_FLUSH)
        return fail(FSN_EINVAL, "slot %d: flag %d is not FSN_SLOT_HOLD (0), FSN_SLOT_STEP (1), FSN_SLOT_START (2) or FSN_SLOT_FLUSH (3)", b, f);
    for (int i = 0; i < CHUNK_PLAN_FIELDS; ++i) p[i] = 0;
    p[CP_ROW0] = row0;
    *n1 = cs->n[b]; *k1 = cs->k[b];
    if (f == FSN_SLOT_HOLD) return FSN_OK;
    const char* name = f == FSN_SLOT_START ? "START" : f == FSN_SLOT_STEP ? "STEP" : "FLUSH";
    if (c < 0 || c > S) return fail(FSN_EINVAL, "slot %d: h_counts = %d: a %s consumes 0 to S = %d samples", b, c, name, S);
    if (f != FSN_SLOT_START && cs->n[b] < 0) return fail(FSN_EINVAL, "slot %d: %s on a slot without a session (START one first)", b, name);
    const int64_t n0 = f == FSN_SLOT_START ? 0 : cs->n[b], k0 = f == FSN_SLOT_START ? 0 : cs->k[b], a0 = k0 * H, n = n0 + c;
    // chunk k is complete once the input reaches k H + C; at FLUSH every chunk that starts before the end is, zero-padded
    const int64_t kend = f == FSN_SLOT_FLUSH ? (n + H - 1) / H : std::max(k0, n / H - 1);
    p[CP_NC] = (int32_t)(kend - k0);
    p[CP_REL0] = (int32_t)(n0 - a0);
    p[CP_REL1] = (int32_t)(n - a0);
    p[CP_LO] = k0 ? -CHUNK_PRE : 0;
    p[CP_PHASE] = (int32_t)(a0 % (cs->C + CHUNK_PRE));
    p[CP_NOUT] = (int32_t)(f == FSN_SLOT_FLUSH ? n - a0 : (kend - k0) * H);
    *n1 = f == FSN_SLOT_FLUSH ? -1 : n;
    *k1 = f == FSN_SLOT_FLUSH ? 0 : kend;
    return FSN_OK;
}

extern "C" int fsn_chunk_stream_create(fsn_model* m, int32_t B, int32_t chunk_samples, fsn_chunk_stream** out) {
    if (!m) return fail(FSN_EINVAL, "m is null");
    if (!out) return fail(FSN_EINVAL, "out is null");
    if (B < 1) return fail(FSN_EINVAL, "B = %d: the handle needs at least one slot", B);
    if (!m->finalized) return fail(FSN_ESTATE, "fsn_model_finalize has not been called");
    const int C = chunk_samples;
    if (int rc = chunk_length_ok(C)) return rc;
    // every batch of the step is fsn_model_enhance_audio on rows of P + C samples: refused here with that call's message
    int T = 0, Lmax = 0;
    bool all = true;
    int rc = audio_check(m->cfg, 1, (int64_t)CHUNK_PRE + C, nullptr, &T, &Lmax, &all);
    if (!rc && m->cfg.output_size != 2) rc = fail(FSN_EINVAL, "the audio call needs output_size 2 (a complex mask)");
    if (rc) {
        char why[512];
        snprintf(why, sizeof(why), "%s", g_err);
        return fail(rc, "chunk_samples = %d: fsn_model_enhance_audio refuses rows of %d + %d samples: %s", C, CHUNK_PRE, C, why);
    }
    fsn_chunk_stream* cs = new fsn_chunk_stream();
    cs->m = m; cs->B = B; cs->C = C;
    cs->n.assign(B, -1);
    cs->k.assign(B, 0);
    std::vector<float> w(C);
    const double pi = std::acos(-1.0);
    for (int i = 0; i < C; ++i) w[i] = (float)(0.5 - 0.5 * std::cos(2.0 * pi * i / C));   // torch.hann_window(C), periodic
    int e = cs->ring.ensure((size_t)B * (C + CHUNK_PRE) * sizeof(float), true);
    e |= cs->tail.ensure((size_t)B * chunk_tail_stride(C) * sizeof(float), true);
    e |= cs->window.ensure((size_t)C * sizeof(float), false);
    e |= cs->plan.ensure((size_t)B * CHUNK_PLAN_FIELDS * sizeof(int32_t), false);
    // the zero-fills and the pageable copy ran on the legacy stream, which a non-blocking stream's first step is not ordered after
    if (e || cudaMemcpy(cs->window.p, w.data(), (size_t)C * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaDeviceSynchronize() != cudaSuccess) {
        fsn_chunk_stream_destroy(cs);
        return fail(FSN_ECUDA, "chunk stream state allocation failed (B = %d, chunk_samples = %d)", B, C);
    }
    *out = cs;
    return FSN_OK;
}

extern "C" void fsn_chunk_stream_destroy(fsn_chunk_stream* cs) {
    if (!cs) return;
    cudaDeviceSynchronize();                                             // nothing in flight may still use the buffers
    for (DevBuf* b : {&cs->ring, &cs->tail, &cs->window, &cs->plan, &cs->rows, &cs->enh, &cs->x_slot}) b->release();
    delete cs;
}

// Every slot's plan is made and checked, then the batch of the completed chunks is checked as the offline audio call, before anything
// is allocated, staged or launched.  Then: the gather, the forward (run_plain: it waits for pipelined batches and plans sub-batches
// under the cap as fsn_model_enhance_audio does; none when no chunk completes), the cross-fade, and the host counters.
extern "C" int fsn_chunk_stream_step(fsn_chunk_stream* cs, const float* d_samples, int32_t S, const int32_t* h_flags,
                                     const int32_t* h_counts, float* d_out, int32_t* h_nout, void* stream) {
    if (!cs) return fail(FSN_EINVAL, "cs is null");
    const int B = cs->B, C = cs->C, W = C + CHUNK_PRE;
    if (!d_samples) return fail(FSN_EINVAL, "d_samples is null ([B, S] float32 on the device)");
    if (!d_out) return fail(FSN_EINVAL, "d_out is null ([B, S + chunk_samples] float32 on the device)");
    if (!h_flags) return fail(FSN_EINVAL, "h_flags is null (one flag per slot, slots 0..%d)", B - 1);
    if (!h_counts) return fail(FSN_EINVAL, "h_counts is null (one sample count per slot, slots 0..%d)", B - 1);
    if (!h_nout) return fail(FSN_EINVAL, "h_nout is null (one result per slot, slots 0..%d)", B - 1);
    if (S < 1) return fail(FSN_EINVAL, "S = %d: a row needs at least one sample", S);
    if ((long long)S + 2LL * W > 0x7fffffffLL)
        return fail(FSN_EINVAL, "S = %d: S + 2 (chunk_samples + %d) exceeds 2^31 - 1", S, CHUNK_PRE);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    std::vector<int32_t> plan((size_t)B * CHUNK_PLAN_FIELDS);
    std::vector<int64_t> n1(B), k1(B);
    int nrows = 0;
    for (int b = 0; b < B; ++b) {
        int32_t* p = plan.data() + (size_t)b * CHUNK_PLAN_FIELDS;
        if (int rc = chunk_slot_plan(cs, b, h_flags[b], h_counts[b], S, nrows, p, &n1[b], &k1[b])) return rc;
        if ((long long)nrows + p[CP_NC] > 0x7fffffffLL / W) return fail(FSN_EINVAL, "more than 2^31 - 1 samples of chunk rows in one call");
        nrows += p[CP_NC];
    }
    // the batch of every completed chunk: rows [nrows, P + C]; the caller's buffers stand in for the rows until they are allocated
    Batch fwd{CALL_AUDIO, nullptr, nullptr, nullptr, nrows, 0, nullptr, nullptr, nullptr, d_samples, d_out, W, nullptr};
    std::vector<int32_t> lens;
    std::vector<float> row_db, row_lam;                                 // each row enhanced with its slot's limit (check_batch drops
    if (nrows && !cs->lam_db.empty()) {                                 // them when none is finite)
        row_db.reserve((size_t)nrows);
        for (int b = 0; b < B; ++b)
            row_db.insert(row_db.end(), (size_t)plan[(size_t)b * CHUNK_PLAN_FIELDS + CP_NC], cs->lam_db[b]);
        fwd.atten_db = row_db.data();
    }
    if (nrows)
        if (int rc = check_batch(cs->m, fwd, &lens, &row_lam)) return rc;
    const size_t rb = (size_t)nrows * W * sizeof(float);
    const int rc = cs->order.run(stream, [&] {
        int e = nrows ? cs->rows.ensure(rb, false, s, cs->m->env_poison) | cs->enh.ensure(rb, false, s, cs->m->env_poison) : 0;
        if (e) return fail(FSN_ECUDA, "chunk row allocation failed (%d rows of %d samples)", nrows, W);
        int32_t* h = nullptr;
        if (int rc = cs->stage.take(plan.size(), &h)) return rc;
        memcpy(h, plan.data(), plan.size() * sizeof(int32_t));
        if (int rc = cs->stage.send(cs->plan.p, plan.size(), s)) return rc;
        ChunkStreamLaunch a{};
        a.plan = static_cast<const int*>(cs->plan.p);
        a.samples = d_samples; a.out = d_out;
        a.ring = static_cast<float*>(cs->ring.p); a.tail = static_cast<float*>(cs->tail.p);
        a.rows = static_cast<float*>(cs->rows.p); a.enh = static_cast<const float*>(cs->enh.p);
        a.window = static_cast<const float*>(cs->window.p);
        a.B = B; a.S = S; a.C = C; a.P = CHUNK_PRE;
        launch_chunk_gather(a, s);
        CK(cudaGetLastError());
        if (nrows) {
            fwd.wave = a.rows; fwd.wave_out = static_cast<float*>(cs->enh.p);
            if (int rc = run_plain(cs->m, fwd, s)) return rc;
        }
        launch_chunk_crossfade(a, s);
        CK(cudaGetLastError());
        return FSN_OK;
    });
    if (rc) return rc;
    for (int b = 0; b < B; ++b) {
        cs->n[b] = n1[b]; cs->k[b] = k1[b];
        h_nout[b] = plan[(size_t)b * CHUNK_PLAN_FIELDS + CP_NOUT];
    }
    return FSN_OK;
}

// The checks of a set_atten_lim call on a handle of B slots (fsn_stream_set_atten_lim, fsn_chunk_stream_set_atten_lim): the arrays, n,
// every slot in range and named once, every limit valid (atten_floor); *lam: the n floors.  Nothing is changed here.
static int slot_limits_ok(int B, int32_t n, const int32_t* h_slots, const float* h_atten_db, std::vector<float>* lam) {
    if (n < 1) return fail(FSN_EINVAL, "n = %d: at least one slot", n);
    if (!h_slots) return fail(FSN_EINVAL, "h_slots is null (n = %d slot indices)", n);
    if (!h_atten_db) return fail(FSN_EINVAL, "h_atten_db is null (n = %d limits in dB)", n);
    std::vector<int> seen(B, -1);
    lam->resize((size_t)n);
    for (int i = 0; i < n; ++i) {
        const int b = h_slots[i];
        if (b < 0 || b >= B) return fail(FSN_EINVAL, "h_slots[%d] = %d is out of range (slots 0..%d)", i, b, B - 1);
        if (seen[b] >= 0) return fail(FSN_EINVAL, "h_slots[%d] = %d: slot %d is named twice (also h_slots[%d])", i, b, b, seen[b]);
        seen[b] = i;
        if (int rc = atten_floor(h_atten_db[i], "slot", b, i, &(*lam)[i])) return rc;
    }
    return FSN_OK;
}

extern "C" int fsn_stream_set_atten_lim(fsn_stream* st, int32_t n, const int32_t* h_slots, const float* h_atten_db) {
    if (!st) return fail(FSN_EINVAL, "st is null");
    std::vector<float> lam;
    if (int rc = slot_limits_ok(st->B, n, h_slots, h_atten_db, &lam)) return rc;
    if (st->lam.empty()) st->lam.assign((size_t)st->B, 0.f);
    for (int i = 0; i < n; ++i) st->lam[h_slots[i]] = lam[i];
    return FSN_OK;
}

extern "C" int fsn_chunk_stream_set_atten_lim(fsn_chunk_stream* cs, int32_t n, const int32_t* h_slots, const float* h_atten_db) {
    if (!cs) return fail(FSN_EINVAL, "cs is null");
    std::vector<float> lam;
    if (int rc = slot_limits_ok(cs->B, n, h_slots, h_atten_db, &lam)) return rc;
    if (cs->lam_db.empty()) cs->lam_db.assign((size_t)cs->B, INFINITY);
    for (int i = 0; i < n; ++i) cs->lam_db[h_slots[i]] = h_atten_db[i];
    return FSN_OK;
}

// ---------------------------------------------------------------------------------------------
// park, resume and move sessions (DESIGN.md §3.11)
// ---------------------------------------------------------------------------------------------
// The payload: the mode's segments of the table STATE in order, each at a 16-byte aligned offset off[i]; ns of them, the stride
// rounded up to 256 bytes
static int state_layout(const fsn_config& c, int mode, size_t* off, int* ns, int64_t* stride) {
    if (int rc = streams_ok(c)) return rc;
    if (mode != FSN_STATE_MODE_MASK && mode != FSN_STATE_MODE_AUDIO)
        return fail(FSN_EINVAL, "mode %d is not FSN_STATE_MODE_MASK (1) or FSN_STATE_MODE_AUDIO (2)", mode);
    if (c.num_freqs < 4 || c.num_freqs > 2048 || c.look_ahead < 0 || c.num_layers < 1 || c.num_layers > 4 || c.fb_hidden < 16 ||
        c.fb_hidden % 16 || c.sb_hidden < 16 || c.sb_hidden % 16)
        return fail(FSN_EINVAL, "bad configuration: num_freqs %d, look_ahead %d, num_layers %d, fb_hidden %d, sb_hidden %d", c.num_freqs,
                    c.look_ahead, c.num_layers, c.fb_hidden, c.sb_hidden);
    if (mode == FSN_STATE_MODE_AUDIO)
        if (int rc = audio_fft_ok(c)) return rc;
    size_t o = 0;
    int k = 0;
    for (; k < NSEG && (mode == FSN_STATE_MODE_AUDIO || !(STATE[k].flags & ST_AUDIO)); ++k) {
        if (off) off[k] = o;
        o += (seg_slot_bytes(c, k) * seg_layers(c, k) + 15) & ~(size_t)15;
    }
    if (ns) *ns = k;
    *stride = (int64_t)((o + 255) & ~(size_t)255);
    return FSN_OK;
}

extern "C" int fsn_stream_state_layout(const fsn_config* cfg, int32_t mode, int64_t* payload_bytes, int32_t* meta_bytes) {
    if (!cfg) return fail(FSN_EINVAL, "cfg is null");
    int64_t stride = 0;
    if (int rc = state_layout(*cfg, mode, nullptr, nullptr, &stride)) return rc;
    if (payload_bytes) *payload_bytes = stride;
    if (meta_bytes) *meta_bytes = (int32_t)sizeof(fsn_slot_meta);
    return FSN_OK;
}

extern "C" uint64_t fsn_model_weights_id(const fsn_model* m) { return m && m->finalized ? m->weights_id : 0; }

extern "C" int64_t fsn_stream_state_bytes(const fsn_stream* st) {
    if (!st) return fail(FSN_EINVAL, "st is null");
    if (!st->mode) return fail(FSN_ESTATE, "the handle has served no call and no load yet: its mode (masks or audio) is not known");
    int64_t stride = 0;
    if (int rc = state_layout(st->m->cfg, st->mode, nullptr, nullptr, &stride)) return rc;
    return stride;
}

// The first configuration field in which a and b differ, lstm_impl excepted (streaming always runs the mma kernels); null if none
static const char* cfg_diff(const fsn_config& a, const fsn_config& b, int* va, int* vb) {
    for (const auto& e : kCfgFields) {
        if (e.off == offsetof(fsn_config, lstm_impl)) continue;
        memcpy(va, reinterpret_cast<const char*>(&a) + e.off, 4);
        memcpy(vb, reinterpret_cast<const char*>(&b) + e.off, 4);
        if (*va != *vb) return e.name;
    }
    return nullptr;
}

// n slot indices of a handle of B slots, distinct when `unique`
static int state_slots_ok(int B, int n, const int32_t* h_slots, bool unique) {
    if (n < 1) return fail(FSN_EINVAL, "n = %d: at least one slot", n);
    if (!h_slots) return fail(FSN_EINVAL, "h_slots is null (n = %d slot indices)", n);
    std::vector<int> seen(unique ? B : 0, -1);
    for (int i = 0; i < n; ++i) {
        const int b = h_slots[i];
        if (b < 0 || b >= B) return fail(FSN_EINVAL, "h_slots[%d] = %d is out of range (slots 0..%d)", i, b, B - 1);
        if (unique && seen[b] >= 0) return fail(FSN_EINVAL, "h_slots[%d] = %d: slot %d is loaded twice (also h_slots[%d])", i, b, b, seen[b]);
        if (unique) seen[b] = i;
    }
    return FSN_OK;
}

// d_state: 256-byte aligned device memory of the device that holds handle_mem, the handle's state
static int state_buffer_ok(const void* handle_mem, const void* d_state) {
    if (!d_state) return fail(FSN_EINVAL, "d_state is null");
    cudaPointerAttributes pa{}, ph{};
    const cudaError_t e = cudaPointerGetAttributes(&pa, d_state);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(FSN_EINVAL, "d_state is not device memory (%s)", cudaGetErrorString(e));
    }
    if (pa.type != cudaMemoryTypeDevice && pa.type != cudaMemoryTypeManaged)
        return fail(FSN_EINVAL, "d_state is not device memory (memory type %d: a host pointer)", (int)pa.type);
    CK(cudaPointerGetAttributes(&ph, handle_mem));
    if (pa.device != ph.device) return fail(FSN_EINVAL, "d_state is memory of device %d, the handle lives on device %d", pa.device, ph.device);
    if (reinterpret_cast<uintptr_t>(d_state) % 256) return fail(FSN_EINVAL, "d_state is not 256-byte aligned");
    return FSN_OK;
}

// One launch of stream_state_copy_kernel for n sessions: the mode's segments between their handle slots h_slots and the payload.
// A lockstep handle switches to per-slot counts first, as at its first slot call.
static int state_copy(fsn_stream* st, int n, const int32_t* h_slots, void* d_state, int mode, int dir, cudaStream_t s) {
    size_t off[NSEG] = {};
    int ns = 0;
    int64_t stride = 0;
    if (int rc = state_layout(st->m->cfg, mode, off, &ns, &stride)) return rc;
    if (mode == FSN_STATE_MODE_MASK) use_slot_counts(st);
    StreamStateLaunch a{};
    state_launch(st, ns, 0, off, a);
    if (st->x_slot.ensure((size_t)(n > st->B ? n : st->B) * sizeof(int32_t), false)) return fail(FSN_ECUDA, "slot-list buffer allocation failed");
    int32_t* h = nullptr;
    if (int rc = st->stage.take(n, &h)) return rc;
    memcpy(h, h_slots, (size_t)n * sizeof(int32_t));
    if (int rc = st->stage.send(st->x_slot.p, n, s)) return rc;
    a.slots = static_cast<const int*>(st->x_slot.p); a.n = n;
    a.payload = static_cast<char*>(d_state); a.stride = (size_t)stride; a.dir = dir;
    const int e = launch_stream_state(a, s);
    if (e) return fail(FSN_ECUDA, "session state copy failed: %s", cudaGetErrorString((cudaError_t)e));
    return FSN_OK;
}

extern "C" int fsn_stream_save_slots(fsn_stream* st, int32_t n, const int32_t* h_slots, void* d_state, fsn_slot_meta* h_meta, void* stream) {
    if (!st) return fail(FSN_EINVAL, "st is null");
    if (int rc = state_slots_ok(st->B, n, h_slots, false)) return rc;
    if (!h_meta) return fail(FSN_EINVAL, "h_meta is null (n = %d metas)", n);
    const int mode = st->mode;
    if (!mode || (mode == FSN_STATE_MODE_AUDIO && st->a_tick.empty()))
        return fail(FSN_ESTATE, "the handle has served no call and no load: it holds no session to save");
    if (int rc = state_buffer_ok(st->cum_in.p, d_state)) return rc;
    int64_t stride = 0;
    if (int rc = state_layout(st->m->cfg, mode, nullptr, nullptr, &stride)) return rc;
    if (int rc = st->order.run(stream, [&] { return state_copy(st, n, h_slots, d_state, mode, STREAM_STATE_SAVE, static_cast<cudaStream_t>(stream)); }))
        return rc;
    for (int i = 0; i < n; ++i) {
        const int b = h_slots[i];
        fsn_slot_meta& q = h_meta[i];
        memset(&q, 0, sizeof(q));
        q.magic = FSN_SLOT_STATE_MAGIC; q.version = FSN_SLOT_STATE_VERSION;
        q.cfg = st->m->cfg; q.weights_id = st->m->weights_id; q.mode = mode;
        if (mode == FSN_STATE_MODE_MASK) q.frames = st->nb[b];
        else { q.tick = st->a_tick[b]; q.hops = st->a_hops[b]; q.frames = st->a_pend[b]; }
        q.payload_bytes = stride;
    }
    return FSN_OK;
}

extern "C" int fsn_stream_load_slots(fsn_stream* st, int32_t n, const int32_t* h_slots, const void* d_state, const fsn_slot_meta* h_meta,
                                     void* stream) {
    if (!st) return fail(FSN_EINVAL, "st is null");
    if (int rc = state_slots_ok(st->B, n, h_slots, true)) return rc;
    if (!h_meta) return fail(FSN_EINVAL, "h_meta is null (n = %d metas)", n);
    const fsn_model* m = st->m;
    const int hmode = st->mode;
    static const char* kModeName[3] = {"", "mask", "audio"};
    for (int i = 0; i < n; ++i) {                                       // every meta is checked before any state changes
        const fsn_slot_meta& q = h_meta[i];
        if (q.magic != FSN_SLOT_STATE_MAGIC) return fail(FSN_EINVAL, "h_meta[%d]: bad magic 0x%08x (not a saved session)", i, q.magic);
        if (q.version != FSN_SLOT_STATE_VERSION)
            return fail(FSN_EINVAL, "h_meta[%d]: version %u, this library reads version %d", i, q.version, FSN_SLOT_STATE_VERSION);
        if (q.mode != FSN_STATE_MODE_MASK && q.mode != FSN_STATE_MODE_AUDIO)
            return fail(FSN_EINVAL, "h_meta[%d]: mode %d is not FSN_STATE_MODE_MASK (1) or FSN_STATE_MODE_AUDIO (2)", i, q.mode);
        const int want = hmode ? hmode : h_meta[0].mode;
        if (q.mode != want)
            return fail(FSN_ESTATE, "h_meta[%d]: a session of the %s call, this handle serves the %s call%s", i, kModeName[q.mode],
                        kModeName[want], hmode ? "" : " (the mode of h_meta[0])");
        int va = 0, vb = 0;
        if (const char* f = cfg_diff(q.cfg, m->cfg, &va, &vb))
            return fail(FSN_EINVAL, "h_meta[%d]: cfg.%s = %d, this handle's model has %d", i, f, va, vb);
        if (q.weights_id != m->weights_id)
            return fail(FSN_EINVAL, "h_meta[%d]: weights_id %016llx, this handle's model has %016llx (other weights)", i,
                        (unsigned long long)q.weights_id, (unsigned long long)m->weights_id);
        int64_t stride = 0;
        if (int rc = state_layout(m->cfg, q.mode, nullptr, nullptr, &stride)) return rc;
        if (q.payload_bytes != stride)
            return fail(FSN_EINVAL, "h_meta[%d]: payload_bytes %lld, this handle's payload is %lld bytes", i, (long long)q.payload_bytes,
                        (long long)stride);
        if (q.mode == FSN_STATE_MODE_MASK ? q.frames < 0 : (q.tick < -1 || q.hops < 0))
            return fail(FSN_EINVAL, "h_meta[%d]: bad counters (frames %d, tick %d, hops %d)", i, q.frames, q.tick, q.hops);
        if (q.mode == FSN_STATE_MODE_AUDIO && q.frames) {               // the samples of a partial hop (fsn_stream_step_audio_samples)
            const int H = m->cfg.num_freqs - 1;
            if (q.frames < 0 || q.frames >= H)
                return fail(FSN_EINVAL, "h_meta[%d]: frames = %d pending samples, outside [0, hop = %d)", i, q.frames, H);
            if (q.tick < 0) return fail(FSN_EINVAL, "h_meta[%d]: frames = %d pending samples on a meta without a session (tick -1)", i, q.frames);
            if (q.hops) return fail(FSN_EINVAL, "h_meta[%d]: frames = %d pending samples after the session's FLUSH (hops %d)", i, q.frames, q.hops);
        }
    }
    if (int rc = state_buffer_ok(st->cum_in.p, d_state)) return rc;
    const int mode = h_meta[0].mode;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (int rc = claim_mode(st, mode)) return rc;
    if (int rc = st->order.run(stream, [&] {
            if (mode == FSN_STATE_MODE_AUDIO && st->a_tick.empty())
                if (int rc = audio_alloc(st, s)) return rc;
            return state_copy(st, n, h_slots, const_cast<void*>(d_state), mode, STREAM_STATE_LOAD, s);
        }))
        return rc;
    for (int i = 0; i < n; ++i) {
        const int b = h_slots[i];
        if (mode == FSN_STATE_MODE_MASK) st->nb[b] = h_meta[i].frames;
        else { st->a_tick[b] = h_meta[i].tick; st->a_hops[b] = h_meta[i].hops; st->a_pend[b] = h_meta[i].frames; }
    }
    return FSN_OK;
}

// ---------------------------------------------------------------------------------------------
// park, resume and move overlapped-chunk sessions (DESIGN.md §3.17)
// ---------------------------------------------------------------------------------------------
// The payload of C: the ring row at 0, the tail row at the next 16-byte boundary, the stride rounded up to 256 bytes.  The copy moves
// the tail's handle row, chunk_tail_stride(C) floats: H floats and the padding up to the payload's next 16-byte boundary.
struct ChunkLayout { size_t ring, tail_off, tail_copy, stride; };
static int chunk_layout(int C, ChunkLayout* l) {
    if (int rc = chunk_length_ok(C)) return rc;
    l->ring = (size_t)(C + CHUNK_PRE) * sizeof(float);
    l->tail_off = (l->ring + 15) & ~(size_t)15;
    l->tail_copy = (size_t)chunk_tail_stride(C) * sizeof(float);
    l->stride = (l->tail_off + (size_t)(C / 2) * sizeof(float) + 255) & ~(size_t)255;
    return FSN_OK;
}

extern "C" int fsn_chunk_stream_state_layout(int32_t chunk_samples, int64_t* payload_bytes, int32_t* meta_bytes) {
    ChunkLayout l{};
    if (int rc = chunk_layout(chunk_samples, &l)) return rc;
    if (payload_bytes) *payload_bytes = (int64_t)l.stride;
    if (meta_bytes) *meta_bytes = (int32_t)sizeof(fsn_chunk_slot_meta);
    return FSN_OK;
}

// One launch of stream_state_copy_kernel for n sessions: the ring and the tail as two segments of one layer each, between the handle
// slots h_slots and the payload.  Ring rows are (C + P) 4 bytes (8-byte multiples when C = 2 mod 4), tail rows 16-byte multiples.
static int chunk_state_copy(fsn_chunk_stream* cs, int n, const int32_t* h_slots, void* d_state, int dir, cudaStream_t s) {
    ChunkLayout l{};
    if (int rc = chunk_layout(cs->C, &l)) return rc;
    StreamStateLaunch a{};
    a.nseg = 2;
    a.seg[0] = StreamStateSeg{static_cast<char*>(cs->ring.p), 0, l.ring, 0, 1, l.ring % 16 ? 8 : 16};
    a.seg[1] = StreamStateSeg{static_cast<char*>(cs->tail.p), 0, l.tail_copy, l.tail_off, 1, 16};
    state_items(a);
    if (cs->x_slot.ensure((size_t)(n > cs->B ? n : cs->B) * sizeof(int32_t), false)) return fail(FSN_ECUDA, "slot-list buffer allocation failed");
    int32_t* h = nullptr;
    if (int rc = cs->stage.take(n, &h)) return rc;
    memcpy(h, h_slots, (size_t)n * sizeof(int32_t));
    if (int rc = cs->stage.send(cs->x_slot.p, n, s)) return rc;
    a.slots = static_cast<const int*>(cs->x_slot.p); a.n = n;
    a.payload = static_cast<char*>(d_state); a.stride = l.stride; a.dir = dir;
    const int e = launch_stream_state(a, s);
    if (e) return fail(FSN_ECUDA, "chunk session state copy failed: %s", cudaGetErrorString((cudaError_t)e));
    return FSN_OK;
}

extern "C" int fsn_chunk_stream_save_slots(fsn_chunk_stream* cs, int32_t n, const int32_t* h_slots, void* d_state, fsn_chunk_slot_meta* h_meta,
                                           void* stream) {
    if (!cs) return fail(FSN_EINVAL, "cs is null");
    if (int rc = state_slots_ok(cs->B, n, h_slots, false)) return rc;
    if (!h_meta) return fail(FSN_EINVAL, "h_meta is null (n = %d metas)", n);
    if (int rc = state_buffer_ok(cs->ring.p, d_state)) return rc;
    ChunkLayout l{};
    if (int rc = chunk_layout(cs->C, &l)) return rc;
    if (int rc = cs->order.run(stream, [&] { return chunk_state_copy(cs, n, h_slots, d_state, STREAM_STATE_SAVE, static_cast<cudaStream_t>(stream)); }))
        return rc;
    const fsn_model* m = cs->m;
    for (int i = 0; i < n; ++i) {
        const int b = h_slots[i];
        fsn_chunk_slot_meta& q = h_meta[i];
        memset(&q, 0, sizeof(q));
        q.magic = FSN_CHUNK_STATE_MAGIC; q.version = FSN_CHUNK_STATE_VERSION;
        q.chunk_samples = cs->C; q.pre_context = CHUNK_PRE;
        q.num_freqs = m->cfg.num_freqs; q.model_kind = m->cfg.model_kind; q.weights_id = m->weights_id;
        q.samples = cs->n[b]; q.chunks = cs->k[b];
        q.payload_bytes = (int64_t)l.stride;
    }
    return FSN_OK;
}

extern "C" int fsn_chunk_stream_load_slots(fsn_chunk_stream* cs, int32_t n, const int32_t* h_slots, const void* d_state,
                                           const fsn_chunk_slot_meta* h_meta, void* stream) {
    if (!cs) return fail(FSN_EINVAL, "cs is null");
    if (int rc = state_slots_ok(cs->B, n, h_slots, true)) return rc;
    if (!h_meta) return fail(FSN_EINVAL, "h_meta is null (n = %d metas)", n);
    ChunkLayout l{};
    if (int rc = chunk_layout(cs->C, &l)) return rc;
    const int64_t H = cs->C / 2;
    for (int i = 0; i < n; ++i) {                                       // every meta is checked before any state changes
        const fsn_chunk_slot_meta& q = h_meta[i];
        if (q.magic != FSN_CHUNK_STATE_MAGIC) return fail(FSN_EINVAL, "h_meta[%d]: bad magic 0x%08x (not a saved chunk session)", i, q.magic);
        if (q.version != FSN_CHUNK_STATE_VERSION)
            return fail(FSN_EINVAL, "h_meta[%d]: version %u, this library reads version %d", i, q.version, FSN_CHUNK_STATE_VERSION);
        if (q.chunk_samples != cs->C)
            return fail(FSN_EINVAL, "h_meta[%d]: chunk_samples %d, this handle's chunks are %d samples", i, q.chunk_samples, cs->C);
        if (q.pre_context != CHUNK_PRE)
            return fail(FSN_EINVAL, "h_meta[%d]: pre_context %d, this handle's pre-context is %d samples", i, q.pre_context, CHUNK_PRE);
        if (q.payload_bytes != (int64_t)l.stride)
            return fail(FSN_EINVAL, "h_meta[%d]: payload_bytes %lld, this handle's payload is %lld bytes", i, (long long)q.payload_bytes,
                        (long long)l.stride);
        if (q.samples < -1 || q.samples > (1LL << 62))
            return fail(FSN_EINVAL, "h_meta[%d]: samples %lld is outside -1 .. 2^62", i, (long long)q.samples);
        const int64_t k = q.samples < 0 ? 0 : std::max<int64_t>(0, q.samples / H - 1);
        if (q.chunks != k)
            return fail(FSN_EINVAL, "h_meta[%d]: chunks %lld, a session of %lld samples has enhanced %lld (max(0, floor(samples / %lld) - 1))",
                        i, (long long)q.chunks, (long long)q.samples, (long long)k, (long long)H);
    }
    if (int rc = state_buffer_ok(cs->ring.p, d_state)) return rc;
    if (int rc = cs->order.run(stream, [&] {
            return chunk_state_copy(cs, n, h_slots, const_cast<void*>(d_state), STREAM_STATE_LOAD, static_cast<cudaStream_t>(stream));
        }))
        return rc;
    for (int i = 0; i < n; ++i) {
        const int b = h_slots[i];
        cs->n[b] = h_meta[i].samples; cs->k[b] = h_meta[i].chunks;
    }
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
extern "C" int fsn_model_last_fb_ws(const fsn_model* m) { return m ? m->last_fb_ws : 0; }

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

extern "C" int fsn_plan_audio(const fsn_config* cfg, int32_t B, int64_t L, const int64_t* h_lengths, double cap_bytes, int32_t force_window,
                              int32_t force_bins, int32_t* Bs, int32_t* Tw, int32_t* Fc, int64_t* bytes) {
    if (!cfg || !Bs || !Tw || !Fc || !(cap_bytes > 0)) return fail(FSN_EINVAL, "bad argument");
    if (force_window < 0 || force_window % 32) return fail(FSN_EINVAL, "force_window must be 0 or a positive multiple of 32");
    if (force_bins < 0) return fail(FSN_EINVAL, "force_bins must be 0 or a positive number of bins");
    if (cfg->num_layers < 1 || cfg->num_layers > 4 || cfg->look_ahead < 0) return fail(FSN_EINVAL, "bad configuration");
    int T = 0, Lmax = 0;
    bool all = true;
    if (int rc = audio_check(*cfg, B, L, h_lengths, &T, &Lmax, &all)) return rc;
    return put_plan(plan_forward(*cfg, runs_layerwise(*cfg, 0), B, T, cap_bytes, force_window, force_bins, true), Bs, Tw, Fc, bytes);
}

extern "C" int fsn_plan_forward(const fsn_config* cfg, int32_t B, int32_t T, double cap_bytes, int32_t force_window, int32_t* Bs, int32_t* Tw,
                                int64_t* bytes) {
    int32_t fc = 0;
    return fsn_plan_forward_bins(cfg, B, T, cap_bytes, force_window, 0, Bs, Tw, &fc, bytes);
}

extern "C" int fsn_model_plan_bins(const fsn_model* m, int32_t B, int32_t T, int32_t* Bs, int32_t* Tw, int32_t* Fc, int64_t* bytes) {
    if (!m || !Bs || !Tw || !Fc || B < 1 || T < 1) return fail(FSN_EINVAL, "bad argument");
    if (int rc = check_length(m->cfg, 1, T)) return rc;
    return put_plan(plan_forward(m->cfg, m->layerwise, B, T, m->ws_cap_bytes, m->env_sb_window, m->env_sb_chunk),
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

// ---- speech metrics (DESIGN.md §3.20): model-free, one score per clip ----------------------------------------------------------

static int metric_check(const char* fn, int32_t B, int64_t L, const int64_t* h_lengths, long long* Lmax) {
    if (B < 1 || B > 65535) return fail(FSN_EINVAL, "%s: B = %d: a batch holds 1 .. 65535 clips", fn, B);
    if (L < 1 || L > 0x7fffffffLL) return fail(FSN_EINVAL, "%s: L = %lld: the row length must be 1 .. 2^31 - 1 samples", fn, (long long)L);
    long long mx = 0;
    for (int b = 0; b < (h_lengths ? B : 1); ++b) {
        const long long n = h_lengths ? h_lengths[b] : L;
        if (n < 1 || n > L)
            return fail(FSN_EINVAL, "%s: clip %d: h_lengths[%d] = %lld is outside 1 .. L = %lld", fn, b, b, n, (long long)L);
        if (n > mx) mx = n;
    }
    *Lmax = mx;
    return FSN_OK;
}

static int metric_sr_check(const char* fn, int32_t sr) {
    if (sr < 8000 || sr > 48000) return fail(FSN_EINVAL, "%s: sr = %d: the sample rate must be 8000 .. 48000 Hz", fn, sr);
    return FSN_OK;
}

static int metric_work_check(const char* fn, const void* d_ref, const void* d_est, const void* d_work, const void* d_out, int64_t work_bytes,
                             size_t need) {
    if (!d_ref || !d_est || !d_out || !d_work) return fail(FSN_EINVAL, "%s: null device pointer", fn);
    if (work_bytes < 0 || (size_t)work_bytes < need)
        return fail(FSN_EINVAL, "%s: work_bytes = %lld, the call needs %zu", fn, (long long)work_bytes, need);
    return FSN_OK;
}

static std::vector<long long> metric_lengths(int32_t B, int64_t L, const int64_t* h_lengths) {
    std::vector<long long> len(B, (long long)L);
    if (h_lengths) for (int b = 0; b < B; ++b) len[b] = h_lengths[b];
    return len;
}

extern "C" int fsn_metric_si_sdr_workspace(int32_t B, int64_t L, const int64_t* h_lengths, int64_t* bytes) {
    long long Lmax = 0;
    if (!bytes) return fail(FSN_EINVAL, "fsn_metric_si_sdr_workspace: null bytes");
    if (int rc = metric_check("fsn_metric_si_sdr_workspace", B, L, h_lengths, &Lmax)) return rc;
    SiSdrLaunch a{};
    *bytes = (int64_t)si_sdr_layout(a, nullptr, B, Lmax);
    return FSN_OK;
}

extern "C" int fsn_metric_si_sdr(const float* d_ref, const float* d_est, int32_t B, int64_t L, const int64_t* h_lengths, void* d_work,
                                 int64_t work_bytes, double* d_out, void* stream) {
    const char* fn = "fsn_metric_si_sdr";
    long long Lmax = 0;
    if (int rc = metric_check(fn, B, L, h_lengths, &Lmax)) return rc;
    SiSdrLaunch a{};
    if (int rc = metric_work_check(fn, d_ref, d_est, d_work, d_out, work_bytes, si_sdr_layout(a, nullptr, B, Lmax))) return rc;
    si_sdr_layout(a, d_work, B, Lmax);
    a.ref = d_ref; a.est = d_est; a.L = L; a.out = d_out;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const std::vector<long long> len = metric_lengths(B, L, h_lengths);
    CK(cudaMemcpyAsync(const_cast<long long*>(a.len), len.data(), len.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
    CK(launch_si_sdr(a, s));
    return FSN_OK;
}

extern "C" int fsn_metric_stoi_workspace(int32_t B, int64_t L, const int64_t* h_lengths, int32_t sr, int64_t* bytes) {
    const char* fn = "fsn_metric_stoi_workspace";
    long long Lmax = 0;
    if (!bytes) return fail(FSN_EINVAL, "%s: null bytes", fn);
    if (int rc = metric_check(fn, B, L, h_lengths, &Lmax)) return rc;
    if (int rc = metric_sr_check(fn, sr)) return rc;
    StoiLaunch a{};
    stoi_geometry(sr, a);
    *bytes = (int64_t)stoi_layout(a, nullptr, B, Lmax);
    return FSN_OK;
}

extern "C" int fsn_metric_stoi(const float* d_ref, const float* d_est, int32_t B, int64_t L, const int64_t* h_lengths, int32_t sr,
                               void* d_work, int64_t work_bytes, double* d_out, void* stream) {
    const char* fn = "fsn_metric_stoi";
    long long Lmax = 0;
    if (int rc = metric_check(fn, B, L, h_lengths, &Lmax)) return rc;
    if (int rc = metric_sr_check(fn, sr)) return rc;
    StoiLaunch a{};
    stoi_geometry(sr, a);
    if (int rc = metric_work_check(fn, d_ref, d_est, d_work, d_out, work_bytes, stoi_layout(a, nullptr, B, Lmax))) return rc;
    stoi_layout(a, d_work, B, Lmax);
    a.x = d_ref; a.y = d_est; a.L = L; a.out = d_out;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const std::vector<long long> len = metric_lengths(B, L, h_lengths);
    std::vector<float> tab;
    stoi_tables(a, tab);
    CK(cudaMemcpyAsync(const_cast<long long*>(a.len), len.data(), len.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(const_cast<float2*>(a.tw), tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice, s));
    CK(launch_stoi(a, s));
    return FSN_OK;
}

extern "C" int fsn_metric_sdr_workspace(int32_t B, int64_t L, const int64_t* h_lengths, int64_t* bytes) {
    const char* fn = "fsn_metric_sdr_workspace";
    long long Lmax = 0;
    if (!bytes) return fail(FSN_EINVAL, "%s: null bytes", fn);
    if (int rc = metric_check(fn, B, L, h_lengths, &Lmax)) return rc;
    SdrLaunch a{};
    *bytes = (int64_t)sdr_layout(a, nullptr, B, Lmax);
    return FSN_OK;
}

extern "C" int fsn_metric_sdr(const float* d_ref, const float* d_est, int32_t B, int64_t L, const int64_t* h_lengths, void* d_work,
                              int64_t work_bytes, double* d_out, void* stream) {
    const char* fn = "fsn_metric_sdr";
    long long Lmax = 0;
    if (int rc = metric_check(fn, B, L, h_lengths, &Lmax)) return rc;
    SdrLaunch a{};
    if (int rc = metric_work_check(fn, d_ref, d_est, d_work, d_out, work_bytes, sdr_layout(a, nullptr, B, Lmax))) return rc;
    sdr_layout(a, d_work, B, Lmax);
    a.ref = d_ref; a.est = d_est; a.L = L; a.out = d_out;
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const std::vector<long long> len = metric_lengths(B, L, h_lengths);
    CK(cudaMemcpyAsync(const_cast<long long*>(a.len), len.data(), len.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
    CK(launch_sdr(a, s));
    return FSN_OK;
}
