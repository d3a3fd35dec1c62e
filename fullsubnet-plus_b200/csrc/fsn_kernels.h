// Internal launch prototypes (host side) of the fsnplus_b200 kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>

namespace fsn {

// Launch a kernel of the front-end chain; when chained launches are on for the calling thread (fsn_chain_launch_set, decided per
// forward from the FSN_PDL knob read at model creation and the batch size) it gets the programmatic-stream-serialization attribute --
// every kernel launched through this helper executes pdl_wait() (fsn_common.cuh).
bool fsn_chain_launch_enabled();
void fsn_chain_launch_set(bool on);
template <typename... KArgs, typename... Args>
inline cudaError_t launch_chain(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at{};
    at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at.val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = &at; cfg.numAttrs = fsn_chain_launch_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ---- k_front.cu ------------------------------------------------------------------------------
struct TsseParams {            // device pointers, one set per branch
    const float* conv_w[3];    // [C, k]
    const float* conv_b[3];    // [C]
    const float* cat_w;        // [3]
    const float* cat_b;        // [1]
    const float* fc1_w;        // [C/2, C]
    const float* fc1_b;        // [C/2]
    const float* fc2_w;        // [C, C/2]
    const float* fc2_b;        // [C]
    const float* eca_w;        // [3]   ChannelECAlayer.conv.weight
};
struct TsseLaunch {
    const float* x[3];         // per branch input [B, F, T]
    TsseParams p[3];
    int nbranch, B, F, T, Tp, P;   // Tp = T + look_ahead, P = row pitch of the output
    int ksz[3];
    int attention;             // 0: norm only (fullsubnet.Model), 1 + FSN_ATTN_*: norm + that channel attention
    float* out;                // [nbranch, B, F, P]
    float* scale;              // [nbranch, B, F] per-row scale handed from the statistics kernel to the apply kernel
    float* amax;               // optional [nbranch, B]: max |out| of the (sample, branch) -- the fp16 store scale of the first TCN block (fp16_store_scale)
    float* rows;               // [nbranch, B, F, 35] row statistics handed from tsse_rowstats_kernel to the gate kernel (tsse_row_floats())
    int prenorm;               // 1: input is already normalised (input_norm_kernel), skip the utterance-mean division
    int sub;                   // subband_num (ECA, mag branch only): channels are groups of `sub` reflect-padded bins (fullsubnet_plus.py:146-153)
    float* out_tm; int Cp;     // optional time-major copy [(branch, b, t), Cp] for the TCN GEMMs (pad columns stay zero)
    const int* tlen;           // optional [nbranch, B] per-sample extent frames[b] + look_ahead (clip_len); null: every sample spans Tp
};
inline size_t tsse_row_floats() { return 3 + 2 * 16; }
void launch_tsse_norm(const TsseLaunch& a, cudaStream_t s);
// norm types other than offline_laplace_norm (reference base_model.py:227-316): y[nbranch, B, F, Tp] = norm(pad(x))
struct NormLaunch { const float* x[3]; float* y; int nbranch, B, F, T, Tp, type; const int* tlen; };   // tlen: as TsseLaunch
void launch_input_norm(const NormLaunch& a, cudaStream_t s);

struct ConvLaunch {          // Y[z] = act(W X[z] + b): output Linear of the full-band LSTM (fullsubnet.Model)
    const float* X;          // [Z, K, P]
    const float* W;          // [M, K]
    const float* bias;       // [M]
    float* Y;                // [Z, M, P]
    int Z, M, K, Tp, P;
    int act;                 // FSN_ACT_*
};
void launch_conv1x1(const ConvLaunch& a, cudaStream_t s);

struct SbPackLaunch {
    const float* win;        // [B, F, Pw] window source (post-attention mag branch, or raw padded mag)
    int Pw;
    const float* fb[3];      // [B, F, P] full-band outputs (nfb of them)
    int nfb, P;
    int B, F, Tp, Ns, Nf;    // neighbours
    float* mu;               // [B] utterance mean of the concatenated sub-band input
    float* sigma;            // [B] unbiased std (offline_gaussian_norm only)
    float* rowsum;           // [B, 1 + nfb, F, 2] scratch: row sums and sums of squares
    int norm_type;           // FSN_NORM_*
    __half* ximg;            // [ntiles, Tw, 128 rows, 64 halves] SWIZZLE_128B images of frames t0 .. t0 + Tw - 1
    int ntiles;
    int t0, Tw;              // frame window of the images (t0 = 0, Tw = Tp: the whole clip); Tw is a multiple of 32 except in the last window
    double* cum;             // cumulative norms, windowed: running (sum, sum of squares) [B*F][2] at the window's end, reloaded when t0 > 0
    float* xtm;              // sub-band TCN input: fp32 time-major [B*Fc*Tp, 64], row (b*Fc + f - f0)*Tp + t, columns >= I zero
    float* amax;             // [B*Fc] max |x| of every sequence of xtm (zeroed by the launcher): block 0's fp16 store scale
    const int* tlen;         // optional [B] per-sample extent in frames of Tp (rows past it are written as zero); null: Tp
    // xtm only: the bins f0 .. f0 + Fc - 1 of every sample (a chunk of the sub-band TCN; f0 = 0, Fc = F: all of them).  Sequence
    // (b, f) is row b * Fc + (f - f0) of xtm and amax; neighbours are still read from the absolute bins, reflected over the whole F
    int f0, Fc;
};
void launch_sb_stats(const SbPackLaunch& a, cudaStream_t s);
void launch_sb_pack(const SbPackLaunch& a, cudaStream_t s);
// the same normalised values as launch_sb_pack, written to a.xtm / a.amax instead of the fp16 images
void launch_sb_pack_tm(const SbPackLaunch& a, cudaStream_t s);
// time-major [Z*Tp, ld] -> [Z, C, Tp] (test hook of the sub-band TCN input)
void launch_tm_to_fm(const float* x, int ld, float* y, int Z, int C, int Tp, cudaStream_t s);
// [B, F, T] fp32 (+ zero look-ahead pad) -> zero-padded copy [B, F, P]; with tlen [B], sample b's input ends at tlen[b] - la
void launch_pad_copy(const float* x, float* y, int B, int F, int T, int P, const int* tlen, int la, cudaStream_t s);
// full-band LSTM input: [B, F, P] fp32 -> [Tp, Bpad, Ipad] fp16 (rows >= B and k >= F zero)
void launch_fb_pack(const float* x, __half* y, int B, int F, int Tp, int P, int rows_pad, int Ipad, cudaStream_t s);

void launch_apply_cirm(const float* crm, const float2* noisy, float2* enh, int B, int F, int T, cudaStream_t s);
// same with the noisy spectrum as two planes [B, F, T] (the model's own real / imag inputs); with tlen [B], frames
// t >= tlen[b] - la are written as zero without reading the planes
void launch_apply_cirm_planar(const float* crm, const float* nreal, const float* nimag, float2* enh, int B, int F, int T, const int* tlen,
                              int la, cudaStream_t s);

// streaming step kernels (k_front.cu): one frame of the cumulative norms with running sums carried in global memory
struct StreamNormLaunch { const float* x; float* y; double* cum; int B, F, P, n, type; };       // x [B,F] -> y [B,F,P] (t = 0)
void launch_stream_norm(const StreamNormLaunch& a, cudaStream_t s);
struct StreamPackLaunch { const float* mag; const float* fb; int Pfb; double* cum; __half* ximg; int B, F, Ns, Nf, n, type; };
void launch_stream_pack(const StreamPackLaunch& a, cudaStream_t s);

// ---- k_lstm_mma.cu ---------------------------------------------------------------------------
struct LstmMmaWeights {       // device, produced by pack (fsn_api.cu)
    const uint4* wfrag[4];    // per layer: [H/8 groups][K/16][32 lanes][2 x uint4]
    const float* bias[4];     // per layer [4H] (b_ih + b_hh), original i,f,g,o order
    const float* fc_w;        // [O, H]
    const float* fc_b;        // [O]
};
struct LstmMmaLaunch {
    LstmMmaWeights w;
    int L, H, I, Ipad;        // Ipad: multiple of 16
    int rows, Tp;
    // input: either SW128 images (img != null; Ipad == 64) or plain [Tp, rows_pad, Ipad]
    const __half* img; int ntiles;
    const __half* xplain; int rows_pad;
    float* cstate;            // [L, rows_alloc, H] scratch (zeroed by the launcher)
    int rows_alloc;
    // output A (fused FC, O <= 8): out[b][o][f][t - la]  (row = b*F + f)
    float* out; int O, F, la, act;
    // output B: top-layer h as fp32 [rows, H, P]
    float* hseq; int P;
    int fast;
    int gru;                  // 1: pseudo-gate GRU cell (gru_cell), cstate carries h in fp32
    // streaming: hidden state carried across launches ([L, rows_alloc, H] fp16); resume = 1 continues from it
    __half* hstate; int resume;
    const int* tlen;          // optional [B] per-sample extent in frames of Tp: output frames t - la >= tlen[b] - la are written as zero
};
size_t lstm_mma_cstate_bytes(int L, int rows, int H, int* rows_alloc);
int launch_lstm_mma(const LstmMmaLaunch& a, cudaStream_t s);   // returns 0 or cudaError

// ---- k_lstm_ws.cu: weight-stationary persistent LSTM for <= 64 rows (full-band LSTM of fullsubnet.Model) ----------
struct LstmWsLaunch {
    const float* w_ih[4]; const float* w_hh[4]; const float* b_ih[4]; const float* b_hh[4];   // reference-layout fp32 parameters (device)
    int L, H, I, Ipad, rows, rows_pad, Tp;
    const __half* x;          // [Tp, rows_pad >= 64, Ipad]
    __half* hbuf;             // [L, 2, 64, H] exchange buffer (zeroed by the caller unless resume)
    float* cbuf;              // [L, 64, H] cell state carried across launches (streaming) or null
    unsigned int* barrier;    // grid barrier counter
    float* hseq; int P;       // top-layer h as fp32 [rows, H, P]
    int fast, resume, t0;     // t0: absolute index of the first step (exchange-buffer parity)
    int gru;                  // 1: pseudo-gate GRU cell, cbuf / cst carry h in fp32
};
bool lstm_ws_supported(int L, int H, int Ipad, int rows, int num_sms);
int launch_lstm_ws(const LstmWsLaunch& a, cudaStream_t s);

// ---- k_lstm_tc5r.cu: single-layer recurrent wgmma kernel, input projection time-batched by launch_gemm_f16 ------------------
struct LstmTc5rLaunch {
    const __half* wstream;    // [H/32 chunks][k-blocks] of 16 KB: W_hh (lstm_tc5r_pack_layer), or [W_ih | W_hh] with ximg (lstm_tc5_pack_first_layer)
    const float* bias;        // [4H] pre-scaled, chunk column order
    const float* fc_w;        // [2][H]   (last layer)
    const float* fc_b;        // [2]
    int H, rows, Tp, ntiles;  // Tp: frames of the whole clip (T + look_ahead)
    // time window of this launch: steps t0 .. t0 + Tw - 1 (t0 = 0, Tw = Tp: the whole clip).  gin / ximg / hseq hold the window only
    // (window-local step index, stride Tw); the output index, the look-ahead test and tlen use the absolute step t0 + t
    int t0, Tw;
    const __half* gin;        // [ntiles_pad * Tw * 128, 4H] fp16 input projection X_l W_ih^T (lstm_tc5r_gin_order), or null with ximg
    const __half* ximg;       // first layer: [ntiles_pad, Tw, 128 rows, 64 halves] SW128 input images; the input projection is then part
                              // of the recurrence, with W_ih as one extra k-block in front of every chunk of the stream
    __half* hseq;             // [ntiles_pad * Tw * 128, H] fp16 output sequence (not the last layer)
    float* cstate;            // [2 ntiles_pad CTAs][H/32 chunks][4][128 threads] float4: c (GRU: h in fp32), read back at t0 > 0
    __half* hstate;           // windowed forwards: this layer's fp16 h [ntiles_pad * 128, H], loaded at entry when t0 > 0 (instead
                              // of h = 0) and stored at exit; null: h starts at zero and is not kept
    float* out; int F, la;    // last layer: mask [B, 2, F, Tp - la]
    int act;                  // FSN_ACT_* on the Linear output (last layer)
    int fast, gru, last;
    // fused post-processing (inferencer.py:152-157): when enh != null the last layer decompresses the cIRM and multiplies it with the
    // noisy spectrum (planes [B, F, T]) instead of writing the mask: enh [B, F, T] complex64 (interleaved re, im)
    const float* nreal; const float* nimag; float2* enh;
    const int* tlen;          // optional [B] per-sample extent in frames of Tp: output frames t - la >= tlen[b] - la are written as zero
};
bool lstm_tc5r_supported(int H, int O);
size_t lstm_tc5r_cstate_bytes(int ntiles, int H);
int64_t lstm_tc5r_weight_stream_bytes(int H);
int launch_lstm_tc5r(const LstmTc5rLaunch& a, cudaStream_t s);
void lstm_tc5r_pack_layer(int H, int Kin, int Kpad, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, bool gru,
                          std::vector<uint16_t>& stream, std::vector<uint16_t>& wih_perm, std::vector<float>& bias);
void lstm_tc5r_gin_order(int H, int Kpad, std::vector<uint16_t>& wih_perm);   // rows of wih_perm -> the Gin column order the kernel reads
void lstm_tc5_pack_first_layer(int I, int H, const float* w_ih0, const float* w_hh0, uint16_t* dst);   // k_lstm_tc5d.cu: [x | hidden] blocks per chunk

// ---- k_gemm_tc5.cu (TCN on wgmma, time-major activations; the input projection of the layer-wise LSTM path) ----------------
// C[M, N] = A[M, K] B[N, K]^T, fp16 in / fp32 accumulate / fp16 out (input projection of the layer-wise path).  tile_n: 0 or 256 =
// 128 x 256 tiles on CTA pairs where the shape allows (gemm_f16_pair_tiles), else 128 x 128; 128 = always 128 x 128 (FSN_GIN_GEMM)
struct GemmF16Launch { long long M; int N, K; __half* C; long long ldc; int tile_n; };
bool gemm_f16_supported(long long M, int N, int K);
bool gemm_f16_pair_tiles(const GemmF16Launch& g);
int launch_gemm_f16(const void* A, const void* B, const GemmF16Launch& a, int num_sms, cudaStream_t s);
int make_tmap_f16_2d(void* out_map /*128 B, 64 B aligned*/, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows);   // box = 64 halves x box_rows, SWIZZLE_128B

enum { EPI5_PRELU_STATS = 1, EPI5_GLN_RES = 2, EPI5_OUT = 3, EPI5_F16OUT = 4, EPI5_GLN_HEAD = 5 };
struct GemmTc5Launch {
    int Kp, NT, nstage, ntiles_n, Npad;        // K (multiple of 32; GLN_RES: fp16 operands, multiple of 64), N tile (64 or 128), ring depth, N tiles and padded N per branch
    int rows_per_branch, tiles_m, nbranch, Tp, B;
    int epi;
    const float* bias[3];                      // PRELU_STATS / OUT: conv bias; GLN_RES: s2 + conv bias
    const float* prelu[3];
    const float* s1[3];                        // GLN_RES: sum_c W'[n, c]
    double* stats_out;                         // [Z, 2]
    const double* stats_in; double count_row;  // GLN_RES / GLN_HEAD: elements per row in stats_in (a group's count: count_row x its frames)
    float* Y; int ldY;                         // GLN_RES: new residual stream (fp32)
    __half* Y16;                               // PRELU_STATS: the hidden activation, fp16 [rows, ldY], stored times fp16_store_scale(amax_in[z]); F16OUT: C
    const float* amax_in;                      // PRELU_STATS: [Z] max |x| of the block's input stream per sample
    float* amax_out;                           // GLN_RES: [Z] max |x| of the new stream per sample (atomicMax on the bit pattern; zeroed by the caller)
    const float* Xold; float* Xrelu;           // GLN_RES: residual input, optional relu'd copy
    float* out; int F, P, act;                 // OUT: [Z, F, P] (frequency-major); GLN_HEAD: mask [B, O, F, Tp - la]
    // GLN_HEAD (last block of the sub-band TCN, one 64-column N tile): GLN_RES's new stream x, then act(Linear(relu(x))) per row;
    // rows are (b * Fg + f - f0) * Tp + t.  With enh != null: decompress_cIRM x the noisy planes [B, F, Tp - la] into enh instead of the mask
    const float* fc_w; const float* fc_b;      // [O, 64] (columns >= I zero), [O]
    int O, la;
    const float* nreal; const float* nimag; float2* enh;
    // optional per-sample extent in frames of Tp, tlen[z / zdiv] for gLN group z (full band: z = branch * B + b, tlen [3][B], zdiv 1;
    // sub band: z = b * F + f, zdiv F).  Rows t >= that extent are written as zero and left out of every statistic and maximum
    const int* tlen; int zdiv;
    // GLN_HEAD: group z is bin f0 + z % Fg of clip z / Fg (a chunk of Fg bins from f0; Fg = F, f0 = 0: every bin).  F still sets the
    // layout of the mask, the enhanced spectrum and the noisy planes
    int Fg, f0;
};
int make_tmap_f32_2d(void* out_map /*128 B, 64 B aligned*/, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows);
int launch_gemm_tc5(const void* mapA, const void* mapB, GemmTc5Launch a, int num_sms, cudaStream_t s);
struct DwTmLaunch {
    const __half* X; __half* Y;                // [Z * Tp, C] hidden activations, fp16
    int Z, B, C, Tp, dilation;                 // Z groups (sequences), branch of group z = z / B
    int causal;                                // 1: taps t-2d, t-d, t (TCNBlock(causal=True)); 0: t-d, t, t+d
    const double* stats_in; double* stats_out;
    const float* amax;                         // [Z]: X holds the activation times fp16_store_scale(amax[z]); the statistics are unscaled
    const float* gamma[3]; const float* beta[3]; const float* w[3]; const float* b[3]; const float* prelu[3];
    const int* tlen; int zdiv;                 // as GemmTc5Launch: taps past the extent read zero, rows past it are written as zero
};
int launch_dwconv_tm(const DwTmLaunch& a, cudaStream_t s);

}  // namespace fsn
