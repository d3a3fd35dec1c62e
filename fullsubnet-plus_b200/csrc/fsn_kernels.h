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
// dynamic shared memory of tsse_norm_kernel in bytes at F bins: 5 F + F / 2 + 8 floats (46 KB at F = 2048)
size_t tsse_norm_smem(int F);
// The front end's launchers return null, or the name of the kernel whose launch (or cudaFuncSetAttribute) failed with *err
const char* launch_tsse_norm(const TsseLaunch& a, cudaStream_t s, cudaError_t* err);
// norm types other than offline_laplace_norm (reference base_model.py:227-316): y[nbranch, B, F, Tp] = norm(pad(x)).  frames: scratch
// [nbranch, B, 4, Tp] floats (per-frame sums, sums of squares, scale and shift), input_norm_frames_bytes; the forward lends it the
// lane's full-band output buffer, which is written only after the input norm has run
struct NormLaunch { const float* x[3]; float* y; int nbranch, B, F, T, Tp, type; const int* tlen; float* frames; };   // tlen: as TsseLaunch
inline size_t input_norm_frames_bytes(int nbranch, int B, int Tp) { return (size_t)nbranch * B * 4 * Tp * sizeof(float); }
cudaError_t launch_input_norm(const NormLaunch& a, cudaStream_t s);

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
    // test hook (fsn_model_sb_forward): the sub-band input itself, [B*F, I, Tp] fp32; launch_sb_pack then writes it into the images
    // unnormalised (frames t0 .. t0 + Tw - 1 of every row of the padded tile pairs; rows >= B*F, columns >= I and frames past tlen zero)
    const float* raw;
};
const char* launch_sb_stats(const SbPackLaunch& a, cudaStream_t s, cudaError_t* err);
const char* launch_sb_pack(const SbPackLaunch& a, cudaStream_t s, cudaError_t* err);
// a wide sub-band input (64 < I <= 128): the same values as plain fp16 rows of 128 halves, columns >= I zero.  time_major = false:
// the A operand of layer 0's input-projection GEMM, row (tile * Tw + t - t0) * 128 + r (LstmTc5rLaunch::hseq's order); true: the
// generic kernel's plain input [Tw, ntiles * 128, 128] (LstmMmaLaunch::xplain, rows_pad = ntiles * 128)
const char* launch_sb_pack_wide(const SbPackLaunch& a, bool time_major, cudaStream_t s, cudaError_t* err);
// the same normalised values as launch_sb_pack, written to a.xtm / a.amax instead of the fp16 images
const char* launch_sb_pack_tm(const SbPackLaunch& a, cudaStream_t s, cudaError_t* err);
// time-major [Z*Tp, ld] -> [Z, C, Tp] (test hook of the sub-band TCN input)
void launch_tm_to_fm(const float* x, int ld, float* y, int Z, int C, int Tp, cudaStream_t s);
// [B, F, T] fp32 (+ zero look-ahead pad) -> zero-padded copy [B, F, P]; with tlen [B], sample b's input ends at tlen[b] - la
void launch_pad_copy(const float* x, float* y, int B, int F, int T, int P, const int* tlen, int la, cudaStream_t s);
// full-band LSTM input: [B, F, P] fp32 -> [Tp, Bpad, Ipad] fp16 (rows >= B and k >= F zero)
void launch_fb_pack(const float* x, __half* y, int B, int F, int Tp, int P, int rows_pad, int Ipad, cudaStream_t s);

void launch_apply_cirm(const float* crm, const float2* noisy, float2* enh, int B, int F, int T, cudaStream_t s);
// same with the noisy spectrum as two planes [B, F, T] (the model's own real / imag inputs); with tlen [B], frames
// t >= tlen[b] - la are written as zero without reading the planes; with lam [B] (device, or null: no limit) each clip's mask gets
// its attenuation floor (limit_mask, DESIGN.md §3.18)
void launch_apply_cirm_planar(const float* crm, const float* nreal, const float* nimag, float2* enh, int B, int F, int T, const int* tlen,
                              int la, cudaStream_t s, const float* lam = nullptr);

// streaming step kernels (k_front.cu): K frames of the cumulative norms with running sums carried in global memory, frame after
// frame.  slot: null (every slot is at frame n), or [B] per-slot frame counts of the slot calls, -1 = held: a held slot's frames are
// not read, its sums are untouched and its outputs are zero.  x [B, F, K] -> y [B, F, P] (frames at columns 0 .. K - 1)
// kf: null, or [B] per-slot frame counts (slot calls): a stepping slot runs frames 0 .. kf - 1 only, the rest of its row is zero
struct StreamNormLaunch { const float* x; float* y; double* cum; int B, F, K, P, n, type; const int* slot; const int* kf; };
void launch_stream_norm(const StreamNormLaunch& a, cudaStream_t s);
// frames k0 .. k0 + Kw - 1 of mag [B, F, K] and fb [B, F, Pfb] -> images [tile, Kw, 128 rows, 64 halves].  idx null: row b F + f,
// held rows zero.  idx [B]: row (idx[b] - j0) F + f for the sessions j0 .. j0 + nsess - 1 of a sub-batch, nothing for any other slot.
// K = 1 with idx null runs a one-frame kernel with the same arithmetic in fewer registers (faster at 1024 slots)
struct StreamPackLaunch {
    const float* mag; const float* fb; int Pfb; double* cum; __half* ximg; int B, F, K, Ns, Nf, n, type, k0, Kw; const int* slot;
    const int* idx; int j0, nsess;
    const int* kf;            // null, or [B]: frames k >= kf[b] of a stepping slot are zero images and leave its sums untouched
};
void launch_stream_pack(const StreamPackLaunch& a, cudaStream_t s);
// a wide input (64 < I <= 128) as plain fp16 rows of 128 halves: with idx, row (tile * Kw + k - k0) * 128 + r of the compact rows (layer
// 0's input-projection GEMM); without, time-major [K, ntiles * 128, 128] for the generic kernel (ntiles = ceil(B F / 128))
void launch_stream_pack_wide(const StreamPackLaunch& a, cudaStream_t s);
// compact masks src [nsess, 2, F, K] of the sessions j0 .. j0 + nsess - 1 -> dst [B, 2, F, K] at their slots (idx[b] - j0), leading
// columns with slot[b] + k < la zero; zero_held: also zero the rows of held slots
// src has Ks <= K columns; dst columns k >= Ks of the sub-batch's slots are zero
struct StreamChunkScatterLaunch { const float* src; float* dst; const int* slot; const int* idx; int j0, nsess, B, F, K, Ks, la, zero_held; };
void launch_stream_chunk_scatter(const StreamChunkScatterLaunch& a, cudaStream_t s);

// ---- k_stream_state.cu: save / load of streaming sessions (fsn_stream_save_slots, fsn_stream_load_slots), START reset ----------
// One segment of the payload: the handle's rows of one state buffer.  Slot b's rows of layer l start at base + l layer_stride +
// b slot_bytes; in the payload of session i they lie at i stride + pay_off + l slot_bytes.  vec: 16 or 8, the access width every
// handle-side offset is a multiple of.
struct StreamStateSeg { char* base; size_t layer_stride, slot_bytes, pay_off; int L, vec; };
// A work item: bytes [begin, end) of one layer's rows of one segment (multiples of 16, except at the end of an 8-byte segment)
struct StreamStateItem { int seg, layer; uint32_t begin, end; };
constexpr int STREAM_STATE_MAX_SEG = 9, STREAM_STATE_MAX_ITEMS = 96;
enum { STREAM_STATE_LOAD, STREAM_STATE_SAVE, STREAM_STATE_ZERO };
struct StreamStateLaunch {
    StreamStateSeg seg[STREAM_STATE_MAX_SEG]; int nseg;
    StreamStateItem item[STREAM_STATE_MAX_ITEMS]; int nitem;
    const int* slots; int n;  // [n] device: the handle slot of session i
    char* payload; size_t stride;
    int dir;                  // LOAD: payload -> handle (scatter); SAVE: handle -> payload (gather); ZERO: zeros -> handle, no payload
};
int launch_stream_state(const StreamStateLaunch& a, cudaStream_t s);   // returns 0 or cudaError
// The sub-band h / c of n sessions (slots sess[0 .. n - 1]) between the handle ([L, rows_alloc, H] rows b F + f, fp16 h, fp32 c) and
// the layer-wise recurrence's carry (LstmTc5rLaunch::hstate rows j F + f, h_layer halves per layer; cstate in its CTA-private
// order, c_layer floats per layer).  out = 0: handle -> carry; 1: carry -> handle
struct StreamSbCarryLaunch {
    __half* h_handle; float* c_handle; int rows_alloc;
    __half* h_carry; size_t h_layer; float* c_carry; size_t c_layer;
    const int* sess; int n, F, H, L, out;
};
void launch_stream_sb_carry(const StreamSbCarryLaunch& a, cudaStream_t s);

// ---- k_stream_audio.cu: audio in and out of the streaming audio calls (fsn_stream_step_audio_slots, _chunk, _samples) ---------
// Up to K hops per slot (DESIGN.md §3.10, §3.14, §3.19; the per-hop call is K = 1): slot b's active ticks are the first na[b] of the
// call, at slot ticks k0[b] + i; with start[b] its tick 0 is a START (store hop 0, no model frame).  Its first nstore[b] active ticks
// store the row's hops 0 .. nstore - 1.  Every other active tick is a model frame: model column c = i - start, frame
// j = k0 + start - 1 + c, its magnitude and mask at column c of the model's planes [B, F, Km] and [B, 2, F, Km].
struct StreamAudioLaunch {
    const int *k0, *na, *start, *nstore, *hops;   // [B] each; hops: the session's K after this call (0 = not flushed)
    const int *r0, *r;        // [B] each, or null (no partial hops: both 0): samples pending before the call; the trailing partial
                              // hop after it (the next pending count, or at a FLUSH the partial end: L = K hop + r)
    const float* samples;     // [B, S] this call's samples of each row (the hop calls: S = K hop)
    float* out;               // [B, So] output hops, then a FLUSH's last r samples, at the front of each row, zero after them
    int S, So;                // row strides of samples and out (the hop calls: K hop; the sample call: So = S + (la + 3) hop)
    int zero_out;             // the analysis zeroes the output rows (a call with no tick runs no synthesis)
    float* hist;              // [B, 3, hop] history ring: hop q at q % 3
    float2* spec;             // [B, la + 1, F] noisy spectrum ring: frame j at j % (la + 1)
    float* tail;              // [B, hop] second half of the last synthesised windowed frame
    float2* sspec;            // [B, K, F] scratch: the spectrum of each model column's frame
    float* mag;               // model input [B, F, Km]
    const float* mask;        // model output [B, 2, F, Km]
    float* umask;             // [B, 2, F, K] the caller's masks by tick, or null
    const float* window;      // [n_fft] periodic Hann
    const float2* twiddle;    // [n_fft / 2 + 1] exp(-2 pi i k / n_fft)
    const float* inv_env;     // [hop] 1 / (w^2(i) + w^2(i + hop))
    const float* inv_last;    // [hop] 1 / w^2(i + hop)
    int B, K, Km, n_fft, la;  // Km: model columns, the largest frame count of the call; n_fft: power of two, 64 .. 1024
    const float* lam;         // optional [B] attenuation floor of each slot (limit_mask, DESIGN.md §3.18); null: the unlimited synthesis
};
void launch_stream_stft(const StreamAudioLaunch& a, cudaStream_t s);
void launch_stream_istft(const StreamAudioLaunch& a, cudaStream_t s);

// ---- k_audio.cu: audio in and out of the offline forward (fsn_model_enhance_audio), and the tables of both audio paths -------
struct AudioLaunch {
    const float* wave;        // [B, L] input rows (analysis; samples past a clip's length are never read)
    float* out;               // [B, L] output rows (synthesis; samples past a clip's length are written as zero)
    long long L;              // row stride of wave and out
    const int* len;           // [B] samples per clip (device), or null: every clip is Lall samples
    int Lall;
    int B, T, n_fft;          // T: frames of the planes (the batch's longest clip); n_fft: power of two, 64 .. 1024
    float* planes;            // [3][B][F][T] mag, real, imag: analysis output, the forward's input
    const float2* enh;        // [B, F, T] enhanced spectrum: synthesis input, the forward's output
    const float* window; const float2* twiddle; const float* inv_env; const float* inv_last;   // audio_tables
};
// Both put the batch on gridDim.y (B <= 65535, kept by plan_forward); they return the launch's error
cudaError_t launch_audio_stft(const AudioLaunch& a, cudaStream_t s);
cudaError_t launch_audio_istft(const AudioLaunch& a, cudaStream_t s);
// Tables of one n_fft, computed in double, in one array: periodic Hann window w [n_fft] | twiddles exp(-2 pi i k / n_fft) for
// k = 0 .. hop (hop + 1 float2) | 1 / (w^2(i) + w^2(i + hop)) for i < hop | 1 / w^2(i + hop) for i < hop (the last L mod hop samples of a
// clip, which one frame covers)
void audio_tables(int n_fft, std::vector<float>& tab);
struct AudioTables { const float* window; const float2* twiddle; const float* inv_env; const float* inv_last; };
inline AudioTables audio_table_ptrs(const float* tab, int n_fft) {
    const int H = n_fft / 2;
    return {tab, reinterpret_cast<const float2*>(tab + n_fft), tab + n_fft + 2 * (H + 1), tab + n_fft + 2 * (H + 1) + H};
}

// ---- k_chunk_stream.cu: overlapped-chunk sessions around the offline audio forward (fsn_chunk_stream_step, DESIGN.md §3.16) -------
// The per-slot plan, CHUNK_PLAN_FIELDS int32 per slot: the chunks this call completes (nc, at batch rows row0 .. row0 + nc - 1), the
// slot's samples relative to its next chunk's start a0 = k0 H (ring below rel0, the call's row in [rel0, rel1), zero below lo and
// from rel1 on), the ring position of a0 (phase) and the samples emitted (nout).  lo = 0 exactly when that next chunk is chunk 0.
enum { CP_NC, CP_ROW0, CP_REL0, CP_REL1, CP_LO, CP_PHASE, CP_NOUT, CHUNK_PLAN_FIELDS };
// Floats between two slots' tails: C / 2 rounded up to a multiple of 4, so that every slot's tail starts 16-byte aligned and the save /
// load copy (stream_state_copy_kernel) moves it in 16-byte or 8-byte accesses whatever the parity of C / 2 (DESIGN.md §3.17)
__host__ __device__ inline int chunk_tail_stride(int C) { return ((C >> 1) + 3) & ~3; }
struct ChunkStreamLaunch {
    const int* plan;          // [B, CHUNK_PLAN_FIELDS] device
    const float* samples;     // [B, S] this call's samples at the front of each row
    float* ring;              // [B, C + P] the slot's last C + P samples, sample p at p mod (C + P)
    float* rows;              // [n, P + C] the completed chunks' input rows (gather output, the forward's input)
    const float* enh;         // [n, P + C] the forward's output rows
    float* tail;              // [B, chunk_tail_stride(C)] the windowed second half of the slot's last enhanced chunk (C / 2 floats)
    const float* window;      // [C] periodic Hann window
    float* out;               // [B, S + C] emitted samples at the front of each row, zero after them
    int B, S, C, P;
};
void launch_chunk_gather(const ChunkStreamLaunch& a, cudaStream_t s);
void launch_chunk_crossfade(const ChunkStreamLaunch& a, cudaStream_t s);

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
    // optional (streaming slot and chunk calls): per-slot frame counts, -1 = held; row r belongs to slot r / slot_rows.  A held row
    // writes neither cstate nor hstate.  The fused-FC output at step t of a held slot, or of a slot whose frame count + t is below
    // slot_la (still filling its look-ahead), is zero
    const int* slot; int slot_rows, slot_la;
    // optional with slot: [B] per-slot frame counts; a stepping row holds at every step t >= kf (keeps c, carries its h forward,
    // output zero)
    const int* kf;
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
    const int* slot;          // optional (streaming slot call, Tp = 1): [rows] per-slot frame counts, -1 = held: the row keeps its
                              // cell state and carries its previous h into this step's exchange-buffer parity
    const int* kf;            // optional with slot: [rows] per-slot frame counts; a stepping row holds as above at steps t >= kf
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
                              // of the recurrence, with W_ih as one extra k-block in front of every chunk of the stream.  A wide input
                              // (64 < Isb <= 128) is rows of 128 halves in hseq's order instead: the host projects it with the GEMM
                              // (fsn_api.cu, sb_layers) and the kernel gets ximg = null
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
    const float* lam;         // with enh: optional [B] attenuation floor of each clip (limit_mask, DESIGN.md §3.18); null: no limit, and
                              // the launch runs the kernel instantiated without it
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

// EPI5_GLN_HEAD_LIM: EPI5_GLN_HEAD writing the enhanced spectrum with each clip's attenuation floor lam[z / Fg] (a sibling instantiation,
// so the unlimited head is unchanged)
enum { EPI5_PRELU_STATS = 1, EPI5_GLN_RES = 2, EPI5_OUT = 3, EPI5_F16OUT = 4, EPI5_GLN_HEAD = 5, EPI5_GLN_HEAD_LIM = 6 };
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
    const float* lam;                          // GLN_HEAD_LIM: [B] attenuation floor of each clip (limit_mask, DESIGN.md §3.18)
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

// ---- k_metrics.cu (fsn_metric_si_sdr, fsn_metric_stoi, fsn_metric_sdr) -----------------------------------------------------------------------
struct SiSdrLaunch {
    const float* ref; const float* est; long long L; int B;    // [B, L] rows, clip b = the first len[b] samples of its row
    const long long* len;                                      // [B], on the device
    int nchunk; double2* part; double* alpha; double* out;     // partials [B, nchunk], alpha [B], scores [B]
};
// Sets a's workspace pointers (ws = nullptr: offsets from 0) for B clips of at most Lmax samples; returns the bytes.
size_t si_sdr_layout(SiSdrLaunch& a, void* ws, int B, long long Lmax);
cudaError_t launch_si_sdr(const SiSdrLaunch& a, cudaStream_t s);

struct StoiLaunch {
    const float* x; const float* y; long long L; int B;        // reference and estimate rows
    const long long* len;                                      // [B], on the device
    int up, down, half, ntap;                                  // 10 kHz = sr up / down; filter taps 2 half + 1, ntap per phase
    const float* poly; const float* win; const float2* tw;     // stoi_tables, in the workspace
    long long F; long long P;                                  // frame stride (the longest clip's frames), partial stride
    double* energy; int* kept; int* nkept; double* env; double* part; double* out;
};
void stoi_geometry(int sr, StoiLaunch& a);                         // up, down, half, ntap of sr
size_t stoi_table_floats(const StoiLaunch& a);
void stoi_tables(const StoiLaunch& a, std::vector<float>& tab);   // what the workspace's table segment holds
size_t stoi_layout(StoiLaunch& a, void* ws, int B, long long Lmax);  // as si_sdr_layout, after stoi_geometry
cudaError_t launch_stoi(const StoiLaunch& a, cudaStream_t s);

struct SdrLaunch {
    const float* ref; const float* est; long long L; int B;    // as SiSdrLaunch
    const long long* len;                                      // [B], on the device
    long long nct, npt;                                        // correlation / projection tiles of the longest clip (partial strides)
    double* corr;                                              // per-tile partials [B, nct, 1024]: R[0 .. 511], D[0 .. 511]
    double* rd;                                                // their per-clip sums [B, 1024]
    double* coef;                                              // distortion filter c [B, 512] (NaN where the solve stopped)
    double2* part; double* out;                                // projection partials [B, npt] (sum P^2, sum (e' - P)^2), scores [B]
};
size_t sdr_layout(SdrLaunch& a, void* ws, int B, long long Lmax);  // as si_sdr_layout
cudaError_t launch_sdr(const SdrLaunch& a, cudaStream_t s);

}  // namespace fsn
