/*
 * fsnplus_b200 -- C ABI of the H100-native (sm_90a) FullSubNet+/FullSubNet inference forward.
 *
 * This is the drop-in boundary for ONE path of RookieJunChen/FullSubNet-plus: the model forward
 *   speech_enhance/fullsubnet_plus/model/fullsubnet_plus.py:122-209  (FullSubNet_Plus.forward)
 *   speech_enhance/fullsubnet/model/fullsubnet.py:68-118             (Model.forward)
 * as called by the inferencer at
 *   speech_enhance/fullsubnet_plus/inferencer/inferencer.py:150 and :123.
 * The reference has no FFI of its own (it is pure Python/PyTorch); the Python mirror in
 * fullsubnet-plus_b200/fsnplus_b200/model.py binds these entry points with ctypes and exposes the
 * reference's nn.Module constructors / forward signatures / state_dict keys (INTEGRATION.md).
 *
 * Conventions: plain C types only; every pointer named d_* is a CUDA device pointer, h_* a host
 * pointer; `stream` is a cudaStream_t passed as void* (NULL = legacy default stream); all entry points
 * return 0 on success or a negative FSN_E* code, with a message available from fsn_last_error().
 * There is no CPU fallback: without a CUDA device every compute entry point fails with FSN_ECUDA.
 */
#ifndef FSNPLUS_B200_H_
#define FSNPLUS_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FSN_OK 0
#define FSN_EINVAL (-1)  /* bad argument / unsupported configuration (the reference raises/asserts) */
#define FSN_ECUDA (-2)   /* CUDA runtime error (including "no device")                              */
#define FSN_ESTATE (-3)  /* call order error (e.g. forward before finalize, missing parameter)      */

/* model_kind */
#define FSN_KIND_PLUS 0 /* fullsubnet_plus.model.fullsubnet_plus.FullSubNet_Plus (fullsubnet_plus.py:16) */
#define FSN_KIND_FSN 1  /* fullsubnet.model.fullsubnet.Model                      (fullsubnet.py:12)      */

/* activations: audio_zen/model/module/sequence_model.py:84-93 */
#define FSN_ACT_NONE 0
#define FSN_ACT_RELU 1
#define FSN_ACT_TANH 2
#define FSN_ACT_RELU6 3

/* norm_type: audio_zen/model/base_model.py:318-330 (norm_wrapper) */
#define FSN_NORM_OFFLINE_LAPLACE 0
#define FSN_NORM_CUMULATIVE_LAPLACE 1
#define FSN_NORM_OFFLINE_GAUSSIAN 2
#define FSN_NORM_CUMULATIVE_LAYER 3

/* channel_attention_model: fullsubnet_plus.py:52-70 (0 keeps a zero-initialised config on the inference.toml default) */
#define FSN_ATTN_TSSE 0    /* ChannelTimeSenseSELayer  attention_model.py:43-104  */
#define FSN_ATTN_SE 1      /* ChannelSELayer           attention_model.py:6-40    */
#define FSN_ATTN_CBAM 2    /* ChannelCBAMLayer         attention_model.py:296-334 */
#define FSN_ATTN_ECA 3     /* ChannelECAlayer          attention_model.py:337-359 */

/* sequence_model of the recurrent modules: sequence_model.py:31-46 */
#define FSN_RNN_LSTM 0
#define FSN_RNN_GRU 1      /* runs on the LSTM kernels as pseudo-gates (r, z, n_x, n_h) with a GRU cell */

/* lstm_impl */
#define FSN_LSTM_AUTO 0
#define FSN_LSTM_MMA 1     /* generic mma.sync kernel (any hidden size / layer count)               */
#define FSN_LSTM_TCGEN05 2 /* tensor-core path (historical name): layer-wise wgmma kernels, hidden % 64 == 0 and <= 512, input <= 64, output_size 2 */
#define FSN_LSTM_TCN 3     /* reported by fsn_model_last_lstm_impl only: the sub-band model is the TCN (fsn_config.sb_tcn)   */

typedef struct fsn_config {
    int32_t model_kind;
    int32_t num_freqs;        /* F                                   (config/inference.toml:33) */
    int32_t look_ahead;       /*                                      (:34)                      */
    int32_t sb_num_neighbors; /*                                      (:31)                      */
    int32_t fb_num_neighbors; /*                                      (:32)                      */
    int32_t fb_hidden;        /* fb_model_hidden_size (LSTM full band; ignored by the TCN)       */
    int32_t sb_hidden;        /* sb_model_hidden_size                 (:40)                      */
    int32_t num_layers;       /* 2 in the reference (fullsubnet_plus.py:76,106); additive knob   */
    int32_t output_size;      /* 2                                    (fullsubnet_plus.py:31)    */
    int32_t fb_act;           /* fb_output_activate_function          (:36)                      */
    int32_t sb_act;           /* sb_output_activate_function          (:37)                      */
    int32_t norm_type;        /*                                      (:42)                      */
    int32_t kersize[3];       /* TSSE kernel sizes                    (:44)                      */
    int32_t lstm_impl;        /* FSN_LSTM_*                                                      */
    int32_t fast_math;        /* 0: ex2/rcp gates; 1: tanh.approx gates (the Python mirror's default) */
    int32_t channel_attention;/* FSN_ATTN_*  channel_attention_model  (:38)                      */
    int32_t rnn_type;         /* FSN_RNN_*   sequence_model           (:35)                      */
    int32_t subband_num;      /* 0 or 1: off; > 1 needs FSN_ATTN_ECA (the only attention whose
                                 reference forward runs in that mode, fullsubnet_plus.py:146-163) */
    int32_t tcn_causal;       /* 0: TCNBlock(causal=False), what SequenceModel("TCN") builds (sequence_model.py:47-58);
                                 1: TCNBlock(causal=True) in the three full-band models (causal_conv.py:74-75,104-105):
                                 depth-wise taps t-2d, t-d, t instead of t-d, t, t+d.  Additive knob (SURVEY.md 8f rank 2) */
    int32_t sb_tcn;           /* 0: the sub-band model is the LSTM / GRU of rnn_type; 1: sequence_model = "TCN" of FullSubNet_Plus
                                 (fullsubnet_plus.py:102-110): 8 non-causal TCNBlock(Isb -> 512 -> Isb) + ReLU + Linear(Isb -> output_size).
                                 sb_hidden, num_layers, rnn_type, lstm_impl and fast_math do not apply to it */
} fsn_config;

typedef struct fsn_model fsn_model;

int fsn_version(void);
const char* fsn_last_error(void);

/* Replaces FullSubNet_Plus.__init__ / Model.__init__ (fullsubnet_plus.py:17-120, fullsubnet.py:13-66):
 * validates the configuration and creates an empty parameter store on the current CUDA device. */
int fsn_model_create(const fsn_config* cfg, fsn_model** out);
void fsn_model_destroy(fsn_model* m);

/* Replaces nn.Module.load_state_dict for this module tree (audio_zen/inferencer/base_inferencer.py:104):
 * `key` is the reference state_dict key, `h_data` float32 host data in the reference's shape. */
int fsn_model_set_param(fsn_model* m, const char* key, const float* h_data, int64_t numel);
/* Number of keys the configuration expects / i-th expected key and its element count. */
int fsn_model_num_params(const fsn_model* m);
int fsn_model_param_info(const fsn_model* m, int index, const char** key, int64_t* numel);
/* Re-orders / converts the parameters into the kernel layouts (fp16 gate-interleaved LSTM images, ...). */
int fsn_model_finalize(fsn_model* m);

/* Replaces FullSubNet_Plus.forward(noisy_mag, noisy_real, noisy_imag) (fullsubnet_plus.py:122-209) and
 * Model.forward(noisy_mag) (fullsubnet.py:68-118; pass d_real = d_imag = NULL).
 * Inputs: [B, 1, F, T] float32, contiguous, device.  Output: [B, output_size, F, T] float32, contiguous,
 * device, caller-owned.  Every sample is processed independently (the eval semantics of the reference
 * called with batch 1; the training-only drop_band of fullsubnet_plus.py:192-196 is never applied).  Because of that a
 * batch whose workspace would exceed FSN_WS_CAP_GB (default 24) is run as equal sub-batches on `stream`, with identical results. */
int fsn_model_forward(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                      float* d_out, void* stream);
/* The model call PLUS the two lines that follow it in the reference's inferencer methods (fullsubnet_plus/inferencer/inferencer.py:152-157,
 * audio_zen/acoustics/mask.py:60-63): decompress_cIRM and the complex multiplication with the noisy spectrum, fused into the epilogue
 * of the sub-band LSTM kernel -- the mask never goes to memory.  d_real / d_imag are the planes the model takes anyway (required
 * here also for fullsubnet.Model, which does not read them in its forward); d_enh: [B, F, T] complex64 (interleaved re, im) =
 * the argument of the inferencer's iSTFT. */
int fsn_model_forward_enhance(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                              float* d_enh, void* stream);
/* Ragged batches: fsn_model_forward / fsn_model_forward_enhance for clips of different lengths stored in one [B, 1, F, T] batch.
 * h_frames: HOST array of B frame counts, 1 <= h_frames[b] <= T (with the TSSE attention also h_frames[b] + look_ahead >= every
 * kersize), else FSN_EINVAL naming the sample.  Sample b is its first h_frames[b] frames followed by the look_ahead zero frames of
 * the reference's right padding: every time reduction, norm and convolution tap of the forward stops at h_frames[b] + look_ahead.
 * Inputs at t >= h_frames[b] are never read (they may hold anything, NaN included); outputs there are exact zeros, and
 * out[b, ..., :h_frames[b]] equals the forward of that clip alone up to floating-point reordering.  h_frames may be reused as soon as
 * the call returns (the counts go to the device through pinned staging slots; no stream is synchronised).  h_frames == NULL, or
 * every count equal to T, runs the unragged forward unchanged. */
int fsn_model_forward_ragged(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                             const int32_t* h_frames, float* d_out, void* stream);
int fsn_model_forward_enhance_ragged(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                     const int32_t* h_frames, float* d_enh, void* stream);
/* Same call with HOST buffers (pinned or pageable): H2D copies, the forward and the D2H copy of the
 * mask are all enqueued on `stream` and the call returns after the result is in h_out. */
int fsn_model_forward_host(fsn_model* m, const float* h_mag, const float* h_real, const float* h_imag, int32_t B, int32_t T,
                           float* h_out, void* stream);

/* Pipelined variants for STREAMS OF BATCHES (the reference's inferencer loop, base_inferencer.py:133-160, issues one forward
 * after the other; the outputs of a batch are only needed when its files are written).  The forward is split at the one point
 * where it changes character: the full-band front end (norm, attention, TCN / full-band LSTM, sub-band statistics + packing) is
 * bandwidth/latency-bound and occupies the whole GPU for a short time, the sub-band LSTM is tensor-bound and occupies the SMs for
 * a long time.  Both entry points run the front end of batch i+1 on an internal stream, into the second of two
 * workspace lanes, WHILE the sub-band LSTM of batch i runs on another internal stream: the front end fills the idle SMs.
 *
 * fsn_model_submit: device buffers.  The inputs must be complete in `stream` order at the time of the call and stay untouched,
 * d_out unread, until fsn_model_wait(m, stream) has been called (it makes `stream` wait for every submitted batch; it does not
 * block the host) or fsn_model_sync_host(m) has returned.  A plain fsn_model_forward on any stream first waits for the pipeline.
 *
 * fsn_model_forward_host_async: pinned host buffers; additionally the H2D copy of batch i+1 and the D2H copy of batch i-1
 * overlap on two copy streams.  `stream` is ignored (host memory carries no stream order).  The host buffers must stay
 * untouched (h_out unread) until fsn_model_sync_host() returns. */
int fsn_model_submit(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                     float* d_out, void* stream);
int fsn_model_submit_enhance(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                             float* d_enh, void* stream);   /* pipelined fsn_model_forward_enhance */
int fsn_model_wait(fsn_model* m, void* stream);
/* Finer-grained completion for consumers that post-process batch i while batch i+1 runs: the workspace lane (0 / 1) the LAST
 * fsn_model_submit used, and a wait on the batch most recently submitted into one lane (valid until the next submit into it). */
int fsn_model_last_lane(const fsn_model* m);
int fsn_model_wait_lane(fsn_model* m, int32_t lane, void* stream);
int fsn_model_forward_host_async(fsn_model* m, const float* h_mag, const float* h_real, const float* h_imag, int32_t B, int32_t T,
                                 float* h_out, void* stream);
int fsn_model_sync_host(fsn_model* m);

/* Streaming (frame-by-frame) inference for the causal configuration (BASELINE config #4): fullsubnet.Model with
 * norm_type cumulative_laplace_norm or cumulative_layer_norm.  State carried between calls: running norm sums, (h, c) of the
 * full-band and sub-band LSTMs.  Call n consumes magnitude frame n ([B, F] float32, device) and writes the cIRM of frame
 * n - look_ahead to d_mask ([B, 2, F]); *h_valid = 0 for the first look_ahead calls.  Feeding look_ahead zero frames at the
 * end flushes the tail, exactly like the reference's right padding (fullsubnet.py:81). */
typedef struct fsn_stream fsn_stream;
int fsn_stream_create(fsn_model* m, int32_t B, fsn_stream** out);
int fsn_stream_step(fsn_stream* st, const float* d_mag_frame, float* d_mask, int32_t* h_valid, void* stream);
void fsn_stream_destroy(fsn_stream* st);

/* Fused post-processing of the inferencer method (fullsubnet_plus/inferencer/inferencer.py:152-157 and
 * audio_zen/acoustics/mask.py:60-63): decompress_cIRM (K = 10, limit = 9.9) + complex multiply with the noisy spectrum.
 * d_crm [B, 2, F, T] float32 (model output), d_noisy / d_enh [B, F, T] complex64 (interleaved re, im). */
int fsn_apply_cirm(const float* d_crm, const float* d_noisy, float* d_enh, int32_t B, int32_t F, int32_t T, void* stream);

/* Test hooks: copy an intermediate of the LAST forward to a device buffer.
 *   "fb_in"  [nbranch, B, F, T+look_ahead]  post-norm (and post-attention) full-band inputs
 *   "fb_out" [nbranch, B, F, T+look_ahead]  full-band model outputs
 *   "sb_mu"  [B]                            utterance mean of the (un-normalised) sub-band input
 *   "sb_in"  [B, F, Isb, T+look_ahead]       normalised sub-band input (sub-band TCN only) */
int fsn_model_get_stage(fsn_model* m, const char* name, float* d_dst, int64_t numel, void* stream);
/* Kernels launched by the last forward (bench.py reports it as gpu_launches). */
int64_t fsn_model_last_launch_count(const fsn_model* m);
/* Device time (ms, CUDA events on the forward's stream) of the sub-band model (LSTM kernels or the TCN) of the last forward;
 * synchronises on the closing event.  < 0 if no forward has run. */
float fsn_model_last_lstm_ms(fsn_model* m);
/* Same for the last n forwards (n <= 32, oldest first); returns how many were written.  Synchronises. */
int fsn_model_lstm_ms_history(fsn_model* m, float* h_ms, int32_t n);
/* Device timeline of the last n forwards (n <= 32, oldest first): 4 floats each = front-end start, front-end end, sub-band
 * LSTM start, LSTM end in ms relative to the oldest one's front-end start (CUDA events on the streams the phases run on).  With
 * the pipelined entry points the front end of batch i+1 lies inside the LSTM interval of batch i.  Returns the count; synchronises. */
int fsn_model_timeline(fsn_model* m, float* h_ms4, int32_t n);
/* Which implementation the last forward used for the sub-band model (FSN_LSTM_MMA / _TCGEN05 / _TCN). */
int fsn_model_last_lstm_impl(const fsn_model* m);

/* Long clips (DESIGN.md §3.7).  The plain entry points (fsn_model_forward, _enhance, both _ragged ones, fsn_model_forward_host) plan
 * every call so that its forward workspace stays within FSN_WS_CAP_GB (default 24): a batch that fits runs whole or as equal
 * sub-batches, exactly as before; when one sub-batch would still exceed the cap, the layer-wise sub-band LSTM runs in time windows
 * of Tw frames (a multiple of 32), carrying h and c exactly from one window to the next, so the result is bit-identical to the
 * unwindowed forward and the sub-band memory is O(Tw).  Everything that needs the whole utterance (norms, attention pooling, the
 * full-band model, the sub-band statistics) stays whole-clip at about 26 KB per frame (FullSubNet+) or 41 KB (fullsubnet.Model).
 * FSN_SB_WINDOW=<frames> (a positive multiple of 32, read at fsn_model_create, else FSN_EINVAL) forces windows of that length.
 * Windows apply to the layer-wise path only: lstm_impl = FSN_LSTM_MMA and the pipelined entry points run unwindowed, and the sub-band
 * TCN runs in bin chunks instead (DESIGN.md §3.8): when one sub-batch would exceed the cap, its B x num_freqs sequences run Fc bins at
 * a time (the last chunk takes the remainder), each sequence with exactly its own arithmetic, so the sub-band memory is O(Fc x T').
 * FSN_SB_CHUNK=<bins> (a positive integer, read at fsn_model_create, else FSN_EINVAL) forces chunks of that many bins on every plain
 * forward of a sub-band TCN model (>= num_freqs: unchunked); LSTM / GRU models ignore it.  The pipelined entry points run unchunked.
 * Length limits (FSN_EINVAL naming the limit, from every forward entry point and fsn_plan_forward): T + look_ahead <= 16 776 960
 * frames (65535 x 256, the TCN depth-wise convolution's grid), num_freqs x (T + look_ahead) <= 2^31 - 1 (the per-clip plane index), and
 * for FullSubNet+ 3 x B x (T + look_ahead) + 128 <= 2^31 - 1 (the full-band TCN's rows; the planner keeps sub-batches below it).  At
 * num_freqs = 257 that is 8 355 967 frames, about 37 hours at 16 kHz / hop 256.  Memory binds first: the whole-clip part, ~26 KB
 * (FullSubNet+) / ~40 KB (fullsubnet.Model) per frame, leaves room in the 24 GB default cap for one clip of up to 4.0 / 2.6 hours
 * (T = 915 689 / 599 084, windows then down to 32 frames); a longer clip runs with 256-frame windows and allocates past the cap.  A 2-hour
 * clip (T = 450 000) plans 6016- / 2944-frame windows within the default cap; the planner keeps every sub-band TCN chunk run below its
 * Bs * Fc * (T + look_ahead) + 128 < 2^31 row limit.
 * After a windowed or chunked forward the model holds at most the plan's bytes: it first gives back whatever earlier forwards grew
 * beyond them.
 *
 * fsn_plan_forward: the plan, from the configuration alone (its lstm_impl; no environment knob), for B clips of T frames under
 * cap_bytes: *Bs clips per sub-batch, *Tw frames per window (0: unwindowed), *bytes (may be NULL) the workspace it requests.
 * force_window: 0, or the FSN_SB_WINDOW value.  No GPU needed.  For a sub-band TCN configuration that chunks, *bytes is the chunked
 * request (fsn_plan_forward_bins gives the chunk). */
int fsn_plan_forward(const fsn_config* cfg, int32_t B, int32_t T, double cap_bytes, int32_t force_window, int32_t* Bs, int32_t* Tw,
                     int64_t* bytes);
/* The same plan with the sub-band TCN's bin chunk: *Fc bins per chunk (0: unchunked; always 0 for LSTM / GRU).  force_bins: 0, or the
 * FSN_SB_CHUNK value. */
int fsn_plan_forward_bins(const fsn_config* cfg, int32_t B, int32_t T, double cap_bytes, int32_t force_window, int32_t force_bins,
                          int32_t* Bs, int32_t* Tw, int32_t* Fc, int64_t* bytes);
/* Bytes the model currently holds in forward workspaces: both lanes plus the sub-band scratch (parameters and host-entry staging excluded). */
int64_t fsn_model_workspace_bytes(const fsn_model* m);
/* Plan of the last plain forward: sub-batch and window (Tw = 0: unwindowed). */
int fsn_model_last_plan(const fsn_model* m, int32_t* Bs, int32_t* Tw);
/* The same with the bin chunk of the sub-band TCN (Fc = 0: unchunked). */
int fsn_model_last_plan_bins(const fsn_model* m, int32_t* Bs, int32_t* Tw, int32_t* Fc);
/* The plan the model's next plain forward of B clips of T frames will use: fsn_plan_forward with the knobs the model read at create
 * (FSN_WS_CAP_GB, FSN_SB_WINDOW, FSN_SB_CHUNK, FSN_LSTM_IMPL).  Host only; enqueues nothing. */
int fsn_model_plan(const fsn_model* m, int32_t B, int32_t T, int32_t* Bs, int32_t* Tw, int64_t* bytes);
/* The same with the bin chunk of the sub-band TCN (Fc = 0: unchunked). */
int fsn_model_plan_bins(const fsn_model* m, int32_t B, int32_t T, int32_t* Bs, int32_t* Tw, int32_t* Fc, int64_t* bytes);
/* Synchronises the device and frees every forward workspace of the model (fsn_model_workspace_bytes drops to 0); the next forward
 * allocates what it needs again.  For callers that keep several models and run a capped (windowed) forward on one of them. */
int fsn_model_release_workspace(fsn_model* m);

/* Host-side packers exposed for CPU tests of the kernel layouts (no GPU needed). */
/* 128-row x 64-half tile with the SWIZZLE_128B layout: byte offset of element (row, k). */
uint32_t fsn_sw128_offset(uint32_t row, uint32_t k);
/* Size in bytes and content of the packed two-layer weight stream (128 gate columns x 64 k SWIZZLE_128B stages, consumption order). */
int64_t fsn_tc5_weight_stream_bytes(int32_t input_size, int32_t hidden);
/* weight row (in [W_i; W_f; W_g; W_o] order) that gate column n (0..127) of 32-unit chunk j maps to */
int32_t fsn_tc5_gate_row(int32_t hidden, int32_t chunk, int32_t n);
int fsn_tc5_pack_weights(int32_t input_size, int32_t hidden, const float* w_ih0, const float* w_hh0, const float* w_ih1,
                         const float* w_hh1, uint16_t* h_dst /* fp16 bits */);

/* Layer-wise wgmma path (DESIGN.md 3.3), one layer: recurrent stream (hidden/32 chunks x hidden/64 tiles of 16 KB), the
 * input-projection matrix for the GEMM ([4 hidden, k_pad] fp16, rows in chunk column order) and the pre-scaled biases
 * ([4 hidden] in the same order; gru != 0 scales pseudo-gate 3 like a tanh argument).  b_ih / b_hh in the nn.LSTM 4-block layout. */
int64_t fsn_tc5r_weight_stream_bytes(int32_t hidden);
int fsn_tc5r_pack_layer(int32_t hidden, int32_t k_in, int32_t k_pad, const float* w_ih, const float* w_hh, const float* b_ih,
                        const float* b_hh, int32_t gru, uint16_t* h_stream, uint16_t* h_wih, float* h_bias);

/* The layer-wise path's input-projection GEMM alone (test / bench hook): d_c[M, N] = d_a[M, K] d_b[N, K]^T, fp16 row-major device
 * buffers, fp32 accumulation, enqueued on `stream`.  M % 128 == 0, N % 128 == 0, K % 64 == 0.  tile_n: 0 (or 256) = 128 x 256 tiles
 * on CTA pairs where N % 256 == 0 and M / 128 is even, else 128 x 128; 128 = always 128 x 128 (what FSN_GIN_GEMM=128 selects). */
int fsn_gemm_f16(const void* d_a, const void* d_b, void* d_c, int64_t M, int32_t N, int32_t K, int32_t tile_n, void* stream);
/* The N tile (128 or 256) fsn_gemm_f16 runs that shape with, or FSN_EINVAL for a shape it rejects; host only. */
int32_t fsn_gemm_f16_tile_n(int64_t M, int32_t N, int32_t K, int32_t tile_n);

#ifdef __cplusplus
}
#endif
#endif /* FSNPLUS_B200_H_ */
