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
 *
 * Stream order.  A call that takes `stream` reads its device inputs and writes its device outputs in `stream` order, and returns
 * without synchronising it, unless its comment says otherwise (fsn_model_forward_host, which returns with the result).  The calls of
 * one handle (a model, a streaming handle, a chunk handle) run in the order they are made whatever streams they are issued on: each
 * call waits on the device for the handle's previous call, so one handle may be driven from several streams (from one host thread at
 * a time).  The calls without a stream -- fsn_model_finalize, fsn_model_load, fsn_stream_create, fsn_chunk_stream_create and the
 * destroys -- synchronise the device before they return, so a handle is ready for a first call on any stream and freed only once
 * nothing in flight uses it.
 * Queue depth: host arrays (h_frames, h_lengths, h_atten_db, h_flags, h_hops, h_counts, slot lists) go to the device through a ring of
 * 4 pinned staging slots per handle, and are free when the call returns.  Every streaming slot call (all but fsn_stream_step before
 * the handle's first slot call), chunk step, save and load takes one slot of its handle; an offline call with host arrays takes one of
 * the model's per sub-batch (a chunk step whose chunks complete also takes the model's, one per sub-batch).  So 4 such calls may be
 * queued ahead of the GPU; the 5th waits on the host until the GPU has read the slot it reuses, i.e. reached the first of them.
 * A call that stages more values than any call before it on the handle grows the 4 slots, a call that grows a workspace frees the
 * old one, and a forward at another batch geometry (clips, frames, window, bin chunk) than the model's previous one frees part of
 * it: each synchronises the device.  So a first call, a call at a larger shape, and a chunk step whose completed-row count differs
 * from the model's previous forward may wait.
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
 * validates the configuration and creates an empty parameter store on the current CUDA device.  The sub-band input size
 * Isb = (2 sb_num_neighbors + 1) + k (2 fb_num_neighbors + 1) (k = 3 for FSN_KIND_PLUS, 1 for FSN_KIND_FSN) must be <= 128 for an LSTM /
 * GRU sub band and <= 64 for the sub-band TCN, else FSN_EINVAL naming the limit (DESIGN.md §3.3). */
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

/* Model files (DESIGN.md §3.15, INTEGRATION.md): a configuration and its reference state_dict in one file, so a C or C++ program gets a
 * ready handle without Python.  Little-endian, all integers unsigned unless noted:
 *   magic       8 bytes "FSNMODEL"
 *   version     u32 = 1
 *   config      u32 count, then per field: u16 name length, the name (an fsn_config member: "num_freqs", "kersize[0]", ...), i32 value
 *   parameters  u32 count, then per key: u16 key length (1..255), the key, i64 numel, numel float32 values in the reference's shape
 *               order.  The keys are exactly those fsn_model_param_info lists for the configuration, in that order.
 *   checksum    u64: h = 0xcbf29ce484222325 (the FNV-1a basis); for each 8-byte little-endian word w of every preceding byte (the
 *               last word zero-padded): h = (h ^ w) * 0x100000001b3 mod 2^64, h ^= h >> 29.
 * A config field the file does not name takes 0 (the zero-initialised default); a field name this library does not know is refused.
 *
 * fsn_model_file_write: writes cfg and the n parameters (keys[i], h_data[i]: numel[i] float32 host values in the reference's shape) to
 * path.  Host only, no GPU.  cfg is checked as fsn_model_create checks it, with the same codes and messages; the keys must be exactly the
 * configuration's, in any order, each with its size (FSN_EINVAL naming the unexpected, duplicate, mis-sized or missing key).  The file is
 * written to path + ".tmp" and renamed over path: a failed write (FSN_EINVAL naming the file and the cause) leaves no file at path. */
int fsn_model_file_write(const char* path, const fsn_config* cfg, int32_t n, const char* const* keys, const float* const* h_data,
                         const int64_t* numel);
/* Reads and verifies the whole file -- magic, version, bounds, trailing bytes, checksum, config fields, the configuration as
 * fsn_model_create checks it, the key set and every size -- and returns its configuration, e.g. for fsn_plan_audio or
 * fsn_stream_state_layout before a GPU is touched.  Host only.  A malformed file is FSN_EINVAL with a message naming the file and what
 * is wrong (for a truncation, the byte offset); a configuration create refuses gives create's code and message. */
int fsn_model_file_config(const char* path, fsn_config* cfg);
/* The same verification, then fsn_model_create, fsn_model_set_param for every record and fsn_model_finalize: a finalized handle whose
 * fsn_model_weights_id equals that of any handle built from the same configuration and parameters (so sessions saved from a handle
 * built in Python load into it).  *out is set to NULL first and stays NULL on any error; no handle leaks. */
int fsn_model_load(const char* path, fsn_model** out);

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
/* Waveforms in, waveforms out (DESIGN.md §3.12): the inferencer's whole method -- STFT, model, decompress_cIRM x noisy spectrum,
 * iSTFT -- for a batch of clips, with both transforms on the device (no FFT library, no torch).  Clip b's output is
 *   torch.istft(decompress_cIRM(model(|X|, Re X, Im X)) * X, n_fft, hop, n_fft, hann, length = L_b)
 *   X = torch.stft(x_b, n_fft, hop, n_fft, window = torch.hann_window(n_fft) (periodic), center = True, pad_mode = "reflect")
 * of that clip alone, T_b = L_b / hop + 1 frames (fullsubnet.Model: model(|X|)), up to fp32 rounding.  Every clip is reflected at its
 * own end and synthesised over its own frames only; the window envelope of its last L_b mod hop samples is the one frame that covers
 * them, as in torch.istft.
 * Geometry from the model: n_fft = 2 (num_freqs - 1), a power of two from 64 to 1024; hop = n_fft / 2; win_length = n_fft.
 * d_wave, d_out: [B, L] float32 device.  Clip b is the first h_lengths[b] samples of its row (h_lengths: HOST array of B counts, free
 * when the call returns; NULL: every clip is L samples).  Samples past a clip's length are never read (NaN there does not matter);
 * its output samples there are exact zeros.
 * FSN_EINVAL, naming the clip: h_lengths[b] <= n_fft / 2 (the reflect padding needs more), h_lengths[b] > L, or too few frames for the
 * TSSE kernels (the clip needs (max kersize - look_ahead - 1) hop samples).  FSN_EINVAL for another num_freqs (naming it), null
 * pointers, B < 1, L outside 1 .. 2^31 - 1, and the length limits below on T = max_b L_b / hop + 1.
 * The call is a plain forward: it plans sub-batches, sub-band time windows and bin chunks under FSN_WS_CAP_GB (fsn_plan_audio) with
 * its own workspace counted (20 bytes per bin and frame of each clip: the mag / real / imag planes and the enhanced spectrum).  Per
 * sub-batch: one analysis launch, the forward (unmasked when every clip has the longest clip's length, as fsn_model_forward_ragged),
 * one synthesis launch.  The call does not synchronise the stream. */
int fsn_model_enhance_audio(fsn_model* m, const float* d_wave, int32_t B, int64_t L, const int64_t* h_lengths, float* d_out, void* stream);

/* Attenuation limits (DESIGN.md §3.18): how much noise suppression may take away, per clip or per live session.  A limit of L dB
 * (L >= 0, or +inf) has the floor lam = 10^(-L / 20), computed in double and rounded to float.  After decompress_cIRM the complex mask
 * M of every bin and frame becomes M' = M where |M| >= lam (always at lam = 0, i.e. L = +inf: no limit), lam M / |M| where
 * 0 < |M| < lam (the mask's phase, its magnitude raised to lam), (lam, 0) where M = 0; then Y = M' X as without a limit.  So
 * |Y| >= lam |X| in every bin: no bin loses more than L dB.  A mask that amplifies is never touched; L = 0 attenuates no bin.
 * The limit acts only where the library forms the enhanced spectrum or audio: every mask output (fsn_model_forward*, the streaming
 * d_mask) stays the model's raw cIRM.  A negative or NaN limit is FSN_EINVAL naming the clip or slot and the value.  A call whose
 * limits are all +inf runs exactly the unlimited call: the same kernels, bits and launch counts.
 *
 * Offline: h_atten_db is a HOST array of B floats, one per clip (NULL: no limit), free when the call returns; it reaches the device
 * with the clips' lengths (one copy per sub-batch).  fsn_model_forward_enhance_lim is fsn_model_forward_enhance (h_frames NULL) or
 * fsn_model_forward_enhance_ragged with limits; fsn_model_enhance_audio_lim is fsn_model_enhance_audio with limits.  Both plan, check
 * and run exactly as those calls; with h_atten_db NULL they are those calls.  The pipelined entry points and fsn_apply_cirm take no
 * limit. */
int fsn_model_forward_enhance_lim(fsn_model* m, const float* d_mag, const float* d_real, const float* d_imag, int32_t B, int32_t T,
                                  const int32_t* h_frames, const float* h_atten_db, float* d_enh, void* stream);
int fsn_model_enhance_audio_lim(fsn_model* m, const float* d_wave, int32_t B, int64_t L, const int64_t* h_lengths, const float* h_atten_db,
                                float* d_out, void* stream);
/* The plan of fsn_model_enhance_audio for these clips (fsn_plan_forward_bins with the audio workspace counted), after the same checks
 * of the configuration and lengths, with the same FSN_EINVAL messages.  Host only, no GPU. */
int fsn_plan_audio(const fsn_config* cfg, int32_t B, int64_t L, const int64_t* h_lengths, double cap_bytes, int32_t force_window,
                   int32_t force_bins, int32_t* Bs, int32_t* Tw, int32_t* Fc, int64_t* bytes);
/* Same call with HOST buffers (pinned or pageable): H2D copies, the forward and the D2H copy of the
 * mask are all enqueued on `stream` and the call returns after the result is in h_out.  Its arguments are checked as
 * fsn_model_forward checks them, before anything is staged, copied or synchronised. */
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
 * block the host) or fsn_model_sync_host(m) has returned.  A plain fsn_model_forward on any stream first waits for the pipeline, and
 * a submit waits for the last plain call (the model's calls run in call order on the device; "Stream order" above).
 *
 * fsn_model_forward_host_async: pinned host buffers; additionally the H2D copy of batch i+1 and the D2H copy of batch i-1
 * overlap on two copy streams.  `stream` is ignored (host memory carries no stream order).  The host buffers must stay
 * untouched (h_out unread) until fsn_model_sync_host() returns.  Both pipelined calls check their arguments as fsn_model_forward
 * does (with the length limits of the whole batch) before they record, wait on, allocate or copy anything. */
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

/* Independent sessions on one handle (DESIGN.md §3.9): each of the B slots serves its own session, which starts, pauses and ends on
 * its own schedule and gets exactly the masks it would get streamed alone.  h_flags: HOST array of B flags for this tick. */
#define FSN_SLOT_HOLD 0   /* no frame this tick: the slot's state is unchanged, its frame is never read, its mask row is zero */
#define FSN_SLOT_STEP 1   /* consume the slot's frame, advance its state by one frame                                         */
#define FSN_SLOT_START 2  /* reset the slot's state (norm sums, frame count, h and c of every layer of both LSTMs), then STEP  */
/* h_valid (HOST, [B]): h_valid[b] = 1 when slot b stepped at this tick and has consumed more than look_ahead frames since its last
 * START; d_mask[b] is then the mask of the slot's frame n_b - look_ahead (n_b: frames consumed, this one included).  Otherwise
 * h_valid[b] = 0 and d_mask[b] is zero.  To end a session feed look_ahead zero frames with STEP (the reference's right padding), then
 * HOLD the slot until a START reuses it.  A slot that has never been started behaves as if it had just been reset.
 * FSN_EINVAL, naming the slot, for a flag outside {0, 1, 2}; FSN_EINVAL for a null h_flags or h_valid.  The flags are staged through
 * pinned buffers, so both arrays are free when the call returns; the call does not synchronise the stream.
 * fsn_stream_step on a handle that has never used the slot call runs exactly as before.  Once the handle has used it,
 * fsn_stream_step is the slot call with every flag FSN_SLOT_STEP, and *h_valid is 1 when every slot's mask is valid. */
int fsn_stream_step_slots(fsn_stream* st, const float* d_mag_frame, float* d_mask, const int32_t* h_flags, int32_t* h_valid,
                          void* stream);

/* Many frames per call (DESIGN.md §3.13): K fsn_stream_step_slots ticks in one call, for callers that take 8-64 frames at a time or
 * catch a session up on a backlog.  d_mag [B, F, K] float32 device: slot b's next K magnitude frames along the last axis (rows of
 * HOLD slots are never read).  h_flags: HOST, B flags as in fsn_stream_step_slots; STEP and START consume K frames, HOLD leaves the
 * slot's state (frame count and norm sums included) unchanged.  d_mask [B, 2, F, K] float32 device: with n_b the frames slot b had
 * consumed since its START before this call (0 on START), column k is the mask of frame n_b + k - look_ahead when that index is >= 0,
 * else zero; rows of held slots are zero.  h_valid (HOST, [B]): the number of valid columns, always the trailing ones:
 * clamp(n_b + K - look_ahead, 0, K) for a stepping slot, 0 for a held one.  The call may be mixed freely with fsn_stream_step /
 * fsn_stream_step_slots and save / load on the same handle; the session state and its payload are the per-frame step's.
 * The sub-band stage runs on the offline forward's path: the layer-wise tensor-core kernels when the configuration takes them
 * (then only the stepping sessions run, in sub-batches and time windows under FSN_WS_CAP_GB, fsn_stream_chunk_plan; the result does
 * not depend on the split, but it is not the per-frame step's bits: both meet the same accuracy), else the per-frame step's kernel
 * over K steps, bit-identical to K fsn_stream_step_slots calls.  The scratch belongs to the handle: allocated at the first call,
 * grow-only, freed by fsn_stream_destroy.
 * FSN_EINVAL naming the slot for a flag outside {0, 1, 2}; naming the argument for K < 1 or a null array; naming the limit for K past
 * 65535 x 256 - 4 frames or num_freqs x K past 2^31 - 1.  FSN_ESTATE on a handle that serves the audio call.  A failed call changes no
 * state.  Both host arrays are free when the call returns; the call does not synchronise the stream. */
int fsn_stream_step_chunk(fsn_stream* st, const float* d_mag, int32_t K, float* d_mask, const int32_t* h_flags, int32_t* h_valid,
                          void* stream);
/* The chunk call's sub-band plan for n_active stepping sessions of K frames under cap_bytes: sessions per sub-batch *Bs, window *Tw
 * (0: the whole chunk) and the scratch *bytes of one sub-batch (layer-wise path: images, Gin, layer output, h / c carry, compact
 * masks; generic path: one piece, the images).  Same FSN_EINVAL messages as the call, plus a non-streaming configuration and
 * n_active < 1.  Host only, no GPU. */
int fsn_stream_chunk_plan(const fsn_config* cfg, int32_t n_active, int32_t K, double cap_bytes, int32_t* Bs, int32_t* Tw, int64_t* bytes);

/* Audio in, audio out (DESIGN.md §3.10): the slot call with the STFT before the model step and decompress_cIRM x noisy spectrum,
 * inverse FFT and overlap-add after it, on the device.  Each slot's waveform equals the offline enhancement of its session's audio
 * (torch.stft(center=True, reflect) -> model -> decompress_cIRM x spectrum -> torch.istft(length = L)).
 * Geometry from the model: n_fft = 2 (num_freqs - 1), a power of two from 64 to 1024; hop = n_fft / 2; periodic Hann window of n_fft.
 * Any other num_freqs is FSN_EINVAL, naming it.
 * d_samples [B, hop] float32 device: one hop of new samples per slot (rows of HOLD and FLUSH slots are never read).
 * d_out [B, hop] float32 device: one hop of enhanced audio per slot.  h_flags: HOST, B flags of FSN_SLOT_HOLD / STEP / START and: */
#define FSN_SLOT_FLUSH 3  /* audio call only: no samples this tick; the session's input has ended, advance its tail                   */
/* A START resets the slot's audio and model state and consumes the session's first hop; STEP consumes the next hop; HOLD is no tick
 * (state unchanged, output row zero).  A session of K >= 2 hops (L = K hop samples; a session of any other length runs through
 * fsn_stream_step_audio_samples below) ends with exactly look_ahead + 2 FLUSH ticks; further FLUSH ticks act as HOLD until a START
 * reuses the slot.
 * h_valid (HOST, [B]): h_valid[b] = 1 when d_out[b] holds hop q of the slot's session; hop q comes out at the slot's tick
 * q + look_ahead + 2 (ticks counted from 0 at the START, HOLD ticks excluded): the algorithmic latency is look_ahead + 2 hops.
 * Every other output row is zero.  d_mask: null, or [B, 2, F] float32 device, which receives at slot tick k the cIRM of the slot's
 * frame k - look_ahead - 1 when that index is >= 0, and zero otherwise.
 * FSN_EINVAL, naming the slot, for a flag outside {0, 1, 2, 3}, a STEP after the session's first FLUSH, a STEP or FLUSH on a slot
 * that has no session, and a FLUSH after fewer than 2 hops; FSN_EINVAL, naming the argument, for a null array.  A handle serves
 * either the mask calls (fsn_stream_step, fsn_stream_step_slots) or this call: mixing them is FSN_ESTATE.  The audio state
 * (history, spectrum ring, overlap tail) and the scratch shared with fsn_stream_step_audio_chunk are allocated at the first call.
 * Per tick: one H2D copy and 8 kernels (+ the reset kernel on ticks where a session's model row starts, + the grid-barrier memset of
 * the full-band step at B <= 64; 2 kernels when no slot has a model frame).  The call does not synchronise the stream. */
int fsn_stream_step_audio_slots(fsn_stream* st, const float* d_samples, float* d_out, const int32_t* h_flags, int32_t* h_valid,
                                float* d_mask, void* stream);

/* Many hops per call (DESIGN.md §3.14): audio in and out, K hops per slot, for callers that hold audio buffers of 8-64 hops or catch
 * a session up after a stall.  For slot b the call is exactly K fsn_stream_step_audio_slots ticks on that slot, by h_flags[b] and
 * n = h_hops[b] (HOST arrays of B values):
 *   HOLD: HOLD x K (h_hops ignored);  START (1 <= n <= K): START, STEP x (n - 1), HOLD x (K - n);  STEP (1 <= n <= K): STEP x n,
 *   HOLD x (K - n);  FLUSH (0 <= n <= K): STEP x n, FLUSH x (K - n) -- the input ends after these n hops.
 * A session ends within a FLUSH call when n + look_ahead + 2 <= K; otherwise further FLUSH calls with n = 0 complete it.  A session
 * that STARTs and FLUSHes takes two calls.
 * d_samples [B, K hop] float32 device: slot b's n new hops at the front of its row; no other sample is read.  d_out [B, K hop] float32
 * device: the hops those ticks emit, in order, at the front of the row, zero after them; h_nout (HOST, [B]) their count.  d_mask: null,
 * or [B, 2, F, K] float32 device, whose column i is the mask row of tick i (zero on HOLD ticks, the START tick and before frame 0).
 * The slot's state and counters afterwards are those the K ticks leave, so this call, fsn_stream_step_audio_slots and save / load mix
 * freely on one handle.  The model steps each session's frames of the call on the chunk call's path (fsn_stream_step_chunk: the
 * layer-wise sub band where the configuration takes it, else bit-identical to the per-hop call).  The scratch belongs to the handle:
 * allocated at the first call, grow-only, freed by fsn_stream_destroy.
 * FSN_EINVAL naming the slot for a flag outside {0, 1, 2, 3}, h_hops outside the range above, a STEP or FLUSH on a slot that has no
 * session, a STEP or a FLUSH with n > 0 after the session's FLUSH, and a FLUSH that would end a session of fewer than 2 hops; naming the
 * argument for a null array and K < 1; naming the limit for K past fsn_stream_step_chunk's limits or K x hop past 2^31 - 1.  FSN_ESTATE
 * on a handle that serves the mask calls.  A failed call changes no state.  The host arrays are free when the call returns; the call
 * does not synchronise the stream. */
int fsn_stream_step_audio_chunk(fsn_stream* st, const float* d_samples, int32_t K, const int32_t* h_flags, const int32_t* h_hops,
                                float* d_out, int32_t* h_nout, float* d_mask, void* stream);

/* Any number of samples per slot and call (DESIGN.md §3.19), with fsn_chunk_stream_step's call shape: packets of 10 ms, 20 ms or
 * whatever a transport delivers, and sessions of any length.  hop = n_fft / 2, la = look_ahead.
 * d_samples [B, S] float32 device: slot b reads its first h_counts[b] samples (0 <= h_counts[b] <= S); no other sample is read.
 * h_flags (HOST, B values): HOLD no change (h_counts ignored); START resets the slot, then consumes its samples; STEP consumes; FLUSH
 * consumes, then ends the session: every remaining output sample through L comes out in this call and the slot has no live session
 * after it (a later FLUSH of 0 samples acts as HOLD, a START reuses the slot).
 * d_out [B, S + (la + 3) hop] float32 device: each slot's newly final samples at the front of its row, zero after them; h_nout (HOST,
 * [B]) their count.  The bound: before a call a session has read t hop + r0 samples (t whole hops, r0 < hop) and emitted
 * max(0, t - la - 2) hops, so it lags by at most (la + 2) hop + r0 < (la + 3) hop; a call adds at most S.
 * Result: a session's outputs concatenated over its calls are fsn_model_enhance_audio of its input x[0, L), up to fp32 rounding, for
 * every L > n_fft / 2 (the offline call's minimum) and any schedule of counts, holds and calls.
 * Timing: output sample n is final in the call where the session's input reaches (floor(n / hop) + la + 3) hop samples, or at its FLUSH
 * -- the hop calls' latency of la + 2 hops, counted from the end of the hop the sample is in.
 * Equivalence: completed hops drive exactly the ticks of the hop calls.  A call that completes at most one hop per slot and FLUSHes
 * no live session runs fsn_stream_step_audio_slots' path; any other call runs fsn_stream_step_audio_chunk's path with each slot's hop
 * count and K = the most ticks of any slot, bit-identical to that hop call.  So a session fed whole hops and ended on a hop boundary
 * gives the hop calls' bits.  A session ending at L = K hop + r, 0 < r < hop, has K + 1 frames: frame K is analysed from its r real
 * samples reflected at L - 1, and after it is synthesised the last r samples are its tail times 1 / w^2(i + hop), as offline.
 * Between calls the r < hop samples of a partial hop wait in the history-ring slot the next hop takes (the payload layout does not
 * change); a session started with fewer than hop samples exists at tick 0 and its first whole hop runs the START tick.
 * Mixing: the hop calls and this call mix freely on one audio handle, except that a hop call's STEP or FLUSH on a slot holding a
 * partial hop is FSN_EINVAL naming the slot (a START discards the partial hop); a FLUSH of 0 samples from this call completes a
 * session a hop call left mid-flush.  fsn_stream_set_atten_lim applies to every frame this call synthesises.  No mask output: the
 * hop calls provide it.
 * Launches: a call in which no slot completes a hop or FLUSHes launches one kernel (the partial-hop store, which also zeroes d_out),
 * and a call in which no slot consumes a sample launches none (d_out is cleared by a memset).  Otherwise as the hop call it runs.
 * Errors, all checked before any state changes (a failed call changes nothing): FSN_EINVAL naming the slot for a flag outside
 * {0, 1, 2, 3}, a count outside [0, S], a STEP or FLUSH on a slot without a session, a STEP or a FLUSH with a count > 0 after the
 * session's FLUSH, and a FLUSH that would end a session of L <= n_fft / 2 samples; naming the argument for a null array and S < 1;
 * naming the limit for a derived K past fsn_stream_step_audio_chunk's limits and for S + (la + 3) hop past 2^31 - 1.  FSN_ESTATE on a
 * handle that serves the mask calls.  The host arrays are free when the call returns; the call does not synchronise the stream. */
int fsn_stream_step_audio_samples(fsn_stream* st, const float* d_samples, int32_t S, const int32_t* h_flags, const int32_t* h_counts,
                                  float* d_out, int32_t* h_nout, void* stream);

/* Per-slot attenuation limits of the streaming audio calls (semantics: fsn_model_enhance_audio_lim above): slot h_slots[i] gets
 * h_atten_db[i] dB (+inf: no limit), kept until it is set again.  fsn_stream_step_audio_slots and fsn_stream_step_audio_chunk apply it
 * to every frame they synthesise after this call; the mask calls and every d_mask ignore it.  A fresh handle has no limit on any slot;
 * START and fsn_stream_load_slots leave a slot's limit as it is, and the limit is not part of a saved session (payload and meta are
 * unchanged): a caller who moves a session sets the limit of the slot it loads into.  Host only: it enqueues nothing, the next step
 * stages the limits with its plan.  Errors, checked before anything changes: FSN_EINVAL for a null array, n < 1, a slot out of range, a
 * slot twice in one call (naming the index) and a negative or NaN limit (naming the slot and the value).  Both arrays are free when
 * the call returns. */
int fsn_stream_set_atten_lim(fsn_stream* st, int32_t n, const int32_t* h_slots, const float* h_atten_db);

/* Overlapped-chunk sessions (DESIGN.md §3.16): live audio for any model fsn_model_enhance_audio runs -- FullSubNet+ with any attention
 * and norm, the sub-band TCN, fullsubnet.Model with any norm -- by the reference's overlapped_chunk inferencer
 * (fullsubnet_plus/inferencer/inferencer.py:191-250).  With C = chunk_samples (even), H = C / 2, P = 256 samples of pre-context and
 * w = torch.hann_window(C) (periodic), a session's input x[0, L) is cut into chunks k = 0 .. ceil(L / H) - 1 of rows
 * x[k H - P, k H + C) (zero before 0 and past L), each enhanced by fsn_model_enhance_audio, its first P output samples dropped: e_k.
 * Output region y[k H, (k + 1) H) is e_0[0, H) for k = 0 and e_k[0, H) w[0, H) + e_{k-1}[H, C) w[H, C) after it; the output is y[0, L).
 * Chunk k completes once the input reaches k H + C (at FLUSH: every chunk, zero-padded), and region k is emitted with it, so the
 * output lags the input by H to 2H samples.  Every chunk completed by every slot in one call runs as ONE batch of rows of P + C
 * samples through the offline audio call (sub-batches under FSN_WS_CAP_GB, fsn_plan_audio; no forward when none completes).
 * fsn_chunk_stream_create: FSN_EINVAL naming the argument for a null m or out and B < 1; naming the limit for an odd C, H < P, and
 * rows of P + C samples that fsn_model_enhance_audio refuses for this model (its message); FSN_ESTATE before fsn_model_finalize.  The
 * handle keeps per slot a ring of C + P samples and a tail of H samples, and the window, allocated here; the staged plan and the
 * batch's rows are allocated at first use, grow-only.  fsn_chunk_stream_destroy frees them all.
 * fsn_chunk_stream_step: d_samples [B, S] float32 device, slot b reading its first h_counts[b] samples (0 <= h_counts[b] <= S; no other
 * sample is read).  h_flags (HOST, B values of FSN_SLOT_*): HOLD no samples, no change (h_counts ignored); START resets the slot,
 * then consumes; STEP consumes; FLUSH consumes, then ends the session (the remaining chunks are enhanced and y through L is emitted),
 * leaving the slot without a session.  d_out [B, S + C] float32 device: each slot's newly final samples at the front of its row,
 * zero after them; h_nout (HOST, [B]) their count.  A session's outputs concatenated over its calls are y[0, L).
 * FSN_EINVAL naming the slot for a flag outside {0, 1, 2, 3}, a count outside [0, S], a STEP or FLUSH on a slot without a session;
 * naming the argument for a null array and S < 1; naming the limit for S + 2 (C + P) past 2^31 - 1 and for chunk rows of more than
 * 2^31 - 1 samples in one call.  A failed call changes no state.
 * The host arrays are free when the call returns; the call does not synchronise the stream. */
typedef struct fsn_chunk_stream fsn_chunk_stream;
int fsn_chunk_stream_create(fsn_model* m, int32_t B, int32_t chunk_samples, fsn_chunk_stream** out);
int fsn_chunk_stream_step(fsn_chunk_stream* cs, const float* d_samples, int32_t S, const int32_t* h_flags, const int32_t* h_counts,
                          float* d_out, int32_t* h_nout, void* stream);
void fsn_chunk_stream_destroy(fsn_chunk_stream* cs);
/* Per-slot attenuation limits of overlapped-chunk sessions, with fsn_stream_set_atten_lim's rules: every chunk row a slot completes in a
 * later fsn_chunk_stream_step is enhanced with that slot's limit in the call's one audio batch (fsn_model_enhance_audio_lim).  The
 * cross-fade is linear, so a session whose limit never changes gets exactly the overlapped-chunk output of the limited enhancement. */
int fsn_chunk_stream_set_atten_lim(fsn_chunk_stream* cs, int32_t n, const int32_t* h_slots, const float* h_atten_db);

/* Park, resume and move overlapped-chunk sessions (DESIGN.md §3.17): save the state of some slots of a chunk handle to a device buffer
 * and load it into any slot of any chunk handle with the same chunk_samples -- the same one, one with another B, one on another device
 * after the caller has copied the payload there, or one of ANOTHER MODEL.
 *
 * A session's state holds no model state: the sample ring, the overlap tail and two host counters.  A saved session is a payload row
 * of payload_bytes (d_state [n, payload_bytes], device) plus a host fsn_chunk_slot_meta.  The payload, one layout per C:
 *   bytes [0, (C + P) 4)            the ring, float32: session sample p at float p mod (C + P) (the last C + P samples the slot read)
 *   bytes [t, t + H 4)              the tail, float32 (H = C / 2), t = (C + P) 4 rounded up to 16: the windowed second half of the
 *                                   session's last enhanced chunk
 *   payload_bytes = t + H 4 rounded up to 256.
 * The bytes between the ring and the tail and after the tail are padding: a save writes them with unspecified values, a load never
 * reads what lies between the ring and the tail and writes what follows the tail only to the handle's own padding, which nothing
 * reads.  The ring is indexed by absolute session position, so a raw copy of the rows is canonical: independent of B, of the slot and
 * of the device.
 *
 * Model identity is NOT checked: a session saved from one model continues on another (other weights, the sub-band TCN, fullsubnet.Model)
 * -- the chunks enhanced before the load come from the saving model, the rest from the loading one, cross-faded by the usual rule.
 * num_freqs, model_kind and weights_id are in the meta for the caller to enforce its own policy.
 *
 * fsn_chunk_stream_save_slots is a snapshot: the slots are unchanged and may keep stepping (a fork) or START other sessions.  h_meta[i]
 * describes session i, saved from slot h_slots[i]; a slot without a session saves as samples = -1, chunks = 0.
 * fsn_chunk_stream_load_slots replaces a START: it overwrites the state of slot h_slots[i] with session i, host counters included, and
 * the slot's next call is a STEP or FLUSH that continues the session.  Loading a meta with samples = -1 leaves the slot without a
 * session.
 * Both calls are ordered on `stream` like the step: h_meta is filled (save) or validated (load) on the host before the call returns,
 * the payload copy (one kernel for the n sessions) is enqueued and the stream is not synchronised; h_slots and h_meta are free on
 * return.
 * Every check runs before any state changes or launch: a failed call changes nothing.  FSN_EINVAL, naming the index or field: a null
 * array, n < 1, a slot out of range, a slot twice in one load, a bad magic or version, a chunk_samples, pre_context or payload_bytes
 * other than this handle's, samples outside -1 .. 2^62, chunks other than max(0, floor(samples / H) - 1) (0 when samples = -1), a
 * d_state that is not 256-byte aligned device memory of the handle's device. */
#define FSN_CHUNK_STATE_VERSION 1
#define FSN_CHUNK_STATE_MAGIC 0x434E5346u  /* the bytes 'F' 'S' 'N' 'C' */
typedef struct fsn_chunk_slot_meta { /* host-side description of one saved overlapped-chunk session                   */
    uint32_t magic, version;         /* FSN_CHUNK_STATE_MAGIC, FSN_CHUNK_STATE_VERSION                                */
    int32_t chunk_samples, pre_context; /* C and P (256) of the saving handle                                         */
    int32_t num_freqs, model_kind;   /* the saving model: for the caller, not checked at a load                       */
    uint64_t weights_id;             /* fsn_model_weights_id of the saving model: for the caller, not checked         */
    int64_t samples;                 /* n: samples since START, -1 = the slot had no session                          */
    int64_t chunks;                  /* k: chunks enhanced (max(0, floor(n / H) - 1) for a live session)              */
    int64_t payload_bytes;           /* stride of one session in d_state                                              */
} fsn_chunk_slot_meta;
/* Payload stride for chunk_samples and sizeof(fsn_chunk_slot_meta).  Host only, no GPU.  FSN_EINVAL naming the limit for a
 * chunk_samples that fsn_chunk_stream_create refuses on its own (odd, H < P, past 2^30 - 1 - P). */
int fsn_chunk_stream_state_layout(int32_t chunk_samples, int64_t* payload_bytes, int32_t* meta_bytes);
int fsn_chunk_stream_save_slots(fsn_chunk_stream* cs, int32_t n, const int32_t* h_slots, void* d_state, fsn_chunk_slot_meta* h_meta,
                                void* stream);
int fsn_chunk_stream_load_slots(fsn_chunk_stream* cs, int32_t n, const int32_t* h_slots, const void* d_state,
                                const fsn_chunk_slot_meta* h_meta, void* stream);

/* Park, resume and move sessions (DESIGN.md §3.11): save the state of some slots to a device buffer and load it into any slot of a
 * compatible handle -- the same one, another with a different B or full-band kernel, or one on another device after the caller has
 * copied the payload there.
 *
 * A saved session is a payload row of payload_bytes (d_state [n, payload_bytes], device) plus a host fsn_slot_meta.  The payload is
 * canonical: one layout per (configuration, mode), independent of B, of the slot, of the full-band kernel (weight-stationary at B <= 64,
 * generic above) and of the handle's tick parity.  Segments in this order, each at a 16-byte aligned offset: cum_in (2 fp64), cum_sb
 * (num_freqs x 2 fp64), full-band h (fp16, every layer) and c (fp32, every layer; the GRU keeps its fp32 h there), sub-band h and c
 * (num_freqs rows per layer each), then in audio mode the history ring, the spectrum ring and the overlap tail.  payload_bytes is a
 * multiple of 256.
 *
 * fsn_stream_save_slots is a snapshot: the slots are unchanged and may keep stepping (a fork) or START other sessions.  h_meta[i]
 * describes session i, saved from slot h_slots[i].
 * fsn_stream_load_slots replaces a START: it overwrites the whole state of slot h_slots[i] with session i, host counters included, and
 * the slot's next tick is a STEP (or FLUSH).  A START after a load discards the loaded state like any other.
 * Both calls are ordered on `stream` like the step calls: h_meta is filled (save) or validated (load) on the host before the call
 * returns, the payload copy (one kernel) is enqueued and the stream is not synchronised; h_slots and h_meta are free on return.
 * A handle that has served no call yet takes the meta's mode at a load (and allocates its audio state in audio mode); a handle that
 * has only used fsn_stream_step switches to per-slot counts at a save or load, as at its first slot call.
 * Errors change no state.  FSN_EINVAL, naming the index or field: a null array, n < 1, a slot out of range, a slot twice in one load, a
 * bad magic or version, an audio meta's frames outside [0, hop) or > 0 with tick -1 or hops > 0, a payload_bytes other than this
 * handle's, a configuration field that differs (lstm_impl excepted: streaming
 * always runs the mma kernels), a weights_id that differs, a d_state that is not 256-byte aligned device memory of the handle's
 * device.  FSN_ESTATE: a meta whose mode is not the handle's, a save on a handle that has served no call. */
#define FSN_SLOT_STATE_VERSION 1
#define FSN_SLOT_STATE_MAGIC 0x534E5346u   /* the bytes 'F' 'S' 'N' 'S' */
#define FSN_STATE_MODE_MASK 1              /* saved from a handle serving fsn_stream_step / fsn_stream_step_slots */
#define FSN_STATE_MODE_AUDIO 2             /* saved from a handle serving fsn_stream_step_audio_slots             */
typedef struct fsn_slot_meta {      /* host-side description of one saved session                                  */
    uint32_t magic, version;        /* FSN_SLOT_STATE_MAGIC, FSN_SLOT_STATE_VERSION                                 */
    fsn_config cfg;                 /* the saving model's configuration                                             */
    uint64_t weights_id;            /* fsn_model_weights_id of the saving model                                     */
    int32_t mode;                   /* FSN_STATE_MODE_MASK or FSN_STATE_MODE_AUDIO                                  */
    int32_t frames;                 /* mask mode: frames the slot consumed since its START; audio mode: the samples r of a
                                       partial hop (fsn_stream_step_audio_samples), 0 <= r < hop, 0 without a session or after its FLUSH */
    int32_t tick, hops;             /* audio mode: the slot's tick count (-1 = no session) and hops K (0 before its first FLUSH); 0 in mask mode */
    int64_t payload_bytes;          /* stride of one session in d_state                                             */
} fsn_slot_meta;
/* Payload stride of this handle's mode; FSN_ESTATE before the handle has served a call or a load. */
int64_t fsn_stream_state_bytes(const fsn_stream* st);
/* Payload stride of a (configuration, mode) and sizeof(fsn_slot_meta).  Host only, no GPU.  FSN_EINVAL for a configuration that cannot
 * stream (FullSubNet+, a non-cumulative norm), a mode other than 1 or 2, or an audio mode whose num_freqs the audio call rejects. */
int fsn_stream_state_layout(const fsn_config* cfg, int32_t mode, int64_t* payload_bytes, int32_t* meta_bytes);
/* 64-bit hash of every parameter (key and fp32 bytes) of a finalized model: equal weights give equal ids.  0 before fsn_model_finalize. */
uint64_t fsn_model_weights_id(const fsn_model* m);
int fsn_stream_save_slots(fsn_stream* st, int32_t n, const int32_t* h_slots, void* d_state, fsn_slot_meta* h_meta, void* stream);
int fsn_stream_load_slots(fsn_stream* st, int32_t n, const int32_t* h_slots, const void* d_state, const fsn_slot_meta* h_meta,
                          void* stream);

/* Fused post-processing of the inferencer method (fullsubnet_plus/inferencer/inferencer.py:152-157 and
 * audio_zen/acoustics/mask.py:60-63): decompress_cIRM (K = 10, limit = 9.9) + complex multiply with the noisy spectrum.
 * d_crm [B, 2, F, T] float32 (model output), d_noisy / d_enh [B, F, T] complex64 (interleaved re, im). */
int fsn_apply_cirm(const float* d_crm, const float* d_noisy, float* d_enh, int32_t B, int32_t F, int32_t T, void* stream);

/* Test hooks: copy an intermediate of the LAST forward to a device buffer.
 *   "fb_in"  [nbranch, B, F, T+look_ahead]  post-norm (and post-attention) full-band inputs
 *   "fb_out" [nbranch, B, F, T+look_ahead]  full-band model outputs
 *   "sb_mu"  [B]                            utterance mean of the (un-normalised) sub-band input
 *   "sb_in"  [B, F, Isb, T+look_ahead]       normalised sub-band input (sub-band TCN only)
 *   "stft"   [3, B, 1, F, T]                 the mag / real / imag planes the audio call's forward read
 *   "enh"    [B, F, T] complex64 (2 floats)  the enhanced spectrum the audio call synthesised
 *   "sb_img" raw bytes, numel = bytes / 4    the fp16 sub-band input of the LSTM / GRU (not the TCN: FSN_EINVAL) as the last
 *            forward packed it, with np = ceil(B*F / 128) rounded up to even tiles and T' = T + look_ahead:
 *              Isb <= 64:                 SWIZZLE_128B images [np, T', 128 rows, 64 halves]: row r's 16-byte chunk k / 8 sits
 *                                         at chunk (k / 8) ^ (r % 8) of its 128-byte line
 *              Isb > 64, layer-wise path: rows of 128 halves, sequence `row` at frame t is row ((row / 128) * T' + t) * 128 + row % 128
 *              Isb > 64, generic kernel:  time-major rows of 128 halves [T', ceil(B*F / 128) * 128, 128] (the rest of the buffer unused)
 *            (fsn_model_last_lstm_impl tells the path); bytes = np * T' * 128 * (128 or 256).  Rows >= B*F, channels >= Isb and
 *            frames past a clip's extent are zero.  FSN_ESTATE after a forward that packed the images in time windows.
 * "stft" and "enh" are kept only when the last forward was an audio call that ran as one sub-batch; FSN_ESTATE otherwise. */
int fsn_model_get_stage(fsn_model* m, const char* name, float* d_dst, int64_t numel, void* stream);
/* Test hook of the streaming handle: copy an intermediate of the LAST step call that stepped the model (fsn_stream_step, _step_slots,
 * _step_chunk, _step_audio_slots, _step_audio_chunk, _step_audio_samples) to a device buffer.  K: that call's frames (the audio calls:
 * its largest model frame count per slot); every slot's row, held ones included.  In the audio calls slot b's frames are columns
 * 0 .. k_b - 1 (k_b: the frames it stepped in the call); its columns past k_b hold no frame of the call.
 *   "fb_in"  [B, F, K]                 the cumulative-norm output, the full band's input
 *   "fb_out" [B, F, K]                 the full band's output
 *   "sb_img" raw bytes, numel = bytes / 4  the fp16 sub-band input of the generic kernel: SWIZZLE_128B images [nt, K, 128, 64] (Isb <= 64)
 *            or time-major rows of 128 halves [K, nt * 128, 128] (Isb > 64), nt = ceil(B*F / 128), bytes = nt * K * 128 * (128 or 256)
 *   "mag"    [B, F, K]                 the audio calls only: the magnitude frames the model stepped
 *   "mask"   [B, 2, F, K]              the audio calls only: the model's cIRM columns (the mask each column's synthesis reads; the
 *                                      sample call returns no masks)
 *   "spec"   [B, K, F] complex64       the audio calls only: the noisy spectra of the frames the call analysed (numel = 2 B K F floats)
 * FSN_ESTATE before any step, after a step call that failed, after an audio call that stepped no frame, for "sb_img" after a step whose sub band ran layer-wise
 * (its images are compact rows per group, sub-batch and window) and for "mag", "mask" and "spec" after a mask call.  FSN_EINVAL for a null argument,
 * an unknown name or a numel other than the one the message names.  Reading it changes nothing on any step path. */
int fsn_stream_get_stage(fsn_stream* st, const char* name, float* d_dst, int64_t numel, void* stream);
/* Test-only: 1 if the handle's full-band step runs on the weight-stationary kernel (k_lstm_ws.cu), 0 if on the generic mma kernel
 * (fixed at fsn_stream_create: B <= 64 slots on a shape lstm_ws_supported takes, and FSN_NO_WS unset) or for a null handle. */
int fsn_stream_fb_ws(const fsn_stream* st);
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
/* Test-only: 1 if the last forward of a fullsubnet.Model ran its full-band LSTM on the weight-stationary kernel (k_lstm_ws.cu), 0 if
 * on the generic mma kernel, for a FullSubNet_Plus (whose full band is the TCN) or before any forward.  Lets the element-wise tests
 * assert which kernel they checked. */
int fsn_model_last_fb_ws(const fsn_model* m);

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
/* The input-projection matrix of a deeper layer exactly as fsn_model_finalize uploads it: [4 hidden, k_pad] fp16 whose row c gives
 * Gin column c, in the order the recurrent kernel reads (column j*128 + p*32 + cg*8 + q*2 + e = gate q of unit 32 j + 8 cg + 2 p + e). */
int fsn_tc5r_gin_weights(int32_t hidden, int32_t k_in, int32_t k_pad, const float* w_ih, uint16_t* h_wih);
/* Weight-ring slots (shared-memory plan) of the layer-wise kernel for one layer role: first = input projection in the recurrence,
 * last = fused output Linear.  FSN_EINVAL for a hidden size it does not take. */
int32_t fsn_tc5r_ring_stages(int32_t hidden, int32_t first, int32_t last);
/* Sequences per CTA (64, 32 or 16) the generic mma.sync kernel runs a stack of `layers` layers with (0: none fits). */
int32_t fsn_lstm_mma_rows(int32_t layers, int32_t hidden, int32_t input_pad, int32_t output_size);

/* Test hook: the sub-band LSTM / GRU stage of a finalized model alone, on a given sub-band input, through the forward's own layer and
 * window loop (GEMM dispatch, per-layer cell / hidden state, fused epilogues); only the packer differs.
 * d_x: [B, F, Isb, T + look_ahead] float32, device -- the normalised input sb_model receives (same layout as get_stage "sb_in"; any
 * Isb the model takes, up to 128);
 * rounded to fp16 (nearest) like the forward's packed input.
 * Tw: 0 = one launch per layer over all frames; else windows of Tw frames (positive multiple of 32; layer-wise path only).
 * h_frames: NULL or B host frame counts, as fsn_model_forward_ragged.  Output: d_out [B, 2, F, T] (mask), or, when d_enh != NULL,
 * the enhanced spectrum [B, F, T] complex64 from d_real / d_imag [B, F, T], as fsn_model_forward_enhance.
 * FSN_EINVAL for a sub-band TCN model, a bad window or frame count; FSN_ESTATE before fsn_model_finalize. */
int fsn_model_sb_forward(fsn_model* m, const float* d_x, int32_t B, int32_t T, int32_t Tw, const int32_t* h_frames,
                         float* d_out, const float* d_real, const float* d_imag, float* d_enh, void* stream);

/* The layer-wise path's input-projection GEMM alone (test / bench hook): d_c[M, N] = d_a[M, K] d_b[N, K]^T, fp16 row-major device
 * buffers, fp32 accumulation, enqueued on `stream`.  M % 128 == 0, N % 128 == 0, K % 64 == 0.  tile_n: 0 (or 256) = 128 x 256 tiles
 * on CTA pairs where N % 256 == 0 and M / 128 is even, else 128 x 128; 128 = always 128 x 128 (what FSN_GIN_GEMM=128 selects). */
int fsn_gemm_f16(const void* d_a, const void* d_b, void* d_c, int64_t M, int32_t N, int32_t K, int32_t tile_n, void* stream);
/* The N tile (128 or 256) fsn_gemm_f16 runs that shape with, or FSN_EINVAL for a shape it rejects; host only. */
int32_t fsn_gemm_f16_tile_n(int64_t M, int32_t N, int32_t K, int32_t tile_n);

/* ---- Speech metrics (DESIGN.md §3.20): no model, no weights ----------------------------------------------------------------
 * Objective scores of an estimate against its clean reference, one float64 score per clip.  d_ref and d_est are [B, L] float32 device
 * rows; clip b is the first h_lengths[b] samples of its rows (h_lengths == NULL: every clip is L samples).  No reduction crosses clips:
 * a clip's score is bit-identical whatever else is in the batch.  d_work is a device buffer of at least the bytes the matching
 * *_workspace call reports for the same B, L, h_lengths (and sr); the call enqueues on `stream` and returns before the scores exist.
 * Every argument is checked before any device work: FSN_EINVAL, naming the argument, for B outside 1 .. 65535, L outside
 * 1 .. 2^31 - 1, a clip length outside 1 .. L (naming the clip), sr outside 8000 .. 48000, a null pointer or too small a workspace. */

/* SI-SDR in dB: 10 log10(|a r|^2 / |e - a r|^2), a = <r, e> / <r, r>, accumulated in fp64 over two passes.  A silent reference
 * gives NaN, an estimate equal to the reference +inf (as the float64 formula does).  Workspace: B (16 ceil(max L_b / 16384) + 16)
 * bytes, rounded up. */
int fsn_metric_si_sdr_workspace(int32_t B, int64_t L, const int64_t* h_lengths, int64_t* bytes);
int fsn_metric_si_sdr(const float* d_ref, const float* d_est, int32_t B, int64_t L, const int64_t* h_lengths, void* d_work,
                      int64_t work_bytes, double* d_out, void* stream);

/* Classic STOI (Taal et al. 2011) as pystoi 0.3.3's stoi(ref, est, sr, extended=False) computes it: resampling to 10 kHz, removal of
 * the frames more than 40 dB below the reference's loudest, 15 one-third-octave band envelopes, 30-frame segments.  A clip with fewer
 * than 30 envelope frames after silent-frame removal, or with no frame at all, scores 1e-5.  Workspace: about 270 bytes per 128
 * samples at 10 kHz of the longest clip, per clip, plus the resampling filter. */
int fsn_metric_stoi_workspace(int32_t B, int64_t L, const int64_t* h_lengths, int32_t sr, int64_t* bytes);
int fsn_metric_stoi(const float* d_ref, const float* d_est, int32_t B, int64_t L, const int64_t* h_lengths, int32_t sr, void* d_work,
                    int64_t work_bytes, double* d_out, void* stream);

/* SDR in dB as BSS Eval v3 computes it for one source with a 512-tap distortion filter (mir_eval's bss_eval_sources; DESIGN.md
 * §3.21): with r, e zero-extended, R[k] = sum r[n] r[n + k], D[k] = sum r[n] e[n + k] (k < 512), G c = D for G[i][j] = R[|i - j|],
 * P = c * r over n < L_b + 511 and SDR = 10 log10(sum P^2 / sum (e' - P)^2), e' = e followed by 511 zeros.  fp64 throughout (a
 * Levinson solve per clip); no sample rate.  A silent reference or a silent estimate gives NaN, and so does a reference whose
 * Levinson recursion meets a prediction error that is not a positive finite number (numerically singular); a zero denominator gives
 * +inf.  Scores above 100 dB (est = ref, clips of a few samples) measure rounding noise.  Workspace: B (8192 ceil(max L_b / 3584)
 * + 16 ceil((max L_b + 511) / 4096) + 12296) bytes, each of its five segments rounded up to 256 bytes. */
int fsn_metric_sdr_workspace(int32_t B, int64_t L, const int64_t* h_lengths, int64_t* bytes);
int fsn_metric_sdr(const float* d_ref, const float* d_est, int32_t B, int64_t L, const int64_t* h_lengths, void* d_work,
                   int64_t work_bytes, double* d_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FSNPLUS_B200_H_ */
