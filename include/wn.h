/* wn.h — C ABI of libwn.so, the H100 (sm_90a) autoregressive WaveNet synthesis engine.
 *
 * This is the drop-in boundary for ONE path of r9y9/wavenet_vocoder: everything
 * WaveNet.incremental_forward() does per generated sample (reference wavenet.py:215-343),
 * i.e. the first 1x1 conv, the dilated gated residual stack with its cached queues
 * (modules.py:112-163, conv.py:17-46), the 1x1 head, and the output sampler
 * (mixture.py:118-156, :221-270, wavenet.py:332-335).  The reference has no FFI for this path
 * (it is pure Python on ATen); the entry points below are what a ctypes binding inside
 * wavenet_vocoder/wavenet.py would call instead of its Python loop -- see INTEGRATION.md.
 *
 * Conventions
 *   - plain C, no torch types.  All `const float*` marked DEVICE are CUDA device pointers on the
 *     handle's device; those marked HOST are ordinary host pointers.
 *   - every function returns 0 on success, a negative wn_status otherwise, and records a
 *     message retrievable with wn_last_error() (thread local).
 *   - one handle per GPU, one generate call in flight per handle (like the reference module,
 *     which owns its queues and is not re-entrant, wavenet.py:241,342).
 *   - there is NO CPU fallback: without a usable CUDA device wn_create() fails.
 */
#ifndef WN_H_
#define WN_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 3 = 2 plus streaming (wn_stream_*, wn_upsample_cone, wn_decode_stream); no struct of version 2 changed, and
 * wn_create accepts a wn_config that says 2 */
#define WN_ABI_VERSION 3

typedef enum wn_status {
    WN_OK = 0,
    WN_ERR_INVALID = -1,     /* bad argument / unsupported shape            */
    WN_ERR_CUDA = -2,        /* CUDA runtime error (message has the detail) */
    WN_ERR_STATE = -3,       /* call order (e.g. generate before weights)   */
    WN_ERR_DEVICE = -4,      /* kernel reported a fault or watchdog timeout */
    WN_ERR_NOMEM = -5
} wn_status;

/* input of the first 1x1 conv (wavenet.py:119-122) */
enum { WN_INPUT_SCALAR = 0, WN_INPUT_ONEHOT = 1 };
/* output head / sampler (wavenet.py:322-335) */
enum { WN_HEAD_MOL = 0,      /* sample_from_discretized_mix_logistic, mixture.py:118-156 */
       WN_HEAD_GAUSS = 1,    /* sample_from_mix_gaussian, mixture.py:221-270             */
       WN_HEAD_SOFTMAX = 2   /* softmax + OneHotCategorical, wavenet.py:332-335          */ };
/* sampler noise source */
enum { WN_NOISE_REPLAY = 0,  /* caller supplies the draws (bit-parity with torch's CPU RNG) */
       WN_NOISE_PHILOX = 1   /* counter-based generator on the device                       */ };

/* generate flags */
#define WN_FLAG_SOFTMAX   1u  /* wavenet.py:217 softmax=True  */
#define WN_FLAG_QUANTIZE  2u  /* wavenet.py:217 quantize=True */

/* Shape of the model == constructor arguments of the reference WaveNet (wavenet.py:98-111). */
typedef struct wn_config {
    int32_t abi_version;          /* WN_ABI_VERSION */
    int32_t layers;               /* L                                   */
    int32_t stacks;               /* dilation cycles; d_l = 2^(l mod L/stacks), wavenet.py:125-126 */
    int32_t residual_channels;    /* R */
    int32_t gate_channels;        /* G (even) */
    int32_t skip_channels;        /* S */
    int32_t out_channels;         /* O */
    int32_t kernel_size;          /* kw >= 1 */
    int32_t cin_channels;         /* C, 0 = no local conditioning  */
    int32_t gin_channels;         /* gin, 0 = no global conditioning */
    int32_t input_kind;           /* WN_INPUT_*  */
    int32_t head_kind;            /* WN_HEAD_*   */
    int32_t device;               /* CUDA ordinal */
    int32_t num_ctas;             /* 0 = choose; else number of cooperating thread blocks */
    int32_t exchange_copies;      /* 0 = choose; replicas of each exchange vector in L2   */
    int32_t ring_slots;           /* 0 = choose; streaming weight slots in shared memory  */
    int32_t poll_warps;           /* 0 = choose; warps that poll the exchange into shared memory (2..12) */
    int32_t reserved[7];
} wn_config;

/* One residual layer, HOST pointers, fp32, weight-norm already folded (modules.py:13-18).
 * conv_w is linearised exactly as conv.py:51-62: (G, kw*R), column k*R + r, tap k=0 oldest. */
typedef struct wn_layer_weights {
    const float* conv_w;   /* (G, kw*R) */
    const float* conv_b;   /* (G)       */
    const float* cond_w;   /* (G, C)   or NULL, no bias (modules.py:94)  */
    const float* gcond_w;  /* (G, gin) or NULL, no bias (modules.py:100) */
    const float* out_w;    /* (R, G/2) */
    const float* out_b;    /* (R)      */
    const float* skip_w;   /* (S, G/2) */
    const float* skip_b;   /* (S)      */
} wn_layer_weights;

typedef struct wn_weights {
    const float* first_w;    /* (R, 1) scalar input or (R, O) one-hot input, wavenet.py:119-122 */
    const float* first_b;    /* (R) */
    const float* last_a_w;   /* (S, S)  last_conv_layers[1], wavenet.py:136-141 */
    const float* last_a_b;   /* (S)  */
    const float* last_b_w;   /* (O, S)  last_conv_layers[3] */
    const float* last_b_b;   /* (O)  */
    const wn_layer_weights* layers;   /* [L] */
} wn_weights;

/* One synthesis call == one WaveNet.incremental_forward() (wavenet.py:215-343).
 * All pointers are DEVICE pointers unless noted; NULL where not applicable. */
typedef struct wn_generate_args {
    int32_t B;                 /* utterances (rows of the batch); any B >= 1               */
    int32_t T;                 /* samples to generate per utterance                         */
    const float* c;            /* (B,T,C) local conditioning at SAMPLE rate (after upsample, wavenet.py:272-278) */
    const float* c_frames;     /* or: (B,C,n_frames) conditioning FRAMES, upsampled on the device by the network given to
                                  wn_load_upsampler (upsample.py:29-85, wavenet.py:274-276); exclusive with `c`          */
    int32_t n_frames;
    const float* g;            /* (B,gin) global conditioning vector (after embedding, wavenet.py:263-268)       */
    const float* initial;      /* scalar input: (B) ; one-hot input: NULL (default index) -- wavenet.py:281-292   */
    int32_t initial_index;     /* one-hot input: start class (reference default 127, wavenet.py:286); <0 = 127     */
    const int32_t* initial_rows;   /* one-hot input: (B) start class per utterance, overrides initial_index; or NULL */
    const float* initial_dense;    /* one-hot input: (B,O) dense start vector fed as is (wavenet.py:281-292); or NULL */
    int32_t T_test;            /* teacher-forcing length (wavenet.py:247-258), 0 = free running                    */
    const float* test_scalar;  /* scalar input: (B,T_test)                                   */
    const int32_t* test_index; /* one-hot input given as class ids: (B,T_test)               */
    const float* test_dense;   /* one-hot input given as dense rows: (B,T_test,O)            */
    uint32_t flags;            /* WN_FLAG_*                                                   */
    int32_t noise_kind;        /* WN_NOISE_*                                                  */
    uint64_t seed;             /* WN_NOISE_PHILOX                                             */
    const float* noise_u1;     /* REPLAY: (T,B,K) uniforms for the mixture pick, mixture.py:138   */
    const float* noise_u2;     /* REPLAY: (T,B) uniforms for the logistic draw, mixture.py:151    */
    const float* noise_z;      /* REPLAY: (T,B) standard normals, mixture.py:265-267              */
    const float* noise_e;      /* REPLAY: (T,B,O) Exp(1) draws of multinomial, wavenet.py:334-335 */
    float* out_scalar;         /* scalar input: (B,T) samples in [-1,1]                       */
    int32_t* out_index;        /* one-hot input + QUANTIZE: (B,T) sampled class               */
    float* out_dense;          /* one-hot input, no QUANTIZE: (B,O,T) probabilities / logits  */
    float* params_out;         /* optional (B,O,T): head output per step (sampler input)      */
    void* stream;              /* cudaStream_t, NULL = default stream                         */
    int32_t philox_row0;       /* WN_NOISE_PHILOX: utterance b of this call draws the noise of row philox_row0 + b
                                * (a batch split over several handles / calls then draws what one call would)  */
    int32_t reserved[7];
} wn_generate_args;

/* What the planner decided (for tests, DESIGN.md numbers and the roofline arithmetic). */
typedef struct wn_plan_info {
    int32_t num_ctas, threads_per_cta, batch_tile;
    int32_t rows_y, rows_x, rows_skip, rows_head_a, rows_head_b;   /* max rows owned per CTA */
    int32_t resident_blobs, ring_slots, blobs_per_step;
    int32_t exchange_copies, exchanges_per_step;
    int32_t rings_in_smem;
    int64_t smem_bytes, layer_blob_bytes, head_blob_bytes, packed_bytes_per_cta;
    int64_t weight_bytes_per_step;     /* algorithmic fp32 weight bytes one step must touch */
    int64_t flops_per_sample;          /* 2*MAC per generated sample per utterance           */
    int64_t streamed_bytes_per_step;   /* bytes the TMA pipeline moves per step (all CTAs)   */
    int64_t launches;                  /* kernels launched by this handle so far             */
    int64_t cond_packed_bytes_per_cta; /* size of the conditioning-weight image of one block */
    int64_t bias_packed_bytes_per_cta; /* size of the bias image of one block (cluster engine) */
    int64_t num_clusters, cluster_size, num_passes, engine;   /* clusters are not used by the current engine: P, 1 */
    int64_t poll_warps;
} wn_plan_info;

int32_t wn_abi_version(void);
/* sizeof() of the structs of this header as the library was compiled, in the order wn_config, wn_weights,
 * wn_generate_args, wn_plan_info, wn_upsampler, wn_stream_open_args, wn_stream_chunk; n = capacity of `out`, the
 * return value the number written.  Lets a binding
 * that transcribes the structs (ctypes, cgo, JNI) check its layout before the first real call. */
int32_t wn_struct_sizes(int32_t* out, int32_t n);
const char* wn_last_error(void);

/* Create an engine for one model shape on one GPU.  Fails (WN_ERR_CUDA) without a device. */
int32_t wn_create(const wn_config* cfg, void** handle);
int32_t wn_destroy(void* handle);

/* Upload weights (HOST fp32, folded).  Packs them per thread block and copies to the device. */
int32_t wn_load_weights(void* handle, const wn_weights* w);

/* Local-conditioning upsampler (reference upsample.py): optional conv_in over frames, then per scale a
 * nearest-neighbour stretch and a 1 x (2s+1) smoothing filter shared by all channels.  HOST pointers, weight norm
 * already folded.  Only the common configuration is supported natively (freq_axis_kernel_size 1, no activation,
 * nearest mode, every scale >= 2); callers keep other variants on their own side and pass `c`. */
typedef struct wn_upsampler {
    int32_t channels;          /* C (== cin_channels)                                                      */
    int32_t n_scales;          /* <= 8                                                                     */
    const int32_t* scales;     /* [n_scales] upsample_scales                                               */
    const float* filters;      /* concatenated smoothing filters, 2*s_j+1 taps each (Conv2d weight (1,1,1,2s+1)) */
    const float* conv_in_w;    /* (C,C,conv_in_ks) ConvInUpsampleNetwork.conv_in.weight, or NULL           */
    int32_t conv_in_ks;        /* 2*cin_pad+1, or 0                                                        */
    int32_t indent;            /* samples trimmed at both ends: cin_pad*prod(scales) for UpsampleNetwork, else 0 */
    int32_t reserved[5];
} wn_upsampler;
int32_t wn_load_upsampler(void* handle, const wn_upsampler* u);
/* Run only the upsampler: c_frames (B,C,n_frames) -> out (B,T,C), DEVICE pointers, T = upsampled length. */
int32_t wn_upsample(void* handle, const float* c_frames, int32_t B, int32_t n_frames, int32_t T, float* out,
                    void* stream);

/* Decode synthesis output to audio (synthesis.py:66-84 + evaluate.py:43-48,247-251): inverse mu-law for
 * input_type 1 ("mulaw", y_scalar) / 2 ("mulaw-quantize", y_index), nothing for 0 ("raw"); then
 * inv_preemphasis (preemphasis_coef != 0), division by global_gain_scale (> 0), and -- for out_pcm16 -- trimming to
 * lengths[b] (zeros beyond), clip to [-1,1] and (x*32767) truncated to int16.  DEVICE pointers; (B,T) each. */
enum { WN_DECODE_RAW = 0, WN_DECODE_MULAW = 1, WN_DECODE_MULAW_QUANTIZE = 2 };
int32_t wn_decode(const float* y_scalar, const int32_t* y_index, int32_t B, int32_t T, const int32_t* lengths,
                  int32_t input_type, int32_t quantize_channels, float preemphasis_coef, float global_gain_scale,
                  float* out_float, int16_t* out_pcm16, void* stream);

/* Run one synthesis call; returns after the launch is enqueued on args->stream.
 * wn_sync() waits for it and reports a device-side fault/timeout as WN_ERR_DEVICE. */
int32_t wn_generate(void* handle, const wn_generate_args* args);
int32_t wn_sync(void* handle);

/* Same call with HOST buffers everywhere a DEVICE pointer is expected above (inputs are copied
 * in, results copied out, synchronous). */
int32_t wn_generate_host(void* handle, const wn_generate_args* args);

int32_t wn_get_plan(void* handle, int32_t batch, wn_plan_info* out);

/* ---- Streaming (ABI 3): one utterance made in consecutive chunks, bit-identical to one wn_generate call over the
 * whole utterance with the same weights, noise and conditioning, for any split.  What links step t to step t+1 --
 * the older-tap history rings, the fed-back sample, the Philox step -- stays in a device buffer the stream owns.
 * Engine 5 only, at most one batch tile (4 utterances), no teacher forcing.  Several streams may be open on one
 * handle and called in turn; the handle still runs one call at a time, and wn_sync(handle) waits for a chunk. */
typedef struct wn_stream_open_args {
    int32_t B;                     /* utterances, 1..4                                                             */
    const float* g;                /* DEVICE (B,gin) or NULL; read once, at open                                    */
    const float* initial;          /* DEVICE, as wn_generate_args; copied at open                                   */
    int32_t initial_index;
    const int32_t* initial_rows;
    const float* initial_dense;
    uint32_t flags;                /* WN_FLAG_*                                                                     */
    int32_t noise_kind;            /* WN_NOISE_*: PHILOX draws the noise of the absolute step; REPLAY takes each
                                      chunk's (T,B,.) rows from the chunk's wn_generate_args                        */
    uint64_t seed;
    int32_t philox_row0;
    void* stream;                  /* cudaStream_t of the open (it returns after the set-up is complete)            */
    int32_t reserved[6];
} wn_stream_open_args;

/* Where a chunk's conditioning FRAMES (wn_generate_args.c_frames, n_frames of them) sit in the utterance. */
typedef struct wn_stream_chunk {
    int64_t frame_offset;          /* utterance frame index of c_frames[..., 0]                                      */
    int64_t frames_total;          /* frames of the utterance received so far                                       */
    int32_t final;                 /* 1: frames_total is the whole utterance; no chunk may follow this one          */
    int32_t reserved[5];
} wn_stream_chunk;

int32_t wn_stream_open(void* handle, const wn_stream_open_args* args, void** stream);
/* Generate the next chunk->T samples.  chunk: B as opened; T; c (B,T,C) sample-rate conditioning of these samples
 * or c_frames + n_frames with `where`; replay noise (T,B,.); outputs and params_out (B,.,T) of this chunk;
 * g, initial*, T_test and test_* unset.  `where` may be NULL without c_frames (then it can still mark the end).
 * WN_ERR_STATE after wn_load_weights changed the handle's weights or after a final chunk. */
int32_t wn_stream_generate(void* stream, const wn_generate_args* chunk, const wn_stream_chunk* where);
/* Absolute step of the next sample (samples generated so far). */
int64_t wn_stream_position(void* stream);
int32_t wn_stream_close(void* stream);

/* Device-less: the conditioning frames [*f_lo, *f_hi) that samples [t_lo, t_hi) of an utterance need, given n_frames
 * received (final = 1: that is all of them), and *n_ready = how many samples from the start are known from those
 * frames whatever follows (for final, the upsampled length).  Only scales, conv_in_ks and indent of `u` are read.  */
int32_t wn_upsample_cone(const wn_upsampler* u, int64_t n_frames, int32_t final, int64_t t_lo, int64_t t_hi,
                         int64_t* f_lo, int64_t* f_hi, int64_t* n_ready);

/* wn_decode over one chunk of an utterance: `carry` (DEVICE, B floats, zero before the first chunk) holds the
 * inv_preemphasis recursion between chunks; lengths are relative to the chunk. */
int32_t wn_decode_stream(const float* y_scalar, const int32_t* y_index, int32_t B, int32_t T, const int32_t* lengths,
                         int32_t input_type, int32_t quantize_channels, float preemphasis_coef, float global_gain_scale,
                         float* out_float, int16_t* out_pcm16, float* carry, void* stream);

/* Device-less planning + packing, for host-logic tests and tooling: computes the plan for
 * `cfg` assuming `num_sms` SMs / `smem_per_cta` bytes, and (if `packed` != NULL) writes the
 * packed weight image of thread block `cta` into `packed`: packed_bytes_per_cta bytes (layer
 * blobs + head blob) followed, if the buffer has room, by cond_packed_bytes_per_cta bytes (the
 * local-conditioning rows the conditioning warp reads from L2) and bias_packed_bytes_per_cta bytes
 * (biases of the rows the block owns). */
int32_t wn_plan_only(const wn_config* cfg, int32_t batch, int32_t num_sms, int64_t smem_per_cta,
                     wn_plan_info* out);
int32_t wn_pack_cta(const wn_config* cfg, int32_t batch, int32_t num_sms, int64_t smem_per_cta,
                    const wn_weights* w, int32_t cta, float* packed, int64_t packed_floats);

/* The raw execution plan (struct Wn7Plan of csrc/wn7_plan.h as int32 words) and its pass table (struct Wn7Pass,
 * 12 bytes each), for tools and the host tests that replay the packed image.
 * Returns the number of passes (>= 0) or a negative wn_status. */
int32_t wn_plan_passes(const wn_config* cfg, int32_t batch, int32_t num_sms, int64_t smem_per_cta,
                       int32_t* plan_words, int32_t max_plan_words, void* passes, int32_t max_passes);

/* ---- Teacher-forced scoring (added in ABI 3 without changing WN_ABI_VERSION or any struct: wn_struct_sizes still
 * reports 7 structs; a binding detects these two entry points by their presence in the library).
 *
 * Teacher-forced batch forward (reference WaveNet.forward): writes params_out (B,O,T), the head output a fully
 * teacher-forced wn_generate would write, computed in parallel over time (dense 3xTF32 GEMMs, csrc/wn_dense.cuh).
 * Reads B, T, T_test (== T) and exactly one of test_scalar / test_index / test_dense; c or c_frames (through the loaded
 * upsampler) and g as wn_generate does; flags (WN_FLAG_SOFTMAX only: a softmax over O); params_out; stream.  Refused
 * with WN_ERR_INVALID: any noise_* or out_* pointer, initial / initial_rows / initial_dense, T_test != T.
 * initial_index is not read.  Returns after the launches are enqueued; wn_sync(handle) waits for them.  The activation
 * scratch grows as needed (WN_ERR_NOMEM says how many bytes were needed). */
int32_t wn_forward(void* handle, const wn_generate_args* a);
/* Per-sample negative log-likelihood of y_target (B,T) [MoL, Gauss] or class_target (B,T) [softmax] under the
 * head outputs y_bot (B,O,T); DEVICE pointers; out (B,T).  The reference's discretized_mix_logistic_loss
 * (mixture.py:26-106, num_classes and log_scale_min as given), mix_gaussian_loss (mixture.py:161-218) and the
 * cross-entropy of the softmax head (train.py:346-362), each with reduce=False.  num_classes >= 2 (read by MoL only);
 * a class outside [0,O) gives NaN.  The arguments are checked before the device is touched. */
int32_t wn_nll(const float* y_bot, int32_t head_kind, int32_t B, int32_t O, int32_t T, const float* y_target,
               const int32_t* class_target, int32_t num_classes, float log_scale_min, float* out_bt, void* stream);

/* Stand-alone samplers over a (B,O,T) head-output tensor (DEVICE), the reference's
 * mixture.py entry points; noise is REPLAY layout with T as given. out: (B,T). */
int32_t wn_sample_mol(const float* y_bot, int32_t B, int32_t O, int32_t T,
                      const float* u1_tbk, const float* u2_tb, float* out_bt, void* stream);
int32_t wn_sample_gauss(const float* y_bot, int32_t B, int32_t O, int32_t T,
                        const float* u1_tbk, const float* z_tb, float* out_bt, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* WN_H_ */
