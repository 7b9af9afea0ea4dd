/*
 * sopro_b200 — C-ABI of the H100-native Sopro hot path.
 *
 * The reference (samuel-vitorino/sopro) is pure Python/PyTorch and has no FFI;
 * every entry point below names the reference interface it replaces
 * (paths relative to the reference's src/sopro/).  Plain pointers and sizes
 * only, no torch types.  Unless a parameter says "host", pointers are CUDA
 * device pointers owned by the caller; `stream` is a cudaStream_t passed as
 * void* (NULL = legacy default stream).  Every function returns 0 on success
 * or a negative sopro_status; sopro_last_error() gives the message for the
 * calling thread.  There is no CPU fallback: creating an engine on a device
 * that is not sm_90 fails.
 */
#ifndef SOPRO_B200_H_
#define SOPRO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SOPRO_MAX_AR_LAYERS 16

enum sopro_status {
  SOPRO_OK = 0,
  SOPRO_ERR_INVALID = -1,     /* bad argument / unsupported geometry */
  SOPRO_ERR_CUDA = -2,        /* a CUDA runtime call failed */
  SOPRO_ERR_UNSUPPORTED = -3, /* device is not sm_90, or feature not built */
  SOPRO_ERR_STATE = -4        /* call out of order */
};

enum sopro_wdtype { SOPRO_W_F32 = 0, SOPRO_W_BF16 = 1 };

/* Geometry of the AR generator.  Replaces the fields of SoproTTSConfig the AR
 * path reads (config.py:14-27) + the literals in nn/generator.py:12-42. */
typedef struct sopro_ar_config {
  int32_t d_model;                          /* cfg.d_model (384) */
  int32_t n_layers;                         /* cfg.n_layers_ar (6) */
  int32_t kernel;                           /* cfg.ar_kernel (13) */
  int32_t n_heads;                          /* 4, nn/generator.py:36 */
  int32_t vocab;                            /* codebook_size + 1 (2049), model.py:83 */
  int32_t eos_id;                           /* codebook_size, model.py:59 */
  int32_t dilation[SOPRO_MAX_AR_LAYERS];    /* nn/generator.py:16-20 */
  int32_t has_attn[SOPRO_MAX_AR_LAYERS];    /* 1 if a TextXAttnBlock follows block i */
  int32_t weight_dtype;                     /* sopro_wdtype: storage of the matrices */
} sopro_ar_config_t;

/* HOST pointers to fp32 tensors in the reference's state_dict layout. */
typedef struct sopro_ar_layer_weights {
  const float* norm_w;    /* ar.blocks.i.norm.weight      [D]        nn/blocks.py:123 */
  const float* glu_w;     /* ar.blocks.i.glu.pro.weight   [2D, D]    nn/blocks.py:19 */
  const float* glu_b;     /* ar.blocks.i.glu.pro.bias     [2D] */
  const float* dw_w;      /* ar.blocks.i.dw.dw.weight     [D, 1, k]  nn/blocks.py:48 */
  const float* dw_b;      /* ar.blocks.i.dw.dw.bias       [D] */
  const float* ffn_norm_w;/* ar.blocks.i.ff.0.weight      [D]        nn/blocks.py:129 */
  const float* ffn_w1;    /* ar.blocks.i.ff.1.weight      [4D, D] */
  const float* ffn_b1;    /* ar.blocks.i.ff.1.bias        [4D] */
  const float* ffn_w2;    /* ar.blocks.i.ff.3.weight      [D, 4D] */
  const float* ffn_b2;    /* ar.blocks.i.ff.3.bias        [D] */
  /* cross-attention after block i (NULL when has_attn[i] == 0)  nn/text.py:57-65 */
  const float* nq_w;      /* ar.x_attns.i.nq.weight       [D] */
  const float* nkv_w;     /* ar.x_attns.i.nkv.weight      [D] */
  const float* q_w;       /* ar.x_attns.i.q_proj.weight   [D, D] */
  const float* k_w;       /* ar.x_attns.i.k_proj.weight   [D, D] */
  const float* v_w;       /* ar.x_attns.i.v_proj.weight   [D, D] */
  const float* o_w;       /* ar.x_attns.i.out_proj.weight [D, D] */
  float gate_tanh;        /* tanh(ar.x_attns.i.gate), evaluated by the caller in fp32 (nn/text.py:131) */
} sopro_ar_layer_weights_t;

typedef struct sopro_ar_weights {
  sopro_ar_layer_weights_t layer[SOPRO_MAX_AR_LAYERS];
  const float* final_norm_w; /* ar.norm.weight  [D]      nn/generator.py:41 */
  const float* head_w;       /* ar.head.weight  [V, D]   nn/generator.py:42 */
  const float* head_b;       /* ar.head.bias    [V] */
  const float* cb_embed;     /* cb_embed.emb.weight [Q*V'+1, D]  nn/embeddings.py:47-49 */
  int64_t cb_embed_rows;     /* Q*codebook_size + 1 */
  int64_t bos_row;           /* Q*codebook_size, nn/embeddings.py:49 */
} sopro_ar_weights_t;

/* Per-utterance sampling knobs: kwargs of SoproTTSModel.ar_stream (model.py:218-231)
 * plus the literals it passes to sample_token (model.py:284-291). */
typedef struct sopro_ar_sampling {
  float top_p;               /* 0.9 */
  float temperature;         /* 1.05 */
  float recovery_top_p;      /* 0.85 */
  float recovery_temp;       /* 1.2 */
  float repetition_penalty;  /* 1.1 */
  int32_t top_k;             /* 50; must be in [1, 64] */
  int32_t anti_loop;         /* 1 */
  int32_t loop_streak;       /* 8 */
  int32_t min_gen_frames;    /* cfg.min_gen_frames (12) */
  int32_t stop_on_first_eos; /* 1 = what generate_tokens/stream consumers do (model.py:382-383,
                                streaming.py:114-115); 0 = ar_stream's own rule (model.py:304) */
} sopro_ar_sampling_t;

typedef struct sopro_engine sopro_engine_t;
typedef struct sopro_ar_session sopro_ar_session_t;

const char* sopro_last_error(void);
const char* sopro_version(void);

/* Engine = device-resident copy of the AR step weights (converted to
 * cfg->weight_dtype).  Replaces SoproTTSModel.ar + cb_embed residency after
 * SoproTTS.from_pretrained (model.py:443-446). */
int sopro_engine_create(const sopro_ar_config_t* cfg, const sopro_ar_weights_t* host_weights,
                        int device, sopro_engine_t** out);
int sopro_engine_destroy(sopro_engine_t* e);
/* bytes of step-resident weights as stored on the device (W_step of SURVEY.md §8d) */
int64_t sopro_engine_step_weight_bytes(const sopro_engine_t* e);
int sopro_engine_num_sms(const sopro_engine_t* e);

/* Session = state of a batch of independent utterances: conv ring buffers, text
 * K/V, history, outputs.  Replaces ARRVQ1Generator.init_stream_state
 * (nn/generator.py:44-68) and the locals of ar_stream (model.py:242-255). */
int sopro_ar_session_create(sopro_engine_t* e, int max_batch, int max_steps, int max_text_len,
                            sopro_ar_session_t** out);
int sopro_ar_session_destroy(sopro_ar_session_t* s);

/* Launch geometry override (0 = automatic): utterances per CTA team. */
int sopro_ar_session_set_team(sopro_ar_session_t* s, int utts_per_team);

/* Start `batch` utterances.  Zeroes the rings, builds the text K/V caches on the
 * device (TextXAttnBlock.build_kv_cache, nn/text.py:75-83), resets history.
 *   cond_ar   [batch, steps, D] f32   prep["cond_ar"] rows 0..steps-1 (model.py:272)
 *   txt_seq   [batch, text_stride, D] f32   prep["txt_seq"], padded to text_stride rows
 *   text_len  [batch] i32 HOST        valid rows per utterance (text_mask, model.py:186)
 *   noise     [batch, steps, noise_k] f32   Exp(1) draws: what torch.multinomial would
 *             consume at each step, q of argmax(p/q); noise_k >= top_k when top_p < 1
 *             (rank-aligned, sampling.py:83-84), noise_k >= vocab otherwise (sampling.py:93)
 *   sampling  [batch] HOST
 */
int sopro_ar_begin(sopro_ar_session_t* s, int batch, int steps, const float* cond_ar,
                   const float* txt_seq, int text_stride, const int32_t* text_len,
                   const float* noise, int noise_k, const sopro_ar_sampling_t* sampling,
                   void* stream);

/* Advance every live utterance by up to n_steps frames (the body of the
 * `for t in range(max_steps)` loop, model.py:265-305) in ONE persistent kernel.
 * Asynchronous on `stream`. Returns after enqueueing. */
int sopro_ar_run(sopro_ar_session_t* s, int n_steps, void* stream);

/* Device views of the outputs (valid until the session is destroyed):
 *   tokens   [batch, steps] i32   token per step: what ar_stream yields (model.py:302)
 *   n_tokens [batch] i32          steps taken so far;   done [batch] i32 */
int sopro_ar_outputs(sopro_ar_session_t* s, const int32_t** tokens, const int32_t** n_tokens,
                     const int32_t** done);
/* Synchronous copy to HOST buffers (tokens row stride = steps given to begin). */
int sopro_ar_read(sopro_ar_session_t* s, int32_t* tokens_host, int32_t* n_tokens_host,
                  int32_t* done_host, void* stream);
/* steps the slowest live utterance has reached (host value, after the last run completes) */
int sopro_ar_position(sopro_ar_session_t* s);

/* One-call host-buffer path (what a ctypes/cgo caller with numpy-like buffers uses;
 * bench.py's e2e leg): H2D of cond/text/noise, begin, run to completion, D2H of
 * tokens, synchronises `stream`.  All pointers HOST. */
int sopro_ar_generate_host(sopro_ar_session_t* s, int batch, int steps, const float* cond_ar,
                           const float* txt_seq, int text_stride, const int32_t* text_len,
                           const float* noise, int noise_k, const sopro_ar_sampling_t* sampling,
                           int32_t* tokens_out, int32_t* n_tokens_out, void* stream);

/* ---- host-side noise tapes --------------------------------------------------------------------------------------
 * The Exp(1) draws torch.multinomial consumes on the CPU (reference sampling.py:83-93: multinomial == argmax(p / q),
 * q ~ Exp(1) from torch's CPU generator, `vocab` draws per step), reproduced bit for bit by a host-side mt19937 for a
 * PRIVATE generator seeded like torch.manual_seed(seed).  Only the first `keep` columns of each [vocab] row are
 * materialised (the sampler reads top_k of them); the generator still advances by the whole row.  Pure host code. */
typedef struct sopro_noise sopro_noise_t;
int sopro_noise_create(uint64_t seed, sopro_noise_t** out);
/* next n_rows rows of the tape -> out [n_rows, keep] f32 (host) */
int sopro_noise_rows(sopro_noise_t* g, int n_rows, int vocab, int keep, float* out);
int sopro_noise_destroy(sopro_noise_t* g);

/* ---- test / debug hooks (used by tests/, not by the product path) ---- */
/* teacher forcing: token fed back at step t is forced[b, t]; the sampled one goes to
 * `sampled` (sopro_ar_debug_sampled).  NULL disables. [batch, steps] i32 device. */
int sopro_ar_set_forced_tokens(sopro_ar_session_t* s, const int32_t* forced);
/* trace_blocks [steps, n_layers, batch, D] f32 (residual stream after block i incl. its
 * cross-attention), trace_logits [steps, batch, V] f32; NULL disables. device. */
int sopro_ar_set_trace(sopro_ar_session_t* s, float* trace_blocks, float* trace_logits);
/* clock64 stamps of one step: buf [grid, 224] i64 device (grid = SM count): one stamp at step
 * start, then five per stage (activations staged, weight tiles done, whole CTA done, barrier
 * arrival posted, barrier released). NULL = off */
int sopro_ar_set_timing(sopro_ar_session_t* s, int64_t* buf, int step);
/* word timestamps: every later launch stores the text cross-attention weights it applies into probs (device f32,
 * [steps][n_attn][batch][H][ld], n_attn = the attention layers in ascending order): for every step it computes and every
 * key l < text_len[b], exp(s_l - max) / sum, a non-finite weight stored as 0.  Entries at l >= text_len[b], and steps a
 * launch skips (every utterance of a team done), are not written.  The sampled tokens do not change.  NULL = off.
 * ld < 1 with a buffer is SOPRO_ERR_INVALID; sopro_ar_begin and sopro_ar_run refuse ld < the batch's longest text
 * (SOPRO_ERR_INVALID, before any launch). */
int sopro_ar_set_attn_trace(sopro_ar_session_t* s, float* probs, int64_t ld);
/* the same into a ring of `ring` step rows: step t goes to row t % ring of probs [ring][n_attn][batch][H][ld] (a stream
 * consumes each launch's rows before the next launch overwrites them).  sopro_ar_set_attn_trace is the case ring =
 * the session's steps.  ring < 1 with a buffer is SOPRO_ERR_INVALID; sopro_ar_run refuses a launch of more than `ring`
 * steps (SOPRO_ERR_INVALID, before any launch). */
int sopro_ar_set_attn_trace_ring(sopro_ar_session_t* s, float* probs, int64_t ld, int32_t ring);
/* warp task shape of the GEMV stages of later launches: 0 = picked per stage from the launch geometry (the default),
 * 1 = always R rows x TU utterances (wide), 2 = R x TU/2 (narrow) in every GEMV stage but GLU (teams of one utterance
 * stay wide).  The outputs are bit-identical in every mode. */
int sopro_ar_session_set_task_shape(sopro_ar_session_t* s, int mode);
/* the stage program of the last launch: kinds[i] (0 GLU, 1 FFN1, 2 FFN2, 3 Q, 4 O, 5 HEAD, 6 ATT, 7 SAMPLE, 8 fused
 * Q+ATT) and shapes[i] (0 wide, 1 narrow) of its first min(cap, *n_stage) stages; *n_stage = 0 before any launch.  HOST. */
int sopro_ar_session_stage_shapes(sopro_ar_session_t* s, int32_t* kinds, int32_t* shapes, int cap, int32_t* n_stage);
/* copy the sampled (pre-forcing) tokens into dst [batch, steps] i32 (device) */
int sopro_ar_debug_sampled(sopro_ar_session_t* s, int32_t* dst, void* stream);
/* copy the text K/V built by sopro_ar_begin into k_dst / v_dst, each
 * [n_attn_layers, batch, H, Lpad, Dh] f32 (device), Lpad = max_text_len rounded up to 4 */
int sopro_ar_debug_kv(sopro_ar_session_t* s, float* k_dst, float* v_dst, void* stream);
/* Host-only view of an operand image the NAR engine builds (no device needed): W6 [N][6K] of W [N][K] (bf16 terms of the
 * six product pairs mm, lh, hl, mh, hm, hh). */
int sopro_debug_pack_w6(const float* W, int N, int K, uint16_t* out);
/* The kernel's sampler (sample_token, sampling.py:24-93) on ONE logits row, outside the step: HOST buffers; `hist` = the
 * n_hist tokens generated so far (repetition penalty looks at the last 50), `noise` = the Exp(1) draws of this step (first
 * noise_k columns of the tape row: >= top_k when top_p < 1, vocab otherwise), `recovery` != 0 samples with the recovery
 * (top_p, temperature).  -> token_out.  Needs a device but no engine. */
int sopro_debug_sample(const float* logits, int vocab, const int32_t* hist, int n_hist, const float* noise, int noise_k,
                       const sopro_ar_sampling_t* sampling, int recovery, int device, int32_t* token_out);


/* ======================= Mimi codec decode (codes -> waveform) =======================
 * Replaces transformers.MimiModel.decode as the reference calls it: MimiCodec.decode_full
 * (codec/mimi.py:65-72) and, through it, MimiStreamDecoder.decode_step (codec/mimi.py:115-181).
 * Citations below are transformers/models/mimi/modeling_mimi.py (5.5.0). */
#define SOPRO_MIMI_MAX_LAYERS 16
#define SOPRO_MIMI_MAX_RATIOS 8

typedef struct sopro_mimi_config {
  int32_t hidden;        /* 512  MimiConfig.hidden_size */
  int32_t codebook_dim;  /* 256  (hidden == 2*codebook_dim: the two 1x1 output projections are fused) */
  int32_t n_q;           /* 32   num_quantizers */
  int32_t n_sem;         /* 1    num_semantic_quantizers */
  int32_t vocab;         /* 2048 codebook_size */
  int32_t n_layers;      /* 8 */
  int32_t n_heads;       /* 8 */
  int32_t ffn;           /* 2048 intermediate_size */
  int32_t window;        /* 250  sliding_window */
  int32_t num_filters;   /* 64 */
  int32_t kernel;        /* 7 */
  int32_t last_kernel;   /* 3 */
  int32_t res_kernel;    /* 3 */
  int32_t compress;      /* 2 */
  int32_t n_ratios;      /* 4 */
  int32_t ratios[SOPRO_MIMI_MAX_RATIOS]; /* 8,6,5,4 */
  float norm_eps;        /* 1e-5 */
  float rope_theta;      /* 10000 */
} sopro_mimi_config_t;

/* HOST fp32 pointers, state_dict layouts. */
typedef struct sopro_mimi_layer_weights {
  const float *ln1_w, *ln1_b;            /* input_layernorm                 :933 */
  const float *q_w, *k_w, *v_w, *o_w;    /* self_attn.*_proj.weight [C,C]    :676-679 */
  const float* ls1;                      /* self_attn_layer_scale.scale     :935 */
  const float *ln2_w, *ln2_b;            /* post_attention_layernorm        :934 */
  const float *fc1_w, *fc2_w;            /* mlp.fc1 [F,C], mlp.fc2 [C,F] */
  const float* ls2;                      /* mlp_layer_scale.scale */
} sopro_mimi_layer_weights_t;

typedef struct sopro_mimi_stage_weights {
  const float *convt_w, *convt_b;        /* decoder.layers.{i}.conv: ConvTranspose1d [Cin, Cout, 2r], [Cout] */
  const float *res1_w, *res1_b;          /* ...block.1.conv [Cout/2, Cout, 3] */
  const float *res2_w, *res2_b;          /* ...block.3.conv [Cout, Cout/2, 1] */
} sopro_mimi_stage_weights_t;

typedef struct sopro_mimi_weights {
  const float* embed;         /* [n_q, vocab, codebook_dim]: embed_sum / clamp(cluster_usage, 1e-5)  (:1192-1196),
                                 semantic codebooks first, then acoustic */
  const float* sem_out_proj;  /* quantizer.semantic_residual_vector_quantizer.output_proj.weight [C, Dc] */
  const float* ac_out_proj;   /* quantizer.acoustic_...output_proj.weight [C, Dc] */
  const float* upsample_w;    /* upsample.conv.weight [C, 1, 4] */
  sopro_mimi_layer_weights_t layer[SOPRO_MIMI_MAX_LAYERS];
  const float *conv0_w, *conv0_b; /* decoder.layers.0.conv [16F, C, 7] */
  sopro_mimi_stage_weights_t stage[SOPRO_MIMI_MAX_RATIOS];
  const float *last_w, *last_b;   /* decoder.layers.14.conv [1, F, 3] */
} sopro_mimi_weights_t;

typedef struct sopro_mimi sopro_mimi_t;

int sopro_mimi_create(const sopro_mimi_config_t* cfg, const sopro_mimi_weights_t* host_weights, int device,
                      sopro_mimi_t** out);
int sopro_mimi_destroy(sopro_mimi_t* m);
int64_t sopro_mimi_samples_per_frame(const sopro_mimi_t* m); /* 1920 */
/* codes [B, n_q, T] i32 (device) -> wav [B, T*1920] f32 (device).  MimiModel.decode (:1633-1680). */
int sopro_mimi_decode(sopro_mimi_t* m, const int32_t* codes, int B, int T, float* wav, void* stream);
/* same with HOST buffers; synchronises the stream */
int sopro_mimi_decode_host(sopro_mimi_t* m, const int32_t* codes_host, int B, int T, float* wav_host, void* stream);

/* Arithmetic of the dense blocks (transformer linears, SEANet Conv1d / ConvTranspose1d).
 *   SOPRO_MIMI_BF16_TC (default): bf16 operands on the tensor cores (wgmma), fp32 accumulation,
 *     fp32 residual streams / LayerNorm / softmax; within 2e-2 * max|wav| of the fp32 reference.
 *   SOPRO_MIMI_FP32: every contraction in fp32 on the FMA pipe; within 1e-4 of the reference
 *     (what transformers computes on CPU, modeling_mimi.py). */
#define SOPRO_MIMI_FP32 0
#define SOPRO_MIMI_BF16_TC 1
int sopro_mimi_set_precision(sopro_mimi_t* m, int precision);
/* Decodes of at most 64 frames (B*T: streaming chunks, time-to-first-audio) are launch-bound (~100 kernels); they
 * are captured once per (B, T, precision) into a CUDA graph over internal static buffers and replayed (default on).
 * Results are identical to the plain path. */
int sopro_mimi_set_graphs(sopro_mimi_t* m, int enabled);

/* A decode that meets a code outside [0, vocab) (e.g. an uncut EOS id) clamps it and sets a sticky flag instead of
 * reading outside the codebook (the reference's embedding lookup raises IndexError, modeling_mimi.py:1192-1196).
 * sopro_mimi_check synchronises `stream`, returns SOPRO_ERR_INVALID if the flag was set since the last check, and
 * clears it.  The *_host entry points validate their host buffers up front instead. */
int sopro_mimi_check(sopro_mimi_t* m, void* stream);

/* ---- streaming decode with persistent state: MimiStreamDecoder.decode_step / MimiDecodeState (reference
 * codec/mimi.py:75-181).  A stream carries one K/V ring per transformer layer (the last `window` positions), the
 * previous RVQ frame of the upsampler and the (taps-1) left-context rows of every causal conv (what transformers'
 * MimiConv1dPaddingCache holds, modeling_mimi.py:77-170), so a chunk costs O(chunk) and, decoder being causal, the
 * chunks concatenate to exactly what sopro_mimi_decode gives for the whole sequence (bit-identical in SOPRO_MIMI_FP32
 * mode; within the tensor-core mode's stated tolerance otherwise).  The reference instead re-decodes 2 overlap frames
 * on top of a transformers KV cache with no conv context and documents its stream as not bit-exact (README.md:151).
 * One stream = one utterance; streams of one decoder are independent; the arithmetic mode is the decoder's at
 * create / reset time. */
typedef struct sopro_mimi_stream sopro_mimi_stream_t;
/* A stream of `rows` utterances in [1, 65535] decoded side by side: every step advances all rows by the same number of
 * frames, and each row's state sits in its own slice of every buffer, so each kernel reads and writes only its own
 * row and sums in a fixed order: row b's samples equal a one-row stream fed row b's codes, bit for bit, in both
 * arithmetic modes.  A row whose utterance has ended can be fed code 0 and its samples dropped (the decoder is causal:
 * its earlier samples do not change).  Device memory grows linearly with rows (sopro_mimi_stream_bytes). */
int sopro_mimi_stream_create_rows(sopro_mimi_t* m, int max_chunk_frames, int rows, sopro_mimi_stream_t** out);
int sopro_mimi_stream_create(sopro_mimi_t* m, int max_chunk_frames, sopro_mimi_stream_t** out);  /* rows = 1 */
int sopro_mimi_stream_destroy(sopro_mimi_stream_t* s);
int sopro_mimi_stream_reset(sopro_mimi_stream_t* s, void* stream);     /* back to frame 0 (MimiDecodeState()) */
int64_t sopro_mimi_stream_frames(const sopro_mimi_stream_t* s);        /* MimiDecodeState.frames_seen */
int64_t sopro_mimi_stream_rows(const sopro_mimi_stream_t* s);
int64_t sopro_mimi_stream_bytes(const sopro_mimi_stream_t* s);         /* device bytes the stream holds */
/* the next n frames of every row: codes [rows, n_q, n] i32 (device) -> wav [rows, n*1920] f32 (device); any n >= 1
 * (longer than max_chunk_frames is processed in pieces).  One row: codes [n_q, n] -> wav [n*1920]. */
int sopro_mimi_decode_step(sopro_mimi_stream_t* s, const int32_t* codes, int n, float* wav, void* stream);
int sopro_mimi_decode_step_host(sopro_mimi_stream_t* s, const int32_t* codes_host, int n, float* wav_host, void* stream);

/* ---- Mimi ENCODE (waveform -> codes): MimiCodec.encode_file's model call (reference codec/mimi.py:41-63 ->
 * MimiModel.encode, modeling_mimi.py:1455-1488, 1522-1611), once per reference voice.  SEANet encoder (:454-497:
 * conv k7, 4 x [ResnetBlock, ELU, strided conv kernel 2r stride r] with r = reversed(ratios), ELU, conv k3), the
 * encoder transformer (same layer as the decoder's), the 25 -> 12.5 Hz conv (kernel 4, stride 2, replicate padding,
 * :1419-1429) and the split residual vector quantizer's nearest-neighbour search (:1262-1280, :1311-1338).  fp32
 * throughout (the codes are an argmin): batch 1, any sample count >= 1; every strided conv pads its input on the right
 * to a full window (MimiConv1d._get_extra_padding_for_conv1d, :273-285), so T = ceil(ceil(..ceil(n/4)../8)/2).
 * HOST fp32 pointers in state_dict layouts; `cfg` is the decoder's sopro_mimi_config_t. */
typedef struct sopro_mimi_enc_stage_weights {
  const float *res1_w, *res1_b;   /* encoder.layers.{1+3s}.block.1.conv [C/2, C, 3], [C/2]   (C = 64 << s) */
  const float *res2_w, *res2_b;   /* encoder.layers.{1+3s}.block.3.conv [C, C/2, 1], [C] */
  const float *down_w, *down_b;   /* encoder.layers.{3+3s}.conv [2C, C, 2r], [2C],  r = ratios[n_ratios-1-s] */
} sopro_mimi_enc_stage_weights_t;

typedef struct sopro_mimi_encoder_weights {
  const float *conv0_w, *conv0_b;                    /* encoder.layers.0.conv [F, 1, 7], [F] */
  sopro_mimi_enc_stage_weights_t stage[SOPRO_MIMI_MAX_RATIOS];
  const float *last_w, *last_b;                      /* encoder.layers.14.conv [hidden, 16F, 3], [hidden] */
  sopro_mimi_layer_weights_t layer[SOPRO_MIMI_MAX_LAYERS]; /* encoder_transformer.layers.* */
  const float* downsample_w;                         /* downsample.conv.weight [hidden, hidden, 4], no bias */
  const float* sem_in_proj;                          /* quantizer.semantic_...input_proj.weight [Dc, hidden] */
  const float* ac_in_proj;                           /* quantizer.acoustic_...input_proj.weight [Dc, hidden] */
  const float* embed;                                /* [n_q, vocab, Dc] as in sopro_mimi_weights_t */
} sopro_mimi_encoder_weights_t;

typedef struct sopro_mimi_encoder sopro_mimi_encoder_t;
int sopro_mimi_encoder_create(const sopro_mimi_config_t* cfg, const sopro_mimi_encoder_weights_t* host_weights, int device,
                              sopro_mimi_encoder_t** out);
int sopro_mimi_encoder_destroy(sopro_mimi_encoder_t* e);
/* MimiModel.get_encoded_length (:1490-1503): frames produced for n_samples input samples; < 0 on bad arguments */
int64_t sopro_mimi_encoded_frames(const sopro_mimi_encoder_t* e, int64_t n_samples);
/* wav [n_samples] f32 @24 kHz (device) -> codes [n_q, T] i32 (device), T = sopro_mimi_encoded_frames(n_samples).
 * `latent` (optional, device [T, hidden] f32) receives the pre-quantizer embeddings (tests compare them with the
 * oracle's; the codes are their nearest neighbours). */
int sopro_mimi_encode(sopro_mimi_encoder_t* e, const float* wav, int64_t n_samples, int32_t* codes, float* latent, void* stream);
/* same with HOST buffers; synchronises the stream */
int sopro_mimi_encode_host(sopro_mimi_encoder_t* e, const float* wav_host, int64_t n_samples, int32_t* codes_host,
                           float* latent_host, void* stream);
/* A ragged batch of clips in one pass: row b of wav [B][stride] f32 @24 kHz (device) has lens_host[b] samples (HOST i64,
 * each in [1, 14 400 000]); samples past lens[b] are not read.  Tmax = sopro_mimi_encoded_frames(longest row) -> codes
 * [B][n_q][Tmax] i32 (device): row b's first T_b = sopro_mimi_encoded_frames(lens[b]) frames are written, the rest
 * are left as they were.  `latent` (optional, device [B][Tmax][hidden] f32): rows past T_b hold padding values.
 * Row b equals sopro_mimi_encode of that clip alone, codes and latent, bit for bit.  The batch is padded to the longest
 * row rounded up to 2 * prod(ratios) samples; B times that must be at most 14 400 000 (the single call's bound).
 * B < 1, a length out of range, stride < the longest row, an oversized batch or a null pointer: SOPRO_ERR_INVALID
 * before any launch.  Uploads the B lengths (HOST -> device copy on `stream`); no synchronisation. */
int sopro_mimi_encode_batch(sopro_mimi_encoder_t* e, const float* wav, int32_t B, int64_t stride, const int64_t* lens_host,
                            int32_t* codes, float* latent, void* stream);

/* ---- voice ingestion (MimiCodec.encode_file's host-side preparation, reference codec/mimi.py:44-57, on the device for
 * a ragged batch of clips, each at its own sample rate; no reference counterpart for the batch).
 *   Trim: the energy VAD of the reference's trim_silence_energy (audio.py:30-87) at the clip's rate sr:
 *   flen = max(1, floor(sr * 25 / 1000)), hop = max(1, floor(sr * 10 / 1000)), pad = floor(sr * 30 / 1000); frames
 *   k < K = floor((n - flen) / hop) + 1; e_k = sum x^2 / flen summed in fp64 (a fixed order per frame), dB_k =
 *   10 log10(e_k + 1e-10); thr = max(max_k dB_k - 40, -40); frame k is voiced when dB_k > thr; start = max(0, first hop
 *   - pad), end = min(n, last hop + flen + pad).  The extent is (0, n) when n < floor(sr * 0.1) or n < flen, no frame
 *   is voiced, or end - start < floor(sr / 2).  The reference sums in fp32, so a frame whose dB lies within rounding of
 *   the threshold may be classified differently there.
 *   Pack: row b of dst [B][dst_stride] = the lens_host[b] samples at src[b], zeros up to dst_stride. */
/* rows: HOST array of B device pointers, row b of lens_host[b] samples (HOST i64) at rates_host[b] Hz (HOST i32, in
 * [4000, 192000]) -> ext [B][2] (device i64).  One launch per 64 rows; no call synchronises or allocates. */
int sopro_ingest_trim(const float* const* rows, int32_t B, const int64_t* lens_host, const int32_t* rates_host, int64_t* ext,
                      void* stream);
/* src: HOST array of B device pointers (row b's first sample, read in place); lens_host[b] in [0, dst_stride].  One
 * launch per 128 rows; no call synchronises or allocates. */
int sopro_ingest_pack(const float* const* src, int32_t B, const int64_t* lens_host, float* dst, int64_t dst_stride, void* stream);

/* ------------------------------------------------------------------------------------------------
 * NAR refiner: SoproTTSModel.nar_refine (reference model.py:307-347) over NARSinglePass.forward_stage
 * (nn/nar.py:89-116), NARStageAdapter (nn/nar.py:13-32), SSMLiteBlock.forward (nn/blocks.py:143-148) and
 * CodebookEmbedding.sum_embed_subset (nn/embeddings.py:77-112).  Given the AR tokens (codebook 0) and the
 * conditioning rows it fills codebooks 1..Q-1 stage by stage (argmax).  fp32 throughout: the ids equal the
 * reference's.  HOST fp32 pointers in state_dict layouts; the engine uploads its own copy.
 * ------------------------------------------------------------------------------------------------ */
#define SOPRO_MAX_SSM_LAYERS 16
#define SOPRO_NAR_MAX_STAGES 8
#define SOPRO_NAR_MAX_CODEBOOKS 64

typedef struct sopro_ssm_block_weights { /* SSMLiteBlock (nn/blocks.py:113-133) */
  const float* norm_w;              /* norm.weight [D] */
  const float *glu_w, *glu_b;       /* glu.pro [2D, D], [2D] */
  const float *dw_w, *dw_b;         /* dw.dw [D, 1, k], [D] */
  const float* ffn_norm_w;          /* ff.0.weight [D] */
  const float *ffn_w1, *ffn_b1;     /* ff.1 [4D, D], [4D] */
  const float *ffn_w2, *ffn_b2;     /* ff.3 [D, 4D], [D] */
} sopro_ssm_block_weights_t;

typedef struct sopro_nar_config {
  int32_t d_model;        /* 384 */
  int32_t n_layers;       /* cfg.n_layers_nar (6) */
  int32_t kernel;         /* cfg.nar_kernel_size (11) */
  int32_t dilation[SOPRO_MAX_SSM_LAYERS]; /* nn/nar.py:47-52 */
  int32_t n_codebooks;    /* Q = 32 */
  int32_t codebook_size;  /* V = 2048 */
  int32_t head_dim;       /* cfg.nar_head_dim (256) */
  int32_t adapter_hidden; /* 256 (nn/nar.py:14) */
  int32_t n_stages;       /* non-empty stages of B, C, D, E (nn/nar.py:41-44) */
  int32_t stage_first[SOPRO_NAR_MAX_STAGES]; /* first codebook of the stage; stages cover 1..Q-1 consecutively */
  int32_t stage_count[SOPRO_NAR_MAX_STAGES];
} sopro_nar_config_t;

typedef struct sopro_nar_weights {
  sopro_ssm_block_weights_t block[SOPRO_MAX_SSM_LAYERS];  /* nar.blocks.{i} */
  const float* norm_w;                     /* nar.norm.weight [D] */
  const float *pre_w, *pre_b;              /* nar.pre [Hn, D], [Hn] */
  const float* stage_emb;                  /* nar.stage_emb.weight [n_stages, D] */
  const float* adapter_norm_w;             /* nar.adapter.norm.weight [D] */
  const float *adapter_w0, *adapter_b0;    /* nar.adapter.mlp.0 [256, D], [256] */
  const float *adapter_w2, *adapter_b2;    /* nar.adapter.mlp.2 [2D, 256], [2D] */
  const float* head_w[SOPRO_NAR_MAX_CODEBOOKS]; /* nar.heads.{stage}.{j}.weight [V, Hn], indexed by CODEBOOK (1..Q-1) */
  const float* head_b[SOPRO_NAR_MAX_CODEBOOKS];
  const float* head_id_emb[SOPRO_NAR_MAX_STAGES]; /* nar.head_id_emb.{stage}.weight [count, Hn] */
  const float* mix[SOPRO_NAR_MAX_STAGES];         /* nar.mix.{stage} [2] (softmaxed, model.py:335-337) */
  const float* prev_cb_weights;            /* nar_prev_cb_weights [Q] (model.py:70-72) */
  const float* cb_embed;                   /* cb_embed.emb.weight [Q*V + 1, D] */
} sopro_nar_weights_t;

typedef struct sopro_nar sopro_nar_t;
int sopro_nar_create(const sopro_nar_config_t* cfg, const sopro_nar_weights_t* host_weights, int device, sopro_nar_t** out);
int sopro_nar_destroy(sopro_nar_t* n);
/* cond: rows [b][t][d_model] f32 (device), utterance b starting at cond + b*cond_batch_stride (floats) -- cond_ar[:, :T]
 * of the prefill; rvq1 [B, Tmax] i32 (device): the AR tokens; lens [B] i32 (device) or NULL: valid frames per
 * utterance (the refiner is not causal: rows >= lens[b] are padding and act as the zero padding of the convs);
 * codes [B, Tmax, Q] i32 (device) out: codebook 0 = rvq1, 1..Q-1 refined (rows >= lens[b] are undefined). */
int sopro_nar_refine(sopro_nar_t* n, const float* cond, int64_t cond_batch_stride, const int32_t* rvq1, const int32_t* lens,
                     int B, int Tmax, int32_t* codes, void* stream);
/* test hook (teacher forcing): when non-NULL, every stage conditions on the previous codebooks of forced_codes
 * [B, Tmax, Q] i32 (device) instead of on its own argmax results, so one near-tie flip cannot cascade. */
int sopro_nar_set_forced(sopro_nar_t* n, const int32_t* forced_codes);
/* Arithmetic unit of the refiner's contractions: -1 = automatic (tensor cores -- wgmma, every fp32 operand split into
 * three exact bf16 terms, the six products that reach fp32's last bit, fp32 accumulation -- whenever more than 16 rows are
 * refined; the fp32 FMA skinny kernel below that), 0 = fp32 FMA kernels only (also: environment SOPRO_NAR_TC=0), 1 = as -1
 * but fails if the geometry has no tensor-core images. */
int sopro_nar_set_contraction(sopro_nar_t* n, int mode);
/* One utterance's streaming windows (B == 1, <= 256 frames, no lens / forced codes) are replayed from CUDA graphs captured
 * over internal static buffers (a window is 113..217 launches): identical results, launch overhead removed.  Default on. */
int sopro_nar_set_graphs(sopro_nar_t* n, int enabled);
/* test hook: when non-NULL, every stage's pre-head activation z (nar.pre's output, before the head id embedding) is
 * copied to z + s*B*Tmax*head_dim, layout [n_stages][B][Tmax][head_dim] f32 (device).  Bypasses the graph replay. */
int sopro_nar_set_trace(sopro_nar_t* n, float* z);

/* test hooks: the refiner's and the prefill's kernels one launch at a time, with the engine's own launchers.  Device
 * pointers, no allocation; a shape the kernel does not take returns SOPRO_ERR_INVALID and launches nothing.
 *
 * One fp32 contraction (dense_f32.cuh DenseOp): C[m][n] = epi(prologue(A)[m] . W[n] + bias[n]) with the RMSNorm prologue
 * (norm_w) and/or a_add; epi 0 bias, 1 bias+GELU, 2 R + acc, 3 GLU (C [M][ldc >= N/2]), 4 argmax, 5 R + gate*acc.
 * kernel: 0 = the engine's choice, 16 = the skinny kernel (M <= 16, K <= 2048), 32 / 64 / 128 = that tile edge (not 32 for
 * GLU).  groups > 1 (argmax only): group z uses W + z*zW, bias + z*zBias, a_add + z*zAdd.  Argmax: ids [M][groups] i32
 * gets the first maximum of each row and group, through a workspace ws of >= 8*groups*M*ceil(N/8) bytes. */
int sopro_debug_dense(const float* A, const float* W, const float* bias, const float* norm_w, const float* a_add, const float* R,
                      float* C, float gate, int M, int N, int K, int ldc, int epi, int groups, int64_t zW, int64_t zBias,
                      int64_t zAdd, int kernel, int32_t* ids, void* ws, int64_t ws_bytes, void* stream);
/* The tensor-core contraction of the refiner: X [M][K] fp32 (optionally RMS-normalised by norm_w) is split into
 * A3 [M][3K] bf16 = [h | m | l], then C [M][N] = epi(six products of A3 and W6 + bias); W6 [N][6K] as
 * sopro_debug_pack_w6 builds it; epi 0 none, 1 GELU, 3 R + acc (R may alias C). */
int sopro_debug_tc6(const float* X, const float* norm_w, const uint16_t* W6, const float* bias, const float* R, float* C, void* A3,
                    int64_t M, int N, int K, int epi, void* stream);
/* depthwise conv + residual of an SSMLiteBlock: out[b][t] = x[b][t] + bias + sum_j h[b][t + j*dil - left] * w[:, j] for
 * t < lens[b] (rows outside [0, lens[b]) count as zero and are not read; output rows >= lens[b] are not written);
 * rows [B][Tmax][D], lens NULL = Tmax. */
int sopro_debug_dwconv_res(const float* h, const float* x, const float* w, const float* bias, float* out, const int32_t* lens, int B,
                           int Tmax, int D, int k, int dil, int left, void* stream);
/* first maximum of each head's V logits: logits [rows][heads][V] -> codes[r*Q + head] */
int sopro_debug_argmax_heads(const float* logits, int64_t rows, int heads, int V, int32_t* codes, int Q, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Prefill: SoproTTSModel.prepare_conditioning (reference model.py:172-216) for B texts that share one prepared
 * reference voice: TextEncoder (nn/text.py:16-44) -> txt_seq, txt_pool; base = txt_pool + frame sinusoid;
 * SpeakerFiLM (nn/speaker.py:64-85); RefXAttnStack with cached K/V (nn/ref.py:57-108, 111-160); cond_norm -> cond_ar.
 * fp32 (cond_ar / txt_seq feed the id-exact AR kernel).  HOST fp32 weight pointers, state_dict layouts.
 * prepare_reference (once per voice: Token2SV, reference encoder, K/V projections) is sopro_refprep_* below.
 * ------------------------------------------------------------------------------------------------ */
#define SOPRO_PREFILL_MAX_REF_LAYERS 8
#define SOPRO_PREFILL_MAX_BLEND_SEGMENTS 16  /* segments of one blended voice (sopro_prefill_run_blends) */

typedef struct sopro_prefill_config {
  int32_t d_model;        /* 384 */
  int32_t n_layers_text;  /* cfg.n_layers_text (2) */
  int32_t text_kernel;    /* 7 (nn/text.py:24) */
  int32_t text_vocab;     /* rows of text_enc.embed.emb.weight */
  int32_t sv_dim;         /* cfg.sv_student_dim (192) */
  int32_t ref_layers;     /* cfg.ref_xattn_layers (3) */
  int32_t ref_heads;      /* cfg.ref_xattn_heads (2) */
  float ref_gmax;         /* cfg.ref_xattn_gmax */
  int32_t max_text_len;   /* rows of text_pos */
  int32_t max_frames_pos; /* rows of frame_pos */
} sopro_prefill_config_t;

typedef struct sopro_prefill_ref_layer {
  const float* nq_w;      /* ref_xattn.blocks.{i}.nq.weight [D] */
  const float* q_w;       /* ...q_proj.weight [D, D] */
  const float* o_w;       /* ...out_proj.weight [D, D] */
  float gate;             /* ...gate (scalar; gmax * tanh(gate) is applied, nn/ref.py:105) */
} sopro_prefill_ref_layer_t;

typedef struct sopro_prefill_weights {
  const float* text_emb;   /* text_enc.embed.emb.weight [vocab, D] */
  const float* text_pos;   /* sinusoid table [max_text_len, D] (nn/embeddings.py:11-25; a non-persistent buffer) */
  const float* frame_pos;  /* sinusoid table [max_frames_pos, D] */
  sopro_ssm_block_weights_t text_block[SOPRO_MAX_SSM_LAYERS]; /* text_enc.layers.{i} */
  const float* text_norm_w;             /* text_enc.norm.weight */
  const float *film_w0, *film_b0;       /* spk_film.mlp.0 [D, sv], [D] */
  const float *film_w2, *film_b2;       /* spk_film.mlp.2 [2D, D], [2D] */
  const float *film_norm_w, *film_norm_b; /* spk_film.norm (LayerNorm) */
  sopro_prefill_ref_layer_t ref_layer[SOPRO_PREFILL_MAX_REF_LAYERS];
  const float* cond_norm_w;             /* cond_norm.weight */
} sopro_prefill_weights_t;

typedef struct sopro_prefill sopro_prefill_t;
int sopro_prefill_create(const sopro_prefill_config_t* cfg, const sopro_prefill_weights_t* host_weights, int device,
                         sopro_prefill_t** out);
int sopro_prefill_destroy(sopro_prefill_t* p);
/* All pointers below are DEVICE pointers.  text_ids [B, Lmax] i32 (padded), text_len [B] i32; sv [B or 1, sv_dim]
 * (sv_shared != 0: one speaker vector for the batch); ref_k / ref_v: HOST arrays of ref_layers device pointers to the
 * prepared reference's cached K / V [H, Tr, D/H] (PreparedReference.ref_kv_caches, model.py:45-50);
 * n_frames = max_frames + 1.  Outputs: txt_seq [B, Lmax, D] (rows >= text_len[b] undefined), txt_pool [B, D],
 * cond_ar [B, n_frames, D] -- the `prep` dict of model.py:210-216. */
int sopro_prefill_run(sopro_prefill_t* p, const int32_t* text_ids, const int32_t* text_len, int B, int Lmax, const float* sv,
                      int sv_shared, const float* const* ref_k, const float* const* ref_v, int Tr, float style_strength,
                      int n_frames, float* txt_seq, float* txt_pool, float* cond_ar, void* stream);
/* The same prefill with a voice per text: B texts over a table of n_voices (1 <= n_voices <= B) prepared references.
 * voice_of: HOST int32 [B], text b speaks voice voice_of[b] in [0, n_voices); sv: DEVICE f32 [n_voices, sv_dim], voice v's
 * speaker vector; tr: HOST int32 [n_voices], voice v's reference frames, each in [1, 4096]; ref_k / ref_v: HOST arrays of
 * ref_layers * n_voices device pointers, entry i * n_voices + v = voice v's cached K / V of reference layer i [H, tr[v], D/H].
 * The other arguments and the outputs are sopro_prefill_run's.  Text b's rows equal, bit for bit, the rows of a
 * sopro_prefill_run of the same texts with voice voice_of[b] alone (sv_shared = 1).  The table is copied to the device
 * on `stream` with no host synchronisation; the host arrays may be released when the call returns. */
int sopro_prefill_run_voices(sopro_prefill_t* p, const int32_t* text_ids, const int32_t* text_len, int B, int Lmax, int n_voices,
                             const int32_t* voice_of, const float* sv, const int32_t* tr, const float* const* ref_k,
                             const float* const* ref_v, float style_strength, int n_frames, float* txt_seq, float* txt_pool,
                             float* cond_ar, void* stream);
/* The voice-table prefill over blended voices (SoproTTS.blend_voices, sopro_b200/voices.py).  Voice v's K / V are
 * n_seg[v] segments one after another along the frame axis: its tr[v] frames split into seg_frames[...] frames each, with
 * weights seg_w[...].  n_seg: HOST int32 [n_voices], each in [1, SOPRO_PREFILL_MAX_BLEND_SEGMENTS]; seg_frames: HOST int32,
 * voice 0's n_seg[0] entries, then voice 1's, ..., each >= 1 and summing to tr[v] per voice; seg_w: HOST f32 in the same
 * order, each finite and > 0 (the caller normalises them).  In each reference cross-attention layer a row of voice v
 * attends to each segment on its own (its own softmax; non-finite outputs zeroed) and mixes the read-outs,
 * a = sum_s seg_w[s] a_s in segment order, before the RMS match, out_proj and the gate.  The other arguments and the
 * outputs are sopro_prefill_run_voices's; anything else in the table returns SOPRO_ERR_INVALID with nothing launched.
 * A voice of one segment with weight 1.0f gives the rows sopro_prefill_run_voices gives it, bit for bit, and a row equals
 * the row of a launch with its voice alone.  The segment table travels to the device with the voice table (no host
 * synchronisation); the host arrays may be released when the call returns. */
int sopro_prefill_run_blends(sopro_prefill_t* p, const int32_t* text_ids, const int32_t* text_len, int B, int Lmax, int n_voices,
                             const int32_t* voice_of, const float* sv, const int32_t* tr, const float* const* ref_k,
                             const float* const* ref_v, const int32_t* n_seg, const int32_t* seg_frames, const float* seg_w,
                             float style_strength, int n_frames, float* txt_seq, float* txt_pool, float* cond_ar, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Reference preparation: SoproTTSModel.prepare_reference (reference model.py:152-170), once per voice, from the
 * voice's codes: Token2SV (nn/speaker.py:12-61, AttentiveStatsPool nn/blocks.py:165-188) -> sv_ref;
 * _encode_reference_seq (model.py:136-150) -> ref_seq; RefXAttnStack.build_kv_caches (nn/ref.py) -> the K / V the
 * prefill engine reads.  fp32.  HOST fp32 weight pointers, state_dict layouts.
 * ------------------------------------------------------------------------------------------------ */
typedef struct sopro_refprep_config {
  int32_t d_model;        /* 384 */
  int32_t sv_embed_dim;   /* 192: Token2SV's d */
  int32_t sv_dim;         /* cfg.sv_student_dim (192) */
  int32_t n_codebooks;    /* 32 */
  int32_t codebook_size;  /* 2048 */
  int32_t sv_kernel;      /* 7 (nn/speaker.py:24,27) */
  int32_t ref_enc_layers; /* cfg.ref_enc_layers (2) */
  int32_t ref_enc_kernel; /* 7 */
  int32_t ref_layers;     /* cfg.ref_xattn_layers (3) */
  int32_t ref_heads;      /* cfg.ref_xattn_heads (2) */
} sopro_refprep_config_t;

typedef struct sopro_refprep_kv_layer {
  const float* nkv_w;     /* ref_xattn.blocks.{i}.nkv.weight [D] */
  const float* k_w;       /* ...k_proj.weight [D, D] */
  const float* v_w;       /* ...v_proj.weight [D, D] */
} sopro_refprep_kv_layer_t;

typedef struct sopro_refprep_weights {
  const float* sv_emb;          /* token2sv.emb.weight [Q*V, d] */
  const float* sv_cb_weights;   /* token2sv.cb_weights [Q] (softmax taken by the engine) */
  const float *sv_dw0_w, *sv_dw0_b; /* token2sv.enc.0.dw [d, 1, k], [d] */
  const float *sv_dw1_w, *sv_dw1_b; /* token2sv.enc.3.dw */
  const float *pool_w0, *pool_b0;   /* token2sv.pool.attn.0 [d, d], [d] */
  const float* pool_w2;             /* token2sv.pool.attn.2.weight [1, d] */
  float pool_b2;                    /* token2sv.pool.attn.2.bias */
  const float *proj_w, *proj_b;     /* token2sv.proj [sv, 2d], [sv] */
  const float* cb_embed;            /* cb_embed.emb.weight [>= Q*V, D] (the first Q*V rows are read) */
  const float* ref_cb_weights;      /* ref_cb_weights [Q] */
  sopro_ssm_block_weights_t ref_block[SOPRO_MAX_SSM_LAYERS]; /* ref_enc_blocks.{i} */
  const float* ref_norm_w;          /* ref_enc_norm.weight */
  sopro_refprep_kv_layer_t layer[SOPRO_PREFILL_MAX_REF_LAYERS];
} sopro_refprep_weights_t;

typedef struct sopro_refprep sopro_refprep_t;
int sopro_refprep_create(const sopro_refprep_config_t* cfg, const sopro_refprep_weights_t* host_weights, int device,
                         sopro_refprep_t** out);
int sopro_refprep_destroy(sopro_refprep_t* p);
/* DEVICE pointers: tokens [Tr, Q] i32 -> sv [sv_dim], ref_seq [Tr, D]; ref_k / ref_v: HOST arrays of ref_layers device
 * pointers, each [H, Tr, D/H] (PreparedReference.ref_kv_caches[i]["k"/"v"], model.py:45-50). */
int sopro_refprep_run(sopro_refprep_t* p, const int32_t* tokens, int Tr, float* sv, float* ref_seq, float* const* ref_k,
                      float* const* ref_v, void* stream);
/* Token2SV alone over a ragged batch (best-of-N synthesis scores its takes with it): B code sequences -> B unit speaker
 * vectors, and optionally their cosine with one reference vector.  tokens: device int32 [B][Tmax][Q]; lens_host: B ints
 * in [1, Tmax], Tmax <= 4096; sv: device f32 [B][sv_dim]; ref_sv: device f32 [sv_dim] or NULL; cos: device f32 [B]
 * (written only when ref_sv is given).  Row b equals, bit for bit, the sv sopro_refprep_run gives for its lens_host[b]
 * frames alone.  Codes outside [0, codebook_size) are reported by sopro_refprep_check. */
int sopro_refprep_speaker_vectors(sopro_refprep_t* p, const int32_t* tokens, int32_t B, int32_t Tmax, const int32_t* lens_host,
                                  float* sv, const float* ref_sv, float* cos, void* stream);
/* sopro_refprep_speaker_vectors scored against a reference vector per row (best-of-N over texts in different voices):
 * ref_sv: device f32 [B][sv_dim], cos[b] = sv[b] . ref_sv[b]; both required.  Each row's sv and cos equal, bit for bit,
 * those of sopro_refprep_speaker_vectors with ref_sv[b] as its one vector. */
int sopro_refprep_speaker_vectors_per_row(sopro_refprep_t* p, const int32_t* tokens, int32_t B, int32_t Tmax, const int32_t* lens_host,
                                          float* sv, const float* ref_sv, float* cos, void* stream);
/* synchronises `stream`; SOPRO_ERR_INVALID if a run since the last check met a code outside [0, codebook_size) (the
 * reference's embedding lookup raises IndexError); clears the flag */
int sopro_refprep_check(sopro_refprep_t* p, void* stream);

/* test hook: one tensor-core implicit GEMM (no reference counterpart), launched through the decoder's own launcher in
 * its operand geometry.  X bf16 (device): item b at X + b*a_pitch*cin, ctx context rows then M rows of cin channels
 * (a_pitch >= ctx + M; rows [ctx + M, a_pitch) are never read); W bf16 [N][taps*cin] (device).
 *   y[b][m][n] = epi(sum_j sum_ci X_b[m + ctx + j - (taps-1)][ci] * W[n][j*cin + ci] + bias[n % bias_mod])
 * with rows before X_b's first context row read as zero (the causal pad); epi: 0 none, 1 GELU(erf),
 * 2 R' + scale[n]*acc, 3 R' + acc with R'[b][m][n] = R[(b*r_pitch + m)*N + n] (R may equal out_f32: in place).
 * out_f32[(b*c_pitch + m)*N + n] = y; out_bf16 at the same offsets gets bf16(y), through ELU when out_elu; either
 * output may be null.  Nothing outside rows [0, M) of an item is written.  bias may be null (else bias_mod in [4, N], a
 * multiple of 4); 0 <= ctx <= taps-1, c_pitch >= M, r_pitch >= M (epi 2, 3), pointers 16-byte aligned.  A shape the
 * kernel does not take returns SOPRO_ERR_INVALID and launches nothing. */
int sopro_debug_tc_gemm_pitched(const void* X, int B, int M, int ctx, int64_t a_pitch, int cin, int taps, const void* W, int N,
                                const float* bias, int bias_mod, int epi, const float* R, int64_t r_pitch, const float* scale,
                                float* out_f32, void* out_bf16, int64_t c_pitch, int out_elu, void* stream);
/* the same launch in the one-shot decode's packed geometry: X bf16 [B][rows][cin], R and the outputs [B][rows][N], no
 * context rows (ctx = 0, every pitch = rows); bias_mod <= 0 means N.  Only dil = 1 and pad = taps - 1 are taken (the
 * geometry the decoder issues); anything else returns SOPRO_ERR_INVALID. */
int sopro_debug_tc_gemm(const void* X, int B, int64_t rows, int cin, int taps, int dil, int pad, const void* W, int N,
                        const float* bias, int bias_mod, int epi, const float* R, const float* scale, float* out_f32,
                        void* out_bf16, int out_elu, void* stream);

/* test hooks: single tensor-core-mode kernels of the Mimi decoder (no reference counterpart).  Device pointers, no
 * allocation; a shape the kernel does not take returns SOPRO_ERR_INVALID and launches nothing.
 *
 * sliding-window attention: q, k bf16 [B][T2][C] (rotated), vt bf16 [B][C][T2p] (v transposed, T2p >= T2 and a multiple
 * of 8), out bf16 [B][T2][C]; C = 64*H, 1 <= window <= 257; query i attends to keys (i - window, i]. */
int sopro_debug_tc_attn(const void* q, const void* k, const void* vt, void* out, int B, int T2, int64_t T2p, int C, int H, int window,
                        void* stream);
/* fused ResnetBlock: out = Z + W2 . bf16(ELU(conv_taps(X; W1) + bias1)) + bias2.  X bf16 [B][ctx + M][2*hid] (its first
 * ctx rows are left context, 0 <= ctx <= taps-1; the causal zero pad supplies the other taps-1-ctx rows), W1 bf16
 * [hid][taps*2*hid], W2 bf16 [2*hid][hid], bias1 [hid], bias2 [2*hid], Z fp32 [B][M][2*hid]; out_f32 / out_bf16
 * [B][M][2*hid], either may be null, out_elu applies ELU to the bf16 copy only.  hid in {32, 64, 128}, 2*hid*taps a
 * multiple of 64.  Items packed back to back. */
int sopro_debug_tc_resblock(const void* X, const void* W1, const void* W2, const float* bias1, const float* bias2, const float* Z,
                            float* out_f32, void* out_bf16, int B, int M, int ctx, int hid, int taps, int out_elu, void* stream);
/* the same launch over pitched items (a stream's buffers): item b of X, Z and the outputs starts a_pitch >= ctx + M,
 * z_pitch >= M and o_pitch >= M rows after item b - 1; nothing outside rows [0, M) of an output item is written. */
int sopro_debug_tc_resblock_pitched(const void* X, const void* W1, const void* W2, const float* bias1, const float* bias2,
                                    const float* Z, float* out_f32, void* out_bf16, int B, int M, int ctx, int64_t a_pitch, int64_t z_pitch,
                                    int64_t o_pitch, int hid, int taps, int out_elu, void* stream);
/* attention operands from fp32 QKV rows [B][T2][3C]: rotated q -> qh, rotated k -> kh (bf16 [B][T2][C]), v -> vt (bf16
 * [B][C][T2p], T2p = T2 rounded up to 8, pad columns zero).  table: RoPE table of tab_T2 >= T2 positions,
 * [cos rows 0..tab_T2) | sin rows 0..tab_T2)] of 32 floats each; C = 64*H. */
int sopro_debug_rope_pack(const float* qkv, const float* table, int tab_T2, void* qh, void* kh, void* vt, int B, int T2, int C, int H,
                          void* stream);

/* test hooks: single fp32 kernels of the Mimi decoder and encoder (no reference counterpart), each launched with the
 * launch geometry the codec uses.  Device pointers, no allocation; a shape the kernel does not take returns
 * SOPRO_ERR_INVALID and launches nothing.
 *
 * implicit GEMM: out[b][m][n] (at out + b*c_bs + m*ldc + n) = epi(sum_{j, ci} act(A'[m + j*dil - pad][ci]) * W[n][j*Cin + ci]
 * + bias[n % bias_mod]), A' = A + b*a_bs read as [Min][Cin] (rows outside [0, Min) are zero), act = ELU when a_elu;
 * epi 0 none, 1 GELU(erf), 2 R' + scale[n]*acc, 3 R' + acc with R'[m][n] = R[b*r_bs + m*N + n].  Each output is one fma
 * chain over ascending k = j*Cin + ci.  K = taps*Cin, K % 16 == 0, Cin % 4 == 0, Min >= M, ldc >= N, a_bs % 4 == 0;
 * N % 64 != 0 and N <= 32 takes the 32-column tile. */
int sopro_debug_mimi_gemm(const float* A, const float* W, const float* bias, const float* R, const float* scale, float* out, int B, int M,
                          int N, int K, int Min, int Cin, int taps, int dil, int pad, int ldc, int bias_mod, int epi, int a_elu,
                          int64_t a_bs, int64_t c_bs, int64_t r_bs, void* stream);
/* RVQ lookup-sum: codes i32 [B][Q][code_T] (frames [0, T) read, code_T >= T), embed [Q][vocab][Dc] -> S [B][T][2*Dc] =
 * [sum of codebooks q < n_sem | sum of the others], each summed in q order.  A code outside [0, vocab) is clamped and
 * sets *bad (device i32, sticky). */
int sopro_debug_mimi_rvq_gather(const int32_t* codes, const float* embed, float* S, int B, int Q, int T, int code_T, int Dc, int vocab,
                                int n_sem, int32_t* bad, void* stream);
/* depthwise causal ConvTranspose k=4 s=2: x [B][T][C], w [C][4] -> y [B][2T][C]; y[2t+r] = x[t]*w[r] + x[t-1]*w[r+2],
 * x[-1] = prev[b] (device [B][C]) or zero when prev is NULL. */
int sopro_debug_mimi_upsample(const float* x, const float* w, float* y, const float* prev, int B, int T, int C, void* stream);
/* LayerNorm over C of rows x [rows][C] -> y [rows][C], fp32 (out_bf16 = 0) or bf16. */
int sopro_debug_mimi_layernorm(const float* x, const float* w, const float* b, void* y, int64_t rows, int C, float eps, int out_bf16,
                               void* stream);
/* RoPE then causal sliding-window attention in fp32 over qkv [B][T2][3C] (q and k rotated in place), row t at position
 * pos0 + t; table [cos rows | sin rows] of tab_T2 >= pos0 + T2 positions, Dh/2 floats each; out [B][T2][C] fp32 or bf16.
 * Query at position p attends to positions (p - window, p].  With kring / vring (device [B][R][C], both or neither,
 * R >= T2 + window - 1), each rotated key and value is first written to slot position % R and the keys and values are
 * read from the rings; without them pos0 = 0.  C % H == 0, (C/H) % 4 == 0. */
int sopro_debug_mimi_attn(float* qkv, const float* table, int tab_T2, void* out, int B, int T2, int C, int H, int window, int pos0,
                          float* kring, float* vring, int R, int out_bf16, void* stream);
/* final conv Cin -> 1, taps in [1, 8]: y[b][t] = bias + sum_j sum_c act(x[b][t + j - (taps-1)][c]) * w[j*Cin + c] over rows
 * >= lo (lo in [-(taps-1), 0]: rows lo..-1 are context in front of x), item b at x + b*x_bs, y + b*y_bs.  x_bf16 = 0: x
 * fp32 and act = ELU (final_conv_kernel, Cin % 4 == 0); x_bf16 = 1: x bf16 already ELU'd (final_conv_h_kernel,
 * Cin % 8 == 0). */
int sopro_debug_mimi_final_conv(const void* x, int x_bf16, const float* w, const float* bias, float* y, int B, int64_t Tn, int Cin,
                                int taps, int lo, int64_t x_bs, int64_t y_bs, void* stream);
/* residual codeword search of the encoder (Dc = 256): proj [B][T][512] = [semantic | acoustic] projections, embed
 * [n_q][V][256] -> codes i32 [B][n_q][T]; codebooks q < n_sem search from the semantic half, the rest from the acoustic
 * half, each code torch.argmin of the squared distances to the running residual (the first NaN, else the lowest index of
 * the minimum: always in [0, V)).  frames: device i32 [B] or NULL; frames of clip b at or past frames[b] are not written. */
int sopro_debug_mimi_rvq_encode(const float* proj, const float* embed, int32_t* codes, int T, int n_q, int n_sem, int V,
                                const int32_t* frames, int B, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Output resampling (no reference counterpart: the reference always returns 24 kHz): band-limited resampling of a
 * waveform from sr_in to sr_out with torchaudio.functional.resample's default filter (sinc_interp_hann,
 * lowpass_filter_width 6, rolloff 0.99).  With g = gcd(sr_in, sr_out), o = sr_in / g, n = sr_out / g,
 * base = 0.99 * min(o, n), width = ceil(6 o / base): output j = q n + p is sum_i k[p][i] * x[q o - width + i] over the
 * phase's nonzero taps (x = 0 outside [0, N)), ceil(n N / o) outputs.  Supported: integer rates in [4000, 192000], unequal,
 * whose reduced o and n are both <= 4096; anything else is SOPRO_ERR_INVALID before any allocation or launch.
 * fp32 accumulation, one FMA chain per output in increasing input index, shared by the one-shot and the stream paths. */
typedef struct sopro_resampler sopro_resampler_t;
typedef struct sopro_resampler_stream sopro_resampler_stream_t;
/* host-only: the filter.  geometry [4] HOST out = (o, n, width, S), S = the longest nonzero span; when non-NULL,
 * first [n], span [n] (i32) and taps [n][S] (f32, zero past each span) receive phase p's nonzero taps
 * k[p][first[p] .. first[p] + span[p]) (evaluated in double, rounded to fp32 once). */
int sopro_resampler_filter(int32_t sr_in, int32_t sr_out, int32_t* geometry, int32_t* first, int32_t* span, float* taps);
/* host-only: ceil(n * n_in / o), the outputs of n_in input samples; < 0 for a refused rate pair or n_in < 0 */
int64_t sopro_resampled_length(int32_t sr_in, int32_t sr_out, int64_t n_in);
int sopro_resampler_create(int32_t sr_in, int32_t sr_out, int device, sopro_resampler_t** out);
/* (destroy a resampler's streams first) */
int sopro_resampler_destroy(sopro_resampler_t* r);
/* one-shot, ragged batch: row b of x [B][x_stride] f32 (device) has lens_host[b] samples (HOST i64; NULL = x_stride each);
 * samples at or past lens[b] are not read.  Row b's ceil(n lens[b] / o) outputs go to y + b * y_stride (device; y_stride
 * >= the longest row's outputs when B > 1); the rest of the row is not written.  Row b equals that row resampled alone. */
int sopro_resample(sopro_resampler_t* r, const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, float* y,
                   int64_t y_stride, void* stream);
/* Streaming: one utterance pushed in chunks of at most max_chunk samples.  After N input samples the pushes have emitted
 * n * max(0, floor((N - width) / o)) outputs -- every block whose whole window [q o - width, q o + width + o) has arrived --
 * and finish emits the rest up to ceil(n N / o).  The concatenated outputs equal sopro_resample of the concatenated input
 * bit for bit, under any chunk schedule.  The state carries fewer than 2 width + o input samples on the device; output
 * counts are host arithmetic (no call synchronises).  Calls on one stream state must be ordered (one CUDA stream). */
int sopro_resampler_stream_create(sopro_resampler_t* r, int64_t max_chunk, sopro_resampler_stream_t** out);
int sopro_resampler_stream_destroy(sopro_resampler_stream_t* s);
/* back to sample 0 (host-only; also clears the finished state) */
int sopro_resampler_stream_reset(sopro_resampler_stream_t* s);
/* outputs the next call writes: a push of n_more samples (final == 0), or a push of n_more samples followed by finish
 * (final != 0); < 0 on bad arguments or after finish */
int64_t sopro_resampler_stream_ready(const sopro_resampler_stream_t* s, int64_t n_more, int final);
/* x [n] f32 (device) -> y (device) receives stream_ready(s, n, 0) outputs.  n > max_chunk: SOPRO_ERR_INVALID, nothing
 * launched, state unchanged.  After finish: SOPRO_ERR_STATE until a reset. */
int sopro_resampler_push(sopro_resampler_stream_t* s, const float* x, int64_t n, float* y, void* stream);
/* the remaining stream_ready(s, 0, 1) outputs (the input's end is zero padded) -> y (device); SOPRO_ERR_STATE when
 * called twice without a reset */
int sopro_resampler_finish(sopro_resampler_stream_t* s, float* y, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Speaking rate (no reference counterpart: the reference has no rate control): pitch-preserving time-scale
 * modification of a 24 kHz waveform by WSOLA.  Frame N = 480, synthesis hop Hs = 240, search tolerance D = 160,
 * periodic Hann window w[n] = sin^2(pi n / N).  The speed is quantised to S = round(speed * 65536) (half to even),
 * S in [16384, 262144] (speed 0.25 .. 4.0).  For L input samples (x = 0 outside [0, L)):
 *   M = ceil(L * 65536 / S) outputs, K = ceil(M / Hs) + 1 frames (0 when M = 0), a_k = floor((k Hs S + 32768) / 65536);
 *   d_0 = 0; for k >= 1, with p_{k-1} = a_{k-1} + d_{k-1}: d_k = argmax over d in [-D, D] of
 *   sum_n x[p_{k-1} + n] x[a_k + d - N/2 + n] (ties: smallest |d|, then the negative one);
 *   y[m] = sum_k w[m - k Hs + N/2] x[p_k + m - k Hs] over the two frames covering m, in increasing k, for m in [0, M).
 * fp32 arithmetic; one device function computes a frame for both the one-shot and the stream paths. */
typedef struct sopro_stretch_stream sopro_stretch_stream_t;
/* host-only: validates and quantises a speed; SOPRO_ERR_INVALID for NaN, +-inf or anything outside [0.25, 4.0] */
int sopro_stretch_speed(double speed, int32_t* S);
/* host-only: M = ceil(n_in * 65536 / S); < 0 for a refused S or n_in < 0 */
int64_t sopro_stretched_length(int32_t S, int64_t n_in);
/* host-only: returns K, the frames of n_in input samples, and (when a is non-NULL) writes their nominal analysis
 * positions a[0 .. K) (i64); < 0 for a refused S or n_in < 0 */
int64_t sopro_stretch_positions(int32_t S, int64_t n_in, int64_t* a);
/* host-only: the N = 480 window taps, sin^2(pi n / N) evaluated in double and rounded to fp32 once -> w [480] */
int sopro_stretch_window(float* w);
/* one-shot, ragged batch, one CTA per row: row b of x [B][x_stride] f32 (device) has lens_host[b] samples (HOST i64;
 * NULL = x_stride each); samples at or past lens[b] are not read.  Row b's M_b outputs go to y + b * y_stride (device;
 * y_stride >= the longest row's outputs when B > 1); the rest of the row is not written.  offsets (nullable, device
 * i32 [B][K_max], K_max = the longest row's frame count) receives every d_k: a test hook. */
int sopro_stretch(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int32_t S, float* y, int64_t y_stride,
                  int32_t* offsets, void* stream);
/* as sopro_stretch, with a speed per row: S_host (HOST i32 [B]) holds each row's S.  Row b produces
 * sopro_stretched_length(S_host[b], lens[b]) outputs.  A row with S_b = 65536 is copied through unchanged (M_b = lens[b])
 * and runs no frames; any other row's outputs (and offsets) equal sopro_stretch of that row alone at S_b, bit for bit.
 * One launch covers the whole batch (the rows' lengths and speeds reach it through one stream-ordered copy).
 * y_stride >= the longest row's outputs when B > 1; offsets: K_max = n_frames of the longest row's outputs, and a
 * copied row writes none.  Refused before any launch: sopro_stretch's refusals, a null S_host, and an S_b outside
 * [16384, 262144] in any row. */
int sopro_stretch_rows(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, const int32_t* S_host, float* y,
                       int64_t y_stride, int32_t* offsets, void* stream);
/* Streaming: one utterance pushed in chunks of at most max_chunk samples.  Frame k is ready once
 * max(a_k + D + N/2, a_{k-1} + D + Hs + N/2) input samples have arrived (a_0 + D + N/2 for frame 0); with frames
 * [0, k_done) done, the pushes have emitted the outputs below max(0, k_done - 1) * Hs, and finish emits the rest up to
 * M.  The concatenated outputs equal sopro_stretch of the concatenated input bit for bit, under any chunk schedule.
 * The state on the device: the last p, the Hs pending overlap-add samples, and fewer than 2048 carried input samples;
 * output counts are host arithmetic (no call synchronises).  Calls on one state must be ordered (one CUDA stream). */
int sopro_stretch_stream_create(int64_t max_chunk, int device, sopro_stretch_stream_t** out);
int sopro_stretch_stream_destroy(sopro_stretch_stream_t* s);
/* back to sample 0 at speed S (host-only; also clears the finished state).  A new state takes no push until its first
 * reset; one state serves every speed. */
int sopro_stretch_stream_reset(sopro_stretch_stream_t* s, int32_t S);
/* outputs the next call writes: a push of n_more samples (final == 0), or a push of n_more samples followed by finish
 * (final != 0); < 0 on bad arguments, before the first reset or after finish */
int64_t sopro_stretch_stream_ready(const sopro_stretch_stream_t* s, int64_t n_more, int final);
/* x [n] f32 (device) -> y (device) receives stream_ready(s, n, 0) outputs.  n > max_chunk: SOPRO_ERR_INVALID, nothing
 * launched, state unchanged.  After finish: SOPRO_ERR_STATE until a reset. */
int sopro_stretch_push(sopro_stretch_stream_t* s, const float* x, int64_t n, float* y, void* stream);
/* the remaining stream_ready(s, 0, 1) outputs (the input's end is zero padded) -> y (device); SOPRO_ERR_STATE when
 * called twice without a reset */
int sopro_stretch_finish(sopro_stretch_stream_t* s, float* y, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Loudness normalisation (no reference counterpart: the reference's output level follows its reference recording):
 * ITU-R BS.1770-4 integrated loudness of mono rows x[0, n) at a rate sr, an integer in [4000, 192000], and a gain to
 * a target T.
 *   K-weighting: two biquads in cascade, zero initial state, x = 0 before sample 0; libebur128's coefficients from the
 *   analog prototype, evaluated on the host in double (K = tan(pi f0 / sr), a0 = 1 + K/Q + K^2):
 *     shelf: f0 = 1681.974450955533, G = 3.999843853973347 dB, Q = 0.7071752369554196, Vh = 10^(G/20),
 *            Vb = Vh^0.4996667741545416; b = [Vh + Vb K/Q + K^2, 2 (K^2 - Vh), Vh - Vb K/Q + K^2] / a0,
 *            a = [1, 2 (K^2 - 1) / a0, (1 - K/Q + K^2) / a0];
 *     high-pass: f0 = 38.13547087602444, Q = 0.5003270373238773; b = [1, -2, 1], a as above with its own K and a0.
 *   Blocks: sub-block s = floor((sr + 5) / 10) samples; block j = sub-blocks j .. j + 3 for j in [0, J),
 *   J = max(0, floor(n / s) - 3); z_j = sum y^2 over the block / (4 s); l_j = -0.691 + 10 log10 z_j; a trailing partial
 *   sub-block belongs to no block.
 *   Gating: absolute, l_j > -70; Gamma_r = -0.691 + 10 log10(mean z over those blocks) - 10; L = -0.691 +
 *   10 log10(mean z over the blocks with l_j > -70 and l_j > Gamma_r), compared as energies (thresholds converted once
 *   in double); L = -inf when no block passes (silence, or n < 4 s).
 *   Gain: g = fp32(min(10^((T - L) / 20), 10^(-1/20) / max|x|)), rounded once, toward zero, so that the fixed -1 dBFS
 *   sample-peak ceiling holds in fp32: max|y| <= fp32(10^(-1/20)); g = 1 when L = -inf; y = g * x, one fp32 multiply.
 * The filter, the y^2 sums, the block energies and the gating run in fp64 on the device; every sum has a fixed order,
 * so a row's L, g and y depend only on its own samples.  No call synchronises with the host or allocates. */
/* host-only: the K-weighting coefficients at sr -> c[10] = shelf b0, b1, b2, a1, a2, then high-pass b0, b1, b2, a1, a2
 * (a0 = 1); SOPRO_ERR_INVALID for a rate outside [4000, 192000] */
int sopro_loudness_filter(int32_t sr, double* c);
/* host-only: SOPRO_OK for a target in [-60, 0] LUFS, SOPRO_ERR_INVALID otherwise (NaN and +-inf included) */
int sopro_loudness_target(double T);
/* host-only: the workspace bytes for B rows of at most max_len samples at sr; < 0 for bad arguments */
int64_t sopro_loudness_workspace(int32_t B, int64_t max_len, int32_t sr);
/* ragged batch: row b of x [B][x_stride] f32 (device) has lens_host[b] samples (HOST i64; NULL = x_stride each);
 * samples at or past lens[b] are not read.  ws: device, at least loudness_workspace(B, max lens, sr) bytes.
 * L of row b -> lufs_dev[b] (device f64; -inf when no block passes the gates). */
int sopro_loudness_measure(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int32_t sr, void* ws,
                           double* lufs_dev, void* stream);
/* as the measure, then y + b * y_stride (device; y_stride >= the longest row when B > 1) receives g_b * x over
 * [0, lens[b]); the rest of the row is not written.  y may alias x (y_stride = x_stride).  lufs_dev (nullable) receives
 * L, gain_dev (nullable, device f32 [B]) receives g: a test hook.  A refused T is SOPRO_ERR_INVALID before any launch. */
int sopro_loudness_normalize(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int32_t sr, double T,
                             float* y, int64_t y_stride, void* ws, double* lufs_dev, float* gain_dev, void* stream);

/* Live loudness: a causal leveller for audio that is still arriving.  It levels a passage, not each moment (it is not
 * an AGC): the gain follows the integrated loudness of everything so far.  One row x at rate sr (as above) and a target
 * T in [-60, 0] LUFS; the K-weighting (fp64, zero initial state), s, the blocks z_j and both gates are the meter's
 * above.  Sub-block k is x[k s, (k + 1) s).
 *   Meter: for k >= 3, M_k is the integrated loudness over blocks 0 .. k - 3, the meter's L of the prefix
 *   x[0, (k + 1) s); -inf when no block passes the gates.
 *   Gain: a_k = min(10^((T - M_k) / 20), 10^(B / 20)) for finite M_k, 1 when M_k = -inf.  B = 30 dB, the largest boost:
 *   a first block that barely passes the -70 LUFS gate (a breath, room tone) is not raised by 50 dB or more before any
 *   speech has been metered.
 *   Release: nothing before sub-block 3 is complete (4 s samples); then sub-blocks 0 .. 3 go out at the constant gain
 *   a_3, and each later sub-block k as soon as it is complete, under the ramp r(i) = a_{k-1} + (a_k - a_{k-1}) (i + 1) / s
 *   in double, i the index inside the sub-block.
 *   Ceiling: c_k = 10^(-1/20) / max|x| over sub-block k; y = fp32_rz(min(r(i), c_k)) * x, one fp32 multiply, the gain
 *   rounded toward zero, so that max|y| <= fp32(10^(-1/20)) everywhere.
 *   End: the finish releases what is held: a row of fewer than 4 sub-blocks at gain 1 under each sub-block's ceiling,
 *   then the partial tail (< s samples) at the last a (1 when there is none) under the tail's own ceiling.
 * Order: the filter's state at the end of sub-block k is s_k = A^s s_{k-1} + agg_k (A the filter's one-sample
 * transition, agg_k the state sub-block k leaves from zero state); a sub-block's y^2 sum, the absolute gate's running
 * sum (in increasing j) and M_k's relative-gated sum each have an order set by k alone.  So the output is a function of
 * the row's samples only: a stream's concatenated output equals sopro_level of the concatenated input bit for bit
 * under any push schedule, and a row of a ragged batch equals that row alone. */
/* host-only: the workspace bytes of sopro_level for B rows of at most max_len samples at sr; < 0 for bad arguments */
int64_t sopro_level_workspace(int32_t B, int64_t max_len, int32_t sr);
/* one-shot, ragged batch: row b of x [B][x_stride] f32 (device) has lens_host[b] samples (HOST i64; NULL = x_stride
 * each); samples at or past lens[b] are not read.  y + b * y_stride (device; y_stride >= the longest row when B > 1)
 * receives the levelled row over [0, lens[b]); the rest of the row is not written.  meter_dev and gain_dev (nullable,
 * device f64 [B][floor(max lens / s)]) receive M_k and a_k of every complete sub-block (NaN for k < 3): a test hook.
 * A refused T or rate is SOPRO_ERR_INVALID before any launch.  No call synchronises or allocates. */
int sopro_level(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int32_t sr, double T, float* y,
                int64_t y_stride, void* ws, double* meter_dev, double* gain_dev, void* stream);
/* Streaming: one utterance pushed in chunks of at most max_chunk samples.  After N input samples the pushes have
 * released floor(N / s) s samples once floor(N / s) >= 4 and none before, and finish releases the rest up to N.  One launch per push that completes a sub-block.  The state on the device: the filter
 * state, fewer than 4 s + 2 held input samples, the absolute gate's sum and count, a_{k-1}, and every sub-block's y^2
 * sum (8 bytes per 100 ms) in a store that starts at ten minutes and doubles in stream order.  Create allocates and
 * synchronises; output counts are host arithmetic and no other call synchronises.  Calls on one state are ordered on
 * one CUDA stream. */
typedef struct sopro_level_stream sopro_level_stream_t;
int sopro_level_stream_create(int64_t max_chunk, int32_t sr, int device, sopro_level_stream_t** out);
int sopro_level_stream_destroy(sopro_level_stream_t* s);
/* back to sample 0 with target T (host-only; also clears the finished state).  A new state takes no push until its
 * first reset; SOPRO_ERR_INVALID for a refused T. */
int sopro_level_stream_reset(sopro_level_stream_t* s, double T);
/* outputs the next call writes: a push of n_more samples (final == 0), or a push of n_more samples followed by finish
 * (final != 0); < 0 on bad arguments, before the first reset or after finish */
int64_t sopro_level_stream_ready(const sopro_level_stream_t* s, int64_t n_more, int final);
/* x [n] f32 (device) -> y (device) receives stream_ready(s, n, 0) outputs.  n > max_chunk: SOPRO_ERR_INVALID, nothing
 * launched, state unchanged.  After finish: SOPRO_ERR_STATE until a reset. */
int sopro_level_push(sopro_level_stream_t* s, const float* x, int64_t n, float* y, void* stream);
/* the remaining stream_ready(s, 0, 1) outputs -> y (device); SOPRO_ERR_STATE when called twice without a reset */
int sopro_level_finish(sopro_level_stream_t* s, float* y, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Long-form synthesis (no reference counterpart: the reference speaks one utterance of at most max_frames): the speech
 * extent of each segment's decoded 24 kHz row, and the join of those extents into one waveform.
 *   Extents: the energy trim of the reference's trim_silence_energy at 24 kHz.  For a row of n samples, frames of 600
 *   samples every 240, K = floor((n - 600) / 240) + 1; e_k = sum x^2 / 600 and dB_k = 10 log10(e_k + 1e-10), in fp64;
 *   thr = max(max_k dB_k - 40, -40); frame k is voiced when dB_k > thr; start = max(0, first * 240 - 720),
 *   end = min(n, last * 240 + 600 + 720).  The extent is (0, n) when n < 2400, no frame is voiced, or end - start < 12000.
 *   Each frame's sum has a fixed order, so a row gets the same extent alone or in any ragged batch.
 *   Join: for each non-empty extent in order, x[start, end) with its first and last F = min(240, floor(span / 2)) samples
 *   faded: y = x * f[i] for the i-th sample from the span's start and from its end, one fp32 multiply, with
 *   f[i] = 0.5 - 0.5 cos(pi (i + 0.5) / F) evaluated in double on the host and rounded to fp32 once; P zero samples
 *   between consecutive spans, none before the first or after the last.  The output has sum(spans) + (spans - 1) P
 *   samples. */
/* host-only: the fade's F taps -> f [F]; SOPRO_ERR_INVALID for F outside [0, 240] */
int sopro_longform_fade(int32_t F, float* f);
/* ragged batch, one launch per 128 rows: row b of x [B][x_stride] f32 (device) has lens_host[b] samples (HOST i64;
 * NULL = x_stride each); samples at or past lens[b] are not read.  (start, end) of row b -> ext [B][2] (device i64).
 * No call synchronises or allocates. */
int sopro_longform_extents(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int64_t* ext, void* stream);
/* src: HOST array of n_seg device pointers, segment i's row of lens_host[i] samples (HOST i64), read in place;
 * ext_host: HOST i64 [n_seg][2], each 0 <= start <= end <= lens[i] (an empty extent is skipped, its src may be NULL);
 * pause: P in [0, 48000] samples.  y (device f32) receives the joined waveform; y_len must equal its length.  Bad
 * geometry is SOPRO_ERR_INVALID before any launch.  No call synchronises or allocates. */
int sopro_longform_join(const float* const* src, int32_t n_seg, const int64_t* lens_host, const int64_t* ext_host, int64_t pause,
                        float* y, int64_t y_len, void* stream);
/* as sopro_longform_join, but pauses_host: HOST i64 [n_nonempty - 1], the zeros before each non-empty span after the
 * first, each in [0, 48000] (NULL when at most one span is non-empty); gain: DEVICE f32 [n_seg] or NULL (= 1); span i's
 * samples are gain[i] * (w * x), the faded product rounded first, exactly as sopro_loudness_normalize scales an
 * already-joined row, so a run of spans with one gain g equals that run joined alone and scaled by g, bit for bit.
 * sopro_longform_join is this entry point with every pause equal to `pause` and gain = NULL.  The dialogue join uses
 * it with a sentence pause inside a turn, a turn pause between turns and one loudness gain per turn. */
int sopro_longform_join_gaps(const float* const* src, int32_t n_seg, const int64_t* lens_host, const int64_t* ext_host,
                             const int64_t* pauses_host, const float* gain, float* y, int64_t y_len, void* stream);
/* Streaming trim: the extent of a row decided while its samples arrive, and the join emitted piece by piece.
 *   Causal rule: frame k (complete once 240 k + 600 samples have arrived) is classified once, when it completes, against
 *   thr_k = max(M_k - 40, -40), M_k the largest dB among frames 0 .. k; an earlier decision is never revisited.  When
 *   no frame of the row is above 0 dB (M <= 0) every thr_k is -40, the one-shot threshold, so the final extent is the
 *   one-shot extent above and the emitted pieces concatenate to the join bit for bit.  Louder rows get the causal
 *   rule's extent, which can start earlier than the one-shot one.
 *   Certain prefix: with f and l the first and last voiced frame so far and n the samples so far, start =
 *   max(0, 240 f - 720) and end_p = min(n, 240 l + 1320).  end_p only grows and start is fixed once f is, so once
 *   end_p - start >= 12000 the row is certain to be trimmed to a span of at least 12000 samples, F = 240, and
 *   [start, end_p - 240) is beyond the reach of its fade-out: that is the available bound.  Before that nothing is
 *   available.  When the row is final its extent is the one-shot rule's over its n samples (the whole row when
 *   n < 2400, nothing is voiced or the span is under 12000), and all of it is available.
 *   Status, per row i64 [5]: n, decided (start is known), start, the available bound (0 when undecided; the extent's
 *   end once final), final.
 * A state holds `rows` rows of at most max_len samples each on the device (rows <= 256, max_len <= 2^31); create
 * allocates and synchronises, and no other call does either.  Calls on one state are ordered on one CUDA stream, or
 * ordered by the caller. */
typedef struct sopro_longform_stream sopro_longform_stream_t;
int sopro_longform_stream_create(int32_t rows, int64_t max_len, int device, sopro_longform_stream_t** out);
int sopro_longform_stream_destroy(sopro_longform_stream_t* s);
/* rows [row0, row0 + n_rows) back to no samples (one launch) */
int sopro_longform_stream_reset(sopro_longform_stream_t* s, int32_t row0, int32_t n_rows, void* stream);
/* one launch for rows [row0, row0 + n_rows): row row0 + i appends counts_host[i] (HOST i64; 0 = the row did not run)
 * samples from x + i * x_stride (device f32), classifies its newly complete frames, and becomes final when
 * final_host[i] (HOST i32) is non-zero; then its status is written on the device.  A count past the capacity, a push
 * to a final row, or x_stride below the largest count (when n_rows > 1) is SOPRO_ERR_INVALID before any launch. */
int sopro_longform_stream_push(sopro_longform_stream_t* s, const float* x, int64_t x_stride, int32_t row0, int32_t n_rows,
                               const int64_t* counts_host, const int32_t* final_host, void* stream);
/* the status rows [row0, row0 + n_rows) -> status_host (HOST i64 [n_rows][5], pinned for an asynchronous copy) */
int sopro_longform_stream_status(const sopro_longform_stream_t* s, int32_t row0, int32_t n_rows, int64_t* status_host,
                                 void* stream);
/* pieces_host: HOST i64 [n_pieces][5] = (row, a, b, start, end); y (device f32, y_len = the pieces' total) receives,
 * back to back, samples [a, b) of the row's span [start, end) as the join writes them (fade-in over the span's first F
 * samples, fade-out over its last F, F = min(240, (end - start) / 2)), or, for end = -1, of a span whose end is not
 * known yet (F = 240, no fade-out: b must lie within the available bound); row = -1 is b - a pause zeros (a = 0).
 * Pieces outside the samples pushed are SOPRO_ERR_INVALID before any launch.  One launch per 48 pieces. */
int sopro_longform_stream_emit(const sopro_longform_stream_t* s, const int64_t* pieces_host, int32_t n_pieces, float* y,
                               int64_t y_len, void* stream);
/* Timeline mix (timed synthesis): n_items rows placed at absolute sample offsets and summed where they overlap.
 * src: HOST array of n_items device pointers, item i's row of lens_host[i] samples (HOST i64), read in place and placed
 * at offs_host[i] (HOST i64).  With i1 < i2 < ... the items covering sample t, in item order, y[t] (device f32 [y_len])
 * is src[i1][t - offs[i1]], then each later covering item's sample added with one round-to-nearest fp32 add, in item
 * order; 0 where no item covers t.  Every sample of y is written (the caller does not zero it); a sample covered by a
 * single item equals that item's sample bit for bit; the result depends only on the items, not on the tiling.
 * One launch for any item count: each 4096-sample tile's covering items reach the device through one stream-ordered
 * copy.  Refused before any launch: n_items < 0, a null src / lens_host / offs_host with items, a null source for a
 * non-empty item, a negative length or offset, offs + lens > y_len, y_len outside [0, 2^40], a null y with
 * y_len > 0. */
int sopro_timeline_mix(const float* const* src, int32_t n_items, const int64_t* lens_host, const int64_t* offs_host, float* y,
                       int64_t y_len, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Lossless FLAC output (RFC 9639; no reference counterpart: the reference's demo sends PCM16): mono, 16 bits per sample,
 * at a rate sr, an integer in [4000, 192000].  Every choice is fixed, so the device's bytes equal
 * oracle/flac_oracle.py's.
 *   Input: each fp32 sample -> trunc(clamp(x, -1, 1) * 32767.0f) (wire.float_to_pcm16le's rule); NaN -> 0.
 *   Stream: "fLaC", one metadata header (last 1, type 0, length 34), STREAMINFO: min / max block size (u16), min / max
 *   frame bytes (u24), sr (u20), channels - 1 = 0 (u3), bits - 1 = 15 (u5), total samples (u36), MD5 all zero ("not
 *   computed").  One-shot: fixed blocking, 4096-sample blocks (the last may be shorter), min = max block 4096, the exact
 *   frame sizes (0 with no frame) and total.  Stream: variable blocking, min block 16, max 4096, frame sizes and total 0.
 *   Frame header: 0xFF, 0xF8 (fixed) / 0xF9 (variable); block-size code 1100 for 4096, else 0110 + u8 (n - 1) when
 *   n <= 256, else 0111 + u16 (n - 1); rate code 0100 8k, 0101 16k, 0110 22.05k, 0111 24k, 1000 32k, 1001 44.1k,
 *   1010 48k, 1011 96k, 0001 88.2k, 0010 176.4k, 0011 192k, any other 0000 (from STREAMINFO); channels 0000, size
 *   100, reserved 0; the frame number (fixed) or first sample's number (variable) in FLAC's UTF-8 coding; the block-size
 *   bytes; CRC-8 (poly 0x07, init 0) over the header.
 *   Subframe: 0, 6-bit type, wasted-bits flag 0.  Candidates in order CONSTANT (all samples equal), FIXED 0-4, LPC 1-12,
 *   VERBATIM, order p only when p <= n; each sized exactly, the smallest wins, ties to the earlier.
 *   LPC: R[l] = sum s[n] s[n - l] (l = 0 .. 12, int64, exact in double); none when R[0] = 0.  Levinson-Durbin in double,
 *   one IEEE rounding per operation, err = R[0], for p = 1 .. 12: stop if !(err > 0) or err not finite;
 *   acc = R[p] - a[j] R[p-1-j] (j = 0 .. p-2, in order); k = acc / err; a[j] -= k a[p-2-j] (from the old a); a[p-1] = k;
 *   stop if any of these is not finite; err *= (1 - k k).  Precision 12: e = frexp exponent of max|a|,
 *   shift = min(11 - e, 15), the order skipped when max|a| = 0 or shift < 0; error-feedback rounding
 *   err' += a[j] 2^shift, q = clamp(round(err') (halves away from zero), -2048, 2047), err' -= q.  Residual
 *   s[n] - ((sum q[j] s[n-1-j]) >> shift), arithmetic shift; fields precision - 1 (u4), shift (s5), q[0 .. p-1] (s12).
 *   Residual coding: partitioned Rice, u = 2e or -2e - 1; a partition of m residuals costs m (k + 1) + sum(u >> k), k
 *   the cheapest in 0 .. 14 (method 00, 4-bit parameters) or 0 .. 30 (method 01, 5-bit), ties to the smaller k, no
 *   escapes; partition order o in 0 .. 8 with n % 2^o = 0 and (n >> o) >= p; per o the cheaper method (ties to 00), then
 *   the cheapest o (ties to the smaller).  Zero pad to a byte, then CRC-16 (poly 0x8005, init 0) over the frame.
 * A row's bytes depend only on its own samples. */
typedef struct SoproFlacStream SoproFlacStream;
/* host-only: the workspace bytes and the output bound (every row's worst case, VERBATIM plus headers) of one encode of
 * B rows of at most max_len samples; SOPRO_ERR_INVALID for a refused rate or geometry (max_len < 2^36) */
int sopro_flac_sizes(int32_t B, int64_t max_len, int32_t sr, int64_t* ws_bytes, int64_t* out_bytes);
/* ragged batch, one launch of each kernel per 128 rows: row b of x [B][x_stride] f32 (device) has lens_host[b] samples
 * (HOST i64; NULL = x_stride each); samples at or past lens[b] are not read.  ws: device, sopro_flac_sizes' bytes; out:
 * device, at least its bound.  Row b's complete stream lands at out + row_off[b], row_bytes[b] bytes (device i64 [B]),
 * the rows back to back in order.  A refused rate or geometry is SOPRO_ERR_INVALID before any launch.  No call
 * synchronises or allocates. */
int sopro_flac_encode(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, int32_t sr, void* ws,
                      uint8_t* out, int64_t* row_off, int64_t* row_bytes, void* stream);
/* a stream of frames (variable blocking; the header is the stream STREAMINFO above).  Each push of n samples, after the
 * carried ones, becomes 4096-sample frames and one remainder frame; a remainder under 16 samples (frames that short may
 * only end a stream) is carried on the device to the next push.  push: ws / out sized by sopro_flac_sizes(1, n + 15);
 * the frames' bytes -> out, their count -> *nbytes (device i64).  finish: the carried samples as the last frame (none
 * when nothing is carried), then the state starts over at sample 0.  create allocates the 2 x 16-sample carry. */
int sopro_flac_stream_create(int32_t sr, SoproFlacStream** out);
int sopro_flac_stream_destroy(SoproFlacStream* s);
int sopro_flac_stream_reset(SoproFlacStream* s, int32_t sr);
/* host-only: samples carried to the next push (0 .. 15); -1 for NULL */
int64_t sopro_flac_stream_carried(const SoproFlacStream* s);
int sopro_flac_stream_push(SoproFlacStream* s, const float* x, int64_t n, void* ws, uint8_t* out, int64_t* nbytes, void* stream);
int sopro_flac_stream_finish(SoproFlacStream* s, void* ws, uint8_t* out, int64_t* nbytes, void* stream);

/* ---- word alignment (no reference counterpart): the monotonic token -> frame path through the AR step's text
 * cross-attention weights (sopro_ar_set_attn_trace).  Per utterance b of L = text_len[b] tokens and T = frames[b] frames:
 *   A[t][l] = sum over s ascending, then h ascending, of (double) probs[t][s][b][h][l], starting from 0.0;
 *   S[0][0] = A[0][0], S[0][l > 0] = -inf; for t >= 1 S[t][l] = A[t][l] + max(S[t-1][l], S[t-1][l-1]) (S[t-1][-1] = -inf),
 *   the stay predecessor l winning ties; backtrack from (T-1, L-1).
 * first [B][ld] (device i32): first[b][l] = the first frame of token l, which owns frames [first[l], first[l+1]) with
 * first[L] := T; every token gets at least one frame.  Entries l >= L are -1, and so is the whole row when there is no
 * path (T < L or T == 0, or a path that does not start at (0, 0)).  IEEE double additions and comparisons only. */
/* host-only: the workspace bytes of one alignment; SOPRO_ERR_INVALID for bad geometry */
int sopro_align_sizes(int32_t B, int32_t steps, int64_t ld, int64_t* ws_bytes);
/* probs: device f32 [steps][n_attn][B][H][ld]; text_len_host, frames_host: HOST i32 [B], 1 <= text_len <= min(ld, 2048),
 * 0 <= frames <= steps; ws: device, sopro_align_sizes' bytes.  One CTA per utterance, one launch per 128 utterances.
 * Bad geometry is SOPRO_ERR_INVALID before any launch.  No call synchronises or allocates. */
int sopro_align(const float* probs, int32_t steps, int32_t n_attn, int32_t B, int32_t H, int64_t ld, const int32_t* text_len_host,
                const int32_t* frames_host, void* ws, int32_t* first, void* stream);

/* ---- streaming word alignment: a causal restatement of the one above, for streams.  Fixed-lag Viterbi with binding
 * commits, per row of L tokens and a lag of D >= 1 frames (oracle/align_stream_oracle.py::StreamAlign in float64):
 *   A[t][l] and S[t][l] are the one-shot's (same summation order, the stay predecessor winning ties).
 *   Commit: after S[t] for t >= D, frame c = t - D is committed.  l* = the lowest l with the largest finite S[t][l];
 *     the backtrack from (t, l*) to frame c gives token k_c; a token whose first frame is <= c on that path has that
 *     first frame, final (so first[k_c] = c when k_c moved past k_{c-1}; first[0] = 0 at c = 0).
 *   Prune: S[t][l] = -inf for every l whose backtrack to frame c is not k_c.  Every later path then extends the
 *     committed prefix: no commit is ever revised.
 *   End, with T = the row's frames: backtrack from (T-1, L-1) if that state is finite, else from the highest l whose
 *     S[T-1][l] is finite; tokens past the end state start at T (zero length).  T == 0 gives no path (first all -1).
 *   With no commit (T <= D) and T >= L the path is the one-shot path.  Unlike the one-shot, T < L still gives a path:
 *     the committed tokens, then zero-length ones.
 * The state lives in a caller-allocated device buffer of sopro_align_stream_sizes' bytes; its first
 * rows x (2 + ld) i32 are, per row, {F = frames committed, K = tokens whose first frame is final, first[ld]}: first[l]
 * is -1 until committed, and past the row's end F = T, K = L and first is the whole path (-1 from L on, or the whole row
 * when there is no path).  A stream of several rows: rows <= 256; a row's frames t come from the ring trace of
 * sopro_ar_set_attn_trace_ring, slot t % ring.  No call synchronises; only create and destroy touch the heap, on the host. */
typedef struct sopro_align_stream sopro_align_stream_t;
/* host-only: the device state bytes; SOPRO_ERR_INVALID for bad geometry (rows not in [1, 256], ld, lag or max_frames < 1) */
int sopro_align_stream_sizes(int32_t rows, int64_t ld, int32_t lag, int32_t max_frames, int64_t* state_bytes);
/* state: device, sopro_align_stream_sizes' bytes, owned by the caller for the stream's life; max_frames: the most frames
 * a row takes between two begins */
int sopro_align_stream_create(int32_t rows, int64_t ld, int32_t lag, int32_t max_frames, void* state,
                              sopro_align_stream_t** out);
int sopro_align_stream_destroy(sopro_align_stream_t* s);
/* every row starts over with text_len_host[b] (HOST i32 [rows], in [1, min(ld, 2048)]) tokens: one reset launch */
int sopro_align_stream_begin(sopro_align_stream_t* s, const int32_t* text_len_host, void* stream);
/* probs: the ring trace, device f32 [ring][n_attn][B][H][ld] with B = rows and ld = the state's; frames_host[b] (HOST,
 * in [0, ring]): row b's new frames, which sit in the ring now; end_host[b] (HOST): nonzero when the row ends after them.
 * One launch for every row (one CTA per row; none when no row has work).  A row that has ended takes no frames and no
 * second end until the next begin; a row's frames past max_frames, bad geometry and a null probs with frames are
 * SOPRO_ERR_INVALID, before any launch. */
int sopro_align_stream_push(sopro_align_stream_t* s, const float* probs, int32_t ring, int32_t n_attn, int32_t B, int32_t H,
                            int64_t ld, const int32_t* frames_host, const int32_t* end_host, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Watermark (no reference counterpart): a keyed spread-spectrum mark on 24 kHz audio, and its detector.  A key is an
 * integer in [0, 2^32).
 *   Pattern: P = SOPRO_WATERMARK_PERIOD samples.  The real-DFT bins k with LO_HZ <= k 24000 / P <= HI_HZ (k = 342 ..
 *   1194) get unit magnitude and phase 2 pi u_k, u_k = (z >> 11) 2^-53 for splitmix64's outputs z seeded with the key,
 *   one per bin in bin order; every other bin is zero.  p[n] = sum_k cos(2 pi k n / P + 2 pi u_k) in double, scaled to
 *   unit RMS, rounded to fp32 once.
 *   Embed: blocks of SOPRO_WATERMARK_BLOCK samples from the utterance's first sample; r_j = sqrt(sum x^2 / count) over
 *   block j (a trailing partial block over its own samples), summed in double in a fixed order that depends only on
 *   the block's samples; g_j = fp32(a min(r_{j-1}, r_j)), r_{-1} = 0, a = 10^(LEVEL_DB / 20);
 *   y[n] = fma(g_{j(n)}, p[n mod P], x[n]), and y = x bit for bit where g = 0.
 *   Detect: r_j as above from the clip's first sample; w_j = 1 / r_j where r_j > max(10^(FLOOR_DB / 20) max_j r_j, 1e-6),
 *   else 0; F[k] = sum over n = k (mod P) of w_{j(n)} x[n] (double, stored fp32); c[l] = sum_k F[k] p[(k + l) mod P]
 *   for every lag l (fp32, direct); score = max c / sqrt(mean c^2) (0 when c = 0), offset = the first argmax (the
 *   pattern's phase at the clip's first sample), detected = score >= THRESHOLD.
 * A row's results depend only on its own samples.  No call synchronises or allocates, except stream_create. */
#define SOPRO_WATERMARK_PERIOD 8192
#define SOPRO_WATERMARK_BLOCK 240
#define SOPRO_WATERMARK_LO_HZ 1000
#define SOPRO_WATERMARK_HI_HZ 3500
#define SOPRO_WATERMARK_LEVEL_DB (-30.0)
#define SOPRO_WATERMARK_FLOOR_DB (-40.0)
#define SOPRO_WATERMARK_THRESHOLD 7.0
typedef struct sopro_watermark_stream sopro_watermark_stream_t;
/* host-only: the key's pattern -> out [P] f32 (host); SOPRO_ERR_INVALID for a key outside [0, 2^32) */
int sopro_watermark_pattern(int64_t key, float* out);
/* host-only: the device workspace bytes of one embed / one detect of B rows of at most max_len samples (either
 * pointer may be NULL); SOPRO_ERR_INVALID for bad geometry */
int sopro_watermark_sizes(int32_t B, int64_t max_len, int64_t* embed_ws, int64_t* detect_ws);
/* ragged batch, two launches per 128 rows: row b of x [B][x_stride] f32 (device) has lens_host[b] samples (HOST i64;
 * NULL = x_stride each); samples at or past lens[b] are not read.  pattern: device f32 [P].  Row b's marked samples go to
 * y + b * y_stride (device; y_stride >= the longest row when B > 1); the rest of the row is not written. */
int sopro_watermark_embed(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, const float* pattern, float* y,
                          int64_t y_stride, void* ws, void* stream);
/* ragged batch as the embed; per row score -> score [B] (device f32), offset -> offset [B] (device i64), the decision
 * -> detected [B] (device u8, 0 or 1).  Four launches per 128 rows. */
int sopro_watermark_detect(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, const float* pattern, void* ws,
                           float* score, int64_t* offset, uint8_t* detected, void* stream);
/* Streaming embed: one utterance pushed in chunks of at most max_chunk samples.  A push emits every complete block
 * (held + n rounded down to a multiple of BLOCK), holding back at most BLOCK - 1 samples; finish emits the held ones as
 * the last, partial block.  The concatenated outputs equal sopro_watermark_embed of the concatenated input bit for bit,
 * under any chunk schedule.  The state on the device: the held samples and the last block's r; output counts are host
 * arithmetic.  Calls on one state must be ordered (one CUDA stream). */
int sopro_watermark_stream_create(int64_t max_chunk, int device, sopro_watermark_stream_t** out);
int sopro_watermark_stream_destroy(sopro_watermark_stream_t* s);
/* back to sample 0 with this key's pattern (device f32 [P], kept alive by the caller until the next reset; host-only).
 * A new state takes no push until its first reset. */
int sopro_watermark_stream_reset(sopro_watermark_stream_t* s, const float* pattern);
/* outputs the next call writes: a push of n_more samples (final == 0), or a push followed by finish (final != 0); < 0 on
 * bad arguments, before the first reset or after finish */
int64_t sopro_watermark_stream_ready(const sopro_watermark_stream_t* s, int64_t n_more, int final);
/* x [n] f32 (device) -> y (device) receives stream_ready(s, n, 0) outputs.  n > max_chunk: SOPRO_ERR_INVALID, nothing
 * launched, state unchanged.  After finish: SOPRO_ERR_STATE until a reset. */
int sopro_watermark_push(sopro_watermark_stream_t* s, const float* x, int64_t n, float* y, void* stream);
/* the held samples, marked -> y (device); SOPRO_ERR_STATE when called twice without a reset */
int sopro_watermark_finish(sopro_watermark_stream_t* s, float* y, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Reference-voice denoising (no reference counterpart): a stationary-noise Wiener suppressor with the decision-directed
 * a priori SNR estimate (Ephraim-Malah), for SoproTTS.prepare_references(denoise=True).  Each row of n samples at
 * 24 kHz on its own:
 *   Frames: N = SOPRO_DENOISE_FRAME, R = SOPRO_DENOISE_HOP; w[j] = sqrt(0.5 - 0.5 cos(2 pi j / N)) (periodic sqrt-Hann)
 *   for analysis and synthesis; M = ceil(n / R) + 1 frames, frame m covering samples [(m - 1) R, (m + 1) R) with zeros
 *   outside [0, n); X[m][k], k = 0 .. N/2, and P[m][k] = |X|^2.
 *   Noise, once per row: E[m] = sum of P[m][k], in double with k ascending.  Of the C = floor(n / R) - 1 frames wholly
 *   inside the row (m = 1 .. C), the K = max(1, floor(C / 10)) with the smallest E, ties to the lower m; lambda[k] = the
 *   mean of their P[m][k], summed in double with m ascending.
 *   Gain, per bin, in double: gamma = P / lambda; xi[0] = max(gamma[0] - 1, 0);
 *   xi[m] = 0.98 G[m-1]^2 gamma[m-1] + 0.02 max(gamma[m] - 1, 0); G[m] = max(xi / (1 + xi), 0.1) (a -20 dB floor);
 *   G = 1 in every frame of a bin where lambda = 0.
 *   Synthesis: G X, inverse real FFT, times w; y[i] = frame q's second half + frame q + 1's first half, q = floor(i / R),
 *   added in that order.
 *   A row with n < N or a non-finite E[m] comes back unchanged.  w^2 at hop N/2 sums to 1, so G = 1 reconstructs the
 *   input in exact arithmetic.
 * The device FFT is a 512-point shared-memory radix-2 transform in fp32 (twiddles and window computed in double, rounded
 * once); E, lambda and the recursion run in double.  Every sum runs in an order fixed by the row's own positions, so a
 * row's output is the same alone and in any batch, bit for bit.  No call synchronises or allocates. */
#define SOPRO_DENOISE_FRAME 512
#define SOPRO_DENOISE_HOP 256
/* host-only: the device workspace bytes of one call over B rows of at most max_len samples; SOPRO_ERR_INVALID for bad
 * geometry (B < 1, max_len outside [0, 2^36]) or a null ws_bytes */
int sopro_denoise_sizes(int32_t B, int64_t max_len, int64_t* ws_bytes);
/* ragged batch, five launches per 128 rows: row b of x [B][x_stride] f32 (device) has lens_host[b] samples (HOST i64;
 * NULL = x_stride each); samples at or past lens[b] are not read.  Row b of y (device, y + b * y_stride, y_stride >=
 * x_stride when B > 1) receives lens[b] outputs, then zeros up to x_stride.  ws: device, sopro_denoise_sizes(B, the
 * longest row) bytes; on return it begins with sel [B][Kmax] i32, Kmax = K of the longest row (1 below N): row b's
 * selected noise frames in ascending order, then -1 (all -1 for a row that passed through) -- a test hook.  y must not
 * overlap x.  Bad geometry or a null pointer is SOPRO_ERR_INVALID before any launch. */
int sopro_denoise(const float* x, int32_t B, int64_t x_stride, const int64_t* lens_host, void* ws, float* y, int64_t y_stride,
                  void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SOPRO_B200_H_ */
