// Host side of the AR engine + the C-ABI declared in include/sopro_b200.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/sopro_b200.h"
#include "common.cuh"
#include "ar_kernel.cuh"

using namespace sopro;

namespace {

thread_local std::string g_err;

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

uint16_t f32_to_bf16_rne(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);  // NaN
  const uint32_t lsb = (u >> 16) & 1u;
  u += 0x7fffu + lsb;
  return (uint16_t)(u >> 16);
}

struct Arena {
  std::vector<unsigned char> host;
  size_t add(size_t bytes) {
    const size_t off = align_up(host.size(), 256);
    host.resize(off + bytes);
    return off;
  }
  size_t add_f32(const float* src, size_t n) {
    const size_t off = add(n * 4);
    memcpy(host.data() + off, src, n * 4);
    return off;
  }
  size_t add_mat(const float* src, size_t n, int wdtype) {
    if (wdtype == SOPRO_W_F32) return add_f32(src, n);
    const size_t off = add(n * 2);
    uint16_t* d = reinterpret_cast<uint16_t*>(host.data() + off);
    for (size_t i = 0; i < n; ++i) d[i] = f32_to_bf16_rne(src[i]);
    return off;
  }
};

}  // namespace

namespace mimi {
void set_error(const char* msg) { g_err = msg; }
}  // namespace mimi

struct sopro_engine {
  int device = 0;
  int n_sms = 0;
  sopro_ar_config_t cfg{};
  int D = 0, F = 0, V = 0, Vpad = 0, H = 0, Dh = 0, Kc = 0, n_layers = 0, n_attn = 0;
  unsigned char* dev = nullptr;  // weight arena
  size_t dev_bytes = 0;
  int64_t step_weight_bytes = 0;
  LayerDev layer[kMaxLayers]{};
  const float* nkv_w[kMaxLayers]{};  // per attn slot
  const void* wk[kMaxLayers]{};
  const void* wv[kMaxLayers]{};
  const float* final_norm_w = nullptr;
  const void* head_w = nullptr;
  const float* head_b = nullptr;
  const float* emb = nullptr;
  const float* epi[kMaxLayers]{};  // packed [D][KcE]: dwconv taps, dwconv bias, GLU value bias, GLU gate bias
  int KcP = 0, KcE = 0;
  long long ring_floats_per_utt = 0;
};

struct sopro_ar_session {
  sopro_engine* e = nullptr;
  int max_batch = 0, max_steps = 0, Lmax = 0;
  int utts_per_team = 0;  // 0 = auto
  int task_shape = 0;     // 0 = picked per stage by launch_ar, 1 = always wide, 2 = always narrow (test hook)
  StageOp last_prog[kMaxStages]{};  // the stage program of the last launch (with each stage's task shape)
  int last_n_stage = 0;
  // device buffers
  float *ring = nullptr, *xa = nullptr, *xb = nullptr, *hbuf = nullptr, *qbuf = nullptr, *abuf = nullptr,
        *logits = nullptr, *kc = nullptr, *vc = nullptr;
  int *tokens = nullptr, *sampled = nullptr, *text_len = nullptr, *n_tokens = nullptr, *done = nullptr;
  UttState* st = nullptr;
  SamplingDev* samp = nullptr;
  unsigned* barrier = nullptr;
  unsigned* tok_ll = nullptr;
  unsigned seq_base = 0;
  TileDesc* tiles = nullptr;  // [n_sms][kMaxTilesPerStep]
  int* n_tiles = nullptr;     // [n_sms]
  unsigned char* stage_tiles = nullptr;  // [n_sms][kMaxStages]
  std::vector<unsigned char> h_stage_tiles;
  int tile_P = -1, tile_wbuf = -1, tile_qatt = -1;
  bool qatt = false;  // this launch geometry uses the fused q + attention stage
  std::vector<TileDesc> h_tiles;
  std::vector<int> h_ntiles;
  // staging for the host-buffer path
  float *h_cond = nullptr, *h_txt = nullptr, *h_noise = nullptr;
  size_t h_cond_cap = 0, h_txt_cap = 0, h_noise_cap = 0;
  // current batch
  int B = 0, steps = 0, noise_k = 0, t_pos = 0;
  const float* cond = nullptr;
  const float* noise = nullptr;
  const int* forced = nullptr;
  float* trace_blocks = nullptr;
  float* trace_logits = nullptr;
  long long* timing = nullptr;
  int timing_step = -1;
  float* attn_trace = nullptr;  // word timestamps: [steps][n_attn][B][H][attn_ld] (null = off)
  int64_t attn_ld = 0;
  int attn_ring = 0;  // the trace's step rows: step t goes to row t % attn_ring (0 = the batch's steps, no ring)
  int max_len = 0;  // longest text of the current batch
  bool begun = false;
  std::vector<UttState> host_st;
  // pinned staging of begin()'s small uploads (text lengths, sampler parameters, initial states): the copies are asynchronous
  // and begin() does not wait for the stream (it used to synchronise because the sources were pageable vectors)
  unsigned char* pin = nullptr;
  size_t pin_bytes = 0;
  cudaEvent_t pin_done = nullptr;  // last begin()'s uploads have left the staging buffer
};

extern "C" {

const char* sopro_last_error(void) { return g_err.c_str(); }
const char* sopro_version(void) { return "sopro_b200 0.1 (sm_90a)"; }

int sopro_engine_create(const sopro_ar_config_t* cfg, const sopro_ar_weights_t* w, int device,
                        sopro_engine_t** out) {
  if (!cfg || !w || !out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  const int rc = open_device(device, "the AR engine");
  if (rc != SOPRO_OK) return rc;
  const int D = cfg->d_model, NL = cfg->n_layers, Kc = cfg->kernel, H = cfg->n_heads, V = cfg->vocab;
  if (D <= 0 || D % 4 != 0) return fail(SOPRO_ERR_INVALID, "d_model must be a positive multiple of 4 (got %d)", D);
  if (NL <= 0 || NL > kMaxLayers) return fail(SOPRO_ERR_INVALID, "n_layers must be in [1,%d]", kMaxLayers);
  if (H <= 0 || D % H != 0 || (D / H) % 4 != 0 || D / H > 128)
    return fail(SOPRO_ERR_INVALID, "bad head geometry D=%d H=%d (head_dim must be a multiple of 4, <= 128)", D, H);
  if (Kc < 1 || Kc > 64) return fail(SOPRO_ERR_INVALID, "kernel must be in [1,64]");
  if (V < 2 || V > kMaxVocab) return fail(SOPRO_ERR_INVALID, "vocab must be in [2,%d]", kMaxVocab);
  if (cfg->eos_id < 0 || cfg->eos_id >= V) return fail(SOPRO_ERR_INVALID, "eos_id out of range");
  if (cfg->weight_dtype != SOPRO_W_F32 && cfg->weight_dtype != SOPRO_W_BF16)
    return fail(SOPRO_ERR_INVALID, "weight_dtype must be 0 (f32) or 1 (bf16)");
  if (w->cb_embed_rows < V || w->bos_row < 0 || w->bos_row >= w->cb_embed_rows)
    return fail(SOPRO_ERR_INVALID, "cb_embed has %lld rows, need >= vocab %d and a valid bos_row",
                (long long)w->cb_embed_rows, V);
  int n_sms = 0;
  CK(cudaDeviceGetAttribute(&n_sms, cudaDevAttrMultiProcessorCount, device));

  sopro_engine* e = new sopro_engine();
  e->device = device;
  e->n_sms = n_sms;
  e->cfg = *cfg;
  e->D = D;
  e->F = 4 * D;
  e->V = V;
  e->Vpad = (int)align_up((size_t)V, 4);
  e->H = H;
  e->Dh = D / H;
  e->Kc = Kc;
  e->n_layers = NL;
  e->KcP = (int)align_up((size_t)Kc, 4);
  e->KcE = (int)align_up((size_t)Kc + 3, 4);
  const int wd = cfg->weight_dtype;
  const size_t wsz = wd == SOPRO_W_F32 ? 4 : 2;

  Arena A;
  struct Off {
    size_t norm_w, glu_w, glu_b, dw_w, dw_b, ffn_norm_w, w1, b1, w2, b2, nq_w, nkv_w, wq, wk, wv, wo, epi;
  } off[kMaxLayers];
  int64_t step_bytes = 0;
  int n_attn = 0;
  long long ring_off = 0;
  for (int i = 0; i < NL; ++i) {
    const sopro_ar_layer_weights_t& L = w->layer[i];
    if (!L.norm_w || !L.glu_w || !L.glu_b || !L.dw_w || !L.dw_b || !L.ffn_norm_w || !L.ffn_w1 || !L.ffn_b1 ||
        !L.ffn_w2 || !L.ffn_b2) {
      delete e;
      return fail(SOPRO_ERR_INVALID, "layer %d: null weight pointer", i);
    }
    if (cfg->dilation[i] < 1) {
      delete e;
      return fail(SOPRO_ERR_INVALID, "layer %d: dilation must be >= 1", i);
    }
    off[i].norm_w = A.add_f32(L.norm_w, D);
    off[i].glu_w = A.add_mat(L.glu_w, (size_t)2 * D * D, wd);
    off[i].glu_b = A.add_f32(L.glu_b, 2 * D);
    off[i].dw_w = A.add_f32(L.dw_w, (size_t)D * Kc);
    off[i].dw_b = A.add_f32(L.dw_b, D);
    off[i].ffn_norm_w = A.add_f32(L.ffn_norm_w, D);
    off[i].w1 = A.add_mat(L.ffn_w1, (size_t)4 * D * D, wd);
    off[i].b1 = A.add_f32(L.ffn_b1, 4 * D);
    off[i].w2 = A.add_mat(L.ffn_w2, (size_t)4 * D * D, wd);
    off[i].b2 = A.add_f32(L.ffn_b2, D);
    {
      std::vector<float> er((size_t)D * e->KcE, 0.f);
      for (int c = 0; c < D; ++c) {
        float* r = er.data() + (size_t)c * e->KcE;
        for (int j = 0; j < Kc; ++j) r[j] = L.dw_w[(size_t)c * Kc + j];
        r[Kc] = L.dw_b[c];
        r[Kc + 1] = L.glu_b[c];
        r[Kc + 2] = L.glu_b[c + D];
      }
      off[i].epi = A.add_f32(er.data(), er.size());
    }
    step_bytes += (int64_t)(D + 2 * D + (size_t)D * Kc + D + D + 4 * D + D) * 4 + (int64_t)(2 + 4 + 4) * D * D * wsz;
    if (cfg->has_attn[i]) {
      if (!L.nq_w || !L.nkv_w || !L.q_w || !L.k_w || !L.v_w || !L.o_w) {
        delete e;
        return fail(SOPRO_ERR_INVALID, "layer %d: has_attn set but attention weights are null", i);
      }
      off[i].nq_w = A.add_f32(L.nq_w, D);
      off[i].nkv_w = A.add_f32(L.nkv_w, D);
      off[i].wq = A.add_mat(L.q_w, (size_t)D * D, wd);
      off[i].wk = A.add_mat(L.k_w, (size_t)D * D, wd);
      off[i].wv = A.add_mat(L.v_w, (size_t)D * D, wd);
      off[i].wo = A.add_mat(L.o_w, (size_t)D * D, wd);
      step_bytes += (int64_t)D * 4 + (int64_t)2 * D * D * wsz + 4;
    }
  }
  const size_t off_fn = A.add_f32(w->final_norm_w, D);
  const size_t off_hw = A.add_mat(w->head_w, (size_t)V * D, wd);
  const size_t off_hb = A.add_f32(w->head_b, V);
  step_bytes += (int64_t)D * 4 + (int64_t)V * D * wsz + (int64_t)V * 4;
  // compact embedding table: rows 0..V-1 (cb_index 0 -> row == token id, nn/embeddings.py:51-55;
  // row V-1 == table row 2048 is what an early EOS feeds back) + the BOS row
  const size_t off_emb = A.add((size_t)(V + 1) * D * 4);
  memcpy(A.host.data() + off_emb, w->cb_embed, (size_t)V * D * 4);
  memcpy(A.host.data() + off_emb + (size_t)V * D * 4, w->cb_embed + (size_t)w->bos_row * D, (size_t)D * 4);

  e->dev_bytes = align_up(A.host.size(), 256);
  cudaError_t err = cudaMalloc(&e->dev, e->dev_bytes);
  if (err != cudaSuccess) {
    delete e;
    return fail(SOPRO_ERR_CUDA, "cudaMalloc(%zu) failed: %s", e->dev_bytes, cudaGetErrorString(err));
  }
  err = cudaMemcpy(e->dev, A.host.data(), A.host.size(), cudaMemcpyHostToDevice);
  if (err != cudaSuccess) {
    cudaFree(e->dev);
    delete e;
    return fail(SOPRO_ERR_CUDA, "weight upload failed: %s", cudaGetErrorString(err));
  }
  auto F32 = [&](size_t o) { return reinterpret_cast<const float*>(e->dev + o); };
  auto PTR = [&](size_t o) { return reinterpret_cast<const void*>(e->dev + o); };
  for (int i = 0; i < NL; ++i) {
    LayerDev& L = e->layer[i];
    L.norm_w = F32(off[i].norm_w);
    L.glu_w = PTR(off[i].glu_w);
    L.glu_b = F32(off[i].glu_b);
    L.dw_w = F32(off[i].dw_w);
    L.dw_b = F32(off[i].dw_b);
    L.ffn_norm_w = F32(off[i].ffn_norm_w);
    L.w1 = PTR(off[i].w1);
    L.b1 = F32(off[i].b1);
    L.w2 = PTR(off[i].w2);
    L.b2 = F32(off[i].b2);
    e->epi[i] = F32(off[i].epi);
    L.dil = cfg->dilation[i];
    L.ring_len = (Kc - 1) * L.dil + 1;
    L.has_attn = cfg->has_attn[i] ? 1 : 0;
    L.attn_slot = -1;
    if (L.has_attn) {
      L.nq_w = F32(off[i].nq_w);
      L.wq = PTR(off[i].wq);
      L.wo = PTR(off[i].wo);
      L.gate_tanh = w->layer[i].gate_tanh;
      L.attn_slot = n_attn;
      e->nkv_w[n_attn] = F32(off[i].nkv_w);
      e->wk[n_attn] = PTR(off[i].wk);
      e->wv[n_attn] = PTR(off[i].wv);
      ++n_attn;
    }
    ring_off += (long long)D * L.dil * e->KcP;  // conv state per utterance: [D][dil][KcP]
  }
  e->n_attn = n_attn;
  e->ring_floats_per_utt = ring_off;
  e->final_norm_w = F32(off_fn);
  e->head_w = PTR(off_hw);
  e->head_b = F32(off_hb);
  e->emb = F32(off_emb);
  e->step_weight_bytes = step_bytes;
  *out = e;
  return SOPRO_OK;
}

int sopro_engine_destroy(sopro_engine_t* e) {
  if (!e) return SOPRO_OK;
  cudaSetDevice(e->device);
  if (e->dev) cudaFree(e->dev);
  delete e;
  return SOPRO_OK;
}

int64_t sopro_engine_step_weight_bytes(const sopro_engine_t* e) { return e ? e->step_weight_bytes : 0; }
int sopro_engine_num_sms(const sopro_engine_t* e) { return e ? e->n_sms : 0; }

static void session_free(sopro_ar_session* s) {
  cudaFree(s->ring);
  cudaFree(s->xa);
  cudaFree(s->xb);
  cudaFree(s->hbuf);
  cudaFree(s->qbuf);
  cudaFree(s->abuf);
  cudaFree(s->logits);
  cudaFree(s->kc);
  cudaFree(s->vc);
  cudaFree(s->tokens);
  cudaFree(s->sampled);
  cudaFree(s->text_len);
  cudaFree(s->n_tokens);
  cudaFree(s->done);
  cudaFree(s->st);
  cudaFree(s->samp);
  cudaFree(s->barrier);
  cudaFree(s->tok_ll);
  cudaFree(s->tiles);
  cudaFree(s->n_tiles);
  cudaFree(s->stage_tiles);
  if (s->pin) cudaFreeHost(s->pin);
  if (s->pin_done) cudaEventDestroy(s->pin_done);
  cudaFree(s->h_cond);
  cudaFree(s->h_txt);
  cudaFree(s->h_noise);
}

int sopro_ar_session_create(sopro_engine_t* e, int max_batch, int max_steps, int max_text_len,
                            sopro_ar_session_t** out) {
  if (!e || !out) return fail(SOPRO_ERR_INVALID, "null argument");
  *out = nullptr;
  if (max_batch < 1 || max_steps < 1 || max_text_len < 1)
    return fail(SOPRO_ERR_INVALID, "max_batch, max_steps, max_text_len must be >= 1");
  if (max_batch > e->n_sms * 16)
    return fail(SOPRO_ERR_INVALID, "max_batch %d exceeds %d (SMs x %d utterances per team)", max_batch,
                e->n_sms * 16, 16);
  CK(cudaSetDevice(e->device));
  sopro_ar_session* s = new sopro_ar_session();
  s->e = e;
  s->max_batch = max_batch;
  s->max_steps = max_steps;
  s->Lmax = (int)align_up((size_t)max_text_len, 4);
  const size_t B = max_batch, D = e->D, F = e->F;
  const size_t kv = (size_t)std::max(e->n_attn, 1) * B * s->Lmax * D;
  cudaError_t err = cudaSuccess;
  auto A = [&](void** p, size_t bytes) {
    if (err == cudaSuccess) err = cudaMalloc(p, std::max<size_t>(bytes, 256));
  };
  A((void**)&s->ring, (size_t)e->ring_floats_per_utt * B * 4);
  // exchange buffers are sized for the LL layout (value + flag per element)
  A((void**)&s->xa, B * D * 8);
  A((void**)&s->xb, B * D * 8);
  A((void**)&s->hbuf, B * F * 8);
  A((void**)&s->qbuf, B * D * 8);
  A((void**)&s->abuf, B * D * 8);
  A((void**)&s->logits, B * e->Vpad * 8);
  A((void**)&s->tok_ll, B * 8);
  A((void**)&s->kc, kv * 4);
  A((void**)&s->vc, kv * 4);
  A((void**)&s->tokens, B * max_steps * 4);
  A((void**)&s->sampled, B * max_steps * 4);
  A((void**)&s->text_len, B * 4);
  A((void**)&s->n_tokens, B * 4);
  A((void**)&s->done, B * 4);
  A((void**)&s->st, B * sizeof(UttState));
  A((void**)&s->samp, B * sizeof(SamplingDev));
  A((void**)&s->barrier, (size_t)e->n_sms * 32 * 4);
  A((void**)&s->tiles, (size_t)e->n_sms * kMaxTilesPerStep * sizeof(TileDesc));
  A((void**)&s->n_tiles, (size_t)e->n_sms * 4);
  A((void**)&s->stage_tiles, (size_t)e->n_sms * kMaxStages);
  if (err != cudaSuccess) {
    session_free(s);
    delete s;
    return fail(SOPRO_ERR_CUDA, "session allocation failed: %s", cudaGetErrorString(err));
  }
  *out = s;
  return SOPRO_OK;
}

int sopro_ar_session_destroy(sopro_ar_session_t* s) {
  if (!s) return SOPRO_OK;
  cudaSetDevice(s->e->device);
  session_free(s);
  delete s;
  return SOPRO_OK;
}

int sopro_ar_session_set_team(sopro_ar_session_t* s, int utts_per_team) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null session");
  if (utts_per_team < 0 || utts_per_team > kMaxUttPerTeam)
    return fail(SOPRO_ERR_INVALID, "utts_per_team must be in [0,%d]", kMaxUttPerTeam);
  s->utts_per_team = utts_per_team;
  return SOPRO_OK;
}

int sopro_ar_session_set_task_shape(sopro_ar_session_t* s, int mode) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null session");
  if (mode < 0 || mode > 2) return fail(SOPRO_ERR_INVALID, "task shape mode must be 0 (auto), 1 (wide) or 2 (narrow)");
  s->task_shape = mode;
  return SOPRO_OK;
}

int sopro_ar_session_stage_shapes(sopro_ar_session_t* s, int32_t* kinds, int32_t* shapes, int cap, int32_t* n_stage) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null session");
  if (cap < 0 || (cap > 0 && (!kinds || !shapes))) return fail(SOPRO_ERR_INVALID, "stage_shapes: bad output buffers");
  for (int i = 0; i < s->last_n_stage && i < cap; ++i) {
    kinds[i] = s->last_prog[i].kind;
    shapes[i] = s->last_prog[i].shape;
  }
  if (n_stage) *n_stage = s->last_n_stage;
  return SOPRO_OK;
}

}  // extern "C"

template <typename WT>
static int launch_kv(sopro_ar_session* s, const float* txt, int text_stride, const std::vector<int>& lens,
                     cudaStream_t st) {
  sopro_engine* e = s->e;
  if (e->n_attn == 0) return SOPRO_OK;
  KvParams kp{};
  kp.D = e->D;
  kp.H = e->H;
  kp.Dh = e->Dh;
  kp.B = s->B;
  kp.Lmax = s->Lmax;
  kp.text_stride = text_stride;
  kp.n_attn = e->n_attn;
  kp.txt = txt;
  kp.text_len = s->text_len;
  for (int i = 0; i < e->n_attn; ++i) {
    kp.nkv_w[i] = e->nkv_w[i];
    kp.wk[i] = e->wk[i];
    kp.wv[i] = e->wv[i];
  }
  kp.kc = s->kc;
  kp.vc = s->vc;
  int maxlen = 0;
  for (int v : lens) maxlen = std::max(maxlen, v);
  dim3 grid((maxlen + 15) / 16, s->B, e->n_attn);
  const size_t smem = (size_t)16 * e->D * 4;
  CK(cudaFuncSetAttribute(kv_build_kernel<WT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kv_build_kernel<WT><<<grid, kThreads, smem, st>>>(kp);
  CK(cudaGetLastError());
  return SOPRO_OK;
}

extern "C" {

int sopro_ar_begin(sopro_ar_session_t* s, int batch, int steps, const float* cond_ar, const float* txt_seq,
                   int text_stride, const int32_t* text_len, const float* noise, int noise_k,
                   const sopro_ar_sampling_t* sampling, void* stream) {
  if (!s || !cond_ar || !txt_seq || !text_len || !noise || !sampling)
    return fail(SOPRO_ERR_INVALID, "null argument");
  sopro_engine* e = s->e;
  if (batch < 1 || batch > s->max_batch) return fail(SOPRO_ERR_INVALID, "batch %d not in [1,%d]", batch, s->max_batch);
  if (steps < 1 || steps > s->max_steps) return fail(SOPRO_ERR_INVALID, "steps %d not in [1,%d]", steps, s->max_steps);
  if (text_stride < 1) return fail(SOPRO_ERR_INVALID, "text_stride must be >= 1");
  std::vector<int> lens(batch);
  std::vector<SamplingDev> sd(batch);
  for (int b = 0; b < batch; ++b) {
    lens[b] = text_len[b];
    if (lens[b] < 1 || lens[b] > s->Lmax || lens[b] > text_stride)
      return fail(SOPRO_ERR_INVALID, "text_len[%d]=%d not in [1,min(%d,%d)]", b, lens[b], s->Lmax, text_stride);
    const sopro_ar_sampling_t& q = sampling[b];
    if (q.top_k < 1 || q.top_k > kMaxTopK)
      return fail(SOPRO_ERR_INVALID, "sampling[%d].top_k=%d not in [1,%d] (top_k=0 is not on the ar_stream path)", b,
                  q.top_k, kMaxTopK);
    const int need = (q.top_p < 1.0f && q.recovery_top_p < 1.0f) ? std::min(q.top_k, e->V) : e->V;
    if (noise_k < need)
      return fail(SOPRO_ERR_INVALID, "noise_k=%d too small: utterance %d needs %d draws per step", noise_k, b, need);
    sd[b].top_p = q.top_p;
    sd[b].temperature = q.temperature;
    sd[b].rec_top_p = q.recovery_top_p;
    sd[b].rec_temp = q.recovery_temp;
    sd[b].rep_pen = q.repetition_penalty;
    sd[b].top_k = q.top_k;
    sd[b].anti_loop = q.anti_loop;
    sd[b].loop_streak = q.loop_streak;
    sd[b].min_gen = q.min_gen_frames;
    sd[b].stop_on_first_eos = q.stop_on_first_eos;
  }
  const int max_len = *std::max_element(lens.begin(), lens.end());
  if (s->attn_trace && s->attn_ld < max_len)
    return fail(SOPRO_ERR_INVALID, "attention trace row stride %lld < longest text %d", (long long)s->attn_ld, max_len);
  CK(cudaSetDevice(e->device));
  s->max_len = max_len;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  s->B = batch;
  s->steps = steps;
  s->noise_k = noise_k;
  s->cond = cond_ar;
  s->noise = noise;
  s->t_pos = 0;
  s->host_st.assign(batch, UttState{0, -1, 0, 0, 0, {0, 0, 0}});
  {
    const size_t b_len = align_up((size_t)batch * 4, 64), b_samp = align_up((size_t)batch * sizeof(SamplingDev), 64),
                 b_st = (size_t)batch * sizeof(UttState);
    if (s->pin_bytes < b_len + b_samp + b_st) {
      if (s->pin_done) CK(cudaEventSynchronize(s->pin_done));
      if (s->pin) cudaFreeHost(s->pin);
      s->pin = nullptr;
      s->pin_bytes = 0;
      CK(cudaMallocHost(reinterpret_cast<void**>(&s->pin), b_len + b_samp + b_st));
      s->pin_bytes = b_len + b_samp + b_st;
    }
    if (!s->pin_done) CK(cudaEventCreateWithFlags(&s->pin_done, cudaEventDisableTiming));
    else CK(cudaEventSynchronize(s->pin_done));  // the previous begin()'s copies have read the staging buffer (normally long ago)
    memcpy(s->pin, lens.data(), (size_t)batch * 4);
    memcpy(s->pin + b_len, sd.data(), (size_t)batch * sizeof(SamplingDev));
    memcpy(s->pin + b_len + b_samp, s->host_st.data(), b_st);
    CK(cudaMemcpyAsync(s->text_len, s->pin, (size_t)batch * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(s->samp, s->pin + b_len, (size_t)batch * sizeof(SamplingDev), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(s->st, s->pin + b_len + b_samp, b_st, cudaMemcpyHostToDevice, st));
    CK(cudaEventRecord(s->pin_done, st));
  }
  CK(cudaMemsetAsync(s->ring, 0, (size_t)e->ring_floats_per_utt * batch * 4, st));
  CK(cudaMemsetAsync(s->tokens, 0, (size_t)batch * steps * 4, st));
  CK(cudaMemsetAsync(s->sampled, 0, (size_t)batch * steps * 4, st));
  {
    const size_t Bz = (size_t)batch, Dz = (size_t)e->D;
    CK(cudaMemsetAsync(s->xa, 0, Bz * Dz * 8, st));
    CK(cudaMemsetAsync(s->xb, 0, Bz * Dz * 8, st));
    CK(cudaMemsetAsync(s->hbuf, 0, Bz * e->F * 8, st));
    CK(cudaMemsetAsync(s->qbuf, 0, Bz * Dz * 8, st));
    CK(cudaMemsetAsync(s->abuf, 0, Bz * Dz * 8, st));
    CK(cudaMemsetAsync(s->logits, 0, Bz * e->Vpad * 8, st));
    CK(cudaMemsetAsync(s->tok_ll, 0, Bz * 8, st));
    s->seq_base = 0;
  }
  CK(cudaMemsetAsync(s->n_tokens, 0, (size_t)batch * 4, st));
  CK(cudaMemsetAsync(s->done, 0, (size_t)batch * 4, st));
  const size_t kv = (size_t)std::max(e->n_attn, 1) * batch * s->Lmax * e->D;
  CK(cudaMemsetAsync(s->kc, 0, kv * 4, st));
  CK(cudaMemsetAsync(s->vc, 0, kv * 4, st));
  int rc = e->cfg.weight_dtype == SOPRO_W_F32 ? launch_kv<float>(s, txt_seq, text_stride, lens, st)
                                               : launch_kv<__nv_bfloat16>(s, txt_seq, text_stride, lens, st);
  if (rc != SOPRO_OK) return rc;
  s->begun = true;
  return SOPRO_OK;
}

}  // extern "C"

// ---- weight-tile schedule of one AR step for every team rank (consumption order of the kernel)
struct StageW {
  int stage;          // index in the kernel's stage program
  const void* w;
  int N, K, parts;    // parts = 2 for the GLU (value rows + gate rows of the same channels)
  const float* epi;   // GLU: packed [D][KcE] epilogue rows; else the bias vector [N] (or null)
  bool by_head;       // fused q + attention stage: rank r gets ALL rows of head r % H (ranks >= H * (P / H): none)
};

// the fused q-projection + attention stage needs at least one CTA per head
static bool use_qatt(const sopro_engine* e, int P) {
  static const bool off = getenv("SOPRO_AR_QATT") && atoi(getenv("SOPRO_AR_QATT")) == 0;
  return !off && P >= e->H;
}

static int build_tiles(sopro_ar_session* s, int P, int wbuf, cudaStream_t st) {
  sopro_engine* e = s->e;
  const bool qatt = s->qatt;
  if (s->tile_P == P && s->tile_wbuf == wbuf && s->tile_qatt == (int)qatt) return SOPRO_OK;
  const size_t wsz = e->cfg.weight_dtype == SOPRO_W_F32 ? 4 : 2;
  std::vector<StageW> prog;
  int si = 0;  // must mirror the stage program built in launch_ar
  for (int i = 0; i < e->n_layers; ++i) {
    const LayerDev& L = e->layer[i];
    prog.push_back({si++, L.glu_w, e->D, e->D, 2, e->epi[i], false});
    prog.push_back({si++, L.w1, e->F, e->D, 1, L.b1, false});
    prog.push_back({si++, L.w2, e->D, e->F, 1, L.b2, false});
    if (L.has_attn) {
      if (qatt) {
        prog.push_back({si++, L.wq, e->D, e->D, 1, nullptr, true});
      } else {
        prog.push_back({si++, L.wq, e->D, e->D, 1, nullptr, false});
        si++;  // attention core: no weights
      }
      prog.push_back({si++, L.wo, e->D, e->D, 1, nullptr, false});
    }
  }
  prog.push_back({si++, e->head_w, e->V, e->D, 1, e->head_b, false});
  s->h_stage_tiles.assign((size_t)P * kMaxStages, 0);
  s->h_tiles.assign((size_t)P * kMaxTilesPerStep, TileDesc{});
  s->h_ntiles.assign(P, 0);
  for (int r = 0; r < P; ++r) {
    int n = 0;
    for (const StageW& sw : prog) {
      int n0 = (int)(((long long)sw.N * r) / P), n1 = (int)(((long long)sw.N * (r + 1)) / P);
      if (sw.by_head) {
        const int PH = P / e->H;
        n0 = r < e->H * PH ? (r % e->H) * e->Dh : 0;
        n1 = r < e->H * PH ? n0 + e->Dh : 0;
      }
      const size_t row_bytes = (size_t)sw.K * wsz;
      // per row: weights (x parts) + epilogue constants (GLU: KcE floats; else 1 bias float, +32 B span slack)
      const size_t epi_row = sw.parts == 2 ? (size_t)e->KcE * 4 : (sw.epi ? 4 : 0);
      const int rpt = (int)(((size_t)wbuf - 32) / (row_bytes * sw.parts + epi_row));
      if (rpt < 1) return fail(SOPRO_ERR_INVALID, "weight buffer %d B cannot hold one row (%zu B x %d)", wbuf, row_bytes, sw.parts);
      for (int a = n0; a < n1; a += rpt) {
        const int nr = std::min(rpt, n1 - a);
        if (n >= kMaxTilesPerStep) return fail(SOPRO_ERR_INVALID, "more than %d weight tiles per step (P=%d, wbuf=%d)", kMaxTilesPerStep, P, wbuf);
        TileDesc& t = s->h_tiles[(size_t)r * kMaxTilesPerStep + n++];
        const unsigned char* base = reinterpret_cast<const unsigned char*>(sw.w);
        t.src0 = reinterpret_cast<unsigned long long>(base + (size_t)a * row_bytes);
        t.bytes0 = (unsigned)((size_t)nr * row_bytes);
        t.src1 = sw.parts == 2 ? reinterpret_cast<unsigned long long>(base + (size_t)(a + sw.N) * row_bytes) : 0ull;
        t.bytes1 = sw.parts == 2 ? t.bytes0 : 0u;
        t.src2 = 0;
        t.bytes2 = 0;
        t.off2 = 0;
        if (sw.parts == 2) {
          t.src2 = reinterpret_cast<unsigned long long>(sw.epi + (size_t)a * e->KcE);
          t.bytes2 = (unsigned)((size_t)nr * e->KcE * 4);
        } else if (sw.epi) {
          const int lo = a / 4 * 4, hi = (a + nr + 3) / 4 * 4;  // 16-byte aligned span (vectors are padded)
          t.src2 = reinterpret_cast<unsigned long long>(sw.epi + lo);
          t.bytes2 = (unsigned)((hi - lo) * 4);
          t.off2 = a - lo;
        }
        t.row0 = a;
        t.nrows = nr;
        if (++s->h_stage_tiles[(size_t)r * kMaxStages + sw.stage] == 255)
          return fail(SOPRO_ERR_INVALID, "more than 254 weight tiles in one stage");
      }
    }
    s->h_ntiles[r] = n;
  }
  CK(cudaMemcpyAsync(s->tiles, s->h_tiles.data(), s->h_tiles.size() * sizeof(TileDesc), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s->n_tiles, s->h_ntiles.data(), (size_t)P * 4, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s->stage_tiles, s->h_stage_tiles.data(), s->h_stage_tiles.size(), cudaMemcpyHostToDevice, st));
  s->tile_P = P;
  s->tile_wbuf = wbuf;
  s->tile_qatt = (int)qatt;
  return SOPRO_OK;
}

// Task shape of every weight stage (ar_kernel.cuh, TaskShape).  Task i of a tile runs on warp i mod 16, and warp w issues
// from scheduler w mod 4, so scheduler 0 carries ceil(tasks / 4) tasks of R x TUE outputs x K MACs each.  A stage takes
// narrow when its busiest scheduler, summed over the stage's tiles and maximised over the team's ranks, carries less
// work even after weighting by its 1.2x shared-memory bytes per MAC (1.5 against 1.25 B): measured at batch 64 (DESIGN.md
// §3), a narrow HEAD (272 against 288 output-units per scheduler) is slower, FFN2 and O (48 against 64) are faster.
// A tie keeps the wide shape.  The fused q + attention stage keeps its own tiles.
static void pick_task_shapes(sopro_ar_session* s, ArParams& p, int P, int TU, int Bt) {
  const int R = TU == 8 ? 4 : 2, RC = R / 2;
  std::vector<int> first(P, 0);  // each rank's first tile of the stage
  for (int si = 0; si < p.n_stage; ++si) {
    StageOp& op = p.prog[si];
    op.shape = SHAPE_WIDE;
    const bool gemv = op.kind <= K_HEAD;
    const int K = op.kind == K_FFN2 ? s->e->F : s->e->D;
    long long load[2] = {0, 0};  // [wide, narrow]
    for (int r = 0; r < P; ++r) {
      const int nt = s->h_stage_tiles[(size_t)r * kMaxStages + si];
      long long l[2] = {0, 0};
      for (int j = 0; gemv && j < nt; ++j) {
        const int nr = s->h_tiles[(size_t)r * kMaxTilesPerStep + first[r] + j].nrows;
        const int n_rt = op.kind == K_GLU ? (nr + RC - 1) / RC : (nr + R - 1) / R;
        for (int w = 0; w < 2; ++w) {
          const int tue = w ? std::max(TU / 2, 1) : TU;
          const long long tasks = (long long)n_rt * ((Bt + tue - 1) / tue);
          l[w] += (tasks + 3) / 4 * R * tue * K;
        }
      }
      first[r] += nt;
      load[0] = std::max(load[0], l[0]);
      load[1] = std::max(load[1], l[1]);
    }
    if (!gemv || TU < 2 || op.kind == K_GLU) continue;  // GLU is always wide: its narrow tiles measured slower
    if (s->task_shape == 2 || (s->task_shape == 0 && 6 * load[1] < 5 * load[0])) op.shape = SHAPE_NARROW;
  }
  std::copy(p.prog, p.prog + p.n_stage, s->last_prog);
  s->last_n_stage = p.n_stage;
}

template <typename WT, int TU, bool LL>
static int launch_ar_tu(sopro_ar_session* s, ArParams& p, size_t smem, int grid, cudaStream_t st) {
  // the attention-trace export is its own instantiation, so the untraced kernel's code is not touched by it
  auto kern = p.attn_trace ? ar_persistent_kernel<WT, TU, LL, true> : ar_persistent_kernel<WT, TU, LL, false>;
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kThreads, smem));
  if (occ < 1) return fail(SOPRO_ERR_CUDA, "persistent kernel does not fit an SM (smem %zu)", smem);
  CK(cudaMemsetAsync(s->barrier, 0, (size_t)s->e->n_sms * 32 * 4, st));
  void* args[] = {(void*)&p};
  CK(cudaLaunchCooperativeKernel((const void*)kern, dim3(grid), dim3(kThreads), args, smem, st));
  s->seq_base += (unsigned)((p.t_end - p.t_begin) * p.n_stage);
  return SOPRO_OK;
}

template <typename WT>
static int launch_ar(sopro_ar_session* s, int t_begin, int t_end, cudaStream_t st) {
  sopro_engine* e = s->e;
  ArParams p{};
  p.D = e->D;
  p.F = e->F;
  p.V = e->V;
  p.Vpad = e->Vpad;
  p.H = e->H;
  p.Dh = e->Dh;
  p.Kc = e->Kc;
  p.KcP = e->KcP;
  p.KcE = e->KcE;
  p.n_layers = e->n_layers;
  p.eos_id = e->cfg.eos_id;
  long long roff = 0;
  for (int i = 0; i < e->n_layers; ++i) {
    p.layer[i] = e->layer[i];
    p.layer[i].ring_off = roff;
    roff += (long long)e->D * e->layer[i].dil * e->KcP * s->B;
  }
  p.final_norm_w = e->final_norm_w;
  p.head_w = e->head_w;
  p.head_b = e->head_b;
  p.emb = e->emb;
  p.B = s->B;
  p.steps = s->steps;
  p.Lmax = s->Lmax;
  p.noise_k = s->noise_k;
  p.cond = s->cond;
  p.noise = s->noise;
  p.kc = s->kc;
  p.vc = s->vc;
  p.text_len = s->text_len;
  p.ring = s->ring;
  p.xa = s->xa;
  p.xb = s->xb;
  p.hbuf = s->hbuf;
  p.qbuf = s->qbuf;
  p.abuf = s->abuf;
  p.logits = s->logits;
  p.tokens = s->tokens;
  p.sampled = s->sampled;
  p.n_tokens = s->n_tokens;
  p.done = s->done;
  p.forced = s->forced;
  p.st = s->st;
  p.samp = s->samp;
  p.trace_blocks = s->trace_blocks;
  p.trace_logits = s->trace_logits;
  p.barrier = s->barrier;
  p.tok_ll = s->tok_ll;
  p.seq_base = s->seq_base;
  p.timing = s->timing;
  p.timing_step = s->timing_step;
  p.attn_trace = s->attn_trace;
  p.attn_ld = s->attn_ld;
  p.attn_step = (long long)e->n_attn * s->B * e->H * s->attn_ld;
  p.attn_ring = s->attn_ring > 0 ? s->attn_ring : s->steps;
  // ---- team geometry: g teams x P CTAs, Bt utterances per team
  int Bt = s->utts_per_team;
  if (Bt <= 0) {
    if (const char* env = getenv("SOPRO_AR_UTTS_PER_TEAM")) Bt = atoi(env);
  }
  if (Bt <= 0) Bt = std::min(s->B, 8);  // measured at B=64: 8 utterances/team + LL = 362k cycles/step, 16 + barrier = 429k
  // activations ([Bt][F] fp32) may use at most ~120 KB of shared memory; the rest is the weight ring
  const int bt_cap = std::min(kMaxUttPerTeam, std::max(1, (int)((120 * 1024) / ((size_t)e->F * 4))));
  Bt = std::min(Bt, bt_cap);
  int g = (s->B + Bt - 1) / Bt;
  if (g > e->n_sms) {
    Bt = bt_cap;
    g = (s->B + Bt - 1) / Bt;
  }
  if (g > e->n_sms) return fail(SOPRO_ERR_INVALID, "batch %d needs %d teams > %d SMs", s->B, g, e->n_sms);
  Bt = (s->B + g - 1) / g;  // balance
  g = (s->B + Bt - 1) / Bt;
  int P = e->n_sms / g;
  if (const char* env = getenv("SOPRO_AR_MAX_P")) {  // experiment knob: fewer CTAs per team (larger slices, fewer exchange partners)
    const int cap = atoi(env);
    if (cap >= 1) P = std::min(P, cap);
  }
  p.g = g;
  p.P = P;
  p.Bt = Bt;
  p.t_begin = t_begin;
  p.t_end = t_end;
  const size_t kSmemCap = 213 * 1024;  // 227 KB minus static shared memory (sampler scratch, mbarriers) and alignment slack
  const size_t table_bytes = (size_t)kMaxTilesPerStep * sizeof(TileDesc);
  const size_t wsz = e->cfg.weight_dtype == SOPRO_W_F32 ? 4 : 2;
  // attention: per 256-thread group q[Dh] + scores[Lmax] + partial outputs; K / V are read straight from L2
  const size_t need_att_base = (size_t)2 * (e->Dh + att_group_floats(s->Lmax, e->Dh)) * 4;
  const size_t need_smp = (size_t)e->Vpad * 8 + e->Vpad + 16;
  size_t act_bytes = 0, wbuf = 0;
  int nbuf = 0, PH = 1;
  bool qatt = use_qatt(e, P);
  const size_t need_act = std::max((size_t)Bt * e->F * 4, (size_t)2 * Bt * e->D * 4 + (size_t)kWarps * kTapSlots * e->KcP * 4);
  auto slice_bytes = [&](int N, int K, int parts) {
    const size_t rows = (size_t)((N + P - 1) / P);
    return rows * K * wsz * parts + (parts == 2 ? rows * e->KcE * 4 : rows * 4) + 32;
  };
  size_t full = std::max(std::max(slice_bytes(e->D, e->D, 2), slice_bytes(e->F, e->D, 1)),
                         std::max(slice_bytes(e->D, e->F, 1), slice_bytes(e->V, e->D, 1)));
  full = align_up(full, 128);
  // The fused q + attention stage (one exchange and one GEMV stage fewer per attention layer) streams a whole head's
  // Wq rows through every serving CTA: taken when that head tile fits at most two ring buffers (batched launches); a
  // batch-1 launch, whose CTAs (one per SM) hold slivers of every matrix, keeps the q stage spread over all CTAs.
  for (;;) {
    size_t need_att = need_att_base;
    PH = qatt ? P / e->H : 1;
    if (qatt) need_att += (size_t)((Bt + PH - 1) / PH) * (e->D + e->Dh) * 4;  // + the fused stage's x rows and q rows
    act_bytes = align_up(std::max(need_act, std::max(need_att, need_smp)), 128);
    if (act_bytes + table_bytes + 2 * 4096 > kSmemCap) {
      if (qatt) {
        qatt = false;
        continue;
      }
      return fail(SOPRO_ERR_INVALID, "shared memory: activations need %zu B (Bt=%d, Lmax=%d), nothing left for weights",
                  act_bytes, Bt, s->Lmax);
    }
    const size_t avail = kSmemCap - act_bytes - table_bytes;
    if (2 * full <= avail) {
      wbuf = full;
      nbuf = (int)std::min<size_t>(kMaxWBuf, avail / wbuf);
    } else {
      wbuf = (avail / 2) / 128 * 128;
      nbuf = 2;
    }
    if (qatt && (size_t)e->Dh * e->D * wsz + 64 > 2 * wbuf) {
      qatt = false;
      continue;
    }
    break;
  }
  p.PH = PH;
  s->qatt = qatt;
  int rc = build_tiles(s, P, (int)wbuf, st);
  if (rc != SOPRO_OK) return rc;
  p.tiles = s->tiles;
  p.n_tiles = s->n_tiles;
  p.stage_tiles = s->stage_tiles;
  p.nbuf = nbuf;
  p.wbuf_bytes = (int)wbuf;
  p.act_bytes = (int)act_bytes;
  p.ring_off = (int)act_bytes;
  p.table_off = (int)(act_bytes + (size_t)nbuf * wbuf);
  const size_t smem = act_bytes + (size_t)nbuf * wbuf + table_bytes + 1024;  // + slack for the 1024-byte alignment
  // ---- stage program of one step
  {
    int n = 0;
    for (int i = 0; i < e->n_layers; ++i) {
      p.prog[n++] = {K_GLU, (unsigned char)i};
      p.prog[n++] = {K_FFN1, (unsigned char)i};
      p.prog[n++] = {K_FFN2, (unsigned char)i};
      if (e->layer[i].has_attn) {
        if (qatt) {
          p.prog[n++] = {K_QATT, (unsigned char)i};
        } else {
          p.prog[n++] = {K_Q, (unsigned char)i};
          p.prog[n++] = {K_ATT, (unsigned char)i};
        }
        p.prog[n++] = {K_O, (unsigned char)i};
      }
    }
    p.prog[n++] = {K_HEAD, 0};
    p.prog[n++] = {K_SAMPLE, 0};
    p.n_stage = n;
  }
  const int TU = Bt >= 8 ? 8 : Bt >= 4 ? 4 : Bt >= 2 ? 2 : 1;
  pick_task_shapes(s, p, P, TU, Bt);
  const int grid = g * P;
  // activation exchange: LL protocol (flag-in-data, no barrier) for small teams, where the step is latency
  // bound; team barrier for large teams, where LL's doubled activation traffic costs more than the barrier
  // (measured: B=64 429k vs 446k cycles/step).  SOPRO_AR_SYNC=ll|barrier overrides.
  const char* sync_env = getenv("SOPRO_AR_SYNC");
  bool ll = Bt <= 8;
  if (sync_env && strcmp(sync_env, "barrier") == 0) ll = false;
  if (sync_env && strcmp(sync_env, "ll") == 0) ll = true;
  if (ll) {
    if (TU == 8) return launch_ar_tu<WT, 8, true>(s, p, smem, grid, st);
    if (TU == 4) return launch_ar_tu<WT, 4, true>(s, p, smem, grid, st);
    if (TU == 2) return launch_ar_tu<WT, 2, true>(s, p, smem, grid, st);
    return launch_ar_tu<WT, 1, true>(s, p, smem, grid, st);
  }
  if (TU == 8) return launch_ar_tu<WT, 8, false>(s, p, smem, grid, st);
  if (TU == 4) return launch_ar_tu<WT, 4, false>(s, p, smem, grid, st);
  if (TU == 2) return launch_ar_tu<WT, 2, false>(s, p, smem, grid, st);
  return launch_ar_tu<WT, 1, false>(s, p, smem, grid, st);
}

extern "C" {

int sopro_ar_run(sopro_ar_session_t* s, int n_steps, void* stream) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null session");
  if (!s->begun) return fail(SOPRO_ERR_STATE, "sopro_ar_run before sopro_ar_begin");
  if (n_steps < 1) return fail(SOPRO_ERR_INVALID, "n_steps must be >= 1");
  sopro_engine* e = s->e;
  CK(cudaSetDevice(e->device));
  const int t0 = s->t_pos;
  const int t1 = std::min(s->steps, t0 + n_steps);
  if (t0 >= t1) return SOPRO_OK;
  if (s->attn_trace && s->attn_ld < s->max_len)  // a trace set after sopro_ar_begin
    return fail(SOPRO_ERR_INVALID, "attention trace row stride %lld < longest text %d", (long long)s->attn_ld, s->max_len);
  if (s->attn_trace && s->attn_ring > 0 && t1 - t0 > s->attn_ring)  // the launch would overwrite its own first steps
    return fail(SOPRO_ERR_INVALID, "a launch of %d steps into an attention trace ring of %d", t1 - t0, s->attn_ring);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int rc = e->cfg.weight_dtype == SOPRO_W_F32 ? launch_ar<float>(s, t0, t1, st)
                                               : launch_ar<__nv_bfloat16>(s, t0, t1, st);
  if (rc != SOPRO_OK) return rc;
  s->t_pos = t1;
  return SOPRO_OK;
}

int sopro_ar_outputs(sopro_ar_session_t* s, const int32_t** tokens, const int32_t** n_tokens,
                     const int32_t** done) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null session");
  if (tokens) *tokens = s->tokens;
  if (n_tokens) *n_tokens = s->n_tokens;
  if (done) *done = s->done;
  return SOPRO_OK;
}

int sopro_ar_read(sopro_ar_session_t* s, int32_t* tokens_host, int32_t* n_tokens_host, int32_t* done_host,
                  void* stream) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null session");
  if (!s->begun) return fail(SOPRO_ERR_STATE, "sopro_ar_read before sopro_ar_begin");
  CK(cudaSetDevice(s->e->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (tokens_host)
    CK(cudaMemcpyAsync(tokens_host, s->tokens, (size_t)s->B * s->steps * 4, cudaMemcpyDeviceToHost, st));
  s->host_st.resize(s->B);
  CK(cudaMemcpyAsync(s->host_st.data(), s->st, (size_t)s->B * sizeof(UttState), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (int b = 0; b < s->B; ++b) {
    if (n_tokens_host) n_tokens_host[b] = s->host_st[b].len;
    if (done_host) done_host[b] = s->host_st[b].done;
  }
  return SOPRO_OK;
}

int sopro_ar_position(sopro_ar_session_t* s) { return s ? s->t_pos : -1; }

static int ensure(float** p, size_t* cap, size_t bytes) {
  if (*cap >= bytes) return SOPRO_OK;
  if (*p) cudaFree(*p);
  *p = nullptr;
  *cap = 0;
  cudaError_t e = cudaMalloc((void**)p, bytes);
  if (e != cudaSuccess) return fail(SOPRO_ERR_CUDA, "staging alloc %zu failed: %s", bytes, cudaGetErrorString(e));
  *cap = bytes;
  return SOPRO_OK;
}

int sopro_ar_generate_host(sopro_ar_session_t* s, int batch, int steps, const float* cond_ar, const float* txt_seq,
                           int text_stride, const int32_t* text_len, const float* noise, int noise_k,
                           const sopro_ar_sampling_t* sampling, int32_t* tokens_out, int32_t* n_tokens_out,
                           void* stream) {
  if (!s || !cond_ar || !txt_seq || !text_len || !noise || !sampling || !tokens_out)
    return fail(SOPRO_ERR_INVALID, "null argument");
  if (batch < 1 || batch > s->max_batch || steps < 1 || steps > s->max_steps || text_stride < 1 || noise_k < 1)
    return fail(SOPRO_ERR_INVALID, "bad batch/steps/text_stride/noise_k");
  sopro_engine* e = s->e;
  CK(cudaSetDevice(e->device));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t nc = (size_t)batch * steps * e->D * 4, nt = (size_t)batch * text_stride * e->D * 4,
               nn = (size_t)batch * steps * noise_k * 4;
  int rc;
  if ((rc = ensure(&s->h_cond, &s->h_cond_cap, nc)) != SOPRO_OK) return rc;
  if ((rc = ensure(&s->h_txt, &s->h_txt_cap, nt)) != SOPRO_OK) return rc;
  if ((rc = ensure(&s->h_noise, &s->h_noise_cap, nn)) != SOPRO_OK) return rc;
  CK(cudaMemcpyAsync(s->h_cond, cond_ar, nc, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s->h_txt, txt_seq, nt, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(s->h_noise, noise, nn, cudaMemcpyHostToDevice, st));
  rc = sopro_ar_begin(s, batch, steps, s->h_cond, s->h_txt, text_stride, text_len, s->h_noise, noise_k, sampling,
                      stream);
  if (rc != SOPRO_OK) return rc;
  rc = sopro_ar_run(s, steps, stream);
  if (rc != SOPRO_OK) return rc;
  return sopro_ar_read(s, tokens_out, n_tokens_out, nullptr, stream);
}

int sopro_ar_set_forced_tokens(sopro_ar_session_t* s, const int32_t* forced) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null session");
  s->forced = forced;
  return SOPRO_OK;
}

int sopro_ar_set_trace(sopro_ar_session_t* s, float* trace_blocks, float* trace_logits) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null session");
  s->trace_blocks = trace_blocks;
  s->trace_logits = trace_logits;
  return SOPRO_OK;
}

int sopro_ar_set_attn_trace(sopro_ar_session_t* s, float* probs, int64_t ld) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null session");
  if (probs && ld < 1) return fail(SOPRO_ERR_INVALID, "attention trace row stride must be >= 1 (got %lld)", (long long)ld);
  s->attn_trace = probs;
  s->attn_ld = probs ? ld : 0;
  s->attn_ring = 0;
  return SOPRO_OK;
}

int sopro_ar_set_attn_trace_ring(sopro_ar_session_t* s, float* probs, int64_t ld, int32_t ring) {
  if (probs && ring < 1) return fail(SOPRO_ERR_INVALID, "attention trace ring must be >= 1 step (got %d)", ring);
  const int rc = sopro_ar_set_attn_trace(s, probs, ld);
  if (rc != SOPRO_OK) return rc;
  s->attn_ring = probs ? ring : 0;
  return SOPRO_OK;
}

int sopro_ar_set_timing(sopro_ar_session_t* s, int64_t* buf, int step) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null session");
  s->timing = reinterpret_cast<long long*>(buf);
  s->timing_step = step;
  return SOPRO_OK;
}

int sopro_ar_debug_sampled(sopro_ar_session_t* s, int32_t* dst, void* stream) {
  if (!s || !dst) return fail(SOPRO_ERR_INVALID, "null argument");
  CK(cudaMemcpyAsync(dst, s->sampled, (size_t)s->B * s->steps * 4, cudaMemcpyDeviceToDevice,
                     reinterpret_cast<cudaStream_t>(stream)));
  return SOPRO_OK;
}

}  // extern "C"

namespace {
__global__ void __launch_bounds__(kThreads, 1) sampler_debug_kernel(const __grid_constant__ ArParams p, int t) {
  extern __shared__ __align__(16) unsigned char dbg_smem[];
  __shared__ SamplerSmem ssm;
  float* sx = reinterpret_cast<float*>(dbg_smem);
  float* sp = sx + p.Vpad;
  unsigned char* flags = reinterpret_cast<unsigned char*>(sx + 2 * p.Vpad);
  sample_utterance(p, 0, t, sx, sp, flags, ssm, 0, 0u, 0u);
}
}  // namespace

extern "C" {

int sopro_debug_sample(const float* logits, int vocab, const int32_t* hist, int n_hist, const float* noise, int noise_k,
                       const sopro_ar_sampling_t* q, int recovery, int device, int32_t* token_out) {
  if (!logits || !noise || !q || !token_out || (n_hist > 0 && !hist)) return fail(SOPRO_ERR_INVALID, "null argument");
  if (vocab < 2 || vocab > kMaxVocab || n_hist < 0 || q->top_k < 1 || q->top_k > kMaxTopK)
    return fail(SOPRO_ERR_INVALID, "sampler hook: vocab in [2,%d], top_k in [1,%d]", kMaxVocab, kMaxTopK);
  const int need = (q->top_p < 1.0f && q->recovery_top_p < 1.0f) ? std::min(q->top_k, vocab) : vocab;
  if (noise_k < need) return fail(SOPRO_ERR_INVALID, "sampler hook: noise_k=%d, need %d", noise_k, need);
  CK(cudaSetDevice(device));
  const int Vpad = (int)align_up((size_t)vocab, 4), steps = n_hist + 1;
  float *d_logits = nullptr, *d_noise = nullptr;
  int *d_tok = nullptr, *d_sampled = nullptr, *d_n = nullptr, *d_done = nullptr;
  UttState* d_st = nullptr;
  SamplingDev* d_samp = nullptr;
  unsigned* d_ll = nullptr;
  auto cleanup = [&]() {
    cudaFree(d_logits); cudaFree(d_noise); cudaFree(d_tok); cudaFree(d_sampled); cudaFree(d_n); cudaFree(d_done);
    cudaFree(d_st); cudaFree(d_samp); cudaFree(d_ll);
  };
  cudaError_t err = cudaMalloc(&d_logits, (size_t)Vpad * 4);
  if (err == cudaSuccess) err = cudaMalloc(&d_noise, (size_t)steps * noise_k * 4);
  if (err == cudaSuccess) err = cudaMalloc(&d_tok, (size_t)steps * 4);
  if (err == cudaSuccess) err = cudaMalloc(&d_sampled, (size_t)steps * 4);
  if (err == cudaSuccess) err = cudaMalloc(&d_n, 4);
  if (err == cudaSuccess) err = cudaMalloc(&d_done, 4);
  if (err == cudaSuccess) err = cudaMalloc(&d_st, sizeof(UttState));
  if (err == cudaSuccess) err = cudaMalloc(&d_samp, sizeof(SamplingDev));
  if (err == cudaSuccess) err = cudaMalloc(&d_ll, 8);
  if (err == cudaSuccess) err = cudaMemset(d_logits, 0, (size_t)Vpad * 4);
  if (err == cudaSuccess) err = cudaMemcpy(d_logits, logits, (size_t)vocab * 4, cudaMemcpyHostToDevice);
  if (err == cudaSuccess) err = cudaMemset(d_noise, 0, (size_t)steps * noise_k * 4);
  if (err == cudaSuccess) err = cudaMemcpy(d_noise + (size_t)n_hist * noise_k, noise, (size_t)noise_k * 4, cudaMemcpyHostToDevice);
  if (err == cudaSuccess) err = cudaMemset(d_tok, 0, (size_t)steps * 4);
  if (err == cudaSuccess && n_hist) err = cudaMemcpy(d_tok, hist, (size_t)n_hist * 4, cudaMemcpyHostToDevice);
  UttState st{n_hist, n_hist ? hist[n_hist - 1] : -1, 0, recovery ? 1 : 0, 0, {0, 0, 0}};
  SamplingDev sd{q->top_p, q->temperature, q->recovery_top_p, q->recovery_temp, q->repetition_penalty, q->top_k, 0, q->loop_streak,
                 q->min_gen_frames, q->stop_on_first_eos};
  if (err == cudaSuccess) err = cudaMemcpy(d_st, &st, sizeof(st), cudaMemcpyHostToDevice);
  if (err == cudaSuccess) err = cudaMemcpy(d_samp, &sd, sizeof(sd), cudaMemcpyHostToDevice);
  if (err != cudaSuccess) {
    cleanup();
    return fail(SOPRO_ERR_CUDA, "sampler hook: %s", cudaGetErrorString(err));
  }
  ArParams p{};
  p.V = vocab;
  p.Vpad = Vpad;
  p.eos_id = vocab - 1;
  p.B = 1;
  p.steps = steps;
  p.noise_k = noise_k;
  p.noise = d_noise;
  p.logits = d_logits;
  p.tokens = d_tok;
  p.sampled = d_sampled;
  p.n_tokens = d_n;
  p.done = d_done;
  p.st = d_st;
  p.samp = d_samp;
  p.tok_ll = d_ll;
  const size_t smem = (size_t)Vpad * 8 + Vpad + 16;
  sampler_debug_kernel<<<1, kThreads, smem>>>(p, n_hist);
  err = cudaGetLastError();
  if (err == cudaSuccess) err = cudaDeviceSynchronize();
  if (err == cudaSuccess) err = cudaMemcpy(token_out, d_sampled + n_hist, 4, cudaMemcpyDeviceToHost);
  cleanup();
  if (err != cudaSuccess) return fail(SOPRO_ERR_CUDA, "sampler hook: %s", cudaGetErrorString(err));
  return SOPRO_OK;
}

int sopro_ar_debug_kv(sopro_ar_session_t* s, float* k_dst, float* v_dst, void* stream) {
  if (!s) return fail(SOPRO_ERR_INVALID, "null argument");
  const size_t n = (size_t)s->e->n_attn * s->B * s->Lmax * s->e->D * 4;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (k_dst) CK(cudaMemcpyAsync(k_dst, s->kc, n, cudaMemcpyDeviceToDevice, st));
  if (v_dst) CK(cudaMemcpyAsync(v_dst, s->vc, n, cudaMemcpyDeviceToDevice, st));
  return SOPRO_OK;
}

}  // extern "C"
