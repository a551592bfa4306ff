// Engine behind the C ABI (include/vcla.h): device arenas, weight registry / repacking, and the orchestration of
// the three phases of the path -- vision encode, prefill, decode step (CUDA-graph captured).
#include "../../include/vcla.h"
#include "kernels.h"

#include <dlfcn.h>
#include <math.h>
#include <nccl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <thread>
#include <map>
#include <string>
#include <tuple>
#include <vector>

using namespace vcla;

namespace {

enum SlotKind { SLOT_MAT = 0, SLOT_VEC = 1, SLOT_Q8 = 2 };   // SLOT_Q8: int8 rows + fp32 row scales (weight_format 1)
enum SlotLayout { LAY_PLAIN = 0, LAY_INTERLEAVE32 = 1 };

struct Slot {
  std::string name;
  int64_t shape[4] = {0, 0, 0, 0};
  int ndim = 0;
  int kind = SLOT_MAT;
  int layout = LAY_PLAIN;
  int which = 0;           // interleave: 0 gate, 1 up
  int64_t rows = 0, cols = 0;  // 2D view of the logical tensor
  void* dst = nullptr;     // storage (bf16 for MAT, f32 for VEC) at the slot's first row
  int ld = 0;              // storage row pitch (elements) for MAT
  void* dst2 = nullptr;    // optional second copy (resampler k/v also live in the all-layer KV weight)
  float* scale = nullptr;  // SLOT_Q8: row scales, indexed like the stored rows
  double std = 0.0; float mean = 0.f;
};

struct VisionLayer {
  float *ln1_w, *ln1_b, *ln2_w, *ln2_b, *bqkv, *bo, *b1, *b2;
  bf16 *wqkv, *wo, *w1, *w2;
};
struct ResamplerLayer {
  bf16 *wqkv, *wo, *wi, *wo2;
  float *bqkv, *bo, *ln1_w, *ln1_b, *bi, *bo2, *ln2_w, *ln2_b;
};
struct TextLayer {
  float *ln1, *ln2;
  bf16 *wqkv, *wo, *wgu, *wd;                 // weight_format 0
  int8_t *qqkv, *qo, *qgu, *qd;               // weight_format 1: int8 rows (k in the decode kernel's fragment order, quant.cu) ...
  float *sqkv, *so, *sgu, *sd;                //                  ... and their fp32 scales
};

struct GraphKey {
  int B; const void* tok_in; const void* logits; const void* tok_out; int n_steps = 1; int dp = 0; int samp = 0; int beam = 0;
  int stream = 0;   // captured armed: every step publishes into the token stream ring
  int lookup = 0;   // prompt lookup: rows per verification step (0: plain decode steps)
  auto fields() const { return std::tie(B, tok_in, logits, tok_out, n_steps, dp, samp, beam, stream, lookup); }
  bool operator<(const GraphKey& o) const { return fields() < o.fields(); }
};
struct DecodeGraph {
  cudaGraphExec_t exec; int64_t launches; uint64_t last_use;   // launches: kernels one replay enqueues (vcla_kernel_launches)
};

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

uint32_t fnv1a32(const char* s) {
  uint32_t h = 0x811C9DC5u;
  for (; *s; ++s) { h ^= (uint8_t)*s; h *= 0x01000193u; }
  return h;
}

}  // namespace

struct vcla_ctx {
  vcla_config cfg;
  int v_tokens = 0, kpatch = 0, kpad = 0, hd_t = 0;
  // arenas
  uint8_t* w_arena = nullptr; size_t w_bytes = 0, w_off = 0;
  uint8_t* a_arena = nullptr; size_t a_bytes = 0, a_off = 0;
  size_t kv_bytes = 0;
  KvFormat kv_format() const { return (KvFormat)cfg.kv_format; }
  std::vector<Slot> slots;
  std::map<std::string, int> slot_index;
  // vision weights
  bf16* patch_w = nullptr; float *cls = nullptr, *pos = nullptr, *pre_w = nullptr, *pre_b = nullptr, *post_w = nullptr, *post_b = nullptr;
  std::vector<VisionLayer> vl;
  // resampler
  float* rq = nullptr; bf16* r_wkv_all = nullptr; float* r_bkv_all = nullptr;
  std::vector<ResamplerLayer> rl;
  bf16* proj_w = nullptr; float* proj_b = nullptr;
  // text
  bf16 *embed = nullptr, *lm_head = nullptr; float* final_norm = nullptr;
  std::vector<TextLayer> tl;
  // kv cache: pages owned by the pool view (kv.pages is the arena of every layer) and handed to sequences round-robin as they grow by
  // the device-side allocator (elementwise.cu: kv_reset / kv_reserve / advance_seq), so a sequence's pages are NOT contiguous; all
  // stream-ordered and graph-capturable.  kv_order: the order in which a reset stacks the free pages.
  KvCache kv;
  int32_t *seq_len = nullptr, *img_row_default = nullptr, *kv_order = nullptr;
  // RoPE tables and argmax scratch are per context (another context may use another theta / device / stream)
  float *rope_cos = nullptr, *rope_sin = nullptr, *cand_val = nullptr; int32_t* cand_idx = nullptr;
  int attn_persistent_mode = 1, attn_persistent_grid = 0;
  // data parallel (vcla_nccl_init): per-step all-gather of the chosen tokens, captured inside the decode graph on a forked branch
  ncclComm_t comm = nullptr; int dp_rank = 0, dp_world = 1, dp_width = 0; bool dp_active = false;
  bool dp_on() const { return comm != nullptr && dp_active; }
  int32_t *dp_send = nullptr, *dp_recv = nullptr, *dp_hist = nullptr, *dp_step = nullptr;
  cudaStream_t dp_stream = nullptr; cudaEvent_t dp_fork = nullptr, dp_join = nullptr; bool dp_pending = false;
  // device-side sampling (vcla_set_sampler): replaces the argmax by the fused logits-processor chain + draw
  SamplerParams* samp_params = nullptr; float* samp_logits = nullptr; int32_t* finished = nullptr; bool samp_on = false;
  // beam search (vcla_set_beam): the beam kernels replace the argmax, and the K/V of the chosen beams are rearranged through the
  // page table after every step (beam_K rows per batch item, sharing their parents' pages copy-on-write)
  BeamParams* beam_params = nullptr; bool beam_on = false; int beam_K = 0, beam_max_new = 0;
  float *beam_cand_val = nullptr, *beam_run = nullptr, *hyp_score = nullptr;
  int32_t *beam_cand_tok = nullptr, *beam_parent = nullptr, *hyp_len = nullptr, *hyp_fin = nullptr, *hyp_tok = nullptr, *hyp_tmp = nullptr;
  int32_t *beam_state = nullptr, *beam_copy = nullptr, *beam_table_tmp = nullptr;
  unsigned long long* beam_cow_bytes = nullptr;
  // fan-out (vcla_set_fanout): vcla_prefill forks each prompt to `fanout` rows through the beam reorder (parent r / fanout); forked:
  // the resident rows came from such a fork (cleared by vcla_reset)
  int fanout = 1; bool forked = false;
  // token streaming (vcla_stream_*): ring in pinned, mapped host memory; stream_done is recorded after every armed enqueue
  StreamRing *ring_host = nullptr, *ring_dev = nullptr; bool stream_armed = false;
  cudaEvent_t stream_done = nullptr; bool stream_pending = false;
  StreamRing* ring() const { return stream_armed ? ring_dev : nullptr; }
  // prompt lookup decoding (vcla_set_lookup): verification steps of lk_rows rows replace the decode steps of the one resident sequence
  bool lk_on = false, lk_primed = false; int lk_rows = 0, lk_max_new = 0;
  int64_t* lk_prompt = nullptr; int32_t *lk_tok = nullptr, *lk_pick = nullptr; LookupState* lk_state = nullptr;
  int64_t len_bound = 0;   // host-side upper bound of the cached tokens per sequence (prefill S + decode steps issued since)
  int resident_b = 0;      // sequences resident since the last vcla_prefill (0 after vcla_reset)
  // vision activations
  bf16 *v_im2col = nullptr, *v_norm = nullptr, *v_qkv = nullptr, *v_attn = nullptr, *v_ffn = nullptr;
  float *v_hidden = nullptr, *v_postln_f32 = nullptr;
  float *r_hidden = nullptr, *img_embeds = nullptr;
  bf16 *r_hidden_bf16 = nullptr, *r_qkv = nullptr, *r_kvimg = nullptr, *r_ctx = nullptr, *r_ffn = nullptr;
  // prefill activations
  float* resid = nullptr; bf16 *xn = nullptr, *qkv = nullptr, *attn = nullptr, *hmid = nullptr;
  float* p_ssq = nullptr;    // [max_prefill_tokens][t_hidden / 64] row statistics of the deferred-RMSNorm prefill schedule
  bf16* q8_wide = nullptr;   // weight_format 1: bf16(q) of the projection the prefill GEMM runs next (largest: gate/up)
  // decode activations
  float* d_resid = nullptr; bf16 *d_xn = nullptr, *d_attn = nullptr, *d_h = nullptr;
  float *ws_qkv = nullptr, *ws_o = nullptr, *ws_gu = nullptr, *ws_d = nullptr, *ws_lm = nullptr;
  float* attn_scratch = nullptr; int32_t* attn_counters = nullptr;
  float* pa_part = nullptr; int32_t* pa_counters = nullptr;   // split-KV partials / arrival counters of the paged prefill attention
  int32_t* d_tok = nullptr;
  int32_t *tok_hist = nullptr, *step_idx = nullptr;
  float* d_ssq = nullptr;    // [64][t_hidden / 128] row statistics of the deferred-RMSNorm decode schedule (cluster split-K)
  int csk_qkv = 0, csk_o = 0, csk_gu = 0, csk_d = 0, csk_lm = 0;   // CTAs per cluster (= K splits), chosen per batch on first use
  int csk_batch = 0;
  int sp_qkv = 1, sp_o = 1, sp_gu = 1, sp_d = 1, sp_lm = 1, kv_splits = 1;
  int l2_prefetch_kb = 0;    // decode GEMMs: weight k-blocks per CTA prefetched into L2 during the dependency wait (VCLA_L2_PREFETCH_KB).
                             // Off by default: the prefetch traffic can delay the latency-critical consumer kernel in front of the GEMM.
  // graphs
  std::map<GraphKey, DecodeGraph> graphs;   // bounded (kMaxGraphs) so a caller with ever-new buffers cannot grow it
  uint64_t graph_uses = 0;                  // clock of DecodeGraph::last_use
  int64_t launches = 0;
  void* staging = nullptr; size_t staging_bytes = 0;
  void* trace_buf = nullptr; unsigned long long trace_cap = 0;
  cudaStream_t cap_stream = nullptr;   // graph capture is illegal on the legacy default stream torch uses
};

namespace {

template <typename T>
T* w_alloc(vcla_ctx* c, size_t n) {
  size_t bytes = align_up(n * sizeof(T), 256);
  if (c->w_arena == nullptr) { c->w_off += bytes; return nullptr; }   // sizing pass
  T* p = reinterpret_cast<T*>(c->w_arena + c->w_off);
  c->w_off += bytes;
  return p;
}
template <typename T>
T* a_alloc(vcla_ctx* c, size_t n) {
  size_t bytes = align_up(n * sizeof(T), 1024);
  if (c->a_arena == nullptr) { c->a_off += bytes; return nullptr; }
  T* p = reinterpret_cast<T*>(c->a_arena + c->a_off);
  c->a_off += bytes;
  return p;
}

void add_slot(vcla_ctx* c, const std::string& name, std::initializer_list<int64_t> shape, int kind, void* dst, int ld, double std_,
              float mean_, int layout = LAY_PLAIN, int which = 0, void* dst2 = nullptr) {
  if (c->w_arena == nullptr) return;  // sizing pass: no registry
  Slot s;
  s.name = name; s.kind = kind; s.layout = layout; s.which = which; s.dst = dst; s.ld = ld; s.dst2 = dst2; s.std = std_; s.mean = mean_;
  s.ndim = (int)shape.size();
  int i = 0; int64_t numel = 1;
  for (int64_t d : shape) { s.shape[i++] = d; numel *= d; }
  s.rows = shape.size() ? *shape.begin() : 1;
  s.cols = s.rows ? numel / s.rows : 0;
  if (kind == SLOT_VEC) { s.rows = 1; s.cols = numel; }
  c->slot_index[name] = (int)c->slots.size();
  c->slots.push_back(s);
}

// Lays out every weight in the arena.  Called twice: once with w_arena == nullptr to size, once to assign.
// std / mean per tensor follow oracle/visualcla_oracle.py:weight_specs exactly.
void layout_weights(vcla_ctx* c) {
  const vcla_config& g = c->cfg;
  c->w_off = 0;
  const int D = g.v_hidden, Fv = g.v_ffn;
  const std::string vp = "vision_model.vision_model.";
  c->cls = w_alloc<float>(c, D);
  add_slot(c, vp + "embeddings.class_embedding", {D}, SLOT_VEC, c->cls, 0, 1.0, 0.f);
  c->patch_w = w_alloc<bf16>(c, (size_t)D * c->kpad);
  add_slot(c, vp + "embeddings.patch_embedding.weight", {D, 3, g.v_patch, g.v_patch}, SLOT_MAT, c->patch_w, c->kpad, 1.0 / sqrt((double)c->kpatch), 0.f);
  c->pos = w_alloc<float>(c, (size_t)c->v_tokens * D);
  add_slot(c, vp + "embeddings.position_embedding.weight", {c->v_tokens, D}, SLOT_VEC, c->pos, 0, 0.5, 0.f);
  c->pre_w = w_alloc<float>(c, D); add_slot(c, vp + "pre_layrnorm.weight", {D}, SLOT_VEC, c->pre_w, 0, 0.1, 1.f);
  c->pre_b = w_alloc<float>(c, D); add_slot(c, vp + "pre_layrnorm.bias", {D}, SLOT_VEC, c->pre_b, 0, 0.1, 0.f);
  c->vl.resize(g.v_layers);
  for (int i = 0; i < g.v_layers; ++i) {
    VisionLayer& L = c->vl[i];
    const std::string lp = vp + "encoder.layers." + std::to_string(i) + ".";
    L.ln1_w = w_alloc<float>(c, D); add_slot(c, lp + "layer_norm1.weight", {D}, SLOT_VEC, L.ln1_w, 0, 0.1, 1.f);
    L.ln1_b = w_alloc<float>(c, D); add_slot(c, lp + "layer_norm1.bias", {D}, SLOT_VEC, L.ln1_b, 0, 0.1, 0.f);
    L.ln2_w = w_alloc<float>(c, D); add_slot(c, lp + "layer_norm2.weight", {D}, SLOT_VEC, L.ln2_w, 0, 0.1, 1.f);
    L.ln2_b = w_alloc<float>(c, D); add_slot(c, lp + "layer_norm2.bias", {D}, SLOT_VEC, L.ln2_b, 0, 0.1, 0.f);
    L.wqkv = w_alloc<bf16>(c, (size_t)3 * D * D);
    L.bqkv = w_alloc<float>(c, 3 * D);
    const char* pr[3] = {"q_proj", "k_proj", "v_proj"};
    for (int j = 0; j < 3; ++j) {
      add_slot(c, lp + "self_attn." + pr[j] + ".weight", {D, D}, SLOT_MAT, L.wqkv ? L.wqkv + (size_t)j * D * D : nullptr, D, 1.5 / sqrt((double)D), 0.f);
      add_slot(c, lp + "self_attn." + pr[j] + ".bias", {D}, SLOT_VEC, L.bqkv ? L.bqkv + j * D : nullptr, 0, 0.1, 0.f);
    }
    L.wo = w_alloc<bf16>(c, (size_t)D * D); add_slot(c, lp + "self_attn.out_proj.weight", {D, D}, SLOT_MAT, L.wo, D, 0.5 / sqrt((double)D), 0.f);
    L.bo = w_alloc<float>(c, D); add_slot(c, lp + "self_attn.out_proj.bias", {D}, SLOT_VEC, L.bo, 0, 0.05, 0.f);
    L.w1 = w_alloc<bf16>(c, (size_t)Fv * D); add_slot(c, lp + "mlp.fc1.weight", {Fv, D}, SLOT_MAT, L.w1, D, 1.0 / sqrt((double)D), 0.f);
    L.b1 = w_alloc<float>(c, Fv); add_slot(c, lp + "mlp.fc1.bias", {Fv}, SLOT_VEC, L.b1, 0, 0.1, 0.f);
    L.w2 = w_alloc<bf16>(c, (size_t)D * Fv); add_slot(c, lp + "mlp.fc2.weight", {D, Fv}, SLOT_MAT, L.w2, Fv, 0.5 / sqrt((double)Fv), 0.f);
    L.b2 = w_alloc<float>(c, D); add_slot(c, lp + "mlp.fc2.bias", {D}, SLOT_VEC, L.b2, 0, 0.05, 0.f);
  }
  c->post_w = w_alloc<float>(c, D); add_slot(c, vp + "post_layernorm.weight", {D}, SLOT_VEC, c->post_w, 0, 0.1, 1.f);
  c->post_b = w_alloc<float>(c, D); add_slot(c, vp + "post_layernorm.bias", {D}, SLOT_VEC, c->post_b, 0, 0.1, 0.f);

  const int R = g.r_hidden, Fr = g.r_ffn, Q = g.r_queries, RL = g.r_layers;
  const std::string rp = "visual_resampler.";
  c->rq = w_alloc<float>(c, (size_t)Q * R); add_slot(c, rp + "query_embeddding", {1, Q, R}, SLOT_VEC, c->rq, 0, 1.0, 0.f);
  c->r_wkv_all = w_alloc<bf16>(c, (size_t)RL * 2 * R * R);
  c->r_bkv_all = w_alloc<float>(c, (size_t)RL * 2 * R);
  c->rl.resize(RL);
  for (int i = 0; i < RL; ++i) {
    ResamplerLayer& L = c->rl[i];
    const std::string lp = rp + "encoder.layer." + std::to_string(i) + ".";
    L.wqkv = w_alloc<bf16>(c, (size_t)3 * R * R);
    L.bqkv = w_alloc<float>(c, 3 * R);
    const char* pr[3] = {"query", "key", "value"};
    for (int j = 0; j < 3; ++j) {
      // key/value additionally live in the all-layer [RL*2R, R] matrix used for the layer-invariant image rows
      void* d2w = (j > 0 && c->r_wkv_all) ? (void*)(c->r_wkv_all + ((size_t)i * 2 + (j - 1)) * R * R) : nullptr;
      void* d2b = (j > 0 && c->r_bkv_all) ? (void*)(c->r_bkv_all + ((size_t)i * 2 + (j - 1)) * R) : nullptr;
      add_slot(c, lp + "crossattention.self." + pr[j] + ".weight", {R, R}, SLOT_MAT, L.wqkv ? L.wqkv + (size_t)j * R * R : nullptr, R, 1.5 / sqrt((double)R), 0.f, LAY_PLAIN, 0, d2w);
      add_slot(c, lp + "crossattention.self." + pr[j] + ".bias", {R}, SLOT_VEC, L.bqkv ? L.bqkv + j * R : nullptr, 0, 0.1, 0.f, LAY_PLAIN, 0, d2b);
    }
    L.wo = w_alloc<bf16>(c, (size_t)R * R); add_slot(c, lp + "crossattention.output.dense.weight", {R, R}, SLOT_MAT, L.wo, R, 1.0 / sqrt((double)R), 0.f);
    L.bo = w_alloc<float>(c, R); add_slot(c, lp + "crossattention.output.dense.bias", {R}, SLOT_VEC, L.bo, 0, 0.05, 0.f);
    L.ln1_w = w_alloc<float>(c, R); add_slot(c, lp + "crossattention.output.LayerNorm.weight", {R}, SLOT_VEC, L.ln1_w, 0, 0.1, 1.f);
    L.ln1_b = w_alloc<float>(c, R); add_slot(c, lp + "crossattention.output.LayerNorm.bias", {R}, SLOT_VEC, L.ln1_b, 0, 0.1, 0.f);
    L.wi = w_alloc<bf16>(c, (size_t)Fr * R); add_slot(c, lp + "intermediate.dense.weight", {Fr, R}, SLOT_MAT, L.wi, R, 1.0 / sqrt((double)R), 0.f);
    L.bi = w_alloc<float>(c, Fr); add_slot(c, lp + "intermediate.dense.bias", {Fr}, SLOT_VEC, L.bi, 0, 0.1, 0.f);
    L.wo2 = w_alloc<bf16>(c, (size_t)R * Fr); add_slot(c, lp + "output.dense.weight", {R, Fr}, SLOT_MAT, L.wo2, Fr, 1.0 / sqrt((double)Fr), 0.f);
    L.bo2 = w_alloc<float>(c, R); add_slot(c, lp + "output.dense.bias", {R}, SLOT_VEC, L.bo2, 0, 0.05, 0.f);
    L.ln2_w = w_alloc<float>(c, R); add_slot(c, lp + "output.LayerNorm.weight", {R}, SLOT_VEC, L.ln2_w, 0, 0.1, 1.f);
    L.ln2_b = w_alloc<float>(c, R); add_slot(c, lp + "output.LayerNorm.bias", {R}, SLOT_VEC, L.ln2_b, 0, 0.1, 0.f);
  }
  const int T = g.t_hidden, Ft = g.t_ffn, V = g.t_vocab, TL = g.t_layers;
  c->proj_w = w_alloc<bf16>(c, (size_t)T * R); add_slot(c, "image_projection_layer.weight", {T, R}, SLOT_MAT, c->proj_w, R, 1.0 / sqrt((double)R), 0.f);
  c->proj_b = w_alloc<float>(c, T); add_slot(c, "image_projection_layer.bias", {T}, SLOT_VEC, c->proj_b, 0, 0.1, 0.f);

  const std::string tp = "text_model.model.";
  const double res_gain = 1.0 / sqrt(2.0 * (double)TL);
  c->embed = w_alloc<bf16>(c, (size_t)V * T); add_slot(c, tp + "embed_tokens.weight", {V, T}, SLOT_MAT, c->embed, T, 1.0, 0.f);
  c->tl.resize(TL);
  for (int i = 0; i < TL; ++i) {
    TextLayer& L = c->tl[i];
    const std::string lp = tp + "layers." + std::to_string(i) + ".";
    L.ln1 = w_alloc<float>(c, T); add_slot(c, lp + "input_layernorm.weight", {T}, SLOT_VEC, L.ln1, 0, 0.1, 1.f);
    L.ln2 = w_alloc<float>(c, T); add_slot(c, lp + "post_attention_layernorm.weight", {T}, SLOT_VEC, L.ln2, 0, 0.1, 1.f);
    if (g.weight_format == 1) {
      // load_in_8bit: the seven projections as int8 rows + row scales (q/k/v and gate/up are quantised per slot)
      L.wqkv = L.wo = L.wgu = L.wd = nullptr;
      auto q8 = [&](const std::string& name, int64_t rows, int64_t cols, int8_t* q, float* sc, double std_, int layout, int which) {
        add_slot(c, name, {rows, cols}, SLOT_Q8, q, (int)cols, std_, 0.f, layout, which);
        if (c->w_arena != nullptr) c->slots.back().scale = sc;
      };
      L.qqkv = w_alloc<int8_t>(c, (size_t)3 * T * T); L.sqkv = w_alloc<float>(c, (size_t)3 * T);
      const char* pr[3] = {"q_proj", "k_proj", "v_proj"};
      const double sd[3] = {1.5, 1.5, 1.0};
      for (int j = 0; j < 3; ++j)
        q8(lp + "self_attn." + pr[j] + ".weight", T, T, L.qqkv ? L.qqkv + (size_t)j * T * T : nullptr, L.sqkv ? L.sqkv + (size_t)j * T : nullptr,
           sd[j] / sqrt((double)T), LAY_PLAIN, 0);
      L.qo = w_alloc<int8_t>(c, (size_t)T * T); L.so = w_alloc<float>(c, T);
      q8(lp + "self_attn.o_proj.weight", T, T, L.qo, L.so, res_gain * 2.0 / sqrt((double)T), LAY_PLAIN, 0);
      L.qgu = w_alloc<int8_t>(c, (size_t)2 * Ft * T); L.sgu = w_alloc<float>(c, (size_t)2 * Ft);
      q8(lp + "mlp.gate_proj.weight", Ft, T, L.qgu, L.sgu, 1.0 / sqrt((double)T), LAY_INTERLEAVE32, 0);
      q8(lp + "mlp.up_proj.weight", Ft, T, L.qgu, L.sgu, 1.0 / sqrt((double)T), LAY_INTERLEAVE32, 1);
      L.qd = w_alloc<int8_t>(c, (size_t)T * Ft); L.sd = w_alloc<float>(c, T);
      q8(lp + "mlp.down_proj.weight", T, Ft, L.qd, L.sd, res_gain * 4.0 / sqrt((double)Ft), LAY_PLAIN, 0);
      continue;
    }
    L.qqkv = L.qo = L.qgu = L.qd = nullptr; L.sqkv = L.so = L.sgu = L.sd = nullptr;
    L.wqkv = w_alloc<bf16>(c, (size_t)3 * T * T);
    add_slot(c, lp + "self_attn.q_proj.weight", {T, T}, SLOT_MAT, L.wqkv, T, 1.5 / sqrt((double)T), 0.f);
    add_slot(c, lp + "self_attn.k_proj.weight", {T, T}, SLOT_MAT, L.wqkv ? L.wqkv + (size_t)T * T : nullptr, T, 1.5 / sqrt((double)T), 0.f);
    add_slot(c, lp + "self_attn.v_proj.weight", {T, T}, SLOT_MAT, L.wqkv ? L.wqkv + (size_t)2 * T * T : nullptr, T, 1.0 / sqrt((double)T), 0.f);
    L.wo = w_alloc<bf16>(c, (size_t)T * T); add_slot(c, lp + "self_attn.o_proj.weight", {T, T}, SLOT_MAT, L.wo, T, res_gain * 2.0 / sqrt((double)T), 0.f);
    L.wgu = w_alloc<bf16>(c, (size_t)2 * Ft * T);
    add_slot(c, lp + "mlp.gate_proj.weight", {Ft, T}, SLOT_MAT, L.wgu, T, 1.0 / sqrt((double)T), 0.f, LAY_INTERLEAVE32, 0);
    add_slot(c, lp + "mlp.up_proj.weight", {Ft, T}, SLOT_MAT, L.wgu, T, 1.0 / sqrt((double)T), 0.f, LAY_INTERLEAVE32, 1);
    L.wd = w_alloc<bf16>(c, (size_t)T * Ft); add_slot(c, lp + "mlp.down_proj.weight", {T, Ft}, SLOT_MAT, L.wd, Ft, res_gain * 4.0 / sqrt((double)Ft), 0.f);
  }
  c->final_norm = w_alloc<float>(c, T); add_slot(c, tp + "norm.weight", {T}, SLOT_VEC, c->final_norm, 0, 0.1, 1.f);
  c->lm_head = w_alloc<bf16>(c, (size_t)V * T); add_slot(c, "text_model.lm_head.weight", {V, T}, SLOT_MAT, c->lm_head, T, 4.0 / sqrt((double)T), 0.f);
}

void layout_activations(vcla_ctx* c) {
  const vcla_config& g = c->cfg;
  c->a_off = 0;
  const size_t Bv = g.max_batch, VT = (size_t)Bv * c->v_tokens, D = g.v_hidden, gg = (size_t)(c->v_tokens - 1);
  c->v_im2col = a_alloc<bf16>(c, Bv * gg * c->kpad);
  c->v_hidden = a_alloc<float>(c, VT * D);
  c->v_norm = a_alloc<bf16>(c, VT * D);
  c->v_qkv = a_alloc<bf16>(c, VT * 3 * D);
  c->v_attn = a_alloc<bf16>(c, VT * D);
  c->v_ffn = a_alloc<bf16>(c, VT * g.v_ffn);
  c->v_postln_f32 = a_alloc<float>(c, VT * D);
  const size_t RQ = (size_t)Bv * g.r_queries, R = g.r_hidden;
  c->r_hidden = a_alloc<float>(c, RQ * R);
  c->r_hidden_bf16 = a_alloc<bf16>(c, RQ * R);
  c->r_qkv = a_alloc<bf16>(c, RQ * 3 * R);
  c->r_kvimg = a_alloc<bf16>(c, VT * (size_t)g.r_layers * 2 * R);
  c->r_ctx = a_alloc<bf16>(c, RQ * R);
  c->r_ffn = a_alloc<bf16>(c, RQ * g.r_ffn);
  c->img_embeds = a_alloc<float>(c, RQ * g.t_hidden);
  const size_t Tk = g.max_prefill_tokens, T = g.t_hidden, F = g.t_ffn;
  c->resid = a_alloc<float>(c, Tk * T);
  c->xn = a_alloc<bf16>(c, Tk * T);
  c->qkv = a_alloc<bf16>(c, Tk * 3 * T);
  c->attn = a_alloc<bf16>(c, Tk * T);
  c->hmid = a_alloc<bf16>(c, Tk * F);
  c->p_ssq = a_alloc<float>(c, Tk * ((T + 63) / 64));
  if (g.weight_format == 1) c->q8_wide = a_alloc<bf16>(c, std::max((size_t)3 * T * T, (size_t)2 * F * T));
  const size_t Bp = 64;  // decode operand rows (batch is processed in chunks of <= 64)
  c->d_resid = a_alloc<float>(c, Bp * T);
  c->d_xn = a_alloc<bf16>(c, Bp * T);
  c->d_attn = a_alloc<bf16>(c, Bp * T);
  c->d_h = a_alloc<bf16>(c, Bp * F);
  c->ws_qkv = a_alloc<float>(c, (size_t)c->sp_qkv * Bp * 3 * T);
  c->ws_o = a_alloc<float>(c, (size_t)c->sp_o * Bp * T);
  c->ws_gu = a_alloc<float>(c, (size_t)c->sp_gu * Bp * 2 * F);
  c->ws_d = a_alloc<float>(c, (size_t)c->sp_d * Bp * T);
  c->ws_lm = a_alloc<float>(c, (size_t)c->sp_lm * Bp * g.t_vocab);
  c->attn_scratch = a_alloc<float>(c, (size_t)Bp * g.t_heads * 8 * (128 + 2));   // up to 8 KV splits
  c->attn_counters = a_alloc<int32_t>(c, (size_t)Bp * g.t_heads);
  c->pa_part = a_alloc<float>(c, (size_t)attention_paged_partials() * kAttnPartialFloats);
  c->pa_counters = a_alloc<int32_t>(c, (size_t)attention_paged_partials());
  c->d_tok = a_alloc<int32_t>(c, Bp);
  c->tok_hist = a_alloc<int32_t>(c, (size_t)(g.max_seq + 2) * Bp);
  c->step_idx = a_alloc<int32_t>(c, 16);
  c->d_ssq = a_alloc<float>(c, Bp * ((T + 127) / 128));
  c->kv.table = a_alloc<int32_t>(c, (size_t)g.max_batch * c->kv.pages_per_seq);
  c->seq_len = a_alloc<int32_t>(c, g.max_batch);
  c->img_row_default = a_alloc<int32_t>(c, g.max_batch);
  c->kv.free_stack = a_alloc<int32_t>(c, (size_t)c->kv.total_pages);
  c->kv_order = a_alloc<int32_t>(c, (size_t)c->kv.total_pages);
  c->kv.state = a_alloc<int32_t>(c, 4);
  c->kv.npages = a_alloc<int32_t>(c, g.max_batch);
  c->rope_cos = a_alloc<float>(c, (size_t)(g.max_seq + 1) * 64);
  c->rope_sin = a_alloc<float>(c, (size_t)(g.max_seq + 1) * 64);
  c->cand_val = a_alloc<float>(c, Bp * kArgmaxChunks);
  c->cand_idx = a_alloc<int32_t>(c, Bp * kArgmaxChunks);
  c->samp_params = a_alloc<SamplerParams>(c, 1);
  c->samp_logits = a_alloc<float>(c, Bp * (size_t)g.t_vocab);
  c->finished = a_alloc<int32_t>(c, Bp);
  c->beam_params = a_alloc<BeamParams>(c, 1);
  c->beam_cand_val = a_alloc<float>(c, Bp * kBeamMaxCand);
  c->beam_cand_tok = a_alloc<int32_t>(c, Bp * kBeamMaxCand);
  c->beam_run = a_alloc<float>(c, Bp);
  c->beam_parent = a_alloc<int32_t>(c, Bp);
  c->hyp_score = a_alloc<float>(c, Bp);
  c->hyp_len = a_alloc<int32_t>(c, Bp);
  c->hyp_fin = a_alloc<int32_t>(c, Bp);
  c->hyp_tok = a_alloc<int32_t>(c, Bp * (size_t)g.max_seq);
  c->hyp_tmp = a_alloc<int32_t>(c, Bp * (size_t)g.max_seq);
  c->beam_state = a_alloc<int32_t>(c, Bp * 2);
  c->beam_copy = a_alloc<int32_t>(c, 1 + 3 * Bp);
  c->beam_table_tmp = a_alloc<int32_t>(c, (size_t)g.max_batch * c->kv.pages_per_seq);
  c->beam_cow_bytes = a_alloc<unsigned long long>(c, 1);
  c->lk_prompt = a_alloc<int64_t>(c, (size_t)g.max_seq);
  c->lk_tok = a_alloc<int32_t>(c, 16);
  c->lk_pick = a_alloc<int32_t>(c, 16);
  c->lk_state = a_alloc<LookupState>(c, 1);
}

// Split-K factor of a decode GEMM (row tiles of 128 x `splits` work units on 2 persistent CTAs per SM).  A thin last wave is
// latency-bound (one lone CTA streams a small fraction of HBM bandwidth), and a single wave of one-tile CTAs loses the
// epilogue/load overlap -> prefer >= ~2 waves with a last wave that is >= 60 % full.
int pick_splits(int n_out, int K) {
  const int tiles = (n_out + 127) / 128;
  const int kb = (K + 63) / 64;
  const double slots = 2.0 * num_sms();
  int best = 1;
  double best_score = 1e9;
  for (int want = 1; want <= 40; ++want) {
    if (kb / want < 4 && want > 1) break;               // at least 4 k-blocks per work unit
    const int per = (kb + want - 1) / want;
    const int s = (kb + per - 1) / per;                 // realisable: every split non-empty
    if (s != want) continue;
    const double w = tiles * (double)s / slots;
    const double f = w - floor(w);
    double score;
    if (w < 1.0) score = (1.0 - w) + 0.15;
    else if (f < 1e-9) score = 0.0;
    else if (f >= 0.6) score = (1.0 - f) * 0.3;
    else score = (0.6 - f) + 0.2;
    score += 0.01 * s;                                  // fewer partials for the consumers when otherwise equal
    if (score < best_score) { best_score = score; best = s; }
  }
  return best;
}

int count(vcla_ctx* c, int n = 1) { c->launches += n; return 0; }

// Destroys every captured decode graph, so the next decode call captures one with the current settings.
int drop_graphs(vcla_ctx* c) {
  if (c->graphs.empty()) return 0;
  const cudaError_t e = cudaDeviceSynchronize();   // a launch of one of them may still be in flight
  for (auto& kv : c->graphs) cudaGraphExecDestroy(kv.second.exec);
  c->graphs.clear();
  if (e != cudaSuccess) { set_error("drop_graphs: device error %s", cudaGetErrorString(e)); return -1; }
  return 0;
}

// Points the in-kernel timeline of every kernel family at buf (nullptr: tracing off).
int trace_set_all(void* buf, unsigned long long cap) {
  int rc = 0;
  rc |= trace_set_gemm(buf, cap);
  rc |= trace_set_attention_tc(buf, cap);
  rc |= trace_set_gemm_decode(buf, cap);
  rc |= trace_set_sampler(buf, cap);
  rc |= trace_set_beam(buf, cap);
  rc |= trace_set_attention(buf, cap);
  rc |= trace_set_elementwise(buf, cap);
  return rc;
}

}  // namespace

// ---- NCCL, bound at run time ------------------------------------------------------------------------------------
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi g_nccl;
// NCCL is bound at run time (dlopen by soname: inside a torch process this resolves to the libnccl torch already loaded), so
// libvcla.so itself has no link-time dependency on it and single-GPU users never touch it.
static int nccl_api() {
  if (g_nccl.lib) return 0;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) { set_error("NCCL not found (dlopen libnccl.so.2: %s)", dlerror()); return -1; }
  g_nccl.GetUniqueId = (decltype(g_nccl.GetUniqueId))dlsym(h, "ncclGetUniqueId");
  g_nccl.CommInitRank = (decltype(g_nccl.CommInitRank))dlsym(h, "ncclCommInitRank");
  g_nccl.AllGather = (decltype(g_nccl.AllGather))dlsym(h, "ncclAllGather");
  g_nccl.CommDestroy = (decltype(g_nccl.CommDestroy))dlsym(h, "ncclCommDestroy");
  g_nccl.GetErrorString = (decltype(g_nccl.GetErrorString))dlsym(h, "ncclGetErrorString");
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllGather || !g_nccl.CommDestroy || !g_nccl.GetErrorString) {
    set_error("NCCL library lacks an expected symbol"); return -1;
  }
  g_nccl.lib = h;
  return 0;
}
#define VCLA_NCCL_OK(expr)                                                                                   \
  do {                                                                                                       \
    ncclResult_t _r = (expr);                                                                                \
    if (_r != ncclSuccess) { set_error("%s failed: %s", #expr, g_nccl.GetErrorString(_r)); return -1; }      \
  } while (0)


// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

const char* vcla_last_error(void) { return get_error(); }
const char* vcla_version(void) { return "vcla-h100 0.1 (sm_90a, wgmma/TMA)"; }
void vcla_set_pdl(int on) { set_pdl(on != 0); }

int vcla_create(const vcla_config* cfg, vcla_ctx** out) {
  if (!cfg || !out) { set_error("vcla_create: null argument"); return -1; }
  // Switches of removed schedules: refuse them, or a stale A/B script would measure the default and report it as the alternative.
  for (const char* v : {"VCLA_DECODE_SCHEDULE", "VCLA_FUSED_DECODE"}) {
    if (getenv(v)) {
      set_error("vcla_create: %s is set, but the decode schedules it selected were removed (the batch size picks the schedule)", v);
      return -1;
    }
  }
  if (const char* e = getenv("VCLA_PREFILL_FUSED")) {
    if (atoi(e) == 0) { set_error("vcla_create: VCLA_PREFILL_FUSED=0 is set, but the 8-kernel prefill schedule was removed"); return -1; }
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_error("vcla_create: no CUDA device (this library has no CPU fallback)");
    return -1;
  }
  vcla_ctx* c = new vcla_ctx();
  c->cfg = *cfg;
  vcla_config& g = c->cfg;
  if (g.page_tokens <= 0) g.page_tokens = 64;
  auto bad = [&](const char* why) { set_error("vcla_create: %s", why); delete c; return -1; };
  if (g.t_hidden % g.t_heads || g.t_hidden / g.t_heads != 128) return bad("LLaMA head_dim must be 128");
  if (g.v_hidden % g.v_heads || g.v_hidden / g.v_heads != 64) return bad("ViT head_dim must be 64");
  if (g.r_hidden % g.r_heads || g.r_hidden / g.r_heads != 64) return bad("Resampler head_dim must be 64");
  if (g.t_ffn % 32) return bad("LLaMA ffn must be a multiple of 32");
  if (g.v_hidden % 8 || g.r_hidden % 8 || g.t_hidden % 8 || g.v_ffn % 8 || g.r_ffn % 8 || g.t_ffn % 8) return bad("hidden sizes must be multiples of 8");
  if (g.v_image % g.v_patch) return bad("image size must be a multiple of the patch size");
  if (g.max_batch < 1 || g.max_seq < 1 || g.max_prefill_tokens < 1) return bad("capacities must be positive");
  if (g.max_seq > 1 << 20) return bad("max_seq too large");
  if (g.page_tokens > 64 || g.page_tokens % 8) return bad("page_tokens must be a multiple of 8 and <= 64");
  if (g.weight_format != 0 && g.weight_format != 1) return bad("weight_format must be 0 (bf16) or 1 (int8 LLaMA projections)");
  if (g.weight_format == 1 && (g.t_hidden % 64 || g.t_ffn % 64)) return bad("int8 projections need LLaMA hidden and ffn sizes that are multiples of 64");
  if (g.kv_format != KV_BF16 && g.kv_format != KV_INT8) return bad("kv_format must be 0 (bf16) or 1 (int8 rows + fp32 row scales)");
  c->v_tokens = (g.v_image / g.v_patch) * (g.v_image / g.v_patch) + 1;
  c->kpatch = 3 * g.v_patch * g.v_patch;
  c->kpad = (c->kpatch + 63) / 64 * 64;
  c->hd_t = 128;
  c->kv.heads = g.t_heads; c->kv.page_tokens = g.page_tokens; c->kv.layers = g.t_layers;
  c->kv.pages_per_seq = (g.max_seq + g.page_tokens - 1) / g.page_tokens;
  c->kv.total_pages = c->kv.pages_per_seq * g.max_batch;
  c->kv.layer_elems = g.kv_format == KV_INT8 ? c->kv.row(c->kv.total_pages, 0, 0) * (kKvQ8RowBytes / 2) : c->kv.row(c->kv.total_pages, 0, 0) * 128;
  c->sp_qkv = pick_splits(3 * g.t_hidden, g.t_hidden);
  c->sp_o = pick_splits(g.t_hidden, g.t_hidden);
  c->sp_gu = pick_splits(2 * g.t_ffn, g.t_hidden);
  c->sp_d = pick_splits(g.t_hidden, g.t_ffn);
  c->sp_lm = pick_splits(g.t_vocab, g.t_hidden);
  if (const char* e = getenv("VCLA_L2_PREFETCH_KB")) c->l2_prefetch_kb = atoi(e);
  c->kv_splits = g.max_seq >= 1536 ? 4 : (g.max_seq >= 768 ? 2 : 1);   // context-driven minimum; raised per call for small batches
  if (const char* e = getenv("VCLA_KV_SPLITS")) { const int v = atoi(e); if (v >= 1 && v <= 8) c->kv_splits = v; }   // tuning override

  if (gemm_init()) { delete c; return -1; }
  // sizing passes
  layout_weights(c); c->w_bytes = c->w_off;
  layout_activations(c); c->a_bytes = c->a_off;
  c->kv_bytes = c->kv.layer_elems * g.t_layers * sizeof(bf16);
  cudaError_t e;
  if ((e = cudaMalloc(&c->w_arena, c->w_bytes)) != cudaSuccess || (e = cudaMalloc(&c->a_arena, c->a_bytes)) != cudaSuccess ||
      (e = cudaMalloc(&c->kv.pages, c->kv_bytes)) != cudaSuccess) {
    (void)cudaGetLastError();   // a failed allocation must not surface as the error of the next context's first launch
    set_error("vcla_create: cudaMalloc failed (%s): weights %.2f GB, activations %.2f GB, kv %.2f GB", cudaGetErrorString(e),
              c->w_bytes / 1e9, c->a_bytes / 1e9, c->kv_bytes / 1e9);
    vcla_destroy(c);
    return -1;
  }
  cudaMemset(c->w_arena, 0, c->w_bytes);
  cudaMemset(c->a_arena, 0, c->a_bytes);
  layout_weights(c);
  layout_activations(c);
  // page allocation order: physical pages 0,1,2,... are handed out in this order after every reset (vcla_kv_debug_shuffle permutes it)
  std::vector<int32_t> order((size_t)c->kv.total_pages);
  for (size_t i = 0; i < order.size(); ++i) order[i] = (int32_t)i;
  cudaMemcpy(c->kv_order, order.data(), order.size() * 4, cudaMemcpyHostToDevice);
  std::vector<int32_t> two(g.max_batch, 2);
  cudaMemcpy(c->img_row_default, two.data(), two.size() * 4, cudaMemcpyHostToDevice);
  if (const char* e = getenv("VCLA_ATTN_PERSISTENT")) c->attn_persistent_mode = atoi(e);
  if (const char* e = getenv("VCLA_ATTN_PERSISTENT_GRID")) c->attn_persistent_grid = atoi(e);
  if (rope_fill_tables(g.max_seq + 1, 128, g.rope_theta, c->rope_cos, c->rope_sin) || attention_init() || sampler_init() || beam_init() || vcla_reset(c, nullptr)) { vcla_destroy(c); return -1; }
  if (cudaDeviceSynchronize() != cudaSuccess) { set_error("vcla_create: device error %s", cudaGetErrorString(cudaGetLastError())); vcla_destroy(c); return -1; }
  *out = c;
  return 0;
}

void vcla_destroy(vcla_ctx* c) {
  if (!c) return;
  drop_graphs(c);
  if (c->w_arena) cudaFree(c->w_arena);
  if (c->a_arena) cudaFree(c->a_arena);
  if (c->kv.pages) cudaFree(c->kv.pages);
  if (c->staging) cudaFree(c->staging);
  if (c->comm) { cudaDeviceSynchronize(); g_nccl.CommDestroy(c->comm); c->comm = nullptr; }
  if (c->dp_send) cudaFree(c->dp_send);
  if (c->dp_stream) cudaStreamDestroy(c->dp_stream);
  if (c->dp_fork) cudaEventDestroy(c->dp_fork);
  if (c->dp_join) cudaEventDestroy(c->dp_join);
  if (c->cap_stream) cudaStreamDestroy(c->cap_stream);
  if (c->trace_buf) { trace_set_all(nullptr, 0); cudaFree(c->trace_buf); }
  if (c->ring_host) { if (c->stream_pending) cudaEventSynchronize(c->stream_done); cudaFreeHost(c->ring_host); }
  if (c->stream_done) cudaEventDestroy(c->stream_done);
  delete c;
}

int vcla_get_config(const vcla_ctx* c, vcla_config* out) { if (!c || !out) return -1; *out = c->cfg; return 0; }
int vcla_memory_bytes(const vcla_ctx* c, int64_t* w, int64_t* kv, int64_t* a) {
  if (!c) return -1;
  if (w) *w = (int64_t)c->w_bytes;
  if (kv) *kv = (int64_t)c->kv_bytes;
  if (a) *a = (int64_t)c->a_bytes;
  return 0;
}
int64_t vcla_kernel_launches(vcla_ctx* c, int reset) { int64_t v = c->launches; if (reset) c->launches = 0; return v; }

int vcla_weight_count(const vcla_ctx* c) { return c ? (int)c->slots.size() : 0; }
int vcla_weight_info(const vcla_ctx* c, int index, const char** name, int64_t shape[4], int* ndim, int* kind) {
  if (!c || index < 0 || index >= (int)c->slots.size()) { set_error("vcla_weight_info: bad index"); return -1; }
  const Slot& s = c->slots[index];
  if (name) *name = s.name.c_str();
  if (shape) for (int i = 0; i < 4; ++i) shape[i] = s.shape[i];
  if (ndim) *ndim = s.ndim;
  if (kind) *kind = s.kind;
  return 0;
}

static int ensure_staging(vcla_ctx* c, size_t bytes) {
  if (c->staging_bytes >= bytes) return 0;
  if (c->staging) cudaFree(c->staging);
  c->staging = nullptr; c->staging_bytes = 0;
  VCLA_CUDA_OK(cudaMalloc(&c->staging, bytes));
  c->staging_bytes = bytes;
  return 0;
}

// place a contiguous bf16 [rows, cols] device matrix into a slot's storage
static int place_matrix(const Slot& s, const bf16* src, cudaStream_t st) {
  if (s.layout == LAY_INTERLEAVE32) return interleave_rows32(src, (int)s.rows, (int)s.cols, s.which, (bf16*)s.dst, st);
  if (copy_rows_bf16(src, (int)s.rows, (int)s.cols, (bf16*)s.dst, s.ld, st)) return -1;
  if (s.dst2) return copy_rows_bf16(src, (int)s.rows, (int)s.cols, (bf16*)s.dst2, (int)s.cols, st);
  return 0;
}

static int q8_which(const Slot& s) { return s.layout == LAY_INTERLEAVE32 ? s.which : -1; }

int vcla_load_weight(vcla_ctx* c, const char* name, const void* src, int dtype, int64_t numel, int on_device, vcla_stream stream) {
  cudaStream_t st = (cudaStream_t)stream;
  auto it = c->slot_index.find(name);
  if (it == c->slot_index.end()) { set_error("vcla_load_weight: unknown tensor '%s'", name); return -1; }
  const Slot& s = c->slots[it->second];
  const size_t n = (size_t)s.rows * s.cols;
  if (src == nullptr || numel != (int64_t)n) {
    set_error("vcla_load_weight: '%s' holds %lld elements, the caller passed %lld (checkpoint / config shape mismatch)", name, (long long)n, (long long)numel);
    return -1;
  }
  const size_t esz = dtype == VCLA_F32 ? 4 : 2;
  if (dtype < 0 || dtype > 2) { set_error("vcla_load_weight: bad dtype"); return -1; }
  // staging: [raw source copy][bf16 contiguous]
  const size_t raw_bytes = align_up(n * esz, 256);
  if (ensure_staging(c, raw_bytes + n * 2 + 256)) return -1;
  const void* dsrc = src;
  if (!on_device) {
    VCLA_CUDA_OK(cudaMemcpyAsync(c->staging, src, n * esz, cudaMemcpyHostToDevice, st));
    dsrc = c->staging;
  }
  if (s.kind == SLOT_VEC) {
    if (convert_to_f32(dsrc, dtype, (int64_t)n, (float*)s.dst, st)) return -1;
    if (s.dst2 && convert_to_f32(dsrc, dtype, (int64_t)n, (float*)s.dst2, st)) return -1;
  } else if (s.kind == SLOT_Q8) {
    // quantised from the source values themselves (fp32 / fp16 / bf16), not from a bf16 copy
    if (quantize_rows_q8(dsrc, dtype, (int)s.rows, (int)s.cols, q8_which(s), (int8_t*)s.dst, s.scale, st)) return -1;
  } else {
    bf16* tmp = reinterpret_cast<bf16*>((uint8_t*)c->staging + raw_bytes);
    if (convert_to_bf16(dsrc, dtype, (int64_t)n, tmp, st)) return -1;
    if (place_matrix(s, tmp, st)) return -1;
  }
  VCLA_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

int vcla_read_weight(vcla_ctx* c, const char* name, void* dst_host, vcla_stream stream) {
  cudaStream_t st = (cudaStream_t)stream;
  auto it = c->slot_index.find(name);
  if (it == c->slot_index.end()) { set_error("vcla_read_weight: unknown tensor '%s'", name); return -1; }
  const Slot& s = c->slots[it->second];
  if (s.kind == SLOT_VEC) {
    VCLA_CUDA_OK(cudaMemcpyAsync(dst_host, s.dst, (size_t)s.cols * 4, cudaMemcpyDeviceToHost, st));
  } else if (s.kind == SLOT_Q8) {
    const size_t n = (size_t)s.rows * s.cols;
    if (ensure_staging(c, n * 4)) return -1;
    if (read_rows_q8((const int8_t*)s.dst, s.scale, (int)s.rows, (int)s.cols, q8_which(s), nullptr, nullptr, (float*)c->staging, st)) return -1;
    VCLA_CUDA_OK(cudaMemcpyAsync(dst_host, c->staging, n * 4, cudaMemcpyDeviceToHost, st));
  } else if (s.layout == LAY_INTERLEAVE32) {
    for (int64_t j0 = 0; j0 < s.rows; j0 += 32) {
      const int64_t nr = (s.rows - j0) < 32 ? (s.rows - j0) : 32;
      const bf16* srcp = (const bf16*)s.dst + ((j0 / 32) * 64 + (int64_t)s.which * 32) * s.cols;
      VCLA_CUDA_OK(cudaMemcpyAsync((bf16*)dst_host + j0 * s.cols, srcp, (size_t)nr * s.cols * 2, cudaMemcpyDeviceToHost, st));
    }
  } else {
    VCLA_CUDA_OK(cudaMemcpy2DAsync(dst_host, (size_t)s.cols * 2, s.dst, (size_t)s.ld * 2, (size_t)s.cols * 2, (size_t)s.rows, cudaMemcpyDeviceToHost, st));
  }
  VCLA_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

static const Slot* q8_slot(vcla_ctx* c, const char* name, const char* what) {
  auto it = c->slot_index.find(name);
  if (it == c->slot_index.end()) { set_error("%s: unknown tensor '%s'", what, name); return nullptr; }
  const Slot& s = c->slots[it->second];
  if (s.kind != SLOT_Q8) { set_error("%s: '%s' is not stored as int8 (weight_format 1 stores the LLaMA projections so)", what, name); return nullptr; }
  return &s;
}

int vcla_read_weight_q8(vcla_ctx* c, const char* name, int8_t* q_host, float* scale_host, vcla_stream stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const Slot* s = q8_slot(c, name, "vcla_read_weight_q8");
  if (s == nullptr) return -1;
  const size_t n = (size_t)s->rows * s->cols, qbytes = align_up(n, 256);
  if (ensure_staging(c, qbytes + (size_t)s->rows * 4)) return -1;
  int8_t* q = (int8_t*)c->staging;
  float* sc = (float*)((uint8_t*)c->staging + qbytes);
  if (read_rows_q8((const int8_t*)s->dst, s->scale, (int)s->rows, (int)s->cols, q8_which(*s), q, sc, nullptr, st)) return -1;
  if (q_host) VCLA_CUDA_OK(cudaMemcpyAsync(q_host, q, n, cudaMemcpyDeviceToHost, st));
  if (scale_host) VCLA_CUDA_OK(cudaMemcpyAsync(scale_host, sc, (size_t)s->rows * 4, cudaMemcpyDeviceToHost, st));
  VCLA_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

int vcla_load_weight_q8(vcla_ctx* c, const char* name, const int8_t* q, const float* scale, int on_device, vcla_stream stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const Slot* s = q8_slot(c, name, "vcla_load_weight_q8");
  if (s == nullptr) return -1;
  if (q == nullptr || scale == nullptr) { set_error("vcla_load_weight_q8: null source"); return -1; }
  const size_t n = (size_t)s->rows * s->cols, qbytes = align_up(n, 256);
  const int8_t* dq = q; const float* ds = scale;
  if (!on_device) {
    if (ensure_staging(c, qbytes + (size_t)s->rows * 4)) return -1;
    VCLA_CUDA_OK(cudaMemcpyAsync(c->staging, q, n, cudaMemcpyHostToDevice, st));
    VCLA_CUDA_OK(cudaMemcpyAsync((uint8_t*)c->staging + qbytes, scale, (size_t)s->rows * 4, cudaMemcpyHostToDevice, st));
    dq = (const int8_t*)c->staging; ds = (const float*)((uint8_t*)c->staging + qbytes);
  }
  if (place_rows_q8(dq, ds, (int)s->rows, (int)s->cols, q8_which(*s), (int8_t*)s->dst, s->scale, st)) return -1;
  VCLA_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

int vcla_init_synthetic(vcla_ctx* c, uint32_t seed, vcla_stream stream) {
  cudaStream_t st = (cudaStream_t)stream;
  size_t max_n = 0;
  for (const Slot& s : c->slots) if (s.kind != SLOT_VEC) max_n = std::max(max_n, (size_t)s.rows * s.cols);
  if (ensure_staging(c, max_n * 2 + 256)) return -1;
  const double sigma = 65536.0 / sqrt(3.0);
  for (const Slot& s : c->slots) {
    const int64_t n = s.rows * s.cols;
    const uint32_t sd = fnv1a32(s.name.c_str()) ^ (uint32_t)(seed * 0x9E3779B1u);
    const float mul = (float)(s.std / sigma);
    if (s.kind == SLOT_VEC) {
      if (fill_hash_normal(nullptr, (float*)s.dst, n, sd, mul, s.mean, st)) return -1;
      if (s.dst2 && fill_hash_normal(nullptr, (float*)s.dst2, n, sd, mul, s.mean, st)) return -1;
    } else {
      bf16* tmp = (bf16*)c->staging;
      if (fill_hash_normal(tmp, nullptr, n, sd, mul, s.mean, st)) return -1;
      if (s.kind == SLOT_Q8) {
        if (quantize_rows_q8(tmp, VCLA_BF16, (int)s.rows, (int)s.cols, q8_which(s), (int8_t*)s.dst, s.scale, st)) return -1;
      } else if (place_matrix(s, tmp, st)) return -1;
    }
  }
  VCLA_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

int vcla_reset(vcla_ctx* c, vcla_stream stream) {
  VCLA_CUDA_OK(cudaMemsetAsync(c->seq_len, 0, (size_t)c->cfg.max_batch * 4, (cudaStream_t)stream));
  VCLA_CUDA_OK(cudaMemsetAsync(c->attn_counters, 0, (size_t)64 * c->cfg.t_heads * 4, (cudaStream_t)stream));
  VCLA_CUDA_OK(cudaMemsetAsync(c->step_idx, 0, 4, (cudaStream_t)stream));
  // every page back on the free stack, no sequence owns any
  if (kv_reset(c->kv, c->kv_order, c->cfg.max_batch, (cudaStream_t)stream)) return -1;
  if (c->dp_step) VCLA_CUDA_OK(cudaMemsetAsync(c->dp_step, 0, 4, (cudaStream_t)stream));
  VCLA_CUDA_OK(cudaMemsetAsync(c->finished, 0, 64 * 4, (cudaStream_t)stream));
  c->len_bound = 0;
  c->resident_b = 0;
  c->forked = false;
  return 0;
}

int vcla_kv_truncate(vcla_ctx* c, const int32_t* len_host, int B, vcla_stream stream) {
  if (!c || !len_host) { set_error("vcla_kv_truncate: null arguments"); return -1; }
  if (c->resident_b <= 0) { set_error("vcla_kv_truncate: no resident sequences (call vcla_prefill first)"); return -1; }
  if (B != c->resident_b) { set_error("vcla_kv_truncate: batch %d differs from the %d resident sequences", B, c->resident_b); return -1; }
  int64_t longest = 0;
  for (int b = 0; b < B; ++b) {
    if (len_host[b] < 0) { set_error("vcla_kv_truncate: negative length %d for sequence %d", len_host[b], b); return -1; }
    longest = std::max<int64_t>(longest, len_host[b]);
  }
  count(c); if (kv_truncate(c->seq_len, len_host, B, (cudaStream_t)stream)) return -1;
  c->len_bound = std::min(c->len_bound, longest);
  return 0;
}

int vcla_kv_debug_shuffle(vcla_ctx* c, uint32_t seed) {
  // test hook: permute the order in which physical pages are handed out (Fisher-Yates over an LCG); takes effect at the next reset
  std::vector<int32_t> order((size_t)c->kv.total_pages);
  for (size_t i = 0; i < order.size(); ++i) order[i] = (int32_t)i;
  uint64_t x = 0x9E3779B97F4A7C15ull ^ seed;
  for (size_t i = order.size(); i > 1; --i) {
    x = x * 6364136223846793005ull + 1442695040888963407ull;
    std::swap(order[i - 1], order[(size_t)((x >> 33) % i)]);
  }
  VCLA_CUDA_OK(cudaDeviceSynchronize());
  VCLA_CUDA_OK(cudaMemcpy(c->kv_order, order.data(), order.size() * 4, cudaMemcpyHostToDevice));
  return vcla_reset(c, nullptr);
}

int vcla_kv_read_pages(vcla_ctx* c, int32_t* table_host, int32_t* npages_host, int32_t* state_host) {
  // synchronous copy of the page table [max_batch][pages_per_seq], the per-sequence page counts and {free pages, error flag}
  VCLA_CUDA_OK(cudaDeviceSynchronize());
  if (table_host) VCLA_CUDA_OK(cudaMemcpy(table_host, c->kv.table, (size_t)c->cfg.max_batch * c->kv.pages_per_seq * 4, cudaMemcpyDeviceToHost));
  if (npages_host) VCLA_CUDA_OK(cudaMemcpy(npages_host, c->kv.npages, (size_t)c->cfg.max_batch * 4, cudaMemcpyDeviceToHost));
  if (state_host) VCLA_CUDA_OK(cudaMemcpy(state_host, c->kv.state, 8, cudaMemcpyDeviceToHost));
  return 0;
}
int vcla_kv_read_layer(vcla_ctx* c, int layer, void* host) {
  if (!c || !host || layer < 0 || layer >= c->kv.layers) { set_error("vcla_kv_read_layer: bad arguments"); return -1; }
  VCLA_CUDA_OK(cudaDeviceSynchronize());
  VCLA_CUDA_OK(cudaMemcpy(host, c->kv.layer(layer).pages, c->kv_bytes / c->kv.layers, cudaMemcpyDeviceToHost));
  return 0;
}
int vcla_kv_geometry(const vcla_ctx* c, int* pages_per_seq, int* total_pages, int* page_tokens) {
  if (!c) return -1;
  if (pages_per_seq) *pages_per_seq = c->kv.pages_per_seq;
  if (total_pages) *total_pages = c->kv.total_pages;
  if (page_tokens) *page_tokens = c->kv.page_tokens;
  return 0;
}

// -------------------------------------------------------------------------------------------------
// vision encode
// -------------------------------------------------------------------------------------------------
static int gemm_bf16(vcla_ctx* c, const bf16* A, int M, int K, int lda, const bf16* W, int N, int ldw, const float* bias, int act, bf16* out, int ldo, cudaStream_t st) {
  GemmCall g; g.A = A; g.B = W; g.M = M; g.N = N; g.K = K; g.lda = lda; g.ldb = ldw; g.mode = GEMM_STORE_BF16; g.out = out; g.ldo = ldo; g.bias = bias; g.act = act;
  count(c); return gemm_tc(g, st);
}
static int gemm_f32(vcla_ctx* c, const bf16* A, int M, int K, int lda, const bf16* W, int N, int ldw, const float* bias, int accumulate, float* out, int ldo, cudaStream_t st) {
  GemmCall g; g.A = A; g.B = W; g.M = M; g.N = N; g.K = K; g.lda = lda; g.ldb = ldw; g.mode = GEMM_ADD_F32; g.out = out; g.ldo = ldo; g.bias = bias; g.accumulate = accumulate;
  count(c); return gemm_tc(g, st);
}

int vcla_vision_encode(vcla_ctx* c, const void* pixels, int pixel_dtype, int B, float* out_dev, vcla_stream stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const vcla_config& g = c->cfg;
  if (B < 1 || B > g.max_batch) { set_error("vision_encode: batch %d exceeds capacity %d", B, g.max_batch); return -1; }
  const int D = g.v_hidden, NT = c->v_tokens, NP = NT - 1, rows = B * NT;
  // patch embedding: im2col + GEMM; epilogue adds the position embedding and scatters to token rows 1..NP
  count(c); if (im2col(pixels, pixel_dtype, B, g.v_image, g.v_patch, c->kpad, c->v_im2col, st)) return -1;
  {
    GemmCall gc; gc.A = c->v_im2col; gc.B = c->patch_w; gc.M = B * NP; gc.N = D; gc.K = c->kpad; gc.lda = c->kpad; gc.ldb = c->kpad;
    gc.mode = GEMM_ADD_F32; gc.out = c->v_hidden; gc.ldo = D; gc.rowtab = c->pos + D; gc.rowtab_period = NP;
    gc.rows_per_group = NP; gc.group_stride = NT; gc.row_offset = 1;
    count(c); if (gemm_tc(gc, st)) return -1;
  }
  count(c); if (vit_cls_rows(c->v_hidden, B, NT, D, c->cls, c->pos, st)) return -1;
  count(c); if (layernorm(c->v_hidden, rows, D, c->pre_w, c->pre_b, g.v_eps, nullptr, c->v_hidden, st)) return -1;
  const float vscale = 1.0f / sqrtf(64.f);
  for (int i = 0; i < g.v_layers; ++i) {
    const VisionLayer& L = c->vl[i];
    count(c); if (layernorm(c->v_hidden, rows, D, L.ln1_w, L.ln1_b, g.v_eps, c->v_norm, nullptr, st)) return -1;
    if (gemm_bf16(c, c->v_norm, rows, D, D, L.wqkv, 3 * D, D, L.bqkv, ACT_NONE, c->v_qkv, 3 * D, st)) return -1;
    AttnCall a; a.q = c->v_qkv; a.q_stride = 3 * D; a.k0 = c->v_qkv + D; a.v0 = c->v_qkv + 2 * D; a.kv0_stride = 3 * D; a.n0 = NT;
    a.out = c->v_attn; a.o_stride = D; a.B = B; a.H = g.v_heads; a.Sq = NT; a.HD = 64; a.scale = vscale; a.causal = 0;
    count(c); if (attention_prefill(a, st)) return -1;
    if (gemm_f32(c, c->v_attn, rows, D, D, L.wo, D, D, L.bo, 1, c->v_hidden, D, st)) return -1;
    count(c); if (layernorm(c->v_hidden, rows, D, L.ln2_w, L.ln2_b, g.v_eps, c->v_norm, nullptr, st)) return -1;
    if (gemm_bf16(c, c->v_norm, rows, D, D, L.w1, g.v_ffn, D, L.b1, ACT_QUICK_GELU, c->v_ffn, g.v_ffn, st)) return -1;
    if (gemm_f32(c, c->v_ffn, rows, g.v_ffn, g.v_ffn, L.w2, D, g.v_ffn, L.b2, 1, c->v_hidden, D, st)) return -1;
  }
  // post_layernorm on ALL tokens (what the reference does, modeling_visualcla.py:284/350)
  count(c); if (layernorm(c->v_hidden, rows, D, c->post_w, c->post_b, g.v_eps, c->v_norm, c->v_postln_f32, st)) return -1;

  // ---- Resampler
  const int R = g.r_hidden, Q = g.r_queries, RL = g.r_layers, qrows = B * Q;
  count(c); if (broadcast_rows(c->rq, Q, R, B, c->r_hidden, c->r_hidden_bf16, st)) return -1;
  // K/V of the (layer-invariant) image rows for all layers in one GEMM
  if (gemm_bf16(c, c->v_norm, rows, R, R, c->r_wkv_all, RL * 2 * R, R, c->r_bkv_all, ACT_NONE, c->r_kvimg, RL * 2 * R, st)) return -1;
  const float rscale = 1.0f / sqrtf(64.f);
  for (int i = 0; i < RL; ++i) {
    const ResamplerLayer& L = c->rl[i];
    if (gemm_bf16(c, c->r_hidden_bf16, qrows, R, R, L.wqkv, 3 * R, R, L.bqkv, ACT_NONE, c->r_qkv, 3 * R, st)) return -1;
    AttnCall a; a.q = c->r_qkv; a.q_stride = 3 * R;
    a.k0 = c->r_qkv + R; a.v0 = c->r_qkv + 2 * R; a.kv0_stride = 3 * R; a.n0 = Q;          // the query rows themselves (:315 cat)
    a.k1 = c->r_kvimg + (size_t)i * 2 * R; a.v1 = a.k1 + R; a.kv1_stride = RL * 2 * R; a.n1 = NT;   // image rows
    a.out = c->r_ctx; a.o_stride = R; a.B = B; a.H = g.r_heads; a.Sq = Q; a.HD = 64; a.scale = rscale; a.causal = 0;
    count(c); if (attention_prefill(a, st)) return -1;
    if (gemm_f32(c, c->r_ctx, qrows, R, R, L.wo, R, R, L.bo, 1, c->r_hidden, R, st)) return -1;           // dense + residual
    count(c); if (layernorm(c->r_hidden, qrows, R, L.ln1_w, L.ln1_b, g.r_eps, c->r_hidden_bf16, c->r_hidden, st)) return -1;  // post-LN
    if (gemm_bf16(c, c->r_hidden_bf16, qrows, R, R, L.wi, g.r_ffn, R, L.bi, ACT_GELU_ERF, c->r_ffn, g.r_ffn, st)) return -1;
    if (gemm_f32(c, c->r_ffn, qrows, g.r_ffn, g.r_ffn, L.wo2, R, g.r_ffn, L.bo2, 1, c->r_hidden, R, st)) return -1;
    count(c); if (layernorm(c->r_hidden, qrows, R, L.ln2_w, L.ln2_b, g.r_eps, c->r_hidden_bf16, c->r_hidden, st)) return -1;
  }
  // projector -> fp32 image embeddings
  if (gemm_f32(c, c->r_hidden_bf16, qrows, R, R, c->proj_w, g.t_hidden, R, c->proj_b, 0, c->img_embeds, g.t_hidden, st)) return -1;
  if (out_dev) VCLA_CUDA_OK(cudaMemcpyAsync(out_dev, c->img_embeds, (size_t)qrows * g.t_hidden * 4, cudaMemcpyDeviceToDevice, st));
  return 0;
}

// -------------------------------------------------------------------------------------------------
// decode launches (the prefill's last-position lm_head uses the workspace one too)
// -------------------------------------------------------------------------------------------------
// The batch size picks the decode schedule: up to 32 rows the cluster split-K GEMMs with fused consumers (5 kernels
// per layer); 33..64 rows split-K partials in an L2 workspace reduced by separate consumer kernels (8 kernels per layer).
// int8 projections (weight_format 1) run the cluster split-K schedule at every batch: its int8 kernel has a 64-column batch tile.
static bool decode_uses_csk(const vcla_ctx* c, int B) { return B <= 32 || c->cfg.weight_format == 1; }
static int csk_max_batch(const vcla_ctx* c) { return c->cfg.weight_format == 1 ? 64 : 32; }
// The bf16 lm_head of a decode step runs on the cluster kernel up to 32 rows, beyond on the workspace GEMM (one stream of its weights
// over all rows).  The prefill's last-row head always takes the workspace GEMM (lm_head_last).
static bool lm_head_uses_csk(int B) { return B <= 32; }

// The five weight-streaming GEMMs of a decode step (numbering of vcla_bench_decode_gemm's `which`).
enum DecodeGemm { DG_QKV = 0, DG_O = 1, DG_GATE_UP = 2, DG_DOWN = 3, DG_LM_HEAD = 4 };

// GEMM `which` of decode layer i (i is ignored for the lm_head) on the workspace schedule: swap-AB split-K partials of
// the d_xn / d_attn / d_h rows into that GEMM's fp32 L2 workspace, reduced by the next consumer kernel.
static int ws_gemm(vcla_ctx* c, int which, int i, int B, cudaStream_t st) {
  const vcla_config& g = c->cfg;
  const int TH = g.t_hidden, F = g.t_ffn;
  const TextLayer* L = which == DG_LM_HEAD ? nullptr : &c->tl[i];
  GemmCall gc; gc.N = B; gc.mode = GEMM_PARTIAL_F32; gc.ws_rows = B; gc.weights_are_A = 1; gc.l2_prefetch_kb = c->l2_prefetch_kb;
  switch (which) {
    case DG_QKV: gc.A = L->wqkv; gc.B = c->d_xn; gc.M = 3 * TH; gc.K = TH; gc.splits = c->sp_qkv; gc.out = c->ws_qkv; break;
    case DG_O: gc.A = L->wo; gc.B = c->d_attn; gc.M = TH; gc.K = TH; gc.splits = c->sp_o; gc.out = c->ws_o; break;
    case DG_GATE_UP: gc.A = L->wgu; gc.B = c->d_xn; gc.M = 2 * F; gc.K = TH; gc.splits = c->sp_gu; gc.out = c->ws_gu; break;
    case DG_DOWN: gc.A = L->wd; gc.B = c->d_h; gc.M = TH; gc.K = F; gc.splits = c->sp_d; gc.out = c->ws_d; break;
    default: gc.A = c->lm_head; gc.B = c->d_xn; gc.M = g.t_vocab; gc.K = TH; gc.splits = c->sp_lm; gc.out = c->ws_lm; break;
  }
  gc.lda = gc.ldb = gc.K; gc.ldo = gc.M;
  count(c); return gemm_tc(gc, st);
}

// GEMM `which` of decode layer i on the cluster split-K schedule (gemm_decode.cu): the split-K reduction and the consumer run
// inside the GEMM, with RMSNorm's row scale deferred to the next GEMM through the per-row sums of squares in d_ssq.
static int csk_gemm(vcla_ctx* c, int which, int i, int B, cudaStream_t st) {
  const vcla_config& g = c->cfg;
  const int TH = g.t_hidden, F = g.t_ffn;
  const TextLayer* L = which == DG_LM_HEAD ? nullptr : &c->tl[i];
  CskCall k; k.B = B; k.inv_dim = 1.0f / (float)TH; k.eps = g.t_eps;
  switch (which) {
    case DG_QKV: k.W = L->wqkv; k.Wq = L->qqkv; k.wscale = L->sqkv; k.X = c->d_xn; k.M = 3 * TH; k.K = TH; k.splits = c->csk_qkv; k.mode = CSK_OUT_F32; k.out = c->ws_qkv; break;
    case DG_O: k.W = L->wo; k.Wq = L->qo; k.wscale = L->so; k.X = c->d_attn; k.M = TH; k.K = TH; k.splits = c->csk_o; k.mode = CSK_RESID; k.norm_w = L->ln2; break;
    case DG_GATE_UP: k.W = L->wgu; k.Wq = L->qgu; k.wscale = L->sgu; k.X = c->d_xn; k.M = 2 * F; k.K = TH; k.splits = c->csk_gu; k.mode = CSK_SWIGLU; k.h = c->d_h; break;
    case DG_DOWN: k.W = L->wd; k.Wq = L->qd; k.wscale = L->sd; k.X = c->d_h; k.M = TH; k.K = F; k.splits = c->csk_d; k.mode = CSK_RESID;
      k.norm_w = (i + 1 < g.t_layers) ? c->tl[i + 1].ln1 : c->final_norm; break;
    default: k.W = c->lm_head; k.X = c->d_xn; k.M = g.t_vocab; k.K = TH; k.splits = c->csk_lm; k.mode = CSK_OUT_F32; k.out = c->ws_lm; break;
  }
  if (k.mode == CSK_OUT_F32) k.ldo = k.M;
  if (k.mode == CSK_RESID) {
    k.resid = c->d_resid; k.xw = c->d_xn; k.ssq_out = c->d_ssq;
  } else {
    k.ssq_in = c->d_ssq; k.ssq_slots = (TH + 127) / 128;   // one slot per 128-row tile of the o / down projections
  }
  count(c); return gemm_csk(k, st);
}

// Decode attention of layer L over the paged KV cache, reading the fused QKV projection from ws_qkv (qkv_splits partials).
static DecodeAttnCall decode_attn_call(const vcla_ctx* c, int layer, int B, int qkv_splits) {
  const vcla_config& g = c->cfg;
  DecodeAttnCall a; a.qkv_partial = c->ws_qkv; a.splits = qkv_splits; a.ws_rows = B; a.kv = c->kv.layer(layer);
  a.seq_len = c->seq_len; a.out = c->d_attn; a.scratch = c->attn_scratch;
  a.counters = c->attn_counters; a.B = B; a.HD = 128; a.scale = 1.0f / sqrtf(128.f); a.rope_theta = g.rope_theta;
  a.rope_cos = c->rope_cos; a.rope_sin = c->rope_sin; a.persistent_mode = c->attn_persistent_mode; a.persistent_grid = c->attn_persistent_grid;
  // enough CTAs to cover the SMs for small batches; long contexts split so a CTA streams <= ~12 pages
  const int want = (num_sms() + B * g.t_heads - 1) / (B * g.t_heads);
  a.kv_splits = std::min(8, std::max(want, c->kv_splits));
  return a;
}

// ---- data parallel token exchange -------------------------------------------------------------------------------
// One all-gather of this rank's `dp_width` token slots + append to the global history.  fork != 0: on the side stream, joined by
// the next dp_wait() (the exchange is off the step's critical path: only the caller, not the next step, consumes it).
static int dp_gather(vcla_ctx* c, cudaStream_t st, int fork) {
  cudaStream_t gs = st;
  if (fork) {
    VCLA_CUDA_OK(cudaEventRecord(c->dp_fork, st));
    VCLA_CUDA_OK(cudaStreamWaitEvent(c->dp_stream, c->dp_fork, 0));
    gs = c->dp_stream;
  }
  VCLA_NCCL_OK(g_nccl.AllGather(c->dp_send, c->dp_recv, (size_t)c->dp_width, ncclInt32, c->comm, gs));
  count(c); if (dp_unpack(c->dp_recv, c->dp_world * c->dp_width, c->dp_hist, c->dp_step, gs)) return -1;
  if (fork) { VCLA_CUDA_OK(cudaEventRecord(c->dp_join, gs)); c->dp_pending = true; }
  return 0;
}
static int dp_wait(vcla_ctx* c, cudaStream_t st) {
  if (!c->dp_pending) return 0;
  VCLA_CUDA_OK(cudaStreamWaitEvent(st, c->dp_join, 0));
  c->dp_pending = false;
  return 0;
}

// The token pick of one step from the lm_splits partials the lm_head left in ws_lm: beam search, the sampler or the argmax (+ the
// token exchange when data parallel).  fork == 0: the prefill's pick (beam search's first step, the exchange inline; with fan-out the
// sampler draws fanout picks from each of the B prompts' logits rows).  lookup: the picks of all B rows of a prompt lookup verification
// step into lk_pick, without history, step, finished-flag or exchange writes.
static int pick(vcla_ctx* c, int B, int lm_splits, float* logits, int32_t* tok, int fork, bool lookup, cudaStream_t st) {
  const vcla_config& g = c->cfg;
  if (lookup) {
    const int V = g.t_vocab;
    count(c, 2);
    if (c->samp_on) {
      if (dec_logits_reduce(c->ws_lm, lm_splits, B, V, B, V, c->samp_logits, V, c->cand_val, c->cand_idx, st)) return -1;
      return dec_sample_lookup(c->samp_logits, V, V, B, c->tok_hist, c->step_idx, c->samp_params, c->lk_pick, st);
    }
    return dec_logits_argmax(c->ws_lm, lm_splits, B, V, B, V, nullptr, V, c->lk_pick, nullptr, nullptr, c->cand_val, c->cand_idx, nullptr, st);
  }
  if (c->dp_on() && dp_wait(c, st)) return -1;            // the previous step's exchange must have read dp_send before it is rewritten
  if (c->beam_on) {
    // B rows: the prompts at the prefill (fork == 0; every item's beams are still its prompt), else B / K items of K beams
    float* lg = logits ? logits : c->samp_logits;
    const bool first = fork == 0;
    const int R = first ? 1 : c->beam_K, items = B / R;
    count(c, 3);
    if (dec_logits_reduce(c->ws_lm, lm_splits, B, g.t_vocab, B, g.t_vocab, lg, g.t_vocab, c->cand_val, c->cand_idx, st)) return -1;
    if (dec_beam_step(lg, g.t_vocab, g.t_vocab, B, c->tok_hist, c->step_idx, c->beam_params, first ? nullptr : c->beam_run, c->beam_cand_val,
                      c->beam_cand_tok, st)) return -1;
    return dec_beam_select(c->beam_params, items, R, g.t_vocab, c->step_idx, c->beam_cand_val, c->beam_cand_tok, c->tok_hist, c->beam_run,
                           c->beam_parent, tok, c->hyp_score, c->hyp_len, c->hyp_fin, c->hyp_tok, c->hyp_tmp, c->cfg.max_seq, c->beam_state, nullptr, st);
  }
  if (c->samp_on) {
    // logits -> [repetition penalty, no-repeat-ngram, temperature, top-k, top-p, draw] in one kernel; raw logits stay available
    float* lg = logits ? logits : c->samp_logits;
    const int n = fork == 0 ? c->fanout : 1;
    count(c, 2);
    if (dec_logits_reduce(c->ws_lm, lm_splits, B, g.t_vocab, B, g.t_vocab, lg, g.t_vocab, c->cand_val, c->cand_idx, st)) return -1;
    if (dec_sample(lg, g.t_vocab, g.t_vocab, B * n, c->tok_hist, c->step_idx, c->samp_params, tok, c->tok_hist, c->dp_on() ? c->dp_send : nullptr,
                   c->finished, nullptr, st, n)) return -1;
    if (c->dp_on()) return dp_gather(c, st, fork);
    return 0;
  }
  count(c, 2);
  if (dec_logits_argmax(c->ws_lm, lm_splits, B, g.t_vocab, B, g.t_vocab, logits, g.t_vocab, tok, c->tok_hist, c->step_idx, c->cand_val, c->cand_idx,
                        c->dp_on() ? c->dp_send : nullptr, st)) return -1;
  if (c->dp_on()) return dp_gather(c, st, fork);
  return 0;
}

static int lm_head_last(vcla_ctx* c, int B, float* logits_dev, int32_t* tok_dev, cudaStream_t st) {
  // d_resid[B, T] holds the hidden state of the positions to score
  const vcla_config& g = c->cfg;
  count(c); if (dec_resid_norm(nullptr, 0, B, c->d_resid, B, g.t_hidden, c->final_norm, g.t_eps, c->d_xn, st)) return -1;
  if (ws_gemm(c, DG_LM_HEAD, 0, B, st)) return -1;
  return pick(c, B, c->sp_lm, logits_dev, tok_dev ? tok_dev : c->d_tok, 0, false, st);
}

// The LLaMA stack over the B x S rows already embedded in c->resid.  base_len == nullptr: a whole prompt (causal attention over its
// own rows); otherwise a chunk appended to the base_len[b] cached tokens of each sequence (RoPE positions and cache slots start at
// base_len[b], attention reads the cached prefix from the page pool).
static int prefill_layers(vcla_ctx* c, int B, int S, const int32_t* left_pad, int pos_from_mask, const int32_t* base_len, cudaStream_t st) {
  const vcla_config& g = c->cfg;
  const int TH = g.t_hidden, F = g.t_ffn, H = g.t_heads;
  const int rows = B * S;
  const float scale = 1.0f / sqrtf(128.f);
  // 5 kernels per layer: RMSNorm is deferred (operand = bf16(resid * norm_w); the row scale commutes with the GEMM and is applied in
  // the consuming GEMM's epilogue from the per-tile sums of squares the producing GEMM wrote), RoPE + KV-cache append run in the
  // QKV GEMM's epilogue on the fp32 accumulator, SwiGLU in the gate/up epilogue, the residual add in the O / down epilogues.
  const int slots = (TH + gemm_pick_bn(rows, TH) - 1) / gemm_pick_bn(rows, TH);
  GemmRowScale rsc; rsc.ssq = c->p_ssq; rsc.slots = slots; rsc.inv_dim = 1.0f / (float)TH; rsc.eps = g.t_eps;
  count(c); if (prenorm_rows(c->resid, rows, TH, c->tl[0].ln1, c->xn, c->p_ssq, slots, st)) return -1;
  // int8 projections: each GEMM first expands its int8 rows to bf16(q) (exact) in q8_wide and takes the row scales as column scales,
  // so the prefill computes sum(q x) * s like the decode kernel
  const bool q8 = g.weight_format == 1;
  auto weight = [&](const bf16* w, const int8_t* q, int n, int k, GemmCall& gc, const float* sc) -> int {
    if (!q8) { gc.B = w; return 0; }
    count(c); if (expand_rows_q8(q, n, k, 1, c->q8_wide, st)) return -1;
    gc.B = c->q8_wide; gc.colscale = sc;
    return 0;
  };
  for (int i = 0; i < g.t_layers; ++i) {
    const TextLayer& L = c->tl[i];
    {
      GemmCall gc; if (weight(L.wqkv, L.qqkv, 3 * TH, TH, gc, L.sqkv)) return -1;
      gc.A = c->xn; gc.M = rows; gc.N = 3 * TH; gc.K = TH; gc.lda = TH; gc.ldb = TH; gc.mode = GEMM_STORE_BF16; gc.out = c->qkv; gc.ldo = 3 * TH;
      gc.rowscale = rsc;
      gc.rope.cos = c->rope_cos; gc.rope.sin = c->rope_sin; gc.rope.kv = c->kv.layer(i);
      gc.rope.S = S; gc.rope.T = TH; gc.rope.left_pad = left_pad; gc.rope.pos_from_mask = pos_from_mask;
      gc.rope.base_len = base_len;
      gc.kv_format = c->kv_format();
      count(c); if (gemm_tc(gc, st)) return -1;
    }
    if (base_len == nullptr) {
      AttnCall a; a.q = c->qkv; a.q_stride = 3 * TH; a.k0 = c->qkv + TH; a.v0 = c->qkv + 2 * TH; a.kv0_stride = 3 * TH; a.n0 = S;
      a.out = c->attn; a.o_stride = TH; a.B = B; a.H = H; a.Sq = S; a.HD = 128; a.scale = scale; a.causal = 1; a.kv_start = left_pad;
      count(c); if (attention_prefill(a, st)) return -1;
    } else {
      AttnPagedCall a; a.q = c->qkv; a.q_stride = 3 * TH; a.kv = c->kv.layer(i); a.base_len = base_len; a.max_kv = (int)c->len_bound + S;
      a.out = c->attn; a.o_stride = TH; a.B = B; a.T = S; a.scale = scale; a.part = c->pa_part; a.counters = c->pa_counters;
      count(c); if (attention_paged(a, st, c->kv_format())) return -1;
    }
    {
      GemmCall gc; if (weight(L.wo, L.qo, TH, TH, gc, L.so)) return -1;
      gc.A = c->attn; gc.M = rows; gc.N = TH; gc.K = TH; gc.lda = TH; gc.ldb = TH; gc.mode = GEMM_ADD_F32; gc.accumulate = 1; gc.out = c->resid; gc.ldo = TH;
      gc.emit.norm_w = L.ln2; gc.emit.xw = c->xn; gc.emit.ldxw = TH; gc.emit.ssq_out = c->p_ssq;
      count(c); if (gemm_tc(gc, st)) return -1;
    }
    {
      GemmCall gc; if (weight(L.wgu, L.qgu, 2 * F, TH, gc, L.sgu)) return -1;
      gc.A = c->xn; gc.M = rows; gc.N = 2 * F; gc.K = TH; gc.lda = TH; gc.ldb = TH; gc.mode = GEMM_SWIGLU_BF16; gc.out = c->hmid; gc.ldo = F;
      gc.rowscale = rsc;
      count(c); if (gemm_tc(gc, st)) return -1;
    }
    {
      GemmCall gc; if (weight(L.wd, L.qd, TH, F, gc, L.sd)) return -1;
      gc.A = c->hmid; gc.M = rows; gc.N = TH; gc.K = F; gc.lda = F; gc.ldb = F; gc.mode = GEMM_ADD_F32; gc.accumulate = 1; gc.out = c->resid; gc.ldo = TH;
      gc.emit.norm_w = (i + 1 < g.t_layers) ? c->tl[i + 1].ln1 : c->final_norm; gc.emit.xw = c->xn; gc.emit.ldxw = TH; gc.emit.ssq_out = c->p_ssq;
      count(c); if (gemm_tc(gc, st)) return -1;
    }
  }
  return 0;
}

// logits of every row (optional) and of each sequence's last row (+ the argmax / sampler pick), from the final residual stream
static int prefill_logits(vcla_ctx* c, int B, int S, float* logits_all, float* last_logits, int32_t* next_tok, cudaStream_t st) {
  const vcla_config& g = c->cfg;
  const int TH = g.t_hidden, rows = B * S;
  if (logits_all) {
    count(c); if (rmsnorm(c->resid, rows, TH, c->final_norm, g.t_eps, c->xn, st)) return -1;
    if (gemm_f32(c, c->xn, rows, TH, TH, c->lm_head, g.t_vocab, TH, nullptr, 0, logits_all, g.t_vocab, st)) return -1;
  }
  count(c); if (gather_last_rows(c->resid, B, S, TH, c->d_resid, st)) return -1;
  return lm_head_last(c, B, last_logits, next_tok, st);
}

static int beam_reorder(vcla_ctx* c, int rows_old, int rows_new, const int32_t* tok, cudaStream_t st);

// after every enqueue that publishes into the token stream ring: lets vcla_stream_wait tell "not yet" from "never"
static int stream_mark(vcla_ctx* c, cudaStream_t st) {
  if (!c->stream_armed) return 0;
  VCLA_CUDA_OK(cudaEventRecord(c->stream_done, st));
  c->stream_pending = true;
  return 0;
}

int vcla_prefill(vcla_ctx* c, const int64_t* ids, int B, int T, int image_mode, const int32_t* img_row, const int32_t* left_pad,
                 int pos_from_mask, float* logits_all, float* last_logits, int32_t* next_tok, vcla_stream stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const vcla_config& g = c->cfg;
  const int nq = g.r_queries, TH = g.t_hidden;
  const int S = (image_mode == VCLA_IMAGE_AT_HEAD) ? T + nq : T;
  if (B < 1 || B > g.max_batch || B > 64) { set_error("prefill: batch %d exceeds capacity (max_batch %d, <= 64 per call)", B, g.max_batch); return -1; }
  if ((long)B * S > g.max_prefill_tokens) { set_error("prefill: %d x %d tokens exceed max_prefill_tokens %d", B, S, g.max_prefill_tokens); return -1; }
  if (S > g.max_seq) { set_error("prefill: sequence %d exceeds max_seq %d", S, g.max_seq); return -1; }
  if (image_mode == VCLA_IMAGE_AT_HEAD && T < 2) { set_error("prefill: image_at_head needs >= 2 text tokens"); return -1; }
  if (image_mode == VCLA_IMAGE_AT_HEAD && left_pad != nullptr) { set_error("prefill: left padding is not defined for the image_at_head layout"); return -1; }
  if (c->beam_on) {
    // each prompt is prefilled once and forked to K rows afterwards
    const int rows = B * c->beam_K, cap = std::min(g.max_batch, 64);
    if (rows > cap) { set_error("prefill: %d prompts x %d beams exceed %d rows (min(max_batch, 64))", B, c->beam_K, cap); return -1; }
    if ((long)S + c->beam_max_new > g.max_seq) { set_error("prefill: prompt %d + %d new tokens exceed max_seq %d", S, c->beam_max_new, g.max_seq); return -1; }
    if (c->dp_on()) { set_error("prefill: beam search is not available while the data-parallel token exchange is active"); return -1; }
  }
  const int n = c->fanout, rows = B * n;
  if (n > 1) {
    // each prompt is prefilled once and forked to n rows after the first pick
    const int cap = std::min(g.max_batch, 64);
    if (rows > cap) { set_error("prefill: %d prompts x %d replies exceed %d rows (min(max_batch, 64))", B, n, cap); return -1; }
    if (c->beam_on) { set_error("prefill: fan-out (vcla_set_fanout) is not available with beam search"); return -1; }
    if (c->dp_on()) { set_error("prefill: fan-out is not available while the data-parallel token exchange is active"); return -1; }
  }
  if (vcla_reset(c, stream)) return -1;
  // pages for the prompt's tokens (real tokens only: left padding is never cached)
  count(c); if (kv_reserve(c->kv, B, S, left_pad, st)) return -1;
  count(c); if (embed_tokens(ids, B, T, S, TH, c->embed, g.t_vocab, image_mode == VCLA_IMAGE_AT_HEAD ? 1 : 0, nq, c->resid, st)) return -1;
  if (image_mode != VCLA_TEXT_ONLY) {
    const int32_t* rs = (image_mode == VCLA_IMAGE_AT_HEAD || img_row == nullptr) ? c->img_row_default : img_row;
    count(c); if (scatter_image_rows(c->img_embeds, B, nq, TH, rs, S, c->resid, st)) return -1;
  }
  if (prefill_layers(c, B, S, left_pad, pos_from_mask, nullptr, st) || prefill_logits(c, B, S, logits_all, last_logits, next_tok, st)) return -1;
  int32_t* picks = next_tok ? next_tok : c->d_tok;
  // fan-out: the parent map of the fork; the argmax picked once per prompt, so its picks (and history row 0) are widened to the rows
  if (n > 1) { count(c); if (fanout_rows(n, rows, c->beam_parent, c->samp_on ? nullptr : picks, c->tok_hist, st)) return -1; }
  // sequence lengths become S - pad; the page the first decoded token will be appended to is reserved here.  The step published to the
  // token stream is history row 0 of all the rows.
  count(c); if (advance_seq(c->seq_len, B, S, left_pad, c->step_idx, c->kv, st, c->ring(), c->tok_hist, rows)) return -1;
  if (c->beam_on && beam_reorder(c, B, B * c->beam_K, picks, st)) return -1;
  // fan-out: row r continues prompt r / n -- it shares the prompt's full pages, and every row but the first of a prompt gets its own copy
  // of the partly filled page it writes next
  if (n > 1 && beam_reorder(c, B, rows, picks, st)) return -1;
  c->len_bound = S;
  c->resident_b = c->beam_on ? B * c->beam_K : rows;
  c->forked = n > 1;
  c->lk_primed = false;
  return stream_mark(c, st);
}

int vcla_prefill_extend(vcla_ctx* c, const int64_t* ids, int B, int T, float* logits_all, float* last_logits, int32_t* next_tok, vcla_stream stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const vcla_config& g = c->cfg;
  if (!ids || T < 1) { set_error("prefill_extend: no tokens"); return -1; }
  if (c->resident_b <= 0) { set_error("prefill_extend: no resident sequences (call vcla_prefill first)"); return -1; }
  if (B != c->resident_b) { set_error("prefill_extend: batch %d differs from the %d resident sequences", B, c->resident_b); return -1; }
  if (c->dp_on()) { set_error("prefill_extend: not available while the data-parallel token exchange is active"); return -1; }
  if (c->beam_on) { set_error("prefill_extend: not available in beam-search mode"); return -1; }
  if (c->fanout > 1 || c->forked) { set_error("prefill_extend: not available in fan-out mode or while forked rows are resident"); return -1; }
  if ((long)B * T > g.max_prefill_tokens) { set_error("prefill_extend: %d x %d tokens exceed max_prefill_tokens %d", B, T, g.max_prefill_tokens); return -1; }
  if (c->len_bound + T > g.max_seq) {
    set_error("prefill_extend: %lld cached tokens + %d exceed the context capacity max_seq=%d", (long long)c->len_bound, T, g.max_seq);
    return -1;
  }
  // like vcla_prefill: the token history, the step counter and the finished flags start over with this call's pick
  VCLA_CUDA_OK(cudaMemsetAsync(c->step_idx, 0, 4, st));
  VCLA_CUDA_OK(cudaMemsetAsync(c->finished, 0, 64 * 4, st));
  count(c); if (kv_reserve(c->kv, B, T, nullptr, st, c->seq_len)) return -1;
  count(c); if (embed_tokens(ids, B, T, T, g.t_hidden, c->embed, g.t_vocab, 0, g.r_queries, c->resid, st)) return -1;
  if (prefill_layers(c, B, T, nullptr, 1, c->seq_len, st) || prefill_logits(c, B, T, logits_all, last_logits, next_tok, st)) return -1;
  count(c); if (advance_seq(c->seq_len, B, T, nullptr, c->step_idx, c->kv, st, c->ring(), c->tok_hist)) return -1;
  c->len_bound += T;
  c->lk_primed = false;
  return stream_mark(c, st);
}

// Beam search: rows_new rows continue the rows_old rows (beam_parent, written by the select kernel) with the tokens `tok`; then the
// copy-on-write rows of the pages written next are copied for every layer.
static int beam_reorder(vcla_ctx* c, int rows_old, int rows_new, const int32_t* tok, cudaStream_t st) {
  count(c, 2);
  if (kv_beam_reorder(rows_old, rows_new, c->beam_parent, tok, c->seq_len, c->kv, c->beam_table_tmp, c->tok_hist, c->step_idx, c->beam_copy,
                      c->beam_cow_bytes, st, c->kv_format()))
    return -1;
  return kv_page_copy(c->kv, c->beam_copy, rows_new, st, c->kv_format());
}

// -------------------------------------------------------------------------------------------------
// decode
// -------------------------------------------------------------------------------------------------
// CTAs per cluster for a [M, K] weight at batch B: the choice that keeps the largest share of the 2 x SMs CTA slots busy over whole
// rounds of cluster-tiles (clusters are gang-scheduled: floor(slots / S) of them are resident).  q8: the int8 kernel's batch tiles.
static int csk_pick(int M, int K, int B, bool q8 = false) {
  const int tiles = (M + 127) / 128, kb = (K + 63) / 64, bn = B <= 16 ? 16 : (B <= 32 || !q8 ? 32 : 64);
  int best = 1; double best_score = -1.0;
  for (int S = 1; S <= 8; ++S) {
    const int per = (kb + S - 1) / S;
    if ((kb + per - 1) / per != S) continue;                 // every K slice non-empty
    if (S > 1 && kb / S < 2) break;
    if (((B + S - 1) / S) * S > bn + 4) continue;            // reduce buffer columns
    int ncl = gemm_csk_clusters(B, S, q8);
    if (ncl <= 0) continue;
    if (ncl > tiles) ncl = tiles;
    const int rounds = (tiles + ncl - 1) / ncl;
    double score = (double)tiles * S / ((double)rounds * 2.0 * num_sms());
    if (rounds >= 2) score += 0.02;                          // a second tile per CTA overlaps its loads with the first one's epilogue
    if (score > best_score) { best_score = score; best = S; }
  }
  return best;
}
static int csk_prepare(vcla_ctx* c, int B) {
  if (c->csk_batch == B) return 0;
  const vcla_config& g = c->cfg;
  const bool q8 = g.weight_format == 1;
  int v[5] = {csk_pick(3 * g.t_hidden, g.t_hidden, B, q8), csk_pick(g.t_hidden, g.t_hidden, B, q8), csk_pick(2 * g.t_ffn, g.t_hidden, B, q8),
              csk_pick(g.t_hidden, g.t_ffn, B, q8), lm_head_uses_csk(B) ? csk_pick(g.t_vocab, g.t_hidden, B) : 1};
  if (const char* e = getenv("VCLA_CSK_SPLITS")) {            // tuning override: "qkv,o,gu,d,lm"
    int o[5];
    if (sscanf(e, "%d,%d,%d,%d,%d", &o[0], &o[1], &o[2], &o[3], &o[4]) == 5) for (int i = 0; i < 5; ++i) if (o[i] >= 1 && o[i] <= 8) v[i] = o[i];
  }
  c->csk_qkv = v[0]; c->csk_o = v[1]; c->csk_gu = v[2]; c->csk_d = v[3]; c->csk_lm = v[4];
  c->csk_batch = B;
  return 0;
}

// Workspace layer stack (bf16 at 33..64 rows), 8 kernels per layer: split-K partials in L2 workspaces reduced by separate consumer
// kernels.  Ends with the final norm, so d_xn holds the normalised rows for the lm_head.
static int ws_stack(vcla_ctx* c, const int32_t* tok_in, int B, cudaStream_t st) {
  const vcla_config& g = c->cfg;
  const int TH = g.t_hidden, F = g.t_ffn;
  count(c); if (embed_tokens_i32(tok_in, B, TH, c->embed, g.t_vocab, c->d_resid, st)) return -1;
  for (int i = 0; i < g.t_layers; ++i) {
    const TextLayer& L = c->tl[i];
    count(c); if (dec_resid_norm(i == 0 ? nullptr : c->ws_d, c->sp_d, B, c->d_resid, B, TH, L.ln1, g.t_eps, c->d_xn, st)) return -1;
    if (ws_gemm(c, DG_QKV, i, B, st)) return -1;
    count(c); if (attention_decode(decode_attn_call(c, i, B, c->sp_qkv), st, c->kv_format())) return -1;
    if (ws_gemm(c, DG_O, i, B, st)) return -1;
    count(c); if (dec_resid_norm(c->ws_o, c->sp_o, B, c->d_resid, B, TH, L.ln2, g.t_eps, c->d_xn, st)) return -1;
    if (ws_gemm(c, DG_GATE_UP, i, B, st)) return -1;
    count(c); if (dec_silu_mul(c->ws_gu, c->sp_gu, B, B, F, c->d_h, st)) return -1;
    if (ws_gemm(c, DG_DOWN, i, B, st)) return -1;
  }
  count(c); return dec_resid_norm(c->ws_d, c->sp_d, B, c->d_resid, B, TH, c->final_norm, g.t_eps, c->d_xn, st);
}

// Cluster split-K layer stack (batches <= 32, every batch with int8 projections), 5 kernels per layer:  QKV GEMM [rstd] ->
// attention(+RoPE, append) -> O GEMM [+residual, norm weight, sum sq] -> gate/up GEMM [rstd, SiLU*mul] -> down GEMM [+residual, next
// norm weight, sum sq].  The bracketed consumers run inside the GEMM after the cluster's split-K reduction; RMSNorm's per-row scale
// rstd is deferred to the consuming GEMM.  lookup: a verification step over B rows of the one resident sequence, whose attention is
// the multi-query mode with the one-row KV split count.
static int csk_stack(vcla_ctx* c, const int32_t* tok_in, int B, bool lookup, cudaStream_t st) {
  const vcla_config& g = c->cfg;
  const int TH = g.t_hidden;
  count(c); if (dec_embed(tok_in, B, TH, c->embed, g.t_vocab, c->d_resid, c->tl[0].ln1, c->d_xn, c->d_ssq, (TH + 127) / 128, st)) return -1;
  for (int i = 0; i < g.t_layers; ++i) {
    if (csk_gemm(c, DG_QKV, i, B, st)) return -1;
    if (lookup) {
      DecodeAttnCall a = decode_attn_call(c, i, 1, 1);
      a.B = B; a.ws_rows = B;
      count(c, 2); if (attention_decode_lookup(a, st, c->kv_format())) return -1;
    } else {
      count(c); if (attention_decode(decode_attn_call(c, i, B, 1), st, c->kv_format())) return -1;
    }
    if (csk_gemm(c, DG_O, i, B, st) || csk_gemm(c, DG_GATE_UP, i, B, st) || csk_gemm(c, DG_DOWN, i, B, st)) return -1;
  }
  return 0;
}

// The lm_head of a decode step over B rows.  -> the split-K partials it left in ws_lm (1: the cluster kernel reduced them), -1 on
// error.  The workspace GEMM reads normalised rows: after the cluster stack (rows_normed false) d_resid is normalised first.
static int lm_head(vcla_ctx* c, int B, bool rows_normed, cudaStream_t st) {
  if (lm_head_uses_csk(B)) return csk_gemm(c, DG_LM_HEAD, 0, B, st) ? -1 : 1;
  if (!rows_normed) {
    const vcla_config& g = c->cfg;
    count(c); if (dec_resid_norm(nullptr, 0, B, c->d_resid, B, g.t_hidden, c->final_norm, g.t_eps, c->d_xn, st)) return -1;
  }
  return ws_gemm(c, DG_LM_HEAD, 0, B, st) ? -1 : c->sp_lm;
}

static LookupCall lookup_call(vcla_ctx* c) {
  LookupCall k; k.R = c->lk_rows; k.prompt = c->lk_prompt;
  k.tok = c->lk_tok; k.pick = c->lk_pick; k.history = c->tok_hist; k.step_idx = c->step_idx; k.seq_len = c->seq_len; k.finished = c->finished;
  k.samp = c->samp_on ? c->samp_params : nullptr; k.state = c->lk_state;
  k.kv = c->kv; k.ring = c->ring();
  return k;
}

// The B sequences take the step's tokens: their lengths grow by one and the page the next token goes to is reserved (beam search then
// rearranges the rows after their parents).  lookup: accept the verified picks, advance, and draft the next step's rows instead.
static int advance(vcla_ctx* c, int B, const int32_t* tok, bool lookup, cudaStream_t st) {
  count(c);
  if (lookup) return lookup_accept(lookup_call(c), 0, st);
  if (advance_seq(c->seq_len, B, 1, nullptr, c->step_idx, c->kv, st, c->ring(), c->tok_hist)) return -1;
  return c->beam_on ? beam_reorder(c, B, B, tok, st) : 0;
}

// One decode step: the layer stack of the batch's schedule, the lm_head, the pick and the advance.  With prompt lookup set, the step
// verifies the lk_rows rows in lk_tok of the one resident sequence on the cluster stack at the split counts of a one-row step
// (csk_prepare(c, 1)), so every row's logits are those of a one-token step.
static int enqueue_decode_step(vcla_ctx* c, const int32_t* tok_in, int B, float* logits, int32_t* tok_out, cudaStream_t st) {
  const bool lookup = c->lk_on, csk = lookup || decode_uses_csk(c, B);
  const int rows = lookup ? c->lk_rows : B;
  if (csk ? csk_stack(c, lookup ? c->lk_tok : tok_in, rows, lookup, st) : ws_stack(c, tok_in, B, st)) return -1;
  const int lm_splits = lm_head(c, rows, !csk, st);
  if (lm_splits < 0 || pick(c, rows, lm_splits, logits, tok_out, 1, lookup, st)) return -1;
  return advance(c, B, tok_out, lookup, st);
}

// The key of a captured decode graph: the call's buffers and step count, and every mode that changes the captured work.
static GraphKey graph_key(const vcla_ctx* c, const int32_t* tok_in, int B, const float* logits, const int32_t* tok_out, int n_steps) {
  return GraphKey{B, tok_in, logits, tok_out, n_steps, c->dp_on() ? 1 : 0, c->samp_on ? 1 : 0, c->beam_on ? c->beam_K : 0, c->stream_armed ? 1 : 0,
                  c->lk_on ? c->lk_rows : 0};
}

static int decode_graph(vcla_ctx* c, const int32_t* tok_in, int B, float* logits, int32_t* tok_out, int n_steps, cudaStream_t st) {
  const GraphKey key = graph_key(c, tok_in, B, logits, tok_out, n_steps);
  auto it = c->graphs.find(key);
  if (it == c->graphs.end()) {
    const int64_t before = c->launches;
    cudaGraph_t graph = nullptr;
    if (!c->cap_stream) VCLA_CUDA_OK(cudaStreamCreateWithFlags(&c->cap_stream, cudaStreamNonBlocking));
    VCLA_CUDA_OK(cudaStreamBeginCapture(c->cap_stream, cudaStreamCaptureModeThreadLocal));
    int rc = 0;
    for (int i = 0; i < n_steps && rc == 0; ++i) rc = enqueue_decode_step(c, tok_in, B, logits, tok_out, c->cap_stream);
    if (rc == 0 && c->dp_on()) rc = dp_wait(c, c->cap_stream);      // a captured graph must join its forked exchange branch
    cudaError_t e = cudaStreamEndCapture(c->cap_stream, &graph);
    if (rc != 0) { if (graph) cudaGraphDestroy(graph); (void)cudaGetLastError(); return -1; }
    if (e != cudaSuccess) { set_error("decode: graph capture failed: %s", cudaGetErrorString(e)); return -1; }
    cudaGraphExec_t exec = nullptr;
    e = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) { set_error("decode: graph instantiate failed: %s", cudaGetErrorString(e)); return -1; }
    const int64_t launches = c->launches - before;
    c->launches = before;  // capture enqueued nothing
    // bounded cache: a caller that keeps passing fresh buffers evicts the least recently used graph instead of growing forever.
    // (Evicting while an older launch of that graph may still be in flight needs the device to be idle first.)
    constexpr size_t kMaxGraphs = 24;
    if (c->graphs.size() >= kMaxGraphs) {
      const auto victim = std::min_element(c->graphs.begin(), c->graphs.end(),
                                           [](const auto& x, const auto& y) { return x.second.last_use < y.second.last_use; });
      VCLA_CUDA_OK(cudaDeviceSynchronize());
      cudaGraphExecDestroy(victim->second.exec);
      c->graphs.erase(victim);
    }
    it = c->graphs.emplace(key, DecodeGraph{exec, launches, 0}).first;
  }
  it->second.last_use = ++c->graph_uses;
  VCLA_CUDA_OK(cudaGraphLaunch(it->second.exec, st));
  c->launches += it->second.launches;
  return 0;
}

// What a decode call needs after its argument checks, and the split counts of its cluster split-K GEMMs (occupancy queries: never
// inside a capture).  Every decode step appends one token per sequence: refuse the call instead of running past the context
// capacity (the kernels index the page table, the RoPE table and the token history by the sequence length).
static int decode_begin(vcla_ctx* c, int n_steps, int B) {
  if (c->len_bound <= 0) { set_error("decode: no prefilled sequences (call vcla_prefill first)"); return -1; }
  if (c->lk_on) {
    if (B != 1 || c->resident_b != 1) { set_error("decode: prompt lookup steps one resident sequence (got B=%d, %d resident)", B, c->resident_b); return -1; }
    return csk_prepare(c, 1);
  }
  if (c->beam_on && B != c->resident_b) {
    // the beams of an item share pages: a step advances exactly the rows the prefill forked
    set_error("decode: beam search steps all %d rows the prefill forked (got %d)", c->resident_b, B);
    return -1;
  }
  if (c->len_bound + n_steps > c->cfg.max_seq) {
    set_error("decode: %lld cached tokens + %d steps exceed the context capacity max_seq=%d", (long long)c->len_bound, n_steps, c->cfg.max_seq);
    return -1;
  }
  return decode_uses_csk(c, B) ? csk_prepare(c, B) : 0;
}

// After a decode call enqueued its work (rc == 0): the bound on the cached tokens grows by the steps it issued, and the token
// stream records the work that publishes into it.
static int decode_end(vcla_ctx* c, int rc, int n_steps, cudaStream_t st) {
  if (rc != 0) return rc;
  c->len_bound += n_steps;
  return stream_mark(c, st);
}

int vcla_decode_step(vcla_ctx* c, const int32_t* tok_in, int B, float* logits, int32_t* tok_out, int use_graph, vcla_stream stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (B < 1 || B > c->cfg.max_batch || B > 64) { set_error("decode: batch %d unsupported", B); return -1; }
  if (!tok_in || !tok_out) { set_error("decode: null token buffers"); return -1; }
  if (c->lk_on) { set_error("decode: prompt lookup verification steps run through vcla_decode_multi"); return -1; }
  if (decode_begin(c, 1, B)) return -1;
  int rc = use_graph ? decode_graph(c, tok_in, B, logits, tok_out, 1, st) : enqueue_decode_step(c, tok_in, B, logits, tok_out, st);
  if (rc == 0 && !use_graph && c->dp_on()) rc = dp_wait(c, st);
  return decode_end(c, rc, 1, st);
}

int vcla_decode_multi(vcla_ctx* c, int32_t* tok_inout, int B, int n_steps, vcla_stream stream) {
  // n_steps greedy decode steps captured back to back in ONE CUDA graph (the token buffer is consumed and rewritten in place,
  // every chosen token is appended to the device-side history): amortises the gap between consecutive graph launches.
  cudaStream_t st = (cudaStream_t)stream;
  if (B < 1 || B > c->cfg.max_batch || B > 64) { set_error("decode: batch %d unsupported", B); return -1; }
  if (!tok_inout || n_steps < 1 || n_steps > 64) { set_error("decode_multi: bad arguments"); return -1; }
  if (decode_begin(c, n_steps, B)) return -1;
  if (c->lk_on && !c->lk_primed) {
    // right after the prefill: history rows = the prefill's pick, seq_len = the prompt
    if (c->len_bound + c->lk_max_new + c->lk_rows - 1 > c->cfg.max_seq) {
      set_error("decode: %lld cached tokens + max_new %d + %d drafts exceed the context capacity max_seq=%d", (long long)c->len_bound,
                c->lk_max_new, c->lk_rows - 1, c->cfg.max_seq);
      return -1;
    }
    count(c); if (lookup_accept(lookup_call(c), 1, st)) return -1;
    c->lk_primed = true;
    c->len_bound += c->lk_max_new - 1;     // upper bound: at most max_new - 1 decoded tokens are cached
  }
  const int rc = decode_graph(c, tok_inout, B, nullptr, tok_inout, n_steps, st);
  return decode_end(c, rc, c->lk_on ? 0 : n_steps, st);   // lookup: the priming above bounded every step's tokens
}

// -------------------------------------------------------------------------------------------------
// device-side sampling (SURVEY 8f-1)
// -------------------------------------------------------------------------------------------------
static int sampler_to_params(const vcla_sampler* s, SamplerParams* p) {
  if (s->n_eos < 0 || s->n_eos > 4) { set_error("sampler: at most 4 eos ids"); return -1; }
  if (s->do_sample && (s->top_k < 1 || s->top_k > 1024)) { set_error("sampler: the device path needs 1 <= top_k <= 1024 (got %d)", s->top_k); return -1; }
  if (s->do_sample && !(s->temperature > 0.f)) { set_error("sampler: temperature must be > 0"); return -1; }
  if (!(s->repetition_penalty > 0.f)) { set_error("sampler: repetition_penalty must be > 0"); return -1; }
  if (s->top_p <= 0.f || s->top_p > 1.f) { set_error("sampler: top_p must be in (0, 1]"); return -1; }
  memset(p, 0, sizeof(*p));
  p->do_sample = s->do_sample ? 1 : 0;
  p->rep_penalty = s->repetition_penalty; p->no_repeat_ngram = s->no_repeat_ngram_size > 0 ? s->no_repeat_ngram_size : 0;
  p->temperature = s->temperature; p->top_k = s->top_k; p->top_p = s->top_p;
  p->one_minus_top_p = (float)(1.0 - (double)s->top_p);
  p->min_new_tokens = s->min_new_tokens; p->n_eos = s->n_eos; p->pad_id = s->pad_token_id;
  for (int i = 0; i < s->n_eos; ++i) p->eos[i] = s->eos_token_id[i];
  p->seed = s->seed;
  return 0;
}

int vcla_sampler_supported(const vcla_ctx* c) { return c ? sampler_supported(c->cfg.t_vocab) : 0; }

int vcla_set_sampler(vcla_ctx* c, const vcla_sampler* s, vcla_stream stream) {
  if (!c) return -1;
  if (s == nullptr) { c->samp_on = false; return 0; }
  if (!sampler_supported(c->cfg.t_vocab)) { set_error("sampler: vocabulary %d does not fit the device sampler", c->cfg.t_vocab); return -1; }
  SamplerParams p;
  if (sampler_to_params(s, &p)) return -1;
  // pageable source: the driver stages it before returning, so `p` may go out of scope
  VCLA_CUDA_OK(cudaMemcpyAsync(c->samp_params, &p, sizeof(p), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  c->samp_on = true;
  return 0;
}

int vcla_read_finished(vcla_ctx* c, int32_t* dst_dev, int B, vcla_stream stream) {
  if (!c || !dst_dev || B < 1 || B > 64) { set_error("vcla_read_finished: bad arguments"); return -1; }
  VCLA_CUDA_OK(cudaMemcpyAsync(dst_dev, c->finished, (size_t)B * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

int vcla_op_sample(const float* logits_dev, int B, int V, const int32_t* history_dev, int L, const vcla_sampler* s, int32_t* tok_dev,
                   float* scores_out_dev, vcla_stream stream) {
  if (!logits_dev || !s || B < 1 || V < 1 || L < 0 || (L > 0 && !history_dev)) { set_error("vcla_op_sample: bad arguments"); return -1; }
  SamplerParams p;
  if (sampler_to_params(s, &p) || sampler_init()) return -1;
  uint8_t* scratch = nullptr;
  VCLA_CUDA_OK(cudaMalloc(&scratch, sizeof(SamplerParams) + 16));
  cudaStream_t st = (cudaStream_t)stream;
  VCLA_CUDA_OK(cudaMemcpyAsync(scratch, &p, sizeof(p), cudaMemcpyHostToDevice, st));
  VCLA_CUDA_OK(cudaMemcpyAsync(scratch + sizeof(SamplerParams), &L, 4, cudaMemcpyHostToDevice, st));
  const int rc = dec_sample(logits_dev, V, V, B, history_dev, (const int32_t*)(scratch + sizeof(SamplerParams)), (const SamplerParams*)scratch, tok_dev, nullptr,
                            nullptr, nullptr, scores_out_dev, st);
  cudaStreamSynchronize(st);
  cudaFree(scratch);
  return rc;
}

// -------------------------------------------------------------------------------------------------
// prompt lookup decoding
// -------------------------------------------------------------------------------------------------
// Rows a verification step may run: k + 1 <= 16 (the 16-column batch tile), and every one-row split count S must reduce the rows
// together: S * ceil(rows / S) <= 20 reduce-buffer columns of that tile (gemm_csk).  Fewer rows change the speed, never the tokens.
static int lookup_rows(vcla_ctx* c, int k) {
  if (csk_prepare(c, 1)) return -1;
  const int splits[5] = {c->csk_qkv, c->csk_o, c->csk_gu, c->csk_d, c->csk_lm};
  int rows = std::min(k, 15) + 1;
  for (; rows > 2; --rows) {
    bool ok = true;
    for (int s : splits) ok = ok && ((rows + s - 1) / s) * s <= 20;
    if (ok) break;
  }
  return rows;
}

int vcla_set_lookup(vcla_ctx* c, const vcla_lookup* lk, vcla_stream stream) {
  if (!c) return -1;
  if (lk == nullptr) {
    c->lk_on = false;
    return 0;
  }
  if (lk->k < 1 || lk->n < 1 || lk->max_new < 1 || lk->prompt_len < 0 || lk->prompt_len > c->cfg.max_seq || (lk->prompt_len > 0 && !lk->prompt_ids)) {
    set_error("vcla_set_lookup: bad arguments (k >= 1, n >= 1, max_new >= 1, 0 <= prompt_len <= max_seq)"); return -1;
  }
  if (c->beam_on) { set_error("vcla_set_lookup: not available in beam-search mode"); return -1; }
  if (c->dp_on()) { set_error("vcla_set_lookup: not available while the data-parallel token exchange is active"); return -1; }
  if (c->resident_b > 1) { set_error("vcla_set_lookup: prompt lookup decodes one sequence (%d resident)", c->resident_b); return -1; }
  const int rows = lookup_rows(c, lk->k);
  if (rows < 0) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  if (lk->prompt_len > 0) VCLA_CUDA_OK(cudaMemcpyAsync(c->lk_prompt, lk->prompt_ids, (size_t)lk->prompt_len * 8, cudaMemcpyDeviceToDevice, st));
  LookupState init;
  memset(&init, 0, sizeof(init));
  // n-grams longer than 16 are searched as 16: the one-CTA search costs ~n^2 * len / 256 per step, and n changes the drafts only
  init.n = std::min(lk->n, 16); init.max_new = lk->max_new; init.prompt_len = lk->prompt_len;
  // pageable source: staged by the driver before the call returns
  VCLA_CUDA_OK(cudaMemcpyAsync(c->lk_state, &init, sizeof(init), cudaMemcpyHostToDevice, st));
  c->lk_rows = rows; c->lk_max_new = lk->max_new;
  c->lk_on = true; c->lk_primed = false;
  return 0;
}

int vcla_read_lookup_stats(vcla_ctx* c, int64_t* out, vcla_stream stream) {
  if (!c || !out) { set_error("vcla_read_lookup_stats: null argument"); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  int32_t step = 0, fin = 0;
  LookupState s;
  VCLA_CUDA_OK(cudaMemcpyAsync(&step, c->step_idx, 4, cudaMemcpyDeviceToHost, st));
  VCLA_CUDA_OK(cudaMemcpyAsync(&fin, c->finished, 4, cudaMemcpyDeviceToHost, st));
  VCLA_CUDA_OK(cudaMemcpyAsync(&s, c->lk_state, sizeof(s), cudaMemcpyDeviceToHost, st));
  VCLA_CUDA_OK(cudaStreamSynchronize(st));
  out[0] = step; out[1] = fin; out[2] = (int64_t)s.steps; out[3] = (int64_t)s.drafted; out[4] = (int64_t)s.accepted; out[5] = c->lk_rows;
  return 0;
}

// -------------------------------------------------------------------------------------------------
// beam search
// -------------------------------------------------------------------------------------------------
static int beam_to_params(const vcla_beam* s, int V, BeamParams* p) {
  if (s->num_beams < 2 || s->num_beams > kBeamMaxK) { set_error("beam: num_beams must be in 2..%d (got %d)", kBeamMaxK, s->num_beams); return -1; }
  if (s->n_eos < 0 || s->n_eos > 4) { set_error("beam: at most 4 eos ids"); return -1; }
  if (s->early_stopping < 0 || s->early_stopping > 2) { set_error("beam: early_stopping must be 0 (False), 1 (True) or 2 (\"never\")"); return -1; }
  if (s->max_new_tokens < 1) { set_error("beam: max_new_tokens must be >= 1"); return -1; }
  if (!(s->repetition_penalty > 0.f)) { set_error("beam: repetition_penalty must be > 0"); return -1; }
  memset(p, 0, sizeof(*p));
  p->K = s->num_beams;
  p->M = std::max(2, 1 + s->n_eos) * s->num_beams;
  if (p->M > V) { set_error("beam: %d candidates per step exceed the vocabulary %d", p->M, V); return -1; }
  p->n_eos = s->n_eos;
  for (int i = 0; i < s->n_eos; ++i) p->eos[i] = s->eos_token_id[i];
  p->length_penalty = s->length_penalty; p->early_stopping = s->early_stopping; p->max_new = s->max_new_tokens;
  p->rep_penalty = s->repetition_penalty; p->no_repeat_ngram = s->no_repeat_ngram_size > 0 ? s->no_repeat_ngram_size : 0;
  p->min_new_tokens = s->min_new_tokens;
  return 0;
}

int vcla_set_beam(vcla_ctx* c, const vcla_beam* s) {
  if (!c) return -1;
  if (s == nullptr) { c->beam_on = false; c->beam_K = 0; return 0; }
  if (!beam_supported(c->cfg.t_vocab)) { set_error("beam: vocabulary %d does not fit the beam-step kernel", c->cfg.t_vocab); return -1; }
  if (c->dp_on()) { set_error("beam: not available while the data-parallel token exchange is active"); return -1; }
  if (c->stream_armed) { set_error("beam: not available while token streaming is armed (vcla_stream_arm)"); return -1; }
  if (c->lk_on) { set_error("beam: not available while prompt lookup is set (vcla_set_lookup)"); return -1; }
  BeamParams p;
  if (beam_to_params(s, c->cfg.t_vocab, &p)) return -1;
  if (p.K > std::min(c->cfg.max_batch, 64)) { set_error("beam: %d beams exceed min(max_batch, 64) = %d rows", p.K, std::min(c->cfg.max_batch, 64)); return -1; }
  if (p.max_new > c->cfg.max_seq) { set_error("beam: max_new_tokens %d exceeds max_seq %d", p.max_new, c->cfg.max_seq); return -1; }
  VCLA_CUDA_OK(cudaMemcpy(c->beam_params, &p, sizeof(p), cudaMemcpyHostToDevice));
  c->beam_on = true; c->beam_K = p.K; c->beam_max_new = p.max_new;
  return 0;
}

int vcla_set_fanout(vcla_ctx* c, int n) {
  if (!c) return -1;
  if (n < 1 || n > 64) { set_error("vcla_set_fanout: %d replies per prompt not in 1..64", n); return -1; }
  c->fanout = n;
  return 0;
}

int vcla_read_beams(vcla_ctx* c, int32_t* tokens_host, int32_t* lengths_host, float* scores_host, int32_t* done_host) {
  if (!c || !c->beam_on || c->resident_b <= 0) { set_error("vcla_read_beams: no beam search is resident (vcla_set_beam, then vcla_prefill)"); return -1; }
  const int K = c->beam_K, items = c->resident_b / K, cap = c->cfg.max_seq;
  VCLA_CUDA_OK(cudaDeviceSynchronize());
  if (tokens_host) {
    VCLA_CUDA_OK(cudaMemcpy2D(tokens_host, (size_t)c->beam_max_new * 4, c->hyp_tok, (size_t)cap * 4, (size_t)c->beam_max_new * 4, (size_t)items * K,
                              cudaMemcpyDeviceToHost));
  }
  if (lengths_host) VCLA_CUDA_OK(cudaMemcpy(lengths_host, c->hyp_len, (size_t)items * K * 4, cudaMemcpyDeviceToHost));
  if (scores_host) VCLA_CUDA_OK(cudaMemcpy(scores_host, c->hyp_score, (size_t)items * K * 4, cudaMemcpyDeviceToHost));
  if (done_host) {
    std::vector<int32_t> st((size_t)items * 2);
    VCLA_CUDA_OK(cudaMemcpy(st.data(), c->beam_state, st.size() * 4, cudaMemcpyDeviceToHost));
    for (int b = 0; b < items; ++b) done_host[b] = st[(size_t)b * 2 + 1];
  }
  return 0;
}

int vcla_beam_cow_bytes(vcla_ctx* c, int64_t* bytes, int reset) {
  if (!c) return -1;
  unsigned long long v = 0;
  VCLA_CUDA_OK(cudaDeviceSynchronize());
  VCLA_CUDA_OK(cudaMemcpy(&v, c->beam_cow_bytes, 8, cudaMemcpyDeviceToHost));
  if (bytes) *bytes = (int64_t)v;
  if (reset) VCLA_CUDA_OK(cudaMemset(c->beam_cow_bytes, 0, 8));
  return 0;
}

int vcla_op_beam_step(const float* logits_dev, int B, int V, const int32_t* history_dev, int t, const vcla_beam* beam, float* run_scores_dev,
                      float* hyp_scores_dev, int32_t* hyp_lens_dev, int32_t* hyp_fin_dev, int32_t* hyp_tokens_dev, int32_t* item_state_dev,
                      int32_t* parent_dev, int32_t* token_dev, int32_t* cand_dev, vcla_stream stream) {
  if (!logits_dev || !beam || B < 1 || V < 1 || t < 0 || (t > 0 && !history_dev) || !run_scores_dev || !hyp_scores_dev || !hyp_lens_dev ||
      !hyp_fin_dev || !hyp_tokens_dev || !item_state_dev || !parent_dev || !token_dev) {
    set_error("vcla_op_beam_step: bad arguments"); return -1;
  }
  BeamParams p;
  if (beam_to_params(beam, V, &p) || beam_init()) return -1;
  if (B * p.K > 64) { set_error("vcla_op_beam_step: %d x %d rows exceed 64", B, p.K); return -1; }
  if (t >= p.max_new) { set_error("vcla_op_beam_step: step %d is past max_new_tokens %d", t, p.max_new); return -1; }
  const int R = t == 0 ? 1 : p.K, rows = B * R;
  const size_t n_cand = (size_t)rows * p.M, n_tmp = (size_t)B * p.K * p.max_new;
  uint8_t* scratch = nullptr;
  VCLA_CUDA_OK(cudaMalloc(&scratch, 256 + n_cand * 8 + n_tmp * 4));
  BeamParams* pd = reinterpret_cast<BeamParams*>(scratch);
  int32_t* step = reinterpret_cast<int32_t*>(scratch + 128);
  float* cv = reinterpret_cast<float*>(scratch + 256);
  int32_t* ct = reinterpret_cast<int32_t*>(cv + n_cand);
  int32_t* tmp = ct + n_cand;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = 0;
  if (cudaMemcpyAsync(pd, &p, sizeof(p), cudaMemcpyHostToDevice, st) != cudaSuccess || cudaMemcpyAsync(step, &t, 4, cudaMemcpyHostToDevice, st) != cudaSuccess) {
    set_error("vcla_op_beam_step: upload failed"); rc = -1;
  }
  if (rc == 0) rc = dec_beam_step(logits_dev, V, V, rows, history_dev, step, pd, t == 0 ? nullptr : run_scores_dev, cv, ct, st);
  if (rc == 0) rc = dec_beam_select(pd, B, R, V, step, cv, ct, history_dev, run_scores_dev, parent_dev, token_dev, hyp_scores_dev, hyp_lens_dev, hyp_fin_dev,
                                    hyp_tokens_dev, tmp, p.max_new, item_state_dev, cand_dev, st);
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == 0) { set_error("vcla_op_beam_step: %s", cudaGetErrorString(cudaGetLastError())); rc = -1; }
  cudaFree(scratch);
  return rc;
}

// -------------------------------------------------------------------------------------------------
// data parallel (SURVEY 8e): NCCL communicator owned by the context, token all-gather inside the decode graph
// -------------------------------------------------------------------------------------------------
int vcla_nccl_unique_id(uint8_t* out128) {
  if (!out128) { set_error("vcla_nccl_unique_id: null"); return -1; }
  if (nccl_api()) return -1;
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId id;
  VCLA_NCCL_OK(g_nccl.GetUniqueId(&id));
  memcpy(out128, &id, 128);
  return 0;
}

int vcla_nccl_init(vcla_ctx* c, const uint8_t* id128, int rank, int world, int width) {
  if (!c || !id128 || world < 1 || rank < 0 || rank >= world || width < 1 || width > 64) { set_error("vcla_nccl_init: bad arguments"); return -1; }
  if (c->comm) { set_error("vcla_nccl_init: context already has a communicator"); return -1; }
  if (nccl_api()) return -1;
  ncclUniqueId id;
  memcpy(&id, id128, 128);
  VCLA_NCCL_OK(g_nccl.CommInitRank(&c->comm, world, id, rank));
  c->dp_rank = rank; c->dp_world = world; c->dp_width = width;
  const size_t n_send = 64, n_recv = (size_t)world * 64, n_hist = (size_t)(c->cfg.max_seq + 2) * world * width;
  VCLA_CUDA_OK(cudaMalloc(&c->dp_send, (n_send + n_recv + n_hist + 4) * 4));
  VCLA_CUDA_OK(cudaMemset(c->dp_send, 0, (n_send + n_recv + n_hist + 4) * 4));
  c->dp_recv = c->dp_send + n_send; c->dp_hist = c->dp_recv + n_recv; c->dp_step = c->dp_hist + n_hist;
  VCLA_CUDA_OK(cudaStreamCreateWithFlags(&c->dp_stream, cudaStreamNonBlocking));
  VCLA_CUDA_OK(cudaEventCreateWithFlags(&c->dp_fork, cudaEventDisableTiming));
  VCLA_CUDA_OK(cudaEventCreateWithFlags(&c->dp_join, cudaEventDisableTiming));
  // graphs captured before the communicator existed do not contain the exchange
  return drop_graphs(c);
}

int vcla_allgather_tokens(vcla_ctx* c, const int32_t* local_dev, int n, int32_t* all_dev, vcla_stream stream) {
  if (!c || !c->comm) { set_error("vcla_allgather_tokens: call vcla_nccl_init first"); return -1; }
  if (!local_dev || !all_dev || n < 1) { set_error("vcla_allgather_tokens: bad arguments"); return -1; }
  VCLA_NCCL_OK(g_nccl.AllGather(local_dev, all_dev, (size_t)n, ncclInt32, c->comm, (cudaStream_t)stream));
  return 0;
}

int vcla_dp_set_active(vcla_ctx* c, int on) {
  // the exchange is part of prefill / decode only while active (every rank of the communicator must then make the same calls);
  // a rank-local generate() on a context that owns a communicator runs with it off
  if (!c) return -1;
  if (on && !c->comm) { set_error("vcla_dp_set_active: call vcla_nccl_init first"); return -1; }
  if (on && c->stream_armed) { set_error("vcla_dp_set_active: not available while token streaming is armed (vcla_stream_arm)"); return -1; }
  if (on && c->lk_on) { set_error("vcla_dp_set_active: not available while prompt lookup is set (vcla_set_lookup)"); return -1; }
  c->dp_active = on != 0;
  return 0;
}

int vcla_dp_exchange(vcla_ctx* c, vcla_stream stream) {
  // the exchange of one step without any compute: for a rank that holds no requests (global batch < world size)
  if (!c || !c->comm) { set_error("vcla_dp_exchange: call vcla_nccl_init first"); return -1; }
  return dp_gather(c, (cudaStream_t)stream, 0);
}

int vcla_read_history_dp(vcla_ctx* c, int32_t* dst_dev, int n_steps, vcla_stream stream) {
  // [n_steps][world * width] int32: the tokens every rank chose at the prefill (row 0) and each decode step since
  if (!c || !c->comm) { set_error("vcla_read_history_dp: call vcla_nccl_init first"); return -1; }
  if (n_steps < 0 || n_steps > c->cfg.max_seq + 1) { set_error("vcla_read_history_dp: bad arguments"); return -1; }
  VCLA_CUDA_OK(cudaMemcpyAsync(dst_dev, c->dp_hist, (size_t)n_steps * c->dp_world * c->dp_width * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

// -------------------------------------------------------------------------------------------------
// introspection + operator-level entry points
// -------------------------------------------------------------------------------------------------
int vcla_read_stage(vcla_ctx* c, const char* stage, int B, float* dst, vcla_stream stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const vcla_config& g = c->cfg;
  const float* src = nullptr; size_t n = 0;
  if (!strcmp(stage, "vit_out")) { src = c->v_hidden; n = (size_t)B * c->v_tokens * g.v_hidden; }
  else if (!strcmp(stage, "post_ln")) { src = c->v_postln_f32; n = (size_t)B * c->v_tokens * g.v_hidden; }
  else if (!strcmp(stage, "resampler_out")) { src = c->r_hidden; n = (size_t)B * g.r_queries * g.r_hidden; }
  else if (!strcmp(stage, "projector_out")) { src = c->img_embeds; n = (size_t)B * g.r_queries * g.t_hidden; }
  else if (!strcmp(stage, "step_logits")) { src = c->ws_lm; n = (size_t)B * g.t_vocab; }   // B <= 32 rows of the last one-split lm_head
  else if (!strcmp(stage, "lookup_tokens")) { src = reinterpret_cast<const float*>(c->lk_tok); n = (size_t)B; }   // int32 bits
  else { set_error("vcla_read_stage: unknown stage '%s'", stage); return -1; }
  VCLA_CUDA_OK(cudaMemcpyAsync(dst, src, n * 4, cudaMemcpyDeviceToHost, st));
  VCLA_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

int vcla_bench_decode_gemm(vcla_ctx* c, int which, int B, int reps, float* avg_us, int64_t* weight_bytes, vcla_stream stream) {
  // Times one decode weight-streaming GEMM shape over all layers' (distinct) weights, reps times, with CUDA events on
  // the launching stream.  13 GB of weights >> 126 MB L2, so every launch streams from HBM.
  cudaStream_t st = (cudaStream_t)stream;
  const vcla_config& g = c->cfg;
  if (B < 1 || B > 64 || which < 0 || which > 4 || reps < 1) { set_error("bench_decode_gemm: bad arguments"); return -1; }
  const int TH = g.t_hidden, F = g.t_ffn;
  cudaEvent_t e0, e1;
  VCLA_CUDA_OK(cudaEventCreate(&e0));
  VCLA_CUDA_OK(cudaEventCreate(&e1));
  const bool csk = which == DG_LM_HEAD ? lm_head_uses_csk(B) : decode_uses_csk(c, B);
  if (csk && csk_prepare(c, B)) return -1;
  auto run_all = [&]() -> int {
    const int layers = which == DG_LM_HEAD ? 1 : g.t_layers;
    for (int i = 0; i < layers; ++i) if (csk ? csk_gemm(c, which, i, B, st) : ws_gemm(c, which, i, B, st)) return -1;
    return 0;
  };
  if (run_all()) return -1;  // warm-up
  VCLA_CUDA_OK(cudaEventRecord(e0, st));
  for (int r = 0; r < reps; ++r) if (run_all()) return -1;
  VCLA_CUDA_OK(cudaEventRecord(e1, st));
  VCLA_CUDA_OK(cudaEventSynchronize(e1));
  float ms = 0.f;
  VCLA_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
  const int per = which == 4 ? 1 : g.t_layers;
  if (avg_us) *avg_us = ms * 1000.f / (float)(reps * per);
  if (weight_bytes) {
    const int64_t n[5] = {(int64_t)3 * TH * TH, (int64_t)TH * TH, (int64_t)2 * F * TH, (int64_t)TH * F, (int64_t)g.t_vocab * TH};
    const int64_t rows[5] = {(int64_t)3 * TH, TH, (int64_t)2 * F, TH, g.t_vocab};
    // int8 projections: one byte per weight + one fp32 scale per row
    *weight_bytes = (g.weight_format == 1 && which != DG_LM_HEAD) ? n[which] + rows[which] * 4 : n[which] * 2;
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  return 0;
}

int vcla_read_history(vcla_ctx* c, int32_t* dst_dev, int B, int n_steps, vcla_stream stream) {
  // tokens chosen by the prefill (step 0) and every decode step since, as a device [n_steps, B] int32 array
  if (n_steps < 0 || n_steps > c->cfg.max_seq + 1 || B < 1 || B > 64) { set_error("vcla_read_history: bad arguments"); return -1; }
  VCLA_CUDA_OK(cudaMemcpyAsync(dst_dev, c->tok_hist, (size_t)n_steps * B * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

// ---- token streaming: the ring is written by advance_seq_kernel (elementwise.cu) and read here ------------------------------------
static int stream_published(const vcla_ctx* c) { return __atomic_load_n(&c->ring_host->published, __ATOMIC_ACQUIRE); }

// 1 when every armed enqueue so far has completed, 0 when some is in flight, -1 on a device error
static int stream_drained(vcla_ctx* c) {
  if (!c->stream_pending) return 1;
  const cudaError_t e = cudaEventQuery(c->stream_done);
  if (e == cudaSuccess) { c->stream_pending = false; return 1; }
  if (e == cudaErrorNotReady) { (void)cudaGetLastError(); return 0; }
  set_error("token stream: device error %s", cudaGetErrorString(e));
  return -1;
}

int vcla_stream_arm(vcla_ctx* c, int on) {
  if (!c) return -1;
  if (!on) { c->stream_armed = false; return 0; }
  if (c->beam_on) { set_error("vcla_stream_arm: streaming is not available with beam search"); return -1; }
  if (c->dp_on()) { set_error("vcla_stream_arm: streaming is not available while the data-parallel token exchange is active"); return -1; }
  const int d = stream_drained(c);
  if (d < 0) return -1;
  if (d == 0) { set_error("vcla_stream_arm: armed work is still in flight (wait for it before arming again)"); return -1; }
  if (c->ring_host == nullptr) {
    const int rows = c->cfg.max_seq + 2;      // as many rows as the device token history
    void* p = nullptr;
    VCLA_CUDA_OK(cudaHostAlloc(&p, stream_ring_bytes(rows), cudaHostAllocMapped | cudaHostAllocPortable));
    memset(p, 0, stream_ring_bytes(rows));
    void* dp = nullptr;
    const cudaError_t e = cudaHostGetDevicePointer(&dp, p, 0);
    if (e == cudaSuccess && c->stream_done == nullptr) {
      const cudaError_t e2 = cudaEventCreateWithFlags(&c->stream_done, cudaEventDisableTiming);
      if (e2 != cudaSuccess) { cudaFreeHost(p); set_error("vcla_stream_arm: %s", cudaGetErrorString(e2)); return -1; }
    }
    if (e != cudaSuccess) { cudaFreeHost(p); set_error("vcla_stream_arm: %s", cudaGetErrorString(e)); return -1; }
    c->ring_host = (StreamRing*)p;
    c->ring_dev = (StreamRing*)dp;
    c->ring_host->rows = rows;
  }
  __atomic_store_n(&c->ring_host->published, 0, __ATOMIC_RELEASE);
  c->ring_host->epoch += 1;
  c->stream_armed = true;
  return 0;
}

int vcla_stream_wait(vcla_ctx* c, int target, int timeout_us, int* published) {
  if (!c || !c->ring_host) { set_error("vcla_stream_wait: streaming was never armed (vcla_stream_arm)"); return -1; }
  if (target < 0 || target > c->ring_host->rows) { set_error("vcla_stream_wait: target %d outside 0..%d", target, c->ring_host->rows); return -1; }
  const auto t0 = std::chrono::steady_clock::now();
  for (long it = 0;; ++it) {
    int p = stream_published(c);
    if (published) *published = p;
    if (p >= target) return 0;
    if (it < 4096 && (it & 63) != 63) continue;          // spin briefly: a step at 7B widths is a few milliseconds
    const int d = stream_drained(c);
    if (d < 0) return -1;
    if (d == 1) {
      p = stream_published(c);                             // the event completed after the last publish: read the count again
      if (published) *published = p;
      if (p >= target) return 0;
      set_error("vcla_stream_wait: step %d will never be published: all armed work has completed with %d steps published", target, p);
      return -1;
    }
    if (timeout_us >= 0 &&
        std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count() >= timeout_us)
      return 0;
    if (it >= 4096) std::this_thread::sleep_for(std::chrono::microseconds(20));
  }
}

int vcla_stream_read(vcla_ctx* c, int from, int to, int B, int32_t* dst_host) {
  if (!c || !c->ring_host) { set_error("vcla_stream_read: streaming was never armed (vcla_stream_arm)"); return -1; }
  const int p = stream_published(c);
  if (from < 0 || to < from || to > p || B < 1 || B > 64 || (to > from && !dst_host)) {
    set_error("vcla_stream_read: steps [%d, %d) x %d not within the %d published steps", from, to, B, p);
    return -1;
  }
  for (int s = from; s < to; ++s) memcpy(dst_host + (size_t)(s - from) * B, c->ring_host->tokens + (size_t)s * 64, (size_t)B * 4);
  return 0;
}

int vcla_trace_enable(vcla_ctx* c, int max_events) {
  // installs (max_events > 0) or removes (0) the timeline buffer every kernel's CTA 0 appends to
  VCLA_CUDA_OK(cudaDeviceSynchronize());
  if (c->trace_buf) { trace_set_all(nullptr, 0); cudaFree(c->trace_buf); c->trace_buf = nullptr; c->trace_cap = 0; }
  if (max_events <= 0) return 0;
  const size_t bytes = 8 + (size_t)max_events * 32;
  VCLA_CUDA_OK(cudaMalloc(&c->trace_buf, bytes));
  VCLA_CUDA_OK(cudaMemset(c->trace_buf, 0, bytes));
  c->trace_cap = (unsigned long long)max_events;
  if (trace_set_all(c->trace_buf, c->trace_cap)) {
    set_error("vcla_trace_enable: cudaMemcpyToSymbol failed");
    return -1;
  }
  return 0;
}
int vcla_trace_read(vcla_ctx* c, uint64_t* dst_host, int max_events, int* n_events) {
  // copies [tag, t_entry_ns, t_dep_ns, t_exit_ns] x n to the host and clears the buffer.  Synchronises.
  if (!c->trace_buf) { set_error("vcla_trace_read: tracing is off"); return -1; }
  VCLA_CUDA_OK(cudaDeviceSynchronize());
  unsigned long long cnt = 0;
  VCLA_CUDA_OK(cudaMemcpy(&cnt, c->trace_buf, 8, cudaMemcpyDeviceToHost));
  if (cnt > c->trace_cap) cnt = c->trace_cap;
  if (cnt > (unsigned long long)max_events) cnt = (unsigned long long)max_events;
  VCLA_CUDA_OK(cudaMemcpy(dst_host, (uint8_t*)c->trace_buf + 8, cnt * 32, cudaMemcpyDeviceToHost));
  VCLA_CUDA_OK(cudaMemset(c->trace_buf, 0, 8));
  if (n_events) *n_events = (int)cnt;
  return 0;
}

int vcla_op_gemm(const void* A, const void* W, int M, int N, int K, int mode, int act, int accumulate, const float* bias, void* out,
                 int ldo, int splits, int tile_n, int use_reference, vcla_stream stream) {
  GemmCall g;
  g.A = (const bf16*)A; g.B = (const bf16*)W; g.M = M; g.N = N; g.K = K; g.lda = K; g.ldb = K; g.mode = mode; g.act = act; g.accumulate = accumulate;
  g.bias = bias; g.out = out; g.ldo = ldo; g.splits = splits; g.ws_rows = N; g.bn = tile_n; g.weights_are_A = (mode == GEMM_PARTIAL_F32);
  return use_reference ? gemm_naive(g, (cudaStream_t)stream) : gemm_tc(g, (cudaStream_t)stream);
}
int vcla_op_gemm_csk(const void* W, const void* X, int M, int B, int K, int splits, int mode, float* out_or_resid, const float* norm_w, void* xw_or_h,
                     float* ssq_out, const float* ssq_in, int ssq_slots, float inv_dim, float eps, vcla_stream stream) {
  CskCall k; k.W = (const bf16*)W; k.X = (const bf16*)X; k.M = M; k.B = B; k.K = K; k.splits = splits; k.mode = mode;
  k.ssq_in = ssq_in; k.ssq_slots = ssq_slots; k.inv_dim = inv_dim; k.eps = eps;
  if (mode == CSK_OUT_F32) { k.out = out_or_resid; k.ldo = M; }
  else if (mode == CSK_RESID) { k.resid = out_or_resid; k.norm_w = norm_w; k.xw = (bf16*)xw_or_h; k.ssq_out = ssq_out; }
  else if (mode == CSK_SWIGLU) { k.h = (bf16*)xw_or_h; }
  else { set_error("vcla_op_gemm_csk: unknown mode %d", mode); return -1; }
  return gemm_csk(k, (cudaStream_t)stream);
}
int vcla_op_gemm_csk_q8(const int8_t* Wq, const float* wscale, const void* X, int M, int B, int K, int splits, int mode, float* out_or_resid,
                        const float* norm_w, void* xw_or_h, float* ssq_out, const float* ssq_in, int ssq_slots, float inv_dim, float eps,
                        vcla_stream stream) {
  // caller rows are in logical order: put them into the stored (fragment) order in a scratch, run, free.  Synchronises.
  if (!Wq || !wscale || !X || M < 1 || K < 1) { set_error("vcla_op_gemm_csk_q8: bad arguments"); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t qbytes = align_up((size_t)M * K, 256);
  uint8_t* scratch = nullptr;
  VCLA_CUDA_OK(cudaMalloc(&scratch, qbytes + (size_t)M * 4));
  CskCall k; k.Wq = (const int8_t*)scratch; k.wscale = (const float*)(scratch + qbytes); k.X = (const bf16*)X; k.M = M; k.B = B; k.K = K;
  k.splits = splits; k.mode = mode; k.ssq_in = ssq_in; k.ssq_slots = ssq_slots; k.inv_dim = inv_dim; k.eps = eps;
  int rc = 0;
  if (mode == CSK_OUT_F32) { k.out = out_or_resid; k.ldo = M; }
  else if (mode == CSK_RESID) { k.resid = out_or_resid; k.norm_w = norm_w; k.xw = (bf16*)xw_or_h; k.ssq_out = ssq_out; }
  else if (mode == CSK_SWIGLU) { k.h = (bf16*)xw_or_h; }
  else { set_error("vcla_op_gemm_csk_q8: unknown mode %d", mode); rc = -1; }
  if (rc == 0) rc = place_rows_q8(Wq, wscale, M, K, -1, (int8_t*)scratch, (float*)(scratch + qbytes), st);
  if (rc == 0) rc = gemm_csk(k, st);
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == 0) { set_error("vcla_op_gemm_csk_q8: %s", cudaGetErrorString(cudaGetLastError())); rc = -1; }
  cudaFree(scratch);
  return rc;
}
int vcla_op_gemm_q8(const void* A, const int8_t* Wq, const float* wscale, int M, int N, int K, int mode, int accumulate, void* out, int ldo,
                    const float* norm_w, void* xw, float* ssq_out, vcla_stream stream) {
  // bf16(q) of the caller's logical rows into a scratch, then the prefill GEMM with the row scales as column scales.  Synchronises.
  if (!A || !Wq || !wscale || !out || M < 1 || N < 1 || K < 1) { set_error("vcla_op_gemm_q8: bad arguments"); return -1; }
  if (mode != GEMM_STORE_BF16 && mode != GEMM_ADD_F32 && mode != GEMM_SWIGLU_BF16) { set_error("vcla_op_gemm_q8: unknown mode %d", mode); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  bf16* wide = nullptr;
  VCLA_CUDA_OK(cudaMalloc(&wide, (size_t)N * K * 2));
  GemmCall g; g.A = (const bf16*)A; g.B = wide; g.M = M; g.N = N; g.K = K; g.lda = K; g.ldb = K; g.mode = mode; g.accumulate = accumulate;
  g.out = out; g.ldo = ldo; g.colscale = wscale;
  if (norm_w != nullptr) { g.emit.norm_w = norm_w; g.emit.xw = (bf16*)xw; g.emit.ldxw = N; g.emit.ssq_out = ssq_out; }
  int rc = expand_rows_q8(Wq, N, K, 0, wide, st);
  if (rc == 0) rc = gemm_tc(g, st);
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == 0) { set_error("vcla_op_gemm_q8: %s", cudaGetErrorString(cudaGetLastError())); rc = -1; }
  cudaFree(wide);
  return rc;
}
int vcla_debug_set_csk_splits(vcla_ctx* c, int B, int qkv, int o, int gu, int d, int lm) {
  // tuning hook: CTAs per cluster of the five decode GEMM shapes at batch B (0 = keep the automatic choice); drops the captured graphs.
  // Batches 33..64 run the cluster schedule only with int8 projections, whose lm_head then is the workspace GEMM (lm is ignored).
  if (!c || B < 1 || B > csk_max_batch(c)) { set_error("vcla_debug_set_csk_splits: bad arguments"); return -1; }
  c->csk_batch = 0;
  if (csk_prepare(c, B)) return -1;
  int* dst[5] = {&c->csk_qkv, &c->csk_o, &c->csk_gu, &c->csk_d, &c->csk_lm};
  const int v[5] = {qkv, o, gu, d, lm};
  for (int i = 0; i < 5; ++i) if (v[i] >= 1 && v[i] <= 8) *dst[i] = v[i];
  return drop_graphs(c);
}
int vcla_debug_get_csk_splits(vcla_ctx* c, int B, int* out5) {
  if (!c || !out5 || B < 1 || B > csk_max_batch(c)) return -1;
  if (c->csk_batch != B && csk_prepare(c, B)) return -1;
  out5[0] = c->csk_qkv; out5[1] = c->csk_o; out5[2] = c->csk_gu; out5[3] = c->csk_d; out5[4] = c->csk_lm;
  return 0;
}
int vcla_debug_decode_ctas_per_sm(vcla_ctx* c, int B, int* out2) {
  if (!c || !out2 || B < 1 || B > csk_max_batch(c)) { set_error("vcla_debug_decode_ctas_per_sm: bad arguments"); return -1; }
  out2[0] = gemm_csk_ctas_per_sm(B, c->cfg.weight_format == 1);
  out2[1] = attention_decode_ctas_per_sm(decode_attn_call(c, 0, B, 1), c->kv_format());
  return out2[0] > 0 && out2[1] > 0 ? 0 : -1;
}
int vcla_op_gemm_csk_clusters(int B, int splits) { return gemm_csk_clusters(B, splits); }
void vcla_set_attention_tc(int on) { attention_set_tc(on); }
int vcla_op_attention(const void* q, int q_stride, const void* k0, const void* v0, int kv0_stride, int n0, const void* k1, const void* v1,
                      int kv1_stride, int n1, void* out, int o_stride, int B, int H, int Sq, int HD, float scale, int causal, vcla_stream stream,
                      const int32_t* kv_start_dev) {
  // operator entry for tests: the left padding is read back and checked before the launch.  Synchronises.
  if (!q || !k0 || !v0 || !out || (n1 > 0 && (!k1 || !v1)) || B < 1 || H < 1 || Sq < 1 || n0 < 0 || n1 < 0) {
    set_error("vcla_op_attention: bad arguments"); return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (kv_start_dev) {
    std::vector<int32_t> kv_start((size_t)B);
    VCLA_CUDA_OK(cudaStreamSynchronize(st));
    VCLA_CUDA_OK(cudaMemcpy(kv_start.data(), kv_start_dev, kv_start.size() * 4, cudaMemcpyDeviceToHost));
    for (int b = 0; b < B; ++b) {
      if (kv_start[b] < 0 || kv_start[b] > n0 + n1) {
        set_error("vcla_op_attention: kv_start[%d] = %d outside [0, %d]", b, kv_start[b], n0 + n1); return -1;
      }
    }
  }
  AttnCall a; a.q = (const bf16*)q; a.q_stride = q_stride; a.k0 = (const bf16*)k0; a.v0 = (const bf16*)v0; a.kv0_stride = kv0_stride; a.n0 = n0;
  a.k1 = (const bf16*)k1; a.v1 = (const bf16*)v1; a.kv1_stride = kv1_stride; a.n1 = n1; a.out = (bf16*)out; a.o_stride = o_stride;
  a.B = B; a.H = H; a.Sq = Sq; a.HD = HD; a.scale = scale; a.causal = causal; a.kv_start = kv_start_dev;
  int rc = attention_prefill(a, st);
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == 0) { set_error("vcla_op_attention: %s", cudaGetErrorString(cudaGetLastError())); rc = -1; }
  return rc;
}
// Operator entries on a caller's pool: read back the page table [B][kv.pages_per_seq] and the lengths len_dev [B] (synchronising st) and
// refuse, before any launch, a length below 0, a sequence whose len + rows tokens do not fit its table row, and a negative page among
// the entries the launch reads.  Raises kv.total_pages to the pool extent (largest page read + 1).  -> the longest length, -1 if refused.
static int op_check_pages(const char* who, KvPool& kv, const int32_t* len_dev, int B, int rows, cudaStream_t st) {
  std::vector<int32_t> table((size_t)B * kv.pages_per_seq), len((size_t)B);
  VCLA_CUDA_OK(cudaStreamSynchronize(st));
  VCLA_CUDA_OK(cudaMemcpy(table.data(), kv.table, table.size() * 4, cudaMemcpyDeviceToHost));
  VCLA_CUDA_OK(cudaMemcpy(len.data(), len_dev, len.size() * 4, cudaMemcpyDeviceToHost));
  int longest = 0;
  for (int b = 0; b < B; ++b) {
    if (len[b] < 0 || (int64_t)len[b] + rows > (int64_t)kv.pages_per_seq * kv.page_tokens) {
      set_error("%s: sequence %d (%d + %d tokens) exceeds its table row (%d pages of %d)", who, b, len[b], rows, kv.pages_per_seq, kv.page_tokens);
      return -1;
    }
    for (int i = 0; i < kv.pages_for(len[b] + rows); ++i) {
      const int32_t page = table[(size_t)b * kv.pages_per_seq + i];
      if (page < 0) { set_error("%s: sequence %d has no page %d", who, b, i); return -1; }
      kv.total_pages = std::max(kv.total_pages, page + 1);
    }
    longest = std::max(longest, len[b]);
  }
  return longest;
}
static KvPool op_pool(const void* pages, const int32_t* table, int pages_per_seq, int page_tokens, int heads) {
  KvPool kv; kv.pages = (bf16*)pages; kv.table = const_cast<int32_t*>(table);
  kv.heads = heads; kv.page_tokens = page_tokens; kv.pages_per_seq = pages_per_seq;
  return kv;
}

// int8 pools: the caller's total_pages places the scale region, so every page the call reads must lie below it
static int op_check_q8_extent(const char* who, KvFormat fmt, const KvPool& kv, int total_pages) {
  if (fmt == KV_INT8 && kv.total_pages > total_pages) {
    set_error("%s: page %d is outside the %d-page int8 pool", who, kv.total_pages - 1, total_pages); return -1;
  }
  return 0;
}
static int op_attention_paged(KvFormat fmt, const void* q, int q_stride, const void* kv_pages, int total_pages, const int32_t* page_table,
                              int pages_per_seq, int page_tokens, const int32_t* base_len_dev, void* out, int o_stride, int B, int H, int T,
                              float scale, vcla_stream stream) {
  // operator entry for tests: the pool extent (bf16) and the longest sequence are read back from the caller's table and lengths, the
  // split-KV scratch is allocated for the call.  Synchronises.
  if (!q || !kv_pages || !page_table || !base_len_dev || !out || B < 1 || B > 64 || H < 1 || T < 1 || pages_per_seq < 1 ||
      (fmt == KV_INT8 && total_pages < 1)) {
    set_error("vcla_op_attention_paged: bad arguments"); return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  KvPool kv = op_pool(kv_pages, page_table, pages_per_seq, page_tokens, H);
  const int longest = op_check_pages("vcla_op_attention_paged", kv, base_len_dev, B, T, st);
  if (longest < 0 || op_check_q8_extent("vcla_op_attention_paged", fmt, kv, total_pages)) return -1;
  if (fmt == KV_INT8) kv.total_pages = total_pages;
  const int n = attention_paged_partials();
  void* scratch = nullptr;
  VCLA_CUDA_OK(cudaMalloc(&scratch, (size_t)n * kAttnPartialFloats * 4 + (size_t)n * 4));
  int32_t* counters = reinterpret_cast<int32_t*>(reinterpret_cast<float*>(scratch) + (size_t)n * kAttnPartialFloats);
  AttnPagedCall a; a.q = (const bf16*)q; a.q_stride = q_stride; a.kv = kv; a.base_len = base_len_dev; a.max_kv = longest + T;
  a.out = (bf16*)out; a.o_stride = o_stride; a.B = B; a.T = T; a.scale = scale; a.part = reinterpret_cast<float*>(scratch); a.counters = counters;
  int rc = cudaMemsetAsync(counters, 0, (size_t)n * 4, st) == cudaSuccess ? attention_paged(a, st, fmt) : -1;
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == 0) { set_error("vcla_op_attention_paged: %s", cudaGetErrorString(cudaGetLastError())); rc = -1; }
  cudaFree(scratch);
  return rc;
}
int vcla_op_attention_paged(const void* q, int q_stride, const void* kv_pages, const int32_t* page_table, int pages_per_seq, int page_tokens,
                            const int32_t* base_len_dev, void* out, int o_stride, int B, int H, int T, float scale, vcla_stream stream) {
  return op_attention_paged(KV_BF16, q, q_stride, kv_pages, 0, page_table, pages_per_seq, page_tokens, base_len_dev, out, o_stride, B, H, T,
                            scale, stream);
}
int vcla_op_attention_paged_q8(const void* q, int q_stride, const void* kv_pool, int total_pages, const int32_t* page_table, int pages_per_seq,
                               int page_tokens, const int32_t* base_len_dev, void* out, int o_stride, int B, int H, int T, float scale,
                               vcla_stream stream) {
  return op_attention_paged(KV_INT8, q, q_stride, kv_pool, total_pages, page_table, pages_per_seq, page_tokens, base_len_dev, out, o_stride, B,
                            H, T, scale, stream);
}
static int op_attention_decode(KvFormat fmt, const float* qkv_partial, int splits, void* kv_pages, int total_pages, const int32_t* page_table,
                               int pages_per_seq, int page_tokens, const int32_t* seq_len_dev, void* out, int B, int H, int kv_splits, float scale,
                               float rope_theta, int persistent, int persistent_grid, int launches, vcla_stream stream) {
  // operator entry for tests: goes through attention_decode() (the dispatch is under test too); the RoPE tables, the combine scratch
  // and the arrival counters are made for the call.  Everything a kernel would index with is checked here first.  Synchronises.
  if (!qkv_partial || !kv_pages || !page_table || !seq_len_dev || !out || splits < 1 || B < 1 || B > 64 || H < 1 || pages_per_seq < 1 ||
      page_tokens < 1 || launches < 1 || persistent_grid < 0 || !(rope_theta > 0.f) || (fmt == KV_INT8 && total_pages < 1)) {
    set_error("vcla_op_attention_decode: bad arguments"); return -1;
  }
  if (kv_splits < 1 || kv_splits > 8) { set_error("vcla_op_attention_decode: kv_splits %d outside 1..8", kv_splits); return -1; }
  if (persistent != 0 && persistent != 1) { set_error("vcla_op_attention_decode: persistent must be 0 or 1"); return -1; }
  if (persistent && kv_splits != 1) { set_error("vcla_op_attention_decode: the persistent kernel requires kv_splits == 1 (got %d)", kv_splits); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  KvPool kv = op_pool(kv_pages, page_table, pages_per_seq, page_tokens, H);
  const int max_len = op_check_pages("vcla_op_attention_decode", kv, seq_len_dev, B, 1, st);
  if (max_len < 0 || op_check_q8_extent("vcla_op_attention_decode", fmt, kv, total_pages)) return -1;
  if (fmt == KV_INT8) kv.total_pages = total_pages;
  const size_t rope_floats = (size_t)(max_len + 1) * 64, scratch_floats = (size_t)B * H * kv_splits * (128 + 2);
  float* buf = nullptr;
  VCLA_CUDA_OK(cudaMalloc(&buf, (2 * rope_floats + scratch_floats + (size_t)B * H) * 4));
  DecodeAttnCall a; a.qkv_partial = qkv_partial; a.splits = splits; a.ws_rows = B; a.kv = kv;
  a.seq_len = seq_len_dev; a.out = (bf16*)out; a.B = B; a.HD = 128;
  a.kv_splits = kv_splits; a.scale = scale; a.rope_theta = rope_theta; a.rope_cos = buf; a.rope_sin = buf + rope_floats;
  a.scratch = buf + 2 * rope_floats; a.counters = reinterpret_cast<int32_t*>(a.scratch + scratch_floats);
  a.persistent_mode = persistent ? 2 : 0; a.persistent_grid = persistent_grid;
  int rc = rope_fill_tables(max_len + 1, 128, rope_theta, buf, buf + rope_floats);
  if (rc == 0 && cudaMemsetAsync(a.scratch, 0, (scratch_floats + (size_t)B * H) * 4, st) != cudaSuccess) { set_error("vcla_op_attention_decode: memset failed"); rc = -1; }
  // every launch runs over the same scratch and counters, as the replays of a decode graph do; out is NaN before each, so an
  // element the last launch did not write cannot pass for one an earlier launch wrote
  for (int i = 0; i < launches && rc == 0; ++i) {
    if (cudaMemsetAsync(out, 0xff, (size_t)B * H * 128 * 2, st) != cudaSuccess) { set_error("vcla_op_attention_decode: memset failed"); rc = -1; break; }
    rc = attention_decode(a, st, fmt);
  }
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == 0) { set_error("vcla_op_attention_decode: %s", cudaGetErrorString(cudaGetLastError())); rc = -1; }
  cudaFree(buf);
  return rc;
}
int vcla_op_attention_decode(const float* qkv_partial, int splits, void* kv_pages, const int32_t* page_table, int pages_per_seq, int page_tokens,
                             const int32_t* seq_len_dev, void* out, int B, int H, int kv_splits, float scale, float rope_theta, int persistent,
                             int persistent_grid, int launches, vcla_stream stream) {
  return op_attention_decode(KV_BF16, qkv_partial, splits, kv_pages, 0, page_table, pages_per_seq, page_tokens, seq_len_dev, out, B, H, kv_splits,
                             scale, rope_theta, persistent, persistent_grid, launches, stream);
}
int vcla_op_attention_decode_q8(const float* qkv_partial, int splits, void* kv_pool, int total_pages, const int32_t* page_table, int pages_per_seq,
                                int page_tokens, const int32_t* seq_len_dev, void* out, int B, int H, int kv_splits, float scale, float rope_theta,
                                int persistent, int persistent_grid, int launches, vcla_stream stream) {
  return op_attention_decode(KV_INT8, qkv_partial, splits, kv_pool, total_pages, page_table, pages_per_seq, page_tokens, seq_len_dev, out, B, H,
                             kv_splits, scale, rope_theta, persistent, persistent_grid, launches, stream);
}
static int op_attention_decode_lookup(KvFormat fmt, const float* qkv_partial, int splits, void* kv_pages, int total_pages, const int32_t* page_table,
                                      int pages_per_seq, int page_tokens, const int32_t* seq_len_dev, void* out, int rows, int H, int kv_splits,
                                      float scale, float rope_theta, vcla_stream stream) {
  // operator entry for tests: attention_decode_lookup on caller buffers; the RoPE tables, scratch and counters are made for the call.
  if (!qkv_partial || !kv_pages || !page_table || !seq_len_dev || !out || splits < 1 || rows < 2 || rows > 16 || H < 1 || pages_per_seq < 1 ||
      page_tokens < 1 || !(rope_theta > 0.f) || (fmt == KV_INT8 && total_pages < 1)) {
    set_error("vcla_op_attention_decode_lookup: bad arguments"); return -1;
  }
  if (kv_splits < 1 || kv_splits > 8) { set_error("vcla_op_attention_decode_lookup: kv_splits %d outside 1..8", kv_splits); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  KvPool kv = op_pool(kv_pages, page_table, pages_per_seq, page_tokens, H);
  const int len = op_check_pages("vcla_op_attention_decode_lookup", kv, seq_len_dev, 1, rows, st);
  if (len < 0 || op_check_q8_extent("vcla_op_attention_decode_lookup", fmt, kv, total_pages)) return -1;
  if (fmt == KV_INT8) kv.total_pages = total_pages;
  const size_t rope_floats = (size_t)(len + rows) * 64, scratch_floats = (size_t)rows * H * kv_splits * (128 + 2);
  float* buf = nullptr;
  VCLA_CUDA_OK(cudaMalloc(&buf, (2 * rope_floats + scratch_floats + (size_t)rows * H) * 4));
  DecodeAttnCall a; a.qkv_partial = qkv_partial; a.splits = splits; a.ws_rows = rows; a.kv = kv;
  a.seq_len = seq_len_dev; a.out = (bf16*)out; a.B = rows; a.HD = 128;
  a.kv_splits = kv_splits; a.scale = scale; a.rope_theta = rope_theta; a.rope_cos = buf; a.rope_sin = buf + rope_floats;
  a.scratch = buf + 2 * rope_floats; a.counters = reinterpret_cast<int32_t*>(a.scratch + scratch_floats);
  int rc = rope_fill_tables(len + rows, 128, rope_theta, buf, buf + rope_floats);
  if (rc == 0 && cudaMemsetAsync(a.scratch, 0, (scratch_floats + (size_t)rows * H) * 4, st) != cudaSuccess) { set_error("vcla_op_attention_decode_lookup: memset failed"); rc = -1; }
  if (rc == 0) rc = attention_decode_lookup(a, st, fmt);
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == 0) { set_error("vcla_op_attention_decode_lookup: %s", cudaGetErrorString(cudaGetLastError())); rc = -1; }
  cudaFree(buf);
  return rc;
}
int vcla_op_attention_decode_lookup(const float* qkv_partial, int splits, void* kv_pages, const int32_t* page_table, int pages_per_seq,
                                    int page_tokens, const int32_t* seq_len_dev, void* out, int rows, int H, int kv_splits, float scale,
                                    float rope_theta, vcla_stream stream) {
  return op_attention_decode_lookup(KV_BF16, qkv_partial, splits, kv_pages, 0, page_table, pages_per_seq, page_tokens, seq_len_dev, out, rows, H,
                                    kv_splits, scale, rope_theta, stream);
}
int vcla_op_attention_decode_lookup_q8(const float* qkv_partial, int splits, void* kv_pool, int total_pages, const int32_t* page_table,
                                       int pages_per_seq, int page_tokens, const int32_t* seq_len_dev, void* out, int rows, int H, int kv_splits,
                                       float scale, float rope_theta, vcla_stream stream) {
  return op_attention_decode_lookup(KV_INT8, qkv_partial, splits, kv_pool, total_pages, page_table, pages_per_seq, page_tokens, seq_len_dev, out,
                                    rows, H, kv_splits, scale, rope_theta, stream);
}
int vcla_op_logits_argmax(const float* partial, int splits, int ldp, int B, int V, float* logits_out, int32_t* tok_out, vcla_stream stream) {
  // operator entry for tests: dec_logits_argmax without token history or data-parallel send buffer.  Synchronises.
  if (!partial || !tok_out || splits < 1 || B < 1 || V < 1 || ldp < V) { set_error("vcla_op_logits_argmax: bad arguments"); return -1; }
  cudaStream_t st = (cudaStream_t)stream;
  float* cand = nullptr;
  VCLA_CUDA_OK(cudaMalloc(&cand, (size_t)B * kArgmaxChunks * 8));
  int rc = dec_logits_argmax(partial, splits, B, ldp, B, V, logits_out, V, tok_out, nullptr, nullptr, cand,
                             reinterpret_cast<int32_t*>(cand + (size_t)B * kArgmaxChunks), nullptr, st);
  if (cudaStreamSynchronize(st) != cudaSuccess && rc == 0) { set_error("vcla_op_logits_argmax: %s", cudaGetErrorString(cudaGetLastError())); rc = -1; }
  cudaFree(cand);
  return rc;
}
int vcla_op_layernorm(const float* x, int rows, int D, const float* w, const float* b, float eps, void* y_bf16, float* y_f32, vcla_stream stream) {
  return layernorm(x, rows, D, w, b, eps, (bf16*)y_bf16, y_f32, (cudaStream_t)stream);
}
int vcla_op_rmsnorm(const float* x, int rows, int D, const float* w, float eps, void* y_bf16, vcla_stream stream) {
  return rmsnorm(x, rows, D, w, eps, (bf16*)y_bf16, (cudaStream_t)stream);
}

}  // extern "C"
