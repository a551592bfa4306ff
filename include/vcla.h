/*
 * vcla.h -- C ABI of the H100-native VisualCLA multimodal forward path (libvcla.so).
 *
 * This is the drop-in boundary for ONE hot path of airaria/Visual-Chinese-LLaMA-Alpaca:
 *   image + prompt -> CLIP-ViT-L/14 -> post_layernorm -> 6-layer Resampler -> projector
 *   -> splice into the text embeddings -> LLaMA-7B prefill + KV-cache greedy decode.
 * The reference is pure Python and has no FFI of its own (SURVEY.md section 8b); each entry point
 * below names the reference code it replaces (paths relative to the reference repo root, `HF:` =
 * transformers 5.5.0).  The Python package `visualcla` (visual-chinese-llama-alpaca_b200/visualcla)
 * binds these with ctypes and exposes the reference's own API (VisualCLAModel.generate/.forward,
 * chat, get_model_and_tokenizer_and_processor).  See INTEGRATION.md for the binding stub.
 *
 * Conventions: plain pointers and sizes, no torch / C++ types; every function returns 0 on success,
 * non-zero on failure with a message retrievable through vcla_last_error() (thread-local); nothing
 * throws across the ABI.  "dev" pointers are CUDA device pointers on the context's device; the
 * library never frees caller memory.  One context per GPU, calls externally serialised.  Every call
 * that takes a `stream` only enqueues work on it (no host synchronisation) unless documented.
 */
#ifndef VCLA_H_
#define VCLA_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vcla_ctx vcla_ctx;
typedef void* vcla_stream; /* cudaStream_t */

/* element types of caller buffers */
enum { VCLA_F32 = 0, VCLA_F16 = 1, VCLA_BF16 = 2 };

/* image layouts of the prompt (models/visualcla/modeling_visualcla.py:290-305 / :356-370) */
enum {
  VCLA_TEXT_ONLY = 0,       /* pixel_values=None: multimodal_embeds = input_embeds (:378-380) */
  VCLA_IMAGE_AT_HEAD = 1,   /* [e0,e1, img x nq, e2...]  (:291/:357); S = T + nq */
  VCLA_IMAGE_PLACEHOLDER = 2 /* image rows replace the nq <img_token> slots after <img> (:293-305); S = T */
};

/* Shapes of the path.  Mirrors VisualCLAConfig / VisualResamplerConfig / the HF CLIP + LLaMA configs
 * (models/visualcla/configuration_visualcla.py:10-39, modeling_visual_resampler.py:90-129). */
typedef struct {
  /* CLIP-ViT (HF:models/clip/modeling_clip.py) */
  int v_hidden, v_layers, v_heads, v_ffn, v_patch, v_image;
  float v_eps;
  /* Resampler (models/visualcla/modeling_visual_resampler.py) */
  int r_hidden, r_layers, r_heads, r_ffn, r_queries;
  float r_eps;
  /* LLaMA (HF:models/llama/modeling_llama.py) */
  int t_hidden, t_layers, t_heads, t_ffn, t_vocab;
  float t_eps, rope_theta;
  /* capacity of this context */
  int max_batch;           /* sequences resident at once (per GPU) */
  int max_seq;             /* prompt + generated tokens per sequence */
  int max_prefill_tokens;  /* max B*S of one prefill call */
  int page_tokens;         /* tokens per KV-cache page (default 64 if 0) */
  /* storage of the LLaMA projections: 0 = bf16 (default), 1 = weight-only int8 (load_in_8bit, below) */
  int weight_format;
  /* storage of the paged KV cache: 0 = bf16 (default), 1 = int8 rows + one fp32 scale per row (kv_cache_dtype="int8", below) */
  int kv_format;
} vcla_config;

const char* vcla_last_error(void);
const char* vcla_version(void);

/* ---- lifetime -------------------------------------------------------------------------------- */
/* Allocates the weight arena, paged KV cache and activation buffers on the current CUDA device.
 * Replaces model construction: VisualCLAModel.__init__ (modeling_visualcla.py:70-108). */
int vcla_create(const vcla_config* cfg, vcla_ctx** out);
void vcla_destroy(vcla_ctx* ctx);
int vcla_get_config(const vcla_ctx* ctx, vcla_config* out);
/* bytes of device memory held by the context (weights, kv, activations) */
int vcla_memory_bytes(const vcla_ctx* ctx, int64_t* weights, int64_t* kv, int64_t* activations);

/* ---- weights ---------------------------------------------------------------------------------- */
/* The logical tensors are addressed by the reference's own state-dict names
 * (VisualCLAModel.state_dict(): "vision_model.vision_model.*", "visual_resampler.*",
 * "image_projection_layer.*", "text_model.model.*", "text_model.lm_head.weight"; merged checkpoint
 * layout scripts/merge_llama_with_visualcla_lora.py:92-97, read back at modeling_visualcla.py:141-179). */
int vcla_weight_count(const vcla_ctx* ctx);
/* kind: 0 = matrix stored bf16, 1 = vector/table stored f32.  shape has up to 4 dims. */
int vcla_weight_info(const vcla_ctx* ctx, int index, const char** name, int64_t shape[4], int* ndim, int* kind);
/* Copy + repack one tensor into the arena (fused QKV, gate/up interleave, K padding).  `src` is a host
 * pointer (on_device = 0) or device pointer (on_device = 1) to the contiguous tensor in `dtype` holding `numel`
 * elements; the call fails (nothing is read) unless numel equals the element count of the named tensor, so a
 * checkpoint whose shape disagrees with the config is an error, never an out-of-bounds read.
 * Replaces from_merged_pretrained's loading (modeling_visualcla.py:120-181).  Synchronises the stream. */
int vcla_load_weight(vcla_ctx* ctx, const char* name, const void* src, int dtype, int64_t numel, int on_device,
                     vcla_stream stream);
/* Copy one logical tensor back to host: bf16 for kind 0, f32 for kind 1 (state_dict() equivalent). */
int vcla_read_weight(vcla_ctx* ctx, const char* name, void* dst_host, vcla_stream stream);
/* Deterministic synthetic weights: w = mean + std * IrwinHall4(hash(name, seed, index)), bit-identical
 * to oracle/visualcla_oracle.py:hash_normal_bf16 (std/mean per tensor as in oracle weight_specs).  With weight_format 1 the
 * int8 tensors are quantised from these bf16 values. */
int vcla_init_synthetic(vcla_ctx* ctx, uint32_t seed, vcla_stream stream);

/* ---- load_in_8bit: weight-only int8 LLaMA projections (weight_format 1) -------------------------------------------------------
 * The reference passes load_in_8bit only to LlamaForCausalLM.from_pretrained (models/visualcla/modeling_visualcla.py:151-156,
 * :242-247), where bitsandbytes replaces the seven nn.Linear of every LLaMA layer (q, k, v, o, gate, up, down); embed_tokens,
 * lm_head, the norms, CLIP, the Resampler and the projector stay as they are.  Here those seven tensors are stored as int8 rows with
 * one fp32 scale per row (kind 2 in vcla_weight_info): a = max|w_row| in fp32, s = a / 127, q = clamp(rint(w * (127 / a)), -127, 127)
 * (half to even; a zero row gives s = 0, q = 0), w = the source values in fp32.  The effective weight is q * s; activations stay
 * bf16 with fp32 accumulation.  This is the weight half of LLM.int8 only (no activation-outlier decomposition), so results are not
 * bit-equal to bitsandbytes.  vcla_load_weight quantises on the device; vcla_read_weight returns fp32 q * s for kind 2.
 *   vcla_read_weight_q8  the stored int8 rows (rows x cols, host) and row scales (rows, host), exactly; synchronises
 *   vcla_load_weight_q8  stores caller int8 rows + scales exactly (host or device pointers); synchronises */
int vcla_read_weight_q8(vcla_ctx* ctx, const char* name, int8_t* q_host, float* scale_host, vcla_stream stream);
int vcla_load_weight_q8(vcla_ctx* ctx, const char* name, const int8_t* q, const float* scale, int on_device, vcla_stream stream);

/* ---- the hot path ----------------------------------------------------------------------------- */
/* Drop all sequences (KV cache lengths -> 0, every KV page back on the free stack). */
int vcla_reset(vcla_ctx* ctx, vcla_stream stream);

/* Paged KV cache (the reference's DynamicCache, HF:cache_utils.py:88-120, re-designed): physical pages of `page_tokens`
 * tokens are handed to sequences on demand by a device-side allocator that runs inside the stream / the decode CUDA graph
 * (pages are assigned round-robin as sequences grow, so one sequence's pages are NOT contiguous; every kernel goes through
 * the page table).  vcla_decode_* fail with an error instead of running past max_seq.
 *   vcla_kv_geometry     pages per sequence (table row length), pages in the pool, tokens per page
 *   vcla_kv_read_pages   synchronous copy to the host of the page table (max_batch x pages_per_seq int32), the pages owned
 *                        per sequence (max_batch int32) and {free pages, exhausted flag} (2 int32); any pointer may be NULL
 *   vcla_kv_debug_shuffle  test hook: permute the order in which free pages are handed out (then resets the context) */
int vcla_kv_geometry(const vcla_ctx* ctx, int* pages_per_seq, int* total_pages, int* page_tokens);
int vcla_kv_read_pages(vcla_ctx* ctx, int32_t* table_host, int32_t* npages_host, int32_t* state_host);
int vcla_kv_debug_shuffle(vcla_ctx* ctx, uint32_t seed);
/* int8 KV cache (kv_format 1).  The reference keeps K/V in its DynamicCache as the model dtype (HF:cache_utils.py:88-120,
 * DynamicCache.update: torch.cat of the new key_states / value_states); HF's QuantizedCache (HF:cache_utils.py, QuantizedCache) and
 * vLLM's kv_cache_dtype store them in fewer bits instead.  Here every LLaMA K row (after RoPE) and V row is replaced, per head, by its
 * int8 round trip the moment it is computed, with the load_in_8bit rule applied to the row's 128 fp32 values: a = max|x|,
 * s = a / 127, q = clamp(rint(x * (127 / a)), -127, 127) (half to even; a = 0 gives s = q = 0).  Every attention reads q * s: the
 * prefill QKV epilogue also writes bf16(q * s) into the K/V columns its own attention reads, the decode step quantises the new row
 * before attending to it.  Per layer the pool holds the int8 rows [total_pages][K|V][heads][page_tokens][128] followed by their fp32
 * scales [total_pages][K|V][heads][page_tokens]: 132 bytes per row instead of 256 (0.516x).  The page table, allocator, truncate /
 * extend and copy-on-write are those of the bf16 cache; vcla_beam_cow_bytes counts 132 bytes per copied row.
 *   vcla_kv_read_layer   synchronous copy of one layer's pool bytes (vcla_memory_bytes' kv / layers) to the host */
int vcla_kv_read_layer(vcla_ctx* ctx, int layer, void* host);
/* Keep each resident sequence's first min(current length, len_host[b]) cached tokens (b < B, B = the batch of the last
 * vcla_prefill) and forget the rest; the pages stay owned by the sequence (vcla_reset returns them).  With vcla_prefill_extend this
 * reuses the common prefix of a conversation: HF DynamicCache.crop (HF:cache_utils.py) before generate(past_key_values=...). */
int vcla_kv_truncate(vcla_ctx* ctx, const int32_t* len_host, int B, vcla_stream stream);

/* pixels (B,3,I,I) NCHW -> image embeddings (B, r_queries, t_hidden), kept inside the context for the
 * next vcla_prefill and optionally copied to `out_dev_f32`.  Replaces
 *   vision_model(pixel_values) -> post_layernorm -> visual_resampler -> image_projection_layer
 * (modeling_visualcla.py:283-288 / :349-354; HF:models/clip/modeling_clip.py:667-692;
 *  modeling_visual_resampler.py:609-737). */
int vcla_vision_encode(vcla_ctx* ctx, const void* pixels_dev, int pixel_dtype, int B, float* out_dev_f32, vcla_stream stream);

/* Prefill B prompts of T tokens each (equal length, unpadded; position_ids = arange).
 *   ids_dev        int64 (B,T) device
 *   image_mode     VCLA_TEXT_ONLY / VCLA_IMAGE_AT_HEAD / VCLA_IMAGE_PLACEHOLDER
 *   img_row_dev    int32 (B) device: first row of the image block inside each sequence (index of <img> + 1),
 *                  -1 = no image for this sample; ignored for TEXT_ONLY; for AT_HEAD pass NULL (row 2)
 *   left_pad_dev   int32 (B) device or NULL: number of LEFT padding tokens per sequence (attention_mask = [0]*p + [1]*(T-p),
 *                  what HF generate expects for batched prompts of different lengths): pad keys are masked, the KV cache
 *                  holds only the real tokens.  pos_from_mask != 0: RoPE positions count real tokens from 0
 *                  (HF generate: position_ids = attention_mask.cumsum(-1) - 1); 0: positions are arange(S) (plain forward(),
 *                  which the reference calls without position_ids, modeling_visualcla.py:321-328).  Not with IMAGE_AT_HEAD.
 *   logits_all_dev f32 (B,S,V) or NULL   -- VisualCLAModel.forward(...).logits (modeling_visualcla.py:321-328)
 *   last_logits_dev f32 (B,V) or NULL    -- logits of the last position (what generate() samples from)
 *   next_tok_dev   int32 (B) or NULL     -- argmax of last_logits (greedy)
 * Fills the KV cache; sequence length becomes S.  Replaces the splice (modeling_visualcla.py:290-312 /
 * :356-377) + LlamaForCausalLM prefill (HF:models/llama/modeling_llama.py:375-501). */
int vcla_prefill(vcla_ctx* ctx, const int64_t* ids_dev, int B, int T, int image_mode, const int32_t* img_row_dev,
                 const int32_t* left_pad_dev, int pos_from_mask, float* logits_all_dev, float* last_logits_dev,
                 int32_t* next_tok_dev, vcla_stream stream);

/* Append T text tokens (ids_dev int64 (B,T)) to each of the B sequences resident since the last vcla_prefill (same B): the chunk
 * row t of sequence b is token L_b + t (RoPE position and cache slot; L_b = its current cached length) and attends to all L_b
 * cached tokens plus the chunk's rows up to itself.  No vision work: the cached prefix keeps its image rows.  Outputs as
 * vcla_prefill, over the chunk's rows only (logits_all_dev f32 (B,T,V)); lengths grow by T.  Like vcla_prefill it restarts the
 * token history (row 0 = this call's pick), the sampler's step counter and the finished flags.  Fails when nothing is resident,
 * while the data-parallel exchange is active, when B*T > max_prefill_tokens or when a sequence could pass max_seq.  Replaces HF
 * generate(input_ids, past_key_values=cache): the forward over the uncached tail of the prompt (HF:generation/utils.py,
 * HF:models/llama/modeling_llama.py with past_key_values). */
int vcla_prefill_extend(vcla_ctx* ctx, const int64_t* ids_dev, int B, int T, float* logits_all_dev, float* last_logits_dev,
                        int32_t* next_tok_dev, vcla_stream stream);

/* One greedy decode step for the B resident sequences: consumes tok_in_dev (int32 (B)), appends its K/V,
 * writes logits (f32 (B,V), optional) and the argmax (int32 (B)).  Captured into a CUDA graph on first use
 * (per distinct argument tuple) when use_graph != 0.  Replaces one iteration of
 * GenerationMixin._sample (HF:generation/utils.py:2743-2810) incl. DynamicCache.update (HF:cache_utils.py:119-120). */
int vcla_decode_step(vcla_ctx* ctx, const int32_t* tok_in_dev, int B, float* logits_dev, int32_t* tok_out_dev, int use_graph,
                     vcla_stream stream);

/* n_steps (1..64) greedy decode steps replayed as ONE CUDA graph; tok_inout_dev (int32 (B)) is consumed and rewritten in place by
 * every step and every chosen token is appended to the history (vcla_read_history).  Same arithmetic as n_steps calls of
 * vcla_decode_step; amortises the launch gap between steps. */
int vcla_decode_multi(vcla_ctx* ctx, int32_t* tok_inout_dev, int B, int n_steps, vcla_stream stream);

/* Tokens chosen so far: row 0 = the prefill's argmax, row s = decode step s.  Copies [n_steps, B] int32 to a DEVICE buffer
 * (async on `stream`): lets a greedy loop run as pure graph replays with no per-step host or torch work. */
int vcla_read_history(vcla_ctx* ctx, int32_t* dst_dev, int B, int n_steps, vcla_stream stream);

/* ---- device-side sampling (SURVEY.md section 8f-1) ---------------------------------------------------------------------
 * chat()'s real default is sampling (models/visualcla/modeling_utils.py:36-47: temperature 0.5, top_k 40, top_p 0.9,
 * repetition_penalty 1.1, no_repeat_ngram_size 15).  With a sampler set, vcla_prefill / vcla_decode_step / vcla_decode_multi
 * replace the argmax by ONE fused kernel per step -- HF's processor chain in HF's order (RepetitionPenalty, NoRepeatNGram,
 * min_new_tokens EOS mask, Temperature, TopK, TopP; HF:generation/logits_process.py) + a Philox-keyed multinomial draw -- on the
 * device token history (with inputs_embeds HF's processors only see the new tokens), inside the captured CUDA graph: no logits
 * leave the device, no host work per token.  do_sample = 0 takes the argmax of the processed scores (greedy + penalties).
 * A sequence that emitted an EOS id keeps producing pad_token_id (sticky per-sequence flag, vcla_read_finished).
 * The parameters live in device memory: changing them does not re-capture graphs.
 * The draw (do_sample = 1), for sequence b after L generated tokens (L = 0 at the prefill's pick):
 *   x0   = word 0 of Philox4x32-10 (Random123) with counter words (L, b, 0, 0) and key words (seed & 0xffffffff, seed >> 32)
 *   u    = (x0 >> 8) * 2^-24, a 24-bit uniform in [0, 1)
 *   the candidates -- the top-k set, every tie at the k-th value included -- sorted by (score descending, token id ascending); top-p
 *   keeps ranks 0 .. keep-1 (rank r >= 1 goes when the fp32 sum of the probabilities of ranks r .. last is <= 1 - top_p)
 *   e_r  = expf(s_r - s_0), tot = e_0 + ... + e_{keep-1} (fp32, in rank order)
 *   pick = the first rank r with e_0 + ... + e_r > u * tot, else rank keep-1
 * Prompt lookup verification (vcla_lookup) draws row r of a step that starts at L generated tokens with counter (L + r, 0): the draw
 * one-token decoding makes at that length.  The candidate buffer holds 1024 entries: a row with more than 1024 tokens tied at the
 * k-th value draws among 1024 of them, which ones and in which order undefined. */
typedef struct {
  int do_sample;
  float repetition_penalty;     /* 1 = off */
  int no_repeat_ngram_size;     /* 0 = off */
  float temperature;            /* 1 = off */
  int top_k;                    /* 1..1024, required when do_sample */
  float top_p;                  /* 1 = off */
  int min_new_tokens;
  int n_eos;                    /* <= 4 */
  int eos_token_id[4];
  int pad_token_id;
  uint64_t seed;                /* the Philox key: the draw above */
} vcla_sampler;
int vcla_sampler_supported(const vcla_ctx* ctx);   /* 1 when the vocabulary row fits one CTA's shared memory */
int vcla_set_sampler(vcla_ctx* ctx, const vcla_sampler* sampler_or_null, vcla_stream stream);   /* NULL: back to greedy argmax */
int vcla_read_finished(vcla_ctx* ctx, int32_t* dst_dev, int B, vcla_stream stream);
/* Operator-level entry (parity tests): the same kernel on caller logits (B,V) f32 and a token history [L][B] int32; writes the
 * chosen tokens (B) and, if not NULL, the processed scores (B,V) (-inf = filtered) exactly as HF's chain would return them.
 * Synchronises. */
int vcla_op_sample(const float* logits_dev, int B, int V, const int32_t* history_dev, int L, const vcla_sampler* sampler,
                   int32_t* tok_dev, float* scores_out_dev, vcla_stream stream);

/* ---- prompt lookup decoding (HF GenerationConfig.prompt_lookup_num_tokens / max_matching_ngram_size) ------------------------------
 * One resident sequence (B = 1).  With a lookup set, every step of vcla_decode_multi is a verification step: k + 1 rows -- the last
 * emitted token and up to k tokens copied from earlier text -- run through one decode step (the split counts of a one-row step, so
 * each row's logits are bit-identical to a one-token step at that position), each row is picked by the argmax or, with a sampler set,
 * by the sampler at that row's length (draw counter (length, 0), history extended by the drafts it verifies), and the picks up to and
 * including the first one that differs from the next draft are emitted (HF:generation/utils.py _assisted_decoding), stopping after an
 * EOS id and at max_new history rows.  The next drafts follow HF:generation/candidate_generator.py
 * PromptLookupCandidateGenerator.get_candidates over prompt_ids ++ the emitted tokens: for g = min(n, len - 1) .. 1 the leftmost
 * earlier window equal to the last g tokens, up to k tokens of its continuation, clamped to max_new - emitted - 1.  A step emits 1 to
 * k + 1 tokens, the same tokens one-token decoding emits; steps after the end emit nothing.  The first decode call after a prefill
 * reserves pages and drafts the first step.  k is clamped to 15 and further to the rows the one-row split counts can reduce together.
 * With the token stream armed, each verification step publishes the tokens it emits (vcla_stream_wait counts history rows).
 * vcla_set_lookup refuses beam search, the data-parallel exchange and more than one resident sequence; vcla_decode_multi refuses
 * B != 1 and prefill length + max_new + k > max_seq.  n above 16 is searched as 16 (drafts only).  prompt_ids is copied.
 * Restates HF:generation/utils.py:3603-3620 and HF:generation/candidate_generator.py:1057-1149.  NULL: off (plain decode steps). */
typedef struct {
  int k;                        /* drafted tokens per step, >= 1 */
  int n;                        /* largest n-gram matched, >= 1 (HF default 2) */
  int max_new;                  /* max_new_tokens: history rows after which steps emit nothing */
  const int64_t* prompt_ids;    /* device int64 (prompt_len): the text searched before the emitted tokens */
  int prompt_len;
} vcla_lookup;
int vcla_set_lookup(vcla_ctx* ctx, const vcla_lookup* lookup_or_null, vcla_stream stream);
/* Synchronises.  out[0] = history rows (emitted tokens incl. the prefill's pick), out[1] = finished flag, out[2] = verification steps
 * that emitted, out[3] = drafts offered, out[4] = drafts emitted (counters since vcla_set_lookup), out[5] = rows per verification step. */
int vcla_read_lookup_stats(vcla_ctx* ctx, int64_t* out6_host, vcla_stream stream);

/* ---- beam search without sampling (HF:generation/utils.py:2876-3395, the vectorised _beam_search; reached from the reference's
 * generate(num_beams=...), models/visualcla/modeling_visualcla.py:382-391) ---------------------------------------------------------
 * With beam mode set, vcla_prefill prefills each of its B prompts once, runs the first selection on the prompts' last logits and forks
 * every prompt to K = num_beams rows (row b * K + j) that share the prompt's KV-cache pages; next_tok_dev (if not NULL) then receives
 * the B * K first tokens.  vcla_decode_step / vcla_decode_multi step all B * K rows: per step one kernel per beam row (log_softmax,
 * repetition penalty / no-repeat-ngram / min_new_tokens EOS mask on that beam's own history, + its running score, top-M of the row),
 * one kernel per item (the item's top M = max(2, 1 + n_eos) * K candidates over K * V, stopping-criteria hits, the next K beams, the
 * finished-hypothesis store, the early-stop heuristic) and, after the sequence lengths advance, the page-table reorder: a beam continues
 * its parent's pages; only the partly filled page it writes next is copied, when several beams continue one parent.  All of it is
 * captured in the decode graphs.  Refused: B * K > min(max_batch, 64), prompt + max_new_tokens > max_seq, the data-parallel exchange.
 *   vcla_set_beam        NULL: off (argmax / sampler again).  early_stopping: 0 False, 1 True, 2 "never" (HF's three settings)
 *   vcla_read_beams      synchronous copy to the host of the store of the B items: tokens [B][K][max_new_tokens] int32 (the first
 *                        lengths[b][k] are valid), lengths [B][K] int32, scores [B][K] f32 (length-penalised, best first), done [B]
 *                        int32 (HF's stopping condition holds for the item); any pointer may be NULL
 *   vcla_beam_cow_bytes  bytes of K/V copied copy-on-write since the last reset (counted on the device); synchronises
 *   vcla_op_beam_step    the two selection kernels on caller buffers (operator tests): logits (t == 0: B rows, the prompts; else B * K
 *                        rows) f32 (rows, V); history [t][rows] int32; run_scores [rows] in (ignored at t == 0), [B * K] out; the store
 *                        hyp_scores / hyp_lens / hyp_fin [B][K] and hyp_tokens [B][K][max_new_tokens] and item_state [B][2] = {heuristic
 *                        unsatisfied, done} are initialised at t == 0 and updated; parent (the logits row each new beam continues), token
 *                        [B * K]; cand (nullable) [B][M][2] = {k * V + v, hit} of the item's top M.  Synchronises. */
typedef struct {
  int num_beams;                /* 2..16 */
  float length_penalty;
  int early_stopping;           /* 0 False, 1 True, 2 "never" */
  int max_new_tokens;
  int n_eos;                    /* <= 4 */
  int eos_token_id[4];
  float repetition_penalty;     /* 1 = off */
  int no_repeat_ngram_size;     /* 0 = off */
  int min_new_tokens;
} vcla_beam;
int vcla_set_beam(vcla_ctx* ctx, const vcla_beam* beam_or_null);
/* ---- fan-out: n sampled replies per prompt from one prefill (HF generate(do_sample=True, num_return_sequences=n)) ------------------
 * With n > 1 set, vcla_prefill prefills each of its B prompts once and forks prompt b to rows b * n .. b * n + n - 1 (the order of HF's
 * repeat_interleave) through the beam search page-table reorder: the rows share every full page of the prompt, and every row but the
 * first of a prompt gets its own copy of the partly filled page it writes next (vcla_beam_cow_bytes counts those rows).  The first pick
 * is the sampler's over B * n rows, row r scoring the last logits of prompt r / n with its own draw counter (0, r) -- so siblings draw
 * independently and a row's draw and processed scores are exactly those of an unforked row r with the same logits; without a sampler
 * each row takes its prompt's argmax.  next_tok_dev (if not NULL) receives the B * n picks and last_logits_dev stays (B, V); the token
 * history, the finished flags, the sequence lengths and the page table then describe B * n resident rows, which vcla_decode_step /
 * vcla_decode_multi step like a batch, and an armed token stream receives the B * n picks as the prefill's step.  n = 1: off (the
 * default).  Refused by vcla_prefill: B * n > min(max_batch, 64), beam mode, the data-parallel exchange.  vcla_prefill_extend is refused
 * in fan-out mode and while forked rows are resident (until the next vcla_prefill or vcla_reset). */
int vcla_set_fanout(vcla_ctx* ctx, int n);
int vcla_read_beams(vcla_ctx* ctx, int32_t* tokens_host, int32_t* lengths_host, float* scores_host, int32_t* done_host);
int vcla_beam_cow_bytes(vcla_ctx* ctx, int64_t* bytes, int reset);
int vcla_op_beam_step(const float* logits_dev, int B, int V, const int32_t* history_dev, int t, const vcla_beam* beam, float* run_scores_dev,
                      float* hyp_scores_dev, int32_t* hyp_lens_dev, int32_t* hyp_fin_dev, int32_t* hyp_tokens_dev, int32_t* item_state_dev,
                      int32_t* parent_dev, int32_t* token_dev, int32_t* cand_dev, vcla_stream stream);

/* ---- data parallel over the GPUs of one box (SURVEY.md section 8e; the reference has no DP of its own) ----------------
 * Requests are independent through the whole path, so each rank (one process + one context per GPU) runs a contiguous slice of
 * the batch and the ONLY exchange is one NCCL all-gather of the chosen token ids per decode step.  After vcla_nccl_init the
 * exchange is part of the path itself: vcla_prefill and every decode step (also inside the CUDA graphs of vcla_decode_multi)
 * all-gather `width` int32 slots per rank on a forked stream branch -- off the step's critical path, joined before the send
 * buffer is rewritten -- and append them to a device-side global history.
 *   vcla_nccl_unique_id   rank 0 creates the 128-byte ncclUniqueId and ships it to the other ranks by any means
 *   vcla_nccl_init        width = slots per rank (the largest shard's batch, <= 64); collective over all ranks
 *   vcla_allgather_tokens plain all-gather of n int32 per rank on `stream` (the non-graph building block)
 *   vcla_dp_set_active    the exchange is part of vcla_prefill / vcla_decode_* only while active (off after init): every rank must
 *                         then make the same sequence of calls; a rank-local generation runs with it off
 *   vcla_dp_exchange      one step's exchange without compute (a rank that holds no requests: global batch < world size)
 *   vcla_read_history_dp  [n_steps][world * width] int32 -> device buffer: row 0 = prefill argmax of every rank, row s = step s
 * NCCL is bound with dlopen("libnccl.so.2") at the first of these calls; single-GPU use never loads it. */
int vcla_nccl_unique_id(uint8_t* out128);
int vcla_nccl_init(vcla_ctx* ctx, const uint8_t* id128, int rank, int world, int width);
int vcla_allgather_tokens(vcla_ctx* ctx, const int32_t* local_dev, int n, int32_t* all_dev, vcla_stream stream);
int vcla_dp_set_active(vcla_ctx* ctx, int on);
int vcla_dp_exchange(vcla_ctx* ctx, vcla_stream stream);
int vcla_read_history_dp(vcla_ctx* ctx, int32_t* dst_dev, int n_steps, vcla_stream stream);

/* ---- token streaming (models/visualcla/modeling_utils.py:180-247 chat_in_stream; HF generate(streamer=...)) -------------------
 * While armed, the kernel that advances the sequence lengths after every token choice (the prefill / extend pick and every decode
 * step, also inside the CUDA graphs) copies that step's tokens into a ring in pinned, mapped host memory and then publishes the step
 * with a system-scope release store of its counter: the host sees each token as soon as the device has it, with no copy, graph
 * break or synchronisation per token.  The token-choosing kernels are the same armed or not, so streaming never changes a token.
 *   vcla_stream_arm    on != 0: allocate the ring (once), reset the published-step counter, bump the epoch; refused while earlier
 *                      armed work is still in flight, in beam mode and while the data-parallel exchange is active.  on == 0: later
 *                      enqueues stop publishing (graphs captured armed and disarmed are cached apart)
 *   vcla_stream_wait   wait until at least `target` steps are published (acquire load); *published = the count seen.  Returns 0
 *                      on success or when timeout_us (< 0: no limit) expires first (then *published < target); returns an error
 *                      when all armed work enqueued so far has completed and the count is still below target (it never will be)
 *   vcla_stream_read   copy published steps [from, to) of B tokens each to a host buffer ([to - from][B] int32) */
int vcla_stream_arm(vcla_ctx* ctx, int on);
int vcla_stream_wait(vcla_ctx* ctx, int target, int timeout_us, int* published);
int vcla_stream_read(vcla_ctx* ctx, int from, int to, int B, int32_t* dst_host);

/* number of this library's kernels launched by the context since the last call with reset != 0 */
int64_t vcla_kernel_launches(vcla_ctx* ctx, int reset);

/* ---- introspection for parity tests ---------------------------------------------------------- */
/* Copy an internal fp32 activation to the host (synchronises): "vit_out" (B,tokens,v_hidden), "post_ln",
 * "resampler_out" (B,nq,r_hidden), "projector_out" (B,nq,t_hidden), "inputs_embeds" n/a after prefill; "step_logits" (B,V): the
 * logits rows of the last decode or verification step on the cluster split-K schedule (B <= 32 rows); "lookup_tokens" (B): the int32
 * input tokens (bit patterns in the f32 buffer) of the next prompt lookup verification step. */
int vcla_read_stage(vcla_ctx* ctx, const char* stage, int B, float* dst_host, vcla_stream stream);

/* ---- operator-level entry points (kernel parity tests, micro-benchmarks) ---------------------- */
/* D = A[M,K] * W[N,K]^T on the wgmma path.  mode: 0 store bf16 (act: 0 none, 1 quick_gelu, 2 gelu),
 * 1 fp32 (accumulate flag), 2 SwiGLU (W rows interleaved [32 gate|32 up]), 3 swap-AB split-K partials
 * (out f32 [splits][M_b][N] with A = weights).  use_reference != 0 runs the naive CUDA-core kernel instead. */
int vcla_op_gemm(const void* A_dev_bf16, const void* W_dev_bf16, int M, int N, int K, int mode, int act, int accumulate,
                 const float* bias_dev, void* out_dev, int ldo, int splits, int tile_n, int use_reference, vcla_stream stream);
/* Decode GEMM with the split-K reduction inside a thread-block cluster (csrc/gemm_decode.cu): out[b, n] = sum_k W[n, k] X[b, k], W (M, K)
 * bf16 streamed once, X (B <= 32, K) bf16, `splits` CTAs per cluster (1..8).  mode 0: out_or_resid = out f32 (B, M) = rstd[b] * acc;
 * mode 1: out_or_resid = resid f32 (B, M) += acc, xw_or_h = bf16 (B, M) = resid * norm_w, ssq_out f32 (B, ceil(M / 128)) = per-tile sums of
 * squares; mode 2: W rows interleaved [32 gate | 32 up], xw_or_h = h bf16 (B, M / 2) = silu(rstd * g) * (rstd * u).
 * rstd[b] = rsqrt(sum_slots ssq_in[b][slot] * inv_dim + eps), 1 when ssq_in is NULL.  vcla_op_gemm_csk_clusters: co-resident clusters. */
int vcla_op_gemm_csk(const void* W_dev_bf16, const void* X_dev_bf16, int M, int B, int K, int splits, int mode, float* out_or_resid,
                     const float* norm_w, void* xw_or_h, float* ssq_out, const float* ssq_in, int ssq_slots, float inv_dim, float eps,
                     vcla_stream stream);
int vcla_op_gemm_csk_clusters(int B, int splits);
/* The int8 variant of vcla_op_gemm_csk (the decode GEMMs of weight_format 1, replacing bitsandbytes' Linear8bitLt forward behind
 * models/visualcla/modeling_visualcla.py:151-156): Wq int8 (M, K) row-major, wscale f32 (M) (device); K % 64 == 0; B <= 64 (a 64-column
 * batch tile serves 33..64).  The row scale is applied after the fixed-order cluster reduction: mode 0 out = rstd * s * acc, mode 1
 * resid += s * acc, mode 2 gate and up rows each take their own scale.  Synchronises. */
int vcla_op_gemm_csk_q8(const int8_t* Wq_dev, const float* wscale_dev, const void* X_dev_bf16, int M, int B, int K, int splits, int mode,
                        float* out_or_resid, const float* norm_w, void* xw_or_h, float* ssq_out, const float* ssq_in, int ssq_slots,
                        float inv_dim, float eps, vcla_stream stream);
/* The prefill GEMM of weight_format 1 (same replacement): bf16(Wq) (N, K) int8 row-major is expanded exactly, then
 * D = A[M,K] * bf16(Wq)^T * diag(wscale) on the wgmma path.  mode 0 store bf16, 1 fp32 (accumulate flag; with norm_w not NULL also
 * xw = bf16(out * norm_w) (M, N) and ssq_out (M, ceil(N / tile width)) as vcla_prefill's residual GEMMs; the GEMM picks a tile width of
 * 64, 128 or 256 from M and N), 2 SwiGLU (rows interleaved [32 gate|32 up]).
 * Synchronises. */
int vcla_op_gemm_q8(const void* A_dev_bf16, const int8_t* Wq_dev, const float* wscale_dev, int M, int N, int K, int mode, int accumulate,
                    void* out_dev, int ldo, const float* norm_w, void* xw_dev, float* ssq_out, vcla_stream stream);
/* tuning hooks: read / override the CTAs-per-cluster of the five decode GEMM shapes {qkv, o, gate_up, down, lm_head} at batch B
 * (B <= 32; with weight_format 1 B <= 64, where at 33..64 the lm_head runs on the workspace GEMM and its entry is ignored) */
int vcla_debug_set_csk_splits(vcla_ctx* ctx, int B, int qkv, int o, int gate_up, int down, int lm_head);
int vcla_debug_get_csk_splits(vcla_ctx* ctx, int B, int* out5);
/* test hook: resident CTAs per SM (occupancy query) of the two decode kernels a step at batch B launches with this context's weights and
 * cache: out2[0] the cluster split-K GEMM, out2[1] decode attention */
int vcla_debug_decode_ctas_per_sm(vcla_ctx* ctx, int B, int* out2);
/* prefill attention kernel: 0 = the mma.sync kernel everywhere, 1 (default) = wgmma flash attention (QK^T / PV on the warpgroup tensor
 * cores, S and O in registers, TMA operands) at head dim 128 (LLaMA prefill) and mma.sync at head dim 64 (ViT / Resampler), 2 = wgmma everywhere */
void vcla_set_attention_tc(int mode);
/* The prefill attention of vcla_vision_encode and vcla_prefill on caller buffers, through the same dispatch (vcla_set_attention_tc).
 * All operands bf16, head h at columns [h*HD, (h+1)*HD) of a row; HD 64 or 128; strides in elements.
 *   q        B*Sq rows: query i of sequence b is row b*Sq + i (q_stride)
 *   k0, v0   segment 0, B*n0 rows: key j < n0 of sequence b is row b*n0 + j (kv0_stride)
 *   k1, v1   segment 1, B*n1 rows (NULL when n1 = 0): key n0 + j of sequence b is row b*n1 + j (kv1_stride)
 *   out      B*Sq rows (o_stride): out = softmax(scale * q k^T) v over the keys visible to the query; only the H*HD columns of
 *            the B*Sq rows are written
 * Key j of sequence b is visible to query i iff kv_start[b] <= j < n0 + n1 and, when causal, j <= i + n0 + n1 - Sq.  kv_start_dev is
 * int32 (B) in device memory (left padding: the first kv_start[b] keys of sequence b are hidden), NULL for none.  A query that sees no
 * key gets a row of zeros.  Hidden keys that share a 64-key tile with visible ones are still loaded, and a zero probability does not
 * cancel a NaN in P*V: such K/V rows -- the left padding, the causal future, the rows after a sequence's last key up to its tile's end
 * (the next sequence's first rows, or the allocation's) -- must be finite.  Causal attention takes one KV segment on the wgmma kernel;
 * a call that kernel cannot describe (a pitch or an output stride that is not a multiple of 8, causal with two segments) runs on the
 * mma.sync kernel.  Refused on the host, before any launch: a NULL q, k0, v0 or out (k1, v1 when n1 > 0), B, H or Sq below 1, and
 * kv_start[b] outside [0, n0 + n1] (read back after synchronising the stream).  Synchronises. */
int vcla_op_attention(const void* q, int q_stride, const void* k0, const void* v0, int kv0_stride, int n0, const void* k1,
                      const void* v1, int kv1_stride, int n1, void* out, int o_stride, int B, int H, int Sq, int HD, float scale,
                      int causal, vcla_stream stream, const int32_t* kv_start_dev);
/* The paged prefill attention of vcla_prefill_extend on caller buffers (head dim 128): q (B*T rows, q_stride) bf16; kv_pages a layer
 * pool [pages][K|V][H][page_tokens][128] bf16; page_table int32 (B, pages_per_seq); base_len_dev int32 (B) cached tokens before the
 * chunk (the chunk's own K/V must already be in the pool at slots base_len .. base_len + T - 1); out (B*T rows, o_stride) bf16.
 * Key j is visible to chunk row t iff j <= base_len[b] + t.  Refused on the host, before any launch: base_len[b] < 0,
 * base_len[b] + T > pages_per_seq * page_tokens, a negative page among the entries the chunk reads.  Synchronises. */
int vcla_op_attention_paged(const void* q, int q_stride, const void* kv_pages, const int32_t* page_table, int pages_per_seq,
                            int page_tokens, const int32_t* base_len_dev, void* out, int o_stride, int B, int H, int T, float scale,
                            vcla_stream stream);
/* The decode attention of vcla_decode_step on caller buffers (head dim 128), context-free: one new token per sequence.  In one launch
 * it sums the fused-QKV split-K partials qkv_partial f32 [splits][B][3*H*128] (q | k | v, split order 0..splits-1), applies RoPE at
 * position seq_len[b] to q and k, rounds k and v to bf16 and WRITES them into the pool at (page_table[b][seq_len[b] / page_tokens], slot
 * seq_len[b] % page_tokens) -- nothing else in the pool is written --, and attends over the seq_len[b] cached rows plus the new one.
 *   kv_pages      the layer pool [pages][K|V][H][page_tokens][128] bf16, read and written
 *   page_table    int32 (B, pages_per_seq); only entries 0 .. seq_len[b] / page_tokens of a row are read
 *   seq_len_dev   int32 (B): cached tokens per sequence, 0 allowed (the output is then the new token's v); not advanced by the call
 *   out           bf16 (B, H*128)
 *   kv_splits     1..8 CTAs per (sequence, head), combined in split order through a scratch and self-resetting counters
 *   persistent    0 = the one-shot kernel, 1 = the persistent kernel (kv_splits must be 1) on a grid of persistent_grid CTAs (0 = default)
 *   launches      >= 1: the kernel is enqueued that many times over the same scratch and counters, as graph replays do; the append is
 *                 idempotent while seq_len is unchanged, so out and the pool do not depend on it.  out is filled with NaN before every
 *                 launch: what the last launch leaves unwritten stays NaN
 * The RoPE tables (positions 0 .. max seq_len), scratch and counters are made for the call.  Refused on the host, before any launch:
 * seq_len[b] < 0 or seq_len[b] + 1 > pages_per_seq * page_tokens, a negative page among the entries read, page_tokens not a multiple of 8
 * in 8..64, kv_splits outside 1..8, persistent with kv_splits > 1, B > 64.  Synchronises. */
int vcla_op_attention_decode(const float* qkv_partial, int splits, void* kv_pages, const int32_t* page_table, int pages_per_seq,
                             int page_tokens, const int32_t* seq_len_dev, void* out, int B, int H, int kv_splits, float scale,
                             float rope_theta, int persistent, int persistent_grid, int launches, vcla_stream stream);
/* Operator entry of the verification attention (tests): rows (2..16) query rows of ONE sequence of length seq_len_dev[0] cached tokens;
 * row r at position seq_len + r appends its K/V, then attends over keys [0, seq_len + r] with the one-token kernel's arithmetic at
 * length seq_len + r + 1 and kv_splits splits.  qkv_partial [splits][rows][3 * H * 128], out [rows][H * 128].  Synchronises. */
int vcla_op_attention_decode_lookup(const float* qkv_partial, int splits, void* kv_pages, const int32_t* page_table, int pages_per_seq,
                                    int page_tokens, const int32_t* seq_len_dev, void* out, int rows, int H, int kv_splits, float scale,
                                    float rope_theta, vcla_stream stream);
/* The paged prefill attention and the two decode entries on a pool in the int8 layout (kv_format 1, above): int8 rows of the
 * total_pages pages, then their fp32 scales (the scale region starts total_pages * 2 * H * page_tokens * 128 bytes in).  Keys and
 * values are read as q * s; the decode entries quantise the new row per head and write it as q and s.  Same refusals as the bf16
 * entries, plus total_pages < 1 and a page the call reads at or beyond total_pages. */
int vcla_op_attention_paged_q8(const void* q, int q_stride, const void* kv_pool, int total_pages, const int32_t* page_table,
                               int pages_per_seq, int page_tokens, const int32_t* base_len_dev, void* out, int o_stride, int B, int H, int T,
                               float scale, vcla_stream stream);
int vcla_op_attention_decode_q8(const float* qkv_partial, int splits, void* kv_pool, int total_pages, const int32_t* page_table,
                                int pages_per_seq, int page_tokens, const int32_t* seq_len_dev, void* out, int B, int H, int kv_splits,
                                float scale, float rope_theta, int persistent, int persistent_grid, int launches, vcla_stream stream);
int vcla_op_attention_decode_lookup_q8(const float* qkv_partial, int splits, void* kv_pool, int total_pages, const int32_t* page_table,
                                       int pages_per_seq, int page_tokens, const int32_t* seq_len_dev, void* out, int rows, int H,
                                       int kv_splits, float scale, float rope_theta, vcla_stream stream);
/* The greedy pick of vcla_decode_step on caller buffers: logits_out f32 (B, V) or NULL = sum over splits (in split order) of partial f32
 * [splits][B][ldp] (ldp >= V; columns >= V are not read), tok_out int32 (B) = its argmax, the smallest index among equal maxima as
 * torch.argmax; a row that is -inf everywhere gives 0.  Synchronises. */
int vcla_op_logits_argmax(const float* partial, int splits, int ldp, int B, int V, float* logits_out, int32_t* tok_out, vcla_stream stream);
int vcla_op_layernorm(const float* x, int rows, int D, const float* w, const float* b, float eps, void* y_bf16, float* y_f32,
                      vcla_stream stream);
int vcla_op_rmsnorm(const float* x, int rows, int D, const float* w, float eps, void* y_bf16, vcla_stream stream);
/* Micro-benchmark of ONE decode weight-streaming GEMM shape (which: 0 fused QKV, 1 o_proj, 2 fused gate/up, 3 down_proj,
 * 4 lm_head) over every layer's distinct weights with batch B, timed with CUDA events on `stream`; returns the mean
 * microseconds per kernel launch and the algorithmic weight bytes one launch streams (weight_format 1: the int8 kernel, one byte
 * per weight + 4 per row scale, for shapes 0..3).  Synchronises. */
int vcla_bench_decode_gemm(vcla_ctx* ctx, int which, int B, int reps, float* avg_us, int64_t* weight_bytes, vcla_stream stream);
/* Timeline trace for profiles/: when enabled, CTA (0,0,0) of every kernel appends {tag, t_entry, t_dependency_resolved, t_exit}
 * (%globaltimer, ns).  Tags: 1 swap-AB GEMM, 2 GEMM, 3 prefill attention, 4 decode attention, 5 layernorm, 6 rmsnorm, 7 rope+cache,
 * 8 resid+rmsnorm, 9 silu*mul, 10/11 logits+argmax, 12 advance, 13 embed, 14 sampler, 15 beam step, 16 beam select, 17 beam page
 * reorder, 18 beam page copy, 21 fan-out row map.  vcla_trace_read synchronises and clears. */
int vcla_trace_enable(vcla_ctx* ctx, int max_events);
int vcla_trace_read(vcla_ctx* ctx, uint64_t* dst_host, int max_events, int* n_events);
/* enable/disable programmatic dependent launch for subsequently enqueued kernels (process-wide) */
void vcla_set_pdl(int on);

/* ---- image pre-processing (the step before the path; SURVEY.md §8(f) row 3) ------------------------ */
/* Replaces HF CLIPImageProcessor's PIL pipeline as the reference calls it for every request
 * (models/visualcla/modeling_utils.py:130 builds it, :150-152 / :187-189 call it):
 *   resize(shortest_edge = out_size, BICUBIC) -> center_crop(out_size) -> x * 1/255 -> (x - mean) / std
 * The resize is Pillow's 8-bit ImagingResample (antialiased separable bicubic, 22-bit taps, clip after each pass,
 * horizontal first) and the result is bit-identical to it.  No context needed: the caller owns every buffer.
 *
 * vcla_preprocess_workspace_bytes: device scratch one call needs for a (height, width) picture; -1 if unsupported
 *   (sides 1..32768, out_size 1..4096, resized long side <= 65536).  Host-only, no GPU needed.
 * vcla_resample_taps: Pillow's tap table of one axis (host-only): first[out], count[out], taps[out][ksize] with 22
 *   fractional bits.  Returns ksize; with all three pointers NULL only returns ksize.  -1 on error.
 * vcla_preprocess_image: rgb_dev = (height, width, 3) uint8 RGB in device memory; pixel_values_dev = (3, out_size,
 *   out_size) in `dtype` (VCLA_F32 / F16 / BF16, round-to-nearest from the float32 result); mean3/std3 = host floats.
 *   Builds the tap tables on the host, uploads them into the workspace and enqueues two kernels on `stream`.  The
 *   workspace must be 16-byte aligned and stay untouched until the stream has run them. */
int64_t vcla_preprocess_workspace_bytes(int height, int width, int out_size);
int vcla_resample_taps(int in_size, int out_size, int32_t* first, int32_t* count, int32_t* taps, int ksize_capacity);
int vcla_preprocess_image(const uint8_t* rgb_dev, int height, int width, int out_size, const float* mean3,
                          const float* std3, void* workspace_dev, int64_t workspace_bytes, void* pixel_values_dev,
                          int dtype, vcla_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* VCLA_H_ */
