"""Beam search of VisualCLAModel.generate(num_beams=K, do_sample=False) in fp32 on the CPU (ref: modeling_visualcla.py:382-391 forwards
num_beams to HF generate(inputs_embeds=...) -> HF:generation/utils.py:2876-3395, the vectorised _beam_search of transformers 5.5), on
top of the path restatement in visualcla_oracle.py.  With inputs_embeds the prompt is not part of input_ids: decoder_prompt_len = 0,
the processors see only the generated tokens, the length penalty divides by the generated length.  Ties between equal scores go to
the lower index (stable sorts), as on the device."""
from __future__ import annotations

from typing import Optional

import torch

from visualcla_oracle import KVCache, PathConfig, llama_forward, special_ids, splice, vision_encode


class BeamState:
    """Per-item beam-search state [B][K]: running scores, the finished-hypothesis store (scores, lengths, finished flags, token
    rows) and the early-stop / done flags (HF:3197-3219)."""

    def __init__(self, B: int, K: int, max_new: int):
        self.B, self.K, self.max_new = B, K, max_new
        self.run = torch.zeros(B, K)
        self.run[:, 1:] = -1e9                                              # :3200-3201
        self.scores = torch.full((B, K), -1e9)                               # :3202
        self.lens = torch.zeros(B, K, dtype=torch.long)
        self.fin = torch.zeros(B, K, dtype=torch.bool)                       # :3205
        self.tokens = torch.zeros(B, K, max_new, dtype=torch.long)
        self.unsat = torch.ones(B, dtype=torch.bool)                         # :3208
        self.done = torch.zeros(B, dtype=torch.bool)
        self.hist = torch.zeros(B, K, 0, dtype=torch.long)                   # running beams' generated tokens


def _topk_stable(x: torch.Tensor, k: int):
    v, i = torch.sort(x, dim=-1, descending=True, stable=True)
    return v[..., :k], i[..., :k]


def beam_step(st: BeamState, logits: torch.Tensor, t: int, n_eos_ids, length_penalty: float, early_stopping,
              repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0, min_new_tokens: int = 0) -> dict:
    """One iteration of the loop body (HF:3252-3371) on fp32 logits of the B*K running beams (t == 0: the B prompts; HF starts
    beams 1..K-1 at -1e9, so only beam 0 of each item can be picked, and all K beams share the prompt's logits).
    -> {parent (B,K) beam index continued, token (B,K), cand (B,M) flat indices k*V+v, hit (B,M)}; updates `st`."""
    from transformers.generation import logits_process as lp
    B, K = st.B, st.K
    eos = list(n_eos_ids)
    M = max(2, 1 + len(eos)) * K                                             # :3154
    V = logits.shape[-1]
    lg = logits.float()
    if t == 0:
        lg = lg.repeat_interleave(K, dim=0)
    log_probs = torch.log_softmax(lg, dim=-1)                                # :3256
    ids = st.hist.reshape(B * K, t)
    procs = []                                                               # :3257 (HF:_get_logits_processor order)
    if min_new_tokens and eos:
        procs.append(lp.MinNewTokensLengthLogitsProcessor(0, min_new_tokens, eos))
    if repetition_penalty != 1.0:
        procs.append(lp.RepetitionPenaltyLogitsProcessor(penalty=repetition_penalty))
    if no_repeat_ngram_size:
        procs.append(lp.NoRepeatNGramLogitsProcessor(no_repeat_ngram_size))
    for p in procs:
        log_probs = p(ids, log_probs)
    log_probs = log_probs.view(B, K, V) + st.run[:, :, None]                 # :3286-3287
    log_probs = log_probs.reshape(B, K * V)                                  # :3288
    topk_lp, topk_idx = _topk_stable(log_probs, M)                           # :2981
    nxt_lp, _ = _topk_stable(log_probs, M + 1)
    margin = nxt_lp[:, M - 1] - nxt_lp[:, M]                                 # how decisive the choice of the M candidates was
    beam = topk_idx // V                                                     # :2984
    tok = topk_idx % V                                                       # :2987
    seqs = torch.cat([torch.gather(st.hist, 1, beam[:, :, None].expand(B, M, t)), tok[:, :, None]], dim=2)
    hit = torch.full((B, M), t + 1 >= st.max_new)                           # :3306 MaxLengthCriteria
    for e in eos:
        hit |= tok == e                                                      # EosTokenCriteria
    # next running beams (:3013-3018)
    run_lp = topk_lp + hit.to(torch.float32) * -1.0e9
    _, nxt = _topk_stable(run_lp, K)
    st.run = torch.gather(run_lp, 1, nxt)
    parent = torch.gather(beam, 1, nxt)
    token = torch.gather(tok, 1, nxt)
    new_hist = torch.gather(seqs, 1, nxt[:, :, None].expand(B, K, t + 1))
    # finished hypotheses (:3046-3071)
    top_mask = torch.arange(M) < K
    did = hit & top_mask[None, :]
    sc = topk_lp / ((t + 1) ** length_penalty)
    full = st.fin.all(dim=-1, keepdim=True) & (early_stopping is True)
    sc += full.to(torch.float32) * -1.0e9
    sc += (~st.unsat[:, None]).to(torch.float32) * -1.0e9
    sc += (~did) * -1.0e9
    pad_seqs = torch.zeros(B, M, st.max_new, dtype=torch.long)
    pad_seqs[:, :, : t + 1] = seqs
    m_scores = torch.cat([st.scores, sc], dim=1)
    m_tokens = torch.cat([st.tokens, pad_seqs], dim=1)
    m_lens = torch.cat([st.lens, torch.full((B, M), t + 1, dtype=torch.long)], dim=1)
    m_fin = torch.cat([st.fin, did], dim=1)
    _, keep = _topk_stable(m_scores, K)
    st.scores = torch.gather(m_scores, 1, keep)
    st.tokens = torch.gather(m_tokens, 1, keep[:, :, None].expand(B, K, st.max_new))
    st.lens = torch.gather(m_lens, 1, keep)
    st.fin = torch.gather(m_fin, 1, keep)
    # early-stop heuristic at cur_len = t + 1 (:2912-2920) and each item's share of the loop condition (:2933-2943)
    cur = t + 1
    hyp_len = st.max_new if (early_stopping == "never" and length_penalty > 0.0) else cur
    best = st.run[:, :1] / (hyp_len ** length_penalty)
    worst = torch.where(st.fin, torch.min(st.scores, dim=1, keepdim=True)[0], torch.tensor(-1.0e9))
    st.unsat = st.unsat & torch.any(best > worst, dim=-1)
    st.done = st.done | ~st.unsat | (st.fin.all(-1) & (early_stopping is True)) | hit.all(-1)
    st.hist = new_hist
    return dict(parent=parent, token=token, cand=topk_idx, hit=hit, cand_scores=topk_lp, margin=margin)


def beam_output(st: BeamState, num_return_sequences: int, fill: int):
    """HF:3375-3385: the best num_return_sequences hypotheses per item, cut to the longest returned length, filled with `fill`
    (HF:3187 output_fill_value)."""
    B, R = st.B, num_return_sequences
    lens = st.lens[:, :R].reshape(-1)
    L = int(lens.max())
    out = torch.full((B * R, L), fill, dtype=torch.long)
    toks = st.tokens[:, :R].reshape(B * R, -1)
    for i in range(B * R):
        out[i, : int(lens[i])] = toks[i, : int(lens[i])]
    return out, st.scores[:, :R].reshape(-1).clone()


def output_fill_value(pad_token_id, eos_ids) -> int:
    """HF:3187 `pad_token_id or eos_token_id[0] if eos_token_id is not None else -1` (a conditional expression around the `or`)."""
    if eos_ids:
        return int(pad_token_id) if pad_token_id else int(eos_ids[0])
    return -1


def beam_search(w, cfg: PathConfig, input_ids, pixel_values, num_beams: int, max_new_tokens: int, image_at_head: bool = True,
                left_pad: Optional[torch.Tensor] = None, eos_token_id=(), pad_token_id=None, length_penalty: float = 1.0,
                early_stopping=False, num_return_sequences: int = 1, repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0,
                min_new_tokens: int = 0):
    """VisualCLAModel.generate(num_beams=K, do_sample=False) in fp32: the prompt is prefilled once per item and its KV cache
    repeated for the K beams; after every step the cache rows are gathered by parent (HF reorder_cache).
    -> (sequences (B * num_return_sequences, L) int64, scores (B * num_return_sequences,) fp32, per-step records)."""
    s0, s1, _, s3 = special_ids(cfg)
    img = vision_encode(w, cfg, pixel_values) if pixel_values is not None else None
    x = splice(w, cfg, input_ids, img, image_at_head, s0, s1, s3)
    B, K = input_ids.shape[0], num_beams
    cache = KVCache(cfg.t_layers)
    logits = llama_forward(w, cfg, x, cache, last_only=True, left_pad=left_pad)[:, -1]
    pads = None if left_pad is None else left_pad.repeat_interleave(K)
    st = BeamState(B, K, max_new_tokens)
    steps = []
    for t in range(max_new_tokens):
        r = beam_step(st, logits, t, eos_token_id, length_penalty, early_stopping, repetition_penalty, no_repeat_ngram_size, min_new_tokens)
        r["logits"] = logits
        steps.append(r)
        if bool(st.done.all()):
            break
        rows = (torch.arange(B)[:, None] * (1 if t == 0 else K) + r["parent"]).reshape(-1)
        for i in range(cfg.t_layers):
            cache.k[i] = cache.k[i].index_select(0, rows)
            cache.v[i] = cache.v[i].index_select(0, rows)
        e = w["text_model.model.embed_tokens.weight"][r["token"].reshape(-1)].float().unsqueeze(1)
        logits = llama_forward(w, cfg, e, cache, last_only=True, left_pad=pads)[:, -1]
    seqs, scores = beam_output(st, num_return_sequences, output_fill_value(pad_token_id, list(eos_token_id)))
    return seqs, scores, steps


def beam_rescore(w, cfg: PathConfig, input_ids, pixel_values, tokens: torch.Tensor, image_at_head: bool = True,
                 left_pad: Optional[torch.Tensor] = None, length_penalty: float = 1.0) -> torch.Tensor:
    """Teacher-forced score of given continuations (B, L) (no processors): sum of log_softmax over the tokens / L^length_penalty,
    the score beam search gives a finished hypothesis of that length."""
    s0, s1, _, s3 = special_ids(cfg)
    img = vision_encode(w, cfg, pixel_values) if pixel_values is not None else None
    x = splice(w, cfg, input_ids, img, image_at_head, s0, s1, s3)
    cache = KVCache(cfg.t_layers)
    logits = llama_forward(w, cfg, x, cache, last_only=True, left_pad=left_pad)[:, -1]
    total = torch.zeros(tokens.shape[0])
    for j in range(tokens.shape[1]):
        total += torch.log_softmax(logits.float(), -1).gather(1, tokens[:, j:j + 1]).squeeze(1)
        if j + 1 < tokens.shape[1]:
            e = w["text_model.model.embed_tokens.weight"][tokens[:, j]].float().unsqueeze(1)
            logits = llama_forward(w, cfg, e, cache, last_only=True, left_pad=left_pad)[:, -1]
    return total / (tokens.shape[1] ** length_penalty)
