"""CPU oracle for the VisualCLA multimodal forward path  --  TEST INFRASTRUCTURE ONLY.

This file is a plain fp32 CPU restatement (torch CPU tensor ops, no nn.Module,
no HF classes) of the one hot path this repo accelerates:

    image + prompt -> CLIP-ViT-L/14 -> post_layernorm -> 6-layer Resampler
    -> projector -> splice into text embeddings -> LLaMA prefill + greedy decode

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` legs may import it.  The product package
(`visual-chinese-llama-alpaca_b200/visualcla`) never does.

Pinning status: the reference repo has no tests / golden vectors of its own
(SURVEY.md section 4, 8c).  This oracle is pinned against *outputs of the reference
itself* run in the authoring container: `oracle/gen_golden.py` imports the
unmodified reference (`models/visualcla` of a reference checkout, behind the import shim
in `oracle/ref_shim.py`) plus HF transformers 5.5.0 CLIP/LLaMA, runs
`VisualCLAModel.forward/.generate` on seeded weights and writes
`tests/golden/*.npz`; `tests/test_oracle_golden.py` checks this restatement
against those files.

Every function cites the reference lines it restates.  `ref:` paths are relative
to the reference repository's root, `HF:` paths to site-packages/transformers (5.5.0).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field, asdict
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------
# host threads: torch's intra-op pool degrades badly when os.cpu_count() exceeds the cores this process
# may actually use (observed: 128 "cpus" on the GPU box -> 30x slower than 8 threads) -> calibrate once
# --------------------------------------------------------------------------------------
_THREADS = None


def pick_threads(candidates=(8, 16, 32, 64)) -> int:
    """Set torch's intra-op thread count to the fastest of `candidates` for a 7B-shaped matmul; returns it."""
    global _THREADS
    if _THREADS is not None:
        torch.set_num_threads(_THREADS)
        return _THREADS
    import os
    import time
    try:
        avail = len(os.sched_getaffinity(0))
    except Exception:
        avail = os.cpu_count() or 1
    a, b = torch.randn(256, 4096), torch.randn(4096, 4096)
    best, best_t = 1, float("inf")
    for n in sorted({c for c in candidates if c <= avail} | {min(avail, 8)}):
        torch.set_num_threads(n)
        a @ b
        t0 = time.perf_counter()
        for _ in range(3):
            a @ b
        dt = time.perf_counter() - t0
        if dt < best_t * 0.95:
            best, best_t = n, dt
    _THREADS = best
    torch.set_num_threads(best)
    return best


# --------------------------------------------------------------------------------------
# configuration
# --------------------------------------------------------------------------------------
@dataclass
class PathConfig:
    """Shapes of the path.  Defaults = VisualCLA-7B-v0.1 (SURVEY.md section 8 constants)."""
    # CLIP-ViT-L/14  (HF:models/clip/modeling_clip.py:138-219,354-386,647-692)
    v_hidden: int = 1024
    v_layers: int = 24
    v_heads: int = 16
    v_ffn: int = 4096
    v_patch: int = 14
    v_image: int = 224
    v_eps: float = 1e-5
    # Resampler (ref: models/visualcla/modeling_visual_resampler.py:90-129)
    r_hidden: int = 1024
    r_layers: int = 6
    r_heads: int = 16
    r_ffn: int = 4096
    r_queries: int = 64
    r_eps: float = 1e-12
    # LLaMA-7B (HF:models/llama/modeling_llama.py)
    t_hidden: int = 4096
    t_layers: int = 32
    t_heads: int = 32
    t_ffn: int = 11008
    t_vocab: int = 49958
    t_eps: float = 1e-6
    rope_theta: float = 10000.0

    @property
    def v_tokens(self) -> int:
        return (self.v_image // self.v_patch) ** 2 + 1

    @property
    def t_head_dim(self) -> int:
        return self.t_hidden // self.t_heads

    def to_dict(self):
        return asdict(self)


def tiny_config() -> PathConfig:
    """Small config used for the golden fixtures (keeps the kernel-specialised head dims:
    64 for ViT/Resampler, 128 for LLaMA; deliberately awkward vocab / ffn sizes)."""
    return PathConfig(
        v_hidden=128, v_layers=2, v_heads=2, v_ffn=256, v_patch=14, v_image=56,
        r_hidden=128, r_layers=2, r_heads=2, r_ffn=320, r_queries=8,
        t_hidden=256, t_layers=2, t_heads=2, t_ffn=448, t_vocab=1003,
    )


# --------------------------------------------------------------------------------------
# deterministic synthetic weights (integer hash -> Irwin-Hall(4) pseudo-normal)
# bit-identical to the device generator `fill_hash_normal_kernel` in csrc/elementwise.cu (pure integer
# arithmetic + one fp32 multiply + one fp32 add + RNE round to bf16).
# --------------------------------------------------------------------------------------
_IH_SIGMA = 65536.0 / math.sqrt(3.0)      # std of the sum of four uniform u16


def fnv1a32(name: str) -> int:
    h = 0x811C9DC5
    for c in name.encode("utf-8"):
        h ^= c
        h = (h * 0x01000193) & 0xFFFFFFFF
    return h


def _fmix32(h: np.ndarray) -> np.ndarray:
    h = h.copy()
    h ^= h >> np.uint32(16)
    h *= np.uint32(0x85EBCA6B)
    h ^= h >> np.uint32(13)
    h *= np.uint32(0xC2B2AE35)
    h ^= h >> np.uint32(16)
    return h


def hash_normal_bf16(name: str, numel: int, scale: float, seed: int = 0, offset: float = 0.0) -> torch.Tensor:
    """numel pseudo-normal values, std ~= scale, mean = offset, rounded to bf16; returned as
    fp32 holding exactly the bf16 values."""
    with np.errstate(over="ignore"):
        s = np.uint32((fnv1a32(name) ^ (seed * 0x9E3779B1)) & 0xFFFFFFFF)
        idx = np.arange(numel, dtype=np.uint32)
        a = _fmix32(idx * np.uint32(0x9E3779B1) + s)
        b = _fmix32(a ^ np.uint32(0x7F4A7C15))
    tot = ((a & np.uint32(0xFFFF)).astype(np.int64) + (a >> np.uint32(16)).astype(np.int64)
           + (b & np.uint32(0xFFFF)).astype(np.int64) + (b >> np.uint32(16)).astype(np.int64) - 131070)
    mul = np.float32(scale / _IH_SIGMA)
    val = tot.astype(np.float32) * mul + np.float32(offset)
    t = torch.from_numpy(val.astype(np.float32))
    return t.to(torch.bfloat16).to(torch.float32)


def weight_specs(cfg: PathConfig) -> List[Tuple[str, Tuple[int, ...], float, float]]:
    """(state-dict name, shape, std, mean) for every tensor on the path.  Names are the
    reference's `VisualCLAModel.state_dict()` keys (ref: modeling_visualcla.py:70-108;
    merged-dir layout ref: scripts/merge_llama_with_visualcla_lora.py:92-97).
    Scales are fan-in based so activations stay O(1) and attention is non-uniform
    (a std-0.02 init makes every softmax flat and hides bugs)."""
    sp: List[Tuple[str, Tuple[int, ...], float, float]] = []
    D, Fv = cfg.v_hidden, cfg.v_ffn
    vp = "vision_model.vision_model."
    kpatch = 3 * cfg.v_patch * cfg.v_patch
    sp.append((vp + "embeddings.class_embedding", (D,), 1.0, 0.0))
    sp.append((vp + "embeddings.patch_embedding.weight", (D, 3, cfg.v_patch, cfg.v_patch), 1.0 / math.sqrt(kpatch), 0.0))
    sp.append((vp + "embeddings.position_embedding.weight", (cfg.v_tokens, D), 0.5, 0.0))
    sp.append((vp + "pre_layrnorm.weight", (D,), 0.1, 1.0))
    sp.append((vp + "pre_layrnorm.bias", (D,), 0.1, 0.0))
    for i in range(cfg.v_layers):
        lp = f"{vp}encoder.layers.{i}."
        for ln in ("layer_norm1", "layer_norm2"):
            sp.append((lp + ln + ".weight", (D,), 0.1, 1.0))
            sp.append((lp + ln + ".bias", (D,), 0.1, 0.0))
        for pr in ("q_proj", "k_proj", "v_proj"):
            sp.append((lp + f"self_attn.{pr}.weight", (D, D), 1.5 / math.sqrt(D), 0.0))
            sp.append((lp + f"self_attn.{pr}.bias", (D,), 0.1, 0.0))
        sp.append((lp + "self_attn.out_proj.weight", (D, D), 0.5 / math.sqrt(D), 0.0))
        sp.append((lp + "self_attn.out_proj.bias", (D,), 0.05, 0.0))
        sp.append((lp + "mlp.fc1.weight", (Fv, D), 1.0 / math.sqrt(D), 0.0))
        sp.append((lp + "mlp.fc1.bias", (Fv,), 0.1, 0.0))
        sp.append((lp + "mlp.fc2.weight", (D, Fv), 0.5 / math.sqrt(Fv), 0.0))
        sp.append((lp + "mlp.fc2.bias", (D,), 0.05, 0.0))
    sp.append((vp + "post_layernorm.weight", (D,), 0.1, 1.0))
    sp.append((vp + "post_layernorm.bias", (D,), 0.1, 0.0))

    R, Fr = cfg.r_hidden, cfg.r_ffn
    rp = "visual_resampler."
    sp.append((rp + "query_embeddding", (1, cfg.r_queries, R), 1.0, 0.0))
    for i in range(cfg.r_layers):
        lp = f"{rp}encoder.layer.{i}."
        for pr in ("query", "key", "value"):
            sp.append((lp + f"crossattention.self.{pr}.weight", (R, R), 1.5 / math.sqrt(R), 0.0))
            sp.append((lp + f"crossattention.self.{pr}.bias", (R,), 0.1, 0.0))
        sp.append((lp + "crossattention.output.dense.weight", (R, R), 1.0 / math.sqrt(R), 0.0))
        sp.append((lp + "crossattention.output.dense.bias", (R,), 0.05, 0.0))
        sp.append((lp + "crossattention.output.LayerNorm.weight", (R,), 0.1, 1.0))
        sp.append((lp + "crossattention.output.LayerNorm.bias", (R,), 0.1, 0.0))
        sp.append((lp + "intermediate.dense.weight", (Fr, R), 1.0 / math.sqrt(R), 0.0))
        sp.append((lp + "intermediate.dense.bias", (Fr,), 0.1, 0.0))
        sp.append((lp + "output.dense.weight", (R, Fr), 1.0 / math.sqrt(Fr), 0.0))
        sp.append((lp + "output.dense.bias", (R,), 0.05, 0.0))
        sp.append((lp + "output.LayerNorm.weight", (R,), 0.1, 1.0))
        sp.append((lp + "output.LayerNorm.bias", (R,), 0.1, 0.0))
    sp.append(("image_projection_layer.weight", (cfg.t_hidden, R), 1.0 / math.sqrt(R), 0.0))
    sp.append(("image_projection_layer.bias", (cfg.t_hidden,), 0.1, 0.0))

    T, Ft, V = cfg.t_hidden, cfg.t_ffn, cfg.t_vocab
    tp = "text_model.model."
    res_gain = 1.0 / math.sqrt(2.0 * cfg.t_layers)
    sp.append((tp + "embed_tokens.weight", (V, T), 1.0, 0.0))
    for i in range(cfg.t_layers):
        lp = f"{tp}layers.{i}."
        sp.append((lp + "input_layernorm.weight", (T,), 0.1, 1.0))
        sp.append((lp + "post_attention_layernorm.weight", (T,), 0.1, 1.0))
        for pr in ("q_proj", "k_proj"):
            sp.append((lp + f"self_attn.{pr}.weight", (T, T), 1.5 / math.sqrt(T), 0.0))
        sp.append((lp + "self_attn.v_proj.weight", (T, T), 1.0 / math.sqrt(T), 0.0))
        sp.append((lp + "self_attn.o_proj.weight", (T, T), res_gain * 2.0 / math.sqrt(T), 0.0))
        sp.append((lp + "mlp.gate_proj.weight", (Ft, T), 1.0 / math.sqrt(T), 0.0))
        sp.append((lp + "mlp.up_proj.weight", (Ft, T), 1.0 / math.sqrt(T), 0.0))
        sp.append((lp + "mlp.down_proj.weight", (T, Ft), res_gain * 4.0 / math.sqrt(Ft), 0.0))
    sp.append((tp + "norm.weight", (T,), 0.1, 1.0))
    sp.append(("text_model.lm_head.weight", (V, T), 4.0 / math.sqrt(T), 0.0))
    return sp


def make_weights(cfg: PathConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    out = {}
    for name, shape, std, mean in weight_specs(cfg):
        n = int(np.prod(shape))
        out[name] = hash_normal_bf16(name, n, std, seed, mean).reshape(shape)
    return out


def make_inputs(cfg: PathConfig, batch: int, t_text: int, seed: int = 1234,
                img_start_id: Optional[int] = None, img_end_id: Optional[int] = None):
    """Synthetic inputs of SURVEY.md section 8(d): randn pixels, ids = [BOS, <img>, </img>, random...]."""
    g = torch.Generator().manual_seed(seed)
    pixels = torch.randn(batch, 3, cfg.v_image, cfg.v_image, generator=g)
    pixels = pixels.to(torch.bfloat16).to(torch.float32)
    V = cfg.t_vocab
    img_start_id = V - 4 if img_start_id is None else img_start_id
    img_end_id = V - 3 if img_end_id is None else img_end_id
    ids = torch.empty(batch, t_text, dtype=torch.long)
    for b in range(batch):
        gb = torch.Generator().manual_seed(seed + 1 + b)
        ids[b] = torch.randint(3, V - 4, (t_text,), generator=gb)
    ids[:, 0] = 1
    ids[:, 1] = img_start_id
    ids[:, 2] = img_end_id
    return pixels, ids


# --------------------------------------------------------------------------------------
# CLIP vision tower
# --------------------------------------------------------------------------------------
def quick_gelu(x: torch.Tensor) -> torch.Tensor:
    # HF:activations.py QuickGELUActivation: x * sigmoid(1.702 x)
    return x * torch.sigmoid(1.702 * x)


def _mha(q, k, v, heads: int, scale: float, causal: bool = False):
    """softmax(q k^T * scale) v, fp32.  q (B,Sq,D), k/v (B,Sk,D)."""
    B, Sq, D = q.shape
    Sk = k.shape[1]
    hd = D // heads
    qh = q.view(B, Sq, heads, hd).transpose(1, 2)
    kh = k.view(B, Sk, heads, hd).transpose(1, 2)
    vh = v.view(B, Sk, heads, hd).transpose(1, 2)
    s = torch.matmul(qh, kh.transpose(-1, -2)) * scale
    if causal:
        off = Sk - Sq
        m = torch.ones(Sq, Sk, dtype=torch.bool).tril(diagonal=off)
        s = s.masked_fill(~m, float("-inf"))
    p = torch.softmax(s, dim=-1)
    o = torch.matmul(p, vh)
    return o.transpose(1, 2).reshape(B, Sq, D)


def clip_vision_forward(w: Dict[str, torch.Tensor], cfg: PathConfig, pixel_values: torch.Tensor) -> torch.Tensor:
    """CLIPVisionModel(pixel_values)[0]  == last_hidden_state BEFORE post_layernorm.
    HF:models/clip/modeling_clip.py:202-218 (embeddings), :677 (pre_layrnorm),
    :363-385 (encoder layer, pre-LN), :262-279 (attention), :343-351 (MLP).
    Called at ref: models/visualcla/modeling_visualcla.py:283/349."""
    vp = "vision_model.vision_model."
    B = pixel_values.shape[0]
    D = cfg.v_hidden
    # patch embedding: Conv2d(3, D, k=p, s=p, bias=False) == unfold + matmul  (:148-154,:208-210)
    P = cfg.v_patch
    g = cfg.v_image // P
    x = pixel_values.float().view(B, 3, g, P, g, P).permute(0, 2, 4, 1, 3, 5).reshape(B, g * g, 3 * P * P)
    wp = w[vp + "embeddings.patch_embedding.weight"].reshape(D, 3 * P * P)
    patches = x @ wp.t()
    cls = w[vp + "embeddings.class_embedding"].view(1, 1, D).expand(B, 1, D)
    h = torch.cat([cls, patches], dim=1) + w[vp + "embeddings.position_embedding.weight"].unsqueeze(0)  # :212-217
    h = F.layer_norm(h, (D,), w[vp + "pre_layrnorm.weight"], w[vp + "pre_layrnorm.bias"], cfg.v_eps)   # :677
    scale = (D // cfg.v_heads) ** -0.5
    for i in range(cfg.v_layers):
        lp = f"{vp}encoder.layers.{i}."
        r = h
        y = F.layer_norm(h, (D,), w[lp + "layer_norm1.weight"], w[lp + "layer_norm1.bias"], cfg.v_eps)
        q = y @ w[lp + "self_attn.q_proj.weight"].t() + w[lp + "self_attn.q_proj.bias"]
        k = y @ w[lp + "self_attn.k_proj.weight"].t() + w[lp + "self_attn.k_proj.bias"]
        v = y @ w[lp + "self_attn.v_proj.weight"].t() + w[lp + "self_attn.v_proj.bias"]
        a = _mha(q, k, v, cfg.v_heads, scale)
        a = a @ w[lp + "self_attn.out_proj.weight"].t() + w[lp + "self_attn.out_proj.bias"]
        h = r + a
        r = h
        y = F.layer_norm(h, (D,), w[lp + "layer_norm2.weight"], w[lp + "layer_norm2.bias"], cfg.v_eps)
        y = quick_gelu(y @ w[lp + "mlp.fc1.weight"].t() + w[lp + "mlp.fc1.bias"])
        y = y @ w[lp + "mlp.fc2.weight"].t() + w[lp + "mlp.fc2.bias"]
        h = r + y
    return h


def clip_post_layernorm(w, cfg: PathConfig, h: torch.Tensor) -> torch.Tensor:
    """ref: modeling_visualcla.py:284/350 -- post_layernorm applied by the *reference* to all tokens."""
    vp = "vision_model.vision_model."
    return F.layer_norm(h, (cfg.v_hidden,), w[vp + "post_layernorm.weight"], w[vp + "post_layernorm.bias"], cfg.v_eps)


# --------------------------------------------------------------------------------------
# Resampler  (the only arithmetic that lives in the reference tree)
# --------------------------------------------------------------------------------------
def resampler_forward(w, cfg: PathConfig, image_tokens: torch.Tensor) -> torch.Tensor:
    """VisualResamplerModel(encoder_hidden_states=image_tokens).last_hidden_state
    ref: modeling_visual_resampler.py:609-737.  Per layer (:371-416):
      kv_src = cat([queries, image_tokens])                     (:315)
      Q = query(h); K = key(kv_src); V = value(kv_src)          (:174,:186-189)
      ctx = softmax(Q K^T / sqrt(hd) + 0) V                     (:213,:237,:240,:243,:253)
      h = LN(dense(ctx) + h)                                    (:273-277)
      h = LN(dense2(gelu(dense1(h))) + h)                       (:340-343,:353-357)
    masks are identically zero (:672-694), dropout is identity in eval, pooler (:725) is
    dead compute (only .last_hidden_state is read, ref: modeling_visualcla.py:287/353)."""
    rp = "visual_resampler."
    B = image_tokens.shape[0]
    R = cfg.r_hidden
    h = w[rp + "query_embeddding"].expand(B, -1, -1)          # :661
    scale = 1.0 / math.sqrt(R // cfg.r_heads)
    for i in range(cfg.r_layers):
        lp = f"{rp}encoder.layer.{i}."
        src = torch.cat([h, image_tokens], dim=1)
        q = h @ w[lp + "crossattention.self.query.weight"].t() + w[lp + "crossattention.self.query.bias"]
        k = src @ w[lp + "crossattention.self.key.weight"].t() + w[lp + "crossattention.self.key.bias"]
        v = src @ w[lp + "crossattention.self.value.weight"].t() + w[lp + "crossattention.self.value.bias"]
        ctx = _mha(q, k, v, cfg.r_heads, scale)
        a = ctx @ w[lp + "crossattention.output.dense.weight"].t() + w[lp + "crossattention.output.dense.bias"]
        h = F.layer_norm(a + h, (R,), w[lp + "crossattention.output.LayerNorm.weight"],
                         w[lp + "crossattention.output.LayerNorm.bias"], cfg.r_eps)
        y = F.gelu(h @ w[lp + "intermediate.dense.weight"].t() + w[lp + "intermediate.dense.bias"])   # erf gelu
        y = y @ w[lp + "output.dense.weight"].t() + w[lp + "output.dense.bias"]
        h = F.layer_norm(y + h, (R,), w[lp + "output.LayerNorm.weight"], w[lp + "output.LayerNorm.bias"], cfg.r_eps)
    return h


def project(w, image_embeds: torch.Tensor) -> torch.Tensor:
    """ref: modeling_visualcla.py:288/354  image_projection_layer (Linear R -> T, with bias)."""
    return image_embeds @ w["image_projection_layer.weight"].t() + w["image_projection_layer.bias"]


def vision_encode(w, cfg: PathConfig, pixel_values: torch.Tensor, stages: Optional[dict] = None) -> torch.Tensor:
    """pixels -> (B, r_queries, t_hidden) image embeddings (ref: modeling_visualcla.py:346-354)."""
    vit = clip_vision_forward(w, cfg, pixel_values)
    post = clip_post_layernorm(w, cfg, vit)
    res = resampler_forward(w, cfg, post)
    proj = project(w, res)
    if stages is not None:
        stages.update(vit_out=vit, post_ln=post, resampler_out=res, projector_out=proj)
    return proj


# --------------------------------------------------------------------------------------
# splice (ref: modeling_visualcla.py:290-312 / :356-377)
# --------------------------------------------------------------------------------------
def splice(w, cfg: PathConfig, input_ids: torch.Tensor, image_embeds: Optional[torch.Tensor],
           image_at_head: bool, img_start_id: int, img_end_id: int, img_token_id: int) -> torch.Tensor:
    emb = w["text_model.model.embed_tokens.weight"][input_ids]          # :280/346
    if image_embeds is None:
        return emb
    if image_at_head:
        return torch.cat([emb[:, :2], image_embeds, emb[:, 2:]], dim=1)  # :291/357
    outs = []
    nq = image_embeds.shape[1]
    for b in range(input_ids.shape[0]):                                    # :293-305/:359-370
        pos = torch.where(input_ids[b] == img_start_id)[0]
        if len(pos) == 0:
            outs.append(emb[b])
            continue
        p = int(pos[0])
        if int(input_ids[b, p + nq + 1]) != img_end_id:
            raise ValueError(f"Num of patch ({nq}) is not equal to the length of pre-filled image patch tokens.")
        outs.append(torch.cat([emb[b, :p + 1], image_embeds[b], emb[b, p + nq + 1:]], dim=0))
    return torch.stack(outs, dim=0)


# --------------------------------------------------------------------------------------
# LLaMA
# --------------------------------------------------------------------------------------
def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    # HF:models/llama/modeling_llama.py:62-67
    var = x.pow(2).mean(-1, keepdim=True)
    return weight * (x * torch.rsqrt(var + eps))


def rope_tables(cfg: PathConfig, positions: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    # HF:models/llama/modeling_llama.py:98-141 (default rope, fp32)
    hd = cfg.t_head_dim
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))
    fr = positions.float()[:, None] * inv[None, :]
    emb = torch.cat([fr, fr], dim=-1)
    return emb.cos(), emb.sin()


def apply_rope(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """x (B,H,S,hd); cos/sin (S,hd) or (B,1,S,hd).  HF:models/llama/modeling_llama.py:144-170 (rotate_half)."""
    h = x.shape[-1] // 2
    rot = torch.cat([-x[..., h:], x[..., :h]], dim=-1)
    return x * cos + rot * sin


class KVCache:
    def __init__(self, n_layers: int):
        self.k: List[Optional[torch.Tensor]] = [None] * n_layers
        self.v: List[Optional[torch.Tensor]] = [None] * n_layers

    @property
    def length(self) -> int:
        return 0 if self.k[0] is None else self.k[0].shape[2]


def llama_forward(w, cfg: PathConfig, embeds: torch.Tensor, cache: Optional[KVCache] = None,
                  last_only: bool = False, weights_bf16: Optional[dict] = None,
                  left_pad: Optional[torch.Tensor] = None, pos_from_mask: bool = True) -> torch.Tensor:
    """LlamaForCausalLM.forward(inputs_embeds=...) with causal mask.  Without `left_pad`: position_ids = arange
    (equal-length, unpadded prompts).  HF:models/llama/modeling_llama.py:375-425 (model),
    :303-332 (layer), :251-289 (attention), :173-186 (MLP), :486-487 (lm_head).
    With a cache: appends K,V (HF:cache_utils.py:119-120) and attends over past+new.
    `left_pad` (B,) = number of left padding tokens per sequence (attention_mask = [0]*p + [1]*(S-p)): pad keys are
    masked; with pos_from_mask (what generate() does: position_ids = attention_mask.cumsum(-1) - 1,
    HF:generation/utils.py prepare_inputs_for_generation) real tokens are numbered from 0, otherwise (plain forward(), which
    the reference calls without position_ids, ref: modeling_visualcla.py:321-328) positions are arange(S)."""
    tp = "text_model.model."
    B, S, T = embeds.shape
    H, hd = cfg.t_heads, cfg.t_head_dim
    past = cache.length if cache is not None else 0
    pad = torch.zeros(B, dtype=torch.long) if left_pad is None else left_pad.long()
    pos = torch.arange(past, past + S)[None, :].expand(B, S)
    if pos_from_mask:
        pos = (pos - pad[:, None]).clamp(min=0)
    cosb, sinb = rope_tables(cfg, pos.reshape(-1))
    cosb, sinb = cosb.view(B, 1, S, hd), sinb.view(B, 1, S, hd)
    h = embeds.float()
    scale = hd ** -0.5

    def W(name):
        t = w[name]
        return t if t.dtype == torch.float32 else t.float()

    for i in range(cfg.t_layers):
        lp = f"{tp}layers.{i}."
        r = h
        y = rmsnorm(h, W(lp + "input_layernorm.weight"), cfg.t_eps)
        q = (y @ W(lp + "self_attn.q_proj.weight").t()).view(B, S, H, hd).transpose(1, 2)
        k = (y @ W(lp + "self_attn.k_proj.weight").t()).view(B, S, H, hd).transpose(1, 2)
        v = (y @ W(lp + "self_attn.v_proj.weight").t()).view(B, S, H, hd).transpose(1, 2)
        q = apply_rope(q, cosb, sinb)
        k = apply_rope(k, cosb, sinb)
        if cache is not None:
            if cache.k[i] is not None:
                k = torch.cat([cache.k[i], k], dim=2)
                v = torch.cat([cache.v[i], v], dim=2)
            cache.k[i], cache.v[i] = k, v
        Sk = k.shape[2]
        s = torch.matmul(q, k.transpose(-1, -2)) * scale
        visible = torch.ones(S, Sk, dtype=torch.bool).tril(diagonal=Sk - S)[None, None]
        if left_pad is not None:
            visible = visible & (torch.arange(Sk)[None, :] >= pad[:, None])[:, None, None, :]
        s = s.masked_fill(~visible, float("-inf"))
        p = torch.softmax(s, dim=-1)
        p = torch.nan_to_num(p, nan=0.0)          # fully masked rows (queries inside the padding) produce garbage in HF; zero here
        a = torch.matmul(p, v).transpose(1, 2).reshape(B, S, T)
        h = r + a @ W(lp + "self_attn.o_proj.weight").t()
        r = h
        y = rmsnorm(h, W(lp + "post_attention_layernorm.weight"), cfg.t_eps)
        g = y @ W(lp + "mlp.gate_proj.weight").t()
        u = y @ W(lp + "mlp.up_proj.weight").t()
        h = r + (F.silu(g) * u) @ W(lp + "mlp.down_proj.weight").t()
    if last_only:
        h = h[:, -1:, :]
    h = rmsnorm(h, W(tp + "norm.weight"), cfg.t_eps)
    return h @ W("text_model.lm_head.weight").t()


# --------------------------------------------------------------------------------------
# the two public entry points of the path
# --------------------------------------------------------------------------------------
def special_ids(cfg: PathConfig) -> Tuple[int, int, int, int]:
    """(<img>, </img>, <pad>, <img_token>) = the 4 ids appended to the base vocab
    (ref: modeling_utils.py:95-102; visualcla.py:146-148 pins <img_token>=49957)."""
    V = cfg.t_vocab
    return V - 4, V - 3, V - 2, V - 1


def forward_logits(w, cfg: PathConfig, input_ids, pixel_values, image_at_head: bool = True,
                   stages: Optional[dict] = None) -> torch.Tensor:
    """VisualCLAModel.forward(...).logits  (ref: modeling_visualcla.py:264-330)."""
    s0, s1, _, s3 = special_ids(cfg)
    img = vision_encode(w, cfg, pixel_values, stages) if pixel_values is not None else None
    x = splice(w, cfg, input_ids, img, image_at_head, s0, s1, s3)
    if stages is not None:
        stages["inputs_embeds"] = x
    return llama_forward(w, cfg, x)


def causal_lm_loss(logits: torch.Tensor, labels: torch.Tensor, n_image_rows: int = 0) -> torch.Tensor:
    """forward(labels=...).loss.  In the image_at_head layout the reference widens the labels with -100 over the image block
    after the first label (ref: modeling_visualcla.py:313-315); LlamaForCausalLM then shifts by one and averages the
    cross-entropy over the positions whose label is not -100 (HF:models/llama/modeling_llama.py:489-491 ->
    HF:loss/loss_utils.py ForCausalLMLoss: logits upcast to fp32, labels padded with -100 and shifted, mean reduction)."""
    if n_image_rows > 0:
        fill = torch.full((labels.shape[0], n_image_rows), -100, dtype=labels.dtype)
        labels = torch.cat([labels[:, :1], fill, labels[:, 1:]], dim=1)
    lg = logits.float()[:, :-1].reshape(-1, logits.shape[-1])
    tgt = labels[:, 1:].reshape(-1)
    keep = tgt != -100
    logp = torch.log_softmax(lg[keep], dim=-1)
    return -(logp.gather(1, tgt[keep].unsqueeze(1)).squeeze(1)).mean()


def generate_greedy(w, cfg: PathConfig, input_ids, pixel_values, max_new_tokens: int,
                    image_at_head: bool = True, forced_tokens: Optional[torch.Tensor] = None,
                    return_logits: bool = True, left_pad: Optional[torch.Tensor] = None):
    """VisualCLAModel.generate(do_sample=False, eos disabled): returns ONLY the new tokens
    (ref: modeling_visualcla.py:333-392 -> HF:generation/utils.py:2658-2810, argmax of the
    fp32 copy of the last-position logits :2762,:2793).
    Returns (tokens (B,N) int64, logits (B,N,V) fp32 or None).  With forced_tokens the
    oracle is teacher-forced (its own argmax is still what `tokens` reports)."""
    s0, s1, _, s3 = special_ids(cfg)
    img = vision_encode(w, cfg, pixel_values) if pixel_values is not None else None
    x = splice(w, cfg, input_ids, img, image_at_head, s0, s1, s3)
    cache = KVCache(cfg.t_layers)
    logits = llama_forward(w, cfg, x, cache, last_only=True, left_pad=left_pad)[:, -1]
    toks, logs = [], []
    for step in range(max_new_tokens):
        nxt = logits.argmax(-1)
        toks.append(nxt)
        if return_logits:
            logs.append(logits)
        if step == max_new_tokens - 1:
            break
        feed = nxt if forced_tokens is None else forced_tokens[:, step]
        e = w["text_model.model.embed_tokens.weight"][feed].float().unsqueeze(1)
        logits = llama_forward(w, cfg, e, cache, last_only=True, left_pad=left_pad)[:, -1]
    return torch.stack(toks, 1), (torch.stack(logs, 1) if return_logits else None)
