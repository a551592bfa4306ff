"""Reference of the int8 KV cache (kv_cache_dtype="int8"), shared by tests/test_kv_int8_oracle.py and tests/test_kv_int8_gpu.py.

One rule defines the model: every LLaMA K row (after RoPE) and V row is replaced, per head, by its int8 round trip the moment it is
computed -- load_in_8bit's row quantiser (oracle/int8_oracle.py:quantize) applied to the row's 128 fp32 values -- and every attention
reads q * s.  `llama_forward_q8` is oracle/visualcla_oracle.py:llama_forward with that round trip applied to k and v right after RoPE
(kv_hook=None gives llama_forward's computation, which tests/test_kv_int8_oracle.py checks bit for bit)."""
from typing import Optional

import torch
import torch.nn.functional as F

import int8_oracle as Q
import visualcla_oracle as O

HD = 128


def quantize_rows(x: torch.Tensor):
    """x (..., 128) any float dtype -> (q int8 (..., 128), s float32 (...)), the rule of int8_oracle.quantize on each row."""
    shape = x.shape
    q, s = Q.quantize(x.detach().float().reshape(-1, shape[-1]))
    return torch.from_numpy(q).view(shape), torch.from_numpy(s).view(shape[:-1])


def dequantize_rows(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """q * s in fp32 (what every attention of the int8 cache reads)."""
    return q.float() * s.float()[..., None]


def kv_round_trip(x: torch.Tensor) -> torch.Tensor:
    """The hook: x (B, H, S, 128) fp32 -> q * s of each row, fp32."""
    q, s = quantize_rows(x)
    return dequantize_rows(q, s)


def llama_forward_q8(w, cfg, embeds: torch.Tensor, cache: Optional[O.KVCache] = None, last_only: bool = False,
                     left_pad: Optional[torch.Tensor] = None, pos_from_mask: bool = True, kv_hook=kv_round_trip) -> torch.Tensor:
    """oracle llama_forward (same arguments, same operations) with k and v passed through kv_hook after RoPE."""
    tp = "text_model.model."
    B, S, T = embeds.shape
    H, hd = cfg.t_heads, cfg.t_head_dim
    past = cache.length if cache is not None else 0
    pad = torch.zeros(B, dtype=torch.long) if left_pad is None else left_pad.long()
    pos = torch.arange(past, past + S)[None, :].expand(B, S)
    if pos_from_mask:
        pos = (pos - pad[:, None]).clamp(min=0)
    cosb, sinb = O.rope_tables(cfg, pos.reshape(-1))
    cosb, sinb = cosb.view(B, 1, S, hd), sinb.view(B, 1, S, hd)
    h = embeds.float()
    scale = hd ** -0.5

    def W(name):
        t = w[name]
        return t if t.dtype == torch.float32 else t.float()

    for i in range(cfg.t_layers):
        lp = f"{tp}layers.{i}."
        r = h
        y = O.rmsnorm(h, W(lp + "input_layernorm.weight"), cfg.t_eps)
        q = (y @ W(lp + "self_attn.q_proj.weight").t()).view(B, S, H, hd).transpose(1, 2)
        k = (y @ W(lp + "self_attn.k_proj.weight").t()).view(B, S, H, hd).transpose(1, 2)
        v = (y @ W(lp + "self_attn.v_proj.weight").t()).view(B, S, H, hd).transpose(1, 2)
        q = O.apply_rope(q, cosb, sinb)
        k = O.apply_rope(k, cosb, sinb)
        if kv_hook is not None:
            k, v = kv_hook(k), kv_hook(v)
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
        p = torch.nan_to_num(p, nan=0.0)
        a = torch.matmul(p, v).transpose(1, 2).reshape(B, S, T)
        h = r + a @ W(lp + "self_attn.o_proj.weight").t()
        r = h
        y = O.rmsnorm(h, W(lp + "post_attention_layernorm.weight"), cfg.t_eps)
        g = y @ W(lp + "mlp.gate_proj.weight").t()
        u = y @ W(lp + "mlp.up_proj.weight").t()
        h = r + (F.silu(g) * u) @ W(lp + "mlp.down_proj.weight").t()
    if last_only:
        h = h[:, -1:, :]
    h = O.rmsnorm(h, W(tp + "norm.weight"), cfg.t_eps)
    return h @ W("text_model.lm_head.weight").t()


def generate_greedy_q8(w, cfg, input_ids, pixel_values, max_new_tokens: int, image_at_head: bool = True, kv_hook=kv_round_trip,
                       forced_tokens: Optional[torch.Tensor] = None, left_pad: Optional[torch.Tensor] = None, cache=None):
    """oracle generate_greedy on llama_forward_q8: (new tokens (B, N), logits (B, N, V)).  `cache` (a KVCache) receives the K/V."""
    s0, s1, _, s3 = O.special_ids(cfg)
    img = O.vision_encode(w, cfg, pixel_values) if pixel_values is not None else None
    x = O.splice(w, cfg, input_ids, img, image_at_head, s0, s1, s3)
    cache = O.KVCache(cfg.t_layers) if cache is None else cache
    logits = llama_forward_q8(w, cfg, x, cache, last_only=True, left_pad=left_pad, kv_hook=kv_hook)[:, -1]
    toks, logs = [], []
    for step in range(max_new_tokens):
        nxt = logits.argmax(-1)
        toks.append(nxt)
        logs.append(logits)
        if step == max_new_tokens - 1:
            break
        feed = nxt if forced_tokens is None else forced_tokens[:, step]
        e = w["text_model.model.embed_tokens.weight"][feed].float().unsqueeze(1)
        logits = llama_forward_q8(w, cfg, e, cache, last_only=True, left_pad=left_pad, kv_hook=kv_hook)[:, -1]
    return torch.stack(toks, 1), torch.stack(logs, 1)


def split_pool(raw: torch.Tensor, total_pages: int, H: int, pt: int):
    """A layer's int8 pool bytes (uint8) -> (q int8 [pages][2][H][pt][128], s float32 [pages][2][H][pt]) views."""
    n_rows = total_pages * 2 * H * pt
    q = raw[:n_rows * HD].view(torch.int8).view(total_pages, 2, H, pt, HD)
    s = raw[n_rows * HD:n_rows * (HD + 4)].view(torch.float32).view(total_pages, 2, H, pt)
    return q, s


def pool_bytes(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """Inverse of split_pool: one contiguous uint8 buffer (int8 rows, then fp32 scales)."""
    return torch.cat([q.contiguous().view(torch.uint8).reshape(-1), s.contiguous().view(torch.uint8).reshape(-1)])


def ulp_distance(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """|a - b| in units in the last place of fp32 (same-sign finite values)."""
    ai = a.contiguous().view(torch.int32).long()
    bi = b.contiguous().view(torch.int32).long()
    return (ai - bi).abs()


__all__ = ["quantize_rows", "dequantize_rows", "kv_round_trip", "llama_forward_q8", "generate_greedy_q8", "split_pool", "pool_bytes",
           "ulp_distance"]
