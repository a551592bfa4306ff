"""LoRA folding at load time, without `peft` (SURVEY.md section 8f-2).

The reference ships VisualCLA-7B as LoRA deltas + full Resampler / projector / embedding / lm_head tensors in one
`adapter_model.bin` (key layout: ref scripts/inference/text_generation_webui/convert_ckpt_for_tgwebui.py:31-71; targets
`(q|k|v|o|gate|down|up)_proj` of LLaMA and the CLIP attention/MLP linears, `modules_to_save = [embed_tokens, lm_head]`)
and merges them offline with `PeftModel.merge_and_unload()` (ref scripts/merge_llama_with_visualcla_lora.py:78-85).
Here the merge  W <- W + (lora_alpha / r) * B @ A  is done while loading, on the device the weights already live on.
"""
from __future__ import annotations

import json
import os
import re
from typing import Dict, Tuple

import torch

_PREFIX = "base_model.model."


def normalise_key(k: str) -> str:
    """adapter_model.bin key -> VisualCLAModel.state_dict() key (+ '.lora_A' / '.lora_B' marker kept)."""
    if k.startswith(_PREFIX):
        k = k[len(_PREFIX):]
    k = re.sub(r"\.modules_to_save\.[^.]+\.", ".", k)       # peft >= 0.4 infix for fully-trained modules
    k = re.sub(r"\.(lora_[AB])\.[^.]+\.weight$", r".\1.weight", k)   # adapter-name infix ("default")
    k = k.replace(".original_module.", ".")
    return k


def plan(keys) -> Tuple[Dict[str, Dict[str, str]], Dict[str, str]]:
    """-> ({target weight name: {'A': key, 'B': key}}, {target name: key}) for LoRA pairs and fully-replaced tensors."""
    pairs: Dict[str, Dict[str, str]] = {}
    full: Dict[str, str] = {}
    for k in keys:
        n = normalise_key(k)
        m = re.match(r"(.*)\.lora_([AB])\.weight$", n)
        if m:
            pairs.setdefault(m.group(1) + ".weight", {})[m.group(2)] = k
        elif "lora_" in n:
            raise ValueError(f"unsupported LoRA tensor {k} (only lora_A / lora_B weights are handled)")
        else:
            full[n] = k
    for name, ab in pairs.items():
        if set(ab) != {"A", "B"}:
            raise ValueError(f"incomplete LoRA pair for {name}: {sorted(ab)}")
    return pairs, full


def fold(w: torch.Tensor, A: torch.Tensor, B: torch.Tensor, scaling: float, fan_in_fan_out: bool = False) -> torch.Tensor:
    """W + scaling * B @ A in fp32 (A: [r, in], B: [out, r])."""
    delta = (B.float() @ A.float()) * scaling
    if fan_in_fan_out:
        delta = delta.t()
    return w.float() + delta


def load_lora(model, lora_dir: str, strict: bool = True):
    """Fold an unmerged VisualCLA LoRA checkpoint directory (adapter_config.json + adapter_model.bin) into `model`.

    On a load_in_8bit model the int8 projections are folded as quantise(q * s + scaling * B @ A): the delta is added to the
    dequantised weight and the sum is quantised again.  PEFT instead keeps the delta unmerged beside the int8 base, so the two
    differ by the int8 rounding of the delta."""
    with open(os.path.join(lora_dir, "adapter_config.json")) as f:
        cfg = json.load(f)
    scaling = float(cfg["lora_alpha"]) / float(cfg["r"])
    fifo = bool(cfg.get("fan_in_fan_out", False))
    path = os.path.join(lora_dir, "adapter_model.bin")
    if os.path.exists(path):
        sd = torch.load(path, map_location="cpu", weights_only=True)
    else:
        from safetensors.torch import load_file
        sd = load_file(os.path.join(lora_dir, "adapter_model.safetensors"), device="cpu")
    pairs, full = plan(sd.keys())
    eng = model._engine
    table = {n: s for n, s, _k in eng.weight_table()}
    # vocabulary growth first (ref inference.py:69: resize_token_embeddings(len(tokenizer)) before the adapter is applied)
    emb = "text_model.model.embed_tokens.weight"
    if emb in full and sd[full[emb]].shape[0] != table[emb][0]:
        model.resize_token_embeddings(sd[full[emb]].shape[0])
        eng = model._engine
        table = {n: s for n, s, _k in eng.weight_table()}
    unknown = [n for n in list(pairs) + list(full) if n not in table and "pooler" not in n and "position_ids" not in n]
    if unknown and strict:
        raise KeyError(f"LoRA checkpoint has tensors the model does not know: {unknown[:4]} ... ({len(unknown)})")
    dev = eng.device
    for name, ab in pairs.items():
        if name not in table:
            continue
        w = eng.read_weight(name).to(dev)
        eng.load_weight(name, fold(w, sd[ab["A"]].to(dev), sd[ab["B"]].to(dev), scaling, fifo))
    for name, k in full.items():
        if name in table:
            eng.load_weight(name, sd[k])
    return {"folded": len(pairs), "replaced": sum(1 for n in full if n in table), "scaling": scaling}
