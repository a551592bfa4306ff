"""fp32 restatement of the weight-only int8 quantiser of load_in_8bit (csrc/quant.cu), in the same operation order:

    a = max_k |w[r, k]|           (fp32; w = the source tensor converted to fp32)
    s = a / 127                   (fp32, round to nearest)
    q = clamp(rint(w * (127 / a)), -127, 127)    (127 / a in fp32, the product in fp32, rint = round half to even)
    a == 0: s = 0, q = 0

The effective weight is q * s.  `quantized_weights` turns an oracle weight dict into the one the int8 engine computes with: the seven
LLaMA projections of every layer replaced by q * s, everything else unchanged (what bitsandbytes converts under load_in_8bit, minus
its activation-outlier decomposition)."""
from typing import Dict, Tuple

import numpy as np
import torch

Q8_SUFFIXES = ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight", "self_attn.o_proj.weight",
               "mlp.gate_proj.weight", "mlp.up_proj.weight", "mlp.down_proj.weight")


def is_q8(name: str) -> bool:
    return name.startswith("text_model.model.layers.") and name.endswith(Q8_SUFFIXES)


def quantize(w) -> Tuple[np.ndarray, np.ndarray]:
    """w: (rows, cols) array / tensor of any float dtype -> (q int8 (rows, cols), s float32 (rows,))."""
    if isinstance(w, torch.Tensor):
        w = w.detach().float().cpu().numpy()
    w = np.asarray(w, dtype=np.float32)
    a = np.max(np.abs(w), axis=1).astype(np.float32)
    s = (a / np.float32(127.0)).astype(np.float32)
    with np.errstate(divide="ignore"):
        inv = np.where(a > 0, np.float32(127.0) / a, np.float32(0.0)).astype(np.float32)
    q = np.clip(np.rint((w * inv[:, None]).astype(np.float32)), -127, 127).astype(np.int8)
    return q, s


def dequantize(q: np.ndarray, s: np.ndarray) -> np.ndarray:
    return (q.astype(np.float32) * s.astype(np.float32)[:, None]).astype(np.float32)


def quantized_weights(w: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    out = {}
    for k, v in w.items():
        if is_q8(k):
            q, s = quantize(v)
            out[k] = torch.from_numpy(dequantize(q, s))
        else:
            out[k] = v
    return out
