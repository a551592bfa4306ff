"""bf16 vs load_in_8bit (weight-only int8 LLaMA projections) at VisualCLA-7B shapes, in one process, alternating the two engines.

Reports per format: decode step time (CUDA-graph replay) at B = 1, 8, 32, 64 and the achieved GB/s against the step's byte floor (the
weights every step streams: projections + lm_head; KV and activations excluded), the prefill time of 8 images + 64-token prompts,
vcla_memory_bytes, and the greedy-token agreement of the two formats on the same seeded prompts.  Prints the card name and power limit.

    python tools/int8_bench.py [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))

import torch  # noqa: E402

from visualcla import VisualCLAModel  # noqa: E402
from visualcla.engine import path_config_7b  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:      # the numbers still stand; say what is missing
        return f"unknown ({e})"


def floor_bytes(p, fmt):
    T, F, V, L = p["t_hidden"], p["t_ffn"], p["t_vocab"], p["t_layers"]
    n = 4 * T * T + 3 * T * F
    rows = 3 * T + T + 2 * F + T
    proj = L * (n + 4 * rows) if fmt == 1 else L * 2 * n
    return proj + 2 * V * T


def time_decode(m, B, steps, reps):
    eng = m._engine
    ids = torch.randint(100, 30000, (B, 16), device="cuda")
    eng.prefill(ids, 0)
    tok = eng.token_buffer(B)
    tok.fill_(1)
    eng.decode_many(tok, steps)              # captures the graphs
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = []
    for _ in range(reps):
        eng.prefill(ids, 0)
        e0.record()
        eng.decode_many(tok, steps)
        e1.record()
        torch.cuda.synchronize()
        best.append(e0.elapsed_time(e1) / steps)
    best.sort()
    return best[len(best) // 2]


def time_prefill(m, reps):
    eng = m._engine
    g = torch.Generator().manual_seed(0)
    px = torch.randn(8, 3, 224, 224, generator=g).cuda()
    ids = torch.randint(100, 30000, (8, 64), generator=g).cuda()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(reps + 1):
        e0.record()
        eng.vision_encode(px)
        eng.prefill(ids, 1)
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    out = sorted(out[1:])
    return out[len(out) // 2]


def agreement(m8, m16, steps=32):
    g = torch.Generator().manual_seed(1)
    px = torch.randn(8, 3, 224, 224, generator=g).cuda()
    ids = torch.randint(100, 30000, (8, 64), generator=g).cuda()
    kw = dict(input_ids=ids, pixel_values=px, do_sample=False, max_new_tokens=steps, eos_token_id=None, pad_token_id=0)
    a, b = m8.generate(**kw), m16.generate(**kw)
    first = (a != b).int().argmax(1).where((a != b).any(1), torch.full((8,), steps, device=a.device))
    return {"tokens_equal": float((a == b).float().mean()), "steps_before_first_difference": first.tolist()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    p = path_config_7b()
    models = {fmt: VisualCLAModel.from_synthetic(p, seed=0, max_batch=64, max_seq=168,
                                                 max_prefill_tokens=64 * 128, load_in_8bit=fmt == 1) for fmt in (0, 1)}
    res = {"card (name, power limit)": card(), "decode": {}, "prefill_ms": {}, "memory_bytes": {}}
    for fmt, m in models.items():
        w, kv, act = m._engine.memory_bytes()
        res["memory_bytes"][("bf16", "int8")[fmt]] = {"weights": w, "kv": kv, "activations": act}
    for B in (1, 8, 32, 64):
        row = {}
        for rep in range(2):                 # alternate the engines twice: both see the same machine state
            for fmt, m in models.items():
                ms = time_decode(m, B, a.steps, a.reps)
                key = ("bf16", "int8")[fmt]
                if rep == 1 or key not in row:
                    row[key] = {"step_ms": ms, "GB/s_vs_floor": floor_bytes(p, fmt) / (ms * 1e-3) / 1e9, "floor_GB": floor_bytes(p, fmt) / 1e9}
        res["decode"][f"B{B}"] = row
        print(json.dumps({f"B{B}": row}), flush=True)
    for rep in range(2):
        for fmt, m in models.items():
            res["prefill_ms"][("bf16", "int8")[fmt]] = time_prefill(m, a.reps)
    res["greedy_agreement_int8_vs_bf16"] = agreement(models[1], models[0])
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "int8_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
