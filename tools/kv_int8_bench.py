"""bf16 vs int8 KV cache (kv_cache_dtype="int8") at VisualCLA-7B widths, in one process, alternating the two formats.

Reports per format: the decode step time by CUDA-graph replay at B = 1, 8, 32, 64 x context 256, 1024, 1984 (shapes whose cache does
not fit the card are skipped), each step's byte floor (LLaMA weights + the KV rows the step reads) and the achieved fraction of
3.35 TB/s, vcla_memory_bytes, whether a max_batch 64 x max_seq 2048 context can be created, and the greedy-token agreement of the two
formats over 256 tokens, and the extension time of a reused chat turn (256 new tokens after a 1024-token cached conversation, B = 1).
Prints the card name and power limit.

    python tools/kv_int8_bench.py [--reps 5] [--out DIR]
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
from visualcla import _native as N  # noqa: E402
from visualcla.engine import path_config_7b  # noqa: E402

FORMATS = {"bf16": None, "int8": "int8"}
ROW_BYTES = {"bf16": 256, "int8": 132}
HBM = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:
        return f"unknown ({e})"


def weight_bytes(p):
    T, F, V, L = p["t_hidden"], p["t_ffn"], p["t_vocab"], p["t_layers"]
    return L * 2 * (4 * T * T + 3 * T * F) + 2 * V * T


def kv_read_bytes(p, fmt, B, ctx):
    return B * (ctx + 1) * p["t_layers"] * 2 * p["t_heads"] * ROW_BYTES[fmt]


def model(fmt, B, max_seq, prefill_tokens):
    return VisualCLAModel.from_synthetic(path_config_7b(), seed=0, max_batch=B, max_seq=max_seq, max_prefill_tokens=prefill_tokens,
                                         kv_cache_dtype=FORMATS[fmt])


def time_decode(m, B, ctx, steps, reps):
    eng = m._engine
    ids = torch.randint(100, 30000, (B, ctx), generator=torch.Generator().manual_seed(B + ctx)).cuda()
    tok = eng.token_buffer(B)
    out = []
    for r in range(reps + 1):                     # the first round captures the graphs
        eng.prefill(ids, 0, last_logits=False)
        tok.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.decode_many(tok, steps)
        e1.record()
        torch.cuda.synchronize()
        if r > 0:
            out.append(e0.elapsed_time(e1) / steps)
    out.sort()
    return out[len(out) // 2]


def time_extend(fmt, reps, ctx=1024, new=256):
    m = model(fmt, 1, ctx + new + 8, ctx + new)
    eng = m._engine
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(100, 30000, (1, ctx), generator=g).cuda()
    turn = torch.randint(100, 30000, (1, new), generator=g).cuda()
    eng.prefill(ids, 0, last_logits=False)
    out = []
    for r in range(reps + 1):
        eng.truncate([ctx])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.extend(turn)
        e1.record()
        torch.cuda.synchronize()
        if r > 0:
            out.append(e0.elapsed_time(e1))
    eng.close()
    out.sort()
    return round(out[len(out) // 2], 3)


def agreement(steps=256):
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(100, 30000, (8, 64), generator=g).cuda()
    kw = dict(input_ids=ids, do_sample=False, max_new_tokens=steps, eos_token_id=None, pad_token_id=0)
    outs = {}
    for fmt in FORMATS:
        m = model(fmt, 8, 64 + steps, 8 * 64)
        outs[fmt] = m.generate(**kw)[:, -steps:]
        m._engine.close()
        del m
    a, b = outs["int8"], outs["bf16"]
    first = (a != b).int().argmax(1).where((a != b).any(1), torch.full((8,), steps, device=a.device))
    return {"tokens_equal": float((a == b).float().mean()), "steps_before_first_difference": first.tolist()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    p = path_config_7b()
    res = {"card (name, power limit)": card(), "decode": {}, "memory_bytes": {}, "capacity_64x2048": {}}
    for B in (1, 8, 32, 64):
        for ctx in (256, 1024, 1984):
            row = {}
            for fmt in FORMATS:
                try:
                    m = model(fmt, B, ctx + a.steps + 8, B * ctx)
                except N.NativeError as e:
                    row[fmt] = {"skipped": str(e).split(":")[-1].strip()[:120]}
                    continue
                ms = time_decode(m, B, ctx, a.steps, a.reps)
                floor = weight_bytes(p) + kv_read_bytes(p, fmt, B, ctx + a.steps // 2)
                row[fmt] = {"step_ms": round(ms, 3), "floor_GB": round(floor / 1e9, 2), "floor_ms": round(floor / HBM * 1e3, 3),
                            "frac_of_floor": round(floor / HBM * 1e3 / ms, 3)}
                m._engine.close()
                del m
                torch.cuda.empty_cache()
            res["decode"][f"B{B}_ctx{ctx}"] = row
            print(json.dumps({f"B{B}_ctx{ctx}": row}), flush=True)
    for fmt in FORMATS:
        try:
            m = model(fmt, 64, 2048, 64 * 32)
            w, kv, act = m._engine.memory_bytes()
            res["capacity_64x2048"][fmt] = {"created": True, "weights": w, "kv": kv, "activations": act}
            m._engine.close()
            del m
        except N.NativeError as e:
            res["capacity_64x2048"][fmt] = {"created": False, "error": str(e)[:200]}
        torch.cuda.empty_cache()
    res["extend_ms_1024_cached_plus_256"] = {fmt: time_extend(fmt, a.reps) for fmt in FORMATS}
    res["greedy_agreement_int8_vs_bf16_256_tokens"] = agreement()
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "kv_int8_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
