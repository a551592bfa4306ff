"""Beam search at 7B widths (synthetic weights, text-only prompts): ms per decode step of beam search against a greedy run at the same
number of rows (B prompts x K beams), the in-kernel trace times of the beam kernels, and the K/V bytes copied copy-on-write per step
(counted on the device), with the bound (K - 1) * B partial pages per step.  Prints the card name and power limit with the numbers.

    python tools/beam_bench.py [--steps 32] [--prompt 64] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))

TAGS = {15: "beam_step", 16: "beam_select", 17: "page_reorder", 18: "page_copy"}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:                      # the numbers still carry the device name torch reports
        return f"{torch.cuda.get_device_name(0)} (power limit unavailable: {e})"


def timed(eng, tok, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    done = 0
    while done < steps:
        eng.decode_many(tok, 8)
        done += 8
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / done


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--prompt", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from visualcla.engine import Engine, path_config_7b
    assert torch.cuda.is_available(), "beam_bench needs the GPU"
    torch.cuda.set_device(0)
    steps = (a.steps + 7) // 8 * 8
    max_new = steps + 16 + 1
    eng = Engine(path_config_7b(), max_batch=64, max_seq=a.prompt + max_new + 8)
    eng.init_synthetic(0)
    _, _, pt = eng.kv_geometry()
    pc = eng.path_cfg
    bytes_per_token = pc["t_layers"] * 2 * pc["t_hidden"] * 2
    g = torch.Generator().manual_seed(0)
    info = dict(card=card(), torch_device=torch.cuda.get_device_name(0), prompt=a.prompt, steps=steps, page_tokens=pt,
                kv_bytes_per_token=bytes_per_token, rows=[])
    print(f"[beam_bench] {info['card']}; prompt {a.prompt} tokens, {steps} timed steps, page {pt} tokens, "
          f"{bytes_per_token / 2 ** 20:.2f} MiB K/V per cached token")
    for B in (1, 8):
        for K in (2, 4, 8):
            R = B * K
            ids = torch.randint(0, pc["t_vocab"] - 8, (R, a.prompt), generator=g)
            # greedy at the same rows
            _, first, _ = eng.prefill(ids, 0, None, last_logits=False)
            tok = eng.token_buffer(R)
            tok.copy_(first)
            eng.decode_many(tok, 8)                                       # warm-up: captures the graphs
            greedy_ms = timed(eng, tok, steps)
            # beam search: B prompts, K beams
            eng.set_beam(eng.beam_spec(K, max_new))
            try:
                _, first, _ = eng.prefill(ids[:B], 0, None, last_logits=False)
                bt = eng.token_buffer(R)
                bt.copy_(first)
                eng.decode_many(bt, 8)
                eng.beam_cow_bytes(reset=True)
                beam_ms = timed(eng, bt, steps)
                cow = eng.beam_cow_bytes(reset=True) / steps
                eng.trace_enable(4096)
                eng.decode_many(bt, 8)
                ev = eng.trace_read(4096)
                eng.trace_enable(0)
            finally:
                eng.set_beam(None)
            kt = {}
            for tag, name in TAGS.items():
                d = [(x[3] - x[1]) / 1e3 for x in ev if x[0] == tag and x[3] > x[1]]
                kt[name] = round(sum(d) / len(d), 2) if d else None
            bound = (K - 1) * B * (pt - 1) * bytes_per_token
            row = dict(B=B, K=K, rows=R, greedy_ms_per_step=round(greedy_ms, 3), beam_ms_per_step=round(beam_ms, 3),
                       overhead_pct=round(100 * (beam_ms / greedy_ms - 1), 2), kernel_us=kt, cow_bytes_per_step=int(cow),
                       cow_bound_bytes_per_step=int(bound))
            info["rows"].append(row)
            print(f"[beam_bench] B={B} K={K} rows={R}: greedy {greedy_ms:.3f} ms/step, beam {beam_ms:.3f} ms/step "
                  f"({row['overhead_pct']:+.2f} %); kernels (us, CTA 0 trace) {kt}; copy-on-write {cow / 2 ** 20:.2f} MiB/step "
                  f"(bound {bound / 2 ** 20:.1f} MiB)")
    print(json.dumps(info))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "beam_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
