"""N sampled replies per prompt at 7B widths (synthetic weights, one image at the head and a chat-length prompt, the reference's chat
sampling knobs): generate(num_return_sequences=N), which encodes and prefills the prompt once and forks its KV pages to N rows, against the
expanded batch -- the prompt and its pixels repeated N times, num_return_sequences=1 -- at N = 1, 4, 8, 16.  Per arm: time to first token
(a call with max_new_tokens=1: vision encode, prefill, first pick), the whole call at a fixed max_new_tokens, and the KV pages in use right
after the prefill and at the end of the call (vcla_kv_read_pages).  Times are host clocks around calls that end in a device synchronise,
the median of --reps runs after one warm-up run that captures the decode graphs.  Prints the card name and power limit with the numbers.

    python tools/return_sequences_bench.py [--new 64] [--prompt 48] [--reps 3] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))

CHAT = dict(do_sample=True, repetition_penalty=1.1, no_repeat_ngram_size=15, temperature=0.5, top_k=40, top_p=0.9)   # DEFAULT_GENERATION_CONFIG


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                      # the numbers still carry the device name torch reports
        return f"{torch.cuda.get_device_name(0)} (power limit unavailable: {e})"


def timed_call(fn, reps):
    """median wall-clock ms of fn() over reps runs, each ended by a device synchronise, after one warm-up run"""
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def pages_in_use(eng):
    _, _, free, exhausted = eng.kv_pages()
    assert not exhausted
    return eng.kv_geometry()[1] - free


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=64, help="max_new_tokens of the whole call")
    ap.add_argument("--prompt", type=int, default=48, help="text tokens of the prompt (the image adds 64 rows at its head)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import visualcla
    from visualcla.engine import path_config_7b
    assert torch.cuda.is_available(), "return_sequences_bench needs the GPU"
    torch.cuda.set_device(0)
    pc = path_config_7b()
    ns = (1, 4, 8, 16)
    m = visualcla.VisualCLAModel.from_synthetic(pc, seed=0, max_batch=max(ns), max_seq=a.prompt + pc["r_queries"] + a.new + 8)
    eng = m._engine
    _, total, pt = eng.kv_geometry()
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(3, pc["t_vocab"] - 8, (1, a.prompt), generator=g)
    ids[0, 0] = 1
    px = torch.randn(1, 3, pc["v_image"], pc["v_image"], generator=g).to(torch.bfloat16).float().cuda()
    ids = ids.cuda()
    S = a.prompt + pc["r_queries"]
    info = dict(card=card(), torch_device=torch.cuda.get_device_name(0), prompt_rows=S, max_new_tokens=a.new, page_tokens=pt,
                total_pages=total, reps=a.reps, rows=[])
    print(f"[return_sequences_bench] {info['card']}; prompt {S} rows (64 image + {a.prompt} text), {a.new} new tokens, "
          f"page {pt} tokens, median of {a.reps} after a warm-up")

    def run(n, fork, max_new):
        kw = dict(max_new_tokens=max_new, eos_token_id=None, pad_token_id=0, **CHAT)
        if fork:
            return m.generate(input_ids=ids, pixel_values=px, num_return_sequences=n, **kw)
        return m.generate(input_ids=ids.repeat(n, 1), pixel_values=px.repeat(n, 1, 1, 1), **kw)

    for n in ns:
        row = dict(N=n)
        for arm, fork in (("fork", True), ("expanded", False)):
            torch.manual_seed(0)
            ttft = timed_call(lambda: run(n, fork, 1), a.reps)
            pages_prefill = pages_in_use(eng)
            full = timed_call(lambda: run(n, fork, a.new), a.reps)
            out = run(n, fork, a.new)
            torch.cuda.synchronize()
            assert out.shape == (n, a.new)
            row[arm] = dict(ttft_ms=round(ttft, 2), call_ms=round(full, 2), ms_per_token_row=round(full / a.new, 3),
                            pages_after_prefill=pages_prefill, pages_at_end=pages_in_use(eng))
        info["rows"].append(row)
    base = info["rows"][0]["fork"]["call_ms"]
    for row in info["rows"]:
        row["call_vs_n1_fork"] = round(row["fork"]["call_ms"] / base, 3)
        f, x = row["fork"], row["expanded"]
        print(f"[return_sequences_bench] N={row['N']:2d}: fork ttft {f['ttft_ms']:.1f} ms, call {f['call_ms']:.1f} ms "
              f"({row['call_vs_n1_fork']:.2f}x N=1), pages {f['pages_after_prefill']} -> {f['pages_at_end']} | expanded ttft "
              f"{x['ttft_ms']:.1f} ms, call {x['call_ms']:.1f} ms, pages {x['pages_after_prefill']} -> {x['pages_at_end']}")
    print(json.dumps(info))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "return_sequences_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
