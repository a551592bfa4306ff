"""Prompt lookup decoding at 7B widths (synthetic weights, B = 1): the plain decode step and the verification step of k drafts at two
context lengths, the break-even acceptance (t_k / t_plain - 1 accepted drafts per step), and tokens/s of greedy generate() with and
without prompt_lookup_num_tokens on the synthetic model's output, with the acceptance it got, and on a cyclic output (o_proj and
down_proj zeroed) as a labelled upper bound; the in-situ attention share of each step from the kernel trace.  Synthetic weights say
nothing about the acceptance on real answers, so none of these tokens/s is an estimate of the speedup there.
Usage: python tools/lookup_bench.py [out.json]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))
import torch  # noqa: E402
import visualcla  # noqa: E402

KS = [1, 3, 7, 10, 15]
REPS = 8          # graph replays of 8 steps per measurement


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def attention_share(eng, tok):
    """In-situ share of the attention kernels (one-token: tag 4; verification: append 19 + attend 4) in ONE graph-replayed step, from the
    %globaltimer trace: a kernel's duration is its successor's dependency-resolved time minus its own (bench.py's rule)."""
    eng.decode_many(tok, 1)                                        # capture the one-step graph untraced
    eng.trace_enable(8192)
    eng.decode_many(tok, 1)
    torch.cuda.synchronize()
    ev = sorted((r for r in eng.trace_read(8192) if r[2]), key=lambda r: r[2])
    eng.trace_enable(0)
    span = ev[-1][2] - ev[0][2]
    attn = sum(ev[i + 1][2] - ev[i][2] for i in range(len(ev) - 1) if ev[i][0] in (4, 19))
    return attn / span


def main():
    m = visualcla.VisualCLAModel.from_synthetic("7b", seed=0, max_batch=1, max_seq=1400)
    eng = m._engine
    res = dict(gpu=gpu_name(), steps={})
    for ctx in (260, 1100):
        ids = torch.randint(3, 49954, (1, ctx), device="cuda")
        row = {}
        tok = torch.zeros(1, dtype=torch.int32, device="cuda")

        def prefill():
            _, first, _ = eng.prefill(ids, 0, None, last_logits=False)
            tok.copy_(first)
        prefill()
        eng.decode_many(tok, 8)                                       # capture + warm up
        prefill()
        row["plain_ms"] = timed(lambda: eng.decode_many(tok, 8), REPS) / 8
        row["plain_attention_share"] = attention_share(eng, tok)
        for k in KS:
            prefill()
            eng.set_lookup(ids[0], k, 2, eng.max_seq - ctx - 16)
            eng.decode_many(tok, 8)
            t = timed(lambda: eng.decode_many(tok, 8), REPS) / 8
            row[f"k{k}_attention_share"] = attention_share(eng, tok)
            eng.set_lookup(None)
            row[f"k{k}_ms"] = t
            row[f"k{k}_break_even_accepted_per_step"] = t / row["plain_ms"] - 1.0
        res["steps"][ctx] = row
        print(ctx, json.dumps(row), flush=True)
    # tokens/s of greedy generate() on the synthetic output (its acceptance is reported beside it)
    ids = torch.randint(3, 49954, (1, 260), device="cuda")
    kw = dict(do_sample=False, eos_token_id=None, pad_token_id=0, max_new_tokens=256)
    plain = m.generate(input_ids=ids, **kw)
    look = m.generate(input_ids=ids, prompt_lookup_num_tokens=10, **kw)
    assert torch.equal(plain, look)
    for name, extra in (("plain", {}), ("lookup_k10", dict(prompt_lookup_num_tokens=10))):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.generate(input_ids=ids, **kw, **extra)
        torch.cuda.synchronize()
        res[f"synthetic_tok_s_{name}"] = 256 / (time.perf_counter() - t0)
    res["synthetic_lookup_stats"] = dict(zip(("produced", "finished", "steps", "drafted", "accepted", "rows"), eng.lookup_stats()))
    # upper bound: with o_proj and down_proj zeroed the next token depends on the current one only, so the output cycles and lookup
    # copies it; real answers accept fewer drafts
    T, F = 4096, 11008
    for i in range(32):
        p = f"text_model.model.layers.{i}."
        eng.load_weight(p + "self_attn.o_proj.weight", torch.zeros(T, T, dtype=torch.bfloat16, device="cuda"))
        eng.load_weight(p + "mlp.down_proj.weight", torch.zeros(T, F, dtype=torch.bfloat16, device="cuda"))
    # the next token is now a function of the current one: a prompt that holds the greedy continuation of its last token lets every
    # draft be accepted
    g = m.generate(input_ids=ids, **dict(kw, max_new_tokens=600))
    ids = torch.cat([ids, g, ids[:, -1:]], 1)
    kw["max_new_tokens"] = 512
    for name, extra in (("plain", {}), ("lookup_k10", dict(prompt_lookup_num_tokens=10)), ("lookup_k15", dict(prompt_lookup_num_tokens=15))):
        m.generate(input_ids=ids, **kw, **extra)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = m.generate(input_ids=ids, **kw, **extra)
        torch.cuda.synchronize()
        res[f"cyclic_upper_bound_tok_s_{name}"] = 512 / (time.perf_counter() - t0)
        if extra:
            res[f"cyclic_upper_bound_stats_{name}"] = dict(zip(("produced", "finished", "steps", "drafted", "accepted", "rows"), eng.lookup_stats()))
    print(json.dumps(res, indent=1))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
