"""Time to the first token of a chat turn, with the KV cache of the conversation reused and with a full re-prefill.

    python tools/chat_turn_bench.py [--layers 32] [--lengths 256,1024,1792] [--instr 32] [--reply 48] [--warmup 2] [--reps 5]

The 7B-width synthetic model (random weights, placeholder image layout), one image, a scripted conversation: each turn appends an
instruction of --instr tokens and the model's greedy reply of --reply tokens, driven through generate(past_key_values=...) the way
chat() does with reuse_kv_cache=True, until the prompt reaches each of --lengths tokens.  There, the first token of the next turn
is timed with CUDA events (after --warmup untimed runs, mean of --reps):
  full_ms    vision tower + prefill of the whole conversation (what every turn costs without reuse)
  reuse_ms   truncate to the cached conversation + extend by the new instruction (vcla_kv_truncate + vcla_prefill_extend)
  attn_us    one launch of the paged prefill attention (the new instruction over the cached conversation, one layer), device time
             from torch.profiler; attn_gbps = the K/V bytes it must read (every cached token, all heads) / attn_us
One JSON line per length, the card name and power limit first.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))
import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        out = ""
    return {"device": name, "power_limit": out or "unknown"}


def cuda_ms(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        start.record()
        fn()
        end.record()
        end.synchronize()
        times.append(start.elapsed_time(end))
    return sum(times) / len(times)


def attention_us(lib, N, prefix, T, H, page_tokens, reps):
    """Device time of one paged attention launch: T new rows over prefix cached tokens, H heads of 128, one sequence."""
    pps = (prefix + T + page_tokens - 1) // page_tokens
    pool = torch.randn(pps, 2, H, page_tokens, 128, device="cuda").to(torch.bfloat16)
    table = torch.randperm(pps, device="cuda").to(torch.int32)
    q = torch.randn(T, H * 128, device="cuda").to(torch.bfloat16)
    out = torch.empty_like(q)
    base = torch.tensor([prefix], dtype=torch.int32, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run():
        N.check(lib.vcla_op_attention_paged(N.ptr(q), H * 128, N.ptr(pool), N.ptr(table), pps, page_tokens, N.ptr(base), N.ptr(out),
                                            H * 128, 1, H, T, C.c_float(128 ** -0.5), st), "vcla_op_attention_paged")
    run()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            run()
    total = sum(e.device_time_total for e in prof.key_averages() if "attn_prefill_tc_kernel" in e.key)
    return total / reps, 2 * (prefix + T) * H * 128 * 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--lengths", default="256,1024,1792")
    ap.add_argument("--instr", type=int, default=32)
    ap.add_argument("--reply", type=int, default=48)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import visualcla
    from visualcla import _native as N
    from visualcla.engine import path_config_7b
    lengths = sorted(int(x) for x in a.lengths.split(","))
    print(json.dumps(card()), flush=True)
    cfg = dict(path_config_7b(), t_layers=a.layers)
    max_seq = lengths[-1] + a.instr + a.reply + 64
    m = visualcla.VisualCLAModel.from_synthetic(cfg, seed=0, max_batch=1, max_seq=max_seq)
    eng = m._engine
    V, nq = cfg["t_vocab"], cfg["r_queries"]
    img0, img1, imgt = V - 4, V - 3, V - 1
    m.image_at_head = False
    m.tokenizer = types.SimpleNamespace(img_start_token_id=img0, img_end_token_id=img1, img_token_id=imgt)
    g = torch.Generator().manual_seed(0)
    text = lambda n: torch.randint(3, V - 4, (1, n), generator=g)
    px = torch.randn(1, 3, cfg["v_image"], cfg["v_image"], generator=g).cuda()
    conv = torch.cat([torch.tensor([[1, img0]]), torch.full((1, nq), imgt), torch.tensor([[img1]]), text(a.instr)], 1)
    greedy = dict(do_sample=False, eos_token_id=None, pad_token_id=0, return_dict_in_generate=True)
    handle = None
    for target in lengths:
        while conv.shape[1] + (a.reply + a.instr) // 2 < target:     # stop within half a turn of the target length
            r = m.generate(input_ids=conv.cuda(), pixel_values=px, max_new_tokens=a.reply, past_key_values=handle, **greedy)
            handle = r.past_key_values
            conv = torch.cat([conv, r.sequences.cpu(), text(a.instr)], 1)
        # the cache now holds the conversation up to the last reply; the next turn's prompt adds one instruction
        cached = len(handle)
        new = conv[:, cached:]
        ids = conv.cuda()

        def full():
            eng.vision_encode(px)
            eng.prefill(ids, N.IMAGE_PLACEHOLDER, torch.tensor([2], dtype=torch.int32), last_logits=False)

        def reuse():
            eng.truncate([cached])
            eng.extend(new, last_logits=False)

        reuse_ms = cuda_ms(reuse, a.warmup, a.reps)      # the handle's cache is resident: time extend first, then overwrite it
        full_ms = cuda_ms(full, a.warmup, a.reps)
        attn_us, kv_bytes = attention_us(eng.lib, N, cached, new.shape[1], cfg["t_heads"], eng.kv_geometry()[2], a.reps)
        # a current handle for the next, longer turn
        r = m.generate(input_ids=conv.cuda(), pixel_values=px, max_new_tokens=a.reply, **greedy)
        handle = r.past_key_values
        conv = torch.cat([conv, r.sequences.cpu(), text(a.instr)], 1)
        print(json.dumps({"prompt_tokens": int(ids.shape[1]), "cached_tokens": cached, "new_tokens": int(new.shape[1]), "layers": a.layers,
                          "full_ms": round(full_ms, 3), "reuse_ms": round(reuse_ms, 3), "speedup": round(full_ms / reuse_ms, 2),
                          "attn_us": round(attn_us, 2), "attn_gbps": round(kv_bytes / attn_us / 1e3, 1)}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
