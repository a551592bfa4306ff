"""Timeline of ONE graph-replayed decode step (real 7B shapes) from the in-kernel %globaltimer trace."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))
import torch  # noqa: E402
import visualcla  # noqa: E402
from visualcla import _native as N  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
pdl = int(sys.argv[2]) if len(sys.argv) > 2 else 1
out_path = sys.argv[3] if len(sys.argv) > 3 else None
N.load().vcla_set_pdl(pdl)
TAGS = {1: "gemm_swap", 2: "gemm", 3: "attn_prefill", 4: "attn_decode", 5: "layernorm", 6: "rmsnorm", 7: "rope_cache", 8: "resid_norm",
        9: "silu_mul", 10: "logits1", 11: "logits2", 12: "advance", 13: "embed", 14: "sampler", 19: "attn_lookup_append", 20: "lookup_accept"}
m = visualcla.VisualCLAModel.from_synthetic("7b", seed=0, max_batch=B, max_seq=400, max_prefill_tokens=B * 128)
m.image_at_head = True
eng = m._engine
px = torch.randn(B, 3, 224, 224, device="cuda").half()
ids = torch.randint(3, 49954, (B, 64), device="cuda")
eng.vision_encode(px)
_, tok, _ = eng.prefill(ids, 1, None, last_logits=False)
tok = tok.clone()
for _ in range(4):
    eng.decode_step(tok, tok, None)      # captures the graph, warms up
torch.cuda.synchronize()
eng.trace_enable(4096)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
eng.decode_step(tok, tok, None)
e1.record()
torch.cuda.synchronize()
ev = eng.trace_read()
eng.trace_enable(0)
ev.sort(key=lambda r: r[1])
t0 = ev[0][1]
print(f"decode step B={B} pdl={pdl}: {len(ev)} kernels, CUDA-event time {e0.elapsed_time(e1) * 1000:.1f} us, trace span {(max(r[3] or r[2] for r in ev) - t0) / 1000:.1f} us")
print(" idx kernel        entry_us   dep_us  exit_us | wait(dep-entry) run(exit-dep)")
rows = []
for i, (tag, a, b, c) in enumerate(ev):
    rows.append({"kernel": TAGS.get(tag, str(tag)), "entry_us": (a - t0) / 1e3, "dep_us": (b - t0) / 1e3 if b else None, "exit_us": (c - t0) / 1e3 if c else None})
    if i < 40 or i > len(ev) - 12:
        r = rows[-1]
        d = f"{r['dep_us']:8.1f}" if r["dep_us"] is not None else "       -"
        x = f"{r['exit_us']:8.1f}" if r["exit_us"] is not None else "       -"
        w = f"{r['dep_us'] - r['entry_us']:7.1f}" if r["dep_us"] is not None else "      -"
        run = f"{r['exit_us'] - r['dep_us']:7.1f}" if (r["exit_us"] is not None and r["dep_us"] is not None) else "      -"
        print(f"{i:4d} {r['kernel']:12s} {r['entry_us']:8.1f} {d} {x} | {w} {run}")
# how early do kernels start relative to their predecessor's dependency resolution?
early = [rows[i]["dep_us"] - rows[i]["entry_us"] for i in range(1, len(rows)) if rows[i]["dep_us"] is not None]
print(f"mean (dep - entry) = {sum(early) / len(early):.2f} us  (time a kernel's CTA 0 is resident before its inputs are ready)")
# in-situ duration of a kernel = its successor's dependency-resolved time - its own (the launch gap included): they add up to the step
deps = [(r["kernel"], r["dep_us"]) for r in rows if r["dep_us"] is not None]
deps.sort(key=lambda x: x[1])
per = {}
gi = 0
for i in range(len(deps) - 1):
    k = deps[i][0]
    if k == "gemm_swap":
        k = ["gemm_qkv", "gemm_o", "gemm_gate_up", "gemm_down"][gi % 4] if gi < 128 else "gemm_lm_head"
        gi += 1
    per.setdefault(k, []).append(deps[i + 1][1] - deps[i][1])
print("in-situ mean us per kernel kind:", {k: round(sum(v) / len(v), 2) for k, v in per.items()})
print("per layer (sum of the per-layer kernels):", round(sum(sum(v) / len(v) for k, v in per.items() if len(v) >= 32), 2), "us")
if out_path:
    json.dump({"B": B, "pdl": pdl, "event_us": e0.elapsed_time(e1) * 1000, "insitu_mean_us": {k: sum(v) / len(v) for k, v in per.items()},
               "schedule": "csk" if B <= 32 else "workspace", "events": rows}, open(out_path, "w"))
