"""Where a graph-replayed decode step loses time at kernel boundaries (7B shapes, bench.py's workload at batch B).

For each of the five per-layer decode kernels: in-situ time (successor's dependency-resolved time - own, the launch gap included, as
bench.py's roofline.in_step_us), byte floor at a streaming rate, and the loss = in-situ - floor.  For each boundary: the entry gap =
successor CTA 0 entry - predecessor CTA 0 exit (negative: the successor was resident before its predecessor's first CTA left).

  python tools/decode_boundaries.py [--batch 8] [--rate GBps] [--out file.json]

--rate defaults to the best rate any decode GEMM reaches in this trace (the stream rate the hardware showed it can sustain inside a step).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (bench.py puts the package on sys.path)

KINDS = ["qkv", "attn_decode", "o_proj", "gate_up", "down_proj"]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=10).stdout.strip()
        return out or None
    except Exception:  # noqa: BLE001
        return None


def trace_step(B, n_layers=32):
    """One graph-replayed decode step at mid-generation context (bench.py's in-situ point) -> (labelled events, context, event time us)."""
    import torch
    import visualcla
    S = bench.T_TEXT + bench.NQ
    model = visualcla.VisualCLAModel.from_synthetic("7b", seed=0, max_batch=B, max_seq=S + bench.N_NEW + 1, max_prefill_tokens=B * S)
    model.image_at_head = True
    eng = model._engine
    px, ids = bench.synth_inputs(B)
    px, ids = px.cuda(), ids.cuda()
    tok = eng.token_buffer(B)
    mode, rows = model._image_layout(ids, px)
    eng.vision_encode(px)
    _, first, _ = eng.prefill(ids, mode, rows, all_logits=False, last_logits=False)
    tok.copy_(first)
    eng.decode_many(tok, bench.N_NEW // 2)
    for _ in range(3):
        eng.decode_step(tok, tok, None)           # single-step graph: captured + warm
    torch.cuda.synchronize()
    eng.trace_enable(4096)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    eng.decode_step(tok, tok, None)
    e1.record()
    torch.cuda.synchronize()
    ev = eng.trace_read()
    eng.trace_enable(0)
    ctx = S + bench.N_NEW // 2 + 3
    eng.close()
    ev = [e for e in ev if e[2]]
    ev.sort(key=lambda r: r[2])
    names, gi = [], 0
    for tag, _a, _b, _c in ev:
        if tag == 1:
            names.append(["qkv", "o_proj", "gate_up", "down_proj"][gi % 4] if gi < 4 * n_layers else "lm_head")
            gi += 1
        else:
            names.append(bench.TRACE_TAGS.get(tag, str(tag)))
    rows = [{"kernel": n, "entry": a / 1e3, "dep": b / 1e3, "exit": (c / 1e3) if c else None} for n, (_t, a, b, c) in zip(names, ev)]
    return rows, ctx, e0.elapsed_time(e1) * 1000


def analyse(rows, B, ctx, rate=None, n_layers=32):
    nbytes = dict(bench.GEMM_BYTES)
    nbytes["attn_decode"] = B * (ctx + 1) * bench.KV_BYTES_PER_TOKEN / n_layers
    insitu, gaps = {}, {}
    for i in range(len(rows) - 1):
        a, b = rows[i], rows[i + 1]
        insitu.setdefault(a["kernel"], []).append(b["dep"] - a["dep"])
        if a["exit"] is not None:
            gaps.setdefault(f"{a['kernel']}->{b['kernel']}", []).append(b["entry"] - a["exit"])
    mean = {k: statistics.mean(v) for k, v in insitu.items()}
    if rate is None:
        rate = max(nbytes[k] / mean[k] / 1e3 for k in ("qkv", "o_proj", "gate_up", "down_proj", "lm_head") if k in mean)
    table = {}
    for k in KINDS:
        if k not in mean:
            continue
        floor = nbytes[k] / rate / 1e3
        table[k] = {"n": len(insitu[k]), "insitu_us": mean[k], "floor_us": floor, "loss_us": mean[k] - floor}
    per_layer = sum(r["loss_us"] for r in table.values())
    layer_gaps = {}
    for k, v in gaps.items():
        if len(v) >= n_layers - 1:
            layer_gaps[k] = {"n": len(v), "mean_us": statistics.mean(v), "min_us": min(v), "max_us": max(v)}
    step_us = rows[-1]["dep"] - rows[0]["dep"]
    return {"B": B, "ctx": ctx, "rate_GBps": rate, "kernels": table, "loss_per_layer_us": per_layer, "loss_per_step_us": per_layer * n_layers,
            "gaps": layer_gaps, "traced_step_us": step_us, "insitu_other_us": {k: v for k, v in mean.items() if k not in KINDS}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--rate", type=float, default=None, help="GB/s for the byte floors (default: the best in-step GEMM rate)")
    ap.add_argument("--pdl", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("decode_boundaries.py needs a CUDA device")
    from visualcla import _native
    _native.load().vcla_set_pdl(args.pdl)
    rows, ctx, ev_us = trace_step(args.batch)
    r = analyse(rows, args.batch, ctx, args.rate)
    r["event_us"], r["card"] = ev_us, card()
    print(f"decode step B={r['B']} ctx={ctx}: {ev_us:.1f} us (CUDA events), traced {r['traced_step_us']:.1f} us; card: {r['card']}")
    print(f"byte floors at {r['rate_GBps']:.0f} GB/s")
    print(f"{'kernel':12s} {'in-situ us':>10s} {'floor us':>9s} {'loss us':>8s}")
    for k, t in r["kernels"].items():
        print(f"{k:12s} {t['insitu_us']:10.2f} {t['floor_us']:9.2f} {t['loss_us']:8.2f}")
    print(f"boundary loss: {r['loss_per_layer_us']:.2f} us per layer, {r['loss_per_step_us'] / 1e3:.3f} ms per step")
    print(f"{'boundary':26s} {'entry gap us (mean / min / max)':>32s}")
    for k, g in r["gaps"].items():
        print(f"{k:26s} {g['mean_us']:10.2f} {g['min_us']:10.2f} {g['max_us']:10.2f}")
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"summary": r, "events": rows}, f)


if __name__ == "__main__":
    main()
