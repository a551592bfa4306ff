"""Tuning sweep of the cluster split-K decode GEMMs (csrc/gemm_decode.cu) on one GPU: for every decode GEMM shape and every cluster size S,
the kernel timed alone over 32 layers' distinct weights (vcla_bench_decode_gemm), then whole decode steps for a few S combinations.
    python tools/csk_sweep.py <batch> [out.json]
"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))
import torch  # noqa: E402
import visualcla  # noqa: E402
from visualcla import _native as N  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
out_path = sys.argv[2] if len(sys.argv) > 2 else None
N.load().vcla_set_pdl(1)
m = visualcla.VisualCLAModel.from_synthetic("7b", seed=0, max_batch=B, max_seq=512, max_prefill_tokens=B * 128)
m.image_at_head = True
eng = m._engine
lib = eng.lib
px = torch.randn(B, 3, 224, 224, device="cuda").half()
ids = torch.randint(3, 49954, (B, 64), device="cuda")


def get():
    a = (C.c_int * 5)()
    N.check(lib.vcla_debug_get_csk_splits(eng._ctx, B, C.byref(a)), "get")
    return list(a)


def setv(v):
    N.check(lib.vcla_debug_set_csk_splits(eng._ctx, B, *v), "set")


auto = get()
names = ["qkv", "o_proj", "gate_up", "down_proj", "lm_head"]
res = {"B": B, "auto": auto, "isolated_us": {}, "steps": []}
print("auto splits", dict(zip(names, auto)), "clusters", {s: lib.vcla_op_gemm_csk_clusters(B, s) for s in range(1, 9)})
for w, nm in enumerate(names):
    row = {}
    for S in range(1, 9):
        v = [0] * 5
        v[w] = S
        try:
            setv(v)
            if get()[w] != S:
                continue
            us, nbytes = eng.bench_decode_gemm(w, B, reps=3)
            row[S] = round(us, 2)
        except Exception as e:  # noqa: BLE001
            row[S] = "err: " + str(e)[:60]
    setv(auto)
    res["isolated_us"][nm] = row
    print(f"{nm:10s}", row)


def step_ms(v, n=48):
    setv(v)
    eng.vision_encode(px)
    _, tok, _ = eng.prefill(ids, 1, None, last_logits=False)
    tok = tok.clone()
    eng.decode_many(tok, 16)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    eng.decode_many(tok, n)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


best = [min((us, S) for S, us in res["isolated_us"][nm].items() if isinstance(us, float))[1] for nm in names]
combos = [auto, best]
for extra in ([6, 8, 5, 8, 3], [3, 8, 5, 8, 3], [6, 4, 5, 4, 3], [3, 4, 3, 4, 3], [4, 8, 4, 8, 4], [2, 4, 2, 4, 2], [6, 8, 6, 8, 6]):
    if extra not in combos:
        combos.append(extra)
for v in combos:
    try:
        ms = step_ms(v)
        res["steps"].append({"splits": v, "ms_per_token": ms})
        print("step", v, f"{ms:.4f} ms/token")
    except Exception as e:  # noqa: BLE001
        print("step", v, "err", str(e)[:100])
if out_path:
    json.dump(res, open(out_path, "w"), indent=1)
