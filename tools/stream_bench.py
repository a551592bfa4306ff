"""Cost of token streaming at 7B widths (synthetic weights): one image + a 64-token prompt (configs[1]-shaped), B = 1 and 8,
DEFAULT_GENERATION_CONFIG (sampling, repetition penalty, no-repeat-ngram), 256 new tokens.

    python tools/stream_bench.py [--batches 1 8] [--new 256] [--reps 12]

(a) decode step time with the token ring armed vs disarmed: CUDA events around replays of the same 8-step decode graph, the two
    arms alternating in one run; median and spread (min..max) per step.
(b) whole generations as a streaming consumer sees them, for the device streaming path (generate(streamer=...)), the per-step
    host loop (VCLA_HOST_SAMPLER=1) and non-streamed device generate(): wall time, time to first token, p50 / p99 of the gaps
    between the tokens the consumer receives.  Prints one JSON line per measurement.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(round(q / 100 * (len(xs) - 1))))]


class Clock:
    """streamer: arrival time of every put after the first (the empty prompt put)."""

    def __init__(self, t0):
        self.t0, self.times, self.first = t0, [], True

    def put(self, value):
        if self.first:
            self.first = False
            return
        self.times.append(time.perf_counter())

    def end(self):
        pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--skip-host", action="store_true")
    a = ap.parse_args()
    import visualcla
    from visualcla import _native as N
    from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG
    print(json.dumps(dict(card=card())), flush=True)
    torch.cuda.set_device(0)
    T, nq = 64, 64
    model = visualcla.VisualCLAModel.from_synthetic("7b", seed=0, max_batch=max(a.batches), max_seq=T + nq + a.new + 8)
    eng = model._engine
    cfg = model.config.to_path_config()
    gen = torch.Generator().manual_seed(0)
    for B in a.batches:
        px = torch.randn(B, 3, cfg["v_image"], cfg["v_image"], generator=gen).cuda()
        ids = torch.randint(3, 30000, (B, T), generator=gen)
        ids[:, 0] = 1
        ids = ids.cuda()
        # ---- (a) step time, armed vs disarmed ----
        eng.vision_encode(px)
        spec = eng.sampler_spec(do_sample=True, repetition_penalty=1.1, no_repeat_ngram_size=15, temperature=0.5, top_k=40, top_p=0.9, seed=1)
        eng.set_sampler(spec)
        tok = eng.token_buffer(B)
        times = {False: [], True: []}
        for rep in range(a.reps + 2):
            for armed in ((False, True) if rep % 2 == 0 else (True, False)):
                eng.stream_arm(armed)
                _, first, _ = eng.prefill(ids, N.IMAGE_AT_HEAD, None, last_logits=False)
                tok.copy_(first)
                eng.decode_many(tok, 8)                     # warm: the graph exists and the pages are reserved
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(4):
                    eng.decode_many(tok, 8)
                e1.record()
                torch.cuda.synchronize()
                eng.stream_arm(False)
                if rep >= 2:
                    times[armed].append(e0.elapsed_time(e1) * 1e3 / 32)
        eng.set_sampler(None)
        for armed in (False, True):
            xs = times[armed]
            print(json.dumps(dict(B=B, what="decode_step_us", armed=armed, median=round(pct(xs, 50), 1), min=round(min(xs), 1),
                                  max=round(max(xs), 1), n=len(xs))), flush=True)
        # ---- (b) whole generations ----
        gc = DEFAULT_GENERATION_CONFIG.__class__(**{**DEFAULT_GENERATION_CONFIG.to_dict(), "max_new_tokens": a.new, "pad_token_id": 0})
        modes = [("device_streamed", True, None), ("device_plain", False, None)] + ([] if a.skip_host else [("host_loop_streamed", True, "1")])
        for rep in range(3):
            for name, stream, host in modes:
                if host:
                    os.environ["VCLA_HOST_SAMPLER"] = host
                torch.manual_seed(rep)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                clk = Clock(t0)
                out = model.generate(input_ids=ids, pixel_values=px, generation_config=gc, **(dict(streamer=clk) if stream else {}))
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                os.environ.pop("VCLA_HOST_SAMPLER", None)
                if rep == 0:
                    continue                                # warm-up (graph capture, allocations)
                ts = clk.times
                gaps = [(y - x) * 1e3 for x, y in zip(ts, ts[1:])]
                print(json.dumps(dict(B=B, what="generate", mode=name, rep=rep, tokens=int(out.shape[1]), wall_ms=round((t1 - t0) * 1e3, 1),
                                      ttft_ms=round(((ts[0] if ts else t1) - t0) * 1e3, 1),
                                      gap_p50_ms=round(pct(gaps, 50), 3) if gaps else None,
                                      gap_p99_ms=round(pct(gaps, 99), 3) if gaps else None)), flush=True)


if __name__ == "__main__":
    main()
