"""Measure the device image pre-processing (csrc/preprocess.cu) on one GPU with the reference's CPU path timed beside it.

    python tools/preprocess_bench.py [--sizes 480x640,1080x1920,3000x4000] [--reps 200]

Per picture size one JSON line:
  device_us        both kernels + the tap-table upload, CUDA events on the launching stream, picture already in HBM
  e2e_us           host uint8 picture -> pixel_values in HBM through VclaImageProcessor.__call__ (H2D copy inside)
  algorithmic_mb   source window read + 8-bit intermediate written and read + planar float32 result written (DESIGN.md §3)
  gbps / frac      algorithmic bytes / device time against MEASURED_PEAKS.json's HBM copy bandwidth
  pil_us           the reference's path for the same picture: transformers' PIL-backed CLIPImageProcessor on one host core
The CPU leg is the reference's own dependency (Pillow via HF), not the oracle; it is the baseline, not the product.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from visualcla.image_processing_vcla import VclaImageProcessor  # noqa: E402


def hbm_peak_gbps():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as fh:
            d = json.load(fh)
        for k in ("hbm_gbs", "hbm_gbps", "hbm_copy_gbps"):
            if k in d:
                v = d[k]
                return float(v["burst"] if isinstance(v, dict) and "burst" in v else v), "MEASURED_PEAKS.json"
    except Exception:
        pass
    return 3350.0, "H100 SXM data-sheet"


def algorithmic_bytes(proc, h, w, side=224):
    first_h, count_h, _ = proc.resample_taps(w, _resized(h, w, side)[1])
    first_v, count_v, _ = proc.resample_taps(h, _resized(h, w, side)[0])
    rh, rw = _resized(h, w, side)
    top, left = (rh - side) // 2, (rw - side) // 2
    cols = int(first_h[left + side - 1] + count_h[left + side - 1] - first_h[left])
    rows = int(first_v[top + side - 1] + count_v[top + side - 1] - first_v[top])
    return 3 * rows * cols + 2 * 3 * rows * side + 3 * side * side * 4, rows, cols


def _resized(h, w, side):
    short, long = (w, h) if w <= h else (h, w)
    new_long = int(side * long / short)
    return (new_long, side) if w <= h else (side, new_long)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="224x224,480x640,1080x1920,3000x4000")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--no-pil", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    proc = VclaImageProcessor()
    peak, peak_src = hbm_peak_gbps()
    pil = None
    if not args.no_pil:
        try:
            from transformers.models.clip import CLIPImageProcessorPil as PilProcessor
        except ImportError:
            from transformers import CLIPImageProcessor as PilProcessor
        pil = PilProcessor()
        torch.set_num_threads(1)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")       # > 126 MB L2
    rng = np.random.default_rng(0)
    for tok in args.sizes.split(","):
        h, w = (int(v) for v in tok.lower().split("x"))
        img = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        dev_img = torch.from_numpy(img).cuda()
        for _ in range(5):
            proc(dev_img)
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            flush.zero_()                                                   # cold L2 for every timed call
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            proc(dev_img)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) * 1e3)
        device_us = float(np.median(times))
        t0 = time.perf_counter()
        n_e2e = max(10, args.reps // 10)
        for _ in range(n_e2e):
            proc(img)
        torch.cuda.synchronize()
        e2e_us = (time.perf_counter() - t0) / n_e2e * 1e6
        nbytes, rows, cols = algorithmic_bytes(proc, h, w)
        line = {"op": "clip_preprocess", "picture": f"{h}x{w}", "source_window": f"{rows}x{cols}", "device_us": round(device_us, 2),
                "e2e_us": round(e2e_us, 1), "algorithmic_mb": round(nbytes / 1e6, 3), "gbps": round(nbytes / device_us / 1e3, 1),
                "peak_gbps": peak, "peak_source": peak_src, "frac": round(nbytes / device_us / 1e3 / peak, 4),
                "timing": "CUDA events, median of %d, L2 flushed before each call" % args.reps, "gpu_launches_per_picture": 2}
        if pil is not None:
            from PIL import Image
            im = Image.fromarray(img)
            pil(images=im, return_tensors="pt")
            t0 = time.perf_counter()
            n = 0
            while time.perf_counter() - t0 < 2.0:
                pil(images=im, return_tensors="pt")
                n += 1
            line["pil_us"] = round((time.perf_counter() - t0) / n * 1e6, 1)
            line["cpu_baseline"] = {"kind": "reference", "cores": 1, "sample": f"{n} calls of transformers' PIL-backed CLIPImageProcessor"}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
