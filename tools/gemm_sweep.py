"""Tile-shape sweep of the prefill wgmma GEMM on the path's shapes (TFLOP/s per tile N)."""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))
import torch  # noqa: E402
from visualcla import _native as N  # noqa: E402

lib = N.load()
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
shapes = [("qkv", 1024, 12288, 4096), ("o", 1024, 4096, 4096), ("gate_up", 1024, 22016, 4096), ("down", 1024, 4096, 11008),
          ("qkv32", 6144, 12288, 4096), ("o32", 6144, 4096, 4096), ("gate_up32", 6144, 22016, 4096), ("down32", 6144, 4096, 11008),
          ("vit_qkv", 2056, 3072, 1024), ("vit_fc1", 2056, 4096, 1024), ("vit_fc2", 2056, 1024, 4096), ("vit_qkv32", 8224, 3072, 1024)]
for name, M, Nn, K in shapes:
    A = torch.randn(M, K, device="cuda").bfloat16()
    W = (torch.randn(Nn, K, device="cuda") / 64).bfloat16()
    out = torch.empty(M, Nn, device="cuda", dtype=torch.bfloat16)
    res = []
    for tn in (64, 128, 256):
        def run():
            rc = lib.vcla_op_gemm(C.c_void_p(A.data_ptr()), C.c_void_p(W.data_ptr()), M, Nn, K, 0, 0, 0, None, C.c_void_p(out.data_ptr()), Nn, 1, tn, 0, st)
            assert rc == 0
        for _ in range(3):
            run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            run()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        res.append(f"bn{tn}: {ms * 1000:7.1f} us {2 * M * Nn * K / ms / 1e9:7.1f} TF/s")
    print(f"{name:10s} M={M:5d} N={Nn:5d} K={K:5d} | " + " | ".join(res), flush=True)
