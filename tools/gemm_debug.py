"""On-GPU diagnosis of the wgmma GEMM: runs a ladder of shapes from a single MMA k-block upwards and, on mismatch,
prints a coarse error map so descriptor / swizzle / pipeline bugs can be told apart in one run."""
import ctypes as C
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))
from visualcla import _native as N  # noqa: E402

lib = N.load()
st = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
p = lambda t: None if t is None else C.c_void_p(t.data_ptr())


def run(M, Nn, K, mode=1, tile_n=0, splits=1, pattern="rand"):
    g = torch.Generator().manual_seed(M * 7 + Nn * 3 + K)
    if pattern == "rand":
        A = torch.randn(M, K, generator=g)
        W = torch.randn(Nn, K, generator=g) / math.sqrt(K)
    else:  # structured: A[m,k] = 1 if k == m % K ; W[n,k] = n + k/1024  -> out[m,n] = W[n, m%K]
        A = torch.zeros(M, K)
        A[torch.arange(M), torch.arange(M) % K] = 1.0
        W = (torch.arange(Nn)[:, None] % 64).float() + (torch.arange(K)[None, :].float() / 256.0)
    A, W = A.to(torch.bfloat16).cuda(), W.to(torch.bfloat16).cuda()
    ref = A.float() @ W.float().t()
    try:
        if mode == 3:
            ws = torch.full((splits, Nn, M), float("nan"), device="cuda")   # here "A" = weights [M,K], W = batch rows [Nn,K]
            rc = lib.vcla_op_gemm(p(A), p(W), M, Nn, K, 3, 0, 0, None, p(ws), M, splits, 0, 0, st())
            torch.cuda.synchronize()
            out = ws.sum(0).t()
        else:
            out = torch.full((M, Nn), float("nan"), device="cuda")
            rc = lib.vcla_op_gemm(p(A), p(W), M, Nn, K, 1, 0, 0, None, p(out), Nn, 1, tile_n, 0, st())
            torch.cuda.synchronize()
    except Exception as e:  # noqa: BLE001
        print(f"  M={M} N={Nn} K={K} mode={mode} tile={tile_n}: EXCEPTION {e}")
        return False
    if rc != 0:
        print(f"  M={M} N={Nn} K={K} mode={mode} tile={tile_n}: rc={rc} {lib.vcla_last_error().decode()}")
        return False
    err = (out - ref).abs()
    nan = torch.isnan(out).float().mean().item()
    mx = torch.nan_to_num(err, nan=1e9).max().item()
    ok = mx <= 2e-2 * max(1.0, ref.abs().max().item())
    print(f"  M={M:5d} N={Nn:5d} K={K:5d} mode={mode} tile={tile_n:3d} splits={splits} {pattern:6s}: max err {mx:.3e} nan {nan:.3f} -> {'ok' if ok else 'BAD'}")
    if not ok:
        e = torch.nan_to_num(err, nan=99.0)
        rb, cb = max(1, M // 8), max(1, Nn // 8)
        print("    coarse error map (rows x cols, 8x8 blocks, max err per block):")
        for i in range(0, M, rb):
            print("    " + " ".join(f"{e[i:i + rb, j:j + cb].max().item():8.2e}" for j in range(0, Nn, cb)))
        if pattern != "rand":
            print("    out[0:4, 0:8]:", out[:4, :8].tolist())
            print("    ref[0:4, 0:8]:", ref[:4, :8].tolist())
    return ok


def main():
    print(lib.vcla_version().decode(), torch.cuda.get_device_name(0))
    allok = True
    print("[1] single tile, single k-block")
    allok &= run(128, 64, 64, tile_n=64, pattern="struct")
    allok &= run(128, 64, 64, tile_n=64)
    print("[2] K loop (multi k-block, pipeline wrap)")
    allok &= run(128, 64, 128, tile_n=64)
    allok &= run(128, 64, 1024, tile_n=64)
    print("[3] wider tiles")
    allok &= run(128, 128, 256, tile_n=128)
    allok &= run(128, 256, 256, tile_n=256)
    print("[4] multiple tiles / persistence / tails")
    allok &= run(512, 512, 512, tile_n=256)
    allok &= run(4096, 4096, 1024, tile_n=256)
    allok &= run(300, 392, 640, tile_n=0)
    print("[5] swap-AB split-K (decode)")
    allok &= run(128, 16, 64, mode=3)
    allok &= run(256, 8, 512, mode=3, splits=2)
    allok &= run(4096, 32, 4096, mode=3, splits=4)
    allok &= run(1003, 3, 256, mode=3)
    allok &= run(4096, 64, 1024, mode=3, splits=2)
    print("ALL OK" if allok else "SOME FAILED")
    return 0 if allok else 1


if __name__ == "__main__":
    sys.exit(main())
