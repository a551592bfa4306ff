"""Targets for ncu: runs only the kernel of interest so `ncu -k regex:... -s N -c 3` lands on it.
  python tools/profile_gemm.py decode [which] [B]   -> decode swap-AB weight-streaming GEMM over the 32 layers' weights
  python tools/profile_gemm.py prefill              -> prefill wgmma GEMM  (1024 x 12288 x 4096, tile 64x256)
  python tools/profile_gemm.py step [B]             -> one full prefill + 4 decode steps (launch list)"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "visual-chinese-llama-alpaca_b200"))
import torch  # noqa: E402
import visualcla  # noqa: E402
from visualcla import _native as N  # noqa: E402

mode = sys.argv[1] if len(sys.argv) > 1 else "decode"
if mode == "prefill":
    lib = N.load()
    M, Nn, K = 1024, 12288, 4096
    A = torch.randn(M, K, device="cuda").bfloat16()
    W = (torch.randn(Nn, K, device="cuda") / 64).bfloat16()
    out = torch.empty(M, Nn, device="cuda", dtype=torch.bfloat16)
    for _ in range(6):
        rc = lib.vcla_op_gemm(C.c_void_p(A.data_ptr()), C.c_void_p(W.data_ptr()), M, Nn, K, 0, 0, 0, None, C.c_void_p(out.data_ptr()), Nn, 1, 0, 0,
                              C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, lib.vcla_last_error()
    torch.cuda.synchronize()
    print("prefill gemm done")
else:
    B = int(sys.argv[3]) if len(sys.argv) > 3 else 8
    m = visualcla.VisualCLAModel.from_synthetic("7b", seed=0, max_batch=B, max_seq=400, max_prefill_tokens=B * 128)
    if mode == "decode":
        which = int(sys.argv[2]) if len(sys.argv) > 2 else 2
        us, nbytes = m._engine.bench_decode_gemm(which, B, reps=1)
        print(f"decode gemm which={which} B={B}: {us:.2f} us/launch, {nbytes / us / 1e3:.1f} GB/s")
    else:
        B = int(sys.argv[2]) if len(sys.argv) > 2 else 8
        px = torch.randn(B, 3, 224, 224, device="cuda").half()
        ids = torch.randint(3, 49954, (B, 64), device="cuda")
        m.image_at_head = True
        out = m.generate(input_ids=ids, pixel_values=px, do_sample=False, max_new_tokens=5, eos_token_id=None, pad_token_id=0)
        torch.cuda.synchronize()
        print("step done", out.shape)
