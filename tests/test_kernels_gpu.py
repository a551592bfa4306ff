"""Operator-level parity of the CUDA kernels, called through the C ABI (include/vcla.h) and checked against plain
torch fp32 math on the same bf16-rounded inputs.  GPU only."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from visualcla import _native as N
    return N.load()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _check(lib, rc):
    assert rc == 0, lib.vcla_last_error().decode()


def _rand(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).cuda()


def _gemm(lib, A, W, mode, act=0, accumulate=0, bias=None, out=None, ldo=None, splits=1, tile_n=0, ref=0):
    M, K = A.shape
    N = W.shape[0]
    _check(lib, lib.vcla_op_gemm(_p(A), _p(W), M, N, K, mode, act, accumulate, _p(bias), _p(out), ldo, splits, tile_n, ref, _stream()))
    torch.cuda.synchronize()


GEMM_SHAPES = [
    (128, 256, 64), (128, 256, 512), (257, 1024, 1024), (300, 392, 640), (64, 4096, 1024),
    (1024, 12288, 4096), (96, 1003, 256), (17, 64, 128), (514, 3072, 1024),
]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
@pytest.mark.parametrize("tile_n", [0, 64, 128, 256])
def test_gemm_store_bf16(lib, M, N, K, tile_n):
    A, W = _rand((M, K), 1.0, 1), _rand((N, K), 1.0 / math.sqrt(K), 2)
    bias = torch.randn(N, device="cuda")
    out = torch.full((M, N), float("nan"), dtype=torch.bfloat16, device="cuda")
    _gemm(lib, A, W, 0, act=0, bias=bias, out=out, ldo=N, tile_n=tile_n)
    ref = A.float() @ W.float().t() + bias
    err = (out.float() - ref).abs().max().item()
    assert err <= 2e-2 * max(1.0, ref.abs().max().item()), f"max err {err}"


@pytest.mark.parametrize("act", [1, 2])
def test_gemm_activations(lib, act):
    M, N, K = 257, 512, 256
    A, W = _rand((M, K), 1.0, 3), _rand((N, K), 1.0 / math.sqrt(K), 4)
    bias = torch.randn(N, device="cuda") * 0.5
    out = torch.empty((M, N), dtype=torch.bfloat16, device="cuda")
    _gemm(lib, A, W, 0, act=act, bias=bias, out=out, ldo=N)
    x = A.float() @ W.float().t() + bias
    ref = x * torch.sigmoid(1.702 * x) if act == 1 else torch.nn.functional.gelu(x)
    assert (out.float() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("M,N,K", [(257, 1024, 4096), (130, 1003, 256), (128, 4096, 11008)])
@pytest.mark.parametrize("accumulate", [0, 1])
def test_gemm_f32_residual(lib, M, N, K, accumulate):
    A, W = _rand((M, K), 1.0, 5), _rand((N, K), 1.0 / math.sqrt(K), 6)
    bias = torch.randn(N, device="cuda")
    base = torch.randn(M, N, device="cuda")
    out = base.clone()
    _gemm(lib, A, W, 1, accumulate=accumulate, bias=bias, out=out, ldo=N)
    ref = A.float() @ W.float().t() + bias + (base if accumulate else 0)
    err = (out - ref).abs().max().item()
    assert err <= 2e-3 * max(1.0, ref.abs().max().item()), f"max err {err}"


def test_gemm_matches_naive_kernel(lib):
    """wgmma path vs the CUDA-core reference kernel inside the library (same epilogue semantics)."""
    M, N, K = 200, 320, 448
    A, W = _rand((M, K), 1.0, 7), _rand((N, K), 1.0 / math.sqrt(K), 8)
    o1 = torch.zeros((M, N), device="cuda")
    o2 = torch.zeros((M, N), device="cuda")
    _gemm(lib, A, W, 1, out=o1, ldo=N)
    _gemm(lib, A, W, 1, out=o2, ldo=N, ref=1)
    assert (o1 - o2).abs().max().item() <= 1e-3


@pytest.mark.parametrize("M,F,K", [(128, 448, 256), (300, 11008, 4096)])
def test_gemm_swiglu(lib, M, F, K):
    A = _rand((M, K), 1.0, 9)
    Wg, Wu = _rand((F, K), 1.0 / math.sqrt(K), 10), _rand((F, K), 1.0 / math.sqrt(K), 11)
    # interleave [32 gate | 32 up]
    W = torch.empty(2 * F, K, dtype=torch.bfloat16, device="cuda")
    Wv = W.view(F // 32, 2, 32, K)
    Wv[:, 0] = Wg.view(F // 32, 32, K)
    Wv[:, 1] = Wu.view(F // 32, 32, K)
    out = torch.empty((M, F), dtype=torch.bfloat16, device="cuda")
    _gemm(lib, A, W, 2, out=out, ldo=F)
    g, u = A.float() @ Wg.float().t(), A.float() @ Wu.float().t()
    ref = torch.nn.functional.silu(g) * u
    assert (out.float() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("Nout,K,B,splits", [(4096, 4096, 8, 4), (12288, 4096, 1, 4), (4096, 11008, 32, 9), (1003, 256, 3, 1),
                                              (22016, 4096, 16, 2), (49958, 4096, 64, 2), (512, 448, 5, 7)])
def test_gemm_swap_ab_splitk(lib, Nout, K, B, splits):
    """decode GEMM: A = weights [Nout,K] streamed once, B = activations [B,K]; fp32 partials [splits][B][Nout]."""
    Wt, X = _rand((Nout, K), 1.0 / math.sqrt(K), 12), _rand((B, K), 1.0, 13)
    ws = torch.full((splits, B, Nout), float("nan"), device="cuda")
    _check(lib, lib.vcla_op_gemm(_p(Wt), _p(X), Nout, B, K, 3, 0, 0, None, _p(ws), Nout, splits, 0, 0, _stream()))
    torch.cuda.synchronize()
    got = ws.sum(0)
    ref = X.float() @ Wt.float().t()
    assert not torch.isnan(ws).any()
    err = (got - ref).abs().max().item()
    assert err <= 2e-3 * max(1.0, ref.abs().max().item()), f"max err {err}"


@pytest.mark.parametrize("rows,D", [(514, 1024), (7, 128), (96, 4096)])
def test_layernorm_rmsnorm(lib, rows, D):
    x = torch.randn(rows, D, device="cuda") * 3 + 0.5
    w, b = torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    yb = torch.empty(rows, D, dtype=torch.bfloat16, device="cuda")
    yf = torch.empty(rows, D, device="cuda")
    _check(lib, lib.vcla_op_layernorm(_p(x), rows, D, _p(w), _p(b), 1e-5, _p(yb), _p(yf), _stream()))
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x, (D,), w, b, 1e-5)
    assert (yf - ref).abs().max().item() <= 1e-4
    assert (yb.float() - ref).abs().max().item() <= 4e-2
    _check(lib, lib.vcla_op_rmsnorm(_p(x), rows, D, _p(w), 1e-6, _p(yb), _stream()))
    torch.cuda.synchronize()
    ref = w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6))
    assert (yb.float() - ref).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())


# ---------------------------------------------------------------------------------------------------------------
# decode GEMM with the split-K reduction inside a thread-block cluster (csrc/gemm_decode.cu)
# ---------------------------------------------------------------------------------------------------------------
def _csk(lib, W, X, splits, mode, out_or_resid=None, norm_w=None, xw_or_h=None, ssq_out=None, ssq_in=None, slots=0, inv_dim=0.0, eps=0.0):
    M, K = W.shape
    B = X.shape[0]
    _check(lib, lib.vcla_op_gemm_csk(_p(W), _p(X), M, B, K, splits, mode, _p(out_or_resid), _p(norm_w), _p(xw_or_h), _p(ssq_out), _p(ssq_in), slots,
                                     inv_dim, eps, _stream()))
    torch.cuda.synchronize()


CSK_CASES = [(4096, 4096, 8, 8), (4096, 4096, 1, 8), (12288, 4096, 8, 6), (12288, 4096, 3, 3), (4096, 11008, 8, 8), (1003, 256, 5, 2), (4096, 4096, 16, 8),
             (4096, 4096, 17, 8), (12288, 4096, 32, 5), (4096, 11008, 29, 7), (49958, 4096, 8, 3), (640, 1024, 13, 1)]


@pytest.mark.parametrize("M,K,B,S", CSK_CASES)
def test_csk_out_f32_with_deferred_scale(lib, M, K, B, S):
    W, X = _rand((M, K), 1.0 / math.sqrt(K), 11), _rand((B, K), 1.0, 12)
    slots = 7
    ssq = torch.rand(B, slots, device="cuda") * 50.0
    out = torch.full((B, M), float("nan"), device="cuda")
    _csk(lib, W, X, S, 0, out_or_resid=out, ssq_in=ssq, slots=slots, inv_dim=1.0 / K, eps=1e-6)
    rstd = torch.rsqrt(ssq.sum(1) / K + 1e-6)
    ref = (X.float() @ W.float().t()) * rstd[:, None]
    err = (out - ref).abs().max().item()
    assert err <= 2e-3 * max(1.0, ref.abs().max().item()), f"max err {err}"
    out2 = torch.empty_like(out)
    _csk(lib, W, X, S, 0, out_or_resid=out2, ssq_in=ssq, slots=slots, inv_dim=1.0 / K, eps=1e-6)
    assert torch.equal(out, out2), "fixed reduction order: bit-identical run to run"


@pytest.mark.parametrize("M,K,B,S", [(4096, 4096, 8, 8), (4096, 11008, 8, 8), (4096, 4096, 32, 8), (1024, 2752, 5, 4), (4096, 11008, 19, 6)])
def test_csk_residual_next_operand_and_row_statistics(lib, M, K, B, S):
    W, X = _rand((M, K), 1.0 / math.sqrt(K), 13), _rand((B, K), 1.0, 14)
    resid0 = torch.randn(B, M, device="cuda")
    norm_w = torch.randn(M, device="cuda") * 0.1 + 1.0
    resid = resid0.clone()
    xw = torch.empty(B, M, dtype=torch.bfloat16, device="cuda")
    tiles = (M + 127) // 128
    ssq = torch.full((B, tiles), float("nan"), device="cuda")
    _csk(lib, W, X, S, 1, out_or_resid=resid, norm_w=norm_w, xw_or_h=xw, ssq_out=ssq)
    ref = resid0 + X.float() @ W.float().t()
    assert (resid - ref).abs().max().item() <= 2e-3 * max(1.0, ref.abs().max().item())
    assert (xw.float() - resid * norm_w).abs().max().item() <= 1e-2 * (resid * norm_w).abs().max().item()
    want = torch.nn.functional.pad(resid, (0, tiles * 128 - M)).view(B, tiles, 128).pow(2).sum(-1)
    assert (ssq - want).abs().max().item() <= 1e-4 * want.max().item()


@pytest.mark.parametrize("F,K,B,S", [(11008, 4096, 8, 5), (11008, 4096, 32, 5), (1408, 512, 3, 2), (2752, 1024, 17, 4)])
def test_csk_swiglu(lib, F, K, B, S):
    g, u = _rand((F, K), 1.0 / math.sqrt(K), 15), _rand((F, K), 1.0 / math.sqrt(K), 16)
    assert F % 32 == 0
    W = torch.stack([g.view(F // 32, 32, K), u.view(F // 32, 32, K)], 1).reshape(2 * F, K).contiguous()     # [32 gate | 32 up] blocks
    X = _rand((B, K), 1.0, 17)
    ssq = torch.rand(B, 3, device="cuda") * 30.0
    h = torch.empty(B, F, dtype=torch.bfloat16, device="cuda")
    _csk(lib, W, X, S, 2, xw_or_h=h, ssq_in=ssq, slots=3, inv_dim=1.0 / K, eps=1e-6)
    rstd = torch.rsqrt(ssq.sum(1) / K + 1e-6)[:, None]
    ref = torch.nn.functional.silu((X.float() @ g.float().t()) * rstd) * ((X.float() @ u.float().t()) * rstd)
    assert (h.float() - ref).abs().max().item() <= 1.5e-2 * max(1.0, ref.abs().max().item())
