"""Decode kernels of the 16-column batch tile (B <= 16) fit three CTAs per SM: the cluster split-K GEMM and the one-shot decode
attention, whose grids of about two CTAs per SM leave a slot where, under PDL, the next kernel becomes resident (and starts its weight
stream) before the previous one drains.  Residency, grid and load order change, the arithmetic does not: graph-replayed decode equals
eager decode bit for bit, replays repeat exactly, and the split counts the schedule picks are the ones it picked before."""
import ctypes as C

import pytest
import torch

import visualcla_oracle as O

pytestmark = pytest.mark.gpu

STEPS = 64


@pytest.fixture(scope="module")
def eng():
    from visualcla.engine import Engine
    cfg = O.PathConfig(v_layers=1, r_layers=1, t_layers=8)          # 7B LLaMA widths, 8 layers
    e = Engine(cfg.to_dict(), max_batch=32, max_seq=STEPS + 40, page_tokens=64)
    e.init_synthetic(0)
    yield e
    e.close()


def _prompt(B, T=24):
    g = torch.Generator().manual_seed(1000 + B)
    return torch.randint(3, 49954, (B, T), generator=g)


def _decode(eng, B, use_graph):
    """Prefill B text prompts, then STEPS greedy steps one launch sequence (or one single-step graph replay) at a time ->
    (tokens (STEPS, B), logits (STEPS, B, V))."""
    _, first, _ = eng.prefill(_prompt(B), 0, None, last_logits=False)
    tok = eng.token_buffer(B)
    tok.copy_(first)
    logits = torch.empty(B, eng.vocab, dtype=torch.float32, device=eng.device)
    toks, logs = [], []
    for _ in range(STEPS):
        eng.decode_step(tok, tok, logits, use_graph=use_graph)
        toks.append(tok.clone())
        logs.append(logits.clone())
    torch.cuda.synchronize()
    return torch.stack(toks), torch.stack(logs)


@pytest.mark.parametrize("B", [1, 8, 16, 17, 32])
def test_graph_replayed_decode_equals_eager_bitwise(eng, B):
    """B <= 16 runs the kernels sized for a free third slot; B = 17 and 32 (the 32-column tile, the persistent attention) are
    checked the same way on their unchanged path."""
    t_eager, l_eager = _decode(eng, B, use_graph=False)
    t_graph, l_graph = _decode(eng, B, use_graph=True)
    assert torch.equal(t_eager, t_graph)
    assert torch.equal(l_eager.view(torch.int32), l_graph.view(torch.int32)), "logits differ in their bits"


@pytest.mark.parametrize("B", [1, 8, 16])
def test_sixteen_step_graph_replays_repeat_exactly(eng, B):
    runs = []
    for _ in range(10):
        _, first, _ = eng.prefill(_prompt(B), 0, None, last_logits=False)
        tok = eng.token_buffer(B)
        tok.copy_(first)
        eng.decode_many(tok, 16)
        runs.append(eng.read_history(B, 17).cpu())
    for r in runs[1:]:
        assert torch.equal(r, runs[0])


def _ctas_per_sm(eng, B):
    out = (C.c_int * 2)()
    assert eng.lib.vcla_debug_decode_ctas_per_sm(eng._ctx, B, C.byref(out)) == 0, eng.lib.vcla_last_error()
    return list(out)


def test_small_batch_decode_kernels_leave_a_third_slot(eng):
    """The GEMM of every B <= 16 and the one-shot attention (B = 1, 8: one wave at two CTAs per SM) fit three CTAs per SM.  At
    B = 16 attention is the persistent kernel (512 (sequence, head) items > 2 x SMs), which keeps two; so does everything of B > 16."""
    for B in (1, 2, 4, 8, 12, 16):
        gemm, attn = _ctas_per_sm(eng, B)
        assert gemm >= 3, f"B={B}: gemm_csk {gemm} CTAs/SM"
        if B <= 8:
            assert attn >= 3, f"B={B}: attention {attn} CTAs/SM"
    for B in (17, 32):
        assert _ctas_per_sm(eng, B) == [2, 2]


def test_split_counts_unchanged(eng):
    """The bound on clusters per launch that csk_pick chooses from is what the two-CTA configuration it replaced had, and so are the
    split counts it picks, which set the fp32 summation order.  Values for the 132-SM H100 SXM."""
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("split counts pinned for a 132-SM H100")
    want = {1: [8, 8, 8, 8, 8], 8: [8, 8, 8, 8, 8], 16: [8, 8, 8, 8, 8]}
    for B, v in want.items():
        got = (C.c_int * 5)()
        assert eng.lib.vcla_debug_get_csk_splits(eng._ctx, B, C.byref(got)) == 0
        assert list(got) == v, f"B={B}: splits {list(got)} (qkv, o, gate_up, down, lm_head), expected {v}"
        clusters = [eng.lib.vcla_op_gemm_csk_clusters(B, S) for S in range(1, 9)]
        assert clusters == [528, 264, 158, 124, 94, 78, 64, 60], f"B={B}: cluster bound for S = 1..8 CTAs per cluster {clusters}"
