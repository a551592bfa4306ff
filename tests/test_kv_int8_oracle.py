"""CPU checks of the int8 KV cache reference (tests/kv_int8_reference.py): the hooked LLaMA forward without its hook is the oracle's
forward bit for bit, the row quantiser is load_in_8bit's (zero rows, exact .5 ties, the +-127 clamp), and attention over the
dequantised rows is scaled_dot_product_attention's."""
import numpy as np
import torch
import torch.nn.functional as F

import int8_oracle as Q
import visualcla_oracle as O
from kv_int8_reference import dequantize_rows, generate_greedy_q8, llama_forward_q8, quantize_rows


def test_hook_off_is_the_oracle_bit_for_bit():
    cfg = O.tiny_config()
    w = O.make_weights(cfg, 0)
    px, ids = O.make_inputs(cfg, 2, 12, seed=1234)
    x = O.splice(w, cfg, ids, O.vision_encode(w, cfg, px), True, *[O.special_ids(cfg)[i] for i in (0, 1, 3)])
    assert torch.equal(llama_forward_q8(w, cfg, x, kv_hook=None), O.llama_forward(w, cfg, x))
    tok_ref, log_ref = O.generate_greedy(w, cfg, ids, px, 4)
    tok, log = generate_greedy_q8(w, cfg, ids, px, 4, kv_hook=None)
    assert torch.equal(tok, tok_ref) and torch.equal(log, log_ref)


def test_hook_on_changes_the_model_slightly():
    cfg = O.tiny_config()
    w = O.make_weights(cfg, 0)
    px, ids = O.make_inputs(cfg, 2, 12, seed=1234)
    _, log_ref = O.generate_greedy(w, cfg, ids, px, 3)
    _, log = generate_greedy_q8(w, cfg, ids, px, 3)
    err = ((log - log_ref).abs().max() / log_ref.abs().max()).item()
    assert 0 < err < 5e-2


def test_row_quantiser_edge_cases():
    x = torch.zeros(4, 128)
    x[1, 0] = 127.0                     # a = 127: s = 1, so x = k + 0.5 is an exact tie that rounds to even
    x[1, 1:6] = torch.tensor([0.5, 1.5, 2.5, -0.5, -2.5])
    x[2] = torch.linspace(-3.0, 3.0, 128)
    x[3, 5] = -1e-30                    # tiny rows quantise to +-127 at their absmax
    q, s = quantize_rows(x)
    assert s[0] == 0 and not q[0].any()
    assert s[1] == 1.0 and q[1, :6].tolist() == [127, 0, 2, 2, 0, -2]
    assert q[2].abs().max() == 127 and q[2, 0] == -127 and q[2, -1] == 127
    assert q[3, 5] == -127
    assert q.abs().max() <= 127


def test_row_quantiser_is_the_weight_quantiser():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(64, 128, generator=g) * torch.logspace(-3, 3, 64)[:, None]
    q, s = quantize_rows(x.view(4, 16, 128))
    qw, sw = Q.quantize(x)
    assert np.array_equal(q.reshape(64, 128).numpy(), qw) and np.array_equal(s.reshape(64).numpy(), sw)
    assert torch.equal(dequantize_rows(q, s).reshape(64, 128), torch.from_numpy(Q.dequantize(qw, sw)))


def test_decode_reference_is_sdpa_on_dequantised_rows():
    g = torch.Generator().manual_seed(5)
    H, L = 4, 37
    q = torch.randn(H, 128, generator=g, dtype=torch.float64)
    kq, ks = quantize_rows(torch.randn(L, H, 128, generator=g))
    vq, vs = quantize_rows(torch.randn(L, H, 128, generator=g))
    K, V = kq.double() * ks.double()[..., None], vq.double() * vs.double()[..., None]
    # the kernels' form: s_k * sum q k for the score, (p s_v) v for the accumulator
    score = torch.einsum("hd,lhd->hl", q, kq.double()) * ks.double().T * 128 ** -0.5
    p = torch.softmax(score, dim=-1)
    out = torch.einsum("hl,lhd->hd", p * vs.double().T, vq.double())
    ref = F.scaled_dot_product_attention(q[:, None, None], K.permute(1, 0, 2)[:, None], V.permute(1, 0, 2)[:, None])[:, 0, 0]
    assert torch.allclose(out, ref, rtol=1e-12, atol=1e-12)
