"""The fp32 restatement of the load_in_8bit quantiser (oracle/int8_oracle.py), pinned on its edge cases.  CPU only."""
import numpy as np

import int8_oracle as Q


def test_ties_round_half_to_even():
    # absmax 127 makes 127 / a == 1 exactly, so w * (127 / a) == w and the ties are the inputs themselves
    w = np.array([[127.0, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 3.5]], dtype=np.float32)
    q, s = Q.quantize(w)
    assert s[0] == np.float32(1.0)
    assert q.tolist() == [[127, 0, 2, 2, 0, -2, -2, 4]]


def test_zero_row_and_absmax():
    rng = np.random.default_rng(0)
    w = rng.standard_normal((5, 64)).astype(np.float32)
    w[2] = 0.0
    w[3, 7] = -10.0          # negative absmax maps to -127
    q, s = Q.quantize(w)
    assert s[2] == 0.0 and not q[2].any()
    assert q[3, 7] == -127
    for r in (0, 1, 3, 4):
        assert np.abs(q[r]).max() == 127
        assert s[r] == np.float32(np.abs(w[r]).max() / np.float32(127.0))
    assert q.dtype == np.int8 and s.dtype == np.float32


def test_quantize_of_dequantized_is_idempotent():
    rng = np.random.default_rng(1)
    w = (rng.standard_normal((64, 256)) * rng.uniform(1e-3, 10.0, (64, 1))).astype(np.float32)
    q, s = Q.quantize(w)
    q2, s2 = Q.quantize(Q.dequantize(q, s))
    assert np.array_equal(q2, q)
    assert np.allclose(s2, s, rtol=2 ** -23, atol=0)


def test_quantized_weights_replace_only_the_projections():
    import torch
    w = {"text_model.model.layers.0.self_attn.q_proj.weight": torch.randn(8, 64),
         "text_model.model.layers.0.mlp.down_proj.weight": torch.randn(8, 64),
         "text_model.lm_head.weight": torch.randn(8, 64),
         "text_model.model.embed_tokens.weight": torch.randn(8, 64),
         "visual_resampler.encoder.layer.0.crossattention.self.query.weight": torch.randn(8, 64)}
    out = Q.quantized_weights(w)
    for k in w:
        assert torch.equal(out[k], w[k]) != Q.is_q8(k), k
