"""Host side of generate(num_beams=K) on the CPU with a fake engine that has the beam surface: every refusal, num_return_sequences >
num_beams, chunking of batches by max_batch // K, output shapes and HF's fill value, and that num_beams=1 makes exactly the engine calls
it made before beam search existed."""
import types

import pytest
import torch

from visualcla import _native as N
from visualcla.modeling_visualcla import VclaKVCache, VisualCLAModel

V = 50


class BeamEngine:
    """Fake engine: prefill of n prompts forks to n * K rows; the store of item b holds K hypotheses whose tokens derive from the
    prompt's last id; hypothesis k of item b has length max_new - k (clamped to 1) and every item is done after the first poll."""
    device = torch.device("cpu")
    vocab, nq, max_batch, max_seq, max_prefill_tokens = V, 4, 8, 256, 256

    def __init__(self):
        self.calls, self.session, self._beam = [], 0, None

    @staticmethod
    def beam_spec(num_beams, max_new_tokens, **kw):
        return types.SimpleNamespace(num_beams=num_beams, max_new_tokens=max_new_tokens, **kw)

    def set_beam(self, spec):
        self.calls.append(("set_beam", None if spec is None else spec.num_beams))
        self._beam = spec

    def vision_encode(self, px, return_embeds=False):
        self.calls.append(("vision_encode",))

    def prefill(self, ids, mode, rows, all_logits=False, last_logits=True, left_pad=None, pos_from_mask=True):
        self.session += 1
        K = self._beam.num_beams if self._beam is not None else 1
        self.calls.append(("prefill", tuple(ids.shape), K))
        self.last = ids[:, -1].clone()
        first = (ids[:, -1] % V).to(torch.int32).repeat_interleave(K)
        return (torch.zeros(ids.shape[0], V) if last_logits else None), first, None

    def token_buffer(self, n):
        return torch.zeros(n, dtype=torch.int32)

    def decode_many(self, tok, n):
        self.session += 1
        self.calls.append(("decode_many", tok.numel(), n))
        self.hist.extend([tok.clone()] * n)

    def decode_step(self, tok_in, tok_out, logits=None, use_graph=True):
        self.calls.append(("decode_step", tok_in.numel()))
        tok_out.copy_((tok_in * 7 + 3) % V)

    def read_history(self, B, n):
        return torch.stack([torch.arange(B, dtype=torch.int32) + i for i in range(n)], 0)

    def read_beam_done(self, n):
        self.calls.append(("read_beam_done", n))
        return torch.ones(n, dtype=torch.int32)

    def read_beams(self, n):
        K, m = self._beam.num_beams, self._beam.max_new_tokens
        tok = torch.zeros(n, K, m, dtype=torch.int32)
        lens = torch.zeros(n, K, dtype=torch.int32)
        for b in range(n):
            for k in range(K):
                tok[b, k] = (int(self.last[b]) * 10 + k * 100 + torch.arange(m)) % 1000
                lens[b, k] = max(1, m - k)
        return tok, lens, torch.zeros(n, K), torch.ones(n, dtype=torch.int32)

    hist = []


def make_model():
    m = object.__new__(VisualCLAModel)
    m._engine = BeamEngine()
    m._tok_buf = {}
    m.image_at_head = True
    m.tokenizer = None
    return m


IDS = torch.tensor([[1, 5, 9], [1, 6, 8], [1, 7, 7], [1, 8, 6], [1, 9, 5]])


@pytest.mark.parametrize("kw", [dict(do_sample=True), dict(output_scores=True, return_dict_in_generate=True), dict(output_logits=True),
                                dict(num_beam_groups=2, diversity_penalty=0.5), dict(eos_token_id=[1, 2, 3, 4, 5]), dict(num_beams=16)],
                         ids=["sampling", "output_scores", "output_logits", "diverse", "five_eos", "too_many_beams"])
def test_refusals(kw):
    m = make_model()
    args = dict(num_beams=2, max_new_tokens=4, pad_token_id=0)
    args.update(kw)
    with pytest.raises(NotImplementedError):
        m.generate(input_ids=IDS[:1], **args)
    assert not any(c[0] == "prefill" for c in m._engine.calls)


def test_refusals_of_processors_criteria_and_streaming():
    m = make_model()
    with pytest.raises(NotImplementedError):
        m.generate(input_ids=IDS[:1], num_beams=2, max_new_tokens=4, logits_processor=[lambda i, s: s])
    with pytest.raises(NotImplementedError):
        m.generate(input_ids=IDS[:1], num_beams=2, max_new_tokens=4, stopping_criteria=[lambda i, s: False])
    with pytest.raises(NotImplementedError):
        m.generate(input_ids=IDS[:1], num_beams=2, max_new_tokens=4, streamer=object())


def test_num_return_sequences_above_num_beams_is_a_value_error():
    with pytest.raises(ValueError, match="num_return_sequences"):
        make_model().generate(input_ids=IDS[:1], num_beams=2, num_return_sequences=3, max_new_tokens=4)


def test_chunks_shapes_and_fill():
    m = make_model()
    out = m.generate(input_ids=IDS, num_beams=4, num_return_sequences=2, max_new_tokens=6, eos_token_id=40, pad_token_id=0)
    eng = m._engine
    prefills = [c for c in eng.calls if c[0] == "prefill"]
    assert [p[1][0] for p in prefills] == [2, 2, 1] and all(p[2] == 4 for p in prefills)       # max_batch 8 // 4 beams = 2 prompts
    assert ("set_beam", None) in eng.calls and eng._beam is None                              # beam mode is off afterwards
    assert out.shape == (5 * 2, 6) and out.dtype == torch.int64
    # hypothesis 1 of each item is one token shorter: filled with eos[0], because pad 0 is falsy (HF's output_fill_value)
    assert (out[1::2, 5] == 40).all() and (out[0::2, 5] != 40).all()
    assert int(out[0, 0]) == 90 and int(out[1, 0]) == 190
    m2 = make_model()
    o2 = m2.generate(input_ids=IDS[:1], num_beams=3, num_return_sequences=3, max_new_tokens=5, eos_token_id=None, pad_token_id=0)
    assert o2.shape == (3, 5) and int(o2[2, 4]) == -1                                          # no EOS: filled with -1
    m3 = make_model()
    o3 = m3.generate(input_ids=IDS[:1], num_beams=2, num_return_sequences=2, max_new_tokens=5, eos_token_id=40, pad_token_id=7)
    assert int(o3[1, 4]) == 7


def test_polls_between_graphs_of_eight_steps_and_returns_a_non_reusable_handle():
    m = make_model()
    eng = m._engine
    eng.read_beam_done = lambda n: (eng.calls.append(("read_beam_done", n)), torch.zeros(n, dtype=torch.int32))[1]
    r = m.generate(input_ids=IDS[:2], num_beams=2, max_new_tokens=20, eos_token_id=40, pad_token_id=0, return_dict_in_generate=True)
    steps = [c[2] for c in eng.calls if c[0] == "decode_many"]
    assert steps == [8, 8, 3] and all(c[1] == 4 for c in eng.calls if c[0] == "decode_many")
    assert sum(c[0] == "read_beam_done" for c in eng.calls) == 3
    assert r.sequences.shape == (2, 20)
    assert isinstance(r.past_key_values, VclaKVCache) and r.past_key_values.ids is None


def test_num_beams_one_makes_the_same_engine_calls():
    a, b = make_model(), make_model()
    ra = a.generate(input_ids=IDS[:2], max_new_tokens=5, eos_token_id=None, pad_token_id=0)
    rb = b.generate(input_ids=IDS[:2], num_beams=1, max_new_tokens=5, eos_token_id=None, pad_token_id=0)
    assert torch.equal(ra, rb)
    assert a._engine.calls == b._engine.calls
    assert not any(c[0] == "set_beam" for c in b._engine.calls)
    with pytest.raises(ValueError):                          # as before (HF's own check): several sequences need beam search
        make_model().generate(input_ids=IDS[:1], num_return_sequences=2, max_new_tokens=4)
