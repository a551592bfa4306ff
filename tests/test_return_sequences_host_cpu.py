"""generate(do_sample=True, num_return_sequences=N) on the CPU: the engine traffic of the fork, without a GPU.  A fake engine with the
fan-out surface (set_fanout, a prefill that returns B * N first picks and (B, V) last logits, decode over B * N rows, the device
sampler's EOS semantics and the token ring) records every call.  Checked: one set_fanout + one prefill per chunk, decode over B * N
rows, the row order b * N + j, the EOS cut over all rows, chunking above the row bound, the host loop prefilling once, the refusals,
and that a call with num_return_sequences=1 makes exactly the engine calls of tests/golden/generate_trace.json."""
import json
import os
import types

import pytest
import torch

from visualcla.engine import Engine
from visualcla.modeling_visualcla import VclaKVCache, VisualCLAModel

V, NQ = 50, 4
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "generate_trace.json")


class FanoutEngine:
    """Toy model: row r of prompt b = r // N starts with (7 * last_id[b] + 3 + r) % V and continues with (5 * prev + 1 + step + r) % V,
    so every row of a prompt draws its own tokens.  `eos_at[r]` (optional) makes row r emit token 0 at that step.  With a sampler spec a
    finished row emits pad.  Work is synchronous: everything enqueued is published to the ring at once."""
    device = torch.device("cpu")
    vocab, nq, max_seq, max_prefill_tokens = V, NQ, 64, 1024
    sampler_spec = staticmethod(Engine.sampler_spec)

    def __init__(self, log, max_batch=8, eos_at=None):
        self.log, self.max_batch, self.eos_at = log, max_batch, eos_at or {}
        self.session = 0
        self.fan, self.spec = 1, None
        self.armed, self.ring = False, []
        self.hist, self.finished = [], torch.zeros(0, dtype=torch.bool)
        self.bufs = {}

    def _buf(self, t):
        return self.bufs.setdefault(t.data_ptr(), len(self.bufs))

    def _finish(self, nxt):
        step = len(self.hist)
        for r, at in self.eos_at.items():
            if r < nxt.numel() and step == at:
                nxt[r] = 0
        s = self.spec
        if s is not None and s.n_eos:
            nxt = torch.where(self.finished, torch.full_like(nxt, s.pad_token_id), nxt)
            self.finished |= torch.isin(nxt.long(), torch.tensor(list(s.eos_token_id)[: s.n_eos]))
        return nxt

    def _emit(self, t):
        self.hist.append(t.clone())
        if self.armed:
            self.ring.append(t.clone())

    @staticmethod
    def first_pick(last_ids, n):
        r = torch.arange(last_ids.numel() * n)
        return ((last_ids.long().repeat_interleave(n) * 7 + 3 + r) % V).to(torch.int32)

    def vision_encode(self, px, return_embeds=False):
        self.log.append(["vision_encode", list(px.shape)])

    def set_fanout(self, n):
        self.log.append(["set_fanout", n])
        self.fan = n

    def set_sampler(self, spec):
        self.log.append(["set_sampler", spec is not None])
        self.spec = spec

    def sampler_supported(self):
        return True

    def prefill(self, ids, mode, rows, all_logits=False, last_logits=True, left_pad=None, pos_from_mask=True):
        B = ids.shape[0]
        self.log.append(["prefill", list(ids.shape), self.fan])
        self.session += 1
        self.hist, self.finished = [], torch.zeros(B * self.fan, dtype=torch.bool)
        first = self._finish(self.first_pick(ids[:, -1], self.fan))
        self._emit(first)
        ll = None
        if last_logits:
            ll = torch.zeros(B, V)
            ll[torch.arange(B), ids[:, -1].long() % V] = 5.0
        return ll, first, None

    def _step(self, tok_in, tok_out, logits=None):
        r = torch.arange(tok_in.numel())
        nxt = self._finish(((tok_in.long() * 5 + 1 + len(self.hist) + r) % V).to(torch.int32))
        if logits is not None:
            logits.zero_()
            logits[r, nxt.long()] = 5.0
        tok_out.copy_(nxt)
        self._emit(nxt)

    def decode_step(self, tok_in, tok_out, logits=None, use_graph=True):
        self.log.append(["decode_step", tok_in.numel(), logits is not None and list(logits.shape)])
        self._step(tok_in, tok_out, logits)

    def decode_many(self, tok, n):
        self.log.append(["decode_many", self._buf(tok), tok.numel(), n])
        self.session += 1
        for _ in range(n):
            self._step(tok, tok)

    def read_history(self, B, n):
        self.log.append(["read_history", B, n])
        return torch.stack(self.hist[:n], 0)[:, :B]

    def read_finished(self, B):
        self.log.append(["read_finished", B])
        return self.finished[:B].to(torch.int32)

    def stream_supported(self):
        return True

    def stream_arm(self, on):
        self.log.append(["stream_arm", bool(on)])
        self.armed = bool(on)
        if on:
            self.ring = []

    def stream_wait(self, target, timeout_us=-1):
        if len(self.ring) < target:
            raise RuntimeError(f"step {target} will never be published")
        return len(self.ring)

    def stream_read(self, lo, hi, B):
        self.log.append(["stream_read", lo, hi, B])
        return torch.stack(self.ring[lo:hi], 0)[:, :B]


def _model(eng):
    m = object.__new__(VisualCLAModel)
    m._engine, m._tok_buf = eng, {}
    m.image_at_head = False
    m.tokenizer = types.SimpleNamespace(img_start_token_id=40, img_end_token_id=41, img_token_id=42)
    return m


IDS = torch.tensor([[1, 5, 9, 12, 3], [1, 6, 11, 2, 8]])
SAMPLE = dict(do_sample=True, top_k=5, eos_token_id=None, pad_token_id=0)


def _calls(log, kind):
    return [c for c in log if c[0] == kind]


def _reference_rows(ids, n, steps, eos_at=None, eos=None):
    """the fake engine's tokens, computed row by row without it"""
    eng = FanoutEngine([], eos_at=eos_at)
    if eos:
        eng.spec = Engine.sampler_spec(do_sample=True, top_k=5, eos_token_id=eos, pad_token_id=0)
    eng.fan = n
    eng.prefill(ids, 0, None, last_logits=False)
    tok = eng.hist[0].clone()
    for _ in range(steps - 1):
        eng._step(tok, tok)
    return torch.stack(eng.hist, 1).long()


@pytest.fixture(autouse=True)
def _no_host_sampler_env(monkeypatch):
    monkeypatch.delenv("VCLA_HOST_SAMPLER", raising=False)


def test_device_graphs_fork_once_and_decode_all_rows():
    log = []
    eng = FanoutEngine(log)
    torch.manual_seed(0)
    out = _model(eng).generate(input_ids=IDS, **SAMPLE, num_return_sequences=3, max_new_tokens=9)
    assert out.shape == (6, 9) and out.dtype == torch.int64
    assert _calls(log, "set_fanout") == [["set_fanout", 3], ["set_fanout", 1]]
    assert _calls(log, "prefill") == [["prefill", [2, 5], 3]]
    # the fan-out brackets the prefill only; the sampler is set around all of it
    kinds = [c[0] for c in log]
    assert kinds[:4] == ["set_sampler", "set_fanout", "prefill", "set_fanout"] and kinds[-1] == "set_sampler"
    assert all(c[2] == 6 for c in _calls(log, "decode_many"))
    assert sum(c[3] for c in _calls(log, "decode_many")) == 8
    assert _calls(log, "read_history") == [["read_history", 6, 9]]
    assert torch.equal(out, _reference_rows(IDS, 3, 9))


def test_row_order_is_repeat_interleave():
    log = []
    torch.manual_seed(0)
    out = _model(FanoutEngine(log)).generate(input_ids=IDS, **SAMPLE, num_return_sequences=4, max_new_tokens=3)
    first = FanoutEngine.first_pick(IDS[:, -1], 4)
    for b in range(2):
        for j in range(4):
            assert int(out[b * 4 + j, 0]) == int(first[b * 4 + j]) == (7 * int(IDS[b, -1]) + 3 + b * 4 + j) % V
    assert len(set(out[:4, 0].tolist())) == 4          # the siblings of a prompt start with different tokens


def test_eos_cut_over_all_rows():
    log = []
    eos_at = {0: 2, 1: 4, 2: 3, 3: 1, 4: 6, 5: 5}     # row 4 finishes last, at step 6
    torch.manual_seed(0)
    kw = dict(SAMPLE, eos_token_id=[0], min_new_tokens=1)
    out = _model(FanoutEngine(log, eos_at=eos_at)).generate(input_ids=IDS, **kw, num_return_sequences=3, max_new_tokens=20)
    assert out.shape == (6, 7)
    for r, at in eos_at.items():
        assert int(out[r, at]) == 0 and bool((out[r, at + 1:] == 0).all())
    assert all(c[1] == 6 for c in _calls(log, "read_finished"))
    assert _calls(log, "prefill") == [["prefill", [2, 5], 3]]


def test_chunks_when_rows_exceed_the_bound():
    log = []
    ids = torch.tensor([[1, 5 + i, 9, 12 - i, 3 + i] for i in range(5)])
    torch.manual_seed(0)
    out = _model(FanoutEngine(log, max_batch=8)).generate(input_ids=ids, **SAMPLE, num_return_sequences=3, max_new_tokens=4)
    # 8 rows hold 2 prompts x 3 replies: chunks of 2, 2, 1 prompts, one fork and one prefill each
    assert _calls(log, "prefill") == [["prefill", [2, 5], 3], ["prefill", [2, 5], 3], ["prefill", [1, 5], 3]]
    assert _calls(log, "set_fanout") == [["set_fanout", 3], ["set_fanout", 1]] * 3
    assert [c[2] for c in _calls(log, "decode_many")] == [6, 6, 3]
    assert out.shape == (15, 4)
    for c, sl in enumerate([slice(0, 2), slice(2, 4), slice(4, 5)]):
        assert torch.equal(out[sl.start * 3: sl.stop * 3], _reference_rows(ids[sl], 3, 4))


def test_host_loop_prefills_once_and_decodes_all_rows():
    log = []
    torch.manual_seed(0)
    out = _model(FanoutEngine(log)).generate(input_ids=IDS, **SAMPLE, tfs=0.9, num_return_sequences=3, max_new_tokens=5,
                                             output_logits=True, return_dict_in_generate=True)
    assert _calls(log, "set_sampler") == []
    assert _calls(log, "prefill") == [["prefill", [2, 5], 3]]
    assert _calls(log, "set_fanout") == [["set_fanout", 3], ["set_fanout", 1]]
    assert _calls(log, "decode_step") == [["decode_step", 6, [6, V]]] * 4
    assert out.sequences.shape == (6, 5)
    assert [tuple(t.shape) for t in out.logits] == [(6, V)] * 5
    # step 0 scores the prompts' last logits once per reply
    assert torch.equal(out.logits[0][0], out.logits[0][2]) and torch.equal(out.logits[0][3], out.logits[0][5])
    assert out.past_key_values.ids is None


def test_streamed_puts_every_row():
    log = []
    puts = []

    class Streamer:
        def put(self, v):
            puts.append(tuple(v.shape))

        def end(self):
            puts.append("end")

    torch.manual_seed(0)
    out = _model(FanoutEngine(log)).generate(input_ids=IDS[:1], **SAMPLE, num_return_sequences=3, max_new_tokens=6, streamer=Streamer())
    assert puts == [(3, 0)] + [(3,)] * 6 + ["end"]
    assert all(c[3] == 3 for c in _calls(log, "stream_read"))
    assert _calls(log, "prefill") == [["prefill", [1, 5], 3]]
    assert torch.equal(out.cpu(), _reference_rows(IDS[:1], 3, 6))


def test_cache_handle_is_not_reusable_and_is_not_reused():
    log = []
    eng = FanoutEngine(log)
    m = _model(eng)
    torch.manual_seed(0)
    one = m.generate(input_ids=IDS[:1], **SAMPLE, max_new_tokens=3, return_dict_in_generate=True)
    assert one.past_key_values.ids is not None
    log.clear()
    nxt = torch.cat([IDS[:1], one.sequences[:, :2].cpu(), torch.tensor([[7, 8]])], 1)
    two = m.generate(input_ids=nxt, **SAMPLE, num_return_sequences=2, max_new_tokens=3, past_key_values=one.past_key_values,
                     return_dict_in_generate=True)
    assert _calls(log, "prefill") == [["prefill", [1, 9], 2]] and not any(c[0] in ("truncate", "extend") for c in log)
    assert isinstance(two.past_key_values, VclaKVCache) and two.past_key_values.ids is None
    assert two.sequences.shape == (2, 3)


def test_prompt_lookup_is_ignored_with_several_rows():
    log = []
    torch.manual_seed(0)
    out = _model(FanoutEngine(log)).generate(input_ids=IDS[:1], **SAMPLE, num_return_sequences=2, max_new_tokens=5,
                                             prompt_lookup_num_tokens=3)
    assert out.shape == (2, 5) and not any(c[0] == "set_lookup" for c in log)


@pytest.mark.parametrize("kw, exc, msg", [
    (dict(SAMPLE, num_return_sequences=9, max_new_tokens=4), NotImplementedError, "num_return_sequences=9 exceeds"),
    (dict(SAMPLE, num_return_sequences=3, max_new_tokens=4, streamer="streamer"), NotImplementedError, "streaming 3 prompts x 3"),
    (dict(do_sample=False, num_return_sequences=2, max_new_tokens=4), ValueError, "Greedy methods"),
])
def test_refusals(kw, exc, msg):
    log = []

    class Streamer:
        def put(self, v):
            pass

        def end(self):
            pass

    kw = {k: (Streamer() if v == "streamer" else v) for k, v in kw.items()}
    ids = torch.tensor([[1, 5 + i, 9, 12 - i, 3 + i] for i in range(3)])
    with pytest.raises(exc, match=msg):
        _model(FanoutEngine(log)).generate(input_ids=ids, **kw)
    assert log == []


@pytest.mark.parametrize("name", ["greedy_eos", "sample_top_k", "sample_top_k_eos", "host_tfs", "streamer", "streamer_sampled",
                                  "lookup_sampled", "kv_reuse", "above_max_batch", "beams_eos"])
def test_one_return_sequence_makes_todays_engine_calls(name, monkeypatch):
    """num_return_sequences=1 passed explicitly: exactly the engine calls (and results) the trace golden pins for the call without it"""
    import test_generate_trace_cpu as T
    kind, rows, kw, extra = T.CASES[name]
    if "num_return_sequences" not in kw:
        kw = dict(kw, num_return_sequences=1)
    monkeypatch.setitem(T.CASES, name, (kind, rows, kw, extra))
    with open(GOLDEN) as f:
        golden = json.load(f)[name]
    assert T.run_case(name) == golden
