"""Host side of streaming generation (generate(streamer=...), Stream stopping criteria, chat_in_stream) on the CPU, with a fake
engine that emulates the device token ring (include/vcla.h, token streaming): every token choice publishes its step while armed.
Covers which calls stream on the device, the HF order of streamer.put / criteria / end, the cut at EOS and at a consumer stop, the
bound on decode steps run past the cut, the KV-cache handle, and -- against tests/golden/tiny_stream.npz, recorded from the
reference -- the exact event list a streamer and a criterion observe."""
import json
import os
import types

import numpy as np
import pytest
import torch

from visualcla import _native as N
from visualcla.engine import Engine
from visualcla.modeling_utils import Stream
from visualcla.modeling_visualcla import VclaKVCache, VisualCLAModel

V, NQ = 50, 4
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_stream.npz")


class RingEngine:
    """Deterministic toy model (next token = (7 * previous + 3) % V, or a fixed script per step) with the device sampler's EOS
    semantics (a finished row emits pad) and an emulated stream ring.  Work is synchronous: everything enqueued is published."""
    device = torch.device("cpu")
    vocab, nq, max_batch, max_seq, max_prefill_tokens = V, NQ, 4, 256, 1024
    sampler_spec = staticmethod(Engine.sampler_spec)

    def __init__(self, script=None):
        self.script = script            # (B, L) tokens of step 0..L-1; later steps emit 0
        self.session = 0
        self.armed = False
        self.ring = []
        self.spec = None
        self.calls = []
        self.decode_steps = 0
        self.truncated = None

    # ---- token choice -------------------------------------------------------------------------
    def _pick(self, prev, first=False):
        step = len(self.hist)
        if self.script is not None:
            nxt = self.script[:, step] if step < self.script.shape[1] else torch.zeros(self.script.shape[0], dtype=torch.int64)
            nxt = nxt.to(torch.int32)
        else:
            nxt = prev if first else ((prev.long() * 7 + 3) % V).to(torch.int32)
        s = self.spec
        if s is not None and s.n_eos:
            eos = torch.tensor(list(s.eos_token_id)[: s.n_eos])
            nxt = torch.where(self.finished, torch.full_like(nxt, s.pad_token_id), nxt)
            self.finished |= torch.isin(nxt.long(), eos)
        return nxt

    def _choose(self, tok):
        self.hist.append(tok.clone())
        if self.armed:
            self.ring.append(tok.clone())

    def _start(self, first):
        self.hist = []
        self.finished = torch.zeros(first.shape[0], dtype=torch.bool)
        first = self._pick(first, first=True)
        self._choose(first)
        return first

    def vision_encode(self, px, return_embeds=False):
        self.calls.append("vision")

    def prefill(self, ids, mode, rows, all_logits=False, last_logits=True, left_pad=None, pos_from_mask=True):
        self.calls.append("prefill")
        self.session += 1
        first = self._start((ids[:, -1] % V).to(torch.int32))
        ll = torch.zeros(ids.shape[0], V) if last_logits else None
        if ll is not None:
            ll[torch.arange(ids.shape[0]), first.long()] = 5.0
        return ll, first, None

    def extend(self, ids, all_logits=False, last_logits=True):
        self.calls.append("extend")
        self.session += 1
        return None, self._start((ids[:, -1] % V).to(torch.int32)), None

    def truncate(self, lengths):
        self.truncated = list(lengths)

    def decode_step(self, tok_in, tok_out, logits=None, use_graph=True):
        self.decode_steps += 1
        nxt = self._pick(tok_in)
        if logits is not None:
            logits.zero_()
            logits[torch.arange(nxt.shape[0]), nxt.long()] = 5.0
        tok_out.copy_(nxt)
        self._choose(nxt)

    def decode_many(self, tok, n):
        for _ in range(n):
            self.decode_step(tok, tok)

    def read_history(self, B, n):
        return torch.stack(self.hist[:n], 0)

    # ---- device sampler -----------------------------------------------------------------------
    def sampler_supported(self):
        return True

    def set_sampler(self, spec):
        self.spec = spec
        self.calls.append("set_sampler" if spec is not None else "unset_sampler")

    def read_finished(self, B):
        return self.finished[:B].to(torch.int32)

    # ---- the ring -------------------------------------------------------------------------------
    def stream_supported(self):
        return True

    def stream_arm(self, on):
        self.calls.append("arm" if on else "disarm")
        self.armed = bool(on)
        if on:
            self.ring = []

    def stream_wait(self, target, timeout_us=-1):
        if len(self.ring) < target:
            raise N.NativeError(f"vcla_stream_wait: step {target} will never be published")
        return len(self.ring)

    def stream_read(self, lo, hi, B):
        return torch.stack(self.ring[lo:hi], 0)[:, :B] if hi > lo else torch.empty(0, B, dtype=torch.int32)


class NoRingEngine(RingEngine):
    stream_supported = None

    def __getattribute__(self, name):
        if name == "stream_supported":
            raise AttributeError(name)
        return super().__getattribute__(name)


def make_model(engine=None):
    m = object.__new__(VisualCLAModel)
    m._engine = engine if engine is not None else RingEngine()
    m._tok_buf = {}
    m.image_at_head = False
    m.tokenizer = types.SimpleNamespace(img_start_token_id=40, img_end_token_id=41, img_token_id=42)
    return m


class Recorder:
    """streamer + Stream-criterion recording in one event list (the golden's format)."""

    def __init__(self):
        self.events = []

    def put(self, value):
        self.events.append(dict(kind="put", shape=list(value.shape), dtype=str(value.dtype), device=str(value.device),
                                values=value.reshape(-1).tolist()))

    def end(self):
        self.events.append(dict(kind="end"))

    def criterion(self, stop_after=None):
        rec = self

        class RecStream(Stream):
            def __call__(self, input_ids, scores):
                rec.events.append(dict(kind="criterion", length=int(input_ids.shape[-1]), batch=int(input_ids.shape[0])))
                return stop_after is not None and input_ids.shape[-1] >= stop_after
        return RecStream()


def chain(first, n):
    out = [int(first)]
    for _ in range(n - 1):
        out.append((out[-1] * 7 + 3) % V)
    return out


IDS = torch.tensor([[1, 5, 9], [1, 6, 11]])


def test_which_calls_stream_on_the_device(monkeypatch):
    def armed(engine=None, **kw):
        m = make_model(engine)
        m.generate(input_ids=IDS[:1], max_new_tokens=6, pad_token_id=0, **kw)
        return "arm" in m._engine.calls

    assert armed(do_sample=False, eos_token_id=None, streamer=Recorder())                        # argmax graphs
    assert armed(do_sample=False, eos_token_id=7, streamer=Recorder())                           # device sampler
    assert armed(do_sample=True, top_k=5, eos_token_id=None, stopping_criteria=[Stream(lambda ids: None)])
    assert not armed(do_sample=False, eos_token_id=None)                                         # nothing to stream
    assert not armed(do_sample=False, eos_token_id=None, stopping_criteria=[lambda i, s: False])  # arbitrary criteria: host loop
    assert not armed(do_sample=False, eos_token_id=None, streamer=Recorder(), stopping_criteria=[Stream(), lambda i, s: False])
    assert not armed(do_sample=True, top_k=5, tfs=0.9, eos_token_id=None, streamer=Recorder())   # host-only sampler knob
    assert not armed(NoRingEngine(), do_sample=False, eos_token_id=None, streamer=Recorder())    # engine without a ring
    monkeypatch.setenv("VCLA_HOST_SAMPLER", "1")
    assert not armed(do_sample=True, top_k=5, eos_token_id=None, streamer=Recorder())
    with pytest.raises(NotImplementedError):
        make_model().generate(input_ids=IDS[:1], num_beams=2, do_sample=False, max_new_tokens=4, streamer=Recorder())


@pytest.mark.parametrize("device", [True, False])
def test_put_before_criteria_and_one_end(device):
    rec = Recorder()
    m = make_model(RingEngine() if device else NoRingEngine())
    out = m.generate(input_ids=IDS, do_sample=False, max_new_tokens=5, eos_token_id=None, pad_token_id=0, streamer=rec,
                     stopping_criteria=[rec.criterion()])
    ev = rec.events
    assert ev[0] == dict(kind="put", shape=[2, 0], dtype="torch.int64", device="cpu", values=[])
    assert [e["kind"] for e in ev[1:]] == ["put", "criterion"] * 5 + ["end"]
    puts = [e for e in ev[1:] if e["kind"] == "put"]
    assert all(p["shape"] == [2] and p["dtype"] == "torch.int64" and p["device"] == "cpu" for p in puts)
    assert torch.equal(torch.tensor([p["values"] for p in puts]).t(), out.cpu())
    assert [e["length"] for e in ev if e["kind"] == "criterion"] == [1, 2, 3, 4, 5]
    assert out[0].tolist() == chain(9, 5) and out[1].tolist() == chain(11, 5)
    assert ("arm" in m._engine.calls) == device and (not device or m._engine.calls[-1] == "disarm")


def test_cut_at_eos_pads_the_finished_row():
    full = make_model().generate(input_ids=IDS, do_sample=False, max_new_tokens=20, eos_token_id=None, pad_token_id=0)
    for eos in (int(full[0, 2]), int(full[1, 10]), [int(full[0, 1]), int(full[1, 4])]):
        host = make_model(NoRingEngine()).generate(input_ids=IDS, do_sample=False, max_new_tokens=20, eos_token_id=eos, pad_token_id=49)
        rec = Recorder()
        m = make_model()
        dev = m.generate(input_ids=IDS, do_sample=False, max_new_tokens=20, eos_token_id=eos, pad_token_id=49, streamer=rec)
        assert "arm" in m._engine.calls and torch.equal(dev, host), (eos, dev.tolist(), host.tolist())
        puts = [e["values"] for e in rec.events[1:] if e["kind"] == "put"]
        assert torch.equal(torch.tensor(puts).t(), dev) and rec.events[-1]["kind"] == "end"


@pytest.mark.parametrize("k", [1, 2, 5, 7, 8, 9, 13, 16, 17, 30])
def test_consumer_stop_cuts_and_bounds_the_steps_run_past_it(k):
    rec = Recorder()
    m = make_model()
    out = m.generate(input_ids=IDS, do_sample=True, top_k=5, max_new_tokens=40, eos_token_id=None, pad_token_id=0, streamer=rec,
                     stopping_criteria=[rec.criterion(stop_after=k)])
    assert out.shape == (2, k)
    assert [e["length"] for e in rec.events if e["kind"] == "criterion"] == list(range(1, k + 1))
    steps_run = 1 + m._engine.decode_steps
    assert 0 <= steps_run - k <= 9, (k, steps_run)
    assert m._engine.calls[-2:] == ["disarm", "unset_sampler"]


def test_launch_ahead_keeps_a_chunk_queued():
    """Each further graph is enqueued when the second-to-last step of the running one is published, before its callbacks."""
    seen = []
    m = make_model()

    def cb(ids):
        seen.append((int(ids.shape[-1]), 1 + m._engine.decode_steps))
    m.generate(input_ids=IDS[:1], do_sample=False, max_new_tokens=30, eos_token_id=None, pad_token_id=0,
               stopping_criteria=[Stream(cb)])
    for n_seen, launched in seen:
        assert launched >= min(30, n_seen + 2) or launched == 30, (n_seen, launched)
    assert seen[-1] == (30, 30)


def test_cache_handle_records_the_fed_tokens_up_to_the_cut():
    m = make_model()
    stop = Stream(lambda ids: (_ for _ in ()).throw(StopIteration) if ids.shape[-1] >= 4 else None)
    out = m.generate(input_ids=IDS[:1], do_sample=False, max_new_tokens=30, eos_token_id=None, pad_token_id=0,
                     stopping_criteria=[stop], return_dict_in_generate=True)
    assert out.sequences.shape == (1, 4)
    cache = out.past_key_values
    assert isinstance(cache, VclaKVCache)
    assert cache.ids.tolist() == IDS[0].tolist() + out.sequences[0, :3].tolist()
    assert m._engine.decode_steps > 3                            # steps past the cut ran, but lie beyond the handle
    # the next turn keeps the common prefix and truncates what the cut dropped
    nxt = torch.cat([IDS[:1], out.sequences[:, :3].cpu(), torch.tensor([[7, 8]])], 1)
    m.generate(input_ids=nxt, do_sample=False, max_new_tokens=3, eos_token_id=None, pad_token_id=0, past_key_values=cache,
               streamer=Recorder())
    assert m._engine.truncated == [len(cache)] and m._engine.calls.count("extend") == 1


@pytest.mark.parametrize("kw", [dict(do_sample=True, top_k=5, tfs=0.9), dict(do_sample=False, output_logits=True, return_dict_in_generate=True),
                                dict(do_sample=True, top_k=5, top_a=0.5), dict(do_sample=False, logits_processor=[lambda i, s: s])])
def test_streamer_on_the_host_loop(kw):
    rec = Recorder()
    m = make_model()
    out = m.generate(input_ids=IDS, max_new_tokens=6, eos_token_id=None, pad_token_id=0, streamer=rec, **kw)
    seq = out.sequences if hasattr(out, "sequences") else out
    assert "arm" not in m._engine.calls
    assert rec.events[0]["shape"] == [2, 0] and rec.events[-1] == dict(kind="end")
    puts = [e["values"] for e in rec.events[1:-1]]
    assert torch.equal(torch.tensor(puts).t(), seq.cpu())


def _golden_cases():
    z = np.load(GOLDEN)
    return z, json.loads(str(z["cases"]))


@pytest.mark.parametrize("device", [True, False])
@pytest.mark.parametrize("name", ["b1", "b1_eos", "b2_padded_eos"])
def test_streamer_protocol_matches_the_reference(name, device):
    z, cases = _golden_cases()
    case = next(c for c in cases if c["name"] == name)
    seqs = torch.from_numpy(z[f"{name}_sequences"])
    rec = Recorder()
    m = make_model((RingEngine if device else NoRingEngine)(script=seqs))
    m.image_at_head = case["image_at_head"]
    ids = torch.from_numpy(z[f"{name}_input_ids"])
    out = m.generate(input_ids=ids, attention_mask=torch.from_numpy(z[f"{name}_attention_mask"]), do_sample=False,
                     max_new_tokens=case["max_new_tokens"], eos_token_id=case["eos"] or None, pad_token_id=case["pad_token_id"],
                     streamer=rec, stopping_criteria=[rec.criterion()])
    assert ("arm" in m._engine.calls) == device
    assert rec.events == case["events"]
    assert torch.equal(out.cpu(), seqs)
