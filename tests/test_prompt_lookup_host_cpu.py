"""Host side of prompt lookup decoding (generate(prompt_lookup_num_tokens=k[, max_matching_ngram_size=n])) on the CPU, with a fake
engine that emulates the verification steps of include/vcla.h (drafts by the rule of oracle/prompt_lookup_oracle.py, a step emits the
leading matching picks plus one, stopping after an EOS id and at max_new).  Covers which calls take the path and that every other call
makes exactly the engine calls it makes without the option, the k clamp, the result / EOS cut / cache handle against the call without
the option, and the draft rule against HF's PromptLookupCandidateGenerator."""
import types

import pytest
import torch

from prompt_lookup_oracle import draft
from visualcla.engine import Engine
from visualcla.modeling_visualcla import VisualCLAModel

V, NQ = 50, 4


class LookupEngine:
    """Deterministic toy model: next token = (7 * previous + 3) % V, or the cyclic script[step % len]; the device sampler's EOS
    semantics (a finished row emits pad).  With a lookup set, decode_many runs verification steps as the device does."""
    device = torch.device("cpu")
    vocab, nq, max_batch, max_seq, max_prefill_tokens = V, NQ, 4, 64, 1024
    sampler_spec = staticmethod(Engine.sampler_spec)

    def __init__(self, script=None):
        self.script = script
        self.armed = False
        self.ring = []
        self.session = 0
        self.spec = None
        self.lookup = None
        self.calls = []
        self.steps = self.drafted = self.accepted = 0

    def _pick(self, prev):
        step = len(self.hist)
        if self.script is not None:
            nxt = torch.full_like(prev, self.script[step % len(self.script)])
        else:
            nxt = ((prev.long() * 7 + 3) % V).to(torch.int32)
        s = self.spec
        if s is not None and s.n_eos:
            eos = torch.tensor(list(s.eos_token_id)[: s.n_eos])
            nxt = torch.where(self.finished, torch.full_like(nxt, s.pad_token_id), nxt)
            self.finished |= torch.isin(nxt.long(), eos)
        return nxt

    def _start(self, ids):
        self.hist = []
        self.finished = torch.zeros(ids.shape[0], dtype=torch.bool)
        first = self._pick((ids[:, -1] % V).to(torch.int32))
        self._emit(first)
        return first

    def _emit(self, t):
        self.hist.append(t.clone())
        if self.armed:
            self.ring.append(t.clone())

    def vision_encode(self, px, return_embeds=False):
        self.calls.append("vision")

    def prefill(self, ids, mode, rows, all_logits=False, last_logits=True, left_pad=None, pos_from_mask=True):
        self.calls.append("prefill")
        self.session += 1
        first = self._start(ids)
        return (torch.zeros(ids.shape[0], V) if last_logits else None), first, None

    def extend(self, ids, all_logits=False, last_logits=True):
        self.calls.append("extend")
        self.session += 1
        return None, self._start(ids), None

    def truncate(self, lengths):
        self.calls.append(("truncate", list(lengths)))

    def decode_step(self, tok_in, tok_out, logits=None, use_graph=True):
        nxt = self._pick(tok_in)
        if logits is not None:
            logits.zero_()
            logits[torch.arange(nxt.shape[0]), nxt.long()] = 5.0
        tok_out.copy_(nxt)
        self._emit(nxt)

    def _verify(self):
        prompt, k, n, max_new = self.lookup
        produced = len(self.hist)
        if produced >= max_new or bool(self.finished[0]):
            return
        text = prompt + [int(t) for t in self.hist]
        d = draft(text, k, n, max_new - produced - 1)
        a = 0
        cnt = 0
        fin = False
        while True:
            t = self._pick(self.hist[-1])
            self._emit(t)
            cnt += 1
            fin = bool(self.finished[0])
            if fin or len(self.hist) >= max_new or a >= len(d) or int(t[0]) != d[a]:
                break
            a += 1
        self.steps += 1
        self.drafted += len(d)
        self.accepted += cnt - 1

    def decode_many(self, tok, n):
        self.calls.append(("decode_many", n))
        for _ in range(n):
            if self.lookup is not None:
                self._verify()
            else:
                self.decode_step(tok, tok)

    def read_history(self, B, n):
        return torch.stack(self.hist[:n], 0)

    def set_lookup(self, prompt_ids, k=0, n=2, max_new=0):
        self.calls.append(("set_lookup", k, n, max_new) if prompt_ids is not None else "unset_lookup")
        self.lookup = None if prompt_ids is None else ([int(t) for t in prompt_ids], k, n, max_new)
        if prompt_ids is not None:
            self.steps = self.drafted = self.accepted = 0

    def lookup_stats(self):
        return len(self.hist), bool(self.finished[0]), self.steps, self.drafted, self.accepted, self.lookup[1] + 1 if self.lookup else 0

    def sampler_supported(self):
        return True

    def set_sampler(self, spec):
        self.spec = spec
        self.calls.append("set_sampler" if spec is not None else "unset_sampler")

    def read_finished(self, B):
        return self.finished[:B].to(torch.int32)

    # ---- the token ring (work is synchronous: everything enqueued is published and every event has run) -------------------------
    def stream_supported(self):
        return True

    def stream_arm(self, on):
        self.calls.append("arm" if on else "disarm")
        self.armed = bool(on)
        if on:
            self.ring = []

    def stream_wait(self, target, timeout_us=-1):
        if len(self.ring) < target:
            raise RuntimeError(f"step {target} will never be published")
        return len(self.ring)

    def stream_read(self, lo, hi, B):
        return torch.stack(self.ring[lo:hi], 0)[:, :B]

    def record_event(self):
        return types.SimpleNamespace(query=lambda: True, synchronize=lambda: None)


def make_model(engine=None):
    m = object.__new__(VisualCLAModel)
    m._engine = engine if engine is not None else LookupEngine()
    m._tok_buf = {}
    m.image_at_head = False
    m.tokenizer = types.SimpleNamespace(img_start_token_id=40, img_end_token_id=41, img_token_id=42)
    return m


IDS = torch.tensor([[1, 5, 9, 12, 3], [1, 6, 11, 2, 8]])
CYCLE = [4, 8, 15, 16, 23, 42]


def _run(kw, ids=IDS[:1], engine=None):
    torch.manual_seed(0)
    m = make_model(engine)
    out = m.generate(input_ids=ids, pad_token_id=0, **kw)
    return out, m._engine.calls


def _lookup_set(calls):
    return [c for c in calls if isinstance(c, tuple) and c[0] == "set_lookup"]


@pytest.mark.parametrize("kw", [dict(do_sample=False, eos_token_id=None),                   # argmax graphs
                                dict(do_sample=False, eos_token_id=7),                      # device sampler, greedy + EOS
                                dict(do_sample=True, top_k=5, eos_token_id=None),           # device sampler, sampling
                                dict(do_sample=False, repetition_penalty=1.2, no_repeat_ngram_size=3, eos_token_id=None)])
def test_device_calls_take_the_path(kw):
    out, calls = _run(dict(kw, max_new_tokens=12, prompt_lookup_num_tokens=3), engine=LookupEngine(CYCLE))
    assert _lookup_set(calls) == [("set_lookup", 3, 2, 12)]
    assert calls[-1] in ("unset_lookup", "unset_sampler")
    ref, _ = _run(dict(kw, max_new_tokens=12), engine=LookupEngine(CYCLE))
    assert torch.equal(out, ref)


def test_max_matching_ngram_size_is_passed():
    _, calls = _run(dict(do_sample=False, eos_token_id=None, max_new_tokens=8, prompt_lookup_num_tokens=4, max_matching_ngram_size=3))
    assert _lookup_set(calls) == [("set_lookup", 4, 3, 8)]


@pytest.mark.parametrize("case", ["batch", "host_sampler_env", "host_only_knob", "logits", "criteria", "capacity", "max_new_1", "k0"])
def test_other_calls_ignore_the_option(case, monkeypatch):
    kw = dict(do_sample=False, eos_token_id=None, max_new_tokens=10)
    ids = IDS[:1]
    if case == "batch":
        ids = IDS
    elif case == "host_sampler_env":
        monkeypatch.setenv("VCLA_HOST_SAMPLER", "1")
        kw.update(eos_token_id=7)
    elif case == "host_only_knob":
        kw.update(do_sample=True, top_k=5, tfs=0.9)
    elif case == "logits":
        kw.update(output_logits=True, return_dict_in_generate=True)
    elif case == "criteria":
        kw.update(stopping_criteria=[lambda i, s: False])
    elif case == "capacity":
        kw.update(max_new_tokens=LookupEngine.max_seq - ids.shape[1] - 2)     # + k = 3 exceeds max_seq
    elif case == "max_new_1":
        kw.update(max_new_tokens=1)
    with_k = dict(kw, prompt_lookup_num_tokens=0 if case == "k0" else 3)
    out, calls = _run(with_k, ids=ids)
    ref, ref_calls = _run(kw, ids=ids)
    assert calls == ref_calls and not _lookup_set(calls)
    if isinstance(out, torch.Tensor):
        assert torch.equal(out, ref)
    else:
        assert torch.equal(out.sequences, ref.sequences)


def test_beam_calls_ignore_the_option(monkeypatch):
    seen = []
    monkeypatch.setattr(VisualCLAModel, "_generate_beams", lambda self, gc, *a: seen.append(gc.prompt_lookup_num_tokens) or "beams")
    m = make_model()
    assert m.generate(input_ids=IDS[:1], num_beams=2, max_new_tokens=4, prompt_lookup_num_tokens=3) == "beams"
    assert seen == [3]


class Rec:
    """streamer + Stream-criterion recording in one event list"""

    def __init__(self):
        self.events = []

    def put(self, v):
        self.events.append(("put", tuple(v.shape), v.dtype, str(v.device), v.reshape(-1).tolist()))

    def end(self):
        self.events.append(("end",))

    def criterion(self, stop_after=None):
        from visualcla.modeling_utils import Stream
        rec = self

        class RecStream(Stream):
            def __call__(self, input_ids, scores):
                rec.events.append(("criterion", int(input_ids.shape[-1])))
                return stop_after is not None and input_ids.shape[-1] >= stop_after
        return RecStream()


@pytest.mark.parametrize("kw", [dict(do_sample=False, eos_token_id=None), dict(do_sample=False, eos_token_id=23),
                                dict(do_sample=True, top_k=5, eos_token_id=None)])
def test_streamed_calls_take_the_path_and_keep_the_put_protocol(kw):
    for max_new in (5, 13, 30):
        for stop_after in (None, 7):
            rec = Rec()
            crit = [rec.criterion(stop_after)]
            base = dict(kw, max_new_tokens=max_new, streamer=rec, stopping_criteria=crit)
            out, calls = _run(dict(base, prompt_lookup_num_tokens=5), engine=LookupEngine(CYCLE))
            assert _lookup_set(calls) == [("set_lookup", 5, 2, max_new)] and "arm" in calls
            ref_rec = Rec()
            ref, _ = _run(dict(kw, max_new_tokens=max_new, streamer=ref_rec, stopping_criteria=[ref_rec.criterion(stop_after)]),
                          engine=LookupEngine(CYCLE))
            if stop_after is None:
                assert torch.equal(out, ref), (kw, max_new, stop_after)
            else:
                # a stopping criterion sees whole puts (HF _assisted_decoding): the row ends at the end of the put it stopped on, so
                # it extends the one-token stream's row and is a prefix of the unstopped row
                full, _ = _run(dict(kw, max_new_tokens=max_new), engine=LookupEngine(CYCLE))
                assert out.shape[1] >= ref.shape[1] and torch.equal(out[:, : ref.shape[1]], ref)
                assert torch.equal(full[:, : out.shape[1]], out)
            ev = rec.events
            assert ev[0][:2] == ("put", (1, 0)) and ev[-1] == ("end",)
            puts = [e for e in ev[1:] if e[0] == "put"]
            assert all(p[1][0] == 1 and p[1][1] >= 1 and p[2] == torch.int64 and p[3] == "cpu" for p in puts)
            assert sum((p[4] for p in puts), []) == out[0].tolist()            # the puts concatenate to the returned row
            # the criteria run once per put, on everything put so far
            crit_ev = [e for e in ev if e[0] == "criterion"]
            assert len(crit_ev) == len(puts)
            lengths = [sum(len(p[4]) for p in puts[: i + 1]) for i in range(len(puts))]
            assert [c[1] for c in crit_ev] == lengths
            assert len(puts) < len(out[0]) or len(out[0]) <= 2                 # accepted drafts arrive several per put


def test_streamed_calls_on_the_host_path_ignore_the_option():
    rec, ref_rec = Rec(), Rec()
    kw = dict(do_sample=False, eos_token_id=None, max_new_tokens=6)
    out, calls = _run(dict(kw, prompt_lookup_num_tokens=3, streamer=rec, stopping_criteria=[lambda i, s: False]))
    ref, ref_calls = _run(dict(kw, streamer=ref_rec, stopping_criteria=[lambda i, s: False]))
    assert calls == ref_calls and torch.equal(out, ref) and not _lookup_set(calls)


def test_k_is_clamped_to_15():
    _, calls = _run(dict(do_sample=False, eos_token_id=None, max_new_tokens=20, prompt_lookup_num_tokens=40))
    assert _lookup_set(calls) == [("set_lookup", 15, 2, 20)]
    # the capacity check uses the clamped k: S + max_new + 15 == max_seq still runs
    _, calls = _run(dict(do_sample=False, eos_token_id=None, max_new_tokens=LookupEngine.max_seq - 5 - 15, prompt_lookup_num_tokens=40))
    assert _lookup_set(calls)


@pytest.mark.parametrize("k", [1, 2, 7, 15])
@pytest.mark.parametrize("n", [1, 2, 3])
def test_result_eos_cut_and_cache_handle_match_plain(k, n):
    for script, kw in ((CYCLE, dict(do_sample=False, eos_token_id=None)),
                       (CYCLE, dict(do_sample=False, eos_token_id=23)),                # EOS inside an accepted run
                       (CYCLE, dict(do_sample=False, eos_token_id=23, min_new_tokens=2)),
                       (None, dict(do_sample=False, eos_token_id=None))):              # nothing to copy: one token per step
        for max_new in (5, 13, 24):
            base = dict(kw, max_new_tokens=max_new, return_dict_in_generate=True)
            out, _ = _run(dict(base, prompt_lookup_num_tokens=k, max_matching_ngram_size=n), engine=LookupEngine(script))
            ref, _ = _run(base, engine=LookupEngine(script))
            assert torch.equal(out.sequences, ref.sequences), (script, kw, max_new)
            assert out.past_key_values.ids.tolist() == ref.past_key_values.ids.tolist()[: len(out.past_key_values.ids)]
            assert len(out.past_key_values.ids) == IDS.shape[1] + out.sequences.shape[1] - 1


def test_cycle_is_verified_in_fewer_steps():
    e = LookupEngine(CYCLE)
    m = make_model(e)
    m.generate(input_ids=IDS[:1], do_sample=False, eos_token_id=None, pad_token_id=0, max_new_tokens=40, prompt_lookup_num_tokens=7)
    steps, accepted = e.steps, e.accepted
    assert accepted > 0 and steps < 39


# ---- the draft rule against HF's PromptLookupCandidateGenerator ---------------------------------------------------------------------
def _hf_draft(text, k, n):
    from transformers.generation.candidate_generator import PromptLookupCandidateGenerator
    # no EOS id in the text: HF would crop a draft at its first EOS (the device emits up to an EOS anyway, so drafts past it never count)
    g = PromptLookupCandidateGenerator(eos_token_id=torch.tensor([-1]), num_output_tokens=k, max_matching_ngram_size=n, max_length=10 ** 6)
    ids = torch.tensor([text], dtype=torch.long)
    cand = g.get_candidates(ids)[0]
    return cand[0, len(text):].tolist()


@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_draft_rule_matches_hf(n):
    gen = torch.Generator().manual_seed(n)
    for trial in range(200):
        length = int(torch.randint(1, 60, (1,), generator=gen))
        vocab = int(torch.randint(2, 12, (1,), generator=gen))       # small vocabularies: many matches, ties broken leftmost
        text = torch.randint(0, vocab, (length,), generator=gen).tolist()
        k = int(torch.randint(1, 16, (1,), generator=gen))
        assert draft(text, k, n) == _hf_draft(text, k, n), (text, k, n)


def test_draft_rule_edge_cases():
    assert draft([5, 6, 7], 3, 2) == [] == _hf_draft([5, 6, 7], 3, 2)                  # no match
    assert draft([9], 3, 2) == [] == _hf_draft([9], 3, 2)                               # nothing before the tail
    assert draft([1, 2, 3, 1, 2], 3, 2) == [3, 1, 2] == _hf_draft([1, 2, 3, 1, 2], 3, 2)
    assert draft([1, 2, 1, 2], 5, 2) == [1, 2] == _hf_draft([1, 2, 1, 2], 5, 2)          # the match runs to the very end
    assert draft([4, 1, 2, 3, 1, 2], 3, 2) == [3, 1, 2]                                 # leftmost of the longest n-gram
    assert draft([7, 3, 7, 1, 2, 7], 2, 2) == [3, 7] == _hf_draft([7, 3, 7, 1, 2, 7], 2, 2)   # falls back to g = 1, leftmost
    for room in range(0, 5):                                                             # max_new clamp
        assert draft([1, 2, 3, 4, 5, 1, 2], 4, 2, room) == [3, 4, 5, 1][:room]
