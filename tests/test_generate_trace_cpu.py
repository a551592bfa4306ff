"""generate()'s exact engine traffic on the CPU, against tests/golden/generate_trace.json.  A recording fake engine (a toy model with
the device sampler's EOS semantics, prompt lookup verification steps, the token ring and the beam surface) logs every call generate()
makes -- prefill / extend / truncate shapes, decode_step and decode_many counts and token buffers, sampler / lookup / beam specs,
arm / disarm, stream waits and the finished / lookup / beam-done polls -- interleaved with what a streamer and the stopping criteria
observe.  Each case also stores the returned tokens, the cache handle's ids, or the refusal's type and message.  The golden pins the
dispatch between the host loop and the device drivers, the launch pattern and the put protocol, so host-side refactors of generate()
can be checked to change none of them.

    python tests/test_generate_trace_cpu.py --record     rewrites the golden from the current code"""
import json
import os
import sys
import types

import pytest
import torch

if __name__ == "__main__":
    _root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [os.path.join(_root, "visual-chinese-llama-alpaca_b200"), os.path.join(_root, "oracle")]

from prompt_lookup_oracle import draft
from visualcla.engine import Engine
from visualcla.modeling_utils import Stream
from visualcla.modeling_visualcla import VisualCLAModel

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "generate_trace.json")
V, NQ = 50, 4
CYCLE = [4, 8, 15, 16, 23, 42]


def _spec_fields(spec):
    out = {}
    for name, _ in spec._fields_:
        v = getattr(spec, name)
        if name == "eos_token_id":
            v = list(v)[: spec.n_eos]
        elif isinstance(v, float):
            v = round(v, 6)
        out[name] = v
    return out


class _Event:
    def __init__(self, log, i):
        self.log, self.i = log, i

    def query(self):
        self.log.append(["event_query", self.i])
        return True

    def synchronize(self):
        self.log.append(["event_synchronize", self.i])


class TraceEngine:
    """Toy model: next token = (7 * previous + 3 + step) % V, or script[step % len(script)]; with a sampler spec a finished row emits pad.
    Work is synchronous: everything enqueued is published to the ring at once and every event has run."""
    device = torch.device("cpu")
    vocab, nq, max_batch, max_seq, max_prefill_tokens = V, NQ, 4, 64, 1024
    sampler_spec = staticmethod(Engine.sampler_spec)
    beam_spec = staticmethod(Engine.beam_spec)

    def __init__(self, log, script=None):
        self.log, self.script = log, script
        self.session = 0
        self.armed, self.ring = False, []
        self.spec = self.lookup = self.beam = None
        self.hist, self.finished = [], torch.zeros(0, dtype=torch.bool)
        self.bufs, self.tok_bufs, self.events = {}, {}, 0
        self.beam_polls = 0
        self.steps = self.drafted = self.accepted = 0

    def _buf(self, t):
        """the first-seen index of a token buffer: the same index means the same persistent buffer"""
        return self.bufs.setdefault(t.data_ptr(), len(self.bufs))

    # ---- token choice ----------------------------------------------------------------------------
    def _pick(self, prev):
        if self.script is not None:
            nxt = torch.full_like(prev, self.script[len(self.hist) % len(self.script)])
        else:
            nxt = ((prev.long() * 7 + 3 + len(self.hist)) % V).to(torch.int32)
        s = self.spec
        if s is not None and s.n_eos:
            nxt = torch.where(self.finished, torch.full_like(nxt, s.pad_token_id), nxt)
            self.finished |= torch.isin(nxt.long(), torch.tensor(list(s.eos_token_id)[: s.n_eos]))
        return nxt

    def _emit(self, t):
        self.hist.append(t.clone())
        if self.armed:
            self.ring.append(t.clone())

    def _start(self, ids):
        K = self.beam.num_beams if self.beam is not None else 1
        self.session += 1
        self.hist = []
        self.finished = torch.zeros(ids.shape[0] * K, dtype=torch.bool)
        self.beam_polls = 0
        self.last = ids[:, -1].clone()
        first = self._pick((ids[:, -1] % V).to(torch.int32).repeat_interleave(K))
        self._emit(first)
        return first

    def _logits(self, tok):
        lg = torch.zeros(tok.shape[0], V)
        lg[torch.arange(tok.shape[0]), tok.long()] = 5.0
        return lg

    # ---- prefill / decode --------------------------------------------------------------------------
    def vision_encode(self, px, return_embeds=False):
        self.log.append(["vision_encode", list(px.shape)])

    def prefill(self, ids, mode, rows, all_logits=False, last_logits=True, left_pad=None, pos_from_mask=True):
        self.log.append(["prefill", list(ids.shape), int(mode), None if rows is None else rows.tolist(), all_logits, last_logits,
                         None if left_pad is None else left_pad.tolist(), pos_from_mask])
        first = self._start(ids)
        return (self._logits(first) if last_logits else None), first, None

    def extend(self, ids, all_logits=False, last_logits=True):
        self.log.append(["extend", ids.tolist(), all_logits, last_logits])
        first = self._start(ids)
        return (self._logits(first) if last_logits else None), first, None

    def truncate(self, lengths):
        self.log.append(["truncate", list(lengths)])

    def decode_step(self, tok_in, tok_out, logits=None, use_graph=True):
        self.log.append(["decode_step", self._buf(tok_in), self._buf(tok_out), logits is not None])
        self._step(tok_in, tok_out, logits)

    def _step(self, tok_in, tok_out, logits=None):
        nxt = self._pick(tok_in)
        if logits is not None:
            logits.copy_(self._logits(nxt))
        tok_out.copy_(nxt)
        self._emit(nxt)

    def decode_many(self, tok, n):
        self.log.append(["decode_many", self._buf(tok), tok.numel(), n])
        self.session += 1
        for _ in range(n):
            if self.lookup is not None:
                self._verify()
            else:
                self._step(tok, tok)

    def read_history(self, B, n):
        self.log.append(["read_history", B, n])
        return torch.stack(self.hist[:n], 0)[:, :B]

    def token_buffer(self, n):
        self.log.append(["token_buffer", n])
        return self.tok_bufs.setdefault(n, torch.zeros(n, dtype=torch.int32))

    # ---- device sampler ----------------------------------------------------------------------------
    def sampler_supported(self):
        return True

    def set_sampler(self, spec):
        self.log.append(["set_sampler", None if spec is None else _spec_fields(spec)])
        self.spec = spec

    def read_finished(self, B):
        self.log.append(["read_finished", B])
        return self.finished[:B].to(torch.int32)

    # ---- prompt lookup -----------------------------------------------------------------------------
    def set_lookup(self, prompt_ids, k=0, n=2, max_new=0):
        self.log.append(["set_lookup", None] if prompt_ids is None else ["set_lookup", prompt_ids.tolist(), k, n, max_new])
        self.lookup = None if prompt_ids is None else ([int(t) for t in prompt_ids], k, n, max_new)

    def _verify(self):
        prompt, k, n, max_new = self.lookup
        if len(self.hist) >= max_new or bool(self.finished[0]):
            return
        d = draft(prompt + [int(t) for t in self.hist], k, n, max_new - len(self.hist) - 1)
        a = 0
        while True:
            t = self._pick(self.hist[-1])
            self._emit(t)
            if bool(self.finished[0]) or len(self.hist) >= max_new or a >= len(d) or int(t[0]) != d[a]:
                break
            a += 1
        self.steps += 1
        self.drafted += len(d)
        self.accepted += a

    def lookup_stats(self):
        self.log.append(["lookup_stats"])
        return len(self.hist), bool(self.finished[0]), self.steps, self.drafted, self.accepted, self.lookup[1] + 1

    def record_event(self):
        self.events += 1
        self.log.append(["record_event", self.events])
        return _Event(self.log, self.events)

    # ---- the ring ------------------------------------------------------------------------------------
    def stream_supported(self):
        return True

    def stream_arm(self, on):
        self.log.append(["stream_arm", bool(on)])
        self.armed = bool(on)
        if on:
            self.ring = []

    def stream_wait(self, target, timeout_us=-1):
        self.log.append(["stream_wait", target])
        if len(self.ring) < target:
            raise RuntimeError(f"step {target} will never be published")
        return len(self.ring)

    def stream_read(self, lo, hi, B):
        self.log.append(["stream_read", lo, hi, B])
        return torch.stack(self.ring[lo:hi], 0)[:, :B]

    # ---- beam search: item b's K hypotheses derive from its prompt's last id; every item is done at the second poll ---------
    def set_beam(self, spec):
        self.log.append(["set_beam", None if spec is None else _spec_fields(spec)])
        self.beam = spec

    def read_beam_done(self, n):
        self.log.append(["read_beam_done", n])
        self.beam_polls += 1
        return torch.full((n,), int(self.beam_polls >= 2), dtype=torch.int32)

    def read_beams(self, n):
        self.log.append(["read_beams", n])
        K, m = self.beam.num_beams, self.beam.max_new_tokens
        tok = torch.zeros(n, K, m, dtype=torch.int32)
        lens = torch.zeros(n, K, dtype=torch.int32)
        for b in range(n):
            for k in range(K):
                tok[b, k] = (int(self.last[b]) * 10 + k * 100 + torch.arange(m)) % 1000
                lens[b, k] = max(1, m - 3 * k)
        return tok, lens, torch.zeros(n, K), torch.ones(n, dtype=torch.int32)


class NoRingEngine(TraceEngine):
    def __getattribute__(self, name):
        if name == "stream_supported":
            raise AttributeError(name)
        return super().__getattribute__(name)


class Streamer:
    def __init__(self, log):
        self.log = log

    def put(self, v):
        self.log.append(["put", list(v.shape), str(v.dtype), str(v.device), v.reshape(-1).tolist()])

    def end(self):
        self.log.append(["end"])


def _criterion(log, stream, stop_at=None):
    def call(ids, scores):
        log.append(["criterion", list(ids.shape), ids.reshape(-1).tolist(), scores is None])
        return stop_at is not None and ids.shape[-1] >= stop_at
    if not stream:
        return call

    class RecStream(Stream):
        def __call__(self, ids, scores):
            return call(ids, scores)
    return RecStream()


def _tensor_criterion(log):
    """a criterion returning one flag per row (HF's StoppingCriteria since 4.39): stops once both rows passed 6 tokens"""
    def call(ids, scores):
        log.append(["criterion", list(ids.shape), None, scores is None])
        return torch.full((ids.shape[0],), ids.shape[-1] >= 6)
    return call


def _processor(log):
    def proc(ids, scores):
        log.append(["processor", list(ids.shape)])
        s = scores.clone()
        s[:, 3] += 1.0
        return s
    return proc


IDS = [[1, 5, 9, 12, 3], [1, 6, 11, 2, 8]]
IDS6 = [[1, 5 + i, 9, 12 - i, 3 + i] for i in range(6)]
GREEDY = dict(do_sample=False, eos_token_id=None, pad_token_id=0)
EOS_B2 = dict(do_sample=False, eos_token_id=[19, 7], pad_token_id=0)       # greedy: row 0 emits 19 at step 3, row 1 emits 7 at step 12
SAMPLE = dict(do_sample=True, top_k=5, eos_token_id=None, pad_token_id=0)

# name -> (engine kind, input rows, generate kwargs, extra); a kwarg value that is a string starting with "@" is built per run
CASES = {
    "greedy": ("ring", IDS, dict(GREEDY, max_new_tokens=10), {}),
    "greedy_eos": ("ring", IDS, dict(EOS_B2, max_new_tokens=24), {}),
    "greedy_eos_return_dict": ("ring", IDS[:1], dict(EOS_B2, max_new_tokens=24, return_dict_in_generate=True), {}),
    "penalties": ("ring", IDS, dict(GREEDY, max_new_tokens=9, repetition_penalty=1.2, no_repeat_ngram_size=3), {}),
    "sample_top_k": ("ring", IDS, dict(SAMPLE, max_new_tokens=9, temperature=0.7, top_p=0.9), {}),
    "sample_top_k_eos": ("ring", IDS, dict(SAMPLE, eos_token_id=[19, 7], min_new_tokens=2, max_new_tokens=20), {}),
    "host_tfs": ("ring", IDS, dict(SAMPLE, tfs=0.9, max_new_tokens=7), {}),
    "host_output_scores": ("ring", IDS, dict(GREEDY, output_scores=True, output_logits=True, return_dict_in_generate=True,
                                             max_new_tokens=5), {}),
    "host_processor_eos": ("ring", IDS, dict(EOS_B2, max_new_tokens=20, logits_processor="@processor"), {}),
    "host_criteria": ("ring", IDS, dict(GREEDY, max_new_tokens=9, stopping_criteria="@criteria"), {}),
    "host_tensor_criteria_eos": ("ring", IDS, dict(EOS_B2, max_new_tokens=20, stopping_criteria="@tensor_criteria"), {}),
    "host_streamer_eos": ("ring", IDS, dict(EOS_B2, max_new_tokens=20, streamer="@streamer", stopping_criteria="@criteria"), {}),
    "stream_criteria_only": ("ring", IDS, dict(GREEDY, max_new_tokens=20, stopping_criteria="@stream_criteria"), {}),
    "streamer": ("ring", IDS, dict(EOS_B2, max_new_tokens=20, streamer="@streamer"), {}),
    "streamer_sampled": ("ring", IDS[:1], dict(SAMPLE, max_new_tokens=11, streamer="@streamer"), {}),
    "streamer_early_stop": ("ring", IDS, dict(GREEDY, max_new_tokens=30, streamer="@streamer", stopping_criteria="@stream_stop_13"), {}),
    "streamer_max_new_1": ("ring", IDS[:1], dict(GREEDY, max_new_tokens=1, streamer="@streamer"), {}),
    "lookup": ("cycle", IDS[:1], dict(GREEDY, max_new_tokens=20, prompt_lookup_num_tokens=3), {}),
    "lookup_sampled": ("cycle", IDS[:1], dict(SAMPLE, max_new_tokens=20, prompt_lookup_num_tokens=4, max_matching_ngram_size=3), {}),
    "lookup_eos": ("cycle", IDS[:1], dict(GREEDY, eos_token_id=23, max_new_tokens=30, prompt_lookup_num_tokens=5,
                                          return_dict_in_generate=True), {}),
    "lookup_streamed": ("cycle", IDS[:1], dict(GREEDY, max_new_tokens=30, prompt_lookup_num_tokens=5, streamer="@streamer",
                                               stopping_criteria="@stream_criteria"), {}),
    "lookup_streamed_stop": ("cycle", IDS[:1], dict(GREEDY, eos_token_id=23, max_new_tokens=40, prompt_lookup_num_tokens=2,
                                                    stopping_criteria="@stream_stop_13"), {}),
    "lookup_b2": ("cycle", IDS, dict(GREEDY, max_new_tokens=12, prompt_lookup_num_tokens=3), {}),
    "lookup_over_capacity": ("cycle", IDS[:1], dict(GREEDY, max_new_tokens=57, prompt_lookup_num_tokens=3), {}),
    "lookup_max_new_1": ("cycle", IDS[:1], dict(GREEDY, eos_token_id=23, max_new_tokens=1, prompt_lookup_num_tokens=3), {}),
    "host_sampler_env_greedy": ("ring", IDS, dict(GREEDY, max_new_tokens=8, prompt_lookup_num_tokens=3), dict(host_sampler=True)),
    "host_sampler_env_eos": ("ring", IDS, dict(EOS_B2, max_new_tokens=20), dict(host_sampler=True)),
    "host_sampler_env_sampled": ("ring", IDS, dict(SAMPLE, max_new_tokens=6), dict(host_sampler=True)),
    "host_sampler_env_streamed": ("ring", IDS, dict(GREEDY, max_new_tokens=6, streamer="@streamer"), dict(host_sampler=True)),
    "kv_reuse": ("ring", IDS[:1], dict(GREEDY, max_new_tokens=6, return_dict_in_generate=True), dict(second_turn=True)),
    "kv_reuse_streamed": ("ring", IDS[:1], dict(EOS_B2, max_new_tokens=12, return_dict_in_generate=True, streamer="@streamer"),
                          dict(second_turn=True)),
    "image_placeholder": ("ring", [[1, 40, 42, 42, 42, 42, 41, 7]], dict(EOS_B2, max_new_tokens=6), dict(pixels=True)),
    "above_max_batch": ("ring", IDS6, dict(EOS_B2, max_new_tokens=16), {}),
    "above_max_batch_greedy": ("ring", IDS6, dict(GREEDY, max_new_tokens=5), {}),
    "beams_eos": ("ring", IDS, dict(num_beams=2, num_return_sequences=2, eos_token_id=40, pad_token_id=0, max_new_tokens=20,
                                    return_dict_in_generate=True), {}),
    "beams_chunked": ("ring", IDS6, dict(num_beams=2, eos_token_id=None, pad_token_id=0, max_new_tokens=5), {}),
    "no_ring_streamer": ("no_ring", IDS, dict(SAMPLE, max_new_tokens=6, streamer="@streamer"), {}),
    "no_ring_stream_criteria": ("no_ring", IDS, dict(GREEDY, max_new_tokens=6, stopping_criteria="@stream_stop_4"), {}),
    # refusals
    "refuse_capacity": ("ring", IDS, dict(GREEDY, max_new_tokens=60), {}),
    "refuse_prefix_fn": ("ring", IDS, dict(GREEDY, max_new_tokens=4, prefix_allowed_tokens_fn="@prefix_fn"), {}),
    "refuse_unknown_argument": ("ring", IDS, dict(GREEDY, max_new_tokens=4, foo_bar=3), {}),
    "refuse_stream_above_max_batch": ("ring", IDS6, dict(GREEDY, max_new_tokens=4, streamer="@streamer"), {}),
    "refuse_nrs_without_beams": ("ring", IDS, dict(GREEDY, max_new_tokens=4, num_return_sequences=2), {}),
    "refuse_beams_streamer": ("ring", IDS, dict(num_beams=2, max_new_tokens=4, streamer="@streamer"), {}),
    "refuse_beams_capacity": ("ring", IDS, dict(num_beams=2, max_new_tokens=60), {}),
}


def _build(v, log):
    if not (isinstance(v, str) and v.startswith("@")):
        return v
    v = v[1:]
    if v == "streamer":
        return Streamer(log)
    if v == "processor":
        return [_processor(log)]
    if v == "criteria":
        return [_criterion(log, stream=False)]
    if v == "tensor_criteria":
        return [_tensor_criterion(log)]
    if v == "stream_criteria":
        return [_criterion(log, stream=True)]
    if v.startswith("stream_stop_"):
        return [_criterion(log, stream=True, stop_at=int(v.rsplit("_", 1)[1]))]
    if v == "prefix_fn":
        return lambda b, ids: list(range(V))
    raise KeyError(v)


def _result(out):
    if isinstance(out, torch.Tensor):
        return dict(sequences=out.tolist())
    cache = out.past_key_values
    return dict(sequences=out.sequences.tolist(), cache_ids=None if cache.ids is None else cache.ids.tolist(), cache_len=len(cache),
                cache_mode=cache.mode, cache_pixels=cache.pixel_values is not None,
                logits=None if out.logits is None else [list(t.shape) for t in out.logits])


def run_case(name):
    kind, rows, kw, extra = CASES[name]
    log = []
    eng = {"ring": TraceEngine, "cycle": TraceEngine, "no_ring": NoRingEngine}[kind](log, CYCLE if kind == "cycle" else None)
    m = object.__new__(VisualCLAModel)
    m._engine, m._tok_buf = eng, {}
    m.image_at_head = False
    m.tokenizer = types.SimpleNamespace(img_start_token_id=40, img_end_token_id=41, img_token_id=42)
    ids = torch.tensor(rows)
    px = torch.zeros(ids.shape[0], 3, 4, 4) if extra.get("pixels") else None
    saved = os.environ.pop("VCLA_HOST_SAMPLER", None)
    if extra.get("host_sampler"):
        os.environ["VCLA_HOST_SAMPLER"] = "1"
    rec = dict(calls=log)
    try:
        torch.manual_seed(7)
        args = {k: _build(v, log) for k, v in kw.items()}
        try:
            out = m.generate(input_ids=ids, pixel_values=px, **args)
        except Exception as e:                                # a refusal: its type and message
            rec["error"] = [type(e).__name__, str(e)]
            return rec
        rec.update(_result(out))
        if extra.get("second_turn"):
            log.append(["second_turn"])
            nxt = torch.cat([ids, out.sequences[:, :2].cpu(), torch.tensor([[7, 8]])], 1)
            args = {k: _build(v, log) for k, v in kw.items()}
            rec["second"] = _result(m.generate(input_ids=nxt, pixel_values=px, past_key_values=out.past_key_values, **args))
    finally:
        os.environ.pop("VCLA_HOST_SAMPLER", None)
        if saved is not None:
            os.environ["VCLA_HOST_SAMPLER"] = saved
    return json.loads(json.dumps(rec))


def _dump(cases):
    lines = ["{"]
    for i, (name, rec) in enumerate(cases.items()):
        lines.append(f"  {json.dumps(name)}: {{")
        keys = list(rec)
        for j, k in enumerate(keys):
            end = "," if j + 1 < len(keys) else ""
            if k == "calls":
                lines.append('    "calls": [')
                lines += [f"      {json.dumps(c)}{',' if n + 1 < len(rec[k]) else ''}" for n, c in enumerate(rec[k])]
                lines.append(f"    ]{end}")
            else:
                lines.append(f"    {json.dumps(k)}: {json.dumps(rec[k])}{end}")
        lines.append("  }" + ("," if i + 1 < len(cases) else ""))
    lines.append("}")
    return "\n".join(lines) + "\n"


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_golden_covers_every_case():
    assert sorted(_golden()) == sorted(CASES)


@pytest.mark.parametrize("name", sorted(CASES))
def test_trace_matches_golden(name):
    assert run_case(name) == _golden()[name]


if __name__ == "__main__":
    if sys.argv[1:] != ["--record"]:
        sys.exit(__doc__)
    with open(GOLDEN, "w") as f:
        f.write(_dump({name: run_case(name) for name in CASES}))
    print(f"wrote {GOLDEN}: {len(CASES)} cases")
