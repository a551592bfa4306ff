"""What every native decode step enqueues, against tests/golden/decode_schedule.json.  Each case starts from a fresh prefill and runs
eager steps, graph captures and replays of one decode mode -- argmax, the device sampler, beam search, prompt lookup verification
steps, extend then decode, the data-parallel token exchange on a one-rank communicator, mode flips on one token buffer and more
token buffers than the graph cache holds -- at batches on both sides of every schedule choice, in bf16 and int8 at tiny widths and
in bf16 at 7B widths.

Recorded per case:
  - structural fields, compared on any H100: the kernel launches of the prefill, of each eager step, capture and replay, and the
    kernel tag sequence of one eager step and one graph replay (trace buffer order: the order in which each kernel's CTA 0 entered;
    left out for data parallel, whose exchange runs on a side stream);
  - device-dependent fields, compared only on the device the golden was recorded on (name and SM count): the tokens, the SHA-256
    of the logits' bytes and the prompt lookup statistics.  Split counts, and with them the fp32 summation order and lookup's rows
    per step, follow the SM count.

    python tests/test_decode_schedule_gpu.py --record     rewrites the golden on the current device"""
import hashlib
import json
import os
import sys

import pytest
import torch

if __name__ == "__main__":
    _root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [os.path.join(_root, "visual-chinese-llama-alpaca_b200"), os.path.join(_root, "oracle")]

import visualcla_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decode_schedule.json")
TINY = dict(v_layers=1, r_layers=1, t_hidden=256, t_heads=2, t_ffn=448, t_layers=2, t_vocab=1003)
CONTEXTS = {
    "tiny_bf16": dict(cfg=O.PathConfig(**TINY), load_in_8bit=False),
    "tiny_int8": dict(cfg=O.PathConfig(**TINY), load_in_8bit=True),
    "7b_bf16": dict(cfg=O.PathConfig(v_layers=1, r_layers=1, t_layers=2), load_in_8bit=False),
}
MAX_BATCH, MAX_SEQ, PROMPT = 64, 128, 12
EOS = 7


def _cases():
    out = {}
    for ctx in ("tiny_bf16", "tiny_int8"):
        for mode in ("argmax", "sampler"):
            for B in (1, 4, 16, 17, 32, 33, 64):
                for armed in ((0, 1) if B in (1, 4) else (0,)):
                    out[f"{ctx}/plain/{mode}/B{B}" + ("/armed" if armed else "")] = dict(ctx=ctx, kind="plain", mode=mode, B=B, armed=armed)
            for k in (1, 7, 15):
                for armed in (0, 1):
                    out[f"{ctx}/lookup/{mode}/k{k}" + ("/armed" if armed else "")] = dict(ctx=ctx, kind="lookup", mode=mode, k=k, armed=armed)
            for B in (8, 40):
                out[f"{ctx}/dp/{mode}/B{B}"] = dict(ctx=ctx, kind="dp", mode=mode, B=B)
        for B in (4, 16, 32, 64):
            out[f"{ctx}/beam/B{B}"] = dict(ctx=ctx, kind="beam", B=B)
        out[f"{ctx}/extend/B4"] = dict(ctx=ctx, kind="extend", B=4)
        out[f"{ctx}/mode_flips/B4"] = dict(ctx=ctx, kind="flips", B=4)
        out[f"{ctx}/eviction/B1"] = dict(ctx=ctx, kind="eviction", B=1)
    for B in (16, 32, 64):
        out[f"7b_bf16/plain/argmax/B{B}"] = dict(ctx="7b_bf16", kind="plain", mode="argmax", B=B, armed=0)
    return out


CASES = _cases()
_ENGINES = {}


def _engine(ctx):
    if ctx not in _ENGINES:
        for other in list(_ENGINES):
            _ENGINES.pop(other).close()          # one context at a time
        torch.cuda.empty_cache()
        import visualcla
        spec = CONTEXTS[ctx]
        m = visualcla.VisualCLAModel.from_synthetic(spec["cfg"].to_dict(), seed=0, max_batch=MAX_BATCH, max_seq=MAX_SEQ,
                                                    load_in_8bit=spec["load_in_8bit"])
        _ENGINES[ctx] = m._engine
    return _ENGINES[ctx]


def _sampler():
    from visualcla.engine import Engine
    return Engine.sampler_spec(do_sample=True, temperature=0.8, top_k=50, min_new_tokens=3, eos_token_id=[EOS], pad_token_id=0, seed=1234)


def _prompt(eng, B, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(10, eng.vocab - 10, (B, PROMPT), generator=g)


def _sha(t):
    torch.cuda.synchronize()
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


class _Rec:
    """Collects one case's structural and device-dependent fields."""

    def __init__(self, eng, trace):
        self.eng, self.trace, self.struct, self.dev = eng, trace, {}, {}

    def launches(self, name, fn):
        self.eng.kernel_launches(reset=True)
        fn()
        torch.cuda.synchronize()
        self.struct[f"launches/{name}"] = self.eng.kernel_launches(reset=True)

    def traced(self, name, fn):
        if not self.trace:
            return self.launches(name, fn)
        self.eng.trace_enable(4096)
        try:
            self.launches(name, fn)
            self.struct[f"tags/{name}"] = [ev[0] for ev in self.eng.trace_read(4096)]
        finally:
            self.eng.trace_enable(0)

    def result(self):
        return {"struct": self.struct, "device": self.dev}


def _prefill(rec, ids, **kw):
    out = {}
    rec.launches("prefill", lambda: out.update(zip(("ll", "tok", "la"), rec.eng.prefill(ids, 0, None, **kw))))
    if out["ll"] is not None:
        rec.dev["prefill_logits"] = _sha(out["ll"])
    return out["tok"]


def _steps(rec, B, tok):
    """One eager step with logits, one graph step with logits (its capture), one traced replay, then decode_many(tok, 8)."""
    eng = rec.eng
    logits = torch.empty(B, eng.vocab, dtype=torch.float32, device=eng.device)
    rec.traced("eager", lambda: eng.decode_step(tok, tok, logits, use_graph=False))
    rec.dev["eager_logits"] = _sha(logits)
    rec.launches("capture", lambda: eng.decode_step(tok, tok, logits, use_graph=True))
    rec.dev["capture_logits"] = _sha(logits)
    rec.traced("replay", lambda: eng.decode_step(tok, tok, logits, use_graph=True))
    rec.dev["replay_logits"] = _sha(logits)
    rec.launches("decode_many8", lambda: eng.decode_many(tok, 8))
    return 1 + 3 + 8          # history rows: the prefill's (or extend's) pick and 11 steps


def _history(rec, B, rows):
    rec.dev["tokens"] = rec.eng.read_history(B, rows).cpu().tolist()


def _disarm(eng, armed):
    torch.cuda.synchronize()
    if armed:
        eng.stream_arm(False)


def _case_plain(rec, c, seed):
    eng, B = rec.eng, c["B"]
    if c["mode"] == "sampler":
        eng.set_sampler(_sampler())
    if c["armed"]:
        eng.stream_arm(True)
    try:
        tok = torch.zeros(B, dtype=torch.int32, device=eng.device)
        tok.copy_(_prefill(rec, _prompt(eng, B, seed)))
        _history(rec, B, _steps(rec, B, tok))
        if c["armed"]:
            rec.dev["published"] = eng.stream_wait(0, 0)
    finally:
        _disarm(eng, c["armed"])
        eng.set_sampler(None)


def _case_beam(rec, c, seed):
    from visualcla.engine import Engine
    eng, B, K = rec.eng, c["B"], 4
    eng.set_beam(Engine.beam_spec(K, 10, length_penalty=0.7, eos_token_id=[EOS]))
    try:
        first = _prefill(rec, _prompt(eng, B // K, seed))
        tok = torch.zeros(B, dtype=torch.int32, device=eng.device)
        tok.copy_(first)
        logits = torch.empty(B, eng.vocab, dtype=torch.float32, device=eng.device)
        rec.traced("eager", lambda: eng.decode_step(tok, tok, logits, use_graph=False))
        rec.dev["eager_logits"] = _sha(logits)
        rec.launches("capture", lambda: eng.decode_step(tok, tok, logits, use_graph=True))
        rec.dev["capture_logits"] = _sha(logits)
        rec.traced("replay", lambda: eng.decode_step(tok, tok, logits, use_graph=True))
        rec.dev["replay_logits"] = _sha(logits)
        rec.launches("decode_many4", lambda: eng.decode_many(tok, 4))
        _history(rec, B, 8)
        toks, lens, scores, done = eng.read_beams(B // K)
        rec.dev["beams"] = [toks.tolist(), lens.tolist(), [hashlib.sha256(scores.numpy().tobytes()).hexdigest()], done.tolist()]
    finally:
        torch.cuda.synchronize()
        eng.set_beam(None)


def _case_lookup(rec, c, seed):
    eng = rec.eng
    if c["mode"] == "sampler":
        eng.set_sampler(_sampler())
    if c["armed"]:
        eng.stream_arm(True)
    try:
        base = _prompt(eng, 1, seed)[:, :4]
        ids = base.repeat(1, PROMPT // 4)                 # a repeating prompt, so that some steps verify drafts
        tok = torch.zeros(1, dtype=torch.int32, device=eng.device)
        tok.copy_(_prefill(rec, ids))
        eng.set_lookup(ids, k=c["k"], n=2, max_new=40)
        try:
            eng.decode_step(tok, tok, None, use_graph=False)
            rec.struct["decode_step_refusal"] = None
        except Exception as e:                            # noqa: BLE001 -- the refusal's message is part of the record
            rec.struct["decode_step_refusal"] = str(e)
        rec.launches("prime_capture4", lambda: eng.decode_many(tok, 4))
        rec.traced("replay4", lambda: eng.decode_many(tok, 4))
        rec.launches("capture8", lambda: eng.decode_many(tok, 8))
        stats = eng.lookup_stats()
        rec.dev["lookup_stats"] = list(stats)
        _history(rec, 1, stats[0])
        if c["armed"]:
            rec.dev["published"] = eng.stream_wait(0, 0)
    finally:
        _disarm(eng, c["armed"])
        eng.set_lookup(None)
        eng.set_sampler(None)


def _case_extend(rec, c, seed):
    eng, B = rec.eng, c["B"]
    tok = torch.zeros(B, dtype=torch.int32, device=eng.device)
    _prefill(rec, _prompt(eng, B, seed))
    out = {}
    rec.launches("extend", lambda: out.update(zip(("ll", "tok", "la"), eng.extend(_prompt(eng, B, seed + 1)[:, :5]))))
    rec.dev["extend_logits"] = _sha(out["ll"])
    tok.copy_(out["tok"])
    _history(rec, B, _steps(rec, B, tok))


def _dp_on(eng):
    """A one-rank communicator on this context (once), then the exchange switched on."""
    if not getattr(eng, "_schedule_test_comm", False):
        from visualcla import _native as N
        uid = torch.zeros(128, dtype=torch.uint8)
        if eng.lib.vcla_nccl_unique_id(N.ptr(uid)) != 0 or eng.lib.vcla_nccl_init(eng._ctx, N.ptr(uid), 0, 1, 64) != 0:
            pytest.skip(f"NCCL cannot create a one-rank communicator here: {eng.lib.vcla_last_error().decode()}")
        eng._schedule_test_comm = True
    eng.dp_set_active(True)


def _case_dp(rec, c, seed):
    from visualcla import _native as N
    eng, B = rec.eng, c["B"]
    _dp_on(eng)
    if c["mode"] == "sampler":
        eng.set_sampler(_sampler())
    try:
        tok = torch.zeros(B, dtype=torch.int32, device=eng.device)
        tok.copy_(_prefill(rec, _prompt(eng, B, seed)))
        logits = torch.empty(B, eng.vocab, dtype=torch.float32, device=eng.device)
        for i in range(2):
            rec.launches(f"eager{i}", lambda: eng.decode_step(tok, tok, logits, use_graph=False))
            rec.dev[f"eager{i}_logits"] = _sha(logits)
        for name in ("capture", "replay"):
            rec.launches(name, lambda: eng.decode_step(tok, tok, logits, use_graph=True))
            rec.dev[f"{name}_logits"] = _sha(logits)
        rec.launches("decode_many8", lambda: eng.decode_many(tok, 8))
        _history(rec, B, 13)
        hist = torch.zeros(13, 64, dtype=torch.int32, device=eng.device)
        N.check(eng.lib.vcla_read_history_dp(eng._ctx, N.ptr(hist), 13, eng._stream()), "vcla_read_history_dp")
        rec.dev["dp_history"] = hist[:, :B].cpu().tolist()
    finally:
        torch.cuda.synchronize()
        eng.set_sampler(None)
        eng.dp_set_active(False)


def _case_flips(rec, c, seed):
    """argmax graph, sampler graph, argmax graph on one token buffer: the graph key keeps the modes apart."""
    eng, B = rec.eng, c["B"]
    tok = torch.zeros(B, dtype=torch.int32, device=eng.device)
    tok.copy_(_prefill(rec, _prompt(eng, B, seed)))
    try:
        for i, mode in enumerate(("argmax", "sampler", "argmax")):
            eng.set_sampler(_sampler() if mode == "sampler" else None)
            rec.launches(f"{i}_{mode}_capture", lambda: eng.decode_step(tok, tok, None, use_graph=True))
            rec.traced(f"{i}_{mode}_replay", lambda: eng.decode_step(tok, tok, None, use_graph=True))
    finally:
        eng.set_sampler(None)
    _history(rec, B, 7)


def _case_eviction(rec, c, seed):
    """26 distinct token buffers through graphs in turn (more than the cache holds), then the first one again."""
    eng = rec.eng
    bufs = [torch.zeros(1, dtype=torch.int32, device=eng.device) for _ in range(26)]
    prev = _prefill(rec, _prompt(eng, 1, seed))
    for i, b in enumerate(bufs + bufs[:1]):
        b.copy_(prev)
        rec.launches(f"graph{i}", lambda: eng.decode_step(b, b, None, use_graph=True))
        prev = b
    _history(rec, 1, 28)


RUNNERS = dict(plain=_case_plain, beam=_case_beam, lookup=_case_lookup, extend=_case_extend, dp=_case_dp, flips=_case_flips,
               eviction=_case_eviction)


def run_case(name):
    c = CASES[name]
    eng = _engine(c["ctx"])
    rec = _Rec(eng, trace=c["kind"] != "dp")
    seed = int(hashlib.sha256(name.encode()).hexdigest()[:8], 16)
    RUNNERS[c["kind"]](rec, c, seed)
    torch.cuda.synchronize()
    return json.loads(json.dumps(rec.result()))


def _device():
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    return {"name": p.name, "sms": p.multi_processor_count}


def _dump(device, cases):
    lines = ["{", f'  "device": {json.dumps(device)},', '  "cases": {']
    for i, (name, rec) in enumerate(cases.items()):
        lines.append(f"    {json.dumps(name)}: {json.dumps(rec, sort_keys=True)}" + ("," if i + 1 < len(cases) else ""))
    lines += ["  }", "}"]
    return "\n".join(lines) + "\n"


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_golden_covers_every_case():
    assert sorted(_golden()["cases"]) == sorted(CASES)


@pytest.mark.parametrize("name", list(CASES))
def test_decode_schedule_matches_golden(name):
    golden = _golden()
    want = golden["cases"][name]
    got = run_case(name)
    assert got["struct"] == want["struct"]
    if golden["device"] == _device():
        assert got["device"] == want["device"]


if __name__ == "__main__":
    if sys.argv[1:] != ["--record"]:
        sys.exit(__doc__)
    recs = {}
    for name in CASES:
        try:
            recs[name] = run_case(name)
        except pytest.skip.Exception as e:
            sys.exit(f"{name}: {e}")
    with open(GOLDEN, "w") as f:
        f.write(_dump(_device(), recs))
    print(f"wrote {GOLDEN}: {len(CASES)} cases on {_device()}")
