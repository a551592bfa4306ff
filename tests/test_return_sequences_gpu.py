"""generate(do_sample=True, num_return_sequences=N) on the device, at 7B widths with 8 LLaMA layers (every prefill GEMM of the LLaMA stack
then takes the 256-wide tile whatever its row count, so a B-row and a B*N-row prefill compute each row alike).

- every token of every forked row against the float64 restatement of the device sampler (oracle/sampler_oracle.py) on the device's own
  raw logits and history, with the draw counter (L, b * N + j), for an image batch under the reference's chat config, with EOS and
  min_new_tokens, and with int8 projections;
- the fork is exact: the first pick's logits are the unforked prefill's, and every decode step's raw logits, teacher-forced with the
  recorded tokens, are bit-equal to the expanded batch's (each prompt repeated N times, no fork) -- on text prompts, because the vision
  tower's 1024-wide GEMMs pick their tile width by row count;
- the pages right after the fork: siblings share every full prompt page and own distinct pages from the partly filled one on, pages in
  use = B x (full prompt pages) + B*N x (the rest), fewer than the expanded batch holds, and vcla_reset returns all of them;
- streaming: a streamed call returns the rows of the same call without a streamer, and the streamer gets (B*N,) puts."""
import os

import pytest
import torch

import visualcla_oracle as O
from test_sampler_draw_gpu import _check_every_token
from test_sampler_gpu import DrawStats
from visualcla import _native as N

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(os.environ.get("VCLA_SKIP_7B") == "1", reason="VCLA_SKIP_7B=1")]
CFG = O.PathConfig(t_layers=8)
STEPS = 32
CHAT = dict(do_sample=True, repetition_penalty=1.1, no_repeat_ngram_size=15, temperature=0.5, top_k=40, top_p=0.9)   # DEFAULT_GENERATION_CONFIG


def _make(load_in_8bit=False):
    import visualcla
    return visualcla.VisualCLAModel.from_synthetic(CFG.to_dict(), seed=0, max_batch=16, max_seq=192, load_in_8bit=load_in_8bit)


@pytest.fixture(scope="module")
def model():
    m = _make()
    yield m
    m._engine.close()


def _generate_spec(monkeypatch, m, **kw):
    """generate(**kw) on the device, recording the sampler spec it builds -> (tokens, spec)"""
    from visualcla.engine import Engine
    built = []
    make = Engine.sampler_spec

    def spy(*a, **k):
        built.append(make(*a, **k))
        return built[-1]
    monkeypatch.setattr(Engine, "sampler_spec", staticmethod(spy))
    out = m.generate(**kw)
    monkeypatch.setattr(Engine, "sampler_spec", staticmethod(make))
    assert len(built) == 1, "generate() ran on the device sampler"
    return out.cpu(), built[0]


def _prefill(m, ids, px, n, last_logits=True):
    """vcla_prefill of the B prompts, forked to n rows each when n > 1 -> (last logits (B, V), first picks (B * n,))"""
    eng = m._engine
    mode, rows = m._image_layout(ids, px)
    if px is not None:
        eng.vision_encode(px)
    eng.set_fanout(n)
    try:
        ll, first, _ = eng.prefill(ids, mode, rows, last_logits=last_logits)
    finally:
        eng.set_fanout(1)
    return ll, first


def _eager_fork(m, ids, px, spec, n, steps=STEPS):
    """The forked prefill, then one decode_step per token with the logits buffer, the sampler set -> (raw logits (R, steps, V) with the
    prompts' last logits repeated for step 0, tokens (R, steps), finished (R,)), on the host."""
    eng = m._engine
    R = ids.shape[0] * n
    eng.set_sampler(spec)
    try:
        ll, first = _prefill(m, ids, px, n)
        tok = first.clone()
        lg = torch.empty(R, eng.vocab, dtype=torch.float32, device=eng.device)
        logits, toks = [ll.repeat_interleave(n, 0).cpu()], [first.cpu()]
        for _ in range(1, steps):
            eng.decode_step(tok, tok, lg)
            logits.append(lg.cpu())
            toks.append(tok.cpu())
        fin = eng.read_finished(R).cpu()
    finally:
        eng.set_sampler(None)
    return torch.stack(logits, 1), torch.stack(toks, 1).long(), fin


def _siblings_differ(toks, n):
    for b in range(toks.shape[0] // n):
        rows = {tuple(r) for r in toks[b * n:(b + 1) * n].tolist()}
        assert len(rows) == n, f"prompt {b}: its {n} replies are not all different"


def test_image_chat_default_every_token(monkeypatch, model):
    """3 prompts with an image x N = 4 under DEFAULT_GENERATION_CONFIG: generate() (graph replays) returns the eager loop's 12 rows in the
    order b * 4 + j, every token is the reference draw with counter (L, b * 4 + j), and the siblings are different replies."""
    from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG
    px, ids = O.make_inputs(CFG, 3, 16, seed=21)
    ids, px = ids.cuda(), px.cuda()
    torch.manual_seed(4)
    out, spec = _generate_spec(monkeypatch, model, input_ids=ids, pixel_values=px, generation_config=DEFAULT_GENERATION_CONFIG,
                               num_return_sequences=4, max_new_tokens=STEPS, eos_token_id=None, pad_token_id=0)
    assert out.shape == (12, STEPS) and out.dtype == torch.int64
    logits, toks, _ = _eager_fork(model, ids, px, spec, 4)
    stats = DrawStats()
    _check_every_token(logits, toks, spec, stats, "N=4, B=3 image, chat default")
    print(f"[return sequences, B=3 x N=4 image, chat default] {stats.line()}")
    assert torch.equal(out, toks), f"graph replays {out.tolist()} vs eager steps {toks.tolist()}"
    _siblings_differ(toks, 4)


def test_eos_min_new_tokens_every_token(monkeypatch, model):
    """An EOS id row 0 draws at a step >= 5 (new to the row, outside its kept set while min_new_tokens masks it), so row 0 repeats the
    run without EOS up to it and finishes there: every row pads after its EOS, read_finished reports exactly the rows that emitted one,
    every token before is the reference draw, and generate() returns the eager rows cut where the last row finished."""
    px, ids = O.make_inputs(CFG, 3, 16, seed=23)
    ids, px = ids.cuda(), px.cuda()
    min_new, pad = 4, 7
    torch.manual_seed(9)
    out0, spec0 = _generate_spec(monkeypatch, model, input_ids=ids, pixel_values=px, num_return_sequences=4, max_new_tokens=STEPS,
                                 eos_token_id=None, pad_token_id=pad, **CHAT)
    logits0, toks0, fin0 = _eager_fork(model, ids, px, spec0, 4)
    assert torch.equal(out0, toks0) and not bool(fin0.any())
    from sampler_oracle import processed_scores
    kept0 = [processed_scores(logits0[0, L].numpy(), toks0[0, :L].numpy(), spec0)[1] for L in range(min_new)]
    s0 = next(s for s in range(5, STEPS) if int(toks0[0, s]) not in toks0[0, :s].tolist()
              and all(kept0[L][int(toks0[0, s])] == float("-inf") for L in range(min_new)))
    eos = int(toks0[0, s0])
    torch.manual_seed(9)                                   # the same Philox key
    out, spec = _generate_spec(monkeypatch, model, input_ids=ids, pixel_values=px, num_return_sequences=4, max_new_tokens=STEPS,
                               eos_token_id=eos, pad_token_id=pad, min_new_tokens=min_new, **CHAT)
    assert spec.seed == spec0.seed
    logits, toks, fin = _eager_fork(model, ids, px, spec, 4)
    assert torch.equal(toks[0, :s0 + 1], toks0[0, :s0 + 1]), "row 0 repeats the first run up to its EOS"
    assert toks[0, s0 + 1:].eq(pad).all(), "row 0 pads after its EOS"
    stats = DrawStats()
    finished = _check_every_token(logits, toks, spec, stats, "N=4 EOS + min_new_tokens")
    assert fin.tolist() == [int(x) for x in finished] and finished[0], (fin.tolist(), finished)
    from visualcla.modeling_visualcla import VisualCLAModel
    assert torch.equal(out, VisualCLAModel._cut_at_eos(toks, [eos])), "generate() rows vs the eager rows cut at the last EOS"
    print(f"[return sequences, EOS at step {s0}, {sum(finished)} of 12 rows finished] {stats.line()}")


def test_fork_is_exact_and_shares_pages(model):
    """Text prompts of 150 tokens (two full 64-token pages and a partly filled one), B = 2 x N = 4."""
    eng = model._engine
    n, B, T, steps = 4, 2, 150, 16
    R = B * n
    _, ids = O.make_inputs(CFG, B, T, seed=31)
    ids = ids.cuda()
    pps, total, pt = eng.kv_geometry()
    full = T // pt
    spec = eng.sampler_spec(seed=(3 << 33) + 5, pad_token_id=0, **CHAT)
    eng.set_sampler(spec)
    try:
        ll_fork, first = _prefill(model, ids, None, n)
        # ---- pages right after the fork
        table, owned, free, exhausted = eng.kv_pages()
        assert not exhausted
        rest = eng_pages_for(T + 1, pt) - full
        assert owned[:R].tolist() == [full + rest] * R and owned[R:].eq(0).all()
        for b in range(B):
            sib = table[b * n:(b + 1) * n]
            assert (sib[:, :full] == sib[0, :full]).all(), f"prompt {b}: siblings share its full pages"
        assert len(set(table[:R, :full].reshape(-1).tolist())) == B * full, "prompts do not share pages"
        own = table[:R, full:full + rest].reshape(-1).tolist()
        assert len(set(own)) == R * rest, "every row owns its pages from the partly filled one on"
        assert not set(own) & set(table[:R, :full].reshape(-1).tolist())
        used_fork = total - free
        assert used_fork == B * full + R * rest, (used_fork, B, full, R, rest)
        # ---- the forked rows decode; raw logits and tokens recorded
        tok = first.clone()
        lg = torch.empty(R, eng.vocab, dtype=torch.float32, device=eng.device)
        logits, toks = [], [first.cpu()]
        for _ in range(1, steps):
            eng.decode_step(tok, tok, lg)
            logits.append(lg.cpu())
            toks.append(tok.cpu())
        toks = torch.stack(toks, 1)
    finally:
        eng.set_sampler(None)
    _siblings_differ(toks, n)
    # ---- the first pick's logits are those of the unforked B-row prefill
    ll_plain, _ = _prefill(model, ids, None, 1)
    assert torch.equal(ll_fork, ll_plain), "forked vs unforked prefill: last logits differ"
    # ---- the expanded batch (each prompt n times, no fork), teacher-forced with the recorded tokens
    ll_exp, _ = _prefill(model, ids.repeat_interleave(n, 0), None, 1)
    assert torch.equal(ll_exp, ll_plain.repeat_interleave(n, 0)), "expanded batch: prefill last logits differ"
    _, owned_x, free_x, _ = eng.kv_pages()
    used_exp = total - free_x
    assert used_exp == R * (full + rest) and used_fork < used_exp
    t_in = torch.zeros(R, dtype=torch.int32, device=eng.device)
    t_out = torch.zeros(R, dtype=torch.int32, device=eng.device)
    for s in range(1, steps):
        t_in.copy_(toks[:, s - 1])
        eng.decode_step(t_in, t_out, lg)
        assert torch.equal(lg.cpu(), logits[s - 1]), f"step {s}: raw logits of the forked rows differ from the expanded batch's"
    print(f"[return sequences, fork B={B} x N={n}, prompt {T}] pages in use {used_fork} forked vs {used_exp} expanded; "
          f"{steps - 1} teacher-forced steps bit-equal")
    # ---- vcla_reset returns every page
    eng.reset()
    _, owned_r, free_r, _ = eng.kv_pages()
    assert free_r == total and owned_r.eq(0).all()


def eng_pages_for(tokens, pt):
    return (tokens + pt - 1) // pt


def test_streamed_equals_plain(model):
    """N = 3, two text prompts, the chat knobs: a streamed call returns the rows of the call without a streamer under the same seed, and
    its streamer gets an empty (6, 0) put, then one (6,) int64 put per step, then end()."""
    _, ids = O.make_inputs(CFG, 2, 20, seed=41)
    ids = ids.cuda()
    puts = []

    class Streamer:
        def put(self, v):
            puts.append((tuple(v.shape), v.dtype))

        def end(self):
            puts.append("end")

    kw = dict(input_ids=ids, num_return_sequences=3, max_new_tokens=24, eos_token_id=None, pad_token_id=0, **CHAT)
    torch.manual_seed(12)
    plain = model.generate(**kw).cpu()
    torch.manual_seed(12)
    streamed = model.generate(streamer=Streamer(), **kw).cpu()
    assert plain.shape == (6, 24)
    assert torch.equal(streamed, plain)
    assert puts == [((6, 0), torch.int64)] + [((6,), torch.int64)] * 24 + ["end"]
    _siblings_differ(plain, 3)


def test_refusals(model):
    """The fan-out mode's refusals on the engine: more rows than min(max_batch, 64), beam mode, an extend of forked rows."""
    eng = model._engine
    _, ids = O.make_inputs(CFG, 5, 12, seed=51)
    with pytest.raises(N.NativeError, match="exceed 16 rows"):
        _prefill(model, ids.cuda(), None, 4)
    eng.set_beam(eng.beam_spec(2, 4))
    try:
        with pytest.raises(N.NativeError, match="beam search"):
            _prefill(model, ids[:2].cuda(), None, 2)
    finally:
        eng.set_beam(None)
    _prefill(model, ids[:2].cuda(), None, 2)
    with pytest.raises(N.NativeError, match="forked rows"):
        eng.extend(ids[:4, :3].cuda())
    with pytest.raises(N.NativeError, match="1..64"):
        eng.set_fanout(65)


def test_int8_every_token(monkeypatch, model):
    """load_in_8bit: 2 prompts with an image x N = 3, every token against the reference draw on the device's raw logits."""
    m8 = _make(load_in_8bit=True)
    try:
        px, ids = O.make_inputs(CFG, 2, 16, seed=61)
        ids, px = ids.cuda(), px.cuda()
        torch.manual_seed(6)
        out, spec = _generate_spec(monkeypatch, m8, input_ids=ids, pixel_values=px, num_return_sequences=3, max_new_tokens=24,
                                   eos_token_id=None, pad_token_id=0, **CHAT)
        logits, toks, _ = _eager_fork(m8, ids, px, spec, 3, steps=24)
        stats = DrawStats()
        _check_every_token(logits, toks, spec, stats, "int8, N=3, B=2 image")
        print(f"[return sequences, int8, B=2 x N=3 image] {stats.line()}")
        assert torch.equal(out, toks)
        _siblings_differ(toks, 3)
    finally:
        m8._engine.close()
