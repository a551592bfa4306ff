"""Sampled decoding end to end, every token against the float64 restatement of the device sampler (oracle/sampler_oracle.py).

An eager loop -- prefill with the last logits, then one decode_step per token with the logits buffer -- yields each step's raw logits
and the token the fused sampler drew from them; the token at step L of row b must be predict(raw logits, the row's first L tokens, spec,
L, b): transformers' processors, then the Philox4x32-10 inverse-CDF draw.  The loop feeds the device's own tokens back, so every step is
comparable.  generate()'s graph replays must give the eager loop's tokens for the spec generate() built, and the raw logits of the
sampler path must be bit-equal to the greedy path's fed the same tokens (dec_logits_reduce vs stage 1 of dec_logits_argmax)."""
import pytest
import torch

import sampler_oracle as SO
import visualcla_oracle as O
from test_sampler_gpu import DrawStats

pytestmark = pytest.mark.gpu
STEPS = 48
CFG = O.tiny_config()
CHAT = dict(do_sample=True, repetition_penalty=1.1, no_repeat_ngram_size=15, temperature=0.5, top_k=40, top_p=0.9)   # DEFAULT_GENERATION_CONFIG


def _model(max_batch):
    import visualcla
    return visualcla.VisualCLAModel.from_synthetic(CFG.to_dict(), seed=3, max_batch=max_batch, max_seq=128)


@pytest.fixture(scope="module")
def image_b3():
    m = _model(3)
    px, ids = O.make_inputs(CFG, 3, 12, seed=5)
    yield m, ids.cuda(), px.cuda()
    m._engine.close()


def _eager(m, ids, px, spec, steps=STEPS):
    """Prefill + one decode_step per token with the sampler set -> (raw logits (B, steps, V), tokens (B, steps), finished (B,)), on the host."""
    eng = m._engine
    B = ids.shape[0]
    mode, rows = m._image_layout(ids, px)
    if px is not None:
        eng.vision_encode(px)
    eng.set_sampler(spec)
    try:
        ll, first, _ = eng.prefill(ids, mode, rows, last_logits=True)
        tok = first.clone()
        lg = torch.empty(B, eng.vocab, dtype=torch.float32, device=eng.device)
        logits, toks = [ll.clone()], [first.clone()]
        for _ in range(1, steps):
            eng.decode_step(tok, tok, lg)
            logits.append(lg.clone())
            toks.append(tok.clone())
        fin = eng.read_finished(B).cpu()
    finally:
        eng.set_sampler(None)
    return torch.stack(logits, 1).cpu(), torch.stack(toks, 1).cpu().long(), fin


def _check_every_token(logits, toks, spec, stats, what):
    """predict() at every step of every row; a row that emitted an EOS id must emit pad_token_id from then on.  -> rows that finished."""
    f = SO.spec_fields(spec)
    B, n, _ = logits.shape
    finished = [False] * B
    for b in range(B):
        for L in range(n):
            t = int(toks[b, L])
            if finished[b]:
                assert t == int(spec.pad_token_id), f"{what}: row {b} step {L} after its EOS: {t}, not the pad id"
                continue
            p = SO.predict(logits[b, L].numpy(), toks[b, :L].numpy(), spec, L, b)
            stats.add(t, p.token, p.ambiguous, p.accept, p.rank, p.margin, f"{what}: row {b} step {L}")
            finished[b] = t in f["eos"]
    return finished


def _greedy_logits_equal(m, ids, px, toks, logits, what):
    """The sampler off, the same tokens fed: the raw logits of every step are bit-equal to the sampled run's."""
    eng = m._engine
    B, n = toks.shape
    mode, rows = m._image_layout(ids, px)
    if px is not None:
        eng.vision_encode(px)
    ll, _, _ = eng.prefill(ids, mode, rows, last_logits=True)
    assert torch.equal(ll.cpu(), logits[:, 0]), f"{what}: prefill logits"
    t_in = torch.zeros(B, dtype=torch.int32, device=eng.device)
    t_out = torch.zeros(B, dtype=torch.int32, device=eng.device)
    lg = torch.empty(B, eng.vocab, dtype=torch.float32, device=eng.device)
    for s in range(1, n):
        t_in.copy_(toks[:, s - 1])
        eng.decode_step(t_in, t_out, lg)
        assert torch.equal(lg.cpu(), logits[:, s]), f"{what}: step {s} logits differ from the greedy path's"


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


def test_chat_default_with_image_every_token(monkeypatch, image_b3):
    """B = 3, image at the head, the reference's DEFAULT_GENERATION_CONFIG: generate() (graph replays of up to 16 steps) equals the eager
    loop under the spec it built, every token equals the reference draw, and the raw logits equal the greedy path's."""
    from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG
    m, ids, px = image_b3
    torch.manual_seed(4)
    out, spec = _generate_spec(monkeypatch, m, input_ids=ids, pixel_values=px, generation_config=DEFAULT_GENERATION_CONFIG,
                               max_new_tokens=STEPS, eos_token_id=None, pad_token_id=0)
    f = SO.spec_fields(spec)
    assert f["do_sample"] and (f["top_k"], f["no_repeat_ngram_size"]) == (40, 15) and f["temperature"] == 0.5
    logits, toks, _ = _eager(m, ids, px, spec)
    stats = DrawStats()
    _check_every_token(logits, toks, spec, stats, "chat default, B=3, image")
    print(f"[sampled decoding, B=3 image, chat default] {stats.line()}")
    assert torch.equal(out, toks), f"graph replays {out.tolist()} vs eager steps {toks.tolist()}"
    _greedy_logits_equal(m, ids, px, toks, logits, "B=3 image")


def test_eos_min_new_tokens_every_token(image_b3):
    """An EOS id that occurs: row 0's draw at the first step >= 5 whose token is new to the row and lay outside the row's kept set while
    min_new_tokens masked it.  With that EOS id row 0 repeats its tokens up to that step and finishes there; every row pads after its
    EOS, read_finished reports exactly the rows that emitted one, and every token before equals the reference draw."""
    m, ids, px = image_b3
    eng = m._engine
    min_new, pad = 4, 7
    spec0 = eng.sampler_spec(seed=(5 << 40) + 11, pad_token_id=pad, **CHAT)
    logits0, toks0, fin0 = _eager(m, ids, px, spec0)
    assert not bool(fin0.any())
    kept0 = [SO.processed_scores(logits0[0, L].numpy(), toks0[0, :L].numpy(), spec0)[1] for L in range(min_new)]
    s0 = next(s for s in range(5, STEPS) if int(toks0[0, s]) not in toks0[0, :s].tolist()
              and all(kept0[L][int(toks0[0, s])] == float("-inf") for L in range(min_new)))
    eos = int(toks0[0, s0])
    spec = eng.sampler_spec(seed=spec0.seed, pad_token_id=pad, min_new_tokens=min_new, eos_token_id=[eos], **CHAT)
    logits, toks, fin = _eager(m, ids, px, spec)
    assert torch.equal(toks[0, :s0 + 1], toks0[0, :s0 + 1]), "row 0 repeats the first run up to its EOS"
    assert toks[0, s0 + 1:].eq(pad).all(), "row 0 pads after its EOS"
    stats = DrawStats()
    finished = _check_every_token(logits, toks, spec, stats, "EOS + min_new_tokens")
    assert fin.tolist() == [int(x) for x in finished] and finished[0], (fin.tolist(), finished)
    print(f"[sampled decoding, EOS at step {s0}] {stats.line()}")


def test_text_b40_every_token(monkeypatch):
    """B = 40, text only: the 33..64-row decode schedule (dec_logits_reduce, then the sampler at sequence counters >= 32)."""
    m = _model(40)
    _, ids = O.make_inputs(CFG, 40, 10, seed=6)
    ids = ids.cuda()
    torch.manual_seed(8)
    knobs = dict(do_sample=True, temperature=0.8, top_k=50, top_p=0.9, repetition_penalty=1.5, no_repeat_ngram_size=3)
    out, spec = _generate_spec(monkeypatch, m, input_ids=ids, max_new_tokens=STEPS, eos_token_id=None, pad_token_id=0, **knobs)
    logits, toks, _ = _eager(m, ids, None, spec)
    stats = DrawStats()
    _check_every_token(logits, toks, spec, stats, "B=40 text")
    print(f"[sampled decoding, B=40 text] {stats.line()}")
    assert stats.ambiguous <= 0.05 * stats.n and stats.above_top >= 0.25 * stats.n, stats.line()
    assert torch.equal(out, toks), "graph replays vs eager steps"
    _greedy_logits_equal(m, ids, None, toks, logits, "B=40 text")
    m._engine.close()
