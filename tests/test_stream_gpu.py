"""Token streaming on the device (include/vcla.h, token streaming): generate(streamer=...) and Stream criteria replay the same decode
graphs armed, so every step's tokens reach the host through the pinned ring as they are chosen.  Checks that streaming changes no
token and no kernel count, that chat_in_stream ends on chat()'s reply, the reference's streamer protocol (tests/golden/tiny_stream.npz),
a consumer that stops early (with the KV cache reused by the next turn), and that waiting for a step that never comes fails fast."""
import json
import os
import time
import types

import numpy as np
import pytest
import torch

import visualcla_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_stream.npz")
MID = O.PathConfig(v_layers=2, r_layers=2, t_hidden=1024, t_heads=8, t_ffn=2752, t_layers=3, t_vocab=5003)


def _model(cfg, max_batch=4, max_seq=192, seed=0):
    import visualcla
    return visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=seed, max_batch=max_batch, max_seq=max_seq)


class Recorder:
    def __init__(self):
        self.events = []

    def put(self, value):
        self.events.append(dict(kind="put", shape=list(value.shape), dtype=str(value.dtype), device=str(value.device),
                                values=value.reshape(-1).tolist()))

    def end(self):
        self.events.append(dict(kind="end"))

    def criterion(self, stop_after=None):
        from visualcla.modeling_utils import Stream
        rec = self

        class RecStream(Stream):
            def __call__(self, input_ids, scores):
                rec.events.append(dict(kind="criterion", length=int(input_ids.shape[-1]), batch=int(input_ids.shape[0])))
                return stop_after is not None and input_ids.shape[-1] >= stop_after
        return RecStream()

    def puts(self):
        return torch.tensor([e["values"] for e in self.events[1:] if e["kind"] == "put"], dtype=torch.int64).t()


def _modes(m, ids, px):
    """(name, generate kwargs): greedy without EOS (argmax graphs), greedy with an EOS the run emits, the chat default sampler."""
    from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG
    full = m.generate(input_ids=ids, pixel_values=px, do_sample=False, max_new_tokens=24, eos_token_id=None, pad_token_id=0)
    eos = int(full[0, 5])
    gc = DEFAULT_GENERATION_CONFIG.__class__(**{**DEFAULT_GENERATION_CONFIG.to_dict(), "max_new_tokens": 24, "pad_token_id": 0})
    return [("greedy", dict(do_sample=False, max_new_tokens=24, eos_token_id=None, pad_token_id=0)),
            ("greedy_eos", dict(do_sample=False, max_new_tokens=24, eos_token_id=eos, pad_token_id=0)),
            ("default_sampler", dict(generation_config=gc))]


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("width", ["tiny", "mid"])
def test_streamed_tokens_are_bit_identical(width, B):
    cfg = O.tiny_config() if width == "tiny" else MID
    m = _model(cfg)
    px, ids = O.make_inputs(cfg, B, 12, seed=77)
    px, ids = px.cuda(), ids.cuda()
    m.image_at_head = True
    eng = m._engine
    for name, kw in _modes(m, ids, px):
        torch.manual_seed(1234)
        plain = m.generate(input_ids=ids, pixel_values=px, **kw)
        torch.manual_seed(1234)
        rec = Recorder()
        calls = []
        orig = eng.stream_arm
        eng.stream_arm = lambda on: (calls.append(on), orig(on))[1]
        try:
            streamed = m.generate(input_ids=ids, pixel_values=px, streamer=rec, **kw)
        finally:
            eng.stream_arm = orig
        assert calls == [True, False], (name, calls)                  # it ran on the device, armed
        assert torch.equal(streamed, plain), (width, B, name, streamed.tolist(), plain.tolist())
        assert torch.equal(rec.puts(), streamed.cpu()), name           # the streamer received exactly the rows of the result
        assert rec.events[0]["shape"] == [B, 0] and rec.events[-1] == dict(kind="end")


def test_chat_in_stream_ends_on_chats_reply():
    import visualcla
    from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG
    cfg = O.tiny_config()
    m = _model(cfg, max_batch=1, max_seq=512)
    s0, s1, s2, s3 = O.special_ids(cfg)

    class Tok:
        bos_token, pad_token, bos_token_id, eos_token_id = "<s>", "<pad>", 1, 2
        img_start_token, img_end_token, img_token = "<img>", "</img>", "<img_token>"
        img_start_token_id, img_end_token_id, img_token_id = s0, s1, s3

        def __call__(self, text, return_tensors=None, add_special_tokens=None):
            from transformers import BatchEncoding
            special = {"<s>": 1, "<img>": s0, "</img>": s1, "<img_token>": s3}
            ids, i = [], 0
            while i < len(text):
                for k, v in special.items():
                    if text.startswith(k, i):
                        ids.append(v); i += len(k); break
                else:
                    ids.append(3 + (ord(text[i]) % 900)); i += 1
            t = torch.tensor([ids])
            return BatchEncoding({"input_ids": t, "attention_mask": torch.ones_like(t)})

        def decode(self, ids, skip_special_tokens=True):
            return " ".join(str(int(x)) for x in ids)

    m.tokenizer, m.image_at_head, m.num_patch = Tok(), False, cfg.r_queries
    px = torch.randn(1, 3, cfg.v_image, cfg.v_image, generator=torch.Generator().manual_seed(5))
    gc = DEFAULT_GENERATION_CONFIG.__class__(**{**DEFAULT_GENERATION_CONFIG.to_dict(), "max_new_tokens": 40})
    torch.manual_seed(99)
    resp, _ = visualcla.chat(m, image=px, text="describe", history=[], generation_config=gc)
    torch.manual_seed(99)
    chunks = list(visualcla.chat_in_stream(m, image=px, text="describe", history=[], generation_config=gc))
    assert len(chunks) == 40 and chunks[-1][0] == resp


def _decisive_ok(cfg, got, ids, px, at_head, pads, eos):
    """device tokens vs the fp32 oracle teacher-forced on them: equal wherever the oracle's top-1/top-2 margin is decisive
    (> 2x the logit tolerance), up to each row's EOS (the rule of tests/test_parity_gpu.py)."""
    w = O.make_weights(cfg, 0)
    n = got.shape[1]
    _, lg = O.generate_greedy(w, cfg, ids, px, n, image_at_head=at_head, forced_tokens=got, left_pad=pads)
    tol = 1.5e-2 * lg.abs().max().item()
    top2 = lg.topk(2, dim=-1)
    decisive = (top2.values[..., 0] - top2.values[..., 1]) > 2 * tol
    live = torch.ones_like(got, dtype=torch.bool)
    for b in range(got.shape[0]):
        row = got[b].tolist()
        for e in eos:
            if e in row:
                live[b, row.index(e) + 1:] = False
    return int((decisive & live & (got != top2.indices[..., 0])).sum()) == 0


@pytest.mark.parametrize("name", ["b1", "b1_eos", "b2_padded_eos"])
def test_reference_streamer_protocol_on_the_device(name):
    z = np.load(GOLDEN)
    case = next(c for c in json.loads(str(z["cases"])) if c["name"] == name)
    cfg = O.tiny_config()
    m = _model(cfg)
    s0, s1, _, s3 = O.special_ids(cfg)
    m.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
    m.image_at_head = case["image_at_head"]
    ids, mask, px = (torch.from_numpy(z[f"{name}_{k}"]) for k in ("input_ids", "attention_mask", "pixel_values"))
    rec = Recorder()
    out = m.generate(input_ids=ids.cuda(), pixel_values=px.cuda(), attention_mask=mask.cuda(), do_sample=False,
                     max_new_tokens=case["max_new_tokens"], eos_token_id=case["eos"] or None, pad_token_id=case["pad_token_id"],
                     streamer=rec, stopping_criteria=[rec.criterion()]).cpu()
    ref = case["events"]
    strip = lambda ev: [(e["kind"], e.get("shape"), e.get("dtype"), e.get("length")) for e in ev]   # noqa: E731
    assert strip(rec.events[:1]) == strip(ref[:1])                   # the first put: (B, 0) int64, before any token
    if torch.equal(out, torch.from_numpy(z[f"{name}_sequences"])):
        assert rec.events == ref
    else:                                                              # a non-decisive step may differ; the structure then
        assert [e["kind"] for e in rec.events] == [k for k, *_ in strip(rec.events)]
        pads = (mask == 0).sum(1).to(torch.int32) if bool((mask == 0).any()) else None
        assert _decisive_ok(cfg, out, ids, px, case["image_at_head"], pads, case["eos"])
    assert torch.equal(rec.puts(), out)


@pytest.mark.parametrize("B", [1, 4])
def test_arming_changes_no_launch_count(B):
    cfg = O.tiny_config()
    m = _model(cfg)
    eng = m._engine
    px, ids = O.make_inputs(cfg, B, 12, seed=3)
    eng.vision_encode(px.cuda())
    counts = {}
    for armed in (False, True, False, True):
        eng.stream_arm(armed)
        eng.kernel_launches(reset=True)
        _, first, _ = eng.prefill(ids.cuda(), 1, None, last_logits=False)
        n_prefill = eng.kernel_launches(reset=True)
        eng.extend(ids[:, -3:].cuda(), last_logits=False)
        n_extend = eng.kernel_launches(reset=True)
        tok = eng.token_buffer(B)
        tok.copy_(first)
        eng.decode_many(tok, 8)
        n_decode = eng.kernel_launches(reset=True)
        if armed:
            assert eng.stream_wait(9) == 9                             # extend's pick (step 0) and the 8 decode steps
        torch.cuda.synchronize()
        eng.stream_arm(False)
        counts.setdefault(armed, []).append((n_prefill, n_extend, n_decode))
    assert counts[True][0] == counts[False][0] == counts[True][1] == counts[False][1]


def test_consumer_stop_then_next_turn_extends_the_cache():
    from visualcla.modeling_utils import Stream
    cfg = MID
    m = _model(cfg, max_batch=1, max_seq=256)
    s0, s1, _, s3 = O.special_ids(cfg)
    m.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
    m.image_at_head = False
    px, ids = O.make_inputs(cfg, 1, 10, seed=11)
    ids = torch.cat([ids[:, :2], torch.full((1, cfg.r_queries), s3), ids[:, 2:]], 1)
    ids[0, 1], ids[0, 2 + cfg.r_queries] = s0, s1
    px, ids = px.cuda(), ids.cuda()
    eng = m._engine
    steps = []
    orig = eng.decode_many
    eng.decode_many = lambda tok, n: (steps.append(n), orig(tok, n))[1]
    k = 5

    def cb(x):
        if x.shape[-1] >= k:
            raise StopIteration
    out = m.generate(input_ids=ids, pixel_values=px, do_sample=False, max_new_tokens=60, eos_token_id=None, pad_token_id=0,
                     stopping_criteria=[Stream(cb)], return_dict_in_generate=True)
    eng.decode_many = orig
    assert out.sequences.shape == (1, k)
    assert 1 + sum(steps) - k <= 9, steps
    cache = out.past_key_values
    assert len(cache) == ids.shape[1] + k - 1
    # next turn: the conversation so far plus a new instruction extends the cache -- no vision tower, no full prefill
    nxt = torch.cat([ids, out.sequences, torch.tensor([[7, 8, 9, 10]], device=ids.device)], 1)
    seen = []
    for name in ("vision_encode", "prefill", "extend"):
        f = getattr(eng, name)
        setattr(eng, name, (lambda f, name: lambda *a, **kw: (seen.append(name), f(*a, **kw))[1])(f, name))
    turn = m.generate(input_ids=nxt, pixel_values=px, do_sample=False, max_new_tokens=8, eos_token_id=None, pad_token_id=0,
                      past_key_values=cache, return_dict_in_generate=True)
    for name in ("vision_encode", "prefill", "extend"):
        delattr(eng, name)
    assert seen == ["extend"], seen
    assert _decisive_ok(cfg, turn.sequences.cpu(), nxt.cpu(), px.cpu(), False, None, [])


def test_wait_for_a_step_that_never_comes_fails_fast():
    from visualcla import _native as N
    cfg = O.tiny_config()
    m = _model(cfg)
    eng = m._engine
    px, ids = O.make_inputs(cfg, 1, 12, seed=3)
    eng.vision_encode(px.cuda())
    eng.stream_arm(True)
    try:
        eng.prefill(ids.cuda(), 1, None, last_logits=False)
        assert eng.stream_wait(1) >= 1
        t0 = time.perf_counter()
        with pytest.raises(N.NativeError, match="never be published"):
            eng.stream_wait(3)                                         # only the prefill's step was enqueued
        assert time.perf_counter() - t0 < 5.0
    finally:
        eng.stream_arm(False)
    with pytest.raises(N.NativeError):                                 # beam mode refuses arming
        eng.set_beam(eng.beam_spec(2, 4))
        try:
            eng.stream_arm(True)
        finally:
            eng.set_beam(None)
