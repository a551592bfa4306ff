"""Host side of KV-cache reuse across generate() calls / chat turns, on the CPU with a fake engine that keeps the token ids it
"caches" (a deterministic toy model: the first pick is a function of the prompt's last id, then next = f(previous)).  Checks which
engine calls happen (full prefill vs truncate + extend), every condition that must fall back to a full prefill, the ids the cache
handle records, and that reuse never changes what generate() returns."""
import types

import pytest
import torch

from visualcla import _native as N
from visualcla import modeling_utils as mu
from visualcla.modeling_visualcla import VclaKVCache, VisualCLAModel

V, NQ = 50, 4
IMG0, IMG1, IMGT = 40, 41, 42


class CacheEngine:
    """Fake engine with the cache surface: prefill / extend / truncate / decode keep `self.cache` (the ids whose K/V a real engine
    holds, batch 1 rows only) and bump `session` like the native engine wrapper does."""
    device = torch.device("cpu")
    vocab, nq, max_batch, max_seq, max_prefill_tokens = V, NQ, 4, 256, 256

    def __init__(self, sampler=False):
        self.calls, self.session, self.cache, self.spec = [], 0, None, None
        self._sampler = sampler

    # ---- device sampler surface (EOS flags, pad after EOS), only when constructed with sampler=True
    def sampler_supported(self):
        return self._sampler

    @staticmethod
    def sampler_spec(**kw):
        return dict(kw)

    def set_sampler(self, spec):
        self.spec = spec

    def read_finished(self, B):
        return self.fin.to(torch.int32)

    def _start(self, first):
        self.hist = [first.clone()]
        self.fin = torch.zeros(first.shape[0], dtype=torch.bool)
        self._mark(first)

    def _mark(self, tok):
        for e in (self.spec or {}).get("eos_token_id", ()):
            self.fin |= tok.long() == e

    def vision_encode(self, px, return_embeds=False):
        self.calls.append(("vision_encode",))

    def prefill(self, ids, mode, rows, all_logits=False, last_logits=True, left_pad=None, pos_from_mask=True):
        self.session += 1
        self.calls.append(("prefill", ids.shape[1]))
        self.cache = [list(map(int, r)) for r in ids]
        first = (ids[:, -1] % V).to(torch.int32)
        self._start(first)
        ll = torch.zeros(ids.shape[0], V)
        ll[torch.arange(ids.shape[0]), first.long()] = 5.0
        return (ll if last_logits else None), first, None

    def truncate(self, lengths):
        self.session += 1
        self.calls.append(("truncate", list(lengths)))
        self.cache = [c[:min(len(c), int(n))] for c, n in zip(self.cache, lengths)]

    def extend(self, ids, all_logits=False, last_logits=True):
        self.session += 1
        self.calls.append(("extend", ids.shape[1]))
        for c, r in zip(self.cache, ids):
            c.extend(map(int, r))
        first = (ids[:, -1] % V).to(torch.int32)
        self._start(first)
        ll = torch.zeros(ids.shape[0], V)
        ll[torch.arange(ids.shape[0]), first.long()] = 5.0
        return (ll if last_logits else None), first, None

    def decode_step(self, tok_in, tok_out, logits=None, use_graph=True):
        self.session += 1
        for c, t in zip(self.cache, tok_in):
            c.append(int(t))
        was = self.fin.clone()
        nxt = ((tok_in.long() * 7 + 3) % V).to(torch.int32)
        if logits is not None:
            lg = torch.zeros(tok_in.shape[0], V)
            lg[torch.arange(tok_in.shape[0]), nxt.long()] = 5.0
            logits.copy_(lg)
        if self.spec is not None:
            nxt[was] = self.spec["pad_token_id"]
            self._mark(torch.where(was, torch.full_like(nxt, -1), nxt))
        tok_out.copy_(nxt)
        self.hist.append(tok_out.clone())

    def decode_many(self, tok, n):
        for _ in range(n):
            self.decode_step(tok, tok)

    def read_history(self, B, n):
        return torch.stack(self.hist[:n], 0)


def make_model(sampler=False, image_at_head=False):
    m = object.__new__(VisualCLAModel)
    m._engine = CacheEngine(sampler)
    m._tok_buf = {}
    m.image_at_head = image_at_head
    m.tokenizer = types.SimpleNamespace(img_start_token_id=IMG0, img_end_token_id=IMG1, img_token_id=IMGT)
    return m


def prompt(*text):
    """[BOS, <img>, 4 x <img_token>, </img>, text...] (placeholder layout, image rows 2..5, block ends at index 7)"""
    return torch.tensor([[1, IMG0] + [IMGT] * NQ + [IMG1] + list(text)])


PX = torch.arange(12, dtype=torch.float32).reshape(1, 3, 2, 2)
GREEDY = dict(do_sample=False, max_new_tokens=5, eos_token_id=None, pad_token_id=0)


def kinds(eng):
    return [c[0] for c in eng.calls]


def test_handle_records_the_cached_ids_and_turn_two_extends():
    m = make_model()
    eng = m._engine
    p1 = prompt(5, 6, 7)
    r1 = m.generate(input_ids=p1, pixel_values=PX, return_dict_in_generate=True, **GREEDY)
    h = r1.past_key_values
    assert isinstance(h, VclaKVCache) and h.is_current(eng)
    # the prompt, then the 4 tokens fed to decode steps; the 5th pick was never fed
    assert h.ids.tolist() == p1[0].tolist() + r1.sequences[0, :4].tolist() == eng.cache[0]
    p2 = torch.cat([p1, r1.sequences[:, :3], torch.tensor([[9, 10, 11]])], 1)     # history re-tokenized differently after 3 tokens
    eng.calls.clear()
    r2 = m.generate(input_ids=p2, pixel_values=PX.clone(), past_key_values=h, return_dict_in_generate=True, **GREEDY)
    keep = p1.shape[1] + 3
    assert eng.calls[:2] == [("truncate", [keep]), ("extend", p2.shape[1] - keep)]
    assert "vision_encode" not in kinds(eng) and "prefill" not in kinds(eng)
    assert eng.cache[0][: p2.shape[1]] == p2[0].tolist()
    fresh = make_model().generate(input_ids=p2, pixel_values=PX, return_dict_in_generate=True, **GREEDY)
    assert torch.equal(r2.sequences, fresh.sequences)
    assert r2.past_key_values.ids.tolist() == eng.cache[0]
    assert not h.is_current(eng), "the old handle went stale with the second call"


def test_reuse_is_off_by_default_in_chat_and_on_when_asked():
    def run(reuse):
        m = make_model()
        m.reuse_kv_cache = reuse
        history, turns = [], []
        for text in ([5, 6], [7, 8, 9], [10]):
            ids = prompt(*sum(([t] for t in text), []))
            if history:
                ids = torch.cat([history[-1], torch.tensor([text])], 1)
            out = m.generate(input_ids=ids, pixel_values=PX, **(mu._cache_kwargs(m)), **GREEDY)
            out = mu._keep_cache(m, out)
            history.append(torch.cat([ids, out], 1))
            turns.append(out)
        return m._engine, turns

    off_eng, off = run(False)
    assert kinds(off_eng).count("prefill") == 3 and kinds(off_eng).count("vision_encode") == 3 and "extend" not in kinds(off_eng)
    on_eng, on = run(True)
    assert kinds(on_eng).count("prefill") == 1 and kinds(on_eng).count("vision_encode") == 1
    assert kinds(on_eng).count("truncate") == 2 and kinds(on_eng).count("extend") == 2
    assert all(torch.equal(a, b) for a, b in zip(on, off))


def test_chat_keeps_the_handle_on_the_model():
    class Tok:
        bos_token, bos_token_id, eos_token_id = "", 1, 2
        img_start_token, img_end_token, img_token = "<img>", "</img>", "<img_token>"
        img_start_token_id, img_end_token_id, img_token_id = IMG0, IMG1, IMGT

        def __call__(self, text, return_tensors=None, add_special_tokens=None):
            from transformers import BatchEncoding
            n = len(text) % 7 + 3
            ids = prompt(*range(3, 3 + n))
            return BatchEncoding({"input_ids": ids, "attention_mask": torch.ones_like(ids)})

        def decode(self, ids, skip_special_tokens=True):
            return " ".join(map(str, ids.tolist()))

    m = make_model()
    m.tokenizer = Tok()
    m.num_patch = NQ
    from transformers import GenerationConfig
    gc = GenerationConfig(do_sample=False, max_new_tokens=4)
    mu.chat(m, PX, "hi", history=[], generation_config=gc)
    assert not hasattr(m, "_chat_kv_cache")
    m.reuse_kv_cache = True
    mu.chat(m, PX, "hi", history=[], generation_config=gc)
    assert isinstance(m._chat_kv_cache, VclaKVCache) and m._chat_kv_cache.is_current(m._engine)


@pytest.mark.parametrize("case", ["image", "stale", "batch", "left_pad", "image_at_head", "text_only_vs_image", "short_lcp"])
def test_fallbacks_to_a_full_prefill(case):
    m = make_model(image_at_head=(case == "image_at_head"))
    eng = m._engine
    p1 = prompt(5, 6, 7)
    h = m.generate(input_ids=p1, pixel_values=PX, return_dict_in_generate=True, **GREEDY).past_key_values
    p2 = torch.cat([p1, torch.tensor([[8, 9]])], 1)
    px, mask = PX, None
    if case == "image":
        px = PX + 1
    elif case == "stale":
        eng.prefill(p1, N.IMAGE_PLACEHOLDER, None)
    elif case == "batch":
        p2 = p2.repeat(2, 1)
        px = PX.repeat(2, 1, 1, 1)
    elif case == "left_pad":
        p2 = torch.cat([torch.tensor([[0]]), p2], 1)
        mask = torch.ones_like(p2)
        mask[0, 0] = 0
    elif case == "text_only_vs_image":
        px = None
    elif case == "short_lcp":
        p2 = p2.clone()
        p2[0, 4] = 3                                  # differs inside the image block
    eng.calls.clear()
    out = m.generate(input_ids=p2, pixel_values=px, attention_mask=mask, past_key_values=h, **GREEDY)
    assert "prefill" in kinds(eng) and "extend" not in kinds(eng) and "truncate" not in kinds(eng), eng.calls
    ref = make_model(image_at_head=(case == "image_at_head")).generate(input_ids=p2, pixel_values=px, attention_mask=mask, **GREEDY)
    assert torch.equal(out, ref)


def test_prompt_that_is_a_prefix_of_the_cache_re_extends_one_token():
    m = make_model()
    eng = m._engine
    p1 = prompt(5, 6, 7)
    r1 = m.generate(input_ids=p1, pixel_values=PX, return_dict_in_generate=True, **GREEDY)
    for p2 in (p1, torch.cat([p1, r1.sequences[:, :2]], 1)):
        h = m.generate(input_ids=p1, pixel_values=PX, return_dict_in_generate=True, **GREEDY).past_key_values
        eng.calls.clear()
        out = m.generate(input_ids=p2, pixel_values=PX, past_key_values=h, **GREEDY)
        assert eng.calls[:2] == [("truncate", [p2.shape[1] - 1]), ("extend", 1)]
        assert torch.equal(out, make_model().generate(input_ids=p2, pixel_values=PX, **GREEDY))


def test_text_only_conversation_reuses_too():
    m = make_model()
    eng = m._engine
    p1 = torch.tensor([[1, 5, 6, 7]])
    h = m.generate(input_ids=p1, return_dict_in_generate=True, **GREEDY).past_key_values
    assert h.pixel_values is None and h.mode == N.TEXT_ONLY
    eng.calls.clear()
    m.generate(input_ids=torch.cat([p1, torch.tensor([[9]])], 1), past_key_values=h, **GREEDY)
    assert kinds(eng)[:2] == ["truncate", "extend"]


def test_cached_ids_include_the_pad_steps_past_eos_on_the_device_path():
    """Greedy + EOS on the device sampler: graphs of 8 steps keep running past EOS (emitting pad), and every fed token is in the
    cache; the returned sequence is cut at EOS exactly as without a handle."""
    base = make_model().generate(input_ids=prompt(5, 6, 7), pixel_values=PX, **dict(GREEDY, max_new_tokens=20))
    eos = int(base[0, 2])
    m = make_model(sampler=True)
    eng = m._engine
    r = m.generate(input_ids=prompt(5, 6, 7), pixel_values=PX, return_dict_in_generate=True,
                   **dict(GREEDY, max_new_tokens=20, eos_token_id=eos, pad_token_id=49))
    assert r.sequences[0].tolist() == base[0, :3].tolist()
    h = r.past_key_values
    n_fed = len(eng.hist) - 1                                  # decode steps run (a whole graph of 8 past the first pick)
    assert n_fed == 8 and h.ids.tolist() == eng.cache[0]
    assert h.ids[-n_fed:].tolist() == [int(t) for t in torch.stack(eng.hist[:n_fed])[:, 0]]
    assert h.ids[-1].item() == 49, "the pad steps after EOS were fed too"
    eng.calls.clear()
    p2 = torch.cat([prompt(5, 6, 7), r.sequences, torch.tensor([[12, 13]])], 1)
    out = m.generate(input_ids=p2, pixel_values=PX, past_key_values=h, **dict(GREEDY, eos_token_id=eos, pad_token_id=49))
    assert kinds(eng)[:2] == ["truncate", "extend"] and eng.calls[0][1] == [prompt(5, 6, 7).shape[1] + 3]
    ref = make_model(sampler=True).generate(input_ids=p2, pixel_values=PX, **dict(GREEDY, eos_token_id=eos, pad_token_id=49))
    assert torch.equal(out, ref)


def test_host_loop_path_records_what_it_fed():
    m = make_model()
    eng = m._engine
    r = m.generate(input_ids=prompt(5, 6), pixel_values=PX, return_dict_in_generate=True, output_logits=True, **GREEDY)
    assert r.past_key_values.ids.tolist() == eng.cache[0] and len(r.logits) == 5
    assert r.past_key_values.ids[-4:].tolist() == r.sequences[0, :4].tolist()


class CharTok:
    """Character-level stand-in for the tokenizer: special tokens keep their ids, every other character maps to 3..32, and decode
    does not invert encode (like SentencePiece around a reply, the re-tokenized history differs from the generated ids)."""
    bos_token, bos_token_id = "", 1
    img_start_token, img_end_token, img_token = "<img>", "</img>", "<img_token>"
    img_start_token_id, img_end_token_id, img_token_id = IMG0, IMG1, IMGT

    def __init__(self, eos):
        self.eos_token_id = eos

    def __call__(self, text, return_tensors=None, add_special_tokens=None):
        import re
        from transformers import BatchEncoding
        special = {"<img>": IMG0, "</img>": IMG1, "<img_token>": IMGT}
        ids = [1]
        for part in re.split(r"(<img>|</img>|<img_token>)", text):
            ids += [special[part]] if part in special else [ord(c) % 30 + 3 for c in part]
        t = torch.tensor([ids])
        return BatchEncoding({"input_ids": t, "attention_mask": torch.ones_like(t)})

    def decode(self, ids, skip_special_tokens=True):
        return "".join(chr(ord("a") + int(i) % 26) for i in ids if int(i) != self.eos_token_id)


def test_streamed_turn_that_ends_on_eos_keeps_the_cache_for_the_next_turn():
    """chat_in_stream stops listening at the EOS id; generation must then end normally (not be aborted), so the cache handle of the
    streamed turn is stored before the generator finishes and the next turn extends it instead of running the vision tower again."""
    from transformers import GenerationConfig
    m = make_model()
    eng = m._engine
    m.num_patch, m.reuse_kv_cache = NQ, True
    m.tokenizer = CharTok(eos=0)
    history = []
    mu.chat(m, PX, "hi", history=history, generation_config=GenerationConfig(do_sample=False, max_new_tokens=4))
    # the streamed turn's reply: first pick = last prompt id (':' -> 31), then the toy chain 31 -> 20 -> 43 -> ...; 43 plays EOS
    m.tokenizer = CharTok(eos=43)
    gc = GenerationConfig(do_sample=False, max_new_tokens=12, eos_token_id=43, pad_token_id=0)
    eng.calls.clear()
    out = list(mu.chat_in_stream(m, PX, "more", history=history, generation_config=gc))
    assert [r for r, _ in out] == ["f", "fu"], out          # ids 31, 20; the consumer stopped at 43
    assert "extend" in kinds(eng)
    h = m._chat_kv_cache
    assert h.is_current(eng), "the streamed turn's handle survives the consumer stopping at EOS"
    ids = h.ids.tolist()
    assert ids == eng.cache[0] and any(ids[i:i + 3] == [31, 31, 20] for i in range(len(ids))), "prompt end ':', then the fed 31, 20"
    history = out[-1][1]
    eng.calls.clear()
    mu.chat(m, PX, "again", history=history, generation_config=GenerationConfig(do_sample=False, max_new_tokens=4))
    assert kinds(eng)[:2] == ["truncate", "extend"] and "vision_encode" not in kinds(eng) and "prefill" not in kinds(eng)
