"""Prompt lookup decoding on the device (include/vcla.h, prompt lookup decoding).  The verification attention (attn_decode_kernel in its
append + attend modes through vcla_op_attention_decode_lookup) gives every row r the one-token kernel's bits at length seq_len + r + 1
and is within the decode tolerance of an fp64 reference; generate(prompt_lookup_num_tokens=k) returns exactly the tokens of the same
call without it (argmax graphs, the device sampler with EOS / min_new_tokens / penalties / the chat default, bf16 and int8 projections,
text-only and image-at-head layouts, a reused KV cache); and on a cyclic output the drafts are accepted, in fewer steps than tokens."""
import ctypes as C
import types

import pytest
import torch

import visualcla_oracle as O
from test_decode_attention_gpu import HD, OUT_TOL, SCALE, decode_ref, make_case

pytestmark = pytest.mark.gpu

MID = O.PathConfig(v_layers=2, r_layers=2, t_hidden=1024, t_heads=8, t_ffn=2752, t_layers=3, t_vocab=5003)
KS = [1, 2, 7, 10, 15, 20]


def _one_token(partial, pool, table, L, pt, H, kv_splits, theta):
    from visualcla import _native as N
    pool_d, part_d, table_d = pool.cuda(), partial.cuda(), table.cuda()
    len_d = torch.tensor([L], dtype=torch.int32, device="cuda")
    out = torch.zeros(1, H * HD, dtype=torch.bfloat16, device="cuda")
    N.check(N.load().vcla_op_attention_decode(N.ptr(part_d), partial.shape[0], N.ptr(pool_d), N.ptr(table_d), table.shape[1], pt, N.ptr(len_d),
                                              N.ptr(out), 1, H, kv_splits, C.c_float(SCALE), C.c_float(theta), 0, 0, 1,
                                              C.c_void_p(torch.cuda.current_stream().cuda_stream)), "vcla_op_attention_decode")
    return out.cpu(), pool_d.cpu()


@pytest.mark.parametrize("pt", [8, 16, 32, 64])
def test_lookup_attention_rows_are_one_token_steps(pt):
    from visualcla import _native as N
    H, theta, splits = 4, 10000.0, 2
    for R in (2, 5, 16):
        for P in (1, pt - 1, pt, 3 * pt - 2, 5 * pt + 3):
            for kv_splits in (1, 3, 8):
                case = make_case(pt, [P], H, splits, seed=P * 131 + R, steps=R)
                partial = torch.randn(splits, R, 3 * H * HD, generator=torch.Generator().manual_seed(R + P)) / 2 ** 0.5
                pool_d, part_d, table_d = case.pool.cuda(), partial.cuda(), case.table.cuda()
                len_d = torch.tensor([P], dtype=torch.int32, device="cuda")
                out = torch.zeros(R, H * HD, dtype=torch.bfloat16, device="cuda")
                N.check(N.load().vcla_op_attention_decode_lookup(N.ptr(part_d), splits, N.ptr(pool_d), N.ptr(table_d), case.table.shape[1], pt,
                                                                 N.ptr(len_d), N.ptr(out), R, H, kv_splits, C.c_float(SCALE), C.c_float(theta),
                                                                 C.c_void_p(torch.cuda.current_stream().cuda_stream)), "lookup attention")
                out, pool = out.cpu(), pool_d.cpu()
                what = f"pt {pt} rows {R} seq_len {P} kv_splits {kv_splits}"
                for r in range(R):
                    # the one-token kernel at length P + r + 1 over the rows the lookup call appended before row r
                    o1, pool1 = _one_token(partial[:, r:r + 1], pool, case.table, P + r, pt, H, kv_splits, theta)
                    assert torch.equal(o1.view(torch.int16), out[r:r + 1].view(torch.int16)), f"{what}: row {r} differs from the one-token step"
                    assert torch.equal(pool1.view(torch.int16), pool.view(torch.int16)), f"{what}: appended row {r} differs from the one-token append"
                    ref, _, _ = decode_ref(partial[:, r:r + 1], pool, case.table, [P + r], pt, H, SCALE, theta)
                    err = (out[r].view(H, HD).double() - ref[0]).abs().max().item() / max(1.0, ref[0].abs().max().item())
                    assert err <= OUT_TOL, f"{what}: row {r} max |out - ref| = {err:.3e}"


def _model(load_in_8bit=False, max_seq=256):
    import visualcla
    return visualcla.VisualCLAModel.from_synthetic(MID.to_dict(), seed=0, max_batch=2, max_seq=max_seq, load_in_8bit=load_in_8bit)


def _modes(m, ids, px):
    from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG
    full = m.generate(input_ids=ids, pixel_values=px, do_sample=False, max_new_tokens=40, eos_token_id=None, pad_token_id=0)
    eos = int(full[0, 17])
    gc = DEFAULT_GENERATION_CONFIG.__class__(**{**DEFAULT_GENERATION_CONFIG.to_dict(), "max_new_tokens": 40, "pad_token_id": 0})
    return [dict(do_sample=False, max_new_tokens=40, eos_token_id=None, pad_token_id=0),
            dict(do_sample=False, max_new_tokens=37, eos_token_id=None, pad_token_id=0),            # max_new inside an accepted run
            dict(do_sample=False, max_new_tokens=40, eos_token_id=eos, pad_token_id=0),
            dict(do_sample=False, max_new_tokens=40, eos_token_id=eos, pad_token_id=0, min_new_tokens=25),
            dict(do_sample=False, max_new_tokens=40, repetition_penalty=1.3, no_repeat_ngram_size=3, eos_token_id=None, pad_token_id=0),
            dict(generation_config=gc)]


@pytest.mark.parametrize("int8", [False, True])
@pytest.mark.parametrize("k", KS)
def test_generate_equals_plain(k, int8):
    m = _model(load_in_8bit=int8)
    eng = m._engine
    for layout in ("text", "head"):
        px, ids = O.make_inputs(MID, 1, 24, seed=11)
        m.image_at_head = layout == "head"
        px = px.cuda() if layout == "head" else None
        ids = ids.cuda()
        for kw in _modes(m, ids, px):
            torch.manual_seed(99)
            plain = m.generate(input_ids=ids, pixel_values=px, **kw)
            for n in (1, 2, 3):
                torch.manual_seed(99)
                out = m.generate(input_ids=ids, pixel_values=px, prompt_lookup_num_tokens=k, max_matching_ngram_size=n, **kw)
                assert torch.equal(out, plain), (k, n, int8, layout, kw, out.tolist(), plain.tolist())
                assert eng.lookup_stats()[2] > 0, "the call ran verification steps"
    eng.close()


def test_reused_cache_turn_equals_plain():
    m = _model()
    cfg = MID
    s0, s1, _, s3 = O.special_ids(cfg)
    m.image_at_head = False
    m.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
    px, _ = O.make_inputs(cfg, 1, 8, seed=77)
    g = torch.Generator().manual_seed(3)
    t1, t2 = torch.randint(3, cfg.t_vocab - 4, (1, 20), generator=g), torch.randint(3, cfg.t_vocab - 4, (1, 15), generator=g)
    p1 = torch.cat([torch.tensor([[1, s0]]), torch.full((1, cfg.r_queries), s3), torch.tensor([[s1]]), t1], 1)
    kw = dict(do_sample=False, eos_token_id=None, pad_token_id=0, return_dict_in_generate=True)
    runs = {}
    for k in (0, 7):
        r1 = m.generate(input_ids=p1.cuda(), pixel_values=px.cuda(), max_new_tokens=20, prompt_lookup_num_tokens=k, **kw)
        p2 = torch.cat([p1, r1.sequences.cpu(), t2], 1)
        r2 = m.generate(input_ids=p2.cuda(), pixel_values=px.cuda(), max_new_tokens=20, past_key_values=r1.past_key_values,
                        prompt_lookup_num_tokens=k, **kw)
        runs[k] = (r1.sequences, r2.sequences, r1.past_key_values.ids)
    assert torch.equal(runs[0][0], runs[7][0]) and torch.equal(runs[0][1], runs[7][1])
    assert torch.equal(runs[0][2], runs[7][2])
    m._engine.close()


def _cycle_period(row, tail=128):
    t = row[-tail:].tolist()
    for p in range(1, tail // 2):
        if all(t[i] == t[i + p] for i in range(tail - p)):
            return p
    return 0


def test_lookup_accepts_drafts_on_a_cycle():
    # with o_proj and down_proj zeroed the next greedy token is a function of the current one, so the output must end in a cycle
    m = _model(max_seq=512)
    eng = m._engine
    T, F = MID.t_hidden, MID.t_ffn
    for i in range(MID.t_layers):
        p = f"text_model.model.layers.{i}."
        eng.load_weight(p + "self_attn.o_proj.weight", torch.zeros(T, T, dtype=torch.bfloat16, device="cuda"))
        eng.load_weight(p + "mlp.down_proj.weight", torch.zeros(T, F, dtype=torch.bfloat16, device="cuda"))
    kw = dict(do_sample=False, eos_token_id=None, pad_token_id=0, max_new_tokens=300)
    _, ids = O.make_inputs(MID, 1, 16, seed=5)
    plain = m.generate(input_ids=ids.cuda(), **kw)
    assert _cycle_period(plain[0]), "the greedy output does not end in a cycle"
    out = m.generate(input_ids=ids.cuda(), prompt_lookup_num_tokens=10, **kw)
    assert torch.equal(out, plain)
    produced, fin, steps, drafted, accepted, _ = eng.lookup_stats()
    assert produced == 300 and accepted > 0 and steps < produced - 1, (steps, drafted, accepted)
    eng.close()


@pytest.mark.parametrize("int8", [False, True])
def test_verification_step_logits_are_one_token_logits(int8):
    """The logits of one verification step over R rows are bit-equal, row by row, to R one-token steps fed the same tokens."""
    m = _model(load_in_8bit=int8)
    eng = m._engine
    V = MID.t_vocab
    _, ids = O.make_inputs(MID, 1, 24, seed=11)
    ids = ids.cuda()
    t_in = torch.zeros(1, dtype=torch.int32, device="cuda")
    t_out = torch.zeros(1, dtype=torch.int32, device="cuda")
    lg = torch.empty(1, V, dtype=torch.float32, device="cuda")
    for k in (1, 7, 15):
        _, first, _ = eng.prefill(ids, 0, None, last_logits=False)
        t_in.copy_(first)
        eng.set_lookup(ids[0], k, 2, 100)
        eng.decode_many(t_in, 3)                                  # a few verification steps: the step under test starts later
        produced, _, _, _, _, R = eng.lookup_stats()
        hist = eng.read_history(1, produced)[:, 0].cpu()
        rows_tok = eng.read_stage("lookup_tokens", R).view(torch.int32)
        assert int(rows_tok[0]) == int(hist[-1])
        eng.decode_many(t_in, 1)
        step = eng.read_stage("step_logits", R)
        eng.set_lookup(None)
        _, first, _ = eng.prefill(ids, 0, None, last_logits=False)
        for t in hist[:-1].tolist():
            t_in.fill_(t)
            eng.decode_step(t_in, t_out, lg)
        for r in range(R):
            t_in.fill_(int(rows_tok[r]))
            eng.decode_step(t_in, t_out, lg)
            assert torch.equal(lg.cpu()[0], step[r]), f"k {k} int8 {int8}: row {r} of {R} differs from the one-token step"
    eng.close()


def _cyclic_model():
    # with o_proj and down_proj zeroed the next token's logits depend on the current token only: outputs keep repeating earlier text
    m = _model(max_seq=512)
    T, F = MID.t_hidden, MID.t_ffn
    for i in range(MID.t_layers):
        p = f"text_model.model.layers.{i}."
        m._engine.load_weight(p + "self_attn.o_proj.weight", torch.zeros(T, T, dtype=torch.bfloat16, device="cuda"))
        m._engine.load_weight(p + "mlp.down_proj.weight", torch.zeros(T, F, dtype=torch.bfloat16, device="cuda"))
    return m


def test_device_sampler_accepts_drafts_on_a_cycle():
    """Drafts accepted on the device sampler's path (rows >= 1 drawn with counter (L + r, 0) over the provisional drafts), with the
    same tokens as the call without lookup."""
    from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG
    m = _cyclic_model()
    eng = m._engine
    _, ids = O.make_inputs(MID, 1, 16, seed=5)
    greedy = m.generate(input_ids=ids.cuda(), do_sample=False, max_new_tokens=150, eos_token_id=None, pad_token_id=0).cpu()
    # the greedy continuation of the last prompt token is in the prompt: the drafts are the greedy tokens
    ids = torch.cat([ids, greedy, ids[:, -1:]], 1).cuda()
    eos = next(t for t in range(3, MID.t_vocab) if t not in set(greedy[0].tolist()))
    base = dict(max_new_tokens=120, pad_token_id=0)
    modes = [dict(base, do_sample=False, eos_token_id=eos, min_new_tokens=30),
             dict(base, do_sample=False, repetition_penalty=1.1, eos_token_id=None),
             dict(base, do_sample=True, temperature=0.5, top_k=40, top_p=0.9, eos_token_id=None),
             dict(generation_config=DEFAULT_GENERATION_CONFIG.__class__(**{**DEFAULT_GENERATION_CONFIG.to_dict(), **base}))]
    for i, kw in enumerate(modes):
        for k in (3, 10, 15):
            torch.manual_seed(7)
            plain = m.generate(input_ids=ids, **kw)
            torch.manual_seed(7)
            out = m.generate(input_ids=ids, prompt_lookup_num_tokens=k, **kw)
            assert torch.equal(out, plain), (i, k, out.tolist(), plain.tolist())
            produced, _, steps, drafted, accepted, _ = eng.lookup_stats()
            if i < 3:                              # the chat default bans repeated 15-grams: its acceptance is not asserted
                assert accepted > 0 and steps < produced - 1, (i, k, steps, drafted, accepted)
    eng.close()


def test_streamed_lookup_equals_plain_and_chat_in_stream_ends_on_chats_reply():
    import visualcla
    from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG
    m = _cyclic_model()
    eng = m._engine
    _, ids = O.make_inputs(MID, 1, 16, seed=5)
    ids = ids.cuda()

    class Rec:
        def __init__(self):
            self.puts = []

        def put(self, v):
            self.puts.append(v.clone())

        def end(self):
            pass
    greedy = m.generate(input_ids=ids, do_sample=False, max_new_tokens=120, eos_token_id=None, pad_token_id=0)
    for kw in (dict(do_sample=False, eos_token_id=None), dict(do_sample=False, eos_token_id=int(greedy[0, 90])),
               dict(do_sample=True, temperature=0.5, top_k=40, eos_token_id=None)):
        torch.manual_seed(3)
        plain = m.generate(input_ids=ids, max_new_tokens=120, pad_token_id=0, **kw)
        torch.manual_seed(3)
        rec = Rec()
        out = m.generate(input_ids=ids, max_new_tokens=120, pad_token_id=0, prompt_lookup_num_tokens=10, streamer=rec, **kw)
        assert torch.equal(out, plain), kw
        puts = rec.puts[1:]
        assert rec.puts[0].shape == (1, 0) and all(p.shape[0] == 1 and p.shape[1] >= 1 and p.dtype == torch.int64 for p in puts)
        assert torch.cat(puts, 1).tolist() == out.cpu().tolist()
        assert len(puts) < out.shape[1], "accepted drafts arrive several per put"
    eng.close()


def test_chat_in_stream_with_lookup_ends_on_chats_reply():
    import visualcla
    from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG
    cfg = O.tiny_config()
    m = visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=0, max_batch=1, max_seq=512)
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
    for extra in (dict(do_sample=False, repetition_penalty=1.0, no_repeat_ngram_size=0), dict()):
        gc = DEFAULT_GENERATION_CONFIG.__class__(**{**DEFAULT_GENERATION_CONFIG.to_dict(), "max_new_tokens": 40,
                                                    "prompt_lookup_num_tokens": 10, **extra})
        torch.manual_seed(99)
        resp, _ = visualcla.chat(m, image=px, text="describe the describe", history=[], generation_config=gc)
        torch.manual_seed(99)
        chunks = list(visualcla.chat_in_stream(m, image=px, text="describe the describe", history=[], generation_config=gc))
        assert chunks[-1][0] == resp, (extra, chunks[-1][0], resp)
    m._engine.close()
