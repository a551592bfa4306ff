"""Extending resident sequences from the paged KV cache (vcla_prefill_extend / vcla_kv_truncate) and reusing it across generate()
calls and chat turns, on the device: the paged prefill attention operator against a torch fp32 reference, the engine against the
oracle's forward of the concatenated sequence, page accounting, 7B widths, and chat() with a real tokenizer."""
import copy
import ctypes as C
import math

import pytest
import torch

import visualcla_oracle as O

pytestmark = pytest.mark.gpu

LOGIT_TOL = 1.5e-2        # relative to max |logit| (as in test_parity_gpu)
LOGIT_TOL_TINY = 3.0e-2   # the 2-layer tiny configuration (as in test_parity_gpu)


def _margin_ok_tokens(dev_tokens, ora_tokens, ora_logits, tol_abs, free_running=False):
    """Tokens must be equal wherever the oracle's top1-top2 margin exceeds 2*tol_abs (free-running: up to the first mismatch)."""
    top2 = ora_logits.topk(2, dim=-1).values
    decisive = (top2[..., 0] - top2[..., 1]) > 2 * tol_abs
    diff = dev_tokens.cpu() != ora_tokens.cpu()
    if free_running:
        decisive = decisive & (torch.cumsum(torch.cumsum(diff.long(), 1), 1) <= 1)
    bad = diff & decisive
    return int(bad.sum()), int(decisive.sum()), int(decisive.numel())


def _rel(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    return (a - b).abs().max().item() / max(1e-6, b.abs().max().item())


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. the operator
# ---------------------------------------------------------------------------------------------------------------------------------
def _paged_case(pt, lens, T, H, seed):
    """Random q / K / V, the K/V of sequence b's first lens[b] + T tokens scattered over a permuted page pool whose other slots
    hold NaN (unwritten cache slots may hold anything)."""
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    pps = max(1, math.ceil((max(lens) + T) / pt))
    n_pages = B * pps + 3
    table = torch.randperm(n_pages, generator=g)[: B * pps].view(B, pps).to(torch.int32)
    pool = torch.full((n_pages, 2, H, pt, 128), float("nan"), dtype=torch.bfloat16)
    q = torch.randn(B, T, H, 128, generator=g).to(torch.bfloat16)
    ks, vs = [], []
    for b, L in enumerate(lens):
        k = torch.randn(L + T, H, 128, generator=g).to(torch.bfloat16)
        v = torch.randn(L + T, H, 128, generator=g).to(torch.bfloat16)
        j = torch.arange(L + T)
        pages, slots = table[b, j // pt].long(), j % pt
        pool[pages, 0, :, slots] = k
        pool[pages, 1, :, slots] = v
        ks.append(k)
        vs.append(v)
    return q, pool, table, ks, vs


def _paged_ref(q, ks, vs, lens, scale):
    B, T, H, _ = q.shape
    out = torch.empty(B, T, H, 128)
    for b, L in enumerate(lens):
        qf, kf, vf = q[b].float().transpose(0, 1), ks[b].float().transpose(0, 1), vs[b].float().transpose(0, 1)   # (H, rows, 128)
        s = qf @ kf.transpose(1, 2) * scale
        vis = torch.arange(L + T)[None, :] <= (L + torch.arange(T))[:, None]
        s = s.masked_fill(~vis[None], float("-inf"))
        out[b] = (torch.softmax(s, -1) @ vf).transpose(0, 1)
    return out


def _row_err(got, ref):
    """max over (sequence, row, head) of the error relative to that output row's largest |value|.  bf16 rounding of P and of the
    output stays below ~0.5 %; one key wrongly visible or masked moves a row by > 10 % even behind a 1500-token prefix (an
    absolute bound would not see it there: those outputs are ~1e-2 and the change ~1e-3 absolute)."""
    return ((got - ref).abs().amax(-1) / ref.abs().amax(-1).clamp_min(1e-6)).max().item()


PAGED_TOL = 2e-2


def _paged_run(q, pool, table, lens, pt):
    from visualcla import _native as N
    lib = N.load()
    B, T, H, _ = q.shape
    qd, pd, td = q.reshape(B * T, H * 128).cuda(), pool.cuda(), table.cuda()
    ld = torch.tensor(lens, dtype=torch.int32, device="cuda")
    out = torch.zeros(B * T, H * 128, dtype=torch.bfloat16, device="cuda")
    N.check(lib.vcla_op_attention_paged(N.ptr(qd), H * 128, N.ptr(pd), N.ptr(td), table.shape[1], pt, N.ptr(ld), N.ptr(out), H * 128,
                                        B, H, T, C.c_float(128 ** -0.5), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
            "vcla_op_attention_paged")
    return out.view(B, T, H, 128).float().cpu()


def test_paged_attention_operator_refuses_a_negative_page():
    """A negative table entry among those the chunk reads is refused on the host, before any launch."""
    from visualcla import _native as N
    lens, T, pt = [20, 3], 5, 8
    q, pool, table, _ks, _vs = _paged_case(pt, lens, T, 2, seed=3)
    table[1, 0] = -1                                   # sequence 1 reads page 0 only (3 + 5 tokens)
    with pytest.raises(N.NativeError, match="no page 0"):
        _paged_run(q, pool, table, lens, pt)


@pytest.mark.parametrize("pt", [8, 16, 32, 64])
@pytest.mark.parametrize("prefix", [0, 1, 63, 64, 65, 1500])
def test_paged_attention_operator(pt, prefix):
    """B = 3 sequences with different cached lengths, chunks of 1 / 17 / 64 / 130 rows; H = 4 heads leaves SMs idle, so every
    launch with more than two key tiles takes the split-KV path."""
    for T in (1, 17, 64, 130):
        lens = [prefix, prefix // 2, prefix + 7]
        q, pool, table, ks, vs = _paged_case(pt, lens, T, 4, seed=pt * 1000 + prefix + T)
        got = _paged_run(q, pool, table, lens, pt)
        ref = _paged_ref(q, ks, vs, lens, 128 ** -0.5)
        assert torch.isfinite(got).all(), (pt, prefix, T)
        err = _row_err(got, ref)
        assert err <= PAGED_TOL, f"page_tokens {pt} prefix {prefix} chunk {T}: row-relative err {err:.3e}"


@pytest.mark.parametrize("pt", [16, 64])
def test_paged_attention_full_grid_and_split_determinism(pt):
    """32 heads x 3 sequences x 3 query tiles cover the SMs (no split); one sequence, one row over a ~1500-token prefix splits the
    keys over many CTAs -- run twice, the combine in split order must give bit-identical output."""
    lens = [600, 13, 1100]
    q, pool, table, ks, vs = _paged_case(pt, lens, 130, 32, seed=5 + pt)
    err = _row_err(_paged_run(q, pool, table, lens, pt), _paged_ref(q, ks, vs, lens, 128 ** -0.5))
    assert err <= PAGED_TOL, f"full grid: row-relative err {err:.3e}"
    lens = [1499]
    q, pool, table, ks, vs = _paged_case(pt, lens, 1, 32, seed=9 + pt)
    a = _paged_run(q, pool, table, lens, pt)
    b = _paged_run(q, pool, table, lens, pt)
    assert torch.equal(a, b), "split-KV combine must be deterministic"
    assert _row_err(a, _paged_ref(q, ks, vs, lens, 128 ** -0.5)) <= PAGED_TOL


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. / 3. the engine against the oracle, page accounting
# ---------------------------------------------------------------------------------------------------------------------------------
MID = O.PathConfig(v_layers=2, r_layers=2, t_hidden=1024, t_heads=8, t_ffn=2752, t_layers=3, t_vocab=5003)


def _model(cfg, seed, max_batch, max_seq):
    import visualcla
    return visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=seed, max_batch=max_batch, max_seq=max_seq)


def _emb(w, ids):
    return w["text_model.model.embed_tokens.weight"][ids].float()


def _check_pages(eng, lens):
    _pps, total, pt = eng.kv_geometry()
    _table, owned, free, exhausted = eng.kv_pages()
    for b, n in enumerate(lens):
        assert int(owned[b]) >= math.ceil((n + 1) / pt), (b, n, owned.tolist())
    assert free + int(owned.sum()) == total and exhausted == 0


def test_extend_in_chunks_matches_the_oracle():
    """Prefill with an image (at-head layout), then extend in three chunks with all logits: each chunk's logits equal the oracle's
    forward of the whole concatenated sequence at those positions.  Pages are handed out in a permuted order."""
    from visualcla import _native as N
    cfg, seed = MID, 5
    m = _model(cfg, seed, 1, 512)
    eng = m._engine
    eng.kv_debug_shuffle(11)
    w = O.make_weights(cfg, seed)
    px, ids = O.make_inputs(cfg, 1, 40, seed=3)
    g = torch.Generator().manual_seed(8)
    chunks = [torch.randint(3, cfg.t_vocab - 4, (1, n), generator=g) for n in (17, 64, 130)]
    eng.vision_encode(px.cuda())
    eng.prefill(ids.cuda(), N.IMAGE_AT_HEAD, None)
    s0, s1, _, s3 = O.special_ids(cfg)
    x = O.splice(w, cfg, ids, O.vision_encode(w, cfg, px), True, s0, s1, s3)
    full = torch.cat([x] + [_emb(w, c) for c in chunks], 1)
    ref = O.llama_forward(w, cfg, full)
    pos = x.shape[1]
    for c in chunks:
        last, tok, la = eng.extend(c.cuda(), all_logits=True)
        r = ref[:, pos:pos + c.shape[1]]
        assert _rel(la, r) <= LOGIT_TOL, f"chunk at {pos}: rel err {_rel(la, r):.3e}"
        assert _rel(last, r[:, -1]) <= LOGIT_TOL                  # the last row again, through the decode-side lm_head
        assert int(tok[0]) == int(last[0].argmax())
        pos += c.shape[1]
    _check_pages(eng, [pos])


def test_extend_after_a_left_padded_batch():
    """A left-padded B = 2 first prefill leaves different cached lengths per sequence; the chunk of each starts at its own length."""
    cfg, seed = MID, 6
    m = _model(cfg, seed, 2, 256)
    eng = m._engine
    w = O.make_weights(cfg, seed)
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(3, cfg.t_vocab - 4, (2, 50), generator=g)
    pads = torch.tensor([0, 19], dtype=torch.int32)
    ids[1, :19] = 0
    from visualcla import _native as N
    eng.prefill(ids.cuda(), N.TEXT_ONLY, None, left_pad=pads, pos_from_mask=True)
    chunks = [torch.randint(3, cfg.t_vocab - 4, (2, n), generator=g) for n in (9, 70)]
    lens = [50, 31]
    for i, c in enumerate(chunks):
        _, _, la = eng.extend(c.cuda(), all_logits=True)
        for b in range(2):
            seq = torch.cat([ids[b, int(pads[b]):]] + [cc[b] for cc in chunks[: i + 1]])
            ref = O.llama_forward(w, cfg, _emb(w, seq[None]))[0, -c.shape[1]:]
            assert _rel(la[b], ref) <= LOGIT_TOL, f"sequence {b}: rel err {_rel(la[b], ref):.3e}"
        lens = [n + c.shape[1] for n in lens]
    _check_pages(eng, lens)


def _oracle_greedy_from(w, cfg, embeds, n):
    cache = O.KVCache(cfg.t_layers)
    logits = O.llama_forward(w, cfg, embeds, cache, last_only=True)[:, -1]
    toks, logs = [], []
    for step in range(n):
        nxt = logits.argmax(-1)
        toks.append(nxt)
        logs.append(logits)
        if step < n - 1:
            logits = O.llama_forward(w, cfg, _emb(w, nxt)[:, None], cache, last_only=True)[:, -1]
    return torch.stack(toks, 1), torch.stack(logs, 1)


def test_decode_truncate_extend_matches_the_oracle():
    """prefill, 20 greedy decode steps, truncate back to the prompt + 10 of them, extend by a new chunk, decode again: the extend
    logits and the greedy tokens after it follow the oracle of the kept sequence + the chunk."""
    from visualcla import _native as N
    cfg, seed = MID, 7
    m = _model(cfg, seed, 1, 512)
    eng = m._engine
    w = O.make_weights(cfg, seed)
    px, ids = O.make_inputs(cfg, 1, 33, seed=4)
    eng.vision_encode(px.cuda())
    _, tok0, _ = eng.prefill(ids.cuda(), N.IMAGE_AT_HEAD, None)
    tok = tok0.clone()
    fed = []
    for _ in range(20):
        fed.append(int(tok[0]))
        eng.decode_step(tok, tok, None)
    S = ids.shape[1] + cfg.r_queries
    eng.truncate([S + 10])
    chunk = torch.randint(3, cfg.t_vocab - 4, (1, 23), generator=torch.Generator().manual_seed(1))
    last, first, la = eng.extend(chunk.cuda(), all_logits=True)
    s0, s1, _, s3 = O.special_ids(cfg)
    x = O.splice(w, cfg, ids, O.vision_encode(w, cfg, px), True, s0, s1, s3)
    full = torch.cat([x, _emb(w, torch.tensor([fed[:10]])), _emb(w, chunk)], 1)
    ref = O.llama_forward(w, cfg, full)[:, -chunk.shape[1]:]
    assert _rel(la, ref) <= LOGIT_TOL, f"extend after truncate: rel err {_rel(la, ref):.3e}"
    n = 12
    tok.copy_(first)
    eng.decode_many(tok, n - 1)
    dev = eng.read_history(1, n).t().long().cpu()
    o_tok, o_log = _oracle_greedy_from(w, cfg, full, n)
    nbad, ndec, ntot = _margin_ok_tokens(dev, o_tok, o_log, LOGIT_TOL * o_log.abs().max().item(), free_running=True)
    assert nbad == 0, f"{nbad} decisive greedy tokens differ ({ndec}/{ntot} decisive)"
    _check_pages(eng, [S + 10 + chunk.shape[1] + n - 1])


def test_extend_is_refused_when_it_cannot_run():
    from visualcla import _native as N
    cfg = O.tiny_config()
    m = _model(cfg, 0, 2, 48)
    eng = m._engine
    one = torch.ones(1, 4, dtype=torch.int64)
    with pytest.raises(N.NativeError, match="resident"):
        eng.extend(one)
    with pytest.raises(N.NativeError, match="resident"):
        eng.truncate([3])
    ids = torch.randint(3, 50, (2, 20))
    eng.prefill(ids.cuda(), N.TEXT_ONLY, None)
    with pytest.raises(N.NativeError, match="batch"):
        eng.extend(one)
    with pytest.raises(N.NativeError, match="max_seq"):
        eng.extend(torch.ones(2, 29, dtype=torch.int64))
    eng.extend(torch.ones(2, 28, dtype=torch.int64))             # exactly fills max_seq = 48
    eng.truncate([10, 40])
    eng.extend(torch.ones(2, 8, dtype=torch.int64))              # the bound follows the longest kept sequence
    eng.reset()
    with pytest.raises(N.NativeError, match="resident"):
        eng.extend(torch.ones(2, 2, dtype=torch.int64))
    # B * T over max_prefill_tokens, with max_seq leaving room
    import visualcla
    eng2 = visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=0, max_batch=2, max_seq=128, max_prefill_tokens=50)._engine
    eng2.prefill(ids.cuda(), N.TEXT_ONLY, None)
    with pytest.raises(N.NativeError, match="max_prefill_tokens"):
        eng2.extend(torch.ones(2, 26, dtype=torch.int64))
    eng2.extend(torch.ones(2, 25, dtype=torch.int64))


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. 7B widths
# ---------------------------------------------------------------------------------------------------------------------------------
def test_two_turn_conversation_at_7b_widths():
    """configs[0] widths, 8 of the 32 LLaMA layers: turn 2 passes turn 1's cache handle; its first-step logits equal the oracle's
    full forward of the turn-2 prompt and the greedy tokens follow the oracle wherever decisive."""
    import types
    cfg = O.PathConfig(t_layers=8)
    m = _model(cfg, 0, 1, 512)
    eng = m._engine
    s0, s1, _, s3 = O.special_ids(cfg)
    m.image_at_head = False
    m.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
    px, _ = O.make_inputs(cfg, 1, 8, seed=77)
    g = torch.Generator().manual_seed(3)
    text = lambda n: torch.randint(3, cfg.t_vocab - 4, (1, n), generator=g)
    p1 = torch.cat([torch.tensor([[1, s0]]), torch.full((1, cfg.r_queries), s3), torch.tensor([[s1]]), text(30)], 1)
    kw = dict(do_sample=False, eos_token_id=None, pad_token_id=0)
    r1 = m.generate(input_ids=p1.cuda(), pixel_values=px.cuda(), max_new_tokens=8, return_dict_in_generate=True, **kw)
    p2 = torch.cat([p1, r1.sequences.cpu(), text(25)], 1)
    extends = []
    orig = eng.extend
    eng.extend = lambda *a, **k: (extends.append(1), orig(*a, **k))[1]
    r2 = m.generate(input_ids=p2.cuda(), pixel_values=px.cuda(), max_new_tokens=6, past_key_values=r1.past_key_values,
                    output_logits=True, return_dict_in_generate=True, **kw)
    assert extends, "turn 2 extends the cached conversation"
    w = {k: v.float() for k, v in m.state_dict().items()}
    o_tok, o_log = O.generate_greedy(w, cfg, p2, px, 6, image_at_head=False)
    err = _rel(r2.logits[0], o_log[:, 0])
    assert err <= LOGIT_TOL, f"turn-2 first-step logits rel err {err:.3e}"
    nbad, ndec, ntot = _margin_ok_tokens(r2.sequences, o_tok, o_log, LOGIT_TOL * o_log.abs().max().item(), free_running=True)
    assert nbad == 0, f"{nbad} decisive tokens differ ({ndec}/{ntot} decisive)"
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# 5. chat() with a real tokenizer
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def merged_dir(tmp_path_factory):
    import sentencepiece as spm
    import visualcla
    from transformers import CLIPImageProcessor, LlamaTokenizer
    root = tmp_path_factory.mktemp("merged_kv")
    tokdir = root / "tok"
    tokdir.mkdir()
    corpus = "\n".join(["the quick brown fox jumps over the lazy dog", "a picture of a cat sitting on a mat", "describe the image in detail please",
                        "what colour is the car", "图片里有什么", "请描述这张图片", "hello world this is a test of the tokenizer"] * 20)
    (tokdir / "corpus.txt").write_text(corpus)
    spm.SentencePieceTrainer.train(input=str(tokdir / "corpus.txt"), model_prefix=str(tokdir / "tokenizer"), vocab_size=400, model_type="bpe",
                                   character_coverage=1.0, bos_id=1, eos_id=2, unk_id=0, pad_id=-1, byte_fallback=True, minloglevel=2)
    tok = LlamaTokenizer.from_pretrained(str(tokdir))
    tok.add_special_tokens({"additional_special_tokens": ["<img>", "</img>", "<pad>", "<img_token>"]})
    cfg = O.PathConfig(**dict(O.tiny_config().to_dict(), t_vocab=len(tok)))
    model = visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=3, max_batch=1, max_seq=512)
    out = root / "visualcla-tiny"
    model.save_merged_pretrained(str(out))
    tok.save_pretrained(str(out))
    proc = CLIPImageProcessor(size={"shortest_edge": cfg.v_image}, crop_size={"height": cfg.v_image, "width": cfg.v_image})
    proc.save_pretrained(str(out))
    proc.save_pretrained(str(out / "vision_encoder"))
    model._engine.close()
    return str(out), cfg


def _image(seed=0):
    import numpy as np
    from PIL import Image
    rng = np.random.default_rng(seed)
    return Image.fromarray(rng.integers(0, 255, (50, 70, 3), dtype=np.uint8))


def test_chat_turns_reuse_the_cache(merged_dir):
    import visualcla
    from transformers import GenerationConfig
    from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG, encoding_text
    path, cfg = merged_dir
    load = dict(torch_dtype=torch.float16, default_device=None, device_map=None, load_in_8bit=False, max_batch=1, max_seq=512)
    m_r, tok, proc = visualcla.get_model_and_tokenizer_and_processor(visualcla_model=path, reuse_kv_cache=True, **load)
    m_n, _, _ = visualcla.get_model_and_tokenizer_and_processor(visualcla_model=path, **load)
    assert m_r.reuse_kv_cache and not m_n.reuse_kv_cache
    s2 = tok.convert_tokens_to_ids("<pad>")
    gc = GenerationConfig(do_sample=False, max_new_tokens=8, eos_token_id=None, pad_token_id=s2)
    img = _image()
    px = proc(img, return_tensors="pt").pixel_values
    w = {k: v.float() for k, v in m_n.state_dict().items()}
    captured = {}
    for name, m in (("r", m_r), ("n", m_n)):
        orig = m.generate

        def gen(*a, _orig=orig, _name=name, **k):
            r = _orig(*a, **k)
            captured[_name] = r.sequences if hasattr(r, "sequences") else r
            return r
        m.generate = gen
    e_r = m_r._engine
    n_vis = (m_n._engine.kernel_launches(reset=True), m_n._engine.vision_encode(px.cuda()), m_n._engine.kernel_launches(reset=True))[2]
    assert n_vis > 0
    history = []
    launches = []
    for turn, text in enumerate(["describe the image", "and the background?", "what colour is the car"]):
        before = copy.deepcopy(history)
        e_r.kernel_launches(reset=True)
        resp_r, _ = visualcla.chat(m_r, image=img, text=text, history=copy.deepcopy(before), generation_config=gc)
        launches.append(e_r.kernel_launches(reset=True))
        resp_n, history = visualcla.chat(m_n, image=img, text=text, history=history, generation_config=gc)
        ids = encoding_text(before, text, m_n.num_patch, tok).input_ids
        o_tok, o_log = O.generate_greedy(w, cfg, ids, px.float(), 8, image_at_head=False, forced_tokens=captured["n"].cpu())
        nbad, ndec, ntot = _margin_ok_tokens(captured["r"][:, :8], captured["n"][:, :8], o_log, LOGIT_TOL_TINY * o_log.abs().max().item(),
                                             free_running=True)
        assert nbad == 0, f"turn {turn}: {nbad} decisive tokens differ between reuse and a fresh prefill ({ndec}/{ntot} decisive)"
        if turn > 0:
            assert launches[turn] <= launches[0] - n_vis + 2, f"turn {turn} ran the vision tower again: {launches}"
    # the reference's default (sampling) config runs through the device sampler after an extend
    extends, samplers = [], []
    orig_extend, orig_set = e_r.extend, e_r.set_sampler
    e_r.extend = lambda *a, **k: (extends.append(1), orig_extend(*a, **k))[1]
    e_r.set_sampler = lambda spec: (samplers.append(spec), orig_set(spec))[1]
    dgc = copy.deepcopy(DEFAULT_GENERATION_CONFIG)
    dgc.max_new_tokens = 12
    resp, h4 = visualcla.chat(m_r, image=img, text="again", history=copy.deepcopy(history), generation_config=dgc)
    assert isinstance(resp, str) and extends and samplers and samplers[0] is not None
    # and one streamed turn (host loop with a stopping criterion) extends too
    extends.clear()
    out = list(visualcla.chat_in_stream(m_r, image=img, text="one more", history=h4, generation_config=gc))
    assert extends and all(isinstance(r, str) for r, _ in out)


class _EosAs:
    """The loaded tokenizer with another EOS id (what chat_in_stream stops listening at)."""

    def __init__(self, tok, eos):
        self._tok, self.eos_token_id = tok, eos

    def __getattr__(self, name):
        return getattr(self._tok, name)

    def __call__(self, *a, **k):
        return self._tok(*a, **k)


def test_streamed_turn_ending_on_eos_is_extended_by_the_next_turn(merged_dir):
    """A chat_in_stream turn whose reply ends on EOS: the consumer stops listening there, generation ends normally and keeps its
    cache handle, and the next turn extends the cache instead of running the vision tower and a full prefill.  With an all-zero
    lm_head every pick is id 0 (the first of equal logits), which plays EOS here."""
    import visualcla
    from transformers import GenerationConfig
    path, cfg = merged_dir
    m, tok, _ = visualcla.get_model_and_tokenizer_and_processor(visualcla_model=path, torch_dtype=torch.float16, default_device=None,
                                                               device_map=None, load_in_8bit=False, reuse_kv_cache=True, max_batch=1,
                                                               max_seq=512)
    eng = m._engine
    eng.load_weight("text_model.lm_head.weight", torch.zeros(cfg.t_vocab, cfg.t_hidden))
    m.tokenizer = _EosAs(tok, 0)
    gc = GenerationConfig(do_sample=False, max_new_tokens=8, eos_token_id=0, pad_token_id=tok.convert_tokens_to_ids("<pad>"))
    img = _image()
    history = []
    visualcla.chat(m, image=img, text="describe the image", history=history, generation_config=gc)
    assert m._chat_kv_cache.is_current(eng)
    out = list(visualcla.chat_in_stream(m, image=img, text="and the background?", history=history, generation_config=gc))
    assert out == [], "the reply's first id is EOS: nothing is streamed"
    assert m._chat_kv_cache.is_current(eng), "the streamed turn kept its cache handle"
    history.append({"type": "response", "value": ""})
    calls = []
    for name in ("vision_encode", "prefill", "extend"):
        orig = getattr(eng, name)
        setattr(eng, name, lambda *a, _o=orig, _n=name, **k: (calls.append(_n), _o(*a, **k))[1])
    visualcla.chat(m, image=img, text="what colour is the car", history=history, generation_config=gc)
    assert calls == ["extend"], calls
