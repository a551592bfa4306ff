"""Beam search on the device: the selection kernels against the oracle's step, the KV cache shared between beams (copy-on-write
pages), the page accounting, end-to-end generate(num_beams=...) against the reference's fixtures and the oracle, determinism, and
that greedy / sampled decode steps launch exactly the kernels they launched before beam search existed."""
import json
import os

import numpy as np
import pytest
import torch

import beam_oracle as BO
import visualcla_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_beams.npz")


def _engine(cfg, max_batch=8, max_seq=96, page_tokens=64, seed=0):
    from visualcla.engine import Engine
    eng = Engine(cfg.to_dict(), max_batch=max_batch, max_seq=max_seq, page_tokens=page_tokens)
    eng.init_synthetic(seed)
    return eng


def _model(cfg, max_batch=8, max_seq=96, page_tokens=64, seed=0):
    import visualcla
    m = visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=seed, max_batch=max_batch, max_seq=max_seq)
    if page_tokens != 64:
        m._engine = _engine(cfg, max_batch, max_seq, page_tokens, seed)
    return m


# ---- operator ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,n_eos,procs", [(2, 0, False), (4, 1, True), (4, 4, False), (16, 2, True)])
def test_op_beam_step_matches_oracle(K, n_eos, procs):
    """The two selection kernels on seeded random logits, step by step up to and including the max-length step, against the oracle's
    step on the same logits and histories: parents, tokens, candidates, hits and the hypothesis store identical, scores within a
    relative 1e-6."""
    from visualcla.engine import Engine
    torch.manual_seed(100 + K + n_eos)
    cfg = O.tiny_config()
    eng = _engine(cfg, max_batch=64, max_seq=32)
    B, V, max_new = (4 if K * 4 <= 64 else 2), 1003, 7
    eos = list(range(5, 5 + n_eos))
    kw = dict(repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=2) if procs else {}
    spec = Engine.beam_spec(K, max_new, length_penalty=0.7, early_stopping=False, eos_token_id=eos, **kw)
    st = BO.BeamState(B, K, max_new)
    dev_state = {}
    for t in range(max_new):
        rows = B if t == 0 else B * K
        logits = torch.randn(rows, V) * 3.0
        if eos:
            logits[:, eos] += 3.0                  # EOS among the candidates: hypotheses finish early
        hist = st.hist.reshape(B * K, t)
        r = BO.beam_step(st, logits, t, eos, 0.7, False, **kw)
        d = eng.op_beam_step(logits, hist if t else None, t, spec, dev_state)
        R = 1 if t == 0 else K
        par = d["parent"].cpu().long().view(B, K) - torch.arange(B)[:, None] * R
        assert torch.equal(par, r["parent"]), f"step {t}"
        assert torch.equal(d["token"].cpu().long().view(B, K), r["token"]), f"step {t}"
        cand = d["cand"].cpu().long()
        assert torch.equal(cand[..., 0], r["cand"]) and torch.equal(cand[..., 1].bool(), r["hit"]), f"step {t}"
        assert torch.equal(dev_state["lens"].cpu().long(), st.lens) and torch.equal(dev_state["fin"].cpu().bool(), st.fin), f"step {t}"
        torch.testing.assert_close(dev_state["scores"].cpu(), st.scores, rtol=1e-6, atol=0)
        torch.testing.assert_close(dev_state["run"].cpu().view(B, K), st.run, rtol=1e-6, atol=0)
        tok = dev_state["tokens"].cpu().long()
        for b in range(B):
            for k in range(K):
                if st.fin[b, k]:
                    n = int(st.lens[b, k])
                    assert torch.equal(tok[b, k, :n], st.tokens[b, k, :n]), f"step {t} item {b} hyp {k}"
        items = dev_state["items"].cpu()
        assert torch.equal(items[:, 0].bool(), st.unsat) and torch.equal(items[:, 1].bool(), st.done), f"step {t}"


# ---- cache correctness under sharing + page accounting -------------------------------------------------------------------------
@pytest.mark.parametrize("page_tokens", [8, 64])
def test_beams_share_pages_copy_on_write(page_tokens):
    """After every step each running beam's logits equal a fresh prefill of prompt + that beam's tokens (the beams read their
    parents' pages and their own copies of the page written next), no page at a write position belongs to two beams, and free pages +
    distinct referenced pages = the pool.  A shuffled page hand-out order gives identical tokens; vcla_reset frees every page."""
    cfg = O.PathConfig(v_layers=1, r_layers=1, t_hidden=512, t_heads=4, t_ffn=1408, t_layers=2, t_vocab=2003)
    B, K, T, steps = 2, 4, 13, 12
    eng = _engine(cfg, max_batch=8, max_seq=64, page_tokens=page_tokens, seed=3)
    ref = _engine(cfg, max_batch=8, max_seq=64, page_tokens=page_tokens, seed=3)
    _, ids = O.make_inputs(cfg, B, T, seed=77)
    pps, total, pt = eng.kv_geometry()

    def run(check):
        spec = eng.beam_spec(K, steps + 1, eos_token_id=())
        eng.set_beam(spec)
        try:
            _, first, _ = eng.prefill(ids, 0, None, last_logits=False)
            tok = eng.token_buffer(B * K)
            tok.copy_(first)
            logits = torch.empty(B * K, eng.vocab, dtype=torch.float32, device=eng.device)
            for s in range(1, steps + 1):
                hist = eng.read_history(B * K, s).t().cpu().long()          # each row's tokens, the last one is fed now
                eng.decode_step(tok, tok, logits, use_graph=(s % 2 == 0))
                if not check:
                    continue
                table, owned, free, exhausted = eng.kv_pages()
                assert exhausted == 0
                L = T + s                                                  # cached tokens per row; the next one is written at L
                pw = L // pt
                at_write = [int(table[j, pw]) for j in range(B * K)]
                assert len(set(at_write)) == B * K, f"step {s}: a write page is shared {at_write}"
                refd = set()
                for j in range(B * K):
                    assert int(owned[j]) == pw + 1
                    refd |= set(table[j, : int(owned[j])].tolist())
                assert free + len(refd) == total, f"step {s}: {free} free + {len(refd)} referenced != {total}"
                want, _, _ = ref.prefill(torch.cat([ids.repeat_interleave(K, 0), hist], 1), 0, None)
                scale = float(want.abs().max())
                err = float((logits - want).abs().max()) / scale
                assert err < 1.5e-2, f"step {s}: beam logits differ from a fresh prefill by {err:.3e} (relative)"
            hyp = eng.read_beams(B)
        finally:
            eng.set_beam(None)
        return hyp

    base = run(True)
    eng.reset()
    assert eng.kv_pages()[2] == total
    eng.kv_debug_shuffle(5)
    again = run(False)
    assert torch.equal(again[0], base[0]) and torch.equal(again[1], base[1])
    assert int(eng.kv_pages()[2]) < total
    eng.reset()
    assert eng.kv_pages()[2] == total


# ---- end to end ----------------------------------------------------------------------------------------------------------------
def _case_kwargs(c):
    kw = dict(num_beams=c["num_beams"], do_sample=False, max_new_tokens=c["max_new_tokens"], pad_token_id=c["pad_token_id"],
              eos_token_id=(c["eos"] or None))
    for k in ("early_stopping", "length_penalty", "num_return_sequences", "repetition_penalty", "no_repeat_ngram_size"):
        if k in c:
            kw[k] = c[k]
    return kw


def _oracle_kwargs(c):
    return dict(eos_token_id=c["eos"], pad_token_id=c["pad_token_id"], length_penalty=c.get("length_penalty", 1.0),
                early_stopping=c.get("early_stopping", False), num_return_sequences=c.get("num_return_sequences", 1),
                repetition_penalty=c.get("repetition_penalty", 1.0), no_repeat_ngram_size=c.get("no_repeat_ngram_size", 0))


def _check_against_oracle(w, cfg, got, ids, px, at_head, pads, K, n_new, okw, tol, ref_seqs=None):
    """Equal sequences wherever every step's margin between candidates M and M+1 exceeds 2 x tol; otherwise the device's best
    hypothesis, re-scored teacher-forced by the oracle, is within tol of the oracle's best score."""
    seqs, scores, steps = BO.beam_search(w, cfg, ids, px, K, n_new, image_at_head=at_head, left_pad=pads, **okw)
    if ref_seqs is not None:
        assert torch.equal(seqs, ref_seqs), "the oracle no longer reproduces the reference fixture"
    decisive = all(bool((r["margin"] > 2 * tol).all()) for r in steps)
    if decisive:
        assert got.shape == seqs.shape and torch.equal(got, seqs)
        return "equal"
    nrs = okw.get("num_return_sequences", 1)
    eos = okw.get("eos_token_id", ())
    for b in range(ids.shape[0]):
        row = got[b * nrs].tolist()
        n = next((i + 1 for i, v in enumerate(row) if v in list(eos)), len(row))   # a hypothesis ends at its first EOS
        best = torch.tensor(row[:n]).unsqueeze(0)
        rs = BO.beam_rescore(w, cfg, ids[b:b + 1], None if px is None else px[b:b + 1], best, image_at_head=at_head,
                            left_pad=None if pads is None else pads[b:b + 1], length_penalty=okw.get("length_penalty", 1.0))
        if okw.get("repetition_penalty", 1.0) == 1.0 and not okw.get("no_repeat_ngram_size"):
            assert abs(float(rs[0]) - float(scores[b * nrs])) <= tol, f"item {b}: re-scored {float(rs[0])} vs oracle {float(scores[b * nrs])}"
    return "rescored"


def test_tiny_beams_against_reference_fixture():
    z = np.load(GOLDEN)
    cfg = O.tiny_config()
    w = O.make_weights(cfg, int(z["seed"]))
    m = _model(cfg, max_batch=8, max_seq=64)
    s0, s1, _, s3 = O.special_ids(cfg)
    import types
    m.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
    px = torch.from_numpy(z["pixel_values"])
    head_ids = torch.from_numpy(z["k4_input_ids"])
    tol = 1.5e-2 * float(O.forward_logits(w, cfg, head_ids, px)[:, -1].abs().max())
    outcomes = {}
    for c in json.loads(str(z["cases"])):
        n = c["name"]
        ids = torch.from_numpy(z[f"{n}_input_ids"])
        mask = torch.from_numpy(z[f"{n}_attention_mask"])
        at_head = c["layout"] in ("head", "text")
        m.image_at_head = at_head
        p = None if c["layout"] == "text" else px
        got = m.generate(input_ids=ids.cuda(), pixel_values=None if p is None else p.cuda(), attention_mask=mask.cuda(), **_case_kwargs(c)).cpu()
        pads = (mask == 0).sum(1) if bool((mask == 0).any()) else None
        ref = torch.from_numpy(z[f"{n}_sequences"])
        outcomes[n] = _check_against_oracle(w, cfg, got, ids, p, at_head, pads, c["num_beams"], c["max_new_tokens"], _oracle_kwargs(c),
                                            tol=tol, ref_seqs=ref)
    print("[beams] tiny fixture:", outcomes)


def test_wide_config_against_oracle_and_deterministic():
    cfg = O.PathConfig(v_layers=1, r_layers=1, t_hidden=1024, t_heads=8, t_ffn=2816, t_layers=2, t_vocab=4001)
    m = _model(cfg, max_batch=8, max_seq=96, seed=5)
    w = O.make_weights(cfg, 5)
    px, ids = O.make_inputs(cfg, 2, 11, seed=9)
    kw = dict(num_beams=4, do_sample=False, max_new_tokens=12, eos_token_id=[int(7)], pad_token_id=0, length_penalty=1.3)
    got = m.generate(input_ids=ids.cuda(), pixel_values=px.cuda(), **kw).cpu()
    again = m.generate(input_ids=ids.cuda(), pixel_values=px.cuda(), **kw).cpu()
    assert torch.equal(got, again), "two runs differ"
    logits = O.forward_logits(w, cfg, ids, px)[:, -1]
    tol = 1.5e-2 * float(logits.abs().max())
    okw = dict(eos_token_id=[7], pad_token_id=0, length_penalty=1.3)
    print("[beams] 1024-wide:", _check_against_oracle(w, cfg, got, ids, px, True, None, 4, 12, okw, tol))


# ---- unchanged paths -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [4, 40])
def test_greedy_and_sampled_steps_launch_what_they_launched_before(B):
    """A greedy or sampled decode step launches 5 kernels per layer + 5 (batches <= 32) or 8 per layer + 6 (33..64), as before beam
    search existed; a beam step adds the beam-step kernel and the reorder + page copy."""
    cfg = O.PathConfig(v_layers=1, r_layers=1, t_hidden=256, t_heads=2, t_ffn=448, t_layers=2, t_vocab=1003)
    eng = _engine(cfg, max_batch=64, max_seq=32)
    ids = torch.randint(0, 1000, (B, 5))
    want = 5 * cfg.t_layers + 5 if B <= 32 else 8 * cfg.t_layers + 6
    tok = eng.token_buffer(B)
    _, first, _ = eng.prefill(ids, 0, None)
    tok.copy_(first)
    eng.kernel_launches(reset=True)
    eng.decode_step(tok, tok, use_graph=False)
    assert eng.kernel_launches(reset=True) == want
    eng.set_sampler(eng.sampler_spec(do_sample=True, top_k=5, temperature=0.7, seed=1))
    try:
        eng.prefill(ids, 0, None)
        eng.kernel_launches(reset=True)
        eng.decode_step(tok, tok, use_graph=False)
        assert eng.kernel_launches(reset=True) == want
    finally:
        eng.set_sampler(None)
    eng.set_beam(eng.beam_spec(4, 4))
    try:
        _, first, _ = eng.prefill(ids[: B // 4], 0, None)
        bt = eng.token_buffer(B)
        bt.copy_(first)
        eng.kernel_launches(reset=True)
        eng.decode_step(bt, bt, use_graph=False)
        assert eng.kernel_launches(reset=True) == want + 3
    finally:
        eng.set_beam(None)


def test_beam_refusals_on_the_device():
    from visualcla import _native as N
    cfg = O.tiny_config()
    eng = _engine(cfg, max_batch=8, max_seq=32)
    with pytest.raises(N.NativeError, match="exceed"):
        eng.set_beam(eng.beam_spec(16, 4))                   # 16 rows > max_batch 8
    eng.set_beam(eng.beam_spec(4, 8))
    try:
        with pytest.raises(N.NativeError, match="exceed"):
            eng.prefill(torch.randint(0, 900, (3, 5)), 0, None)   # 12 rows > 8
        with pytest.raises(N.NativeError, match="max_seq"):
            eng.prefill(torch.randint(0, 900, (1, 30)), 0, None)  # 30 + 8 > 32
    finally:
        eng.set_beam(None)


@pytest.mark.skipif(os.environ.get("VCLA_SKIP_7B") == "1", reason="VCLA_SKIP_7B=1")
def test_7b_widths_against_oracle():
    """7B widths, 8 LLaMA layers, B=2 text prompts, K=4, 64 new tokens: equal to the fp32 oracle's beam search where every step is
    decisive, else the device's best hypothesis re-scored by the oracle is within the logit tolerance of the oracle's best score."""
    cfg = O.PathConfig(t_layers=8)
    m = _model(cfg, max_batch=8, max_seq=160, seed=0)
    w = {k: v.float() for k, v in m.state_dict().items()}
    _, ids = O.make_inputs(cfg, 2, 24, seed=3)
    got = m.generate(input_ids=ids.cuda(), num_beams=4, do_sample=False, max_new_tokens=64, eos_token_id=None, pad_token_id=0).cpu()
    assert got.shape == (2, 64)
    tol = 1.5e-2 * float(O.forward_logits(w, cfg, ids, None)[:, -1].abs().max())
    print("[beams] 7B widths:", _check_against_oracle(w, cfg, got, ids, None, True, None, 4, 64, dict(eos_token_id=[], pad_token_id=0), tol))
    m._engine.close()
