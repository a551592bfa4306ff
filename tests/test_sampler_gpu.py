"""Device-side sampling stack (csrc/sampler.cu through the C ABI) against the processors HF's generate() builds for the reference's
DEFAULT_GENERATION_CONFIG (ref models/visualcla/modeling_utils.py:36-47): processed scores must have the identical kept set and
equal values; every drawn token must be the pick of the float64 restatement of the draw (oracle/sampler_oracle.py: Philox4x32-10
uniform, inverse CDF over the sorted kept set) -- bit for bit where the cumulative sums are exact integers, and outside the fp32
ambiguity window elsewhere; the draw frequencies and the deterministic corners are checked too."""
import os

import numpy as np
import pytest
import torch

import sampler_oracle as SO
import visualcla_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VAL_TOL = 2e-6


@pytest.fixture(scope="module")
def eng():
    import visualcla
    m = visualcla.VisualCLAModel.from_synthetic(O.tiny_config().to_dict(), seed=0, max_batch=2, max_seq=64)
    return m._engine


def _same_scores(got, want, what):
    got, want = got.float().cpu(), torch.as_tensor(np.asarray(want)).float()
    kg, kw = torch.isfinite(got), torch.isfinite(want)
    assert torch.equal(kg, kw), f"{what}: kept sets differ ({int(kg.sum())} vs {int(kw.sum())} finite entries)"
    err = (got[kg] - want[kw]).abs().max().item() if bool(kg.any()) else 0.0
    assert err <= VAL_TOL * max(1.0, want[kw].abs().max().item()), f"{what}: max abs diff {err:.3e}"


LIVE_KNOBS = ((1.1, 15, 0.5, 40, 0.9), (1.3, 4, 1.0, 1, 1.0), (1.0, 0, 0.7, 100, 0.5), (1.2, 2, 1.5, 1000, 0.95), (1.0, 0, 1.0, 5, 0.3))


@pytest.mark.parametrize("n_gram", [3, 15])
def test_chain_matches_hf_golden(eng, n_gram):
    g = np.load(os.path.join(ROOT, "tests", "golden", "samplers.npz"))
    logits, hist = torch.from_numpy(g["chain_logits"]), torch.from_numpy(g["chain_history"])
    S = eng.sampler_spec
    _, sc = eng.op_sample(logits, hist, S(do_sample=False, repetition_penalty=1.1))
    _same_scores(sc, g[f"n{n_gram}_rep"], "repetition penalty")
    tok, sc = eng.op_sample(logits, hist, S(do_sample=False, repetition_penalty=1.1, no_repeat_ngram_size=n_gram))
    _same_scores(sc, g[f"n{n_gram}_ngram"], "penalty + no-repeat-ngram")
    assert torch.equal(tok.cpu().long(), torch.from_numpy(g[f"n{n_gram}_ngram"]).argmax(-1)), "greedy over the processed scores"
    _, sc = eng.op_sample(logits, hist, S(do_sample=True, repetition_penalty=1.1, no_repeat_ngram_size=n_gram, temperature=0.5, top_k=40, top_p=1.0, seed=1))
    _same_scores(sc, g[f"n{n_gram}_topk"], "... + temperature + top-k")
    tok, sc = eng.op_sample(logits, hist, S(do_sample=True, repetition_penalty=1.1, no_repeat_ngram_size=n_gram, temperature=0.5, top_k=40, top_p=0.9, seed=1))
    _same_scores(sc, g[f"n{n_gram}_topp"], "full default chain")
    kept = torch.isfinite(torch.from_numpy(g[f"n{n_gram}_topp"]))
    assert bool(kept[torch.arange(4), tok.cpu().long()].all()), "the drawn token belongs to the kept set"
    if n_gram == 3:
        assert not bool(torch.isfinite(sc[0, hist[0, 4]])) and not bool(torch.isfinite(sc[0, hist[0, 12]])), "both continuations of the repeated bigram are banned"


def test_chain_matches_hf_live_at_model_vocab(eng):
    """Fresh random logits at the real vocabulary (49958), long histories with repeats, several knob settings, against transformers'
    own processors run here."""
    g = torch.Generator().manual_seed(5)
    V, B, L = 49958, 6, 300
    logits = torch.randn(B, V, generator=g) * 3.0
    hist = torch.randint(0, V, (B, L), generator=g)
    hist[:, 200:230] = hist[:, 20:50]                       # long repeats: n-gram bans fire for n <= 31
    hist[:, -14:] = hist[:, 20:34]                          # ... and the current suffix matches them
    for rp, ng, t, k, p in LIVE_KNOBS:
        x = _hf(logits, hist, rp=rp, ng=ng, t=t, k=k, p=p)
        tok, sc = eng.op_sample(logits, hist, eng.sampler_spec(do_sample=True, repetition_penalty=rp, no_repeat_ngram_size=ng, temperature=t, top_k=k, top_p=p, seed=3))
        _same_scores(sc, x, f"rp={rp} ngram={ng} T={t} k={k} p={p}")
        assert bool(torch.isfinite(x)[torch.arange(B), tok.cpu().long()].all())


def _hf(logits, hist, rp=1.0, ng=0, t=1.0, k=0, p=1.0, min_new=0, eos=()):
    """transformers' processors in the kernel's order (k = 0: no top-k, i.e. the greedy path's full processed row)"""
    from transformers.generation import logits_process as lp
    h = torch.zeros(logits.shape[0], 0, dtype=torch.long) if hist is None else hist.long()
    x = logits.clone()
    if rp != 1.0:
        x = lp.RepetitionPenaltyLogitsProcessor(penalty=rp)(h, x)
    if ng:
        x = lp.NoRepeatNGramLogitsProcessor(ng)(h, x)
    if eos and min_new:
        x = lp.MinNewTokensLengthLogitsProcessor(prompt_length_to_skip=0, min_new_tokens=min_new, eos_token_id=list(eos))(h, x)
    if t != 1.0:
        x = lp.TemperatureLogitsWarper(t)(h, x)
    if k:
        x = lp.TopKLogitsWarper(top_k=k, min_tokens_to_keep=1)(h, x)
    if p < 1.0:
        x = lp.TopPLogitsWarper(top_p=p, min_tokens_to_keep=1)(h, x)
    return x


class DrawStats:
    """Counts over checked draws: ambiguous ones (u * tot within the fp32 window of a boundary), picks above rank 0, and the largest
    distance to a boundary seen on a draw where the kernel took the neighbouring rank."""
    def __init__(self):
        self.n = self.ambiguous = self.above_top = self.mismatch = 0
        self.worst = 0.0

    def add(self, got, want, ambiguous, accept, rank, margin, what):
        self.n += 1
        self.ambiguous += ambiguous
        self.above_top += rank > 0
        if ambiguous and got in accept:
            if got != want:
                self.mismatch += 1
                self.worst = max(self.worst, margin)
            return
        assert got == want, f"{what}: the kernel picked {got}, the reference draw is {want} (rank {rank}, acceptable {accept})"

    def line(self):
        return (f"{self.n} draws, {self.ambiguous} ambiguous ({self.ambiguous / max(1, self.n):.2%}), {self.above_top} at rank > 0, "
                f"{self.mismatch} took the neighbour (largest distance {self.worst:.2e} of tot)")


def check_draws(tok, scores, seed, L, stats, what=""):
    """Each row's pick must be the float64 draw over the kernel's own processed scores (kept set and values), with u = uniform(seed,
    L, row); within the ambiguity window either neighbouring rank is accepted."""
    tok, scores = tok.cpu().long().tolist(), scores.cpu().numpy()
    u = SO.uniform(seed, L, np.arange(len(tok)))
    for b, t in enumerate(tok):
        d = SO.draw(scores[b], float(u[b]))
        stats.add(t, d.token, d.ambiguous, d.accept, d.rank, d.margin, f"{what} row {b} L={L} seed={seed:#x} u={u[b]!r}")


PHILOX_SEEDS = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 62 - 1, (1 << 63) | 0x0123456789ABCDEF]


def test_philox_draw_bit_exact(eng):
    """1024 equal logits at scattered ids per row, all others far below, top_k = 1024, T = 1, no top-p: tot = 1024 and every partial
    sum is an exact integer in fp32, so the kernel must pick rank x0 >> 22 of the tie (ranked by index) -- 10 bits of Philox output
    per draw, compared exactly.  Sequence counters 0..63, step counters up to the high half-word, both key words."""
    V = 3000
    g = torch.Generator().manual_seed(17)
    for B in (1, 7, 64):
        ids = torch.stack([torch.randperm(V, generator=g)[:1024].sort().values for _ in range(B)])
        logits = torch.full((B, V), -40.0).scatter_(1, ids, 0.75)
        for L in (0, 1, 2, 1000, 65537):
            hist = torch.zeros(B, L, dtype=torch.int32, device="cuda") if L else None   # penalties off: never read
            for seed in PHILOX_SEEDS:
                tok, _ = eng.op_sample(logits, hist, eng.sampler_spec(do_sample=True, top_k=1024, seed=seed), return_scores=False)
                rank = torch.from_numpy((SO.word0(seed, L, np.arange(B)) >> 22).astype(np.int64))
                want = ids[torch.arange(B), rank]
                assert torch.equal(tok.cpu().long(), want), f"B={B} L={L} seed={seed:#x}: {tok.cpu().tolist()} vs {want.tolist()}"


def test_default_chain_draws_match_reference_at_model_vocab(eng):
    """The knob settings of test_chain_matches_hf_live_at_model_vocab, 40 fresh logit sets and seeds each (200 x 6 draws): every pick
    is the float64 draw over the kernel's processed scores with the Philox uniform of (seed, L, row)."""
    V, B, L = 49958, 6, 300
    stats = DrawStats()
    for i, (rp, ng, t, k, p) in enumerate(LIVE_KNOBS):
        for s in range(40):
            g = torch.Generator().manual_seed(100 * i + s)
            logits = torch.randn(B, V, generator=g) * 3.0
            hist = torch.randint(0, V, (B, L), generator=g)
            hist[:, 200:230] = hist[:, 20:50]
            hist[:, -14:] = hist[:, 20:34]
            seed = (0x9E3779B97F4A7C15 * (40 * i + s + 1)) & (2 ** 64 - 1)
            spec = eng.sampler_spec(do_sample=True, repetition_penalty=rp, no_repeat_ngram_size=ng, temperature=t, top_k=k, top_p=p, seed=seed)
            tok, sc = eng.op_sample(logits, hist, spec)
            check_draws(tok, sc, seed, L, stats, f"rp={rp} ngram={ng} T={t} k={k} p={p}")
    print(f"[sampler draws, model vocabulary] {stats.line()}")
    assert stats.ambiguous <= 0.05 * stats.n, stats.line()
    assert stats.above_top >= 0.25 * stats.n, stats.line()


def test_kept_set_edges_match_hf(eng):
    """Kept sets at the edges of top-k, min_new_tokens and no-repeat-ngram, against transformers' processors; the draws over them
    against the float64 draw."""
    stats = DrawStats()
    g = torch.Generator().manual_seed(23)

    def run(logits, hist, what, seed=5, **kw):
        spec = eng.sampler_spec(do_sample=kw.get("k", 0) > 0, repetition_penalty=kw.get("rp", 1.0), no_repeat_ngram_size=kw.get("ng", 0),
                                temperature=kw.get("t", 1.0), top_k=kw.get("k", 0), top_p=kw.get("p", 1.0), min_new_tokens=kw.get("min_new", 0),
                                eos_token_id=kw.get("eos", ()), seed=seed)
        tok, sc = eng.op_sample(logits, hist, spec)
        _same_scores(sc, _hf(logits, hist, **kw), what)
        if kw.get("k", 0) > 0:
            check_draws(tok, sc, seed, 0 if hist is None else hist.shape[1], stats, what)
        return tok.cpu(), sc.cpu()

    # ties straddling the k-th value: every tie is kept (k + ties), as HF's threshold comparison does
    V, B, k = 2000, 4, 40
    logits = torch.randn(B, V, generator=g)
    order = logits.argsort(1, descending=True)
    for b in range(B):
        lo, hi = 30 + 2 * b, 45 + b                        # ranks lo .. hi-1 tie, the k-th (rank 39) among them
        logits[b, order[b, lo:hi]] = float(logits[b, order[b, lo]])
    _, sc = run(logits, None, "ties at the k-th value", k=k, t=0.5)
    assert torch.isfinite(sc).sum(1).tolist() == [45 + b for b in range(B)]
    top = logits.max(1, keepdim=True).values
    tied_max = torch.where(torch.arange(V)[None, :] % 500 == 3, top + 1.0, logits)       # 4 equal maxima, top_k = 1
    _, sc = run(tied_max, None, "top_k = 1 with 4 tied maxima", k=1)
    assert torch.isfinite(sc).sum(1).tolist() == [4] * B
    # top_k at the top of the kernel's range, at the model vocabulary, with and without top-p
    logits = torch.randn(B, 49958, generator=g) * 3.0
    for p in (1.0, 0.95):
        _, sc = run(logits, None, f"top_k = 1024, top_p = {p}", k=1024, t=1.5, p=p, seed=9)
    # top_k >= V
    logits = torch.randn(B, 7, generator=g)
    for kk in (7, 8, 1024):
        _, sc = run(logits, None, f"top_k = {kk} at V = 7", k=kk, seed=kk)
        assert bool(torch.isfinite(sc).all())
    # min_new_tokens: four EOS ids (the four largest logits) masked while L < min_new, no longer at L = min_new
    V = 2000
    logits = torch.randn(B, V, generator=g)
    eos = (11, 700, 1500, 1999)
    logits[:, list(eos)] = 6.0
    for L in (3, 4, 5):
        hist = torch.randint(0, V, (B, L), generator=g)
        for kk in (0, 50):
            _, sc = run(logits, hist, f"min_new_tokens 4, L {L}, k {kk}", k=kk, min_new=4, eos=eos, seed=L)
            assert bool(torch.isfinite(sc[:, list(eos)]).all()) == (L >= 4), f"EOS ids at L={L}"
    # no-repeat-ngram: a constant history can first be banned at L = n (the n-gram t..t exists); at L = n - 1 nothing is banned
    logits = torch.randn(B, V, generator=g)
    for n in (2, 3, 15):
        for L in (n - 1, n):
            hist = torch.full((B, L), 123)
            for kk in (0, 200):
                _, sc = run(logits, hist, f"ngram {n}, L {L}, k {kk}", k=kk, ng=n, rp=1.1, seed=n)
                if kk == 0:
                    assert bool(torch.isfinite(sc[:, 123]).all()) == (L < n), f"ngram {n} at L={L}"
    print(f"[sampler draws, kept-set edges] {stats.line()}")


def test_draw_distribution_and_determinism(eng):
    V, B = 1000, 64
    base = torch.full((V,), -20.0)
    probs = torch.tensor([0.4, 0.25, 0.15, 0.1, 0.06, 0.04])
    ids = torch.tensor([7, 300, 41, 999, 0, 512])
    base[ids] = probs.log()
    logits = base.repeat(B, 1)
    counts = torch.zeros(V)
    n_calls = 60
    for s in range(n_calls):
        tok, _ = eng.op_sample(logits, None, eng.sampler_spec(do_sample=True, top_k=6, seed=1000 + s), return_scores=False)
        counts += torch.bincount(tok.cpu().long(), minlength=V).float()
    n = n_calls * B
    assert counts.sum() == n and counts[ids].sum() == n, "only the top-k tokens are ever drawn"
    freq = counts[ids] / n
    sigma = (probs * (1 - probs) / n).sqrt()
    assert bool(((freq - probs).abs() < 5 * sigma).all()), f"draw frequencies {freq.tolist()} vs probabilities {probs.tolist()}"
    a, _ = eng.op_sample(logits, None, eng.sampler_spec(do_sample=True, top_k=6, seed=42), return_scores=False)
    b, _ = eng.op_sample(logits, None, eng.sampler_spec(do_sample=True, top_k=6, seed=42), return_scores=False)
    c, _ = eng.op_sample(logits, None, eng.sampler_spec(do_sample=True, top_k=6, seed=43), return_scores=False)
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert len(set(a.tolist())) > 1, "sequences draw independently (counter = (step, sequence))"
    one, _ = eng.op_sample(torch.randn(5, V), None, eng.sampler_spec(do_sample=True, top_k=1, temperature=0.3, top_p=0.2, seed=9), return_scores=False)
    assert one.shape == (5,)


def _model():
    import visualcla
    cfg = O.PathConfig(v_layers=1, r_layers=1, t_hidden=512, t_heads=4, t_ffn=1408, t_layers=2, t_vocab=2003)
    m = visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=9, max_batch=4, max_seq=200)
    px, ids = O.make_inputs(cfg, 3, 20, seed=5)
    return m, ids.cuda(), px.cuda()


def test_generate_device_path_equals_host_processor_path(monkeypatch):
    """Deterministic knobs (greedy + repetition penalty + n-gram ban, EOS with padding, top_k=1 'sampling'): the in-graph device
    sampler must produce exactly the tokens of the per-step host path that runs HF's processors on the returned logits."""
    m, ids, px = _model()
    kw = dict(input_ids=ids, pixel_values=px, max_new_tokens=40, pad_token_id=0)
    plain = m.generate(do_sample=False, eos_token_id=None, **kw)
    launches0 = m._engine.kernel_launches(reset=True)
    cases = [dict(do_sample=False, eos_token_id=None, repetition_penalty=1.3, no_repeat_ngram_size=2),
             dict(do_sample=True, top_k=1, temperature=0.7, top_p=0.9, eos_token_id=None, repetition_penalty=1.1, no_repeat_ngram_size=15),
             dict(do_sample=False, eos_token_id=int(plain[0, 5]), repetition_penalty=1.0),
             dict(do_sample=False, eos_token_id=[int(plain[0, 3]), int(plain[1, 9]), int(plain[2, 20])], min_new_tokens=6, repetition_penalty=1.2)]
    for c in cases:
        monkeypatch.delenv("VCLA_HOST_SAMPLER", raising=False)
        dev = m.generate(**c, **kw)
        monkeypatch.setenv("VCLA_HOST_SAMPLER", "1")
        host = m.generate(**c, **kw)
        assert dev.shape == host.shape and torch.equal(dev, host), f"{c}: device {dev.tolist()} vs host {host.tolist()}"
    monkeypatch.delenv("VCLA_HOST_SAMPLER", raising=False)
    assert not torch.equal(m.generate(do_sample=False, eos_token_id=None, repetition_penalty=1.3, no_repeat_ngram_size=2, **kw), plain)
    assert launches0 > 0


def test_generate_default_chat_config_on_device():
    """The reference's DEFAULT_GENERATION_CONFIG runs as graph replays with the sampler inside; seeded runs repeat, the tokens
    respect the no-repeat-ngram constraint, and Mirostat / TFS (host path) still work."""
    from visualcla.modeling_utils import DEFAULT_GENERATION_CONFIG
    m, ids, px = _model()
    gc = DEFAULT_GENERATION_CONFIG
    kw = dict(input_ids=ids, pixel_values=px, generation_config=gc, max_new_tokens=48, eos_token_id=None, pad_token_id=0)
    torch.manual_seed(1)
    a = m.generate(**kw)
    torch.manual_seed(1)
    b = m.generate(**kw)
    torch.manual_seed(2)
    c = m.generate(**kw)
    assert a.shape == (3, 48) and torch.equal(a, b) and not torch.equal(a, c)
    small = m.generate(input_ids=ids, pixel_values=px, do_sample=True, top_k=3, temperature=2.0, no_repeat_ngram_size=2, max_new_tokens=60,
                       eos_token_id=None, pad_token_id=0)
    for row in small.tolist():
        bigrams = list(zip(row, row[1:]))
        assert len(bigrams) == len(set(bigrams)), "no bigram may repeat with no_repeat_ngram_size=2"
    mir = m.generate(input_ids=ids[:1], pixel_values=px[:1], do_sample=True, temperature=0.8, top_k=40, top_p=0.9, mirostat_mode=2, mirostat_tau=5,
                     mirostat_eta=0.1, max_new_tokens=6, eos_token_id=None, pad_token_id=0)
    tfs = m.generate(input_ids=ids, pixel_values=px, do_sample=True, temperature=0.8, top_k=40, tfs=0.9, max_new_tokens=6, eos_token_id=None, pad_token_id=0)
    assert mir.shape == (1, 6) and tfs.shape == (3, 6)
