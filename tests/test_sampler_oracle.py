"""The host restatement of the device sampler's draw (oracle/sampler_oracle.py) pinned on its own, so that it cannot be wrong behind a
skipped GPU test: Random123's Philox4x32-10 known-answer vectors, the 24-bit uniform, hand-worked inverse-CDF draws (ties, the
last-rank fallback, the ambiguity window) and the top-p keep counts."""
import numpy as np
import pytest

import sampler_oracle as S

NEG = -np.inf


@pytest.mark.parametrize("ctr, key, want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(x) for x in S.philox4x32_10(ctr, key)) == want


def test_philox_broadcasts_like_scalar_calls():
    steps, seqs = np.arange(5)[:, None], np.arange(3)[None, :]
    got = S.philox4x32_10((steps, seqs, 0, 0), (7, 1 << 31))
    assert got.shape == (4, 5, 3) and got.dtype == np.uint32
    for s in range(5):
        for b in range(3):
            assert tuple(got[:, s, b]) == tuple(S.philox4x32_10((s, b, 0, 0), (7, 1 << 31)))


def test_key_words_and_counter_words_are_distinct_inputs():
    seed = (0x89ABCDEF << 32) | 0x01234567
    assert S.key_words(seed) == (0x01234567, 0x89ABCDEF)
    x = int(S.word0(seed, 3, 5))
    assert x == int(S.philox4x32_10((3, 5, 0, 0), (0x01234567, 0x89ABCDEF))[0])
    assert x != int(S.word0(seed, 5, 3)), "step and sequence are different counter words"
    assert x != int(S.word0((0x01234567 << 32) | 0x89ABCDEF, 3, 5)), "the two seed halves are different key words"
    assert int(S.word0(seed, 1 << 16, 0)) != int(S.word0(seed, 0, 0)), "the step's high half-word reaches the counter"


def test_uniform_range_and_resolution():
    steps = np.arange(4096)[:, None]
    seqs = np.arange(64)[None, :]
    u = S.uniform(12345, steps, seqs)
    assert u.shape == (4096, 64) and float(u.min()) >= 0.0 and float(u.max()) < 1.0
    ints = u * 2.0 ** 24
    assert np.array_equal(ints, np.floor(ints)), "u is a 24-bit integer times 2**-24"
    assert int(np.bitwise_or.reduce(ints.astype(np.int64).ravel())) == (1 << 24) - 1, "all 24 bits are used"
    assert abs(float(u.mean()) - 0.5) < 0.01
    x0 = S.word0(12345, 17, 9)
    assert S.uniform(12345, 17, 9) == float(int(x0) >> 8) / 2 ** 24
    assert S.uniform(0, 0, 0) == float(0x6627E8D5 >> 8) / 2 ** 24


def test_draw_single_kept_token():
    row = np.full(10, NEG)
    row[6] = -3.0
    for u in (0.0, 0.5, 1 - 2 ** -24):
        d = S.draw(row, u)
        assert (d.token, d.rank, d.ambiguous, d.accept) == (6, 0, False, (6,))


def test_draw_two_equal_tokens_split_at_one_half():
    row = np.full(8, NEG)
    row[[2, 5]] = 1.5
    below, above = 0.5 - 2 * S.EPS, 0.5 + 2 * S.EPS
    assert (S.draw(row, below).token, S.draw(row, below).rank) == (2, 0)
    assert (S.draw(row, above).token, S.draw(row, above).rank) == (5, 1)
    assert not S.draw(row, below).ambiguous and not S.draw(row, above).ambiguous
    # exactly at the boundary: e_0 = 1 is not > u * tot = 1, so the pick is rank 1
    assert S.draw(row, 0.5).token == 5 and S.draw(row, 0.5).ambiguous


def test_draw_ties_are_ranked_by_index():
    row = np.array([0.0, 2.0, NEG, 2.0, 1.0, 2.0])
    ids, v = S.sorted_kept(row)
    assert ids.tolist() == [1, 3, 5, 4, 0] and v.tolist() == [2.0, 2.0, 2.0, 1.0, 0.0]
    e = np.exp(np.array([0.0, 0.0, 0.0, -1.0, -2.0]))
    cum = np.cumsum(e) / e.sum()
    for r in range(5):
        lo = 0.0 if r == 0 else cum[r - 1]
        u = (lo + cum[r]) / 2
        assert S.draw(row, u).rank == r and S.draw(row, u).token == ids[r]


def test_draw_last_rank_fallback():
    row = np.full(4, NEG)
    row[[0, 1, 3]] = [0.0, -1.0, -200.0]     # the last term underflows below the others' rounding: cum[1] == cum[2] == tot
    e = np.exp(np.array([0.0, -1.0, -200.0]))
    assert np.cumsum(e)[1] == np.cumsum(e)[2]
    d = S.draw(row, 1.0)                     # no cumulative sum exceeds u * tot: the last rank
    assert d.rank == 2 and d.token == 3
    d = S.draw(row, 1 - 2 ** -24)
    assert d.rank == 1 and d.token == 1


def test_draw_ambiguity_window_is_exactly_eps():
    row = np.full(6, NEG)
    row[[1, 4]] = 0.0                         # tot = 2, the one interior boundary at u = 0.5
    inside, outside = 0.5 - 0.99 * S.EPS, 0.5 - 1.01 * S.EPS
    d = S.draw(row, inside)
    assert d.ambiguous and d.token == 1 and d.accept == (1, 4) and d.margin == pytest.approx(0.99 * S.EPS)
    d = S.draw(row, outside)
    assert not d.ambiguous and d.accept == (1,) and d.margin == pytest.approx(1.01 * S.EPS)
    d = S.draw(row, 0.5 + 0.99 * S.EPS)
    assert d.ambiguous and d.token == 4 and d.accept == (1, 4)
    d = S.draw(row, 0.5 + 1.01 * S.EPS)
    assert not d.ambiguous and d.accept == (4,)
    # u near 0 or near 1 is no boundary of a different pick
    assert not S.draw(row, 0.0).ambiguous and not S.draw(row, 1 - 2 ** -24).ambiguous


def test_top_p_keep_counts():
    # probabilities 0.5, 0.3, 0.2 (sorted); tails: ranks 1.. = 0.5, rank 2 = 0.2
    row = np.log(np.array([0.3, 0.5, 0.2]))
    assert S.top_p_keep_counts(row, 0.9) == (3,)          # 1 - top_p = 0.1 < 0.2: nothing removed
    assert S.top_p_keep_counts(row, 0.6) == (2,)          # 0.4: rank 2 (0.2) removed, rank 1 (0.5) kept
    assert S.top_p_keep_counts(row, 0.4) == (1,)          # 0.6: ranks 1, 2 removed
    assert S.top_p_keep_counts(row, 0.8) == (2, 3)        # 0.2 = the tail of rank 2: within eps, both counts
    assert S.keep_top(row, 2).tolist() == [row[0], row[1], NEG]
    assert S.top_p_threshold(0.9) == float(np.float32(1.0 - float(np.float32(0.9))))


class _Spec:
    do_sample, repetition_penalty, no_repeat_ngram_size, temperature, top_k, top_p = 1, 1.0, 0, 1.0, 3, 1.0
    min_new_tokens, n_eos, eos_token_id, pad_token_id, seed = 0, 0, (0, 0, 0, 0), 0, 0

    def __init__(self, **kw):
        self.__dict__.update(kw)


def test_spec_fields_reads_a_sampler_spec():
    f = S.spec_fields(_Spec(repetition_penalty=1.1, no_repeat_ngram_size=15, n_eos=2, eos_token_id=(7, 9, 0, 0), seed=2 ** 63 + 5))
    assert f["eos"] == [7, 9] and f["seed"] == 2 ** 63 + 5 and f["no_repeat_ngram_size"] == 15


def test_predict_chains_the_processors_and_the_draw():
    pytest.importorskip("transformers")
    logits = np.array([0.0, np.log(3.0), 5.0, np.log(2.0), -1.0], dtype=np.float32)
    # step 0, no history: token 2 is banned by nothing and dominates; with min_new_tokens it is masked as an EOS id
    spec = _Spec(top_k=3, seed=11)
    u = S.uniform(11, 0, 1)
    p = S.predict(logits, [], spec, 0, 1)
    assert p.token == S.draw(p.scores, u).token and np.isfinite(p.scores).sum() == 3
    masked = S.predict(logits, [], _Spec(top_k=3, seed=11, min_new_tokens=1, n_eos=1, eos_token_id=(2, 0, 0, 0)), 0, 1)
    assert not np.isfinite(masked.scores[2]) and np.isfinite(masked.scores[[1, 3, 0]]).all()
    # probabilities 3/6, 2/6, 1/6 over tokens 1, 3, 0: the draw follows u
    e = np.array([3.0, 2.0, 1.0]) / 6
    want = [1, 3, 0][int(np.searchsorted(np.cumsum(e), u, side="right"))]
    assert masked.token == want or masked.ambiguous
    # no-repeat-ngram with n = 2 after history [4, 1, 4]: token 1 is banned; repetition penalty divides the positive repeats
    p = S.predict(logits, [4, 1, 4], _Spec(top_k=5, no_repeat_ngram_size=2, repetition_penalty=2.0, seed=3), 3, 0)
    assert not np.isfinite(p.scores[1]) and p.scores[2] == np.float32(5.0) and p.scores[4] == np.float32(-2.0)
