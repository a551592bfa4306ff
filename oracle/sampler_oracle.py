"""The device sampler's draw (csrc/sampler.cu, dec_sample_kernel) restated on the host in float64, so that every sampled token can be
checked against what the rule says it must be.

The rule (include/vcla.h, vcla_sampler):
  counter = (step, sequence, 0, 0), key = (seed & 0xffffffff, seed >> 32)      step = tokens generated so far, sequence = batch row
  x0      = word 0 of Philox4x32-10(counter, key)                              (Salmon et al. 2011, the Random123 generator)
  u       = (x0 >> 8) * 2**-24                                                 a 24-bit uniform in [0, 1)
  kept set, sorted by (value descending, index ascending); e_r = exp(x_r - x_0), tot = sum e_r
  pick    = the first rank r with e_0 + ... + e_r > u * tot, else the last rank

The kernel sums at most 1024 terms in fp32 with expf, so its cumulative sums carry a relative error of about 1024 * 2**-24 ~ 6e-5
plus a few expf ulps.  A draw whose u * tot lies within EPS * tot of a cumulative boundary is therefore ambiguous: both neighbouring
ranks are acceptable.  top-p's keep count is an fp32 comparison in the kernel too (cum <= 1 - top_p): top_p_keep_counts lists every
count within EPS of that threshold.

philox4x32_10, uniform, draw and top_p_keep_counts need numpy only; predict runs transformers' processors and imports them itself."""
from typing import NamedTuple, Sequence, Tuple

import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57          # round multipliers
W0, W1 = 0x9E3779B9, 0xBB67AE85          # key increments (the golden ratio and sqrt(3) - 1)
EPS = 1e-4
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr: Sequence, key: Sequence) -> np.ndarray:
    """Philox4x32-10 of the four counter words and two key words (each an int or a broadcastable integer array) -> uint32 (4, ...).
    Each round maps (c0, c1, c2, c3) to (hi(M1*c2) ^ c1 ^ k0, lo(M1*c2), hi(M0*c0) ^ c3 ^ k1, lo(M0*c0)), then bumps the key."""
    c = np.broadcast_arrays(*[np.asarray(x, dtype=np.uint64) & _MASK for x in ctr], *[np.asarray(k, dtype=np.uint64) & _MASK for k in key])
    c0, c1, c2, c3, k0, k1 = (a.copy() for a in c)
    m0, m1, w0, w1 = np.uint64(M0), np.uint64(M1), np.uint64(W0), np.uint64(W1)
    for _ in range(10):
        p0, p1 = m0 * c0, m1 * c2                 # 32 x 32 -> 64 bit products: exact in uint64
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK
        k0, k1 = (k0 + w0) & _MASK, (k1 + w1) & _MASK
    return np.stack([c0, c1, c2, c3]).astype(np.uint32)


def key_words(seed: int) -> Tuple[int, int]:
    seed = int(seed) & (2 ** 64 - 1)
    return seed & 0xFFFFFFFF, seed >> 32


def word0(seed: int, step, seq) -> np.ndarray:
    """x0 = word 0 of Philox4x32-10((step, seq, 0, 0), seed): uint32, broadcast over step / seq."""
    return philox4x32_10((step, seq, 0, 0), key_words(seed))[0]


def uniform(seed: int, step, seq):
    """The kernel's uniform for (seed, step, sequence): (x0 >> 8) * 2**-24, exact in float64 (and in fp32)."""
    u = (word0(seed, step, seq) >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
    return float(u) if u.ndim == 0 else u


class Draw(NamedTuple):
    token: int                # the pick
    rank: int                 # its rank in the sorted kept set
    ambiguous: bool           # u * tot within eps * tot of an interior cumulative boundary
    accept: Tuple[int, ...]   # every token the kernel may pick within its fp32 error (the pick and, if ambiguous, its neighbours)
    margin: float             # min |u * tot - boundary| / tot over the interior boundaries (inf with one kept token)


def sorted_kept(scores) -> Tuple[np.ndarray, np.ndarray]:
    """The finite entries of one row, sorted by (value descending, index ascending) -> (ids, float64 values)."""
    x = np.asarray(scores, dtype=np.float64).reshape(-1)
    idx = np.flatnonzero(np.isfinite(x))
    order = np.lexsort((idx, -x[idx]))
    ids = idx[order]
    return ids, x[ids]


def draw(scores, u: float, eps: float = EPS) -> Draw:
    """The inverse-CDF draw over one row of processed scores (the finite entries are the kept set), in float64."""
    ids, v = sorted_kept(scores)
    if ids.size == 0:
        raise ValueError("draw: the row keeps no token")
    e = np.exp(v - v[0])
    cum = np.cumsum(e)
    tot = cum[-1]
    target = u * tot
    hit = np.flatnonzero(cum > target)
    r = int(hit[0]) if hit.size else ids.size - 1
    # interior boundaries only: below the first one the pick is rank 0 either way, and at the last one the kernel falls back to the
    # last rank when its running sum never exceeds u * tot
    dist = np.abs(cum[:-1] - target)
    near = np.flatnonzero(dist < eps * tot)
    ranks = {r} | {int(j) for j in near} | {int(j) + 1 for j in near}
    margin = float(dist.min() / tot) if dist.size else float("inf")
    return Draw(int(ids[r]), r, bool(near.size), tuple(sorted(int(ids[j]) for j in ranks)), margin)


def top_p_threshold(top_p: float) -> float:
    """1 - top_p as the kernel holds it: top_p arrives as fp32, the difference is taken in double and rounded to fp32."""
    return float(np.float32(1.0 - float(np.float32(top_p))))


def top_p_keep_counts(scores, top_p: float, eps: float = EPS) -> Tuple[int, ...]:
    """Keep counts of the top-p filter over one row of top-k scores (finite = kept), computed in float64: rank r >= 1 of the sorted kept
    set is removed when the ascending cumulative probability of ranks r .. c-1 is <= 1 - top_p; the largest is always kept.  Every
    count whose boundary lies within eps of the threshold is listed (the kernel's cumulative sum is fp32)."""
    ids, v = sorted_kept(scores)
    p = np.exp(v - v[0])
    p /= p.sum()
    tail = np.cumsum(p[::-1])[::-1][1:]          # tail[r - 1] = p_r + ... + p_{c-1}, r = 1 .. c-1
    thr = top_p_threshold(top_p)
    lo = 1 + int(np.count_nonzero(tail > thr + eps))
    hi = 1 + int(np.count_nonzero(tail > thr - eps))
    return tuple(range(lo, hi + 1))


def keep_top(scores, count: int) -> np.ndarray:
    """The row with only its `count` highest-ranked finite entries kept (the rest -inf)."""
    ids, _ = sorted_kept(scores)
    out = np.full(np.asarray(scores).reshape(-1).shape, -np.inf)
    out[ids[:count]] = np.asarray(scores, dtype=np.float64).reshape(-1)[ids[:count]]
    return out


class Prediction(NamedTuple):
    token: int                # the draw over the kept set transformers' processors return
    ambiguous: bool           # more than one token is acceptable
    accept: Tuple[int, ...]   # every acceptable token (draw windows and top-p keep counts within eps)
    rank: int
    margin: float
    scores: np.ndarray        # the processed scores (transformers), float32


def spec_fields(spec) -> dict:
    """A native vcla_sampler (or any object with the same attribute names) -> plain Python values."""
    n_eos = int(spec.n_eos)
    return dict(do_sample=bool(spec.do_sample), repetition_penalty=float(spec.repetition_penalty), no_repeat_ngram_size=int(spec.no_repeat_ngram_size),
                temperature=float(spec.temperature), top_k=int(spec.top_k), top_p=float(spec.top_p), min_new_tokens=int(spec.min_new_tokens),
                eos=[int(spec.eos_token_id[i]) for i in range(n_eos)], seed=int(spec.seed))


def processed_scores(logits_row, history, spec):
    """transformers' processors on one row, in the order sampler.cu applies them: repetition penalty, no-repeat-ngram, the
    min_new_tokens EOS mask, temperature, top-k, top-p.  -> (scores before top-p, scores after top-p), float32 (V,) numpy."""
    import torch
    from transformers.generation import logits_process as lp
    f = spec_fields(spec)
    x = torch.as_tensor(np.asarray(logits_row, dtype=np.float32)).reshape(1, -1).clone()
    h = torch.as_tensor(np.asarray(history, dtype=np.int64)).reshape(1, -1)
    if f["repetition_penalty"] != 1.0:
        x = lp.RepetitionPenaltyLogitsProcessor(penalty=f["repetition_penalty"])(h, x)
    if f["no_repeat_ngram_size"] > 0:
        x = lp.NoRepeatNGramLogitsProcessor(f["no_repeat_ngram_size"])(h, x)
    if f["eos"] and f["min_new_tokens"] > 0:
        x = lp.MinNewTokensLengthLogitsProcessor(prompt_length_to_skip=0, min_new_tokens=f["min_new_tokens"], eos_token_id=f["eos"])(h, x)
    if f["temperature"] != 1.0:
        x = lp.TemperatureLogitsWarper(f["temperature"])(h, x)
    x = lp.TopKLogitsWarper(top_k=f["top_k"], min_tokens_to_keep=1)(h, x)
    before = x
    if f["top_p"] < 1.0:
        x = lp.TopPLogitsWarper(top_p=f["top_p"], min_tokens_to_keep=1)(h, x)
    return before[0].numpy(), x[0].numpy()


def predict(logits_row, history, spec, step: int, seq: int, eps: float = EPS) -> Prediction:
    """The token the device sampler must draw at `step` (= len(history)) of batch row `seq` from raw logits and the row's generated
    tokens so far: transformers' processors, then draw() with uniform(seed, step, seq).  The pick is made on the kept set
    transformers returns; accept also covers the picks on every top-p keep count within eps of the threshold."""
    f = spec_fields(spec)
    if not f["do_sample"]:
        raise ValueError("predict: the draw rule applies to do_sample only")
    before, after = processed_scores(logits_row, history, spec)
    u = uniform(f["seed"], step, seq)
    d = draw(after, u, eps)
    accept = set(d.accept)
    ambiguous = d.ambiguous
    if f["top_p"] < 1.0:
        counts = top_p_keep_counts(before, f["top_p"], eps)
        if len(counts) > 1:
            ambiguous = True
        for c in counts:
            accept.update(draw(keep_top(before, c), u, eps).accept)
    return Prediction(d.token, ambiguous or len(accept) > 1, tuple(sorted(accept)), d.rank, d.margin, after)
