"""The two kernels every generated token passes through, at operator level: the decode attention (attn_decode_kernel and
attn_decode_persistent_kernel through vcla_op_attention_decode) and the greedy pick (dec_logits_stage1/2 through
vcla_op_logits_argmax), each against a plain torch reference written from the definition.

Decode attention.  The reference sums the split-K partials in fp32 in split order (what the kernels specify; it makes the appended V
exact), applies RoPE in float64 in HF's rotate_half form at HF's angle -- inv_freq and position * inv_freq in fp32, which is how the
model is defined --, rounds the new K/V row to bf16 and takes a float64 softmax over the cached rows (gathered through the page table)
plus the new row.  The pool is larger than the batch needs, the page tables are a seeded permutation with unused entries set to -1 (by
reading, neither kernel dereferences an entry beyond seq_len / page_tokens, and the entry checks the ones it will read), and every
element that is not a valid cached row -- the slots from seq_len on in each last page, the pages nobody owns -- holds a bf16 NaN, so
a read past the valid tokens poisons the output and a write anywhere but the appended row changes the pool.  seq_len = 0 does not occur
in the engine (a prefill always precedes) but both kernels handle it (the output is the new token's v) and it is tested.

The tests marked `gpu` need a device; the unmarked ones check the reference itself on the CPU (against
torch.nn.functional.scaled_dot_product_attention in float64 and the oracle's RoPE), so a wrong reference cannot hide behind a skip."""
import ctypes as C
import math
from types import SimpleNamespace

import pytest
import torch

import visualcla_oracle as O

gpu = pytest.mark.gpu

HD = 128
SCALE = HD ** -0.5
NAN_BITS = 0x7FC1          # a bf16 NaN; as int16 it is positive, and no kernel produces this payload
# |out - ref| <= OUT_TOL * max(1, max |ref|).  out is one bf16 rounding of an fp32 result: half an ulp is up to 2^-8 = 3.9e-3 of the
# value.  Largest values observed (H100 80GB HBM3, 700 W): 3.2e-3 in the geometry sweep, 3.0e-3 mixed lengths, 3.2e-3 persistent ring,
# 1.9e-3 production shapes, 3.4e-3 in step 2 of the two-step test (whose cached K row may sit one ulp from the reference's), 1.0e-3 and
# less in the numerics cases.  Twice the largest would pass the starting bound of 3 * 2^-9 = 5.9e-3, so that bound stays.
OUT_TOL = 3 * 2.0 ** -9

_observed = {}


def _note(group, err):
    _observed[group] = max(_observed.get(group, 0.0), err)


@pytest.fixture(scope="module", autouse=True)
def _report_observed():
    yield
    for group in sorted(_observed):
        print(f"\n[decode-attention] largest error, {group}: {_observed[group]:.3e}", end="")
    print()


# ---------------------------------------------------------------------------------------------------------------------------------
# reference
# ---------------------------------------------------------------------------------------------------------------------------------
def sum_splits(partial):
    """fp32 sum over dim 0 in split order, starting from 0 as the kernels do."""
    acc = torch.zeros_like(partial[0])
    for s in range(partial.shape[0]):
        acc = acc + partial[s]
    return acc


def rope_ref(x, pos, theta):
    """x (..., 128) float64 at position pos: x * cos + rotate_half(x) * sin, pairs (d, d + 64); the angle is HF's fp32 one."""
    power = (torch.tensor(float(theta), dtype=torch.float64) ** (torch.arange(0, HD, 2, dtype=torch.float64) / HD)).float()
    inv = 1.0 / power            # HF: inv_freq = 1 / base ** (arange(0, dim, 2) / dim) in fp32, here with every step correctly rounded
    ang = (torch.tensor(float(pos), dtype=torch.float32) * inv).double()
    cos, sin = torch.cat([ang.cos(), ang.cos()]), torch.cat([ang.sin(), ang.sin()])
    rot = torch.cat([-x[..., HD // 2:], x[..., :HD // 2]], dim=-1)
    return x * cos + rot * sin


def gather_rows(pool, table_row, n, pt):
    """The first n cached rows of one sequence: K, V (n, H, 128) in the pool's bf16."""
    j = torch.arange(n)
    rows = pool[table_row[j // pt].long(), :, :, j % pt]          # (n, 2, H, 128)
    return rows[:, 0], rows[:, 1]


def decode_ref(partial, pool, table, lens, pt, H, scale, theta):
    """out (B, H, 128) float64 and the appended rows k_new, v_new (B, H, 128) bf16."""
    B = len(lens)
    qkv = sum_splits(partial).view(B, 3, H, HD)
    out = torch.empty(B, H, HD, dtype=torch.float64)
    k_new = torch.empty(B, H, HD, dtype=torch.bfloat16)
    v_new = torch.empty(B, H, HD, dtype=torch.bfloat16)
    for b, L in enumerate(lens):
        q = rope_ref(qkv[b, 0].double(), L, theta)
        k_new[b] = rope_ref(qkv[b, 1].double(), L, theta).float().to(torch.bfloat16)
        v_new[b] = qkv[b, 2].to(torch.bfloat16)
        kc, vc = gather_rows(pool, table[b], L, pt)
        K = torch.cat([kc.double(), k_new[b].double()[None]])      # (L + 1, H, 128)
        V = torch.cat([vc.double(), v_new[b].double()[None]])
        p = torch.softmax(torch.einsum("hd,lhd->hl", q, K) * scale, dim=-1)
        out[b] = torch.einsum("hl,lhd->hd", p, V)
    return out, k_new, v_new


# ---------------------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------------------
def make_case(pt, lens, H, splits, seed, theta=10000.0, k_std=1.0, spare_entries=2, steps=1):
    """Seeded partials and a NaN-filled pool holding lens[b] cached rows per sequence behind a permuted, partly unused page table.
    Each sequence owns the pages of its cached rows and of the `steps` rows to be appended."""
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    owned = [(L + steps - 1) // pt + 1 for L in lens]
    pps = max(owned) + spare_entries
    n_pages = sum(owned) + 3
    perm = torch.randperm(n_pages, generator=g).to(torch.int32)
    table = torch.full((B, pps), -1, dtype=torch.int32)
    pool = torch.full((n_pages, 2, H, pt, HD), NAN_BITS, dtype=torch.int16).view(torch.bfloat16)
    at = 0
    for b, L in enumerate(lens):
        table[b, :owned[b]] = perm[at:at + owned[b]]
        at += owned[b]
        j = torch.arange(L)
        pages, slots = table[b, j // pt].long(), j % pt
        pool[pages, 0, :, slots] = (torch.randn(L, H, HD, generator=g) * k_std).to(torch.bfloat16)
        pool[pages, 1, :, slots] = torch.randn(L, H, HD, generator=g).to(torch.bfloat16)
    partial = torch.randn(splits, B, 3 * H * HD, generator=g) / math.sqrt(splits)
    return SimpleNamespace(pt=pt, lens=list(lens), H=H, B=B, theta=theta, partial=partial, pool=pool, table=table)


def q_rotated(case):
    """The rotated, unscaled query of every (sequence, head), float64 (B, H, 128)."""
    q = sum_splits(case.partial).view(case.B, 3, case.H, HD)[:, 0].double()
    return torch.stack([rope_ref(q[b], L, case.theta) for b, L in enumerate(case.lens)])


def set_key_scores(case, b, rows, score):
    """Overwrite cached K rows `rows` of sequence b by the multiple of each head's rotated query that scores `score`."""
    qr = q_rotated(case)[b]                                        # (H, 128)
    key = (qr * (score / SCALE) / (qr * qr).sum(-1, keepdim=True)).float().to(torch.bfloat16)
    j = torch.as_tensor(rows)
    case.pool[case.table[b, j // case.pt].long(), 0, :, j % case.pt] = key[None].expand(len(j), -1, -1)


def set_new_key_score(case, score):
    """Make the new token's key a multiple of its query: k = a * q commutes with RoPE, and q . q is about 128 per head."""
    T = case.H * HD
    case.partial[:, :, T:2 * T] = case.partial[:, :, :T] * (score / (SCALE * HD))


def ordered_bits(x):
    """bf16 -> int32 that grows with the value, so that neighbours differ by one (both zeros give 0)."""
    bits = x.contiguous().view(torch.int16).to(torch.int32)
    mag = bits & 0x7FFF
    return torch.where(bits < 0, -mag, mag)


def new_row_index(case):
    b = torch.arange(case.B)
    L = torch.tensor(case.lens)
    return case.table[b, L // case.pt].long(), L % case.pt


def check_result(case, out, pool_after, ref, group, what):
    """Assertions 1-3 of a call: the output, the appended row, and nothing else written."""
    r_out, k_new, v_new = ref
    got = out.view(case.B, case.H, HD).double()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    err = (got - r_out).abs().max().item() / max(1.0, r_out.abs().max().item())
    _note(group, err)
    assert err <= OUT_TOL, f"{what}: max |out - ref| / max(1, max |ref|) = {err:.3e}"
    pages, slots = new_row_index(case)
    k_got, v_got = pool_after[pages, 0, :, slots], pool_after[pages, 1, :, slots]          # (B, H, 128)
    assert torch.equal(v_got.view(torch.int16), v_new.view(torch.int16)), f"{what}: appended V row is not bf16(v)"
    # one bf16 ulp; where x cos and rotate_half(x) sin cancel the result is far smaller than the fp32 rounding of its terms, so an
    # element also passes within 2^-20 of the row's scale
    ulps = (ordered_bits(k_got) - ordered_bits(k_new)).abs()
    far = (ulps > 1) & ((k_got.double() - k_new.double()).abs() > 2.0 ** -20 * max(1.0, k_new.float().abs().max().item()))
    assert not far.any(), f"{what}: appended K row is {int(ulps[far].max())} bf16 ulps from the reference"
    same = (ulps == 0).float().mean().item()
    assert same >= 0.99, f"{what}: only {same:.4f} of the appended K row is bit-equal to the reference"
    expect = case.pool.clone()
    expect[pages, 0, :, slots] = k_got
    expect[pages, 1, :, slots] = v_got
    assert torch.equal(expect.view(torch.int16), pool_after.view(torch.int16)), f"{what}: the pool changed outside the appended row"
    return err


def run_op(case, kv_splits=1, persistent=0, grid=0, launches=1, lens=None, pool=None, pt=None):
    """-> (rc, out (B, H*128) bf16 on the host, the pool after the call on the host)."""
    from visualcla import _native as N
    lib = N.load()
    pool_d = (case.pool if pool is None else pool).cuda()
    part_d, table_d = case.partial.cuda(), case.table.cuda()
    len_d = torch.tensor(case.lens if lens is None else lens, dtype=torch.int32, device="cuda")
    out = torch.zeros(case.B, case.H * HD, dtype=torch.bfloat16, device="cuda")
    rc = lib.vcla_op_attention_decode(N.ptr(part_d), case.partial.shape[0], N.ptr(pool_d), N.ptr(table_d), case.table.shape[1],
                                      case.pt if pt is None else pt, N.ptr(len_d), N.ptr(out), case.B, case.H, kv_splits,
                                      C.c_float(SCALE), C.c_float(case.theta), persistent, grid, launches,
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, out.cpu(), pool_d.cpu()


def run_ok(case, **kw):
    from visualcla import _native as N
    rc, out, pool = run_op(case, **kw)
    N.check(rc, "vcla_op_attention_decode")
    return out, pool


def check_variants(case, variants, group):
    """Every (kv_splits, persistent, grid) variant against the reference (assertions 1-3); for each, two launches over the same scratch
    and counters and a second call must reproduce output and pool bit for bit (4); the variants agree with each other (5)."""
    ref = decode_ref(case.partial, case.pool, case.table, case.lens, case.pt, case.H, SCALE, case.theta)
    outs = []
    for kv_splits, persistent, grid in variants:
        what = f"{group}: page_tokens {case.pt} seq_len {case.lens} H {case.H} qkv splits {case.partial.shape[0]} kv_splits {kv_splits} " \
               f"persistent {persistent} grid {grid}"
        out, pool = run_ok(case, kv_splits=kv_splits, persistent=persistent, grid=grid)
        check_result(case, out, pool, ref, group, what)
        out2, pool2 = run_ok(case, kv_splits=kv_splits, persistent=persistent, grid=grid, launches=2)
        assert torch.equal(out2.view(torch.int16), out.view(torch.int16)), f"{what}: a second launch over the same counters changed the output"
        assert torch.equal(pool2.view(torch.int16), pool.view(torch.int16)), f"{what}: a second launch changed the pool"
        out3, pool3 = run_ok(case, kv_splits=kv_splits, persistent=persistent, grid=grid)
        assert torch.equal(out3.view(torch.int16), out.view(torch.int16)) and torch.equal(pool3.view(torch.int16), pool.view(torch.int16)), \
            f"{what}: two calls differ"
        outs.append(out.double())
    bound = OUT_TOL * max(1.0, ref[0].abs().max().item())
    for o in outs[1:]:
        assert (o - outs[0]).abs().max().item() <= bound, f"{group}: variants {variants} disagree on seq_len {case.lens}"
    return ref


ONE_SHOT = [(1, 0, 0), (2, 0, 0), (3, 0, 0), (4, 0, 0), (8, 0, 0)]
PERSISTENT = [(1, 1, 1), (1, 1, 2), (1, 1, 5), (1, 1, 0)]


# ---------------------------------------------------------------------------------------------------------------------------------
# the reference itself (CPU)
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("theta", [10000.0, 500.0])
def test_rope_reference_equals_oracle(theta):
    cfg = O.PathConfig(t_hidden=2 * HD, t_heads=2, rope_theta=theta)
    x = torch.randn(3, 2, HD, generator=torch.Generator().manual_seed(1))
    for pos in (0, 1, 65, 1500):
        cos, sin = O.rope_tables(cfg, torch.tensor([pos]))
        want = O.apply_rope(x[:, :, None, :], cos, sin)[:, :, 0]
        # the oracle's cos / sin are fp32, and its fp32 pow may round inv_freq one ulp away, which the position multiplies
        assert (rope_ref(x.double(), pos, theta) - want.double()).abs().max().item() < 2e-6 + pos * 2.0 ** -22
    # the pairing and the sign, spelled out: at angle a, (x_d, x_{d+64}) -> (x_d cos a - x_{d+64} sin a, x_{d+64} cos a + x_d sin a)
    e = torch.zeros(HD, dtype=torch.float64)
    e[0] = 1.0
    r = rope_ref(e, 1, theta)                                      # pair 0 turns at inv_freq 1: angle = 1 rad
    assert abs(r[0].item() - math.cos(1.0)) < 1e-12 and abs(r[64].item() - math.sin(1.0)) < 1e-12 and r.abs().sum().item() < 1.5


@pytest.mark.parametrize("pt", [8, 64])
def test_decode_reference_equals_sdpa(pt):
    """kv lengths 1 and 65 (seq_len 0 and 64): the reference's output is float64 scaled_dot_product_attention over the gathered rows
    plus the row it says is appended, with the q / k the oracle's RoPE gives."""
    lens, H, theta = [0, 64], 2, 10000.0
    case = make_case(pt, lens, H, splits=3, seed=11 + pt)
    out, k_new, v_new = decode_ref(case.partial, case.pool, case.table, lens, pt, H, SCALE, theta)
    qkv = sum_splits(case.partial).view(2, 3, H, HD)
    assert (qkv.double() - case.partial.double().sum(0).view(2, 3, H, HD)).abs().max().item() < 1e-5
    cfg = O.PathConfig(t_hidden=H * HD, t_heads=H, rope_theta=theta)
    for b, L in enumerate(lens):
        cos, sin = O.rope_tables(cfg, torch.tensor([L]))
        q = O.apply_rope(qkv[b, 0][:, None, :], cos, sin)          # (H, 1, 128)
        k = O.apply_rope(qkv[b, 1][:, None, :], cos, sin)
        assert (k[:, 0] - k_new[b].float()).abs().max().item() <= 2.0 ** -8 * k.abs().max().item()
        assert torch.equal(v_new[b], qkv[b, 2].to(torch.bfloat16))
        kc, vc = gather_rows(case.pool, case.table[b], L, pt)
        assert kc.shape == (L, H, HD) and not torch.isnan(kc.float()).any() and not torch.isnan(vc.float()).any()
        K = torch.cat([kc, k_new[b][None]]).double().transpose(0, 1)   # (H, L + 1, 128)
        V = torch.cat([vc, v_new[b][None]]).double().transpose(0, 1)
        want = torch.nn.functional.scaled_dot_product_attention(q.double(), K, V, scale=SCALE)[:, 0]
        assert (out[b] - want).abs().max().item() < 1e-5           # q from the oracle's fp32 tables
        mine = torch.nn.functional.scaled_dot_product_attention(rope_ref(qkv[b, 0].double(), L, theta)[:, None], K, V, scale=SCALE)[:, 0]
        assert (out[b] - mine).abs().max().item() < 1e-12


def test_case_pool_is_nan_outside_the_cached_rows():
    case = make_case(16, [0, 5, 16, 40], 2, splits=2, seed=3)
    valid = torch.zeros(case.pool.shape[0], case.pt, dtype=torch.bool)
    for b, L in enumerate(case.lens):
        j = torch.arange(L)
        valid[case.table[b, j // case.pt].long(), j % case.pt] = True
        used = L // case.pt + 1
        assert (case.table[b, :used] >= 0).all() and (case.table[b, used:] == -1).all()
    nan = torch.isnan(case.pool.float())                           # (pages, 2, H, pt, 128)
    assert int(valid.sum()) == sum(case.lens)
    assert not nan[valid[:, None, None, :, None].expand_as(nan)].any() and nan[~valid[:, None, None, :, None].expand_as(nan)].all()
    used_pages = case.table[case.table >= 0]
    assert used_pages.unique().numel() == used_pages.numel() < case.pool.shape[0]
    x = torch.tensor([-1.0, -0.0, 0.0, 1.0], dtype=torch.bfloat16)
    assert ordered_bits(x).tolist() == [-0x3F80, 0, 0, 0x3F80]
    assert int(ordered_bits(torch.tensor([1.0078125], dtype=torch.bfloat16)) - ordered_bits(x[3:])) == 1


# ---------------------------------------------------------------------------------------------------------------------------------
# decode attention on the device
# ---------------------------------------------------------------------------------------------------------------------------------
def _sweep_lengths(pt):
    return [0, 1, pt - 1, pt, pt + 1, 2 * pt - 1, 2 * pt, 3 * pt + 5, 7 * pt, 1500]


@gpu
@pytest.mark.parametrize("pt", [8, 16, 32, 64])
@pytest.mark.parametrize("li", range(10))
def test_decode_attention_split_geometry(pt, li):
    """Both kernels over page size x cached length x kv_splits.  chunk = roundup(ceil((L + 1) / kv_splits), page_tokens): L = 0, 1,
    page_tokens - 1 leave more splits than pages (empty CTAs enter the combine with m = -inf, l = 0); L = page_tokens with 2 splits,
    2 * page_tokens with 3 / 4 / 8 and 7 * page_tokens with 8 are exact multiples of the chunk, so the new token sits alone in a CTA
    that streams no page."""
    L = _sweep_lengths(pt)[li]
    case = make_case(pt, [L, 2 * L // 3], 2, splits=1 + li % 4, seed=1000 * pt + L)
    check_variants(case, ONE_SHOT + [(1, 1, 1), (1, 1, 0)], "geometry sweep")


@gpu
@pytest.mark.parametrize("pt", [16, 64])
def test_decode_attention_mixed_lengths(pt):
    """Every row has its own chunking and page count, as after left-padded prefills, kv_truncate and beam search."""
    case = make_case(pt, [1, 63, 64, 65, 700, 5, 1500, 128], 3, splits=4, seed=77 + pt)
    check_variants(case, [(1, 0, 0), (4, 0, 0), (8, 0, 0)] + PERSISTENT, "mixed lengths")


@gpu
@pytest.mark.parametrize("pt", [8, 64])
@pytest.mark.parametrize("H", [1, 3])
def test_decode_attention_persistent_ring(pt, H):
    """Items whose page counts (0, 1, 2, 4, 5, 7, 3, 1, 8, 2) are not multiples of the 3 ring stages follow each other on one CTA, so
    the stage index and the mbarrier parities wrap inside and across items; qkv split counts 1, 2, 3, 5, 8 take both halves of the
    q/k/v producer's two-at-a-time loads."""
    lens = [0, pt, 2 * pt, 4 * pt - 3, 5 * pt, 7 * pt - 1, 3 * pt, 1, 8 * pt, pt + 1]
    for (grid, splits) in [(1, 1), (2, 2), (5, 3), (0, 5), (1, 8), (3, 3)]:
        case = make_case(pt, lens, H, splits=splits, seed=10 * pt + H + splits)
        check_variants(case, [(1, 1, grid), (1, 0, 0)], "persistent ring")


@gpu
@pytest.mark.parametrize("B", [1, 8, 32, 64])
def test_decode_attention_production_shapes(B):
    """LLaMA-7B's 32 heads at page size 64, about 300 cached tokens, with kv_splits and the kernel the engine picks for the batch:
    decode_attn_call takes kv_splits = min(8, max(ceil(SMs / (B * H)), context minimum)) from B and H = 32 (the minimum is 1 below 768
    tokens of context, 4 from 1536), and attention_decode runs the persistent kernel when kv_splits is 1 and B * H exceeds 2 CTAs per SM."""
    H, sms = 32, torch.cuda.get_device_properties(0).multi_processor_count
    lens = [300 + (37 * b) % 64 - 32 for b in range(B)]
    case = make_case(64, lens, H, splits=4, seed=500 + B)
    variants = []
    for context_min in (1, 4):
        kv_splits = min(8, max((sms + B * H - 1) // (B * H), context_min))
        variant = (kv_splits, int(kv_splits == 1 and B * H > 2 * sms), 0)
        if variant not in variants:
            variants.append(variant)
    check_variants(case, variants, "production shapes")


@gpu
@pytest.mark.parametrize("where", ["first split", "last split", "new token"])
def test_decode_attention_one_dominant_key(where):
    """One key scores about 80 above the rest: the softmax is that key's V row, wherever the key sits."""
    pt, lens = 16, [200, 90]
    case = make_case(pt, lens, 2, splits=2, seed=31, k_std=0.05)
    if where == "new token":
        set_new_key_score(case, 80.0)
    else:
        for b, L in enumerate(lens):
            set_key_scores(case, b, [3 if where == "first split" else L - 2], 80.0)
    ref = check_variants(case, [(1, 0, 0), (4, 0, 0), (8, 0, 0), (1, 1, 1)], "dominant key")
    for b, L in enumerate(lens):
        row = ref[2][b] if where == "new token" else gather_rows(case.pool, case.table[b], L, pt)[1][3 if where == "first split" else L - 2]
        assert (ref[0][b] - row.double()).abs().max().item() < 1e-6      # the case is what it claims to be


@gpu
def test_decode_attention_vanishing_first_pages():
    """Every key of the first pages scores about 100 below the later ones: their partial (m = -100) must vanish in the merges across
    token groups, warps and CTAs, not turn into NaN or inf."""
    pt, lens = 16, [160, 96]
    case = make_case(pt, lens, 2, splits=1, seed=32, k_std=0.05)
    for b, L in enumerate(lens):
        set_key_scores(case, b, list(range(L // 2)), -100.0)
    ref = check_variants(case, [(1, 0, 0), (2, 0, 0), (4, 0, 0), (8, 0, 0), (1, 1, 2)], "vanishing pages")
    for b, L in enumerate(lens):                                   # the case is what it claims to be: only the later rows count
        kc, vc = gather_rows(case.pool, case.table[b], L, pt)
        K = torch.cat([kc[L // 2:].double(), ref[1][b].double()[None]])
        V = torch.cat([vc[L // 2:].double(), ref[2][b].double()[None]])
        p = torch.softmax(torch.einsum("hd,lhd->hl", q_rotated(case)[b], K) * SCALE, dim=-1)
        assert (ref[0][b] - torch.einsum("hl,lhd->hd", p, V)).abs().max().item() < 1e-12


@gpu
def test_decode_attention_equal_scores():
    """q = 0: every score is 0 and the output is the plain average of the L + 1 V rows."""
    pt, lens, H = 32, [0, 31, 100, 257], 2
    case = make_case(pt, lens, H, splits=3, seed=33)
    case.partial[:, :, :H * HD] = 0.0
    ref = check_variants(case, [(1, 0, 0), (3, 0, 0), (8, 0, 0), (1, 1, 1)], "equal scores")
    for b, L in enumerate(lens):
        mean = torch.cat([gather_rows(case.pool, case.table[b], L, pt)[1].double(), ref[2][b].double()[None]]).mean(0)
        assert (ref[0][b] - mean).abs().max().item() < 1e-12


@gpu
@pytest.mark.parametrize("theta", [10000.0, 500.0])
@pytest.mark.parametrize("kernel", ["one-shot", "split", "persistent"])
def test_decode_attention_appended_row_is_what_the_next_step_reads(theta, kernel):
    """Step 1 appends a row at seq_len; step 2 runs at seq_len + 1 on the pool step 1 left, with a new q, against the reference on a
    pool holding the *reference's* row.  Step 2's own key and value are 0 and one sequence has a single cached key, so its output is
    decided by the score of the appended key and by its V."""
    pt, lens, H = 16, [1, 15, 16, 47, 300], 2
    kv_splits, persistent, grid = {"one-shot": (1, 0, 0), "split": (4, 0, 0), "persistent": (1, 1, 2)}[kernel]
    case = make_case(pt, lens, H, splits=2, seed=41, theta=theta, steps=2)
    ref1 = decode_ref(case.partial, case.pool, case.table, lens, pt, H, SCALE, theta)
    out1, pool1 = run_ok(case, kv_splits=kv_splits, persistent=persistent, grid=grid)
    check_result(case, out1, pool1, ref1, "two steps", f"step 1, {kernel}, theta {theta}")
    pages, slots = new_row_index(case)
    step2 = SimpleNamespace(**vars(case))
    step2.lens = [L + 1 for L in lens]
    step2.pool = case.pool.clone()
    step2.pool[pages, 0, :, slots] = ref1[1]
    step2.pool[pages, 1, :, slots] = ref1[2]
    step2.partial = torch.randn(case.partial.shape, generator=torch.Generator().manual_seed(42)) * 2.0
    step2.partial[:, :, H * HD:] = 0.0
    ref2 = decode_ref(step2.partial, step2.pool, step2.table, step2.lens, pt, H, SCALE, theta)
    out2, _ = run_ok(step2, kv_splits=kv_splits, persistent=persistent, grid=grid, pool=pool1)
    got = out2.view(len(lens), H, HD).double()
    err = (got - ref2[0]).abs().max().item() / max(1.0, ref2[0].abs().max().item())
    _note("two steps", err)
    assert torch.isfinite(got).all() and err <= OUT_TOL, f"step 2 after {kernel} step 1, theta {theta}: err {err:.3e}"


@gpu
@pytest.mark.parametrize("bad", ["seq_len beyond the table row", "negative seq_len", "page_tokens 12", "page_tokens 128", "page_tokens 0",
                                 "kv_splits 9", "kv_splits 0", "persistent with kv_splits 2", "unowned page", "launches 0"])
def test_decode_attention_refuses_bad_arguments(bad):
    """Refused on the host with a message; nothing is launched, so the pool is untouched."""
    from visualcla import _native as N
    case = make_case(16, [5, 10], 2, splits=2, seed=51)
    rows = case.table.shape[1] * 16
    kw = {"seq_len beyond the table row": dict(lens=[5, rows]), "negative seq_len": dict(lens=[-1, 10]),
          "page_tokens 12": dict(pt=12), "page_tokens 128": dict(pt=128), "page_tokens 0": dict(pt=0), "kv_splits 9": dict(kv_splits=9),
          "kv_splits 0": dict(kv_splits=0), "persistent with kv_splits 2": dict(kv_splits=2, persistent=1),
          "unowned page": dict(lens=[5, 16]), "launches 0": dict(launches=0)}[bad]
    rc, _, pool = run_op(case, **kw)
    assert rc != 0 and len(N.load().vcla_last_error()) > 10, bad
    assert torch.equal(pool.view(torch.int16), case.pool.view(torch.int16)), f"{bad}: the pool was written"
    out, _ = run_ok(case)                                          # and the next valid call works
    assert torch.isfinite(out.float()).all()


# ---------------------------------------------------------------------------------------------------------------------------------
# greedy argmax: logits = the fp32 sum of the partials in split order, token = the first index of the maximum.  A row that is -inf
# everywhere gives 0, as torch.argmax does: a column of the row, which the next step's embedding lookup can index.
# ---------------------------------------------------------------------------------------------------------------------------------
def argmax_op(partial, V, want_logits=True):
    from visualcla import _native as N
    lib = N.load()
    S, B, ldp = partial.shape
    part_d = partial.cuda()
    logits = torch.full((B, V), float("nan"), device="cuda") if want_logits else None
    tok = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    N.check(lib.vcla_op_logits_argmax(N.ptr(part_d), S, ldp, B, V, N.ptr(logits), N.ptr(tok), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
            "vcla_op_logits_argmax")
    torch.cuda.synchronize()
    return (logits.cpu() if want_logits else None), tok.cpu().long()


def tie_rows(V):
    """Integer-valued rows (sums of integer partials are exact) whose maximum is duplicated, with the index that must win.  Stage 1
    gives chunk c the columns [c * per, (c + 1) * per), per = ceil(V / 32), and thread t of 256 the columns c * per + t + 256 i; the
    names describe V = 32000 and 49958 (per >= 264), at a smaller V the same columns tie across other units."""
    per = (V + 31) // 32
    places = {"two lanes of a warp": (5, 9), "two warps of a chunk": (10, 200), "one thread, two trips": (7, 263),
              "two chunks": (per + 3, 20 * per + 1), "first and last column": (0, V - 1),
              "a later chunk, lanes": (17 * per + 33, 17 * per + 40), "a later chunk, warps": (17 * per + 2, 17 * per + 130),
              "chunk border": (per - 1, per), "three chunks": (3 * per + 1, 9 * per, 31 * per)}
    g = torch.Generator().manual_seed(V)
    rows, want, names = [], [], []
    for name, at in places.items():
        if max(at) >= V or len(set(at)) < len(at):
            continue
        row = torch.randint(-50, 50, (V,), generator=g).float()
        row[list(at)] = 100.0
        rows.append(row); want.append(min(at)); names.append(name)
    rows.append(torch.full((V,), 3.0)); want.append(0); names.append("constant row")
    return torch.stack(rows), torch.tensor(want), names


def split_integers(rows, splits, seed):
    """Integer partials [splits][B][V] whose sum is `rows`."""
    g = torch.Generator().manual_seed(seed)
    parts = [torch.randint(-20, 20, rows.shape, generator=g).float() for _ in range(splits - 1)]
    return torch.stack(parts + [rows - sum(parts)]) if parts else rows[None].clone()


@pytest.mark.parametrize("V", [33, 1003, 32000, 49958])
def test_tie_rows_are_what_they_claim(V):
    rows, want, names = tie_rows(V)
    assert len(names) >= (3 if V == 33 else 6)
    assert torch.equal(torch.argmax(rows, dim=-1), want)
    assert torch.equal((rows == rows.max(-1, keepdim=True).values).sum(-1) >= 2, torch.ones(len(names), dtype=torch.bool))
    assert torch.equal(sum_splits(split_integers(rows, 7, 1)), rows)
    assert int(torch.argmax(torch.full((V,), float("-inf")))) == 0


@gpu
@pytest.mark.parametrize("V", [7, 31, 33, 1003, 5003, 32000, 49958])
def test_logits_argmax_sweep(V):
    """Vocabulary sizes that leave trailing chunks empty (7, 31), ragged (33, 1003, 5003, 49958) or even (32000); the padding columns
    of the partials hold +inf and NaN and must not be read."""
    for splits in (1, 2, 7):
        for B in (1, 5, 64):
            g = torch.Generator().manual_seed(V + 100 * splits + B)
            ldp = V + 5
            partial = torch.empty(splits, B, ldp)
            partial[:, :, :V] = torch.randn(splits, B, V, generator=g)
            partial[:, :, V:] = torch.tensor([float("inf"), float("nan"), float("inf"), float("nan"), float("inf")])
            want = sum_splits(partial[:, :, :V].contiguous())
            logits, tok = argmax_op(partial, V)
            assert torch.equal(logits.view(torch.int32), want.view(torch.int32)), (V, splits, B)
            assert torch.equal(tok, torch.argmax(want, dim=-1)), (V, splits, B)
            _, tok2 = argmax_op(partial, V, want_logits=False)
            assert torch.equal(tok2, tok), (V, splits, B)


@gpu
@pytest.mark.parametrize("V", [33, 1003, 32000, 49958])
@pytest.mark.parametrize("splits", [1, 3])
def test_logits_argmax_ties(V, splits):
    """The smallest index wins among equal maxima: across lanes, warps, a thread's trips, the 32 chunks and stage 2."""
    rows, want, names = tie_rows(V)
    logits, tok = argmax_op(split_integers(rows, splits, V + splits), V)
    assert torch.equal(logits, rows)
    for name, t, w in zip(names, tok.tolist(), want.tolist()):
        assert t == w, f"V {V}, maximum in {name}: token {t}, want {w}"


@gpu
@pytest.mark.parametrize("V", [7, 1003, 32000])
@pytest.mark.parametrize("splits", [1, 2])
def test_logits_argmax_minus_infinity(V, splits):
    ninf = float("-inf")
    rows = torch.full((4, V), ninf)
    rows[0, V - 2] = -5.0                                         # one finite entry, in the last non-empty chunk
    rows[1, V // 2] = -1e30
    rows[3, :V // 2] = -3.0                                       # -inf tail
    partial = torch.stack([rows] + [torch.where(rows == ninf, rows, torch.zeros_like(rows))] * (splits - 1))
    logits, tok = argmax_op(partial, V)
    assert torch.equal(logits, rows)
    assert tok.tolist() == [V - 2, V // 2, 0, 0] == torch.argmax(rows, dim=-1).tolist()
