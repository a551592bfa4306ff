"""The two prefill attention kernels at operator level: attn_prefill_kernel (mma.sync, csrc/attention.cu: the ViT, the Resampler and
every call the wgmma kernel cannot describe) and attn_prefill_tc_kernel (wgmma, csrc/attention_tc.cu: LLaMA's causal prefill), both
through vcla_op_attention, against a float64 reference written from the definition.

Key j of sequence b is visible to query i iff kv_start[b] <= j < n0 + n1 and, when causal, j <= i + n0 + n1 - Sq; the softmax runs
over the visible keys and a query that sees none gets a row of zeros.

Hidden keys that share a 64-key tile with visible ones are loaded, so they cannot be NaN (P = 0 does not cancel a NaN in P V).
Instead they are decoys that a leak cannot hide: the last head dimension is a decoy channel -- every query has 1 there, every visible
key 0 --, and a decoy key is 0 everywhere except that channel, where it holds a power of two that scores 12 above the case's highest
visible score; its V row is DECOY_V in every column, far from the N(0, 1) visible values.  One leaked decoy then takes nearly all of
a row's weight.  Decoys fill the left padding of every sequence and 64 rows after the last sequence of every allocation.  In the
non-paged layout the rows after sequence b's end are sequence b + 1's first rows, so the multi-sequence cases left-pad the later
sequences and those rows are decoys too.  Causal-future keys are also visible keys of later rows, so they cannot be constant
decoys: the `ramp` cases give every key a score that rises by more than 1.4 per key (two more channels), so each key a row must not
see outscores every key it sees.

The metric is row-relative: the largest |out - ref| over a (sequence, query, head) row over the largest |ref| of that row (an
absolute bound would not see one leaked or dropped key behind a few hundred visible ones).  Rows with no visible key must be exactly
0.  out has a gap of columns after H * HD and rows after B * Sq, filled with a NaN pattern that must survive; every call runs twice
and must give the same bits.

The tests marked `gpu` need a device; the unmarked ones check the reference and the cases on the CPU (the reference against float64
torch.nn.functional.scaled_dot_product_attention), so a wrong reference cannot hide behind a skip."""
import ctypes as C
import math
import os
from types import SimpleNamespace

import pytest
import torch

gpu = pytest.mark.gpu

NAN_BITS = 0x7FC1          # a bf16 NaN; no kernel produces this payload
DECOY_V = 8.0
DECOY_MARGIN = 12.0        # a decoy scores this much above the case's highest visible score (natural log units)
PAD_ROWS = 64              # decoy rows after the last sequence of every K/V allocation
# max |out - ref| over a row / max |ref| of the row.  The output is one bf16 rounding of an fp32 result (up to 2^-8 = 3.9e-3 of the
# row's largest value) and P is rounded to bf16 before P V.  Largest values observed over both kernels (H100 80GB HBM3, 700 W):
# 6.0e-3 geometry sweep, 6.0e-3 left padding, 5.9e-3 production shapes, 5.9e-3 [q | k | v] layout, 5.4e-3 numerics,
# 5.2e-3 two segments, 5.1e-3 dispatch, 4.7e-3 causal future decoys, 4.6e-3 causal Sq < Sk.  The starting bound of 1e-2 is 1.66 times
# the largest and stays: what the cases catch is far larger (a leaked decoy takes most of a row; a dropped key moves a row that sees
# at most 1088 keys by about 1 / sqrt(1088) = 3e-2).
ROW_TOL = 1e-2

_observed = {}


def _note(group, err):
    _observed[group] = max(_observed.get(group, 0.0), err)


@pytest.fixture(scope="module", autouse=True)
def _report_observed():
    yield
    for group in sorted(_observed):
        print(f"\n[prefill-attention] largest row-relative error, {group}: {_observed[group]:.3e}", end="")
    print()


# ---------------------------------------------------------------------------------------------------------------------------------
# reference
# ---------------------------------------------------------------------------------------------------------------------------------
def visible(Sq, Sk, causal, kv0, device="cpu"):
    """(Sq, Sk) bool: key j visible to query i."""
    i = torch.arange(Sq, device=device)[:, None]
    j = torch.arange(Sk, device=device)[None, :]
    vis = (j >= kv0) & (j < Sk) & (i >= 0)
    if causal:
        vis = vis & (j <= i + (Sk - Sq))
    return vis


def attention_ref(q, k, v, kv_start, causal, scale):
    """q (B, Sq, H, HD), k / v (B, Sk, H, HD) on any device -> float64 (B, Sq, H, HD); rows with no visible key are 0."""
    B, Sq, H, HD = q.shape
    Sk = k.shape[1]
    out = torch.zeros(B, Sq, H, HD, dtype=torch.float64, device=q.device)
    for b in range(B):
        vis = visible(Sq, Sk, causal, 0 if kv_start is None else kv_start[b], q.device)
        s = torch.einsum("ihd,jhd->hij", q[b].double(), k[b].double()) * scale
        s = s.masked_fill(~vis, float("-inf"))
        m = s.amax(-1, keepdim=True)
        p = torch.exp(s - torch.where(torch.isfinite(m), m, torch.zeros_like(m)))
        l = p.sum(-1, keepdim=True)
        o = torch.einsum("hij,jhd->hid", p, v[b].double())
        out[b] = torch.where(l > 0, o / torch.where(l > 0, l, torch.ones_like(l)), torch.zeros_like(o)).transpose(0, 1)
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------------------
def later_pads(B, Sk):
    """Left padding of a multi-sequence case: sequence 0 none, the later ones min(63, Sk - 1), so that the rows after a sequence's end
    are decoys."""
    return None if B == 1 else [0] + [min(63, max(Sk - 1, 0))] * (B - 1)


def make_case(B, H, HD, Sq, n0, n1=0, causal=0, kv_start=None, scale=None, seed=0, q_std=1.0, k_std=1.0, ramp=0):
    """Seeded bf16 Q (B, Sq, H, HD) and K, V (B, n0 + n1, H, HD) with the decoy channel set; decoys are placed by finish()."""
    g = torch.Generator().manual_seed(seed)
    Sk = n0 + n1
    q = torch.randn(B, Sq, H, HD, generator=g) * q_std
    k = torch.randn(B, Sk, H, HD, generator=g) * k_std
    v = torch.randn(B, Sk, H, HD, generator=g)
    q[..., -1] = 1.0
    k[..., -1] = 0.0
    if ramp:
        # raw score ramp * j from two channels that bf16 holds exactly: 16 ramp * (j // 16) and ramp * (j % 16)
        j = torch.arange(Sk, dtype=torch.float32)
        q[..., -3:-1] = 1.0
        k[..., -2] = (ramp * 16 * (j // 16))[None, :, None]
        k[..., -3] = (ramp * (j % 16))[None, :, None]
    return SimpleNamespace(B=B, H=H, HD=HD, Sq=Sq, n0=n0, n1=n1, Sk=Sk, causal=causal, kv_start=kv_start,
                           scale=HD ** -0.5 if scale is None else scale, q=q.to(torch.bfloat16), k=k.to(torch.bfloat16),
                           v=v.to(torch.bfloat16), decoy=None)


def visible_all(case):
    """(B, Sq, Sk) bool."""
    return torch.stack([visible(case.Sq, case.Sk, case.causal, 0 if case.kv_start is None else case.kv_start[b]) for b in range(case.B)])


def raw_scores(case):
    """float64 q . k (B, H, Sq, Sk), unscaled."""
    return torch.einsum("bihd,bjhd->bhij", case.q.double(), case.k.double())


def finish(case):
    """Place the decoys: the key row (0 ..., A) with A a power of two that scores DECOY_MARGIN above every visible score of the case,
    the value row DECOY_V; in the left padding of every sequence and in the PAD_ROWS rows after the last one."""
    dev = "cuda" if torch.cuda.is_available() else "cpu"
    top = 0.0
    for b in range(case.B):
        vis = visible(case.Sq, case.Sk, case.causal, 0 if case.kv_start is None else case.kv_start[b], dev)
        if vis.any():
            s = torch.einsum("ihd,jhd->hij", case.q[b].to(dev).double(), case.k[b].to(dev).double())
            top = max(top, s[:, vis].max().item())
    A = 2.0 ** math.ceil(math.log2(top + DECOY_MARGIN / case.scale))
    case.decoy = torch.zeros(case.H, case.HD, dtype=torch.bfloat16)
    case.decoy[:, -1] = A
    assert case.decoy[0, -1].item() == A
    for b in range(case.B):
        p = 0 if case.kv_start is None else case.kv_start[b]
        case.k[b, :p] = case.decoy
        case.v[b, :p] = DECOY_V
    return case


def check_decoys(case):
    """Every decoy key outscores every visible key of every row by DECOY_MARGIN; with a ramp, every causal-future key of a row
    outscores every key the row sees."""
    s = raw_scores(case) * case.scale
    vis = visible_all(case)[:, None].expand_as(s)
    decoy_score = case.decoy[0, -1].double().item() * case.scale
    assert not vis.any() or decoy_score >= s[vis].max().item() + DECOY_MARGIN
    for b in range(case.B):
        p = 0 if case.kv_start is None else case.kv_start[b]
        assert (s[b, :, :, :p] == decoy_score).all()
    if case.causal:
        fut = torch.ones(case.Sq, case.Sk, dtype=torch.bool).triu(case.Sk - case.Sq + 1)
        return fut, s
    return None, s


# ---------------------------------------------------------------------------------------------------------------------------------
# the operator
# ---------------------------------------------------------------------------------------------------------------------------------
def _segment(k, v, stride, pad_value_k, pad_value_v, col0=0):
    """One K/V allocation: rows b * n + j hold K at columns [col0, col0 + D), V at [col0 + D, col0 + 2 D); PAD_ROWS decoy rows after."""
    B, n, H, HD = k.shape
    D = H * HD
    buf = torch.zeros(B * n + PAD_ROWS, stride, dtype=torch.bfloat16)
    buf[:B * n, col0:col0 + D] = k.reshape(B * n, D)
    buf[:B * n, col0 + D:col0 + 2 * D] = v.reshape(B * n, D)
    buf[B * n:, col0:col0 + D] = pad_value_k.reshape(D)
    buf[B * n:, col0 + D:col0 + 2 * D] = pad_value_v
    return buf


def run_op(case, o_stride=None, layout="split", seg1_layers=1, seg1_layer=0, kv_start=None, raw=False):
    """-> the output allocation (B * Sq + 8 rows, o_stride) bf16 on the device, or the return code when raw.
    layout "split": q (q_stride = D + 16) and [K | V] per segment (stride 2 D + 24); "qkv": one [q | k | v] buffer of stride 3 D, the
    vcla_vision_encode / vcla_prefill layout (self-attention, one segment).  seg1_layers > 1 puts segment 1 at layer `seg1_layer` of a
    [layers][K | V] row, the Resampler's image K/V."""
    from visualcla import _native as N
    lib = N.load()
    B, Sq, H, HD, n0, n1 = case.B, case.Sq, case.H, case.HD, case.n0, case.n1
    D = H * HD
    o_stride = D + 8 if o_stride is None else o_stride
    dv = torch.full((D,), DECOY_V, dtype=torch.bfloat16)
    keep = []
    if layout == "qkv":
        assert Sq == n0 and n1 == 0
        buf = _segment(case.k[:, :n0], case.v[:, :n0], 3 * D, case.decoy, dv, col0=D)
        buf[:B * Sq, :D] = case.q.reshape(B * Sq, D)
        buf = buf.cuda()
        keep.append(buf)
        base = buf.data_ptr()
        q_ptr, q_stride, k0, v0, kv0_stride = base, 3 * D, base + 2 * D, base + 4 * D, 3 * D
    else:
        qb = torch.randn(B * Sq + PAD_ROWS, D + 16, generator=torch.Generator().manual_seed(7)).to(torch.bfloat16)
        qb[:B * Sq, :D] = case.q.reshape(B * Sq, D)
        s0 = _segment(case.k[:, :n0], case.v[:, :n0], 2 * D + 24, case.decoy, dv)
        qb, s0 = qb.cuda(), s0.cuda()
        keep += [qb, s0]
        q_ptr, q_stride, k0, v0, kv0_stride = qb.data_ptr(), D + 16, s0.data_ptr(), s0.data_ptr() + 2 * D, 2 * D + 24
    k1 = v1 = None
    kv1_stride = 0
    if n1 > 0:
        stride1 = seg1_layers * 2 * D + (0 if seg1_layers > 1 else 8)
        s1 = _segment(case.k[:, n0:], case.v[:, n0:], stride1, case.decoy, dv, col0=seg1_layer * 2 * D).cuda()
        keep.append(s1)
        k1, v1, kv1_stride = s1.data_ptr() + seg1_layer * 4 * D, s1.data_ptr() + (seg1_layer * 2 + 1) * 2 * D, stride1
    ks = case.kv_start if kv_start is None else kv_start
    ks_d = None if ks is None else torch.tensor(ks, dtype=torch.int32, device="cuda")
    out = torch.full((B * Sq + 8, o_stride), NAN_BITS, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    rc = lib.vcla_op_attention(C.c_void_p(q_ptr), q_stride, C.c_void_p(k0), C.c_void_p(v0), kv0_stride, n0, C.c_void_p(k1) if k1 else None,
                               C.c_void_p(v1) if v1 else None, kv1_stride, n1, N.ptr(out), o_stride, B, H, Sq, HD, C.c_float(case.scale),
                               case.causal, C.c_void_p(torch.cuda.current_stream().cuda_stream), N.ptr(ks_d))
    torch.cuda.synchronize()
    if raw:
        return rc, out
    N.check(rc, "vcla_op_attention")
    return out


def row_err(got, ref):
    """max over (sequence, query, head) rows with a visible key of max |got - ref| / max |ref| of the row."""
    scale = ref.abs().amax(-1)
    live = scale > 0
    if not live.any():
        return 0.0
    return ((got - ref).abs().amax(-1)[live] / scale[live]).max().item()


def check(case, group, modes=None, **kw):
    """Run the case under every mode of `modes` (default: the current one) twice each and check it: -> {mode: output allocation}."""
    ref = attention_ref(case.q.cuda(), case.k.cuda(), case.v.cuda(), case.kv_start, case.causal, case.scale)
    empty = torch.stack([visible_all(case)[b].any(-1) for b in range(case.B)]).logical_not().cuda()   # (B, Sq) rows that see no key
    D = case.H * case.HD
    what = f"{group}: B {case.B} H {case.H} HD {case.HD} Sq {case.Sq} n0 {case.n0} n1 {case.n1} causal {case.causal} " \
           f"kv_start {case.kv_start} scale {case.scale:.4g}"
    out = run_op(case, **kw)
    again = run_op(case, **kw)
    assert torch.equal(out.view(torch.int16), again.view(torch.int16)), f"{what}: two calls differ"
    o_bits = out.view(torch.int16)
    assert (o_bits[:, D:] == NAN_BITS).all(), f"{what}: a column after H * HD was written"
    assert (o_bits[case.B * case.Sq:] == NAN_BITS).all(), f"{what}: a row after B * Sq was written"
    got = out[:case.B * case.Sq, :D].view(case.B, case.Sq, case.H, case.HD).double()
    assert torch.isfinite(got).all(), f"{what}: {int((~torch.isfinite(got)).sum())} elements not written or not finite"
    assert (got[empty] == 0).all(), f"{what}: a query that sees no key has a nonzero output"
    err = row_err(got, ref)
    _note(group, err)
    assert err <= ROW_TOL, f"{what}: row-relative error {err:.3e}"
    return out


@pytest.fixture(scope="module")
def lib():
    from visualcla import _native as N
    return N.load()


def _restore_mode(lib):
    lib.vcla_set_attention_tc(int(os.environ.get("VCLA_ATTN_TC", "1")))


@pytest.fixture(params=[0, 2], ids=["mma_sync", "wgmma"])
def kernel(request, lib):
    """Mode 0 runs every call on the mma.sync kernel, mode 2 every call the wgmma kernel can describe on the wgmma kernel."""
    lib.vcla_set_attention_tc(request.param)
    yield request.param
    _restore_mode(lib)


# ---------------------------------------------------------------------------------------------------------------------------------
# the reference and the cases themselves (CPU)
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Sq,n0,n1,causal,kv_start,scale", [
    (65, 65, 0, 1, [0, 1, 64, 65], None), (17, 200, 0, 1, [0, 3, 150, 200], None), (1, 65, 0, 1, [0, 64, 65, 2], 0.3),
    (64, 64, 257, 0, [0, 63, 100, 321], None), (70, 130, 0, 0, [0, 129, 130, 5], 0.01), (9, 17, 100, 1, None, None)])
def test_reference_equals_sdpa(Sq, n0, n1, causal, kv_start, scale):
    """Rows with a visible key: float64 scaled_dot_product_attention with the boolean mask; rows without one: exactly 0."""
    B, H, HD = (4 if kv_start else 2), 2, 64
    case = make_case(B, H, HD, Sq, n0, n1, causal, kv_start, scale, seed=Sq + n0)
    ref = attention_ref(case.q, case.k, case.v, kv_start, causal, case.scale)
    q, k, v = (t.double().transpose(1, 2) for t in (case.q, case.k, case.v))
    for b in range(B):
        vis = visible(Sq, n0 + n1, causal, 0 if kv_start is None else kv_start[b])
        live = vis.any(-1)
        want = torch.nn.functional.scaled_dot_product_attention(q[b], k[b], v[b], attn_mask=vis, scale=case.scale).transpose(0, 1)
        assert (ref[b][live] - want[live]).abs().max().item() < 1e-12 if live.any() else True
        assert (ref[b][~live] == 0).all()
    if kv_start:
        assert any(not visible(Sq, n0 + n1, causal, p).any(-1).all() for p in kv_start), "the case has rows that see no key"


def test_reference_softmax_is_plain():
    """Hand-sized: keys of scores 0, ln 3 and 50.  Causal with Sq = 2 < Sk = 3, query 0 sees keys 0 and 1 (weights 1/4 and 3/4) and
    query 1 all three; kv_start 1 leaves query 0 key 1 alone, kv_start 3 leaves nothing."""
    q = torch.zeros(1, 1, 1, 2, dtype=torch.float64)
    q[..., 0] = 1.0
    k = torch.tensor([[0.0, 0.0], [math.log(3.0), 0.0], [50.0, 0.0]], dtype=torch.float64).view(1, 3, 1, 2)
    v = torch.tensor([[4.0, 0.0], [0.0, 8.0], [1e3, 1e3]], dtype=torch.float64).view(1, 3, 1, 2)
    q2 = torch.cat([q, q], 1)
    out = attention_ref(q2, k, v, None, 1, 1.0)
    assert torch.allclose(out[0, 1, 0], torch.softmax(torch.tensor([0.0, math.log(3.0), 50.0], dtype=torch.float64), 0) @ v[0, :, 0])
    assert torch.allclose(out[0, 0, 0], torch.tensor([1.0, 6.0], dtype=torch.float64))
    out = attention_ref(q2, k, v, [1], 1, 1.0)                  # kv_start 1: query 0 sees key 1 alone
    assert torch.allclose(out[0, 0, 0], torch.tensor([0.0, 8.0], dtype=torch.float64))
    assert torch.equal(attention_ref(q2, k, v, [3], 1, 1.0), torch.zeros(1, 2, 1, 2, dtype=torch.float64))


@pytest.mark.parametrize("HD", [64, 128])
def test_decoys_outscore_visible_keys(HD):
    """The decoys of a left-padded causal case and the ramp of a ramp case are what they claim."""
    case = finish(make_case(3, 2, HD, 130, 130, causal=1, kv_start=[0, 63, 65], seed=HD))
    check_decoys(case)
    case = finish(make_case(2, 2, HD, 90, 200, causal=1, kv_start=[0, 70], seed=HD + 1, q_std=0.25, k_std=0.25, ramp=16))
    fut, s = check_decoys(case)
    vis = visible_all(case)
    for b in range(case.B):
        for i in range(case.Sq):
            if vis[b, i].any() and fut[i].any():
                # the first hidden key alone outweighs everything the row sees: a leak of it moves the row by O(1)
                gap = s[b, :, i, fut[i]].min(-1).values - s[b, :, i, vis[b, i]].max(-1).values
                assert gap.min().item() >= 0.5
                assert (torch.exp(s[b, :, i, fut[i]][:, 0]) > torch.exp(s[b, :, i, vis[b, i]]).sum(-1)).all()


# ---------------------------------------------------------------------------------------------------------------------------------
# geometry (both kernels)
# ---------------------------------------------------------------------------------------------------------------------------------
SWEEP_S = [1, 2, 63, 64, 65, 127, 128, 129, 257, 300, 640, 1088]


@gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("S", SWEEP_S)
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("HD", [64, 128])
def test_prefill_geometry(kernel, HD, causal, S, B):
    """Self-attention over S keys: one partial or full query tile, one partial or full key tile, and up to 17 of each.  B = 3 left-pads
    sequences 1 and 2, so the tile tail after sequence 0 and 1 reads decoys."""
    case = finish(make_case(B, 2, HD, S, S, causal=causal, kv_start=later_pads(B, S), seed=S * 10 + HD + causal + B))
    check(case, "geometry")


@gpu
@pytest.mark.parametrize("B,H,S,HD,causal", [(2, 16, 257, 64, 0), (3, 2, 17, 64, 0), (2, 32, 96, 128, 1), (1, 4, 200, 128, 1),
                                              (2, 2, 64, 128, 1), (1, 2, 1, 128, 1), (2, 4, 128, 128, 1), (1, 2, 1088, 128, 1),
                                              (2, 3, 300, 64, 1), (1, 2, 640, 64, 0)])
def test_prefill_self_attention_qkv_layout(kernel, B, H, S, HD, causal):
    """Interleaved [q | k | v] rows of stride 3 H HD, without padding."""
    case = finish(make_case(B, H, HD, S, S, causal=causal, seed=20 + S + H))
    check(case, "qkv layout", layout="qkv")


# ---------------------------------------------------------------------------------------------------------------------------------
# left padding
# ---------------------------------------------------------------------------------------------------------------------------------
def _pads(S):
    """Per-sequence left padding around the tile boundaries, largest first so that most tile tails read the next sequence's decoys."""
    return sorted({min(p, S) for p in (0, 1, 63, 64, 65, 127, S - 1, S)}, reverse=True)


@gpu
@pytest.mark.parametrize("S", [65, 200, 1088])
def test_prefill_left_padding_causal(kernel, S):
    """Causal, head dim 128: kv_start at and around tile boundaries (key tiles left of kv_start are skipped, the first kept one is
    partly hidden), S - 1 (one key: the last query's own) and S (every row 0, no key tile at all when S is a multiple of 64)."""
    pads = _pads(S)
    case = finish(make_case(len(pads), 2, 128, S, S, causal=1, kv_start=pads, seed=300 + S))
    check(case, "left padding")


@gpu
@pytest.mark.parametrize("S", [65, 257])
def test_prefill_left_padding_noncausal(kernel, S):
    pads = _pads(S)
    case = finish(make_case(len(pads), 2, 64, S, S, causal=0, kv_start=pads, seed=400 + S))
    check(case, "left padding")


@gpu
@pytest.mark.parametrize("HD", [64, 128])
@pytest.mark.parametrize("Sq,n0", [(17, 200), (64, 129), (1, 65)])
def test_prefill_causal_fewer_queries(kernel, HD, Sq, n0):
    """Sq < Sk: query i sees keys up to i + Sk - Sq, so the last query sees every key."""
    case = finish(make_case(2, 2, HD, Sq, n0, causal=1, kv_start=[0, min(63, n0 - 1)], seed=500 + Sq + HD))
    check(case, "causal Sq < Sk")


@gpu
@pytest.mark.parametrize("HD", [64, 128])
@pytest.mark.parametrize("Sq,n0", [(65, 65), (300, 300), (17, 200), (129, 129)])
def test_prefill_causal_future_decoys(kernel, HD, Sq, n0):
    """Scores ramp up by more than 1.4 per key: every key past a row's diagonal, in the diagonal tile, outscores every key the row
    sees, and a row's weight sits on its last few visible keys."""
    case = finish(make_case(2, 2, HD, Sq, n0, causal=1, kv_start=[0, min(70, n0 - 1)], seed=600 + Sq + HD, q_std=0.25, k_std=0.25,
                            ramp=16))
    check(case, "causal future decoys")


# ---------------------------------------------------------------------------------------------------------------------------------
# two KV segments
# ---------------------------------------------------------------------------------------------------------------------------------
@gpu
def test_prefill_two_segments_resampler(kernel):
    """vcla_vision_encode's Resampler call: 64 queries over [their own 64 rows ; 257 image rows], H = 16, head dim 64; the image K/V
    are layer 1 of a [3 layers][K | V] row."""
    case = finish(make_case(2, 16, 64, 64, 64, 257, seed=21))
    check(case, "two segments", layout="split", seg1_layers=3, seg1_layer=1)


@gpu
@pytest.mark.parametrize("n0,n1", [(17, 100), (65, 1), (1, 257)])
def test_prefill_two_segments_unaligned(kernel, n0, n1):
    case = finish(make_case(3, 2, 64, n0, n0, n1, kv_start=later_pads(3, n0 + n1), seed=700 + n0 + n1))
    check(case, "two segments")


# ---------------------------------------------------------------------------------------------------------------------------------
# numerics
# ---------------------------------------------------------------------------------------------------------------------------------
def _boost(case, keys, score):
    """Keys `keys` of every sequence score about `score` more than the rest for every query (channel HD - 2)."""
    case.q[..., -2] = 1.0
    case.k[..., -2] = 0.0
    case.k[:, keys, :, -2] = score / case.scale
    return case


@gpu
@pytest.mark.parametrize("HD", [64, 128])
@pytest.mark.parametrize("where", ["first tile", "last partial tile"])
def test_prefill_one_dominant_key(kernel, HD, where):
    """One key scores about 80 above the rest: every row is that key's V row."""
    Sk = 300
    j = 2 if where == "first tile" else Sk - 3
    case = finish(_boost(make_case(2, 2, HD, 65, Sk, seed=800 + HD, k_std=0.05), [j], 80.0))
    ref = attention_ref(case.q, case.k, case.v, None, 0, case.scale)
    assert (ref - case.v[:, j][:, None].double()).abs().max().item() < 1e-12          # the case is what it claims to be
    check(case, "numerics")


@gpu
@pytest.mark.parametrize("HD", [64, 128])
@pytest.mark.parametrize("causal", [0, 1])
@pytest.mark.parametrize("order", ["maximum last", "maximum first"])
def test_prefill_rescale(kernel, HD, causal, order):
    """Ten key tiles; the keys of one tile score about 40 above the others.  Last: every earlier tile's partial sum is rescaled by
    about e^-40 when that tile arrives; first: the later tiles add about e^-40 each."""
    Sk = 640
    keys = list(range(Sk - 64, Sk)) if order == "maximum last" else list(range(64))
    case = finish(_boost(make_case(1, 2, HD, Sk if causal else 64, Sk, causal=causal, seed=900 + HD + causal), keys, 40.0))
    check(case, "numerics")


@gpu
@pytest.mark.parametrize("causal", [0, 1])
def test_prefill_equal_scores(kernel, causal):
    """q = 0 outside the decoy channel: every visible score is 0 and a row is the plain mean of the V rows it sees."""
    case = make_case(3, 2, 128, 200, 200, causal=causal, kv_start=[0, 64, 65], seed=1000 + causal)
    case.q[..., :-1] = 0.0
    finish(case)
    ref = attention_ref(case.q, case.k, case.v, case.kv_start, causal, case.scale)
    for b, p in enumerate(case.kv_start):
        for i in (0, 99, 199):
            hi = i + 1 if causal else 200
            if hi > p:
                assert (ref[b, i] - case.v[b, p:hi].double().mean(0)).abs().max().item() < 1e-12
    check(case, "numerics")


@gpu
@pytest.mark.parametrize("HD", [64, 128])
@pytest.mark.parametrize("scale", [0.3, 0.01])
def test_prefill_scale(kernel, HD, scale):
    """A softmax scale other than HD^-0.5: 0.3 makes the rows peaked, 0.01 nearly flat."""
    case = finish(make_case(2, 2, HD, 129, 129, causal=1, kv_start=[0, 40], scale=scale, seed=1100 + HD))
    check(case, "numerics")


# ---------------------------------------------------------------------------------------------------------------------------------
# production shapes and the dispatch
# ---------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("shape", ["vit B8", "llama B8 padded", "llama B1 S1088", "llama B64"])
def test_prefill_production_shapes(lib, mode, shape):
    """The engine's calls: the ViT's self-attention (257 tokens, 16 heads of 64, [q | k | v] rows) and LLaMA-7B's causal prefill
    (32 heads of 128, [q | k | v] rows, left padding for batched prompts of different lengths), output rows of H HD."""
    B, H, HD, S, causal, pads = {"vit B8": (8, 16, 64, 257, 0, None),
                                 "llama B8 padded": (8, 32, 128, 600, 1, [0, 17, 64, 100, 300, 599, 1, 250]),
                                 "llama B1 S1088": (1, 32, 128, 1088, 1, None),
                                 "llama B64": (64, 32, 128, 48, 1, None)}[shape]
    lib.vcla_set_attention_tc(mode)
    try:
        case = finish(make_case(B, H, HD, S, S, causal=causal, kv_start=pads, seed=1200 + B + S))
        check(case, "production shapes", layout="qkv", o_stride=H * HD)
    finally:
        _restore_mode(lib)


@gpu
@pytest.mark.parametrize("HD,causal,n1", [(128, 1, 0), (64, 0, 0), (64, 1, 100)])
def test_prefill_dispatch_falls_back_to_mma_sync(lib, HD, causal, n1):
    """Mode 2 sends a call the wgmma kernel cannot describe -- an output stride that is not a multiple of 8, or causal attention over
    two segments -- to the mma.sync kernel: the bits are mode 0's.  With a describable call the two kernels' bits differ, so the
    comparison can tell them apart."""
    case = finish(make_case(2, 2, HD, 130, 130, n1, causal=causal, kv_start=[0, 63], seed=1300 + HD + n1))
    D = 2 * HD
    try:
        outs = {}
        for mode in (0, 2):
            lib.vcla_set_attention_tc(mode)
            for o_stride in (D + 2, D + 8):
                outs[mode, o_stride] = check(case, "dispatch", o_stride=o_stride)[:, :D].contiguous().view(torch.int16)
    finally:
        _restore_mode(lib)
    assert torch.equal(outs[2, D + 2], outs[0, D + 2]), "mode 2 with an output stride of D + 2 did not run the mma.sync kernel"
    assert torch.equal(outs[0, D + 8], outs[0, D + 2]), "the mma.sync kernel's result depends on the output stride"
    if n1 == 0:
        assert not torch.equal(outs[2, D + 8], outs[0, D + 8]), "mode 2 with a describable call gave the mma.sync kernel's bits"
    else:
        assert torch.equal(outs[2, D + 8], outs[0, D + 8]), "causal attention over two segments did not run the mma.sync kernel"


@gpu
@pytest.mark.parametrize("bad", ["kv_start -1", "kv_start n0 + n1 + 1"])
def test_prefill_refuses_kv_start_out_of_range(lib, bad):
    """Refused on the host with a message before any launch: the output keeps its NaN pattern; the next valid call works."""
    case = finish(make_case(2, 2, 128, 65, 65, causal=1, kv_start=[0, 3], seed=1400))
    ks = {"kv_start -1": [0, -1], "kv_start n0 + n1 + 1": [66, 0]}[bad]
    rc, out = run_op(case, kv_start=ks, raw=True)
    assert rc != 0 and b"kv_start" in lib.vcla_last_error(), bad
    assert (out.view(torch.int16) == NAN_BITS).all(), f"{bad}: the output was written"
    check(case, "left padding")
