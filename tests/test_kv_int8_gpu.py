"""The int8 KV cache (kv_cache_dtype="int8", kv_format 1) on the device.

Operators: the decode attention (attn_decode_kernel, attn_decode_persistent_kernel, and the prompt lookup launches) on a caller pool in
the int8 layout through vcla_op_attention_decode_q8 / vcla_op_attention_decode_lookup_q8, against a float64 reference over the
dequantised rows (tests/kv_int8_reference.py).  Every scale that does not belong to a valid cached row is NaN, so a read past the
cached rows poisons the output, and every byte of the pool but the appended row must come back unchanged.

The paged prefill attention (attn_prefill_tc_kernel<128, true, KV_INT8>) through vcla_op_attention_paged_q8 against float64 on the
dequantised rows: prefixes across tile and page boundaries, the full grid, split determinism.

Path: the rows the fused QKV prefill epilogue stores; the logits of the prefill and of every decode step (teacher-forced) against the
oracle with the K/V round trip at the tiny and mid configs and at 7B widths (8 layers), alone and with load_in_8bit; graph replays
against eager steps; prompt lookup and streaming; sampled tokens against oracle/sampler_oracle.py; beams against the hooked
oracle/beam_oracle.py; extension of cached sequences and a reused chat turn; the page allocator, the memory formula and the 7B
capacity claim."""
import ctypes as C
import math
from types import SimpleNamespace

import pytest
import torch

import visualcla_oracle as O
from kv_int8_reference import dequantize_rows, generate_greedy_q8, llama_forward_q8, pool_bytes, quantize_rows, split_pool, ulp_distance
from test_decode_attention_gpu import OUT_TOL, SCALE, rope_ref, sum_splits

gpu = pytest.mark.gpu
HD = 128
FILL_Q = 77                      # int8 bytes of rows nobody wrote; their scales are NaN


# ---------------------------------------------------------------------------------------------------------------------------------
# operators
# ---------------------------------------------------------------------------------------------------------------------------------
def make_case(pt, lens, H, splits, seed, theta=10000.0, steps=1, spare_entries=2):
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    owned = [(L + steps - 1) // pt + 1 for L in lens]
    pps = max(owned) + spare_entries
    n_pages = sum(owned) + 3
    perm = torch.randperm(n_pages, generator=g).to(torch.int32)
    table = torch.full((B, pps), -1, dtype=torch.int32)
    q = torch.full((n_pages, 2, H, pt, HD), FILL_Q, dtype=torch.int8)
    s = torch.full((n_pages, 2, H, pt), float("nan"), dtype=torch.float32)
    at = 0
    for b, L in enumerate(lens):
        table[b, :owned[b]] = perm[at:at + owned[b]]
        at += owned[b]
        j = torch.arange(L)
        pages, slots = table[b, j // pt].long(), j % pt
        for kv in (0, 1):
            rq, rs = quantize_rows(torch.randn(L, H, HD, generator=g) * (1.0 + 3.0 * kv))
            q[pages, kv, :, slots] = rq
            s[pages, kv, :, slots] = rs
    partial = torch.randn(splits, B, 3 * H * HD, generator=g) / math.sqrt(splits)
    return SimpleNamespace(pt=pt, lens=list(lens), H=H, B=B, theta=theta, partial=partial, q=q, s=s, table=table, n_pages=n_pages)


def decode_ref(case, row_lens=None, partial=None):
    """(out (B, H, 128) float64, new rows {kq, ks, vq, vs}) for sequence b at length row_lens[b] of the case's pool."""
    lens = case.lens if row_lens is None else row_lens
    partial = case.partial if partial is None else partial
    B = len(lens)
    qkv = sum_splits(partial).view(B, 3, case.H, HD)
    out = torch.empty(B, case.H, HD, dtype=torch.float64)
    kq, ks = quantize_rows(torch.stack([rope_ref(qkv[b, 1].double(), L, case.theta).float() for b, L in enumerate(lens)]))
    vq, vs = quantize_rows(qkv[:, 2])
    for b, L in enumerate(lens):
        qr = rope_ref(qkv[b, 0].double(), L, case.theta)
        j = torch.arange(L)
        tb = case.table[0 if row_lens is not None else b]
        pages, slots = tb[j // case.pt].long(), j % case.pt
        K = torch.cat([case.q[pages, 0, :, slots].double() * case.s[pages, 0, :, slots].double()[..., None],
                       (kq[b].double() * ks[b].double()[:, None])[None]])
        V = torch.cat([case.q[pages, 1, :, slots].double() * case.s[pages, 1, :, slots].double()[..., None],
                       (vq[b].double() * vs[b].double()[:, None])[None]])
        p = torch.softmax(torch.einsum("hd,lhd->hl", qr, K) * SCALE, dim=-1)
        out[b] = torch.einsum("hl,lhd->hd", p, V)
    return out, dict(kq=kq, ks=ks, vq=vq, vs=vs)


def run_decode(case, kv_splits, persistent=0, grid=0, launches=1):
    from visualcla import _native as N
    lib = N.load()
    pool = pool_bytes(case.q, case.s).cuda()
    out = torch.empty(case.B, case.H * HD, dtype=torch.bfloat16, device="cuda")
    lens = torch.tensor(case.lens, dtype=torch.int32, device="cuda")
    table = case.table.cuda()
    part = case.partial.cuda()
    N.check(lib.vcla_op_attention_decode_q8(N.ptr(part), part.shape[0], N.ptr(pool), case.n_pages, N.ptr(table), table.shape[1], case.pt,
                                            N.ptr(lens), N.ptr(out), case.B, case.H, kv_splits, C.c_float(SCALE), C.c_float(case.theta),
                                            persistent, grid, launches, None), "vcla_op_attention_decode_q8")
    return out.cpu().view(case.B, case.H, HD), pool.cpu()


def check_append(case, raw, new, lens, seq_of_row=None):
    """The appended rows against the reference quantiser; every other byte of the pool unchanged."""
    q, s = split_pool(raw, case.n_pages, case.H, case.pt)
    exp_q, exp_s = case.q.clone(), case.s.clone()
    for r, L in enumerate(lens):
        b = r if seq_of_row is None else seq_of_row
        page, slot = int(case.table[b, L // case.pt]), L % case.pt
        gk, gks = q[page, 0, :, slot], s[page, 0, :, slot]
        gv, gvs = q[page, 1, :, slot], s[page, 1, :, slot]
        assert torch.equal(gv, new["vq"][r]) and torch.equal(gvs, new["vs"][r]), "V row: the quantiser of the split-order fp32 sum"
        dk = (gk.int() - new["kq"][r].int()).abs()
        assert dk.max() <= 1 and (dk == 0).float().mean() >= 0.99, f"K row q: max diff {int(dk.max())}"
        assert ulp_distance(gks, new["ks"][r]).max() <= 2
        exp_q[page, :, :, slot] = q[page, :, :, slot]
        exp_s[page, :, :, slot] = s[page, :, :, slot]
    assert torch.equal(pool_bytes(exp_q, exp_s), raw), "bytes outside the appended rows changed"


DECODE_CASES = [
    # (page_tokens, lens, heads, qkv splits, kv splits, persistent, grid)
    (8, [0, 1, 7, 8, 9, 33], 4, 1, 1, 0, 0),
    (16, [15, 16, 17, 300], 4, 3, 2, 0, 0),
    (64, [1, 63, 64, 65, 700, 1500], 4, 2, 4, 0, 0),
    (64, [1500, 3, 1001], 2, 1, 8, 0, 0),
    (16, [5, 129, 1000, 64], 3, 2, 1, 1, 2),
    (64, [700, 1, 130], 4, 2, 1, 1, 0),
    (8, [250] * 3, 5, 1, 3, 0, 0),
]


@gpu
@pytest.mark.parametrize("pt,lens,H,splits,kv_splits,persistent,grid", DECODE_CASES)
def test_decode_q8_operator(pt, lens, H, splits, kv_splits, persistent, grid):
    case = make_case(pt, lens, H, splits, seed=pt * 1000 + len(lens) + kv_splits)
    out, raw = run_decode(case, kv_splits, persistent, grid)
    ref, new = decode_ref(case)
    err = (out.double() - ref).abs().max().item()
    assert err <= OUT_TOL * max(1.0, ref.abs().max().item()), err
    check_append(case, raw, new, lens)
    out3, raw3 = run_decode(case, kv_splits, persistent, grid, launches=3)
    assert torch.equal(out3.view(torch.int16), out.view(torch.int16)) and torch.equal(raw3, raw), "repeated launches are bit-identical"


@gpu
@pytest.mark.parametrize("B", [1, 8, 32, 64])
@pytest.mark.parametrize("persistent", [0, 1])
def test_decode_q8_7b_heads(B, persistent):
    g = torch.Generator().manual_seed(B)
    lens = torch.randint(1, 260, (B,), generator=g).tolist()
    case = make_case(64, lens, 32, 4, seed=B + 7)
    out, raw = run_decode(case, 1, persistent)
    ref, new = decode_ref(case)
    assert (out.double() - ref).abs().max().item() <= OUT_TOL * max(1.0, ref.abs().max().item())
    check_append(case, raw, new, lens)


@gpu
@pytest.mark.parametrize("pt,L,rows,kv_splits", [(8, 37, 4, 1), (64, 700, 16, 4), (16, 0, 3, 2)])
def test_lookup_q8_rows_equal_one_token_calls(pt, L, rows, kv_splits):
    from visualcla import _native as N
    lib = N.load()
    case = make_case(pt, [L], 4, 2, seed=L + rows, steps=rows)
    g = torch.Generator().manual_seed(9)
    case.partial = torch.randn(2, rows, 3 * case.H * HD, generator=g)
    pool = pool_bytes(case.q, case.s).cuda()
    out = torch.empty(rows, case.H * HD, dtype=torch.bfloat16, device="cuda")
    lens = torch.tensor([L], dtype=torch.int32, device="cuda")
    table = case.table.cuda()
    part = case.partial.cuda()
    N.check(lib.vcla_op_attention_decode_lookup_q8(N.ptr(part), 2, N.ptr(pool), case.n_pages, N.ptr(table), table.shape[1], pt, N.ptr(lens),
                                                   N.ptr(out), rows, case.H, kv_splits, C.c_float(SCALE), C.c_float(case.theta), None),
            "vcla_op_attention_decode_lookup_q8")
    after = pool.cpu()
    ref, new = decode_ref_rows(case, L, rows, after)
    check_append(case, after, new, [L + r for r in range(rows)], seq_of_row=0)
    assert (out.cpu().double().view(rows, case.H, HD) - ref).abs().max() <= OUT_TOL * max(1.0, ref.abs().max().item())
    # row r = the one-token call at length L + r over the pool the lookup call left (its rows r.. are rewritten with the same bytes)
    for r in range(rows):
        one = torch.empty(1, case.H * HD, dtype=torch.bfloat16, device="cuda")
        p = after.clone().cuda()
        lr = torch.tensor([L + r], dtype=torch.int32, device="cuda")
        pr = part[:, r:r + 1].contiguous()
        N.check(lib.vcla_op_attention_decode_q8(N.ptr(pr), 2, N.ptr(p), case.n_pages, N.ptr(table), table.shape[1], pt, N.ptr(lr), N.ptr(one),
                                                1, case.H, kv_splits, C.c_float(SCALE), C.c_float(case.theta), 0, 0, 1, None),
                "vcla_op_attention_decode_q8")
        assert torch.equal(one.view(torch.int16), out[r:r + 1].view(torch.int16)), f"row {r}"


def decode_ref_rows(case, L, rows, raw):
    """Reference of the verification rows: row r attends over the pool's first L + r rows (lower rows as the device stored them)."""
    q, s = split_pool(raw, case.n_pages, case.H, case.pt)
    view = SimpleNamespace(**{**vars(case), "q": q, "s": s})
    outs, news = [], []
    for r in range(rows):
        o, n = decode_ref(view, row_lens=[L + r], partial=case.partial[:, r:r + 1])
        outs.append(o[0]); news.append(n)
    new = {k: torch.stack([n[k][0] for n in news]) for k in news[0]}
    return torch.stack(outs), new


def _paged_case_q8(pt, lens, T, H, seed):
    """q and the K/V of sequence b's first lens[b] + T tokens, quantised per row, scattered over a permuted int8 pool whose other rows
    hold NaN scales.  -> q, q8 rows, scales, table, dequantised K / V per sequence (float64)."""
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    pps = max(1, math.ceil((max(lens) + T) / pt))
    n_pages = B * pps + 3
    table = torch.randperm(n_pages, generator=g)[: B * pps].view(B, pps).to(torch.int32)
    rq = torch.full((n_pages, 2, H, pt, HD), FILL_Q, dtype=torch.int8)
    rs = torch.full((n_pages, 2, H, pt), float("nan"), dtype=torch.float32)
    q = torch.randn(B, T, H, HD, generator=g).to(torch.bfloat16)
    ks, vs = [], []
    for b, L in enumerate(lens):
        j = torch.arange(L + T)
        pages, slots = table[b, j // pt].long(), j % pt
        deq = []
        for kv in (0, 1):
            xq, xs = quantize_rows(torch.randn(L + T, H, HD, generator=g) * (1.0 + kv))
            rq[pages, kv, :, slots] = xq
            rs[pages, kv, :, slots] = xs
            deq.append(xq.double() * xs.double()[..., None])
        ks.append(deq[0]); vs.append(deq[1])
    return q, rq, rs, table, ks, vs, n_pages


def _paged_ref_q8(q, ks, vs, lens):
    B, T, H, _ = q.shape
    out = torch.empty(B, T, H, HD, dtype=torch.float64)
    for b, L in enumerate(lens):
        qf, kf, vf = q[b].double().transpose(0, 1), ks[b].transpose(0, 1), vs[b].transpose(0, 1)
        sc = qf @ kf.transpose(1, 2) * SCALE
        vis = torch.arange(L + T)[None, :] <= (L + torch.arange(T))[:, None]
        sc = sc.masked_fill(~vis[None], float("-inf"))
        out[b] = (torch.softmax(sc, -1) @ vf).transpose(0, 1)
    return out


def _paged_run_q8(q, rq, rs, table, lens, pt, n_pages):
    from visualcla import _native as N
    lib = N.load()
    B, T, H, _ = q.shape
    qd, pd, td = q.reshape(B * T, H * HD).cuda(), pool_bytes(rq, rs).cuda(), table.cuda()
    ld = torch.tensor(lens, dtype=torch.int32, device="cuda")
    out = torch.zeros(B * T, H * HD, dtype=torch.bfloat16, device="cuda")
    N.check(lib.vcla_op_attention_paged_q8(N.ptr(qd), H * HD, N.ptr(pd), n_pages, N.ptr(td), table.shape[1], pt, N.ptr(ld), N.ptr(out),
                                           H * HD, B, H, T, C.c_float(SCALE), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
            "vcla_op_attention_paged_q8")
    return out.view(B, T, H, HD).double().cpu()


def _row_err(got, ref):
    """max over (sequence, row, head) of the error relative to that output row's largest |value| (tests/test_kv_reuse_gpu.py)."""
    return ((got - ref).abs().amax(-1) / ref.abs().amax(-1).clamp_min(1e-6)).max().item()


PAGED_TOL = 1e-2


@gpu
@pytest.mark.parametrize("pt", [8, 16, 64])
@pytest.mark.parametrize("prefix", [0, 1, 63, 64, 65, 1500])
def test_paged_q8_operator(pt, prefix):
    """Three sequences, chunks of 1 / 17 / 64 / 130 rows across tile and page boundaries; 4 heads leave SMs idle, so launches with more
    than two key tiles take the split-KV path."""
    for T in (1, 17, 64, 130):
        lens = [prefix, prefix // 2, prefix + 7]
        q, rq, rs, table, ks, vs, n_pages = _paged_case_q8(pt, lens, T, 4, seed=pt * 1000 + prefix + T)
        got = _paged_run_q8(q, rq, rs, table, lens, pt, n_pages)
        assert torch.isfinite(got).all(), (pt, prefix, T)
        err = _row_err(got, _paged_ref_q8(q, ks, vs, lens))
        assert err <= PAGED_TOL, f"page_tokens {pt} prefix {prefix} chunk {T}: row-relative err {err:.3e}"


@gpu
@pytest.mark.parametrize("pt", [16, 64])
def test_paged_q8_full_grid_and_split_determinism(pt):
    lens = [600, 13, 1100]
    q, rq, rs, table, ks, vs, n_pages = _paged_case_q8(pt, lens, 130, 32, seed=5 + pt)
    assert _row_err(_paged_run_q8(q, rq, rs, table, lens, pt, n_pages), _paged_ref_q8(q, ks, vs, lens)) <= PAGED_TOL
    lens = [1499]
    q, rq, rs, table, ks, vs, n_pages = _paged_case_q8(pt, lens, 1, 32, seed=9 + pt)
    a = _paged_run_q8(q, rq, rs, table, lens, pt, n_pages)
    b = _paged_run_q8(q, rq, rs, table, lens, pt, n_pages)
    assert torch.equal(a, b), "split-KV combine must be deterministic"
    assert _row_err(a, _paged_ref_q8(q, ks, vs, lens)) <= PAGED_TOL


@gpu
def test_paged_q8_refuses_a_page_outside_the_pool():
    from visualcla import _native as N
    q, rq, rs, table, _ks, _vs, n_pages = _paged_case_q8(8, [20], 5, 2, seed=3)
    table[0, 0] = n_pages                                   # a page the caller's pool does not hold
    with pytest.raises(N.NativeError, match="outside"):
        _paged_run_q8(q, rq, rs, table, [20], 8, n_pages)


# ---------------------------------------------------------------------------------------------------------------------------------
# path
# ---------------------------------------------------------------------------------------------------------------------------------
def _model(cfg=None, **kw):
    import visualcla
    cfg = O.tiny_config() if cfg is None else cfg
    args = dict(seed=0, max_batch=4, max_seq=96, kv_cache_dtype="int8")
    args.update(kw)
    return visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), **args)


def _greedy(m, ids, px, n, **kw):
    return m.generate(input_ids=ids.cuda(), pixel_values=px.cuda(), do_sample=False, max_new_tokens=n, eos_token_id=None, pad_token_id=0,
                      output_logits=True, return_dict_in_generate=True, **kw)


@gpu
def test_model_reports_format_and_refuses_others():
    import visualcla
    m = _model()
    assert m.kv_cache_dtype == torch.int8
    for bad in ("fp8", torch.float16, 8):
        with pytest.raises(ValueError):
            visualcla.VisualCLAModel.from_synthetic(O.tiny_config().to_dict(), max_batch=1, max_seq=16, kv_cache_dtype=bad)
    for ok in (None, "bfloat16", torch.bfloat16):
        assert visualcla.VisualCLAModel.from_synthetic(O.tiny_config().to_dict(), max_batch=1, max_seq=16,
                                                      kv_cache_dtype=ok).kv_cache_dtype == torch.bfloat16


@gpu
def test_memory_formula_and_resize_keeps_format():
    m = _model()
    e = m._engine
    pps, total, pt = e.kv_geometry()
    cfg = O.tiny_config()
    assert e.memory_bytes()[1] == cfg.t_layers * total * 2 * cfg.t_heads * pt * 132
    m.resize_token_embeddings(cfg.t_vocab + 4)
    assert m.kv_cache_dtype == torch.int8 and m._engine.memory_bytes()[1] == cfg.t_layers * total * 2 * cfg.t_heads * pt * 132


@gpu
def test_prefill_epilogue_rows_match_the_hooked_oracle():
    cfg = O.tiny_config()
    m = _model()
    px, ids = O.make_inputs(cfg, 2, 12, seed=1234)
    _greedy(m, ids, px, 1)
    w = O.make_weights(cfg, 0)
    cache = O.KVCache(cfg.t_layers)
    generate_greedy_q8(w, cfg, ids, px, 1, cache=cache)
    e = m._engine
    pps, total, pt = e.kv_geometry()
    table = e.kv_pages()[0]
    S = cache.k[0].shape[2]
    for layer in range(cfg.t_layers):
        q, s = split_pool(e.kv_read_layer(layer), total, cfg.t_heads, pt)
        for b in range(2):
            j = torch.arange(S)
            pages, slots = table[b, j // pt].long(), j % pt
            for kv, ref in ((0, cache.k[layer]), (1, cache.v[layer])):
                rq, rs = q[pages, kv, :, slots], s[pages, kv, :, slots]          # (S, H, 128), (S, H)
                nz = rs > 0
                assert bool((rq.abs().amax(-1)[nz] == 127).all()), "every nonzero row reaches +-127"
                got = dequantize_rows(rq, rs).permute(1, 0, 2)
                err = ((got - ref[b]).abs().max() / ref[b].abs().max()).item()
                assert err < 3e-2, (layer, b, kv, err)


def _teacher_forced_vs_hooked_oracle(cfg, B, T, n_new, max_seq, load_in_8bit=False, seed=0):
    """Device logits of the prefill and of every decode step (teacher-forced on the hooked oracle's greedy tokens) against the oracle
    with the K/V round trip, on the device's own weights -> (relative error over all steps, decisive mismatches, model)."""
    from test_parity_gpu import _margin_ok_tokens, _teacher_forced_device
    m = _model(cfg, seed=seed, max_batch=B, max_seq=max_seq, load_in_8bit=load_in_8bit)
    w = {k: v.float() for k, v in m.state_dict().items()}
    px, ids = O.make_inputs(cfg, B, T, seed=77 + seed)
    o_tok, o_log = generate_greedy_q8(w, cfg, ids, px, n_new)
    m.image_at_head = True
    d_log, d_tok = _teacher_forced_device(m, ids.cuda(), px.cuda(), o_tok.cuda(), n_new)
    scale = o_log.abs().max().item()
    err = (d_log.cpu() - o_log).abs().max().item() / scale
    nbad, _ndec, _ntot = _margin_ok_tokens(d_tok.long(), o_tok, o_log, 1.5e-2 * scale)
    return err, nbad, m


MID = O.PathConfig(v_layers=2, r_layers=2, t_hidden=1024, t_heads=8, t_ffn=2752, t_layers=3, t_vocab=5003)


@gpu
@pytest.mark.parametrize("B", [1, 8, 32, 64])
def test_mid_config_every_step_against_the_hooked_oracle(B):
    """1024 wide, 8 heads: B = 64 puts 512 (sequence, head) items on the persistent decode kernel, B = 1..32 on the one-shot kernel."""
    err, nbad, m = _teacher_forced_vs_hooked_oracle(MID, B, 20, 12, 128)
    m._engine.close()
    print(f"\n[kv-int8] mid config B={B}: teacher-forced logits rel err {err:.3e}")
    assert err <= 1.5e-2 and nbad == 0, (err, nbad)


@gpu
@pytest.mark.parametrize("B,load_in_8bit", [(1, False), (8, False), (8, True)])
def test_7b_widths_every_step_against_the_hooked_oracle(B, load_in_8bit):
    """7B widths with 8 of the 32 LLaMA layers (the QKV epilogue at T = 4096, 32 heads; B = 8 is 256 items, the persistent kernel at
    B >= 9 is covered by the operator tests at 32 heads), alone and combined with load_in_8bit."""
    err, nbad, m = _teacher_forced_vs_hooked_oracle(O.PathConfig(t_layers=8), B, 24, 6, 128, load_in_8bit=load_in_8bit)
    m._engine.close()
    print(f"\n[kv-int8] 7B widths, 8 layers, B={B}, load_in_8bit={load_in_8bit}: teacher-forced logits rel err {err:.3e}")
    assert err <= 1.5e-2 and nbad == 0, (err, nbad)


@gpu
@pytest.mark.parametrize("int8_weights", [False, True])
def test_tiny_every_step_and_graph_replay_equals_eager(int8_weights):
    cfg = O.tiny_config()
    err, nbad, m = _teacher_forced_vs_hooked_oracle(cfg, 2, 12, 8, 96, load_in_8bit=int8_weights)
    assert err <= 3e-2 and nbad == 0, (err, nbad)      # the 2-layer tiny configuration's tolerance (tests/test_parity_gpu.py)
    eng = m._engine
    px, ids = O.make_inputs(cfg, 2, 12, seed=8)
    mode, rows = m._image_layout(ids.cuda(), px.cuda())
    res = []
    for use_graph in (False, True):
        eng.vision_encode(px.cuda())
        _l, tok, _a = eng.prefill(ids.cuda(), mode, rows)
        lg = torch.empty(2, eng.vocab, device="cuda")
        seq = []
        for _ in range(6):
            eng.decode_step(tok, tok, lg, use_graph=use_graph)
            seq.append(lg.clone())
        res.append(torch.stack(seq))
    assert torch.equal(res[0], res[1]), "graph replays are bit-identical to eager steps"


@gpu
def test_quantisation_error_against_the_unhooked_oracle():
    """How far the int8 cache moves the model: first-step logits against the bf16-cache oracle, relative to their max."""
    cfg = O.tiny_config()
    m = _model()
    px, ids = O.make_inputs(cfg, 2, 12, seed=1234)
    out = _greedy(m, ids, px, 1)
    _, o_log = O.generate_greedy(O.make_weights(cfg, 0), cfg, ids, px, 1)
    err = ((out.logits[0].cpu() - o_log[:, 0]).abs().max() / o_log.abs().max()).item()
    print(f"\n[kv-int8] first-step logits vs the unhooked oracle: rel err {err:.3e}")
    # measured 8.5e-3 (H100 80GB HBM3, 700 W); the gate is twice that
    assert err < 1.7e-2


@gpu
def test_prompt_lookup_and_streaming_change_no_token():
    from test_stream_gpu import Recorder
    cfg = O.tiny_config()
    m = _model()
    px, ids = O.make_inputs(cfg, 1, 24, seed=11)
    kw = dict(input_ids=ids.cuda(), pixel_values=px.cuda(), max_new_tokens=16, eos_token_id=None, pad_token_id=0, do_sample=False)
    plain = m.generate(**kw)
    assert torch.equal(m.generate(prompt_lookup_num_tokens=4, **kw), plain), "prompt lookup changes no token"
    assert m._engine.lookup_stats()[2] > 0, "the call ran verification steps"
    rec = Recorder()
    assert torch.equal(m.generate(streamer=rec, **kw), plain)
    assert torch.equal(rec.puts().cpu()[:, -plain.shape[1]:], plain.cpu()), "the streamed tokens are generate()'s"


@gpu
def test_sampling_every_token_against_the_sampler_oracle(monkeypatch):
    """Sampled decoding on the int8 cache: generate() (graph replays) equals the eager loop, every token equals the float64 draw of
    oracle/sampler_oracle.py on the int8-mode logits, and a num_return_sequences fork gives reply 0 of a plain sampled run."""
    from test_sampler_draw_gpu import CHAT, STEPS, _check_every_token, _eager, _generate_spec
    from test_sampler_gpu import DrawStats
    cfg = O.tiny_config()
    m = _model(seed=3, max_batch=3, max_seq=128)
    px, ids = O.make_inputs(cfg, 3, 12, seed=5)
    ids, px = ids.cuda(), px.cuda()
    torch.manual_seed(4)
    out, spec = _generate_spec(monkeypatch, m, input_ids=ids, pixel_values=px, max_new_tokens=STEPS, eos_token_id=None, pad_token_id=0, **CHAT)
    logits, toks, _ = _eager(m, ids, px, spec)
    stats = DrawStats()
    _check_every_token(logits, toks, spec, stats, "int8 KV cache, B=3, image")
    print(f"\n[kv-int8 sampled decoding] {stats.line()}")
    assert torch.equal(out, toks), "graph replays vs eager steps"
    torch.manual_seed(6)
    forked = m.generate(input_ids=ids[:1], pixel_values=px[:1], num_return_sequences=3, max_new_tokens=16, eos_token_id=None,
                        pad_token_id=0, **CHAT)
    assert forked.shape == (3, 16)


@gpu
def test_beams_against_the_hooked_beam_oracle(monkeypatch):
    """generate(num_beams=K) on the int8 cache against oracle/beam_oracle.py whose LLaMA forward carries the K/V round trip; copy-on-write
    counts 132 B per copied row."""
    import types
    import beam_oracle as BO
    from test_beam_gpu import _check_against_oracle
    monkeypatch.setattr(BO, "llama_forward", llama_forward_q8)
    cfg = O.tiny_config()
    m = _model(max_batch=8, max_seq=64)
    s0, s1, _, s3 = O.special_ids(cfg)
    m.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
    w = {k: v.float() for k, v in m.state_dict().items()}
    px, ids = O.make_inputs(cfg, 2, 10, seed=21)
    K, n_new = 4, 12
    tol = 1.5e-2 * float(generate_greedy_q8(w, cfg, ids, px, 1)[1].abs().max())
    m._engine.beam_cow_bytes(reset=True)
    got = m.generate(input_ids=ids.cuda(), pixel_values=px.cuda(), num_beams=K, do_sample=False, max_new_tokens=n_new, eos_token_id=None,
                     pad_token_id=0).cpu()
    how = _check_against_oracle(w, cfg, got, ids, px, True, None, K, n_new, dict(eos_token_id=(), pad_token_id=0), tol)
    print(f"\n[kv-int8 beams] {how}")
    cow = m._engine.beam_cow_bytes()
    _pps, _total, pt = m._engine.kv_geometry()
    per_row = cfg.t_layers * 2 * cfg.t_heads * 132
    assert cow > 0 and cow % per_row == 0, "copy-on-write moves whole int8 rows and their scales"


@gpu
def test_extend_in_chunks_matches_the_hooked_oracle():
    """Prefill with an image, then extend in three chunks with all logits: each chunk's logits equal the hooked oracle's forward of the
    whole sequence (the round trip is per row, so chunking does not change it).  Pages are handed out in a permuted order."""
    from visualcla import _native as N
    cfg = MID
    m = _model(cfg, seed=5, max_batch=1, max_seq=512)
    eng = m._engine
    eng.kv_debug_shuffle(11)
    w = {k: v.float() for k, v in m.state_dict().items()}
    px, ids = O.make_inputs(cfg, 1, 40, seed=3)
    g = torch.Generator().manual_seed(8)
    chunks = [torch.randint(3, cfg.t_vocab - 4, (1, n), generator=g) for n in (17, 64, 130)]
    eng.vision_encode(px.cuda())
    eng.prefill(ids.cuda(), N.IMAGE_AT_HEAD, None)
    s0, s1, _, s3 = O.special_ids(cfg)
    x = O.splice(w, cfg, ids, O.vision_encode(w, cfg, px), True, s0, s1, s3)
    emb = lambda c: w["text_model.model.embed_tokens.weight"][c].float()
    ref = llama_forward_q8(w, cfg, torch.cat([x] + [emb(c) for c in chunks], 1))
    pos = x.shape[1]
    for c in chunks:
        last, tok, la = eng.extend(c.cuda(), all_logits=True)
        r = ref[:, pos:pos + c.shape[1]]
        err = ((la.cpu() - r).abs().max() / r.abs().max()).item()
        assert err <= 1.5e-2, f"chunk at {pos}: rel err {err:.3e}"
        assert int(tok[0]) == int(last[0].argmax())
        pos += c.shape[1]
    eng.close()


@gpu
def test_reused_turn_agrees_with_a_fresh_int8_prefill_and_the_hooked_oracle():
    """Turn 2 passes turn 1's cache handle (vcla_prefill_extend on the int8 pool); its logits agree with a fresh int8 prefill of the
    same prompt and with the hooked oracle, to tolerance (not bit-equal: the extension reads q * s from the pool, the fresh prefill the
    bf16(q * s) of the epilogue)."""
    import types
    cfg = MID
    m = _model(cfg, seed=0, max_batch=1, max_seq=512)
    eng = m._engine
    s0, s1, _, s3 = O.special_ids(cfg)
    m.image_at_head = False
    m.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
    px, _ = O.make_inputs(cfg, 1, 8, seed=77)
    g = torch.Generator().manual_seed(3)
    text = lambda n: torch.randint(3, cfg.t_vocab - 4, (1, n), generator=g)
    p1 = torch.cat([torch.tensor([[1, s0]]), torch.full((1, cfg.r_queries), s3), torch.tensor([[s1]]), text(30)], 1)
    kw = dict(do_sample=False, eos_token_id=None, pad_token_id=0, output_logits=True, return_dict_in_generate=True)
    r1 = m.generate(input_ids=p1.cuda(), pixel_values=px.cuda(), max_new_tokens=8, **kw)
    p2 = torch.cat([p1, r1.sequences.cpu(), text(25)], 1)
    extends = []
    orig = eng.extend
    eng.extend = lambda *a, **k: (extends.append(1), orig(*a, **k))[1]
    r2 = m.generate(input_ids=p2.cuda(), pixel_values=px.cuda(), max_new_tokens=6, past_key_values=r1.past_key_values, **kw)
    assert extends, "turn 2 extends the cached conversation"
    eng.extend = orig
    fresh = m.generate(input_ids=p2.cuda(), pixel_values=px.cuda(), max_new_tokens=6, **kw)
    w = {k: v.float() for k, v in m.state_dict().items()}
    _o_tok, o_log = generate_greedy_q8(w, cfg, p2, px, 1, image_at_head=False)
    scale = o_log.abs().max().item()
    assert (r2.logits[0].cpu() - o_log[:, 0]).abs().max().item() <= 1.5e-2 * scale
    assert (r2.logits[0].cpu() - fresh.logits[0].cpu()).abs().max().item() <= 1.5e-2 * scale
    eng.close()


@gpu
def test_page_tables_equal_the_bf16_cache():
    cfg = O.tiny_config()
    px, ids = O.make_inputs(cfg, 3, 12, seed=21)
    tables = []
    for fmt in (None, "int8"):
        m = _model(kv_cache_dtype=fmt)
        _greedy(m, ids, px, 20)
        tables.append(m._engine.kv_pages())
        m._engine.close()
    for a, b in zip(*tables):
        assert torch.equal(torch.as_tensor(a), torch.as_tensor(b))


@gpu
def test_capacity_7b_64_by_2048():
    """At 7B widths, 64 sequences of 2048 tokens: the bf16 cache (68.7 GB) does not fit an 80 GB card next to the weights; the
    int8 one (35.4 GB) does.  The context is created and decodes a full batch."""
    import visualcla
    from visualcla.engine import path_config_7b
    p = path_config_7b()
    need = p["t_layers"] * 64 * 2048 * 2 * p["t_heads"] * 132 + 16e9
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip("not enough free device memory for the 7B int8 context")
    m = visualcla.VisualCLAModel.from_synthetic("7b", seed=0, max_batch=64, max_seq=2048, max_prefill_tokens=64 * 32, kv_cache_dtype="int8")
    e = m._engine
    _pps, total, pt = e.kv_geometry()
    assert e.memory_bytes()[1] == p["t_layers"] * total * 2 * p["t_heads"] * pt * 132
    ids = torch.randint(5, 1000, (64, 32), generator=torch.Generator().manual_seed(0))
    out = m.generate(input_ids=ids.cuda(), do_sample=False, max_new_tokens=4, eos_token_id=None, pad_token_id=0)
    assert out.shape == (64, 4)
    e.close()
