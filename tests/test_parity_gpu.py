"""End-to-end parity of the CUDA path (through the Python drop-in API -> C ABI) against
  (a) the golden fixtures produced by the UNMODIFIED reference (tests/golden, tiny config), and
  (b) the CPU oracle (oracle/visualcla_oracle.py) at larger shapes, incl. the real VisualCLA-7B widths.

Tolerances: the device path rounds GEMM operands / KV cache / attention probabilities to bf16 (fp32 accumulation, fp32
residual stream, fp32 softmax + norm statistics); the oracle is fp32 end to end.  bf16 has 8 mantissa bits
(rel. 2^-9 per rounding), so logits agree to ~1e-2 of the logit scale, not 1e-3 (DESIGN.md "Numerics").  Greedy tokens
must match exactly wherever the oracle's top-1/top-2 margin exceeds the logit tolerance."""
import ast
import os
import types

import numpy as np
import pytest
import torch

import visualcla_oracle as O

pytestmark = pytest.mark.gpu

# Gates = ~1.5x the measured error (every run appends its measured values to $VCLA_PARITY_LOG when set).  north_star's "1e-3" is below what ANY bf16 path reaches against an fp32 oracle -- see
# test_7b_error_not_worse_than_hf_bf16, which measures HF's own bf16 path on the same GPU, weights and inputs.
STAGE_TOL = {"vit_out": 6e-3, "post_ln": 6e-3, "resampler_out": 1.7e-2, "projector_out": 1.5e-2}   # relative to the stage's max |value|
LOGIT_TOL = 1.5e-2    # relative to max |logit|
LOGIT_TOL_TINY = 3.0e-2   # the 2-layer tiny reference goldens measure 1.3e-2 .. 2.05e-2 depending on the attention kernel (few, narrow layers:
                          # a max-abs metric over little averaging of the bf16 roundings)
LOSS_TOL = 3e-2       # absolute, cross-entropy in nats (measured 1.3e-2 on the tiny goldens: ~1 % logit error at |logit| ~ 17)


def _record(key, value):
    path = os.environ.get("VCLA_PARITY_LOG")
    if path:
        import json
        with open(path, "a") as f:
            f.write(json.dumps({"key": key, "value": value}) + "\n")


def _rel_err(a, b):
    a = a.detach().float().cpu() if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a)).float()
    b = b.detach().float().cpu() if isinstance(b, torch.Tensor) else torch.as_tensor(np.asarray(b)).float()
    assert a.shape == b.shape, (a.shape, b.shape)
    return (a - b).abs().max().item() / max(1e-6, b.abs().max().item())


def _margin_ok_tokens(dev_tokens, ora_tokens, ora_logits, tol_abs, free_running=False):
    """Tokens must be equal wherever the oracle's top1-top2 margin is larger than 2*tol_abs.  Teacher-forced runs are
    comparable at every step; in a free-running run only the steps up to (and including) a sequence's first mismatch
    are, because after it the two runs condition on different prefixes."""
    top2 = ora_logits.topk(2, dim=-1).values
    margin = top2[..., 0] - top2[..., 1]
    decisive = margin > 2 * tol_abs
    diff = dev_tokens.cpu() != ora_tokens.cpu()
    if free_running:
        comparable = torch.cumsum(torch.cumsum(diff.long(), 1), 1) <= 1     # prefix up to the first mismatch
        decisive = decisive & comparable
    bad = diff & decisive
    return int(bad.sum()), int(decisive.sum()), int(decisive.numel())


def _model(cfg: O.PathConfig, seed, max_batch, max_seq):
    import visualcla
    return visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=seed, max_batch=max_batch, max_seq=max_seq)


def _load_golden(golden_dir, name):
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    return g, O.PathConfig(**ast.literal_eval(str(g["config"])))


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tiny_b2_t12", "tiny_b3_t7"])
def test_device_weights_equal_oracle_generator(golden_dir, name):
    g, cfg = _load_golden(golden_dir, name)
    m = _model(cfg, int(g["seed"]), 4, 64)
    w = O.make_weights(cfg, int(g["seed"]))
    sd = m.state_dict()
    assert set(sd) == set(w)
    for k in w:
        assert torch.equal(sd[k].float().reshape(w[k].shape), w[k]), k


@pytest.mark.parametrize("name", ["tiny_b2_t12", "tiny_b3_t7"])
def test_tiny_against_reference_golden(golden_dir, name):
    """Reference-pinned: stages, logits in all three layouts, greedy tokens -- vs the unmodified reference's outputs."""
    g, cfg = _load_golden(golden_dir, name)
    m = _model(cfg, int(g["seed"]), 4, 64)
    px = torch.from_numpy(g["pixel_values"]).cuda()
    ids = torch.from_numpy(g["input_ids"]).cuda()
    B = ids.shape[0]
    m.image_at_head = True
    out = m.forward(input_ids=ids, pixel_values=px, attention_mask=torch.ones_like(ids), labels=ids)
    for st in ("vit_out", "post_ln", "resampler_out", "projector_out"):
        e = _rel_err(m._engine.read_stage(st, B), g[st])
        _record(f"{name}.{st}", e)
        assert e <= STAGE_TOL[st], f"{st}: rel err {e:.3e}"
    e = _rel_err(out.logits, g["logits_at_head"])
    _record(f"{name}.logits_at_head", e)
    assert e <= LOGIT_TOL_TINY, f"logits_at_head rel err {e:.3e}"
    assert _rel_err(m.embed_images(px), g["projector_out"]) <= STAGE_TOL["projector_out"]      # tg-webui entry point (embed_images)
    # forward(labels=...).loss vs the reference's own loss: -100 fill over the image block (ref :313-315), ignored labels
    _record(f"{name}.loss_at_head", abs(float(out.loss) - float(g["loss_at_head"])))
    assert abs(float(out.loss) - float(g["loss_at_head"])) <= LOSS_TOL
    lm = m.forward(input_ids=ids, pixel_values=px, attention_mask=torch.ones_like(ids), labels=torch.from_numpy(g["labels_masked"]).cuda()).loss
    assert abs(float(lm) - float(g["loss_at_head_masked"])) <= LOSS_TOL
    # placeholder layout (what get_model_and_tokenizer_and_processor configures)
    s0, s1, _, s3 = O.special_ids(cfg)
    m.image_at_head = False
    m.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
    ids_ph = torch.from_numpy(g["input_ids_placeholder"]).cuda()
    out_ph = m.forward(input_ids=ids_ph, pixel_values=px, attention_mask=torch.ones_like(ids_ph), labels=ids_ph)
    assert _rel_err(out_ph.logits, g["logits_placeholder"]) <= LOGIT_TOL_TINY
    assert torch.equal(out_ph.logits, out.logits), "layout equivalence (SURVEY 4-iv) must be bit-exact on the device too"
    assert abs(float(out_ph.loss) - float(g["loss_placeholder"])) <= LOSS_TOL
    out_txt = m.forward(input_ids=ids, pixel_values=None, attention_mask=torch.ones_like(ids), labels=ids)
    assert _rel_err(out_txt.logits, g["logits_text_only"]) <= LOGIT_TOL_TINY
    assert abs(float(out_txt.loss) - float(g["loss_text_only"])) <= LOSS_TOL
    # greedy generation: only the new tokens come back
    n = g["gen_tokens"].shape[1]
    m.image_at_head = True
    res = m.generate(input_ids=ids, pixel_values=px, attention_mask=torch.ones_like(ids), do_sample=False, max_new_tokens=n,
                     eos_token_id=None, pad_token_id=0, output_logits=True, return_dict_in_generate=True)
    assert res.sequences.shape == (B, n)
    glog = torch.from_numpy(g["gen_logits"])
    scale = glog.abs().max().item()
    nbad, ndec, ntot = _margin_ok_tokens(res.sequences, torch.from_numpy(g["gen_tokens"]), glog, LOGIT_TOL_TINY * scale, free_running=True)
    assert nbad == 0, f"{nbad} decisive greedy tokens differ ({ndec}/{ntot} decisive)"
    # fast greedy path (device argmax, CUDA graph) gives the same tokens as the logits path
    fast = m.generate(input_ids=ids, pixel_values=px, do_sample=False, max_new_tokens=n, eos_token_id=None, pad_token_id=0)
    assert torch.equal(fast, res.sequences)


def _teacher_forced_device(m, ids, px, forced, n_new):
    """Run the device path feeding the oracle's tokens; return per-step logits (B, n_new, V) and device argmax tokens."""
    eng = m._engine
    from visualcla import _native as N
    B = ids.shape[0]
    mode, rows = m._image_layout(ids, px)
    eng.vision_encode(px)
    last, tok0, _ = eng.prefill(ids, mode, rows, all_logits=False, last_logits=True)
    logits = [last.clone()]
    toks = [tok0.clone()]
    tok = torch.zeros(B, dtype=torch.int32, device=eng.device)
    lg = torch.empty(B, eng.vocab, dtype=torch.float32, device=eng.device)
    for s in range(1, n_new):
        tok.copy_(forced[:, s - 1].to(torch.int32))
        eng.decode_step(tok, tok, lg)
        logits.append(lg.clone())
        toks.append(tok.clone())
    return torch.stack(logits, 1), torch.stack(toks, 1)


def _run_vs_oracle(cfg, seed, B, T, n_new, max_seq, logit_tol=LOGIT_TOL, weights=None):
    m = _model(cfg, seed, B, max_seq)
    w = O.make_weights(cfg, seed) if weights is None else weights(m)
    px, ids = O.make_inputs(cfg, B, T, seed=77 + seed)
    o_tok, o_log = O.generate_greedy(w, cfg, ids, px, n_new, image_at_head=True)
    m.image_at_head = True
    d_log, d_tok = _teacher_forced_device(m, ids.cuda(), px.cuda(), o_tok.cuda(), n_new)
    scale = o_log.abs().max().item()
    err = (d_log.cpu() - o_log).abs().max().item() / scale
    nbad, ndec, ntot = _margin_ok_tokens(d_tok.long(), o_tok, o_log, logit_tol * scale)
    _record(f"vs_oracle.hidden{cfg.t_hidden}.layers{cfg.t_layers}.B{B}.T{T}.steps{n_new}", err)
    return m, err, nbad, ndec, ntot, o_tok, o_log


def test_mid_config_vs_oracle():
    """ViT/Resampler at real width but few layers, LLaMA at 1024 width: exercises 257-token ViT, 64x321 resampler
    attention, multi-tile GEMMs, multi-page KV cache and 40 decode steps."""
    cfg = O.PathConfig(v_layers=2, r_layers=2, t_hidden=1024, t_heads=8, t_ffn=2752, t_layers=3, t_vocab=5003)
    m, err, nbad, ndec, ntot, o_tok, o_log = _run_vs_oracle(cfg, 5, 3, 70, 40, 256)
    assert err <= LOGIT_TOL, f"teacher-forced logits rel err {err:.3e}"
    assert nbad == 0, f"{nbad} decisive tokens differ ({ndec}/{ntot} decisive)"
    # free-running greedy on the device == oracle tokens wherever decisive (here: compare the prefix up to first diff)
    px, ids = O.make_inputs(cfg, 3, 70, seed=77 + 5)
    out = m.generate(input_ids=ids.cuda(), pixel_values=px.cuda(), do_sample=False, max_new_tokens=40, eos_token_id=None, pad_token_id=0)
    assert out.shape == (3, 40)
    # free-running: every sequence must follow the oracle up to its first mismatch, and that mismatch must be a
    # non-decisive step (top-1/top-2 margin within the logit tolerance); later steps condition on different prefixes
    nbad, ndec, ntot = _margin_ok_tokens(out, o_tok, o_log, LOGIT_TOL * o_log.abs().max().item(), free_running=True)
    assert nbad == 0, f"free-running: {nbad} decisive tokens differ before the first divergence ({ndec}/{ntot} decisive)"


def test_long_context_vs_oracle():
    """BASELINE configs[4] in miniature: long prompt (S = 64 + 900), multi-page KV cache, 4-way split-KV decode attention
    (max_seq >= 1536 selects 4 KV splits), causal prefill attention over 16 KV tiles."""
    cfg = O.PathConfig(v_layers=1, r_layers=1, t_hidden=512, t_heads=4, t_ffn=1408, t_layers=2, t_vocab=3001)
    m, err, nbad, ndec, ntot, _, _ = _run_vs_oracle(cfg, 11, 2, 900, 12, 1600)
    assert err <= LOGIT_TOL, f"teacher-forced logits rel err {err:.3e}"
    assert nbad == 0, f"{nbad} decisive tokens differ ({ndec}/{ntot} decisive)"


def test_persistent_decode_attention(monkeypatch):
    """The warp-specialised persistent decode-attention kernel (used when sequences x heads outnumber the resident CTAs, e.g.
    batch 32 x 32 heads) forced onto a small problem with 5 CTAs, so every CTA walks several (sequence, head) items and the
    KV ring wraps across items."""
    monkeypatch.setenv("VCLA_ATTN_PERSISTENT", "2")
    monkeypatch.setenv("VCLA_ATTN_PERSISTENT_GRID", "5")
    cfg = O.PathConfig(v_layers=1, r_layers=1, t_hidden=1024, t_heads=8, t_ffn=1408, t_layers=2, t_vocab=2003)
    m, err, nbad, ndec, ntot, _, _ = _run_vs_oracle(cfg, 17, 4, 150, 20, 512)
    assert err <= LOGIT_TOL, f"teacher-forced logits rel err {err:.3e}"
    assert nbad == 0, f"{nbad} decisive tokens differ ({ndec}/{ntot} decisive)"


def test_chat_api_on_device():
    """The reference's chat()/chat_in_stream() entry points (ref: modeling_utils.py:143-247) drive the CUDA path end to end
    (stub tokenizer / image processor: no tokenizer files exist offline)."""
    import visualcla
    from transformers import GenerationConfig

    cfg = O.tiny_config()
    m = visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=0, max_batch=1, max_seq=256)
    s0, s1, s2, s3 = O.special_ids(cfg)

    class Tok:
        bos_token, pad_token, bos_token_id, eos_token_id = "<s>", "<pad>", 1, 2
        img_start_token, img_end_token, img_token = "<img>", "</img>", "<img_token>"
        img_start_token_id, img_end_token_id, img_token_id = s0, s1, s3

        def __call__(self, text, return_tensors=None, add_special_tokens=None):
            from transformers import BatchEncoding
            ids, i = [], 0
            special = {"<s>": 1, "<img>": s0, "</img>": s1, "<img_token>": s3}
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
    m.image_processor = lambda img, return_tensors=None: types.SimpleNamespace(pixel_values=torch.randn(1, 3, cfg.v_image, cfg.v_image))
    px = torch.randn(1, 3, cfg.v_image, cfg.v_image)
    gc = GenerationConfig(do_sample=False, max_new_tokens=5, eos_token_id=None, pad_token_id=0)
    hist = []
    resp, hist = visualcla.chat(m, image=px, text="hello", history=hist, generation_config=gc)
    assert len(resp.split()) == 5 and hist[0].get("first_instruction") and hist[-1]["type"] == "response"
    resp2, hist = visualcla.chat(m, image=px, text="more", history=hist, generation_config=gc)       # multi-turn: image block only in turn 1
    assert len(hist) == 4
    # default (sampling) config path: temperature/top-k/top-p/repetition penalty/no-repeat-ngram on the returned logits
    gs = GenerationConfig(do_sample=True, top_k=40, top_p=0.9, temperature=0.5, repetition_penalty=1.1, no_repeat_ngram_size=15,
                          max_new_tokens=6, eos_token_id=None, pad_token_id=0)
    resp3, _ = visualcla.chat(m, image=px, text="again", history=[], generation_config=gs)
    assert len(resp3.split()) == 6
    chunks = list(visualcla.chat_in_stream(m, image=px, text="stream", history=[], generation_config=gc))
    assert len(chunks) == 5 and len(chunks[-1][0].split()) == 5 and chunks[-1][1][-1]["type"] == "response"


def test_left_padded_batch_against_reference_golden(golden_dir):
    """Prompts of different lengths, LEFT padded (HF batching): tokens/logits vs the reference's generate() and forward()
    (tests/golden/tiny_padded.npz), and each padded sequence must equal the same sequence run alone without padding."""
    g, cfg = _load_golden(golden_dir, "tiny_padded")
    m = _model(cfg, int(g["seed"]), 4, 96)
    s0, s1, s2, s3 = O.special_ids(cfg)
    m.image_at_head = False
    m.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
    px = torch.from_numpy(g["pixel_values"]).cuda()
    ids = torch.from_numpy(g["input_ids"]).cuda()
    mask = torch.from_numpy(g["attention_mask"]).cuda()
    pads = g["pads"].tolist()
    n = g["gen_tokens"].shape[1]
    kw = dict(do_sample=False, max_new_tokens=n, eos_token_id=None, pad_token_id=s2)
    res = m.generate(input_ids=ids, pixel_values=px, attention_mask=mask, output_logits=True, return_dict_in_generate=True, **kw)
    glog = torch.from_numpy(g["gen_logits"])
    scale = glog.abs().max().item()
    e0 = (res.logits[0].cpu() - glog[:, 0]).abs().max().item() / scale
    assert e0 <= LOGIT_TOL_TINY, f"prefill-step logits rel err {e0:.3e}"
    nbad, ndec, ntot = _margin_ok_tokens(res.sequences, torch.from_numpy(g["gen_tokens"]), glog, LOGIT_TOL_TINY * scale, free_running=True)
    assert nbad == 0, f"{nbad} decisive tokens differ ({ndec}/{ntot} decisive)"
    # forward(): arange positions, pad keys masked; only real rows are defined
    fwd = m.forward(input_ids=ids, pixel_values=px, attention_mask=mask).logits.cpu()
    ref = torch.from_numpy(g["forward_logits"])
    for b, p in enumerate(pads):
        assert _rel_err(fwd[b, p:], ref[b, p:]) <= LOGIT_TOL_TINY
    # padding invariance on the device: sequence b alone (unpadded) generates the same tokens as inside the padded batch
    fast = m.generate(input_ids=ids, pixel_values=px, attention_mask=mask, **kw)
    assert torch.equal(fast, res.sequences)
    for b, p in enumerate(pads):
        alone = m.generate(input_ids=ids[b:b + 1, p:], pixel_values=px[b:b + 1], **kw)
        assert torch.equal(alone[0], fast[b]), f"sequence {b} (pad {p}) differs from its unpadded run"
    with pytest.raises(NotImplementedError):
        bad = mask.clone(); bad[0, -1] = 0
        m.generate(input_ids=ids, pixel_values=px, attention_mask=bad, **kw)


def test_lora_fold_at_load(tmp_path):
    """Unmerged checkpoint path without peft: fold synthetic LoRA deltas + replaced tensors, compare with the oracle run on the
    explicitly merged weights (what PeftModel.merge_and_unload would have produced)."""
    import json
    import visualcla
    cfg = O.tiny_config()
    m = visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=4, max_batch=2, max_seq=64)
    w = O.make_weights(cfg, 4)
    g = torch.Generator().manual_seed(1)
    r, alpha = 4, 8
    sd = {}
    targets = ["text_model.model.layers.0.self_attn.q_proj.weight", "text_model.model.layers.1.mlp.gate_proj.weight",
               "text_model.model.layers.1.mlp.down_proj.weight", "vision_model.vision_model.encoder.layers.0.self_attn.v_proj.weight",
               "vision_model.vision_model.encoder.layers.1.mlp.fc2.weight"]
    for t in targets:
        out_f, in_f = w[t].shape
        A, B = torch.randn(r, in_f, generator=g) * 0.05, torch.randn(out_f, r, generator=g) * 0.05
        base = "base_model.model." + t[: -len(".weight")]
        sd[base + ".lora_A.weight"], sd[base + ".lora_B.weight"] = A, B
        w[t] = (w[t] + (alpha / r) * (B @ A)).to(torch.bfloat16).float()
    newq = (torch.randn(1, cfg.r_queries, cfg.r_hidden, generator=g)).to(torch.bfloat16).float()
    sd["base_model.model.visual_resampler.query_embeddding"] = newq
    w["visual_resampler.query_embeddding"] = newq
    torch.save(sd, tmp_path / "adapter_model.bin")
    json.dump({"r": r, "lora_alpha": alpha, "fan_in_fan_out": False}, open(tmp_path / "adapter_config.json", "w"))
    info = visualcla.load_lora(m, str(tmp_path))
    assert info["folded"] == len(targets) and info["replaced"] == 1
    px, ids = O.make_inputs(cfg, 2, 10, seed=6)
    got = m.forward(input_ids=ids.cuda(), pixel_values=px.cuda(), labels=ids.cuda()).logits
    ref = O.forward_logits(w, cfg, ids, px, image_at_head=True)
    assert _rel_err(got, ref) <= LOGIT_TOL


# "tcgen05" is the stable id of VCLA_ATTN_TC mode 2, the tensor-core kernel of csrc/attention_tc.cu (wgmma on sm_90a)
@pytest.mark.parametrize("impl", [0, 2], ids=["mma_sync", "tcgen05"])
def test_prefill_attention_kernels_end_to_end(golden_dir, impl):
    """Both prefill attention kernels through the whole path: ViT (257 tokens, hd 64), Resampler (two KV segments), LLaMA causal
    prefill over several KV tiles, and left padding (kv_start) against the reference's padded golden."""
    from visualcla import _native as N
    lib = N.load()
    lib.vcla_set_attention_tc(impl)
    try:
        cfg = O.PathConfig(v_layers=2, r_layers=2, t_hidden=1024, t_heads=8, t_ffn=2752, t_layers=3, t_vocab=5003)
        m, err, nbad, ndec, ntot, _, _ = _run_vs_oracle(cfg, 5, 3, 300, 6, 512)
        assert err <= LOGIT_TOL, f"teacher-forced logits rel err {err:.3e}"
        assert nbad == 0
        g, gcfg = _load_golden(golden_dir, "tiny_padded")
        mp = _model(gcfg, int(g["seed"]), 4, 96)
        s0, s1, s2, s3 = O.special_ids(gcfg)
        mp.image_at_head = False
        mp.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
        px, ids, mask = (torch.from_numpy(g[k]).cuda() for k in ("pixel_values", "input_ids", "attention_mask"))
        fwd = mp.forward(input_ids=ids, pixel_values=px, attention_mask=mask).logits.cpu()
        ref = torch.from_numpy(g["forward_logits"])
        for b, p in enumerate(g["pads"].tolist()):
            assert _rel_err(fwd[b, p:], ref[b, p:]) <= LOGIT_TOL_TINY
    finally:
        lib.vcla_set_attention_tc(int(os.environ.get("VCLA_ATTN_TC", "1")))


@pytest.mark.parametrize("B", [1, 5, 16, 17, 32, 33, 64])
def test_decode_over_batch_sizes(B):
    """Both decode schedules against the oracle, each chosen by the batch size as in use.  Batches <= 32, cluster split-K
    decode GEMMs: every batch tile (16 / 32 columns), uneven column ownership (batch not a multiple of the cluster size,
    clusters larger than the batch) and multi-round cluster walks.  Batches 33..64 (both ends): split-K partials in the L2
    workspaces with separate consumer kernels."""
    cfg = O.PathConfig(v_layers=1, r_layers=1, t_hidden=1024, t_heads=8, t_ffn=2752, t_layers=2, t_vocab=5003)
    m, err, nbad, ndec, ntot, _, _ = _run_vs_oracle(cfg, 19, B, 24, 8, 128)
    assert err <= LOGIT_TOL, f"teacher-forced logits rel err {err:.3e}"
    assert nbad == 0, f"{nbad} decisive tokens differ ({ndec}/{ntot} decisive)"


def test_batch_invariance_row_for_row():
    """DP correctness premise (SURVEY 4-v): a sample's tokens do not depend on what else is in the batch."""
    cfg = O.PathConfig(v_layers=1, r_layers=1, t_hidden=512, t_heads=4, t_ffn=1408, t_layers=2, t_vocab=2003)
    import visualcla
    m = visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=9, max_batch=8, max_seq=160)
    px, ids = O.make_inputs(cfg, 6, 20, seed=5)
    full = m.generate(input_ids=ids.cuda(), pixel_values=px.cuda(), do_sample=False, max_new_tokens=24, eos_token_id=None, pad_token_id=0)
    lo = m.generate(input_ids=ids[:2].cuda(), pixel_values=px[:2].cuda(), do_sample=False, max_new_tokens=24, eos_token_id=None, pad_token_id=0)
    hi = m.generate(input_ids=ids[2:].cuda(), pixel_values=px[2:].cuda(), do_sample=False, max_new_tokens=24, eos_token_id=None, pad_token_id=0)
    assert torch.equal(full, torch.cat([lo, hi], 0))


def test_merged_checkpoint_roundtrip(tmp_path):
    """save in the reference's merged-directory layout -> from_merged_pretrained -> identical logits."""
    import visualcla
    cfg = O.tiny_config()
    m = visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=2, max_batch=2, max_seq=64)
    px, ids = O.make_inputs(cfg, 2, 9, seed=3)
    a = m.forward(input_ids=ids.cuda(), pixel_values=px.cuda(), labels=ids.cuda()).logits.clone()
    m.save_merged_pretrained(str(tmp_path))
    m2 = visualcla.VisualCLAModel.from_merged_pretrained(str(tmp_path), torch_dtype=torch.bfloat16, default_device=None, device_map=None,
                                                         load_in_8bit=False, max_batch=2, max_seq=64)
    b = m2.forward(input_ids=ids.cuda(), pixel_values=px.cuda(), labels=ids.cuda()).logits
    assert torch.equal(a, b)
    with pytest.raises(KeyError):
        visualcla.VisualCLAModel.from_merged_pretrained(str(tmp_path))


def test_placeholder_errors_and_eos():
    import visualcla
    cfg = O.tiny_config()
    m = visualcla.VisualCLAModel.from_synthetic(cfg.to_dict(), seed=0, max_batch=2, max_seq=64)
    s0, s1, _, s3 = O.special_ids(cfg)
    m.image_at_head = False
    m.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
    px, _ = O.make_inputs(cfg, 1, 8)
    bad = torch.tensor([[1, s0, s3, s3, s1, 5, 6, 7, 8, 9, 10, 11]]).cuda()
    with pytest.raises(ValueError):
        m.generate(input_ids=bad, pixel_values=px.cuda(), do_sample=False, max_new_tokens=2)
    # EOS: pick the first greedy token as "eos" -> generation stops after one token and pads
    m.image_at_head = True
    px, ids = O.make_inputs(cfg, 2, 8)
    free = m.generate(input_ids=ids.cuda(), pixel_values=px.cuda(), do_sample=False, max_new_tokens=6, eos_token_id=None, pad_token_id=0)
    eos = int(free[0, 0])
    out = m.generate(input_ids=ids.cuda(), pixel_values=px.cuda(), do_sample=False, max_new_tokens=6, eos_token_id=eos, pad_token_id=0)
    assert int(out[0, 0]) == eos and bool((out[0, 1:] == 0).all())
    # sampling path runs and respects top_k=1 == greedy
    samp = m.generate(input_ids=ids.cuda(), pixel_values=px.cuda(), do_sample=True, top_k=1, temperature=0.7, max_new_tokens=6,
                      eos_token_id=None, pad_token_id=0)
    assert torch.equal(samp, free)


# ---------------------------------------------------------------------------------------------------------------
# Real VisualCLA-7B widths (BASELINE.json configs).  The oracle gets the device's own bf16 weights (vcla_read_weight).
# ---------------------------------------------------------------------------------------------------------------
skip7b = pytest.mark.skipif(os.environ.get("VCLA_SKIP_7B") == "1", reason="VCLA_SKIP_7B=1")


def _dl(m):
    return {k: v.float() for k, v in m.state_dict().items()}


def _7b_case(tag, B, T, n_new, max_seq, t_layers=None):
    cfg = O.PathConfig() if t_layers is None else O.PathConfig(t_layers=t_layers)
    print(f"[7B parity {tag}] oracle host threads: {O.pick_threads()}")
    m, err, nbad, ndec, ntot, _, _ = _run_vs_oracle(cfg, 0, B, T, n_new, max_seq, weights=_dl)
    print(f"[7B parity {tag}] teacher-forced logits rel err {err:.3e}; decisive tokens {ndec}/{ntot}, mismatches {nbad}")
    eng = m._engine
    try:
        assert err <= LOGIT_TOL
        assert nbad == 0
    finally:
        eng.close()


@skip7b
def test_config1_7b_logit_parity_gate():
    """BASELINE configs[0]: 1 image + 32-token prompt (S=96), the full 64 greedy tokens teacher-forced, oracle = fp32 on CPU."""
    _7b_case("cfg1", 1, 32, int(os.environ.get("VCLA_7B_STEPS", "64")), 256)


@skip7b
def test_config2_7b_batch8():
    """BASELINE configs[1] shapes at full depth: B=8, S=128 (BN=16 decode tiles, 4-way split-KV one-shot decode attention)."""
    _7b_case("cfg2", 8, 64, 6, 128 + 256 + 1)


@skip7b
def test_config3_7b_batch32():
    """BASELINE configs[2] shapes: B=32, T=128 (S=192): BN=32 decode tiles, persistent decode-attention kernel (32 x 32 items).
    Full widths, 8 of the 32 LLaMA layers by default (every kernel / tile / split choice depends on widths and batch, not on
    depth; depth is covered by cfg1/cfg2) -- VCLA_PARITY_FULL_DEPTH=1 runs all 32."""
    _7b_case("cfg3", 32, 128, 5, 192 + 256 + 1, None if os.environ.get("VCLA_PARITY_FULL_DEPTH") == "1" else 8)


@skip7b
def test_config5_7b_long_context():
    """BASELINE configs[4] shapes: B=16, T=1024 (S=1088): kv_splits=4 decode attention over 17+ pages, 17 KV tiles of causal
    prefill attention.  Full widths, 8 LLaMA layers by default (see cfg3)."""
    _7b_case("cfg5", 16, 1024, 4, 1088 + 512 + 1, None if os.environ.get("VCLA_PARITY_FULL_DEPTH") == "1" else 8)


@skip7b
def test_7b_error_not_worse_than_hf_bf16():
    """north_star asks for logits "within 1e-3 bf16"; a bf16 rounding is 2^-9 = 2e-3, so the honest bar is HF's own bf16 path:
    the very HF classes the reference calls (CLIPVisionModel, LlamaForCausalLM; Resampler = the oracle's torch restatement), in
    bf16 on this GPU, with the same weights and inputs.  err(this repo vs fp32 oracle) must not exceed 1.1 x err(HF-bf16 vs
    fp32 oracle)."""
    from transformers import LlamaConfig, LlamaForCausalLM
    from transformers.models.clip.modeling_clip import CLIPVisionConfig, CLIPVisionModel
    cfg = O.PathConfig()
    m = _model(cfg, 0, 1, 256)
    sd = m.state_dict()                                       # bf16 matrices / fp32 vectors, reference state-dict names
    px, ids = O.make_inputs(cfg, 1, 32, seed=77)
    m.image_at_head = True
    ours = m.forward(input_ids=ids.cuda(), pixel_values=px.cuda(), attention_mask=torch.ones_like(ids).cuda(), labels=ids.cuda()).logits.float().cpu()
    m._engine.close()
    w32 = {k: v.float() for k, v in sd.items()}
    ref = O.forward_logits(w32, cfg, ids, px, image_at_head=True)
    del w32
    dt = torch.bfloat16
    old = torch.get_default_dtype()
    torch.set_default_dtype(dt)
    try:
        with torch.device("cuda"):
            llama = LlamaForCausalLM(LlamaConfig(vocab_size=cfg.t_vocab, hidden_size=cfg.t_hidden, intermediate_size=cfg.t_ffn,
                                                 num_hidden_layers=cfg.t_layers, num_attention_heads=cfg.t_heads, num_key_value_heads=cfg.t_heads,
                                                 rms_norm_eps=cfg.t_eps, rope_theta=cfg.rope_theta, max_position_embeddings=2048,
                                                 tie_word_embeddings=False, pad_token_id=0, bos_token_id=1, eos_token_id=2)).eval()
            clip = CLIPVisionModel(CLIPVisionConfig(hidden_size=cfg.v_hidden, intermediate_size=cfg.v_ffn, num_hidden_layers=cfg.v_layers,
                                                    num_attention_heads=cfg.v_heads, image_size=cfg.v_image, patch_size=cfg.v_patch,
                                                    hidden_act="quick_gelu", layer_norm_eps=cfg.v_eps)).eval()
    finally:
        torch.set_default_dtype(old)
    tsd = {k[len("text_model."):]: v for k, v in sd.items() if k.startswith("text_model.")}
    vsd = {k[len("vision_model."):]: v for k, v in sd.items() if k.startswith("vision_model.")}
    miss = llama.load_state_dict(tsd, strict=False)
    assert not [k for k in miss.missing_keys if "rotary" not in k] and not miss.unexpected_keys, miss
    miss = clip.load_state_dict(vsd, strict=False)
    assert not [k for k in miss.missing_keys if "position_ids" not in k] and not miss.unexpected_keys, miss
    wr = {k: v.cuda().to(dt) for k, v in sd.items() if k.startswith(("visual_resampler.", "image_projection_layer."))}
    with torch.no_grad():
        emb = llama.get_input_embeddings()(ids.cuda())
        vit = clip(pixel_values=px.cuda().to(dt))[0]
        post = clip.vision_model.post_layernorm(vit)
        img = O.project(wr, O.resampler_forward(wr, cfg, post)).to(dt)
        x = torch.cat([emb[:, :2], img, emb[:, 2:]], dim=1)
        hf = llama(inputs_embeds=x, attention_mask=torch.ones(x.shape[:2], dtype=torch.long, device="cuda")).logits.float().cpu()
    scale = ref.abs().max().item()
    e_ours, e_hf = (ours - ref).abs().max().item() / scale, (hf - ref).abs().max().item() / scale
    rms_ours, rms_hf = (ours - ref).pow(2).mean().sqrt().item() / scale, (hf - ref).pow(2).mean().sqrt().item() / scale
    print(f"[7B vs HF-bf16] max rel err: this repo {e_ours:.3e}, HF bf16 {e_hf:.3e}; rms: {rms_ours:.3e} vs {rms_hf:.3e}")
    _record("hf_bf16_comparison", {"ours_max": e_ours, "hf_bf16_max": e_hf, "ours_rms": rms_ours, "hf_bf16_rms": rms_hf})
    assert e_ours <= 1.1 * e_hf, f"this repo {e_ours:.3e} vs HF bf16 {e_hf:.3e}"
    assert e_ours <= LOGIT_TOL
