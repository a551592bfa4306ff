"""Generate tests/golden/tiny_beams.npz by running the UNMODIFIED reference's generate(num_beams=...) (behind oracle/ref_shim.py)
on the tiny config with seeded synthetic weights.  Run in the authoring container only:

    python oracle/gen_golden_beams.py

The fixture pins oracle/beam_oracle.py (tests/test_beam_oracle.py) and, through it, the device beam search
(tests/test_beam_gpu.py).  The model is built exactly as for the other fixtures (oracle/gen_golden.py:build_reference_model).
"""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import visualcla_oracle as O  # noqa: E402
from gen_golden import OUT, build_reference_model  # noqa: E402
from ref_shim import import_reference  # noqa: E402

BEAM_CASES = [   # name, layout, generation-config overrides (num_beams, eos "greedy" = a token the greedy run emits early)
    ("k4", "head", dict(num_beams=4)),
    ("eos_es_true", "head", dict(num_beams=3, eos="greedy", early_stopping=True)),
    ("eos_es_false", "head", dict(num_beams=3, eos="greedy", early_stopping=False)),
    ("eos_es_never", "head", dict(num_beams=3, eos="greedy", early_stopping="never")),
    ("lp_2", "text", dict(num_beams=3, eos="greedy", length_penalty=2.0)),
    ("lp_neg", "text", dict(num_beams=3, eos="greedy", length_penalty=-0.5)),
    ("nrs_2", "placeholder", dict(num_beams=4, eos="greedy", num_return_sequences=2)),
    ("rep_ngram", "head", dict(num_beams=3, eos="greedy", repetition_penalty=1.1, no_repeat_ngram_size=3)),
    ("padded", "padded", dict(num_beams=3, eos="greedy")),
]


@torch.no_grad()
def case_tiny_beams(visualcla, seed=0, n_new=10):
    """Beam search through the reference's generate(num_beams=...) (ref: modeling_visualcla.py:382-391 -> HF:generation/utils.py
    _beam_search) on the tiny config: every case's returned sequences and their scores (HF sequences_scores)."""
    from transformers import GenerationConfig
    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed)
    model = build_reference_model(visualcla, cfg, w)
    s0, s1, s2, s3 = O.special_ids(cfg)
    model.tokenizer = types.SimpleNamespace(img_start_token_id=s0, img_end_token_id=s1, img_token_id=s3)
    B, T, nq = 2, 9, cfg.r_queries
    pixels, ids = O.make_inputs(cfg, B, T, seed=4321 + seed)
    ids_ph = torch.cat([ids[:, :2], torch.full((B, nq), s3, dtype=torch.long), ids[:, 2:]], dim=1)
    pads = [0, 3]
    ids_pad = torch.full((B, T + nq), s2, dtype=torch.long)
    mask_pad = torch.zeros(B, T + nq, dtype=torch.long)
    for b, p in enumerate(pads):
        ids_pad[b, p:] = ids_ph[b, : T + nq - p]
        mask_pad[b, p:] = 1
    # EOS for the EOS cases: the token the greedy run (image at head) emits at step 2 for item 0
    model.image_at_head = True
    greedy = model.generate(input_ids=ids, pixel_values=pixels, attention_mask=torch.ones_like(ids),
                            generation_config=GenerationConfig(do_sample=False, max_new_tokens=4, eos_token_id=None, pad_token_id=0))
    eos_id = int(greedy[0, 2])
    out, meta = {}, []
    for name, layout, over in BEAM_CASES:
        over = dict(over)
        eos = [eos_id] if over.pop("eos", None) == "greedy" else None
        gc = GenerationConfig(do_sample=False, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=0, bos_token_id=1,
                              return_dict_in_generate=True, output_scores=True, **over)
        if layout == "head":
            model.image_at_head, x, px, mask = True, ids, pixels, torch.ones_like(ids)
        elif layout == "text":
            model.image_at_head, x, px, mask = True, ids, None, torch.ones_like(ids)
        elif layout == "placeholder":
            model.image_at_head, x, px, mask = False, ids_ph, pixels, torch.ones_like(ids_ph)
        else:
            model.image_at_head, x, px, mask = False, ids_pad, pixels, mask_pad
        gen = model.generate(input_ids=x, pixel_values=px, attention_mask=mask, generation_config=gc)
        out[f"{name}_input_ids"] = x.numpy()
        out[f"{name}_attention_mask"] = mask.numpy()
        out[f"{name}_sequences"] = gen.sequences.numpy()
        out[f"{name}_scores"] = gen.sequences_scores.float().numpy()
        meta.append(dict(name=name, layout=layout, eos=eos or [], pad_token_id=0, max_new_tokens=n_new, **over))
        print(f"[golden] tiny_beams {name}: sequences {tuple(gen.sequences.shape)} scores {gen.sequences_scores.tolist()}")
    np.savez_compressed(os.path.join(OUT, "tiny_beams.npz"), config=np.array(repr(cfg.to_dict())), seed=np.array(seed),
                        pixel_values=pixels.numpy(), cases=np.array(json.dumps(meta)), **out)


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    case_tiny_beams(import_reference())
