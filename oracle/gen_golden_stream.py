"""Generate tests/golden/tiny_stream.npz by running the UNMODIFIED reference's generate(streamer=..., stopping_criteria=[...])
(behind oracle/ref_shim.py) on the tiny config with seeded synthetic weights.  Run in the authoring container only:

    python oracle/gen_golden_stream.py

The fixture pins the streamer protocol of generate(): which `put` calls a streamer receives (shape, dtype, values), in what
order relative to the stopping-criteria calls (with the length of the ids each one sees), and the single `end`.  The reference
forwards `streamer` and `stopping_criteria` to HF generate(inputs_embeds=...) (ref: modeling_visualcla.py:382-391), which is what
chat_in_stream relies on (ref: modeling_utils.py:180-247).  The model is built exactly as for the other fixtures
(oracle/gen_golden.py:build_reference_model).
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


class RecordingStreamer:
    """HF BaseStreamer shape: put(value) per call, end() once."""

    def __init__(self, events):
        self.events = events

    def put(self, value):
        self.events.append(dict(kind="put", shape=list(value.shape), dtype=str(value.dtype), device=str(value.device),
                                values=value.reshape(-1).tolist()))

    def end(self):
        self.events.append(dict(kind="end"))


def recording_criterion(events):
    from transformers import StoppingCriteria

    class Rec(StoppingCriteria):
        def __call__(self, input_ids, scores, **kwargs):
            events.append(dict(kind="criterion", length=int(input_ids.shape[-1]), batch=int(input_ids.shape[0])))
            return False
    return Rec()


@torch.no_grad()
def case_tiny_stream(visualcla, seed=0, n_new=10):
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

    def greedy(x, px, mask, at_head, eos=None):
        model.image_at_head = at_head
        return model.generate(input_ids=x, pixel_values=px, attention_mask=mask,
                              generation_config=GenerationConfig(do_sample=False, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=0))

    # B = 1 at head: EOS = the token the greedy run emits at step 3 (not earlier)
    g1 = greedy(ids[:1], pixels[:1], torch.ones_like(ids[:1]), True)[0].tolist()
    k = next(i for i in range(3, n_new) if g1[i] not in g1[:i])
    eos_b1 = g1[k]
    # B = 2 padded placeholder: EOS = a token row 0 emits part-way that row 1 never emits
    g2 = greedy(ids_pad, pixels, mask_pad, False)
    r0, r1 = g2[0].tolist(), g2[1].tolist()
    k2 = next(i for i in range(2, n_new - 2) if r0[i] not in r0[:i] and r0[i] not in r1)
    eos_b2 = r0[k2]
    cases = [("b1", True, ids[:1], pixels[:1], torch.ones_like(ids[:1]), None),
             ("b1_eos", True, ids[:1], pixels[:1], torch.ones_like(ids[:1]), [eos_b1]),
             ("b2_padded_eos", False, ids_pad, pixels, mask_pad, [eos_b2])]
    out, meta = {}, []
    for name, at_head, x, px, mask, eos in cases:
        events = []
        model.image_at_head = at_head
        gc = GenerationConfig(do_sample=False, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=0, bos_token_id=1)
        seq = model.generate(input_ids=x, pixel_values=px, attention_mask=mask, generation_config=gc,
                             streamer=RecordingStreamer(events), stopping_criteria=[recording_criterion(events)])
        out[f"{name}_input_ids"] = x.numpy()
        out[f"{name}_attention_mask"] = mask.numpy()
        out[f"{name}_pixel_values"] = px.numpy()
        out[f"{name}_sequences"] = seq.numpy()
        meta.append(dict(name=name, image_at_head=at_head, eos=eos or [], pad_token_id=0, max_new_tokens=n_new, events=events))
        print(f"[golden] tiny_stream {name}: sequences {seq.tolist()} events {len(events)} "
              f"(first put {events[0]['shape']} {events[0]['dtype']})")
    np.savez_compressed(os.path.join(OUT, "tiny_stream.npz"), config=np.array(repr(cfg.to_dict())), seed=np.array(seed),
                        cases=np.array(json.dumps(meta)), **out)


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(os.cpu_count() or 1)
    case_tiny_stream(import_reference())
