"""The oracle's beam search (oracle/beam_oracle.py:beam_search, a restatement of HF 5.5's _beam_search) reproduces every case the
reference's own generate(num_beams=...) produced on the tiny config (tests/golden/tiny_beams.npz): tokens and lengths exactly, the
sequence scores within 1e-5."""
import json
import os

import numpy as np
import pytest
import torch

import beam_oracle as BO
import visualcla_oracle as O

Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_beams.npz"))
CASES = json.loads(str(Z["cases"]))


@pytest.fixture(scope="module")
def weights():
    return O.make_weights(O.tiny_config(), int(Z["seed"]))


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_beam_search_matches_reference(weights, case):
    cfg = O.tiny_config()
    n = case["name"]
    ids = torch.from_numpy(Z[f"{n}_input_ids"])
    mask = torch.from_numpy(Z[f"{n}_attention_mask"])
    pads = (mask == 0).sum(1) if bool((mask == 0).any()) else None
    px = None if case["layout"] == "text" else torch.from_numpy(Z["pixel_values"])
    seqs, scores, _ = BO.beam_search(weights, cfg, ids, px, case["num_beams"], case["max_new_tokens"],
                                    image_at_head=case["layout"] in ("head", "text"), left_pad=pads, eos_token_id=case["eos"],
                                    pad_token_id=case["pad_token_id"], length_penalty=case.get("length_penalty", 1.0),
                                    early_stopping=case.get("early_stopping", False),
                                    num_return_sequences=case.get("num_return_sequences", 1),
                                    repetition_penalty=case.get("repetition_penalty", 1.0),
                                    no_repeat_ngram_size=case.get("no_repeat_ngram_size", 0))
    ref = torch.from_numpy(Z[f"{n}_sequences"])
    assert seqs.shape == ref.shape and torch.equal(seqs, ref)
    assert float((scores - torch.from_numpy(Z[f"{n}_scores"])).abs().max()) <= 1e-5


def test_fixture_covers_the_issue_cases():
    names = {c["name"] for c in CASES}
    assert {"k4", "eos_es_true", "eos_es_false", "eos_es_never", "lp_2", "lp_neg", "nrs_2", "rep_ngram", "padded"} <= names
    eos_case = Z["eos_es_true_sequences"]
    eos = next(c["eos"] for c in CASES if c["name"] == "eos_es_true")[0]
    first = [list(r).index(eos) if eos in r else None for r in eos_case.tolist()]
    assert any(f is not None and f < 5 for f in first), "a hypothesis should finish early on the EOS id"


def test_output_fill_value_precedence():
    assert BO.output_fill_value(0, [64]) == 64          # pad 0 is falsy: `pad or eos[0]`
    assert BO.output_fill_value(7, [64]) == 7
    assert BO.output_fill_value(None, [64, 3]) == 64
    assert BO.output_fill_value(0, []) == -1
