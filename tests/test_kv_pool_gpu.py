"""What the device KV page allocator hands out, against tests/golden/kv_pool.json.  Each scenario runs on a fresh context and takes
snapshots of the allocator after its steps: a prefill with left padding at page_tokens 8 and 64, decode steps that cross page
boundaries at B = 1, 17 and 40 (eager, graph and decode_many steps), truncate then extend, a beam fork whose steps copy pages on write,
prompt lookup verification steps and a prefill after a shuffled hand-out order.

Recorded per snapshot: the page table row of every sequence up to the pages it owns, the owned counts of all max_batch sequences, the
free page count, the exhausted flag, beam_cow_bytes() and, for prompt lookup, lookup_stats().  The allocator is one serial thread, so
its output depends only on the calls and on what it is told: the beam and lookup scenarios hand out pages after the tokens the model
picked (and lookup's rows per step follow the SM count), so their snapshots are compared only on the device the golden was recorded on
(name and SM count); every other scenario is compared on any H100.

    python tests/test_kv_pool_gpu.py --record     rewrites the golden on the current device"""
import json
import os
import sys

import pytest
import torch

if __name__ == "__main__":
    _root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [os.path.join(_root, "visual-chinese-llama-alpaca_b200"), os.path.join(_root, "oracle")]

import visualcla_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kv_pool.json")
CFG = O.PathConfig(v_layers=1, r_layers=1, t_hidden=256, t_heads=2, t_ffn=448, t_layers=2, t_vocab=1003)
TOKEN_DEPENDENT = ("beam", "lookup")


class _Engines:
    """Makes Engine(max_batch, max_seq, page_tokens) contexts with seeded synthetic weights and closes them all at the end."""

    def __init__(self):
        self.made = []

    def __call__(self, max_batch, max_seq, page_tokens):
        from visualcla.engine import Engine
        eng = Engine(CFG.to_dict(), max_batch=max_batch, max_seq=max_seq, page_tokens=page_tokens)
        eng.init_synthetic(0)
        self.made.append(eng)
        return eng

    def close(self):
        torch.cuda.synchronize()
        for eng in self.made:
            eng.close()
        torch.cuda.empty_cache()


@pytest.fixture
def make_engine():
    engines = _Engines()
    yield engines
    engines.close()


def _ids(eng, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(10, eng.vocab - 10, (B, T), generator=g)


def _snap(eng, B, lookup=False):
    torch.cuda.synchronize()
    table, owned, free, exhausted = eng.kv_pages()
    out = dict(rows=[table[b, : int(owned[b])].tolist() for b in range(B)], owned=owned.tolist(), free=free, exhausted=exhausted,
               cow_bytes=eng.beam_cow_bytes())
    if lookup:
        out["lookup_stats"] = list(eng.lookup_stats())
    return out


def _prefill_leftpad(make, pt):
    eng = make(8, 128, pt)
    B, T = 5, 37
    pad = torch.tensor([0, 3, 8, 17, 36], dtype=torch.int32)
    _, tok, _ = eng.prefill(_ids(eng, B, T, 11), 0, None, left_pad=pad)
    snaps = [_snap(eng, B)]
    buf = eng.token_buffer(B)
    buf.copy_(tok)
    for _ in range(3):
        eng.decode_step(buf, buf, None, use_graph=False)
    snaps.append(_snap(eng, B))
    return snaps


def _decode_cross(make, B):
    eng = make(64, 64, 8)
    _, tok, _ = eng.prefill(_ids(eng, B, 5, 100 + B), 0, None)
    snaps = [_snap(eng, B)]
    buf = eng.token_buffer(B)
    buf.copy_(tok)
    for _ in range(3):
        eng.decode_step(buf, buf, None, use_graph=False)
    snaps.append(_snap(eng, B))
    for _ in range(3):
        eng.decode_step(buf, buf, None, use_graph=True)
    snaps.append(_snap(eng, B))
    eng.decode_many(buf, 12)
    snaps.append(_snap(eng, B))
    return snaps


def _truncate_extend(make):
    eng = make(4, 128, 8)
    B = 3
    _, tok, _ = eng.prefill(_ids(eng, B, 21, 5), 0, None)
    buf = eng.token_buffer(B)
    buf.copy_(tok)
    eng.decode_many(buf, 10)
    snaps = [_snap(eng, B)]
    eng.truncate([9, 30, 24])
    snaps.append(_snap(eng, B))
    _, tok, _ = eng.extend(_ids(eng, B, 13, 6))
    snaps.append(_snap(eng, B))
    buf.copy_(tok)
    for _ in range(4):
        eng.decode_step(buf, buf, None, use_graph=False)
    snaps.append(_snap(eng, B))
    return snaps


def _beam(make):
    eng = make(8, 64, 8)
    items, K = 2, 4
    eng.set_beam(eng.beam_spec(K, 14, eos_token_id=()))
    try:
        _, first, _ = eng.prefill(_ids(eng, items, 13, 77), 0, None, last_logits=False)
        snaps = [_snap(eng, items * K)]
        buf = eng.token_buffer(items * K)
        buf.copy_(first)
        for s in range(1, 11):
            eng.decode_step(buf, buf, None, use_graph=(s % 2 == 0))
            snaps.append(_snap(eng, items * K))
    finally:
        torch.cuda.synchronize()
        eng.set_beam(None)
    return snaps


def _lookup(make):
    eng = make(1, 128, 8)
    ids = _ids(eng, 1, 20, 9)
    buf = eng.token_buffer(1)
    _, tok, _ = eng.prefill(ids, 0, None)
    buf.copy_(tok)
    eng.decode_many(buf, 24)
    greedy = eng.read_history(1, 25).cpu().t()
    # searching the prompt followed by its own greedy continuation drafts tokens the verification steps accept
    _, tok, _ = eng.prefill(ids, 0, None)
    buf.copy_(tok)
    eng.set_lookup(torch.cat([ids, greedy.long()], 1), k=7, n=2, max_new=48)
    try:
        snaps = []
        for _ in range(3):
            eng.decode_many(buf, 4)
            snaps.append(_snap(eng, 1, lookup=True))
    finally:
        torch.cuda.synchronize()
        eng.set_lookup(None)
    return snaps


def _shuffled(make):
    eng = make(4, 96, 8)
    eng.kv_debug_shuffle(7)
    B = 3
    pad = torch.tensor([0, 4, 9], dtype=torch.int32)
    _, tok, _ = eng.prefill(_ids(eng, B, 30, 3), 0, None, left_pad=pad)
    snaps = [_snap(eng, B)]
    buf = eng.token_buffer(B)
    buf.copy_(tok)
    eng.decode_many(buf, 8)
    snaps.append(_snap(eng, B))
    return snaps


SCENARIOS = {
    "prefill_leftpad/pt8": lambda make: _prefill_leftpad(make, 8),
    "prefill_leftpad/pt64": lambda make: _prefill_leftpad(make, 64),
    "decode_cross/B1": lambda make: _decode_cross(make, 1),
    "decode_cross/B17": lambda make: _decode_cross(make, 17),
    "decode_cross/B40": lambda make: _decode_cross(make, 40),
    "truncate_extend/B3": _truncate_extend,
    "beam/K4": _beam,
    "lookup/k7": _lookup,
    "shuffled/B3": _shuffled,
}


def _device():
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    return {"name": p.name, "sms": p.multi_processor_count}


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_golden_covers_every_scenario():
    assert sorted(_golden()["scenarios"]) == sorted(SCENARIOS)


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_kv_pool_matches_golden(name, make_engine):
    golden = _golden()
    if name.split("/")[0] in TOKEN_DEPENDENT and golden["device"] != _device():
        pytest.skip(f"{name} depends on picked tokens; the golden was recorded on {golden['device']}")
    got = json.loads(json.dumps(SCENARIOS[name](make_engine)))
    assert got == golden["scenarios"][name]


if __name__ == "__main__":
    if sys.argv[1:] != ["--record"]:
        sys.exit(__doc__)
    recs = {}
    for name, fn in SCENARIOS.items():
        engines = _Engines()
        recs[name] = fn(engines)
        engines.close()
    lines = ["{", f'  "device": {json.dumps(_device())},', '  "scenarios": {']
    for i, (name, rec) in enumerate(recs.items()):
        lines.append(f"    {json.dumps(name)}: {json.dumps(rec, sort_keys=True)}" + ("," if i + 1 < len(recs) else ""))
    lines += ["  }", "}"]
    with open(GOLDEN, "w") as f:
        f.write("\n".join(lines) + "\n")
    print(f"wrote {GOLDEN}: {len(recs)} scenarios on {_device()}")
