"""Draft rule of prompt lookup decoding (HF:generation/candidate_generator.py PromptLookupCandidateGenerator.get_candidates, without its
optional forbidden-token cropping and its cropping at an EOS id: the verification stops at an emitted EOS, so neither changes a token),
restated over a plain list of token ids: the text the device searches is the call's prompt ids
followed by the tokens emitted so far."""
from typing import List, Sequence


def draft(text: Sequence[int], k: int, n: int, room: int = 1 << 30) -> List[int]:
    """For g = min(n, len(text) - 1) .. 1: the leftmost earlier window equal to the last g tokens whose continuation is non-empty;
    the draft is up to k tokens of that continuation, and at most `room` tokens (max_new - emitted - 1).  [] when nothing matches."""
    text = [int(t) for t in text]
    N = len(text)
    for g in range(min(n, N - 1), 0, -1):
        tail = text[N - g:]
        for i in range(0, N - g):
            if text[i:i + g] == tail:
                return text[i + g:i + g + max(0, min(k, room))]
    return []
