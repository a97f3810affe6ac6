"""Per-sequence stops of the batched greedy decode (LlamaDecoder._decode_batched): with an EOS id or a stopping criterion, every
sequence of a generate_batch call is its plain output cut after its own first stop, in graph and in eager mode."""
import pytest
import torch

from tests.test_gpu_packed_decode import _decoder

pytestmark = pytest.mark.gpu
DEV = "cuda"
N = 24


def _cut(ids, eos, stop):
    for k in range(len(ids)):
        if ids[k] in eos or (stop is not None and stop(torch.tensor(ids[:k + 1]))):
            return ids[:k + 1]
    return ids


def _pick_eos(plain):
    """The token whose first occurrences are spread over the most different steps (absent counts as one more)."""
    def spread(t):
        firsts = [p.index(t) if t in p else None for p in plain]
        return len(set(firsts)), sum(f is not None for f in firsts), -t
    return max({t for p in plain for t in p}, key=spread)


def test_batched_decode_stops_each_sequence_on_its_own(monkeypatch):
    dec = _decoder(monkeypatch, True)
    lens = [12, 20, 7, 15]
    x = (torch.randn(sum(lens), 4096, generator=torch.Generator().manual_seed(21)) * 0.3).to(torch.bfloat16).to(DEV)
    plain = [p.tolist() for p in dec.generate_batch(x, lens, N)]
    eos = _pick_eos(plain)
    # a criterion on the history: it fires on these prefixes only, so each sequence stops at its own step (or never)
    targets = lambda lengths: {tuple(p[:n]) for p, n in zip(plain, lengths) if n}  # noqa: E731
    some, every = targets([3, 9, None, 14]), targets([5, 2, 11, 17])
    cases = [
        ([eos], None),
        (None, lambda ids: tuple(ids.tolist()) in some),
        (None, lambda ids: tuple(ids.tolist()) in every),  # all sequences stop before the budget: the loop ends early
        ([eos], lambda ids: tuple(ids.tolist()) in some),
    ]
    for eos_ids, stop in cases:
        want = [_cut(p, eos_ids or [], stop) for p in plain]
        assert len({len(w) for w in want}) >= 2  # the sequences stop at different steps
        for graph in (True, False):
            got = dec.generate_batch(x, lens, N, eos_token_ids=eos_ids, stopping_fn=stop, use_graph=graph)
            assert [g.tolist() for g in got] == want, (eos_ids, graph)
