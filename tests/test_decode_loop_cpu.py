"""The stop predicate every decode loop of LlamaDecoder applies to the ids it has copied to the host (llama_decoder.first_stop):
where a request ends inside a window of generated tokens, by EOS, by a stopping criterion or by the token budget."""
import torch

from spatialrgpt_b200.llama_decoder import eos_list, first_stop

IDS = torch.tensor([5, 9, 2, 7, 9, 3, 8, 1], dtype=torch.int64)


def test_eos_at_the_first_middle_and_last_position_of_a_window():
    assert first_stop(IDS, 1, 4, [9], None, 100) == 2   # first position of [1, 4)
    assert first_stop(IDS, 0, 4, [2], None, 100) == 3   # middle
    assert first_stop(IDS, 2, 6, [3], None, 100) == 6   # last
    assert first_stop(IDS, 2, 6, [9], None, 100) == 5   # the first EOS inside the window, not the one before it


def test_several_eos_ids_stop_at_the_first_of_any():
    assert first_stop(IDS, 0, 8, [8, 7], None, 100) == 4
    assert first_stop(IDS, 0, 8, {3, 1}, None, 100) == 6
    assert first_stop(IDS, 0, 8, [], None, 100) is None


def test_stopping_fn_fires_at_k_and_sees_the_ids_up_to_k():
    seen = []

    def fn(ids):
        seen.append(ids.tolist())
        return len(ids) == 5

    assert first_stop(IDS, 2, 8, [], fn, 100) == 5
    assert seen == [IDS[:3].tolist(), IDS[:4].tolist(), IDS[:5].tolist()]
    assert first_stop(IDS, 0, 8, [1], lambda ids: int(ids[-1]) == 7, 100) == 4  # whichever fires first
    assert first_stop(IDS, 0, 8, [2], lambda ids: int(ids[-1]) == 7, 100) == 3


def test_neither_fires():
    assert first_stop(IDS, 0, 8, [42], lambda ids: False, 100) is None
    assert first_stop(IDS, 3, 8, [42], None, 8) == 8      # the window reaches the budget
    assert first_stop(IDS, 3, 7, [42], None, 8) is None   # it does not
    assert first_stop(IDS, 5, 5, [42], None, 5) == 5      # an empty window at the budget


def test_windows_that_straddle_the_limit():
    # tokens at or past the budget are never inspected: the request returns `limit` tokens whatever they are
    assert first_stop(IDS, 2, 8, [8], None, 5) == 5
    assert first_stop(IDS, 2, 8, [3], None, 5) == 5
    assert first_stop(IDS, 2, 8, [7], None, 5) == 4
    calls = []
    assert first_stop(IDS, 2, 8, [], lambda ids: calls.append(len(ids)), 5) == 5
    assert calls == [3, 4, 5]


def test_eos_list_keeps_the_order():
    assert eos_list(None) == []
    assert eos_list(7) == [7]
    assert eos_list(torch.tensor(7)) == [7]
    assert eos_list([9, 2, 5]) == [9, 2, 5]
    assert eos_list((3, 1)) == [3, 1]
