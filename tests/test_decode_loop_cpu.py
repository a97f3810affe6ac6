"""The stop predicate every decode loop of LlamaDecoder applies to the ids it has copied to the host (llama_decoder.first_stop):
where a request ends inside a window of generated tokens, by EOS, by a stopping criterion or by the token budget.  And the
pipelined loop of the one-token, batched and rows steps (llama_decoder.decode_steps), driven by fake launches and copies."""
import torch

from spatialrgpt_b200.llama_decoder import decode_steps, eos_list, first_stop

IDS = torch.tensor([5, 9, 2, 7, 9, 3, 8, 1], dtype=torch.int64)
UNSEEN = -7  # what a host row holds until its copy has been waited for


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


class FakeDevice:
    """The device side of decode_steps: ``ids`` [T, B] is what the steps produce (row 0 is the first token, already there).
    launch(n) and fetch(n) are logged; a fetched row lands in ``host`` only when its copy is waited for, and a fetch of a row whose
    step was not launched fails."""

    def __init__(self, ids):
        self.ids = torch.tensor(ids, dtype=torch.int64)
        self.host = torch.full(self.ids.shape, UNSEEN, dtype=torch.int64)
        self.log = []

    def launch(self, n):
        assert ("launch", n) not in self.log
        self.log.append(("launch", n))

    def fetch(self, n):
        assert n == 0 or ("launch", n) in self.log, f"row {n} copied before its step was launched"
        self.log.append(("fetch", n))
        dev = self

        class Copy:
            def synchronize(self):
                dev.log.append(("wait", n))
                dev.host[n] = dev.ids[n]
        return Copy()

    def run(self, budgets, eos=(), stopping_fn=None):
        return decode_steps(self.launch, self.fetch, self.host, budgets, list(eos), stopping_fn)

    def launches(self):
        return [n for op, n in self.log if op == "launch"]


def rows(*cols):
    """[T, B] ids from B columns of equal length."""
    return [list(r) for r in zip(*cols)]


def test_step_n_is_launched_before_row_n_minus_1_is_inspected():
    dev = FakeDevice(rows([5, 6, 7, 2, 8, 8]))
    assert dev.run([6], eos=[2]) == [4]
    assert dev.log == [("fetch", 0),
                       ("launch", 1), ("fetch", 1), ("wait", 0),
                       ("launch", 2), ("fetch", 2), ("wait", 1),
                       ("launch", 3), ("fetch", 3), ("wait", 2),
                       ("launch", 4), ("fetch", 4), ("wait", 3)]  # the stop is seen while step 4 runs; step 5 is never launched


def test_eos_length_at_every_position():
    col = [11, 12, 13, 14, 15, 16, 17]
    for k in range(7):
        dev = FakeDevice(rows(col))
        assert dev.run([7], eos=[col[k]]) == [k + 1]
        assert dev.launches() == list(range(1, min(k + 2, 7)))  # one step past the stop is in flight, none past the budget
    dev = FakeDevice(rows(col))
    assert dev.run([7], eos=[99]) == [7]


def test_several_eos_ids_and_a_stopping_criterion():
    dev = FakeDevice(rows([4, 3, 9, 8, 7, 6]))
    assert dev.run([6], eos=[7, 8]) == [4]
    seen = []

    def fn(ids):
        seen.append(ids.tolist())
        return int(ids.sum()) >= 16
    dev = FakeDevice(rows([4, 3, 9, 8, 7, 6]))
    assert dev.run([6], stopping_fn=fn) == [3]
    assert seen == [[4], [4, 3], [4, 3, 9]]  # every prefix, each after its last row's copy was waited for
    dev = FakeDevice(rows([4, 3, 9, 8, 7, 6]))
    assert dev.run([6], eos=[3], stopping_fn=fn) == [2]  # whichever fires first


def test_rows_stop_at_their_own_steps_and_stopped_rows_are_ignored():
    ids = rows([1, 2, 0, 0, 0, 0, 0, 0],   # EOS (0) at row 2
               [1, 2, 3, 4, 0, 5, 0, 6],   # at row 4; its later ids are ignored
               [1, 2, 3, 4, 5, 6, 7, 8])   # never
    dev = FakeDevice(ids)
    assert dev.run([8, 8, 8], eos=[0]) == [3, 5, 8]
    assert dev.launches() == list(range(1, 8))
    calls = []

    def fn(ids):
        calls.append(len(ids))
        return False
    dev = FakeDevice(ids)
    assert dev.run([8, 8, 8], eos=[0], stopping_fn=fn) == [3, 5, 8]
    # a stopped row is not inspected again: row 0 is asked about lengths 1-2, row 1 about 1-4, row 2 about 1-7 (its 8th token is the budget)
    assert sorted(calls) == sorted([1, 2] + [1, 2, 3, 4] + list(range(1, 8)))


def test_every_row_stopping_early_ends_the_loop():
    ids = rows([1, 0, 5, 5, 5, 5, 5, 5, 5, 5],
               [1, 2, 3, 0, 5, 5, 5, 5, 5, 5])
    dev = FakeDevice(ids)
    assert dev.run([10, 10], eos=[0]) == [2, 4]
    assert dev.launches() == [1, 2, 3, 4]  # the last stop is row 3, seen while step 4 runs
    assert dev.log[-1] == ("wait", 3)


def test_per_row_budgets():
    ids = rows([1, 2, 3, 4, 5, 6], [1, 2, 3, 4, 5, 6], [1, 2, 0, 4, 5, 6], [1, 2, 3, 4, 5, 6])
    dev = FakeDevice(ids)
    assert dev.run([2, 6, 5, 4], eos=[0]) == [2, 6, 3, 4]
    assert dev.launches() == [1, 2, 3, 4, 5]
    dev = FakeDevice(ids)
    assert dev.run([2, 3, 5, 4], eos=[0]) == [2, 3, 3, 4]  # every row ends by its budget or its EOS: the loop ends early
    assert dev.launches() == [1, 2, 3, 4]
    dev = FakeDevice(rows([1, 2, 3], [1, 2, 3]))
    assert dev.run([2, 3], eos=[3]) == [2, 3]  # row 0's EOS at row 2 is past its budget; row 1's is its last token


def test_budget_of_one_token():
    for eos in ([], [7], [1]):
        dev = FakeDevice(rows([1]))
        assert dev.run([1], eos=eos) == [1]
        assert dev.launches() == []
    dev = FakeDevice(rows([1, 7, 7, 7], [1, 2, 3, 4]))
    assert dev.run([1, 4], eos=[7]) == [1, 4]
    dev = FakeDevice(rows([1, 2, 3, 4], [1, 2, 3, 4]))
    assert dev.run([1, 4]) == [1, 4]


def test_without_a_stop_condition_the_steps_run_back_to_back():
    dev = FakeDevice(rows([1, 0, 0, 0, 0, 0]))
    assert dev.run([6]) == [6]
    assert dev.log == [("launch", n) for n in range(1, 6)]  # max - 1 launches, no copy, no wait
    dev = FakeDevice(rows([1, 0, 0, 0, 0], [1, 0, 0, 0, 0], [1, 0, 0, 0, 0]))
    assert dev.run([5, 2, 4]) == [5, 2, 4]
    assert dev.log == [("launch", n) for n in range(1, 5)]
