"""Beam search over a batch of prompts, on the CPU: the exports and argument checks of the merge and KV-copy kernels, their SASS, a numpy
restatement of the merge against the host order of the batch-1 loop, the per-step KV copy lists, the combinations that still raise,
and the oracle's per-prompt beam search against HF's batched generate (tests/golden/beam_batch_kats.npz, ``make_beam_batch_golden.py``)."""
import os
import subprocess
import types

import numpy as np
import pytest
import torch

from spatialrgpt_b200.llama_decoder import BeamHypotheses, beam_page_pairs

NEW = ("srgpt_beam_select", "srgpt_kv_copy_workspace_bytes", "srgpt_kv_copy_pages")
BAD = -1


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_both_libraries_export_and_check_arguments(elem):
    from spatialrgpt_b200 import _lib
    lib = _lib.load(elem=elem)
    for name in NEW:
        assert hasattr(lib, name), name
    x = 16  # a 16-byte aligned non-NULL address: every call below fails its argument check before any launch
    ok = [x, x, 2, 3, 6, x, x, x, None]
    for i, v in ((0, None), (1, None), (5, None), (6, None), (7, None), (2, 0), (3, 0), (4, 0), (3, 700), (4, 4096)):
        args = list(ok)
        args[i] = v
        assert lib.srgpt_beam_select(*args) == BAD, i
    assert lib.srgpt_kv_copy_workspace_bytes(3, 32, 16, 2048) == 3 * 32 * 2 * 16 * 2048
    assert lib.srgpt_kv_copy_workspace_bytes(-1, 32, 16, 2048) == -1
    ok = [x, 4, 64, 16, 256, x, 5, 0, None, 0, None]
    for i, v in ((0, None), (5, None), (1, 0), (2, 0), (3, 0), (4, 24), (6, 0), (7, 6), (7, -1), (8, 17)):
        args = list(ok)
        args[i] = v
        assert lib.srgpt_kv_copy_pages(*args) == BAD, i
    args = list(ok)
    args[7], args[8], args[9] = 2, x, 2 * 4 * 2 * 16 * 256 - 1  # a workspace one byte short
    assert lib.srgpt_kv_copy_pages(*args) == BAD
    assert "invalid argument" in _lib.last_error()


def test_new_kernels_in_the_sass_without_local_memory():
    from spatialrgpt_b200 import _lib
    for elem in ("bf16", "f16"):
        _lib.load(elem=elem)
        r = subprocess.run(["cuobjdump", "-sass", _lib.lib_path(elem)], capture_output=True, text=True)
        if r.returncode != 0:
            pytest.skip("cuobjdump unavailable")
        funcs, cur = {}, None
        for line in r.stdout.splitlines():
            if "Function : " in line:
                cur = line.split("Function : ")[1].strip()
                funcs[cur] = []
            elif cur is not None:
                funcs[cur].append(line)
        new = [f for f in funcs if "beam_select_kernel" in f or "kv_copy_kernel" in f]
        assert len(new) == 2, new
        for f in new:
            body = "\n".join(funcs[f])
            assert "LDL" not in body and "STL" not in body, f"{f} uses local memory"


# ---- the merge --------------------------------------------------------------------------------------------------------------------
def merge_restated(cs: np.ndarray, ct: np.ndarray, k: int):
    """beam_select_kernel in numpy: each valid candidate's slot is the number of valid candidates of its prompt before it in
    (score desc, beam asc, token asc) order."""
    G, n_cand = cs.shape[0] // k, cs.shape[1]
    out = np.full((G, n_cand), -np.inf, np.float32), np.full((G, n_cand), -1, np.int32), np.full((G, n_cand), -1, np.int32)
    for g in range(G):
        s, t = cs[g * k:(g + 1) * k].reshape(-1), ct[g * k:(g + 1) * k].reshape(-1)
        b = np.arange(s.size) // n_cand
        for i in np.flatnonzero(t >= 0):
            before = (t >= 0) & ((s > s[i]) | ((s == s[i]) & ((b < b[i]) | ((b == b[i]) & (t < t[i])))))
            r = int(before.sum())
            if r < n_cand:
                out[0][g, r], out[1][g, r], out[2][g, r] = s[i], b[i], t[i]
    return out


def host_order(cs, ct, k, g, n_cand):
    """The batch-1 loop's merge (generate_beam) over prompt g's rows."""
    h_s, h_t = cs[g * k:(g + 1) * k], ct[g * k:(g + 1) * k]
    flat = sorted(((-float(h_s[b, j]), b, int(h_t[b, j])) for b in range(k) for j in range(n_cand) if int(h_t[b, j]) >= 0))[:n_cand]
    return [(-neg, b, t) for neg, b, t in flat]


def candidates(rs, G, k, n_cand, V, ties: bool, drop: float):
    """Rows as srgpt_beam_candidates_bf16 writes them: distinct tokens in (score desc, token asc) order, -inf / -1 at the tail."""
    cs = np.full((G * k, n_cand), -np.inf, np.float32)
    ct = np.full((G * k, n_cand), -1, np.int32)
    for r in range(G * k):
        n = n_cand if rs.rand() > drop else rs.randint(0, n_cand)
        toks = rs.choice(V, n, replace=False)
        sc = (rs.randint(-4, 1, n) * 0.5 if ties else rs.randn(n)).astype(np.float32) - np.float32(1e9 if r % k and rs.rand() < 0.2 else 0)
        order = sorted(range(n), key=lambda i: (-sc[i], toks[i]))
        cs[r, :n], ct[r, :n] = sc[order], toks[order]
    return cs, ct


@pytest.mark.parametrize("G,k,n_cand,ties,drop", [(4, 3, 6, True, 0.0), (7, 3, 6, True, 0.5), (3, 4, 12, False, 0.3), (5, 5, 10, True, 0.9),
                                                  (2, 2, 4, True, 1.0)])
def test_merge_restatement_reproduces_the_host_order(G, k, n_cand, ties, drop):
    rs = np.random.RandomState(G * 100 + k)
    for _ in range(20):
        cs, ct = candidates(rs, G, k, n_cand, 50 if ties else 100000, ties, drop)
        s, b, t = merge_restated(cs, ct, k)
        for g in range(G):
            want = host_order(cs, ct, k, g, n_cand)
            got = [(float(s[g, j]), int(b[g, j]), int(t[g, j])) for j in range(n_cand) if t[g, j] >= 0]
            assert got == want, (g, got, want)
            assert all(t[g, j] == -1 and b[g, j] == -1 and s[g, j] == -np.inf for j in range(len(want), n_cand))


# ---- the KV copies of a step ------------------------------------------------------------------------------------------------------
def run_pairs(pages: np.ndarray, pairs, n_staged: int) -> np.ndarray:
    """The two passes of kv_copy_kernel over pages [n_pages, page_rows]: staged pairs to a workspace and the others to their
    destination, then the staged ones from the workspace."""
    ws = [pages[s, lo:lo + n].copy() for s, _, lo, n in pairs[:n_staged]]
    for s, d, lo, n in pairs[n_staged:]:
        pages[d, lo:lo + n] = pages[s, lo:lo + n]
    for (_, d, lo, n), v in zip(pairs[:n_staged], ws):
        pages[d, lo:lo + n] = v
    return pages


def rows_of(tables, starts, n_gen, page_size=16):
    return {r: [(tables[r][p // page_size], p % page_size) for p in range(starts[r], starts[r] + n_gen)] for r in range(len(tables))}


@pytest.mark.parametrize("parents", [[1, 0, 2, 3, 4, 5], [0, 0, 2, 3, 3, 3], [1, 2, 0, 5, 3, 4], [0, 0, 1, 4, 3, 3], [0, 1, 2, 3, 4, 5]])
@pytest.mark.parametrize("n_gen", [1, 5, 16, 17, 40])
def test_page_pairs_copy_only_generated_rows_of_moved_beams(parents, n_gen):
    # two prompts of three beams: rows 0-2 start at 21, rows 3-5 at 16 (a page boundary); pages are scattered over the cache.  The
    # parents hold a 2-cycle, a parent with two children, 3-cycles, a chain, and no move at all.
    starts = [21] * 3 + [16] * 3
    rs = np.random.RandomState(n_gen)
    perm = rs.permutation(96).tolist()
    tables = [perm[16 * r:16 * r + 5] for r in range(6)]
    pages = rs.randint(0, 1 << 30, (96, 16)).astype(np.int64)  # one value per (page, row) stands for its K and V of every layer
    before = pages.copy()
    pairs, n_staged = beam_page_pairs(tables, parents, starts, n_gen)
    moved = [r for r, p in enumerate(parents) if p != r]
    sources = {parents[r] for r in moved}
    # only pages of moved rows are written, only the rows [start, start + n_gen) of each, and a destination that is a source is staged
    dst_rows = {(d, lo + i) for _, d, lo, n in pairs for i in range(n)}
    want_rows = {pr for r in moved for pr in rows_of(tables, starts, n_gen)[r]}
    assert dst_rows == want_rows
    assert all((any(d in tables[r] for r in sources)) == (i < n_staged) for i, (_, d, _, _) in enumerate(pairs))
    after = run_pairs(pages, pairs, n_staged)
    rows = rows_of(tables, starts, n_gen)
    for r in range(6):
        for (pg, j), (ppg, pj) in zip(rows[r], rows[parents[r]]):
            assert after[pg, j] == before[ppg, pj], (r, pg, j)
    untouched = np.ones_like(pages, dtype=bool)
    for d, j in want_rows:
        untouched[d, j] = False
    assert np.array_equal(after[untouched], before[untouched])
    assert beam_page_pairs(tables, parents, starts, 0) == ([], 0)


def test_beam_hypotheses_follow_the_batch_one_rules():
    h = BeamHypotheses(2, [9], 1.0, False)
    assert h.advance([(-0.5, 0, 9), (-0.7, 0, 4), (-0.9, 0, 5), (-1.2, 0, 6)], 1) == [0, 0]  # the EOS of rank 0 closes [] at -0.5
    assert h.hyps == [(-0.5, [])] and h.seqs == [[4], [5]] and h.scores == [-0.7, -0.9] and not h.done
    assert h.advance([(-1.0, 1, 9), (-1.1, 0, 7), (-1.3, 1, 8), (-1.4, 0, 9)], 2) == [0, 1]  # rank-0 EOS kept; a rank >= k EOS is not
    assert h.hyps == [(-0.5, []), (-0.5, [5])] and h.done  # full and the worst kept (-0.5) beats -1.0 / 2
    assert h.best(10) == [9]
    h = BeamHypotheses(2, [], 1.0, False)
    h.advance([(-0.1, 0, 3), (-0.2, 0, 4)], 1)
    assert h.best(1) == [3]
    with pytest.raises(RuntimeError, match="non-EOS"):
        BeamHypotheses(2, [3], 1.0, False).advance([(-0.1, 0, 3), (-0.2, 0, 4)], 1)


# ---- what still raises -------------------------------------------------------------------------------------------------------------
def test_unsupported_combinations_still_raise_before_gpu_work():
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    gen = getattr(getattr(LlavaLlamaModel.generate, "__wrapped__", None), "__wrapped__", None)
    if gen is None or hasattr(gen, "__wrapped__"):
        pytest.skip("generate is not unwrappable here")

    class NoDevice:  # any device work fails the test
        supports_prompt_lookup = supports_logits_processors = supports_prefix_reuse = True

        def generate_beam(self, *a, **k):
            raise AssertionError("reached the decoder")

        def __getattr__(self, name):
            raise AssertionError(f"reached the decoder ({name})")

    m = LlavaLlamaModel.__new__(LlavaLlamaModel)
    m.config = types.SimpleNamespace(llama=types.SimpleNamespace(eos_token_id=2, vocab_size=1000))
    m.llm = NoDevice()
    ids = torch.tensor([[1, 2, 3], [4, 5, 6]])
    for kw, msg in ((dict(do_sample=True, temperature=0.7), "beam search"), (dict(output_logits=True), "beam search"),
                    (dict(repetition_penalty=1.2), "beam"), (dict(prefix_cache=True), "prefix_cache"),
                    (dict(prompt_lookup_num_tokens=3), "beam")):
        with pytest.raises(NotImplementedError, match=msg):
            gen(m, ids, num_beams=3, **kw)
        with pytest.raises(NotImplementedError, match=msg):
            gen(m, ids[:1], num_beams=3, **kw)
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    m.llm = TPLlamaDecoder.__new__(TPLlamaDecoder)
    for b in (1, 2):
        with pytest.raises(NotImplementedError, match="tensor-parallel"):
            gen(m, ids[:b], num_beams=3)


# ---- the fixture ------------------------------------------------------------------------------------------------------------------
def test_oracle_per_prompt_matches_hf_batched_generate(golden_dir):
    """HF's batched beam search treats every prompt on its own: the oracle's batch-1 restatement over each unpadded prompt gives that
    prompt's row of HF's left-padded batch (rows that end early are filled with the EOS id by transformers 5.5)."""
    from oracle import srgpt_oracle as O
    from tests.golden.make_beam_batch_golden import BEAM_BATCH_CASES
    from tests.golden.make_golden import CASES
    from tests.util import load_npz
    g = load_npz(os.path.join(golden_dir, "beam_batch_kats.npz"))
    oc = O.OracleConfig(**CASES["tiny_masks_gqa"][0])
    sd = O.make_weights(oc, seed=int(g["weight_seed"]))
    lens = [int(n) for n in g["seq_lens"]]
    off = np.cumsum([0] + lens)
    short = 0
    for i, (nb, eos, n_new, lp, es) in enumerate(BEAM_BATCH_CASES):
        for b in range(len(lens)):
            ids = O.beam_search_generate(oc, sd["llm"], g["packed_embeds"][off[b]:off[b + 1]], nb, n_new, eos_token_id=eos, length_penalty=lp,
                                         early_stopping=es).tolist()
            ref = g[f"case{i}"][b].tolist()
            assert ids == ref[:len(ids)] and all(t in (0, (eos or [0])[0]) for t in ref[len(ids):]), (i, b, ids, ref)
            short += len(ids) < n_new
    assert short >= 1  # at least one prompt finishes before the others
