"""Beam search over a batch of prompts on the H100 (LlamaDecoder.generate_beam_batch, generate(B > 1, num_beams=k)): the merge and KV-copy
kernels against torch bit for bit, every prompt against HF's batched generate (tests/golden/beam_batch_kats.npz), graph against eager,
the independence of a prompt's ids from the other prompts of its batch, the stopping rules, the multimodal API against the oracle, and
the quantized weight formats."""
import dataclasses
import os

import pytest
import torch

from oracle import srgpt_oracle as O
from tests.golden.make_beam_batch_golden import BEAM_BATCH_CASES
from tests.golden.make_golden import CASES
from tests.util import load_npz

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.bfloat16, torch.float16]


@pytest.mark.parametrize("G,k,n_cand,V", [(1, 3, 6, 1003), (4, 3, 6, 1003), (42, 3, 6, 128259), (8, 4, 12, 32003), (16, 2, 4, 50)])
def test_beam_select_matches_a_torch_sort(G, k, n_cand, V):
    from spatialrgpt_b200 import ops
    g = torch.Generator().manual_seed(G * 7 + V)
    # integer logits tie often; a row of only a few finite logits leaves candidates with token -1
    logits = torch.randint(-3, 3, (G * k, V), generator=g).to(torch.bfloat16)
    logits[1, 4:] = float("-inf") if V > 8 else logits[1, 4:]
    ld = (V + 7) // 8 * 8
    d_logits = torch.zeros(G * k, ld, dtype=torch.bfloat16, device=DEV)[:, :V]
    d_logits.copy_(logits)
    scores = torch.tensor([[0.0, -0.5, -1e9, -0.5][i % 4] for i in range(G * k)], device=DEV)
    cs = torch.empty(G * k, n_cand, dtype=torch.float32, device=DEV)
    ct = torch.empty(G * k, n_cand, dtype=torch.int32, device=DEV)
    ops.beam_candidates(d_logits, scores, cs, ct)
    os_, ob, ot = (torch.empty(G, n_cand, dtype=t, device=DEV) for t in (torch.float32, torch.int32, torch.int32))
    ops.beam_select(cs, ct, k, os_, ob, ot)
    # torch: a stable sort of the negated scores over each prompt's flattened [k x n_cand] table (beam-major, each row token-ascending on
    # ties), invalid candidates last
    flat_s, flat_t = cs.view(G, k * n_cand), ct.view(G, k * n_cand)
    key = torch.where(flat_t >= 0, -flat_s, torch.full_like(flat_s, float("inf")))
    order = torch.sort(key, dim=1, stable=True).indices[:, :n_cand]
    valid = torch.gather(flat_t, 1, order) >= 0
    ref_s = torch.where(valid, torch.gather(flat_s, 1, order), torch.full_like(os_, float("-inf")))
    ref_b = torch.where(valid, (order // n_cand).to(torch.int32), torch.full_like(ob, -1))
    ref_t = torch.where(valid, torch.gather(flat_t, 1, order), torch.full_like(ot, -1))
    assert torch.equal(os_.view(torch.int32), ref_s.view(torch.int32)) and torch.equal(ob, ref_b) and torch.equal(ot, ref_t)


@pytest.mark.parametrize("dtype", DTYPES)
def test_kv_copy_pages_matches_torch_indexing(dtype):
    from spatialrgpt_b200 import ops
    L, n_pages, nkv, hd = 3, 40, 2, 64
    g = torch.Generator().manual_seed(3)
    pages = torch.randn(L, n_pages, 2, 16, nkv, hd, generator=g).to(dtype).to(DEV)
    # a 2-cycle (5 <-> 9) and a 3-cycle (1 -> 2 -> 3 -> 1) staged; a parent with two children (20 -> 21, 20 -> 22) and partial rows direct
    pairs = [(5, 9, 0, 16), (9, 5, 0, 16), (1, 2, 3, 7), (2, 3, 3, 7), (3, 1, 3, 7), (20, 21, 0, 16), (20, 22, 4, 12), (30, 31, 15, 1)]
    n_staged = 5
    ref = pages.clone()
    snap = pages.clone()
    for s, d, lo, n in pairs:  # gather from the state before the copy, then scatter: what pages_all[:, dst] = pages_all[:, src] does
        ref[:, d, :, lo:lo + n] = snap[:, s, :, lo:lo + n]
    ops.kv_copy_pages(pages, pairs, n_staged)
    assert torch.equal(pages.view(torch.int16), ref.view(torch.int16))
    touched = {d for _, d, _, _ in pairs}
    untouched = [p for p in range(n_pages) if p not in touched]
    assert torch.equal(pages[:, untouched].view(torch.int16), snap[:, untouched].view(torch.int16))
    assert torch.equal(pages[:, 3, :, :3].view(torch.int16), snap[:, 3, :, :3].view(torch.int16))  # rows outside a pair's range stay
    # the prompt replication: whole pages from beam 0's pages to the others, nothing staged
    ops.kv_copy_pages(pages, [(0, 35, 0, 16), (0, 36, 0, 16), (4, 37, 0, 9)])
    assert torch.equal(pages[:, 35], pages[:, 0]) and torch.equal(pages[:, 36], pages[:, 0])
    assert torch.equal(pages[:, 37, :, :9], pages[:, 4, :, :9])


def _model(dtype):
    from tests.test_gpu_fp16 import build_model
    g = load_npz(os.path.join(os.path.dirname(__file__), "golden", "beam_batch_kats.npz"))
    oc, sd, model = build_model(CASES["tiny_masks_gqa"][0], int(g["weight_seed"]), dtype=dtype)
    return g, oc, sd, model


def _row_matches(ids, ref, eos):
    """ids equal HF's row up to their length; HF fills the rest with 0 or (transformers 5.5) the EOS id."""
    return ids == ref[:len(ids)] and all(t in (0, (eos or [0])[0]) for t in ref[len(ids):])


@pytest.mark.parametrize("dtype,need", [(torch.float16, 28), (torch.bfloat16, 24)])
def test_beam_batch_matches_hf_batched_generate(dtype, need):
    """fp16 reproduces every prompt of every case; bf16 gets the near-tie allowance test_gpu_beam.py documents for one prompt (the
    reference's own bf16 arithmetic flips near-ties).  Graph and eager steps give equal ids."""
    g, oc, sd, model = _model(dtype)
    packed = g["packed_embeds"].to(DEV)
    lens = [int(n) for n in g["seq_lens"]]
    ok = []
    for i, (nb, eos, n_new, lp, es) in enumerate(BEAM_BATCH_CASES):
        out = model.llm.generate_beam_batch(packed, lens, nb, n_new, eos_token_ids=eos, length_penalty=lp, early_stopping=es)
        eager = model.llm.generate_beam_batch(packed, lens, nb, n_new, eos_token_ids=eos, length_penalty=lp, early_stopping=es, use_graph=False)
        assert [t.tolist() for t in out] == [t.tolist() for t in eager], i
        ok += [_row_matches(out[b].tolist(), g[f"case{i}"][b].tolist(), eos) for b in range(len(lens))]
    print(f"beam batch {dtype}: prompts equal to HF generate: {sum(ok)} of {len(ok)} {ok}")
    assert sum(ok) >= need, ok


def test_stopping_holds_for_every_row_and_finished_prompts_stay_frozen():
    g, oc, sd, model = _model(torch.float16)
    packed = g["packed_embeds"].to(DEV)
    lens = [int(n) for n in g["seq_lens"]]
    nb, eos, n_new, lp, es = BEAM_BATCH_CASES[3]  # prompt 0 closes its hypotheses after 2 tokens, the others run on
    full = [t.tolist() for t in model.llm.generate_beam_batch(packed, lens, nb, n_new, eos_token_ids=eos)]
    assert len(full[0]) == 2 and all(len(t) == n_new for t in full[1:])
    seen = []

    def stop_at_5(ids):
        seen.append(ids.numel())
        return ids.numel() >= 5

    stopped = [t.tolist() for t in model.llm.generate_beam_batch(packed, lens, nb, n_new, eos_token_ids=eos, stopping_fn=stop_at_5)]
    five = [t.tolist() for t in model.llm.generate_beam_batch(packed, lens, nb, 5, eos_token_ids=eos)]
    assert stopped[0] == full[0]  # finished before the stop: frozen
    for b in range(1, len(lens)):  # stopped after 5 tokens: the finalize of a 5-token budget, with the EOS appended as HF does
        assert stopped[b] == (five[b] + [eos[0]] if len(five[b]) == 5 else five[b]), (b, stopped[b], five[b])
    assert max(seen) == 5
    never = [t.tolist() for t in model.llm.generate_beam_batch(packed, lens, nb, n_new, eos_token_ids=eos, stopping_fn=lambda ids: False)]
    assert never == full
    # a criterion that holds for only some rows does not stop the run
    some = [t.tolist() for t in model.llm.generate_beam_batch(packed, lens, nb, n_new, eos_token_ids=eos,
                                                               stopping_fn=lambda ids: ids.numel() >= 5 and int(ids[0]) == full[1][0])]
    assert some == full


def _long_prompts(H, dtype, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, H, generator=g) * 0.3).to(dtype).to(DEV) for n in lens]


def _composition_check(dec, prompts, k, n_new, eos=None):
    """Each prompt's ids do not depend on the other prompts of its batch: every batch has B * k <= 128 rows per step and packs more than
    128 prompt rows, so each GEMM keeps one configuration (whose per-row results do not depend on M) and attention runs per sequence."""
    def run(idx, **kw):
        return dec.generate_beam_batch(torch.cat([prompts[i] for i in idx]), [prompts[i].shape[0] for i in idx], k, n_new, eos_token_ids=eos, **kw)
    n = len(prompts)
    base = run(list(range(n)))
    assert [t.tolist() for t in base] == [t.tolist() for t in run(list(range(n)), use_graph=False)]
    for idx in ([n - 1, 0], list(reversed(range(n))), [1], [2, 0, 3] if n > 3 else [2, 0]):
        for i, t in zip(idx, run(idx)):
            assert t.tolist() == base[i].tolist(), (idx, i)
    return base


@pytest.mark.parametrize("dtype", DTYPES)
def test_batch_composition_invariance(dtype):
    g, oc, sd, model = _model(dtype)
    prompts = _long_prompts(oc.hidden, dtype, [131, 150, 129, 170, 140], 11)
    _composition_check(model.llm, prompts, 3, 12)
    _composition_check(model.llm, prompts[:4], 4, 10, eos=[460])


def test_generate_api_batch_of_multimodal_prompts_equals_the_oracle(golden_dir):
    from tests.test_gpu_fp16 import build_model
    name = "tiny_masks_gqa"
    kw, n_regions, t_text, kind, n_new, depth_on = CASES[name]
    gd = load_npz(os.path.join(golden_dir, name + ".npz"))
    oc, sd, model = build_model(kw, int(gd["weight_seed"]), dtype=torch.float16)
    reqs = [O.synth_request(oc, n_regions, t_text, seed=s, kind=kind) for s in (1234, 1234)]
    # the second request: the same layout with different pixels, depths and masks
    reqs[1] = (reqs[1][0],) + tuple(O.synth_request(oc, n_regions, t_text, seed=77, kind=kind)[1:])
    refs = []
    for input_ids, images, depths, masks in reqs:
        enc = O.encode_multimodal(oc, sd, images, depths, masks)
        embeds = O.splice_embeddings(oc, sd["llm"]["model.embed_tokens.weight"].float(), input_ids, enc["image_features"], enc["mask_embeds"],
                                     enc["depth_embeds"])[0]
        refs.append(O.beam_search_generate(oc, sd["llm"], embeds, 3, 8).tolist())
    h = lambda t: t.to(DEV, torch.float16)  # noqa: E731
    args = dict(images=h(torch.cat([r[1] for r in reqs])), depths=h(torch.cat([r[2] for r in reqs])),
                masks=[h(m) for r in reqs for m in r[3]])
    out = model.generate(torch.cat([r[0] for r in reqs]).to(DEV), num_beams=3, do_sample=False, max_new_tokens=8, **args)
    assert out.shape[0] == 2
    for b in range(2):
        assert out[b].tolist()[:len(refs[b])] == refs[b], (b, out[b].tolist(), refs[b])
    # the text-only path with a left-padded batch: each row equals the batch-1 beam search of its unpadded prompt
    ids = torch.randint(3, 900, (2, 20), generator=torch.Generator().manual_seed(1)).to(DEV)
    mask = torch.ones_like(ids)
    mask[1, :6] = 0
    model.config.llama.tokenizer_padding_side = "left"
    try:
        both = model.generate(ids, attention_mask=mask, num_beams=3, max_new_tokens=6, pad_token_id=0)
        one = [model.generate(ids[0:1], num_beams=3, max_new_tokens=6), model.generate(ids[1:2, 6:], num_beams=3, max_new_tokens=6)]
    finally:
        model.config.llama.tokenizer_padding_side = "right"
    assert both.shape == (2, 6)
    assert [both[b].tolist() for b in range(2)] == [one[b][0].tolist() for b in range(2)]


def _dims():
    from spatialrgpt_b200.config import LlamaDims
    return dataclasses.replace(LlamaDims(), hidden_size=2048, intermediate_size=5120, num_hidden_layers=4, num_attention_heads=16,
                               num_key_value_heads=4, head_dim=128, vocab_size=32003)


@pytest.mark.parametrize("dtype", DTYPES)
def test_fp8_and_nf4_decoders(dtype):
    """The FP8 and NF4 planes-only 4-layer decoders of test_gpu_fp8.py / test_gpu_nf4_planes.py run batched beams through the same step:
    graph equals eager and a prompt's ids do not depend on its batch, and NF4 planes-only equals NF4 copy mode bit for bit."""
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from tests.test_gpu_fp8 import _fp8_llama
    from tests.test_gpu_nf4_planes import _llama, _llm_state_dict
    d = _dims()
    prompts = _long_prompts(d.hidden_size, dtype, [131, 150, 129, 170], 5)
    dec = LlamaDecoder(d, _fp8_llama(d, dtype), max_seq_len=512, max_seqs=2)
    assert dec.fp8
    out = _composition_check(dec, prompts, 3, 10)
    assert all(1 <= t.numel() <= 10 for t in out)
    del dec
    sd = _llm_state_dict(d, 21)
    res = {}
    for copy in (True, False):
        dec = LlamaDecoder(d, _llama(d, sd, dtype, copy), max_seq_len=512, max_seqs=2)
        assert dec.nf4_planes_only == (not copy)
        res[copy] = [t.tolist() for t in _composition_check(dec, prompts, 3, 10)]
        del dec
    assert res[True] == res[False]
