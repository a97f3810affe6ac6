"""Sampled batches on the H100: the multi-row sampler against the one-row kernel bit for bit and against torch's sampling distribution,
the batched sampled step of a 4-layer Llama-3-8B-shaped decoder (graph against eager, seeds, every draw replayed through the one-row
kernel, logits processors, EOS, launches), the FP8 and NF4 decoders, and generate(do_sample=True) over batches and with
num_return_sequences."""
import numpy as np
import pytest
import torch

from spatialrgpt_b200.llama_decoder import sequence_seeds

pytestmark = pytest.mark.gpu
DEV = "cuda"
SETTINGS = [(0.7, 0.9, 50), (1.0, 1.0, 0), (1.3, 0.5, None), (0.2, 0.95, 1), (1.5, 1.0, 7), (0.9, 0.3, 0)]  # None: top_k = V + 5


def _rows(R, V, seed, dtype):
    """R rows of logits with a 16-byte aligned row stride (the batched lm_head's layout), some entries -inf as bad words leave them."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, V, generator=g) * 3
    x[:, 5:40:7] = float("-inf")
    x[torch.arange(R), torch.randint(0, V, (R,), generator=g)] = float("-inf")
    x[0, 100:110] = x[0].max() + 1  # ties at the top
    buf = torch.zeros(R, (V + 7) // 8 * 8, dtype=dtype, device=DEV)
    buf[:, :V].copy_(x.to(dtype))
    return buf[:, :V]


def _one_row(ops, row, params, seed: int, counter: int) -> int:
    out = torch.full((counter + 1,), -7, dtype=torch.int64, device=DEV)
    ops.sample_top_p(row.float().contiguous(), params, seed, torch.tensor([counter], dtype=torch.int32, device=DEV), 0, out)
    return int(out[counter])


@pytest.mark.parametrize("R", [1, 3, 32, 200])
@pytest.mark.parametrize("V", [128256, 1003])
@pytest.mark.parametrize("elem", ["f32", "bf16", "f16"])
def test_sample_rows_equals_the_one_row_kernel(R, V, elem):
    from spatialrgpt_b200 import ops
    dtype = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}[elem]
    with ops.elem_dtype(torch.float16 if elem == "f16" else torch.bfloat16):
        x = _rows(R, V, R * 13 + V, dtype)
        seeds = torch.tensor(sequence_seeds(R * 1000 + V, R), dtype=torch.int64, device=DEV)
        step = torch.tensor([5], dtype=torch.int32, device=DEV)
        for t, p, k in SETTINGS:
            params = torch.tensor([t, p, float(V + 5 if k is None else k)], dtype=torch.float32, device=DEV)
            ids = torch.full((R,), -7, dtype=torch.int64, device=DEV)
            ops.sample_rows(x, params, seeds, step, 2, ids)  # counter 7
            want = [_one_row(ops, x[r], params, int(seeds[r]), 7) for r in range(R)]
            assert ids.tolist() == want, (t, p, k)
            assert all(torch.isfinite(x[r, i].float()) for r, i in enumerate(want))


def test_sample_rows_rejects_bad_arguments():
    from spatialrgpt_b200 import ops
    from spatialrgpt_b200._lib import SrgptError
    x = _rows(4, 1003, 1, torch.bfloat16)
    params = torch.tensor([1.0, 1.0, 0.0], device=DEV)
    seeds, step, ids = torch.zeros(4, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV), torch.zeros(4, dtype=torch.int64, device=DEV)
    for bad in (dict(logits=x.half()), dict(logits=x[0]), dict(logits=x.t()), dict(seeds=seeds[:3]), dict(seeds=seeds.int()),
                dict(ids=ids[:3]), dict(ids=ids.int()), dict(params=params[:2]), dict(step=step.long())):
        a = dict(logits=x, params=params, seeds=seeds, step=step, ids=ids)
        a.update(bad)
        with pytest.raises(SrgptError):
            ops.sample_rows(a["logits"], a["params"], a["seeds"], a["step"], 0, a["ids"])


def _reference_distribution(row: np.ndarray, t: float, p: float, k: int) -> np.ndarray:
    """HF's temperature, top-k and top-p warpers over one fp32 row, in float64: the probabilities of the kept tokens."""
    s = row.astype(np.float64) / t
    if 0 < k < s.size:
        s = np.where(s >= np.sort(s)[-k], s, -np.inf)
    pr = np.exp(s - s.max())
    pr /= pr.sum()
    order = np.argsort(-pr, kind="stable")
    cum = np.cumsum(pr[order])
    keep = order[: int(np.searchsorted(cum, p * cum[-1])) + 1]
    out = np.zeros_like(pr)
    out[keep] = pr[keep]
    return out / out.sum()


@pytest.mark.parametrize("t,p,k", [(0.8, 0.9, 20), (1.2, 1.0, 0), (1.0, 0.7, 50)])
def test_distribution_of_one_launch_over_many_seeds(t, p, k):
    from scipy.stats import chisquare

    from spatialrgpt_b200 import ops
    R, V = 4096, 32003
    g = torch.Generator().manual_seed(3)
    row = torch.randn(V, generator=g) * 0.5
    row[torch.randperm(V, generator=g)[:40]] += torch.linspace(2.0, 5.0, 40)  # 40 tokens carry most of the mass
    x = row.to(DEV)[None].expand(R, V).contiguous()
    seeds = torch.tensor(sequence_seeds(99, R), dtype=torch.int64, device=DEV)
    ids = torch.empty(R, dtype=torch.int64, device=DEV)
    params = torch.tensor([t, p, float(k)], dtype=torch.float32, device=DEV)
    ops.sample_rows(x, params, seeds, torch.zeros(1, dtype=torch.int32, device=DEV), 0, ids)
    ref = _reference_distribution(row.numpy(), t, p, k)
    draws = ids.cpu().numpy()
    assert np.all(ref[draws] > 0), "a draw outside the support"
    counts = np.bincount(draws, minlength=V).astype(np.float64)
    exp = ref * R
    big = exp >= 5
    obs_b = np.append(counts[big], counts[~big].sum())
    exp_b = np.append(exp[big], exp[~big].sum())
    if exp_b[-1] == 0:
        obs_b, exp_b = obs_b[:-1], exp_b[:-1]
    pval = chisquare(obs_b, exp_b).pvalue
    assert pval > 1e-3, (pval, int(big.sum()))


# ---- the decoder -----------------------------------------------------------------------------------------------------------------
LENS = [12, 20, 7]
SMP = dict(temperature=0.9, top_p=0.95, seed=11)


def _dec(monkeypatch):
    from tests.test_gpu_packed_decode import _decoder
    return _decoder(monkeypatch, True, layers=4)


def _x(lens, H=4096, seed=9):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(sum(lens), H, generator=g) * 0.3).to(torch.bfloat16).to(DEV)


def _lists(out):
    return [o.tolist() for o in out]


def test_batched_sampling_graph_eager_seeds_and_replayed_draws(monkeypatch):
    from spatialrgpt_b200 import ops
    dec = _dec(monkeypatch)
    x = _x(LENS)
    a = _lists(dec.generate_batch(x, LENS, 16, sampling=SMP))
    assert [len(o) for o in a] == [16] * 3
    assert _lists(dec.generate_batch(x, LENS, 16, sampling=SMP)) == a
    calls = []
    real = ops.sample_rows

    def spy(logits, params, seeds, step, off, ids):
        real(logits, params, seeds, step, off, ids)
        calls.append((logits.clone(), params.clone(), seeds.tolist(), int(step) + off, ids.tolist()))

    monkeypatch.setattr(ops, "sample_rows", spy)
    eager = _lists(dec.generate_batch(x, LENS, 16, sampling=SMP, use_graph=False))
    monkeypatch.setattr(ops, "sample_rows", real)
    assert eager == a
    assert len(calls) == 16  # the first tokens, then one launch per step
    for t, (lg, params, seeds, ctr, ids) in enumerate(calls):
        assert seeds == sequence_seeds(11, 3) and ctr == t
        assert lg.dtype == torch.bfloat16 and lg.shape == (3, dec.dims.vocab_size)
        with ops.elem_dtype(torch.bfloat16):
            assert ids == [_one_row(ops, lg[b], params, seeds[b], ctr) for b in range(3)], t
        assert ids == [a[b][t] for b in range(3)]
    other = _lists(dec.generate_batch(x, LENS, 16, sampling=dict(SMP, seed=12)))
    assert all(u != v for u, v in zip(a, other))
    # the sequential path (output_logits) draws with the same seeds and counters: where its logits rows equal the batched ones the ids agree
    seq, _ = dec.generate_batch(x, LENS, 1, sampling=SMP, return_logits=True)
    assert [s.tolist() for s in seq] == [[o[0]] for o in a]  # the first tokens come from the same lm_head rows


def test_batched_sampling_with_processors_eos_and_launches(monkeypatch):
    from spatialrgpt_b200 import ops
    dec = _dec(monkeypatch)
    x = _x(LENS)
    smp = dict(temperature=1.0, top_k=8, seed=5)
    plain = _lists(dec.generate_batch(x, LENS, 12, sampling=smp))
    banned = sorted({plain[0][1], plain[1][0], plain[2][3]})
    spec = dict(bad_words_ids=[[t] for t in banned], repetition_penalty=1.2)
    fed = []
    real = ops.sample_rows

    def spy(logits, params, seeds, step, off, ids):
        real(logits, params, seeds, step, off, ids)
        fed.append((logits.clone(), params.clone(), seeds.tolist(), int(step) + off, ids.tolist()))

    monkeypatch.setattr(ops, "sample_rows", spy)
    eager = _lists(dec.generate_batch(x, LENS, 12, sampling=smp, processors=spec, use_graph=False))
    monkeypatch.setattr(ops, "sample_rows", real)
    assert _lists(dec.generate_batch(x, LENS, 12, sampling=smp, processors=spec)) == eager
    assert not any(t in banned for o in eager for t in o)
    for lg, params, seeds, ctr, ids in fed:
        assert lg.dtype == torch.float32  # the processed rows
        assert bool(torch.isinf(lg[:, banned]).all())
        assert ids == [_one_row(ops, lg[b], params, seeds[b], ctr) for b in range(3)]
    # EOS: each row ends at its first EOS, the others run on
    eos = plain[1][4]
    cut = _lists(dec.generate_batch(x, LENS, 12, sampling=smp, eos_token_ids=eos))
    for b in range(3):
        want = plain[b][:plain[b].index(eos) + 1] if eos in plain[b] else plain[b]
        assert cut[b] == want, b
    # launches: one batched step per token after the first, the first tokens in one extra launch over the greedy request
    L = dec.dims.num_hidden_layers
    per_step = dec._batch_kernels_per_layer * L + 4

    def launches(**kw):
        l0 = ops.LAUNCHES
        dec.generate_batch(x, LENS, kw.pop("n"), **kw)
        return ops.LAUNCHES - l0

    for n in (8, 16):
        launches(n=n), launches(n=n, sampling=smp)  # graphs captured
    s8, s16, g16 = launches(n=8, sampling=smp), launches(n=16, sampling=smp), launches(n=16)
    assert s16 - s8 == 8 * per_step
    assert s16 == g16 + 1


def _long_prompts(H, dtype, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.cat([(torch.randn(n, H, generator=g) * 0.3) for n in lens]).to(dtype).to(DEV)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_fp8_and_nf4_decoders(dtype):
    from spatialrgpt_b200.llama_decoder import LlamaDecoder
    from tests.test_gpu_beam_batch import _dims
    from tests.test_gpu_fp8 import _fp8_llama
    from tests.test_gpu_nf4_planes import _llama, _llm_state_dict
    d = _dims()
    lens = [131, 150, 129]
    x = _long_prompts(d.hidden_size, dtype, lens, 5)

    def check(dec):
        a = _lists(dec.generate_batch(x, lens, 10, sampling=SMP))
        assert _lists(dec.generate_batch(x, lens, 10, sampling=SMP, use_graph=False)) == a
        assert _lists(dec.generate_batch(x, lens, 10, sampling=SMP)) == a
        assert _lists(dec.generate_batch(x, lens, 10, sampling=dict(SMP, seed=1))) != a
        return a

    dec = LlamaDecoder(d, _fp8_llama(d, dtype), max_seq_len=512, max_seqs=2)
    assert dec.fp8
    check(dec)
    del dec
    sd = _llm_state_dict(d, 21)
    res = {}
    for copy in (True, False):
        dec = LlamaDecoder(d, _llama(d, sd, dtype, copy), max_seq_len=512, max_seqs=2)
        assert dec.nf4_planes_only == (not copy)
        res[copy] = check(dec)
        del dec
    assert res[True] == res[False]


# ---- generate() ------------------------------------------------------------------------------------------------------------------
def _model():
    from tests.golden.make_golden import CASES
    from tests.test_gpu_fp16 import build_model
    oc, sd, model = build_model(CASES["tiny_masks_gqa"][0], 3, dtype=torch.float16)
    return oc, model


def test_generate_multimodal_and_left_padded_batches():
    from oracle import srgpt_oracle as O
    from tests.golden.make_golden import CASES
    oc, model = _model()
    _, n_regions, t_text, kind, _, _ = CASES["tiny_masks_gqa"]
    reqs = [O.synth_request(oc, n_regions, t_text, seed=s, kind=kind) for s in (1234, 77)]
    h = lambda t: t.to(DEV, torch.float16)  # noqa: E731
    args = dict(images=h(torch.cat([r[1] for r in reqs])), depths=h(torch.cat([r[2] for r in reqs])), masks=[h(m) for r in reqs for m in r[3]])
    ids = torch.cat([reqs[0][0], reqs[0][0]]).to(DEV)
    kw = dict(do_sample=True, temperature=0.8, top_p=0.9, seed=4, max_new_tokens=10, eos_token_id=None)
    a = model.generate(ids, **args, **kw)
    assert a.shape == (2, 10)
    assert torch.equal(model.generate(ids, **args, **kw), a)
    assert torch.equal(model.generate(ids, **args, **kw, use_cuda_graph=False), a)
    assert not torch.equal(model.generate(ids, **args, **dict(kw, seed=5)), a)
    tok = torch.randint(3, 900, (2, 20), generator=torch.Generator().manual_seed(1)).to(DEV)
    mask = torch.ones_like(tok)
    mask[1, :6] = 0
    model.config.llama.tokenizer_padding_side = "left"
    try:
        t = model.generate(tok, attention_mask=mask, **kw)
        assert t.shape == (2, 10)
        assert torch.equal(model.generate(tok, attention_mask=mask, **kw), t)
        assert torch.equal(model.generate(tok, attention_mask=mask, use_cuda_graph=False, **kw), t)
        # row 1 is its unpadded prompt: the same rows as a batch of the unpadded prompts
        both = model.llm.generate_batch(torch.cat([model.llm.embed_tokens(tok[0]), model.llm.embed_tokens(tok[1, 6:])]), [20, 14], 10,
                                        sampling=dict(temperature=0.8, top_p=0.9, seed=4))
        assert [o.tolist() for o in both] == t.tolist()
    finally:
        model.config.llama.tokenizer_padding_side = "right"


def test_num_return_sequences():
    from spatialrgpt_b200 import ops
    oc, model = _model()
    llm = model.llm
    tok = torch.randint(3, 900, (2, 20), generator=torch.Generator().manual_seed(2)).to(DEV)
    mask = torch.ones_like(tok)
    mask[0, :5] = 0
    lens = [15, 20]
    kw = dict(do_sample=True, temperature=1.5, seed=8, max_new_tokens=12, eos_token_id=None, attention_mask=mask)
    model.config.llama.tokenizer_padding_side = "left"
    try:
        prefilled, pages = [], []
        real_prefill = llm.prefill_packed

        def spy_prefill(emb, seq_lens, **k):
            prefilled.append(list(seq_lens))
            return real_prefill(emb, seq_lens, **k)

        real_copy = ops.kv_copy_pages

        def spy_copy(p, pairs, n_staged=0):
            real_copy(p, pairs, n_staged)
            pages.append(list(pairs))

        llm.prefill_packed = spy_prefill
        ops.kv_copy_pages = spy_copy
        try:
            a = model.generate(tok, num_return_sequences=3, **kw)
        finally:
            del llm.prefill_packed
            ops.kv_copy_pages = real_copy
        assert a.shape == (6, 12)
        assert prefilled == [lens] and sum(prefilled[0]) == sum(lens)  # each prompt once
        # the siblings' prompt rows are the first row's, bit for bit
        assert len(pages) == 1
        kv = llm.cache.pages
        for g, n in enumerate(lens):
            for j in (1, 2):
                for pos in range(n):
                    s_pg, d_pg = llm.cache.owned[3 * g][pos // 16], llm.cache.owned[3 * g + j][pos // 16]
                    assert torch.equal(kv[:, d_pg, :, pos % 16].view(torch.int16), kv[:, s_pg, :, pos % 16].view(torch.int16)), (g, j, pos)
        assert torch.equal(model.generate(tok, num_return_sequences=3, **kw), a)
        assert torch.equal(model.generate(tok, num_return_sequences=3, use_cuda_graph=False, **kw), a)
        for g in range(2):  # temperature 1.5: the three answers of a prompt are not all the same
            assert len({tuple(a[3 * g + j].tolist()) for j in range(3)}) > 1, g
        # top_k = 1: every row follows the arg max of the rows it was fed, so a prompt's three rows are its greedy answer
        fed = []
        real = ops.sample_rows

        def spy(logits, params, seeds, step, off, ids):
            real(logits, params, seeds, step, off, ids)
            fed.append((logits.float().clone(), ids.clone()))

        ops.sample_rows = spy
        try:
            k1 = model.generate(tok, num_return_sequences=3, top_k=1, use_cuda_graph=False, **kw)
        finally:
            ops.sample_rows = real
        for lg, ids in fed:
            assert torch.equal(ids, torch.argmax(lg, -1))
        for g in range(2):
            assert all(torch.equal(k1[3 * g + j], k1[3 * g]) for j in (1, 2))
        one = model.generate(tok[1:], attention_mask=mask[1:], num_return_sequences=4, **{k: v for k, v in kw.items() if k != "attention_mask"})
        assert one.shape == (4, 12)
    finally:
        model.config.llama.tokenizer_padding_side = "right"
