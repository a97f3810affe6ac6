"""Per-step scores on the CPU: the return_dict_in_generate / output_scores parsing of generate() over a host-only stand-in decoder,
the output dataclasses' fields, the tensor-parallel refusal, the new entry points' exports and argument checks, compute_transition_scores
against its HF arithmetic, and BeamHypotheses' beam_indices / sequences_scores against a restatement of HF's BeamSearchScorer."""
import dataclasses
import random
import types

import pytest
import torch

from spatialrgpt_b200.llama_decoder import BeamHypotheses
from spatialrgpt_b200.llava_llama import GenerateBeamDecoderOnlyOutput, GenerateDecoderOnlyOutput, compute_transition_scores

V = 11
BAD = -1


class HostDecoder:
    """A stand-in decoder on the host: returns fixed ids and score rows, and records the keyword arguments it was called with."""
    supports_prompt_lookup = supports_logits_processors = supports_prefix_reuse = supports_batch_sampling = True
    supports_output_scores = True
    dims = types.SimpleNamespace(vocab_size=V)

    def __init__(self):
        self.calls = []

    def embed_tokens(self, ids):
        return torch.zeros(ids.numel(), 4)

    def _extra(self, steps, rows):
        return {"scores": torch.arange(steps * rows * V, dtype=torch.float32).view(steps, rows, V)}

    def generate_from_embeds(self, emb, n, **kw):
        self.calls.append(("one", kw))
        ids = torch.arange(n, dtype=torch.int64)
        r = (ids, torch.zeros(n, V)) if kw.get("return_logits") else ids
        return (r, self._extra(n, 1)) if kw.get("output_scores") else r

    def generate_batch(self, packed, lens, n, **kw):
        self.calls.append(("batch", kw))
        outs = [torch.arange(n - b, dtype=torch.int64) for b in range(len(lens))]
        r = (outs, [torch.zeros(o.numel(), V) for o in outs]) if kw.get("return_logits") else outs
        return (r, self._extra(n, len(lens))) if kw.get("output_scores") else r

    def generate_beam(self, emb, k, n, **kw):
        self.calls.append(("beam", kw))
        ids = torch.tensor([3, 4, 5])
        if not kw.get("output_scores"):
            return ids
        return ids, dict(self._extra(3, k), sequence_scores=[-1.5], beam_indices=[[0, 2, 1]])

    def generate_beam_batch(self, packed, lens, k, n, **kw):
        self.calls.append(("beam_batch", kw))
        outs = [torch.tensor([3, 4, 5]), torch.tensor([6, 7])]
        if not kw.get("output_scores"):
            return outs
        return outs, dict(self._extra(3, 2 * k), sequence_scores=[-1.5, -0.25], beam_indices=[[0, 2, 1], [3, 4]])


def _model(dec=None):
    from spatialrgpt_b200.llava_llama import LlavaLlamaModel
    gen = getattr(getattr(LlavaLlamaModel.generate, "__wrapped__", None), "__wrapped__", None)
    if gen is None or hasattr(gen, "__wrapped__"):
        pytest.skip("generate is not unwrappable here")

    class M(LlavaLlamaModel):
        device = torch.device("cpu")

    m = M.__new__(M)
    m.config = types.SimpleNamespace(llama=types.SimpleNamespace(eos_token_id=None, vocab_size=V, pad_token_id=0))
    m.llm = HostDecoder() if dec is None else dec
    return gen, m


def test_dataclass_fields_carry_hf_names():
    assert [f.name for f in dataclasses.fields(GenerateDecoderOnlyOutput)][:3] == ["sequences", "scores", "logits"]
    beam = [f.name for f in dataclasses.fields(GenerateBeamDecoderOnlyOutput)]
    assert beam[:5] == ["sequences", "sequences_scores", "scores", "logits", "beam_indices"]


def test_without_the_dict_generate_returns_what_it_returned_and_ignores_output_scores():
    gen, m = _model()
    one, two = torch.tensor([[5, 6, 7]]), torch.tensor([[5, 6, 7], [1, 2, 3]])
    for kw in ({}, dict(output_scores=True), dict(return_dict_in_generate=False, output_scores=True)):
        out = gen(m, one, max_new_tokens=4, **kw)
        assert isinstance(out, torch.Tensor) and out.tolist() == [[0, 1, 2, 3]]
        out = gen(m, two, max_new_tokens=4, **kw)
        assert isinstance(out, torch.Tensor) and out.tolist() == [[0, 1, 2, 3], [0, 1, 2, 0]]
        out = gen(m, one, max_new_tokens=2, num_beams=3, **kw)
        assert isinstance(out, torch.Tensor) and out.tolist() == [[3, 4, 5]]
    seqs, logits = gen(m, one, max_new_tokens=4, output_logits=True, output_scores=True)
    assert seqs.tolist() == [[0, 1, 2, 3]] and logits[0].shape == (4, V)
    assert all("output_scores" not in kw for _, kw in m.llm.calls)


def test_the_dict_holds_sequences_scores_and_logits():
    gen, m = _model()
    one, two = torch.tensor([[5, 6, 7]]), torch.tensor([[5, 6, 7], [1, 2, 3]])
    out = gen(m, one, max_new_tokens=4, return_dict_in_generate=True)
    assert isinstance(out, GenerateDecoderOnlyOutput) and out.sequences.tolist() == [[0, 1, 2, 3]] and out.scores is None
    out = gen(m, one, max_new_tokens=4, return_dict_in_generate=True, output_scores=True)
    assert len(out.scores) == 4 and all(s.shape == (1, V) and s.dtype == torch.float32 for s in out.scores)
    assert m.llm.calls[-1][1]["output_scores"] is True
    out = gen(m, two, max_new_tokens=4, return_dict_in_generate=True, output_scores=True, output_logits=True)
    assert out.sequences.tolist() == [[0, 1, 2, 3], [0, 1, 2, 0]] and len(out.scores) == 4 and out.scores[0].shape == (2, V)
    assert [lg.shape for lg in out.logits] == [(4, V), (3, V)]
    out = gen(m, one, max_new_tokens=3, num_beams=3, return_dict_in_generate=True)
    assert isinstance(out, GenerateBeamDecoderOnlyOutput) and out.sequences_scores is None and out.beam_indices is None
    out = gen(m, one, max_new_tokens=3, num_beams=3, return_dict_in_generate=True, output_scores=True)
    assert out.beam_indices.tolist() == [[0, 2, 1]] and out.sequences_scores.tolist() == [-1.5] and out.scores[0].shape == (3, V)
    out = gen(m, two, max_new_tokens=3, num_beams=3, return_dict_in_generate=True, output_scores=True)
    assert out.sequences.tolist() == [[3, 4, 5], [6, 7, 0]] and out.beam_indices.tolist() == [[0, 2, 1], [3, 4, -1]]
    assert out.sequences_scores.tolist() == [-1.5, -0.25] and len(out.scores) == 3 and out.scores[0].shape == (6, V)


def test_tensor_parallel_decoder_refuses_output_scores():
    from spatialrgpt_b200.tensor_parallel import TPLlamaDecoder
    assert TPLlamaDecoder.supports_output_scores is False
    dec = HostDecoder()
    dec.supports_output_scores = False
    gen, m = _model(dec)
    with pytest.raises(NotImplementedError, match="tensor-parallel"):
        gen(m, torch.tensor([[5, 6, 7]]), max_new_tokens=4, return_dict_in_generate=True, output_scores=True)
    assert dec.calls == []
    out = gen(m, torch.tensor([[5, 6, 7]]), max_new_tokens=4, return_dict_in_generate=True)  # no scores asked: served
    assert out.scores is None


@pytest.mark.parametrize("elem", ["bf16", "f16"])
def test_entry_points_export_and_check_arguments(elem):
    from spatialrgpt_b200 import _lib
    lib = _lib.load(elem=elem)
    x = 16  # a non-NULL address: every call below fails its argument check before any launch
    ok = [x, 1, 128, 3, 100, x, 0, x, 300, 100, None]
    for i, v in ((0, None), (5, None), (7, None), (1, 2), (2, 99), (3, 0), (3, 65536), (4, 0), (9, 99), (8, -1)):
        args = list(ok)
        args[i] = v
        assert lib.srgpt_step_scores(*args) == BAD, (i, v)
    ok = [x, 1, 128, 3, 100, x, x, x, 0, x, x, 300, None]
    for i, v in ((10, None), (11, 299), (0, None), (3, 0)):
        args = list(ok)
        args[i] = v
        assert lib.srgpt_sample_rows_scores(*args) == BAD, (i, v)
    ok = [x, 100, x, x, x, -1, x, None, None, 0, x, 100, None]
    for i, v in ((10, None), (11, 99), (0, None)):
        args = list(ok)
        args[i] = v
        assert lib.srgpt_sample_top_p_scores_f32(*args) == BAD, (i, v)
    ok = [x, 128, 3, 100, x, 6, x, x, x, 100, None]
    for i, v in ((9, 99), (0, None), (5, 101)):
        args = list(ok)
        args[i] = v
        assert lib.srgpt_beam_candidates_scores_bf16(*args) == BAD, (i, v)


def hf_compute_transition_scores(sequences, scores, beam_indices, normalize_logits):
    """transformers' GenerationMixin.compute_transition_scores, when this image has it."""
    transformers = pytest.importorskip("transformers")
    from transformers.generation.utils import GenerationMixin
    cfg = types.SimpleNamespace(vocab_size=scores[0].shape[-1])
    cfg.get_text_config = lambda **_: cfg
    model = types.SimpleNamespace(config=cfg)
    try:
        return GenerationMixin.compute_transition_scores(model, sequences, scores, beam_indices, normalize_logits)
    except AttributeError as e:  # a newer transformers reads more of the model than this stand-in has
        pytest.skip(f"transformers {transformers.__version__}: {e}")


@pytest.mark.parametrize("normalize", [False, True])
def test_compute_transition_scores_gathers_the_chosen_tokens(normalize):
    g = torch.Generator().manual_seed(3)
    T, R = 5, 4
    scores = tuple(torch.randn(R, V, generator=g) for _ in range(T))
    seqs = torch.randint(0, V, (R, T), generator=g)
    out = compute_transition_scores(seqs, scores, normalize_logits=normalize)
    for r in range(R):
        for t in range(T):
            row = torch.log_softmax(scores[t][r], -1) if normalize else scores[t][r]
            assert torch.allclose(out[r, t], row[seqs[r, t]], rtol=1e-6, atol=1e-6)
    # beams: step t's row is beam_indices[b, t]; -1 pads give 0; the tokens are the last (longest beam) columns of the sequences
    bi = torch.tensor([[0, 2, 1, 3, -1], [1, 1, 0, -1, -1]])
    bseq = torch.randint(0, V, (2, 5), generator=g)
    out = compute_transition_scores(bseq, scores, bi, normalize_logits=normalize)
    assert out.shape == (2, 4)
    for b in range(2):
        for t in range(4):
            tok = bseq[b, 1 + t]
            want = 0.0 if bi[b, t] < 0 else (torch.log_softmax(scores[t][bi[b, t]], -1) if normalize else scores[t][bi[b, t]])[tok]
            assert torch.allclose(out[b, t], torch.as_tensor(want), rtol=1e-6, atol=1e-6)
    ref = hf_compute_transition_scores(bseq, scores, bi, normalize)
    assert torch.equal(out, ref)


# ---- beam_indices / sequences_scores against a restatement of HF 4.37's BeamSearchScorer (process + finalize, beam_indices on) ---------
def hf_beam_search(step_logprobs, B, k, eos, lp, es, max_len):
    """HF's beam_search loop over given per-step log-probabilities [steps][B * k][V] with BeamSearchScorer's bookkeeping."""
    beam_scores = [0.0 if i % k == 0 else -1e9 for i in range(B * k)]
    seqs = [[] for _ in range(B * k)]
    bidx = [[] for _ in range(B * k)]
    hyps = [[] for _ in range(B)]
    done = [False] * B

    def add(g, score, toks, idx, L):
        sc = score / (L ** lp)
        h = hyps[g]
        if len(h) < k or sc > min(x[0] for x in h):
            h.append((sc, toks, idx))
            if len(h) > k:
                h.sort(key=lambda x: x[0])
                del h[0]

    for step, lpr in enumerate(step_logprobs):
        cur = step + 1
        new_scores, new_seqs, new_idx = [], [], []
        for g in range(B):
            flat = sorted(((-(lpr[g * k + i][t] + beam_scores[g * k + i]), i, t) for i in range(k) for t in range(V)))[:2 * k]
            if done[g]:
                new_scores += [0.0] * k
                new_seqs += [seqs[g * k + i] + [0] for i in range(k)]
                new_idx += [bidx[g * k + i] + [g * k + i] for i in range(k)]
                continue
            nxt = []
            for rank, (neg, i, t) in enumerate(flat):
                row = g * k + i
                if t in eos:
                    if rank >= k:
                        continue
                    add(g, -neg, list(seqs[row]), bidx[row] + [row], cur)
                else:
                    nxt.append((-neg, row, t))
                if len(nxt) == k:
                    break
            best = -flat[0][0]
            if len(hyps[g]) >= k and (es or min(x[0] for x in hyps[g]) >= best / (cur ** lp)):
                done[g] = True
            new_scores += [s for s, _, _ in nxt]
            new_seqs += [seqs[row] + [t] for _, row, t in nxt]
            new_idx += [bidx[row] + [row] for _, row, _ in nxt]
        beam_scores, seqs, bidx = new_scores, new_seqs, new_idx
        if all(done) or cur == max_len:
            break
    out = []
    for g in range(B):
        if not done[g]:
            for i in range(k):
                add(g, beam_scores[g * k + i], list(seqs[g * k + i]), list(bidx[g * k + i]), len(seqs[g * k + i]))
        sc, toks, idx = sorted(hyps[g], key=lambda x: x[0])[-1]
        out.append((toks + ([eos[0]] if len(toks) < max_len and eos else []), sc, idx))
    return out


@pytest.mark.parametrize("seed", range(12))
def test_beam_indices_and_sequences_scores_match_hf_bookkeeping(seed):
    rnd = random.Random(seed)
    B, k, max_len = rnd.choice([1, 2, 3]), rnd.choice([2, 3]), rnd.choice([3, 6])
    eos = [rnd.randrange(V)] if seed % 3 else []
    lp, es = rnd.choice([1.0, 0.7, 1.3]), bool(seed % 2)
    g = torch.Generator().manual_seed(seed)
    steps = [torch.log_softmax(torch.randn(B * k, V, generator=g) * 2, -1).tolist() for _ in range(max_len)]
    ref = hf_beam_search(steps, B, k, eos, lp, es, max_len)
    groups = [BeamHypotheses(k, eos, lp, es, row0=gi * k) for gi in range(B)]
    for step in range(max_len):
        for gi, grp in enumerate(groups):
            if grp.done:
                continue
            cand = sorted(((-(steps[step][gi * k + i][t] + grp.scores[i]), i, t) for i in range(k) for t in range(V)))
            grp.advance([(-neg, i, t) for neg, i, t in cand[:max(2, 1 + len(eos)) * k]], step + 1)
        if all(grp.done for grp in groups):
            break
    for gi, grp in enumerate(groups):
        toks = grp.best(max_len)
        assert toks == ref[gi][0], (gi, toks, ref[gi])
        assert grp.best_beams == ref[gi][2], (gi, grp.best_beams, ref[gi][2])
        assert grp.best_score == pytest.approx(ref[gi][1], rel=1e-12, abs=1e-12)
