"""Llama decoder on the sm_90a kernels: prefill (wgmma GEMMs + flash attention), paged KV cache,
and a CUDA-graph-captured decode step made of weight-streaming GEMV kernels.

Reference: llava/train/transformers_replace/models/llama/modeling_llama.py — LlamaModel.forward
(824-936), LlamaDecoderLayer (611-684), LlamaFlashAttention2 (405-566), LlamaMLP (194-223),
LlamaRMSNorm (61-75), rotary embedding (81-130, 160-191), lm_head + float() (1044-1045),
prepare_inputs_for_generation (1112-1149); greedy loop = HF GenerationMixin (llava_llama.py:212).
The reference re-allocates the KV cache with torch.cat every step (451-456) and launches ~25
torch kernels per layer per token; here one token is 5 kernels per layer replayed from a CUDA graph
with the position / step counters living in device memory.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import List, NamedTuple, Optional

import torch

from . import logits_processors, ops
from .config import LlamaDims
from .weights import LlamaW

PAGE_SIZE = 16


def build_rope_tables(dims: LlamaDims, max_pos: int, device, dtype: torch.dtype = torch.bfloat16) -> (torch.Tensor, torch.Tensor):
    """cos/sin exactly as LlamaRotaryEmbedding.forward computes them (modeling_llama.py:86,117-130):
    fp32 inv_freq, fp32 outer product, cos/sin in fp32, cast to the model dtype.  Host-side table build (once)."""
    hd = dims.head_dim
    inv_freq = 1.0 / (dims.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64).float() / hd))
    t = torch.arange(max_pos, dtype=torch.int64).float()
    if getattr(dims, "rope_scaling_factor", 1.0) != 1.0:  # LlamaLinearScalingRotaryEmbedding.forward (modeling_llama.py:136-140)
        t = t / float(dims.rope_scaling_factor)
    freqs = t[:, None] * inv_freq[None, :]
    return freqs.cos().to(dtype).to(device).contiguous(), freqs.sin().to(dtype).to(device).contiguous()


def eos_list(eos_token_ids) -> List[int]:
    """eos_token_ids as generate() takes it (None, one id or several) -> the ids in the given order (beam search appends the first)."""
    if eos_token_ids is None:
        return []
    return [int(e) for e in (eos_token_ids if isinstance(eos_token_ids, (list, tuple, set)) else [eos_token_ids])]


def first_stop(host_ids, lo: int, hi: int, eos, stopping_fn, limit: int) -> Optional[int]:
    """Where a request ends among the generated tokens [lo, hi) already on the host: k + 1 for the first k whose id is in `eos` or for
    which ``stopping_fn(host_ids[:k + 1])`` fires, else `limit` (the token budget) when the window reaches it, else None."""
    for k in range(lo, min(hi, limit)):
        if int(host_ids[k]) in eos or (stopping_fn is not None and stopping_fn(host_ids[:k + 1])):
            return k + 1
    return limit if hi >= limit else None


def decode_steps(launch, fetch, host, budgets: List[int], eos, stopping_fn) -> List[int]:
    """The decode steps of B rows whose token 0 is already generated; returns each row's length.  ``launch(n)`` enqueues the step
    that produces token n of every row; ``fetch(n)`` enqueues the copy of id row n into ``host`` ([T, B], T = max(budgets)) and
    returns what to ``.synchronize()`` on.  With EOS ids or a criterion, step n is enqueued BEFORE row n - 1 is inspected, so the host
    inspects while exactly one step runs, and no host round trip per token stalls the device (HF inspects after every token too, with
    a blocking .item(); the result is the same).  Without either, the steps run back to back with no copy.  A row that has stopped
    stays in the step and its later ids are ignored; the loop ends when every row has stopped or T - 1 steps have run.  A row's
    length is its first stop (first_stop), else its budget: once the budget is spent the last token is returned whatever it is."""
    T = max(budgets)
    if not eos and stopping_fn is None:
        for n in range(1, T):
            launch(n)
        return list(budgets)
    cols = host.unbind(1)
    stops = [None] * len(budgets)
    copied = fetch(0)
    n = 1
    while n < T:
        launch(n)
        nxt = fetch(n)
        copied.synchronize()
        for b, m in enumerate(budgets):
            if stops[b] is None:
                stops[b] = first_stop(cols[b], n - 1, n, eos, stopping_fn, m)
        if None not in stops:
            break
        copied = nxt
        n += 1
    return [m if s is None else s for s, m in zip(stops, budgets)]


class GraphKey(NamedTuple):
    """What a captured graph computes: its kind ("step", "batch", "rows", "beam", "verify" or "contrastive"), its rows (T for a verify
    pass), whether it samples, whether the logits processors run, the (address, step stride) of the score rows it writes (output_scores),
    the n-gram size of a verify pass, the candidates per prompt of a contrastive step (B * k rows), the addresses and layout of the
    hidden states / attentions it records (ops.StepProbe.key; generate(output_hidden_states=, output_attentions=)), and whether its draw
    runs the typical / epsilon / eta warpers (the warped sampler over LlamaDecoder.warp_params)."""
    kind: str
    rows: int = 1
    sample: bool = False
    proc: bool = False
    scores: Optional[tuple] = None
    ngram: int = 0
    group: int = 0
    probe: Optional[tuple] = None
    warp: bool = False


def sampling_warpers(sampling) -> tuple:
    """(typical_p, epsilon_cutoff, eta_cutoff) of a sampling dict, each at its neutral value (1, 0, 0) when absent or when HF leaves the
    warper off: typical_p >= 1, a cutoff outside (0, 1) (transformers 5.5 _get_logits_processor; NaN included).  Raises ValueError where
    HF's TypicalLogitsWarper does: typical_p <= 0."""
    typ, eps, eta = (sampling.get(k) for k in ("typical_p", "epsilon_cutoff", "eta_cutoff"))
    typ = 1.0 if typ is None else float(typ)
    eps = 0.0 if eps is None else float(eps)
    eta = 0.0 if eta is None else float(eta)
    if typ < 1.0 and not typ > 0.0:
        raise ValueError(f"`typical_p` has to be a float > 0 and < 1, but is {typ}")
    return (typ if typ < 1.0 else 1.0, eps if 0.0 < eps < 1.0 else 0.0, eta if 0.0 < eta < 1.0 else 0.0)


class BeamHypotheses:
    """The host bookkeeping of one prompt's beam search (HF BeamSearchScorer.process / finalize for one batch entry): the running beams'
    tokens and scores, the kept hypotheses and the done flag.  ``advance`` takes the prompt's ranked candidates of one step.
    It also records the beam row every token was chosen from (HF's beam_indices: row0 + the beam, row0 being the prompt's first row of
    the step), and ``best`` leaves the chosen hypothesis' score and rows in ``best_score`` / ``best_beams``."""

    def __init__(self, k: int, eos, length_penalty: float, early_stopping: bool, row0: int = 0):
        self.k, self.eos, self.length_penalty, self.early_stopping, self.row0 = k, eos, length_penalty, early_stopping, row0
        self.seqs: List[List[int]] = [[] for _ in range(k)]
        self.beams: List[List[int]] = [[] for _ in range(k)]  # the row of every token of each running beam
        self.scores = [0.0] + [-1e9] * (k - 1)
        self.hyps: List = []  # (score, tokens) of finished hypotheses, at most k kept
        self.hyp_beams: List[List[int]] = []  # the rows of each kept hypothesis, in the order of hyps
        self.worst, self.done = 1e9, False
        self.best_score, self.best_beams = None, None

    def keep(self, score: float, toks: List[int], beams: Optional[List[int]] = None) -> None:
        if len(self.hyps) < self.k or score > self.worst:
            self.hyps.append((score, toks))
            self.hyp_beams.append([] if beams is None else beams)
            if len(self.hyps) > self.k:
                i = min(range(len(self.hyps)), key=lambda j: self.hyps[j][0])
                del self.hyps[i], self.hyp_beams[i]
            self.worst = min(x[0] for x in self.hyps)

    def advance(self, ranked, cur_len: int) -> List[int]:
        """ranked: (score, beam, token) in (score desc, beam asc, token asc) order, at most 2k (or (1 + #EOS) k) of them.  An EOS of rank
        < k closes a hypothesis; the other candidates become the next beams.  Returns each next beam's parent beam."""
        nxt = []
        for rank, (sc, b, t) in enumerate(ranked):
            if t in self.eos:
                if rank >= self.k:
                    continue
                self.keep(sc / (cur_len ** self.length_penalty), list(self.seqs[b]), self.beams[b] + [self.row0 + b])
            else:
                nxt.append((sc, b, t))
            if len(nxt) == self.k:
                break
        if len(nxt) < self.k:
            raise RuntimeError("beam search ran out of non-EOS candidates")  # HF asserts the same
        if len(self.hyps) >= self.k and (self.early_stopping or self.worst >= ranked[0][0] / (cur_len ** self.length_penalty)):
            self.done = True
        self.seqs = [self.seqs[b] + [t] for _, b, t in nxt]
        self.beams = [self.beams[b] + [self.row0 + b] for _, b, _ in nxt]
        self.scores = [sc for sc, _, _ in nxt]
        return [b for _, b, _ in nxt]

    def close(self) -> None:
        """finalize (beam_search.py): unless done, the running beams become hypotheses over their generated length."""
        if not self.done:
            for i in range(self.k):
                self.keep(self.scores[i] / (len(self.seqs[i]) ** self.length_penalty), list(self.seqs[i]), list(self.beams[i]))

    def best(self, max_new_tokens: int) -> List[int]:
        """finalize (beam_search.py): close, then the best hypothesis, with the first EOS appended when it is shorter than max_new_tokens."""
        self.close()
        i = max(range(len(self.hyps)), key=lambda j: self.hyps[j][0])
        self.best_score, self.best_beams = self.hyps[i][0], list(self.hyp_beams[i])
        best = list(self.hyps[i][1])
        if len(best) < max_new_tokens and self.eos:
            best.append(self.eos[0])
        return best


def group_best(groups: List[BeamHypotheses], max_new_tokens: int) -> List[int]:
    """The answer of one prompt of diverse beam search (BeamSearchScorer.finalize with num_beam_groups, transformers 4.37.2): every group
    closes, and of all groups' hypotheses, in group order, a stable sort by score and pop() take the last best one (a tie goes to the
    later group); the first EOS is appended when it is shorter than max_new_tokens."""
    for grp in groups:
        grp.close()
    best = list(sorted((h for grp in groups for h in grp.hyps), key=lambda h: h[0])[-1][1])
    eos = groups[0].eos
    if len(best) < max_new_tokens and eos:
        best.append(eos[0])
    return best


def beam_page_pairs(tables: List[List[int]], parents: List[int], starts: List[int], n_gen: int, page_size: int = PAGE_SIZE):
    """The KV copies that make every moved row (parents[r] != r) hold its parent's generated rows: positions [starts[r], starts[r] + n_gen)
    of each, page by page, as (src page, dst page, first row, rows) over the page tables ``tables``.  Returns (pairs, n_staged): a pair
    whose destination row is itself some row's parent is listed first and staged (kv_copy_pages), so cycles and chains are safe."""
    sources = {p for r, p in enumerate(parents) if p != r}
    staged, direct = [], []
    for r, p in enumerate(parents):
        if p == r or n_gen <= 0:
            continue
        s0, s1 = starts[r], starts[r] + n_gen
        for j in range(s0 // page_size, (s1 - 1) // page_size + 1):
            lo, hi = max(s0, j * page_size) - j * page_size, min(s1, (j + 1) * page_size) - j * page_size
            (staged if r in sources else direct).append((tables[p][j], tables[r][j], lo, hi - lo))
    return staged + direct, len(staged)


def prompt_page_pairs(tables: List[List[int]], seq_lens: List[int], n: int, page_size: int = PAGE_SIZE):
    """The KV copies that give rows g * n + 1 .. g * n + n - 1 the prompt rows [0, seq_lens[g]) of row g * n, which the prefill wrote:
    (src page, dst page, first row, rows) over the page tables ``tables``, page by page.  No destination is a source, so none is staged."""
    return [(tables[g * n][j], tables[g * n + i][j], 0, min(page_size, seq_lens[g] - j * page_size))
            for g in range(len(seq_lens)) for i in range(1, n) for j in range((seq_lens[g] + page_size - 1) // page_size)]


def candidate_pages(S: int, n_rows: int, page_size: int = PAGE_SIZE):
    """A candidate that continues a prompt of S rows with n_rows >= 1 rows (positions [S, S + n_rows)): (shared, own) page counts.  Its
    first S // page_size pages are the prompt's full pages, shared; it owns the pages from the prompt's partial last page (a copy) or
    the first page past the prompt, up to the page of its last row."""
    shared = S // page_size
    return shared, (S + n_rows + page_size - 1) // page_size - shared


def plan_score_passes(seq_lens: List[int], cand_lens: List[int], row_budget: int, free_pages: int, max_chunks: int = 65535,
                      page_size: int = PAGE_SIZE):
    """The passes of LlamaDecoder.score_candidates.  Candidate c of prompt b needs cand_lens[c] - 1 rows (its tokens but the last, at
    positions S_b ..), so a one-token candidate needs none and is in no pass.  Returns a list of passes, each a list of (b, c, first row,
    rows, own pages) in (b, c) order, filled greedily: a pass holds at most ``row_budget`` rows, ``free_pages`` owned pages (the pages
    left after the prompts') and ``max_chunks`` candidates.  Raises when one candidate alone does not fit."""
    passes, cur, rows, pages = [], [], 0, 0
    for b, S in enumerate(seq_lens):
        for c, L in enumerate(cand_lens):
            n = int(L) - 1
            if n < 1:
                continue
            shared, own = candidate_pages(int(S), n, page_size)
            # the rows [S, S + n) land in table entries shared .. shared + own - 1, never in one of the prompt's full (shared) pages
            first, last = int(S) // page_size, (int(S) + n - 1) // page_size
            assert shared <= first and last < shared + own, "a candidate's K/V would land in a shared page"
            if n > row_budget or own > free_pages:
                raise RuntimeError(f"candidate {c} of prompt {b} needs {n} rows and {own} KV pages; a pass has {row_budget} rows and "
                                   f"{free_pages} free pages")
            if cur and (rows + n > row_budget or pages + own > free_pages or len(cur) >= max_chunks):
                passes.append(cur)
                cur, rows, pages = [], 0, 0
            cur.append((b, c, rows, n, own))
            rows += n
            pages += own
    if cur:
        passes.append(cur)
    return passes


SEED_STRIDE = 0x9E3779B97F4A7C15  # the golden-ratio increment of splitmix64
SEED_MASK = 0x7FFFFFFFFFFFFFFF


def sequence_seeds(seed: int, n: int) -> List[int]:
    """The sampling seeds of the n sequences of a sampled batch: sequence b's seed is sequence b - 1's plus SEED_STRIDE * (b + 1) (sequence
    -1's is ``seed``), mod 2^63, i.e. seed + SEED_STRIDE * (b + 1) (b + 2) / 2.  The batched and the one-after-the-other paths both use it,
    so a sequence draws with the same seed on either."""
    out, s = [], int(seed) & SEED_MASK
    for b in range(n):
        s = (s + SEED_STRIDE * (b + 1)) & SEED_MASK
        out.append(s)
    return out


class PagedKVCache:
    """KV pages for all layers: [layers, n_pages, 2 (k,v), PAGE_SIZE, n_kv_heads, head_dim] bf16, a free list
    and per-sequence page tables (int32, device) of fixed capacity so decode graphs stay valid."""

    def __init__(self, dims: LlamaDims, n_pages: int, max_seqs: int, max_pages_per_seq: int, device, dtype: torch.dtype = torch.bfloat16):
        self.dims = dims
        self.n_pages = n_pages
        self.max_pages_per_seq = max_pages_per_seq
        self.pages = torch.zeros((dims.num_hidden_layers, n_pages, 2, PAGE_SIZE, dims.num_key_value_heads, dims.head_dim),
                                 dtype=dtype, device=device)
        # +1 spare column (a measured-and-dropped decode-attention variant read the page id of row pos+1; kept so tables stay 16-byte padded)
        self.page_tables = torch.zeros((max_seqs, max_pages_per_seq + 1), dtype=torch.int32, device=device)
        self.free: List[int] = list(range(n_pages - 1, -1, -1))
        self.owned: List[List[int]] = [[] for _ in range(max_seqs)]
        # forked sequences (fork): id -> (source sequence, shared pages, owned pages); lent: source sequence -> number of live forks.
        # Fork ids start past every slot, so they never name a slot of `owned`.
        self.forks = {}
        self.lent = {}
        self._next_fork = max_seqs

    def reserve(self, seq: int, n_tokens: int) -> None:
        """Make sure sequence `seq` owns pages for positions [0, n_tokens)."""
        need = (n_tokens + PAGE_SIZE - 1) // PAGE_SIZE
        if need > self.max_pages_per_seq:
            raise RuntimeError(f"sequence needs {need} KV pages > capacity {self.max_pages_per_seq}")
        own = self.owned[seq]
        if need > len(own):
            add = need - len(own)
            if add > len(self.free):
                raise RuntimeError("KV cache exhausted")
            new = [self.free.pop() for _ in range(add)]
            start = len(own)
            own.extend(new)
            self.page_tables[seq, start:start + add] = torch.tensor(new, dtype=torch.int32)

    def reserve_many(self, n_tokens: List[int]) -> None:
        """reserve() for sequences 0..len-1 with ONE host->device copy of the page tables (a 32-request batch otherwise issues
        32 tiny copies between the encoders and the prefill)."""
        host = torch.zeros((len(n_tokens), self.page_tables.shape[1]), dtype=torch.int32)
        for seq, n in enumerate(n_tokens):
            need = (n + PAGE_SIZE - 1) // PAGE_SIZE
            if need > self.max_pages_per_seq:
                raise RuntimeError(f"sequence needs {need} KV pages > capacity {self.max_pages_per_seq}")
            own = self.owned[seq]
            if need > len(own):
                if need - len(own) > len(self.free):
                    raise RuntimeError("KV cache exhausted")
                own.extend(self.free.pop() for _ in range(need - len(own)))
            host[seq, :len(own)] = torch.tensor(own, dtype=torch.int32)
        self.page_tables[:len(n_tokens)].copy_(host, non_blocking=True)

    def release(self, seq: int) -> None:
        """Return the pages sequence `seq` owns to the free list (a fork's shared pages stay with their owner)."""
        if seq in self.forks:
            src, _, own = self.forks.pop(seq)
            self.free.extend(reversed(own))
            self.lent[src] -= 1
            return
        if self.lent.get(seq, 0):
            raise RuntimeError(f"sequence {seq} still lends its pages to {self.lent[seq]} forked sequences")
        self.free.extend(reversed(self.owned[seq]))
        self.owned[seq] = []

    def release_all(self, keep: Optional[int] = None) -> None:
        """release() every slot but `keep`: a request starts from an empty cache (a batch leaves pages owned by slots 1..B-1)."""
        for seq in range(len(self.owned)):
            if seq != keep:
                self.release(seq)

    def fork(self, src: int, shared_pages: int, n_tokens: int) -> int:
        """A host-side sequence whose first `shared_pages` pages ARE sequence `src`'s (shared, never written or freed by the fork) and
        which owns new pages for the rest of positions [0, n_tokens).  Returns its id (``table`` gives its page table; the caller builds
        device tables from it).  ``release`` frees only the pages it owns; `src` cannot be released while forks share its pages."""
        if not 0 <= shared_pages <= len(self.owned[src]):
            raise RuntimeError(f"sequence {src} has {len(self.owned[src])} pages, cannot share {shared_pages}")
        need = (n_tokens + PAGE_SIZE - 1) // PAGE_SIZE
        if need > self.max_pages_per_seq:
            raise RuntimeError(f"sequence needs {need} KV pages > capacity {self.max_pages_per_seq}")
        add = max(0, need - shared_pages)
        if add > len(self.free):
            raise RuntimeError("KV cache exhausted")
        fid = self._next_fork
        self._next_fork += 1
        self.forks[fid] = (src, list(self.owned[src][:shared_pages]), [self.free.pop() for _ in range(add)])
        self.lent[src] = self.lent.get(src, 0) + 1
        return fid

    def table(self, seq: int) -> List[int]:
        """Page ids of sequence `seq` by position // PAGE_SIZE (shared pages first for a fork)."""
        if seq in self.forks:
            _, shared, own = self.forks[seq]
            return shared + own
        return list(self.owned[seq])

    def layer(self, l: int) -> torch.Tensor:
        return self.pages[l]


@dataclass
class PrefillProbe:
    """What a probed prefill records (ops.llama_prefill_layers_probe): ``hidden`` [n_layers, B, R, H] receives the rows each layer reads,
    ``attn`` [n_layers, B, n_heads, R, R] each layer's attention probabilities (either may be None); prompt b's rows start at output row
    ``row_off[b]`` (device int32 [B])."""
    row_off: torch.Tensor
    hidden: Optional[torch.Tensor] = None
    attn: Optional[torch.Tensor] = None


@dataclass
class GenerateProbe:
    """What generate(output_hidden_states=, output_attentions=) records: ``prefill`` the prompt step (PrefillProbe over [B, T] padded rows),
    ``final`` [B, T, H] the final norm of the prompt rows (None without hidden states), ``offs`` each prompt's first padded row, and
    ``steps`` the decode steps (ops.StepProbe; None when there are none)."""
    prefill: PrefillProbe
    final: Optional[torch.Tensor]
    offs: List[int]
    steps: Optional[ops.StepProbe]

    def record_final(self, llm: "LlamaDecoder", hidden: torch.Tensor, seq_lens: List[int]) -> None:
        """final[b] at prompt b's rows: the final norm of the prefill's packed residual rows ``hidden`` (forward()'s hidden_states[L])."""
        if self.final is None:
            return
        hn, o = llm.final_norm(hidden), 0
        for b, n in enumerate(seq_lens):
            self.final[b, self.offs[b]:self.offs[b] + n] = hn[o:o + n]
            o += n


class LlamaDecoder:
    def __init__(self, dims: LlamaDims, w: LlamaW, max_seq_len: int = 4096, max_new_tokens_cap: int = 4096, max_seqs: int = 1,
                 kv_pages: Optional[int] = None):
        self.dims = dims
        self.w = w
        dev = w.embed.device
        self.device = dev
        self.max_seq_len = max_seq_len
        self.dtype = w.embed.dtype  # torch.bfloat16 or torch.float16: selects the build of the kernels (ops.elem_dtype)
        self.cos, self.sin = build_rope_tables(dims, max_seq_len, dev, self.dtype)
        ppseq = (max_seq_len + PAGE_SIZE - 1) // PAGE_SIZE
        self.cache = PagedKVCache(dims, kv_pages if kv_pages is not None else ppseq * max_seqs, max_seqs, ppseq, dev, self.dtype)
        # the decode graph reads the page table of the sequence being decoded from this fixed buffer
        self.active_pt = torch.zeros(ppseq + 1, dtype=torch.int32, device=dev)
        H, nh, hd, I = dims.hidden_size, dims.num_attention_heads, dims.head_dim, dims.intermediate_size
        # decode-step state (static addresses -> graph-capturable)
        self.pos = torch.zeros(1, dtype=torch.int32, device=dev)       # position of the token being processed
        self.step = torch.zeros(1, dtype=torch.int32, device=dev)      # number of generated tokens so far
        self.out_ids = torch.zeros(max_new_tokens_cap, dtype=torch.int64, device=dev)
        self.h = torch.zeros(H, dtype=self.dtype, device=dev)      # residual stream of the current token
        self.q_buf = torch.zeros(nh * hd, dtype=self.dtype, device=dev)
        self.attn_buf = torch.zeros(nh * hd, dtype=self.dtype, device=dev)
        self.act_buf = torch.zeros(I, dtype=self.dtype, device=dev)
        self.lm_ws = ops.lm_head_workspace(dims.vocab_size, dev)
        self.scale = hd ** -0.5
        # quantization="fp8" (weights.from_state_dicts): the layers hold only E4M3 codes and row scales; prefill, batched decode and beams
        # run their linears as the activation quantizer + an FP8 GEMM, the one-token step streams the codes through the FP8 GEMV (DESIGN.md
        # §3).  The verify pass of prompt-lookup decoding has no FP8 form.
        self.fp8 = getattr(w, "quantization", None) == "fp8"
        if self.fp8:
            self.supports_prompt_lookup = False
        # quantization="nf4" with nf4_dequantized_copy=False: the matrices with planes have no dequantized copy, so prefill, batched decode,
        # beams and the verify pass read the planes as well (srgpt_gemm_nf4_bf16, srgpt_gemv_multi_nf4_bf16; bit-identical to the copy)
        self.nf4_planes_only = getattr(w, "quantization", None) == "nf4" and not getattr(w, "nf4_dequantized_copy", True)
        if self.nf4_planes_only and os.environ.get("SRGPT_DECODE_NF4", "1") == "0":
            raise ValueError("SRGPT_DECODE_NF4=0 runs the decode step over the dequantized copies, which a model loaded with "
                             "nf4_dequantized_copy=False does not keep")
        # Captured CUDA graphs: GraphKey -> (graph, kernels one replay launches).  A graph holds the addresses of every buffer it reads,
        # so it is dropped whenever one of them is replaced: the KV cache and the layer stack's array (ensure_capacity), the processor
        # spec (_set_processors), the score buffer (_scores_view) and the batched-decode buffers (_batch_state).
        self._graphs = {}
        # sampling mode (do_sample=True): temperature / top_p live in device memory so one captured graph serves any setting
        self.sample_params = torch.tensor([1.0, 1.0, 0.0], dtype=torch.float32, device=dev)
        # with typical_p / epsilon_cutoff / eta_cutoff on, the draws read these 6 floats {T, top_p, top_k, typical_p, epsilon, eta}
        # instead (the warped sampler, its own graphs: GraphKey.warp); with all three off they run exactly as before
        self.warp_params = torch.tensor([1.0, 1.0, 0.0, 1.0, 0.0, 0.0], dtype=torch.float32, device=dev)
        self.warp = False
        self.sample_logits: Optional[torch.Tensor] = None
        self.sample_seed = 0
        self.sample_seed_dev = torch.zeros(1, dtype=torch.int64, device=dev)  # device copy: the captured graph reads the seed at run time
        # logits processors (repetition penalty, no-repeat n-grams, bad words, minimum length; logits_processors.py): the parameters live
        # in device memory so one captured graph per mode serves every setting.  The spec buffer is sized at first use and grown when a
        # request needs more, which drops the graphs that read it.
        self.proc_fparams = torch.ones(2, dtype=torch.float32, device=dev)
        self.proc_spec: Optional[torch.Tensor] = None
        self.proc_logits: Optional[torch.Tensor] = None  # the processed fp32 row of the one-token step (sampling reads it)
        self.proc_ids = torch.zeros(1, dtype=torch.int64, device=dev)
        # Reusable prompt prefix of sequence 0: its first `prefix_rows` positions hold K/V that a batch-1 PREFILL wrote and nothing has
        # overwritten since (generate_from_embeds(reuse_rows=n) continues from them).  Positions written by decode steps are never
        # counted: the reference prefills them again, and the GEMV decode path rounds differently from the prefill GEMMs.
        # `prefix_epoch` changes whenever the record does, so a caller can tell that someone else's request came in between.
        self.prefix_rows = 0
        self.prefix_epoch = 0
        # The batch-1 decode step streams its matrices in the lossless 12-bit packing (DESIGN.md §3): 3/4 of the bytes, bit-identical
        # results.  The bf16 weights stay resident for prefill and batched decode.  decode_pack: matrix -> "packed" or why it is plain.
        self.decode_pack = {}
        # NF4 layer matrices (weights.from_state_dicts(quantization="nf4")): the layer matrices hold the dequantized values for every path,
        # and the batch-1 decode step streams the NF4 planes instead (bit-identical).  decode_quant: matrix -> "nf4" or why the step reads
        # its dequantized copy.  SRGPT_DECODE_NF4=0 runs the usual step over the dequantized copies.
        self.decode_quant = {}
        self._build_stack()
        self.kernels_per_decode_step = self.stack.step_kernels
        self._batch_kernels_per_layer = self.stack.kernels_per_layer  # batched decode step: as a prefill layer

    supports_prefix_reuse = True
    supports_prompt_lookup = True
    supports_logits_processors = True
    supports_batch_sampling = True  # sampled batches run in the batched step (generate_batch), num_return_sequences included
    supports_output_scores = True  # generate(output_scores=True): the decode steps write each token's score row on the device
    supports_batch_invariant = True  # generate(batch_invariant=True): generate_rows, each row bit-identical to batch 1
    supports_contrastive = True  # generate(penalty_alpha=, top_k=): generate_contrastive
    supports_forward_outputs = True  # forward(output_hidden_states=, output_attentions=): the probed prefill (PrefillProbe)
    supports_generate_outputs = True  # generate(output_hidden_states=, output_attentions=): the probed prefill and decode steps
    packs_decode_weights = True
    _vstate = None  # buffers of the verify pass (prompt-lookup speculative decoding), allocated on first use
    _bstate = None  # buffers of the batched decode step, for the batch size of the last batched request
    _rstate = None  # buffers of the batch-invariant rows step (generate_rows), allocated on first use
    _scores = None  # the score buffer of output_scores (_scores_view), allocated on first use
    _host_ids = None  # pinned host copy of generated ids for the stop checks, and the stream that fills it (_pinned_ids)
    _copy_stream = None
    last_speculation = (0, 0, 0)
    nf4_planes_only = False
    stack: Optional[ops.LlamaStack] = None  # the layers as the composite entry points take them (_build_stack)

    @property
    def _packed_array(self):
        """The srgpt_llama_layer_packed[] the decode step streams, None when it streams no packed matrix."""
        return self.stack.packed

    @property
    def _nf4_array(self):
        """The srgpt_llama_layer_nf4[] the decode step streams, None when it streams no NF4 planes."""
        return self.stack.nf4

    @ops.in_own_dtype
    def _build_stack(self) -> None:
        """The layers as the composite entry points take them (ops.LlamaStack), and the reports of what the decode step streams.  FP8 and
        NF4 layers stream their codes or planes; lm_head stays unquantized and is packed in the bf16 build (SRGPT_DECODE_PACK=0: plain).
        Unquantized bf16 layers stream their 12-bit packings, where a matrix has one."""
        w, quant = self.w, getattr(self.w, "quantization", None)
        pack = self.dtype == torch.bfloat16 and os.environ.get("SRGPT_DECODE_PACK", "1") != "0"
        packed, lm_packed = None, None
        if quant == "fp8" or (quant == "nf4" and os.environ.get("SRGPT_DECODE_NF4", "1") != "0"):
            for l, lw in enumerate(w.layers):
                for name in ("qkv", "o", "gateup", "down"):
                    K = getattr(lw, name + "_w").shape[1]
                    self.decode_quant[f"layers.{l}.{name}"] = ("fp8" if quant == "fp8" else "nf4" if lw.nf4[name] is not None else
                                                               f"K = {K} is not a multiple of {ops.NF4_BATCH}")
            if pack:
                lm_packed, why = ops.pack12(w.lm_head)
                self.decode_pack["lm_head"] = why or "packed"
        elif self.packs_decode_weights and pack:
            packed = []
            for l, lw in enumerate(w.layers):
                packed.append({})
                for name in ("qkv", "o", "gateup", "down"):
                    packed[l][name], why = ops.pack12(getattr(lw, name + "_w"))
                    self.decode_pack[f"layers.{l}.{name}"] = why or "packed"
            lm_packed, why = ops.pack12(w.lm_head)
            self.decode_pack["lm_head"] = why or "packed"
            if "packed" not in self.decode_pack.values():
                packed = None
        pages = [self.cache.layer(l) for l in range(self.dims.num_hidden_layers)]
        self.stack = ops.LlamaStack(w.layers, pages, packed=packed, nf4="nf4" in self.decode_quant.values(), planes_only=self.nf4_planes_only,
                                    lm_packed=lm_packed)

    def _record_prefix(self, rows: int) -> None:
        self.prefix_rows = rows
        self.prefix_epoch += 1

    # ---------------------------------------------------------------------------------------------
    @ops.in_own_dtype
    def ensure_capacity(self, n_seqs: int, tokens_per_seq: int) -> None:
        """Grow the paged cache so `n_seqs` sequences of `tokens_per_seq` tokens fit at once (batched prefill).
        Re-allocation drops all cached sequences and the captured graphs (page addresses change)."""
        need_pages = n_seqs * ((tokens_per_seq + PAGE_SIZE - 1) // PAGE_SIZE)
        self._grow_cache(n_seqs, need_pages, f"{n_seqs} x {tokens_per_seq} tokens")

    def _page_bytes(self) -> int:
        d = self.dims
        return 2 * PAGE_SIZE * d.num_key_value_heads * d.head_dim * 2 * d.num_hidden_layers

    def _grow_cache(self, n_seqs: int, need_pages: int, what: str) -> None:
        """Re-allocate the paged cache when it has fewer than `n_seqs` slots or `need_pages` pages (ensure_capacity)."""
        c = self.cache
        if n_seqs <= len(c.owned) and need_pages <= c.n_pages:
            return
        d = self.dims
        per_page = self._page_bytes()
        free_b, _ = torch.cuda.mem_get_info(self.device)
        cur_b = c.pages.numel() * 2
        if need_pages * per_page > free_b + cur_b - (2 << 30):
            raise RuntimeError(f"KV cache for {what} needs {need_pages * per_page >> 20} MiB, not available")
        self._drop_graphs()
        self._record_prefix(0)
        n_pages_old, n_seqs_old = c.n_pages, len(c.owned)
        self.cache = None
        del c
        self.cache = PagedKVCache(d, max(need_pages, n_pages_old), max(n_seqs, n_seqs_old), (self.max_seq_len + PAGE_SIZE - 1) // PAGE_SIZE, self.device, self.dtype)
        self.stack.set_pages([self.cache.layer(l) for l in range(d.num_hidden_layers)])

    @ops.in_own_dtype
    def embed_tokens(self, ids: torch.Tensor) -> torch.Tensor:
        """Embedding gather through the splice kernel (source 0 only)."""
        flat = ids.reshape(-1).to(device=self.device, dtype=torch.int32)
        if flat.numel():  # nn.Embedding raises on an out-of-range id; the gather kernel itself has no bounds check
            lo, hi = int(flat.min()), int(flat.max())
            if lo < 0 or hi >= self.w.embed.shape[0]:
                raise IndexError(f"token id {lo if lo < 0 else hi} is outside the token table [0, {self.w.embed.shape[0]})")
        return ops.splice_rows(self.w.embed, None, None, None, torch.zeros_like(flat), flat)

    @ops.in_own_dtype
    def prefill_hidden(self, inputs_embeds: torch.Tensor, seq: int = 0, start_pos: int = 0, probe: Optional[PrefillProbe] = None) -> torch.Tensor:
        """Run all layers over one sequence's prompt rows [S, H] at positions start_pos .. start_pos + S - 1; fills the KV cache;
        returns the final-layer residual stream [S, H] (before the final norm).  With start_pos > 0 the rows are a chunk that
        continues the sequence: positions [0, start_pos) must already be in its pages, and attention reads them from there.
        ``probe``: record the hidden states / attention probabilities (PrefillProbe; whole prompts only, start_pos 0)."""
        d, w = self.dims, self.w
        S = inputs_embeds.shape[0]
        if start_pos < 0 or start_pos + S > self.max_seq_len:
            raise RuntimeError(f"prompt of {S} tokens at {start_pos} exceeds max_seq_len {self.max_seq_len}")
        if probe is not None and start_pos != 0:
            raise NotImplementedError("hidden states and attentions of a chunked prefill")
        self._record_prefix(0)
        self.cache.reserve(seq, start_pos + S)
        sp = torch.tensor([start_pos], dtype=torch.int32, device=self.device)
        x = inputs_embeds.to(self.dtype).contiguous().clone()
        if start_pos != 0:
            cu = torch.tensor([0, S], dtype=torch.int32, device=self.device)
            return ops.llama_prefill_chunk_layers(x, self.stack, d, self.cos, self.sin, sp, self.cache.page_tables[seq:seq + 1], PAGE_SIZE,
                                                  self.cache.n_pages, cu, S)
        if probe is not None:
            return ops.llama_prefill_layers_probe(x, self.stack, d, self.cos, self.sin, sp, self.cache.page_tables[seq], PAGE_SIZE, probe.row_off,
                                                  probe.hidden, probe.attn)
        return ops.llama_prefill_layers(x, self.stack, d, self.cos, self.sin, sp, self.cache.page_tables[seq], PAGE_SIZE)

    @ops.in_own_dtype
    def prefill_packed(self, packed_embeds: torch.Tensor, seq_lens: List[int], page_tables: Optional[torch.Tensor] = None,
                       probe: Optional[PrefillProbe] = None) -> torch.Tensor:
        """Prefill `len(seq_lens)` prompts packed back to back ([sum S_b, H]) into sequence slots 0..B-1 (or the rows of
        ``page_tables``, a row-strided view of the cache's tables) in ONE pass: every GEMM runs over all rows, attention / RoPE / KV
        append per sequence (the unpadded varlen path of modeling_llama.py:540-562).  The caller has reserved the pages.  Returns the
        final residual stream, packed.  ``probe``: record the hidden states / attention probabilities (PrefillProbe)."""
        d = self.dims
        B = len(seq_lens)
        if packed_embeds.shape[0] != sum(seq_lens) or B < 1 or min(seq_lens) < 1:
            raise RuntimeError("prefill_packed: rows do not match seq_lens")
        if max(seq_lens) > self.max_seq_len:
            raise RuntimeError(f"prompt of {max(seq_lens)} tokens exceeds max_seq_len {self.max_seq_len}")
        self._record_prefix(0)
        cu = torch.tensor([0] + list(torch.tensor(seq_lens).cumsum(0).tolist()), dtype=torch.int32).to(self.device)
        sp = torch.zeros(B, dtype=torch.int32, device=self.device)
        x = packed_embeds.to(self.dtype).contiguous().clone()
        pts = self.cache.page_tables[:B] if page_tables is None else page_tables
        if probe is not None:
            return ops.llama_prefill_layers_probe(x, self.stack, d, self.cos, self.sin, sp, pts, PAGE_SIZE, probe.row_off, probe.hidden, probe.attn,
                                                  cu_seqlens=cu, max_seqlen=max(seq_lens))
        return ops.llama_prefill_layers(x, self.stack, d, self.cos, self.sin, sp, pts, PAGE_SIZE, cu_seqlens=cu, max_seqlen=max(seq_lens))

    @ops.in_own_dtype
    def first_tokens(self, hidden_packed: torch.Tensor, seq_lens: List[int], return_logits: bool = False, repeat: int = 1):
        """Greedy first token of every packed sequence: final norm + lm_head over the B last rows as one GEMM
        (bf16 logits, modeling_llama.py:1044-1045), argmax with the lowest index on ties.  ``repeat=n``: each last row n times
        (B * n rows, row b * n + j from sequence b)."""
        last = (torch.tensor(seq_lens).cumsum(0) - 1).repeat_interleave(repeat).to(torch.int32).to(self.device)
        rows = ops.splice_rows(hidden_packed, None, None, None, torch.zeros_like(last), last)
        hn = ops.rmsnorm(rows, self.w.norm, self.dims.rms_norm_eps)
        lg = ops.gemm(hn, self.w.lm_head, out=self._logits_buffer(hn.shape[0]))
        ids = ops.argmax_bf16(lg)
        return (ids, lg) if return_logits else ids

    def _logits_buffer(self, rows: int) -> torch.Tensor:
        """bf16 [rows, V] view with a 16-byte-aligned row stride (V = 128259 is odd; the GEMM stores 16-byte vectors)."""
        V = self.dims.vocab_size
        return torch.empty((rows, (V + 7) // 8 * 8), dtype=self.dtype, device=self.device)[:, :V]

    @ops.in_own_dtype
    def logits_all(self, hidden: torch.Tensor, normed: Optional[torch.Tensor] = None) -> torch.Tensor:
        """lm_head over every row -> fp32 logits [S, V] (LlamaForCausalLM.forward semantics, 1044-1045)."""
        return self.lm_head_rows(hidden, normed=normed).float()  # bf16 rounding first, then .float()

    @ops.in_own_dtype
    def final_norm(self, hidden: torch.Tensor) -> torch.Tensor:
        """The final RMSNorm of every row of ``hidden``: the rows the lm_head GEMM reads."""
        return ops.rmsnorm(hidden, self.w.norm, self.dims.rms_norm_eps)

    @ops.in_own_dtype
    def lm_head_rows(self, hidden: torch.Tensor, out: Optional[torch.Tensor] = None, normed: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Final norm + lm_head over every row of ``hidden`` -> element-type logits [S, V] (into ``out``, default a fresh
        _logits_buffer).  ``normed``: final_norm(hidden) when the caller has it already."""
        hn = self.final_norm(hidden) if normed is None else normed
        return ops.gemm(hn, self.w.lm_head, out=self._logits_buffer(hn.shape[0]) if out is None else out)

    # ---------------------------------------------------------------------------------------------
    def _decode_step_launch(self, seq: int, logits_out: Optional[torch.Tensor] = None, sample: bool = False, proc: bool = False,
                            scores: Optional[torch.Tensor] = None, probe: Optional[ops.StepProbe] = None) -> None:
        d, w = self.dims, self.w
        if (sample or proc or scores is not None) and logits_out is None:
            logits_out = self._sample_buffer()
        ops.llama_decode_step(self.h, self.stack, self.q_buf, self.attn_buf, self.act_buf, d, self.cos, self.sin, self.pos, self.active_pt, PAGE_SIZE,
                              w.norm, w.lm_head, w.embed, self.lm_ws, self.out_ids, self.step, logits_out,
                              **({} if probe is None else dict(probe=probe)))
        self._choose(logits_out, sample, proc, scores)

    def _choose(self, raw: Optional[torch.Tensor], sample: bool, proc: bool, scores: Optional[torch.Tensor]) -> None:
        """After an lm_head that advanced the step and wrote the greedy choice: the processors and / or the draw replace that choice, and
        with ``scores`` ([T, 1, V] fp32) the row the token was chosen from goes to scores[step - 1] (the raw row when greedy without
        processors, the processed row when greedy with them, the warped row when sampled)."""
        if proc:
            self._process_row(raw, sample, scores)
        elif sample:  # replaces the greedy id / next embedding row the finalize kernel just wrote (step already advanced)
            ops.sample_top_p(raw, self._draw_params, self.sample_seed_dev, self.step, -1, self.out_ids, self.w.embed, self.h,
                             **self._scores_kw(scores, True))
        elif scores is not None:
            ops.step_scores(raw, self.step, -1, scores)

    def _process_row(self, raw: torch.Tensor, sample: bool, scores: Optional[torch.Tensor] = None) -> None:
        """After an lm_head that advanced the step: the processors over the raw fp32 row (history = out_ids[:step - 1]), then the
        processed greedy choice, or a draw from the processed row, replaces out_ids[step - 1] and the next embedding row."""
        w = self.w
        if (sample or scores is not None) and self.proc_logits is None:
            self.proc_logits = torch.empty(self.dims.vocab_size, dtype=torch.float32, device=self.device)
        if sample:
            ops.logits_process(raw, self.out_ids, 0, 1, self.step, -1, self.proc_fparams, self.proc_spec, out=self.proc_logits)
            ops.sample_top_p(self.proc_logits, self._draw_params, self.sample_seed_dev, self.step, -1, self.out_ids, w.embed, self.h,
                             **self._scores_kw(scores, True))
        else:
            ops.logits_process(raw, self.out_ids, 0, 1, self.step, -1, self.proc_fparams, self.proc_spec, ids=self.proc_ids,
                               **({} if scores is None else {"out": self.proc_logits}))
            ops.logits_pick_token(self.proc_ids, self.step, -1, self.out_ids, w.embed, self.h)
            if scores is not None:
                ops.step_scores(self.proc_logits, self.step, -1, scores)

    def _set_processors(self, processors) -> bool:
        """processors = None or a spec of logits_processors.parse / resolve_min_length.  Writes its device encoding; True when on."""
        if not processors:
            return False
        V = self.dims.vocab_size
        if any(t < 0 or t >= V for s in processors.get("bad_words_ids") or [] for t in s):
            raise ValueError(f"bad_words_ids holds a token outside the vocabulary [0, {V})")
        fparams, ints = logits_processors.encode(processors)
        if self.proc_spec is None or self.proc_spec.numel() < ints.size:
            cap = 256
            while cap < ints.size:
                cap *= 2
            self.proc_spec = torch.zeros(cap, dtype=torch.int32, device=self.device)
            self._drop_graphs(lambda key: key.proc)  # the graphs with processing on read the old buffer
        self.proc_spec[: ints.size].copy_(torch.from_numpy(ints))
        self.proc_fparams.copy_(torch.from_numpy(fparams))
        return True

    def _sample_buffer(self) -> torch.Tensor:
        if self.sample_logits is None:
            self.sample_logits = torch.empty(self.dims.vocab_size, dtype=torch.float32, device=self.device)
        return self.sample_logits

    def _scores_view(self, steps: int, rows: int) -> torch.Tensor:
        """fp32 [steps, rows, V] over the decoder's score buffer (output_scores): the captured graphs that write scores hold its address,
        so it lives across requests and grows (dropping those graphs) when a request needs more."""
        need = steps * rows * self.dims.vocab_size
        if self._scores is None or self._scores.numel() < need:
            self._drop_graphs(lambda key: key.scores is not None)
            self._scores = None
            self._scores = torch.empty(need, dtype=torch.float32, device=self.device)
        return self._scores[:need].view(steps, rows, self.dims.vocab_size)

    @staticmethod
    def _scores_kw(scores: Optional[torch.Tensor], strided: bool = False) -> dict:
        """The sampler's keywords for a score buffer view; none without one, so the call is today's call."""
        if scores is None:
            return {}
        return {"scores": scores, "step_stride": scores.stride(0)} if strided else {"scores": scores}

    @staticmethod
    def _scores_key(scores: Optional[torch.Tensor]) -> Optional[tuple]:
        """GraphKey.scores of a score buffer view: a graph holds the address and the step stride it writes to."""
        return None if scores is None else (scores.data_ptr(), scores.stride(0))

    # ---- captured graphs ---------------------------------------------------------------------------------------------------------
    def _capture(self, key, launch, restore, kernels: int) -> torch.cuda.CUDAGraph:
        """The graph stored under `key`, captured from `launch()` if there is none: one warm-up run outside capture (lazy kernel
        attribute setup) on a side stream, the tensors in `restore` put back as they were, then the capture.  `kernels` is what one
        replay launches (ops.LAUNCHES accounting)."""
        if key in self._graphs:
            return self._graphs[key][0]
        if key.probe is not None:  # every request records into new tensors: keep one probed graph, not one per request
            self._drop_graphs(lambda k: k.probe is not None)
        saved = [t.clone() for t in restore]
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream())  # after the clones are enqueued
        with torch.cuda.stream(s):
            launch()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        for t, v in zip(restore, saved):
            t.copy_(v)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            launch()
        self._graphs[key] = (g, kernels)
        return g

    def _replay(self, key) -> None:
        g, kernels = self._graphs[key]
        g.replay()
        ops.LAUNCHES += kernels

    def _drop_graphs(self, match=lambda key: True) -> None:
        """Forget the captured graphs whose key matches (all of them by default)."""
        self._graphs = {k: v for k, v in self._graphs.items() if not match(k)}

    @property
    def _graph(self) -> Optional[torch.cuda.CUDAGraph]:
        """The greedy one-token step graph, once _ensure_graph has captured it."""
        entry = self._graphs.get(GraphKey("step"))
        return None if entry is None else entry[0]

    def _ensure_graph(self, seq: int, sample: bool = False, proc: bool = False, scores: Optional[torch.Tensor] = None,
                      probe: Optional[ops.StepProbe] = None) -> torch.cuda.CUDAGraph:
        """The one-token step graph of this mode.  Sampling adds its kernel; processing adds 1 more when sampling, 3 when greedy
        (processing, key unpack and pick); greedy score rows add their copy (the sampler writes its own); a probe its launches."""
        kernels = self.kernels_per_decode_step + (1 if sample else 0) + ((1 if sample else 3) if proc else 0) + (
            1 if scores is not None and not sample else 0) + (0 if probe is None else probe.kernels(self.dims.num_hidden_layers, final_norm=True))
        return self._capture(GraphKey("step", 1, sample, proc, self._scores_key(scores), probe=None if probe is None else probe.key(),
                                      warp=sample and self.warp),
                             lambda: self._decode_step_launch(seq, sample=sample, proc=proc, **self._scores_kw(scores),
                                                              **({} if probe is None else dict(probe=probe))),
                             (self.pos, self.step, self.h, self.out_ids), kernels)

    # ---- stop checks: generated ids reach the host through pinned memory while the next step runs --------------------------------
    def _pinned_ids(self, n: int) -> torch.Tensor:
        """n elements of pinned int64 host memory, and the copy stream _to_host fills it on; created on first use, grown when a batch
        needs more."""
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        if self._host_ids is None or self._host_ids.numel() < n:
            self._host_ids = torch.empty(max(n, self.out_ids.numel()), dtype=torch.int64, pin_memory=True)
        return self._host_ids[:n]

    def _to_host(self, *copies) -> torch.cuda.Event:
        """Enqueue each (device slice, pinned slice) copy on the copy stream, ordered after the work enqueued so far; returns the event
        that marks their completion."""
        side = self._copy_stream
        e = torch.cuda.Event()
        e.record()
        side.wait_event(e)
        with torch.cuda.stream(side):
            for src, dst in copies:
                dst.copy_(src, non_blocking=True)
            done = torch.cuda.Event()
            done.record(side)
        return done

    def _run_steps(self, launch, out2d: torch.Tensor, budgets: List[int], eos, stopping_fn) -> List[int]:
        """decode_steps over the device ids ``out2d`` ([T, B]); the rows it inspects reach pinned memory on the copy stream."""
        host = self._pinned_ids(out2d.numel()).view(out2d.shape) if eos or stopping_fn is not None else None
        return decode_steps(launch, lambda n: self._to_host((out2d[n], host[n])), host, budgets, eos, stopping_fn)

    def _start_request(self, prompt_lens: List[int], max_new_tokens: int, writes_ids: bool = True, keep: Optional[int] = None,
                       slack: int = 0) -> None:
        """The KV cache of a request whose slot b continues a prompt of prompt_lens[b] rows by up to max_new_tokens tokens: every
        slot but ``keep`` (whose prompt prefix is reused) released, the cache grown to hold the rows, and each row's pages reserved
        with ``slack`` more positions (prompt lookup's verify passes write past the budget).  ``writes_ids``: the ids go to out_ids,
        whose length caps max_new_tokens; beam search keeps its ids on the host."""
        if writes_ids and max_new_tokens > self.out_ids.numel():
            raise RuntimeError(f"max_new_tokens {max_new_tokens} exceeds the decoder's cap {self.out_ids.numel()}")
        S = max(prompt_lens)
        if S + max_new_tokens > self.max_seq_len:  # every row stays in the step until the last one stops
            raise RuntimeError(f"{S} prompt + {max_new_tokens} new tokens exceed max_seq_len {self.max_seq_len}")
        self.cache.release_all(keep)
        if keep is None:  # growing re-allocates the cache, which would lose the kept slot's K/V
            self.ensure_capacity(len(prompt_lens), S + max_new_tokens + slack)
        self.cache.reserve_many([n + max_new_tokens + slack for n in prompt_lens])

    def _prefill_first_token(self, embeds: torch.Tensor, seq: int, reuse_rows: int, logits_row: Optional[torch.Tensor], sample: bool,
                             proc: bool, scores: Optional[torch.Tensor], probe: Optional[GenerateProbe] = None) -> torch.Tensor:
        """Batch 1's prefill of the prompt ``embeds`` [S, H] into sequence `seq` (its first reuse_rows rows are in the pages already)
        and its first token: final norm + lm_head + arg max on the last row, which writes out_ids[0], the token's embedding row (h)
        and pos = S, step = 1; then _choose.  The fp32 logits go to ``logits_row``, or to the sample buffer when the choice reads
        them.  generate_rows starts every row with it, so each row's first token is its batch-1 request's by construction.  Returns
        the prefill's final residual stream of rows reuse_rows .. S - 1.  ``probe``: the prefill records the prompt step (whole prompts)."""
        d, w = self.dims, self.w
        S = embeds.shape[0]
        if probe is None:
            hidden = self.prefill_hidden(embeds[reuse_rows:], seq, reuse_rows)
        else:
            hidden = self.prefill_hidden(embeds[reuse_rows:], seq, reuse_rows, probe=probe.prefill)
            probe.record_final(self, hidden, [S])
        self.pos.fill_(S - 1)
        self.step.zero_()
        if logits_row is None and (sample or proc or scores is not None):
            logits_row = self._sample_buffer()
        ops.lm_head_argmax(hidden[S - 1 - reuse_rows], w.lm_head, w.norm, d.rms_norm_eps, self.lm_ws, self.out_ids, self.step, self.pos,
                           embed_table=w.embed, next_x=self.h, logits_out=logits_row)
        self._choose(logits_row, sample, proc, scores)
        return hidden

    def _set_sampling(self, sampling) -> bool:
        """sampling = None (greedy) or dict(temperature=, top_p=, top_k=, seed=, and optionally typical_p=, epsilon_cutoff=, eta_cutoff=).
        Returns True when tokens are sampled; self.warp tells whether a typical / epsilon / eta warper is on."""
        self.warp = False
        if not sampling:
            return False
        t = float(sampling.get("temperature") or 1.0)
        p = sampling.get("top_p")
        p = 1.0 if p is None else float(p)
        k = sampling.get("top_k")
        k = 50 if k is None else int(k)  # GenerationConfig's default top_k, applied by HF whenever do_sample=True
        if t <= 0.0 or not (0.0 < p <= 1.0) or k < 0:
            raise ValueError(f"sampling needs temperature > 0, 0 < top_p <= 1 and top_k >= 0, got temperature={t}, top_p={p}, top_k={k}")
        warpers = sampling_warpers(sampling)
        self.sample_params.copy_(torch.tensor([t, p, float(k)], dtype=torch.float32))
        self.warp = warpers != (1.0, 0.0, 0.0)
        if self.warp:
            self.warp_params.copy_(torch.tensor([t, p, float(k), *warpers], dtype=torch.float32))
        seed = sampling.get("seed")
        self._set_seed(int(torch.initial_seed() if seed is None else seed))
        return True

    @property
    def _draw_params(self) -> torch.Tensor:
        """The params the draws read: warp_params (the warped sampler) when a warper is on, else sample_params."""
        return self.warp_params if self.warp else self.sample_params

    def _set_seed(self, seed: int) -> None:
        self.sample_seed = seed & 0x7FFFFFFFFFFFFFFF
        self.sample_seed_dev.copy_(torch.tensor([self.sample_seed], dtype=torch.int64))

    @torch.no_grad()
    @ops.in_own_dtype
    def generate_from_embeds(self, inputs_embeds: torch.Tensor, max_new_tokens: int, eos_token_ids=None, stopping_fn=None,
                             use_graph: bool = True, return_logits: bool = False, seq: int = 0, sampling=None, reuse_rows: int = 0,
                             lookup_ids: Optional[torch.Tensor] = None, lookup_k: int = 0, lookup_ngram: int = 2, processors=None,
                             output_scores: bool = False, outputs: Optional[GenerateProbe] = None):
        """Greedy (or, with ``sampling=dict(temperature, top_p, seed)``, nucleus-sampled) decoding started from prompt
        embeddings [S, H].  Returns LongTensor [n_new] (and fp32 logits [n_new, V] when return_logits).
        ``stopping_fn(ids_so_far: LongTensor) -> bool``.
        ``reuse_rows=n`` keeps the K/V of the first n prompt rows of sequence 0 from the previous batch-1 prefill and prefills only
        rows n..S-1 (chunked prefill at start_pos n); the caller vouches that those rows are the same as before.  n must not exceed
        ``prefix_rows`` nor S - 1 (the last prompt row is always computed: the first new token needs its hidden state).
        ``lookup_k=k > 0`` (greedy, sequence 0): prompt-lookup speculative decoding after the first token (_verify_loop).  Each verify
        pass drafts up to k tokens (clamped to ops.SPEC_T_MAX - 1) by n-gram lookup (sizes lookup_ngram .. 1) in ``lookup_ids`` (int,
        negative = a row that never matches) followed by the generated tokens, and keeps the drafts that equal the model's own greedy
        choices plus one token of its own.  The ids and logits are bit-identical to plain greedy decoding whatever the drafts are.
        ``last_speculation`` = (verify passes, tokens drafted, tokens accepted) of the passes up to the last returned token; a
        request whose verify slack does not fit max_seq_len or the decoder's token cap runs the one-token loop and reports (0, 0, 0).
        ``processors`` (a spec of logits_processors.resolve_min_length, or None): HF's repetition penalty / no-repeat n-gram / bad words /
        minimum length over every token's logits, the first one included, before the greedy choice or the sampling warpers; the history
        is the generated tokens.  Returned logits stay raw, as HF's output_logits.
        ``output_scores``: returns (what it returns without, {"scores": fp32 [n_new, 1, V]}), row t being the row token t was chosen from
        (HF's output_scores): the raw row when greedy, the processed row with processors, the warped row (logits / T, -inf where top-k /
        top-p removed the token) when sampled.  The decode graphs write them on the device; prompt-lookup decoding takes them from its
        verify passes' logit rows (greedy without processors: the raw rows).
        ``outputs`` (GenerateProbe of one row; not with reuse_rows or prompt lookup): the prefill records the prompt step and every
        decode step records its hidden rows / attention probabilities at the device step; ids, scores and logits are unchanged."""
        d = self.dims
        S = inputs_embeds.shape[0]
        n_reuse = int(reuse_rows)
        if outputs is not None and (n_reuse != 0 or lookup_k):
            raise NotImplementedError("hidden states / attentions with a reused prompt prefix or prompt lookup")
        if n_reuse != 0 and (seq != 0 or n_reuse < 0 or n_reuse > self.prefix_rows or n_reuse > S - 1):
            raise ValueError(f"reuse_rows={n_reuse} is not a reusable prefix here: sequence {seq}, {self.prefix_rows} recorded prefill rows, "
                             f"{S} prompt rows (at most S - 1 may be reused)")
        if max_new_tokens < 1:
            empty = torch.empty(0, dtype=torch.int64, device=self.device)
            return (empty, {"scores": torch.empty((0, 1, d.vocab_size), dtype=torch.float32, device=self.device)}) if output_scores else empty
        if lookup_k and self.fp8:
            raise NotImplementedError("prompt-lookup decoding (prompt_lookup_num_tokens) has no FP8 verify pass; decode FP8 weights without it")
        eos = eos_list(eos_token_ids)
        k = min(int(lookup_k), ops.SPEC_T_MAX - 1) if lookup_k else 0
        self.last_speculation = (0, 0, 0)
        if k > 0 and (seq != 0 or sampling or int(lookup_ngram) < 1 or processors):
            raise ValueError("prompt-lookup decoding serves greedy decoding of sequence 0 with lookup_ngram >= 1, without logits processors")
        proc = self._set_processors(processors)
        sample = self._set_sampling(sampling)
        # a verify pass writes up to T positions past the last emitted token, and one pass is in flight after the stop is seen
        slack = 2 * ops.SPEC_T_MAX if k > 0 else 0
        if slack and (S + max_new_tokens + slack > self.max_seq_len or max_new_tokens + slack > self.out_ids.numel()):
            k, slack = 0, 0
        # the prompt goes to slot `seq` (the slots before it are reserved alike and stay unused)
        self._start_request([S] * (seq + 1), max_new_tokens, keep=seq if n_reuse else None, slack=slack)
        n_rows = max_new_tokens + slack  # verify passes write accepted logit rows past the budget too
        # prompt lookup's scores are its logit rows (greedy without processors), which the verify passes write on the logits_all route
        lookup_scores = output_scores and k > 0 and max_new_tokens > 1
        logits = torch.empty((n_rows, d.vocab_size), dtype=torch.float32, device=self.device) if return_logits or lookup_scores else None
        scores = self._scores_view(max_new_tokens, 1) if output_scores and not lookup_scores else None
        self._prefill_first_token(inputs_embeds, seq, n_reuse, None if logits is None else logits[0], sample, proc, scores,
                                  **({} if outputs is None else dict(probe=outputs)))
        if seq == 0 and self.supports_prefix_reuse:
            self._record_prefix(S)
        if k > 0 and max_new_tokens > 1:
            r = self._verify_loop(k + 1, int(lookup_ngram), lookup_ids, max_new_tokens, eos, stopping_fn, use_graph, logits)
            if not output_scores:
                return r
            out, lg = r
            return (r, {"scores": lg.unsqueeze(1).clone()}) if return_logits else (out, {"scores": lg.unsqueeze(1)})
        r = self._decode_loop(seq, max_new_tokens, eos, stopping_fn, use_graph, logits, sample, proc, scores,
                              **({} if outputs is None or outputs.steps is None else dict(probe=outputs.steps)))
        if not output_scores:
            return r
        return r, {"scores": scores[:(r[0] if return_logits else r).numel()].clone()}

    # ---- prompt-lookup speculative decoding: verify passes of T = k + 1 tokens, every weight streamed once per pass ---------------
    def _verify_buffers(self):
        st = self._vstate
        if st is not None:
            return st
        d, dev, Tm = self.dims, self.device, ops.SPEC_T_MAX
        H, qd, I = d.hidden_size, d.num_attention_heads * d.head_dim, d.intermediate_size
        z = lambda *shape, dtype=self.dtype: torch.zeros(shape, dtype=dtype, device=dev)  # noqa: E731
        st = dict(h=z(Tm, H), q=z(Tm, qd), attn=z(Tm, qd), act=z(Tm, I), ws=z(Tm * self.lm_ws.numel(), dtype=torch.uint8), logits=None,
                  pos_rows=z(Tm, dtype=torch.int32), draft=z(Tm, dtype=torch.int32), state=z(8, dtype=torch.int32),
                  prompt=z(self.max_seq_len, dtype=torch.int32), prompt_len=z(1, dtype=torch.int32),
                  host_state=torch.zeros((self.out_ids.numel() + 2, 8), dtype=torch.int32, pin_memory=True))
        self._vstate = st
        return st

    def _verify_launch(self, T: int, ngram: int, logits_all: Optional[torch.Tensor] = None) -> None:
        d, w, st = self.dims, self.w, self._vstate
        if logits_all is not None and st["logits"] is None:
            st["logits"] = torch.empty((ops.SPEC_T_MAX, d.vocab_size), dtype=torch.float32, device=self.device)
        ops.llama_verify_step(st["h"], self.stack, st["q"], st["attn"], st["act"], T, d, self.cos, self.sin, self.pos, st["pos_rows"], self.active_pt,
                              PAGE_SIZE, w.norm, w.lm_head, w.embed, st["ws"], st["logits"] if logits_all is not None else None, logits_all,
                              st["prompt"], st["prompt_len"], ngram, st["draft"], self.out_ids, self.step, st["state"])

    def _verify_graph(self, T: int, ngram: int) -> torch.cuda.CUDAGraph:
        """The captured verify pass of this (T, n-gram size); its warm-up writes only this sequence's slack."""
        return self._capture(GraphKey("verify", T, ngram=ngram), lambda: self._verify_launch(T, ngram),
                             (self.pos, self.step, self.out_ids, self._vstate["state"]), self.stack.verify_kernels)

    def _verify_loop(self, T: int, ngram: int, lookup_ids, max_new_tokens: int, eos, stopping_fn, use_graph: bool, logits):
        """Tokens 1.. of sequence 0 by verify passes; pos / step / out_ids[:1] are set by the first token.  After each pass its state
        (passes, drafted, accepted, step) and a window of out_ids go to pinned memory on a side stream, and the host inspects pass r-1
        while pass r runs (the pattern of _decode_loop).  The tokens are cut at the first EOS / stopping criterion / max_new_tokens
        exactly where the one-token loop cuts them; the pass in flight at the stop writes only this sequence's reserved slack."""
        st = self._verify_buffers()
        self.active_pt.copy_(self.cache.page_tables[0])
        ids = torch.zeros(0, dtype=torch.int64) if lookup_ids is None else torch.as_tensor(lookup_ids).reshape(-1).to("cpu", torch.int64)
        ids = ids[-st["prompt"].numel():]
        ids = torch.where(ids < 0, torch.full_like(ids, -1), ids).to(torch.int32)
        if ids.numel():
            st["prompt"][: ids.numel()].copy_(ids)
        st["prompt_len"].fill_(ids.numel())
        st["state"].zero_()
        graph = use_graph and logits is None
        if graph:
            self._verify_graph(T, ngram)
        host, host_state, window = self._pinned_ids(self.out_ids.numel()), st["host_state"], 2 * T
        host[0] = int(self.out_ids[0])  # the first token (one sync, as the one-token loop's first inspection)
        n = first_stop(host, 0, 1, eos, stopping_fn, max_new_tokens)
        stats, known, r, prev = (0, 0, 0), 1, 0, None
        while n is None:
            if graph:
                self._replay(GraphKey("verify", T, ngram=ngram))
            else:
                self._verify_launch(T, ngram, logits)
            # the state after pass r and out_ids[known, + 2T): pass r's tokens lie in [step after r-1, + T), inside [step after r-2, + 2T)
            copied = self._to_host((st["state"], host_state[r]), (self.out_ids[known:known + window], host[known:known + window]))
            if r > 0:
                prev.synchronize()
                cur = int(host_state[r - 1, 6])
                stats = tuple(int(v) for v in host_state[r - 1, :3])
                n = first_stop(host, known, cur, eos, stopping_fn, max_new_tokens)
                known = cur
            prev = copied
            r += 1
        self.last_speculation = stats
        out = self.out_ids[:n].clone()
        if logits is not None:
            return out, logits[:n]
        return out

    def _decode_loop(self, seq: int, max_new_tokens: int, eos, stopping_fn, use_graph: bool, logits, sample: bool = False,
                     proc: bool = False, scores: Optional[torch.Tensor] = None, probe: Optional[ops.StepProbe] = None):
        """Steps 1..max_new_tokens-1 of sequence `seq` (greedy, or sampled; with the logits processors when proc); pos / step / h /
        out_ids[0] are already set.  ``scores`` ([T, 1, V] fp32): each step's score row goes to scores[step].  On a stop, the step in
        flight only touched this sequence's own KV slot and the step counters, which the next request resets."""
        self.active_pt.copy_(self.cache.page_tables[seq])
        graph = use_graph and logits is None
        key = GraphKey("step", 1, sample, proc, self._scores_key(scores), probe=None if probe is None else probe.key(), warp=sample and self.warp)
        probe_kw = {} if probe is None else dict(probe=probe)
        if graph:
            self._ensure_graph(seq, sample, proc, scores, **probe_kw)

        def launch(n: int) -> None:
            if graph:
                self._replay(key)
            else:
                self._decode_step_launch(seq, None if logits is None else logits[n], sample, proc, **self._scores_kw(scores), **probe_kw)

        n = self._run_steps(launch, self.out_ids[:max_new_tokens].view(max_new_tokens, 1), [max_new_tokens], eos, stopping_fn)[0]
        out = self.out_ids[:n].clone()
        if logits is not None:
            return out, logits[:n]
        return out

    # ---- batched decode: B sequences advance one token per step, every weight streamed ONCE for the whole batch ----------------
    def _batch_state(self, B: int):
        st = self._bstate
        if st is not None and st["B"] == B:
            return st
        self._drop_graphs(lambda key: key.kind in ("batch", "beam", "contrastive"))  # they read the buffers replaced here
        d, dev = self.dims, self.device
        H, nh, nkv, hd, I, V = d.hidden_size, d.num_attention_heads, d.num_key_value_heads, d.head_dim, d.intermediate_size, d.vocab_size
        z = lambda *shape, dtype=self.dtype: torch.zeros(shape, dtype=dtype, device=dev)  # noqa: E731
        st = dict(B=B, h=z(B, H), xn=z(B, H), qkv=z(B, (nh + 2 * nkv) * hd), attn=z(B, nh * hd), act=z(B, I),
                  logits=z(B, (V + 7) // 8 * 8), pos=z(B, dtype=torch.int32), step=z(1, dtype=torch.int32), ids=z(B, dtype=torch.int64),
                  out=z(self.out_ids.numel() * B, dtype=torch.int64), ticket=z(1, dtype=torch.int32),
                  cu=torch.arange(B + 1, dtype=torch.int32, device=dev), seeds=z(B, dtype=torch.int64), proc_rows=None)
        if self.stack.quantizes_activations:  # the activation quantizer's codes and row scales
            st.update(q8=z(B, max(H, nh * hd, I), dtype=torch.uint8), s8=z(B, dtype=torch.float32))
        self._bstate = st
        return st

    def _batch_step_launch(self, st, logits_only: bool = False, proc: bool = False, sample: bool = False,
                           scores: Optional[torch.Tensor] = None, probe: Optional[ops.StepProbe] = None) -> None:
        """One decode step of all B sequences (llava_arch.py:549-611 + modeling_llama.py:540-562 semantics without padding): the
        projections are wgmma GEMMs over the B rows (tall stream-K configuration), RoPE / KV append and attention per sequence.
        ``sample``: row b draws its token with st["seeds"][b] at counter step (the counter the one-token loop uses for that token).
        ``scores`` ([T, B, V] fp32): the rows the tokens were chosen from go to scores[step] (the bf16 rows widened, the processed rows,
        or the sampler's warped rows).  ``probe`` (ops.StepProbe of B rows): each layer's input rows and attention probabilities, and
        the final norm rows, go to its outputs at the device step."""
        d, w, B = self.dims, self.w, st["B"]
        nh, nkv, hd, V = d.num_attention_heads, d.num_key_value_heads, d.head_dim, d.vocab_size
        qd = nh * hd
        h, xn, qkv, attn, act = st["h"], st["xn"], st["qkv"], st["attn"], st["act"]
        pts = self.cache.page_tables

        def linear(x, wt, **kw):
            return ops.linear(x, wt, st.get("q8"), st.get("s8"), **kw)
        for l, lw in enumerate(w.layers):
            pages = self.cache.layer(l)
            if probe is not None and probe.hidden is not None:
                ops.store_step_rows(h, st["step"], probe.step_offset, probe.hidden[:, l])
            ops.rmsnorm(h, lw.in_norm, d.rms_norm_eps, out=xn)
            linear(xn, lw.qkv_w, out=qkv)
            ops.rope_kv_append_varlen(qkv, nh, nkv, hd, self.cos, self.sin, st["pos"], pages, pts, PAGE_SIZE, st["cu"])
            ops.attention_decode_batched(qkv[:, :qd], attn, pages, pts, PAGE_SIZE, st["pos"], nh, nkv, hd, self.scale)
            if probe is not None and probe.attn is not None:
                ops.attention_probs_decode(qkv[:, :qd], pages, pts, PAGE_SIZE, st["pos"], nh, nkv, hd, self.scale, probe.off, probe.n_prompt,
                                           probe.T, st["step"], probe.step_offset, probe.attn[:, l], probe.ws)
            linear(attn, lw.o_w, residual=h, epilogue=ops.EPI_BIAS_RESIDUAL, out=h)
            ops.rmsnorm(h, lw.post_norm, d.rms_norm_eps, out=xn)
            linear(xn, lw.gateup_w, epilogue=ops.EPI_SWIGLU, out=act)
            linear(act, lw.down_w, residual=h, epilogue=ops.EPI_BIAS_RESIDUAL, out=h)
        ops.rmsnorm(h, w.norm, d.rms_norm_eps, out=xn)
        if probe is not None and probe.hidden is not None:  # hidden_states[L]: the rows the lm_head GEMM reads
            ops.store_step_rows(xn, st["step"], probe.step_offset, probe.hidden[:, len(w.layers)])
        lg = st["logits"][:, :V]
        ops.gemm(xn, w.lm_head, out=lg)  # bf16 logits (modeling_llama.py:1044), arg max with the lowest index on ties
        if logits_only:  # beam search: the host picks the next tokens from the candidates of these logits
            return
        if sample:  # from the bf16 rows, or from the processed fp32 rows
            if proc:
                ops.logits_process(lg, st["out"], 1, B, st["step"], 0, self.proc_fparams, self.proc_spec, out=st["proc_rows"])
            ops.sample_rows(st["proc_rows"] if proc else lg, self._draw_params, st["seeds"], st["step"], 0, st["ids"], **self._scores_kw(scores))
        elif proc:  # the processors over each sequence's bf16 row and its history st["out"][t * B + b], t < step; then the arg max
            ops.logits_process(lg, st["out"], 1, B, st["step"], 0, self.proc_fparams, self.proc_spec, ids=st["ids"],
                               **({} if scores is None else {"out": st["proc_rows"]}))
            if scores is not None:
                ops.step_scores(st["proc_rows"], st["step"], 0, scores)
        else:
            ops.argmax_bf16(lg, out=st["ids"])
            if scores is not None:
                ops.step_scores(lg, st["step"], 0, scores)
        ops.decode_batch_advance(st["ids"], w.embed, h, st["out"], st["step"], st["pos"], st["ticket"])

    def _decode_batched(self, first: torch.Tensor, seq_lens: List[int], max_new_tokens: int, eos, stopping_fn, use_graph: bool,
                        proc: bool = False, sample_from: Optional[torch.Tensor] = None, seeds: Optional[List[int]] = None,
                        scores: Optional[torch.Tensor] = None, probe: Optional[ops.StepProbe] = None):
        """Decode of B prefilled sequences together: greedy, or sampled when ``sample_from`` holds the B first-token rows to draw from
        ([B, V], the bf16 lm_head rows or the processed fp32 rows) and ``seeds`` the B row seeds.  Returns a list of LongTensor [n_b]
        (each cut at its own stop).  ``scores`` ([T, B, V] fp32; a greedy caller has written row 0): every step's rows go to scores[step].
        A sequence that has stopped stays in the step, so its rows of the later steps hold what the step computed for it."""
        B = len(seq_lens)
        st = self._batch_state(B)
        sample = sample_from is not None
        if proc and st["proc_rows"] is None and (sample or scores is not None):
            st["proc_rows"] = torch.empty((B, self.dims.vocab_size), dtype=torch.float32, device=self.device)
        if sample:  # the first tokens in one launch, at counter 0
            st["seeds"].copy_(torch.tensor(seeds, dtype=torch.int64))
            st["step"].zero_()
            ops.sample_rows(sample_from, self._draw_params, st["seeds"], st["step"], 0, st["ids"], **self._scores_kw(scores))
            first = st["ids"]
        zero = torch.zeros(B, dtype=torch.int32, device=self.device)
        st["out"][:B].copy_(first)
        st["h"].copy_(ops.splice_rows(self.w.embed, None, None, None, zero, first.to(torch.int32)))
        st["pos"].copy_(torch.tensor(seq_lens, dtype=torch.int32))
        st["step"].fill_(1)
        # the graphs that write scores / probes hold the buffers' addresses
        key = GraphKey("batch", B, sample, proc, self._scores_key(scores), probe=None if probe is None else probe.key(),
                       warp=sample and self.warp)
        probe_kw = {} if probe is None else dict(probe=probe)
        if use_graph:  # with processing on, the processing kernel + key unpack replace the arg max (sampling: processing + draw)
            L = self.dims.num_hidden_layers
            self._capture(key, lambda: self._batch_step_launch(st, proc=proc, sample=sample, scores=scores, **probe_kw),
                          (st["h"], st["pos"], st["step"], st["out"]),
                          self._batch_kernels_per_layer * L + (5 if proc else 4) + (1 if scores is not None and not sample else 0) + (
                              0 if probe is None else probe.kernels(L, final_norm=False)))

        def launch(n: int) -> None:
            if use_graph:
                self._replay(key)
            else:
                self._batch_step_launch(st, proc=proc, sample=sample, scores=scores, **probe_kw)

        out2d = st["out"][: max_new_tokens * B].view(max_new_tokens, B)
        lens = self._run_steps(launch, out2d, [max_new_tokens] * B, eos, stopping_fn)
        res = out2d[:max(lens)].t().contiguous()
        return [res[b, :lens[b]].clone() for b in range(B)]

    # ---- batch-invariant decoding: up to SPEC_T_MAX sequences per weight pass, each bit-identical to its batch-1 generate_from_embeds --
    def _rows_state(self):
        """Buffers of the rows step (llama_decode_rows), sized for SPEC_T_MAX rows once, so a captured graph of B rows stays valid."""
        st = self._rstate
        if st is not None:
            return st
        d, dev, R = self.dims, self.device, ops.SPEC_T_MAX
        H, qd, I = d.hidden_size, d.num_attention_heads * d.head_dim, d.intermediate_size
        z = lambda *shape, dtype=self.dtype: torch.zeros(shape, dtype=dtype, device=dev)  # noqa: E731
        st = dict(h=z(R, H), q=z(R, qd), attn=z(R, qd), act=z(R, I), ws=z(R * self.lm_ws.numel(), dtype=torch.uint8),
                  logits=z(R, d.vocab_size, dtype=torch.float32), pos=z(R, dtype=torch.int32), step=z(1, dtype=torch.int32),
                  out=z(self.out_ids.numel() * R, dtype=torch.int64), seeds=z(R, dtype=torch.int64), ids=z(R, dtype=torch.int64))
        self._rstate = st
        return st

    def _guidance_state(self):
        """The rows state's buffers of classifier-free guidance, added on first use: the device scale g and the guided rows of up to
        SPEC_T_MAX / 2 prompts (a captured guided step holds their addresses)."""
        st = self._rows_state()
        if "guided" not in st:
            st["scale"] = torch.ones(1, dtype=torch.float32, device=self.device)
            st["guided"] = torch.empty((ops.SPEC_T_MAX // 2, self.dims.vocab_size), dtype=torch.float32, device=self.device)
        return st

    def _rows_step_launch(self, B: int, sample: bool, guided: bool = False) -> None:
        """The rows step over B rows; ``guided``: B = 2P rows, row P + b the unconditional branch of row b (llama_decode_rows' guidance)."""
        d, w, st = self.dims, self.w, self._rstate
        kw = dict(sample_params=self._draw_params, seeds=st["seeds"], ids=st["ids"]) if sample else {}
        if guided:
            kw.update(ids=st["ids"], guidance=(st["scale"], st["guided"]))
        ops.llama_decode_rows(st["h"][:B], self.stack, st["q"][:B], st["attn"][:B], st["act"][:B], B, d, self.cos, self.sin, st["pos"],
                              self.cache.page_tables, PAGE_SIZE, w.norm, w.lm_head, w.embed, st["ws"], st["out"], st["step"], st["logits"], **kw)

    @torch.no_grad()
    @ops.in_own_dtype
    def generate_rows(self, embeds_list: List[torch.Tensor], max_new_tokens, eos_token_ids=None, stopping_fn=None, use_graph: bool = True,
                      return_logits: bool = False, sampling=None, seeds: Optional[List[int]] = None, guidance_scale: Optional[float] = None,
                      negative_embeds: Optional[List[torch.Tensor]] = None):
        """Decode B <= SPEC_T_MAX prompts (embeddings [S_b, H] each) together, row b bit-identical to ``generate_from_embeds(embeds_list[b],
        max_new_tokens[b], ..., sampling=dict(sampling, seed=seeds[b]))``: each prompt is prefilled and gets its first token with the
        calls batch 1 makes, then every step runs the rows step (llama_decode_rows), which streams each weight once for all rows and
        gives each row the arithmetic of its one-token step.  ``max_new_tokens``: one budget, or one per row.  EOS and ``stopping_fn``
        are checked per row; a row that has stopped stays in the step and its results are ignored.  Returns a list of B LongTensors
        (and a list of B fp32 logits [n_b, V] when return_logits).
        ``negative_embeds`` (B <= SPEC_T_MAX / 2 embeddings [T_b, H]) with ``guidance_scale`` g: classifier-free guidance (HF's
        UnbatchedClassifierFreeGuidanceLogitsProcessor).  Prompt b's unconditional branch is its negative prompt, prefilled batch 1 into
        sequence B + b at positions from 0 and continued by the tokens chosen for prompt b; the 2B rows run the rows step, and each token is
        chosen (greedy arg max, or drawn with seeds[b]) from g * (log_softmax(c) - log_softmax(u)) + log_softmax(u) of the two rows'
        fp32 logits c and u (ops.guidance_rows).  The conditional rows keep their one-token arithmetic, so prompt b's ids and logits equal
        its guided call alone.  EOS and stopping_fn look at the conditional rows; the returned logits are their raw rows."""
        d, B = self.dims, len(embeds_list)
        guided = negative_embeds is not None
        if self.fp8:
            raise NotImplementedError("batch-invariant decoding has no FP8 form (the rows step is a 16-bit, packed or NF4 GEMV)")
        if guided and not 1 <= B <= ops.SPEC_T_MAX // 2:
            raise ValueError(f"guided generate_rows decodes 1 .. {ops.SPEC_T_MAX // 2} prompts at once (each with its unconditional row), got {B}")
        if guided and (len(negative_embeds) != B or guidance_scale is None or min(int(e.shape[0]) for e in negative_embeds) < 1):
            raise ValueError("guided generate_rows needs guidance_scale and one non-empty negative prompt per prompt")
        if not 1 <= B <= ops.SPEC_T_MAX:
            raise ValueError(f"generate_rows decodes 1 .. {ops.SPEC_T_MAX} prompts at once, got {B}")
        budgets = [int(max_new_tokens)] * B if isinstance(max_new_tokens, int) else [int(m) for m in max_new_tokens]
        if len(budgets) != B or min(budgets) < 1:
            raise ValueError("generate_rows needs one budget of at least 1 token per prompt")
        sample = bool(sampling)
        if sample and (seeds is None or len(seeds) != B):
            raise ValueError("sampled generate_rows needs one seed per prompt")
        lens, mx = [int(e.shape[0]) for e in embeds_list], max(budgets)
        R = 2 * B if guided else B  # rows of the step
        eos = eos_list(eos_token_ids)
        self._start_request(lens + ([int(e.shape[0]) for e in negative_embeds] if guided else []), mx)
        self._set_sampling(sampling)
        st = self._guidance_state() if guided else self._rows_state()
        logits = [torch.empty((mx, d.vocab_size), dtype=torch.float32, device=self.device) for _ in range(B)] if return_logits else None
        if guided:  # each prompt and each negative prompt prefilled batch 1; the first token of a pair from its two last rows
            for r, emb in enumerate(list(embeds_list) + list(negative_embeds)):
                self._prefill_first_token(emb, r, 0, st["logits"][r], False, False, None)
            if logits is not None:
                for b in range(B):
                    logits[b][0].copy_(st["logits"][b])
            st["scale"].fill_(float(guidance_scale))
            st["step"].zero_()  # a draw of the first token uses counter 0, as batch 1's
            if sample:
                st["seeds"][:B].copy_(torch.tensor([int(s) & SEED_MASK for s in seeds], dtype=torch.int64))
            ids = st["ids"][:R]
            ops.guidance_rows(st["logits"][:R], st["scale"], st["guided"][:B], ids=None if sample else ids)
            if sample:
                ops.sample_rows(st["guided"][:B], self._draw_params, st["seeds"][:B], st["step"], 0, st["ids"][:B])
                ops.guidance_pair_ids(ids, B)
            st["out"][:R].copy_(ids)
            st["h"][:R].copy_(ops.splice_rows(self.w.embed, None, None, None, torch.zeros(R, dtype=torch.int32, device=self.device),
                                              ids.to(torch.int32)))
            st["pos"][:R].copy_(torch.tensor(lens + [int(e.shape[0]) for e in negative_embeds], dtype=torch.int32))
        else:
            for b, emb in enumerate(embeds_list):  # generate_from_embeds' prefill and first token, into sequence b
                if sample:
                    self._set_seed(int(seeds[b]))
                self._prefill_first_token(emb, b, 0, None if logits is None else logits[b][0], sample, False, None)
                st["out"][b:b + 1].copy_(self.out_ids[:1])
                st["h"][b].copy_(self.h)
            st["pos"][:B].copy_(torch.tensor(lens, dtype=torch.int32))
        st["step"].fill_(1)
        if sample and not guided:
            st["seeds"][:B].copy_(torch.tensor([int(s) & SEED_MASK for s in seeds], dtype=torch.int64))
        key = GraphKey("guided" if guided else "rows", B, sample, warp=sample and self.warp)
        graph = use_graph and logits is None
        if graph:
            self._capture(key, lambda: self._rows_step_launch(R, sample, guided), (st["h"], st["pos"], st["step"], st["out"]),
                          self.stack.rows_kernels + ((3 if sample else 1) if guided else (1 if sample else 0)))

        def launch(n: int) -> None:
            if graph:
                self._replay(key)
                return
            self._rows_step_launch(R, sample, guided)
            if logits is not None:
                for b in range(B):
                    logits[b][n].copy_(st["logits"][b])

        out2d = st["out"][: mx * R].view(mx, R)[:, :B]  # the conditional rows; an unconditional row repeats its prompt's tokens
        lens_out = self._run_steps(launch, out2d, budgets, eos, stopping_fn)
        res = out2d[:max(lens_out)].t().contiguous()
        outs = [res[b, :lens_out[b]].clone() for b in range(B)]
        if logits is not None:
            return outs, [logits[b][:lens_out[b]] for b in range(B)]
        return outs

    @torch.no_grad()
    @ops.in_own_dtype
    def generate_beam(self, inputs_embeds: torch.Tensor, num_beams: int, max_new_tokens: int, eos_token_ids=None, stopping_fn=None,
                      length_penalty: float = 1.0, early_stopping: bool = False, use_graph: bool = True, output_scores: bool = False):
        """Beam search from prompt embeddings [S, H] (HF GenerationMixin.beam_search + BeamSearchScorer behind llava_llama.py:212 when
        the eval scripts pass --num_beams > 1; restated by the CPU checker of the test suite (beam_search_generate), which is pinned to HF's own
        generate()).  Device side: the prompt is prefilled once per beam as one packed batch (HF expands the inputs the same way), every
        step runs the batched decode layers over the num_beams rows, a kernel reduces each row's logits to its 2 x num_beams best
        (log-prob + beam score, token) pairs, and the surviving beams' KV rows are re-ordered page-wise.  Host side: the hypothesis
        bookkeeping on the num_beams x 2 num_beams candidates - the same control logic HF runs in Python.  Returns the NEW ids.
        ``output_scores``: returns (ids, extra) with extra = _beam_extra's dict: every step's log_softmax rows [steps, num_beams, V]
        (HF's output_scores of beam search, written by the candidates kernel), the best hypothesis' score and the beam row of each of
        its tokens."""
        d, w, k = self.dims, self.w, int(num_beams)
        S, V = inputs_embeds.shape[0], d.vocab_size
        if k < 2:
            raise ValueError("generate_beam needs num_beams >= 2")
        if max_new_tokens < 1:
            empty = torch.empty(0, dtype=torch.int64, device=self.device)
            return (empty, self._beam_extra(None, 0, [])) if output_scores else empty
        eos = eos_list(eos_token_ids)
        n_cand = max(2, 1 + len(eos)) * k
        self._start_request([S] * k, max_new_tokens, writes_ids=False)
        hidden = self.prefill_packed(inputs_embeds.to(self.dtype).repeat(k, 1), [S] * k)
        _, lg = self.first_tokens(hidden, [S] * k, return_logits=True)
        st = self._batch_state(k)
        st["logits"][:, :V].copy_(lg)
        dev = self.device
        hyp = BeamHypotheses(k, eos, length_penalty, early_stopping)
        d_scores = torch.tensor(hyp.scores, dtype=torch.float32).to(dev)
        cand_s = torch.empty((k, n_cand), dtype=torch.float32, device=dev)
        cand_t = torch.empty((k, n_cand), dtype=torch.int32, device=dev)
        h_s = torch.empty((k, n_cand), dtype=torch.float32, pin_memory=True)
        h_t = torch.empty((k, n_cand), dtype=torch.int32, pin_memory=True)
        zero = torch.zeros(k, dtype=torch.int32, device=dev)
        tables = [list(self.cache.owned[b]) for b in range(k)]  # page ids by position // PAGE_SIZE
        pages_all = self.cache.pages
        rows_out = self._scores_view(max_new_tokens, k) if output_scores else None

        for step in range(max_new_tokens):
            ops.beam_candidates(st["logits"][:, :V], d_scores, cand_s, cand_t, **self._logprobs_kw(rows_out, step))
            h_s.copy_(cand_s, non_blocking=True)
            h_t.copy_(cand_t, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            # merge the per-beam candidates: (score desc, beam asc, token asc) = the flat-index order of HF's topk on ties
            flat = sorted(((-float(h_s[b, j]), b, int(h_t[b, j])) for b in range(k) for j in range(n_cand) if int(h_t[b, j]) >= 0))[:n_cand]
            parents = hyp.advance([(-neg, b, t) for neg, b, t in flat], step + 1)
            if hyp.done or step == max_new_tokens - 1:
                break
            if stopping_fn is not None and all(stopping_fn(torch.tensor(q, dtype=torch.int64)) for q in hyp.seqs):
                break  # KeywordsStoppingCriteria.__call__ requires every row (beam) to have hit (mm_utils.py:616-617)
            # ---- device state of the next step: KV rows of the generated region follow their parents (HF _reorder_cache,
            #      modeling_llama.py:1151-1158, copies the WHOLE cache; here only the pages that hold generated tokens)
            if step > 0 and any(p != i for i, p in enumerate(parents)):
                j0, j1 = S // PAGE_SIZE, (S + step - 1) // PAGE_SIZE
                src = [tables[p][j] for i, p in enumerate(parents) if p != i for j in range(j0, j1 + 1)]
                dst = [tables[i][j] for i, p in enumerate(parents) if p != i for j in range(j0, j1 + 1)]
                src_t = torch.tensor(src, dtype=torch.int64).to(dev)
                dst_t = torch.tensor(dst, dtype=torch.int64).to(dev)
                pages_all[:, dst_t] = pages_all[:, src_t]  # gather into a temporary, then scatter: permutations are safe
            ids = torch.tensor([q[-1] for q in hyp.seqs], dtype=torch.int32).to(dev)
            st["h"].copy_(ops.splice_rows(w.embed, None, None, None, zero, ids))
            st["pos"].fill_(S + step)
            d_scores.copy_(torch.tensor(hyp.scores, dtype=torch.float32), non_blocking=True)
            if use_graph:  # the warm-up before the capture rewrites only this step's own KV rows
                self._capture(GraphKey("beam", k), lambda: self._batch_step_launch(st, logits_only=True), (st["h"],), self._batch_kernels_per_layer * d.num_hidden_layers + 2)
                self._replay(GraphKey("beam", k))
            else:
                self._batch_step_launch(st, logits_only=True)
        best = torch.tensor(hyp.best(max_new_tokens), dtype=torch.int64, device=dev)
        return (best, self._beam_extra(rows_out, step + 1, [hyp])) if output_scores else best

    # ---- contrastive search: B prompts x k candidates per step in the batched step, the choice made on the device ----------------
    def _contrastive_state(self, B: int, k: int, L_cap: int):
        """The batched step's buffers of B * k rows and contrastive search's own: each prompt's context rows ctx [B, L_cap, H], its
        next-logits row, the candidates, the penalty's chunk maxima and the choice.  A captured step holds their addresses, so they are
        replaced (and the contrastive graphs dropped) only when (B, k) changes or a request needs a longer context."""
        st = self._batch_state(B * k)
        cs = st.get("contrastive")
        if cs is not None and (cs["B"], cs["k"]) == (B, k) and cs["L_cap"] >= L_cap:
            return st, cs
        self._drop_graphs(lambda key: key.kind == "contrastive")
        st["contrastive"] = None
        d, dev = self.dims, self.device
        L_cap = min((L_cap + 127) // 128 * 128, self.max_seq_len)  # a little slack, so nearby request lengths share the graph
        V = d.vocab_size
        cs = dict(B=B, k=k, L_cap=L_cap, ctx=torch.zeros((B, L_cap, d.hidden_size), dtype=self.dtype, device=dev),
                  next=torch.zeros((B, (V + 7) // 8 * 8), dtype=self.dtype, device=dev)[:, :V],
                  zero=torch.zeros(B, dtype=torch.float32, device=dev), cand_s=torch.zeros((B, k), dtype=torch.float32, device=dev),
                  cand_t=torch.zeros((B, k), dtype=torch.int32, device=dev), src_id=torch.zeros(B * k, dtype=torch.int32, device=dev),
                  partial=ops.contrastive_partial(B, k, L_cap, dev), alpha=torch.zeros(2, dtype=torch.float32, device=dev),
                  sel=torch.zeros(B, dtype=torch.int32, device=dev), pen=torch.zeros((B, k), dtype=torch.float32, device=dev),
                  score=torch.zeros((B, k), dtype=torch.float32, device=dev))
        st["contrastive"] = cs
        return st, cs

    def _contrastive_step_launch(self, st, cs, scores: Optional[torch.Tensor] = None) -> None:
        """One contrastive step: (the next-logits rows to scores[step]), their k candidates each, the B * k candidate tokens through the
        batched step, the degeneration penalty, the choice, and the chosen row's K / V at the new position copied into its siblings."""
        k, V = cs["k"], self.dims.vocab_size
        if scores is not None:
            ops.step_scores(cs["next"], st["step"], 0, scores)
        ops.beam_candidates(cs["next"], cs["zero"], cs["cand_s"], cs["cand_t"])
        ops.splice_rows(self.w.embed, None, None, None, cs["src_id"], cs["cand_t"].view(-1), out=st["h"])
        self._batch_step_launch(st, logits_only=True)
        ops.contrastive_penalty(st["xn"], cs["ctx"], st["pos"], k, cs["partial"])
        ops.contrastive_select(cs["cand_s"], cs["cand_t"], cs["partial"], cs["alpha"], st["xn"], st["logits"][:, :V], cs["ctx"], cs["next"],
                               st["pos"], st["out"], st["step"], st["ticket"], cs["sel"], cs["pen"], cs["score"])
        ops.kv_broadcast_rows(self.cache.pages, self.cache.page_tables, st["pos"], -1, cs["sel"], k)

    @torch.no_grad()
    @ops.in_own_dtype
    def generate_contrastive(self, packed_embeds: torch.Tensor, seq_lens: List[int], top_k: int, penalty_alpha: float, max_new_tokens: int,
                             eos_token_ids=None, stopping_fn=None, use_graph: bool = True, output_scores: bool = False):
        """Contrastive search (HF GenerationMixin.contrastive_search + _ranking_fast, transformers 4.37.2) over B prompts packed back to
        back ([sum S_b, H]).  Row g * k + i of every step is candidate i of prompt g: ONE packed prefill into row g * k (B = 1: batch 1's
        prefill and lm_head, so the first logits row is greedy generate()'s), the prompt pages copied into the other k - 1 rows, every
        prompt row's final norm into its context (HF's last_hidden_states), lm_head on the last row into its next-logits row.  Then each
        token is one step (one graph replay): the k most probable tokens of the next-logits row (beam_candidates), all B * k of them
        through the batched step, pen = the largest cosine of each candidate's final-norm row against the prompt's context, score =
        (1 - alpha) * p - alpha * pen, the best candidate emitted (lowest index on ties), its row appended to the context, its logits
        row the next one, and its K / V at the new position copied into its siblings, so the k rows' histories stay identical.
        EOS and ``stopping_fn`` are checked per prompt; a prompt that has stopped keeps its rows in the step.  Returns a list of B
        LongTensors of new ids; ``output_scores``: (ids, {"scores": fp32 [n_max, B, V]}), scores[t, g] the next-logits row token t of
        prompt g was chosen from (widened exactly).  HF pads a batch on the left and its pad rows join the context; packed prompts have
        no pad rows, so the context is the prompt's own rows (the same for batch 1 and unpadded batches)."""
        d, w, k, B = self.dims, self.w, int(top_k), len(seq_lens)
        V, R, dev = d.vocab_size, B * int(top_k), self.device
        seq_lens = [int(n) for n in seq_lens]
        alpha = float(penalty_alpha)
        if not 2 <= k <= 64:
            raise ValueError(f"generate_contrastive needs 2 <= top_k <= 64, got {k}")
        if not 0.0 <= alpha <= 1.0:
            raise ValueError(f"generate_contrastive needs 0 <= penalty_alpha <= 1, got {penalty_alpha}")
        if B < 1 or packed_embeds.shape[0] != sum(seq_lens) or min(seq_lens) < 1:
            raise RuntimeError("generate_contrastive: rows do not match seq_lens")
        if max_new_tokens < 1:
            empty = [torch.empty(0, dtype=torch.int64, device=dev) for _ in range(B)]
            return (empty, {"scores": torch.empty((0, B, V), dtype=torch.float32, device=dev)}) if output_scores else empty
        eos = eos_list(eos_token_ids)
        starts = [n for n in seq_lens for _ in range(k)]  # row g * k + i: the first generated position of prompt g
        self._start_request(starts, max_new_tokens)
        tables = [list(self.cache.owned[r]) for r in range(R)]
        st, cs = self._contrastive_state(B, k, max(seq_lens) + max_new_tokens)
        ctx, nxt = cs["ctx"], cs["next"]
        if B == 1:
            first = self._sample_buffer()
            hidden = self._prefill_first_token(packed_embeds, 0, 0, first, False, False, None)
            nxt[0].copy_(first)  # lm_head_argmax's fp32 row holds element-type values: exact
        else:
            hidden = self.prefill_packed(packed_embeds, seq_lens, page_tables=self.cache.page_tables[:R:k])
        ops.kv_copy_pages(self.cache.pages, prompt_page_pairs(tables, seq_lens, k))
        off = 0
        for g, n in enumerate(seq_lens):
            ops.rmsnorm(hidden[off:off + n], w.norm, d.rms_norm_eps, out=ctx[g, :n])
            off += n
        if B > 1:  # the last prompt rows' final norm is in the context already
            last = torch.tensor([g * cs["L_cap"] + n - 1 for g, n in enumerate(seq_lens)], dtype=torch.int32).to(dev)
            rows = ops.splice_rows(ctx.view(-1, d.hidden_size), None, None, None, torch.zeros_like(last), last)
            ops.gemm(rows, w.lm_head, out=nxt)
        cs["alpha"].copy_(torch.tensor([1.0 - alpha, alpha], dtype=torch.float64).float())
        st["pos"].copy_(torch.tensor(starts, dtype=torch.int32))
        st["step"].zero_()
        scores = self._scores_view(max_new_tokens, B) if output_scores else None
        key = GraphKey("contrastive", R, scores=self._scores_key(scores), group=k)
        if use_graph:  # the warm-up before the capture writes only this step's own rows, which the first replay writes again
            self._capture(key, lambda: self._contrastive_step_launch(st, cs, scores), (st["pos"], st["step"], nxt),
                          self._batch_kernels_per_layer * d.num_hidden_layers + 7 + (1 if scores is not None else 0))

        def launch(n: int) -> None:
            if use_graph:
                self._replay(key)
            else:
                self._contrastive_step_launch(st, cs, scores)

        launch(0)  # token 0 needs a step of its own: the prefill gave only the row its candidates come from
        out2d = st["out"][: max_new_tokens * B].view(max_new_tokens, B)
        lens = self._run_steps(launch, out2d, [max_new_tokens] * B, eos, stopping_fn)
        res = out2d[:max(lens)].t().contiguous()
        outs = [res[b, :lens[b]].clone() for b in range(B)]
        return (outs, {"scores": scores[:max(lens)].clone()}) if output_scores else outs

    @staticmethod
    def _logprobs_kw(rows_out: Optional[torch.Tensor], step: int) -> dict:
        """beam_candidates' keyword for the step's log_softmax rows; none without output_scores, so the call is today's."""
        return {} if rows_out is None else {"logprobs": rows_out[step]}

    def _beam_extra(self, scores: Optional[torch.Tensor], steps: int, groups: List[BeamHypotheses]) -> dict:
        """What a beam search returns with output_scores: scores fp32 [steps, rows, V] (each step's log_softmax rows), and per prompt
        sequence_score (its best hypothesis' score, HF's sequences_scores) and beam_indices (the beam row, counted over all prompts'
        rows, of each token of that hypothesis; HF's beam_indices before padding)."""
        sc = torch.empty((0, 0, self.dims.vocab_size), dtype=torch.float32, device=self.device) if scores is None else scores[:steps].clone()
        return {"scores": sc, "sequence_scores": [g.best_score for g in groups], "beam_indices": [g.best_beams for g in groups]}

    @torch.no_grad()
    @ops.in_own_dtype
    def generate_beam_batch(self, packed_embeds: torch.Tensor, seq_lens: List[int], num_beams: int, max_new_tokens: int, eos_token_ids=None,
                            stopping_fn=None, length_penalty: float = 1.0, early_stopping: bool = False, use_graph: bool = True,
                            output_scores: bool = False, num_beam_groups: int = 1, diversity_penalty: float = 0.0,
                            pad_token_id: Optional[int] = None):
        """Beam search over B prompts packed back to back ([sum S_b, H]) at once (HF beam_search + BeamSearchScorer with batch_size = B).
        Row g * k + i of every step is beam i of prompt g, so one batched decode step serves all B * k beams.  Device side: ONE packed
        prefill of the B prompts, their pages copied into the other k - 1 beams of each (kv_copy_pages), then per step the candidates
        kernel over all rows, the per-prompt merge (beam_select) whose B x n_cand results reach the host through pinned memory, and the
        copy of the generated KV rows of every beam whose parent is another beam.  Host side: one BeamHypotheses per prompt.  A prompt
        that is done keeps its rows in the step (the graph shape stays fixed) and its choices are ignored.  The loop ends when every
        prompt is done, at max_new_tokens, or when ``stopping_fn`` holds for every beam of the prompts still running.  Returns a list
        of B LongTensors of NEW ids, each prompt's best hypothesis.  ``output_scores``: returns (ids, extra) as generate_beam, the score
        rows [steps, B * k, V] in the step's row order (row g * k + i = beam i of prompt g).  A prompt that is done keeps its rows in the
        step, so its rows of the later steps hold what the step computed for them.
        ``num_beam_groups`` G > 1 with ``diversity_penalty`` > 0: diverse beam search (HF group_beam_search, transformers 4.37.2), B = 1
        included.  Beam i of a prompt belongs to group i // (k / G); each (prompt, group) has its own BeamHypotheses, and one kernel
        per step (beam_group_select) takes every prompt's groups in order, each penalised by diversity_penalty per earlier choice of a
        token in this step, and makes HF's choice on the device; the host replays it from the ranked candidates.  A done group emits
        ``pad_token_id`` (default: the first EOS id), which still counts for the later groups; the answer is the best hypothesis over all
        groups (group_best).  Not with output_scores."""
        d, w, k, B = self.dims, self.w, int(num_beams), len(seq_lens)
        V, R, dev = d.vocab_size, B * int(num_beams), self.device
        seq_lens = [int(n) for n in seq_lens]
        G = int(num_beam_groups)
        if k < 2:
            raise ValueError("generate_beam_batch needs num_beams >= 2")
        if G != 1:
            if G < 1 or G > k or k % G:
                raise ValueError(f"num_beams ({k}) must be divisible by num_beam_groups ({G}), and num_beam_groups at most num_beams")
            if not float(diversity_penalty) > 0.0:
                raise ValueError(f"diverse beam search needs diversity_penalty > 0, got {diversity_penalty}")
            if output_scores:
                raise NotImplementedError("output_scores with num_beam_groups > 1")
        if B < 1 or packed_embeds.shape[0] != sum(seq_lens) or min(seq_lens) < 1:
            raise RuntimeError("generate_beam_batch: rows do not match seq_lens")
        if max_new_tokens < 1:
            empty = [torch.empty(0, dtype=torch.int64, device=dev) for _ in range(B)]
            return (empty, self._beam_extra(None, 0, [])) if output_scores else empty
        eos = eos_list(eos_token_ids)
        gs = k // G  # the beams of a group
        n_cand = max(2, 1 + len(eos)) * gs
        starts = [n for n in seq_lens for _ in range(k)]  # row r = g * k + i: the first generated position of its prompt
        self._start_request(starts, max_new_tokens, writes_ids=False)
        tables = [list(self.cache.owned[r]) for r in range(R)]
        # the prompts are prefilled once, into beam 0 of each; the other beams get copies of its prompt rows
        hidden = self.prefill_packed(packed_embeds, seq_lens, page_tables=self.cache.page_tables[:R:k])
        ops.kv_copy_pages(self.cache.pages, prompt_page_pairs(tables, seq_lens, k))
        st = self._batch_state(R)
        # every beam row starts from its prompt's last hidden row: final norm + lm_head over the R rows
        last = torch.tensor([sum(seq_lens[:g + 1]) - 1 for g in range(B) for _ in range(k)], dtype=torch.int32).to(dev)
        rows = ops.splice_rows(hidden, None, None, None, torch.zeros_like(last), last)
        ops.rmsnorm(rows, w.norm, d.rms_norm_eps, out=st["xn"])
        ops.gemm(st["xn"], w.lm_head, out=st["logits"][:, :V])
        # group q = prompt * G + its group owns rows q * gs .. q * gs + gs - 1; G = 1: one per prompt
        groups = [BeamHypotheses(gs, eos, length_penalty, early_stopping, row0=q * gs) for q in range(B * G)]
        rows_out = self._scores_view(max_new_tokens, R) if output_scores else None
        d_scores = torch.tensor([s for grp in groups for s in grp.scores], dtype=torch.float32).to(dev)
        # G > 1: each row's list must outlast the k - gs tokens the earlier groups may penalise (srgpt_beam_group_select)
        n_list = n_cand if G == 1 else min(n_cand + k - gs, V)
        cand_s = torch.empty((R, n_list), dtype=torch.float32, device=dev)
        cand_t = torch.empty((R, n_list), dtype=torch.int32, device=dev)
        n_sel = 3 * B * G * n_cand
        # the merge's scores (as bits), beams, tokens (G > 1: then each beam's parent and token): one copy to the host
        sel_all = torch.empty(n_sel + (2 * R if G > 1 else 0), dtype=torch.int32, device=dev)
        sel = sel_all[:n_sel].view(3, B * G, n_cand)
        h_all = torch.empty(sel_all.shape, dtype=torch.int32, pin_memory=True)
        h_sel = h_all[:n_sel].view(3, B * G, n_cand)
        h_scores = h_sel[0].view(torch.float32)
        if G > 1:
            stats = torch.empty((R, 2), dtype=torch.float32, device=dev)
            d_eos = torch.tensor(eos, dtype=torch.int32).to(dev)
            d_done = torch.zeros((B, G), dtype=torch.int32, device=dev)
            pad = pad_token_id if pad_token_id is not None else (eos[0] if eos else 0)
            nxt = sel_all[n_sel:].view(2, R)
        zero = torch.zeros(R, dtype=torch.int32, device=dev)
        tokens = [0] * R  # the token each row feeds to the next step (a done prompt's rows repeat theirs)
        for step in range(max_new_tokens):
            if G == 1:
                ops.beam_candidates(st["logits"][:, :V], d_scores, cand_s, cand_t, **self._logprobs_kw(rows_out, step))
                ops.beam_select(cand_s, cand_t, k, sel[0].view(torch.float32), sel[1], sel[2])
            else:
                ops.beam_candidates_scored(st["logits"][:, :V], d_scores, cand_s, cand_t, stats)
                ops.beam_group_select(st["logits"][:, :V], stats, d_scores, cand_t, k, G, d_eos, pad, diversity_penalty, d_done,
                                      sel[0].view(torch.float32).view(B, G, n_cand), sel[1].view(B, G, n_cand), sel[2].view(B, G, n_cand),
                                      nxt[0], nxt[1])
            h_all.copy_(sel_all, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            scores, beams, toks = h_scores.tolist(), h_sel[1].tolist(), h_sel[2].tolist()
            chosen = h_all[n_sel:].view(2, R).tolist() if G > 1 else None
            parents = list(range(R))
            for q, grp in enumerate(groups):
                if grp.done:
                    continue
                ranked = [(scores[q][j], beams[q][j], toks[q][j]) for j in range(n_cand) if toks[q][j] >= 0]
                for i, b in enumerate(grp.advance(ranked, step + 1)):
                    parents[q * gs + i] = q * gs + b
                    tokens[q * gs + i] = grp.seqs[i][-1]
                    if G > 1 and (chosen[0][q * gs + i] + q // G * k, chosen[1][q * gs + i]) != (q * gs + b, tokens[q * gs + i]):
                        raise RuntimeError(f"beam_group_select chose beam {chosen[0][q * gs + i]} / token {chosen[1][q * gs + i]} where "
                                           f"BeamSearchScorer.process takes {q * gs + b - q // G * k} / {tokens[q * gs + i]}")
            if all(grp.done for grp in groups) or step == max_new_tokens - 1:
                break
            if stopping_fn is not None and all(stopping_fn(torch.tensor(q, dtype=torch.int64)) for grp in groups if not grp.done for q in grp.seqs):
                break  # HF evaluates the criterion over the whole expanded batch; the rows of a finished prompt no longer matter
            # the generated KV rows [S_g, S_g + step) follow their parents (the prompt rows are the same in every beam of a prompt)
            pairs, n_staged = beam_page_pairs(tables, parents, starts, step)
            ops.kv_copy_pages(self.cache.pages, pairs, n_staged)
            st["h"].copy_(ops.splice_rows(w.embed, None, None, None, zero, torch.tensor(tokens, dtype=torch.int32).to(dev)))
            st["pos"].copy_(torch.tensor([n + step for n in starts], dtype=torch.int32))
            d_scores.copy_(torch.tensor([s for grp in groups for s in grp.scores], dtype=torch.float32))
            if G > 1:
                d_done.copy_(torch.tensor([grp.done for grp in groups], dtype=torch.int32).view(B, G))
            if use_graph:  # keyed by the row count, as generate_beam's graph: the same launch over the same buffers
                self._capture(GraphKey("beam", R), lambda: self._batch_step_launch(st, logits_only=True), (st["h"],),
                              self._batch_kernels_per_layer * d.num_hidden_layers + 2)
                self._replay(GraphKey("beam", R))
            else:
                self._batch_step_launch(st, logits_only=True)
        if G == 1:
            outs = [torch.tensor(grp.best(max_new_tokens), dtype=torch.int64, device=dev) for grp in groups]
        else:
            outs = [torch.tensor(group_best(groups[b * G:(b + 1) * G], max_new_tokens), dtype=torch.int64, device=dev) for b in range(B)]
        return (outs, self._beam_extra(rows_out, step + 1, groups)) if output_scores else outs

    @torch.no_grad()
    @ops.in_own_dtype
    def generate_batch(self, packed_embeds: torch.Tensor, seq_lens: List[int], max_new_tokens: int, eos_token_ids=None,
                       stopping_fn=None, use_graph: bool = True, return_logits: bool = False, sampling=None, processors=None,
                       num_return_sequences: int = 1, output_scores: bool = False, outputs: Optional[GenerateProbe] = None):
        """Decoding of B prompts: ONE packed prefill pass (tensor-core bound, all prompts share every GEMM), one lm_head GEMM for the
        B first tokens, then BATCHED decode: every step advances all B sequences, each weight streamed once per step for the
        whole batch (_decode_batched), greedy or sampled (``sampling``: sequence b draws with sequence_seeds(seed, B)[b]).  With
        ``return_logits`` the sequences are decoded one after the other with the single-sequence weight-streaming step.  Returns a
        list of LongTensor [n_b] (and a list of fp32 logits).
        ``processors``: the logits processors of generate_from_embeds, on every path (the first tokens included).
        ``num_return_sequences=n`` (sampling only): n answers per prompt.  Each prompt is prefilled once, into row b * n; its prompt
        pages are copied into rows b * n + 1 .. b * n + n - 1, and the B * n rows decode in the batched sampled step, row r with
        sequence_seeds(seed, B * n)[r].  Returns B * n lists, row b * n + j being answer j of prompt b.
        ``output_scores``: returns (what it returns without, {"scores": fp32 [n_max, B * n, V]}), scores[t, r] being the row token t of
        row r was chosen from (generate_from_embeds) and n_max the longest row's length.  In the batched step a row that has stopped
        keeps its place, so its later steps hold what the step computed for it; the one-after-the-other path (return_logits) leaves
        them 0.
        ``outputs`` (GenerateProbe of B rows; B > 1, no return_logits, num_return_sequences 1): the packed prefill records the prompt step
        and the batched step every decode step; ids and scores are unchanged."""
        n_ret = int(num_return_sequences)
        if outputs is not None and (return_logits or n_ret != 1 or len(seq_lens) < 2):
            raise NotImplementedError("hidden states / attentions of generate_batch need B > 1 prompts without output_logits or "
                                      "num_return_sequences > 1")
        if n_ret < 1:
            raise ValueError(f"num_return_sequences must be >= 1, got {n_ret}")
        if n_ret > 1:
            if not sampling:
                raise ValueError("num_return_sequences > 1 needs sampling: greedy decoding has one answer per prompt")
            if return_logits:
                raise NotImplementedError("num_return_sequences > 1 with output_logits")
            if not self.supports_batch_sampling:
                raise NotImplementedError("num_return_sequences > 1 on the tensor-parallel decoder (it does not sample)")
        d, w = self.dims, self.w
        B = len(seq_lens) * n_ret
        if max_new_tokens < 1:
            empty = [torch.empty(0, dtype=torch.int64, device=self.device) for _ in range(B)]
            return (empty, {"scores": torch.empty((0, B, d.vocab_size), dtype=torch.float32, device=self.device)}) if output_scores else empty
        eos = eos_list(eos_token_ids)
        proc = self._set_processors(processors)
        row_lens = [int(n) for n in seq_lens for _ in range(n_ret)]  # row b * n_ret + j continues prompt b
        self._start_request(row_lens, max_new_tokens)
        if outputs is not None:
            hidden = self.prefill_packed(packed_embeds, seq_lens, probe=outputs.prefill)
            outputs.record_final(self, hidden, [int(n) for n in seq_lens])
        elif n_ret == 1:
            hidden = self.prefill_packed(packed_embeds, seq_lens)
        else:  # each prompt once, into the first of its rows; the other rows get copies of its prompt pages
            tables = [list(self.cache.owned[r]) for r in range(B)]
            hidden = self.prefill_packed(packed_embeds, seq_lens, page_tables=self.cache.page_tables[:B:n_ret])
            ops.kv_copy_pages(self.cache.pages, prompt_page_pairs(tables, [int(n) for n in seq_lens], n_ret))
        first, lg = self.first_tokens(hidden, seq_lens, return_logits=True, repeat=n_ret)
        seq_lens = row_lens
        outs, all_logits = [], []
        sample = self._set_sampling(sampling)
        scores = self._scores_view(max_new_tokens, B) if output_scores else None
        zero = torch.zeros(1, dtype=torch.int32, device=self.device)
        first_rows = None  # the processed first-token rows a sampled sequence draws from
        if proc:  # the first tokens with an empty history: only the minimum length and single-token bad words act
            first_rows = torch.empty((B, d.vocab_size), dtype=torch.float32, device=self.device) if sample or output_scores else None
            ops.logits_process(lg, None, 0, 1, None, 0, self.proc_fparams, self.proc_spec, out=first_rows, ids=first)
        if scores is not None and not sample:  # the rows the greedy first tokens were chosen from (a sampler writes its own)
            ops.step_scores(first_rows if proc else lg, zero, 0, scores)
        if max_new_tokens == 1 and not return_logits and not sample:
            outs = [first[b:b + 1] for b in range(B)]
            return (outs, {"scores": scores[:1].clone()}) if output_scores else outs
        seeds = sequence_seeds(self.sample_seed, B) if sample else None
        if not return_logits and B > 1 and (not sample or self.supports_batch_sampling):
            outs = self._decode_batched(first, seq_lens, max_new_tokens, eos, stopping_fn, use_graph, proc,
                                        sample_from=(first_rows if proc else lg) if sample else None, seeds=seeds, scores=scores,
                                        **({} if outputs is None or outputs.steps is None else dict(probe=outputs.steps)))
            return (outs, {"scores": scores[:max(o.numel() for o in outs)].clone()}) if output_scores else outs
        if scores is not None and B > 1:  # one row after the other: a row's steps past its stop are never written
            scores.view(max_new_tokens, B * d.vocab_size)[1 if not sample else 0:].zero_()
        for b in range(B):
            col = None if scores is None else scores[:, b:b + 1]  # sequence b's rows: [T, 1, V] with a step stride of B * V
            logits = None
            if return_logits:
                logits = torch.empty((max_new_tokens, d.vocab_size), dtype=torch.float32, device=self.device)
                logits[0].copy_(lg[b])
            # decode state of sequence b: token 0 is known, the next step processes it at position S_b
            self.out_ids[0:1].copy_(first[b:b + 1])
            self.h.copy_(ops.splice_rows(w.embed, None, None, None, zero, first[b:b + 1].to(torch.int32))[0])
            self.pos.fill_(seq_lens[b])
            self.step.fill_(1)
            if sample:  # re-draw the first token of this sequence from its logits row (a different draw per sequence: the seed moves)
                self._set_seed(seeds[b])
                row = first_rows[b] if proc else lg[b].float().contiguous()
                ops.sample_top_p(row, self._draw_params, self.sample_seed_dev, self.step, -1, self.out_ids, w.embed, self.h,
                                 **self._scores_kw(col, True))
            r = self._decode_loop(b, max_new_tokens, eos, stopping_fn, use_graph, logits, sample, proc, col)
            if return_logits:
                outs.append(r[0]); all_logits.append(r[1])
            else:
                outs.append(r)
        r = (outs, all_logits) if return_logits else outs
        return (r, {"scores": scores[:max(o.numel() for o in outs)].clone()}) if output_scores else r

    # ---- likelihood scoring: every candidate continues its prompt from the prompt's own KV pages ------------------------------------
    supports_scoring = True

    @torch.no_grad()
    @ops.in_own_dtype
    def score_candidates(self, packed_embeds: torch.Tensor, seq_lens: List[int], candidates, row_budget: int) -> torch.Tensor:
        """log p(cand_c[j] | prompt_b ++ cand_c[:j]) for B prompts packed back to back ([sum S_b, H]) and N candidate token lists shared by
        every prompt -> fp32 [B, N, L_max], 0 past each candidate's length.
        1. ONE packed prefill of the prompts into slots 0..B-1; final norm + lm_head over their B last rows, and token_logprobs gives
           every log p(cand_c[0]).
        2. Candidates run in passes (plan_score_passes: at most ``row_budget`` rows and the free KV pages each).  Candidate c of prompt b
           is a fork of slot b (PagedKVCache.fork): its table points at the prompt's full pages, the prompt's partial last page is copied
           into a page it owns (kv_copy_pages, rows [0, S_b % PAGE_SIZE)), and its rows cand_c[:-1] run at start_pos S_b.  A pass is one
           llama_prefill_chunk_layers over all its chunks, one lm_head GEMM into a bounded logits buffer and one token_logprobs launch.
        Every page is back on the free list afterwards."""
        d, dev = self.dims, self.device
        seq_lens = [int(n) for n in seq_lens]
        cands = check_candidates(candidates, d.vocab_size)
        B, N = len(seq_lens), len(cands)
        lens = [len(c) for c in cands]
        if B < 1 or packed_embeds.shape[0] != sum(seq_lens) or min(seq_lens) < 1:
            raise RuntimeError("score_candidates: rows do not match seq_lens")
        if max(seq_lens) + max(lens) > self.max_seq_len:
            raise ValueError(f"a prompt of {max(seq_lens)} rows and a candidate of {max(lens)} tokens exceed max_seq_len {self.max_seq_len}")
        if int(row_budget) < max(lens) - 1 or int(row_budget) < 1:
            raise ValueError(f"row_budget {row_budget} is smaller than the longest candidate's {max(lens) - 1} rows")
        L_max = max(lens)
        # pages: the prompts', then as many candidate pages as memory allows (at least the largest single candidate's)
        prompt_pages = sum((S + PAGE_SIZE - 1) // PAGE_SIZE for S in seq_lens)
        tails = [candidate_pages(S, L - 1)[1] for S in seq_lens for L in lens if L > 1]
        self.cache.release_all()
        free_b, _ = torch.cuda.mem_get_info(dev)
        afford = self.cache.n_pages + max(0, free_b - (2 << 30)) // 2 // self._page_bytes()
        self._grow_cache(B, min(prompt_pages + sum(tails), max(afford, prompt_pages + max(tails, default=0))), "scoring")
        self.cache.reserve_many(seq_lens)
        hidden = self.prefill_packed(packed_embeds, seq_lens)
        out = torch.zeros((B, N, L_max), dtype=torch.float32, device=dev)
        last = (torch.tensor(seq_lens).cumsum(0) - 1).to(torch.int32).to(dev)
        lg = self.lm_head_rows(ops.splice_rows(hidden, None, None, None, torch.zeros_like(last), last))
        _, lp, _ = ops.token_logprobs(lg, [b for b in range(B) for _ in range(N)], [c[0] for _ in range(B) for c in cands])
        out[:, :, 0] = lp.view(B, N)
        del hidden, lg
        plan = plan_score_passes(seq_lens, lens, int(row_budget), len(self.cache.free))
        buf = self._logits_buffer(max(sum(it[3] for it in p) for p in plan)) if plan else None
        prompt_tables = [self.cache.table(b) for b in range(B)]
        cap = self.cache.page_tables.shape[1]
        forks = []
        try:
            for items in plan:
                tables, copies, ids, targets, dst = [], [], [], [], []
                for b, c, _, n, _ in items:
                    S = seq_lens[b]
                    shared = S // PAGE_SIZE
                    f = self.cache.fork(b, shared, S + n)
                    forks.append(f)
                    t = self.cache.table(f)
                    assert not set(t[shared:]) & set(prompt_tables[b]), "a candidate's K/V appends would land in a shared page"
                    if S % PAGE_SIZE:
                        copies.append((prompt_tables[b][shared], t[shared], 0, S % PAGE_SIZE))
                    tables.append(t + [0] * (cap - len(t)))
                    ids.extend(cands[c][:-1])
                    targets.extend(cands[c][1:])
                    dst.extend((b * N + c) * L_max + j for j in range(1, n + 1))
                if copies:
                    ops.kv_copy_pages(self.cache.pages, copies)
                R = len(ids)
                cu = torch.tensor([0] + [it[2] + it[3] for it in items], dtype=torch.int32).to(dev)
                sp = torch.tensor([seq_lens[it[0]] for it in items], dtype=torch.int32).to(dev)
                pts = torch.tensor(tables, dtype=torch.int32).to(dev)
                x = self.embed_tokens(torch.tensor(ids, dtype=torch.int64))
                h = ops.llama_prefill_chunk_layers(x, self.stack, d, self.cos, self.sin, sp, pts, PAGE_SIZE, self.cache.n_pages, cu,
                                                   max(it[3] for it in items))
                lg = self.lm_head_rows(h, out=buf[:R])
                _, lp, _ = ops.token_logprobs(lg, list(range(R)), targets)
                out.view(-1)[torch.tensor(dst, dtype=torch.int64).to(dev)] = lp
                while forks:
                    self.cache.release(forks.pop())
        finally:
            while forks:
                self.cache.release(forks.pop())
            for b in range(B):
                self.cache.release(b)
        return out


def check_candidates(candidates, vocab_size: int) -> List[List[int]]:
    """The candidate token lists of a scoring request as lists of ints; raises ValueError on an empty list, an empty candidate or an id
    outside [0, vocab_size)."""
    if candidates is None or len(candidates) == 0:
        raise ValueError("candidates must be a non-empty list of token-id lists")
    out = []
    for i, c in enumerate(candidates):
        ids = [int(t) for t in (c.reshape(-1).tolist() if isinstance(c, torch.Tensor) else c)]
        if not ids:
            raise ValueError(f"candidate {i} is empty")
        bad = [t for t in ids if t < 0 or t >= vocab_size]
        if bad:
            raise ValueError(f"candidate {i} holds token {bad[0]}, outside the vocabulary [0, {vocab_size})")
        out.append(ids)
    return out
