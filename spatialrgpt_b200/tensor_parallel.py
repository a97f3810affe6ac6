"""Tensor-parallel Llama decode (BASELINE.json config c5, SURVEY.md §8e "optional TP"): one process per GPU, `world` ranks.

No reference counterpart (the reference only EMULATES pretraining_tp inside one GPU, modeling_llama.py:206-219); parity target =
the TP-1 decoder of llama_decoder.py.  Megatron-style sharding of the decode step:

  fused QKV (+RMSNorm, RoPE, KV append)   column parallel: a rank owns n_heads/world query heads and n_kv/world kv heads
  paged decode attention                   the rank's own heads only
  o_proj                                   row parallel: K slice = the rank's heads; fp32 partial sums -> ALL-REDUCE -> + residual
  gate/up (+RMSNorm, SwiGLU)               column parallel: I/world interleaved (gate_i, up_i) row pairs
  down_proj                                row parallel -> ALL-REDUCE -> + residual
  lm_head + argmax                         vocabulary parallel: every rank's (best value, global index) -> ALL-GATHER -> pick

The residual stream h, the position / step counters and the generated ids are replicated and stay bit-identical on all ranks
(the all-reduce result and the gathered arg-max candidates are the same everywhere).  The KV cache keeps the FULL layout on every
rank - a rank only reads and writes its own kv heads - so the prompt runs through the replicated, tensor-core bound prefill of
LlamaDecoder unchanged and decode continues from it.

Collectives (2 x layers all-reduces of H fp32 = 16 KB + one 8-byte-per-rank all-gather per token), two implementations:
  comm="p2p"  (default)  FUSED over NVLink peer memory (csrc/tp_comm.cu): the row-parallel GEMV writes its partial sums straight into
              this rank's slot of a symmetric buffer (torch.distributed._symmetric_memory: cuMem allocation mapped into every peer);
              one kernel then signals the peers, waits for their signals, pulls their slots through NVLink, reduces in rank order
              and applies the residual add (the lm_head all-gather kernel also picks the token and advances the step) - no NCCL
              call and no separate reduction kernel on the decode path;
  comm="nccl"             torch.distributed all_reduce / all_gather_into_tensor on the compute stream + the residual / pick kernels:
              the baseline the fused version is measured against (SRGPT_TP_COMM=nccl).
Both run inside ONE CUDA graph per decode step.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import ops
from .config import LlamaDims
from .llama_decoder import PAGE_SIZE, LlamaDecoder
from .weights import LlamaW


def shard_bounds(total: int, world: int, rank: int):
    per = total // world
    if per * world != total:
        raise ValueError(f"{total} is not divisible by the tensor-parallel size {world}")
    return rank * per, (rank + 1) * per


class TPShard:
    """This rank's slices of one decoder layer (contiguous copies in the layouts the GEMV kernels stream)."""

    def __init__(self, dims: LlamaDims, lw, rank: int, world: int):
        nh, nkv, hd, I = dims.num_attention_heads, dims.num_key_value_heads, dims.head_dim, dims.intermediate_size
        q0, q1 = shard_bounds(nh, world, rank)
        k0, k1 = shard_bounds(nkv, world, rank)
        i0, i1 = shard_bounds(I, world, rank)
        qkv = lw.qkv_w
        self.qkv_w = torch.cat([qkv[q0 * hd:q1 * hd], qkv[(nh + k0) * hd:(nh + k1) * hd], qkv[(nh + nkv + k0) * hd:(nh + nkv + k1) * hd]], 0).contiguous()
        self.o_w = lw.o_w[:, q0 * hd:q1 * hd].contiguous()            # [H, nh_local * hd]
        self.gateup_w = lw.gateup_w[2 * i0:2 * i1].contiguous()        # interleaved (gate_i, up_i) rows of the rank's I slice
        self.down_w = lw.down_w[:, i0:i1].contiguous()                # [H, I / world]
        self.in_norm, self.post_norm = lw.in_norm, lw.post_norm


class TPLlamaDecoder(LlamaDecoder):
    supports_prefix_reuse = False  # prompt-prefix reuse is a batch-1, single-GPU feature: nothing is recorded here
    packs_decode_weights = False   # the ranks stream their bf16 shards
    supports_prompt_lookup = False  # the verify pass is a single-GPU kernel sequence
    supports_logits_processors = False  # the logits are vocabulary-parallel: no rank holds a whole row
    supports_batch_sampling = False  # the decoder implements greedy decoding only
    supports_output_scores = False  # the logits are vocabulary-parallel: no rank holds a whole score row
    supports_scoring = False  # likelihood scoring (score_candidates) is a single-GPU path
    supports_batch_invariant = False  # the rows step (generate_rows) is a single-GPU kernel sequence
    supports_contrastive = False  # contrastive search runs the batched step and its choice on one GPU
    supports_forward_outputs = False  # forward()'s attentions need every head, and no rank holds them all
    supports_generate_outputs = False  # generate()'s attentions likewise

    def score_candidates(self, *args, **kwargs):
        raise NotImplementedError("likelihood scoring (score()) on the tensor-parallel decoder")

    def __init__(self, dims: LlamaDims, w: LlamaW, rank: int, world: int, group=None, max_seq_len: int = 4096, comm: Optional[str] = None, **kw):
        if getattr(w, "quantization", None) is not None:
            raise NotImplementedError(f"the tensor-parallel decoder streams unquantized shards; quantization={w.quantization!r} is single-GPU only")
        super().__init__(dims, w, max_seq_len=max_seq_len, **kw)
        if dims.num_attention_heads % world or dims.num_key_value_heads % world or dims.intermediate_size % world:
            raise ValueError(f"heads {dims.num_attention_heads}/{dims.num_key_value_heads} and intermediate size {dims.intermediate_size} must divide by TP={world}")
        self.rank, self.world, self.group = rank, world, group
        dev = self.device
        self.shards: List[TPShard] = [TPShard(dims, lw, rank, world) for lw in w.layers]
        self.nh_local = dims.num_attention_heads // world
        self.nkv_local = dims.num_key_value_heads // world
        self.kv_off = rank * self.nkv_local
        hd = dims.head_dim
        self.q_local = torch.zeros(self.nh_local * hd, dtype=self.dtype, device=dev)
        self.attn_local = torch.zeros(self.nh_local * hd, dtype=self.dtype, device=dev)
        self.act_local = torch.zeros(dims.intermediate_size // world, dtype=self.dtype, device=dev)
        self.partial = torch.zeros(dims.hidden_size, dtype=torch.float32, device=dev)
        # vocabulary-parallel lm_head: contiguous row blocks, the last rank takes the remainder
        V = dims.vocab_size
        per = (V + world - 1) // world
        self.v0, self.v1 = min(V, rank * per), min(V, (rank + 1) * per)
        self.lm_local = w.lm_head[self.v0:self.v1]
        self.lm_ws_local = ops.lm_head_workspace(max(self.v1 - self.v0, 2), dev)
        self.best = torch.zeros(2, dtype=torch.int32, device=dev)
        self.best_all = torch.zeros(2 * world, dtype=torch.int32, device=dev)
        self.kernels_per_decode_step = 7 * dims.num_hidden_layers + 3
        self.allreduce_bytes_per_token = 2 * dims.num_hidden_layers * dims.hidden_size * 4
        import os
        self.comm = (comm or os.environ.get("SRGPT_TP_COMM") or "p2p") if world > 1 else "none"
        self.tp_epoch = torch.zeros(1, dtype=torch.int32, device=dev)
        if self.comm == "p2p":
            self._init_p2p()

    def _init_p2p(self) -> None:
        """Symmetric buffer: flags [world][128] int32 | (2 x layers + 1) slots of H floats; peer-mapped through torch's symmetric
        memory (plumbing: allocation + address exchange only; every byte moved on the decode path is moved by tp_comm.cu)."""
        import ctypes

        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem

        from . import _lib
        lib = _lib.load()
        d = self.dims
        n_slots = 2 * d.num_hidden_layers + 1
        H = d.hidden_size
        nbytes = int(lib.srgpt_tp_comm_bytes(self.world, n_slots, H))
        group = self.group if self.group is not None else dist.group.WORLD
        buf = symm_mem.empty(nbytes // 4, dtype=torch.float32, device=self.device)
        buf.zero_()
        hdl = symm_mem.rendezvous(buf, group)
        torch.cuda.synchronize(self.device)
        dist.barrier(group=group)  # every rank's flags are zero before anybody signals
        self._symm = (buf, hdl)
        self.peer_bases = (ctypes.c_ulonglong * self.world)(*[int(p) for p in hdl.buffer_ptrs])
        self.slot_off = [int(lib.srgpt_tp_comm_slot_offset(self.world, s, H)) for s in range(n_slots)]
        self.slots = [buf[o // 4: o // 4 + H] for o in self.slot_off]
        self.best_slot = self.slots[-1].view(torch.int32)[:2]
        self.kernels_per_decode_step = 6 * d.num_hidden_layers + 2

    def _capture(self, key, launch, restore, kernels: int) -> torch.cuda.CUDAGraph:
        had = key in self._graphs
        g = super()._capture(key, launch, restore, kernels)
        if not had and key.kind == "step":
            # the warm-up step before the capture ran real collectives with the current (epoch, step): retire those flag values
            self.tp_epoch.add_(1)
        return g

    def _decode_loop(self, *args, **kwargs):
        self.tp_epoch.add_(1)  # a new request: flag values of the previous one can never match (tp_comm.cu seq_value)
        return super()._decode_loop(*args, **kwargs)

    # ---- collectives (NCCL through torch.distributed, on the current stream; world 1 = no-ops) ------------------------------
    def _all_reduce(self, t: torch.Tensor) -> None:
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(t, group=self.group)

    def _all_gather(self, out: torch.Tensor, t: torch.Tensor) -> None:
        if self.world > 1:
            import torch.distributed as dist
            dist.all_gather_into_tensor(out, t, group=self.group)
        else:
            out.copy_(t)

    # ---- one decode step of this rank ------------------------------------------------------------------------------------
    def _decode_step_launch(self, seq: int, logits_out: Optional[torch.Tensor] = None, sample: bool = False, proc: bool = False) -> None:
        if sample or proc or logits_out is not None:
            raise NotImplementedError("the tensor-parallel decoder implements greedy decoding without logits processors (the mode config c5 names)")
        d, w = self.dims, self.w
        hd = d.head_dim
        group = d.num_attention_heads // d.num_key_value_heads
        p2p = self.comm == "p2p"
        for l, sh in enumerate(self.shards):
            pages = self.cache.layer(l)
            ops.gemv_tp_qkv(self.h, sh.qkv_w, self.q_local, sh.in_norm, d.rms_norm_eps, self.nh_local, self.nkv_local, hd, self.cos, self.sin,
                            self.pos, pages, self.active_pt, PAGE_SIZE, d.num_key_value_heads, self.kv_off)
            ops.attention_decode_tp(self.q_local, self.attn_local, pages, self.active_pt, PAGE_SIZE, self.pos, self.nh_local, group,
                                    d.num_key_value_heads, self.kv_off, hd, self.scale)
            if p2p:  # partial sums straight into the symmetric slots; reduce + residual fused over NVLink peer memory
                ops.gemv_tp_partial(self.attn_local, sh.o_w, self.slots[2 * l])
                ops.tp_allreduce_residual(self.peer_bases, self.rank, self.world, self.slot_off[2 * l], 2 * l, self.tp_epoch, self.step, self.h)
                ops.gemv(self.h, sh.gateup_w, self.act_local, norm_weight=sh.post_norm, eps=d.rms_norm_eps, mode=ops.GEMV_SWIGLU)
                ops.gemv_tp_partial(self.act_local, sh.down_w, self.slots[2 * l + 1])
                ops.tp_allreduce_residual(self.peer_bases, self.rank, self.world, self.slot_off[2 * l + 1], 2 * l + 1, self.tp_epoch, self.step, self.h)
                continue
            ops.gemv_tp_partial(self.attn_local, sh.o_w, self.partial)
            self._all_reduce(self.partial)
            ops.tp_residual_add(self.h, self.partial)
            ops.gemv(self.h, sh.gateup_w, self.act_local, norm_weight=sh.post_norm, eps=d.rms_norm_eps, mode=ops.GEMV_SWIGLU)
            ops.gemv_tp_partial(self.act_local, sh.down_w, self.partial)
            self._all_reduce(self.partial)
            ops.tp_residual_add(self.h, self.partial)
        if p2p:
            n_coll = 2 * d.num_hidden_layers
            ops.lm_head_local_best(self.h, self.lm_local, w.norm, d.rms_norm_eps, self.lm_ws_local, self.v0, self.best_slot)
            ops.tp_allgather_pick(self.peer_bases, self.rank, self.world, self.slot_off[n_coll], n_coll, self.tp_epoch, w.embed, self.h, self.out_ids,
                                  self.step, self.pos)
            return
        ops.lm_head_local_best(self.h, self.lm_local, w.norm, d.rms_norm_eps, self.lm_ws_local, self.v0, self.best)
        self._all_gather(self.best_all, self.best)
        ops.tp_pick_token(self.best_all, self.world, w.embed, self.h, self.out_ids, self.step, self.pos)
