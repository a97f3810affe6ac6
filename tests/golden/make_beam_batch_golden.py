"""Generate tests/golden/beam_batch_kats.npz: HF ``LlamaForCausalLM.generate(inputs_embeds=..., attention_mask=..., num_beams=k)`` over a
batch of left-padded prompts of several lengths, on a stock LlamaForCausalLM holding the oracle's seeded weights (the model of
``make_golden.py beam``).  fp32 on CPU, transformers of this image:

    python tests/golden/make_beam_batch_golden.py

tests/test_beam_batch_cpu.py pins the oracle's per-prompt beam search against it; tests/test_gpu_beam_batch.py pins
LlamaDecoder.generate_beam_batch.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle import srgpt_oracle as O  # noqa: E402
from tests.golden.make_golden import BEAM_WEIGHT_SEED, CASES  # noqa: E402

# batched beam search: (num_beams, eos_token_id, max_new_tokens, length_penalty, early_stopping) over every prompt of BEAM_BATCH_LENS
BEAM_BATCH_CASES = [
    (3, None, 10, 1.0, False), (3, [460], 10, 1.0, False), (4, [38, 97], 12, 1.0, False), (2, [886], 10, 1.0, False),
    (3, [764], 16, 2.0, False), (3, [764], 16, 0.5, True), (5, [303], 14, 1.0, True),
]
BEAM_BATCH_LENS = [20, 9, 14, 5]  # the first prompt is beam_kats' inputs_embeds


@torch.no_grad()
def run_beam_batch_kats():
    """HF's batched ``generate(inputs_embeds=[B, T, H], attention_mask=, num_beams=k)`` over left-padded prompts of several lengths, on the
    model of ``make_golden.py beam``.  Row b of case i holds prompt b's new ids; the unpadded prompts are stored packed.  transformers 5.5 fills
    a row that ends early with its EOS id rather than pad_token_id, so a reader compares each row up to its own length."""
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = O.OracleConfig(**CASES["tiny_masks_gqa"][0])
    sd = O.make_weights(cfg, seed=BEAM_WEIGHT_SEED)
    lcfg = LlamaConfig(hidden_size=cfg.hidden, intermediate_size=cfg.inter, num_hidden_layers=cfg.layers, num_attention_heads=cfg.heads,
                       num_key_value_heads=cfg.kv_heads, vocab_size=cfg.vocab, rms_norm_eps=cfg.rms_eps, rope_theta=cfg.rope_theta,
                       max_position_embeddings=4096, tie_word_embeddings=False, head_dim=cfg.head_dim, attention_bias=False, mlp_bias=False,
                       bos_token_id=1, eos_token_id=None, pad_token_id=None)
    lcfg._attn_implementation = "eager"
    llm = LlamaForCausalLM(lcfg).float().eval()
    llm.load_state_dict({k: v.float() for k, v in sd["llm"].items()}, strict=True)
    g = torch.Generator().manual_seed(0)
    prompts = [(torch.randn(n, cfg.hidden, generator=g) * 0.3).to(torch.bfloat16).float() for n in BEAM_BATCH_LENS]
    T = max(BEAM_BATCH_LENS)
    emb = torch.zeros(len(prompts), T, cfg.hidden)
    mask = torch.zeros(len(prompts), T, dtype=torch.long)
    for b, p in enumerate(prompts):  # left padding, as a decoder-only batch is padded for generation
        emb[b, T - p.shape[0]:] = p
        mask[b, T - p.shape[0]:] = 1
    arrays = {"packed_embeds": torch.cat(prompts).numpy(), "seq_lens": np.array(BEAM_BATCH_LENS, dtype=np.int64),
              "weight_seed": np.int64(BEAM_WEIGHT_SEED)}
    for i, (nb, eos, n_new, lp, es) in enumerate(BEAM_BATCH_CASES):
        out = llm.generate(inputs_embeds=emb, attention_mask=mask, num_beams=nb, do_sample=False, max_new_tokens=n_new, eos_token_id=eos,
                           pad_token_id=0, early_stopping=es, length_penalty=lp, num_return_sequences=1)
        arrays[f"case{i}"] = out.numpy()
        print(i, nb, eos, n_new, lp, es, out.tolist())
    path = os.path.join(HERE, "beam_batch_kats.npz")
    np.savez_compressed(path, **arrays)
    print(f"beam_batch_kats -> {path}")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    run_beam_batch_kats()
