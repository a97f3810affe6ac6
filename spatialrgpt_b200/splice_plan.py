"""Host-side plan of the embedding splice (llava/model/llava_arch.py:434-539).

The reference embeds the text ids, overwrites the <mask> / <depth> rows with region embeddings and
replaces each <image> slot by that image's feature rows, sample by sample, with torch indexing on
the device.  Here the same decisions are taken on the host from the token ids alone and expressed
as two int32 arrays per packed output row - ``src_id`` (0 token table, 1 image features, 2 mask
embeds, 3 depth embeds) and ``src_row`` (row inside that source) - which one gather kernel
(``srgpt_splice_rows_bf16``) then executes for the whole batch.  Pure torch-CPU code: no CUDA, so it is
covered by the ``-m "not gpu"`` tests against the oracle's ``splice_embeddings``.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import torch

from .constants import IGNORE_INDEX, IMAGE_TOKEN_INDEX

SRC_TOKENS, SRC_IMAGE, SRC_MASK, SRC_DEPTH = 0, 1, 2, 3


@dataclass
class SplicePlan:
    src_id: torch.Tensor        # int32 [sum(lens)]
    src_row: torch.Tensor       # int32 [sum(lens)]
    lens: List[int]             # rows per sample (after the optional truncation)
    labels: List[torch.Tensor]  # int64 per sample, IGNORE_INDEX on the image rows
    images_used: int
    warnings: List[str]


def build_splice_plan(input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor], labels: Optional[torch.Tensor], n_tok: int,
                      region_counts: Sequence[int], region_present: Sequence[bool], mask_token_id: int, depth_token_id: int,
                      region_on: bool, depth_on: bool, max_len: Optional[int] = None, vocab_size: Optional[int] = None) -> SplicePlan:
    """input_ids [B, T] (CPU int64, IMAGE_TOKEN_INDEX marks image slots); region_counts[i] / region_present[i]: number of
    regions of image i and whether its mask list entry was given (None entries write no region rows, base_extractor.py:47-49)."""
    ids_cpu = input_ids.to(torch.int64)
    B, T = ids_cpu.shape
    if vocab_size is not None:
        # the reference's nn.Embedding raises on an out-of-range id (llava_arch.py:436-437); the gather kernel has no bounds check,
        # so the plan is the place to refuse (only IMAGE_TOKEN_INDEX may be negative)
        bad = ((ids_cpu < 0) & (ids_cpu != IMAGE_TOKEN_INDEX)) | (ids_cpu >= vocab_size)
        if bool(bad.any()):
            b, t = [int(v) for v in torch.nonzero(bad)[0]]
            raise IndexError(f"input_ids[{b}, {t}] = {int(ids_cpu[b, t])} is outside the token table [0, {vocab_size})")
    am = torch.ones((B, T), dtype=torch.bool) if attention_mask is None else attention_mask.bool()
    lab_all = torch.full((B, T), IGNORE_INDEX, dtype=torch.int64) if labels is None else labels.to(torch.int64)
    offs = [0]
    for c in region_counts:
        offs.append(offs[-1] + int(c))
    plan_sid, plan_srow, out_labels, warns = [], [], [], []
    cur = 0
    for b in range(B):
        ids = ids_cpu[b][am[b]]
        lab = lab_all[b][am[b]]
        n = ids.shape[0]
        src_id = torch.zeros(n, dtype=torch.int32)
        src_row = ids.clamp(min=0).to(torch.int32)  # image slots -> token 0 (llava_arch.py:436), replaced below
        img_pos = torch.where(ids == IMAGE_TOKEN_INDEX)[0].tolist()
        if img_pos:
            first = cur
            if first >= len(region_counts):
                raise ValueError(f"sample {b} refers to image {first} but only {len(region_counts)} images were given")
            if region_on and region_present[first]:
                pos = torch.where(ids == mask_token_id)[0]
                k = min(pos.numel(), offs[first + 1] - offs[first])
                if pos.numel() > k:
                    warns.append("Error: fewer mask embeds than <mask> tokens")  # llava_arch.py:476-477 prints, no raise
                src_id[pos[:k]] = SRC_MASK
                src_row[pos[:k]] = torch.arange(offs[first], offs[first] + k, dtype=torch.int32)
            elif region_on and int((ids == mask_token_id).sum()) > 0:
                warns.append("Error: mask embed is None, but the num of <mask> is not 0!!!")
            if depth_on and region_present[first]:
                pos = torch.where(ids == depth_token_id)[0]
                k = min(pos.numel(), offs[first + 1] - offs[first])
                src_id[pos[:k]] = SRC_DEPTH
                src_row[pos[:k]] = torch.arange(offs[first], offs[first] + k, dtype=torch.int32)
        sid_parts, srow_parts, lab_parts = [], [], []
        start = 0
        for p in img_pos:  # expand every <image> slot into that image's n_tok feature rows
            sid_parts += [src_id[start:p], torch.full((n_tok,), SRC_IMAGE, dtype=torch.int32)]
            srow_parts += [src_row[start:p], torch.arange(cur * n_tok, (cur + 1) * n_tok, dtype=torch.int32)]
            lab_parts += [lab[start:p], torch.full((n_tok,), IGNORE_INDEX, dtype=torch.int64)]
            cur += 1
            start = p + 1
        sid_parts.append(src_id[start:]); srow_parts.append(src_row[start:]); lab_parts.append(lab[start:])
        sid, srow, lb = torch.cat(sid_parts), torch.cat(srow_parts), torch.cat(lab_parts)
        if max_len is not None:  # llava_arch.py:541-546 truncation to tokenizer_model_max_length
            sid, srow, lb = sid[:max_len], srow[:max_len], lb[:max_len]
        plan_sid.append(sid); plan_srow.append(srow); out_labels.append(lb)
    return SplicePlan(torch.cat(plan_sid), torch.cat(plan_srow), [int(x.numel()) for x in plan_sid], out_labels, cur, warns)


def reusable_prefix(prev_src_id: Optional[torch.Tensor], prev_src_row: Optional[torch.Tensor], src_id: torch.Tensor, src_row: torch.Tensor,
                    n_tok: int, image_equal: Sequence[bool], mask_equal: Sequence[bool], limit: int) -> int:
    """Rows at the start of a batch-1 prompt whose embeddings are the same as in the previous prompt, so that the K/V a prefill
    wrote for them can be kept (generate(prefix_cache=True)).  Both prompts are given by their splice-plan rows (src_id, src_row).
    Row r matches when both requests take it from the same source row and that source is unchanged:
      * a text row: the same token id (src_row is the id);
      * an image row: image_equal[i] for its image i = src_row // n_tok (the caller folds the depth image of the depth branch in);
      * a <mask> / <depth> row: mask_equal[g] for its region g = src_row (the caller folds in the region's image as well).
    Returns the length of the longest matching prefix, at most `limit` (the rows the decoder still holds, capped at S - 1)."""
    if prev_src_id is None or prev_src_row is None:
        return 0
    n = min(int(prev_src_id.numel()), int(src_id.numel()), max(int(limit), 0))
    if n == 0:
        return 0
    sid, srow = src_id[:n].to(torch.int64), src_row[:n].to(torch.int64)
    ok = (prev_src_id[:n].to(torch.int64) == sid) & (prev_src_row[:n].to(torch.int64) == srow)

    def lookup(table: Sequence[bool], idx: torch.Tensor) -> torch.Tensor:
        t = torch.tensor([bool(v) for v in table] + [False], dtype=torch.bool)  # the extra False answers any index out of range
        return t[torch.where((idx >= 0) & (idx < len(table)), idx, len(table))]

    img = sid == SRC_IMAGE
    ok &= ~img | lookup(image_equal, torch.div(srow, max(int(n_tok), 1), rounding_mode="floor"))
    region = (sid == SRC_MASK) | (sid == SRC_DEPTH)
    ok &= ~region | lookup(mask_equal, srow)
    bad = torch.nonzero(~ok)
    return int(bad[0, 0]) if bad.numel() else n
