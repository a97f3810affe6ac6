"""SpatialRGPT-Bench driver over the sm_90a path — the caller of ``generate()`` that the reference ships as
``llava/eval/eval_spatial.py`` (chunking :72-80, region construction :141-190, prompt loop :200-260, JSONL record :246-258)
and launches one process per GPU from ``scripts/srgpt/eval/srgpt_bench.sh:18-35``.

Same command line, same annotation format (``id``, ``image_info``, ``rle`` | ``bbox``, ``conversations``, ``text_q``,
``qa_info``), same answers file.  Differences, all on the host side of the hot path:

* regions: COCO run-length masks are decoded here (``rle_decode``; the reference needs pycocotools) and fall back to the
  boxes exactly where the reference's ``try/except`` does;
* depth: the monocular depth network (DepthAnything) is an external model and out of scope (SURVEY.md §8a row a0); the
  driver takes any ``depth_predictor(rgb uint8 [H, W, 3]) -> float tensor [h', w']`` and does the reference's post-processing
  (bilinear resize, min-max to 0..255, uint8, x3; eval_spatial.py:99-105) with the ``srgpt_depth_to_u8x3`` kernel;
* the benchmark script passes ``--temperature 0``, so its generation is greedy; a positive ``--temperature`` samples with the
  device sampler (temperature, ``--top_p`` and HF's default top-k of 50), seeded from ``torch.initial_seed()``: the same
  distribution as HF's sampling, not the same random stream.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import re
from typing import Any, Callable, Dict, List, Optional, Sequence

import numpy as np
import torch

from .constants import IMAGE_TOKEN_INDEX
from .conversation import SeparatorStyle, conv_templates
from .mm_utils import _mask_processor, get_model_name_from_path, process_images, tokenizer_image_token


# ---- chunking (eval_spatial.py:72-80): one chunk per process / GPU -----------------------------------------------
def split_list(lst: Sequence[Any], n: int) -> List[Sequence[Any]]:
    size = math.ceil(len(lst) / n)
    return [lst[i:i + size] for i in range(0, len(lst), size)]


def get_chunk(lst: Sequence[Any], n: int, k: int) -> Sequence[Any]:
    return split_list(lst, n)[k]


# ---- regions ----------------------------------------------------------------------------------------------------
def clamp_box(bbox: List[float], image_info: Dict[str, Any]) -> None:
    h, w = image_info["height"], image_info["width"]
    bbox[0] = max(min(w, bbox[0]), 0)
    bbox[2] = max(min(w, bbox[2]), 0)
    bbox[1] = max(min(h, bbox[1]), 0)
    bbox[3] = max(min(h, bbox[3]), 0)


def pad_to_square(a: np.ndarray) -> np.ndarray:
    h, w = a.shape
    side = max(h, w)
    out = np.zeros((side, side), dtype=np.uint8)
    out[(side - h) // 2:(side - h) // 2 + h, (side - w) // 2:(side - w) // 2 + w] = a
    return out


def _rle_counts_from_string(s: str) -> List[int]:
    """COCO's compressed run-length string: 5 data bits per character (offset 48), bit 5 = continuation, sign extension from
    bit 4 of the last group, and from the fourth run on each value is a difference to the run two places back."""
    counts: List[int] = []
    p = 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = ord(s[p]) - 48
            x |= (c & 0x1F) << (5 * k)
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(counts) > 2:
            x += counts[-2]
        counts.append(x)
    return counts


def rle_encode_counts(counts: Sequence[int]) -> str:
    """Inverse of ``_rle_counts_from_string`` (used by the tests and by tools that write annotations)."""
    out = []
    for i, x in enumerate(counts):
        x = int(x)
        if i > 2:
            x -= int(counts[i - 2])
        more = True
        while more:
            c = x & 0x1F
            x >>= 5
            more = (x != -1) if (c & 0x10) else (x != 0)
            if more:
                c |= 0x20
            out.append(chr(c + 48))
    return "".join(out)


def rle_decode(rle: Dict[str, Any]) -> np.ndarray:
    """{"size": [h, w], "counts": str | bytes | list} -> uint8 mask [h, w].  Runs alternate 0s and 1s, starting with 0s, over
    the mask flattened in column-major order (the COCO convention)."""
    h, w = int(rle["size"][0]), int(rle["size"][1])
    counts = rle["counts"]
    if isinstance(counts, bytes):
        counts = counts.decode("ascii")
    if isinstance(counts, str):
        counts = _rle_counts_from_string(counts)
    flat = np.zeros(h * w, dtype=np.uint8)
    pos, val = 0, 0
    for c in counts:
        c = int(c)
        if c < 0 or pos + c > h * w:
            raise ValueError("run-length mask does not match its size")
        if val:
            flat[pos:pos + c] = 1
        pos += c
        val ^= 1
    if pos != h * w:
        raise ValueError("run-length mask does not cover its size")
    return flat.reshape(w, h).T.copy()


def regions_for_line(line: Dict[str, Any], use_mask: bool, pad: bool) -> List[np.ndarray]:
    """Region masks of one annotation (eval_spatial.py:141-181): run-length masks when asked for and decodable, otherwise
    the boxes rasterised after clamping; padded to a square when the model pads its images."""
    info = line["image_info"]

    def boxes() -> List[np.ndarray]:
        out = []
        for bbox in line["bbox"]:
            m = np.zeros((info["height"], info["width"]), dtype=np.uint8)
            clamp_box(bbox, info)
            x1, y1, x2, y2 = map(int, bbox)
            m[y1:y2, x1:x2] = 1
            out.append(m)
        return out

    masks: List[np.ndarray]
    if use_mask:
        try:
            masks = [rle_decode(r).astype(np.uint8) for r in line["rle"]]
        except Exception:  # the reference falls back to the boxes on ANY failure (bare except, :156)
            masks = boxes()
    else:
        masks = boxes()
    return [pad_to_square(m) for m in masks] if pad else masks


# ---- prompts ----------------------------------------------------------------------------------------------------
def question_with_depth_tokens(question: str) -> str:
    """Every region reference carries its depth embedding too (eval_spatial.py:207)."""
    return re.sub(r"<mask>", "<mask> <depth>", question)


def stop_string(conv_mode: str) -> str:
    c = conv_templates[conv_mode]
    return c.sep if c.sep_style != SeparatorStyle.TWO else c.sep2


def clean_output(text: str, stop: str) -> str:
    text = text.strip()
    if stop and text.endswith(stop):
        text = text[: -len(stop)]
    return text.strip()


# ---- the loop ---------------------------------------------------------------------------------------------------
def depth_image(raw_rgb: np.ndarray, depth_predictor: Callable[[np.ndarray], torch.Tensor]):
    """rgb uint8 [H, W, 3] -> PIL image of the normalised depth replicated to 3 channels (eval_spatial.py:92-106); the
    resize / min-max / uint8 / x3 part runs in the ``srgpt_depth_to_u8x3`` kernel."""
    from PIL import Image

    from . import ops
    h, w = raw_rgb.shape[:2]
    raw = depth_predictor(raw_rgb)
    if not torch.is_tensor(raw):
        raw = torch.as_tensor(np.asarray(raw))
    raw = raw.to(dtype=torch.float32)
    if not raw.is_cuda:
        raw = raw.cuda()
    u8 = ops.depth_to_u8x3(raw.reshape(raw.shape[-2], raw.shape[-1]), h, w)
    return Image.fromarray(u8.cpu().numpy())


def get_depth_predictor(spec: Optional[str] = None) -> Optional[Callable[[np.ndarray], torch.Tensor]]:
    """The depth network is external to the hot path (eval_spatial.py:29-58 loads DepthAnything from $DEPTH_ANYTHING_PATH).
    ``spec`` = "package.module:factory" names a zero-argument factory returning ``predictor(rgb uint8 [H, W, 3]) -> depth
    [h', w']``; without a spec, $DEPTH_ANYTHING_PATH is used the way the reference uses it (its ``depth_anything`` package,
    ``checkpoints/depth_anything_vitl14.pth`` and the 518-px / multiple-of-14 transform).  Returns None when neither is given."""
    import importlib
    import sys

    if spec:
        mod, _, fn = spec.partition(":")
        return getattr(importlib.import_module(mod), fn or "get_depth_predictor")()
    root = os.environ.get("DEPTH_ANYTHING_PATH")
    if not root:
        return None
    import cv2
    sys.path.append(root)
    from depth_anything.dpt import DepthAnything
    from depth_anything.util.transform import NormalizeImage, PrepareForNet, Resize
    net = DepthAnything({"encoder": "vitl", "features": 256, "out_channels": [256, 512, 1024, 1024], "localhub": False})
    net.load_state_dict(torch.load(os.path.join(root, "checkpoints", "depth_anything_vitl14.pth"), map_location="cpu"))
    net = net.cuda().eval()
    steps = [Resize(width=518, height=518, resize_target=False, keep_aspect_ratio=True, ensure_multiple_of=14,
                    resize_method="lower_bound", image_interpolation_method=cv2.INTER_CUBIC),
             NormalizeImage(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225]), PrepareForNet()]

    @torch.no_grad()
    def predict(rgb: np.ndarray) -> torch.Tensor:
        sample = {"image": rgb / 255.0}
        for t in steps:
            sample = t(sample)
        return net(torch.from_numpy(sample["image"]).unsqueeze(0).cuda())[0]

    return predict


def answer_questions(line: Dict[str, Any], model, tokenizer, image_processor, image, depth, masks: Optional[torch.Tensor], conv_mode: str,
                     model_name: str, image_file: str, max_new_tokens: int = 128, temperature: float = 0.0, top_p=None,
                     num_beams: int = 1, prefix_cache: bool = False, prompt_lookup_num_tokens: int = 0) -> List[Dict[str, Any]]:
    """All question turns of one annotation (the conversation accumulates, as in the reference) -> JSONL records.
    ``prefix_cache``: each turn reuses the previous turn's encoder outputs and prompt K/V and prefills only the new question
    (generate(prefix_cache=True)); answers match a full re-prefill up to bf16 rounding.
    ``prompt_lookup_num_tokens=k > 0``: greedy answers are decoded by prompt lookup with up to k drafts per verify pass
    (generate(prompt_lookup_num_tokens=k)); the answers are the same, bit for bit."""
    dev = model.device
    images_tensor = process_images([image], image_processor, model.config).to(dev, dtype=model.dtype)
    depths_tensor = None if depth is None else process_images([depth], image_processor, model.config).to(dev, dtype=model.dtype)
    conv = conv_templates[conv_mode].copy()
    stop = stop_string(conv_mode)
    conversations = line["conversations"]
    records = []
    for i in range(len(conversations) // 2):
        # <depth> follows <mask> only when a depth image feeds the depth branch: without one the rows would keep the raw
        # token-table embedding of <depth>, which the model was never trained on
        q = conversations[i * 2]["value"]
        conv.append_message(conv.roles[0], question_with_depth_tokens(q) if depth is not None else q)
        conv.append_message(conv.roles[1], None)
        input_ids = tokenizer_image_token(conv.get_prompt(), tokenizer, IMAGE_TOKEN_INDEX, return_tensors="pt").unsqueeze(0).to(dev)
        output_ids = model.generate(input_ids, images=images_tensor, depths=depths_tensor,
                                    masks=None if masks is None else [masks.to(dev, dtype=model.dtype)],
                                    do_sample=temperature > 0, temperature=temperature, top_p=top_p, num_beams=num_beams,
                                    max_new_tokens=max_new_tokens, use_cache=True, **({"prefix_cache": True} if prefix_cache else {}),
                                    **({"prompt_lookup_num_tokens": prompt_lookup_num_tokens} if prompt_lookup_num_tokens else {}))
        pred = clean_output(tokenizer.batch_decode(output_ids, skip_special_tokens=True)[0], stop)
        records.append({"question_id": line["id"], "image": image_file, "question": line["text_q"], "pred": pred,
                        "gt": conversations[i * 2 + 1]["value"], "model_id": model_name, "qa_info": line["qa_info"]})
    return records


def check_batch_size(batch_size: int, **refused) -> None:
    """--batch-size N > 1 answers N annotations per generate(batch_invariant=True) call; the options in ``refused`` (flag name -> whether
    it is on) have no batch-invariant form and are refused with it."""
    if batch_size < 1:
        raise ValueError(f"--batch-size must be at least 1, got {batch_size}")
    on = [name for name, v in refused.items() if v]
    if batch_size > 1 and on:
        raise ValueError(f"--batch-size > 1 cannot be combined with {', '.join(on)}")


def generate_invariant(model, prompts: Sequence[torch.Tensor], images: torch.Tensor, depths: Optional[torch.Tensor], masks, **kw) -> List[torch.Tensor]:
    """generate(batch_invariant=True) over prompts [1, T_b] (one image each, the images [B, 3, R, R], depths the same or None, masks one
    [n_b, R, R] or None per prompt): returns each prompt's ids [1, n_b], equal to a batch-1 generate() of it with the same kwargs.  The
    prompts are right-padded under an attention mask; the result rows are padded with -1, which no token id is, and cut there."""
    T = max(int(p.shape[1]) for p in prompts)
    ids = torch.zeros((len(prompts), T), dtype=torch.int64)
    am = torch.zeros((len(prompts), T), dtype=torch.int64)
    for b, p in enumerate(prompts):
        ids[b, :p.shape[1]] = p[0].cpu()
        am[b, :p.shape[1]] = 1
    mask_list = None if all(m is None for m in masks) else list(masks)
    dev = model.device
    out = model.generate(ids.to(dev), attention_mask=am.to(dev), images=images, depths=depths, masks=mask_list, batch_invariant=True,
                         pad_token_id=-1, **kw)
    return [row[row >= 0][None] for row in out]


def answer_questions_batch(items: Sequence[Dict[str, Any]], model, tokenizer, image_processor, conv_mode: str, model_name: str,
                           max_new_tokens: int = 128, temperature: float = 0.0, top_p=None) -> List[List[Dict[str, Any]]]:
    """answer_questions for several annotations at once: turn i of every annotation that has one is answered by one
    generate(batch_invariant=True) call, each annotation keeping its own conversation.  items: dicts with line, image, depth, masks and
    image_file.  Returns each annotation's records, equal to what answer_questions writes for it."""
    dev = model.device
    imgs = [process_images([it["image"]], image_processor, model.config).to(dev, dtype=model.dtype) for it in items]
    dps = [None if it["depth"] is None else process_images([it["depth"]], image_processor, model.config).to(dev, dtype=model.dtype) for it in items]
    convs = [conv_templates[conv_mode].copy() for _ in items]
    stop = stop_string(conv_mode)
    records: List[List[Dict[str, Any]]] = [[] for _ in items]
    turns = [len(it["line"]["conversations"]) // 2 for it in items]
    kw = dict(do_sample=temperature > 0, temperature=temperature, top_p=top_p, num_beams=1, max_new_tokens=max_new_tokens, use_cache=True)
    for i in range(max(turns, default=0)):
        live = [b for b in range(len(items)) if turns[b] > i]
        prompts = []
        for b in live:
            it, conv = items[b], convs[b]
            q = it["line"]["conversations"][i * 2]["value"]
            conv.append_message(conv.roles[0], question_with_depth_tokens(q) if it["depth"] is not None else q)
            conv.append_message(conv.roles[1], None)
            prompts.append(tokenizer_image_token(conv.get_prompt(), tokenizer, IMAGE_TOKEN_INDEX, return_tensors="pt").unsqueeze(0))
        seed = {"seed": [torch.initial_seed()] * len(live)} if temperature > 0 else {}  # batch 1 draws with the default seed
        outs = generate_invariant(model, prompts, torch.cat([imgs[b] for b in live]),
                                  None if dps[live[0]] is None else torch.cat([dps[b] for b in live]),
                                  [None if items[b]["masks"] is None else items[b]["masks"].to(dev, dtype=model.dtype) for b in live], **kw, **seed)
        for b, output_ids in zip(live, outs):
            line = items[b]["line"]
            pred = clean_output(tokenizer.batch_decode(output_ids, skip_special_tokens=True)[0], stop)
            records[b].append({"question_id": line["id"], "image": items[b]["image_file"], "question": line["text_q"], "pred": pred,
                               "gt": line["conversations"][i * 2 + 1]["value"], "model_id": model_name, "qa_info": line["qa_info"]})
    return records


def eval_model(args, depth_predictor: Optional[Callable[[np.ndarray], torch.Tensor]] = None, loader=None) -> int:
    """Reference ``eval_model`` (eval_spatial.py:109-260).  ``loader`` defaults to ``load_pretrained_model``;
    ``depth_predictor`` is the external depth network (None: the depth branch gets no input)."""
    from PIL import Image
    batch_size = int(getattr(args, "batch_size", 1) or 1)
    check_batch_size(batch_size, **{"--prefix-cache": getattr(args, "prefix_cache", False),
                                    "--prompt-lookup-num-tokens": getattr(args, "prompt_lookup_num_tokens", 0),
                                    "--num_beams > 1": args.num_beams > 1})
    if loader is None:
        from .builder import load_pretrained_model as loader
    model_path = os.path.expanduser(args.model_path)
    model_name = get_model_name_from_path(model_path)
    # --quantization quantizes from (and computes in) the element type it is loaded in, so the model is loaded in bf16 instead of cast to it
    quant = {"quantization": args.quantization, "torch_dtype": torch.bfloat16} if getattr(args, "quantization", None) else {}
    if getattr(args, "nf4_planes_only", False):
        if getattr(args, "quantization", None) != "nf4":
            raise ValueError("--nf4-planes-only needs --quantization nf4")
        quant["nf4_dequantized_copy"] = False
    tokenizer, model, image_processor, _ = loader(model_path, model_name, getattr(args, "model_base", None), **quant)
    model.to(dtype=torch.bfloat16)  # eval_spatial.py:221: the loader returns fp16, this script computes in bf16
    if depth_predictor is None:
        depth_predictor = get_depth_predictor(getattr(args, "depth_predictor", None))
    if depth_predictor is None and getattr(model.config, "enable_depth", False):
        # the reference ALWAYS runs DepthAnything (eval_spatial.py:113); answers without it are not comparable
        if not getattr(args, "allow_no_depth", False):
            raise RuntimeError("this checkpoint has enable_depth=True but no depth network was given: pass --depth-predictor "
                               "module:factory, set DEPTH_ANYTHING_PATH, or accept degraded answers with --allow-no-depth")
        print("WARNING: no depth network: the depth branch gets no input and <depth> tokens are not inserted; answers are NOT "
              "comparable with the reference's", flush=True)
    with open(args.annotation_file) as f:
        questions = get_chunk(json.load(f), args.num_chunks, args.chunk_idx)
    answers_file = os.path.expanduser(args.answers_file)
    os.makedirs(os.path.dirname(answers_file) or ".", exist_ok=True)
    pad = getattr(model.config, "image_aspect_ratio", None) == "pad"
    mask_proc = _mask_processor(image_processor)
    n = 0
    with open(answers_file, "w") as out:
        # --batch-size N: N consecutive annotations at a time, their records written in the original order
        for g in range(0, len(questions), batch_size):
            items = []
            for line in questions[g:g + batch_size]:
                image_file = line["image_info"]["file_path"]
                region_masks = regions_for_line(line, args.use_mask, pad)
                # eval_spatial.py:183-190: the image processor without normalisation / rescaling, one [1, R, R] slice per region
                masks = (torch.vstack([mask_proc.preprocess(m[None, ...], return_tensors="pt")["pixel_values"][0] for m in region_masks]).float()
                         if region_masks else None)
                image = Image.open(os.path.join(args.image_folder, image_file)).convert("RGB")
                depth = depth_image(np.array(image), depth_predictor) if depth_predictor is not None else None
                items.append(dict(line=line, image=image, depth=depth, masks=masks, image_file=image_file))
            if batch_size == 1:
                it = items[0]
                groups = [answer_questions(it["line"], model, tokenizer, image_processor, it["image"], it["depth"], it["masks"], args.conv_mode,
                                           model_name, it["image_file"], temperature=args.temperature, top_p=args.top_p, num_beams=args.num_beams,
                                           prefix_cache=getattr(args, "prefix_cache", False),
                                           prompt_lookup_num_tokens=getattr(args, "prompt_lookup_num_tokens", 0))]
            else:
                groups = answer_questions_batch(items, model, tokenizer, image_processor, args.conv_mode, model_name, temperature=args.temperature,
                                                top_p=args.top_p)
            for recs in groups:
                for rec in recs:
                    out.write(json.dumps(rec) + "\n")
                    n += 1
    return n


def build_arg_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="SpatialRGPT-Bench over the sm_90a generate() path (flags of llava/eval/eval_spatial.py)")
    p.add_argument("--model-path", type=str, required=True)
    p.add_argument("--model-base", type=str, default=None)
    p.add_argument("--image-folder", type=str, default="")
    p.add_argument("--annotation-file", type=str, default="")
    p.add_argument("--answers-file", type=str, default="answer.jsonl")
    p.add_argument("--conv-mode", type=str, default="llava_v1")
    p.add_argument("--num-chunks", type=int, default=1)
    p.add_argument("--chunk-idx", type=int, default=0)
    p.add_argument("--temperature", type=float, default=0.0)  # the reference's default 0.2 samples; its benchmark script passes 0
    p.add_argument("--top_p", type=float, default=None)
    p.add_argument("--num_beams", type=int, default=1)
    p.add_argument("--use-mask", type=lambda s: str(s).lower() not in ("0", "false", "no"), default=True)
    p.add_argument("--depth-predictor", type=str, default=None,
                   help="module:factory of the external depth network (default: DepthAnything from $DEPTH_ANYTHING_PATH, like the reference)")
    p.add_argument("--prefix-cache", action="store_true",
                   help="prefill only the new question of each follow-up turn, reusing the earlier turns' encoder outputs and K/V")
    p.add_argument("--prompt-lookup-num-tokens", type=int, default=0,
                   help="greedy decoding by prompt lookup: draft up to this many tokens per verify pass (0 = off; same answers)")
    p.add_argument("--allow-no-depth", action="store_true", help="run an enable_depth checkpoint without a depth network (degraded answers)")
    p.add_argument("--batch-size", type=int, default=1,
                   help="answer turn i of this many consecutive annotations in one generate(batch_invariant=True) call (same answers file)")
    p.add_argument("--quantization", choices=["nf4", "fp8"], default=None,
                   help="quantization of the LLM's layer matrices: NF4 weight-only, or FP8 (E4M3) weights and activations")
    p.add_argument("--nf4-planes-only", action="store_true",
                   help="with --quantization nf4: keep only the 4-bit planes of the layer matrices, no dequantized copy (same answers)")
    return p


if __name__ == "__main__":
    print(f"wrote {eval_model(build_arg_parser().parse_args())} answers")
